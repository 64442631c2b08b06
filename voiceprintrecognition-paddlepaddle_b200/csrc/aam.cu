// Cosine classifier + AAMLoss (ArcFace) forward / backward (K9 + K10).
// Reference: ppvector/models/fc.py:41-53 (logits = normalize(x) @ normalize(W, axis=0), W [D,S]) and
// ppvector/loss/aamloss.py:34-46 (phi = c cos m - sqrt(1-c^2) sin m; hard-margin fallback c - mmm when
// c <= th; one-hot select; x scale; softmax cross-entropy, mean over the batch, label smoothing).
// The head is small (B x S = 64 x 2796, D = 192: 69 MFLOP) and HBM/latency-bound, so it is plain fp32 SIMT
// with warp / block reductions -- no tensor cores, no one_hot / [B,S] temporaries beyond the logits.
// Deviation from the reference: sqrt(1 - c^2) is clamped at 0 (the reference would produce NaN for |c| > 1
// by rounding); identical otherwise.
#include <math.h>

#include "common.h"
#include "ptx.cuh"

namespace ppv {

// The workspace of aam_forward and aam_backward: the backward reads the e_hat / inv_e / inv_w the forward left in the same workspace.
struct AamWs {
    float *e_hat, *inv_e, *inv_w, *row_loss, *G, *dEh;  // [B,D] | [B] | [S] | [B] | [B,S] | [B,D]
};
static void carve_aam(WsCarver& cv, int B, int D, int S, AamWs* w) {
    auto take = [&](size_t n) { return static_cast<float*>(cv.take(n * sizeof(float))); };
    w->e_hat = take(size_t(B) * D);
    w->inv_e = take(B);
    w->inv_w = take(S);
    w->row_loss = take(B);
    w->G = take(size_t(B) * S);
    w->dEh = take(size_t(B) * D);
}
size_t aam_workspace_bytes(int B, int D, int S) {
    return carve_extent([&](WsCarver& cv) { AamWs w; carve_aam(cv, B, D, S, &w); });
}

__global__ void aam_norm_rows_kernel(const float* __restrict__ emb, int B, int D, float* __restrict__ e_hat, float* __restrict__ inv_e) {
    const int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    if (row >= B) return;
    const float* x = emb + int64_t(row) * D;
    float ss = 0.f;
    for (int i = lane; i < D; i += 32) ss = fmaf(x[i], x[i], ss);
    ss = warp_sum(ss);
    const float inv = 1.f / fmaxf(sqrtf(ss), 1e-12f);  // F.normalize eps
    for (int i = lane; i < D; i += 32) e_hat[int64_t(row) * D + i] = x[i] * inv;
    if (lane == 0) inv_e[row] = inv;
}
// column norms of W [D,S]: thread per column, coalesced over s
__global__ void aam_norm_cols_kernel(const float* __restrict__ W, int D, int S, float* __restrict__ inv_w) {
    const int s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= S) return;
    float ss = 0.f;
    for (int d = 0; d < D; ++d) {
        const float v = W[int64_t(d) * S + s];
        ss = fmaf(v, v, ss);
    }
    inv_w[s] = 1.f / fmaxf(sqrtf(ss), 1e-12f);
}
// logits[b,s] = <e_hat_b, W[:,s]> * inv_w[s]
__global__ void __launch_bounds__(256)
    aam_logits_kernel(const float* __restrict__ e_hat, const float* __restrict__ W, const float* __restrict__ inv_w, int D, int S,
                      float* __restrict__ logits) {
    extern __shared__ float s_e[];
    const int b = blockIdx.y;
    for (int i = threadIdx.x; i < D; i += blockDim.x) s_e[i] = e_hat[int64_t(b) * D + i];
    __syncthreads();
    const int s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= S) return;
    float acc = 0.f;
    for (int d = 0; d < D; ++d) acc = fmaf(s_e[d], W[int64_t(d) * S + s], acc);
    logits[int64_t(b) * S + s] = acc * inv_w[s];
}

__device__ __forceinline__ float aam_margin(float c, bool is_target, float cos_m, float sin_m, float th, float mmm, int easy,
                                            float* dphi_dc) {
    if (!is_target) {
        *dphi_dc = 1.f;
        return c;
    }
    const float sine = sqrtf(fmaxf(1.f - c * c, 0.f));
    const float phi = c * cos_m - sine * sin_m;
    const bool use_phi = easy ? (c > 0.f) : (c > th);
    if (use_phi) {
        *dphi_dc = cos_m + sin_m * c / fmaxf(sine, 1e-6f);
        return phi;
    }
    *dphi_dc = 1.f;
    return easy ? c : c - mmm;
}

// Scaled logit z of one (row, class) entry and dz / dcos for the loss heads of ppvector/loss/: `kind` 0 = AAMLoss (aamloss.py:34-46),
// 1 = AAMLoss(easy_margin=True), 2 = AMLoss (amloss.py:18-24: cos - m on the target), 3 = ARMLoss (armloss.py:18-31: AMLoss, then every
// entry whose scaled value is below the target's is set to 0), 4 = CELoss (celoss.py:16-18: the raw logits, no scale).
__device__ __forceinline__ float head_value(float c, bool is_target, int kind, float cos_m, float sin_m, float th, float mmm, float margin,
                                            float scale, float zy, float* dz_dc) {
    if (kind <= 1) {
        float d;
        const float v = aam_margin(c, is_target, cos_m, sin_m, th, mmm, kind, &d);
        *dz_dc = scale * d;
        return scale * v;
    }
    if (kind == 4) {
        *dz_dc = 1.f;
        return c;
    }
    const float z = scale * (c - (is_target ? margin : 0.f));
    *dz_dc = scale;
    if (kind == 3 && !is_target && z - zy < 0.f) {
        *dz_dc = 0.f;
        return 0.f;
    }
    return z;
}

__device__ __forceinline__ float block_reduce(float v, float* s_red, bool is_max) {
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    v = is_max ? warp_max(v) : warp_sum(v);
    if (lane == 0) s_red[warp] = v;
    __syncthreads();
    float r = s_red[0];
    for (int w = 1; w < (blockDim.x >> 5); ++w) r = is_max ? fmaxf(r, s_red[w]) : r + s_red[w];
    __syncthreads();
    return r;
}

// SubCenterLoss (ppvector/loss/subcenterloss.py:40-43): the classifier holds K sub-centres per class in adjacent columns
// (reshape(-1, S, K)); a class's cosine is the maximum over its K columns, and only that column receives the class's gradient.
__device__ __forceinline__ float class_cosine(const float* __restrict__ c, int cls, int K, int* arg) {
    float best = c[cls * K];
    int a = 0;
    for (int k = 1; k < K; ++k) {
        const float v = c[cls * K + k];
        if (v > best) {
            best = v;
            a = k;
        }
    }
    *arg = a;
    return best;
}

// SphereFace2 (ppvector/loss/sphereface2.py:44-70): NOT a softmax -- one binary logistic loss per (row, class) entry over
// g(z) = 2 ((z + 1) / 2)^t - 1.  Type C: z_p = scale (g(c) - m), z_n = scale (g(c) + m); type A: g applied to the AAM-style shifted
// cosines (cos(theta + m) with the same th / mmm fallback on the target, cos(theta - m) on the others).  Entry loss:
// target lambda * log(1 + exp(-z_p)), others (1 - lambda) * log(1 + exp(z_n)); the loss's bias parameter is created at 0 and is not
// handed to the optimizer in the reference (trainer.py:186-190 passes model.parameters() only), so it stays 0.
// g is the plain polynomial for every z, as in the reference (sphereface2.py:40-42): a Linear layer's logits go below -1, and so does type
// A's fallback c - mmm on the target (c <= th gives c - mmm <= -1), so the base (z + 1) / 2 is negative by design there.
__device__ __forceinline__ float sf2_entry(float c, bool is_target, bool type_a, int t, float lambda, float cos_m, float sin_m, float th,
                                           float mmm, float margin, float scale, float* dl_dc) {
    float inner = c, dinner = 1.f, shift = 0.f;
    if (type_a) {
        const float sine = sqrtf(fmaxf(1.f - c * c, 0.f));
        const float ds = c / fmaxf(sine, 1e-6f);  // -d sine / dc
        if (is_target) {
            if (c > th) {
                inner = c * cos_m - sine * sin_m;
                dinner = cos_m + sin_m * ds;
            } else {
                inner = c - mmm;
            }
        } else {
            inner = c * cos_m + sine * sin_m;
            dinner = cos_m - sin_m * ds;
        }
    } else {
        shift = is_target ? -margin : margin;
    }
    const float h = 0.5f * (inner + 1.f);
    const float hp = powf(h, float(t - 1));  // ((z + 1) / 2)^(t - 1); t - 1 is integral, so powf is exact for a negative h too
    const float g = 2.f * hp * h - 1.f;
    const float dg = float(t) * hp * dinner;  // d g / d c
    const float z = scale * (g + shift);
    const float x = is_target ? -z : z;  // entry loss = w * softplus(x)
    const float w = is_target ? lambda : 1.f - lambda;
    const float sp = x > 20.f ? x : log1pf(expf(x));
    const float sg = 1.f / (1.f + expf(-x));  // softplus'(x)
    *dl_dc = w * sg * (is_target ? -1.f : 1.f) * scale * dg;
    return w * sp;
}

// one block per row: loss_b and (optionally) G[b,s] = d loss / d logit[b,s].  S = classes, K = sub-centres per class (1: plain heads);
// logits and G have S * K columns.  The same kernel reads a Linear layer's raw logits (K = 1).
__global__ void __launch_bounds__(256)
    aam_row_kernel(const float* __restrict__ logits, const int64_t* __restrict__ labels, int B, int S, int K, float cos_m, float sin_m,
                   float th, float mmm, int easy, float scale, float ls, float* __restrict__ row_loss, float* __restrict__ G, float margin) {
    __shared__ float s_red[8];
    const int b = blockIdx.x;
    const int64_t label = labels[b];
    const float* c = logits + int64_t(b) * S * K;
    if (easy & PPV_HEAD_SPHEREFACE2) {  // selector: PPV_HEAD_SPHEREFACE2 | type A bit | t << 5; `ls` carries lambda
        const bool type_a = (easy & 1) != 0;
        const int t = easy >> 5;
        float acc = 0.f;
        const float invB = 1.f / float(B);
        for (int s = threadIdx.x; s < S; s += blockDim.x) {
            float d;
            acc += sf2_entry(c[s], s == label, type_a, t, ls, cos_m, sin_m, th, mmm, margin, scale, &d);
            if (G) G[int64_t(b) * S + s] = d * invB;
        }
        acc = block_reduce(acc, s_red, false);
        if (threadIdx.x == 0) row_loss[b] = acc;
        return;
    }
    int arg;
    const float zy = scale * (class_cosine(c, int(label), K, &arg) - margin);  // ARMLoss: the target's scaled logit is the threshold of its row
    float mx = -INFINITY;
    for (int s = threadIdx.x; s < S; s += blockDim.x) {
        float d;
        mx = fmaxf(mx, head_value(class_cosine(c, s, K, &arg), s == label, easy, cos_m, sin_m, th, mmm, margin, scale, zy, &d));
    }
    mx = block_reduce(mx, s_red, true);
    float se = 0.f, so = 0.f, tgt = 0.f;
    for (int s = threadIdx.x; s < S; s += blockDim.x) {
        float d;
        const float o = head_value(class_cosine(c, s, K, &arg), s == label, easy, cos_m, sin_m, th, mmm, margin, scale, zy, &d);
        se += expf(o - mx);
        so += o;
        if (s == label) tgt = o;
    }
    se = block_reduce(se, s_red, false);
    so = block_reduce(so, s_red, false);
    tgt = block_reduce(tgt, s_red, false);
    const float lse = mx + logf(se);
    // CE with label smoothing: (1-ls) * (lse - o_y) + ls * (lse - mean_s o_s)
    if (threadIdx.x == 0) row_loss[b] = (1.f - ls) * (lse - tgt) + ls * (lse - so / float(S));
    if (G) {
        const float invB = 1.f / float(B);
        for (int s = threadIdx.x; s < S; s += blockDim.x) {
            float d;
            const float o = head_value(class_cosine(c, s, K, &arg), s == label, easy, cos_m, sin_m, th, mmm, margin, scale, zy, &d);
            const float p = expf(o - lse);
            const float t = (s == label ? (1.f - ls) : 0.f) + ls / float(S);
            for (int k = 0; k < K; ++k) G[(int64_t(b) * S + s) * K + k] = k == arg ? (p - t) * invB * d : 0.f;
        }
    }
}
__global__ void aam_mean_kernel(const float* __restrict__ row_loss, int B, float* __restrict__ loss) {
    if (threadIdx.x == 0 && blockIdx.x == 0) {
        float s = 0.f;
        for (int b = 0; b < B; ++b) s += row_loss[b];  // fixed order: deterministic
        *loss = s / float(B);
    }
}

// head selector (the `easy_margin` argument of the ABI): 0-4 = PPV_HEAD_*; PPV_HEAD_SUBCENTER | (K << 5) | easy = SubCenterLoss with K sub-centres
static int decode_head(int sel, int S, int* kind, int* K) {
    *kind = sel;
    *K = 1;
    if (sel & PPV_HEAD_SUBCENTER) {
        *K = sel >> 5;
        *kind = sel & 1;
        PPV_REQUIRE(*K >= 1 && S % *K == 0, "loss head: SubCenterLoss needs classifier columns = classes x K");
    } else if (sel & PPV_HEAD_SPHEREFACE2) {
        PPV_REQUIRE((sel >> 5) >= 1 && (sel >> 5) <= 16, "loss head: SphereFace2 needs 1 <= t <= 16 in the selector");
    } else {
        PPV_REQUIRE(sel >= 0 && sel <= PPV_HEAD_CE, "loss head: unknown selector");
    }
    return PPV_OK;
}

static void margin_consts(float margin, float* cos_m, float* sin_m, float* th, float* mmm) {
    *cos_m = float(cos(double(margin)));
    *sin_m = float(sin(double(margin)));
    *th = float(cos(M_PI - double(margin)));
    *mmm = float(1.0 + cos(M_PI - double(margin)));
}

int aam_forward(const float* emb, const float* W, const int64_t* labels, int B, int D, int S, float margin, float scale,
                int easy_margin, float label_smoothing, float* logits, float* loss, void* ws, size_t ws_bytes, cudaStream_t st) {
    PPV_REQUIRE(emb && W && labels && logits && loss, "aam_forward: null argument");
    PPV_REQUIRE(B > 0 && D > 0 && S > 0, "aam_forward: empty input");
    if (int rc = check_workspace("aam_forward", ws, ws_bytes, aam_workspace_bytes(B, D, S), "ppv_aam_workspace_bytes")) return rc;
    WsCarver cv{static_cast<uint8_t*>(ws)};
    AamWs w;
    carve_aam(cv, B, D, S, &w);
    aam_norm_rows_kernel<<<(B + 7) / 8, 256, 0, st>>>(emb, B, D, w.e_hat, w.inv_e);
    PPV_LAUNCH_OK("aam_norm_rows_kernel");
    aam_norm_cols_kernel<<<(S + 255) / 256, 256, 0, st>>>(W, D, S, w.inv_w);
    PPV_LAUNCH_OK("aam_norm_cols_kernel");
    aam_logits_kernel<<<dim3((S + 255) / 256, B), 256, D * sizeof(float), st>>>(w.e_hat, W, w.inv_w, D, S, logits);
    PPV_LAUNCH_OK("aam_logits_kernel");
    float cm, sm, th, mmm;
    margin_consts(margin, &cm, &sm, &th, &mmm);
    int kind, K;
    int rc = decode_head(easy_margin, S, &kind, &K);
    if (rc) return rc;
    aam_row_kernel<<<B, 256, 0, st>>>(logits, labels, B, S / K, K, cm, sm, th, mmm, kind, scale, label_smoothing, w.row_loss, nullptr, margin);
    PPV_LAUNCH_OK("aam_row_kernel");
    aam_mean_kernel<<<1, 32, 0, st>>>(w.row_loss, B, loss);
    PPV_LAUNCH_OK("aam_mean_kernel");
    return PPV_OK;
}

// dE_hat[b,d] = sum_s G[b,s] * W[d,s] * inv_w[s]   (one warp per (b,d), coalesced over s)
__global__ void __launch_bounds__(256)
    aam_dehat_kernel(const float* __restrict__ G, const float* __restrict__ W, const float* __restrict__ inv_w, int B, int D, int S,
                     float* __restrict__ dEh) {
    const int64_t wid = int64_t(blockIdx.x) * (blockDim.x >> 5) + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    if (wid >= int64_t(B) * D) return;
    const int b = int(wid / D), d = int(wid % D);
    float acc = 0.f;
    for (int s = lane; s < S; s += 32) acc = fmaf(G[int64_t(b) * S + s] * inv_w[s], W[int64_t(d) * S + s], acc);
    acc = warp_sum(acc);
    if (lane == 0) dEh[wid] = acc;
}
// d_emb[b,:] = (dEh_b - e_hat_b <e_hat_b, dEh_b>) * inv_e[b]
__global__ void aam_demb_kernel(const float* __restrict__ dEh, const float* __restrict__ e_hat, const float* __restrict__ inv_e, int B,
                                int D, float* __restrict__ d_emb) {
    const int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    if (row >= B) return;
    float dot = 0.f;
    for (int i = lane; i < D; i += 32) dot = fmaf(dEh[int64_t(row) * D + i], e_hat[int64_t(row) * D + i], dot);
    dot = warp_sum(dot);
    for (int i = lane; i < D; i += 32)
        d_emb[int64_t(row) * D + i] = (dEh[int64_t(row) * D + i] - e_hat[int64_t(row) * D + i] * dot) * inv_e[row];
}
// per column s: dWhat[:,s] = sum_b G[b,s] e_hat[b,:];  dW[:,s] = (dWhat - w_hat <w_hat, dWhat>) * inv_w[s]
// thread per column, loops over d twice (D small); coalesced over s.
__global__ void __launch_bounds__(128)
    aam_dw_kernel(const float* __restrict__ G, const float* __restrict__ e_hat, const float* __restrict__ W, const float* __restrict__ inv_w,
                  int B, int D, int S, float* __restrict__ dW) {
    extern __shared__ float s_eh[];  // [B, D]
    for (int i = threadIdx.x; i < B * D; i += blockDim.x) s_eh[i] = e_hat[i];
    __syncthreads();
    const int s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= S) return;
    const float iw = inv_w[s];
    float dot = 0.f;
    for (int d = 0; d < D; ++d) {
        float g = 0.f;
        for (int b = 0; b < B; ++b) g = fmaf(G[int64_t(b) * S + s], s_eh[b * D + d], g);
        dW[int64_t(d) * S + s] = g;  // stash dWhat
        dot = fmaf(g, W[int64_t(d) * S + s] * iw, dot);
    }
    for (int d = 0; d < D; ++d) {
        const float g = dW[int64_t(d) * S + s];
        dW[int64_t(d) * S + s] = (g - W[int64_t(d) * S + s] * iw * dot) * iw;
    }
}

int aam_backward(const float* emb, const float* W, const int64_t* labels, const float* logits, int B, int D, int S, float margin,
                 float scale, int easy_margin, float label_smoothing, float* d_emb, float* d_W, void* ws, size_t ws_bytes,
                 cudaStream_t st) {
    PPV_REQUIRE(emb && W && labels && logits && d_emb && d_W, "aam_backward: null argument");
    if (int rc = check_workspace("aam_backward", ws, ws_bytes, aam_workspace_bytes(B, D, S), "ppv_aam_workspace_bytes")) return rc;
    PPV_REQUIRE(size_t(B) * D * sizeof(float) <= 200 * 1024, "aam_backward: B*D too large for the shared-memory dW kernel");
    WsCarver cv{static_cast<uint8_t*>(ws)};
    AamWs w;
    carve_aam(cv, B, D, S, &w);  // e_hat / inv_e / inv_w are those of the forward call
    float cm, sm, th, mmm;
    margin_consts(margin, &cm, &sm, &th, &mmm);
    int kind, K;
    int rc = decode_head(easy_margin, S, &kind, &K);
    if (rc) return rc;
    aam_row_kernel<<<B, 256, 0, st>>>(logits, labels, B, S / K, K, cm, sm, th, mmm, kind, scale, label_smoothing, w.row_loss, w.G, margin);
    PPV_LAUNCH_OK("aam_row_kernel(bwd)");
    const int64_t warps = int64_t(B) * D;
    aam_dehat_kernel<<<unsigned((warps + 7) / 8), 256, 0, st>>>(w.G, W, w.inv_w, B, D, S, w.dEh);
    PPV_LAUNCH_OK("aam_dehat_kernel");
    aam_demb_kernel<<<(B + 7) / 8, 256, 0, st>>>(w.dEh, w.e_hat, w.inv_e, B, D, d_emb);
    PPV_LAUNCH_OK("aam_demb_kernel");
    const size_t smem = size_t(B) * D * sizeof(float);
    PPV_ONCE_PER_DEVICE(PPV_CUDA_OK(cudaFuncSetAttribute(aam_dw_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024)));
    aam_dw_kernel<<<(S + 127) / 128, 128, smem, st>>>(w.G, w.e_hat, W, w.inv_w, B, D, S, d_W);
    PPV_LAUNCH_OK("aam_dw_kernel");
    return PPV_OK;
}

// ------------------------------------------------------------------------------------------------ Linear output layer
// fc.py:37-38, 50-51: logits = H @ W + b with W [D, S] (Paddle's Linear layout, the one the cosine head reads) and b [S], no
// normalisation.  The same loss heads then run on the raw logits (aam_row_kernel with K = 1).  Every product below is a fixed-order fp32
// loop: no atomics, the same bits on every run.
constexpr int LIN_ROWS = 8;    // rows of H (or of G) one thread carries: W is read once per LIN_ROWS rows
constexpr int LIN_DCHUNK = 16;  // dW: columns of H one thread carries
constexpr int LIN_BCHUNK = 256; // dW: rows of H staged in shared memory at a time

// logits[b,s] = sum_d H[b,d] W[d,s] + bias[s]: thread per column s, LIN_ROWS rows per block (those rows of H in shared memory)
__global__ void __launch_bounds__(256)
    lin_logits_kernel(const float* __restrict__ H, const float* __restrict__ W, const float* __restrict__ bias, int B, int D, int S,
                      float* __restrict__ logits) {
    extern __shared__ float s_h[];  // [LIN_ROWS][D]
    const int b0 = blockIdx.y * LIN_ROWS, nb = min(LIN_ROWS, B - b0);
    for (int i = threadIdx.x; i < nb * D; i += blockDim.x) s_h[i] = H[int64_t(b0) * D + i];
    __syncthreads();
    const int s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= S) return;
    float acc[LIN_ROWS] = {};
    for (int d = 0; d < D; ++d) {
        const float w = W[int64_t(d) * S + s];
#pragma unroll
        for (int r = 0; r < LIN_ROWS; ++r) acc[r] = fmaf(s_h[(r < nb ? r : 0) * D + d], w, acc[r]);
    }
    const float bs = bias[s];
    for (int r = 0; r < nb; ++r) logits[int64_t(b0 + r) * S + s] = acc[r] + bs;
}
// dH[b,d] = sum_s G[b,s] W[d,s]: one warp per d (coalesced over s), LIN_ROWS rows of G per warp
__global__ void __launch_bounds__(256)
    lin_dh_kernel(const float* __restrict__ G, const float* __restrict__ W, int B, int D, int S, float* __restrict__ dH) {
    const int d = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    const int b0 = blockIdx.y * LIN_ROWS, nb = min(LIN_ROWS, B - b0);
    if (d >= D) return;
    float acc[LIN_ROWS] = {};
    for (int s = lane; s < S; s += 32) {
        const float w = W[int64_t(d) * S + s];
#pragma unroll
        for (int r = 0; r < LIN_ROWS; ++r)
            if (r < nb) acc[r] = fmaf(G[int64_t(b0 + r) * S + s], w, acc[r]);
    }
#pragma unroll
    for (int r = 0; r < LIN_ROWS; ++r) {
        const float v = warp_sum(acc[r]);
        if (lane == 0 && r < nb) dH[int64_t(b0 + r) * D + d] = v;
    }
}
// dW[d,s] = sum_b H[b,d] G[b,s] for LIN_DCHUNK columns d per thread; the blocks of the first d-chunk also write db[s] = sum_b G[b,s]
__global__ void __launch_bounds__(128)
    lin_dw_kernel(const float* __restrict__ G, const float* __restrict__ H, int B, int D, int S, float* __restrict__ dW, float* __restrict__ db) {
    __shared__ float s_h[LIN_BCHUNK * LIN_DCHUNK];
    const int s = blockIdx.x * blockDim.x + threadIdx.x;
    const int d0 = blockIdx.y * LIN_DCHUNK, nd = min(LIN_DCHUNK, D - d0);
    float acc[LIN_DCHUNK] = {};
    float gs = 0.f;
    for (int b0 = 0; b0 < B; b0 += LIN_BCHUNK) {
        const int nb = min(LIN_BCHUNK, B - b0);
        __syncthreads();
        for (int i = threadIdx.x; i < nb * LIN_DCHUNK; i += blockDim.x) {
            const int r = i / LIN_DCHUNK, j = i % LIN_DCHUNK;
            s_h[i] = j < nd ? H[int64_t(b0 + r) * D + d0 + j] : 0.f;
        }
        __syncthreads();
        if (s < S)
            for (int r = 0; r < nb; ++r) {
                const float g = G[int64_t(b0 + r) * S + s];
                gs += g;
#pragma unroll
                for (int j = 0; j < LIN_DCHUNK; ++j) acc[j] = fmaf(g, s_h[r * LIN_DCHUNK + j], acc[j]);
            }
    }
    if (s >= S) return;
    for (int j = 0; j < nd; ++j) dW[int64_t(d0 + j) * S + s] = acc[j];
    if (blockIdx.y == 0) db[s] = gs;
}

// AAMLoss, SubCenterLoss and SphereFace2 type A read the logits as cosines (sqrt(1 - z^2), and SubCenterLoss's K sub-centre columns):
// on raw Linear logits the reference turns NaN as soon as one leaves [-1, 1].  CELoss, AMLoss, ARMLoss and SphereFace2 type C are
// defined for any real logits.
static int linear_head_check(int sel) {
    const bool cosine_only = (sel & PPV_HEAD_SUBCENTER) || ((sel & PPV_HEAD_SPHEREFACE2) && (sel & 1)) ||
                             (!(sel & PPV_HEAD_SPHEREFACE2) && sel <= PPV_HEAD_AAM_EASY);
    if (cosine_only)
        return fail(PPV_EUNSUPPORTED, "Linear classifier: AAMLoss, SubCenterLoss and SphereFace2 type A take sqrt(1 - z^2) of cosine logits; "
                                      "use CELoss, AMLoss, ARMLoss or SphereFace2 type C");
    return PPV_OK;
}

int linear_head_forward(const float* H, const float* W, const float* bias, const int64_t* labels, int B, int D, int S, float margin, float scale,
                        int easy_margin, float label_smoothing, float* logits, float* loss, void* ws, size_t ws_bytes, cudaStream_t st) {
    PPV_REQUIRE(H && W && bias && labels && logits && loss, "linear_head_forward: null argument");
    PPV_REQUIRE(B > 0 && D > 0 && S > 0, "linear_head_forward: empty input");
    if (int rc = check_workspace("linear_head_forward", ws, ws_bytes, aam_workspace_bytes(B, D, S), "ppv_aam_workspace_bytes")) return rc;
    int kind, K;
    int rc = decode_head(easy_margin, S, &kind, &K);
    if (!rc) rc = linear_head_check(easy_margin);
    if (rc) return rc;
    PPV_REQUIRE(size_t(LIN_ROWS) * D * sizeof(float) <= 48 * 1024, "linear_head_forward: input width too large");
    WsCarver cv{static_cast<uint8_t*>(ws)};
    AamWs w;
    carve_aam(cv, B, D, S, &w);
    lin_logits_kernel<<<dim3((S + 255) / 256, (B + LIN_ROWS - 1) / LIN_ROWS), 256, size_t(LIN_ROWS) * D * sizeof(float), st>>>(H, W, bias, B, D, S,
                                                                                                                                logits);
    PPV_LAUNCH_OK("lin_logits_kernel");
    float cm, sm, th, mmm;
    margin_consts(margin, &cm, &sm, &th, &mmm);
    aam_row_kernel<<<B, 256, 0, st>>>(logits, labels, B, S, 1, cm, sm, th, mmm, kind, scale, label_smoothing, w.row_loss, nullptr, margin);
    PPV_LAUNCH_OK("aam_row_kernel");
    aam_mean_kernel<<<1, 32, 0, st>>>(w.row_loss, B, loss);
    PPV_LAUNCH_OK("aam_mean_kernel");
    return PPV_OK;
}

int linear_head_backward(const float* H, const float* W, const int64_t* labels, const float* logits, int B, int D, int S, float margin, float scale,
                         int easy_margin, float label_smoothing, float* d_H, float* d_W, float* d_bias, void* ws, size_t ws_bytes, cudaStream_t st) {
    PPV_REQUIRE(H && W && labels && logits && d_H && d_W && d_bias, "linear_head_backward: null argument");
    if (int rc = check_workspace("linear_head_backward", ws, ws_bytes, aam_workspace_bytes(B, D, S), "ppv_aam_workspace_bytes")) return rc;
    int kind, K;
    int rc = decode_head(easy_margin, S, &kind, &K);
    if (!rc) rc = linear_head_check(easy_margin);
    if (rc) return rc;
    WsCarver cv{static_cast<uint8_t*>(ws)};
    AamWs w;
    carve_aam(cv, B, D, S, &w);
    float cm, sm, th, mmm;
    margin_consts(margin, &cm, &sm, &th, &mmm);
    aam_row_kernel<<<B, 256, 0, st>>>(logits, labels, B, S, 1, cm, sm, th, mmm, kind, scale, label_smoothing, w.row_loss, w.G, margin);
    PPV_LAUNCH_OK("aam_row_kernel(bwd)");
    lin_dh_kernel<<<dim3((D + 7) / 8, (B + LIN_ROWS - 1) / LIN_ROWS), 256, 0, st>>>(w.G, W, B, D, S, d_H);
    PPV_LAUNCH_OK("lin_dh_kernel");
    lin_dw_kernel<<<dim3((S + 127) / 128, (D + LIN_DCHUNK - 1) / LIN_DCHUNK), 128, 0, st>>>(w.G, H, B, D, S, d_W, d_bias);
    PPV_LAUNCH_OK("lin_dw_kernel");
    return PPV_OK;
}

}  // namespace ppv
