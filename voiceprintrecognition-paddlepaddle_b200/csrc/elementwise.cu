// HBM-bound kernels between the tensor-core GEMMs of the ECAPA-TDNN path:
//   pack_features   [B,T,F] fp32 -> split-bf16 planes in the padded time layout (+ reflect halo)
//   se_squeeze      SEBlock mean over time            (ppvector/models/ecapa_tdnn.py:69-78)
//   (SE excite = two small gather-GEMMs with ReLU / sigmoid epilogues, see ecapa.cu)
//   se_scale_res    s * x + residual                  (ecapa_tdnn.py:82, :142)
//   asp_global      global mean / std of ASP          (ppvector/models/pooling.py:89-92, 102-104)
//   asp_pool        masked softmax over time + weighted mean / std + asp_bn (pooling.py:115-123,
//                   ecapa_tdnn.py:271)
//   planes_to_f32   debug taps
// Layout: rows are frames (padded time layout, common.h), channels are contiguous, so a warp reads
// 32 x bf16x2 = 128 contiguous bytes per row; reductions over time keep per-thread fp32 partials and
// finish through shared memory in a fixed order (deterministic).
#include "common.h"
#include "ptx.cuh"

namespace ppv {

__device__ __forceinline__ float2 ld_split2(const __nv_bfloat16* hi, const __nv_bfloat16* lo, int64_t off) {
    const __nv_bfloat162 h = *reinterpret_cast<const __nv_bfloat162*>(hi + off);
    const __nv_bfloat162 l = *reinterpret_cast<const __nv_bfloat162*>(lo + off);
    const float2 hf = __bfloat1622float2(h);
    const float2 lf = __bfloat1622float2(l);
    return make_float2(hf.x + lf.x, hf.y + lf.y);
}
__device__ __forceinline__ void st_split2(__nv_bfloat16* hi, __nv_bfloat16* lo, int64_t off, float a, float b) {
    __nv_bfloat16 h0, l0, h1, l1;
    split_bf16(a, h0, l0);
    split_bf16(b, h1, l1);
    *reinterpret_cast<uint32_t*>(hi + off) = pack_bf16x2(h0, h1);
    *reinterpret_cast<uint32_t*>(lo + off) = pack_bf16x2(l0, l1);
}

// ------------------------------------------------------------------------------------------------
// pack_features: one warp per frame row; channels >= F are zero-filled (K padding of the first conv).
__global__ void pack_features_kernel(const float* __restrict__ feat, int B, int T, int F, Planes out, int P, int Tp) {
    griddep_launch_dependents();
    griddep_wait();
    const int warps_per_block = blockDim.x >> 5;
    const int64_t frame = int64_t(blockIdx.x) * warps_per_block + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    if (frame >= int64_t(B) * T) return;
    const int b = int(frame / T);
    const int t = int(frame - int64_t(b) * T);
    const float* src = feat + frame * F;
    const int64_t row = int64_t(b) * Tp + P + t;
    int64_t rows[3] = {row, -1, -1};
    if (t >= 1 && t <= P) rows[1] = row - 2 * t;
    const int u = T - 1 - t;
    if (u >= 1 && u <= P) rows[2] = row + 2 * u;
    for (int c = 2 * lane; c < out.ld; c += 64) {
        const float a = (c < F) ? src[c] : 0.f;
        const float bb = (c + 1 < F) ? src[c + 1] : 0.f;
#pragma unroll
        for (int k = 0; k < 3; ++k)
            if (rows[k] >= 0) st_split2(out.hi(), out.lo(), rows[k] * out.ld + c, a, bb);
    }
}

int launch_pack_features(const float* feat, int B, int T, int F, const Planes& out, int P, int Tp, cudaStream_t st) {
    const int64_t frames = int64_t(B) * T;
    const int wpb = 8;
    PPV_PDL_OK(launch_pdl(pack_features_kernel, dim3(unsigned((frames + wpb - 1) / wpb)), dim3(wpb * 32), 0, st, feat, B, T, F, out, P, Tp),
               "pack_features_kernel");
    return PPV_OK;
}

// ------------------------------------------------------------------------------------------------
// Column statistics over the valid frames of one utterance.  Block = (utterance b, 64-channel slab),
// 256 threads = 8 warps; warp w takes frames w, w+8, ...; lane l takes channels 2l, 2l+1 of the slab.
constexpr int STAT_WARPS = 8;

__device__ __forceinline__ float2 block_colsum(float2 v, float2 (*s_part)[32], int warp, int lane) {
    s_part[warp][lane] = v;
    __syncthreads();
    float2 r = make_float2(0.f, 0.f);
#pragma unroll
    for (int w = 0; w < STAT_WARPS; ++w) {
        r.x += s_part[w][lane].x;
        r.y += s_part[w][lane].y;
    }
    __syncthreads();
    return r;
}

// mode 0: mean -> out_f32[b, C] and/or planes [B, C]                                  (SE squeeze)
// mode 1: mean and std = sqrt(clip(var, eps)) -> planes [B, 2C] (mean | std)             (ASP global context)
// mode 2: mean and std = sqrt(var_unbiased + eps) -> planes [B, 2C]                       (TSTP, pooling.py:138-146)
// mode 3: mean and var_unbiased -> planes [B, 2C]                                          (TSP, pooling.py:42-45)
// One pass: each thread keeps Welford's running (count, mean, M2) over its frames; the lanes and then the warps are merged with Chan's
// formula in a fixed order (deterministic, no atomics).  A sum of squares about a fixed shift would cancel in fp32 when the shift
// sits far from the channel's mean (a frame 0 at the ReLU floor under a channel 20-50 std above it).
// Each lane owns 8 channels (one 16-byte load per plane), 4 frames per warp, 32 frames per block iteration.
__device__ __forceinline__ void chan_merge(float& na, float& ma, float& qa, float nb, float mb, float qb) {
    const float n = na + nb;
    const float d = mb - ma;
    const float f = n > 0.f ? nb / n : 0.f;
    ma = fmaf(d, f, ma);
    qa = qa + qb + d * d * na * f;
    na = n;
}

__global__ void __launch_bounds__(STAT_WARPS * 32)
    colstats_kernel(Planes x, int col0, int C, int T_all, int P, int Tp, int mode, float eps, float inv_count, float* __restrict__ out_f32,
                    Planes out_pl, const int* __restrict__ nvalid) {
    __shared__ float s_m[STAT_WARPS][64];
    __shared__ float s_q[STAT_WARPS][64];
    __shared__ float s_n[STAT_WARPS];
    griddep_launch_dependents();
    griddep_wait();
    const int b = blockIdx.y;
    // `lengths` of the reference (ecapa_tdnn.py:71-75, pooling.py:96-103): statistics over the first nvalid[b] frames only
    const int T = nvalid ? max(1, min(T_all, nvalid[b])) : T_all;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int cg = lane & 7, rsub = lane >> 3;
    const int c = col0 + blockIdx.x * 64 + cg * 8;
    const int64_t row0 = int64_t(b) * Tp + P;
    auto load8 = [&](int64_t row, float (&v)[8]) {
        const uint4 h = *reinterpret_cast<const uint4*>(x.hi() + row * x.ld + c);
        const uint4 l = *reinterpret_cast<const uint4*>(x.lo() + row * x.ld + c);
        const uint32_t hw[4] = {h.x, h.y, h.z, h.w}, lw[4] = {l.x, l.y, l.z, l.w};
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const float2 hf = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&hw[i]));
            const float2 lf = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&lw[i]));
            v[2 * i] = hf.x + lf.x;
            v[2 * i + 1] = hf.y + lf.y;
        }
    };
    float n = 0.f, m[8], q[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) m[i] = q[i] = 0.f;
#pragma unroll 4
    for (int t = warp * 4 + rsub; t < T; t += STAT_WARPS * 4) {
        float v[8];
        load8(row0 + t, v);
        n += 1.f;
        const float rn = 1.f / n;
#pragma unroll
        for (int i = 0; i < 8; ++i) {
            const float d = v[i] - m[i];
            m[i] = fmaf(d, rn, m[i]);  // the first frame: m = v exactly
            q[i] = fmaf(d, v[i] - m[i], q[i]);
        }
    }
#pragma unroll
    for (int sh = 8; sh <= 16; sh *= 2) {
        const float nb = __shfl_xor_sync(0xffffffffu, n, sh);
#pragma unroll
        for (int i = 0; i < 8; ++i) {
            const float mb = __shfl_xor_sync(0xffffffffu, m[i], sh), qb = __shfl_xor_sync(0xffffffffu, q[i], sh);
            float na = n;
            chan_merge(na, m[i], q[i], nb, mb, qb);
        }
        n += nb;
    }
    if (rsub == 0) {
        if (cg == 0) s_n[warp] = n;
#pragma unroll
        for (int i = 0; i < 8; ++i) {
            s_m[warp][cg * 8 + i] = m[i];
            s_q[warp][cg * 8 + i] = q[i];
        }
    }
    __syncthreads();
    if (threadIdx.x < 64) {
        const int ch = threadIdx.x;  // channel within the slab
        float N = s_n[0], M = s_m[0][ch], Q = s_q[0][ch];
#pragma unroll
        for (int w = 1; w < STAT_WARPS; ++w) chan_merge(N, M, Q, s_n[w], s_m[w][ch], s_q[w][ch]);
        const float inv = inv_count > 0.f ? inv_count : 1.f / float(T);  // inv_count: zero-bordered images are summed whole
        const float mean = inv_count > 0.f ? M * float(T) * inv : M;
        const float ssq = Q;  // sum of squared deviations from the mean
        const int cc = blockIdx.x * 64 + ch;
        if (mode == 0) {
            if (out_f32) out_f32[int64_t(b) * C + cc] = mean;
            if (out_pl.base) {
                __nv_bfloat16 h, l;
                split_bf16(mean, h, l);
                out_pl.hi()[int64_t(b) * out_pl.ld + cc] = h;
                out_pl.lo()[int64_t(b) * out_pl.ld + cc] = l;
            }
        } else {
            // mode 1: ASP global std = sqrt(clip(var_biased, eps)); mode 2: TSTP std = sqrt(var_unbiased + eps)
            // mode 3: unbiased VARIANCE, no square root (TemporalStatisticsPooling, pooling.py:44)
            const float sd = (mode == 2)   ? sqrtf(fmaxf(ssq, 0.f) / float(T > 1 ? T - 1 : 1) + eps)
                             : (mode == 3) ? fmaxf(ssq, 0.f) / float(T > 1 ? T - 1 : 1)
                                           : sqrtf(fmaxf(ssq * inv, eps));
            if (out_f32) {  // fp32 [B][2C] (the training step's TSP pooling)
                out_f32[int64_t(b) * 2 * C + cc] = mean;
                out_f32[int64_t(b) * 2 * C + C + cc] = sd;
            }
            if (!out_pl.base) return;
            __nv_bfloat16 h, l;
            split_bf16(mean, h, l);
            out_pl.hi()[int64_t(b) * out_pl.ld + cc] = h;
            out_pl.lo()[int64_t(b) * out_pl.ld + cc] = l;
            split_bf16(sd, h, l);
            out_pl.hi()[int64_t(b) * out_pl.ld + C + cc] = h;
            out_pl.lo()[int64_t(b) * out_pl.ld + C + cc] = l;
        }
    }
}

// nvalid[b] = #{t in [0,T): float(t) < lengths[b] * float(T)} -- the reference's length_to_mask(lengths * L, max_len=L)
// (ppvector/models/utils.py:8-19) compares a float arange with the float product, no truncation
__global__ void lengths_to_counts_kernel(const float* __restrict__ lengths, int B, int T, int* __restrict__ nvalid) {
    griddep_launch_dependents();
    griddep_wait();
    const int b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= B) return;
    const float lim = lengths[b] * float(T);
    int n = 0;
    for (int t = 0; t < T; ++t) n += (float(t) < lim) ? 1 : 0;
    nvalid[b] = n;
}
int launch_lengths_to_counts(const float* lengths, int B, int T, int* nvalid, cudaStream_t st) {
    PPV_PDL_OK(launch_pdl(lengths_to_counts_kernel, dim3((B + 127) / 128), dim3(128), 0, st, lengths, B, T, nvalid), "lengths_to_counts_kernel");
    return PPV_OK;
}

int launch_colstats(const Planes& x, int col0, int C, int B, int T, int P, int Tp, int mode, float eps, float* out_f32,
                    const Planes& out_pl, cudaStream_t st, float inv_count, const int* nvalid) {
    PPV_REQUIRE(C % 64 == 0 && col0 % 8 == 0 && x.ld % 8 == 0, "colstats: C % 64, col0 % 8, ld % 8 required");
    dim3 grid(C / 64, B);
    PPV_PDL_OK(launch_pdl(colstats_kernel, grid, dim3(STAT_WARPS * 32), 0, st, x, col0, C, T, P, Tp, mode, eps, inv_count, out_f32, out_pl, nvalid),
               "colstats_kernel");
    return PPV_OK;
}

// ------------------------------------------------------------------------------------------------
// out[r, oc0 + c] = scale[b(r), c] * z[r, c] + res[r, rc0 + c]   for every row of the padded layout.
__device__ __forceinline__ void unpack8(const uint4& h, const uint4& l, float (&v)[8]) {
    const uint32_t hw[4] = {h.x, h.y, h.z, h.w}, lw[4] = {l.x, l.y, l.z, l.w};
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const float2 hf = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&hw[i]));
        const float2 lf = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&lw[i]));
        v[2 * i] = hf.x + lf.x;
        v[2 * i + 1] = hf.y + lf.y;
    }
}
// 8 channels (16 bytes per plane) per thread per iteration
__global__ void __launch_bounds__(256)
    se_scale_res_kernel(Planes z, const float* __restrict__ scale, Planes res, int rc0, Planes out, int oc0, int C, int Tp,
                        int64_t rows, int relu, float relu_max) {
    griddep_launch_dependents();
    griddep_wait();
    const int groups = C >> 3;
    const int64_t total = rows * groups;
    for (int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x; i < total; i += int64_t(gridDim.x) * blockDim.x) {
        const int64_t r = i / groups;
        const int c = int(i - r * groups) * 8;
        const int b = int(r / Tp);
        float zv[8], rv[8];
        unpack8(*reinterpret_cast<const uint4*>(z.hi() + r * z.ld + c), *reinterpret_cast<const uint4*>(z.lo() + r * z.ld + c), zv);
        unpack8(*reinterpret_cast<const uint4*>(res.hi() + r * res.ld + rc0 + c),
                *reinterpret_cast<const uint4*>(res.lo() + r * res.ld + rc0 + c), rv);
        float4 s0 = make_float4(1.f, 1.f, 1.f, 1.f), s1 = s0;  // scale == nullptr: plain residual add
        if (scale) {
            s0 = *reinterpret_cast<const float4*>(scale + int64_t(b) * C + c);
            s1 = *reinterpret_cast<const float4*>(scale + int64_t(b) * C + c + 4);
        }
        const float sv[8] = {s0.x, s0.y, s0.z, s0.w, s1.x, s1.y, s1.z, s1.w};
        uint32_t h[4], l[4];
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            __nv_bfloat16 h0, l0, h1, l1;
            float y0 = fmaf(sv[2 * k], zv[2 * k], rv[2 * k]), y1 = fmaf(sv[2 * k + 1], zv[2 * k + 1], rv[2 * k + 1]);
            if (relu) {
                y0 = fmaxf(y0, 0.f);
                y1 = fmaxf(y1, 0.f);
                if (relu_max > 0.f) {
                    y0 = fminf(y0, relu_max);
                    y1 = fminf(y1, relu_max);
                }
            }
            split_bf16(y0, h0, l0);
            split_bf16(y1, h1, l1);
            h[k] = pack_bf16x2(h0, h1);
            l[k] = pack_bf16x2(l0, l1);
        }
        *reinterpret_cast<uint4*>(out.hi() + r * out.ld + oc0 + c) = make_uint4(h[0], h[1], h[2], h[3]);
        *reinterpret_cast<uint4*>(out.lo() + r * out.ld + oc0 + c) = make_uint4(l[0], l[1], l[2], l[3]);
    }
}

int launch_se_scale_res(const Planes& z, const float* scale, const Planes& res, int rc0, const Planes& out, int oc0, int C,
                        int Tp, int64_t rows, int num_sms, cudaStream_t st, int relu, float relu_max) {
    PPV_REQUIRE(C % 8 == 0 && rc0 % 8 == 0 && oc0 % 8 == 0, "se_scale_res: 8-channel alignment required");
    const int64_t total = rows * (C / 8);
    const int64_t want = (total + 255) / 256;
    const int grid = int(std::min<int64_t>(want, int64_t(num_sms) * 16));
    PPV_PDL_OK(launch_pdl(se_scale_res_kernel, dim3(grid), dim3(256), 0, st, z, scale, res, rc0, out, oc0, C, Tp, rows, relu, relu_max), "se_scale_res_kernel");
    return PPV_OK;
}

// ------------------------------------------------------------------------------------------------
// ASP pooling (lengths = None): per (utterance, channel)
//   a_t = softmax_t(logit_t);  mean = sum a_t x_t;  std = sqrt(clip(sum a_t (x_t - mean)^2, eps))
// then asp_bn (eval affine) on the concatenated [mean | std] -> split planes [B, 2C] feeding the fc GEMM.
__global__ void __launch_bounds__(STAT_WARPS * 32)
    asp_pool_kernel(const float* __restrict__ logits, int64_t lg_ld, Planes x, int C, int T, int P, int Tp, float eps,
                    const float* __restrict__ bn_scale, const float* __restrict__ bn_shift, Planes out_pl,
                    float* __restrict__ out_raw) {
    __shared__ float2 s_part[STAT_WARPS][32];
    const int b = blockIdx.y;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int c = blockIdx.x * 64 + 2 * lane;
    const int64_t row0 = int64_t(b) * Tp + P;
    // pass 1: max
    float2 mx = make_float2(-INFINITY, -INFINITY);
    for (int t = warp; t < T; t += STAT_WARPS) {
        const float2 l = *reinterpret_cast<const float2*>(logits + (row0 + t) * lg_ld + c);
        mx.x = fmaxf(mx.x, l.x);
        mx.y = fmaxf(mx.y, l.y);
    }
    s_part[warp][lane] = mx;
    __syncthreads();
#pragma unroll
    for (int w = 0; w < STAT_WARPS; ++w) {
        mx.x = fmaxf(mx.x, s_part[w][lane].x);
        mx.y = fmaxf(mx.y, s_part[w][lane].y);
    }
    __syncthreads();
    // pass 2: sum e, sum e x
    float2 se = make_float2(0.f, 0.f), sx = make_float2(0.f, 0.f);
    for (int t = warp; t < T; t += STAT_WARPS) {
        const float2 l = *reinterpret_cast<const float2*>(logits + (row0 + t) * lg_ld + c);
        const float2 v = ld_split2(x.hi(), x.lo(), (row0 + t) * x.ld + c);
        const float ex = expf(l.x - mx.x), ey = expf(l.y - mx.y);
        se.x += ex;
        se.y += ey;
        sx.x = fmaf(ex, v.x, sx.x);
        sx.y = fmaf(ey, v.y, sx.y);
    }
    se = block_colsum(se, s_part, warp, lane);
    sx = block_colsum(sx, s_part, warp, lane);
    const float2 inv = make_float2(1.f / se.x, 1.f / se.y);
    const float2 mean = make_float2(sx.x * inv.x, sx.y * inv.y);
    // pass 3: weighted variance around the mean
    float2 sv = make_float2(0.f, 0.f);
    for (int t = warp; t < T; t += STAT_WARPS) {
        const float2 l = *reinterpret_cast<const float2*>(logits + (row0 + t) * lg_ld + c);
        const float2 v = ld_split2(x.hi(), x.lo(), (row0 + t) * x.ld + c);
        const float ax = expf(l.x - mx.x) * inv.x, ay = expf(l.y - mx.y) * inv.y;
        const float dx = v.x - mean.x, dy = v.y - mean.y;
        sv.x = fmaf(ax, dx * dx, sv.x);
        sv.y = fmaf(ay, dy * dy, sv.y);
    }
    sv = block_colsum(sv, s_part, warp, lane);
    if (warp == 0) {
        const float stdx = sqrtf(fmaxf(sv.x, eps)), stdy = sqrtf(fmaxf(sv.y, eps));
        if (out_raw) {
            *reinterpret_cast<float2*>(out_raw + int64_t(b) * 2 * C + c) = mean;
            *reinterpret_cast<float2*>(out_raw + int64_t(b) * 2 * C + C + c) = make_float2(stdx, stdy);
        }
        if (!bn_scale || !out_pl.base) return;  // training path: raw statistics only
        const float2 s0 = *reinterpret_cast<const float2*>(bn_scale + c), h0 = *reinterpret_cast<const float2*>(bn_shift + c);
        const float2 s1 = *reinterpret_cast<const float2*>(bn_scale + C + c),
                     h1 = *reinterpret_cast<const float2*>(bn_shift + C + c);
        st_split2(out_pl.hi(), out_pl.lo(), int64_t(b) * out_pl.ld + c, fmaf(mean.x, s0.x, h0.x), fmaf(mean.y, s0.y, h0.y));
        st_split2(out_pl.hi(), out_pl.lo(), int64_t(b) * out_pl.ld + C + c, fmaf(stdx, s1.x, h1.x), fmaf(stdy, s1.y, h1.y));
    }
}

int launch_asp_pool(const float* logits, int64_t lg_ld, const Planes& x, int C, int B, int T, int P, int Tp, float eps,
                    const float* bn_scale, const float* bn_shift, const Planes& out_pl, float* out_raw, cudaStream_t st) {
    PPV_REQUIRE(C % 64 == 0, "asp_pool: C must be a multiple of 64");
    dim3 grid(C / 64, B);
    asp_pool_kernel<<<grid, STAT_WARPS * 32, 0, st>>>(logits, lg_ld, x, C, T, P, Tp, eps, bn_scale, bn_shift, out_pl, out_raw);
    PPV_LAUNCH_OK("asp_pool_kernel");
    return PPV_OK;
}

// ------------------------------------------------------------------------------------------------
// AFF blend: xo = x * (1 + t) + y * (1 - t), 8 channels per thread
__global__ void __launch_bounds__(256)
    aff_combine_kernel(Planes x, int xc0, Planes y, int yc0, Planes t, Planes out, int C, int64_t rows) {
    griddep_launch_dependents();
    griddep_wait();
    const int groups = C >> 3;
    const int64_t total = rows * groups;
    for (int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x; i < total; i += int64_t(gridDim.x) * blockDim.x) {
        const int64_t r = i / groups;
        const int c = int(i - r * groups) * 8;
        float xv[8], yv[8], tv[8];
        unpack8(*reinterpret_cast<const uint4*>(x.hi() + r * x.ld + xc0 + c), *reinterpret_cast<const uint4*>(x.lo() + r * x.ld + xc0 + c), xv);
        unpack8(*reinterpret_cast<const uint4*>(y.hi() + r * y.ld + yc0 + c), *reinterpret_cast<const uint4*>(y.lo() + r * y.ld + yc0 + c), yv);
        unpack8(*reinterpret_cast<const uint4*>(t.hi() + r * t.ld + c), *reinterpret_cast<const uint4*>(t.lo() + r * t.ld + c), tv);
        uint32_t h[4], l[4];
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            __nv_bfloat16 h0, l0, h1, l1;
            split_bf16(fmaf(xv[2 * k], 1.f + tv[2 * k], yv[2 * k] * (1.f - tv[2 * k])), h0, l0);
            split_bf16(fmaf(xv[2 * k + 1], 1.f + tv[2 * k + 1], yv[2 * k + 1] * (1.f - tv[2 * k + 1])), h1, l1);
            h[k] = pack_bf16x2(h0, h1);
            l[k] = pack_bf16x2(l0, l1);
        }
        *reinterpret_cast<uint4*>(out.hi() + r * out.ld + c) = make_uint4(h[0], h[1], h[2], h[3]);
        *reinterpret_cast<uint4*>(out.lo() + r * out.ld + c) = make_uint4(l[0], l[1], l[2], l[3]);
    }
}

int launch_aff_combine(const Planes& x, int xc0, const Planes& y, int yc0, const Planes& t, const Planes& out, int C, int64_t rows, int num_sms,
                       cudaStream_t st) {
    PPV_REQUIRE(C % 8 == 0 && xc0 % 8 == 0 && yc0 % 8 == 0, "aff_combine: 8-channel alignment required");
    const int64_t total = rows * (C / 8);
    const int grid = int(std::min<int64_t>((total + 255) / 256, int64_t(num_sms) * 16));
    PPV_PDL_OK(launch_pdl(aff_combine_kernel, dim3(grid), dim3(256), 0, st, x, xc0, y, yc0, t, out, C, rows), "aff_combine_kernel");
    return PPV_OK;
}

// planes (padded layout, valid frames) -> fp32 [B,T,C]   (debug taps / tests)
__global__ void planes_to_f32_kernel(Planes x, int col0, int C, int B, int T, int P, int Tp, float* __restrict__ out) {
    const int64_t total = int64_t(B) * T * C;
    for (int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x; i < total; i += int64_t(gridDim.x) * blockDim.x) {
        const int c = int(i % C);
        const int64_t f = i / C;
        const int b = int(f / T), t = int(f % T);
        const int64_t off = (int64_t(b) * Tp + P + t) * x.ld + col0 + c;
        out[i] = __bfloat162float(x.hi()[off]) + __bfloat162float(x.lo()[off]);
    }
}

int launch_planes_to_f32(const Planes& x, int col0, int C, int B, int T, int P, int Tp, float* out, cudaStream_t st) {
    const int64_t total = int64_t(B) * T * C;
    const int grid = int(std::min<int64_t>((total + 255) / 256, 132 * 32));
    planes_to_f32_kernel<<<grid, 256, 0, st>>>(x, col0, C, B, T, P, Tp, out);
    PPV_LAUNCH_OK("planes_to_f32_kernel");
    return PPV_OK;
}

// fp32 row-major [rows, cols] -> split planes (test hook + weight upload helper)
__global__ void f32_to_planes_kernel(const float* __restrict__ src, int64_t rows, int cols, Planes out) {
    const int64_t total = rows * cols;
    for (int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x; i < total; i += int64_t(gridDim.x) * blockDim.x) {
        const int64_t r = i / cols;
        const int c = int(i - r * cols);
        __nv_bfloat16 h, l;
        split_bf16(src[i], h, l);
        out.hi()[r * out.ld + c] = h;
        out.lo()[r * out.ld + c] = l;
    }
}

int launch_f32_to_planes(const float* src, int64_t rows, int cols, const Planes& out, cudaStream_t st) {
    const int64_t total = rows * cols;
    const int grid = int(std::min<int64_t>((total + 255) / 256, 132 * 32));
    f32_to_planes_kernel<<<grid, 256, 0, st>>>(src, rows, cols, out);
    PPV_LAUNCH_OK("f32_to_planes_kernel");
    return PPV_OK;
}

}  // namespace ppv
