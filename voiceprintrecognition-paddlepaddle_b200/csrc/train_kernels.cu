// Kernels of the training step that are not tensor-core GEMMs (SURVEY.md §8 row a11; reference ppvector/trainer.py:206-229):
// train-mode BatchNorm (batch statistics over all valid frames, ppvector/models/utils.py:96-119 -> paddle.nn.BatchNorm1D)
// forward and backward fused with the ReLU backward, reflect-padding gradient fold (utils.py:79-93 backward), bias / column
// reductions, plane transposes for the weight-gradient GEMM, the small fp32 dense layers (SE block, fc, per-utterance ASP
// context), ASP softmax-pooling backward, Adam.  Every reduction is two-stage (per-utterance partials, then a finalize
// kernel in a fixed order): no atomics, results are bitwise reproducible.
#include <math.h>

#include "common.h"
#include "ptx.cuh"
#include "train.h"

namespace ppv {

namespace {

constexpr int TR_WARPS = 8;

__device__ __forceinline__ void tr_unpack8(const uint4& h, const uint4& l, float (&v)[8]) {
    const uint32_t hw[4] = {h.x, h.y, h.z, h.w}, lw[4] = {l.x, l.y, l.z, l.w};
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const float2 hf = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&hw[i]));
        const float2 lf = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&lw[i]));
        v[2 * i] = hf.x + lf.x;
        v[2 * i + 1] = hf.y + lf.y;
    }
}
__device__ __forceinline__ void tr_load8(const Planes& p, int64_t row, int col, float (&v)[8]) {
    tr_unpack8(*reinterpret_cast<const uint4*>(p.hi() + row * p.ld + col), *reinterpret_cast<const uint4*>(p.lo() + row * p.ld + col), v);
}
__device__ __forceinline__ void tr_store8(const Planes& p, int64_t row, int col, const float (&v)[8]) {
    uint32_t h[4], l[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        __nv_bfloat16 h0, l0, h1, l1;
        split_bf16(v[2 * k], h0, l0);
        split_bf16(v[2 * k + 1], h1, l1);
        h[k] = pack_bf16x2(h0, h1);
        l[k] = pack_bf16x2(l0, l1);
    }
    *reinterpret_cast<uint4*>(p.hi() + row * p.ld + col) = make_uint4(h[0], h[1], h[2], h[3]);
    *reinterpret_cast<uint4*>(p.lo() + row * p.ld + col) = make_uint4(l[0], l[1], l[2], l[3]);
}
__device__ __forceinline__ void tr_ld8f(const float* p, float (&v)[8]) {
    const float4 a = *reinterpret_cast<const float4*>(p), b = *reinterpret_cast<const float4*>(p + 4);
    v[0] = a.x, v[1] = a.y, v[2] = a.z, v[3] = a.w, v[4] = b.x, v[5] = b.y, v[6] = b.z, v[7] = b.w;
}

// Gradient of a tensor at (utterance b, frame t, channels c..c+7) summed over its sources (train.h: GradSrcList).
__device__ __forceinline__ void tr_load_grad8(const GradSrcList& gl, int b, int t, int T, int P, int Tp, int c, float (&g)[8]) {
    const int64_t row = int64_t(b) * Tp + P + t;
#pragma unroll
    for (int i = 0; i < 8; ++i) g[i] = 0.f;
    for (int s = 0; s < gl.n; ++s) {
        const GradSrc& gs = gl.s[s];
        float v[8];
#pragma unroll
        for (int i = 0; i < 8; ++i) v[i] = 0.f;
        if (gs.t.base) {
            tr_load8(gs.t, row, gs.col0 + c, v);
            if (gs.fold) {  // reflect padding backward: the halo rows that mirror this frame
                float w[8];
                if (t >= 1 && t <= P) {
                    tr_load8(gs.t, row - 2 * t, gs.col0 + c, w);
#pragma unroll
                    for (int i = 0; i < 8; ++i) v[i] += w[i];
                }
                const int u = T - 1 - t;
                if (u >= 1 && u <= P) {
                    tr_load8(gs.t, row + 2 * u, gs.col0 + c, w);
#pragma unroll
                    for (int i = 0; i < 8; ++i) v[i] += w[i];
                }
            }
            if (gs.rowscale) {
                float sc[8];
                tr_ld8f(gs.rowscale + int64_t(b) * gs.row_ld + c, sc);
#pragma unroll
                for (int i = 0; i < 8; ++i) v[i] *= sc[i];
            }
            if (gs.dtanh.base) {
                float y[8];
                tr_load8(gs.dtanh, row, gs.dtanh_col0 + c, y);
#pragma unroll
                for (int i = 0; i < 8; ++i) v[i] *= 1.f - y[i] * y[i];
            }
        }
        if (gs.rowbias) {
            float bi[8];
            tr_ld8f(gs.rowbias + int64_t(b) * gs.row_ld + c, bi);
#pragma unroll
            for (int i = 0; i < 8; ++i) v[i] += bi[i];
        }
#pragma unroll
        for (int i = 0; i < 8; ++i) g[i] += v[i];
    }
}

// Block-level reduction helper: each lane holds NQ x 8 channel values (cg = lane & 7 -> channels cg*8.., rsub = lane >> 3);
// result for channel ch of the 64-wide slab lands in thread ch (< 64).
template <int NQ>
__device__ __forceinline__ void tr_block_reduce(float (&q)[NQ][8], float (*s_buf)[TR_WARPS][64], int warp, int lane, float (&out)[NQ]) {
    const int cg = lane & 7, rsub = lane >> 3;
#pragma unroll
    for (int n = 0; n < NQ; ++n)
#pragma unroll
        for (int i = 0; i < 8; ++i) {
            q[n][i] += __shfl_xor_sync(0xffffffffu, q[n][i], 8);
            q[n][i] += __shfl_xor_sync(0xffffffffu, q[n][i], 16);
        }
    if (rsub == 0) {
#pragma unroll
        for (int n = 0; n < NQ; ++n)
#pragma unroll
            for (int i = 0; i < 8; ++i) s_buf[n][warp][cg * 8 + i] = q[n][i];
    }
    __syncthreads();
    if (threadIdx.x < 64) {
#pragma unroll
        for (int n = 0; n < NQ; ++n) {
            float a = 0.f;
#pragma unroll
            for (int w = 0; w < TR_WARPS; ++w) a += s_buf[n][w][threadIdx.x];
            out[n] = a;
        }
    }
}

// ---------------------------------------------------------------------------------------------- BatchNorm forward
// per (utterance, 64-channel slab): S = sum(a - K), Q = sum((a - K)^2), K = a[first frame]
__global__ void __launch_bounds__(TR_WARPS * 32) bn_stats_kernel(Planes a, int col0, int C, int T, int P, int Tp, float* __restrict__ part) {
    __shared__ float s_buf[2][TR_WARPS][64];
    const int b = blockIdx.y, warp = threadIdx.x >> 5, lane = threadIdx.x & 31, cg = lane & 7, rsub = lane >> 3;
    const int c = blockIdx.x * 64 + cg * 8;
    const int64_t row0 = int64_t(b) * Tp + P;
    float k[8], q[2][8];
    tr_load8(a, row0, col0 + c, k);
#pragma unroll
    for (int i = 0; i < 8; ++i) q[0][i] = q[1][i] = 0.f;
    for (int t = warp * 4 + rsub; t < T; t += TR_WARPS * 4) {
        float v[8];
        tr_load8(a, row0 + t, col0 + c, v);
#pragma unroll
        for (int i = 0; i < 8; ++i) {
            const float d = v[i] - k[i];
            q[0][i] += d;
            q[1][i] = fmaf(d, d, q[1][i]);
        }
    }
    float out[2];
    tr_block_reduce<2>(q, s_buf, warp, lane, out);
    if (threadIdx.x < 64) {
        const int ch = blockIdx.x * 64 + threadIdx.x;
        const int64_t off = row0 * a.ld + col0 + ch;
        const float K = __bfloat162float(a.hi()[off]) + __bfloat162float(a.lo()[off]);
        float* p = part + (int64_t(b) * 3) * C + ch;
        p[0] = out[0];
        p[C] = out[1];
        p[2 * C] = K;
    }
}
// combine the per-utterance partials in double (all utterances hold T frames: mean = avg of the utterance means,
// M2 = sum M2_b + T * sum (mean_b - mean)^2); one warp per channel, lanes stride over the utterances, fixed reduction order.
// y = a * scale + shift with scale = gamma * rstd
__global__ void __launch_bounds__(256)
    bn_stats_finalize_kernel(const float* __restrict__ part, int B, int C, int T, float eps, float momentum, const float* __restrict__ gamma,
                             const float* __restrict__ beta, float* __restrict__ mean_out, float* __restrict__ rstd_out, float* __restrict__ scale,
                             float* __restrict__ shift, float* __restrict__ run_mean, float* __restrict__ run_var) {
    const int ch = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
    if (ch >= C) return;
    const double nb = T;
    double sm = 0.0, sm2 = 0.0;
    for (int b = lane; b < B; b += 32) {
        const float* p = part + (int64_t(b) * 3) * C + ch;
        const double S = p[0], Q = p[C], K = p[2 * C];
        sm += K + S / nb;
        sm2 += Q - S * S / nb;
    }
    for (int o = 16; o > 0; o >>= 1) {
        sm += __shfl_xor_sync(0xffffffffu, sm, o);
        sm2 += __shfl_xor_sync(0xffffffffu, sm2, o);
    }
    const double mean = sm / B;
    double sd = 0.0;
    for (int b = lane; b < B; b += 32) {
        const float* p = part + (int64_t(b) * 3) * C + ch;
        const double d = double(p[2 * C]) + double(p[0]) / nb - mean;
        sd += d * d;
    }
    for (int o = 16; o > 0; o >>= 1) sd += __shfl_xor_sync(0xffffffffu, sd, o);
    if (lane != 0) return;
    const double var = fmax((sm2 + nb * sd) / (nb * B), 0.0);  // biased, as used for the normalisation
    const float rstd = float(1.0 / sqrt(var + double(eps)));
    mean_out[ch] = float(mean);
    rstd_out[ch] = rstd;
    const float sc = gamma[ch] * rstd;
    scale[ch] = sc;
    shift[ch] = beta[ch] - float(mean) * sc;
    if (run_mean) {  // paddle: running = momentum * running + (1 - momentum) * batch (biased batch variance)
        run_mean[ch] = momentum * run_mean[ch] + (1.f - momentum) * float(mean);
        run_var[ch] = momentum * run_var[ch] + (1.f - momentum) * float(var);
    }
}

// y = a * scale + shift (optionally tanh), valid frames + reflect halo rows; optional second output out2 = y + add
__global__ void __launch_bounds__(256) bn_apply_kernel(BnApplyArgs p) {
    const int groups = p.C >> 3;
    const int64_t total = int64_t(p.B) * p.T * groups;
    for (int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x; i < total; i += int64_t(gridDim.x) * blockDim.x) {
        const int c = int(i % groups) * 8;
        const int64_t bt = i / groups;
        const int b = int(bt / p.T), t = int(bt % p.T);
        const int64_t row = int64_t(b) * p.Tp + p.P + t;
        float v[8], sc[8], sh[8];
        tr_load8(p.a, row, p.a_col0 + c, v);
        tr_ld8f(p.scale + c, sc);
        tr_ld8f(p.shift + c, sh);
#pragma unroll
        for (int k = 0; k < 8; ++k) {
            v[k] = fmaf(v[k], sc[k], sh[k]);
            if (p.tanh_) v[k] = tanhf(v[k]);
        }
        int64_t rows[3] = {row, -1, -1};
        if (t >= 1 && t <= p.P) rows[1] = row - 2 * t;
        const int u = p.T - 1 - t;
        if (u >= 1 && u <= p.P) rows[2] = row + 2 * u;
#pragma unroll
        for (int k = 0; k < 3; ++k)
            if (rows[k] >= 0) tr_store8(p.y, rows[k], p.y_col0 + c, v);
        if (p.out2.base) {
            float w[8];
            tr_load8(p.add, row, p.add_col0 + c, w);
#pragma unroll
            for (int k = 0; k < 8; ++k) w[k] += v[k];
#pragma unroll
            for (int k = 0; k < 3; ++k)
                if (rows[k] >= 0) tr_store8(p.out2, rows[k], p.out2_col0 + c, w);
        }
    }
}

// ---------------------------------------------------------------------------------------------- BatchNorm + ReLU backward
// partials per (utterance, channel): s1 = sum dy, s2 = sum dy * xhat,  xhat = (a - mean) * rstd
__global__ void __launch_bounds__(TR_WARPS * 32)
    bn_bwd_reduce_kernel(GradSrcList gl, Planes a, int a_col0, int C, int T, int P, int Tp, const float* __restrict__ mean,
                         const float* __restrict__ rstd, float* __restrict__ part) {
    __shared__ float s_buf[2][TR_WARPS][64];
    // blockIdx.z splits the frames of an utterance (narrow layers would otherwise fill only B CTAs); partial index = b * nz + z
    const int b = blockIdx.y, warp = threadIdx.x >> 5, lane = threadIdx.x & 31, cg = lane & 7, rsub = lane >> 3;
    const int tchunk = (T + gridDim.z - 1) / gridDim.z, t_lo = blockIdx.z * tchunk, t_hi = min(T, t_lo + tchunk);
    const int pb = b * gridDim.z + blockIdx.z;
    const int c = blockIdx.x * 64 + cg * 8;
    const int64_t row0 = int64_t(b) * Tp + P;
    float mu[8], rs[8], q[2][8];
    tr_ld8f(mean + c, mu);
    tr_ld8f(rstd + c, rs);
#pragma unroll
    for (int i = 0; i < 8; ++i) q[0][i] = q[1][i] = 0.f;
    for (int t = t_lo + warp * 4 + rsub; t < t_hi; t += TR_WARPS * 4) {
        float g[8], v[8];
        tr_load_grad8(gl, b, t, T, P, Tp, c, g);
        tr_load8(a, row0 + t, a_col0 + c, v);
#pragma unroll
        for (int i = 0; i < 8; ++i) {
            q[0][i] += g[i];
            q[1][i] = fmaf(g[i], (v[i] - mu[i]) * rs[i], q[1][i]);
        }
    }
    float out[2];
    tr_block_reduce<2>(q, s_buf, warp, lane, out);
    if (threadIdx.x < 64) {
        const int ch = blockIdx.x * 64 + threadIdx.x;
        part[(int64_t(pb) * 2) * C + ch] = out[0];
        part[(int64_t(pb) * 2 + 1) * C + ch] = out[1];
    }
}
// out0[c] = sum_b part[b][0][c] (-> d beta), out1[c] = sum_b part[b][1][c] (-> d gamma); nq = 1 or 2.  One warp per channel.
__global__ void __launch_bounds__(256) part_finalize_kernel(const float* __restrict__ part, int B, int C, int nq, float* __restrict__ out0, float* __restrict__ out1) {
    const int ch = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
    if (ch >= C) return;
    float a0 = 0.f, a1 = 0.f;
    for (int b = lane; b < B; b += 32) {
        a0 += part[(int64_t(b) * nq) * C + ch];
        if (nq == 2) a1 += part[(int64_t(b) * nq + 1) * C + ch];
    }
    for (int o = 16; o > 0; o >>= 1) {
        a0 += __shfl_xor_sync(0xffffffffu, a0, o);
        a1 += __shfl_xor_sync(0xffffffffu, a1, o);
    }
    if (lane != 0) return;
    out0[ch] = a0;
    if (nq == 2 && out1) out1[ch] = a1;
}
// dz = relu'(a) * gamma * rstd * (dy - dbeta / N - xhat * dgamma / N)  -> planes (valid frames only), and per-utterance column
// sums of dz (bias gradient partials)
__global__ void __launch_bounds__(TR_WARPS * 32)
    bn_bwd_apply_kernel(GradSrcList gl, Planes a, int a_col0, int C, int T, int P, int Tp, const float* __restrict__ mean, const float* __restrict__ rstd,
                        const float* __restrict__ gamma, const float* __restrict__ dbeta, const float* __restrict__ dgamma, float inv_n, Planes dz,
                        int dz_col0, float* __restrict__ part) {
    __shared__ float s_buf[1][TR_WARPS][64];
    const int b = blockIdx.y, warp = threadIdx.x >> 5, lane = threadIdx.x & 31, cg = lane & 7, rsub = lane >> 3;
    const int tchunk = (T + gridDim.z - 1) / gridDim.z, t_lo = blockIdx.z * tchunk, t_hi = min(T, t_lo + tchunk);
    const int pb = b * gridDim.z + blockIdx.z;
    const int c = blockIdx.x * 64 + cg * 8;
    const int64_t row0 = int64_t(b) * Tp + P;
    float mu[8], rs[8], ga[8], db[8], dg[8], q[1][8];
    tr_ld8f(mean + c, mu);
    tr_ld8f(rstd + c, rs);
    tr_ld8f(gamma + c, ga);
    tr_ld8f(dbeta + c, db);
    tr_ld8f(dgamma + c, dg);
#pragma unroll
    for (int i = 0; i < 8; ++i) q[0][i] = 0.f;
    for (int t = t_lo + warp * 4 + rsub; t < t_hi; t += TR_WARPS * 4) {
        float g[8], v[8], o[8];
        tr_load_grad8(gl, b, t, T, P, Tp, c, g);
        tr_load8(a, row0 + t, a_col0 + c, v);
#pragma unroll
        for (int i = 0; i < 8; ++i) {
            const float xh = (v[i] - mu[i]) * rs[i];
            const float da = ga[i] * rs[i] * (g[i] - db[i] * inv_n - xh * dg[i] * inv_n);
            o[i] = v[i] > 0.f ? da : 0.f;
            q[0][i] += o[i];
        }
        tr_store8(dz, row0 + t, dz_col0 + c, o);
    }
    float out[1];
    tr_block_reduce<1>(q, s_buf, warp, lane, out);
    if (threadIdx.x < 64) part[int64_t(pb) * C + blockIdx.x * 64 + threadIdx.x] = out[0];
}

// per-utterance column sums of the summed sources: part[b][c] = sum_t grad(b, t, c); optionally also writes the summed
// gradient as planes (valid frames) -- used to materialise d(out_i) = sum of its consumers' gradients
__global__ void __launch_bounds__(TR_WARPS * 32)
    grad_sum_kernel(GradSrcList gl, int C, int T, int P, int Tp, Planes out, int out_col0, float* __restrict__ part) {
    __shared__ float s_buf[1][TR_WARPS][64];
    const int b = blockIdx.y, warp = threadIdx.x >> 5, lane = threadIdx.x & 31, cg = lane & 7, rsub = lane >> 3;
    const int c = blockIdx.x * 64 + cg * 8;
    const int64_t row0 = int64_t(b) * Tp + P;
    float q[1][8];
#pragma unroll
    for (int i = 0; i < 8; ++i) q[0][i] = 0.f;
    for (int t = warp * 4 + rsub; t < T; t += TR_WARPS * 4) {
        float g[8];
        tr_load_grad8(gl, b, t, T, P, Tp, c, g);
#pragma unroll
        for (int i = 0; i < 8; ++i) q[0][i] += g[i];
        if (out.base) tr_store8(out, row0 + t, out_col0 + c, g);
    }
    float o[1];
    tr_block_reduce<1>(q, s_buf, warp, lane, o);
    if (threadIdx.x < 64 && part) part[int64_t(b) * C + blockIdx.x * 64 + threadIdx.x] = o[0];
}

// part[b][c] = sum_t g(b,t,c) * y[b,t,c]   (SE block: d(gate) = sum_t d(out) * y)
__global__ void __launch_bounds__(TR_WARPS * 32)
    grad_dot_kernel(GradSrcList gl, Planes y, int y_col0, int C, int T, int P, int Tp, float* __restrict__ part) {
    __shared__ float s_buf[1][TR_WARPS][64];
    const int b = blockIdx.y, warp = threadIdx.x >> 5, lane = threadIdx.x & 31, cg = lane & 7, rsub = lane >> 3;
    const int c = blockIdx.x * 64 + cg * 8;
    const int64_t row0 = int64_t(b) * Tp + P;
    float q[1][8];
#pragma unroll
    for (int i = 0; i < 8; ++i) q[0][i] = 0.f;
    for (int t = warp * 4 + rsub; t < T; t += TR_WARPS * 4) {
        float g[8], v[8];
        tr_load_grad8(gl, b, t, T, P, Tp, c, g);
        tr_load8(y, row0 + t, y_col0 + c, v);
#pragma unroll
        for (int i = 0; i < 8; ++i) q[0][i] = fmaf(g[i], v[i], q[0][i]);
    }
    float o[1];
    tr_block_reduce<1>(q, s_buf, warp, lane, o);
    if (threadIdx.x < 64) part[int64_t(b) * C + blockIdx.x * 64 + threadIdx.x] = o[0];
}

// ---------------------------------------------------------------------------------------------- transposes
// planes [rows][ld] columns [col0, col0+C) -> planes [C][out.ld] (out.ld >= rows): out[c][r] = in[r + shift][col0 + c], zero
// where r + shift falls outside [0, rows); 32 x 32 tiles, both planes.  (A conv tap of the weight-gradient GEMM is a row shift
// of the layer input: TMA cannot start a tile at an inner coordinate that is not 16-byte aligned, so the shift is applied here.)
__global__ void __launch_bounds__(256) transpose_planes_kernel(Planes in, int col0, int C, int64_t rows, Planes out, int shift0, int shift_step,
                                                               int64_t out_row_step) {
    __shared__ __nv_bfloat16 tile[2][32][33];
    // blockIdx.z = conv tap: shift = shift0 + z * shift_step, output rows start at z * out_row_step
    const int shift = shift0 + int(blockIdx.z) * shift_step;
    out.base += int64_t(blockIdx.z) * out_row_step * out.ld;
    const int64_t r0 = int64_t(blockIdx.x) * 32;
    const int c0 = blockIdx.y * 32;
    const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;  // 32 x 8
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        const int64_t r = r0 + ty + 8 * k + shift;
        const int c = c0 + tx;
        const bool ok = r >= 0 && r < rows && c < C;
        tile[0][ty + 8 * k][tx] = ok ? in.hi()[r * in.ld + col0 + c] : __float2bfloat16_rn(0.f);
        tile[1][ty + 8 * k][tx] = ok ? in.lo()[r * in.ld + col0 + c] : __float2bfloat16_rn(0.f);
    }
    __syncthreads();
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        const int c = c0 + ty + 8 * k;
        const int64_t r = r0 + tx;
        if (c < C && r < out.ld) {
            out.hi()[int64_t(c) * out.ld + r] = tile[0][tx][ty + 8 * k];
            out.lo()[int64_t(c) * out.ld + r] = tile[1][tx][ty + 8 * k];
        }
    }
}

// ---------------------------------------------------------------------------------------------- weights <-> GEMM layouts
// reference conv weight [Cout][Cin][taps] fp32 -> forward planes Wf[n][tap * Cinp + cin] and data-gradient planes
// Wd[cin][tap * Cout + n] (rows cin >= Cin and columns cin >= Cin stay zero)
__global__ void repack_conv_kernel(const float* __restrict__ w, int64_t w_ld, int Cout, int Cin, int Cinp, int taps, Planes wf, Planes wd) {
    const int64_t total = int64_t(Cout) * Cin * taps;
    for (int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x; i < total; i += int64_t(gridDim.x) * blockDim.x) {
        const int tap = int(i % taps);
        const int cin = int((i / taps) % Cin);
        const int n = int(i / (int64_t(taps) * Cin));
        __nv_bfloat16 h, l;
        split_bf16(w[int64_t(n) * w_ld + int64_t(cin) * taps + tap], h, l);
        const int64_t of = int64_t(n) * wf.ld + tap * Cinp + cin;
        wf.hi()[of] = h;
        wf.lo()[of] = l;
        if (wd.base) {
            const int64_t od = int64_t(cin) * wd.ld + tap * Cout + n;
            wd.hi()[od] = h;
            wd.lo()[od] = l;
        }
    }
}
// weight-gradient partials [splits][Cout (split_rows apart)][taps * Cinp] -> reference layout grad[n][cin][tap]
__global__ void wgrad_unpack_kernel(const float* __restrict__ part, int splits, int64_t split_rows, int Cout, int Cin, int Cinp, int taps,
                                    float* __restrict__ grad, int64_t g_ld) {
    const int64_t total = int64_t(Cout) * Cin * taps;
    const int64_t ld = int64_t(taps) * Cinp;
    for (int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x; i < total; i += int64_t(gridDim.x) * blockDim.x) {
        const int tap = int(i % taps);
        const int cin = int((i / taps) % Cin);
        const int n = int(i / (int64_t(taps) * Cin));
        float a = 0.f;
        for (int z = 0; z < splits; ++z) a += part[(int64_t(z) * split_rows + n) * ld + tap * Cinp + cin];
        grad[int64_t(n) * g_ld + int64_t(cin) * taps + tap] = a;
    }
}

// ---------------------------------------------------------------------------------------------- small dense layers (fp32)
// Y[m][n] = act(sum_k X[m][k] W[n][k] + bias[n]); act 0 none, 1 relu, 2 sigmoid.  One warp per output.
__global__ void __launch_bounds__(256) dense_fwd_kernel(const float* __restrict__ X, int64_t x_ld, const float* __restrict__ W, int64_t w_ld,
                                                        const float* __restrict__ bias, int M, int N, int K, int act, float* __restrict__ Y, int64_t y_ld) {
    const int64_t o = int64_t(blockIdx.x) * 8 + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    if (o >= int64_t(M) * N) return;
    const int m = int(o / N), n = int(o % N);
    float a = 0.f;
    for (int k = lane; k < K; k += 32) a = fmaf(X[m * x_ld + k], W[n * w_ld + k], a);
    for (int s = 16; s > 0; s >>= 1) a += __shfl_xor_sync(0xffffffffu, a, s);
    if (lane == 0) {
        a += bias ? bias[n] : 0.f;
        if (act == 1) a = fmaxf(a, 0.f);
        if (act == 2) a = 1.f / (1.f + expf(-a));
        Y[m * y_ld + n] = a;
    }
}
// dX[m][k] = sum_n dY[m][n] W[n][k]
__global__ void __launch_bounds__(256) dense_bwd_x_kernel(const float* __restrict__ dY, int64_t dy_ld, const float* __restrict__ W, int64_t w_ld, int M,
                                                          int N, int K, float* __restrict__ dX, int64_t dx_ld) {
    const int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
    if (i >= int64_t(M) * K) return;
    const int m = int(i / K), k = int(i % K);
    float a = 0.f;
    for (int n = 0; n < N; ++n) a = fmaf(dY[m * dy_ld + n], W[n * w_ld + k], a);
    dX[m * dx_ld + k] = a;
}
// dW[n][k] = sum_m dY[m][n] X[m][k];  db[n] = sum_m dY[m][n]
__global__ void __launch_bounds__(256) dense_bwd_w_kernel(const float* __restrict__ dY, int64_t dy_ld, const float* __restrict__ X, int64_t x_ld, int M,
                                                          int N, int K, float* __restrict__ dW, int64_t dw_ld, float* __restrict__ db) {
    const int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
    if (i >= int64_t(N) * K) return;
    const int n = int(i / K), k = int(i % K);
    float a = 0.f;
    for (int m = 0; m < M; ++m) a = fmaf(dY[m * dy_ld + n], X[m * x_ld + k], a);
    dW[n * dw_ld + k] = a;
    if (db && k == 0) {
        float s = 0.f;
        for (int m = 0; m < M; ++m) s += dY[m * dy_ld + n];
        db[n] = s;
    }
}
// in place: dy *= act'(y); act 1 relu (y > 0), 2 sigmoid (y (1 - y)); act 0: dy *= alpha
__global__ void act_bwd_kernel(float* __restrict__ dy, const float* __restrict__ y, int64_t n, int act, float alpha) {
    const int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
    if (i >= n) return;
    dy[i] = act == 0 ? dy[i] * alpha : act == 1 ? (y[i] > 0.f ? dy[i] : 0.f) : dy[i] * y[i] * (1.f - y[i]);
}

// BatchNorm1D over the batch axis of a [B][C] fp32 matrix (asp_bn), train mode
__global__ void bn1d_fwd_kernel(const float* __restrict__ x, int B, int C, float eps, float momentum, const float* __restrict__ gamma,
                                const float* __restrict__ beta, float* __restrict__ y, float* __restrict__ mean_out, float* __restrict__ rstd_out,
                                float* __restrict__ run_mean, float* __restrict__ run_var) {
    const int c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= C) return;
    double s = 0.0;
    for (int b = 0; b < B; ++b) s += x[int64_t(b) * C + c];
    const double mean = s / B;
    double m2 = 0.0;
    for (int b = 0; b < B; ++b) {
        const double d = x[int64_t(b) * C + c] - mean;
        m2 += d * d;
    }
    const double var = m2 / B;
    const float rstd = float(1.0 / sqrt(var + double(eps)));
    mean_out[c] = float(mean);
    rstd_out[c] = rstd;
    for (int b = 0; b < B; ++b) y[int64_t(b) * C + c] = (x[int64_t(b) * C + c] - float(mean)) * rstd * gamma[c] + beta[c];
    run_mean[c] = momentum * run_mean[c] + (1.f - momentum) * float(mean);
    run_var[c] = momentum * run_var[c] + (1.f - momentum) * float(var);
}
__global__ void bn1d_bwd_kernel(const float* __restrict__ dy, const float* __restrict__ x, int B, int C, const float* __restrict__ gamma,
                                const float* __restrict__ mean, const float* __restrict__ rstd, float* __restrict__ dx, float* __restrict__ dgamma,
                                float* __restrict__ dbeta) {
    const int c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= C) return;
    float s1 = 0.f, s2 = 0.f;
    for (int b = 0; b < B; ++b) {
        const float g = dy[int64_t(b) * C + c], xh = (x[int64_t(b) * C + c] - mean[c]) * rstd[c];
        s1 += g;
        s2 = fmaf(g, xh, s2);
    }
    dbeta[c] = s1;
    dgamma[c] = s2;
    const float inv = 1.f / float(B);
    for (int b = 0; b < B; ++b) {
        const float g = dy[int64_t(b) * C + c], xh = (x[int64_t(b) * C + c] - mean[c]) * rstd[c];
        dx[int64_t(b) * C + c] = gamma[c] * rstd[c] * (g - s1 * inv - xh * s2 * inv);
    }
}

// ---------------------------------------------------------------------------------------------- ASP backward
// Per (utterance, channel): attn = softmax_t(logit); mean = sum attn x; var = sum attn (x - mean)^2; std = sqrt(clamp(var, eps)).
// Given d mean, d std:  dvar = dstd / (2 std) (0 where var <= eps);  dattn_t = dmean x_t + dvar (x_t - mean)^2;
//   dx_t = attn_t (dmean + 2 dvar (x_t - mean));   dlogit_t = attn_t (dattn_t - sum_t' attn_t' dattn_t').
// (pooling.py:91-94, 118-125 with lengths = None).  Block = (utterance, 32-channel slab); warp w strides over frames.
__global__ void __launch_bounds__(256)
    asp_bwd_kernel(const float* __restrict__ logits, int64_t lg_ld, Planes x, int C, int T, int P, int Tp, float eps, const float* __restrict__ pooled,
                   const float* __restrict__ dpooled, Planes dlogits, Planes dx) {
    __shared__ float s_a[8][32], s_b[8][32];
    const int b = blockIdx.y, warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int c = blockIdx.x * 32 + lane;
    const int64_t row0 = int64_t(b) * Tp + P;
    auto xval = [&](int t) {
        const int64_t o = (row0 + t) * x.ld + c;
        return __bfloat162float(x.hi()[o]) + __bfloat162float(x.lo()[o]);
    };
    auto reduce = [&](float v, float (*buf)[32], bool is_max) {
        buf[warp][lane] = v;
        __syncthreads();
        float r = buf[0][lane];
#pragma unroll
        for (int w = 1; w < 8; ++w) r = is_max ? fmaxf(r, buf[w][lane]) : r + buf[w][lane];
        __syncthreads();
        return r;
    };
    float mx = -INFINITY;
    for (int t = warp; t < T; t += 8) mx = fmaxf(mx, logits[(row0 + t) * lg_ld + c]);
    mx = reduce(mx, s_a, true);
    float den = 0.f;
    for (int t = warp; t < T; t += 8) den += expf(logits[(row0 + t) * lg_ld + c] - mx);
    den = reduce(den, s_a, false);
    const float inv_den = 1.f / den;
    const float mean = pooled[int64_t(b) * 2 * C + c], sd = pooled[int64_t(b) * 2 * C + C + c];
    const float dmean = dpooled[int64_t(b) * 2 * C + c], dstd = dpooled[int64_t(b) * 2 * C + C + c];
    const float dvar = (sd * sd > eps) ? dstd / (2.f * sd) : 0.f;  // sd = sqrt(clamp(var, eps)): no gradient through the clamp floor
    float inner = 0.f;
    for (int t = warp; t < T; t += 8) {
        const float at = expf(logits[(row0 + t) * lg_ld + c] - mx) * inv_den, xv = xval(t), d = xv - mean;
        inner = fmaf(at, dmean * xv + dvar * d * d, inner);
    }
    inner = reduce(inner, s_b, false);
    for (int t = warp; t < T; t += 8) {
        const float at = expf(logits[(row0 + t) * lg_ld + c] - mx) * inv_den, xv = xval(t), d = xv - mean;
        const float dl = at * (dmean * xv + dvar * d * d - inner);
        const float dxv = at * (dmean + 2.f * dvar * d);
        __nv_bfloat16 h, l;
        const int64_t o = (row0 + t);
        split_bf16(dl, h, l);
        dlogits.hi()[o * dlogits.ld + c] = h;
        dlogits.lo()[o * dlogits.ld + c] = l;
        split_bf16(dxv, h, l);
        dx.hi()[o * dx.ld + c] = h;
        dx.lo()[o * dx.ld + c] = l;
    }
}
// global context statistics backward as a row scale / row bias on x (gstat = [mean | std] with std = sqrt(clamp(var_biased, eps))):
//   dx_t += dmean / T + dstd (x_t - mean) / (T std)  =  rs * x_t + rb
// No gradient passes through a clamped std.  gstat went through split-bf16 planes (2^-17 relative), so a std clamped to
// sqrt(eps) can read back a few ulps above it; the clamp test allows that rounding.  Otherwise a channel that is constant over an
// utterance (all frames ReLU-dead) gets rs ~ dstd / (T sqrt(eps)), and rs * x_t + rb cancels to fp32 noise of that size.
__global__ void asp_global_bwd_kernel(const float* __restrict__ gstat, const float* __restrict__ dgstat, int B, int C, int T, float eps,
                                      float* __restrict__ rs, float* __restrict__ rb) {
    const int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
    if (i >= int64_t(B) * C) return;
    const int b = int(i / C), c = int(i % C);
    const float mean = gstat[int64_t(b) * 2 * C + c], sd = gstat[int64_t(b) * 2 * C + C + c];
    const float dmean = dgstat[int64_t(b) * 2 * C + c], dstd = dgstat[int64_t(b) * 2 * C + C + c];
    const float s = (sd * sd > eps * (1.f + 0x1p-14f)) ? dstd / (float(T) * sd) : 0.f;
    rs[i] = s;
    rb[i] = dmean / float(T) - s * mean;
}

// ---------------------------------------------------------------------------------------------- TAP / TSP backward
// mean = (1/T) sum_t x_t, var = (1/(T-1)) sum_t (x_t - mean)^2 (pooling.py:8-47): dx_t = dmean / T + dvar * 2 (x_t - mean) / (T - 1)
// (the mean's own gradient through var sums to zero over t).  8 channels per thread, valid frames only; TAP reads no x.  HBM-bound:
// one pass over x and dx.
template <bool VAR>
__global__ void __launch_bounds__(256) pool_stats_bwd_kernel(Planes x, int C, int T, int P, int Tp, int64_t total, const float* __restrict__ pooled,
                                                             const float* __restrict__ dpooled, Planes dx) {
    const int groups = C >> 3, ld = VAR ? 2 * C : C;
    const float inv_t = 1.f / float(T), two_inv_t1 = 2.f / float(T > 1 ? T - 1 : 1);
    for (int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x; i < total; i += int64_t(gridDim.x) * blockDim.x) {
        const int c = int(i % groups) * 8;
        const int64_t bt = i / groups;
        const int b = int(bt / T), t = int(bt % T);
        const int64_t row = int64_t(b) * Tp + P + t;
        float dm[8], g[8];
        tr_ld8f(dpooled + int64_t(b) * ld + c, dm);
#pragma unroll
        for (int k = 0; k < 8; ++k) g[k] = dm[k] * inv_t;
        if (VAR) {
            float v[8], mu[8], dv[8];
            tr_load8(x, row, c, v);
            tr_ld8f(pooled + int64_t(b) * ld + c, mu);
            tr_ld8f(dpooled + int64_t(b) * ld + C + c, dv);
#pragma unroll
            for (int k = 0; k < 8; ++k) g[k] = fmaf(dv[k] * two_inv_t1, v[k] - mu[k], g[k]);
        }
        tr_store8(dx, row, c, g);
    }
}

// ---------------------------------------------------------------------------------------------- Adam
// paddle.optimizer.Adam with weight_decay = coupled L2 (g += wd * p), bias-corrected step (optimizer/__init__.py:12-18)
__global__ void adam_kernel(float* __restrict__ p, const float* __restrict__ g, float* __restrict__ m, float* __restrict__ v, int64_t n, float lr,
                            float beta1, float beta2, float eps, float wd, float bc1, float bc2, float grad_scale) {
    const int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const float gi = g[i] * grad_scale + wd * p[i];
    const float mi = beta1 * m[i] + (1.f - beta1) * gi;
    const float vi = beta2 * v[i] + (1.f - beta2) * gi * gi;
    m[i] = mi;
    v[i] = vi;
    p[i] -= lr * (mi / bc1) / (sqrtf(vi / bc2) + eps);
}

// ---------------------------------------------------------------------------------------------- AdamW / SGD / Momentum / RMSProp
// paddle.optimizer.<name>(**optimizer_args) (optimizer/__init__.py:12-18), Paddle 2.x update rules (include/ppv_b200.h: PPV_OPT_*).  One
// elementwise update per parameter; HBM-bound: (2 + 2 * states) floats moved per parameter.
struct OptimStep {
    float lr, wd, grad_scale, decay;  // decay = 1 - lr wd (AdamW)
    float beta1, beta2, eps, bc1, bc2;
    float mu, rho, rescale;
    int nesterov, centered;
};

template <int KIND>
__device__ __forceinline__ void optim_update(float& p, float g, float& s0, float& s1, float& s2, const OptimStep& a) {
    g *= a.grad_scale;
    if constexpr (KIND == PPV_OPT_SGD) {
        p -= a.lr * (g + a.wd * p);
    } else if constexpr (KIND == PPV_OPT_MOMENTUM) {
        const float gd = g * a.rescale + a.wd * p;
        s0 = a.mu * s0 + gd;
        p -= a.nesterov ? a.lr * (gd + a.mu * s0) : a.lr * s0;
    } else if constexpr (KIND == PPV_OPT_ADAMW) {
        p *= a.decay;
        s0 = a.beta1 * s0 + (1.f - a.beta1) * g;
        s1 = a.beta2 * s1 + (1.f - a.beta2) * g * g;
        p -= a.lr * (s0 / a.bc1) / (sqrtf(s1 / a.bc2) + a.eps);
    } else {  // PPV_OPT_RMSPROP: epsilon inside the square root, lr inside the momentum buffer
        const float gd = g + a.wd * p;
        s0 = a.rho * s0 + (1.f - a.rho) * gd * gd;
        float ms = s0;
        if (a.centered) {
            s2 = a.rho * s2 + (1.f - a.rho) * gd;
            ms -= s2 * s2;
        }
        s1 = a.mu * s1 + a.lr * gd / sqrtf(ms + a.eps);
        p -= s1;
    }
}

// State buffers the kind reads and writes: s0 for all but SGD, s1 for AdamW and RMSProp, s2 for centered RMSProp.
template <int KIND>
__device__ __forceinline__ bool optim_uses(int k, const OptimStep& a) {
    return KIND == PPV_OPT_SGD ? false : k == 0 ? true : k == 1 ? KIND != PPV_OPT_MOMENTUM : (KIND == PPV_OPT_RMSPROP && a.centered);
}

// VEC: every pointer is 16-byte aligned; the first n & ~3 elements go as float4, the tail element by element.  Grid-stride.
template <int KIND, bool VEC>
__global__ void __launch_bounds__(256) optim_kernel(float* __restrict__ p, const float* __restrict__ g, float* __restrict__ s0,
                                                    float* __restrict__ s1, float* __restrict__ s2, int64_t n, OptimStep a) {
    const int64_t stride = int64_t(gridDim.x) * blockDim.x, tid = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
    const bool u0 = optim_uses<KIND>(0, a), u1 = optim_uses<KIND>(1, a), u2 = optim_uses<KIND>(2, a);
    int64_t done = 0;
    if (VEC) {
        const int64_t n4 = n >> 2;
        const float4 zero = make_float4(0.f, 0.f, 0.f, 0.f);
        for (int64_t i = tid; i < n4; i += stride) {
            float4 pv = reinterpret_cast<const float4*>(p)[i];
            const float4 gv = reinterpret_cast<const float4*>(g)[i];
            float4 a0 = u0 ? reinterpret_cast<const float4*>(s0)[i] : zero;
            float4 a1 = u1 ? reinterpret_cast<const float4*>(s1)[i] : zero;
            float4 a2 = u2 ? reinterpret_cast<const float4*>(s2)[i] : zero;
            optim_update<KIND>(pv.x, gv.x, a0.x, a1.x, a2.x, a);
            optim_update<KIND>(pv.y, gv.y, a0.y, a1.y, a2.y, a);
            optim_update<KIND>(pv.z, gv.z, a0.z, a1.z, a2.z, a);
            optim_update<KIND>(pv.w, gv.w, a0.w, a1.w, a2.w, a);
            reinterpret_cast<float4*>(p)[i] = pv;
            if (u0) reinterpret_cast<float4*>(s0)[i] = a0;
            if (u1) reinterpret_cast<float4*>(s1)[i] = a1;
            if (u2) reinterpret_cast<float4*>(s2)[i] = a2;
        }
        done = n4 << 2;
    }
    for (int64_t i = done + tid; i < n; i += stride) {
        float pi = p[i], a0 = u0 ? s0[i] : 0.f, a1 = u1 ? s1[i] : 0.f, a2 = u2 ? s2[i] : 0.f;
        optim_update<KIND>(pi, g[i], a0, a1, a2, a);
        p[i] = pi;
        if (u0) s0[i] = a0;
        if (u1) s1[i] = a1;
        if (u2) s2[i] = a2;
    }
}

}  // namespace

// ================================================================================================ launchers
#define TR_LAUNCH_OK(what) PPV_LAUNCH_OK(what)

int tr_bn_forward(const Planes& a, int a_col0, int C, int B, int T, int P, int Tp, float eps, float momentum, const float* gamma, const float* beta,
                  float* mean, float* rstd, float* scale, float* shift, float* run_mean, float* run_var, float* part, const BnApplyArgs& apply_in,
                  int num_sms, cudaStream_t st) {
    PPV_REQUIRE(C % 64 == 0 && a_col0 % 8 == 0, "bn_forward: C % 64 == 0 required");
    bn_stats_kernel<<<dim3(C / 64, B), TR_WARPS * 32, 0, st>>>(a, a_col0, C, T, P, Tp, part);
    TR_LAUNCH_OK("bn_stats_kernel");
    bn_stats_finalize_kernel<<<(C + 7) / 8, 256, 0, st>>>(part, B, C, T, eps, momentum, gamma, beta, mean, rstd, scale, shift, run_mean, run_var);
    TR_LAUNCH_OK("bn_stats_finalize_kernel");
    BnApplyArgs p = apply_in;
    p.a = a;
    p.a_col0 = a_col0;
    p.C = C;
    p.B = B;
    p.T = T;
    p.P = P;
    p.Tp = Tp;
    p.scale = scale;
    p.shift = shift;
    const int64_t total = int64_t(B) * T * (C / 8);
    bn_apply_kernel<<<int(std::min<int64_t>((total + 255) / 256, int64_t(num_sms) * 16)), 256, 0, st>>>(p);
    TR_LAUNCH_OK("bn_apply_kernel");
    return PPV_OK;
}

int tr_bn_backward(const GradSrcList& gl, const Planes& a, int a_col0, int C, int B, int T, int P, int Tp, const float* mean, const float* rstd,
                   const float* gamma, float* dgamma, float* dbeta, const Planes& dz, int dz_col0, float* dbias, float* part, size_t part_elems,
                   cudaStream_t st, int tsplit) {
    PPV_REQUIRE(C % 64 == 0 && tsplit >= 1 && tsplit <= 8, "bn_backward: C % 64 == 0 and 1 <= tsplit <= 8 required");
    PPV_REQUIRE(size_t(2) * B * tsplit * C <= part_elems, "bn_backward: partial-sum scratch too small for B * tsplit * C");
    bn_bwd_reduce_kernel<<<dim3(C / 64, B, tsplit), TR_WARPS * 32, 0, st>>>(gl, a, a_col0, C, T, P, Tp, mean, rstd, part);
    TR_LAUNCH_OK("bn_bwd_reduce_kernel");
    part_finalize_kernel<<<(C + 7) / 8, 256, 0, st>>>(part, B * tsplit, C, 2, dbeta, dgamma);
    TR_LAUNCH_OK("part_finalize_kernel");
    bn_bwd_apply_kernel<<<dim3(C / 64, B, tsplit), TR_WARPS * 32, 0, st>>>(gl, a, a_col0, C, T, P, Tp, mean, rstd, gamma, dbeta, dgamma,
                                                                          1.f / (float(B) * float(T)), dz, dz_col0, part);
    TR_LAUNCH_OK("bn_bwd_apply_kernel");
    if (dbias) {
        part_finalize_kernel<<<(C + 7) / 8, 256, 0, st>>>(part, B * tsplit, C, 1, dbias, nullptr);
        TR_LAUNCH_OK("part_finalize_kernel");
    }
    return PPV_OK;
}

int tr_grad_sum(const GradSrcList& gl, int C, int B, int T, int P, int Tp, const Planes& out, int out_col0, float* part, float* colsum, cudaStream_t st) {
    PPV_REQUIRE(C % 64 == 0, "grad_sum: C % 64 == 0 required");
    grad_sum_kernel<<<dim3(C / 64, B), TR_WARPS * 32, 0, st>>>(gl, C, T, P, Tp, out, out_col0, part);
    TR_LAUNCH_OK("grad_sum_kernel");
    if (colsum) {
        part_finalize_kernel<<<(C + 7) / 8, 256, 0, st>>>(part, B, C, 1, colsum, nullptr);
        TR_LAUNCH_OK("part_finalize_kernel");
    }
    return PPV_OK;
}
int tr_grad_dot(const GradSrcList& gl, const Planes& y, int y_col0, int C, int B, int T, int P, int Tp, float* out_bc, cudaStream_t st) {
    PPV_REQUIRE(C % 64 == 0, "grad_dot: C % 64 == 0 required");
    grad_dot_kernel<<<dim3(C / 64, B), TR_WARPS * 32, 0, st>>>(gl, y, y_col0, C, T, P, Tp, out_bc);
    TR_LAUNCH_OK("grad_dot_kernel");
    return PPV_OK;
}
int tr_transpose(const Planes& in, int col0, int C, int64_t rows, const Planes& out, int shift, cudaStream_t st, int ntaps, int shift_step,
                 int64_t out_row_step) {
    PPV_REQUIRE(out.ld >= rows && out.rows >= C + (ntaps - 1) * out_row_step, "transpose: output too small");
    transpose_planes_kernel<<<dim3(unsigned((out.ld + 31) / 32), (C + 31) / 32, ntaps), 256, 0, st>>>(in, col0, C, rows, out, shift, shift_step,
                                                                                                      out_row_step);
    TR_LAUNCH_OK("transpose_planes_kernel");
    return PPV_OK;
}
int tr_repack_conv(const float* w, int64_t w_ld, int Cout, int Cin, int Cinp, int taps, const Planes& wf, const Planes& wd, cudaStream_t st) {
    const int64_t total = int64_t(Cout) * Cin * taps;
    repack_conv_kernel<<<int(std::min<int64_t>((total + 255) / 256, 4096)), 256, 0, st>>>(w, w_ld, Cout, Cin, Cinp, taps, wf, wd);
    TR_LAUNCH_OK("repack_conv_kernel");
    return PPV_OK;
}
int tr_wgrad_unpack(const float* part, int splits, int64_t split_rows, int Cout, int Cin, int Cinp, int taps, float* grad, int64_t g_ld,
                    cudaStream_t st) {
    const int64_t total = int64_t(Cout) * Cin * taps;
    wgrad_unpack_kernel<<<int(std::min<int64_t>((total + 255) / 256, 4096)), 256, 0, st>>>(part, splits, split_rows, Cout, Cin, Cinp, taps, grad, g_ld);
    TR_LAUNCH_OK("wgrad_unpack_kernel");
    return PPV_OK;
}
int tr_dense_fwd(const float* X, int64_t x_ld, const float* W, int64_t w_ld, const float* bias, int M, int N, int K, int act, float* Y, int64_t y_ld,
                 cudaStream_t st) {
    const int64_t outs = int64_t(M) * N;
    dense_fwd_kernel<<<unsigned((outs + 7) / 8), 256, 0, st>>>(X, x_ld, W, w_ld, bias, M, N, K, act, Y, y_ld);
    TR_LAUNCH_OK("dense_fwd_kernel");
    return PPV_OK;
}
int tr_dense_bwd(const float* dY, int64_t dy_ld, const float* X, int64_t x_ld, const float* W, int64_t w_ld, int M, int N, int K, float* dX,
                 int64_t dx_ld, float* dW, int64_t dw_ld, float* db, cudaStream_t st) {
    if (dX) {
        dense_bwd_x_kernel<<<unsigned((int64_t(M) * K + 255) / 256), 256, 0, st>>>(dY, dy_ld, W, w_ld, M, N, K, dX, dx_ld);
        TR_LAUNCH_OK("dense_bwd_x_kernel");
    }
    if (dW) {
        dense_bwd_w_kernel<<<unsigned((int64_t(N) * K + 255) / 256), 256, 0, st>>>(dY, dy_ld, X, x_ld, M, N, K, dW, dw_ld, db);
        TR_LAUNCH_OK("dense_bwd_w_kernel");
    }
    return PPV_OK;
}
int tr_act_bwd(float* dy, const float* y, int64_t n, int act, float alpha, cudaStream_t st) {
    act_bwd_kernel<<<unsigned((n + 255) / 256), 256, 0, st>>>(dy, y, n, act, alpha);
    TR_LAUNCH_OK("act_bwd_kernel");
    return PPV_OK;
}
int tr_bn1d_fwd(const float* x, int B, int C, float eps, float momentum, const float* gamma, const float* beta, float* y, float* mean, float* rstd,
                float* run_mean, float* run_var, cudaStream_t st) {
    bn1d_fwd_kernel<<<(C + 127) / 128, 128, 0, st>>>(x, B, C, eps, momentum, gamma, beta, y, mean, rstd, run_mean, run_var);
    TR_LAUNCH_OK("bn1d_fwd_kernel");
    return PPV_OK;
}
int tr_bn1d_bwd(const float* dy, const float* x, int B, int C, const float* gamma, const float* mean, const float* rstd, float* dx, float* dgamma,
                float* dbeta, cudaStream_t st) {
    bn1d_bwd_kernel<<<(C + 127) / 128, 128, 0, st>>>(dy, x, B, C, gamma, mean, rstd, dx, dgamma, dbeta);
    TR_LAUNCH_OK("bn1d_bwd_kernel");
    return PPV_OK;
}
int tr_asp_bwd(const float* logits, int64_t lg_ld, const Planes& x, int C, int B, int T, int P, int Tp, float eps, const float* pooled,
               const float* dpooled, const Planes& dlogits, const Planes& dx, cudaStream_t st) {
    PPV_REQUIRE(C % 32 == 0, "asp_bwd: C % 32 == 0 required");
    asp_bwd_kernel<<<dim3(C / 32, B), 256, 0, st>>>(logits, lg_ld, x, C, T, P, Tp, eps, pooled, dpooled, dlogits, dx);
    TR_LAUNCH_OK("asp_bwd_kernel");
    return PPV_OK;
}
int tr_asp_global_bwd(const float* gstat, const float* dgstat, int B, int C, int T, float eps, float* rs, float* rb, cudaStream_t st) {
    asp_global_bwd_kernel<<<unsigned((int64_t(B) * C + 255) / 256), 256, 0, st>>>(gstat, dgstat, B, C, T, eps, rs, rb);
    TR_LAUNCH_OK("asp_global_bwd_kernel");
    return PPV_OK;
}
int tr_pool_stats_bwd(const Planes& x, int C, int B, int T, int P, int Tp, const float* pooled, const float* dpooled, bool var, const Planes& dx,
                      cudaStream_t st) {
    PPV_REQUIRE(C % 8 == 0 && B > 0 && T > 0 && Tp >= T + 2 * P, "pool_stats_bwd: C % 8 == 0 and Tp >= T + 2P required");
    const int64_t total = int64_t(B) * T * (C / 8);
    const int grid = int(std::min<int64_t>((total + 255) / 256, int64_t(device_sm_count()) * 16));
    if (var)
        pool_stats_bwd_kernel<true><<<grid, 256, 0, st>>>(x, C, T, P, Tp, total, pooled, dpooled, dx);
    else
        pool_stats_bwd_kernel<false><<<grid, 256, 0, st>>>(x, C, T, P, Tp, total, pooled, dpooled, dx);
    TR_LAUNCH_OK("pool_stats_bwd_kernel");
    return PPV_OK;
}
int adam_step(float* params, const float* grads, float* m, float* v, int64_t n, float lr, float beta1, float beta2, float eps, float weight_decay,
              int64_t step, float grad_scale, cudaStream_t st) {
    PPV_REQUIRE(params && grads && m && v && n > 0 && step >= 1, "adam_step: bad argument");
    const float bc1 = float(1.0 - pow(double(beta1), double(step))), bc2 = float(1.0 - pow(double(beta2), double(step)));
    adam_kernel<<<unsigned((n + 255) / 256), 256, 0, st>>>(params, grads, m, v, n, lr, beta1, beta2, eps, weight_decay, bc1, bc2, grad_scale);
    TR_LAUNCH_OK("adam_kernel");
    return PPV_OK;
}

int optimizer_state_count(int kind, int centered) {
    switch (kind) {
        case PPV_OPT_ADAM:
        case PPV_OPT_ADAMW: return 2;
        case PPV_OPT_SGD: return 0;
        case PPV_OPT_MOMENTUM: return 1;
        case PPV_OPT_RMSPROP: return centered ? 3 : 2;
        default: return PPV_EINVAL;
    }
}

namespace {
template <int KIND>
int launch_optim(float* p, const float* g, float* s0, float* s1, float* s2, int64_t n, const OptimStep& a, cudaStream_t st) {
    const bool vec = ((reinterpret_cast<uintptr_t>(p) | reinterpret_cast<uintptr_t>(g) | reinterpret_cast<uintptr_t>(s0) |
                       reinterpret_cast<uintptr_t>(s1) | reinterpret_cast<uintptr_t>(s2)) & 15) == 0;
    const int64_t items = vec ? std::max<int64_t>(n >> 2, 1) : n;
    const int grid = int(std::min<int64_t>((items + 255) / 256, int64_t(device_sm_count()) * 8));
    if (vec)
        optim_kernel<KIND, true><<<grid, 256, 0, st>>>(p, g, s0, s1, s2, n, a);
    else
        optim_kernel<KIND, false><<<grid, 256, 0, st>>>(p, g, s0, s1, s2, n, a);
    TR_LAUNCH_OK("optim_kernel");
    return PPV_OK;
}
}  // namespace

int optimizer_step(int kind, float* params, const float* grads, float* s0, float* s1, float* s2, int64_t n, const ppv_optim_args& args,
                   int64_t step, float grad_scale, cudaStream_t st) {
    const int ns = optimizer_state_count(kind, args.centered);
    PPV_REQUIRE(ns >= 0, "optimizer_step: kind must be one of PPV_OPT_ADAM / _ADAMW / _SGD / _MOMENTUM / _RMSPROP");
    PPV_REQUIRE(params && grads && n > 0 && step >= 1, "optimizer_step: bad argument");
    PPV_REQUIRE((ns < 1 || s0) && (ns < 2 || s1) && (ns < 3 || s2), "optimizer_step: a state buffer the optimizer needs is NULL");
    if (kind == PPV_OPT_ADAM)
        return adam_step(params, grads, s0, s1, n, args.lr, args.beta1, args.beta2, args.epsilon, args.weight_decay, step, grad_scale, st);
    OptimStep a{};
    a.lr = args.lr;
    a.wd = args.weight_decay;
    a.grad_scale = grad_scale;
    a.decay = float(1.0 - double(args.lr) * double(args.weight_decay));
    a.beta1 = args.beta1;
    a.beta2 = args.beta2;
    a.eps = args.epsilon;
    a.bc1 = float(1.0 - pow(double(args.beta1), double(step)));
    a.bc2 = float(1.0 - pow(double(args.beta2), double(step)));
    a.mu = args.momentum;
    a.rho = args.rho;
    a.rescale = args.rescale_grad;
    a.nesterov = args.use_nesterov != 0;
    a.centered = args.centered != 0;
    // the buffers the kind does not read take part in the alignment test as NULL
    if (ns < 1) s0 = nullptr;
    if (ns < 2) s1 = nullptr;
    if (ns < 3) s2 = nullptr;
    switch (kind) {
        case PPV_OPT_ADAMW: return launch_optim<PPV_OPT_ADAMW>(params, grads, s0, s1, s2, n, a, st);
        case PPV_OPT_SGD: return launch_optim<PPV_OPT_SGD>(params, grads, s0, s1, s2, n, a, st);
        case PPV_OPT_MOMENTUM: return launch_optim<PPV_OPT_MOMENTUM>(params, grads, s0, s1, s2, n, a, st);
        default: return launch_optim<PPV_OPT_RMSPROP>(params, grads, s0, s1, s2, n, a, st);
    }
}

}  // namespace ppv
