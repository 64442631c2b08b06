// Skinny linear layers: out[b, n] = act(sum_k x[b, k] W[n, k] + bias[n]) for a handful of rows (one per utterance), K <= 1024.
// In ECAPA-TDNN that is the SE excitation MLP (ppvector/models/ecapa_tdnn.py:79-80): se1 [B x 512] x [512 x 128] with ReLU into
// planes, se2 [B x 128] x [128 x 512] with sigmoid into fp32.  ASP's global-context fold (K = 3072) and the final fc (K = 1536 or
// 3072) run on the gather-GEMM: plan_row_linear chooses by skinny_linear_supported.
//
// On the tensor-core gather-GEMM these layers would occupy 2-6 CTAs: with M = 256 rows there are only two 128-row tiles, and the
// k-loop is a latency chain.  Here every SM takes a 16 x 16 output tile and walks K on the CUDA cores with fp32 FMAs over
// the exact hi + lo values of the split-bf16 operands (at least as accurate as the three-product tensor path).  128-192 CTAs, no
// split-K, no atomics: deterministic.
#include "common.h"
#include "ptx.cuh"

namespace ppv {

namespace {

constexpr int SK_R = 16, SK_C = 16;   // output tile: rows x columns
constexpr int SK_KC = 512;            // K chunk staged in shared memory
constexpr int SK_LD = SK_KC + 4;      // padded row stride (floats): 16 rows land in different banks for 16-byte loads
constexpr int SK_ITERS = (SK_R + SK_C) * (SK_KC / 8) / 256;  // 16-byte operand segments per thread per chunk (8)
constexpr int SK_SMEM = (SK_R + SK_C) * SK_LD * 4;

// The K loop is a latency chain (global load -> shared -> FMA): the next chunk's operand segments are already in flight in registers
// while the current chunk is multiplied.
__global__ void __launch_bounds__(256) skinny_linear_kernel(Planes x, int x_col0, Planes W, int M, int N, int K, Epilogue ep) {
    extern __shared__ __align__(16) float sk_smem[];
    float(*sx)[SK_LD] = reinterpret_cast<float(*)[SK_LD]>(sk_smem);
    float(*sw)[SK_LD] = reinterpret_cast<float(*)[SK_LD]>(sk_smem + SK_R * SK_LD);
    griddep_launch_dependents();
    griddep_wait();
    const int r0 = blockIdx.y * SK_R, c0 = blockIdx.x * SK_C;
    const int tid = threadIdx.x;
    const int lr = tid & 15, lc = tid >> 4;  // this thread's output (row r0 + lr, column c0 + lc)
    uint4 rh[SK_ITERS], rl[SK_ITERS];
    auto fetch = [&](int k0) {  // operand segments of chunk k0 -> registers (hi and lo planes, 8 elements each)
        const int kc = min(SK_KC, K - k0);
#pragma unroll
        for (int it = 0; it < SK_ITERS; ++it) {
            const int i = tid + it * 256;
            const int row = i / (SK_KC / 8), seg = i - row * (SK_KC / 8);
            const bool is_x = row < SK_R;
            const int gr = is_x ? r0 + row : c0 + (row - SK_R);
            rh[it] = rl[it] = make_uint4(0u, 0u, 0u, 0u);
            if (seg * 8 < kc && gr < (is_x ? M : N)) {
                const Planes& p = is_x ? x : W;
                const int64_t off = int64_t(gr) * p.ld + (is_x ? x_col0 : 0) + k0 + seg * 8;
                rh[it] = *reinterpret_cast<const uint4*>(p.hi() + off);
                rl[it] = *reinterpret_cast<const uint4*>(p.lo() + off);
            }
        }
    };
    auto stash = [&]() {  // registers -> shared memory as fp32 (hi + lo)
#pragma unroll
        for (int it = 0; it < SK_ITERS; ++it) {
            const int i = tid + it * 256;
            const int row = i / (SK_KC / 8), seg = i - row * (SK_KC / 8);
            const uint32_t hw[4] = {rh[it].x, rh[it].y, rh[it].z, rh[it].w}, lw[4] = {rl[it].x, rl[it].y, rl[it].z, rl[it].w};
            float v[8];
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                const float2 a = unpack_bf16x2(hw[j]), b = unpack_bf16x2(lw[j]);
                v[2 * j] = a.x + b.x;
                v[2 * j + 1] = a.y + b.y;
            }
            float* dst = row < SK_R ? &sx[row][seg * 8] : &sw[row - SK_R][seg * 8];
            *reinterpret_cast<float4*>(dst) = make_float4(v[0], v[1], v[2], v[3]);
            *reinterpret_cast<float4*>(dst + 4) = make_float4(v[4], v[5], v[6], v[7]);
        }
    };
    float acc0 = 0.f, acc1 = 0.f, acc2 = 0.f, acc3 = 0.f;
    fetch(0);
    for (int k0 = 0; k0 < K; k0 += SK_KC) {
        const int kc = min(SK_KC, K - k0);  // multiple of 8
        stash();
        __syncthreads();
        if (k0 + SK_KC < K) fetch(k0 + SK_KC);
        const float* px = sx[lr];
        const float* pw = sw[lc];
#pragma unroll 4
        for (int k = 0; k < kc; k += 4) {
            const float4 a = *reinterpret_cast<const float4*>(px + k);
            const float4 b = *reinterpret_cast<const float4*>(pw + k);
            acc0 = fmaf(a.x, b.x, acc0);
            acc1 = fmaf(a.y, b.y, acc1);
            acc2 = fmaf(a.z, b.z, acc2);
            acc3 = fmaf(a.w, b.w, acc3);
        }
        __syncthreads();
    }
    const int r = r0 + lr, c = c0 + lc;
    if (r >= M || c >= N) return;
    float y = (acc0 + acc1) + (acc2 + acc3);
    if (ep.bias) y += ep.bias[c];
    if (ep.relu) y = fmaxf(y, 0.f);
    if (ep.sigmoid_) y = 1.f / (1.f + expf(-y));
    if (ep.out_mode == OUT_F32) {
        static_cast<float*>(ep.out)[int64_t(r) * ep.out_ld + ep.out_col0 + c] = y;
    } else {
        __nv_bfloat16 h, l;
        split_bf16(y, h, l);
        __nv_bfloat16* o = static_cast<__nv_bfloat16*>(ep.out) + int64_t(r) * ep.out_ld + ep.out_col0 + c;
        o[0] = h;
        o[ep.out_plane_stride] = l;
    }
}

}  // namespace

// K <= 1024: with 16 x 16 output tiles every CTA re-reads 32 operand rows, so the L2 -> SM traffic is M N K / 2 bytes.
bool skinny_linear_supported(int M, int N, int K, const Epilogue& ep) {
    return M <= 4096 && K % 8 == 0 && K <= 1024 && !ep.rowgrp_bias && !ep.seg_scale && !ep.bn_scale && !ep.tanh_ && !ep.silu_ && ep.Tp == 0 && ep.img_Wp == 0 &&
           ep.relu_max == 0.f;
}

// x: planes [M rows][>= x_col0 + K], W: planes [>= N rows][K] (K-major, as the gather-GEMM keeps it); epilogue: bias, ReLU or sigmoid,
// planes or fp32 output.
int skinny_linear_launch(const Planes& x, int x_col0, const Planes& W, int M, int N, int K, const Epilogue& ep, cudaStream_t st) {
    PPV_REQUIRE(skinny_linear_supported(M, N, K, ep), "skinny_linear: unsupported shape / epilogue");
    PPV_REQUIRE(x.ld % 8 == 0 && x_col0 % 8 == 0 && W.ld == K, "skinny_linear: operand layout");
    dim3 grid((N + SK_C - 1) / SK_C, (M + SK_R - 1) / SK_R);
    PPV_ONCE_PER_DEVICE(PPV_CUDA_OK(cudaFuncSetAttribute(skinny_linear_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, SK_SMEM)));
    PPV_PDL_OK(launch_pdl(skinny_linear_kernel, grid, dim3(256), size_t(SK_SMEM), st, x, x_col0, W, M, N, K, ep), "skinny_linear_kernel");
    return PPV_OK;
}

}  // namespace ppv
