// 1x1 convolutions with K = 32 input channels (one 32-channel source) and N <= 64 output channels over image grids or plain row ranges:
// ERes2Net's layer-1 conv1 / shortcut (ppvector/models/eres2net.py:85-108) and CAM++'s FCM shortcuts (ppvector/models/campplus.py:232-238).
// ResNetSE plans no pointwise step: its 1x1 convs run on the gather-GEMM.
//
// On the tensor-core gather-GEMM these layers run one 128-row tile per pipeline step with a single 32-wide k-step: 49 200 tiles of 16 KB at
// the 80 x 298 resolution, paced by the per-tile epilogue chain rather than by HBM.  Here one thread owns one grid position, keeps its
// 32 input values (exact hi + lo) in registers and walks the fp32 weight matrix in shared memory with broadcast 16-byte loads: 2 K N FLOP
// per position on the FMA pipe.  At K = 64 every 4 FMAs cost one broadcast LDS.128 (4 LSU cycles per warp), so the kernel would be
// shared-memory bound at 4x its FMA time: only K = 32 is routed here.
#include <type_traits>

#include "common.h"
#include "ptx.cuh"

namespace ppv {

namespace {

constexpr int PW_NCH = 32;  // output channels per accumulator pass

struct PwParams {
    Planes src[2];
    int col0[2], ncols[2], nsrc;
    Planes W;  // [>= N][K] split planes, K-major (the gather-GEMM's weight layout)
    int N, K;
    int64_t M;
    Epilogue ep;
};

template <int K>
__global__ void __launch_bounds__(256, 2) pw_conv_kernel(const PwParams p) {
    extern __shared__ __align__(16) float pw_w[];  // [K][N] fp32
    const int N = p.N;
    for (int i = threadIdx.x; i < N * K; i += blockDim.x) {
        const int n = i / K, k = i - n * K;
        const int64_t off = int64_t(n) * p.W.ld + k;
        pw_w[k * N + n] = __bfloat162float(p.W.hi()[off]) + __bfloat162float(p.W.lo()[off]);
    }
    griddep_launch_dependents();
    griddep_wait();
    __syncthreads();
    const Epilogue& ep = p.ep;
    for (int64_t row = int64_t(blockIdx.x) * blockDim.x + threadIdx.x; row < p.M; row += int64_t(gridDim.x) * blockDim.x) {
        // ---- which output row (image mode: interior positions on the stride grid only; the zero border is never written) ----
        int64_t out_row = row;
        if (ep.img_Wp > 0) {
            const int64_t img = int64_t(ep.img_Hp) * ep.img_Wp;
            const int64_t grp = row / img;
            const int rem = int(row - grp * img);
            const int h = rem / ep.img_Wp - 1, w = rem % ep.img_Wp - 1;
            const int sw = ep.img_stride_w ? ep.img_stride_w : ep.img_stride;
            if (h < 0 || h >= ep.img_H || w < 0 || w >= ep.img_W || (h % ep.img_stride) != 0 || (w % sw) != 0) continue;
            out_row = (grp * ep.out_Hp + h / ep.img_stride + 1) * ep.out_Wp + w / sw + 1;
        }
        // ---- the K input values of this position: exact hi + lo ----
        float x[K];
        auto load = [&](const Planes& t, int col0, auto cnt, float* dst) {  // cnt: compile-time channel count (register indices stay static)
            constexpr int CNT = decltype(cnt)::value;
            const __nv_bfloat16* ph = t.hi() + row * t.ld + col0;
            const __nv_bfloat16* pl = t.lo() + row * t.ld + col0;
#pragma unroll
            for (int c = 0; c < CNT; c += 8) {
                const uint4 h4 = *reinterpret_cast<const uint4*>(ph + c);
                const uint4 l4 = *reinterpret_cast<const uint4*>(pl + c);
                const uint32_t hw[4] = {h4.x, h4.y, h4.z, h4.w}, lw[4] = {l4.x, l4.y, l4.z, l4.w};
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                    const float2 a = unpack_bf16x2(hw[j]), b = unpack_bf16x2(lw[j]);
                    dst[c + 2 * j] = a.x + b.x;
                    dst[c + 2 * j + 1] = a.y + b.y;
                }
            }
        };
        load(p.src[0], p.col0[0], std::integral_constant<int, K>{}, x);
        // ---- PW_NCH output channels at a time ----
        for (int n0 = 0; n0 < N; n0 += PW_NCH) {
            float acc[PW_NCH];
#pragma unroll
            for (int j = 0; j < PW_NCH; j += 4) {
                const float4 b4 = ep.bias ? __ldg(reinterpret_cast<const float4*>(ep.bias + n0 + j)) : make_float4(0.f, 0.f, 0.f, 0.f);
                acc[j] = b4.x;
                acc[j + 1] = b4.y;
                acc[j + 2] = b4.z;
                acc[j + 3] = b4.w;
            }
#pragma unroll
            for (int k = 0; k < K; ++k) {
                const float xv = x[k];
                const float4* wr = reinterpret_cast<const float4*>(pw_w + k * N + n0);
#pragma unroll
                for (int j = 0; j < PW_NCH / 4; ++j) {
                    const float4 w4 = wr[j];  // every lane reads the same address: one broadcast wavefront
                    acc[4 * j] = fmaf(xv, w4.x, acc[4 * j]);
                    acc[4 * j + 1] = fmaf(xv, w4.y, acc[4 * j + 1]);
                    acc[4 * j + 2] = fmaf(xv, w4.z, acc[4 * j + 2]);
                    acc[4 * j + 3] = fmaf(xv, w4.w, acc[4 * j + 3]);
                }
            }
            if (ep.relu) {
#pragma unroll
                for (int j = 0; j < PW_NCH; ++j) {
                    acc[j] = fmaxf(acc[j], 0.f);
                    if (ep.relu_max > 0.f) acc[j] = fminf(acc[j], ep.relu_max);
                }
            }
            uint32_t h[PW_NCH / 2], l[PW_NCH / 2];
#pragma unroll
            for (int j = 0; j < PW_NCH / 2; ++j) split_pack_bf16x2(acc[2 * j], acc[2 * j + 1], h[j], l[j]);
            __nv_bfloat16* oh = static_cast<__nv_bfloat16*>(ep.out) + out_row * ep.out_ld + ep.out_col0 + n0;
            __nv_bfloat16* ol = oh + ep.out_plane_stride;
#pragma unroll
            for (int j = 0; j < PW_NCH / 8; ++j) {  // 16-byte stores, 64 B per plane
                *reinterpret_cast<uint4*>(oh + 8 * j) = make_uint4(h[4 * j], h[4 * j + 1], h[4 * j + 2], h[4 * j + 3]);
                *reinterpret_cast<uint4*>(ol + 8 * j) = make_uint4(l[4 * j], l[4 * j + 1], l[4 * j + 2], l[4 * j + 3]);
            }
        }
    }
}

}  // namespace

// A 1x1 conv qualifies when its single source is a 32-column window at row offset 0, N is 32 or 64, the output goes to split planes (plain
// rows or an image grid, any stride) and the epilogue is bias (+ ReLU / clipped ReLU).
static bool pointwise_supported(const GemmSource* srcs, int nsrc, int N, const Epilogue& ep) {
    if (nsrc != 1 || N % 32 != 0 || N > 64) return false;
    if (srcs[0].row_off != 0 || srcs[0].ncols != 32 || srcs[0].col0 % 8 != 0 || srcs[0].t.ld % 8 != 0) return false;
    if (ep.out_mode != OUT_PLANES || ep.rowgrp_bias || ep.seg_scale || ep.bn_scale || ep.tanh_ || ep.sigmoid_ || ep.silu_ || ep.Tp != 0 || ep.halo) return false;
    return (ep.out_ld % 16) == 0 && (ep.out_col0 % 16) == 0 && (ep.out_plane_stride % 16) == 0;
}

int pointwise_launch(const GemmSource* srcs, int nsrc, const Planes& W, int64_t M, int N, const Epilogue& ep, int num_sms, cudaStream_t st) {
    PPV_REQUIRE(pointwise_supported(srcs, nsrc, N, ep), "pointwise: unsupported shape / epilogue");
    PwParams p;
    p.nsrc = nsrc;
    p.K = 0;
    for (int i = 0; i < 2; ++i) {
        p.src[i] = srcs[i < nsrc ? i : 0].t;
        p.col0[i] = srcs[i < nsrc ? i : 0].col0;
        p.ncols[i] = i < nsrc ? srcs[i].ncols : 0;
        if (i < nsrc) p.K += srcs[i].ncols;
    }
    PPV_REQUIRE(W.ld == p.K && W.rows >= N, "pointwise: weight layout");
    p.W = W;
    p.N = N;
    p.M = M;
    p.ep = ep;
    const size_t smem = size_t(p.K) * N * sizeof(float);
    const int grid = int(std::min<int64_t>((M + 255) / 256, int64_t(num_sms) * 8));
    PPV_PDL_OK(launch_pdl(pw_conv_kernel<32>, dim3(grid), dim3(256), smem, st, p), "pw_conv_kernel<32>");
    return PPV_OK;
}

bool pointwise_step_build(PwStep* s, const GemmSource* srcs, int nsrc, const Planes& W, int N, int64_t M, const Epilogue& ep) {
    const char* e = getenv("PPV_POINTWISE");
    if ((e && e[0] == '0') || ep.img_Wp == 0 || !pointwise_supported(srcs, nsrc, N, ep)) return false;
    for (int i = 0; i < nsrc; ++i) s->srcs[i] = srcs[i];
    s->nsrc = nsrc;
    s->N = N;
    s->M = M;
    s->W = W;
    s->ep = ep;
    return true;
}

}  // namespace ppv
