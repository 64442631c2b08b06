// 3x3 conv (padding 1) with 32 input and 32 output channels over zero-bordered NHWC image grids: the stride-1 stages of
// ResNetSE (ppvector/models/resnet_se.py:24-45, conv2 of layer1), CAM++'s FCM head (ppvector/models/campplus.py:211-281) and
// ERes2Net's 32-wide Res2Net convs (ppvector/models/eres2net.py:85-108).  Same contraction as the gather-GEMM of gemm_wgmma.cu
// (M = grid positions, N = 32, K = 9 taps x 32), restructured around what bounds it.  The generic kernel loads every
// activation row nine times from L2 (one TMA tile per tap) for an N = 32 tile: it is L2 -> shared-memory bound.  Here
//   * the whole weight matrix (9 taps x hi/lo x 2 KB = 36 KB) is loaded once per CTA and stays in shared memory;
//   * ONE image patch of 8 x 64 grid positions (6 x 62 outputs + a one-position halo) is loaded per work item by a single 5-D
//     TMA box per plane ({32 ch, 64 w, 8 h}: out-of-range coordinates are zero-filled, and the zero border of the grid is the
//     conv's padding), landing as 512 consecutive 64-byte rows in the SWIZZLE_64B layout;
//   * the nine taps are the SAME shared-memory patch read at row offsets dh * 64 + dw: the wgmma descriptor start address
//     moves by whole 64-byte rows (the swizzle XOR is a function of the absolute shared-memory address, as in res2conv.cu);
//   * three M = 128 accumulator tiles cover the 384 patch rows that hold outputs; the two MMA warpgroups take them in turn
//     (two m64 x n32 accumulators each), and the epilogue maps a patch row back to its grid position (halo columns are
//     computed and dropped).
// L2 -> SM traffic per output position: 512 / 372 = 1.4 rows instead of 9.
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <mutex>

#include "common.h"
#include "gemm_epilogue.cuh"
#include "ptx.cuh"

namespace ppv {

constexpr int C3_PW = 64, C3_PH = 8;                     // patch: grid positions loaded per work item
constexpr int C3_OW = C3_PW - 2, C3_OH = C3_PH - 2;      // outputs per patch: 62 x 6
constexpr int C3_ROWS = C3_PW * C3_PH;                   // 512 shared-memory rows of 64 B
constexpr int C3_TILES = (C3_OH * C3_PW) / GEMM_BM;      // 3 accumulator tiles of 128 patch rows
constexpr int C3_ROW0 = C3_PW + 1;                       // first patch row that holds an output (ph = 1, pw = 1)
constexpr int C3_PLANE_BYTES = C3_ROWS * 64;             // 32 KB per plane
constexpr int C3_W_TILE = 32 * 64;                       // [32 out ch x 32 k] bf16 per tap per plane
constexpr int C3_STAGES = 2;
constexpr int C3_BN = 32;
static_assert((C3_OH * C3_PW) % GEMM_BM == 0, "patch rows with outputs must be whole accumulator tiles");

template <int NSPLIT>
struct C3Cfg {
    static constexpr int NP = (NSPLIT == 3) ? 2 : 1;
    static constexpr int W_BYTES = 9 * NP * C3_W_TILE;
    static constexpr int STAGE_BYTES = NP * C3_PLANE_BYTES;
    // + 1 KB behind the last stage: the last accumulator tile's +1-row taps read two rows past the patch (dropped outputs)
    static constexpr int SMEM_BYTES = 1024 + ((W_BYTES + 1023) & ~1023) + C3_STAGES * STAGE_BYTES + 1024 + 256;
};

__device__ __forceinline__ void tma_load_5d(uint32_t smem_dst, const CUtensorMap* m, uint32_t bar, int c0, int c1, int c2, int c3, int c4) {
    asm volatile(
        "cp.async.bulk.tensor.5d.shared::cluster.global.mbarrier::complete_tx::bytes"
        " [%0], [%1, {%3, %4, %5, %6, %7}], [%2];"
        :
        : "r"(smem_dst), "l"(reinterpret_cast<uint64_t>(m)), "r"(bar), "r"(c0), "r"(c1), "r"(c2), "r"(c3), "r"(c4)
        : "memory");
}

template <int NSPLIT>
__global__ void __launch_bounds__(GEMM_THREADS, 1) conv3x3_c32_kernel(const __grid_constant__ Conv3x3Params cp) {
    using Cfg = C3Cfg<NSPLIT>;
    constexpr int NP = Cfg::NP;
    extern __shared__ uint8_t smem_raw[];
    const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;
    const uint32_t w_base = smem_base;
    const uint32_t a_base = smem_base + ((Cfg::W_BYTES + 1023) & ~1023);
    const uint32_t bar_base = a_base + C3_STAGES * Cfg::STAGE_BYTES + 1024;
    auto full_bar = [&](int s) { return bar_base + 8u * s; };
    auto empty_bar = [&](int s) { return bar_base + 8u * (C3_STAGES + s); };
    const uint32_t w_full = bar_base + 8u * (2 * C3_STAGES);

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    if (warp == 0 && lane == 0) {
        prefetch_tmap(&cp.mapX);
        prefetch_tmap(&cp.mapW);
    }
    if (warp == 1 && lane == 0) {
        for (int s = 0; s < C3_STAGES; ++s) {
            mbar_init(full_bar(s), 1);
            mbar_init(empty_bar(s), GEMM_MMA_THREADS / 128);  // one arrival per MMA warpgroup
        }
        mbar_init(w_full, 1);
        fence_mbar_init();
    }
    __syncthreads();
    griddep_launch_dependents();  // PDL

    const int per_img = cp.nph * cp.npw;
    if (warp == 0) {
        // ===================== TMA producer =====================
        if (lane == 0) {  // weights: once per CTA
            mbar_arrive_expect_tx(w_full, 9 * NP * C3_W_TILE);
            for (int tap = 0; tap < 9; ++tap)
                for (int pl = 0; pl < NP; ++pl) tma_load_3d(w_base + (tap * NP + pl) * C3_W_TILE, &cp.mapW, w_full, tap * 32, 0, pl);
        }
        __syncwarp();
        griddep_wait();  // the weights above are constants; the activations below come from the previous kernel
        int stage = 0;
        uint32_t phase = 0;
        for (int item = blockIdx.x; item < cp.patches; item += gridDim.x) {
            const int b = item / per_img, r = item - b * per_img;
            const int ih = r / cp.npw, iw = r - ih * cp.npw;
            mbar_wait(empty_bar(stage), phase ^ 1u);
            if (lane == 0) {
                mbar_arrive_expect_tx(full_bar(stage), NP * C3_PLANE_BYTES);
                for (int pl = 0; pl < NP; ++pl)
                    tma_load_5d(a_base + stage * Cfg::STAGE_BYTES + pl * C3_PLANE_BYTES, &cp.mapX, full_bar(stage), cp.x_col0, iw * C3_OW,
                                ih * C3_OH, b, pl);
            }
            __syncwarp();
            if (++stage == C3_STAGES) {
                stage = 0;
                phase ^= 1u;
            }
        }
    } else if (warp >= 4) {
        // ===================== MMA + epilogue: warpgroup g takes every other 128-row accumulator tile =====================
        const int g = (warp - 4) >> 2, t = threadIdx.x & 127;
        griddep_wait();  // the epilogue writes buffers that upstream kernels may still be reading
        mbar_wait(w_full, 0);
        int stage = 0;
        uint32_t phase = 0;
        int tcount = 0;  // running accumulator-tile counter of this CTA: tile n goes to warpgroup n & 1
        float acc0[C3_BN / 2], acc1[C3_BN / 2];
#pragma unroll
        for (int i = 0; i < C3_BN / 2; ++i) acc0[i] = acc1[i] = 0.f;
        for (int item = blockIdx.x; item < cp.patches; item += gridDim.x) {
            const int b = item / per_img, r = item - b * per_img;
            const int ih = r / cp.npw, iw = r - ih * cp.npw;
            mbar_wait(full_bar(stage), phase);
            const uint32_t slot = a_base + stage * Cfg::STAGE_BYTES;
            for (int tt = 0; tt < C3_TILES; ++tt, ++tcount) {
                if ((tcount & 1) != g) continue;
                wgmma_fence_acc(acc0);
                wgmma_fence_acc(acc1);
                wgmma_fence();
                auto issue = [&](float (&acc)[C3_BN / 2], int mb) {
#pragma unroll
                    for (int tap = 0; tap < 9; ++tap) {
                        const int roff = C3_ROW0 + tt * GEMM_BM + mb * 64 + (tap / 3 - 1) * C3_PW + (tap % 3 - 1);
                        const uint64_t a_hi = make_sw64_kmajor_desc(slot + uint32_t(roff) * 64u);
                        const uint64_t b_hi = make_sw64_kmajor_desc(w_base + (tap * NP) * C3_W_TILE);
#pragma unroll
                        for (int k = 0; k < 2; ++k) wgmma_bf16<C3_BN>(acc, a_hi + 2 * k, b_hi + 2 * k, (tap > 0 || k > 0) ? 1u : 0u);
                        if (NSPLIT == 3) {
                            const uint64_t a_lo = make_sw64_kmajor_desc(slot + C3_PLANE_BYTES + uint32_t(roff) * 64u);
                            const uint64_t b_lo = make_sw64_kmajor_desc(w_base + (tap * NP + 1) * C3_W_TILE);
#pragma unroll
                            for (int k = 0; k < 2; ++k) wgmma_bf16<C3_BN>(acc, a_lo + 2 * k, b_hi + 2 * k, 1u);
#pragma unroll
                            for (int k = 0; k < 2; ++k) wgmma_bf16<C3_BN>(acc, a_hi + 2 * k, b_lo + 2 * k, 1u);
                        }
                    }
                };
                issue(acc0, 0);
                issue(acc1, 1);
                wgmma_commit();
                wgmma_wait<0>();
                wgmma_fence_acc(acc0);
                wgmma_fence_acc(acc1);
                auto row_of = [&](int mb, int rr) -> int64_t {
                    const int prow = C3_ROW0 + tt * GEMM_BM + mb * 64 + rr;  // patch row of this accumulator row
                    const int ph = prow / C3_PW, pw = prow - ph * C3_PW;
                    const int hp = ih * C3_OH + ph, wp = iw * C3_OW + pw;  // padded grid coordinates
                    if (pw >= 1 && pw <= C3_OW && ph <= C3_OH && hp <= cp.H && wp <= cp.W) return (int64_t(b) * cp.Hp + hp) * cp.Wp + wp;
                    return -1;
                };
                epilogue_frag<C3_BN>(cp.epi, C3_BN, 0, acc0, [&](int rr) { return row_of(0, rr); }, t);
                epilogue_frag<C3_BN>(cp.epi, C3_BN, 0, acc1, [&](int rr) { return row_of(1, rr); }, t);
            }
            if (t == 0) mbar_arrive(empty_bar(stage));  // this warpgroup is done with the patch
            if (++stage == C3_STAGES) {
                stage = 0;
                phase ^= 1u;
            }
        }
    }
}

// ------------------------------------------------------------------------------------------------ host
typedef CUresult (*EncodeTiledFn5)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                   const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion,
                                   CUtensorMapFloatOOBfill);
static EncodeTiledFn5 encode_fn5() {
    static EncodeTiledFn5 fn = nullptr;
    static std::once_flag once;
    std::call_once(once, [] {
        void* p = nullptr;
        cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess && q == cudaDriverEntryPointSuccess)
            fn = reinterpret_cast<EncodeTiledFn5>(p);
    });
    return fn;
}

bool conv3x3_c32_supported(int Cin, int Cout, int H, int W) { return Cin == 32 && Cout == 32 && H >= 1 && W >= 1; }

int conv3x3_build(Conv3x3Params* cp, const Planes& x, int x_col0, const Planes& Wt, int B, int H, int W, int Hp, int Wp, const Epilogue& epi) {
    PPV_REQUIRE(Hp == H + 2 && Wp == W + 2, "conv3x3: the input must be a zero-bordered [B, H+2, W+2, C] grid");
    PPV_REQUIRE(Wt.ld == 9 * 32 && Wt.rows >= 32, "conv3x3: weight layout must be [N >= 32][9 taps x 32]");
    PPV_REQUIRE(x_col0 % 8 == 0 && x.ld % 8 == 0 && x_col0 + 32 <= x.ld, "conv3x3: input column window");
    PPV_REQUIRE(epi.out_mode == OUT_PLANES && epi.img_Wp == Wp && epi.img_Hp == Hp, "conv3x3: image-mode planes epilogue on the input grid");
    PPV_REQUIRE(x.rows >= int64_t(B) * Hp * Wp, "conv3x3: input smaller than the grid");
    memset(static_cast<void*>(cp), 0, sizeof(*cp));
    EncodeTiledFn5 enc = encode_fn5();
    if (!enc) return fail(PPV_ECUDA, "cuTensorMapEncodeTiled entry point not available");
    if ((reinterpret_cast<uintptr_t>(x.base) & 15) || (x.plane_stride % 8)) return fail(PPV_EINVAL, "conv3x3: planes tensor not 16-byte aligned");
    cuuint64_t dims[5] = {cuuint64_t(x.ld), cuuint64_t(Wp), cuuint64_t(Hp), cuuint64_t(B), 2};
    cuuint64_t strides[4] = {cuuint64_t(x.ld) * 2, cuuint64_t(Wp) * x.ld * 2, cuuint64_t(Hp) * Wp * x.ld * 2, cuuint64_t(x.plane_stride) * 2};
    cuuint32_t box[5] = {32, C3_PW, C3_PH, 1, 1};
    cuuint32_t estr[5] = {1, 1, 1, 1, 1};
    CUresult r = enc(&cp->mapX, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 5, x.base, dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                     CU_TENSOR_MAP_SWIZZLE_64B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) return fail(PPV_ECUDA, "conv3x3: cuTensorMapEncodeTiled failed, CUresult " + std::to_string(int(r)));
    int rc = encode_planes_map_ex(&cp->mapW, Wt, 32, 32, 64);
    if (rc) return rc;
    cp->x_col0 = x_col0;
    cp->B = B;
    cp->H = H;
    cp->W = W;
    cp->Hp = Hp;
    cp->Wp = Wp;
    cp->nph = (H + C3_OH - 1) / C3_OH;
    cp->npw = (W + C3_OW - 1) / C3_OW;
    cp->patches = B * cp->nph * cp->npw;
    cp->epi = epi;
    return PPV_OK;
}

template <int NSPLIT>
static int launch_c3(const Conv3x3Params& cp, int num_sms, cudaStream_t st) {
    using Cfg = C3Cfg<NSPLIT>;
    PPV_CUDA_OK(cudaFuncSetAttribute(conv3x3_c32_kernel<NSPLIT>, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::SMEM_BYTES));
    const int grid = std::min(cp.patches, num_sms);
    PPV_PDL_OK(launch_pdl(conv3x3_c32_kernel<NSPLIT>, dim3(grid), dim3(GEMM_THREADS), Cfg::SMEM_BYTES, st, cp), "conv3x3_c32_kernel");
    return PPV_OK;
}

int conv3x3_launch(const Conv3x3Params& cp, int precision, int num_sms, cudaStream_t st) {
    return precision == PPV_PREC_BF16X3 ? launch_c3<3>(cp, num_sms, st) : launch_c3<1>(cp, num_sms, st);
}

}  // namespace ppv
