// Res2Net dilated conv (K3): y_j = BN(ReLU(conv_k3,d(x_j + y_{j-1}))) for one 64-channel chunk.
// Reference: ppvector/models/ecapa_tdnn.py:36-47 (Res2NetBlock.forward) -> TDNNBlock (ppvector/models/utils.py:147).
//
// Same contraction as gemm_wgmma.cu (N = 64, K = nsrc * 3 taps * 64), restructured around what bounds it -- the
// L2 -> shared-memory fill, not the tensor pipe:
//   * the whole weight matrix of the layer (<= 6 k-slices x hi/lo = 96 KB) is loaded ONCE per CTA and stays in
//     shared memory for all of the CTA's tiles (weight-stationary);
//   * per source (x_j, y_{j-1}) ONE tall activation tile of 128 + 2*4 rows is loaded per output tile; the three
//     conv taps are the SAME shared-memory tile read at row offsets 4-d, 4, 4+d: the wgmma descriptor's start
//     address simply moves by whole 128-byte rows (the SWIZZLE_128B XOR is a function of the absolute shared-memory
//     address, exactly as TMA wrote it, so any row of a 1024-byte-aligned slot is a valid matrix start).
// L2 -> SM traffic per 128-row tile: 2 x 2 x 17 KB = 70 KB instead of 288 KB.
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include "common.h"
#include "gemm_epilogue.cuh"
#include "ptx.cuh"

namespace ppv {

constexpr int R2_PAD = 4;                              // halo rows loaded above / below (max dilation)
constexpr int R2_ROWS = GEMM_BM + 2 * R2_PAD;          // 136
constexpr int R2_A_BYTES = R2_ROWS * 128;              // 17408 B landed per plane
constexpr int R2_A_SLOT = 18 * 1024;                   // 1024-aligned slot per plane
constexpr int R2_W_TILE = 64 * 128;                    // [64 out ch x 64 k] bf16

template <int NSPLIT>
struct R2Cfg {
    static constexpr int NP = (NSPLIT == 3) ? 2 : 1;
    static constexpr int W_BYTES = 6 * NP * R2_W_TILE;  // room for 2 sources x 3 taps
    static constexpr int STAGE_BYTES = NP * R2_A_SLOT;
    static constexpr int STAGES = (NSPLIT == 3) ? 3 : 4;
    static constexpr int SMEM_BYTES = 1024 + W_BYTES + STAGES * STAGE_BYTES + 256;
};

template <int NSPLIT>
__global__ void __launch_bounds__(GEMM_THREADS, 1) res2conv_kernel(const __grid_constant__ Res2Params rp) {
    using Cfg = R2Cfg<NSPLIT>;
    constexpr int NP = Cfg::NP, STAGES = Cfg::STAGES, BN = 64;
    extern __shared__ uint8_t smem_raw[];
    const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;
    const uint32_t w_base = smem_base;
    const uint32_t a_base = smem_base + Cfg::W_BYTES;
    const uint32_t bar_base = a_base + STAGES * Cfg::STAGE_BYTES;
    auto full_bar = [&](int s) { return bar_base + 8u * s; };
    auto empty_bar = [&](int s) { return bar_base + 8u * (STAGES + s); };
    const uint32_t w_full = bar_base + 8u * (2 * STAGES);

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    if (warp == 0 && lane == 0) {
        prefetch_tmap(&rp.mapA[0]);
        prefetch_tmap(&rp.mapA[1]);
        prefetch_tmap(&rp.mapW);
    }
    if (warp == 1 && lane == 0) {
        for (int s = 0; s < STAGES; ++s) {
            mbar_init(full_bar(s), 1);
            mbar_init(empty_bar(s), GEMM_MMA_THREADS / 128);  // one arrival per MMA warpgroup
        }
        mbar_init(w_full, 1);
        fence_mbar_init();
    }
    __syncthreads();
    const int nsrc = rp.nsrc;
    const int wslices = nsrc * 3;
    griddep_launch_dependents();  // PDL

    if (warp == 0) {
        // ===================== TMA producer =====================
        if (lane == 0) {  // weights: once per CTA
            mbar_arrive_expect_tx(w_full, wslices * NP * R2_W_TILE);
            for (int ks = 0; ks < wslices; ++ks)
                for (int pl = 0; pl < NP; ++pl) tma_load_3d(w_base + (ks * NP + pl) * R2_W_TILE, &rp.mapW, w_full, ks * 64, 0, pl);
        }
        __syncwarp();
        griddep_wait();  // the weights above are constants; the activations below come from the previous kernel
        int stage = 0;
        uint32_t phase = 0;
        for (int tile = blockIdx.x; tile < rp.m_tiles; tile += gridDim.x) {
            const int m0 = tile * GEMM_BM;
            const int ntile = tile + gridDim.x;
            if (rp.l2_prefetch && ntile < rp.m_tiles && lane < nsrc * NP) {  // next tile's rows: HBM -> L2 ahead of time
                const int s = lane / NP, pl = lane % NP;
                tma_prefetch_l2_3d(&rp.mapA[s], rp.a_col[s], ntile * GEMM_BM - R2_PAD, pl);
            }
            __syncwarp();
            for (int s = 0; s < nsrc; ++s) {
                mbar_wait(empty_bar(stage), phase ^ 1u);
                if (lane == 0) {
                    mbar_arrive_expect_tx(full_bar(stage), NP * R2_A_BYTES);
                    for (int pl = 0; pl < NP; ++pl)
                        tma_load_3d(a_base + stage * Cfg::STAGE_BYTES + pl * R2_A_SLOT, &rp.mapA[s], full_bar(stage), rp.a_col[s],
                                    m0 - R2_PAD, pl);
                }
                __syncwarp();
                if (++stage == STAGES) {
                    stage = 0;
                    phase ^= 1u;
                }
            }
        }
    } else if (warp >= 4) {
        // ===================== MMA + epilogue: warpgroup g owns rows [64 g, 64 g + 64) of every tile =====================
        const int g = (warp - 4) >> 2, t = threadIdx.x & 127;
        griddep_wait();  // the epilogue writes buffers that upstream kernels may still be reading
        mbar_wait(w_full, 0);
        int stage = 0;
        uint32_t phase = 0;
        float acc[BN / 2];
#pragma unroll
        for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
        for (int tile = blockIdx.x; tile < rp.m_tiles; tile += gridDim.x) {
            int prev = -1;
            wgmma_fence_acc(acc);
            for (int s = 0; s < nsrc; ++s) {
                mbar_wait(full_bar(stage), phase);
                const uint32_t slot = a_base + stage * Cfg::STAGE_BYTES;
                wgmma_fence();
#pragma unroll
                for (int tap = 0; tap < 3; ++tap) {
                    // rows [roff, roff + 64) of the tall tile: whole 128-byte rows of a 1024-byte-aligned slot
                    const uint32_t roff = uint32_t(R2_PAD + (tap - 1) * rp.dil + 64 * g);
                    const uint64_t a_hi = make_sw128_kmajor_desc(slot + roff * 128u);
                    const uint64_t b_hi = make_sw128_kmajor_desc(w_base + ((s * 3 + tap) * NP) * R2_W_TILE);
#pragma unroll
                    for (int k = 0; k < 4; ++k) wgmma_bf16<BN>(acc, a_hi + 2 * k, b_hi + 2 * k, (s > 0 || tap > 0 || k > 0) ? 1u : 0u);
                    if (NSPLIT == 3) {
                        const uint64_t a_lo = make_sw128_kmajor_desc(slot + R2_A_SLOT + roff * 128u);
                        const uint64_t b_lo = make_sw128_kmajor_desc(w_base + ((s * 3 + tap) * NP + 1) * R2_W_TILE);
#pragma unroll
                        for (int k = 0; k < 4; ++k) wgmma_bf16<BN>(acc, a_lo + 2 * k, b_hi + 2 * k, 1u);
#pragma unroll
                        for (int k = 0; k < 4; ++k) wgmma_bf16<BN>(acc, a_hi + 2 * k, b_lo + 2 * k, 1u);
                    }
                }
                wgmma_commit();
                wgmma_wait<1>();
                if (prev >= 0 && t == 0) mbar_arrive(empty_bar(prev));
                prev = stage;
                if (++stage == STAGES) {
                    stage = 0;
                    phase ^= 1u;
                }
            }
            wgmma_wait<0>();
            wgmma_fence_acc(acc);
            if (t == 0) mbar_arrive(empty_bar(prev));
            const int rbase = tile * GEMM_BM + 64 * g;
            epilogue_frag<BN>(rp.epi, BN, 0, acc, [&](int r) -> int64_t { return rbase + r < rp.M ? int64_t(rbase + r) : -1; }, t);
        }
    }
}

int res2conv_build(Res2Params* rp, const GemmSource* srcs, int nsrc, const Planes& W, int M, int dil, const Epilogue& epi) {
    PPV_REQUIRE(nsrc == 1 || nsrc == 2, "res2conv: 1 or 2 sources");
    PPV_REQUIRE(dil >= 1 && dil <= R2_PAD, "res2conv: dilation must be in [1,4]");
    PPV_REQUIRE(W.ld == nsrc * 3 * 64 && W.rows >= 64, "res2conv: weight layout mismatch");
    PPV_REQUIRE(epi.out_mode == OUT_PLANES, "res2conv: planes output only");
    memset(static_cast<void*>(rp), 0, sizeof(*rp));
    for (int s = 0; s < nsrc; ++s) {
        PPV_REQUIRE(srcs[s].ncols == 64 && srcs[s].col0 % 8 == 0, "res2conv: each source is one 64-channel chunk");
        int rc = encode_planes_map_ex(&rp->mapA[s], srcs[s].t, 64, R2_ROWS, 128);
        if (rc) return rc;
        rp->a_col[s] = srcs[s].col0;
    }
    if (nsrc == 1) rp->mapA[1] = rp->mapA[0];
    int rc = encode_planes_map(&rp->mapW, W, 64);
    if (rc) return rc;
    rp->nsrc = nsrc;
    rp->dil = dil;
    {
        const char* pf = getenv("PPV_GEMM_NO_L2PREFETCH");
        rp->l2_prefetch = (pf && pf[0] == '1') ? 0 : 1;
    }
    rp->M = M;
    rp->m_tiles = (M + GEMM_BM - 1) / GEMM_BM;
    rp->epi = epi;
    return PPV_OK;
}

template <int NSPLIT>
static int launch_r2(const Res2Params& rp, int num_sms, cudaStream_t st) {
    using Cfg = R2Cfg<NSPLIT>;
    PPV_ONCE_PER_DEVICE(PPV_CUDA_OK(cudaFuncSetAttribute(res2conv_kernel<NSPLIT>, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::SMEM_BYTES)));
    const int grid = std::min(rp.m_tiles, num_sms);
    PPV_PDL_OK(launch_pdl(res2conv_kernel<NSPLIT>, dim3(grid), dim3(GEMM_THREADS), Cfg::SMEM_BYTES, st, rp), "res2conv_kernel");
    return PPV_OK;
}

int res2conv_launch(const Res2Params& rp, int precision, int num_sms, cudaStream_t st) {
    return precision == PPV_PREC_BF16X3 ? launch_r2<3>(rp, num_sms, st) : launch_r2<1>(rp, num_sms, st);
}

}  // namespace ppv
