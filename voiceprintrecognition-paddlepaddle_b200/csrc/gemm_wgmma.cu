// Gather-GEMM on the Hopper tensor cores (wgmma + TMA + mbarrier), the contraction behind every Conv1d / Linear of the
// ppvector hot path (reference: ppvector/models/utils.py:65-77 Conv1d.forward, reached from TDNNBlock utils.py:147,
// Res2NetBlock ecapa_tdnn.py:36-47, ASP pooling.py:107, fc).
//
//   out[r, n] = epilogue( sum_s  A_{map(s)}[r + row_off(s), a_col(s) : a_col(s)+64] . W[n, 64 s : 64 s + 64] )
//
// A "k-step" s is one 64-wide K slice: a conv tap is a row offset in the padded time layout, a channel
// concat is a different source tensor, `x_i + y_{i-1}` (Res2Net) is two sources sharing the same weights.
// Operands are split-bf16 planes (hi, lo); PPV_PREC_BF16X3 issues hi*hi + lo*hi + hi*lo into one fp32
// register accumulator (fp32-grade), PPV_PREC_BF16 issues hi*hi only.
//
// Warp roles (384 threads, 1 CTA / SM, persistent over 128 x BN tiles):
//   warp 0        TMA producer : cp.async.bulk.tensor 3-D tiles (SWIZZLE_128B / 64B) into a STAGES-deep smem ring, in tile order
//   warps 4-7     MMA warpgroup 0 : wgmma m64 x BN x 16 from the ring, then bias / ReLU / BN affine / tanh ->
//   warps 8-11    MMA warpgroup 1   split-bf16 (or fp32) stores incl. the reflect-halo rows
// BN <= 128 (ping-pong): warpgroup g owns the CTA's tiles g, g + 2, ... whole (two m64 accumulators), so one warpgroup's epilogue
// runs while the other's MMAs keep the tensor cores busy.  BN = 256 (cooperative): warpgroup g owns rows [64 g, 64 g + 64) of every
// tile and both run their epilogues together.  The producer warpgroup hands its registers to the MMA warpgroups (setmaxnreg 40 / 232).
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <algorithm>
#include <mutex>

#include "common.h"
#include "gemm_epilogue.cuh"
#include "ptx.cuh"

namespace ppv {

constexpr int GEMM_MAX_STAGES = 8;  // barrier slots

// The shared-memory ring of an n-tile BN wide with BK-element k-steps: bytes per stage (the A and W tiles, hi and, for
// bf16x3, lo planes), as many stages as fit the 227 KB opt-in beside 1024 bytes of alignment slack and 256 of barriers, and
// the dynamic shared memory that takes.
struct GemmRing {
    int stage_bytes, stages, smem_bytes;
};
constexpr GemmRing gemm_ring(int BN, int BK, int nsplit) {
    const int stage_bytes = (nsplit == 3 ? 2 : 1) * (GEMM_BM + BN) * BK * 2;
    const int fit = (232448 - 1024 - 256) / stage_bytes;
    const int stages = fit > GEMM_MAX_STAGES ? GEMM_MAX_STAGES : fit;
    return {stage_bytes, stages, 1024 + stages * stage_bytes + 256};
}

// BK = K elements per pipeline stage: 64 (128-byte rows, SWIZZLE_128B) or 32 (64-byte rows, SWIZZLE_64B).  The smaller
// stage keeps the same bytes per MMA but doubles the number of ring slots, i.e. more TMA bytes in flight for the same
// shared memory.
template <int BN, int NSPLIT, int BK>
struct GemmCfg {
    static constexpr int NA = (NSPLIT == 3) ? 2 : 1;  // A tiles per stage (hi[, lo])
    static constexpr int NB = NA;
    static constexpr int A_BYTES = GEMM_BM * BK * 2;
    static constexpr int B_BYTES = BN * BK * 2;
    static constexpr GemmRing RING = gemm_ring(BN, BK, NSPLIT);
    static constexpr int STAGE_BYTES = RING.stage_bytes;
    static constexpr int STAGES = RING.stages;
    static constexpr int SMEM_BYTES = RING.smem_bytes;
    static_assert(STAGE_BYTES == NA * A_BYTES + NB * B_BYTES, "stage layout");
    // Ping-pong schedule (each MMA warpgroup owns whole tiles, two m64 x BN accumulators) where a tile fits in registers: BN <= 128.
    // BN = 256 would need 256 accumulator registers per thread and keeps the cooperative schedule (both warpgroups share every tile).
    static constexpr bool PINGPONG = BN <= 128;
    static constexpr int EMPTY_ARRIVALS = PINGPONG ? 1 : GEMM_MMA_THREADS / 128;  // consumers that release one ring slot
    static_assert(STAGES >= 2, "need at least a double buffer");
    static_assert(BN == 64 || BN == 128 || BN == 256, "BN");
    static_assert(BK == 64 || BK == 32, "BK");
};

template <int BK>
__device__ __forceinline__ uint64_t make_kmajor_desc(uint32_t smem_addr) {
    return BK == 64 ? make_sw128_kmajor_desc(smem_addr) : make_sw64_kmajor_desc(smem_addr);
}

template <int BN, int NSPLIT, int BK>
__global__ void __launch_bounds__(GEMM_THREADS, 1) gemm_wgmma_kernel(const __grid_constant__ GemmParams gp) {
    using Cfg = GemmCfg<BN, NSPLIT, BK>;
    constexpr int STAGES = Cfg::STAGES;
    extern __shared__ uint8_t smem_raw[];
    // SWIZZLE_128B tiles need 1024-byte alignment.
    const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;
    const uint32_t tiles_base = smem_base;
    const uint32_t bar_base = smem_base + STAGES * Cfg::STAGE_BYTES;
    // barrier layout (8 B each): full[8], empty[8], resident-weights barrier
    constexpr int MAXST = GEMM_MAX_STAGES;
    auto full_bar = [&](int s) { return bar_base + 8u * s; };
    auto empty_bar = [&](int s) { return bar_base + 8u * (MAXST + s); };
    const uint32_t w_full = bar_base + 8u * (2 * MAXST);

    const int warp = threadIdx.x >> 5;
    const int lane = threadIdx.x & 31;
    // Weight-stationary mode (gp.ws, narrow convs with one n-tile and a small K): the whole weight matrix is loaded ONCE per CTA
    // into the upper part of the ring's shared memory and the ring (4 slots) carries activation tiles only -- for the
    // 32-channel 3x3 convs of the 2-D models the per-tile reload of the weights was a third of the L2 -> SM traffic.
    const int nst = gp.ws ? GEMM_WS_STAGES : STAGES;
    const uint32_t w_res = tiles_base + GEMM_WS_STAGES * Cfg::STAGE_BYTES;

    if (warp == 0 && lane == 0) {
        for (int i = 0; i < GEMM_MAX_MAPS; ++i) prefetch_tmap(&gp.mapA[i]);
        prefetch_tmap(&gp.mapB);
    }
    if (warp == 1 && lane == 0) {
        for (int s = 0; s < MAXST; ++s) {
            mbar_init(full_bar(s), 1);
            mbar_init(empty_bar(s), Cfg::EMPTY_ARRIVALS);
        }
        mbar_init(w_full, 1);
        fence_mbar_init();
    }
    __syncthreads();
    griddep_launch_dependents();  // PDL: the next kernel may begin its prologue
    griddep_wait();               // PDL: upstream activations are complete and visible

    // lin_splits > 0: "wgrad" mode -- the contraction runs over the COLUMNS of both operands (two transposed matrices
    // [M][R] and [N][R]), k-step s of split z reads columns (z * nk + s) * BK; there is no k-step table, and split z of
    // tile (m, n) accumulates into its own partial output block (rows shifted by z * lin_split_rows).
    const int mn_tiles = gp.m_tiles * gp.n_tiles;
    const int num_tiles = mn_tiles * (gp.lin_splits > 0 ? gp.lin_splits : 1);
    const int nk = gp.num_ksteps;
    auto tile_m = [&](int t) { return (t % mn_tiles) / gp.n_tiles; };
    auto tile_n = [&](int t) { return (t % mn_tiles) % gp.n_tiles; };
    // PPV_GEMM_TRACE stamps of one CTA (gp.trace_cta; `on`: tracing, this CTA, the stamping thread, local tile in range), GEMM_TRACE_EVENTS
    // per tile.  Producer: 0-2 / 3-5 its ring-slot waits of k-steps 0-2 / nk-3..nk-1 passed, 8-10 / 11-13 their TMA loads issued, 7 of
    // tile 0 the kernel start.  MMA warpgroup: 0 hand-off barrier passed, 1 first `full` wait passed, 2 last
    // k-step issued, 3 wgmma_wait<0> returned, 4 / 5 epilogue start / end, 6-8 / 9-11 the `empty` arrivals releasing k-steps 0-2 /
    // nk-3..nk-1.
    const bool trace_cta = gp.trace != nullptr && int(blockIdx.x) == gp.trace_cta;
    auto stamp = [&](bool on, int role, int local, int ev) {
        if (on) gp.trace[(role * GEMM_TRACE_TILES + local) * GEMM_TRACE_EVENTS + ev] = clock64();
    };
    // the first and last three k-steps of a tile: event base + 0..2 / base + 3..5
    auto stamp_kstep = [&](bool on, int role, int local, int base, int s) {
        if (s >= 0 && s < 3) stamp(on, role, local, base + s);
        if (s >= nk - 3 && s >= 0) stamp(on, role, local, base + 3 + s - (nk - 3));
    };
    auto stamp_release = [&](bool on, int role, int local, int s) { stamp_kstep(on, role, local, 6, s); };
    stamp(trace_cta && threadIdx.x == 0, 0, 0, 7);

    if (warp < 4) {
        setmaxnreg_dec<40>();  // all four producer warps; warps 1-3 have nothing else to do
        if (warp == 0) {
            // ===================== TMA producer =====================
            int stage = 0;
            uint32_t phase = 0;
            if (gp.ws && lane == 0) {  // resident weights: every k-slice, once
                mbar_arrive_expect_tx(w_full, nk * Cfg::NB * Cfg::B_BYTES);
                for (int s = 0; s < nk; ++s)
                    for (int p = 0; p < Cfg::NB; ++p) tma_load_3d(w_res + (s * Cfg::NB + p) * Cfg::B_BYTES, &gp.mapB, w_full, s * BK, 0, p);
            }
            __syncwarp();
            int local = 0;
            for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x, ++local) {
                const bool tr = trace_cta && lane == 0 && local < GEMM_TRACE_TILES;
                const int zsplit = tile / mn_tiles;
                const int m0 = tile_m(tile) * GEMM_BM;
                const int n0 = tile_n(tile) * BN;
                for (int s = 0; s < nk; ++s) {
                    mbar_wait(empty_bar(stage), phase ^ 1u);
                    stamp_kstep(tr, 0, local, 0, s);
                    if (lane == 0) {
                        const uint32_t sa = tiles_base + stage * Cfg::STAGE_BYTES;
                        const uint32_t sb = sa + Cfg::NA * Cfg::A_BYTES;
                        const uint32_t fb = full_bar(stage);
                        mbar_arrive_expect_tx(fb, gp.ws ? Cfg::NA * Cfg::A_BYTES : Cfg::STAGE_BYTES);
                        if (gp.ws) {
                            const KStep ks = gp.ksteps[s];
#pragma unroll
                            for (int p = 0; p < Cfg::NA; ++p) tma_load_3d(sa + p * Cfg::A_BYTES, &gp.mapA[ks.map()], fb, ks.a_col(), m0 + ks.row_off, p);
                        } else if (gp.lin_splits > 0) {
                            const int kcol = (zsplit * nk + s) * BK;
#pragma unroll
                            for (int p = 0; p < Cfg::NA; ++p) tma_load_3d(sa + p * Cfg::A_BYTES, &gp.mapA[0], fb, kcol, m0, p);
#pragma unroll
                            for (int p = 0; p < Cfg::NB; ++p)
                                tma_load_3d(sb + p * Cfg::B_BYTES, &gp.mapB, fb, kcol + gp.lin_b_col0, gp.lin_b_row0 + n0, p);
                        } else {
                            const KStep ks = gp.ksteps[s];
                            const CUtensorMap* ma = &gp.mapA[ks.map()];
#pragma unroll
                            for (int p = 0; p < Cfg::NA; ++p) tma_load_3d(sa + p * Cfg::A_BYTES, ma, fb, ks.a_col(), m0 + ks.row_off, p);
#pragma unroll
                            for (int p = 0; p < Cfg::NB; ++p) tma_load_3d(sb + p * Cfg::B_BYTES, &gp.mapB, fb, s * BK, n0, p);
                        }
                        stamp_kstep(tr, 0, local, 8, s);
                    }
                    __syncwarp();
                    if (++stage == nst) {
                        stage = 0;
                        phase ^= 1u;
                    }
                }
            }
        }
    } else {
        setmaxnreg_inc<232>();  // 128 x 40 + 256 x 232 <= 64 K registers
        // ===================== MMA + epilogue =====================
        // Ping-pong (BN <= 128): warpgroup g owns the CTA's tiles g, g + 2, g + 4, ... whole, as two m64 x BN accumulators (rows 0-63
        // and 64-127), and skips the ring positions of the other's tiles.  The producer fills the ring in tile order and the warpgroup
        // that consumes a slot releases it.  Ordered hand-off: a warpgroup starts its k-loop only once the other has waited for every
        // k-step of the tile before (named barrier 1 + g, arrived at by the other warpgroup).  So the k-loops run one after the other,
        // one warpgroup's epilogue runs under the other's MMAs, and no warpgroup ever waits for a ring slot more than one fill ahead of
        // the last completed one (an mbarrier parity wait cannot tell fill k from fill k + 2).
        // Cooperative (BN = 256): warpgroup g owns rows [64 g, 64 g + 64) of every tile, one accumulator; both release each slot.
        constexpr bool PP = Cfg::PINGPONG;
        constexpr int NACC = PP ? 2 : 1;  // m64 x BN accumulators per warpgroup: acc0[, acc1]
        const int g = (warp - 4) >> 2;
        const int t = threadIdx.x & 127;
        constexpr uint32_t A_M64 = 64 * BK * 2;  // 64 rows of the A tile (a whole number of 8-row swizzle groups)
        auto m64 = [&](int h) { return PP ? h : g; };  // the 64-row block of the tile that accumulator h holds
        const int my_tiles = blockIdx.x < num_tiles ? (num_tiles - 1 - int(blockIdx.x)) / int(gridDim.x) + 1 : 0;
        int stage = 0;
        uint32_t phase = 0;
        float acc0[BN / 2], acc1[BN / 2];
#pragma unroll
        for (int i = 0; i < BN / 2; ++i) acc0[i] = acc1[i] = 0.f;
        // the MMAs of one 16-wide K slice: acc0, then acc1.  K advance inside the swizzle atom: +32 B (16 bf16) per MMA => +2 in the
        // descriptor's start field
        auto mma = [&](uint64_t a0, uint64_t a1, uint64_t b, int k, uint32_t scale_d) {
            wgmma_bf16<BN>(acc0, a0 + 2 * k, b + 2 * k, scale_d);
            if (PP) wgmma_bf16<BN>(acc1, a1 + 2 * k, b + 2 * k, scale_d);
        };
        if (gp.ws) mbar_wait(w_full, 0);
        int local = 0;  // index of the tile among this CTA's tiles
        for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x, ++local) {
            if (PP && (local & 1) != g) {  // the other warpgroup's tile: skip its nk ring positions
                const int adv = stage + nk;
                phase ^= uint32_t((adv / nst) & 1);
                stage = adv % nst;
                continue;
            }
            const int m0 = tile_m(tile) * GEMM_BM;
            const int n0 = tile_n(tile) * BN;
            const bool tr = trace_cta && t == 0 && local < GEMM_TRACE_TILES;
            if (PP) named_bar_sync_if(local > 0, 1 + g, 2 * 128);  // the other warpgroup has taken every k-step of tile local - 1
            stamp(tr, 1 + g, local, 0);
            int prev = -1;
            wgmma_fence_acc(acc0);
            if (PP) wgmma_fence_acc(acc1);
            for (int s = 0; s < nk; ++s) {
                mbar_wait(full_bar(stage), phase);
                stamp(tr && s == 0, 1 + g, local, 1);
                const uint32_t sa = tiles_base + stage * Cfg::STAGE_BYTES;
                const uint32_t sb = gp.ws ? w_res + s * Cfg::NB * Cfg::B_BYTES : sa + Cfg::NA * Cfg::A_BYTES;
                const uint64_t a0_hi = make_kmajor_desc<BK>(sa + m64(0) * A_M64), a1_hi = make_kmajor_desc<BK>(sa + m64(1) * A_M64);
                const uint64_t b_hi = make_kmajor_desc<BK>(sb);
                wgmma_fence();
                // per accumulator hi*hi, lo*hi, hi*lo, k ascending in each
#pragma unroll
                for (int k = 0; k < BK / 16; ++k) mma(a0_hi, a1_hi, b_hi, k, (s > 0 || k > 0) ? 1u : 0u);
                if (NSPLIT == 3) {
                    const uint32_t sa_lo = sa + Cfg::A_BYTES;
                    const uint64_t a0_lo = make_kmajor_desc<BK>(sa_lo + m64(0) * A_M64), a1_lo = make_kmajor_desc<BK>(sa_lo + m64(1) * A_M64);
                    const uint64_t b_lo = make_kmajor_desc<BK>(sb + Cfg::B_BYTES);
#pragma unroll
                    for (int k = 0; k < BK / 16; ++k) mma(a0_lo, a1_lo, b_hi, k, 1u);
#pragma unroll
                    for (int k = 0; k < BK / 16; ++k) mma(a0_hi, a1_hi, b_lo, k, 1u);
                }
                wgmma_commit();
                stamp(tr && s == nk - 1, 1 + g, local, 2);
                wgmma_wait<1>();  // the previous k-step's MMAs have retired: its ring slot is free
                if (prev >= 0 && t == 0) mbar_arrive(empty_bar(prev));
                stamp_release(tr, 1 + g, local, s - 1);
                prev = stage;
                if (++stage == nst) {
                    stage = 0;
                    phase ^= 1u;
                }
            }
            wgmma_wait<0>();
            stamp(tr, 1 + g, local, 3);
            if (PP) named_bar_arrive_if(local + 1 < my_tiles, 1 + (g ^ 1), 2 * 128);  // the other warpgroup may start tile local + 1
            wgmma_fence_acc(acc0);
            if (PP) wgmma_fence_acc(acc1);
            if (t == 0) mbar_arrive(empty_bar(prev));
            stamp_release(tr, 1 + g, local, nk - 1);
            stamp(tr, 1 + g, local, 4);
            const int64_t shift = int64_t(tile / mn_tiles) * gp.lin_split_rows;
            // acc0, then (ping-pong) acc1 moved down into acc0: one copy of the epilogue code
#pragma unroll 1
            for (int h = 0; h < NACC; ++h) {
                const int rbase = m0 + 64 * m64(h);
                gemm_epilogue<BN>(gp.epi, gp.N, n0, acc0, [&](int r) -> int64_t { return rbase + r < gp.M ? int64_t(rbase + r) : -1; }, t, shift);
                if (PP)
#pragma unroll
                    for (int i = 0; i < BN / 2; ++i) acc0[i] = acc1[i];
            }
            stamp(tr, 1 + g, local, 5);
        }
    }
}

// ------------------------------------------------------------------------------------------------ host
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn get_encode_fn() {
    static EncodeTiledFn fn = nullptr;
    static std::once_flag once;
    std::call_once(once, [] {
        void* p = nullptr;
        cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
            q == cudaDriverEntryPointSuccess)
            fn = reinterpret_cast<EncodeTiledFn>(p);
    });
    return fn;
}

int encode_planes_map_ex(CUtensorMap* m, const Planes& t, int box_cols, int box_rows, int swizzle_bytes) {
    EncodeTiledFn enc = get_encode_fn();
    if (!enc) return fail(PPV_ECUDA, "cuTensorMapEncodeTiled entry point not available");
    if ((reinterpret_cast<uintptr_t>(t.base) & 15) || (t.ld % 8) || (t.plane_stride % 8))
        return fail(PPV_EINVAL, "planes tensor not 16-byte aligned");
    cuuint64_t dims[3] = {cuuint64_t(t.ld), cuuint64_t(t.rows), 2};
    cuuint64_t strides[2] = {cuuint64_t(t.ld) * 2, cuuint64_t(t.plane_stride) * 2};
    cuuint32_t box[3] = {cuuint32_t(box_cols), cuuint32_t(box_rows), 1};
    cuuint32_t estr[3] = {1, 1, 1};
    CUresult r = enc(m, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 3, t.base, dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                     swizzle_bytes == 128 ? CU_TENSOR_MAP_SWIZZLE_128B : swizzle_bytes == 64 ? CU_TENSOR_MAP_SWIZZLE_64B : CU_TENSOR_MAP_SWIZZLE_NONE,
                     CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                     CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) return fail(PPV_ECUDA, "cuTensorMapEncodeTiled failed, CUresult " + std::to_string(int(r)));
    return PPV_OK;
}

// 3-D map over split planes [2][rows][ld] bf16, box = {64 cols, box_rows, 1 plane}, SWIZZLE_128B.
int encode_planes_map(CUtensorMap* m, const Planes& t, int box_rows) { return encode_planes_map_ex(m, t, GEMM_BK, box_rows, 128); }

// The set-up both builders share: zeroed parameters; A map 0 in every A-map slot, since the producer prefetches all of them
// (gemm_build overwrites the slots of further A tensors); the tiling and n-tile width; the epilogue, with the test for paired fp32 stores.
static int gemm_params_init(GemmParams* gp, const Planes& a0, int M, int N, int BN, int BK, const Epilogue& epi) {
    memset(gp, 0, sizeof(*gp));
    int rc = encode_planes_map_ex(&gp->mapA[0], a0, BK, GEMM_BM, BK * 2);
    if (rc) return rc;
    for (int j = 1; j < GEMM_MAX_MAPS; ++j) gp->mapA[j] = gp->mapA[0];
    gp->bk = BK;
    gp->M = M;
    gp->N = N;
    gp->m_tiles = (M + GEMM_BM - 1) / GEMM_BM;
    gp->n_tiles = (N + BN - 1) / BN;
    gp->bn = BN;
    gp->epi = epi;
    if (epi.out_mode == OUT_F32)
        gp->epi.f32_vec_ok = ((epi.out_ld % 2) == 0 && (epi.out_col0 % 2) == 0 && (reinterpret_cast<uintptr_t>(epi.out) & 7) == 0) ? 1 : 0;
    return PPV_OK;
}

int gemm_build(GemmParams* gp, const GemmSource* srcs, int nsrc, const Planes& W, int M, int N, const Epilogue& epi,
               int BN, int BK) {
    if (BK == 0) {
        BK = 64;
        for (int i = 0; i < nsrc; ++i)
            if (srcs[i].ncols % 64) BK = 32;
    }
    PPV_REQUIRE(BK == 64 || BK == 32, "gemm_build: BK must be 64 or 32");
    PPV_REQUIRE(BN == 64 || BN == 128 || BN == 256, "gemm_build: BN must be 64/128/256");
    PPV_REQUIRE(epi.out_mode == OUT_F32 || N % 32 == 0, "gemm_build: planes output needs N % 32 == 0");
    PPV_REQUIRE(!epi.rowgrp_bias || N % 32 == 0, "gemm_build: row-group bias needs N % 32 == 0");
    PPV_REQUIRE(nsrc > 0, "gemm_build: empty K");
    int rc = gemm_params_init(gp, srcs[0].t, M, N, BN, BK, epi);
    if (rc) return rc;
    // distinct A tensors -> maps, the first one map 0
    const __nv_bfloat16* bases[GEMM_MAX_MAPS] = {srcs[0].t.base};
    int nmaps = 1;
    int ks = 0;
    for (int i = 0; i < nsrc; ++i) {
        const GemmSource& s = srcs[i];
        PPV_REQUIRE(s.ncols % BK == 0 && s.col0 % 8 == 0, "gemm_build: source K slice must be a multiple of the k-step");
        PPV_REQUIRE(s.col0 + s.ncols <= s.t.ld, "gemm_build: source K slice exceeds the row");
        int mi = -1;
        for (int j = 0; j < nmaps; ++j)
            if (bases[j] == s.t.base) mi = j;
        if (mi < 0) {
            PPV_REQUIRE(nmaps < GEMM_MAX_MAPS, "gemm_build: too many distinct A tensors");
            mi = nmaps++;
            bases[mi] = s.t.base;
            rc = encode_planes_map_ex(&gp->mapA[mi], s.t, BK, GEMM_BM, BK * 2);
            if (rc) return rc;
        }
        for (int c = 0; c < s.ncols; c += BK) {
            PPV_REQUIRE(ks < GEMM_MAX_KSTEPS, "gemm_build: too many k-steps");
            PPV_REQUIRE(s.col0 + c < (1 << 17), "gemm_build: K slice starts past column 131064");
            gp->ksteps[ks].map_col = uint16_t((mi << 14) | ((s.col0 + c) >> 3));
            gp->ksteps[ks].row_off = int16_t(s.row_off);
            ++ks;
        }
    }
    PPV_REQUIRE(ks > 0, "gemm_build: empty K");
    PPV_REQUIRE(W.ld == ks * BK, "gemm_build: weight K does not match the k-steps");
    PPV_REQUIRE(W.rows >= N, "gemm_build: weight rows < N");
    rc = encode_planes_map_ex(&gp->mapB, W, BK, BN, BK * 2);
    if (rc) return rc;
    gp->num_ksteps = ks;
    {
        // weight-stationary: one n-tile, all k-slices of W (both planes) fit next to a GEMM_WS_STAGES-slot ring, and enough tiles per
        // CTA to pay (two per SM of a 132-SM H100).  Sized on the bf16x3 ring: the bf16 ring holds half the bytes in at least as many stages.
        const GemmRing ring = gemm_ring(BN, BK, 3);
        const size_t w_bytes = size_t(ks) * 2 * BN * BK * 2;
        const char* wsenv = getenv("PPV_GEMM_WS");
        gp->ws = (gp->n_tiles == 1 && ring.stages > GEMM_WS_STAGES && w_bytes <= size_t(ring.stages - GEMM_WS_STAGES) * ring.stage_bytes &&
                  gp->m_tiles >= 264 && !(wsenv && wsenv[0] == '0'))
                     ? 1
                     : 0;
    }
    {
        const char* ns = getenv("PPV_GEMM_NOSTORE");
        gp->epi.debug_nostore = (ns && ns[0] == '1') ? 1 : 0;
    }
    if (const char* tr = getenv("PPV_GEMM_TRACE")) {  // debug: leaked on purpose, read back by gemm_trace_dump
        constexpr size_t n = 3 * GEMM_TRACE_TILES * GEMM_TRACE_EVENTS;
        static unsigned long long* buf = nullptr;
        if (!buf) PPV_CUDA_OK(cudaMalloc(reinterpret_cast<void**>(&buf), n * sizeof(unsigned long long)));
        PPV_CUDA_OK(cudaMemset(buf, 0, n * sizeof(unsigned long long)));
        gp->trace = buf;
        gp->trace_cta = atoi(tr);
    }
    if (epi.out_mode == OUT_PLANES) {
        PPV_REQUIRE((epi.out_ld % 16) == 0 && (epi.out_col0 % 16) == 0 && (epi.out_plane_stride % 16) == 0 &&
                        (reinterpret_cast<uintptr_t>(epi.out) & 15) == 0,
                    "gemm_build: planes output must be 16-byte aligned");
        // the layers of the ECAPA plan: the lean epilogue path covers everything they ask for
        gp->epi.lean = (!epi.halo && !epi.zero_invalid && epi.img_Wp == 0 && !epi.seg_scale && !epi.silu_ && !epi.sigmoid_ &&
                        !(epi.relu && epi.relu_max > 0.f) && !gp->epi.debug_nostore)
                           ? 1
                           : 0;
    }
    return PPV_OK;
}

// Weight-gradient GEMM: out[z][m, out_col0 + n] = sum over columns r of split z of  At[m, r] * Bt[b_row0 + n, r + b_col0]
// (At = transposed output gradient [M][R], Bt = transposed layer input [*][R]; b_col0 = conv tap offset in rows of the
// padded time layout).  Partial blocks are `split_rows` output rows apart; the caller sums them.
int gemm_build_wgrad(GemmParams* gp, const Planes& At, const Planes& Bt, int M, int N, int b_row0, int b_col0, int splits, float* out,
                     int64_t out_ld, int out_col0, int64_t split_rows, int BN) {
    PPV_REQUIRE(BN == 64 || BN == 128 || BN == 256, "gemm_build_wgrad: BN must be 64/128/256");
    PPV_REQUIRE(At.ld == Bt.ld && splits >= 1, "gemm_build_wgrad: operands must share the contraction length");
    Epilogue ep;
    ep.out_mode = OUT_F32;
    ep.out = out;
    ep.out_ld = out_ld;
    ep.out_col0 = out_col0;
    int rc = gemm_params_init(gp, At, M, N, BN, GEMM_BK, ep);
    if (rc) return rc;
    rc = encode_planes_map_ex(&gp->mapB, Bt, GEMM_BK, BN, 128);
    if (rc) return rc;
    const int nk_total = (At.ld + GEMM_BK - 1) / GEMM_BK;
    gp->lin_splits = std::min(splits, nk_total);
    gp->num_ksteps = (nk_total + gp->lin_splits - 1) / gp->lin_splits;
    gp->lin_b_row0 = b_row0;
    gp->lin_b_col0 = b_col0;
    gp->lin_split_rows = split_rows;
    PPV_REQUIRE(N % 32 == 0, "gemm_build_wgrad: N % 32 == 0 required");
    return PPV_OK;
}

template <int BN, int NSPLIT, int BK>
static int launch_one(const GemmParams& gp, int num_sms, cudaStream_t stream) {
    using Cfg = GemmCfg<BN, NSPLIT, BK>;
    PPV_ONCE_PER_DEVICE(PPV_CUDA_OK(cudaFuncSetAttribute(gemm_wgmma_kernel<BN, NSPLIT, BK>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                         Cfg::SMEM_BYTES)));
    const int tiles = gp.m_tiles * gp.n_tiles * (gp.lin_splits > 0 ? gp.lin_splits : 1);
    const int grid = std::min(tiles, num_sms);
    PPV_PDL_OK(launch_pdl(gemm_wgmma_kernel<BN, NSPLIT, BK>, dim3(grid), dim3(GEMM_THREADS), Cfg::SMEM_BYTES, stream, gp),
               "gemm_wgmma_kernel");
    return PPV_OK;
}

template <int BN>
static int launch_bn(const GemmParams& gp, bool x3, int num_sms, cudaStream_t stream) {
    if (gp.bk == 32) return x3 ? launch_one<BN, 3, 32>(gp, num_sms, stream) : launch_one<BN, 1, 32>(gp, num_sms, stream);
    return x3 ? launch_one<BN, 3, 64>(gp, num_sms, stream) : launch_one<BN, 1, 64>(gp, num_sms, stream);
}

// Prints the stamps of the last traced launch in cycles from the kernel start, one line per role and tile, with the phases they give:
// wait = hand-off passed -> first `full` passed, kloop = first `full` -> wgmma_wait<0> returned, epi = epilogue start -> end,
// period = this tile's epilogue end - the previous tile's of the same warpgroup.  The producer lines give, for k-steps 0-2 and
// nk-3..nk-1, when its ring-slot wait passed and when the TMA loads were issued; the MMA lines when the consumer released those
// k-steps' slots (`empty` arrival).
void gemm_trace_dump(const GemmParams& gp) {
    if (!gp.trace) return;
    constexpr int E = GEMM_TRACE_EVENTS;
    unsigned long long h[3 * GEMM_TRACE_TILES * E];
    cudaDeviceSynchronize();
    cudaMemcpy(h, gp.trace, sizeof(h), cudaMemcpyDeviceToHost);
    const unsigned long long t0 = h[7];
    auto at = [&](int r, int i, int e) -> long long { const unsigned long long v = h[(r * GEMM_TRACE_TILES + i) * E + e]; return v ? (long long)(v - t0) : -1ll; };
    printf("gemm trace M=%d N=%d nk=%d BN=%d CTA %d (cycles from kernel start)\n", gp.M, gp.N, gp.num_ksteps, gp.bn, gp.trace_cta);
    for (int i = 0; i < GEMM_TRACE_TILES; ++i) {
        if (at(0, i, 0) < 0) continue;
        printf("gemm trace tma  tile %2d: slot passed / loads issued, k-steps 0-2 and last 3:", i);
        for (int e = 0; e < 6; ++e) printf(" %lld/%lld", at(0, i, e), at(0, i, 8 + e));
        printf("\n");
    }
    for (int r = 1; r < 3; ++r) {
        long long prev_end = -1;
        for (int i = 0; i < GEMM_TRACE_TILES; ++i) {
            if (at(r, i, 0) < 0) continue;
            printf("gemm trace wg%d  tile %2d:", r - 1, i);
            for (int e = 0; e < 6; ++e) printf(" %8lld", at(r, i, e));
            printf("   wait %6lld  kloop %6lld  epi %6lld  period %6lld   released", at(r, i, 1) - at(r, i, 0), at(r, i, 3) - at(r, i, 1),
                   at(r, i, 5) - at(r, i, 4), prev_end >= 0 ? at(r, i, 5) - prev_end : -1ll);
            for (int e = 6; e < 12; ++e) printf(" %lld", at(r, i, e));
            printf("\n");
            prev_end = at(r, i, 5);
        }
    }
    fflush(stdout);
}

int gemm_launch(const GemmParams& gp, int precision, int num_sms, cudaStream_t stream) {
    const bool x3 = (precision == PPV_PREC_BF16X3);
    switch (gp.bn) {
        case 64: return launch_bn<64>(gp, x3, num_sms, stream);
        case 128: return launch_bn<128>(gp, x3, num_sms, stream);
        case 256: return launch_bn<256>(gp, x3, num_sms, stream);
    }
    return fail(PPV_EINVAL, "gemm_launch: bad BN");
}

}  // namespace ppv
