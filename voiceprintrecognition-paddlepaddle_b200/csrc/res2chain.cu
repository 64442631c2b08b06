// The whole Res2Net chain of one SE-Res2Net block in ONE kernel: y_1 = f_1(x_1), y_j = f_j(x_j + y_{j-1}), j = 2..7, with
// f_j = BN(ReLU(conv_k3,d(.))) on 64-channel chunks (ppvector/models/ecapa_tdnn.py:36-47, TDNNBlock utils.py:147).
//
// The seven convs are strictly sequential, and as seven launches each one costs a full kernel latency.  Here one CTA owns one
// UTTERANCE: its whole padded time axis (<= 384 rows x 64 channels, split-bf16) lives in shared memory in the SWIZZLE_128B
// layout the wgmma descriptors read, so
//   * conv taps are descriptor row offsets into that resident tile (as in res2conv.cu),
//   * the epilogue of conv j writes BN(ReLU(.)) to HBM once (the tdnn2 GEMM reads it) and writes x_{j+1} + y_j -- including
//     the reflect-padding halo rows -- straight back into the shared-memory tile as the A operand of conv j+1:
//     the intermediate sums never touch HBM and there is no inter-CTA dependency at all,
//   * the 48 KB of weights of conv j+1 stream into the weight slot by TMA while the epilogue of conv j runs.
// Warp roles: warp 0 TMA, warp 3 TMA store, warps 4-15 three MMA warpgroups (512 threads): warpgroup t owns the 128-row
// output tile t of the utterance (two m64 x n64 register accumulators) and runs its epilogue.
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include "common.h"
#include "gemm_epilogue.cuh"
#include "ptx.cuh"

namespace ppv {

constexpr int RC_PAD = 4;                       // rows loaded above the utterance (max dilation)
constexpr int RC_BOX_ROWS = 200;                // TMA box rows (<= 256); 200 * 128 B is a multiple of 1024
constexpr int RC_ROWS = 2 * RC_BOX_ROWS;        // 400 >= 4 + 384 + 4
constexpr int RC_A_PLANE = RC_ROWS * 128;       // 51200 B per plane
constexpr int RC_W_TILE = 64 * 128;             // [64 out ch x 64 k] bf16
constexpr int RC_MAX_TILES = 3;                 // 128-row output tiles per utterance
constexpr int RC_MAX_TP = RC_MAX_TILES * GEMM_BM;  // 384
constexpr int RC_S_PLANE = GEMM_BM * 128;       // staging tile: 128 rows x 64 channels bf16, SWIZZLE_128B
constexpr int RC_MMA_THREADS = 128 * RC_MAX_TILES;  // one MMA warpgroup per 128-row tile
constexpr int RC_THREADS = 128 + RC_MMA_THREADS;

template <int NSPLIT>
struct RCCfg {
    static constexpr int NP = (NSPLIT == 3) ? 2 : 1;
    static constexpr int A_BYTES = NP * RC_A_PLANE;
    static constexpr int W_SLOT = 3 * NP * RC_W_TILE;  // 3 taps x planes, single slot: the next conv's weights load under the epilogue
    static constexpr int S_BYTES = NP * RC_S_PLANE;    // one staging tile (hi, lo)
    static constexpr int SMEM_BYTES = 1024 + A_BYTES + W_SLOT + 2 * S_BYTES + 256;
};

// Predicated stores, in program order (volatile asm is not reordered): with branches around plain stores the scheduler computes
// many columns ahead of their stores and runs out of registers.
__device__ __forceinline__ void rp_st_shared(bool pred, uint32_t a, uint32_t v) {
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %2, 0;\n\t@p st.shared.u32 [%0], %1;\n\t}" ::"r"(a), "r"(v), "r"(uint32_t(pred)) : "memory");
}
// 16-byte variants for the paired kernel's epilogue (8 bf16 columns of one row and plane)
__device__ __forceinline__ void rp_st_global_v4(bool pred, const void* p, uint4 v) {
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %5, 0;\n\t@p st.global.v4.u32 [%0], {%1, %2, %3, %4};\n\t}" ::"l"(p), "r"(v.x), "r"(v.y),
                 "r"(v.z), "r"(v.w), "r"(uint32_t(pred))
                 : "memory");
}
__device__ __forceinline__ void rp_st_shared_v4(bool pred, uint32_t a, uint4 v) {
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %5, 0;\n\t@p st.shared.v4.u32 [%0], {%1, %2, %3, %4};\n\t}" ::"r"(a), "r"(v.x), "r"(v.y),
                 "r"(v.z), "r"(v.w), "r"(uint32_t(pred))
                 : "memory");
}
__device__ __forceinline__ uint4 rp_ld_shared_v4(uint32_t a) {
    uint4 v;
    asm volatile("ld.shared.v4.u32 {%0, %1, %2, %3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "r"(a) : "memory");
    return v;
}

__device__ __forceinline__ uint32_t rc_ld_shared(uint32_t a) {
    uint32_t v;
    asm volatile("ld.shared.u32 %0, [%1];" : "=r"(v) : "r"(a) : "memory");
    return v;
}

#define RC_STAMP(role, conv, ev)                                                                   \
    do {                                                                                          \
        if (cp.trace && blockIdx.x == 0 && b == 0) cp.trace[((role) * 8 + (conv)) * 8 + (ev)] = clock64(); \
    } while (0)

// Per (conv, tile) a 32 KB staging tile S carries both directions of HBM traffic through TMA: the producer loads the slice
// of the NEXT chunk x_{j+2} into it, the epilogue reads its values from it and overwrites them with y_{j+1}, and warp 3
// stores the tile to HBM.  Two staging tiles serve the (up to) three output tiles of a conv: tiles 0 and 1 run their epilogues
// together, tile 2 after them.
template <int NSPLIT>
__global__ void __launch_bounds__(RC_THREADS, 1) res2chain_kernel(const __grid_constant__ Res2ChainParams cp) {
    using Cfg = RCCfg<NSPLIT>;
    constexpr int NP = Cfg::NP, BN = 64;
    extern __shared__ uint8_t smem_raw[];
    const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;
    uint8_t* smem_gen = smem_raw + (smem_base - smem_u32(smem_raw));
    const uint32_t a_base = smem_base;
    const uint32_t w_base = a_base + Cfg::A_BYTES;
    const uint32_t s_base = w_base + Cfg::W_SLOT;
    const uint32_t bar_base = s_base + 2 * Cfg::S_BYTES;
    const uint32_t x_full = bar_base, x_free = bar_base + 24, w_full = bar_base + 32, w_empty = bar_base + 40;
    auto s_full = [&](int i) { return bar_base + 48u + 8u * i; };
    auto s_empty = [&](int i) { return bar_base + 64u + 8u * i; };
    auto y_ready = [&](int i) { return bar_base + 80u + 8u * i; };

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    if (warp == 0 && lane == 0) {
        prefetch_tmap(&cp.mapX);
        prefetch_tmap(&cp.mapXt);
        prefetch_tmap(&cp.mapY);
        prefetch_tmap(&cp.mapYtail);
        for (int j = 0; j < cp.nconv; ++j) prefetch_tmap(&cp.mapW[j]);
    }
    if (warp == 1 && lane == 0) {
        mbar_init(x_full, 1);
        mbar_init(x_free, 1);
        mbar_init(w_full, 1);
        mbar_init(w_empty, 1);
        for (int i = 0; i < 2; ++i) {
            mbar_init(s_full(i), 1);
            mbar_init(s_empty(i), 1);
            mbar_init(y_ready(i), 128);  // the warpgroup of the tile
        }
        fence_mbar_init();
    }
    __syncthreads();
    griddep_launch_dependents();
    const int nconv = cp.nconv, ntiles = cp.ntiles;

    if (warp == 0) {
        // ===================== TMA producer =====================
        if (lane == 0) {
            griddep_wait();  // x comes from the previous kernel
            int g = 0, u = 0;
            uint32_t sn = 0;  // running staging-tile index (buffer = sn & 1)
            for (int b = blockIdx.x; b < cp.B; b += gridDim.x, ++u) {
                if (u > 0) mbar_wait(x_free, uint32_t(u - 1) & 1u);  // the last conv of the previous utterance has read the tile
                mbar_arrive_expect_tx(x_full, NP * 2 * RC_BOX_ROWS * 128);
                for (int pl = 0; pl < NP; ++pl)
                    for (int h = 0; h < 2; ++h)
                        tma_load_3d(a_base + pl * RC_A_PLANE + h * RC_BOX_ROWS * 128, &cp.mapX, x_full, cp.width /* chunk 1 */,
                                    b * cp.Tp - RC_PAD + h * RC_BOX_ROWS, pl);
                for (int j = 0; j < nconv; ++j, ++g) {
                    if (g > 0) mbar_wait(w_empty, uint32_t(g - 1) & 1u);
                    RC_STAMP(0, j, 0);
                    mbar_arrive_expect_tx(w_full, 3 * NP * RC_W_TILE);
                    for (int tap = 0; tap < 3; ++tap)
                        for (int pl = 0; pl < NP; ++pl) tma_load_3d(w_base + (tap * NP + pl) * RC_W_TILE, &cp.mapW[j], w_full, tap * 64, 0, pl);
                    for (int t = 0; t < ntiles; ++t, ++sn) {
                        const int i = sn & 1;
                        if (sn >= 2) mbar_wait(s_empty(i), ((sn >> 1) - 1) & 1u);  // the store of its previous use has read the tile
                        if (j + 1 < nconv) {  // slice of chunk j+2 that the epilogue adds to y_{j+1}
                            mbar_arrive_expect_tx(s_full(i), NP * RC_S_PLANE);
                            for (int pl = 0; pl < NP; ++pl)
                                tma_load_3d(s_base + i * Cfg::S_BYTES + pl * RC_S_PLANE, &cp.mapXt, s_full(i), (j + 2) * cp.width,
                                            b * cp.Tp + t * GEMM_BM, pl);
                        } else {
                            mbar_arrive(s_full(i));  // nothing to add after the last conv; the tile is used for the store only
                        }
                    }
                }
            }
        }
    } else if (warp == 3) {
        // ===================== store warp: staging tile -> HBM =====================
        if (lane == 0) {
            uint32_t sn = 0;
            for (int b = blockIdx.x; b < cp.B; b += gridDim.x) {
                for (int j = 0; j < nconv; ++j) {
                    for (int t = 0; t < ntiles; ++t, ++sn) {
                        const int i = sn & 1;
                        mbar_wait(y_ready(i), (sn >> 1) & 1u);  // all epilogue threads have written (and fenced) their part of the tile
                        const CUtensorMap* my = (t == ntiles - 1) ? &cp.mapYtail : &cp.mapY;  // never store beyond this utterance's rows
                        for (int pl = 0; pl < NP; ++pl)
                            tma_store_3d(my, s_base + i * Cfg::S_BYTES + pl * RC_S_PLANE, (j + 1) * cp.width, b * cp.Tp + t * GEMM_BM, pl);
                        bulk_commit_group();
                        bulk_wait_read0();
                        mbar_arrive(s_empty(i));
                    }
                }
            }
            bulk_wait_all();
        }
    } else if (warp >= 4) {
        // ===================== MMA + epilogue: warpgroup tw owns output tile tw of the utterance =====================
        const int tw = (warp - 4) >> 2, tid = threadIdx.x & 127, w = tid >> 5, l = tid & 31;
        const int e = threadIdx.x - 128;  // 0 .. RC_MMA_THREADS - 1
        const bool has_tile = tw < ntiles;
        griddep_wait();
        uint8_t* const a_gen = smem_gen;  // a_base == smem_base
        float acc0[BN / 2], acc1[BN / 2];
#pragma unroll
        for (int i = 0; i < BN / 2; ++i) acc0[i] = acc1[i] = 0.f;
        uint32_t g = 0, ucount = 0;
        for (int b = blockIdx.x; b < cp.B; b += gridDim.x, ++ucount) {
            {
                // The producing GEMM stores valid frames only: build the reflect halo rows of the resident tile here --
                // 2 P rows x 8 chunks x planes, one 16-byte copy per thread, in the swizzled layout.
                mbar_wait(x_full, ucount & 1u);
                if (e < 2 * cp.P * 8 * NP) {
                    const int pl = e / (2 * cp.P * 8), r = (e / 8) % (2 * cp.P), c = e % 8;
                    const int k = (r % cp.P) + 1;
                    const int dst = (r < cp.P ? cp.P - k : cp.P + cp.T - 1 + k) + RC_PAD, src = (r < cp.P ? cp.P + k : cp.P + cp.T - 1 - k) + RC_PAD;
                    const uint4 val = *reinterpret_cast<const uint4*>(a_gen + pl * RC_A_PLANE + src * 128 + ((c ^ (src & 7)) << 4));
                    *reinterpret_cast<uint4*>(a_gen + pl * RC_A_PLANE + dst * 128 + ((c ^ (dst & 7)) << 4)) = val;
                }
                fence_proxy_async_smem();
                named_bar_sync(1, RC_MMA_THREADS);
            }
            for (int j = 0; j < nconv; ++j, ++g) {
                mbar_wait(w_full, g & 1u);
                if (tid == 0 && tw == 0) RC_STAMP(1, j, 1);  // weights ready
                if (has_tile) {
                    wgmma_fence_acc(acc0);
                    wgmma_fence_acc(acc1);
                    wgmma_fence();
                    auto issue = [&](float (&acc)[BN / 2], int mb) {
#pragma unroll
                        for (int tap = 0; tap < 3; ++tap) {
                            const uint32_t roff = uint32_t(tw * GEMM_BM + mb * 64 + RC_PAD + (tap - 1) * cp.dil);
                            const uint64_t a_hi = make_sw128_kmajor_desc(a_base + roff * 128u);
                            const uint64_t b_hi = make_sw128_kmajor_desc(w_base + (tap * NP) * RC_W_TILE);
#pragma unroll
                            for (int k = 0; k < 4; ++k) wgmma_bf16<BN>(acc, a_hi + 2 * k, b_hi + 2 * k, (tap > 0 || k > 0) ? 1u : 0u);
                            if (NSPLIT == 3) {
                                const uint64_t a_lo = make_sw128_kmajor_desc(a_base + RC_A_PLANE + roff * 128u);
                                const uint64_t b_lo = make_sw128_kmajor_desc(w_base + (tap * NP + 1) * RC_W_TILE);
#pragma unroll
                                for (int k = 0; k < 4; ++k) wgmma_bf16<BN>(acc, a_lo + 2 * k, b_hi + 2 * k, 1u);
#pragma unroll
                                for (int k = 0; k < 4; ++k) wgmma_bf16<BN>(acc, a_hi + 2 * k, b_lo + 2 * k, 1u);
                            }
                        }
                    };
                    issue(acc0, 0);
                    issue(acc1, 1);
                    wgmma_commit();
                    wgmma_wait<0>();
                    wgmma_fence_acc(acc0);
                    wgmma_fence_acc(acc1);
                }
                // every MMA of this conv has read the operand tile and the weights: both may be overwritten now
                named_bar_sync(1, RC_MMA_THREADS);
                if (e == 0) {
                    RC_STAMP(1, j, 2);
                    mbar_arrive(w_empty);
                    if (j == nconv - 1) mbar_arrive(x_free);
                }
                const float* bias = cp.bias[j];
                const float* bsc = cp.bn_scale[j];
                const float* bsh = cp.bn_shift[j];
                const bool has_next = j + 1 < nconv;
                const uint32_t sn = g * uint32_t(ntiles) + uint32_t(tw);
                const int i = sn & 1;
                // One row per trip of a loop that is not unrolled (acc indexed by selects), the mirror rows as scalars and the
                // shared-memory stores predicated in program order: unrolled, the compiler computes values far ahead of their
                // stores and spills.
                auto epilogue = [&](const float (&acc)[BN / 2], int mb) {
#pragma unroll 1
                    for (int h = 0; h < 2; ++h) {
                        const int rloc = mb * 64 + 16 * w + (l >> 2) + 8 * h;  // row inside the 128-row tile
                        const int p = tw * GEMM_BM + rloc;                      // padded row inside the utterance
                        const int tt = p - cp.P, uu = cp.T - 1 - tt;
                        const bool next = has_next && tt >= 0 && tt < cp.T;
                        const int m0 = p + RC_PAD;
                        const int m1 = (tt >= 1 && tt <= cp.P) ? cp.P - tt + RC_PAD : -1;
                        const int m2 = (uu >= 1 && uu <= cp.P) ? cp.P + cp.T - 1 + uu + RC_PAD : -1;
                        const uint32_t srow = s_base + i * Cfg::S_BYTES + rloc * 128 + 4 * (l & 3);
#pragma unroll
                        for (int q = 0; q < BN / 8; ++q) {
                            const int col = 8 * q + 2 * (l & 3);
                            const uint32_t so = srow + ((q ^ (rloc & 7)) << 4);  // SWIZZLE_128B: 16-byte chunk q of the row
                            // bias -> ReLU -> BatchNorm(eval) affine   (TDNNBlock, utils.py:147)
                            const float2 b2 = __ldg(reinterpret_cast<const float2*>(bias + col));
                            const float2 s2 = __ldg(reinterpret_cast<const float2*>(bsc + col));
                            const float2 h2 = __ldg(reinterpret_cast<const float2*>(bsh + col));
                            const float a0 = h ? acc[4 * q + 2] : acc[4 * q], a1 = h ? acc[4 * q + 3] : acc[4 * q + 1];
                            const float x0 = fmaf(fmaxf(a0 + b2.x, 0.f), s2.x, h2.x);
                            const float x1 = fmaf(fmaxf(a1 + b2.y, 0.f), s2.y, h2.y);
                            uint32_t nh = 0, nl = 0;
                            if (has_next) {
                                nh = rc_ld_shared(so);
                                if (NP == 2) nl = rc_ld_shared(so + RC_S_PLANE);
                            }
                            uint32_t yh, yl;  // y_{j+1} -> staging tile (every row: rows outside the valid frames are halo / padding rows of y)
                            split_pack_bf16x2(x0, x1, yh, yl);
                            rp_st_shared(true, so, yh);
                            if (NP == 2) rp_st_shared(true, so + RC_S_PLANE, yl);
                            // x_{j+2} + y_{j+1} -> operand of the next conv, in place, with its reflect halo rows
                            const float2 hf = unpack_bf16x2(nh), lf = unpack_bf16x2(nl);
                            uint32_t oh, ol;
                            split_pack_bf16x2(x0 + (hf.x + lf.x), x1 + (hf.y + lf.y), oh, ol);
                            auto put = [&](bool pred, int row) {
                                const uint32_t d = a_base + row * 128 + ((q ^ (row & 7)) << 4) + 4 * (l & 3);
                                rp_st_shared(pred, d, oh);
                                if (NP == 2) rp_st_shared(pred, d + RC_A_PLANE, ol);
                            };
                            put(next, m0);
                            put(next && m1 >= 0, m1);
                            put(next && m2 >= 0, m2);
                        }
                    }
                };
                // tiles 0 and 1 use the two staging tiles, tile 2 reuses the first one after them
#pragma unroll 1
                for (int round = 0; round < 2; ++round) {
                    if (has_tile && (tw == 2) == (round == 1)) {
                        mbar_wait(s_full(i), (sn >> 1) & 1u);
                        epilogue(acc0, 0);
                        epilogue(acc1, 1);
                        fence_proxy_async_smem();
                        mbar_arrive(y_ready(i));
                    }
                    if (ntiles > 2 && round == 0) named_bar_sync(2, RC_MMA_THREADS);
                }
                if (tid == 0 && tw == 0) RC_STAMP(2, j, 5);  // all tiles written back
                if (has_next) {
                    fence_proxy_async_smem();  // generic-proxy writes -> visible to the tensor core's async-proxy reads
                    named_bar_sync(1, RC_MMA_THREADS);
                }
            }
        }
    }
}

// ---------------------------------------------------------------------------------------------------------------------------
// Paired variant (Tp <= 320): one CTA holds TWO utterances, A and B, resident in shared memory and alternates them through the
// convs, so that the MMAs of one utterance run on the tensor cores while the warps run the epilogue of the other:
//   MMA_A(j) | epilogue_B(j-1)  ->  MMA_B(j) | epilogue_A(j)  ->  W[j+1] lands  ->  MMA_A(j+1) | epilogue_B(j)  -> ...
// B = 256 utterances are 128 CTAs, one wave.  Five MMA warpgroups (640 threads, 96 registers each): warpgroup w owns the
// m64 row block w of BOTH utterances, one 64 x 64 accumulator per utterance.  The operands (2 x 336 rows x planes) and one
// conv's weights (shared by both utterances) leave no room for staging tiles.  Instead, once every MMA of conv j of an
// utterance has retired, its operand tile is dead, and thread 0 loads chunk x_{j+2} into that tile by TMA (prefetched into L2
// when conv j-1 starts).  The epilogue writes y_{j+1} to HBM straight from the registers, then waits for x_{j+2} and overwrites
// the tile in place with x_{j+2} + y_{j+1}.  Both use 16-byte accesses after a transpose inside each quad of lanes.  Per row, the
// MMA order, the epilogue formulas and the reflect halo rows are those of the one-utterance kernel above, so the outputs are
// bitwise equal to its outputs.
constexpr int RP_BLOCKS = 5;                          // m64 row blocks per utterance, one per MMA warpgroup
constexpr int RP_MAX_TP = RP_BLOCKS * 64;             // 320
constexpr int RP_BOX_ROWS = 168;                      // two boxes: 336 >= 4 + 320 + 4 rows; 168 * 128 B is a multiple of 1024
constexpr int RP_A_PLANE = 2 * RP_BOX_ROWS * 128;     // 43008 B per plane
constexpr int RP_THREADS = 128 * RP_BLOCKS;           // 640
constexpr int RP_VEC_FLOATS = 3 * RES2CHAIN_MAX * 64;  // bias, BN scale, BN shift of every conv

template <int NSPLIT>
struct RPCfg {
    static constexpr int NP = (NSPLIT == 3) ? 2 : 1;
    static constexpr int U_BYTES = NP * RP_A_PLANE;     // one utterance's operand tile
    static constexpr int W_SLOT = 3 * NP * RC_W_TILE;   // 3 taps x planes of one conv
    static constexpr int SMEM_BYTES = 1024 + 2 * U_BYTES + W_SLOT + RP_VEC_FLOATS * 4 + 64;
};
static_assert(RPCfg<3>::SMEM_BYTES <= 232448, "paired res2chain exceeds the H100 shared-memory opt-in");

// trace (PPV_RES2_TRACE) of CTA 0's first pair: role 0 / 1 = utterance A / B, events 0 MMA issued, 1 MMA retired (every
// warpgroup), 2 epilogue start, 3 epilogue end, 4 x_{j+2} load issued, 5 y_{j+1} stores done, 6 x_{j+2} barrier passed
// (thread 0); role 2 = weights, events 0 load issued, 1 landed
#define RP_STAMP(role, conv, ev)                                                                                \
    do {                                                                                                        \
        if (trace_on) cp.trace[((role) * 8 + (conv)) * 8 + (ev)] = clock64();                                   \
    } while (0)

// An opaque copy: what is computed from it stays inside the loop that computes it.  Without it the compiler hoists the operand
// descriptors and the row addresses of both utterances out of the conv loop and spills them.
__device__ __forceinline__ int rp_opaque(int v) {
    asm volatile("mov.b32 %0, %0;" : "+r"(v));
    return v;
}

template <int NSPLIT>
__global__ void __launch_bounds__(RP_THREADS, 1) res2chain_pair_kernel(const __grid_constant__ Res2ChainParams cp) {
    using Cfg = RPCfg<NSPLIT>;
    constexpr int NP = Cfg::NP, BN = 64;
    extern __shared__ uint8_t smem_raw[];
    const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;
    uint8_t* const a_gen = smem_raw + (smem_base - smem_u32(smem_raw));  // utterance u's tile at u * U_BYTES, plane pl at + pl * RP_A_PLANE
    const uint32_t w_base = smem_base + 2 * Cfg::U_BYTES;
    float* const vec = reinterpret_cast<float*>(a_gen + 2 * Cfg::U_BYTES + Cfg::W_SLOT);  // [conv][bias, scale, shift][64]
    const uint32_t bar_base = w_base + Cfg::W_SLOT + RP_VEC_FLOATS * 4;
    const uint32_t x_full = bar_base, w_full = bar_base + 8;
    auto x_next = [&](int u) { return bar_base + 16u + 8u * u; };  // x_{j+2} of utterance u has landed in its tile

    const int tid = threadIdx.x, wg = tid >> 7, wq = (tid >> 5) & 3, l = tid & 31;
    const int nconv = cp.nconv, T = cp.T, P = cp.P, Tp = cp.Tp;
    if (tid == 0) {
        prefetch_tmap(&cp.mapX);
        for (int j = 0; j < nconv; ++j) prefetch_tmap(&cp.mapW[j]);
        mbar_init(x_full, 1);
        mbar_init(w_full, 1);
        mbar_init(x_next(0), 1);
        mbar_init(x_next(1), 1);
        fence_mbar_init();
    }
    __syncthreads();
    griddep_launch_dependents();
    griddep_wait();  // x comes from the previous kernel
    for (int i = tid; i < 3 * 64 * nconv; i += RP_THREADS) {
        const int j = i / 192, k = (i / 64) % 3, c = i % 64;
        vec[i] = (k == 0 ? cp.bias[j] : k == 1 ? cp.bn_scale[j] : cp.bn_shift[j])[c];
    }

    auto load_w = [&](int j) {
        mbar_arrive_expect_tx(w_full, 3 * NP * RC_W_TILE);
        for (int tap = 0; tap < 3; ++tap)
            for (int pl = 0; pl < NP; ++pl) tma_load_3d(w_base + (tap * NP + pl) * RC_W_TILE, &cp.mapW[j], w_full, tap * 64, 0, pl);
    };
    // chunk c of utterance b -> slot u's operand tile: rows [-4, 332) around the utterance in two boxes, completing on `bar`.
    // Rows past the end of the batch are filled with zeros by TMA.
    auto load_x = [&](uint32_t bar, int u, int b, int c) {
        for (int pl = 0; pl < NP; ++pl)
            for (int h = 0; h < 2; ++h)
                tma_load_3d(smem_base + u * Cfg::U_BYTES + pl * RP_A_PLANE + h * RP_BOX_ROWS * 128, &cp.mapX, bar, c * cp.width,
                            b * Tp - RC_PAD + h * RP_BOX_ROWS, pl);
    };
    // x_{c} (c = chunk) of both utterances of the pair -> L2, where load_x of x_{c} one conv later finds it
    auto prefetch_chunk = [&](int b0, int c) {
        for (int u = 0; u < 2 && b0 + u < cp.B; ++u)
            for (int pl = 0; pl < NP; ++pl)
                for (int h = 0; h < 2; ++h) tma_prefetch_l2_3d(&cp.mapX, c * cp.width, (b0 + u) * Tp - RC_PAD + h * RP_BOX_ROWS, pl);
    };
    // D(64 x 64) of row block wg of utterance u, conv taps in the one-utterance kernel's order
    auto issue = [&](float (&acc)[BN / 2], int u) {
        wgmma_fence_acc(acc);
        wgmma_fence();
#pragma unroll
        for (int tap = 0; tap < 3; ++tap) {
            const uint32_t a_row = smem_base + rp_opaque(u * Cfg::U_BYTES) + uint32_t(wg * 64 + RC_PAD + (tap - 1) * cp.dil) * 128u;
            const uint64_t a_hi = make_sw128_kmajor_desc(a_row);
            const uint64_t b_hi = make_sw128_kmajor_desc(w_base + (tap * NP) * RC_W_TILE);
#pragma unroll
            for (int k = 0; k < 4; ++k) wgmma_bf16<BN>(acc, a_hi + 2 * k, b_hi + 2 * k, (tap > 0 || k > 0) ? 1u : 0u);
            if (NSPLIT == 3) {
                const uint64_t a_lo = make_sw128_kmajor_desc(a_row + RP_A_PLANE);
                const uint64_t b_lo = make_sw128_kmajor_desc(w_base + (tap * NP + 1) * RC_W_TILE);
#pragma unroll
                for (int k = 0; k < 4; ++k) wgmma_bf16<BN>(acc, a_lo + 2 * k, b_hi + 2 * k, 1u);
#pragma unroll
                for (int k = 0; k < 4; ++k) wgmma_bf16<BN>(acc, a_hi + 2 * k, b_lo + 2 * k, 1u);
            }
        }
        wgmma_commit();
    };
    // conv j of utterance b (slot u): y_{j+1} -> HBM on rows [0, Tp); then, once x_{j+2} has landed in the operand tile (load_x
    // on x_next(u), completion `xpar`), x_{j+2} + y_{j+1} -> the tile in place on the valid rows and their reflect mirrors.  The
    // load also overwrote the halo rows [0, P) and [P + T, Tp), which the mirrors rewrite, and the rows outside [0, Tp), which only
    // feed halo rows of y (discarded by tdnn2).  An absent utterance (odd B) stores nothing and waits for nothing.
    // After quad_transpose_pairs lane q holds columns 32 c + 8 q + [0, 8) of its two rows in half c: one 16-byte access per row,
    // half and plane.  acc is consumed: pass 1 leaves the BN outputs of half c, row h in acc[16 c + 8 h + k] for pass 2.
    bool trace_on = false;
    auto epilogue = [&](float (&acc)[BN / 2], int u, int b, int j, uint32_t xpar) {
        b = rp_opaque(b);
        const bool present = b < cp.B, has_next = j + 1 < nconv;
        j = rp_opaque(j);  // like b: the y column offset is computed here, not before the epilogue and held through it
        const int q = l & 3, r0 = wg * 64 + 16 * wq + (l >> 2);  // padded rows r0 and r0 + 8 inside the utterance
#pragma unroll
        for (int c = 0; c < 2; ++c) {
            float a[8], bb[8];
#pragma unroll
            for (int i = 0; i < 4; ++i)
                a[2 * i] = acc[16 * c + 4 * i], a[2 * i + 1] = acc[16 * c + 4 * i + 1], bb[2 * i] = acc[16 * c + 4 * i + 2],
                bb[2 * i + 1] = acc[16 * c + 4 * i + 3];
            quad_transpose_pairs(a, bb, q);
            // bias -> ReLU -> BatchNorm(eval) affine   (TDNNBlock, utils.py:147)
            const float* const vb = vec + j * 192 + 32 * c + 8 * q;
#pragma unroll
            for (int k4 = 0; k4 < 8; k4 += 4) {
                const float4 b4 = *reinterpret_cast<const float4*>(vb + k4);
                const float4 s4 = *reinterpret_cast<const float4*>(vb + 64 + k4);
                const float4 h4 = *reinterpret_cast<const float4*>(vb + 128 + k4);
                const float bv[4] = {b4.x, b4.y, b4.z, b4.w}, sv[4] = {s4.x, s4.y, s4.z, s4.w}, hv[4] = {h4.x, h4.y, h4.z, h4.w};
#pragma unroll
                for (int k = 0; k < 4; ++k) {
                    acc[16 * c + k4 + k] = fmaf(fmaxf(a[k4 + k] + bv[k], 0.f), sv[k], hv[k]);
                    acc[16 * c + 8 + k4 + k] = fmaf(fmaxf(bb[k4 + k] + bv[k], 0.f), sv[k], hv[k]);
                }
            }
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const float* const v = acc + 16 * c + 8 * h;
                const int r = r0 + 8 * h;
                const __nv_bfloat16* const yp = cp.y.hi() + (int64_t(b) * Tp + r) * cp.y.ld + (j + 1) * cp.width + 32 * c + 8 * q;
                uint4 vh, vl;
                split_pack_bf16x2(v[0], v[1], vh.x, vl.x), split_pack_bf16x2(v[2], v[3], vh.y, vl.y);
                split_pack_bf16x2(v[4], v[5], vh.z, vl.z), split_pack_bf16x2(v[6], v[7], vh.w, vl.w);
                rp_st_global_v4(present && r < Tp, yp, vh);
                if (NP == 2) rp_st_global_v4(present && r < Tp, yp + cp.y.plane_stride, vl);
            }
        }
        RP_STAMP(u, j, 5);
        if (!(present && has_next)) return;  // uniform across the CTA
        mbar_wait(x_next(u), xpar);
        RP_STAMP(u, j, 6);
        const uint32_t tile = smem_base + u * Cfg::U_BYTES;
        const int r1 = rp_opaque(r0);  // the row arithmetic below stays after the wait instead of holding registers through pass 1
#pragma unroll
        for (int c = 0; c < 2; ++c) {
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int r = r1 + 8 * h, tt = r - P, uu = T - 1 - tt;
                const bool next = tt >= 0 && tt < T;
                const int m0 = r + RC_PAD;
                const int m1 = (tt >= 1 && tt <= P) ? P - tt + RC_PAD : -1;
                const int m2 = (uu >= 1 && uu <= P) ? P + T - 1 + uu + RC_PAD : -1;
                const int k16 = 4 * c + q;  // SWIZZLE_128B: 16-byte unit k16 of row m sits at m * 128 + ((k16 ^ (m & 7)) << 4)
                const uint32_t s0 = tile + m0 * 128 + ((k16 ^ (m0 & 7)) << 4);
                const uint4 xh = rp_ld_shared_v4(s0);
                const uint4 xl = NP == 2 ? rp_ld_shared_v4(s0 + RP_A_PLANE) : make_uint4(0u, 0u, 0u, 0u);
                const float* const v = acc + 16 * c + 8 * h;
                uint4 oh, ol;
                auto add = [&](uint32_t nh, uint32_t nl, int k, uint32_t& ph, uint32_t& pl) {
                    const float2 hf = unpack_bf16x2(nh), lf = unpack_bf16x2(nl);
                    split_pack_bf16x2(v[k] + (hf.x + lf.x), v[k + 1] + (hf.y + lf.y), ph, pl);
                };
                add(xh.x, xl.x, 0, oh.x, ol.x), add(xh.y, xl.y, 2, oh.y, ol.y), add(xh.z, xl.z, 4, oh.z, ol.z), add(xh.w, xl.w, 6, oh.w, ol.w);
                auto put = [&](bool pred, int row) {
                    const uint32_t d = tile + row * 128 + ((k16 ^ (row & 7)) << 4);
                    rp_st_shared_v4(pred, d, oh);
                    if (NP == 2) rp_st_shared_v4(pred, d + RP_A_PLANE, ol);
                };
                put(next, m0);
                put(next && m1 >= 0, m1);
                put(next && m2 >= 0, m2);
            }
        }
    };

    float accA[BN / 2], accB[BN / 2];
#pragma unroll
    for (int i = 0; i < BN / 2; ++i) accA[i] = accB[i] = 0.f;
    const int npairs = (cp.B + 1) / 2;
    uint32_t g = 0, it = 0;
    for (int pi = blockIdx.x; pi < npairs; pi += gridDim.x, ++it) {
        const int b0 = 2 * pi;  // utterances b0 (A) and b0 + 1 (B, absent when B is odd and this is the last pair)
        trace_on = cp.trace && blockIdx.x == 0 && it == 0 && tid == 0;
        if (tid == 0) {
            // chunk 1 of both utterances; an absent B loads out-of-range rows, which TMA fills with zeros
            mbar_arrive_expect_tx(x_full, 2 * NP * RP_A_PLANE);
            for (int u = 0; u < 2; ++u) load_x(x_full, u, b0 + u, 1);
            RP_STAMP(2, 0, 0);
            load_w(0);
            for (int c = 2; c <= 3 && c <= nconv; ++c) prefetch_chunk(b0, c);
        }
        {
            // The producing GEMM stores valid frames only: build the reflect halo rows of both resident tiles here --
            // 2 utterances x 2 P rows x 8 chunks x planes, one 16-byte copy per thread, in the swizzled layout.
            mbar_wait(x_full, it & 1u);
            const int per_u = 2 * P * 8 * NP;
            if (tid < 2 * per_u) {
                const int u = tid / per_u, e = tid % per_u;
                const int pl = e / (2 * P * 8), r = (e / 8) % (2 * P), c = e % 8;
                const int k = (r % P) + 1;
                const int dst = (r < P ? P - k : P + T - 1 + k) + RC_PAD, src = (r < P ? P + k : P + T - 1 - k) + RC_PAD;
                uint8_t* const base = a_gen + u * Cfg::U_BYTES + pl * RP_A_PLANE;
                *reinterpret_cast<uint4*>(base + dst * 128 + ((c ^ (dst & 7)) << 4)) =
                    *reinterpret_cast<const uint4*>(base + src * 128 + ((c ^ (src & 7)) << 4));
            }
            fence_proxy_async_smem();
            __syncthreads();
        }
        for (int j = 0; j < nconv; ++j, ++g) {
            mbar_wait(w_full, g & 1u);
            RP_STAMP(2, j, 1);
            if (tid == 0 && j + 3 <= nconv) prefetch_chunk(b0, j + 3);  // one conv ahead of the load_x that reads it
            issue(accA, 0);  // MMA_A(j)
            // MMA_A(j) is the only group in flight, so this returns at once.  It tells ptxas so: without it ptxas waits for MMA_A(j)
            // inside epilogue_B(j-1) below, and that epilogue no longer runs under the MMAs.
            wgmma_wait<1>();
            RP_STAMP(0, j, 0);
            // Each x_{j+2} load completes one phase of x_next(u).  Before conv j's, slot u has had it * (nconv - 1) loads in this
            // CTA's earlier pairs (an absent B is always its CTA's last pair) and j in this one: g - it.
            if (j > 0) {
                RP_STAMP(1, j - 1, 2);
                epilogue(accB, 1, b0 + 1, j - 1, (g - 1 - it) & 1u);  // under MMA_A(j)
                RP_STAMP(1, j - 1, 3);
                fence_proxy_async_smem();
            }
            __syncthreads();  // B's operand of conv j is complete
            issue(accB, 1);   // MMA_B(j)
            RP_STAMP(1, j, 0);
            wgmma_wait<1>();
            wgmma_fence_acc(accA);
            __syncthreads();  // every warpgroup's MMA_A(j) has retired: A's tile may be overwritten
            RP_STAMP(0, j, 1);
            if (tid == 0 && j + 1 < nconv) {
                mbar_arrive_expect_tx(x_next(0), NP * RP_A_PLANE);
                load_x(x_next(0), 0, b0, j + 2);
                RP_STAMP(0, j, 4);
            }
            RP_STAMP(0, j, 2);
            epilogue(accA, 0, b0, j, (g - it) & 1u);  // under MMA_B(j)
            RP_STAMP(0, j, 3);
            fence_proxy_async_smem();
            wgmma_wait<0>();
            wgmma_fence_acc(accB);
            __syncthreads();  // A's operand of conv j+1 is complete, and every MMA_B(j) has retired: the weight slot is free
            RP_STAMP(1, j, 1);
            if (tid == 0 && j + 1 < nconv) {
                RP_STAMP(2, j + 1, 0);
                load_w(j + 1);  // first: MMA_A(j+1) waits for the weights, only B's pass 2 for x
                if (b0 + 1 < cp.B) {  // B's tile is dead as well; its epilogue runs under MMA_A(j+1)
                    mbar_arrive_expect_tx(x_next(1), NP * RP_A_PLANE);
                    load_x(x_next(1), 1, b0 + 1, j + 2);
                    RP_STAMP(1, j, 4);
                }
            }
        }
        RP_STAMP(1, nconv - 1, 2);
        epilogue(accB, 1, b0 + 1, nconv - 1, 0u);  // the last conv: nothing to load
        RP_STAMP(1, nconv - 1, 3);
        __syncthreads();  // the next pair's loads overwrite the tiles and the weight slot
    }
}

int res2chain_build(Res2ChainParams* cp, const Planes& x, const Planes& y, const Planes* W, const float* const* bias, const float* const* bn_scale,
                    const float* const* bn_shift, int nconv, int B, int T, int P, int Tp, int dil, bool paired) {
    PPV_REQUIRE(nconv >= 1 && nconv <= RES2CHAIN_MAX, "res2chain: 1..7 convs");
    PPV_REQUIRE(P == RC_PAD && Tp == T + 2 * P && Tp <= RC_MAX_TP, "res2chain: padded utterance must fit 384 rows with P == 4");
    PPV_REQUIRE(!paired || Tp <= RP_MAX_TP, "res2chain: the paired kernel needs a padded utterance of at most 320 rows");
    PPV_REQUIRE(dil >= 1 && dil <= RC_PAD, "res2chain: dilation must be in [1,4]");
    PPV_REQUIRE(x.ld >= (nconv + 1) * 64 && y.ld >= (nconv + 1) * 64, "res2chain: buffers narrower than the chunks");
    memset(static_cast<void*>(cp), 0, sizeof(*cp));
    int rc = encode_planes_map_ex(&cp->mapX, x, 64, paired ? RP_BOX_ROWS : RC_BOX_ROWS, 128);
    if (rc) return rc;
    const int ntiles = (Tp + GEMM_BM - 1) / GEMM_BM;
    if (paired) {  // the paired kernel stages nothing: its epilogue writes y from the registers, 16 bytes per row and plane
        PPV_REQUIRE(!(reinterpret_cast<uintptr_t>(y.base) & 15) && y.ld % 8 == 0 && y.plane_stride % 8 == 0, "res2chain: y planes not 16-byte aligned");
    } else {
        rc = encode_planes_map_ex(&cp->mapXt, x, 64, GEMM_BM, 128);
        if (rc) return rc;
        rc = encode_planes_map_ex(&cp->mapY, y, 64, GEMM_BM, 128);
        if (rc) return rc;
        rc = encode_planes_map_ex(&cp->mapYtail, y, 64, Tp - (ntiles - 1) * GEMM_BM, 128);
        if (rc) return rc;
    }
    for (int j = 0; j < nconv; ++j) {
        PPV_REQUIRE(W[j].ld >= 192 && W[j].rows >= 64, "res2chain: weight layout mismatch");
        rc = encode_planes_map(&cp->mapW[j], W[j], 64);
        if (rc) return rc;
        cp->bias[j] = bias[j];
        cp->bn_scale[j] = bn_scale[j];
        cp->bn_shift[j] = bn_shift[j];
    }
    cp->x = x;
    cp->y = y;
    cp->nconv = nconv;
    cp->width = 64;
    cp->B = B;
    cp->T = T;
    cp->P = P;
    cp->Tp = Tp;
    cp->dil = dil;
    cp->ntiles = ntiles;
    cp->paired = paired ? 1 : 0;
    if (getenv("PPV_RES2_TRACE")) {  // debug: leaked on purpose, read back by res2chain_trace_dump
        static unsigned long long* buf = nullptr;
        if (!buf) {
            cudaMalloc(reinterpret_cast<void**>(&buf), 3 * 8 * 8 * sizeof(unsigned long long));
            cudaMemset(buf, 0, 3 * 8 * 8 * sizeof(unsigned long long));
        }
        cp->trace = buf;
    }
    return PPV_OK;
}

template <int NSPLIT>
static int launch_rc(const Res2ChainParams& cp, int num_sms, cudaStream_t st) {
    using Cfg = RCCfg<NSPLIT>;
    PPV_ONCE_PER_DEVICE(PPV_CUDA_OK(cudaFuncSetAttribute(res2chain_kernel<NSPLIT>, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::SMEM_BYTES)));
    const int grid = std::min(cp.B, num_sms);
    PPV_PDL_OK(launch_pdl(res2chain_kernel<NSPLIT>, dim3(grid), dim3(RC_THREADS), Cfg::SMEM_BYTES, st, cp), "res2chain_kernel");
    return PPV_OK;
}

template <int NSPLIT>
static int launch_rp(const Res2ChainParams& cp, int num_sms, cudaStream_t st) {
    using Cfg = RPCfg<NSPLIT>;
    PPV_ONCE_PER_DEVICE(PPV_CUDA_OK(cudaFuncSetAttribute(res2chain_pair_kernel<NSPLIT>, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::SMEM_BYTES)));
    const int grid = std::min((cp.B + 1) / 2, num_sms);
    PPV_PDL_OK(launch_pdl(res2chain_pair_kernel<NSPLIT>, dim3(grid), dim3(RP_THREADS), Cfg::SMEM_BYTES, st, cp), "res2chain_pair_kernel");
    return PPV_OK;
}

int res2chain_launch(const Res2ChainParams& cp, int precision, int num_sms, cudaStream_t st) {
    if (cp.paired) return precision == PPV_PREC_BF16X3 ? launch_rp<3>(cp, num_sms, st) : launch_rp<1>(cp, num_sms, st);
    return precision == PPV_PREC_BF16X3 ? launch_rc<3>(cp, num_sms, st) : launch_rc<1>(cp, num_sms, st);
}
void res2chain_trace_dump(const Res2ChainParams& cp) {
    if (!cp.trace) return;
    unsigned long long h[3 * 8 * 8];
    cudaDeviceSynchronize();
    cudaMemcpy(h, cp.trace, sizeof(h), cudaMemcpyDeviceToHost);
    unsigned long long t0 = ~0ull;
    for (unsigned long long v : h)
        if (v && v < t0) t0 = v;
    static const char* const single_roles[3] = {"tma", "mma", "epi"};
    static const char* const pair_roles[3] = {"utt A", "utt B", "weights"};  // see RP_STAMP
    const char* const* roles = cp.paired ? pair_roles : single_roles;
    for (int r = 0; r < 3; ++r)
        for (int j = 0; j < 7; ++j) {
            printf("res2chain trace %s conv %d:", roles[r], j);
            for (int e = 0; e < 8; ++e) printf(" %8lld", h[(r * 8 + j) * 8 + e] ? (long long)(h[(r * 8 + j) * 8 + e] - t0) : -1ll);
            printf("\n");
        }
}
bool res2chain_fits(int T, int P) { return P == RC_PAD && T + 2 * P <= RC_MAX_TP; }
bool res2chain_pair_fits(int T, int P) { return P == RC_PAD && T + 2 * P <= RP_MAX_TP; }

}  // namespace ppv
