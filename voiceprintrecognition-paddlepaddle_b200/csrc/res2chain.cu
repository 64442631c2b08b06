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
        uint8_t* const s_gen = smem_gen + (s_base - smem_base);
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
                uint8_t* const sbuf = s_gen + i * Cfg::S_BYTES;
                auto epilogue = [&](const float (&acc)[BN / 2], int mb) {
#pragma unroll
                    for (int h = 0; h < 2; ++h) {
                        const int rloc = mb * 64 + 16 * w + (l >> 2) + 8 * h;  // row inside the 128-row tile
                        const int p = tw * GEMM_BM + rloc;                      // padded row inside the utterance
                        const int tt = p - cp.P;
                        const bool valid = tt >= 0 && tt < cp.T;
                        int rows[3] = {p + RC_PAD, -1, -1};
                        if (tt >= 1 && tt <= cp.P) rows[1] = cp.P - tt + RC_PAD;
                        const int uu = cp.T - 1 - tt;
                        if (uu >= 1 && uu <= cp.P) rows[2] = cp.P + cp.T - 1 + uu + RC_PAD;
#pragma unroll
                        for (int q = 0; q < BN / 8; ++q) {
                            const int col = 8 * q + 2 * (l & 3);
                            const int off = ((q ^ (rloc & 7)) << 4) + 4 * (l & 3);  // SWIZZLE_128B: 16-byte chunk q of the row
                            // bias -> ReLU -> BatchNorm(eval) affine   (TDNNBlock, utils.py:147)
                            const float2 b2 = __ldg(reinterpret_cast<const float2*>(bias + col));
                            const float2 s2 = __ldg(reinterpret_cast<const float2*>(bsc + col));
                            const float2 h2 = __ldg(reinterpret_cast<const float2*>(bsh + col));
                            const float x0 = fmaf(fmaxf(acc[4 * q + 2 * h] + b2.x, 0.f), s2.x, h2.x);
                            const float x1 = fmaf(fmaxf(acc[4 * q + 2 * h + 1] + b2.y, 0.f), s2.y, h2.y);
                            uint32_t nh = 0, nl = 0;
                            if (has_next) {
                                nh = *reinterpret_cast<const uint32_t*>(sbuf + rloc * 128 + off);
                                if (NP == 2) nl = *reinterpret_cast<const uint32_t*>(sbuf + RC_S_PLANE + rloc * 128 + off);
                            }
                            uint32_t yh, yl;  // y_{j+1} -> staging tile (every row: rows outside the valid frames are halo / padding rows of y)
                            split_pack_bf16x2(x0, x1, yh, yl);
                            *reinterpret_cast<uint32_t*>(sbuf + rloc * 128 + off) = yh;
                            if (NP == 2) *reinterpret_cast<uint32_t*>(sbuf + RC_S_PLANE + rloc * 128 + off) = yl;
                            if (has_next && valid) {  // x_{j+2} + y_{j+1} -> operand of the next conv, in place, with its reflect halo rows
                                const float2 hf = unpack_bf16x2(nh), lf = unpack_bf16x2(nl);
                                uint32_t oh, ol;
                                split_pack_bf16x2(x0 + (hf.x + lf.x), x1 + (hf.y + lf.y), oh, ol);
#pragma unroll
                                for (int r = 0; r < 3; ++r) {
                                    if (rows[r] < 0) continue;
                                    uint8_t* dst = a_gen + rows[r] * 128 + ((q ^ (rows[r] & 7)) << 4) + 4 * (l & 3);
                                    *reinterpret_cast<uint32_t*>(dst) = oh;
                                    if (NP == 2) *reinterpret_cast<uint32_t*>(dst + RC_A_PLANE) = ol;
                                }
                            }
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

int res2chain_build(Res2ChainParams* cp, const Planes& x, const Planes& y, const Planes* W, const float* const* bias, const float* const* bn_scale,
                    const float* const* bn_shift, int nconv, int B, int T, int P, int Tp, int dil) {
    PPV_REQUIRE(nconv >= 1 && nconv <= RES2CHAIN_MAX, "res2chain: 1..7 convs");
    PPV_REQUIRE(P == RC_PAD && Tp == T + 2 * P && Tp <= RC_MAX_TP, "res2chain: padded utterance must fit 384 rows with P == 4");
    PPV_REQUIRE(dil >= 1 && dil <= RC_PAD, "res2chain: dilation must be in [1,4]");
    PPV_REQUIRE(x.ld >= (nconv + 1) * 64 && y.ld >= (nconv + 1) * 64, "res2chain: buffers narrower than the chunks");
    memset(static_cast<void*>(cp), 0, sizeof(*cp));
    int rc = encode_planes_map_ex(&cp->mapX, x, 64, RC_BOX_ROWS, 128);
    if (rc) return rc;
    const int ntiles = (Tp + GEMM_BM - 1) / GEMM_BM;
    rc = encode_planes_map_ex(&cp->mapXt, x, 64, GEMM_BM, 128);
    if (rc) return rc;
    rc = encode_planes_map_ex(&cp->mapY, y, 64, GEMM_BM, 128);
    if (rc) return rc;
    rc = encode_planes_map_ex(&cp->mapYtail, y, 64, Tp - (ntiles - 1) * GEMM_BM, 128);
    if (rc) return rc;
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

int res2chain_launch(const Res2ChainParams& cp, int precision, int num_sms, cudaStream_t st) {
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
    static const char* roles[3] = {"tma", "mma", "epi"};
    for (int r = 0; r < 3; ++r)
        for (int j = 0; j < 7; ++j) {
            printf("res2chain trace %s conv %d:", roles[r], j);
            for (int e = 0; e < 8; ++e) printf(" %8lld", h[(r * 8 + j) * 8 + e] ? (long long)(h[(r * 8 + j) * 8 + e] - t0) : -1ll);
            printf("\n");
        }
}
bool res2chain_fits(int T, int P) { return P == RC_PAD && T + 2 * P <= RC_MAX_TP; }

}  // namespace ppv
