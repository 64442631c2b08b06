// Fused attentive-statistics pooling (K5): attention logits + softmax over time + weighted mean / std + asp_bn in
// ONE kernel; the [frames, 1536] logits never exist in HBM.
// Reference: ppvector/models/pooling.py:107-123 (attn = conv(tanh(tdnn(.))); masked softmax over T;
// mean = sum(a x); std = sqrt(clip(sum(a (x - mean)^2), eps))) and ppvector/models/ecapa_tdnn.py:271 (asp_bn).
//
// The GEMM is TRANSPOSED relative to the other layers: D[channel, frame] = W2[channel, :] . att[frame, :], i.e.
// A = conv weight slab (128 channels x K=128, K-major), B = attention-TDNN activations (64 frames x K, K-major:
// the activation matrix is already laid out that way).  Accumulator rows are then CHANNELS and columns FRAMES: each of the
// two MMA warpgroups owns 64 channels of the slab, and a thread holds two channels x 16 frames of every 64-frame tile
// (wgmma fragment, ptx.cuh).  The softmax over time and the weighted moments are per-thread running sums over the thread's
// frames, merged across the four threads that share a channel at the end of the utterance -- no atomics, deterministic.
//   * online softmax (running max, rescale once per tile)
//   * moments about the channel's global mean g (from asp_global): S0 = sum e, S1 = sum e (x-g), S2 = sum e (x-g)^2,
//     mean = g + S1/S0, var = S2/S0 - (S1/S0)^2   (shifted one-pass; the reference is two-pass)
//   * the conv bias is constant over time and cancels in the softmax: it is not even loaded.
// Work item = (utterance b, 128-channel slab); a CTA keeps the weight slab in smem for the item and streams the
// utterance in 64-frame tiles through a 2-deep TMA ring.  A ring stage carries BOTH the attention activations (the
// MMA's B operand) and the matching [64 frames x 128 channels] tile of x (un-swizzled, read with plain ld.shared), so the
// epilogue never waits on global memory.
#include <stdio.h>
#include <string.h>

#include "common.h"
#include "ptx.cuh"

namespace ppv {

constexpr int AF_NT = 64;                         // frames per tile (MMA N)
constexpr int AF_A_TILE = 128 * 64 * 2;           // weight tile  [128 ch x 64 k]  bf16, SWIZZLE_128B
constexpr int AF_B_TILE = AF_NT * 64 * 2;         // att tile     [64 fr x 64 k]   bf16, SWIZZLE_128B
constexpr int AF_X_TILE = AF_NT * 128 * 2;        // x tile       [64 fr x 128 ch] bf16, no swizzle (one plane)
constexpr int AF_STAGES = 2;
constexpr float LOG2E = 1.4426950408889634f;

template <int NSPLIT>
__global__ void __launch_bounds__(384, 1) asp_fused_kernel(const __grid_constant__ AspFusedParams p) {
    constexpr int NP = (NSPLIT == 3) ? 2 : 1;  // planes loaded per MMA operand
    extern __shared__ uint8_t smem_raw[];
    const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;
    uint8_t* smem_gen = smem_raw + (smem_base - smem_u32(smem_raw));
    const int ksteps = p.K / 64;  // 2 for K = 128
    const int a_bytes = ksteps * NP * AF_A_TILE;
    const int b_bytes = ksteps * NP * AF_B_TILE;
    const int stage_bytes = b_bytes + 2 * AF_X_TILE;  // x always needs hi and lo
    const uint32_t a_base = smem_base;
    const uint32_t s_base = smem_base + a_bytes;
    const uint32_t bar_base = s_base + AF_STAGES * stage_bytes;
    // barriers: a_full, a_empty, b_full[2], b_empty[2]
    const uint32_t a_full = bar_base, a_empty = bar_base + 8;
    auto b_full = [&](int s) { return bar_base + 16u + 8u * s; };
    auto b_empty = [&](int s) { return bar_base + 32u + 8u * s; };

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    if (warp == 0 && lane == 0) {
        prefetch_tmap(&p.mapW);
        prefetch_tmap(&p.mapAtt);
        prefetch_tmap(&p.mapX);
    }
    if (warp == 1 && lane == 0) {
        mbar_init(a_full, 1);
        mbar_init(a_empty, 256);  // every MMA thread, after the last MMA of the slab
        for (int s = 0; s < AF_STAGES; ++s) {
            mbar_init(b_full(s), 1);
            mbar_init(b_empty(s), 256);  // every MMA thread, after its MMAs retired and it has read the x tile
        }
        fence_mbar_init();
    }
    __syncthreads();
    griddep_launch_dependents();  // PDL
    griddep_wait();

    const int slabs = p.C / 128;
    const int items = slabs * p.B;
    const int ntiles = (p.T + AF_NT - 1) / AF_NT;

    if (warp == 0) {
        // ===================== TMA producer =====================
        int stage = 0;
        uint32_t phase = 0, a_phase = 0;
        int cur_slab = -1;
        for (int item = blockIdx.x; item < items; item += gridDim.x) {
            const int b = item / slabs, slab = item - b * slabs;  // utterance-major: att / x rows are shared by neighbouring items (L2)
            if (slab != cur_slab) {  // the weight slab stays in shared memory while consecutive items share it
                mbar_wait(a_empty, a_phase ^ 1u);
                if (lane == 0) {
                    mbar_arrive_expect_tx(a_full, a_bytes);
                    for (int ks = 0; ks < ksteps; ++ks)
                        for (int pl = 0; pl < NP; ++pl)
                            tma_load_3d(a_base + (ks * NP + pl) * AF_A_TILE, &p.mapW, a_full, ks * 64, slab * 128, pl);
                }
                __syncwarp();
                a_phase ^= 1u;
                cur_slab = slab;
            }
            {  // pull the NEXT item's x tiles (HBM) into L2 while this item is processed
                const int nitem = item + gridDim.x;
                if (nitem < items && lane < 2 * ntiles) {
                    const int nb = nitem / slabs, nslab = nitem - nb * slabs;
                    tma_prefetch_l2_3d(&p.mapX, nslab * 128, nb * p.Tp + p.P + (lane >> 1) * AF_NT, lane & 1);
                }
                __syncwarp();
            }
            const int row0 = b * p.Tp + p.P;
            for (int ft = 0; ft < ntiles; ++ft) {
                mbar_wait(b_empty(stage), phase ^ 1u);
                if (lane == 0) {
                    const uint32_t sb = s_base + stage * stage_bytes;
                    mbar_arrive_expect_tx(b_full(stage), stage_bytes);
                    for (int ks = 0; ks < ksteps; ++ks)
                        for (int pl = 0; pl < NP; ++pl)
                            tma_load_3d(sb + (ks * NP + pl) * AF_B_TILE, &p.mapAtt, b_full(stage), ks * 64, row0 + ft * AF_NT, pl);
                    for (int pl = 0; pl < 2; ++pl)
                        tma_load_3d(sb + b_bytes + pl * AF_X_TILE, &p.mapX, b_full(stage), slab * 128, row0 + ft * AF_NT, pl);
                }
                __syncwarp();
                if (++stage == AF_STAGES) {
                    stage = 0;
                    phase ^= 1u;
                }
            }
        }
    } else if (warp >= 4) {
        // ===================== MMA + softmax / moments: warpgroup g owns channels [64 g, 64 g + 64) of the slab =====================
        const int g = (warp - 4) >> 2, t = threadIdx.x & 127, w = t >> 5, l = t & 31;
        const int cl0 = 64 * g + 16 * w + (l >> 2);  // this thread's channels within the slab: cl0 and cl0 + 8
        float acc[AF_NT / 2];
#pragma unroll
        for (int i = 0; i < AF_NT / 2; ++i) acc[i] = 0.f;
        int stage = 0;
        uint32_t phase = 0, a_phase = 0;
        int cur_slab = -1;
        for (int item = blockIdx.x; item < items; item += gridDim.x) {
            const int b = item / slabs, slab = item - b * slabs;
            if (slab != cur_slab) {
                mbar_wait(a_full, a_phase);
                a_phase ^= 1u;
                cur_slab = slab;
            }
            const int nitem = item + gridDim.x;
            const bool last_of_slab = (nitem >= items) || (nitem % slabs != slab);
            float gm[2], m[2], S0[2], S1[2], S2[2];
#pragma unroll
            for (int rr = 0; rr < 2; ++rr) {
                const int64_t goff = int64_t(b) * p.gstat.ld + slab * 128 + cl0 + 8 * rr;
                gm[rr] = __bfloat162float(p.gstat.hi()[goff]) + __bfloat162float(p.gstat.lo()[goff]);
                m[rr] = -INFINITY;
                S0[rr] = S1[rr] = S2[rr] = 0.f;
            }
            const int Tb = p.nvalid ? max(1, min(p.T, p.nvalid[b])) : p.T;  // masked frames: softmax weight exactly 0
            for (int ft = 0; ft < ntiles; ++ft) {
                mbar_wait(b_full(stage), phase);
                const uint32_t sb = s_base + stage * stage_bytes;
                wgmma_fence_acc(acc);
                wgmma_fence();
                for (int ks = 0; ks < ksteps; ++ks) {
                    const uint64_t a_hi = make_sw128_kmajor_desc(a_base + (ks * NP) * AF_A_TILE + g * 64 * 128);
                    const uint64_t b_hi = make_sw128_kmajor_desc(sb + (ks * NP) * AF_B_TILE);
#pragma unroll
                    for (int k = 0; k < 4; ++k) wgmma_bf16<AF_NT>(acc, a_hi + 2 * k, b_hi + 2 * k, (ks > 0 || k > 0) ? 1u : 0u);
                    if (NSPLIT == 3) {
                        const uint64_t a_lo = make_sw128_kmajor_desc(a_base + (ks * NP + 1) * AF_A_TILE + g * 64 * 128);
                        const uint64_t b_lo = make_sw128_kmajor_desc(sb + (ks * NP + 1) * AF_B_TILE);
#pragma unroll
                        for (int k = 0; k < 4; ++k) wgmma_bf16<AF_NT>(acc, a_lo + 2 * k, b_hi + 2 * k, 1u);
#pragma unroll
                        for (int k = 0; k < 4; ++k) wgmma_bf16<AF_NT>(acc, a_hi + 2 * k, b_lo + 2 * k, 1u);
                    }
                }
                wgmma_commit();
                wgmma_wait<0>();
                wgmma_fence_acc(acc);
                if (ft == ntiles - 1 && last_of_slab) mbar_arrive(a_empty);  // weight slab free once its last item's MMAs retired
                const __nv_bfloat16* xs_hi = reinterpret_cast<const __nv_bfloat16*>(smem_gen + (sb - smem_base) + b_bytes);
                const __nv_bfloat16* xs_lo = xs_hi + AF_X_TILE / 2;
                const int f0 = ft * AF_NT;
#pragma unroll
                for (int rr = 0; rr < 2; ++rr) {
                    float cm = -INFINITY;
#pragma unroll
                    for (int i = 0; i < AF_NT / 8; ++i)
#pragma unroll
                        for (int e = 0; e < 2; ++e)
                            if (f0 + 8 * i + 2 * (l & 3) + e < Tb) cm = fmaxf(cm, acc[4 * i + 2 * rr + e]);
                    if (cm > m[rr]) {
                        const float r = exp2f((m[rr] - cm) * LOG2E);  // exp(-inf) = 0 on the first frames
                        S0[rr] *= r;
                        S1[rr] *= r;
                        S2[rr] *= r;
                        m[rr] = cm;
                    }
                    const float ms = m[rr] * LOG2E;
                    const int cl = cl0 + 8 * rr;
#pragma unroll
                    for (int i = 0; i < AF_NT / 8; ++i)
#pragma unroll
                        for (int e = 0; e < 2; ++e) {
                            const int fl = 8 * i + 2 * (l & 3) + e;
                            if (f0 + fl < Tb) {
                                const int o = fl * 128 + cl;
                                const float xv = __bfloat162float(xs_hi[o]) + __bfloat162float(xs_lo[o]);
                                const float ev = exp2f(fmaf(acc[4 * i + 2 * rr + e], LOG2E, -ms));
                                const float d = xv - gm[rr];
                                const float ed = ev * d;
                                S0[rr] += ev;
                                S1[rr] += ed;
                                S2[rr] = fmaf(ed, d, S2[rr]);
                            }
                        }
                }
                mbar_arrive(b_empty(stage));  // done with the att and x tiles of this stage
                if (++stage == AF_STAGES) {
                    stage = 0;
                    phase ^= 1u;
                }
            }
            // merge the four threads of a channel (lanes 4 k .. 4 k + 3 hold the same two channels)
#pragma unroll
            for (int rr = 0; rr < 2; ++rr) {
#pragma unroll
                for (int off = 1; off <= 2; off <<= 1) {
                    const float om = __shfl_xor_sync(0xffffffffu, m[rr], off), o0 = __shfl_xor_sync(0xffffffffu, S0[rr], off),
                                o1 = __shfl_xor_sync(0xffffffffu, S1[rr], off), o2 = __shfl_xor_sync(0xffffffffu, S2[rr], off);
                    const float mm = fmaxf(m[rr], om);
                    const float ra = S0[rr] > 0.f ? exp2f((m[rr] - mm) * LOG2E) : 0.f, rb = o0 > 0.f ? exp2f((om - mm) * LOG2E) : 0.f;
                    S0[rr] = S0[rr] * ra + o0 * rb;
                    S1[rr] = S1[rr] * ra + o1 * rb;
                    S2[rr] = S2[rr] * ra + o2 * rb;
                    m[rr] = mm;
                }
            }
            if ((l & 3) != 0) continue;
            const int C = p.C;
#pragma unroll
            for (int rr = 0; rr < 2; ++rr) {
                const int c = slab * 128 + cl0 + 8 * rr;
                const float inv = 1.f / S0[rr];
                const float dm = S1[rr] * inv;
                const float mean = gm[rr] + dm;
                const float sd = sqrtf(fmaxf(S2[rr] * inv - dm * dm, p.eps));
                if (p.out_raw) {
                    p.out_raw[int64_t(b) * 2 * C + c] = mean;
                    p.out_raw[int64_t(b) * 2 * C + C + c] = sd;
                }
                __nv_bfloat16 h, lo;
                split_bf16(fmaf(mean, p.bn_scale[c], p.bn_shift[c]), h, lo);
                p.out.hi()[int64_t(b) * p.out.ld + c] = h;
                p.out.lo()[int64_t(b) * p.out.ld + c] = lo;
                split_bf16(fmaf(sd, p.bn_scale[C + c], p.bn_shift[C + c]), h, lo);
                p.out.hi()[int64_t(b) * p.out.ld + C + c] = h;
                p.out.lo()[int64_t(b) * p.out.ld + C + c] = lo;
            }
        }
    }
}

int asp_fused_build(AspFusedParams* p, const Planes& W, const Planes& att, const Planes& x, const Planes& gstat, const float* bn_scale,
                    const float* bn_shift, const Planes& out, float* out_raw, int B, int T, int P, int Tp, int C, int K, float eps) {
    PPV_REQUIRE(C % 128 == 0 && K % 64 == 0 && K <= 128, "asp_fused: C % 128 == 0 and K in {64,128} required");
    memset(p, 0, sizeof(*p));
    PPV_REQUIRE(x.ld == C, "asp_fused: x row length must equal C");
    int rc = encode_planes_map(&p->mapW, W, 128);
    if (rc) return rc;
    rc = encode_planes_map(&p->mapAtt, att, AF_NT);
    if (rc) return rc;
    rc = encode_planes_map_ex(&p->mapX, x, 128, AF_NT, 0);
    if (rc) return rc;
    p->x = x;
    p->gstat = gstat;
    p->bn_scale = bn_scale;
    p->bn_shift = bn_shift;
    p->out = out;
    p->out_raw = out_raw;
    p->B = B;
    p->T = T;
    p->P = P;
    p->Tp = Tp;
    p->C = C;
    p->K = K;
    p->eps = eps;
    p->nvalid = nullptr;
    return PPV_OK;
}

int asp_fused_launch(const AspFusedParams& p, int precision, int num_sms, cudaStream_t st) {
    const bool x3 = precision == PPV_PREC_BF16X3;
    const int ksteps = p.K / 64, np = x3 ? 2 : 1;
    const int smem = 1024 + ksteps * np * AF_A_TILE + AF_STAGES * (ksteps * np * AF_B_TILE + 2 * AF_X_TILE) + 96 + 128 * 16 + 64;
    static bool attr3 = false, attr1 = false;
    bool& attr = x3 ? attr3 : attr1;
    if (!attr) {
        if (x3)
            PPV_CUDA_OK(cudaFuncSetAttribute(asp_fused_kernel<3>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
        else
            PPV_CUDA_OK(cudaFuncSetAttribute(asp_fused_kernel<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
        attr = true;
    }
    const int items = (p.C / 128) * p.B;
    const int grid = std::min(items, num_sms);
    if (x3)
        PPV_PDL_OK(launch_pdl(asp_fused_kernel<3>, dim3(grid), dim3(384), size_t(smem), st, p), "asp_fused_kernel");
    else
        PPV_PDL_OK(launch_pdl(asp_fused_kernel<1>, dim3(grid), dim3(384), size_t(smem), st, p), "asp_fused_kernel");
    return PPV_OK;
}

}  // namespace ppv
