// Shared epilogue of the wgmma kernels (gemm_wgmma.cu, res2conv.cu, conv3x3.cu): one warpgroup's 64 x BN fp32 accumulator
// fragment (registers, layout in ptx.cuh) -> bias / per-utterance bias / ReLU / BatchNorm affine / tanh / sigmoid -> split-bf16
// planes (incl. the reflect-halo rows of the padded time layout) or fp32.  Each thread owns two rows and BN / 4 columns of the
// tile, in pairs of adjacent columns; every pair is processed and stored straight from the registers.
// Not tuned on H100: a warp's store covers 16 B of each of 8 rows (half of a 32-byte sector).  Gathering a row's 8 columns into one
// 16-byte store per lane (a 4 x 4 exchange of column pairs inside each quad of lanes) is the obvious next step; it is not measured.
#pragma once
#include "common.h"
#include "ptx.cuh"

namespace ppv {

constexpr int GEMM_MMA_THREADS = 256;                 // two MMA warpgroups (whole tiles in turn, or rows 0-63 / 64-127 of each)
constexpr int GEMM_THREADS = 128 + GEMM_MMA_THREADS;  // + the producer warpgroup (warp 0: TMA)

// per-column epilogue math on one accumulator value of global column `col`.  The per-column vectors are re-read for each of
// the thread's two rows (L1 hits): holding them for all BN / 4 columns costs the BN = 256 tile more spills than the loads cost.
__device__ __forceinline__ float epilogue_math1(const Epilogue& ep, int N, int col, int64_t grp, int64_t sgrp, float x) {
    if (ep.bias) x += __ldg(ep.bias + col);
    if (ep.rowgrp_bias) x += __ldg(ep.rowgrp_bias + grp * N + col);
    if (ep.seg_scale) x *= __ldg(ep.seg_scale + sgrp * N + col);
    if (ep.relu) {
        x = fmaxf(x, 0.f);
        if (ep.relu_max > 0.f) x = fminf(x, ep.relu_max);
    }
    if (ep.silu_) x = x / (1.f + expf(-x));
    if (ep.bn_scale) x = fmaf(x, __ldg(ep.bn_scale + col), __ldg(ep.bn_shift + col));
    if (ep.tanh_) x = tanhf(x);
    if (ep.sigmoid_) x = 1.f / (1.f + expf(-x));
    return x;
}

// Where one GEMM row goes: validity, destination row, reflect-halo mirror rows, per-utterance / per-segment groups.
struct EpiRow {
    bool valid = false;
    int64_t out_row = 0, mirror_a = -1, mirror_b = -1, grp = 0, sgrp = 0;
    int64_t zero_row = -1;  // an invalid row that must hold zeros (ep.zero_invalid: zero-padded convs read it)
};
// row < 0: this accumulator row holds no output
__device__ __forceinline__ EpiRow epilogue_row(const Epilogue& ep, int64_t row, int64_t out_row_shift) {
    EpiRow r;
    r.valid = row >= 0;
    const int64_t row_in = row;
    if (row < 0) row = 0;
    r.out_row = row + out_row_shift;  // wgrad mode: partial block of this K split
    if (ep.img_Wp > 0) {
        const int64_t img = int64_t(ep.img_Hp) * ep.img_Wp;
        r.grp = row / img;
        const int rem = int(row - r.grp * img);
        const int h = rem / ep.img_Wp - 1, w = rem % ep.img_Wp - 1;
        r.valid = r.valid && h >= 0 && h < ep.img_H && w >= 0 && w < ep.img_W;
        const int sw = ep.img_stride_w ? ep.img_stride_w : ep.img_stride;
        r.valid = r.valid && (h % ep.img_stride) == 0 && (w % sw) == 0;
        r.out_row = (r.grp * ep.out_Hp + h / ep.img_stride + 1) * ep.out_Wp + w / sw + 1;
    } else if (ep.Tp > 0) {
        r.grp = row / ep.Tp;
        const int t = int(row - r.grp * ep.Tp) - ep.P;
        r.valid = r.valid && t >= 0 && t < ep.T;
        if (ep.seg_scale && r.valid) r.sgrp = r.grp * ep.nseg + t / ep.seg_len;
        if (ep.halo && r.valid) {
            if (t >= 1 && t <= ep.P) r.mirror_a = row - 2 * t;
            const int u = ep.T - 1 - t;  // distance from the last frame
            if (u >= 1 && u <= ep.P) r.mirror_b = row + 2 * u;
        }
    }
    const bool same_grid = ep.img_Wp == 0 || (ep.img_stride == 1 && ep.img_stride_w <= 1 && ep.out_Hp == ep.img_Hp && ep.out_Wp == ep.img_Wp);
    if (!r.valid && row_in >= 0 && ep.zero_invalid && ep.out_mode == OUT_PLANES && !ep.halo && same_grid) r.zero_row = row_in + out_row_shift;
    return r;
}

// two adjacent columns (col, col + 1) of one row
__device__ __forceinline__ void epilogue_pair(const Epilogue& ep, int N, int col, const EpiRow& r, float a, float b) {
    if (col >= N) return;
    if (!r.valid) {
        if (r.zero_row >= 0) {
            __nv_bfloat16* ph = static_cast<__nv_bfloat16*>(ep.out) + r.zero_row * ep.out_ld + ep.out_col0 + col;
            *reinterpret_cast<uint32_t*>(ph) = 0u;
            *reinterpret_cast<uint32_t*>(ph + ep.out_plane_stride) = 0u;
        }
        return;
    }
    const bool two = col + 1 < N;
    a = epilogue_math1(ep, N, col, r.grp, r.sgrp, a);
    if (two) b = epilogue_math1(ep, N, col + 1, r.grp, r.sgrp, b);
    if (ep.out_mode == OUT_F32) {
        float* dst = static_cast<float*>(ep.out) + r.out_row * ep.out_ld + ep.out_col0 + col;
        if (two && ep.f32_vec_ok) {
            *reinterpret_cast<float2*>(dst) = make_float2(a, b);
        } else {
            dst[0] = a;
            if (two) dst[1] = b;
        }
        return;
    }
    uint32_t h, l;
    split_pack_bf16x2(a, b, h, l);
    __nv_bfloat16* obase = static_cast<__nv_bfloat16*>(ep.out) + ep.out_col0 + col;
    auto store_row = [&](int64_t row) {
        uint32_t* ph = reinterpret_cast<uint32_t*>(obase + row * ep.out_ld);
        ph[0] = h;
        *reinterpret_cast<uint32_t*>(reinterpret_cast<__nv_bfloat16*>(ph) + ep.out_plane_stride) = l;
    };
    store_row(r.out_row);
    if (r.mirror_a >= 0) store_row(r.mirror_a);
    if (r.mirror_b >= 0) store_row(r.mirror_b);
}

// The whole 64 x BN fragment of this warpgroup.  `row_of(r)`, r in [0, 64): the GEMM row of warpgroup-local row r, or -1 if it
// holds no output; `t`: thread index inside the warpgroup; columns are n0 + [0, BN).  The accumulators are consumed: on return
// `acc` holds garbage.
// The fragment is walked EPI_GROUPS column groups (8 columns, 4 registers) at a time by a loop that is not unrolled; after each trip the
// remaining accumulators move down by one chunk (register moves), so the per-pair code exists once per position inside a chunk
// instead of once per column group.  Unrolled over the whole fragment, the BN = 256 epilogue is ~25 k SASS instructions run straight
// through once per tile, and fetching them, not the tensor cores, sets the GEMM's pace (DESIGN.md §5).
template <int BN, typename RowOf>
__device__ __forceinline__ void epilogue_frag(const Epilogue& ep, int N, int n0, float (&acc)[BN / 2], RowOf&& row_of, int t,
                                              int64_t out_row_shift = 0) {
    if (ep.debug_nostore) return;
    const int w = t >> 5, l = t & 31;
    const int r0 = 16 * w + (l >> 2);
    const EpiRow ra = epilogue_row(ep, row_of(r0), out_row_shift);
    const EpiRow rb = epilogue_row(ep, row_of(r0 + 8), out_row_shift);
    constexpr int EPI_GROUPS = BN / 8 < 4 ? BN / 8 : 4;
#pragma unroll 1
    for (int c = 0; c < BN / 8; c += EPI_GROUPS) {
#pragma unroll
        for (int i = 0; i < EPI_GROUPS; ++i) {
            const int col = n0 + 8 * (c + i) + 2 * (l & 3);
            epilogue_pair(ep, N, col, ra, acc[4 * i + 0], acc[4 * i + 1]);
            epilogue_pair(ep, N, col, rb, acc[4 * i + 2], acc[4 * i + 3]);
        }
#pragma unroll
        for (int j = 0; j + 4 * EPI_GROUPS < BN / 2; ++j) acc[j] = acc[j + 4 * EPI_GROUPS];
    }
}

// The epilogues of the ECAPA-TDNN layers (gemm_build sets ep.lean): split-bf16 planes on the input row grid, bias / per-utterance
// bias / ReLU / BN affine / tanh, no halo, mirror or zero rows, no segment scale, SiLU, sigmoid or clipped ReLU.  The two rows'
// mapping and store addresses are computed once per fragment, and each column's bias / BN vectors are loaded once for both rows.
// Per element the arithmetic is epilogue_math1's, in the same order.
template <int BN, typename RowOf>
__device__ __forceinline__ void epilogue_frag_lean(const Epilogue& ep, int N, int n0, float (&acc)[BN / 2], RowOf&& row_of, int t) {
    const int w = t >> 5, l = t & 31;
    const int r0 = 16 * w + (l >> 2);
    const EpiRow ra = epilogue_row(ep, row_of(r0), 0);
    const EpiRow rb = epilogue_row(ep, row_of(r0 + 8), 0);
    const int c0 = n0 + 2 * (l & 3);  // this thread's first column; its columns are c0 + 8 j + {0, 1}
    __nv_bfloat16* const obase = static_cast<__nv_bfloat16*>(ep.out) + ep.out_col0 + c0;
    uint32_t* const pa = reinterpret_cast<uint32_t*>(obase + ra.out_row * ep.out_ld);
    uint32_t* const pb = reinterpret_cast<uint32_t*>(obase + rb.out_row * ep.out_ld);
    const int64_t lo_off = ep.out_plane_stride / 2;  // the lo plane, in 32-bit words (gemm_build: plane stride % 16 == 0)
    const float* const ga = ep.rowgrp_bias ? ep.rowgrp_bias + ra.grp * N + c0 : nullptr;
    const float* const gb = ep.rowgrp_bias ? ep.rowgrp_bias + rb.grp * N + c0 : nullptr;
    constexpr int EPI_GROUPS = BN / 8 < 4 ? BN / 8 : 4;
#pragma unroll 1
    for (int c = 0; c < BN / 8; c += EPI_GROUPS) {
#pragma unroll
        for (int i = 0; i < EPI_GROUPS; ++i) {
            const int j = 8 * (c + i);
            if (c0 + j >= N) continue;  // planes output: N % 32 == 0, so column c0 + j + 1 exists too
            float xa0 = acc[4 * i + 0], xa1 = acc[4 * i + 1], xb0 = acc[4 * i + 2], xb1 = acc[4 * i + 3];
            if (ep.bias) {
                const float b0 = __ldg(ep.bias + c0 + j), b1 = __ldg(ep.bias + c0 + j + 1);
                xa0 += b0, xa1 += b1, xb0 += b0, xb1 += b1;
            }
            if (ga) {
                xa0 += __ldg(ga + j), xa1 += __ldg(ga + j + 1);
                xb0 += __ldg(gb + j), xb1 += __ldg(gb + j + 1);
            }
            if (ep.relu) xa0 = fmaxf(xa0, 0.f), xa1 = fmaxf(xa1, 0.f), xb0 = fmaxf(xb0, 0.f), xb1 = fmaxf(xb1, 0.f);
            if (ep.bn_scale) {
                const float s0 = __ldg(ep.bn_scale + c0 + j), s1 = __ldg(ep.bn_scale + c0 + j + 1);
                const float h0 = __ldg(ep.bn_shift + c0 + j), h1 = __ldg(ep.bn_shift + c0 + j + 1);
                xa0 = fmaf(xa0, s0, h0), xa1 = fmaf(xa1, s1, h1), xb0 = fmaf(xb0, s0, h0), xb1 = fmaf(xb1, s1, h1);
            }
            if (ep.tanh_) xa0 = tanhf(xa0), xa1 = tanhf(xa1), xb0 = tanhf(xb0), xb1 = tanhf(xb1);
            uint32_t h, lo;
            if (ra.valid) {
                split_pack_bf16x2(xa0, xa1, h, lo);
                pa[j / 2] = h;
                pa[j / 2 + lo_off] = lo;
            }
            if (rb.valid) {
                split_pack_bf16x2(xb0, xb1, h, lo);
                pb[j / 2] = h;
                pb[j / 2 + lo_off] = lo;
            }
        }
#pragma unroll
        for (int j = 0; j + 4 * EPI_GROUPS < BN / 2; ++j) acc[j] = acc[j + 4 * EPI_GROUPS];
    }
}

// The lean path where gemm_build selected it, else the general one.
template <int BN, typename RowOf>
__device__ __forceinline__ void gemm_epilogue(const Epilogue& ep, int N, int n0, float (&acc)[BN / 2], RowOf&& row_of, int t,
                                              int64_t out_row_shift) {
    if (ep.lean) epilogue_frag_lean<BN>(ep, N, n0, acc, row_of, t);
    else epilogue_frag<BN>(ep, N, n0, acc, row_of, t, out_row_shift);
}

}  // namespace ppv
