// Shared epilogue of the wgmma kernels (gemm_wgmma.cu, res2conv.cu, conv3x3.cu): one warpgroup's 64 x BN fp32 accumulator
// fragment (registers, layout in ptx.cuh) -> bias / per-utterance bias / ReLU / BatchNorm affine / tanh / sigmoid -> split-bf16
// planes (incl. the reflect-halo rows of the padded time layout) or fp32.  Each thread owns two rows and BN / 4 columns of the
// tile, in pairs of adjacent columns.  The general path (epilogue_frag) stores every pair straight from the registers: a warp's store
// covers 16 B of each of 8 rows (half of a 32-byte sector).  The lean path of the gather-GEMM (epilogue_frag_lean) first exchanges the
// pairs inside each quad of lanes so that every lane stores 8 columns of a row with one 16-byte store per plane.
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

// 4 x 4 transpose of column pairs inside each quad of lanes (two butterfly stages of __shfl_xor_sync), for 16-byte epilogue
// accesses.  On entry a[2 i], a[2 i + 1] are this lane's two columns of 8-column group i of row a (b: row b), i in [0, 4), as the
// wgmma fragment holds them; on return lane q = lane & 3 holds all 8 columns of group q of both rows, a[k] / b[k] = column 8 q + k.
__device__ __forceinline__ void quad_transpose_pairs(float (&a)[8], float (&b)[8], int q) {
    const bool q2 = (q & 2) != 0, q1 = (q & 1) != 0;
    // stage 1, lanes q and q ^ 2 swap 2 x 2 blocks of column pairs; stage 2, lanes q and q ^ 1 swap single pairs
#pragma unroll
    for (int e = 0; e < 4; ++e) {  // e = 2 j + f: pair j in {0, 1}, float f
        const float sa = q2 ? a[e] : a[e + 4], sb = q2 ? b[e] : b[e + 4];
        const float ra_ = __shfl_xor_sync(0xffffffffu, sa, 2), rb_ = __shfl_xor_sync(0xffffffffu, sb, 2);
        if (q2) a[e] = ra_, b[e] = rb_;
        else a[e + 4] = ra_, b[e + 4] = rb_;
    }
#pragma unroll
    for (int e = 0; e < 8; e += 4) {
#pragma unroll
        for (int f = 0; f < 2; ++f) {
            const float sa = q1 ? a[e + f] : a[e + 2 + f], sb = q1 ? b[e + f] : b[e + 2 + f];
            const float ra_ = __shfl_xor_sync(0xffffffffu, sa, 1), rb_ = __shfl_xor_sync(0xffffffffu, sb, 1);
            if (q1) a[e + f] = ra_, b[e + f] = rb_;
            else a[e + 2 + f] = ra_, b[e + 2 + f] = rb_;
        }
    }
}

// The epilogues of the ECAPA-TDNN layers (gemm_build sets ep.lean): split-bf16 planes on the input row grid, bias / per-utterance
// bias / ReLU / BN affine / tanh, no halo, mirror or zero rows, no segment scale, SiLU, sigmoid or clipped ReLU.  Per element the
// arithmetic is epilogue_math1's, in the same order; each column's bias / BN vectors are loaded once for both of a thread's rows.
// The fragment is walked 32 columns (four 8-column groups) per trip.  The four lanes of a quad share two rows and hold two columns of
// each group; a 4 x 4 transpose inside the quad (two butterfly stages of __shfl_xor_sync) gives lane q all 8 columns of group q of
// both rows, so each row leaves as one 16-byte store per plane instead of four 4-byte ones (whole 32-byte sectors per warp store).
template <int BN, typename RowOf>
__device__ __forceinline__ void epilogue_frag_lean(const Epilogue& ep, int N, int n0, float (&acc)[BN / 2], RowOf&& row_of, int t) {
    static_assert(BN % 32 == 0, "lean epilogue: whole 32-column trips");
    const int w = t >> 5, l = t & 31, q = l & 3;
    const int r0 = 16 * w + (l >> 2);
    const EpiRow ra = epilogue_row(ep, row_of(r0), 0);
    const EpiRow rb = epilogue_row(ep, row_of(r0 + 8), 0);
    const int cq = n0 + 8 * q;  // after the transpose this lane's columns are cq + 8 c + [0, 8) in trip c / 4
    __nv_bfloat16* const obase = static_cast<__nv_bfloat16*>(ep.out) + ep.out_col0 + cq;
    __nv_bfloat16* const pa = obase + ra.out_row * ep.out_ld;
    __nv_bfloat16* const pb = obase + rb.out_row * ep.out_ld;
    const int64_t lo_off = ep.out_plane_stride;  // gemm_build: out_ld, out_col0 and the plane stride are multiples of 16 elements
    const float* const ga = ep.rowgrp_bias ? ep.rowgrp_bias + ra.grp * N + cq : nullptr;
    const float* const gb = ep.rowgrp_bias ? ep.rowgrp_bias + rb.grp * N + cq : nullptr;
#pragma unroll 1
    for (int c = 0; c < BN / 8; c += 4) {
        // a[2 i], a[2 i + 1]: this lane's two columns of group i, row a (b: row b)
        float a[8], b[8];
#pragma unroll
        for (int i = 0; i < 4; ++i) a[2 * i] = acc[4 * i], a[2 * i + 1] = acc[4 * i + 1], b[2 * i] = acc[4 * i + 2], b[2 * i + 1] = acc[4 * i + 3];
#pragma unroll
        for (int j = 0; j + 16 < BN / 2; ++j) acc[j] = acc[j + 16];
        quad_transpose_pairs(a, b, q);
        const int j0 = 8 * c;  // this lane's first column of the trip, relative to cq
        if (n0 + j0 >= N) continue;  // planes output: N % 32 == 0, so a trip's 32 columns are all in or all out
#pragma unroll
        for (int k = 0; k < 8; ++k) {
            const int col = cq + j0 + k;
            if (ep.bias) {
                const float bb = __ldg(ep.bias + col);
                a[k] += bb, b[k] += bb;
            }
            if (ga) a[k] += __ldg(ga + j0 + k), b[k] += __ldg(gb + j0 + k);
            if (ep.relu) a[k] = fmaxf(a[k], 0.f), b[k] = fmaxf(b[k], 0.f);
            if (ep.bn_scale) {
                const float sc = __ldg(ep.bn_scale + col), sh = __ldg(ep.bn_shift + col);
                a[k] = fmaf(a[k], sc, sh), b[k] = fmaf(b[k], sc, sh);
            }
            if (ep.tanh_) a[k] = tanhf(a[k]), b[k] = tanhf(b[k]);
        }
        uint4 ha, la, hb, lb;
        split_pack_bf16x2(a[0], a[1], ha.x, la.x), split_pack_bf16x2(a[2], a[3], ha.y, la.y);
        split_pack_bf16x2(a[4], a[5], ha.z, la.z), split_pack_bf16x2(a[6], a[7], ha.w, la.w);
        split_pack_bf16x2(b[0], b[1], hb.x, lb.x), split_pack_bf16x2(b[2], b[3], hb.y, lb.y);
        split_pack_bf16x2(b[4], b[5], hb.z, lb.z), split_pack_bf16x2(b[6], b[7], hb.w, lb.w);
        if (ra.valid) {
            *reinterpret_cast<uint4*>(pa + j0) = ha;
            *reinterpret_cast<uint4*>(pa + j0 + lo_off) = la;
        }
        if (rb.valid) {
            *reinterpret_cast<uint4*>(pb + j0) = hb;
            *reinterpret_cast<uint4*>(pb + j0 + lo_off) = lb;
        }
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
