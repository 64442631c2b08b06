// L2 row normalisation into split-bf16 planes, shared by the cosine scoring (cosine.cu) and the speaker index (speaker_index.cu).
#pragma once
#include "common.h"
#include "ptx.cuh"

namespace ppv {

// One warp: x[0, D) / max(|x|, tiny) -> row `row` of `out` (columns >= D zero).  A zero-norm row comes out as zeros (scores 0).
__device__ __forceinline__ void normalize_row_to_planes(const float* __restrict__ x, int D, const Planes& out, int64_t row, int lane) {
    float ss = 0.f;
    for (int i = lane; i < D; i += 32) ss = fmaf(x[i], x[i], ss);
    ss = warp_sum(ss);
    const float inv = 1.f / fmaxf(sqrtf(ss), 1e-30f);
    for (int i = lane; i < out.ld; i += 32) {
        __nv_bfloat16 h, l;
        split_bf16(i < D ? x[i] * inv : 0.f, h, l);
        out.hi()[row * out.ld + i] = h;
        out.lo()[row * out.ld + i] = l;
    }
}

// one warp per row: X [rows, D] -> planes [>= rows, ld]
static __global__ void normalize_rows_kernel(const float* __restrict__ X, int rows, int D, Planes out) {
    const int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (row >= rows) return;
    normalize_row_to_planes(X + int64_t(row) * D, D, out, row, threadIdx.x & 31);
}

}  // namespace ppv
