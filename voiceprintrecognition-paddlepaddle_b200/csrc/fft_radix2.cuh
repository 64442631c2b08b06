// The radix-2 shared-memory complex FFT shared by the STFT front ends (spectral.cu) and the general Kaldi Fbank kernel (fbank.cu).
// `count` transforms of N = 2^log2n points lie back to back in shared memory, each loaded in bit-reversed order (fft_bitrev); the
// whole block runs the log2n butterfly stages over all of them at once and leaves each transform in natural order.
#pragma once
#include <cuda_runtime.h>

namespace ppv {

__device__ __forceinline__ int fft_bitrev(int i, int log2n) { return int(__brev(unsigned(i)) >> (32 - log2n)); }

// twiddle[k] = exp(-2 pi i k / N), k < N / 2, in global memory.  Every thread of the block calls this; it ends on a __syncthreads.
__device__ __forceinline__ void fft_radix2(float2* z, int log2n, int count, const float2* __restrict__ twiddle) {
    const int N = 1 << log2n;
    const int hmask = (N >> 1) - 1;
    const int nbf = count * (N >> 1);
    for (int s = 1; s <= log2n; ++s) {
        const int half = 1 << (s - 1);
        const int tw_stride = N >> s;
        for (int bf = threadIdx.x; bf < nbf; bf += blockDim.x) {
            const int lb = bf & hmask;  // butterfly inside its transform
            const int pos = lb & (half - 1);
            const int i0 = ((bf >> (log2n - 1)) << log2n) + ((lb >> (s - 1)) << s) + pos;
            const float2 w = __ldg(twiddle + pos * tw_stride);
            const float2 u = z[i0], v0 = z[i0 + half];
            const float2 v = make_float2(v0.x * w.x - v0.y * w.y, v0.x * w.y + v0.y * w.x);
            z[i0] = make_float2(u.x + v.x, u.y + v.y);
            z[i0 + half] = make_float2(u.x - v.x, u.y - v.y);
        }
        __syncthreads();
    }
}

}  // namespace ppv
