// The register-resident 512-point real FFT shared by the Fbank front end (fbank.cu) and the reverb convolution (reverb.cu).
// A 512-point real transform is one 256-point complex FFT of z[n] = y[2n] + i y[2n+1], done by 16 lanes as two radix-16 passes:
//   pass 1: lane q holds v[n1] = z[16 n1 + q]; fft16 over n1; slot r is multiplied by W256^{k1 q}, k1 = fb_k_of_slot(r), and the
//           16 x 16 tile is transposed through shared memory;
//   pass 2: lane q (now k1) holds v[n2] = A[k1][n2]; fft16 over n2; slot r holds Z[q + 16 fb_k_of_slot(r)].
// The real spectrum follows by untangling bins k and 256 - k with W512^k; the inverse runs the same passes on the conjugate.
#pragma once
#include <math.h>

#include <cuda_runtime.h>

namespace ppv {

__device__ __forceinline__ float2 cmul(float2 a, float2 b) {
    return make_float2(a.x * b.x - a.y * b.y, a.x * b.y + a.y * b.x);
}

// a * exp(-2 pi i E / 16), E a compile-time constant: the trivial rotations cost nothing / two adds
template <int E>
__device__ __forceinline__ float2 rot16(float2 a) {
    constexpr int e = E & 15;
    constexpr float R = 0.70710678118654752f, C1 = 0.92387953251128674f, S1 = 0.38268343236508977f;
    if constexpr (e == 0) return a;
    else if constexpr (e == 4) return make_float2(a.y, -a.x);
    else if constexpr (e == 8) return make_float2(-a.x, -a.y);
    else if constexpr (e == 12) return make_float2(-a.y, a.x);
    else if constexpr (e == 2) return make_float2(R * (a.x + a.y), R * (a.y - a.x));
    else if constexpr (e == 6) return make_float2(R * (a.y - a.x), -R * (a.x + a.y));
    else if constexpr (e == 10) return make_float2(-R * (a.x + a.y), R * (a.x - a.y));
    else if constexpr (e == 14) return make_float2(R * (a.x - a.y), R * (a.x + a.y));
    else {
        // (x + iy)(c - is) = (xc + ys) + i(yc - xs), c = cos(2 pi e / 16), s = sin(2 pi e / 16)
        constexpr float c = (e == 1 || e == 15) ? C1 : (e == 3 || e == 13) ? S1 : (e == 5 || e == 11) ? -S1 : -C1;  // e in {1,3,5,7,9,11,13,15}
        constexpr float s = (e == 1 || e == 7) ? S1 : (e == 3 || e == 5) ? C1 : (e == 9 || e == 15) ? -S1 : -C1;
        return make_float2(fmaf(a.x, c, a.y * s), fmaf(a.y, c, -(a.x * s)));
    }
}

// 4-point forward DFT in place: (x0,x1,x2,x3) -> (X0,X1,X2,X3)
__device__ __forceinline__ void dft4(float2& x0, float2& x1, float2& x2, float2& x3) {
    const float2 t0 = make_float2(x0.x + x2.x, x0.y + x2.y), t1 = make_float2(x0.x - x2.x, x0.y - x2.y);
    const float2 t2 = make_float2(x1.x + x3.x, x1.y + x3.y), t3 = make_float2(x1.x - x3.x, x1.y - x3.y);
    x0 = make_float2(t0.x + t2.x, t0.y + t2.y);
    x2 = make_float2(t0.x - t2.x, t0.y - t2.y);
    x1 = make_float2(t1.x + t3.y, t1.y - t3.x);  // t1 - i t3
    x3 = make_float2(t1.x - t3.y, t1.y + t3.x);  // t1 + i t3
}

// 16-point forward DFT in registers (radix 4 x 4).  Input v[n] natural order; on return slot r holds X[fb_k_of_slot(r)].
__device__ __forceinline__ void fft16(float2 (&v)[16]) {
#pragma unroll
    for (int b = 0; b < 4; ++b) dft4(v[b], v[4 + b], v[8 + b], v[12 + b]);  // slot 4c+b = sum_a x[4a+b] W4^{ac}
    v[5] = rot16<1>(v[5]);
    v[6] = rot16<2>(v[6]);
    v[7] = rot16<3>(v[7]);
    v[9] = rot16<2>(v[9]);
    v[10] = rot16<4>(v[10]);
    v[11] = rot16<6>(v[11]);
    v[13] = rot16<3>(v[13]);
    v[14] = rot16<6>(v[14]);
    v[15] = rot16<9>(v[15]);
#pragma unroll
    for (int c = 0; c < 4; ++c) dft4(v[4 * c], v[4 * c + 1], v[4 * c + 2], v[4 * c + 3]);  // slot 4c+d = X[c + 4d]
}
__host__ __device__ constexpr int fb_k_of_slot(int r) { return (r >> 2) + 4 * (r & 3); }

// The twiddle tables: exp(-2 pi i num / den), rounded once from double.  tw256[k1 * 16 + n2] = fft_twiddle(k1 * n2, 256) (pass 1),
// tw512[k] = fft_twiddle(k, 512) (real-FFT untangling).  The host builds the Fbank's uploaded tables with it; kernels without a handle
// (reverb.cu) fill their shared-memory copies with fft_twiddle_tables.
__host__ __device__ inline float2 fft_twiddle(int num, int den) {
#ifdef __CUDA_ARCH__
    double s, c;
    sincospi(-2.0 * double(num) / double(den), &s, &c);
    return make_float2(float(c), float(s));
#else
    return make_float2(float(cos(-2.0 * M_PI * num / double(den))), float(sin(-2.0 * M_PI * num / double(den))));
#endif
}

__device__ __forceinline__ void fft_twiddle_tables(float2* tw256, float2* tw512) {
    for (int i = threadIdx.x; i < 256; i += blockDim.x) {
        tw256[i] = fft_twiddle((i >> 4) * (i & 15), 256);
        tw512[i] = fft_twiddle(i, 512);
    }
}

}  // namespace ppv
