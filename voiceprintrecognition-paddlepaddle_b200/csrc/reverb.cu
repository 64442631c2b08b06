// Reverberation of the batched audio preparation: the full linear convolution y = s * h of each utterance's mixed signal s (speed ->
// volume -> noise, new_len samples) with its room impulse response h (R taps), y of new_len + R - 1 samples, not truncated
// (recalled yeaudio ReverbPerturbAugmentor: scipy.signal.fftconvolve(samples, rir, "full"); tests/reverb_oracle.py).
// Uniformly partitioned overlap-save with block P = 256 and the 512-point real FFT of fft512.cuh:
//   X_i = FFT512(s[(i - 1) P, (i + 1) P))            i = 0 .. ceil(new_len / P)        (rv_forward_kernel, z = 0)
//   H_j = FFT512(h[j P, (j + 1) P) zero-padded)       j = 0 .. ceil(R / P) - 1          (rv_forward_kernel, z = 1)
//   y[m P, (m + 1) P) = the last P samples of IFFT512(sum_j X_{m-j} H_j)                 (rv_conv_kernel)
// s is never stored: the forward pass evaluates it from the raw samples with the gains of the shared gains kernel (audio_prep.cu).
// Only the partitions of the responses this batch drew are transformed (at most B), never the whole bank.  rv_conv_kernel writes y's
// crop window into the output rows and one fp64 sum of y^2 per output block; rv_norm_kernel turns those (fixed order) into the dB
// normalisation gain, which the shared apply kernel multiplies in.
// Spectra are stored with bins 0 and 256 (both real) packed into slot 0 as (X_0, X_256): 256 float2 per block.  The forward transform
// yields 2 X (fbank.cu's untangling); the response is scaled by 1 / 2048 on load (exact), which absorbs that factor on both operands
// and the 1 / 512 of the inverse transform.
#include <math.h>

#include "audio_prep.cuh"
#include "common.h"
#include "fft512.cuh"

namespace ppv {

namespace {

constexpr int RV_P = 256;         // block / partition length (half the FFT)
constexpr int RV_TM = 16;         // output blocks per rv_conv_kernel CTA: 16 inverse transforms on 16 lanes each
constexpr int RV_FRAMES = 16;     // forward transforms per rv_forward_kernel CTA
constexpr int RV_SCR = 17 * 16;   // float2 scratch per transform: [k1][n2] padded to 17 columns
constexpr float RV_H_SCALE = 1.f / 2048.f;

struct RvGeom {  // one item's block counts; valid = false for an item without reverb or with an out-of-range entry
    bool valid;
    int rlen, roff, nx, nj, ly, nm;
};

__device__ __forceinline__ RvGeom rv_geom(const PrepItem& it, const int32_t* rparams, int b, int64_t bank_len, int max_new_len,
                                          int max_rir_len) {
    RvGeom g;
    g.rlen = prep_rir_len(rparams, b);
    g.roff = g.rlen ? rparams[2 * b] : 0;
    g.valid = g.rlen != 0 && prep_rir_valid(rparams, b, bank_len, max_rir_len) && it.new_len >= 0 && it.new_len <= max_new_len;
    g.nx = (max(it.new_len, 0) + RV_P - 1) / RV_P + 1;
    g.nj = (g.rlen + RV_P - 1) / RV_P;
    g.ly = max(it.new_len, 0) + g.rlen - 1;
    g.nm = (g.ly + RV_P - 1) / RV_P;
    return g;
}

// two radix-16 passes of the 256-point complex FFT on 16 lanes (fft512.cuh): v in natural order per lane -> v[r] = Z[q + 16 k2(r)]
__device__ __forceinline__ void rv_fft256(float2 (&v)[16], float2* scr, const float2* tw, int q) {
    fft16(v);
#pragma unroll
    for (int r = 0; r < 16; ++r) {
        const int k1 = fb_k_of_slot(r);
        scr[k1 * 17 + q] = k1 == 0 ? v[r] : cmul(v[r], tw[k1 * 16 + q]);
    }
    __syncwarp();
#pragma unroll
    for (int n2 = 0; n2 < 16; ++n2) v[n2] = scr[q * 17 + n2];
    fft16(v);
    __syncwarp();
}

// forward transforms: blockIdx.z = 0 the input blocks X_i of the mixed signal, 1 the response partitions H_j
__global__ void __launch_bounds__(256) rv_forward_kernel(const float* __restrict__ wav, int64_t wav_ld, const int32_t* __restrict__ ip,
                                                         const float* __restrict__ fp, const float* __restrict__ noise,
                                                         const float* __restrict__ gains, const float* __restrict__ rir, int64_t bank_len,
                                                         const int32_t* __restrict__ rparams, int max_new_len, int max_rir_len, int NX,
                                                         int NJ, float2* __restrict__ xspec, float2* __restrict__ hspec) {
    __shared__ float2 s_tw[256], s_tw512[256];
    __shared__ float2 s_scr[RV_FRAMES][RV_SCR];
    const int b = blockIdx.y, resp = blockIdx.z;
    const PrepItem it = prep_load_item(ip, fp, b);
    const RvGeom g = rv_geom(it, rparams, b, bank_len, max_new_len, max_rir_len);
    const int nblk = resp ? g.nj : g.nx;
    const int f0 = blockIdx.x * RV_FRAMES;
    if (!g.valid || f0 >= nblk) return;
    fft_twiddle_tables(s_tw, s_tw512);
    __syncthreads();
    const int q = threadIdx.x & 15, fl = threadIdx.x >> 4, f = f0 + fl;  // idle frames (f >= nblk) compute zeros, unseen
    const float* x = wav + int64_t(b) * wav_ld;
    const float gs = gains[2 * b], gn = gains[2 * b + 1];
    auto sample = [&](int u) -> float {  // sample u of frame f's 512-point window
        if (resp) {
            const int j = f * RV_P + u;
            return (u < RV_P && j < g.rlen) ? rir[g.roff + j] * RV_H_SCALE : 0.f;
        }
        const int j = (f - 1) * RV_P + u;
        return (j >= 0 && j < it.new_len) ? prep_mixed_sample(x, noise, it, j, gs, gn) : 0.f;
    };
    float2 v[16];
#pragma unroll
    for (int n1 = 0; n1 < 16; ++n1) v[n1] = make_float2(sample(32 * n1 + 2 * q), sample(32 * n1 + 2 * q + 1));
    float2* scr = s_scr[fl];
    rv_fft256(v, scr, s_tw, q);
#pragma unroll
    for (int r = 0; r < 16; ++r) scr[q + 16 * fb_k_of_slot(r)] = v[r];
    __syncwarp();
    if (f >= nblk) return;
    float2* dst = resp ? hspec + (int64_t(b) * NJ + f) * RV_P : xspec + (int64_t(b) * NX + f) * RV_P;
    // 2 X[k] = 2F + W^k 2G, 2F = Z_k + conj Z_{256-k}, 2G = -i (Z_k - conj Z_{256-k}); k = 0 packs (2 X_0, 2 X_256)
#pragma unroll
    for (int i = 0; i < 16; ++i) {
        const int k = q + 16 * i;
        const float2 zk = scr[k], zn = scr[(RV_P - k) & (RV_P - 1)];
        const float2 fr = make_float2(zk.x + zn.x, zk.y - zn.y);
        const float2 gg = make_float2(zk.y + zn.y, zn.x - zk.x);
        if (k == 0) {
            dst[0] = make_float2(fr.x + gg.x, fr.x - gg.x);
        } else {
            const float2 wg = cmul(s_tw512[k], gg);
            dst[k] = make_float2(fr.x + wg.x, fr.y + wg.y);
        }
    }
}

// output blocks m0 .. m0 + RV_TM - 1 of one item: per bin k (= thread) accumulate sum_j X_{m-j} H_j with a register window over the
// X blocks, then one inverse transform per output block on 16 lanes
__global__ void __launch_bounds__(256) rv_conv_kernel(const int32_t* __restrict__ ip, const float* __restrict__ fp,
                                                      const int32_t* __restrict__ rparams, int64_t bank_len, int max_new_len,
                                                      int max_rir_len, int NX, int NJ, int NM, const float2* __restrict__ xspec,
                                                      const float2* __restrict__ hspec, int normalize, int Lout, float* __restrict__ out,
                                                      double* __restrict__ ypart) {
    __shared__ float2 s_tw[256], s_tw512[256];
    __shared__ float2 s_y[RV_TM][RV_SCR];
    const int b = blockIdx.y;
    const PrepItem it = prep_load_item(ip, fp, b);
    const RvGeom g = rv_geom(it, rparams, b, bank_len, max_new_len, max_rir_len);
    const int m0 = blockIdx.x * RV_TM;
    if (!g.valid || m0 >= g.nm) return;
    const int cs = max(it.crop_start, 0), ce = min(it.crop_start + min(it.crop_len, Lout), g.ly);  // [cs, ce): the crop window
    // without normalisation only the crop window matters: tiles outside it have nothing to write
    if (!normalize && (ce <= m0 * RV_P || cs >= (m0 + RV_TM) * RV_P)) return;
    fft_twiddle_tables(s_tw, s_tw512);

    const int k = threadIdx.x;
    const float2* xs = xspec + int64_t(b) * NX * RV_P + k;
    const float2* hs = hspec + int64_t(b) * NJ * RV_P + k;
    auto ldx = [&](int i) { return (i >= 0 && i < g.nx) ? xs[int64_t(i) * RV_P] : make_float2(0.f, 0.f); };
    float2 acc[RV_TM], w[RV_TM];
    const int jlo = max(0, m0 - g.nx + 1), jhi = min(g.nj - 1, m0 + RV_TM - 1);
#pragma unroll
    for (int t = 0; t < RV_TM; ++t) {
        acc[t] = make_float2(0.f, 0.f);
        w[t] = ldx(m0 + t - jlo);  // w[t] = X_{m0 + t - j} at partition j
    }
    float2 h = jlo <= jhi ? hs[int64_t(jlo) * RV_P] : make_float2(0.f, 0.f), xn = ldx(m0 - jlo - 1);
    for (int j = jlo; j <= jhi; ++j) {
        const float2 hc = h, xc = xn;
        if (j < jhi) {
            h = hs[int64_t(j + 1) * RV_P];
            xn = ldx(m0 - j - 2);
        }
        // bin k > 0: complex product; bin 0 holds (X_0, X_256) x (H_0, H_256), both real: componentwise
        const float a = hc.x, bn = k ? -hc.y : 0.f, c = k ? hc.y : 0.f, d = k ? hc.x : hc.y;
#pragma unroll
        for (int t = 0; t < RV_TM; ++t) {
            acc[t].x = fmaf(w[t].x, a, fmaf(w[t].y, bn, acc[t].x));
            acc[t].y = fmaf(w[t].x, c, fmaf(w[t].y, d, acc[t].y));
        }
#pragma unroll
        for (int t = RV_TM - 1; t > 0; --t) w[t] = w[t - 1];
        w[0] = xc;
    }
#pragma unroll
    for (int t = 0; t < RV_TM; ++t) s_y[t][k] = acc[t];
    __syncthreads();

    // inverse: Z_k = (Y_k + conj Y_{256-k}) + i W^{-k} (Y_k - conj Y_{256-k}), z = conj(FFT256(conj Z)), y[2n] + i y[2n+1] = z[n];
    // the overlap-save output is y[256, 512) = z[128, 256)
    const int q = threadIdx.x & 15, t = threadIdx.x >> 4, m = m0 + t;
    float2* scr = s_y[t];
    float2 v[16];
#pragma unroll
    for (int n1 = 0; n1 < 16; ++n1) {
        const int kk = 16 * n1 + q;
        float2 z;
        if (kk == 0) {
            const float2 p = scr[0];
            z = make_float2(p.x + p.y, p.x - p.y);
        } else {
            const float2 yk = scr[kk], yn = scr[RV_P - kk];
            const float2 fr = make_float2(yk.x + yn.x, yk.y - yn.y), dd = make_float2(yk.x - yn.x, yk.y + yn.y);
            const float2 wc = s_tw512[kk];
            const float2 gg = make_float2(dd.x * wc.x + dd.y * wc.y, dd.y * wc.x - dd.x * wc.y);  // dd * conj(W^k)
            z = make_float2(fr.x - gg.y, fr.y + gg.x);
        }
        v[n1] = make_float2(z.x, -z.y);
    }
    __syncwarp();
    rv_fft256(v, scr, s_tw, q);
    double e = 0.0;
    float* dst = out + int64_t(b) * Lout;
#pragma unroll
    for (int r = 0; r < 16; ++r) {
        const int k2 = fb_k_of_slot(r);
        if (k2 < 8) continue;
        const int gi = m * RV_P + 2 * q + 32 * (k2 - 8);
        const float y0 = v[r].x, y1 = -v[r].y;
        if (gi < g.ly) e += double(y0) * double(y0);
        if (gi + 1 < g.ly) e += double(y1) * double(y1);
        if (gi >= cs && gi < ce) dst[gi - it.crop_start] = y0;
        if (gi + 1 >= cs && gi + 1 < ce) dst[gi + 1 - it.crop_start] = y1;
    }
#pragma unroll
    for (int o = 8; o > 0; o >>= 1) e += __shfl_xor_sync(0xffffffffu, e, o);  // within the 16 lanes of this block: fixed order
    if (q == 0 && m < g.nm) ypart[int64_t(b) * NM + m] = e;
}

// reverb items: gains[2b] = the dB normalisation gain of y (1 without normalisation; NaN for an out-of-range entry)
__global__ void __launch_bounds__(256) rv_norm_kernel(const int32_t* __restrict__ ip, const float* __restrict__ fp,
                                                      const int32_t* __restrict__ rparams, int64_t bank_len, int max_new_len,
                                                      int max_rir_len, int NM, const double* __restrict__ ypart, float target_db,
                                                      int normalize, float* __restrict__ gains) {
    __shared__ double red[8];
    const int b = blockIdx.x;
    const PrepItem it = prep_load_item(ip, fp, b);
    const RvGeom g = rv_geom(it, rparams, b, bank_len, max_new_len, max_rir_len);
    if (g.rlen == 0) return;
    if (!g.valid) {
        if (threadIdx.x == 0) gains[2 * b] = __int_as_float(0x7fffffff);
        return;
    }
    if (!normalize) {
        if (threadIdx.x == 0) gains[2 * b] = 1.f;
        return;
    }
    double s = 0.0;
    for (int m = threadIdx.x; m < g.nm; m += blockDim.x) s += ypart[int64_t(b) * NM + m];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = s;
    __syncthreads();
    if (threadIdx.x == 0) {
        double tot = 0.0;
        for (int w = 0; w < 8; ++w) tot += red[w];  // fixed order: deterministic
        const double ms = tot / double(max(g.ly, 1));
        double gnorm = 1.0;
        if (ms > 0.0) gnorm = pow(10.0, fmin(double(target_db) - 10.0 * log10(ms), 300.0) / 20.0);
        gains[2 * b] = float(gnorm);
    }
}

struct RvLayout {  // blocks per item at the batch's maximum lengths: signal blocks, response partitions, output blocks
    int nx, nj, nm;
};

RvLayout rv_layout(int max_new_len, int max_rir_len) {
    RvLayout L;
    L.nx = (max_new_len + RV_P - 1) / RV_P + 1;
    L.nj = (max_rir_len + RV_P - 1) / RV_P;
    L.nm = int((int64_t(max_new_len) + max_rir_len - 1 + RV_P - 1) / RV_P);
    return L;
}

}  // namespace

void carve_reverb(WsCarver& cv, int B, int max_new_len, int max_rir_len, ReverbViews* v) {
    const RvLayout L = rv_layout(max_new_len, max_rir_len);
    v->ypart = static_cast<double*>(cv.take(size_t(B) * L.nm * sizeof(double)));
    v->xspec = static_cast<float2*>(cv.take(size_t(B) * L.nx * RV_P * sizeof(float2)));
    v->hspec = static_cast<float2*>(cv.take(size_t(B) * L.nj * RV_P * sizeof(float2)));
}

int reverb_run(const float* wav, int64_t wav_ld, const int32_t* iparams, const float* fparams, const float* noise, const float* rir_bank,
               int64_t rir_bank_len, const int32_t* rparams, int B, int max_new_len, int max_rir_len, float target_db, int normalize,
               int Lout, float* out, float* gains, const ReverbViews& v, cudaStream_t st) {
    const RvLayout L = rv_layout(max_new_len, max_rir_len);
    const int fx = (std::max(L.nx, L.nj) + RV_FRAMES - 1) / RV_FRAMES;
    rv_forward_kernel<<<dim3(fx, B, 2), 256, 0, st>>>(wav, wav_ld, iparams, fparams, noise, gains, rir_bank, rir_bank_len, rparams, max_new_len,
                                                      max_rir_len, L.nx, L.nj, v.xspec, v.hspec);
    rv_conv_kernel<<<dim3((L.nm + RV_TM - 1) / RV_TM, B), 256, 0, st>>>(iparams, fparams, rparams, rir_bank_len, max_new_len, max_rir_len, L.nx,
                                                                        L.nj, L.nm, v.xspec, v.hspec, normalize, Lout, out, v.ypart);
    rv_norm_kernel<<<B, 256, 0, st>>>(iparams, fparams, rparams, rir_bank_len, max_new_len, max_rir_len, L.nm, v.ypart, target_db, normalize,
                                      gains);
    PPV_LAUNCH_OK("reverb kernels");
    return PPV_OK;
}

}  // namespace ppv
