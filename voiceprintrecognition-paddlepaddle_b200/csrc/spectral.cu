// STFT front ends of the reference other than Kaldi Fbank: Spectrogram, MelSpectrogram, LogMelSpectrogram, MFCC
// (ppvector/data_utils/featurizer.py:20-27 -> paddle.audio.features.*, un-vendored; algorithm = the library's published one:
// centred, reflect-padded STFT with a periodic hann window -> |X|^power -> slaney/htk mel filterbank -> 10 log10(max(amin, .))
// - 10 log10(max(amin, ref)) -> DCT-II (ortho)), followed by AudioFeaturizer.forward's transpose / time-mean subtraction /
// tail mask (featurizer.py:43-59), and SpecAugment masking (ppvector/data_utils/reader.py:105-107).
//
// One CTA owns one frame: windowed samples -> shared memory (bit-reversed) -> radix-2 FFT in shared memory -> power ->
// sparse mel rows -> log -> DCT, all without touching HBM in between.  HBM traffic is the waveform (read ~n_fft/hop times,
// from L2 after the first) and the [B,T,F] feature (written once, then one read-modify-write pass for the mean).
#include <math.h>

#include <vector>

#include "common.h"
#include "fft_radix2.cuh"
#include "ptx.cuh"

namespace ppv {

constexpr int SP_MAX_NFFT = 4096;
constexpr int SP_THREADS = 256;

struct Spectral {
    ppv_spectral_cfg cfg;
    int n_fft = 0, log2n = 0, hop = 0, n_bins = 0, F = 0;
    float* window = nullptr;   // [n_fft] (win_length window centred in n_fft)
    float2* twiddle = nullptr; // [n_fft/2] exp(-2 pi i k / n_fft)
    float* mel_w = nullptr;    // [nnz]
    int* mel_start = nullptr;  // [n_mels]
    int* mel_len = nullptr;
    int* mel_off = nullptr;
    float* dct = nullptr;      // [n_mels][n_mfcc]
    float log_ref = 0.f;       // 10 log10(max(amin, ref_value))
};

struct SpecKernelArgs {
    const float* window;
    const float2* twiddle;
    const float* mel_w;
    const int* mel_start;
    const int* mel_len;
    const int* mel_off;
    const float* dct;
    int n_fft, log2n, hop, n_bins, method, n_mels, n_mfcc, center;
    float power, amin, log_ref;
};

__device__ __forceinline__ int sp_reflect(int i, int L) {  // numpy 'reflect' (no edge repeat); valid for |overhang| < L
    if (i < 0) i = -i;
    if (i >= L) i = 2 * (L - 1) - i;
    return i;
}

// out_raw [B, T, F].  Ragged batches (both optional, nullptr: every row is L samples / T frames): row b is num_samples[b] samples
// long, reflected at its own right edge when centred, and only its first valid_frames[b] frames are computed.  Both are clamped
// ([1, L] and [0, T]) and every index stays inside the row, so a wrong length gives wrong features for that row, never a fault.
__global__ void __launch_bounds__(SP_THREADS) spectral_frame_kernel(const float* __restrict__ wav, int L, int T, int F, SpecKernelArgs a,
                                                                    const int* __restrict__ num_samples, const int* __restrict__ valid_frames,
                                                                    float* __restrict__ out_raw) {
    extern __shared__ __align__(16) uint8_t sp_smem[];
    float2* z = reinterpret_cast<float2*>(sp_smem);              // n_fft
    float* pw = reinterpret_cast<float*>(z + a.n_fft);           // n_bins
    float* melv = pw + a.n_bins;                                 // n_mels
    griddep_launch_dependents();
    griddep_wait();
    const int t = blockIdx.x, b = blockIdx.y;
    if (valid_frames && t >= min(max(valid_frames[b], 0), T)) return;
    const int Lb = num_samples ? min(max(num_samples[b], 1), L) : L;
    const float* x = wav + int64_t(b) * L;
    const int N = a.n_fft;
    const int start = t * a.hop - (a.center ? N / 2 : 0);
    for (int i = threadIdx.x; i < N; i += SP_THREADS) {
        // centred: an identity clamp whenever Lb > N / 2 frames it; non-centred: t < T keeps [start, start + N) inside [0, L)
        const int src = a.center ? min(max(sp_reflect(start + i, Lb), 0), Lb - 1) : start + i;
        z[fft_bitrev(i, a.log2n)] = make_float2(x[src] * a.window[i], 0.f);
    }
    __syncthreads();
    fft_radix2(z, a.log2n, 1, a.twiddle);
    float* dst = out_raw + (int64_t(b) * T + t) * F;
    for (int k = threadIdx.x; k < a.n_bins; k += SP_THREADS) {
        const float m2 = z[k].x * z[k].x + z[k].y * z[k].y;
        const float p = a.power == 2.f ? m2 : a.power == 1.f ? sqrtf(m2) : powf(m2, 0.5f * a.power);
        if (a.method == PPV_SPEC_SPECTROGRAM)
            dst[k] = p;
        else
            pw[k] = p;
    }
    if (a.method == PPV_SPEC_SPECTROGRAM) return;
    __syncthreads();
    for (int m = threadIdx.x; m < a.n_mels; m += SP_THREADS) {
        const int k0 = a.mel_start[m], n = a.mel_len[m];
        const float* w = a.mel_w + a.mel_off[m];
        float acc = 0.f;
        for (int k = 0; k < n; ++k) acc = fmaf(w[k], pw[k0 + k], acc);
        if (a.method != PPV_SPEC_MEL) acc = 10.f * log10f(fmaxf(a.amin, acc)) - a.log_ref;
        if (a.method == PPV_SPEC_MFCC)
            melv[m] = acc;
        else
            dst[m] = acc;
    }
    if (a.method != PPV_SPEC_MFCC) return;
    __syncthreads();
    for (int c = threadIdx.x; c < a.n_mfcc; c += SP_THREADS) {
        float acc = 0.f;
        for (int m = 0; m < a.n_mels; ++m) acc = fmaf(__ldg(a.dct + m * a.n_mfcc + c), melv[m], acc);
        dst[c] = acc;
    }
}

// In place: x[b, t, f] -= mean_t x[b, :, f]; frames t >= int(ratio[b] * T) are zeroed after it (featurizer.py:48-59).
// Ragged batches (valid_frames, optional): the mean of row b runs over its first Tb = valid_frames[b] frames (clamped to [0, T]) in
// the order of a call on that utterance alone, so the row is bitwise what that call gives; frames Tb .. T - 1 are written as zeros
// without being read.  Block = (32-feature slab, utterance): 8 warps stride over time, lane = feature.
__global__ void __launch_bounds__(256) spectral_cmn_kernel(float* __restrict__ x, const float* __restrict__ lens_ratio,
                                                           const int* __restrict__ valid_frames, int T, int F) {
    __shared__ float s_part[8][32];
    griddep_launch_dependents();
    griddep_wait();
    const int b = blockIdx.y, f = blockIdx.x * 32 + (threadIdx.x & 31), warp = threadIdx.x >> 5;
    const int Tb = valid_frames ? min(max(valid_frames[b], 0), T) : T;
    float* base = x + int64_t(b) * T * F;
    float acc = 0.f;
    if (f < F)
        for (int t = warp; t < Tb; t += 8) acc += base[int64_t(t) * F + f];
    s_part[warp][threadIdx.x & 31] = acc;
    __syncthreads();
    float mean = 0.f;
#pragma unroll
    for (int w = 0; w < 8; ++w) mean += s_part[w][threadIdx.x & 31];
    mean /= float(max(Tb, 1));
    const int keep = min(lens_ratio ? int(lens_ratio[b] * float(T)) : T, Tb);
    if (f < F)
        for (int t = warp; t < T; t += 8) base[int64_t(t) * F + f] = t < keep ? base[int64_t(t) * F + f] - mean : 0.f;
}

// SpecAugment masks (reader.py:105-107, configs/augmentation.yml:36-48; max_time_warp 0).  params [B][PPV_SPECAUG_NPARAM] int32:
// {apply, T_b (frames of this utterance), then n_freq x (f0, width), then n_time x (t0, width)} drawn by the host with the
// reference's RNG calls.  fill_mode 0: zeros; 1: the utterance's mean over its T_b x F values BEFORE masking.
__global__ void __launch_bounds__(256) specaug_kernel(float* __restrict__ x, const int* __restrict__ params, int T, int F, int n_freq, int n_time,
                                                      int fill_mode) {
    __shared__ float s_red[8];
    __shared__ float s_fill;
    const int b = blockIdx.x;
    const int* p = params + int64_t(b) * PPV_SPECAUG_NPARAM;
    if (!p[0]) return;
    const int Tb = min(max(p[1], 0), T);
    float* base = x + int64_t(b) * T * F;
    float fill = 0.f;
    if (fill_mode == 1) {
        float acc = 0.f;
        for (int64_t i = threadIdx.x; i < int64_t(Tb) * F; i += 256) acc += base[i];
        for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
        if ((threadIdx.x & 31) == 0) s_red[threadIdx.x >> 5] = acc;
        __syncthreads();
        if (threadIdx.x == 0) {
            float s = 0.f;
            for (int w = 0; w < 8; ++w) s += s_red[w];
            s_fill = Tb > 0 ? s / (float(Tb) * float(F)) : 0.f;
        }
        __syncthreads();
        fill = s_fill;
    }
    for (int i = 0; i < n_freq; ++i) {
        const int f0 = p[2 + 2 * i], fw = p[3 + 2 * i];
        for (int64_t j = threadIdx.x; j < int64_t(Tb) * fw; j += 256) {
            const int t = int(j / fw), f = f0 + int(j % fw);
            if (f >= 0 && f < F) base[int64_t(t) * F + f] = fill;
        }
    }
    __syncthreads();
    for (int i = 0; i < n_time; ++i) {
        const int t0 = p[2 + 2 * n_freq + 2 * i], tw = p[3 + 2 * n_freq + 2 * i];
        for (int64_t j = threadIdx.x; j < int64_t(tw) * F; j += 256) {
            const int t = t0 + int(j / F);
            if (t >= 0 && t < Tb) base[int64_t(t) * F + int(j % F)] = fill;
        }
    }
}

// ------------------------------------------------------------------------------------------------ host
template <typename T>
static int sp_upload(T** dst, const std::vector<T>& v) {
    PPV_CUDA_OK(cudaMalloc(reinterpret_cast<void**>(dst), std::max<size_t>(v.size(), 1) * sizeof(T)));
    if (!v.empty()) PPV_CUDA_OK(cudaMemcpy(*dst, v.data(), v.size() * sizeof(T), cudaMemcpyHostToDevice));
    return PPV_OK;
}

static double sp_hz_to_mel(double f, bool htk) {
    if (htk) return 2595.0 * log10(1.0 + f / 700.0);
    const double f_sp = 200.0 / 3.0, min_log_hz = 1000.0, min_log_mel = min_log_hz / f_sp, logstep = log(6.4) / 27.0;
    return f >= min_log_hz ? min_log_mel + log(f / min_log_hz) / logstep : f / f_sp;
}
static double sp_mel_to_hz(double m, bool htk) {
    if (htk) return 700.0 * (pow(10.0, m / 2595.0) - 1.0);
    const double f_sp = 200.0 / 3.0, min_log_hz = 1000.0, min_log_mel = min_log_hz / f_sp, logstep = log(6.4) / 27.0;
    return m >= min_log_mel ? min_log_hz * exp(logstep * (m - min_log_mel)) : f_sp * m;
}

void spectral_default_cfg(ppv_spectral_cfg* c, int method) {
    c->method = method;
    c->sample_rate = 22050;
    c->n_fft = method == PPV_SPEC_SPECTROGRAM ? 512 : 2048;
    c->hop_length = 512;
    c->win_length = 0;
    c->power = method == PPV_SPEC_SPECTROGRAM ? 1.f : 2.f;
    c->center = 1;
    c->n_mels = 64;
    c->f_min = 50.f;
    c->f_max = 0.f;
    c->htk = 0;
    c->norm_slaney = 1;
    c->ref_value = 1.f;
    c->amin = 1e-10f;
    c->n_mfcc = 40;
}

void spectral_destroy(Spectral* h) {
    if (!h) return;
    cudaFree(h->window);
    cudaFree(h->twiddle);
    cudaFree(h->mel_w);
    cudaFree(h->mel_start);
    cudaFree(h->mel_len);
    cudaFree(h->mel_off);
    cudaFree(h->dct);
    delete h;
}

int spectral_create(const ppv_spectral_cfg* cfg, Spectral** out) {
    PPV_REQUIRE(cfg && out, "spectral_create: null argument");
    if (cfg->method < PPV_SPEC_SPECTROGRAM || cfg->method > PPV_SPEC_MFCC) return fail(PPV_EINVAL, "spectral: unknown method");
    int log2n = 0;
    while ((1 << log2n) < cfg->n_fft) ++log2n;
    if (cfg->n_fft < 32 || cfg->n_fft > SP_MAX_NFFT || (1 << log2n) != cfg->n_fft)
        return fail(PPV_EUNSUPPORTED, "spectral: n_fft must be a power of two in [32, 4096]");
    const int win = cfg->win_length > 0 ? cfg->win_length : cfg->n_fft;
    if (win > cfg->n_fft || cfg->hop_length <= 0) return fail(PPV_EINVAL, "spectral: win_length <= n_fft and hop_length > 0 required");
    if (!(cfg->power > 0.f) || !(cfg->amin > 0.f)) return fail(PPV_EINVAL, "spectral: power > 0 and amin > 0 required");
    Spectral* h = new Spectral();
    h->cfg = *cfg;
    h->n_fft = cfg->n_fft;
    h->log2n = log2n;
    h->hop = cfg->hop_length;
    h->n_bins = cfg->n_fft / 2 + 1;
    const int N = cfg->n_fft;
    // periodic hann of win_length, zero-padded symmetrically to n_fft (paddle.signal.stft)
    std::vector<float> window(N, 0.f);
    const int lpad = (N - win) / 2;
    for (int i = 0; i < win; ++i) window[lpad + i] = float(0.5 - 0.5 * cos(2.0 * M_PI * i / win));
    std::vector<float2> tw(N / 2);
    for (int k = 0; k < N / 2; ++k) tw[k] = make_float2(float(cos(-2.0 * M_PI * k / N)), float(sin(-2.0 * M_PI * k / N)));
    std::vector<float> melw, dct;
    std::vector<int> mstart, mlen, moff;
    h->F = h->n_bins;
    if (cfg->method != PPV_SPEC_SPECTROGRAM) {
        const int nm = cfg->n_mels;
        const double fmax = cfg->f_max > 0.f ? cfg->f_max : 0.5 * cfg->sample_rate;
        if (nm < 1 || nm > 512 || !(cfg->f_min >= 0.f) || !(fmax > cfg->f_min)) {
            delete h;
            return fail(PPV_EINVAL, "spectral: bad n_mels / f_min / f_max");
        }
        // compute_fbank_matrix (librosa-style): triangular filters on the mel scale, slaney area normalisation
        const bool htk = cfg->htk != 0;
        const double m_lo = sp_hz_to_mel(cfg->f_min, htk), m_hi = sp_hz_to_mel(fmax, htk);
        std::vector<double> mel_f(nm + 2);
        for (int i = 0; i < nm + 2; ++i) mel_f[i] = sp_mel_to_hz(m_lo + (m_hi - m_lo) * i / (nm + 1), htk);
        mstart.resize(nm);
        mlen.resize(nm);
        moff.resize(nm);
        for (int m = 0; m < nm; ++m) {
            const double fd0 = mel_f[m + 1] - mel_f[m], fd1 = mel_f[m + 2] - mel_f[m + 1];
            const double enorm = cfg->norm_slaney ? 2.0 / (mel_f[m + 2] - mel_f[m]) : 1.0;
            int first = -1, last = -1;
            std::vector<float> row(h->n_bins, 0.f);
            for (int k = 0; k < h->n_bins; ++k) {
                const double fk = 0.5 * cfg->sample_rate * k / (h->n_bins - 1);
                const double lower = (fk - mel_f[m]) / fd0, upper = (mel_f[m + 2] - fk) / fd1;
                const double w = std::max(0.0, std::min(lower, upper)) * enorm;
                row[k] = float(w);
                if (w > 0.0) {
                    if (first < 0) first = k;
                    last = k;
                }
            }
            mstart[m] = first < 0 ? 0 : first;
            mlen[m] = first < 0 ? 0 : last - first + 1;
            moff[m] = int(melw.size());
            for (int k = 0; k < mlen[m]; ++k) melw.push_back(row[mstart[m] + k]);
        }
        h->F = nm;
        if (cfg->method == PPV_SPEC_MFCC) {
            const int nc = cfg->n_mfcc;
            if (nc < 1 || nc > nm) {
                delete h;
                return fail(PPV_EINVAL, "spectral: 1 <= n_mfcc <= n_mels required");
            }
            dct.resize(size_t(nm) * nc);  // create_dct(norm='ortho'): [n_mels][n_mfcc]
            for (int c = 0; c < nc; ++c)
                for (int m = 0; m < nm; ++m) {
                    double v = cos(M_PI / nm * (m + 0.5) * c) * sqrt(2.0 / nm);
                    if (c == 0) v *= 1.0 / sqrt(2.0);
                    dct[size_t(m) * nc + c] = float(v);
                }
            h->F = nc;
        }
        h->log_ref = float(10.0 * log10(std::max(double(cfg->amin), double(cfg->ref_value))));
    }
    int rc = sp_upload(&h->window, window);
    if (!rc) rc = sp_upload(&h->twiddle, tw);
    if (!rc) rc = sp_upload(&h->mel_w, melw);
    if (!rc) rc = sp_upload(&h->mel_start, mstart);
    if (!rc) rc = sp_upload(&h->mel_len, mlen);
    if (!rc) rc = sp_upload(&h->mel_off, moff);
    if (!rc) rc = sp_upload(&h->dct, dct);
    if (rc) {
        spectral_destroy(h);
        return rc;
    }
    *out = h;
    return PPV_OK;
}

int spectral_num_frames(const Spectral* h, int L) {
    if (h->cfg.center) return L > h->n_fft / 2 ? 1 + L / h->hop : 0;  // reflect padding needs L > n_fft / 2
    return L >= h->n_fft ? 1 + (L - h->n_fft) / h->hop : 0;
}
int spectral_feature_dim(const Spectral* h) { return h->F; }

int spectral_run(Spectral* h, const float* wav, const float* lens_ratio, int B, int L, float* out, cudaStream_t st, const int* valid_frames,
                 const int* num_samples) {
    PPV_REQUIRE(h && wav && out, "spectral_run: null argument");
    PPV_REQUIRE(B > 0 && B <= 65535, "spectral_run: batch must be in [1, 65535]");
    const int T = spectral_num_frames(h, L);
    PPV_REQUIRE(T > 0, "spectral_run: waveform too short for one frame");
    SpecKernelArgs a;
    a.window = h->window;
    a.twiddle = h->twiddle;
    a.mel_w = h->mel_w;
    a.mel_start = h->mel_start;
    a.mel_len = h->mel_len;
    a.mel_off = h->mel_off;
    a.dct = h->dct;
    a.n_fft = h->n_fft;
    a.log2n = h->log2n;
    a.hop = h->hop;
    a.n_bins = h->n_bins;
    a.method = h->cfg.method;
    a.n_mels = h->cfg.n_mels;
    a.n_mfcc = h->cfg.n_mfcc;
    a.center = h->cfg.center;
    a.power = h->cfg.power;
    a.amin = h->cfg.amin;
    a.log_ref = h->log_ref;
    const size_t smem = size_t(h->n_fft) * sizeof(float2) + size_t(h->n_bins) * sizeof(float) + 512 * sizeof(float);
    PPV_ONCE_PER_DEVICE(PPV_CUDA_OK(cudaFuncSetAttribute(spectral_frame_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 64 * 1024)));
    PPV_REQUIRE(smem <= 64 * 1024, "spectral_run: shared memory budget exceeded");
    PPV_PDL_OK(launch_pdl(spectral_frame_kernel, dim3(T, B), dim3(SP_THREADS), smem, st, wav, L, T, h->F, a, num_samples, valid_frames, out),
               "spectral_frame_kernel");
    PPV_PDL_OK(launch_pdl(spectral_cmn_kernel, dim3((h->F + 31) / 32, B), dim3(256), 0, st, out, lens_ratio, valid_frames, T, h->F),
               "spectral_cmn_kernel");
    return PPV_OK;
}

int spec_augment_run(float* feat, const int32_t* params, int B, int T, int F, int n_freq_masks, int n_time_masks, int fill_mode, cudaStream_t st) {
    PPV_REQUIRE(feat && params, "spec_augment: null argument");
    PPV_REQUIRE(B > 0 && T > 0 && F > 0, "spec_augment: empty batch");
    PPV_REQUIRE(n_freq_masks >= 0 && n_time_masks >= 0 && 2 + 2 * (n_freq_masks + n_time_masks) <= PPV_SPECAUG_NPARAM,
                "spec_augment: too many masks for PPV_SPECAUG_NPARAM");
    PPV_REQUIRE(fill_mode == 0 || fill_mode == 1, "spec_augment: fill_mode must be 0 (zeros) or 1 (utterance mean)");
    specaug_kernel<<<B, 256, 0, st>>>(feat, params, T, F, n_freq_masks, n_time_masks, fill_mode);
    PPV_LAUNCH_OK("specaug_kernel");
    return PPV_OK;
}

}  // namespace ppv
