// Batched waveform preparation in front of the feature extractor: speed perturbation -> volume perturbation -> additive noise at a
// drawn SNR -> dB normalisation -> crop / zero-pad, one launch sequence per BATCH.
// Reference: ppvector/data_utils/reader.py:85-104 (resample, augment_audio :153-163, normalize(target_db), crop) -- per utterance, on
// the CPU, inside DataLoader workers, through the un-vendored yeaudio package; configs/augmentation.yml:1-33.  The semantics below
// are RECALLED yeaudio behaviour (SURVEY.md §8c-6; restated in oracle/audio_prep.py), the random draws stay on the host:
//   speed   change_speed(r): new_len = int(len / r), samples = np.interp(linspace(0, len, new_len), arange(len), samples)
//   volume  samples *= 10^(gain_dB / 20)
//   noise   noise gain = min(rms_dB(signal) - rms_dB(noise) - snr_dB, 300) dB; samples += noise * gain (noise tiled over the utterance)
//   reverb  samples = fftconvolve(samples, rir, "full"): new_len + R - 1 samples, response not normalised (audio_prep_reverb only)
//   norm    gain = min(target_dB - rms_dB(samples), 300) dB over the WHOLE utterance (before the crop), rms_dB = 10 log10(mean x^2)
//   crop    [start, start + crop_len) of the result, zero-padded to the batch's output length
// Two passes over the samples: (1) per-utterance sums  S_xx, S_nn, S_xn  of the speed-changed signal and its noise segment, from
// which every gain follows in closed form (the mixture's energy is g^2 S_xx + 2 g g_n S_xn + g_n^2 S_nn); (2) the output.  HBM-bound:
// ~2 reads of the raw samples + 1 write of the crop.  Items with a room response take the volume and noise gains from pass 1, and their
// normalisation from the energy of the reverberant signal, which reverb.cu computes between the two passes.
#include <math.h>

#include "audio_prep.cuh"
#include "common.h"
#include "ptx.cuh"

namespace ppv {

namespace {

constexpr int AP_CHUNK = 8192;  // samples per block in pass 1

__global__ void __launch_bounds__(256) prep_stats_kernel(const float* __restrict__ wav, int64_t wav_ld, const int32_t* __restrict__ ip,
                                                         const float* __restrict__ fp, const float* __restrict__ noise, int nchunk,
                                                         double* __restrict__ partial) {
    __shared__ double red[3][8];
    const int b = blockIdx.y, chunk = blockIdx.x;
    const PrepItem it = prep_load_item(ip, fp, b);
    const float* x = wav + int64_t(b) * wav_ld;
    double sxx = 0.0, snn = 0.0, sxn = 0.0;
    const int j0 = chunk * AP_CHUNK, j1 = min(it.new_len, j0 + AP_CHUNK);
    for (int j = j0 + threadIdx.x; j < j1; j += blockDim.x) {
        const float v = prep_speed_sample(x, it, j);
        sxx += double(v) * double(v);
        if (it.has_noise) {
            const float n = noise[it.noise_off + (j % it.noise_len)];
            snn += double(n) * double(n);
            sxn += double(v) * double(n);
        }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        sxx += __shfl_xor_sync(0xffffffffu, sxx, o);
        snn += __shfl_xor_sync(0xffffffffu, snn, o);
        sxn += __shfl_xor_sync(0xffffffffu, sxn, o);
    }
    if ((threadIdx.x & 31) == 0) {
        red[0][threadIdx.x >> 5] = sxx;
        red[1][threadIdx.x >> 5] = snn;
        red[2][threadIdx.x >> 5] = sxn;
    }
    __syncthreads();
    if (threadIdx.x < 3) {
        double s = 0.0;
        for (int w = 0; w < 8; ++w) s += red[threadIdx.x][w];  // fixed order: deterministic
        partial[(int64_t(b) * nchunk + chunk) * 3 + threadIdx.x] = s;
    }
}

// gains[b] = {signal gain, noise gain} including the dB normalisation -- except for items with a room response (rparams, may be null):
// their normalisation follows the convolution (reverb.cu)
__global__ void prep_gains_kernel(const int32_t* __restrict__ ip, const float* __restrict__ fp, const double* __restrict__ partial, int nchunk,
                                  int B, float target_db, int normalize, const int32_t* __restrict__ rparams, float* __restrict__ gains) {
    const int b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= B) return;
    const PrepItem it = prep_load_item(ip, fp, b);
    double sxx = 0.0, snn = 0.0, sxn = 0.0;
    const int used = (it.new_len + AP_CHUNK - 1) / AP_CHUNK;
    for (int c = 0; c < used; ++c) {
        sxx += partial[(int64_t(b) * nchunk + c) * 3 + 0];
        snn += partial[(int64_t(b) * nchunk + c) * 3 + 1];
        sxn += partial[(int64_t(b) * nchunk + c) * 3 + 2];
    }
    const double n = double(max(it.new_len, 1));
    const double g = pow(10.0, double(it.vol_gain_db) / 20.0);
    double gn = 0.0;
    if (it.has_noise && snn > 0.0 && sxx > 0.0) {
        const double sig_db = 10.0 * log10(g * g * sxx / n), noise_db = 10.0 * log10(snn / n);
        gn = pow(10.0, fmin(sig_db - noise_db - double(it.snr_db), 300.0) / 20.0);
    }
    double gnorm = 1.0;
    if (normalize && prep_rir_len(rparams, b) == 0) {
        const double ms = (g * g * sxx + 2.0 * g * gn * sxn + gn * gn * snn) / n;
        if (ms > 0.0) gnorm = pow(10.0, fmin(double(target_db) - 10.0 * log10(ms), 300.0) / 20.0);
    }
    gains[2 * b] = float(g * gnorm);
    gains[2 * b + 1] = float(gn * gnorm);
}

// out[b] = the crop window of the prepared signal, zero-padded to Lout.  Items with a room response (rparams, may be null) find their
// un-normalised reverberant crop window in out already (reverb.cu) and gains[2b] = its normalisation gain.
__global__ void __launch_bounds__(256) prep_apply_kernel(const float* __restrict__ wav, int64_t wav_ld, const int32_t* __restrict__ ip,
                                                         const float* __restrict__ fp, const float* __restrict__ noise,
                                                         const float* __restrict__ gains, const int32_t* __restrict__ rparams, int Lout,
                                                         float* __restrict__ out) {
    const int b = blockIdx.y;
    const PrepItem it = prep_load_item(ip, fp, b);
    const float* x = wav + int64_t(b) * wav_ld;
    const float gs = gains[2 * b], gn = gains[2 * b + 1];
    float* dst = out + int64_t(b) * Lout;
    const int rlen = prep_rir_len(rparams, b);
    if (rlen != 0) {
        const int ly = it.new_len + rlen - 1;
        for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < Lout; i += gridDim.x * blockDim.x)
            dst[i] = (i < it.crop_len && it.crop_start + i < ly) ? dst[i] * gs : 0.f;
        return;
    }
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < Lout; i += gridDim.x * blockDim.x) {
        float v = 0.f;
        if (i < it.crop_len) v = prep_mixed_sample(x, noise, it, it.crop_start + i, gs, gn);
        dst[i] = v;
    }
}

struct PrepWs {
    double* partial;  // [B][nchunk][3] per-chunk sums of pass 1
    float* gains;     // [B][2]
    ReverbViews rv;   // audio_prep_reverb only
};
// max_rir_len = 0: audio_prep's workspace; > 0: audio_prep_reverb's, the reverb views behind the shared ones
void carve_prep(WsCarver& cv, int B, int max_new_len, int max_rir_len, PrepWs* w) {
    const size_t nchunk = size_t((max_new_len + AP_CHUNK - 1) / AP_CHUNK);
    w->partial = static_cast<double*>(cv.take(size_t(B) * nchunk * 3 * sizeof(double)));
    w->gains = static_cast<float*>(cv.take(size_t(B) * 2 * sizeof(float)));
    if (max_rir_len > 0) carve_reverb(cv, B, max_new_len, max_rir_len, &w->rv);
}

}  // namespace

size_t audio_prep_workspace_bytes(int B, int max_new_len) {
    if (B <= 0 || max_new_len <= 0) return 0;
    return carve_extent([&](WsCarver& cv) { PrepWs w; carve_prep(cv, B, max_new_len, 0, &w); });
}

// wav [B][wav_ld] raw (resampled) samples; iparams [B][PPV_PREP_NI]; fparams [B][PPV_PREP_NF]; noise: concatenated noise clips (may be null
// when no item has noise); out [B][Lout].  max_new_len >= every item's new_len (sizes the workspace).
int audio_prep(const float* wav, int64_t wav_ld, const int32_t* iparams, const float* fparams, const float* noise, int B, int max_new_len,
               float target_db, int normalize, int Lout, float* out, void* ws, size_t ws_bytes, cudaStream_t st) {
    PPV_REQUIRE(wav && iparams && fparams && out, "audio_prep: null argument");
    PPV_REQUIRE(B > 0 && max_new_len > 0 && Lout > 0, "audio_prep: empty batch");
    if (int rc = check_workspace("audio_prep", ws, ws_bytes, audio_prep_workspace_bytes(B, max_new_len), "ppv_audio_prep_workspace_bytes")) return rc;
    WsCarver cv{static_cast<uint8_t*>(ws)};
    PrepWs w;
    carve_prep(cv, B, max_new_len, 0, &w);
    const int nchunk = (max_new_len + AP_CHUNK - 1) / AP_CHUNK;
    prep_stats_kernel<<<dim3(nchunk, B), 256, 0, st>>>(wav, wav_ld, iparams, fparams, noise, nchunk, w.partial);
    prep_gains_kernel<<<(B + 127) / 128, 128, 0, st>>>(iparams, fparams, w.partial, nchunk, B, target_db, normalize, nullptr, w.gains);
    const int gx = std::max(1, std::min((Lout + 255) / 256, 64));
    prep_apply_kernel<<<dim3(gx, B), 256, 0, st>>>(wav, wav_ld, iparams, fparams, noise, w.gains, nullptr, Lout, out);
    PPV_LAUNCH_OK("audio_prep kernels");
    return PPV_OK;
}

size_t audio_prep_reverb_workspace_bytes(int B, int max_new_len, int max_rir_len) {
    if (B <= 0 || max_new_len <= 0 || max_rir_len <= 0) return 0;
    return carve_extent([&](WsCarver& cv) { PrepWs w; carve_prep(cv, B, max_new_len, max_rir_len, &w); });
}

// audio_prep with reverberation after the noise: rparams [B][2] = {rir_off, rir_len} into rir_bank (rir_bank_len samples), rir_len 0 = no
// reverb for that item.  An item with a response has crop_start / crop_len on its reverberant length new_len + rir_len - 1.  Same stats
// and gains passes (reverb items leave the normalisation out), then reverb.cu's convolution and normalisation, then the same apply pass.
int audio_prep_reverb(const float* wav, int64_t wav_ld, const int32_t* iparams, const float* fparams, const float* noise, const float* rir_bank,
                      int64_t rir_bank_len, const int32_t* rparams, int B, int max_new_len, int max_rir_len, float target_db, int normalize,
                      int Lout, float* out, void* ws, size_t ws_bytes, cudaStream_t st) {
    PPV_REQUIRE(wav && iparams && fparams && rir_bank && rparams && out, "audio_prep_reverb: null argument");
    PPV_REQUIRE(B > 0 && max_new_len > 0 && Lout > 0, "audio_prep_reverb: empty batch");
    PPV_REQUIRE(max_rir_len > 0 && int64_t(max_rir_len) <= rir_bank_len, "audio_prep_reverb: max_rir_len outside [1, rir_bank_len]");
    PPV_REQUIRE(int64_t(max_new_len) + max_rir_len - 1 <= INT32_MAX - 512, "audio_prep_reverb: reverberant length exceeds int32");
    if (int rc = check_workspace("audio_prep_reverb", ws, ws_bytes, audio_prep_reverb_workspace_bytes(B, max_new_len, max_rir_len),
                                 "ppv_audio_prep_reverb_workspace_bytes")) return rc;
    WsCarver cv{static_cast<uint8_t*>(ws)};
    PrepWs w;
    carve_prep(cv, B, max_new_len, max_rir_len, &w);
    const int nchunk = (max_new_len + AP_CHUNK - 1) / AP_CHUNK;
    prep_stats_kernel<<<dim3(nchunk, B), 256, 0, st>>>(wav, wav_ld, iparams, fparams, noise, nchunk, w.partial);
    prep_gains_kernel<<<(B + 127) / 128, 128, 0, st>>>(iparams, fparams, w.partial, nchunk, B, target_db, normalize, rparams, w.gains);
    PPV_LAUNCH_OK("audio_prep_reverb stats / gains");
    const int rc = reverb_run(wav, wav_ld, iparams, fparams, noise, rir_bank, rir_bank_len, rparams, B, max_new_len, max_rir_len, target_db,
                              normalize, Lout, out, w.gains, w.rv, st);
    if (rc != PPV_OK) return rc;
    const int gx = std::max(1, std::min((Lout + 255) / 256, 64));
    prep_apply_kernel<<<dim3(gx, B), 256, 0, st>>>(wav, wav_ld, iparams, fparams, noise, w.gains, rparams, Lout, out);
    PPV_LAUNCH_OK("audio_prep_reverb apply");
    return PPV_OK;
}

}  // namespace ppv
