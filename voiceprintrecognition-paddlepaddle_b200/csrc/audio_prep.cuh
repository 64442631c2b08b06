// Per-utterance parameters and the pre-reverb sample expression of the batched audio preparation, shared by audio_prep.cu (stats /
// gains / apply) and reverb.cu (the convolution reads the mixed signal through the same expression the apply pass writes).
#pragma once
#include "common.h"

namespace ppv {

struct PrepItem {
    int raw_len, new_len, crop_start, crop_len, noise_off, noise_len, has_noise;
    float pos_step, vol_gain_db, snr_db;
};

__device__ __forceinline__ PrepItem prep_load_item(const int32_t* ip, const float* fp, int b) {
    PrepItem it;
    const int32_t* i = ip + b * PPV_PREP_NI;
    const float* f = fp + b * PPV_PREP_NF;
    it.raw_len = i[0];
    it.new_len = i[1];
    it.crop_start = i[2];
    it.crop_len = i[3];
    it.noise_off = i[4];
    it.noise_len = i[5];
    it.has_noise = i[6];
    it.pos_step = f[0];
    it.vol_gain_db = f[1];
    it.snr_db = f[2];
    return it;
}

// sample j of the speed-changed signal: np.interp(j * pos_step, arange(raw_len), x) with np.interp's clamping beyond the last index
__device__ __forceinline__ float prep_speed_sample(const float* __restrict__ x, const PrepItem& it, int j) {
    if (it.new_len == it.raw_len) return x[j];
    // linspace(0, raw_len, new_len)[j] in double (a float position loses the fraction beyond ~1e6 samples)
    const double pos = double(j) * (double(it.raw_len) / double(max(it.new_len - 1, 1)));
    int i0 = int(pos);
    if (i0 >= it.raw_len - 1) return x[it.raw_len - 1];
    const float fr = float(pos - double(i0));
    const float a = x[i0], c = x[i0 + 1];
    return a + fr * (c - a);
}

// sample j (< new_len) of the speed-changed, volume-scaled, noise-mixed signal: gs = signal gain, gn = noise gain
__device__ __forceinline__ float prep_mixed_sample(const float* __restrict__ x, const float* __restrict__ noise, const PrepItem& it, int j,
                                                   float gs, float gn) {
    float v = prep_speed_sample(x, it, j) * gs;
    if (it.has_noise) v = fmaf(noise[it.noise_off + (j % it.noise_len)], gn, v);
    return v;
}

// rparams[b] = {rir_off, rir_len}: a response of rir_len >= 1 samples at rir_bank[rir_off]; 0 = no reverb for this item.  An entry outside
// [0, bank_len) or longer than max_rir_len is invalid: the kernels read nothing for it and the item's output row becomes NaN.
__device__ __forceinline__ int prep_rir_len(const int32_t* rparams, int b) { return rparams ? rparams[2 * b + 1] : 0; }
__device__ __forceinline__ bool prep_rir_valid(const int32_t* rparams, int b, int64_t bank_len, int max_rir_len) {
    const int off = rparams[2 * b], len = rparams[2 * b + 1];
    return off >= 0 && len >= 1 && len <= max_rir_len && int64_t(off) + len <= bank_len;
}

}  // namespace ppv
