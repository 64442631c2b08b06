// extern "C" boundary of libppv_b200 (include/ppv_b200.h): argument checking, handle unwrapping, error text.
// No exceptions cross this boundary; everything returns a status code.
#include <string.h>

#include <new>

#include "common.h"
#include "image_plan.h"
#include "model_common.h"
#include "train.h"

namespace ppv {

static thread_local std::string g_last_error;

void set_error(const std::string& msg) { g_last_error = msg; }
int fail(int code, const std::string& msg) {
    g_last_error = msg;
    return code;
}

int device_sm_count() {
    int dev = 0, n = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0) {
        cudaGetLastError();
        return 132;  // H100 SXM
    }
    return n;
}

static int check_device() {
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess) return fail(PPV_ECUDA, "no CUDA device: libppv_b200 has no CPU fallback");
    int major = 0, minor = 0;
    cudaDeviceGetAttribute(&major, cudaDevAttrComputeCapabilityMajor, dev);
    cudaDeviceGetAttribute(&minor, cudaDevAttrComputeCapabilityMinor, dev);
    if (major != 9 || minor != 0) return fail(PPV_EUNSUPPORTED, "libppv_b200 is built for sm_90a only (found sm_" + std::to_string(major * 10 + minor) + ")");
    return PPV_OK;
}

}  // namespace ppv

using namespace ppv;

struct ppv_fbank {
    Fbank* impl;
};
struct ppv_spectral {
    Spectral* impl;
};

struct ppv_trainer {
    Trainer* impl;
};

struct ppv_model {
    Model* m;
};

#define PPV_GUARD_BEGIN try {
#define PPV_GUARD_END                                                        \
    }                                                                        \
    catch (const std::bad_alloc&) { return fail(PPV_ECUDA, "host out of memory"); } \
    catch (const std::exception& e) { return fail(PPV_EINVAL, std::string("exception: ") + e.what()); } \
    catch (...) { return fail(PPV_EINVAL, "unknown exception"); }

extern "C" {

int ppv_version(void) { return 100; }

int ppv_last_error(char* buf, size_t n) {
    const std::string& e = g_last_error;
    if (buf && n > 0) {
        const size_t k = std::min(n - 1, e.size());
        memcpy(buf, e.data(), k);
        buf[k] = 0;
    }
    return int(e.size());
}

int ppv_device_sm_count(void) { return device_sm_count(); }

// ---------------------------------------------------------------- fbank
void ppv_fbank_default_cfg(ppv_fbank_cfg* c) {
    if (!c) return;
    c->sample_rate = 16000;
    c->n_mels = 80;
    c->frame_length_ms = 25.f;
    c->frame_shift_ms = 10.f;
    c->preemph = 0.97f;
    c->low_freq = 20.f;
    c->high_freq = 0.f;
    c->log_floor = 1.1920928955078125e-07f;
    c->window_type = PPV_FBANK_WIN_POVEY;
    c->blackman_coeff = 0.42f;
    c->remove_dc_offset = 1;
    c->snip_edges = 1;
    c->use_power = 1;
    c->use_log_fbank = 1;
    c->vtln_warp = 1.f;
    c->vtln_low = 100.f;
    c->vtln_high = -500.f;
}

int ppv_fbank_create(const ppv_fbank_cfg* cfg, ppv_fbank_t** out) {
    PPV_GUARD_BEGIN
    PPV_REQUIRE(cfg && out, "ppv_fbank_create: null argument");
    int rc = check_device();
    if (rc) return rc;
    Fbank* impl = nullptr;
    rc = fbank_create(cfg, &impl);
    if (rc) return rc;
    *out = new ppv_fbank{impl};
    return PPV_OK;
    PPV_GUARD_END
}
int ppv_fbank_destroy(ppv_fbank_t* h) {
    if (!h) return PPV_OK;
    fbank_destroy(h->impl);
    delete h;
    return PPV_OK;
}
int ppv_fbank_num_frames(const ppv_fbank_t* h, int L) { return h ? fbank_num_frames(h->impl, L) : 0; }
int ppv_fbank_feature_dim(const ppv_fbank_t* h) { return h ? fbank_n_mels(h->impl) : 0; }

int ppv_fbank_forward(ppv_fbank_t* h, const float* wav, const float* lens_ratio, int B, int L, float* out, void* stream) {
    PPV_GUARD_BEGIN
    PPV_REQUIRE(h && wav && out, "ppv_fbank_forward: null argument");
    PPV_REQUIRE(B > 0 && L > 0, "ppv_fbank_forward: empty input");
    // raw log-mel goes to `out`, then CMN is applied in place (each element is read and written by one thread)
    return fbank_run(h->impl, wav, lens_ratio, B, L, out, out, Planes(), 0, 0, static_cast<cudaStream_t>(stream));
    PPV_GUARD_END
}

int ppv_fbank_forward_ragged(ppv_fbank_t* h, const float* wav, const int32_t* valid_frames, int B, int L, float* out, void* stream) {
    PPV_GUARD_BEGIN
    PPV_REQUIRE(h && wav && out && valid_frames, "ppv_fbank_forward_ragged: null argument");
    PPV_REQUIRE(B > 0 && L > 0, "ppv_fbank_forward_ragged: empty input");
    return fbank_run(h->impl, wav, nullptr, B, L, out, out, Planes(), 0, 0, static_cast<cudaStream_t>(stream), valid_frames);
    PPV_GUARD_END
}

int ppv_fbank_forward_ragged_samples(ppv_fbank_t* h, const float* wav, const int32_t* valid_frames, const int32_t* num_samples, int B, int L,
                                     float* out, void* stream) {
    PPV_GUARD_BEGIN
    PPV_REQUIRE(h && wav && out && valid_frames && num_samples, "ppv_fbank_forward_ragged_samples: null argument");
    PPV_REQUIRE(B > 0 && L > 0, "ppv_fbank_forward_ragged_samples: empty input");
    return fbank_run(h->impl, wav, nullptr, B, L, out, out, Planes(), 0, 0, static_cast<cudaStream_t>(stream), valid_frames, num_samples);
    PPV_GUARD_END
}

size_t ppv_audio_prep_workspace_bytes(int B, int max_new_len) { return audio_prep_workspace_bytes(B, max_new_len); }
int ppv_audio_prep(const float* wav, int64_t wav_ld, const int32_t* iparams, const float* fparams, const float* noise, int B, int max_new_len,
                   float target_db, int normalize, int Lout, float* out, void* ws, size_t ws_bytes, void* stream) {
    PPV_GUARD_BEGIN
    return audio_prep(wav, wav_ld, iparams, fparams, noise, B, max_new_len, target_db, normalize, Lout, out, ws, ws_bytes,
                      static_cast<cudaStream_t>(stream));
    PPV_GUARD_END
}

size_t ppv_audio_prep_reverb_workspace_bytes(int B, int max_new_len, int max_rir_len) {
    return audio_prep_reverb_workspace_bytes(B, max_new_len, max_rir_len);
}
int ppv_audio_prep_reverb(const float* wav, int64_t wav_ld, const int32_t* iparams, const float* fparams, const float* noise,
                          const float* rir_bank, int64_t rir_bank_len, const int32_t* rparams, int B, int max_new_len, int max_rir_len,
                          float target_db, int normalize, int Lout, float* out, void* ws, size_t ws_bytes, void* stream) {
    PPV_GUARD_BEGIN
    return audio_prep_reverb(wav, wav_ld, iparams, fparams, noise, rir_bank, rir_bank_len, rparams, B, max_new_len, max_rir_len, target_db,
                             normalize, Lout, out, ws, ws_bytes, static_cast<cudaStream_t>(stream));
    PPV_GUARD_END
}

// ---------------------------------------------------------------- model
void ppv_ecapa_default_cfg(ppv_ecapa_cfg* c) {
    if (c) ppv_ecapa_default_cfg_impl(c);
}
void ppv_eres2net_default_cfg(ppv_eres2net_cfg* c) {
    if (c) ppv_eres2net_default_cfg_impl(c);
}
void ppv_campplus_default_cfg(ppv_campplus_cfg* c) {
    if (c) ppv_campplus_default_cfg_impl(c);
}
void ppv_resnetse_default_cfg(ppv_resnetse_cfg* c) {
    if (c) ppv_resnetse_default_cfg_impl(c);
}
void ppv_res2net_default_cfg(ppv_res2net_cfg* c) {
    if (c) ppv_res2net_default_cfg_impl(c);
}

int ppv_model_create(int kind, const void* cfg, ppv_model_t** out) {
    PPV_GUARD_BEGIN
    PPV_REQUIRE(cfg && out, "ppv_model_create: null argument");
    if (kind != PPV_MODEL_ECAPA_TDNN && kind != PPV_MODEL_RESNET_SE && kind != PPV_MODEL_ERES2NET && kind != PPV_MODEL_CAMPPLUS &&
        kind != PPV_MODEL_RES2NET)
        return fail(PPV_EUNSUPPORTED, "ppv_model_create: implemented kinds are PPV_MODEL_ECAPA_TDNN, PPV_MODEL_RESNET_SE, PPV_MODEL_ERES2NET, "
                                      "PPV_MODEL_CAMPPLUS, PPV_MODEL_RES2NET");
    int rc = check_device();
    if (rc) return rc;
    Model* m = nullptr;
    switch (kind) {
        case PPV_MODEL_ECAPA_TDNN: rc = ecapa_create(static_cast<const ppv_ecapa_cfg*>(cfg), &m); break;
        case PPV_MODEL_RESNET_SE: rc = resnetse_create(static_cast<const ppv_resnetse_cfg*>(cfg), &m); break;
        case PPV_MODEL_ERES2NET: rc = eres2net_create(static_cast<const ppv_eres2net_cfg*>(cfg), &m); break;
        case PPV_MODEL_RES2NET: rc = res2net_create(static_cast<const ppv_res2net_cfg*>(cfg), &m); break;
        default: rc = campplus_create(static_cast<const ppv_campplus_cfg*>(cfg), &m); break;
    }
    if (rc) return rc;
    *out = new ppv_model{m};
    return PPV_OK;
    PPV_GUARD_END
}
int ppv_model_destroy(ppv_model_t* h) {
    if (!h) return PPV_OK;
    delete h->m;
    delete h;
    return PPV_OK;
}
int ppv_model_load_weight(ppv_model_t* h, const char* name, const float* data, const int64_t* shape, int ndim) {
    PPV_GUARD_BEGIN
    PPV_REQUIRE(h, "ppv_model_load_weight: null model");
    return h->m->load_weight(name, data, shape, ndim);
    PPV_GUARD_END
}
int ppv_model_finalize(ppv_model_t* h) {
    PPV_GUARD_BEGIN
    PPV_REQUIRE(h, "ppv_model_finalize: null model");
    return h->m->finalize();
    PPV_GUARD_END
}
int ppv_model_set_precision(ppv_model_t* h, int precision) {
    PPV_REQUIRE(h, "ppv_model_set_precision: null model");
    return h->m->set_precision(precision);
}
int ppv_model_embd_dim(const ppv_model_t* h) { return h ? h->m->embd_dim() : 0; }
size_t ppv_model_workspace_bytes(const ppv_model_t* h, int B, int T) { return h ? h->m->workspace_bytes(B, T) : 0; }

int ppv_model_forward(ppv_model_t* h, const float* feat, int B, int T, float* emb, void* ws, size_t ws_bytes, void* stream) {
    PPV_GUARD_BEGIN
    PPV_REQUIRE(h && feat && emb, "ppv_model_forward: null argument");
    return h->m->forward(ModelInput{feat}, B, T, emb, ws, ws_bytes, static_cast<cudaStream_t>(stream));
    PPV_GUARD_END
}
int ppv_model_forward_lengths(ppv_model_t* h, const float* feat, const float* lengths, int B, int T, float* emb, void* ws, size_t ws_bytes,
                              void* stream) {
    PPV_GUARD_BEGIN
    PPV_REQUIRE(h && feat && emb, "ppv_model_forward_lengths: null argument");
    ModelInput in{feat};
    in.lengths = lengths;
    return h->m->forward(in, B, T, emb, ws, ws_bytes, static_cast<cudaStream_t>(stream));
    PPV_GUARD_END
}
int ppv_model_forward_wav(ppv_model_t* h, ppv_fbank_t* fb, const float* wav, const float* lens_ratio, int B, int L, float* emb,
                          void* ws, size_t ws_bytes, void* stream) {
    PPV_GUARD_BEGIN
    PPV_REQUIRE(h && fb && wav && emb, "ppv_model_forward_wav: null argument");
    return h->m->forward(ModelInput{nullptr, fb->impl, wav, lens_ratio, L}, B, 0, emb, ws, ws_bytes, static_cast<cudaStream_t>(stream));
    PPV_GUARD_END
}
int ppv_model_read_tap(ppv_model_t* h, const char* name, float* out, size_t out_elems, void* stream) {
    PPV_GUARD_BEGIN
    PPV_REQUIRE(h, "ppv_model_read_tap: null model");
    return h->m->read_tap(name, out, out_elems, static_cast<cudaStream_t>(stream));
    PPV_GUARD_END
}

size_t ppv_eer_workspace_bytes(int64_t n) { return eer_workspace_bytes(n); }
int ppv_eer_mindcf(const float* scores, const int32_t* labels, int64_t n, double p_target, double c_miss, double c_fa, double* out4, void* ws,
                   size_t ws_bytes, void* stream) {
    PPV_GUARD_BEGIN
    PPV_REQUIRE(labels, "ppv_eer_mindcf: null labels");
    return eer_mindcf(scores, labels, nullptr, nullptr, 0, n, p_target, c_miss, c_fa, out4, ws, ws_bytes, static_cast<cudaStream_t>(stream));
    PPV_GUARD_END
}
int ppv_eer_mindcf_matrix(const float* scores, const int32_t* trial_labels, const int32_t* enroll_labels, int M, int N, double p_target,
                          double c_miss, double c_fa, double* out4, void* ws, size_t ws_bytes, void* stream) {
    PPV_GUARD_BEGIN
    PPV_REQUIRE(trial_labels && enroll_labels && M > 0 && N > 0, "ppv_eer_mindcf_matrix: bad argument");
    return eer_mindcf(scores, nullptr, trial_labels, enroll_labels, N, int64_t(M) * N, p_target, c_miss, c_fa, out4, ws, ws_bytes,
                      static_cast<cudaStream_t>(stream));
    PPV_GUARD_END
}
int ppv_row_argmax(const float* sim, int rows, int cols, int32_t* idx, float* best, void* stream) {
    PPV_GUARD_BEGIN
    return row_argmax(sim, rows, cols, idx, best, static_cast<cudaStream_t>(stream));
    PPV_GUARD_END
}

// ---------------------------------------------------------------- AS-norm
int ppv_topn_row_stats(const float* scores, int rows, int cols, int64_t ld, int top_n, float* mean, float* std, void* stream) {
    PPV_GUARD_BEGIN
    int rc = check_device();
    if (rc) return rc;
    return topn_row_stats(scores, rows, cols, ld, top_n, mean, std, static_cast<cudaStream_t>(stream));
    PPV_GUARD_END
}
int ppv_as_norm_apply(float* scores, int M, int N, const float* trial_mean, const float* trial_std, const float* enroll_mean,
                      const float* enroll_std, void* stream) {
    PPV_GUARD_BEGIN
    int rc = check_device();
    if (rc) return rc;
    return as_norm_apply(scores, M, N, trial_mean, trial_std, enroll_mean, enroll_std, static_cast<cudaStream_t>(stream));
    PPV_GUARD_END
}

// ---------------------------------------------------------------- energy VAD
void ppv_vad_default_cfg(ppv_vad_cfg* cfg, int sample_rate) {
    if (!cfg) return;
    cfg->window = int(int64_t(sample_rate) * 25 / 1000);
    cfg->shift = int(int64_t(sample_rate) * 10 / 1000);
    cfg->energy_threshold = 5.5f;
    cfg->energy_mean_scale = 0.5f;
    cfg->frames_context = 2;
    cfg->proportion_threshold = 0.12f;
}
int64_t ppv_vad_num_frames(const ppv_vad_cfg* cfg, int64_t L) { return cfg ? vad_num_frames(*cfg, L) : -1; }
size_t ppv_vad_workspace_bytes(const ppv_vad_cfg* cfg, int R, int64_t total_samples) {
    return cfg ? vad_workspace_bytes(*cfg, R, total_samples) : 0;
}
int ppv_vad_energy(const ppv_vad_cfg* cfg, const float* wav, const int64_t* sample_offsets, int R, double* log_energy, uint8_t* voiced,
                   int32_t* runs, int64_t run_cap, int32_t* n_runs, void* ws, size_t ws_bytes, void* stream) {
    PPV_GUARD_BEGIN
    int rc = check_device();
    if (rc) return rc;
    if (!cfg) return fail(PPV_EINVAL, "ppv_vad_energy: null cfg");
    return vad_energy(*cfg, wav, sample_offsets, R, log_energy, voiced, runs, run_cap, n_runs, ws, ws_bytes, static_cast<cudaStream_t>(stream));
    PPV_GUARD_END
}

// ---------------------------------------------------------------- speaker index
size_t ppv_speaker_index_bytes(int U, int D) { return speaker_index_bytes(U, D); }
int ppv_speaker_index_build(const float* E, int n, int D, const int32_t* order, const int32_t* offsets, int U, float* means, void* index,
                            size_t index_bytes, void* stream) {
    PPV_GUARD_BEGIN
    int rc = check_device();
    if (rc) return rc;
    return speaker_index_build(E, n, D, order, offsets, U, means, index, index_bytes, static_cast<cudaStream_t>(stream));
    PPV_GUARD_END
}
size_t ppv_speaker_index_search_workspace_bytes(int Q, int U, int D, int k) { return speaker_index_search_workspace_bytes(Q, U, D, k); }
int ppv_speaker_index_search(const float* queries, int Q, int D, const void* index, size_t index_bytes, int U, int k, int32_t* idx,
                             float* sim, void* ws, size_t ws_bytes, void* stream) {
    PPV_GUARD_BEGIN
    int rc = check_device();
    if (rc) return rc;
    return speaker_index_search(queries, Q, D, index, index_bytes, U, k, idx, sim, ws, ws_bytes, static_cast<cudaStream_t>(stream));
    PPV_GUARD_END
}

// ---------------------------------------------------------------- speaker diarization
int ppv_cluster_prune(float* affinity, int N, double pval, void* stream) {
    PPV_GUARD_BEGIN
    return cluster_prune(affinity, N, pval, static_cast<cudaStream_t>(stream));
    PPV_GUARD_END
}
int ppv_cluster_laplacian(const float* pruned, int N, double* L, void* stream) {
    PPV_GUARD_BEGIN
    return cluster_laplacian(pruned, N, L, static_cast<cudaStream_t>(stream));
    PPV_GUARD_END
}
size_t ppv_sym_eig_workspace_bytes(int N, int m) { return sym_eig_workspace_bytes(N, m); }
int ppv_sym_eig_smallest(double* L, int N, int m, double* evals, double* evecs, void* ws, size_t ws_bytes, void* stream) {
    PPV_GUARD_BEGIN
    return sym_eig_smallest(L, N, m, evals, evecs, ws, ws_bytes, static_cast<cudaStream_t>(stream));
    PPV_GUARD_END
}
size_t ppv_kmeans_workspace_bytes(int N, int k) { return kmeans_workspace_bytes(N, k); }
int ppv_kmeans(const double* X, int ld, int N, int k, const double* uniforms, int n_uniforms, int max_iter, int32_t* labels, double* inertia,
               void* ws, size_t ws_bytes, void* stream) {
    PPV_GUARD_BEGIN
    return kmeans(X, ld, N, k, uniforms, n_uniforms, max_iter, labels, inertia, ws, ws_bytes, static_cast<cudaStream_t>(stream));
    PPV_GUARD_END
}

int ppv_model_profile(ppv_model_t* h, int enable) {
    PPV_REQUIRE(h && h->m->takes_wav(), "ppv_model_profile: ECAPA-TDNN or Res2Net model required");
    h->m->profile(enable != 0);
    return PPV_OK;
}
int ppv_model_profile_read(ppv_model_t* h, double* gemm_ms, double* other_ms, int64_t* gemm_launches, int64_t* other_launches) {
    PPV_GUARD_BEGIN
    PPV_REQUIRE(h && h->m->takes_wav(), "ppv_model_profile_read: ECAPA-TDNN or Res2Net model required");
    PPV_REQUIRE(gemm_ms && other_ms && gemm_launches && other_launches, "ppv_model_profile_read: null argument");
    return h->m->profile_read(gemm_ms, other_ms, gemm_launches, other_launches);
    PPV_GUARD_END
}

// ---------------------------------------------------------------- STFT front ends, SpecAugment
void ppv_spectral_default_cfg(ppv_spectral_cfg* c, int method) {
    if (c) spectral_default_cfg(c, method);
}
int ppv_spectral_create(const ppv_spectral_cfg* cfg, ppv_spectral_t** out) {
    PPV_GUARD_BEGIN
    PPV_REQUIRE(cfg && out, "ppv_spectral_create: null argument");
    int rc = check_device();
    if (rc) return rc;
    Spectral* impl = nullptr;
    rc = spectral_create(cfg, &impl);
    if (rc) return rc;
    *out = new ppv_spectral{impl};
    return PPV_OK;
    PPV_GUARD_END
}
int ppv_spectral_destroy(ppv_spectral_t* h) {
    if (!h) return PPV_OK;
    spectral_destroy(h->impl);
    delete h;
    return PPV_OK;
}
int ppv_spectral_num_frames(const ppv_spectral_t* h, int L) { return h ? spectral_num_frames(h->impl, L) : 0; }
int ppv_spectral_feature_dim(const ppv_spectral_t* h) { return h ? spectral_feature_dim(h->impl) : 0; }
int ppv_spectral_forward(ppv_spectral_t* h, const float* wav, const float* lens_ratio, int B, int L, float* out, void* stream) {
    PPV_GUARD_BEGIN
    PPV_REQUIRE(h && wav && out, "ppv_spectral_forward: null argument");
    PPV_REQUIRE(B > 0 && L > 0, "ppv_spectral_forward: empty input");
    return spectral_run(h->impl, wav, lens_ratio, B, L, out, static_cast<cudaStream_t>(stream));
    PPV_GUARD_END
}
int ppv_spectral_forward_ragged_samples(ppv_spectral_t* h, const float* wav, const int32_t* valid_frames, const int32_t* num_samples, int B,
                                        int L, float* out, void* stream) {
    PPV_GUARD_BEGIN
    PPV_REQUIRE(h && wav && out && valid_frames && num_samples, "ppv_spectral_forward_ragged_samples: null argument");
    PPV_REQUIRE(B > 0 && L > 0, "ppv_spectral_forward_ragged_samples: empty input");
    return spectral_run(h->impl, wav, nullptr, B, L, out, static_cast<cudaStream_t>(stream), valid_frames, num_samples);
    PPV_GUARD_END
}
int ppv_spec_augment(float* feat, const int32_t* params, int B, int T, int F, int n_freq_masks, int n_time_masks, int fill_mode, void* stream) {
    PPV_GUARD_BEGIN
    return spec_augment_run(feat, params, B, T, F, n_freq_masks, n_time_masks, fill_mode, static_cast<cudaStream_t>(stream));
    PPV_GUARD_END
}

// ---------------------------------------------------------------- training step
int ppv_trainer_create(const ppv_ecapa_cfg* cfg, int num_classes, ppv_trainer_t** out) {
    PPV_GUARD_BEGIN
    PPV_REQUIRE(cfg && out, "ppv_trainer_create: null argument");
    int rc = check_device();
    if (rc) return rc;
    Trainer* impl = nullptr;
    rc = trainer_create(cfg, num_classes, PPV_CLASSIFIER_COSINE, 0, 0, &impl);
    if (rc) return rc;
    *out = new ppv_trainer{impl};
    return PPV_OK;
    PPV_GUARD_END
}
int ppv_trainer_create_classifier(const ppv_ecapa_cfg* cfg, int num_classes, int classifier_type, int num_blocks, int inter_dim,
                                  ppv_trainer_t** out) {
    PPV_GUARD_BEGIN
    PPV_REQUIRE(cfg && out, "ppv_trainer_create_classifier: null argument");
    int rc = check_device();
    if (rc) return rc;
    Trainer* impl = nullptr;
    rc = trainer_create(cfg, num_classes, classifier_type, num_blocks, inter_dim, &impl);
    if (rc) return rc;
    *out = new ppv_trainer{impl};
    return PPV_OK;
    PPV_GUARD_END
}
int ppv_trainer_destroy(ppv_trainer_t* h) {
    if (!h) return PPV_OK;
    trainer_destroy(h->impl);
    delete h;
    return PPV_OK;
}
int64_t ppv_trainer_param_count(const ppv_trainer_t* h) { return h ? trainer_param_count(h->impl) : 0; }
int64_t ppv_trainer_stat_count(const ppv_trainer_t* h) { return h ? trainer_stat_count(h->impl) : 0; }
int ppv_trainer_lookup(const ppv_trainer_t* h, const char* name, int64_t* offset, int64_t* numel, int* is_stat) {
    PPV_GUARD_BEGIN
    PPV_REQUIRE(h, "ppv_trainer_lookup: null handle");
    return trainer_lookup(h->impl, name, offset, numel, is_stat);
    PPV_GUARD_END
}
int ppv_set_pdl(int enabled) {
    const int prev = ppv::pdl_enabled();
    ppv::pdl_enabled() = enabled ? 1 : 0;
    return prev;
}
int ppv_trainer_set_precision(ppv_trainer_t* h, int precision) {
    PPV_GUARD_BEGIN
    PPV_REQUIRE(h, "ppv_trainer_set_precision: null handle");
    return trainer_set_precision(h->impl, precision);
    PPV_GUARD_END
}
int ppv_trainer_bind(ppv_trainer_t* h, float* params, float* grads, float* stats) {
    PPV_GUARD_BEGIN
    PPV_REQUIRE(h, "ppv_trainer_bind: null handle");
    return trainer_bind(h->impl, params, grads, stats);
    PPV_GUARD_END
}
size_t ppv_trainer_workspace_bytes(ppv_trainer_t* h, int B, int T) {
    try {
        return h ? trainer_workspace_bytes(h->impl, B, T) : 0;
    } catch (...) {
        return 0;
    }
}
int ppv_trainer_forward_backward(ppv_trainer_t* h, const float* feat, const int64_t* labels, int B, int T, float margin, float scale,
                                 int easy_margin, float label_smoothing, float* loss, float* logits, void* ws, size_t ws_bytes, void* stream) {
    PPV_GUARD_BEGIN
    PPV_REQUIRE(h, "ppv_trainer_forward_backward: null handle");
    return trainer_forward_backward(h->impl, feat, labels, B, T, margin, scale, easy_margin, label_smoothing, loss, logits, ws, ws_bytes,
                                    static_cast<cudaStream_t>(stream));
    PPV_GUARD_END
}
int ppv_trainer_read_tap(ppv_trainer_t* h, const char* name, float* out, size_t out_elems, void* stream) {
    PPV_GUARD_BEGIN
    PPV_REQUIRE(h, "ppv_trainer_read_tap: null handle");
    return trainer_read_tap(h->impl, name, out, out_elems, static_cast<cudaStream_t>(stream));
    PPV_GUARD_END
}
int ppv_adam_step(float* params, const float* grads, float* m, float* v, int64_t n, float lr, float beta1, float beta2, float eps,
                  float weight_decay, int64_t step, float grad_scale, void* stream) {
    PPV_GUARD_BEGIN
    return adam_step(params, grads, m, v, n, lr, beta1, beta2, eps, weight_decay, step, grad_scale, static_cast<cudaStream_t>(stream));
    PPV_GUARD_END
}
int ppv_optimizer_state_count(int kind, int centered) { return optimizer_state_count(kind, centered); }
int ppv_optimizer_step(int kind, float* params, const float* grads, float* state0, float* state1, float* state2, int64_t n,
                       const ppv_optim_args* args, int64_t step, float grad_scale, void* stream) {
    PPV_GUARD_BEGIN
    PPV_REQUIRE(args, "ppv_optimizer_step: null args");
    return optimizer_step(kind, params, grads, state0, state1, state2, n, *args, step, grad_scale, static_cast<cudaStream_t>(stream));
    PPV_GUARD_END
}

// ---------------------------------------------------------------- cosine scoring
size_t ppv_cosine_workspace_bytes(int M, int N, int D) { return cosine_workspace_bytes(M, N, D); }
int ppv_cosine_matrix(const float* A, const float* Bm, int M, int N, int D, float* out, void* ws, size_t ws_bytes, void* stream) {
    PPV_GUARD_BEGIN
    int rc = check_device();
    if (rc) return rc;
    return cosine_matrix(A, Bm, M, N, D, out, ws, ws_bytes, PPV_PREC_BF16X3, static_cast<cudaStream_t>(stream));
    PPV_GUARD_END
}
int ppv_cosine_pairlist(const float* E, const int32_t* idx, int64_t P, int n, int D, float* out, void* stream) {
    PPV_GUARD_BEGIN
    return cosine_pairlist(E, idx, P, n, D, out, static_cast<cudaStream_t>(stream));
    PPV_GUARD_END
}

// ---------------------------------------------------------------- AAM head
size_t ppv_aam_workspace_bytes(int B, int D, int S) { return aam_workspace_bytes(B, D, S); }
int ppv_aam_forward(const float* emb, const float* W, const int64_t* labels, int B, int D, int S, float margin, float scale,
                    int easy_margin, float label_smoothing, float* logits, float* loss, void* ws, size_t ws_bytes, void* stream) {
    PPV_GUARD_BEGIN
    return aam_forward(emb, W, labels, B, D, S, margin, scale, easy_margin, label_smoothing, logits, loss, ws, ws_bytes,
                       static_cast<cudaStream_t>(stream));
    PPV_GUARD_END
}
int ppv_aam_backward(const float* emb, const float* W, const int64_t* labels, const float* logits, int B, int D, int S, float margin,
                     float scale, int easy_margin, float label_smoothing, float* d_emb, float* d_W, void* ws, size_t ws_bytes,
                     void* stream) {
    PPV_GUARD_BEGIN
    return aam_backward(emb, W, labels, logits, B, D, S, margin, scale, easy_margin, label_smoothing, d_emb, d_W, ws, ws_bytes,
                        static_cast<cudaStream_t>(stream));
    PPV_GUARD_END
}
int ppv_linear_head_forward(const float* H, const float* W, const float* bias, const int64_t* labels, int B, int D, int S, float margin,
                            float scale, int easy_margin, float label_smoothing, float* logits, float* loss, void* ws, size_t ws_bytes,
                            void* stream) {
    PPV_GUARD_BEGIN
    return linear_head_forward(H, W, bias, labels, B, D, S, margin, scale, easy_margin, label_smoothing, logits, loss, ws, ws_bytes,
                               static_cast<cudaStream_t>(stream));
    PPV_GUARD_END
}
int ppv_linear_head_backward(const float* H, const float* W, const int64_t* labels, const float* logits, int B, int D, int S, float margin,
                             float scale, int easy_margin, float label_smoothing, float* d_H, float* d_W, float* d_bias, void* ws,
                             size_t ws_bytes, void* stream) {
    PPV_GUARD_BEGIN
    return linear_head_backward(H, W, labels, logits, B, D, S, margin, scale, easy_margin, label_smoothing, d_H, d_W, d_bias, ws, ws_bytes,
                                static_cast<cudaStream_t>(stream));
    PPV_GUARD_END
}

// ---------------------------------------------------------------- GEMM test hook
// Both hooks' operands in the workspace, zero-padded: A as planes [2][pad128(M)][Kp], then W as planes [2][pad256(N)][Kp], Kp = pad64(K).
static void carve_gemm_test(WsCarver& cv, int M, int N, int K, Planes* pa, Planes* pw) {
    const int Kp = int(align_up(size_t(K), 64));
    *pa = cv.planes(M, Kp);
    *pw = cv.planes(int64_t(align_up(size_t(N), 256)), Kp);
}
size_t ppv_gemm_test_workspace_bytes(int M, int N, int K) {
    return carve_extent([&](WsCarver& cv) { Planes pa, pw; carve_gemm_test(cv, M, N, K, &pa, &pw); });
}
static int gemm_test_stage(const float* A, const float* W, int M, int N, int K, void* ws, size_t need, cudaStream_t st, Planes* pa, Planes* pw) {
    WsCarver cv{static_cast<uint8_t*>(ws)};
    carve_gemm_test(cv, M, N, K, pa, pw);
    PPV_CUDA_OK(cudaMemsetAsync(ws, 0, need, st));
    int rc = launch_f32_to_planes(A, M, K, *pa, st);
    if (rc) return rc;
    return launch_f32_to_planes(W, N, K, *pw, st);
}
int ppv_gemm_test(const float* A, const float* W, const float* bias, const float* bn_scale, const float* bn_shift, int relu, int M,
                  int N, int K, int block_n, int block_k, int precision, float* out, void* ws, size_t ws_bytes, void* stream) {
    PPV_GUARD_BEGIN
    PPV_REQUIRE(A && W && out, "ppv_gemm_test: null argument");
    const size_t need = ppv_gemm_test_workspace_bytes(M, N, K);
    if (int rc = check_workspace("ppv_gemm_test", ws, ws_bytes, need, "ppv_gemm_test_workspace_bytes")) return rc;
    int rc = check_device();
    if (rc) return rc;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    Planes pa, pw;
    rc = gemm_test_stage(A, W, M, N, K, ws, need, st, &pa, &pw);
    if (rc) return rc;
    GemmSource src{pa, 0, pa.ld, 0};
    Epilogue ep;
    ep.bias = bias;
    ep.relu = relu;
    ep.bn_scale = bn_scale;
    ep.bn_shift = bn_shift;
    ep.out_mode = OUT_F32;
    ep.out = out;
    ep.out_ld = N;
    GemmParams gp;
    rc = gemm_build(&gp, &src, 1, pw, M, N, ep, block_n, block_k);
    if (rc) return rc;
    return gemm_launch(gp, precision, device_sm_count(), st);
    PPV_GUARD_END
}

// Planes-output variant of the test hook: out is a split-bf16 planes buffer [2][M][N] (N % 32 == 0, 16-byte aligned) written by the
// epilogue the ECAPA layers use: + bias, + rowgrp_bias[row / Tp] (if given), ReLU (if relu), BN affine (if given), tanh (if tanh_).
// Tp > 0: rows follow the padded time layout (Tp = T + 2 P, M % Tp == 0) and only the T valid rows of each group are stored.
int ppv_gemm_test_planes(const float* A, const float* W, const float* bias, const float* rowgrp_bias, const float* bn_scale,
                         const float* bn_shift, int relu, int tanh_, int Tp, int P, int M, int N, int K, int block_n, int precision,
                         void* out, void* ws, size_t ws_bytes, void* stream) {
    PPV_GUARD_BEGIN
    PPV_REQUIRE(A && W && out, "ppv_gemm_test_planes: null argument");
    const size_t need = ppv_gemm_test_workspace_bytes(M, N, K);
    if (int rc = check_workspace("ppv_gemm_test_planes", ws, ws_bytes, need, "ppv_gemm_test_workspace_bytes")) return rc;
    PPV_REQUIRE(N % 32 == 0 && (Tp == 0 || (M % Tp == 0 && Tp > 2 * P)), "ppv_gemm_test_planes: bad shape");
    int rc = check_device();
    if (rc) return rc;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    Planes pa, pw;
    rc = gemm_test_stage(A, W, M, N, K, ws, need, st, &pa, &pw);
    if (rc) return rc;
    GemmSource src{pa, 0, pa.ld, 0};
    const Planes po{static_cast<__nv_bfloat16*>(out), 0, N, int64_t(M) * N};
    Epilogue ep = Tp > 0 ? planes_epilogue(po, 0, Tp, P, Tp - 2 * P) : planes_epilogue(po);
    ep.bias = bias;
    ep.rowgrp_bias = rowgrp_bias;
    ep.relu = relu;
    ep.tanh_ = tanh_;
    ep.bn_scale = bn_scale;
    ep.bn_shift = bn_shift;
    GemmParams gp;
    rc = gemm_build(&gp, &src, 1, pw, M, N, ep, block_n, 64);
    if (rc) return rc;
    return gemm_launch(gp, precision, device_sm_count(), st);
    PPV_GUARD_END
}

// ---------------------------------------------------------------- conv2d test hook
// One conv2d of the 2-D models (ResNetSE, ERes2Net, CAM++) on an input grid laid out as theirs, with their weight reorder, epilogue
// and tap list (image_plan.h, model_common.h); exactly the kernel `path` names runs, or an error is returned.  Workspace: the input grid [2][pad128(B (H+2) (W+2))][x_ld], then the weight planes [2][pad256(Cout)][k k Cin].
static void carve_conv2d_test(WsCarver& cv, int B, int H, int W, int Cin, int Cout, int k, int x_ld, Planes* xp, Planes* wp) {
    *xp = cv.planes(int64_t(B) * (H + 2) * (W + 2), x_ld);
    *wp = cv.planes(int64_t(align_up(size_t(Cout), 256)), k * k * Cin);
}
size_t ppv_conv2d_test_workspace_bytes(int B, int H, int W, int Cin, int Cout, int k, int x_ld) {
    if (x_ld <= 0) x_ld = Cin;
    return carve_extent([&](WsCarver& cv) { Planes xp, wp; carve_conv2d_test(cv, B, H, W, Cin, Cout, k, x_ld, &xp, &wp); });
}
// relu_max > 0: ReLU clipped at relu_max (ERes2Net's Hardtanh(0, 20)), the ppv_conv2d_test_clipped entry point
static int conv2d_test(const float* x, const float* w, const float* bias, int relu, float relu_max, int B, int H, int W, int Cin, int Cout,
                       int k, int stride_h, int stride_w, int x_col0, int x_ld, int path, int precision, void* out, void* ws, size_t ws_bytes,
                       void* stream) {
    PPV_GUARD_BEGIN
    PPV_REQUIRE(x && w && out, "ppv_conv2d_test: null argument");
    if (x_ld <= 0) x_ld = Cin;
    PPV_REQUIRE(B > 0 && H > 0 && W > 0 && Cin > 0 && Cout > 0 && (k == 1 || k == 3) && stride_h >= 1 && stride_w >= 1,
                "ppv_conv2d_test: bad shape");
    PPV_REQUIRE(x_col0 >= 0 && x_col0 + Cin <= x_ld, "ppv_conv2d_test: the input columns exceed x_ld");
    PPV_REQUIRE(path >= 0 && path <= 2, "ppv_conv2d_test: path must be 0 (3x3 patch kernel), 1 (pointwise kernel) or 2 (gather-GEMM)");
    PPV_REQUIRE(precision == PPV_PREC_BF16X3 || precision == PPV_PREC_BF16, "ppv_conv2d_test: bad precision");
    if (int rc = check_workspace("ppv_conv2d_test", ws, ws_bytes, ppv_conv2d_test_workspace_bytes(B, H, W, Cin, Cout, k, x_ld),
                                 "ppv_conv2d_test_workspace_bytes")) return rc;
    const int Hp = H + 2, Wp = W + 2, Ho = (H - 1) / stride_h + 1, Wo = (W - 1) / stride_w + 1;
    const int64_t M = int64_t(B) * Hp * Wp;
    PPV_REQUIRE(M < (int64_t(1) << 31) && Wp + 1 < 32768, "ppv_conv2d_test: grid too large for 32-bit rows / 16-bit tap offsets");
    int rc = check_device();
    if (rc) return rc;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    // input grid: zero border; x at columns [x_col0, x_col0 + Cin) of the interior; the other columns hold 0x3f3f (0.746 in bf16) in
    // both planes, so a kernel that reads outside its column window is visibly wrong
    WsCarver cv{static_cast<uint8_t*>(ws)};
    Planes xp, wp;
    carve_conv2d_test(cv, B, H, W, Cin, Cout, k, x_ld, &xp, &wp);
    PPV_CUDA_OK(cudaMemsetAsync(xp.base, 0, size_t(2 * xp.plane_stride) * sizeof(__nv_bfloat16), st));
    const size_t pitch = size_t(x_ld) * sizeof(__nv_bfloat16), rows2 = size_t(2 * xp.rows);
    if (x_col0 > 0) PPV_CUDA_OK(cudaMemset2DAsync(xp.base, pitch, 0x3f, size_t(x_col0) * sizeof(__nv_bfloat16), rows2, st));
    if (x_col0 + Cin < x_ld)
        PPV_CUDA_OK(cudaMemset2DAsync(xp.base + x_col0 + Cin, pitch, 0x3f, size_t(x_ld - x_col0 - Cin) * sizeof(__nv_bfloat16), rows2, st));
    for (int b = 0; b < B; ++b)
        for (int h = 0; h < H; ++h) {  // one image row: W consecutive grid positions
            Planes row = xp;
            row.base = xp.base + ((int64_t(b) * Hp + h + 1) * Wp + 1) * x_ld + x_col0;
            rc = launch_f32_to_planes(x + (int64_t(b) * H + h) * W * Cin, W, Cin, row, st);
            if (rc) return rc;
        }
    // weights [Cout][Cin][k][k] -> [Cout][tap][Cin], split into planes on the host as the models prepare theirs
    const int K = k * k * Cin;
    std::vector<float> wh(size_t(Cout) * K);
    PPV_CUDA_OK(cudaMemcpyAsync(wh.data(), w, wh.size() * sizeof(float), cudaMemcpyDeviceToHost, st));
    PPV_CUDA_OK(cudaStreamSynchronize(st));
    ArenaBuilder ab;
    GemmWeights gw;
    ab.put_matrix(&gw, conv_weight_matrix(wh.data(), Cout, Cin, k * k, Cout, {{k * k, Cin, 0, Cin, 0}}), Cout, K);
    PPV_CUDA_OK(cudaMemcpyAsync(wp.base, ab.host.data(), ab.host.size(), cudaMemcpyHostToDevice, st));
    PPV_CUDA_OK(cudaStreamSynchronize(st));
    gw.W.base = wp.base;
    // output grid, zeroed as a plan zeroes its workspace: the kernels store interior positions on the stride grid only
    const int64_t out_plane = int64_t(B) * (Ho + 2) * (Wo + 2) * Cout;
    PPV_CUDA_OK(cudaMemsetAsync(out, 0, size_t(2 * out_plane) * sizeof(__nv_bfloat16), st));
    Planes outp;
    outp.base = static_cast<__nv_bfloat16*>(out);
    outp.ld = Cout;
    outp.plane_stride = out_plane;
    const ImageGeo gin{H, W, Hp, Wp}, gout{Ho, Wo, Ho + 2, Wo + 2};
    Epilogue ep = image_epilogue(outp, gin, gout, stride_h, stride_w);
    ep.bias = bias;
    ep.relu = relu ? 1 : 0;
    ep.relu_max = relu_max;
    const int sms = device_sm_count();
    if (path == 0) {
        PPV_REQUIRE(k == 3 && conv3x3_c32_supported(Cin, Cout, H, W), "ppv_conv2d_test: the patch kernel takes 3x3 convs with 32 -> 32 channels only");
        Conv3x3Params cp;
        rc = conv3x3_build(&cp, xp, x_col0, gw.W, B, H, W, Hp, Wp, ep);
        if (rc) return rc;
        return conv3x3_launch(cp, precision, sms, st);
    }
    if (path == 1) {  // fp32 FMAs over the exact hi + lo values whatever the precision
        PPV_REQUIRE(k == 1, "ppv_conv2d_test: the pointwise kernel takes 1x1 convs only");
        const GemmSource src{xp, x_col0, Cin, 0};
        PwStep s;
        if (!pointwise_step_build(&s, &src, 1, gw.W, Cout, M, ep))
            return fail(PPV_EINVAL, "ppv_conv2d_test: the pointwise kernel does not take this conv (or PPV_POINTWISE=0)");
        return pointwise_launch(s, sms, st);
    }
    std::vector<GemmSource> srcs;
    if (k == 3)
        image_taps(&srcs, xp, x_col0, Cin, gin);
    else
        srcs.push_back(GemmSource{xp, x_col0, Cin, 0});
    GemmParams gp;
    rc = gemm_build(&gp, srcs.data(), int(srcs.size()), gw.W, int(M), Cout, ep, gemm_pick_bn(Cout));
    if (rc) return rc;
    return gemm_launch(gp, precision, sms, st);
    PPV_GUARD_END
}
int ppv_conv2d_test(const float* x, const float* w, const float* bias, int relu, int B, int H, int W, int Cin, int Cout, int k,
                    int stride_h, int stride_w, int x_col0, int x_ld, int path, int precision, void* out, void* ws, size_t ws_bytes,
                    void* stream) {
    return conv2d_test(x, w, bias, relu, 0.f, B, H, W, Cin, Cout, k, stride_h, stride_w, x_col0, x_ld, path, precision, out, ws, ws_bytes,
                       stream);
}
int ppv_conv2d_test_clipped(const float* x, const float* w, const float* bias, float relu_max, int B, int H, int W, int Cin, int Cout,
                            int k, int stride_h, int stride_w, int x_col0, int x_ld, int path, int precision, void* out, void* ws,
                            size_t ws_bytes, void* stream) {
    if (!(relu_max > 0.f)) return fail(PPV_EINVAL, "ppv_conv2d_test_clipped: relu_max must be > 0");
    return conv2d_test(x, w, bias, 1, relu_max, B, H, W, Cin, Cout, k, stride_h, stride_w, x_col0, x_ld, path, precision, out, ws, ws_bytes,
                       stream);
}

// Res2Net's fused stem + max-pool (res2net.cu) on features given here: w [32][49] and bias [32] with the BN already folded in.
int ppv_res2net_stem_test(const float* feat, const float* w, const float* bias, int B, int T, int F, void* out, void* stream) {
    PPV_GUARD_BEGIN
    PPV_REQUIRE(feat && w && bias && out && B > 0, "ppv_res2net_stem_test: bad argument");
    if (int rc = check_device()) return rc;
    int H1, W1, Hq, Wq;
    res2net_stem_grids(F, T, &H1, &W1, &Hq, &Wq);
    Planes o;
    o.base = static_cast<__nv_bfloat16*>(out);
    o.ld = 32;
    o.rows = int64_t(B) * (Hq + 2) * (Wq + 2);
    o.plane_stride = o.rows * o.ld;
    const cudaStream_t st = static_cast<cudaStream_t>(stream);
    PPV_CUDA_OK(cudaMemsetAsync(out, 0, size_t(2) * o.plane_stride * sizeof(__nv_bfloat16), st));
    return launch_res2net_stem(feat, B, T, F, w, bias, 32, o, st);
    PPV_GUARD_END
}

// ---------------------------------------------------------------- 2-D models' stem and elementwise test hooks
// The 1 -> C0 stem conv of ResNetSE, ERes2Net and CAM++ (image_plan.cu) on features given here: w [C0][9] and bias [C0] with the BN
// folded in.
int ppv_stem_conv_test(const float* feat, const float* w, const float* bias, int B, int T, int F, int C0, void* out, void* stream) {
    PPV_GUARD_BEGIN
    PPV_REQUIRE(feat && w && bias && out && B > 0 && T > 0 && F > 0, "ppv_stem_conv_test: bad argument");
    if (int rc = check_device()) return rc;
    Planes o;
    o.base = static_cast<__nv_bfloat16*>(out);
    o.ld = C0;
    o.rows = int64_t(B) * (F + 2) * (T + 2);
    o.plane_stride = o.rows * o.ld;
    const cudaStream_t st = static_cast<cudaStream_t>(stream);
    PPV_CUDA_OK(cudaMemsetAsync(out, 0, size_t(2) * o.plane_stride * sizeof(__nv_bfloat16), st));
    return launch_stem_conv(feat, B, T, F, w, bias, C0, o, F + 2, T + 2, st);
    PPV_GUARD_END
}

// The residual add that ends every 2-D block and ECAPA's SE block (launch_se_scale_res).  Workspace: z planes [2][pad128(rows)][C],
// then res planes [2][pad128(rows)][res_ld].
static void carve_scale_res_test(WsCarver& cv, int rows, int C, int res_ld, Planes* zp, Planes* rp) {
    *zp = cv.planes(rows, C);
    *rp = cv.planes(rows, res_ld);
}
size_t ppv_scale_res_test_workspace_bytes(int rows, int C, int res_ld) {
    if (rows <= 0 || C <= 0 || res_ld <= 0) return 0;
    return carve_extent([&](WsCarver& cv) { Planes zp, rp; carve_scale_res_test(cv, rows, C, res_ld, &zp, &rp); });
}
int ppv_scale_res_test(const float* z, const float* scale, const float* res, int res_ld, int rc0, int C, int rows_per_group, int rows,
                       int relu, float relu_max, void* out, int out_ld, int oc0, void* ws, size_t ws_bytes, void* stream) {
    PPV_GUARD_BEGIN
    PPV_REQUIRE(z && res && out, "ppv_scale_res_test: null argument");
    PPV_REQUIRE(rows > 0 && C > 0 && rows_per_group > 0 && rows % rows_per_group == 0 && rc0 >= 0 && rc0 + C <= res_ld && oc0 >= 0 &&
                    oc0 + C <= out_ld && res_ld % 8 == 0 && out_ld % 8 == 0 && relu_max >= 0.f,
                "ppv_scale_res_test: bad shape");
    if (int rc = check_workspace("ppv_scale_res_test", ws, ws_bytes, ppv_scale_res_test_workspace_bytes(rows, C, res_ld),
                                 "ppv_scale_res_test_workspace_bytes"))
        return rc;
    if (int rc = check_device()) return rc;
    const cudaStream_t st = static_cast<cudaStream_t>(stream);
    WsCarver cv{static_cast<uint8_t*>(ws)};
    Planes zp, rp;
    carve_scale_res_test(cv, rows, C, res_ld, &zp, &rp);
    int rc = launch_f32_to_planes(z, rows, C, zp, st);
    if (rc) return rc;
    if ((rc = launch_f32_to_planes(res, rows, res_ld, rp, st))) return rc;
    const Planes op{static_cast<__nv_bfloat16*>(out), rows, out_ld, int64_t(rows) * out_ld};
    return launch_se_scale_res(zp, scale, rp, rc0, op, oc0, C, rows_per_group, rows, device_sm_count(), st, relu, relu_max);
    PPV_GUARD_END
}

// AFF's blend (launch_aff_combine).  Workspace: x planes [2][pad128(rows)][x_ld], y planes [2][pad128(rows)][y_ld], t planes
// [2][pad128(rows)][C].
static void carve_aff_combine_test(WsCarver& cv, int rows, int C, int x_ld, int y_ld, Planes* xp, Planes* yp, Planes* tp) {
    *xp = cv.planes(rows, x_ld);
    *yp = cv.planes(rows, y_ld);
    *tp = cv.planes(rows, C);
}
size_t ppv_aff_combine_test_workspace_bytes(int rows, int C, int x_ld, int y_ld) {
    if (rows <= 0 || C <= 0 || x_ld <= 0 || y_ld <= 0) return 0;
    return carve_extent([&](WsCarver& cv) { Planes xp, yp, tp; carve_aff_combine_test(cv, rows, C, x_ld, y_ld, &xp, &yp, &tp); });
}
int ppv_aff_combine_test(const float* x, int x_ld, int xc0, const float* y, int y_ld, int yc0, const float* t, int C, int rows, void* out,
                         void* ws, size_t ws_bytes, void* stream) {
    PPV_GUARD_BEGIN
    PPV_REQUIRE(x && y && t && out, "ppv_aff_combine_test: null argument");
    PPV_REQUIRE(rows > 0 && C > 0 && xc0 >= 0 && xc0 + C <= x_ld && yc0 >= 0 && yc0 + C <= y_ld && x_ld % 8 == 0 && y_ld % 8 == 0,
                "ppv_aff_combine_test: bad shape");
    if (int rc = check_workspace("ppv_aff_combine_test", ws, ws_bytes, ppv_aff_combine_test_workspace_bytes(rows, C, x_ld, y_ld),
                                 "ppv_aff_combine_test_workspace_bytes"))
        return rc;
    if (int rc = check_device()) return rc;
    const cudaStream_t st = static_cast<cudaStream_t>(stream);
    WsCarver cv{static_cast<uint8_t*>(ws)};
    Planes xp, yp, tp;
    carve_aff_combine_test(cv, rows, C, x_ld, y_ld, &xp, &yp, &tp);
    int rc = launch_f32_to_planes(x, rows, x_ld, xp, st);
    if (rc) return rc;
    if ((rc = launch_f32_to_planes(y, rows, y_ld, yp, st))) return rc;
    if ((rc = launch_f32_to_planes(t, rows, C, tp, st))) return rc;
    const Planes op{static_cast<__nv_bfloat16*>(out), rows, C, int64_t(rows) * C};
    return launch_aff_combine(xp, xc0, yp, yc0, tp, op, C, rows, device_sm_count(), st);
    PPV_GUARD_END
}

// Res2Net's exclusive 3x3 average pool (res2net.cu).  Workspace: the input grid [2][pad128(B (H+2) (W+2))][C].
static void carve_avgpool_test(WsCarver& cv, int B, int H, int W, int C, Planes* xp) { *xp = cv.planes(int64_t(B) * (H + 2) * (W + 2), C); }
size_t ppv_res2net_avgpool_test_workspace_bytes(int B, int H, int W, int C) {
    if (B <= 0 || H <= 0 || W <= 0 || C <= 0) return 0;
    return carve_extent([&](WsCarver& cv) { Planes xp; carve_avgpool_test(cv, B, H, W, C, &xp); });
}
int ppv_res2net_avgpool_test(const float* x, int B, int H, int W, int C, int col0, int ncols, int stride, void* out, void* ws, size_t ws_bytes,
                             void* stream) {
    PPV_GUARD_BEGIN
    PPV_REQUIRE(x && out && B > 0 && H > 0 && W > 0 && C > 0 && col0 >= 0 && ncols > 0 && col0 + ncols <= C, "ppv_res2net_avgpool_test: bad argument");
    if (int rc = check_workspace("ppv_res2net_avgpool_test", ws, ws_bytes, ppv_res2net_avgpool_test_workspace_bytes(B, H, W, C),
                                 "ppv_res2net_avgpool_test_workspace_bytes"))
        return rc;
    if (int rc = check_device()) return rc;
    const cudaStream_t st = static_cast<cudaStream_t>(stream);
    WsCarver cv{static_cast<uint8_t*>(ws)};
    Planes xp;
    carve_avgpool_test(cv, B, H, W, C, &xp);
    int rc = launch_f32_to_planes(x, int64_t(B) * (H + 2) * (W + 2), C, xp, st);
    if (rc) return rc;
    const int Ho = (H - 1) / std::max(stride, 1) + 1, Wo = (W - 1) / std::max(stride, 1) + 1;
    Planes o;
    o.base = static_cast<__nv_bfloat16*>(out);
    o.ld = C;
    o.rows = int64_t(B) * (Ho + 2) * (Wo + 2);
    o.plane_stride = o.rows * o.ld;
    PPV_CUDA_OK(cudaMemsetAsync(out, 0, size_t(2) * o.plane_stride * sizeof(__nv_bfloat16), st));
    return launch_avgpool3x3(xp, col0, B, H, W, stride, ncols, o, col0, device_sm_count(), st);
    PPV_GUARD_END
}

// ---------------------------------------------------------------- fused attentive-statistics pooling test hook
// Workspace: W planes [2][C][K], att planes [2][B Tp + 64][K], x planes [2][B Tp + 64][C], out planes [2][B][2C].  The tensor
// maps of att and x end at row B Tp; the 64 rows behind hold 0x4646 (12672 in bf16) in both planes.
struct AspTestWs {
    Planes w, att, x, out;
};
static void carve_asp_test(WsCarver& cv, int B, int Tp, int C, int K, AspTestWs* v) {
    const int64_t rows = int64_t(B) * Tp;
    auto planes = [&](int64_t nrows, int ld, int64_t alloc_rows) {
        return Planes{static_cast<__nv_bfloat16*>(cv.take(size_t(2 * alloc_rows * ld) * sizeof(__nv_bfloat16))), nrows, ld, alloc_rows * ld};
    };
    v->w = planes(C, K, C);
    v->att = planes(rows, K, rows + 64);
    v->x = planes(rows, C, rows + 64);
    v->out = planes(B, 2 * C, B);
}
size_t ppv_asp_fused_test_workspace_bytes(int B, int Tp, int C, int K) {
    return carve_extent([&](WsCarver& cv) { AspTestWs v; carve_asp_test(cv, B, Tp, C, K, &v); });
}
int ppv_asp_fused_test(const float* W, const float* att, const float* x, const float* bn_scale, const float* bn_shift,
                       const int* nvalid, int B, int T, int P, int Tp, int C, int K, int precision, int max_ctas, float* out_raw,
                       float* out, void* ws, size_t ws_bytes, void* stream) {
    PPV_GUARD_BEGIN
    PPV_REQUIRE(W && att && x && bn_scale && bn_shift && out_raw && out, "ppv_asp_fused_test: null argument");
    PPV_REQUIRE(B > 0 && T > 0 && P >= 0 && Tp >= T + 2 * P && max_ctas >= 0, "ppv_asp_fused_test: bad shape");
    PPV_REQUIRE(precision == PPV_PREC_BF16X3 || precision == PPV_PREC_BF16, "ppv_asp_fused_test: bad precision");
    if (int rc = check_workspace("ppv_asp_fused_test", ws, ws_bytes, ppv_asp_fused_test_workspace_bytes(B, Tp, C, K),
                                 "ppv_asp_fused_test_workspace_bytes")) return rc;
    int rc = check_device();
    if (rc) return rc;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const int64_t rows = int64_t(B) * Tp;
    WsCarver cv{static_cast<uint8_t*>(ws)};
    AspTestWs v;
    carve_asp_test(cv, B, Tp, C, K, &v);
    const Planes &pw = v.w, &pa = v.att, &px = v.x, &po = v.out;
    PPV_CUDA_OK(cudaMemsetAsync(pa.base, 0x46, reinterpret_cast<uint8_t*>(po.base) - reinterpret_cast<uint8_t*>(pa.base), st));
    if ((rc = launch_f32_to_planes(W, C, K, pw, st)) || (rc = launch_f32_to_planes(att, rows, K, pa, st)) ||
        (rc = launch_f32_to_planes(x, rows, C, px, st))) return rc;
    AspFusedParams ap;
    rc = asp_fused_build(&ap, pw, pa, px, bn_scale, bn_shift, po, out_raw, B, T, P, Tp, C, K, 1e-12f);
    if (rc) return rc;
    ap.nvalid = nvalid;
    rc = asp_fused_launch(ap, precision, max_ctas > 0 ? max_ctas : device_sm_count(), st);
    if (rc) return rc;
    return launch_planes_to_f32(po, 0, 2 * C, B, 1, 0, 1, out, st);
    PPV_GUARD_END
}

// ---------------------------------------------------------------- column statistics test hook
// Workspace: x planes [2][B Tp][ld], then the output planes [2][B][C or 2C].
static void carve_colstats_test(WsCarver& cv, int B, int Tp, int ld, int C, __nv_bfloat16** x, __nv_bfloat16** out) {
    *x = static_cast<__nv_bfloat16*>(cv.take(size_t(B) * Tp * ld * 2 * sizeof(__nv_bfloat16)));
    *out = static_cast<__nv_bfloat16*>(cv.take(size_t(B) * 2 * C * 2 * sizeof(__nv_bfloat16)));
}
size_t ppv_colstats_test_workspace_bytes(int B, int Tp, int ld, int C) {
    return carve_extent([&](WsCarver& cv) { __nv_bfloat16 *x, *out; carve_colstats_test(cv, B, Tp, ld, C, &x, &out); });
}
int ppv_colstats_test(const float* x, int B, int T, int P, int Tp, int ld, int col0, int C, int mode, float eps, float inv_count,
                      const int* nvalid, float* out, float* out_f32, void* ws, size_t ws_bytes, void* stream) {
    PPV_GUARD_BEGIN
    PPV_REQUIRE(x && out, "ppv_colstats_test: null argument");
    PPV_REQUIRE(B > 0 && T > 0 && P >= 0 && Tp >= T + 2 * P && C > 0 && col0 >= 0 && col0 + C <= ld, "ppv_colstats_test: bad shape");
    PPV_REQUIRE(mode >= 0 && mode <= 3 && (mode == 0 || !out_f32), "ppv_colstats_test: mode must be 0-3, out_f32 with mode 0 only");
    if (int rc = check_workspace("ppv_colstats_test", ws, ws_bytes, ppv_colstats_test_workspace_bytes(B, Tp, ld, C),
                                 "ppv_colstats_test_workspace_bytes")) return rc;
    int rc = check_device();
    if (rc) return rc;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const int64_t rows = int64_t(B) * Tp;
    const int oc = mode == 0 ? C : 2 * C;
    WsCarver cv{static_cast<uint8_t*>(ws)};
    __nv_bfloat16 *xb, *ob;
    carve_colstats_test(cv, B, Tp, ld, C, &xb, &ob);
    const Planes px{xb, rows, ld, rows * ld};
    const Planes po{ob, B, oc, int64_t(B) * oc};
    if ((rc = launch_f32_to_planes(x, rows, ld, px, st))) return rc;
    if ((rc = launch_colstats(px, col0, C, B, T, P, Tp, mode, eps, out_f32, po, st, inv_count, nvalid))) return rc;
    return launch_planes_to_f32(po, 0, oc, B, 1, 0, 1, out, st);
    PPV_GUARD_END
}

// ---------------------------------------------------------------- TAP / TSP pooling backward test hook
// Workspace: x planes [2][B Tp][C], then the dx planes [2][B Tp][C].
static void carve_pool_stats_bwd_test(WsCarver& cv, int B, int Tp, int C, Planes* x, Planes* dx) {
    *x = cv.planes(int64_t(B) * Tp, C);
    *dx = cv.planes(int64_t(B) * Tp, C);
}
size_t ppv_pool_stats_bwd_test_workspace_bytes(int B, int Tp, int C) {
    if (B <= 0 || Tp <= 0 || C <= 0) return 0;
    return carve_extent([&](WsCarver& cv) { Planes x, dx; carve_pool_stats_bwd_test(cv, B, Tp, C, &x, &dx); });
}
int ppv_pool_stats_bwd_test(const float* x, const float* pooled, const float* dpooled, int B, int T, int P, int Tp, int C, int var, float* dx,
                            void* ws, size_t ws_bytes, void* stream) {
    PPV_GUARD_BEGIN
    PPV_REQUIRE(x && pooled && dpooled && dx, "ppv_pool_stats_bwd_test: null argument");
    PPV_REQUIRE(B > 0 && T > 0 && P >= 0 && Tp >= T + 2 * P && C > 0 && C % 8 == 0, "ppv_pool_stats_bwd_test: bad shape");
    if (int rc = check_workspace("ppv_pool_stats_bwd_test", ws, ws_bytes, ppv_pool_stats_bwd_test_workspace_bytes(B, Tp, C),
                                 "ppv_pool_stats_bwd_test_workspace_bytes")) return rc;
    int rc = check_device();
    if (rc) return rc;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const int64_t rows = int64_t(B) * Tp;
    WsCarver cv{static_cast<uint8_t*>(ws)};
    Planes px, pd;
    carve_pool_stats_bwd_test(cv, B, Tp, C, &px, &pd);
    PPV_CUDA_OK(cudaMemsetAsync(pd.base, 0x46, size_t(2) * pd.plane_stride * sizeof(__nv_bfloat16), st));  // the rows the kernel must not write
    if ((rc = launch_f32_to_planes(x, rows, C, px, st))) return rc;
    if ((rc = tr_pool_stats_bwd(px, C, B, T, P, Tp, pooled, dpooled, var != 0, pd, st))) return rc;
    return launch_planes_to_f32(pd, 0, C, 1, int(rows), 0, int(rows), dx, st);
    PPV_GUARD_END
}

// ---------------------------------------------------------------- CAM++ context mask test hook
// Workspace: h planes [2][B Tp][128], then w1t [128][64], b1 [64], w2t [64][32], b2 [32] fp32.
struct CpContextTestWs {
    __nv_bfloat16* h;
    float *w1t, *b1, *w2t, *b2;
};
static void carve_cp_context_test(WsCarver& cv, int B, int Tp, CpContextTestWs* v) {
    v->h = static_cast<__nv_bfloat16*>(cv.take(size_t(B) * Tp * 128 * 2 * sizeof(__nv_bfloat16)));
    v->w1t = static_cast<float*>(cv.take(128 * 64 * sizeof(float)));
    v->b1 = static_cast<float*>(cv.take(64 * sizeof(float)));
    v->w2t = static_cast<float*>(cv.take(64 * 32 * sizeof(float)));
    v->b2 = static_cast<float*>(cv.take(32 * sizeof(float)));
}
size_t ppv_campplus_context_test_workspace_bytes(int B, int Tp) {
    return carve_extent([&](WsCarver& cv) { CpContextTestWs v; carve_cp_context_test(cv, B, Tp, &v); });
}
int ppv_campplus_context_test(const float* h, int B, int T, int P, int Tp, const float* w1, const float* b1, const float* w2,
                              const float* b2, float* out, void* ws, size_t ws_bytes, void* stream) {
    PPV_GUARD_BEGIN
    PPV_REQUIRE(h && w1 && b1 && w2 && b2 && out, "ppv_campplus_context_test: null argument");
    PPV_REQUIRE(B > 0 && T > 0 && P >= 0 && Tp >= T + 2 * P, "ppv_campplus_context_test: bad shape");
    if (int rc = check_workspace("ppv_campplus_context_test", ws, ws_bytes, ppv_campplus_context_test_workspace_bytes(B, Tp),
                                 "ppv_campplus_context_test_workspace_bytes")) return rc;
    int rc = check_device();
    if (rc) return rc;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const int64_t rows = int64_t(B) * Tp;
    WsCarver cv{static_cast<uint8_t*>(ws)};
    CpContextTestWs v;
    carve_cp_context_test(cv, B, Tp, &v);
    const Planes ph{v.h, rows, 128, rows * 128};
    if ((rc = launch_f32_to_planes(h, rows, 128, ph, st))) return rc;
    std::vector<float> w1h(64 * 128), w2h(32 * 64), w1t, w2t;
    PPV_CUDA_OK(cudaMemcpyAsync(w1h.data(), w1, w1h.size() * sizeof(float), cudaMemcpyDeviceToHost, st));
    PPV_CUDA_OK(cudaMemcpyAsync(w2h.data(), w2, w2h.size() * sizeof(float), cudaMemcpyDeviceToHost, st));
    PPV_CUDA_OK(cudaStreamSynchronize(st));
    campplus_context_weights(w1h.data(), w2h.data(), &w1t, &w2t);
    PPV_CUDA_OK(cudaMemcpyAsync(v.w1t, w1t.data(), w1t.size() * sizeof(float), cudaMemcpyHostToDevice, st));
    PPV_CUDA_OK(cudaMemcpyAsync(v.w2t, w2t.data(), w2t.size() * sizeof(float), cudaMemcpyHostToDevice, st));
    PPV_CUDA_OK(cudaMemcpyAsync(v.b1, b1, 64 * sizeof(float), cudaMemcpyDeviceToDevice, st));
    PPV_CUDA_OK(cudaMemcpyAsync(v.b2, b2, 32 * sizeof(float), cudaMemcpyDeviceToDevice, st));
    rc = campplus_context_launch(ph, B, T, P, Tp, v.w1t, v.b1, v.w2t, v.b2, out, st);
    if (rc) return rc;
    PPV_CUDA_OK(cudaStreamSynchronize(st));  // the host copies of the weights die here
    return PPV_OK;
    PPV_GUARD_END
}

// ---------------------------------------------------------------- time-axis gather-GEMM test hook
// Workspace: each input's planes [2][rows][ld], then W planes [2][pad256(N)][sum ncols] (zero rows past N).
static void carve_taps_test(WsCarver& cv, const ppv_gemm_taps_case* c, Planes* in, Planes* pw) {
    int K = 0;
    for (int i = 0; i < c->ninputs; ++i) {
        in[i] = Planes{nullptr, c->rows[i], c->ld[i], c->rows[i] * c->ld[i]};
        in[i].base = static_cast<__nv_bfloat16*>(cv.take(size_t(2 * in[i].plane_stride) * sizeof(__nv_bfloat16)));
    }
    for (int j = 0; j < c->nsrc; ++j) K += c->src_ncols[j];
    *pw = cv.planes(int64_t(align_up(size_t(c->N), 256)), K);
}
size_t ppv_gemm_test_taps_workspace_bytes(const ppv_gemm_taps_case* c) {
    if (!c || c->ninputs > PPV_TAPS_MAX_INPUTS) return 0;
    return carve_extent([&](WsCarver& cv) { Planes in[PPV_TAPS_MAX_INPUTS], pw; carve_taps_test(cv, c, in, &pw); });
}
int ppv_gemm_test_taps(const ppv_gemm_taps_case* c, void* ws, size_t ws_bytes, void* stream) {
    PPV_GUARD_BEGIN
    PPV_REQUIRE(c && c->W && c->out, "ppv_gemm_test_taps: null argument");
    PPV_REQUIRE(c->ninputs > 0 && c->ninputs <= PPV_TAPS_MAX_INPUTS && c->nsrc > 0 && c->nsrc <= PPV_TAPS_MAX_SOURCES,
                "ppv_gemm_test_taps: 1-4 inputs and 1-16 sources");
    for (int i = 0; i < c->ninputs; ++i) PPV_REQUIRE(c->x[i] && c->rows[i] > 0 && c->ld[i] > 0, "ppv_gemm_test_taps: bad input");
    for (int j = 0; j < c->nsrc; ++j)
        PPV_REQUIRE(c->src_input[j] >= 0 && c->src_input[j] < c->ninputs && c->src_col0[j] >= 0 && c->src_ncols[j] > 0,
                    "ppv_gemm_test_taps: bad source");
    PPV_REQUIRE(c->M > 0 && c->N > 0 && c->out_rows > 0 && c->out_col0 >= 0 && c->out_col0 + c->N <= c->out_ld,
                "ppv_gemm_test_taps: bad output shape");
    PPV_REQUIRE(c->Tp == 0 || (c->T > 0 && c->P >= 0 && c->Tp >= c->T + 2 * c->P && c->M % c->Tp == 0 && c->out_rows >= c->M),
                "ppv_gemm_test_taps: bad time layout");
    PPV_REQUIRE(!c->seg_scale || (c->Tp > 0 && c->seg_len > 0 && c->nseg == (c->T + c->seg_len - 1) / c->seg_len),
                "ppv_gemm_test_taps: seg_scale needs the time layout and nseg = ceil(T / seg_len)");
    PPV_REQUIRE(c->precision == PPV_PREC_BF16X3 || c->precision == PPV_PREC_BF16, "ppv_gemm_test_taps: bad precision");
    if (int rc = check_workspace("ppv_gemm_test_taps", ws, ws_bytes, ppv_gemm_test_taps_workspace_bytes(c),
                                 "ppv_gemm_test_taps_workspace_bytes")) return rc;
    int rc = check_device();
    if (rc) return rc;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    WsCarver cv{static_cast<uint8_t*>(ws)};
    Planes in[PPV_TAPS_MAX_INPUTS], pw;
    carve_taps_test(cv, c, in, &pw);
    for (int i = 0; i < c->ninputs; ++i)
        if ((rc = launch_f32_to_planes(c->x[i], c->rows[i], c->ld[i], in[i], st))) return rc;
    std::vector<GemmSource> srcs;
    for (int j = 0; j < c->nsrc; ++j) srcs.push_back(GemmSource{in[c->src_input[j]], c->src_col0[j], c->src_ncols[j], c->src_row_off[j]});
    PPV_CUDA_OK(cudaMemsetAsync(pw.base, 0, size_t(2 * pw.plane_stride) * sizeof(__nv_bfloat16), st));
    if ((rc = launch_f32_to_planes(c->W, c->N, pw.ld, pw, st))) return rc;
    Epilogue ep;
    if (c->out_f32) {
        ep.out_mode = OUT_F32;
        ep.out = c->out;
        ep.out_ld = c->out_ld;
        ep.out_col0 = c->out_col0;
        ep.Tp = c->Tp;
        ep.P = c->P;
        ep.T = c->T;
    } else {
        const Planes po{static_cast<__nv_bfloat16*>(c->out), c->out_rows, c->out_ld, c->out_rows * c->out_ld};
        ep = planes_epilogue(po, c->out_col0, c->Tp, c->P, c->T);
    }
    ep.bias = c->bias;
    ep.bn_scale = c->bn_scale;
    ep.bn_shift = c->bn_shift;
    ep.relu = c->relu ? 1 : 0;
    ep.seg_scale = c->seg_scale;
    ep.seg_len = c->seg_len;
    ep.nseg = c->nseg;
    ep.halo = c->halo ? 1 : 0;
    ep.zero_invalid = c->zero_invalid ? 1 : 0;
    GemmParams gp;
    rc = gemm_build(&gp, srcs.data(), int(srcs.size()), pw, c->M, c->N, ep, c->block_n > 0 ? c->block_n : gemm_pick_bn(c->N), c->block_k);
    if (rc) return rc;
    return gemm_launch(gp, c->precision, device_sm_count(), st);
    PPV_GUARD_END
}

// ---------------------------------------------------------------- Res2Net test hook
// Workspace: x planes [2][B Tp][ld_x], y planes [2][B Tp + 64][ld_y], then per conv j the weight planes [2][128][(j ? 2 : 1) 192].
// y's tensor maps take in its 64 tail rows, so a store past the last utterance lands where the caller sees it.
struct Res2NetTestWs {
    Planes x, y, w[RES2CHAIN_MAX];
};
static void carve_res2net_test(WsCarver& cv, int nconv, int B, int Tp, int ld_x, int ld_y, Res2NetTestWs* v) {
    const int64_t rows = int64_t(B) * Tp;
    auto planes = [&](int64_t nrows, int ld) {
        return Planes{static_cast<__nv_bfloat16*>(cv.take(size_t(2 * nrows * ld) * sizeof(__nv_bfloat16))), nrows, ld, nrows * ld};
    };
    v->x = planes(rows, ld_x);
    v->y = planes(rows + 64, ld_y);
    for (int j = 0; j < nconv && j < RES2CHAIN_MAX; ++j) v->w[j] = cv.planes(64, (j ? 2 : 1) * 3 * 64);
}
size_t ppv_res2net_test_workspace_bytes(int nconv, int B, int T, int ld_x, int ld_y) {
    return carve_extent([&](WsCarver& cv) { Res2NetTestWs v; carve_res2net_test(cv, nconv, B, T + 8, ld_x, ld_y, &v); });
}
int ppv_res2net_test(float* x, int ld_x, const float* w, const float* bias, const float* bn_scale, const float* bn_shift, int nconv, int B,
                     int T, int dil, int variant, int precision, int max_ctas, float* y, int ld_y, void* ws, size_t ws_bytes, void* stream) {
    PPV_GUARD_BEGIN
    PPV_REQUIRE(x && w && bias && bn_scale && bn_shift && y, "ppv_res2net_test: null argument");
    constexpr int P = 4;  // the padding of every ECAPA-TDNN layer's output: the largest dilation
    PPV_REQUIRE(nconv >= 1 && nconv <= RES2CHAIN_MAX && B > 0 && T > P && max_ctas >= 0, "ppv_res2net_test: bad shape");
    PPV_REQUIRE(ld_x >= 64 * (nconv + 1) && ld_y >= 64 * (nconv + 1) && ld_x % 8 == 0 && ld_y % 8 == 0,
                "ppv_res2net_test: x and y need 64 (nconv + 1) columns and a 16-byte row pitch");
    PPV_REQUIRE(variant >= PPV_RES2_CHAIN && variant <= PPV_RES2_PER_CONV, "ppv_res2net_test: bad variant");
    PPV_REQUIRE(precision == PPV_PREC_BF16X3 || precision == PPV_PREC_BF16, "ppv_res2net_test: bad precision");
    const int Tp = T + 2 * P;
    if (int rc = check_workspace("ppv_res2net_test", ws, ws_bytes, ppv_res2net_test_workspace_bytes(nconv, B, T, ld_x, ld_y),
                                 "ppv_res2net_test_workspace_bytes")) return rc;
    int rc = check_device();
    if (rc) return rc;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    WsCarver cv{static_cast<uint8_t*>(ws)};
    Res2NetTestWs v;
    carve_res2net_test(cv, nconv, B, Tp, ld_x, ld_y, &v);
    const int R = B * Tp;
    // the launches, built as the ECAPA-TDNN plan builds them (ecapa.cu); the builds reject what the kernels do not take, before any launch
    Res2ChainParams cp;
    Res2Params rp[RES2CHAIN_MAX];
    if (variant == PPV_RES2_PER_CONV) {
        for (int j = 1; j <= nconv; ++j) {
            Epilogue ep = planes_epilogue(v.y, j * 64, Tp, P, T);
            ep.halo = 1;
            ep.relu = 1;
            ep.bias = bias + 64 * (j - 1);
            ep.bn_scale = bn_scale + 64 * (j - 1);
            ep.bn_shift = bn_shift + 64 * (j - 1);
            const GemmSource srcs[2] = {GemmSource{v.x, j * 64, 64, 0}, GemmSource{v.y, (j - 1) * 64, 64, 0}};
            if ((rc = res2conv_build(&rp[j - 1], srcs, j >= 2 ? 2 : 1, v.w[j - 1], R, dil, ep))) return rc;
        }
    } else {
        const float *bj[RES2CHAIN_MAX], *sj[RES2CHAIN_MAX], *hj[RES2CHAIN_MAX];
        for (int j = 0; j < nconv; ++j) bj[j] = bias + 64 * j, sj[j] = bn_scale + 64 * j, hj[j] = bn_shift + 64 * j;
        if ((rc = res2chain_build(&cp, v.x, v.y, v.w, bj, sj, hj, nconv, B, T, P, Tp, dil, variant == PPV_RES2_CHAIN_PAIRED))) return rc;
    }
    // weights [nconv][64][64][3] -> the model's matrices: the three taps of chunk j, and from conv 2 the same weights again for the
    // three taps of conv j-1's output
    std::vector<float> wh(size_t(nconv) * 64 * 64 * 3);
    PPV_CUDA_OK(cudaMemcpyAsync(wh.data(), w, wh.size() * sizeof(float), cudaMemcpyDeviceToHost, st));
    PPV_CUDA_OK(cudaStreamSynchronize(st));
    ArenaBuilder ab;
    GemmWeights gw[RES2CHAIN_MAX];
    for (int j = 0; j < nconv; ++j) {
        std::vector<ConvKGroup> groups = {{3, 64, 0, 64, 0}};
        if (j >= 1) groups.push_back({3, 64, 0, 64, 0});
        const std::vector<double> mtx = conv_weight_matrix(wh.data() + size_t(j) * 64 * 64 * 3, 64, 64, 3, 64, groups);
        ab.put_matrix(&gw[j], mtx, 64, int(mtx.size() / 64), 128);
        PPV_REQUIRE(gw[j].W.plane_stride == v.w[j].plane_stride, "ppv_res2net_test: weight layout mismatch");
        PPV_CUDA_OK(cudaMemcpyAsync(v.w[j].base, ab.host.data() + ab.patches[j].off, size_t(2 * v.w[j].plane_stride) * sizeof(__nv_bfloat16),
                                    cudaMemcpyHostToDevice, st));
    }
    PPV_CUDA_OK(cudaStreamSynchronize(st));  // the host matrices die here
    if ((rc = launch_f32_to_planes(x, R, ld_x, v.x, st)) || (rc = launch_f32_to_planes(y, v.y.rows, ld_y, v.y, st))) return rc;
    const int sms = max_ctas > 0 ? max_ctas : device_sm_count();
    if (variant == PPV_RES2_PER_CONV) {
        for (int j = 0; j < nconv; ++j)
            if ((rc = res2conv_launch(rp[j], precision, sms, st))) return rc;
    } else if ((rc = res2chain_launch(cp, precision, sms, st))) {
        return rc;
    }
    if ((rc = launch_planes_to_f32(v.x, 0, ld_x, R, 1, 0, 1, x, st))) return rc;
    // bf16: the convs read only the hi planes, and the chain stores no lo plane; y comes back as its hi plane
    if (precision == PPV_PREC_BF16) PPV_CUDA_OK(cudaMemsetAsync(v.y.lo(), 0, size_t(v.y.plane_stride) * sizeof(__nv_bfloat16), st));
    return launch_planes_to_f32(v.y, 0, ld_y, int(v.y.rows), 1, 0, 1, y, st);
    PPV_GUARD_END
}

// ---------------------------------------------------------------- skinny linear test hook
// Workspace: x planes [2][pad128(M)][ld], W planes [2][pad128(N)][K], output planes [2][pad128(M)][out_ld].
static void carve_skinny_test(WsCarver& cv, int M, int ld, int N, int K, int out_ld, Planes* px, Planes* pw, Planes* po) {
    *px = cv.planes(M, ld);
    *pw = cv.planes(N, K);
    *po = cv.planes(M, out_ld);
}
size_t ppv_skinny_linear_test_workspace_bytes(int M, int ld, int N, int K, int out_ld) {
    return carve_extent([&](WsCarver& cv) { Planes px, pw, po; carve_skinny_test(cv, M, ld, N, K, out_ld, &px, &pw, &po); });
}
int ppv_skinny_linear_test(const float* x, int M, int ld, int x_col0, const float* W, int N, int K, const float* bias, int act, int out_planes,
                           float* out, int out_ld, int out_col0, void* ws, size_t ws_bytes, void* stream) {
    PPV_GUARD_BEGIN
    PPV_REQUIRE(x && W && out, "ppv_skinny_linear_test: null argument");
    PPV_REQUIRE(M > 0 && N > 0 && K > 0 && x_col0 >= 0 && x_col0 + K <= ld && out_col0 >= 0 && out_col0 + N <= out_ld,
                "ppv_skinny_linear_test: bad shape");
    PPV_REQUIRE(act >= 0 && act <= 2, "ppv_skinny_linear_test: act must be 0 (none), 1 (ReLU) or 2 (sigmoid)");
    if (int rc = check_workspace("ppv_skinny_linear_test", ws, ws_bytes, ppv_skinny_linear_test_workspace_bytes(M, ld, N, K, out_ld),
                                 "ppv_skinny_linear_test_workspace_bytes")) return rc;
    int rc = check_device();
    if (rc) return rc;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    WsCarver cv{static_cast<uint8_t*>(ws)};
    Planes px, pw, po;
    carve_skinny_test(cv, M, ld, N, K, out_ld, &px, &pw, &po);
    Epilogue ep;
    if (out_planes) {
        ep = planes_epilogue(po, out_col0);
    } else {
        ep.out_mode = OUT_F32;
        ep.out = out;
        ep.out_ld = out_ld;
        ep.out_col0 = out_col0;
    }
    ep.bias = bias;
    ep.relu = act == 1;
    ep.sigmoid_ = act == 2;
    // what skinny_linear_launch requires, checked before anything is launched: no other kernel stands in
    PPV_REQUIRE(skinny_linear_supported(M, N, K, ep) && ld % 8 == 0 && x_col0 % 8 == 0,
                "ppv_skinny_linear_test: the skinny kernel does not take this shape");
    if ((rc = launch_f32_to_planes(x, M, ld, px, st)) || (rc = launch_f32_to_planes(W, N, K, pw, st))) return rc;
    if (out_planes && (rc = launch_f32_to_planes(out, M, out_ld, po, st))) return rc;
    if ((rc = skinny_linear_launch(px, x_col0, pw, M, N, K, ep, st))) return rc;
    return out_planes ? launch_planes_to_f32(po, 0, out_ld, M, 1, 0, 1, out, st) : PPV_OK;
    PPV_GUARD_END
}

// ppv_gemm_bench's workspace: the GEMM test hooks' operands, then the output [2][pad128(M)][N] (planes or fp32) and the epilogue
// vectors (bias, BN scale / shift, one bias per Tp-row utterance).
static void carve_gemm_bench(WsCarver& cv, int M, int N, int K, int Tp, Planes* pa, Planes* pw, Planes* po, float** vec) {
    carve_gemm_test(cv, M, N, K, pa, pw);
    *po = cv.planes(M, N);
    *vec = static_cast<float*>(cv.take((3 + size_t(M / Tp)) * size_t(N) * sizeof(float)));
}

// Kernel-only timing of the gather-GEMM (tools/gemm_bench.py): operands are converted once, the kernel is launched
// `iters` times between two CUDA events on `stream`; *ms_per_launch receives the average.  planes_out selects the epilogue:
//   0  ReLU, fp32 [M,N];   1  ReLU, split-bf16 planes (the layout every model layer writes);
//   2  the ECAPA TDNN layers: bias + ReLU + BN affine into planes over the padded time layout (Tp = 306, P = 4: T = 298);
//   3  the ASP attention TDNN (att1): bias + per-utterance bias + ReLU + BN affine + tanh, same layout.
// Modes 2 and 3 need M % 306 == 0.
int ppv_gemm_bench(int M, int N, int K, int block_n, int block_k, int precision, int planes_out, int iters, void* ws, size_t ws_bytes,
                   float* ms_per_launch, void* stream) {
    PPV_GUARD_BEGIN
    PPV_REQUIRE(ms_per_launch && iters > 0, "ppv_gemm_bench: bad argument");
    PPV_REQUIRE(planes_out >= 0 && planes_out <= 3, "ppv_gemm_bench: planes_out must be 0-3");
    constexpr int kTp = 306, kP = 4;
    PPV_REQUIRE(planes_out < 2 || M % kTp == 0, "ppv_gemm_bench: model epilogues need M % 306 == 0");
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    WsCarver cv;
    Planes pa, pw, po;
    float* vec;
    carve_gemm_bench(cv, M, N, K, kTp, &pa, &pw, &po, &vec);
    const size_t need = align_up(cv.off, 256);
    if (int rc = check_workspace("ppv_gemm_bench", ws, ws_bytes, need, "see ppv_gemm_bench in ppv_b200.h")) return rc;
    cv = WsCarver{static_cast<uint8_t*>(ws)};
    carve_gemm_bench(cv, M, N, K, kTp, &pa, &pw, &po, &vec);
    PPV_CUDA_OK(cudaMemsetAsync(ws, 0x11, reinterpret_cast<uint8_t*>(po.base) - static_cast<uint8_t*>(ws), st));  // small finite bf16 values
    PPV_CUDA_OK(cudaMemsetAsync(vec, 0x3c, static_cast<uint8_t*>(ws) + need - reinterpret_cast<uint8_t*>(vec), st));  // small finite floats (0.0115)
    GemmSource src{pa, 0, pa.ld, 0};
    Epilogue ep;
    if (planes_out >= 2) {
        ep = planes_epilogue(po, 0, kTp, kP, kTp - 2 * kP);
        ep.bias = vec; ep.bn_scale = vec + N; ep.bn_shift = vec + 2 * N;
        if (planes_out == 3) { ep.rowgrp_bias = vec + 3 * N; ep.tanh_ = 1; }
    } else if (planes_out) {
        ep = planes_epilogue(po);
    } else {
        ep.out_mode = OUT_F32; ep.out = po.base; ep.out_ld = N;
    }
    ep.relu = 1;
    GemmParams gp;
    int rc = gemm_build(&gp, &src, 1, pw, M, N, ep, block_n, block_k);
    if (rc) return rc;
    const int sms = device_sm_count();
    for (int i = 0; i < 3; ++i) { rc = gemm_launch(gp, precision, sms, st); if (rc) return rc; }
    cudaEvent_t e0, e1;
    PPV_CUDA_OK(cudaEventCreate(&e0));
    PPV_CUDA_OK(cudaEventCreate(&e1));
    PPV_CUDA_OK(cudaEventRecord(e0, st));
    for (int i = 0; i < iters; ++i) { rc = gemm_launch(gp, precision, sms, st); if (rc) return rc; }
    PPV_CUDA_OK(cudaEventRecord(e1, st));
    PPV_CUDA_OK(cudaEventSynchronize(e1));
    float ms = 0.f;
    PPV_CUDA_OK(cudaEventElapsedTime(&ms, e0, e1));
    cudaEventDestroy(e0);
    cudaEventDestroy(e1);
    gemm_trace_dump(gp);  // PPV_GEMM_TRACE: the last timed launch
    *ms_per_launch = ms / float(iters);
    return PPV_OK;
    PPV_GUARD_END
}

}  // extern "C"
