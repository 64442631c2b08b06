// extern "C" boundary of libppv_b200 (include/ppv_b200.h): argument checking, handle unwrapping, error text.
// No exceptions cross this boundary; everything returns a status code.
#include <string.h>

#include <new>

#include "common.h"
#include "image_plan.h"
#include "model_common.h"

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
    int kind;
    Model* m;
};

// The model behind an ECAPA-TDNN handle, else null: the entry points that only ECAPA-TDNN has.
static Model* ecapa_of(const ppv_model* h) { return h && h->kind == PPV_MODEL_ECAPA_TDNN ? h->m : nullptr; }

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

int ppv_model_create(int kind, const void* cfg, ppv_model_t** out) {
    PPV_GUARD_BEGIN
    PPV_REQUIRE(cfg && out, "ppv_model_create: null argument");
    if (kind != PPV_MODEL_ECAPA_TDNN && kind != PPV_MODEL_RESNET_SE && kind != PPV_MODEL_ERES2NET && kind != PPV_MODEL_CAMPPLUS)
        return fail(PPV_EUNSUPPORTED,
                    "ppv_model_create: implemented kinds are PPV_MODEL_ECAPA_TDNN, PPV_MODEL_RESNET_SE, PPV_MODEL_ERES2NET, PPV_MODEL_CAMPPLUS");
    int rc = check_device();
    if (rc) return rc;
    Model* m = nullptr;
    switch (kind) {
        case PPV_MODEL_ECAPA_TDNN: rc = ecapa_create(static_cast<const ppv_ecapa_cfg*>(cfg), &m); break;
        case PPV_MODEL_RESNET_SE: rc = resnetse_create(static_cast<const ppv_resnetse_cfg*>(cfg), &m); break;
        case PPV_MODEL_ERES2NET: rc = eres2net_create(static_cast<const ppv_eres2net_cfg*>(cfg), &m); break;
        default: rc = campplus_create(static_cast<const ppv_campplus_cfg*>(cfg), &m); break;
    }
    if (rc) return rc;
    *out = new ppv_model{kind, m};
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
    return h->m->forward(feat, B, T, emb, ws, ws_bytes, static_cast<cudaStream_t>(stream));
    PPV_GUARD_END
}
int ppv_model_forward_lengths(ppv_model_t* h, const float* feat, const float* lengths, int B, int T, float* emb, void* ws, size_t ws_bytes,
                              void* stream) {
    PPV_GUARD_BEGIN
    PPV_REQUIRE(h && feat && emb, "ppv_model_forward_lengths: null argument");
    if (!ecapa_of(h)) return fail(PPV_EUNSUPPORTED, "ppv_model_forward_lengths: only EcapaTdnn.forward takes lengths in the reference");
    return ecapa_forward(h->m, feat, nullptr, nullptr, nullptr, B, T, 0, emb, ws, ws_bytes, static_cast<cudaStream_t>(stream), lengths);
    PPV_GUARD_END
}
int ppv_model_forward_wav(ppv_model_t* h, ppv_fbank_t* fb, const float* wav, const float* lens_ratio, int B, int L, float* emb,
                          void* ws, size_t ws_bytes, void* stream) {
    PPV_GUARD_BEGIN
    PPV_REQUIRE(h && fb && wav && emb, "ppv_model_forward_wav: null argument");
    if (!ecapa_of(h)) return fail(PPV_EUNSUPPORTED, "ppv_model_forward_wav: the fused waveform path exists for ECAPA-TDNN only; call ppv_fbank_forward + ppv_model_forward");
    const int T = fbank_num_frames(fb->impl, L);
    PPV_REQUIRE(T > 0, "ppv_model_forward_wav: waveform shorter than one frame");
    return ecapa_forward(h->m, nullptr, fb->impl, wav, lens_ratio, B, T, L, emb, ws, ws_bytes, static_cast<cudaStream_t>(stream));
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
    PPV_REQUIRE(ecapa_of(h), "ppv_model_profile: ECAPA-TDNN model required");
    return ecapa_profile(h->m, enable);
}
int ppv_model_profile_read(ppv_model_t* h, double* gemm_ms, double* other_ms, int64_t* gemm_launches, int64_t* other_launches) {
    PPV_GUARD_BEGIN
    PPV_REQUIRE(ecapa_of(h), "ppv_model_profile_read: ECAPA-TDNN model required");
    return ecapa_profile_read(h->m, gemm_ms, other_ms, gemm_launches, other_launches);
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
    rc = trainer_create(cfg, num_classes, &impl);
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

// ---------------------------------------------------------------- GEMM test hook
static inline size_t au(size_t x, size_t a) { return (x + a - 1) / a * a; }
size_t ppv_gemm_test_workspace_bytes(int M, int N, int K) {
    const size_t Kp = au(size_t(K), 64);
    return au(au(size_t(M), 128) * Kp * 4, 256) + au(au(size_t(N), 256) * Kp * 4, 256) + 256;
}
// Both hooks' operands in the workspace, zero-padded: A as planes [2][pad128(M)][Kp], then W as planes [2][pad256(N)][Kp], Kp = pad64(K).
static int gemm_test_stage(const float* A, const float* W, int M, int N, int K, void* ws, cudaStream_t st, Planes* pa, Planes* pw) {
    const int Kp = int(au(size_t(K), 64));
    pa->rows = int64_t(au(size_t(M), 128));
    pa->ld = Kp;
    pa->plane_stride = pa->rows * Kp;
    pa->base = static_cast<__nv_bfloat16*>(ws);
    pw->rows = int64_t(au(size_t(N), 256));
    pw->ld = Kp;
    pw->plane_stride = pw->rows * Kp;
    pw->base = reinterpret_cast<__nv_bfloat16*>(static_cast<uint8_t*>(ws) + au(size_t(pa->plane_stride) * 4, 256));
    PPV_CUDA_OK(cudaMemsetAsync(ws, 0, ppv_gemm_test_workspace_bytes(M, N, K), st));
    int rc = launch_f32_to_planes(A, M, K, *pa, st);
    if (rc) return rc;
    return launch_f32_to_planes(W, N, K, *pw, st);
}
int ppv_gemm_test(const float* A, const float* W, const float* bias, const float* bn_scale, const float* bn_shift, int relu, int M,
                  int N, int K, int block_n, int block_k, int precision, float* out, void* ws, size_t ws_bytes, void* stream) {
    PPV_GUARD_BEGIN
    PPV_REQUIRE(A && W && out && ws, "ppv_gemm_test: null argument");
    PPV_REQUIRE(ws_bytes >= ppv_gemm_test_workspace_bytes(M, N, K), "ppv_gemm_test: workspace too small");
    int rc = check_device();
    if (rc) return rc;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    Planes pa, pw;
    rc = gemm_test_stage(A, W, M, N, K, ws, st, &pa, &pw);
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
    PPV_REQUIRE(A && W && out && ws, "ppv_gemm_test_planes: null argument");
    PPV_REQUIRE(ws_bytes >= ppv_gemm_test_workspace_bytes(M, N, K), "ppv_gemm_test_planes: workspace too small");
    PPV_REQUIRE(N % 32 == 0 && (Tp == 0 || (M % Tp == 0 && Tp > 2 * P)), "ppv_gemm_test_planes: bad shape");
    int rc = check_device();
    if (rc) return rc;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    Planes pa, pw;
    rc = gemm_test_stage(A, W, M, N, K, ws, st, &pa, &pw);
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
static size_t conv2d_test_x_bytes(int B, int H, int W, int x_ld) {
    return au(au(size_t(B) * (H + 2) * (W + 2), 128) * size_t(x_ld) * 4, 256);
}
size_t ppv_conv2d_test_workspace_bytes(int B, int H, int W, int Cin, int Cout, int k, int x_ld) {
    if (x_ld <= 0) x_ld = Cin;
    return conv2d_test_x_bytes(B, H, W, x_ld) + au(au(size_t(Cout), 256) * k * k * Cin * 4, 256) + 256;
}
int ppv_conv2d_test(const float* x, const float* w, const float* bias, int relu, int B, int H, int W, int Cin, int Cout, int k,
                    int stride_h, int stride_w, int x_col0, int x_ld, int path, int precision, void* out, void* ws, size_t ws_bytes,
                    void* stream) {
    PPV_GUARD_BEGIN
    PPV_REQUIRE(x && w && out && ws, "ppv_conv2d_test: null argument");
    if (x_ld <= 0) x_ld = Cin;
    PPV_REQUIRE(B > 0 && H > 0 && W > 0 && Cin > 0 && Cout > 0 && (k == 1 || k == 3) && stride_h >= 1 && stride_w >= 1,
                "ppv_conv2d_test: bad shape");
    PPV_REQUIRE(x_col0 >= 0 && x_col0 + Cin <= x_ld, "ppv_conv2d_test: the input columns exceed x_ld");
    PPV_REQUIRE(path >= 0 && path <= 2, "ppv_conv2d_test: path must be 0 (3x3 patch kernel), 1 (pointwise kernel) or 2 (gather-GEMM)");
    PPV_REQUIRE(precision == PPV_PREC_BF16X3 || precision == PPV_PREC_BF16, "ppv_conv2d_test: bad precision");
    PPV_REQUIRE(ws_bytes >= ppv_conv2d_test_workspace_bytes(B, H, W, Cin, Cout, k, x_ld), "ppv_conv2d_test: workspace too small");
    const int Hp = H + 2, Wp = W + 2, Ho = (H - 1) / stride_h + 1, Wo = (W - 1) / stride_w + 1;
    const int64_t M = int64_t(B) * Hp * Wp;
    PPV_REQUIRE(M < (int64_t(1) << 31) && Wp + 1 < 32768, "ppv_conv2d_test: grid too large for 32-bit rows / 16-bit tap offsets");
    int rc = check_device();
    if (rc) return rc;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    // input grid: zero border; x at columns [x_col0, x_col0 + Cin) of the interior; the other columns hold 0x3f3f (0.746 in bf16) in
    // both planes, so a kernel that reads outside its column window is visibly wrong
    Planes xp;
    xp.rows = int64_t(au(size_t(M), 128));
    xp.ld = x_ld;
    xp.plane_stride = xp.rows * x_ld;
    xp.base = static_cast<__nv_bfloat16*>(ws);
    const size_t x_bytes = conv2d_test_x_bytes(B, H, W, x_ld);
    PPV_CUDA_OK(cudaMemsetAsync(ws, 0, x_bytes, st));
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
    uint8_t* wdev = static_cast<uint8_t*>(ws) + x_bytes;
    PPV_CUDA_OK(cudaMemcpyAsync(wdev, ab.host.data(), ab.host.size(), cudaMemcpyHostToDevice, st));
    PPV_CUDA_OK(cudaStreamSynchronize(st));
    gw.W.base = reinterpret_cast<__nv_bfloat16*>(wdev + ab.patches[0].off);
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

// ---------------------------------------------------------------- fused attentive-statistics pooling test hook
// Workspace: W planes [2][C][K], att planes [2][B Tp + 64][K], x planes [2][B Tp + 64][C], out planes [2][B][2C].  The tensor
// maps of att and x end at row B Tp; the 64 rows behind hold 0x4646 (12672 in bf16) in both planes.
static size_t asp_test_sizes(int B, int Tp, int C, int K, size_t* off) {
    const size_t rows = size_t(B) * Tp + 64;
    const size_t sz[4] = {size_t(C) * K, rows * K, rows * C, size_t(B) * 2 * C};
    size_t o = 0;
    for (int i = 0; i < 4; ++i) {
        off[i] = o;
        o += au(2 * sz[i] * sizeof(__nv_bfloat16), 256);
    }
    return o;
}
size_t ppv_asp_fused_test_workspace_bytes(int B, int Tp, int C, int K) {
    size_t off[4];
    return asp_test_sizes(B, Tp, C, K, off);
}
int ppv_asp_fused_test(const float* W, const float* att, const float* x, const float* bn_scale, const float* bn_shift,
                       const int* nvalid, int B, int T, int P, int Tp, int C, int K, int precision, int max_ctas, float* out_raw,
                       float* out, void* ws, size_t ws_bytes, void* stream) {
    PPV_GUARD_BEGIN
    PPV_REQUIRE(W && att && x && bn_scale && bn_shift && out_raw && out && ws, "ppv_asp_fused_test: null argument");
    PPV_REQUIRE(B > 0 && T > 0 && P >= 0 && Tp >= T + 2 * P && max_ctas >= 0, "ppv_asp_fused_test: bad shape");
    PPV_REQUIRE(precision == PPV_PREC_BF16X3 || precision == PPV_PREC_BF16, "ppv_asp_fused_test: bad precision");
    size_t off[4];
    PPV_REQUIRE(ws_bytes >= asp_test_sizes(B, Tp, C, K, off), "ppv_asp_fused_test: workspace too small");
    int rc = check_device();
    if (rc) return rc;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    uint8_t* w8 = static_cast<uint8_t*>(ws);
    const int64_t rows = int64_t(B) * Tp;
    auto planes = [&](int i, int64_t nrows, int ld, int64_t alloc_rows) {
        return Planes{reinterpret_cast<__nv_bfloat16*>(w8 + off[i]), nrows, ld, alloc_rows * ld};
    };
    const Planes pw = planes(0, C, K, C), pa = planes(1, rows, K, rows + 64), px = planes(2, rows, C, rows + 64),
                 po = planes(3, B, 2 * C, B);
    PPV_CUDA_OK(cudaMemsetAsync(w8 + off[1], 0x46, off[3] - off[1], st));
    if ((rc = launch_f32_to_planes(W, C, K, pw, st)) || (rc = launch_f32_to_planes(att, rows, K, pa, st)) ||
        (rc = launch_f32_to_planes(x, rows, C, px, st)))
        return rc;
    AspFusedParams ap;
    rc = asp_fused_build(&ap, pw, pa, px, bn_scale, bn_shift, po, out_raw, B, T, P, Tp, C, K, 1e-12f);
    if (rc) return rc;
    ap.nvalid = nvalid;
    rc = asp_fused_launch(ap, precision, max_ctas > 0 ? max_ctas : device_sm_count(), st);
    if (rc) return rc;
    return launch_planes_to_f32(po, 0, 2 * C, B, 1, 0, 1, out, st);
    PPV_GUARD_END
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
    PPV_REQUIRE(ws && ms_per_launch && iters > 0, "ppv_gemm_bench: bad argument");
    PPV_REQUIRE(planes_out >= 0 && planes_out <= 3, "ppv_gemm_bench: planes_out must be 0-3");
    constexpr int kTp = 306, kP = 4;
    PPV_REQUIRE(planes_out < 2 || M % kTp == 0, "ppv_gemm_bench: model epilogues need M % 306 == 0");
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const size_t Kp = au(size_t(K), 64);
    const size_t a_bytes = au(au(size_t(M), 128) * Kp * 4, 256), w_bytes = au(au(size_t(N), 256) * Kp * 4, 256);
    const size_t o_bytes = au(au(size_t(M), 128) * size_t(N) * 4, 256);
    const size_t v_bytes = au((3 + size_t(M / kTp)) * size_t(N) * 4, 256);  // bias, BN scale / shift, per-utterance bias
    PPV_REQUIRE(ws_bytes >= a_bytes + w_bytes + o_bytes + v_bytes, "ppv_gemm_bench: workspace too small");
    Planes pa, pw, po;
    pa.rows = int64_t(au(size_t(M), 128)); pa.ld = int(Kp); pa.plane_stride = pa.rows * pa.ld; pa.base = static_cast<__nv_bfloat16*>(ws);
    pw.rows = int64_t(au(size_t(N), 256)); pw.ld = int(Kp); pw.plane_stride = pw.rows * pw.ld;
    pw.base = reinterpret_cast<__nv_bfloat16*>(static_cast<uint8_t*>(ws) + a_bytes);
    po.rows = pa.rows; po.ld = N; po.plane_stride = po.rows * po.ld;
    po.base = reinterpret_cast<__nv_bfloat16*>(static_cast<uint8_t*>(ws) + a_bytes + w_bytes);
    PPV_CUDA_OK(cudaMemsetAsync(ws, 0x11, a_bytes + w_bytes, st));  // small finite bf16 values
    float* vec = reinterpret_cast<float*>(static_cast<uint8_t*>(ws) + a_bytes + w_bytes + o_bytes);
    PPV_CUDA_OK(cudaMemsetAsync(vec, 0x3c, v_bytes, st));  // small finite floats (0.0115)
    GemmSource src{pa, 0, int(Kp), 0};
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
