/* libppv_b200 -- C ABI of the H100-native ppvector hot path.
 *
 * The reference (yeyupiaoling/VoiceprintRecognition-PaddlePaddle) has NO plugin / FFI interface:
 * its boundary is the Python class surface.  Each entry point below names the reference
 * call site it sits under (paths relative to the reference checkout); INTEGRATION.md shows the
 * ctypes binding.  Conventions (SURVEY.md §8b):
 *   - plain pointers and sizes only; every tensor pointer is DEVICE memory owned by the caller,
 *     row-major contiguous; the library never frees caller memory and allocates nothing per call
 *     (per-call scratch is the caller's workspace);
 *   - every call is asynchronous on `stream` (a cudaStream_t passed as void*), no hidden sync;
 *   - return value: 0 = PPV_OK, negative = error; ppv_last_error() gives the text;
 *   - sm_90a (H100) only; there is no CPU fallback.
 */
#ifndef PPV_B200_H
#define PPV_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define PPV_OK 0
#define PPV_EINVAL (-1)       /* bad shape / null pointer / alignment */
#define PPV_ECUDA (-2)        /* a CUDA runtime or driver call failed */
#define PPV_EUNSUPPORTED (-3) /* configuration outside what the kernels implement */
#define PPV_ESTATE (-4)       /* call order violated (e.g. forward before finalize) */

/* Tensor-core contraction precision of the model GEMMs. */
#define PPV_PREC_BF16X3 0 /* split-bf16, 3 MMAs per product: fp32-grade (parity mode, default) */
#define PPV_PREC_BF16 1   /* single bf16 MMA: fast mode, ~1e-2 relative on embeddings */

/* EcapaTdnn(pooling_type=...): ASP = attentive statistics (pooling.py:69-125), SAP = self-attentive (:50-66),
 * TAP = temporal average (:8-25), TSP = temporal mean | unbiased variance (:28-47). */
#define PPV_POOL_ASP 0
#define PPV_POOL_SAP 1
#define PPV_POOL_TAP 2
#define PPV_POOL_TSP 3

typedef struct ppv_fbank ppv_fbank_t;
typedef struct ppv_model ppv_model_t;

int ppv_version(void);
/* Copies the calling thread's last error text (NUL-terminated) into buf; returns its length. */
int ppv_last_error(char* buf, size_t n);
/* Device properties the Python host needs without importing torch.cuda: SM count of the current device. */
int ppv_device_sm_count(void);

/* ---------------------------------------------------------------------------------------------
 * Fbank front end.  Replaces ppvector/data_utils/featurizer.py:88-101 (KaldiFbank.forward ->
 * paddleaudio.compliance.kaldi.fbank per utterance) and :33-60 (AudioFeaturizer.forward:
 * transpose, subtract the time mean, optional tail mask).
 *
 * The window is int(sample_rate * frame_length_ms / 1000) samples and is zero-padded to the next power of two, which must lie in
 * [128, 4096].  A 512-point FFT with snip_edges, remove_dc_offset, use_power and use_log_fbank runs on a register-resident kernel
 * built for that size; every other configuration runs on a general per-frame kernel.  ppv_fbank_create picks one from the config.
 * ------------------------------------------------------------------------------------------- */
#define PPV_FBANK_WIN_POVEY 0
#define PPV_FBANK_WIN_HANNING 1
#define PPV_FBANK_WIN_HAMMING 2
#define PPV_FBANK_WIN_RECTANGULAR 3
#define PPV_FBANK_WIN_BLACKMAN 4
typedef struct {
    int sample_rate;       /* 16000 */
    int n_mels;            /* 80 (<= 128) */
    float frame_length_ms; /* 25 */
    float frame_shift_ms;  /* 10 */
    float preemph;         /* 0.97 */
    float low_freq;        /* 20 */
    float high_freq;       /* 0 => Nyquist */
    float log_floor;       /* 1.1920929e-07 (FLT_EPSILON) */
    int window_type;       /* PPV_FBANK_WIN_POVEY */
    float blackman_coeff;  /* 0.42 */
    int remove_dc_offset;  /* 1: subtract each frame's mean */
    int snip_edges;        /* 1: only frames that fit; 0: (L + shift/2) / shift frames over the edge-reflected waveform */
    int use_power;         /* 1: power spectrum; 0: magnitude */
    int use_log_fbank;     /* 1: log(max(mel, log_floor)); 0: linear mel energies */
    float vtln_warp;       /* 1 => no warping */
    float vtln_low;        /* 100 */
    float vtln_high;       /* -500 => offset from Nyquist */
} ppv_fbank_cfg;

void ppv_fbank_default_cfg(ppv_fbank_cfg* cfg);
int ppv_fbank_create(const ppv_fbank_cfg* cfg, ppv_fbank_t** out);
int ppv_fbank_destroy(ppv_fbank_t* h);
/* As ppv_fbank_forward for a zero-padded batch of utterances of DIFFERENT lengths, each featurised as if alone (the training data
 * path, reader.py:101-104 + collate_fn.py:5-23): valid_frames[b] (device int32) frames of utterance b are real; the time mean is taken
 * over those only and frames beyond them are written as zeros.  With snip_edges = 0 the frames at an utterance's end reflect the
 * padding instead of its own samples: use ppv_fbank_forward_ragged_samples there. */
int ppv_fbank_forward_ragged(ppv_fbank_t* h, const float* wav, const int32_t* valid_frames, int B, int L, float* out, void* stream);
/* As ppv_fbank_forward_ragged, and num_samples[b] (device int32, <= L) is utterance b's own length, where its right edge is reflected
 * when snip_edges = 0; valid_frames[b] must be ppv_fbank_num_frames(h, num_samples[b]). */
int ppv_fbank_forward_ragged_samples(ppv_fbank_t* h, const float* wav, const int32_t* valid_frames, const int32_t* num_samples, int B, int L,
                                     float* out, void* stream);
/* Frame count for L samples: snip_edges: 1 + (L - window) / shift (0 if L < window); otherwise (L + shift/2) / shift, or 0 when the
 * reflected waveform is too short to hold the last frame (torchaudio's _get_strided cannot frame it either). */
int ppv_fbank_num_frames(const ppv_fbank_t* h, int L);
int ppv_fbank_feature_dim(const ppv_fbank_t* h);
/* wav [B,L] fp32 in [-1,1] -> out [B,T,n_mels] fp32, time-mean subtracted; if lens_ratio != NULL,
 * frames t >= int(lens_ratio[b] * T) are zeroed AFTER the mean subtraction (featurizer.py:48-59). */
int ppv_fbank_forward(ppv_fbank_t* h, const float* wav, const float* lens_ratio, int B, int L, float* out,
                      void* stream);

/* ---------------------------------------------------------------------------------------------
 * STFT front ends.  Replace paddle.audio.features.{Spectrogram, MelSpectrogram, LogMelSpectrogram, MFCC} as
 * constructed by ppvector/data_utils/featurizer.py:20-27, plus featurizer.py:43-59 (transpose, time-mean
 * subtraction, tail mask).  Defaults of ppv_spectral_default_cfg are the library's own (sr 22050, n_fft 2048
 * (Spectrogram: 512), hop 512, hann, centred with reflect padding, power 2 (Spectrogram: 1), 64 slaney mels from
 * 50 Hz, amin 1e-10, ref 1, top_db None, 40 MFCCs with an orthonormal DCT-II).  top_db is not implemented.
 * ------------------------------------------------------------------------------------------- */
#define PPV_SPEC_SPECTROGRAM 1
#define PPV_SPEC_MEL 2
#define PPV_SPEC_LOGMEL 3
#define PPV_SPEC_MFCC 4
typedef struct {
    int method;      /* PPV_SPEC_* */
    int sample_rate; /* 22050 */
    int n_fft;       /* power of two in [32, 4096] */
    int hop_length;  /* 512 */
    int win_length;  /* 0 => n_fft */
    float power;     /* exponent of |X| */
    int center;      /* 1: reflect-pad n_fft/2 on both sides */
    int n_mels;      /* 64 */
    float f_min;     /* 50 */
    float f_max;     /* 0 => sample_rate / 2 */
    int htk;         /* 0: slaney mel scale */
    int norm_slaney; /* 1: area-normalised filters */
    float ref_value; /* 1 */
    float amin;      /* 1e-10 */
    int n_mfcc;      /* 40 */
} ppv_spectral_cfg;
typedef struct ppv_spectral ppv_spectral_t;
void ppv_spectral_default_cfg(ppv_spectral_cfg* cfg, int method);
int ppv_spectral_create(const ppv_spectral_cfg* cfg, ppv_spectral_t** out);
int ppv_spectral_destroy(ppv_spectral_t* h);
/* centred: 1 + L / hop (needs L > n_fft / 2); else 1 + (L - n_fft) / hop. */
int ppv_spectral_num_frames(const ppv_spectral_t* h, int L);
int ppv_spectral_feature_dim(const ppv_spectral_t* h);
/* wav [B,L] fp32 -> out [B,T,F] fp32, time-mean subtracted, optional tail mask as in ppv_fbank_forward. */
int ppv_spectral_forward(ppv_spectral_t* h, const float* wav, const float* lens_ratio, int B, int L, float* out, void* stream);
/* A zero-padded batch of utterances of DIFFERENT lengths in one launch sequence, as ppv_fbank_forward_ragged_samples.  wav [B,L] fp32;
 * num_samples[b] (device int32, <= L) is utterance b's own length; valid_frames[b] (device int32) must be
 * ppv_spectral_num_frames(h, num_samples[b]).  out [B,T,F], T = ppv_spectral_num_frames(h, L): row b holds utterance b featurised
 * as if alone (centre reflect padding at both of ITS ends, time mean over its own valid_frames[b] frames), zeros beyond.  Lengths
 * out of range are clamped (valid_frames to [0, T], num_samples to [1, L]): that row's features are wrong, nothing outside it is
 * read or written.  PPV_EINVAL for a null pointer, B outside [1, 65535] or L too short for one frame. */
int ppv_spectral_forward_ragged_samples(ppv_spectral_t* h, const float* wav, const int32_t* valid_frames, const int32_t* num_samples,
                                        int B, int L, float* out, void* stream);

/* SpecAugment masking of a feature batch in place (ppvector/data_utils/reader.py:105-107, configs/augmentation.yml:36-48,
 * max_time_warp 0).  The random draws stay on the host, made with the reference's RNG calls; params is int32
 * [B][PPV_SPECAUG_NPARAM] on the device: {apply (0/1), T_b = frames of utterance b, n_freq_masks x (f0, width),
 * n_time_masks x (t0, width)}.  fill_mode 0 writes zeros, 1 the utterance's mean over its T_b x F values before masking. */
#define PPV_SPECAUG_NPARAM 16
int ppv_spec_augment(float* feat, const int32_t* params, int B, int T, int F, int n_freq_masks, int n_time_masks, int fill_mode,
                     void* stream);

/* ---------------------------------------------------------------------------------------------
 * Speaker-embedding model.  Replaces <Model>.forward, reached from
 * ppvector/predict.py:228-233, :265-266 and ppvector/trainer.py:391-410 (eval mode, lengths=None).
 * kind PPV_MODEL_ECAPA_TDNN: ppvector/models/ecapa_tdnn.py:245-276 with
 * pooling.py:86-125 (ASP, global_context) and models/utils.py:65-148.
 * ------------------------------------------------------------------------------------------- */
#define PPV_MODEL_ECAPA_TDNN 1

typedef struct {
    int input_size;  /* 80 */
    int embd_dim;    /* 192 */
    int channels[5]; /* 512,512,512,512,1536 */
    int kernel_sizes[5];
    int dilations[5];
    int attention_channels; /* 128 */
    int res2net_scale;      /* 8 */
    int se_channels;        /* 128 */
    int precision;          /* PPV_PREC_* */
    int pooling;            /* PPV_POOL_*: ecapa_tdnn.py:212-241 pooling_type */
    int global_context;     /* 1 (default): ASP attends over [x; mean; std] (pooling.py:104-107); 0: over x alone */
} ppv_ecapa_cfg;

void ppv_ecapa_default_cfg(ppv_ecapa_cfg* cfg);

/* kind PPV_MODEL_RESNET_SE: ppvector/models/resnet_se.py:121-139 (SEBottleneck :24-45, SELayer :59-63), ASP head. */
#define PPV_MODEL_RESNET_SE 2
typedef struct {
    int input_size;         /* 80 (must be a multiple of 8) */
    int embd_dim;           /* 192 */
    int layers[4];          /* 3,4,6,3 */
    int num_filters[4];     /* 32,64,128,256 */
    int attention_channels; /* 128 */
    int reduction;          /* 8 (SELayer) */
    int precision;          /* PPV_PREC_* */
} ppv_resnetse_cfg;
void ppv_resnetse_default_cfg(ppv_resnetse_cfg* cfg);

/* kind PPV_MODEL_ERES2NET: ppvector/models/eres2net.py:239-263 (blocks :85-108, :147-170, AFF :46-52), TSTP head;
 * scale 2, expansion 2, base_width 32, one embedding layer (configs/eres2net.yml).  version = 2 selects ERes2NetV2
 * (eres2net.py:266-462: the same blocks at base_width 26, i.e. chunk widths 13 / 26 / 52 / 104 zero-padded to 32 / 32 / 64 / 128 columns,
 * AFF blocks in layers 3-4, `layer3_ds` + `fuse34` instead of the three-level bottom-up fusion; state_dict names as the reference's). */
#define PPV_MODEL_ERES2NET 3
typedef struct {
    int input_size;    /* 80 (must be a multiple of 8) */
    int embd_dim;      /* 192 */
    int num_blocks[4]; /* 3,4,6,3 */
    int m_channels;    /* 32 (or 64) */
    int precision;     /* PPV_PREC_* */
    int version;       /* 1 = ERes2Net (default; 0 means 1), 2 = ERes2NetV2 */
    int base_width;    /* 32 for ERes2Net; ERes2NetV2: 26 (0 means the version's default) */
} ppv_eres2net_cfg;
void ppv_eres2net_default_cfg(ppv_eres2net_cfg* cfg);

/* kind PPV_MODEL_CAMPPLUS: ppvector/models/campplus.py:292-346 (FCM head :254-289, CAM dense TDNN layers :67-141,
 * transit :174-186, statistics pooling :24-31, dense :189-204); blocks 12/24/16, dilations 1/2/2 (configs/cam++.yml). */
#define PPV_MODEL_CAMPPLUS 4
typedef struct {
    int input_size;    /* 80 (must be a multiple of 8) */
    int embd_dim;      /* 192 */
    int growth_rate;   /* 32 */
    int bn_size;       /* 4 */
    int init_channels; /* 128 */
    int precision;     /* PPV_PREC_* */
} ppv_campplus_cfg;
void ppv_campplus_default_cfg(ppv_campplus_cfg* cfg);

/* kind PPV_MODEL_RES2NET: ppvector/models/res2net.py:90-167 (Bottle2neck :11-87), ASP head as ResNetSE's; the reference's configs/res2net.yml.
 * scale 2 only (the sp = sp + spx[i] chain of scale > 2 is PPV_EUNSUPPORTED), m_channels 32, every chunk width
 * m_channels * 2^l * base_width / 64 16 or a multiple of 32, and input_size must leave a final grid of input_size / base_width rows
 * (the stem is 7x7 / stride 3 / padding 1 and a 3x3 / 2 max-pool; the reference sizes its head from input_size / base_width). */
#define PPV_MODEL_RES2NET 5
typedef struct {
    int input_size;         /* 80 */
    int embd_dim;           /* 192 */
    int layers[4];          /* 3,4,6,3 */
    int m_channels;         /* 32 */
    int base_width;         /* 32 */
    int scale;              /* 2 */
    int attention_channels; /* 128 */
    int precision;          /* PPV_PREC_* */
} ppv_res2net_cfg;
void ppv_res2net_default_cfg(ppv_res2net_cfg* cfg);
int ppv_model_create(int kind, const void* cfg, ppv_model_t** out);
int ppv_model_destroy(ppv_model_t* h);
/* Weights are COPIED (and re-laid-out for the tensor cores) at finalize; names and shapes are the
 * reference state_dict's (e.g. "blocks.1.tdnn1.conv.conv.weight" [512,512,1], BatchNorm
 * "weight"/"bias"/"_mean"/"_variance").  `data` is fp32, host or device memory. */
int ppv_model_load_weight(ppv_model_t* h, const char* name, const float* data, const int64_t* shape, int ndim);
int ppv_model_finalize(ppv_model_t* h);
int ppv_model_set_precision(ppv_model_t* h, int precision);
int ppv_model_embd_dim(const ppv_model_t* h);
/* Scratch the caller must provide for a batch of B utterances of T frames (256-byte aligned). */
size_t ppv_model_workspace_bytes(const ppv_model_t* h, int B, int T);
/* feat [B,T,input_size] fp32 (AudioFeaturizer output) -> emb [B,embd_dim] fp32. */
int ppv_model_forward(ppv_model_t* h, const float* feat, int B, int T, float* emb, void* ws, size_t ws_bytes,
                      void* stream);
/* ECAPA-TDNN with the reference's optional `lengths` argument (ecapa_tdnn.py:245; relative lengths in (0,1], device fp32 [B]):
 * SEBlock squeezes (ecapa_tdnn.py:71-75) and AttentiveStatisticsPooling pools / masks its softmax (pooling.py:96-115) over the first
 * #{t : t < lengths[b] * T} frames of each utterance.  lengths == NULL is ppv_model_forward. */
int ppv_model_forward_lengths(ppv_model_t* h, const float* feat, const float* lengths, int B, int T, float* emb, void* ws,
                              size_t ws_bytes, void* stream);
/* Fused front end + model: wav [B,L] fp32 -> emb [B,embd_dim]; ECAPA-TDNN and Res2Net.  ECAPA-TDNN: the Fbank features go straight
 * into the first conv's operand layout and never exist as [B,T,F] fp32; Res2Net: they go to the workspace, where its stem reads them.
 * lens_ratio as ppv_fbank_forward. */
int ppv_model_forward_wav(ppv_model_t* h, ppv_fbank_t* fb, const float* wav, const float* lens_ratio, int B, int L,
                          float* emb, void* ws, size_t ws_bytes, void* stream);
/* Debug / parity taps: copy an internal activation (valid frames only) to out as fp32.
 * ECAPA: name in {"feat","blocks.0","blocks.1","blocks.2","blocks.3","mfa","asp"}; out is [B,T,C] ([B,C] for asp).
 * ResNetSE: {"conv1","layer1".."layer4"} -> [B,H,W,C] (H = frequency, W = time); "flat" -> [B,T',C*H]; "asp" -> [B,2*C*H].
 * ERes2Net: {"layer1".."layer4","fuse12","fuse123","fuse1234"} -> [B,H,W,C]; "stats" -> [B, 2*C*H].
 * Res2Net: "stem" (after the max-pool) and "layer1".."layer4" -> [B,H,W,C]; "flat" -> [B,T',C*H]; "asp" -> [B,2*C*H]. */
int ppv_model_read_tap(ppv_model_t* h, const char* name, float* out, size_t out_elems, void* stream);

/* Measurement hooks (bench.py; ECAPA-TDNN and Res2Net): CUDA events around every kernel group of the forward, on the launching stream.
 * profile(h,1) starts recording; profile_read sums the durations since then (tensor-core GEMM launches vs the
 * HBM-bound kernels), reports how many kernels were launched, synchronises on the last event and resets. */
int ppv_model_profile(ppv_model_t* h, int enable);
int ppv_model_profile_read(ppv_model_t* h, double* gemm_ms, double* other_ms, int64_t* gemm_launches,
                           int64_t* other_launches);

/* ---------------------------------------------------------------------------------------------
 * Training step (ECAPA-TDNN).  Replaces the body of PPVectorTrainer.__train_epoch, ppvector/trainer.py:206-229:
 *   outputs = model(features); los = loss(outputs, label); los.backward(); optimizer.step(); optimizer.clear_grad()
 * with the model in TRAIN mode (BatchNorm batch statistics, running statistics updated with momentum 0.9), the classifier
 * ppvector/models/fc.py:41-53 and AAMLoss ppvector/loss/aamloss.py:28-53, Adam ppvector/optimizer/__init__.py:12-18
 * (coupled L2 weight decay).  Parameters / gradients / BatchNorm running statistics are three caller-owned flat fp32 device
 * buffers; ppv_trainer_lookup gives each state_dict tensor's offset ("blocks.1.tdnn1.conv.conv.weight", ...,
 * "classifier.weight" [embd_dim, num_classes]; "*._mean" / "*._variance" live in the statistics buffer).  Data-parallel
 * training is one all-reduce(sum) over the gradient buffer followed by ppv_optimizer_step(grad_scale = 1 / nranks)
 * (the reference's fleet.distributed_model, trainer.py:318-320).
 * ------------------------------------------------------------------------------------------- */
/* Process-wide: 1 (default) = kernels are launched with programmatic dependent launch (the next kernel of a stream starts its prologue while
 * the previous one drains), 0 = plain stream order.  Switch it off while several batches are in flight on different streams (see
 * INTEGRATION.md: lanes): an early-launched dependent CTA occupies a whole SM while it waits.  Returns the previous setting. */
int ppv_set_pdl(int enabled);

typedef struct ppv_trainer ppv_trainer_t;
/* The classifier of ppvector/models/fc.py (model_conf.classifier), Cosine with num_blocks = 0 unless created with
 * ppv_trainer_create_classifier. */
int ppv_trainer_create(const ppv_ecapa_cfg* cfg, int num_classes, ppv_trainer_t** out);
/* classifier_type: the output layer, fc.py:30-40 -- PPV_CLASSIFIER_COSINE ("classifier.weight" [in, num_classes], cosine logits) or
 * PPV_CLASSIFIER_LINEAR ("classifier.output.weight" [in, num_classes] and "classifier.output.bias" [num_classes], logits = h W + b).
 * num_blocks DenseLayers sit between the embedding and the output layer (fc.py:27-29), each Conv1D(in, inter_dim, 1) with bias then
 * BatchNorm1D(inter_dim), no ReLU, batch statistics in training: "classifier.blocks.<i>.linear.{weight [inter_dim, in, 1], bias}",
 * "classifier.blocks.<i>.nonlinear.batchnorm.{weight, bias, _mean, _variance}"; `in` is embd_dim for block 0 and inter_dim after it.
 * A Linear classifier runs with the loss heads defined for any real logits: PPV_HEAD_AM, PPV_HEAD_ARM, PPV_HEAD_CE and SphereFace2
 * type C; ppv_trainer_forward_backward refuses the others.  Taps "classifier.blocks.<i>" and "g:classifier.blocks.<i>" read a block's
 * output and its gradient, [B, inter_dim]. */
#define PPV_CLASSIFIER_COSINE 0
#define PPV_CLASSIFIER_LINEAR 1
int ppv_trainer_create_classifier(const ppv_ecapa_cfg* cfg, int num_classes, int classifier_type, int num_blocks, int inter_dim,
                                  ppv_trainer_t** out);
int ppv_trainer_destroy(ppv_trainer_t* h);
int64_t ppv_trainer_param_count(const ppv_trainer_t* h); /* floats in the parameter / gradient buffers (tensors are 32-byte aligned) */
int64_t ppv_trainer_stat_count(const ppv_trainer_t* h);  /* floats in the running-statistics buffer */
int ppv_trainer_lookup(const ppv_trainer_t* h, const char* name, int64_t* offset, int64_t* numel, int* is_stat);
int ppv_trainer_bind(ppv_trainer_t* h, float* params, float* grads, float* stats);
/* Operand precision of the step's GEMMs (forward, data gradients, weight gradients): PPV_PREC_BF16X3 (default, fp32-grade) or
 * PPV_PREC_BF16 -- the single-pass bf16 form of train_conf.enable_amp (ppvector/trainer.py:167, 209-229: paddle.amp.auto_cast level O1 + GradScaler
 * around the same step): single-pass bf16 operands, fp32 accumulation, fp32 BatchNorm / pooling / loss / master weights / Adam; bf16
 * keeps fp32's exponent range, so there is no loss scaling. */
int ppv_trainer_set_precision(ppv_trainer_t* h, int precision);
size_t ppv_trainer_workspace_bytes(ppv_trainer_t* h, int B, int T);
/* feat [B,T,F] fp32, labels [B] int64 (device).  Overwrites the whole gradient buffer with d(loss)/d(param), updates the
 * running statistics, writes the scalar loss and (optionally) the classifier's logits [B, num_classes] (device pointers). */
int ppv_trainer_forward_backward(ppv_trainer_t* h, const float* feat, const int64_t* labels, int B, int T, float margin, float scale,
                                 int easy_margin, float label_smoothing, float* loss, float* logits, void* ws, size_t ws_bytes, void* stream);
/* forward activations of the last step: "blocks.0".."blocks.3", "mfa" -> [B,T,C]; "asp" -> [B, 2*3C]; "emb" -> [B, embd_dim];
 * "classifier.blocks.<i>" -> [B, inter_dim] */
int ppv_trainer_read_tap(ppv_trainer_t* h, const char* name, float* out, size_t out_elems, void* stream);
/* p -= lr * mhat / (sqrt(vhat) + eps) with g = grads * grad_scale + weight_decay * p; step counts from 1. */
int ppv_adam_step(float* params, const float* grads, float* m, float* v, int64_t n, float lr, float beta1, float beta2, float eps,
                  float weight_decay, int64_t step, float grad_scale, void* stream);

/* The optimizers ppvector/optimizer/__init__.py:12-18 builds by name (paddle.optimizer.<optimizer>(**optimizer_args)), as one fused
 * elementwise step over the flat buffers.  g = grads * grad_scale; weight_decay is coupled L2 except for AdamW:
 *   PPV_OPT_ADAM      the kernel of ppv_adam_step (bitwise the same); state0 = m, state1 = v
 *   PPV_OPT_ADAMW     p *= 1 - lr wd, then the Adam update of ppv_adam_step on the undecayed g; state0 = m, state1 = v
 *   PPV_OPT_SGD       p -= lr (g + wd p); no state
 *   PPV_OPT_MOMENTUM  g' = g rescale_grad + wd p, v = momentum v + g', p -= lr v (use_nesterov: p -= lr (g' + momentum v)); state0 = v
 *   PPV_OPT_RMSPROP   g' = g + wd p, ms = rho ms + (1 - rho) g'^2, centered: mg = rho mg + (1 - rho) g';
 *                     mom = momentum mom + lr g' / sqrt(ms [- mg^2] + epsilon), p -= mom; state0 = ms, state1 = mom, state2 = mg (centered)
 * ppv_optimizer_state_count(kind, centered) is the number of state buffers (n floats each, zero before the first step) the kind reads:
 * state buffers beyond it may be NULL; negative for an unknown kind.  step counts from 1 (used by ADAM / ADAMW only).  Buffers whose
 * addresses are all 16-byte aligned are read and written as float4. */
#define PPV_OPT_ADAM 0
#define PPV_OPT_ADAMW 1
#define PPV_OPT_SGD 2
#define PPV_OPT_MOMENTUM 3
#define PPV_OPT_RMSPROP 4
typedef struct ppv_optim_args {
    float lr;
    float weight_decay;
    float beta1, beta2, epsilon; /* ADAM / ADAMW: epsilon also for RMSPROP */
    float momentum;              /* MOMENTUM / RMSPROP */
    float rho;                   /* RMSPROP */
    float rescale_grad;          /* MOMENTUM */
    int use_nesterov;            /* MOMENTUM */
    int centered;                /* RMSPROP */
} ppv_optim_args;
int ppv_optimizer_state_count(int kind, int centered);
int ppv_optimizer_step(int kind, float* params, const float* grads, float* state0, float* state1, float* state2, int64_t n,
                       const ppv_optim_args* args, int64_t step, float grad_scale, void* stream);

/* ---------------------------------------------------------------------------------------------
 * Cosine scoring.  Replaces ppvector/predict.py:279-283 (contrast), :173-187 (retrieval:
 * sklearn cosine_similarity) and ppvector/trainer.py:416-423 (eval trial x enrol matrix).
 * ------------------------------------------------------------------------------------------- */
/* A [M,D], Bm [N,D] -> out [M,N], out[i,j] = <A_i,B_j> / (|A_i||B_j|).  ws: scratch of
 * ppv_cosine_workspace_bytes(M,N,D) bytes, 256-byte aligned. */
size_t ppv_cosine_workspace_bytes(int M, int N, int D);
int ppv_cosine_matrix(const float* A, const float* Bm, int M, int N, int D, float* out, void* ws, size_t ws_bytes,
                      void* stream);
/* E [n,D], idx [P,2] int32 -> out [P]. */
int ppv_cosine_pairlist(const float* E, const int32_t* idx, int64_t P, int n, int D, float* out, void* stream);

/* ---------------------------------------------------------------------------------------------
 * Batched waveform preparation / augmentation in front of the feature extractor.  Replaces the per-utterance CPU work of
 * ppvector/data_utils/reader.py:85-104, :153-163 (yeaudio: change_speed, gain_db, add noise at an SNR, normalize(target_db), crop)
 * with one launch sequence per batch; the random draws stay on the host (configs/augmentation.yml).
 * Per utterance b: iparams[b] = {raw_len, new_len (= int(raw_len / speed), or raw_len), crop_start, crop_len, noise_off, noise_len,
 * has_noise, 0}; fparams[b] = {reserved, volume gain dB, SNR dB, 0}.  wav [B][wav_ld] fp32, noise = concatenated noise clips (tiled
 * over the utterance from noise_off), out [B][Lout] fp32 zero-padded.  normalize != 0: dB-normalise to target_db over the whole
 * augmented utterance before the crop.
 * ------------------------------------------------------------------------------------------- */
#define PPV_PREP_NI 8
#define PPV_PREP_NF 4
size_t ppv_audio_prep_workspace_bytes(int B, int max_new_len);
int ppv_audio_prep(const float* wav, int64_t wav_ld, const int32_t* iparams, const float* fparams, const float* noise, int B,
                   int max_new_len, float target_db, int normalize, int Lout, float* out, void* ws, size_t ws_bytes, void* stream);
/* The same with reverberation (yeaudio ReverbPerturbAugmentor: full convolution with a room impulse response, not truncated, the
 * response not normalised) after the noise and before the dB normalisation.  rir_bank = concatenated responses (rir_bank_len samples,
 * device); rparams [B][2] int32 (device) = {rir_off, rir_len}, rir_len 0 = no reverb for that item, otherwise 1 <= rir_len <= max_rir_len
 * and rir_off + rir_len <= rir_bank_len.  For an item with a response, crop_start / crop_len in iparams are on its reverberant length
 * new_len + rir_len - 1.  Items without one come out exactly as from ppv_audio_prep.  rparams live on the device, so a violating entry
 * cannot be reported here: the kernels read nothing for it and write NaN over that item's output row.  ws: scratch of
 * ppv_audio_prep_reverb_workspace_bytes(B, max_new_len, max_rir_len) bytes, 256-byte aligned (~2 KB per 256 samples of every
 * utterance and response). */
size_t ppv_audio_prep_reverb_workspace_bytes(int B, int max_new_len, int max_rir_len);
int ppv_audio_prep_reverb(const float* wav, int64_t wav_ld, const int32_t* iparams, const float* fparams, const float* noise,
                          const float* rir_bank, int64_t rir_bank_len, const int32_t* rparams, int B, int max_new_len, int max_rir_len,
                          float target_db, int normalize, int Lout, float* out, void* ws, size_t ws_bytes, void* stream);

/* ---------------------------------------------------------------------------------------------
 * Verification metrics and enrol-DB retrieval on the device.  Replaces ppvector/metric/metrics.py:4-37
 * (compute_fnr_fpr / compute_eer / compute_dcf, called by ppvector/trainer.py:424-431) and the arg-max of
 * ppvector/predict.py:173-187 (__retrieval).
 * ------------------------------------------------------------------------------------------- */
size_t ppv_eer_workspace_bytes(int64_t n);
/* scores [n] fp32, labels [n] int32 (1 = target trial) -> out4 (device double[4]) = {EER, threshold at the EER, minDCF, number of targets}.
 * ws: ppv_eer_workspace_bytes(n) bytes, 256-byte aligned (both forms). */
int ppv_eer_mindcf(const float* scores, const int32_t* labels, int64_t n, double p_target, double c_miss, double c_fa, double* out4,
                   void* ws, size_t ws_bytes, void* stream);
/* The evaluation loop's form (trainer.py:416-423): scores [M,N] of trials x enrolments, label = (trial_labels[i] == enroll_labels[j]). */
int ppv_eer_mindcf_matrix(const float* scores, const int32_t* trial_labels, const int32_t* enroll_labels, int M, int N, double p_target,
                          double c_miss, double c_fa, double* out4, void* ws, size_t ws_bytes, void* stream);
/* sim [rows, cols] fp32 -> idx [rows] (first maximum, like numpy.argmax), best [rows]. */
int ppv_row_argmax(const float* sim, int rows, int cols, int32_t* idx, float* best, void* stream);

/* ---------------------------------------------------------------------------------------------
 * Speaker index: the enrolment database's per-user mean embeddings, searched by cosine top-k.  Replaces the per-user mean loop of
 * ppvector/predict.py:154-163 (__load_audio_db; register :311-320 and remove_user :360-362 update the same means) and the
 * retrieval of :173-187 (__retrieval: sklearn cosine_similarity of the normalised queries against the means, then numpy.argmax).
 * The index is an opaque device buffer of ppv_speaker_index_bytes(U, D) bytes, 256-byte aligned, written by
 * ppv_speaker_index_build and read by ppv_speaker_index_search; its layout belongs to the library.  Limits: 1 <= D <= 256,
 * U >= 1, Q >= 1, 1 <= k <= min(8, U); anything else is PPV_EINVAL.
 * ------------------------------------------------------------------------------------------- */
/* Bytes of the index of U users of dimension D (0 when out of range). */
size_t ppv_speaker_index_bytes(int U, int D);
/* E [n, D] fp32 enrolment embeddings; order [n] int32 = row indices grouped by user (enrolment order within a user), offsets [U+1]
 * int32 (user u owns order[offsets[u] .. offsets[u+1]), every user at least one row) -> means [U, D] fp32, each the fp32 sum of the
 * user's rows in that order divided by the count (bitwise numpy's E[rows].mean(axis=0)), and the index.  Deterministic; one launch. */
int ppv_speaker_index_build(const float* E, int n, int D, const int32_t* order, const int32_t* offsets, int U, float* means, void* index,
                            size_t index_bytes, void* stream);
/* Scratch of ppv_speaker_index_search, 256-byte aligned: O(Q * k * splits), never O(Q * U). */
size_t ppv_speaker_index_search_workspace_bytes(int Q, int U, int D, int k);
/* queries [Q, D] fp32 -> idx [Q, k] int32, sim [Q, k] fp32: per query the k users of highest cosine similarity, descending, equal
 * similarities lowest index first (k = 1: numpy.argmax's first maximum).  A zero-norm query or mean scores 0.  Deterministic. */
int ppv_speaker_index_search(const float* queries, int Q, int D, const void* index, size_t index_bytes, int U, int k, int32_t* idx,
                             float* sim, void* ws, size_t ws_bytes, void* stream);

/* ---------------------------------------------------------------------------------------------
 * Adaptive score normalisation (AS-norm) against a cohort; no counterpart in the reference.  For a query row q (a trial or an
 * enrolment) scored against the cohort, S_q is the multiset of its top_n largest scores (ties by value only: equal scores at the cut
 * count with multiplicity), mean_q = mean(S_q) and std_q = sqrt(sum((x - mean_q)^2) / (top_n - 1)) floored at 1e-6; then
 * s'(t, e) = 0.5 * ((s - mean_e) / std_e + (s - mean_t) / std_t).  Scores must be finite.
 * ------------------------------------------------------------------------------------------- */
/* scores [rows, cols] fp32, row r at scores + r * ld -> mean [rows], std [rows] fp32 of each row's top_n largest values.  Exact
 * selection; fp64 sums about the top_n-th value.  Bitwise reproducible and independent of how rows are batched.  Rows of up to 10240
 * columns are read from HBM once, wider rows four times.  PPV_EINVAL unless rows, cols >= 1, ld >= cols, 2 <= top_n <= cols. */
int ppv_topn_row_stats(const float* scores, int rows, int cols, int64_t ld, int top_n, float* mean, float* std, void* stream);
/* In place on scores [M, N] fp32 (row-major, ld = N) of trials x enrolments: s' from the trial statistics [M] and the enrolment
 * statistics [N] (std floored at 1e-6 again).  One pass. */
int ppv_as_norm_apply(float* scores, int M, int N, const float* trial_mean, const float* trial_std, const float* enroll_mean,
                      const float* enroll_std, void* stream);

/* ---------------------------------------------------------------------------------------------
 * Energy voice-activity detection: Kaldi's compute-vad (src/ivector/voice-activity-detection.cc, ComputeVadEnergy) on the raw log
 * energy of each snip_edges frame, in front of speaker diarization.  The reference runs silero-vad there (a neural network whose
 * weights ship inside yeaudio); this is the classical energy VAD of Kaldi's x-vector recipes instead.  Per recording of L samples:
 * T = 0 if L < window else 1 + (L - window) / shift frames;
 * e_t = ln(max(32768^2 * sum_{n < window} (x[t * shift + n] - mean_t)^2, FLT_EPSILON)) (mean_t the frame's own mean; fp64 sums; no
 * dither, pre-emphasis or window function); thr = energy_threshold + energy_mean_scale * (sum_t e_t) / T (fp64); frame t is voiced iff
 * num >= den * proportion_threshold (product in fp32), where den counts the frames in [t - frames_context, t + frames_context] ∩ [0, T)
 * and num those of them with e_t2 > thr.
 * ------------------------------------------------------------------------------------------- */
typedef struct {
    int window;                 /* samples per frame: sample_rate * 25 / 1000 (400 at 16 kHz); 1..2048 */
    int shift;                  /* samples between frames: sample_rate * 10 / 1000 (160 at 16 kHz); 1..window */
    float energy_threshold;     /* 5.5 */
    float energy_mean_scale;    /* 0.5; >= 0 */
    int frames_context;         /* 2; >= 0 */
    float proportion_threshold; /* 0.12; in (0, 1) */
} ppv_vad_cfg;
/* The defaults of Kaldi's VoxCeleb / SRE16 x-vector recipes (conf/vad.conf) with 25 ms / 10 ms frames at sample_rate. */
void ppv_vad_default_cfg(ppv_vad_cfg* cfg, int sample_rate);
/* T for a recording of L samples; -1 for a configuration out of range or L < 0. */
int64_t ppv_vad_num_frames(const ppv_vad_cfg* cfg, int64_t L);
/* Workspace for R recordings of total_samples samples in all (the last sample offset); 0 for arguments out of range. */
size_t ppv_vad_workspace_bytes(const ppv_vad_cfg* cfg, int R, int64_t total_samples);
/* R recordings, recording r at wav[sample_offsets[r] .. sample_offsets[r + 1]) (fp32, device; sample_offsets is a HOST array of R + 1
 * non-decreasing values).  Frame outputs are concatenated in recording order (recording r's frames start at the sum of the earlier
 * recordings' T): voiced [sum T] uint8 (0 / 1) and, if log_energy != NULL, e_t [sum T] fp64.  runs [run_cap, 3] int32 receives the
 * maximal runs of voiced frames as (recording, first_frame, end_frame) in recording and frame order, frame indices within the
 * recording; *n_runs (device int32) their count.  run_cap >= sum_r ceil(T_r / 2) (the alternating worst case).  A recording with
 * T = 0 yields no run.  ws: ppv_vad_workspace_bytes(cfg, R, sample_offsets[R]) bytes, 256-byte aligned.  Bitwise reproducible and
 * independent of how recordings are batched.  PPV_EINVAL for null pointers, R < 1, decreasing offsets, too small a workspace or run
 * capacity, and configurations out of range. */
int ppv_vad_energy(const ppv_vad_cfg* cfg, const float* wav, const int64_t* sample_offsets, int R, double* log_energy, uint8_t* voiced,
                   int32_t* runs, int64_t run_cap, int32_t* n_runs, void* ws, size_t ws_bytes, void* stream);

/* ---------------------------------------------------------------------------------------------
 * Speaker diarization: spectral clustering of the chunk embeddings.  Replaces
 * ppvector/infer_utils/speaker_diarization.py:219-310 (SpectralCluster: pruning, Laplacian, scipy.linalg.eigh,
 * sklearn k_means).  The affinity is ppv_cosine_matrix of the [N, D] embeddings.  One stage per entry point, so that each
 * can be fed the previous stage's stored output.  All arithmetic after the affinity is fp64 and every sum runs in a fixed
 * order: results are bitwise reproducible.  N (windows) must be 1 <= N <= 8192, else PPV_EINVAL.
 * ------------------------------------------------------------------------------------------- */
/* In place on affinity [N,N] fp32: pval' = 6/N if N*pval < 6 else pval; each row zeroes its int((1-pval')*N) smallest entries
 * (exact ties: the lower column index first). */
int ppv_cluster_prune(float* affinity, int N, double pval, void* stream);
/* pruned [N,N] fp32 -> L [N,N] fp64 = diag(D) - M, M = (P + P^T)/2 with a zero diagonal, D_i = sum_j |M_ij|. */
int ppv_cluster_laplacian(const float* pruned, int N, double* L, void* stream);
/* The m (1 <= m <= min(N, 32)) smallest eigenvalues of the symmetric L [N,N] fp64 (overwritten), ascending -> evals [m], and
 * their eigenvectors -> evecs [N,m] (row-major).  ws: ppv_sym_eig_workspace_bytes(N, m) bytes, 256-byte aligned. */
size_t ppv_sym_eig_workspace_bytes(int N, int m);
int ppv_sym_eig_smallest(double* L, int N, int m, double* evals, double* evecs, void* ws, size_t ws_bytes, void* stream);
/* sklearn k_means(X, k, n_init="auto") of the rows of X [N, >= k] fp64 (row stride ld) -> labels [N] int32, inertia (device
 * double).  k-means++ consumes uniforms [1 + (k-1)(2 + int(log k))] fp64 in [0, 1) in numpy's draw order; 1 <= k <= min(N, 32).
 * ws: ppv_kmeans_workspace_bytes(N, k) bytes, 256-byte aligned. */
size_t ppv_kmeans_workspace_bytes(int N, int k);
int ppv_kmeans(const double* X, int ld, int N, int k, const double* uniforms, int n_uniforms, int max_iter, int32_t* labels, double* inertia,
               void* ws, size_t ws_bytes, void* stream);

/* ---------------------------------------------------------------------------------------------
 * Cosine classifier + AAMLoss.  Replaces ppvector/models/fc.py:41-53 (Cosine, num_blocks=0) and
 * ppvector/loss/aamloss.py:28-46 (mean softmax-CE over scale * margin-adjusted cosines).
 * W is [D,S] (Paddle layout, fc.py:31).  logits [B,S] receives the plain cosines
 * (outputs['logits'] of the reference); loss is a device scalar.
 * The `easy_margin` argument selects the loss head: 0 = AAMLoss, 1 = AAMLoss(easy_margin=True), PPV_HEAD_AM = AMLoss
 * (ppvector/loss/amloss.py:18-24), PPV_HEAD_ARM = ARMLoss (armloss.py:18-31), PPV_HEAD_CE = CELoss (celoss.py:16-18: raw logits,
 * `scale` ignored); label smoothing and the mean over the batch are common to all of them.
 * ------------------------------------------------------------------------------------------- */
#define PPV_HEAD_AAM 0
#define PPV_HEAD_AAM_EASY 1
#define PPV_HEAD_AM 2
#define PPV_HEAD_ARM 3
#define PPV_HEAD_CE 4
/* SubCenterLoss (ppvector/loss/subcenterloss.py:33-54) with K sub-centres per class: pass PPV_HEAD_SUBCENTER | (K << 5) [| 1 for easy_margin];
 * W / logits then have num_classes * K columns (fc.py:33: class c owns columns c*K .. c*K+K-1), a class's cosine is the max over its K. */
#define PPV_HEAD_SUBCENTER 16
/* SphereFace2 (ppvector/loss/sphereface2.py:44-70), a per-entry binary logistic loss, not a softmax: pass PPV_HEAD_SPHEREFACE2 | (t << 5)
 * [| 1 for margin_type 'A'; default 'C'], the `label_smoothing` argument carries lanbuda (the positive / negative weight); the loss's
 * bias stays at its initial 0 as in the reference (it is not among the optimizer's parameters). */
#define PPV_HEAD_SPHEREFACE2 8
/* ws: ppv_aam_workspace_bytes(B, D, S) bytes, 256-byte aligned. */
int ppv_aam_forward(const float* emb, const float* W, const int64_t* labels, int B, int D, int S, float margin,
                    float scale, int easy_margin, float label_smoothing, float* logits, float* loss,
                    void* ws, size_t ws_bytes, void* stream);
size_t ppv_aam_workspace_bytes(int B, int D, int S);
/* Gradients of the mean loss w.r.t. emb [B,D] and W [D,S]; uses logits from ppv_aam_forward and its ws. */
int ppv_aam_backward(const float* emb, const float* W, const int64_t* labels, const float* logits, int B, int D,
                     int S, float margin, float scale, int easy_margin, float label_smoothing, float* d_emb,
                     float* d_W, void* ws, size_t ws_bytes, void* stream);
/* Linear classifier + loss head (ppvector/models/fc.py:37-38, 50-51: logits = H @ W + b, no normalisation; H [B,D], W [D,S], b [S]),
 * the output layer of the ECAPA-TDNN trainer's Linear classifier.  The same loss heads run on the raw logits; only those defined for
 * any real logit are accepted: PPV_HEAD_CE, PPV_HEAD_AM, PPV_HEAD_ARM and PPV_HEAD_SPHEREFACE2 type C (the cosine-only heads return
 * PPV_EUNSUPPORTED).  D <= 1536.  logits [B,S] receives H @ W + b; loss is a device scalar.
 * ws: ppv_aam_workspace_bytes(B, D, S) bytes, 256-byte aligned. */
int ppv_linear_head_forward(const float* H, const float* W, const float* bias, const int64_t* labels, int B, int D, int S, float margin,
                            float scale, int easy_margin, float label_smoothing, float* logits, float* loss, void* ws, size_t ws_bytes,
                            void* stream);
/* Gradients of the mean loss w.r.t. H [B,D], W [D,S] and b [S]; uses logits from ppv_linear_head_forward. */
int ppv_linear_head_backward(const float* H, const float* W, const int64_t* labels, const float* logits, int B, int D, int S, float margin,
                             float scale, int easy_margin, float label_smoothing, float* d_H, float* d_W, float* d_bias, void* ws,
                             size_t ws_bytes, void* stream);

/* ---------------------------------------------------------------------------------------------
 * Test hook for the tensor-core GEMM (not a reference entry point): out[M,N] = A[M,K] * W[N,K]^T
 * (+bias, ReLU, BN affine as flagged) through the same wgmma/TMA kernel the model uses.
 * A, W, out fp32 device; ws >= ppv_gemm_test_workspace_bytes.  block_n in {64,128,256}; block_k in {64,32}
 * (K elements per pipeline stage: SWIZZLE_128B / SWIZZLE_64B tiles).
 * ------------------------------------------------------------------------------------------- */
size_t ppv_gemm_test_workspace_bytes(int M, int N, int K);
int ppv_gemm_test(const float* A, const float* W, const float* bias, const float* bn_scale, const float* bn_shift,
                  int relu, int M, int N, int K, int block_n, int block_k, int precision, float* out, void* ws,
                  size_t ws_bytes, void* stream);

/* The same with split-bf16 planes output out[2][M][N] (bf16, N % 32 == 0, 16-byte aligned) and the epilogue of the ECAPA layers:
 * + bias, + rowgrp_bias[row / Tp] (may be NULL), ReLU (relu), BN affine (may be NULL), tanh (tanh_).  Tp > 0: padded time layout
 * (Tp = T + 2 P, M % Tp == 0), only the T valid rows of each group are written.  block_k is 64. */
int ppv_gemm_test_planes(const float* A, const float* W, const float* bias, const float* rowgrp_bias, const float* bn_scale,
                         const float* bn_shift, int relu, int tanh_, int Tp, int P, int M, int N, int K, int block_n,
                         int precision, void* out, void* ws, size_t ws_bytes, void* stream);

/* Test hook for the conv2d kernels of ResNetSE, ERes2Net and CAM++ (not a reference entry point): one k x k conv (k 1 or 3, padding
 * k / 2, stride (stride_h, stride_w)) of x [B,H,W,Cin] (fp32 NHWC) with w [Cout,Cin,k,k] (fp32), + bias (may be NULL), ReLU (relu).
 * x is written as split planes at columns [x_col0, x_col0 + Cin) of a zero-bordered [B, H+2, W+2, x_ld] grid (x_ld 0: Cin); the
 * other columns hold a non-zero fill.  path 0: the 3x3 patch kernel (32 -> 32 channels); 1: the pointwise kernel (1x1, Cin 32,
 * Cout 32 or 64; it computes in fp32 over the exact hi + lo values at either precision); 2: the gather-GEMM in image mode (k x k
 * row-offset taps).  A conv the chosen kernel does not take is an error.  out: split-bf16 planes [2][B][Ho+2][Wo+2][Cout] with
 * Ho = (H-1)/stride_h + 1, Wo = (W-1)/stride_w + 1, 16-byte aligned; it is zeroed, then the kernel writes the interior positions.
 * ws >= ppv_conv2d_test_workspace_bytes.  Synchronises `stream` while it prepares the weights. */
size_t ppv_conv2d_test_workspace_bytes(int B, int H, int W, int Cin, int Cout, int k, int x_ld);
int ppv_conv2d_test(const float* x, const float* w, const float* bias, int relu, int B, int H, int W, int Cin, int Cout, int k,
                    int stride_h, int stride_w, int x_col0, int x_ld, int path, int precision, void* out, void* ws,
                    size_t ws_bytes, void* stream);
/* Test hook (not a reference entry point): the same conv with the ReLU clipped at relu_max > 0 (ERes2Net's Hardtanh(0, 20)), as the
 * ERes2Net plans ask the kernels for it.  Same workspace as ppv_conv2d_test. */
int ppv_conv2d_test_clipped(const float* x, const float* w, const float* bias, float relu_max, int B, int H, int W, int Cin, int Cout,
                            int k, int stride_h, int stride_w, int x_col0, int x_ld, int path, int precision, void* out, void* ws,
                            size_t ws_bytes, void* stream);

/* Test hooks for the 2-D models' stem conv and two elementwise kernels (not reference entry points).
 * stem: feat [B,T,F] fp32, w [C0][9] and bias [C0] fp32 with the BN folded in -> out: split-bf16 planes [2][B][F+2][T+2][C0] (the image
 * is the features transposed: frequency rows, frame columns), 16-byte aligned; zeroed, then the kernel writes the interior (3x3 conv,
 * padding 1, ReLU).  C0 a multiple of 8 up to 2048.
 * scale_res: out[r, oc0 + c] = z[r, c] * scale[r / rows_per_group, c] + res[r, rc0 + c] for the rows r < rows, then ReLU if relu, clipped
 * at relu_max when relu_max > 0.  z [rows, C], res [rows, res_ld] fp32, split into planes here; scale [rows / rows_per_group, C] fp32
 * (may be NULL: no scale).  out: split-bf16 planes [2][rows][out_ld], 16-byte aligned, not cleared: only columns [oc0, oc0 + C) are
 * written.  C, rc0, oc0, res_ld, out_ld multiples of 8; ws >= ppv_scale_res_test_workspace_bytes.
 * aff_combine: out[r, c] = x[r, xc0 + c] (1 + t[r, c]) + y[r, yc0 + c] (1 - t[r, c]).  x [rows, x_ld], y [rows, y_ld], t [rows, C] fp32,
 * split into planes here.  out: split-bf16 planes [2][rows][C], 16-byte aligned.  C, xc0, yc0, x_ld, y_ld multiples of 8;
 * ws >= ppv_aff_combine_test_workspace_bytes. */
int ppv_stem_conv_test(const float* feat, const float* w, const float* bias, int B, int T, int F, int C0, void* out, void* stream);
size_t ppv_scale_res_test_workspace_bytes(int rows, int C, int res_ld);
int ppv_scale_res_test(const float* z, const float* scale, const float* res, int res_ld, int rc0, int C, int rows_per_group, int rows,
                       int relu, float relu_max, void* out, int out_ld, int oc0, void* ws, size_t ws_bytes, void* stream);
size_t ppv_aff_combine_test_workspace_bytes(int rows, int C, int x_ld, int y_ld);
int ppv_aff_combine_test(const float* x, int x_ld, int xc0, const float* y, int y_ld, int yc0, const float* t, int C, int rows, void* out,
                         void* ws, size_t ws_bytes, void* stream);

/* Test hooks for Res2Net's CUDA-core kernels (not reference entry points).
 * stem: feat [B,T,F] fp32, w [32][49] and bias [32] fp32 with the BN folded in -> out: split-bf16 planes [2][B][Hq+2][Wq+2][32],
 * H1 = (F-5)/3+1, W1 = (T-5)/3+1, Hq = (H1-1)/2+1, Wq = (W1-1)/2+1, 16-byte aligned; zeroed, then the kernel writes the interior
 * (7x7 / 3 conv, ReLU, 3x3 / 2 max-pool).  F, T >= 5.
 * avgpool: x fp32 [B][H+2][W+2][C] (a zero-bordered grid) -> out: split-bf16 planes [2][B][Ho+2][Wo+2][C], Ho = (H-1)/stride+1,
 * Wo = (W-1)/stride+1; zeroed, then columns [col0, col0+ncols) of the interior get the exclusive 3x3 average (stride 1 or 2, padding 1)
 * of the same columns of x.  col0, ncols, C multiples of 8; ws >= ppv_res2net_avgpool_test_workspace_bytes. */
int ppv_res2net_stem_test(const float* feat, const float* w, const float* bias, int B, int T, int F, void* out, void* stream);
size_t ppv_res2net_avgpool_test_workspace_bytes(int B, int H, int W, int C);
int ppv_res2net_avgpool_test(const float* x, int B, int H, int W, int C, int col0, int ncols, int stride, void* out, void* ws,
                             size_t ws_bytes, void* stream);

/* Test hook for the fused attentive-statistics pooling kernel (not a reference entry point): the kernel the ECAPA-TDNN and ResNetSE
 * plans run, on operands given in fp32 and split into planes here.  W [C,K] (attention conv weight), att [B*Tp,K] and x [B*Tp,C] in
 * the padded time layout (row b*Tp + P + t), bn_scale / bn_shift [2C], nvalid [B] int32 (may be NULL: T valid frames).
 * C % 128 == 0, K in {64, 128}.  max_ctas: the grid's CTA count cap (0: every SM).  The 64 plane rows behind att and x hold a large finite value.  out_raw [B,2C] fp32 (mean | std), out [B,2C]: the asp_bn'd split
 * planes decoded as hi + lo.  ws >= ppv_asp_fused_test_workspace_bytes. */
size_t ppv_asp_fused_test_workspace_bytes(int B, int Tp, int C, int K);
int ppv_asp_fused_test(const float* W, const float* att, const float* x, const float* bn_scale, const float* bn_shift,
                       const int* nvalid, int B, int T, int P, int Tp, int C, int K, int precision, int max_ctas,
                       float* out_raw, float* out, void* ws, size_t ws_bytes, void* stream);

/* Test hook for the column-statistics kernel (not a reference entry point): launch_colstats, as the model plans call it, over x
 * [B*Tp, ld] fp32 split into planes here (rows b*Tp + P + t, t < T, of columns [col0, col0 + C); C % 64 == 0, col0 % 8 == 0,
 * ld % 8 == 0).  mode 0: mean; 1: mean | sqrt(max(var, eps)); 2: mean | sqrt(var_unbiased + eps); 3: mean | var_unbiased.
 * inv_count > 0: mean = sum * inv_count.  nvalid [B] int32 (may be NULL): frames pooled per utterance, clamped to [1, T].
 * out [B, C] (mode 0) or [B, 2C]: the output planes decoded as hi + lo; out_f32 [B, C] (mode 0 only, may be NULL otherwise).
 * ws >= ppv_colstats_test_workspace_bytes. */
size_t ppv_colstats_test_workspace_bytes(int B, int Tp, int ld, int C);
int ppv_colstats_test(const float* x, int B, int T, int P, int Tp, int ld, int col0, int C, int mode, float eps, float inv_count,
                      const int* nvalid, float* out, float* out_f32, void* ws, size_t ws_bytes, void* stream);

/* Test hook for the training step's TAP / TSP pooling backward (not a reference entry point): the kernel the ECAPA-TDNN trainer runs,
 * over x [B*Tp, C] fp32 split into planes here (frames t < T at rows b*Tp + P + t; C % 8 == 0).  pooled and dpooled are fp32
 * [B, C] (var == 0: TAP's mean) or [B, 2C] (var != 0: TSP's mean | unbiased variance) and their gradients.  dx [B*Tp, C]: every row
 * of the output planes decoded as hi + lo; the planes are filled with the bytes 0x46 before the launch, so a row the kernel does not
 * write (halo, padding) reads back as 2 * bf16(0x4646).  ws >= ppv_pool_stats_bwd_test_workspace_bytes (0 for an empty shape). */
size_t ppv_pool_stats_bwd_test_workspace_bytes(int B, int Tp, int C);
int ppv_pool_stats_bwd_test(const float* x, const float* pooled, const float* dpooled, int B, int T, int P, int Tp, int C, int var, float* dx,
                            void* ws, size_t ws_bytes, void* stream);

/* Test hook for CAM++'s context mask (not a reference entry point): the dense layers' context kernel over h [B*Tp, 128] fp32 split
 * into planes here (frames t < T at rows b*Tp + P + t), with the MLP w1 [64,128], b1 [64], w2 [32,64], b2 [32] in the reference
 * layout, transposed on the host as the model prepares them.  out [B * ceil(T/100), 32] fp32.  T > 6400 (more than 64 segments)
 * is an error.  ws >= ppv_campplus_context_test_workspace_bytes.  Synchronises `stream` while it prepares the weights. */
size_t ppv_campplus_context_test_workspace_bytes(int B, int Tp);
int ppv_campplus_context_test(const float* h, int B, int T, int P, int Tp, const float* w1, const float* b1, const float* w2,
                              const float* b2, float* out, void* ws, size_t ws_bytes, void* stream);

/* Test hook for the gather-GEMM on the padded time layout (not a reference entry point): one case as a model plans it.
 * x[i] [rows[i], ld[i]] fp32 (every row given, padding rows included) are split into planes here; source j reads columns
 * [src_col0[j], src_col0[j] + src_ncols[j]) of x[src_input[j]] at row offset src_row_off[j].  W [N, sum ncols] fp32 in k-step order.
 * Epilogue: + bias, * seg_scale[(b * nseg + t / seg_len) * N + n] (may be NULL), ReLU, BN affine (may be NULL) on the T valid rows of
 * every Tp = T + 2P (Tp 0: every row valid); halo: also the reflect mirror rows; zero_invalid: zeros on the other rows.  out_f32 0:
 * planes out [2][out_rows][out_ld] bf16, 1: fp32 out [out_rows][out_ld], written from column out_col0; the hook does not clear it.
 * block_n 0: the plans' choice; block_k 0: gemm_build's.  ws >= ppv_gemm_test_taps_workspace_bytes. */
#define PPV_TAPS_MAX_INPUTS 4
#define PPV_TAPS_MAX_SOURCES 16
typedef struct {
    const float* x[PPV_TAPS_MAX_INPUTS];
    int64_t rows[PPV_TAPS_MAX_INPUTS];
    int ld[PPV_TAPS_MAX_INPUTS];
    int ninputs, nsrc;
    int src_input[PPV_TAPS_MAX_SOURCES], src_col0[PPV_TAPS_MAX_SOURCES], src_ncols[PPV_TAPS_MAX_SOURCES],
        src_row_off[PPV_TAPS_MAX_SOURCES];
    const float* W;
    const float *bias, *bn_scale, *bn_shift, *seg_scale;
    int M, N, relu, seg_len, nseg, Tp, P, T, halo, zero_invalid;
    int out_f32;
    void* out;
    int64_t out_rows;
    int out_ld, out_col0, block_n, block_k, precision;
} ppv_gemm_taps_case;
size_t ppv_gemm_test_taps_workspace_bytes(const ppv_gemm_taps_case* c);
int ppv_gemm_test_taps(const ppv_gemm_taps_case* c, void* ws, size_t ws_bytes, void* stream);

/* Test hook for the Res2Net convs of an SE-Res2Net block (not a reference entry point): y_1 = f_1(x_1), y_j = f_j(x_j + y_{j-1}),
 * f_j = BN(ReLU(conv_k3,dil + bias)) on 64-channel chunks, for j = 1..nconv, through the launches the ECAPA-TDNN plan builds.
 * variant PPV_RES2_CHAIN: res2chain_kernel (T + 8 <= 384); PPV_RES2_CHAIN_PAIRED: res2chain_pair_kernel (T + 8 <= 320);
 * PPV_RES2_PER_CONV: one res2conv_kernel per conv.  x [B*Tp, ld_x] fp32 in the padded time layout (Tp = T + 8, P = 4: frame t of
 * utterance b at row b*Tp + 4 + t), chunk c at columns [64c, 64c + 64); the chain builds its reflect halo rows itself, the per-conv
 * path reads them from x.  w [nconv][64][64][3], bias / bn_scale / bn_shift [nconv][64] fp32.  y [B*Tp + 64, ld_y] fp32: conv j
 * writes columns [64j, 64j + 64) of rows [0, B*Tp) (the chain: every row, the per-conv path: the valid rows and their reflect
 * mirrors).  x and y are split into planes here and come back whole, decoded as hi + lo (y with PPV_PREC_BF16: its hi plane, the
 * only one the convs read and the chain stores): a position no kernel stores keeps its value.  max_ctas: the grid's CTA count cap (0: every SM).  A case the builds reject is PPV_EINVAL before any launch.
 * ws >= ppv_res2net_test_workspace_bytes.  Synchronises `stream` while it prepares the weights. */
#define PPV_RES2_CHAIN 0
#define PPV_RES2_CHAIN_PAIRED 1
#define PPV_RES2_PER_CONV 2
size_t ppv_res2net_test_workspace_bytes(int nconv, int B, int T, int ld_x, int ld_y);
int ppv_res2net_test(float* x, int ld_x, const float* w, const float* bias, const float* bn_scale, const float* bn_shift, int nconv,
                     int B, int T, int dil, int variant, int precision, int max_ctas, float* y, int ld_y, void* ws, size_t ws_bytes,
                     void* stream);

/* Test hook for the skinny linear kernel (not a reference entry point): out[m, out_col0 + n] = act(sum_k x[m, x_col0 + k] W[n, k]
 * + bias[n]) through skinny_linear_launch, as the SE excitation runs it.  x [M, ld] and W [N, K] fp32 are split into planes here;
 * bias [N] may be NULL; act 0: none, 1: ReLU, 2: sigmoid.  out [M, out_ld] fp32: out_planes 0 writes it directly, 1 writes
 * split planes initialised from it and decodes them back whole as hi + lo.  A shape the kernel does not take is PPV_EINVAL before
 * any launch.  ws >= ppv_skinny_linear_test_workspace_bytes. */
size_t ppv_skinny_linear_test_workspace_bytes(int M, int ld, int N, int K, int out_ld);
int ppv_skinny_linear_test(const float* x, int M, int ld, int x_col0, const float* W, int N, int K, const float* bias, int act,
                           int out_planes, float* out, int out_ld, int out_col0, void* ws, size_t ws_bytes, void* stream);

/* Kernel-only timing of the gather-GEMM (tools/gemm_bench.py); ws >= 4*(pad128(M)*pad64(K) + pad256(N)*pad64(K) + pad128(M)*N)
 * bytes + 4*(3 + M/306)*N rounded up to 256.  planes_out: 0 ReLU to fp32, 1 ReLU to planes, 2 bias + ReLU + BN to planes over the
 * padded time layout (Tp = 306, P = 4), 3 the same + per-utterance bias + tanh (ASP attention TDNN); 2 and 3 need M % 306 == 0. */
int ppv_gemm_bench(int M, int N, int K, int block_n, int block_k, int precision, int planes_out, int iters, void* ws,
                   size_t ws_bytes, float* ms_per_launch, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* PPV_B200_H */
