// Shared host/device declarations for libppv_b200: status codes, error reporting, tensor views,
// the GEMM launch parameters and the kernel launchers each .cu file exports to the others.
#pragma once
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdlib.h>

#include <algorithm>
#include <string>
#include <utility>

#include "../../include/ppv_b200.h"

namespace ppv {

void set_error(const std::string& msg);
int fail(int code, const std::string& msg);

#define PPV_CUDA_OK(expr)                                                                             \
    do {                                                                                              \
        cudaError_t _e = (expr);                                                                      \
        if (_e != cudaSuccess)                                                                        \
            return ::ppv::fail(PPV_ECUDA, std::string(#expr) + ": " + cudaGetErrorString(_e));        \
    } while (0)
#define PPV_LAUNCH_OK(what)                                                                           \
    do {                                                                                              \
        cudaError_t _e = cudaGetLastError();                                                          \
        if (_e != cudaSuccess) return ::ppv::fail(PPV_ECUDA, std::string(what) + ": " + cudaGetErrorString(_e)); \
    } while (0)
#define PPV_REQUIRE(cond, msg)                                     \
    do {                                                           \
        if (!(cond)) return ::ppv::fail(PPV_EINVAL, std::string(msg)); \
    } while (0)

// Function attributes (the > 48 KB dynamic shared-memory opt-in) are per device: run `stmt` once per device of this process, not once
// per process (a second GPU used by the same process would otherwise launch without the opt-in).
#define PPV_ONCE_PER_DEVICE(stmt)                                    \
    do {                                                             \
        static unsigned long long _ppv_done = 0ull;                  \
        int _ppv_dev = 0;                                            \
        cudaGetDevice(&_ppv_dev);                                    \
        if (!((_ppv_done >> (_ppv_dev & 63)) & 1ull)) {              \
            stmt;                                                    \
            _ppv_done |= 1ull << (_ppv_dev & 63);                    \
        }                                                            \
    } while (0)

// Process-wide switch (ppv_set_pdl): 1 = launches carry the programmatic-stream-serialization attribute (default), 0 = plain stream order.
// With SEVERAL batches in flight on different streams an early-launched dependent CTA sits on an SM (these kernels take a whole SM's shared
// memory) until its primary grid has drained, and that SM is lost to the other streams' runnable kernels: callers that keep lanes busy
// switch the early launch off for the duration (the kernels' griddepcontrol instructions are no-ops then).
inline int& pdl_enabled() {
    static int v = 1;
    return v;
}

// Launch with programmatic dependent launch enabled (see ptx.cuh: griddep_wait / griddep_launch_dependents).
template <typename... KArgs, typename... Args>
inline cudaError_t launch_pdl(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st, Args&&... args) {
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = grid;
    cfg.blockDim = block;
    cfg.dynamicSmemBytes = smem;
    cfg.stream = st;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = pdl_enabled() ? 1 : 0;
    cfg.attrs = attr;
    cfg.numAttrs = 1;
    return cudaLaunchKernelEx(&cfg, kernel, std::forward<Args>(args)...);
}
#define PPV_PDL_OK(call, what)                                                                                     \
    do {                                                                                                           \
        cudaError_t _e = (call);                                                                                   \
        if (_e != cudaSuccess) return ::ppv::fail(PPV_ECUDA, std::string(what) + ": " + cudaGetErrorString(_e));   \
    } while (0)

// ---- activation storage ---------------------------------------------------------------------------
// Activations between kernels are "split planes": two bf16 matrices hi/lo with x ~= hi + lo
// (~2^-17 relative), row-major [2][rows][ld].  Rows are frames in the PADDED time layout
//   row = b * Tp + P + t,  Tp = T + 2P,
// so that a dilated conv tap is a plain row offset and the reflect padding of the reference's Conv1d
// (ppvector/models/utils.py:79-93) is materialised as halo rows written by the producing epilogue.
struct Planes {
    __nv_bfloat16* base = nullptr;
    int64_t rows = 0;
    int ld = 0;                // elements per row
    int64_t plane_stride = 0;  // elements between the hi and the lo plane
    __host__ __device__ __nv_bfloat16* hi() const { return base; }
    __host__ __device__ __nv_bfloat16* lo() const { return base + plane_stride; }
};

struct TimeLayout {  // padded time layout of a batch
    int B = 0, T = 0, P = 0, Tp = 0;
    int64_t rows() const { return int64_t(B) * Tp; }
};

// ---- GEMM -----------------------------------------------------------------------------------------
constexpr int GEMM_BM = 128;
constexpr int GEMM_BK = 64;
constexpr int GEMM_MAX_KSTEPS = 192;
constexpr int GEMM_MAX_MAPS = 4;
constexpr int GEMM_WS_STAGES = 4;  // ring slots in weight-stationary mode (the rest of the ring's shared memory holds W)

struct KStep {
    int16_t map;      // which A tensor map
    int16_t row_off;  // row offset (conv tap * dilation)
    int32_t a_col;    // first column of the 64-wide K slice in that A tensor
};

enum OutMode : int { OUT_PLANES = 0, OUT_F32 = 1 };

struct Epilogue {
    const float* bias = nullptr;         // [N]
    const float* rowgrp_bias = nullptr;  // [rows / rows_per_group][N]  (per-utterance bias)
    const float* bn_scale = nullptr;     // [N]  y = y * scale + shift  (BatchNorm eval, after ReLU)
    const float* bn_shift = nullptr;     // [N]
    int relu = 0;
    int tanh_ = 0;
    int sigmoid_ = 0;
    int silu_ = 0;
    float relu_max = 0.f;  // > 0: clipped ReLU (Hardtanh(0, relu_max), ERes2Net) applied where `relu` is set
    int out_mode = OUT_PLANES;
    void* out = nullptr;            // Planes base (bf16) or float*
    int64_t out_ld = 0;             // elements
    int64_t out_plane_stride = 0;   // elements (OUT_PLANES)
    int out_col0 = 0;
    // row validity: Tp == 0 -> rows [0, M) are all valid (plain matrix); else padded time layout.
    int Tp = 0, P = 0, T = 0;
    int halo = 0;  // also write the reflect halo rows (output feeds a dilated conv)
    // 2-D image layout (conv2d models): GEMM rows are positions of a zero-bordered [B, img_Hp, img_Wp] grid; a row is
    // stored iff it is an interior position on the output stride grid, at its position in the [B, out_Hp, out_Wp] grid.
    int img_Hp = 0, img_Wp = 0, img_H = 0, img_W = 0, img_stride = 1, out_Hp = 0, out_Wp = 0;
    int img_stride_w = 0;  // 0: same as img_stride; CAM++'s FCM strides the frequency axis only (campplus.py:223-224)
    // per-(utterance, time segment) output scale, padded time layout only: y *= seg_scale[(b * nseg + t / seg_len) * N + n]
    // (context-aware mask of CAM++, campplus.py:88-93); applied after the biases, before the activations
    const float* seg_scale = nullptr;
    int seg_len = 0, nseg = 0;
    int zero_invalid = 0;  // planes output without halo on the input grid: rows outside the valid frames are stored as zeros (zero-padded convs read them)
    int f32_vec_ok = 0;  // set by gemm_build: OUT_F32 rows and columns are 8-byte aligned (paired stores)
    int debug_nostore = 0;  // PPV_GEMM_NOSTORE=1 (tools/gemm_bench.py only): skip the epilogue stores
    int lean = 0;  // set by gemm_build: the epilogue needs only what epilogue_frag_lean does (gemm_epilogue.cuh)
};

// An epilogue that writes split-bf16 planes `out` from column col0: on every row, or with Tp > 0 on the padded time layout (the T
// valid rows of every Tp = T + 2P).
inline Epilogue planes_epilogue(const Planes& out, int col0 = 0, int Tp = 0, int P = 0, int T = 0) {
    Epilogue ep;
    ep.out_mode = OUT_PLANES;
    ep.out = out.base;
    ep.out_ld = out.ld;
    ep.out_plane_stride = out.plane_stride;
    ep.out_col0 = col0;
    ep.Tp = Tp;
    ep.P = P;
    ep.T = T;
    return ep;
}

constexpr int GEMM_TRACE_TILES = 16;   // PPV_GEMM_TRACE: the traced CTA's first tiles stamped
constexpr int GEMM_TRACE_EVENTS = 16;  // stamps per role and tile

struct GemmParams {
    CUtensorMap mapA[GEMM_MAX_MAPS];
    CUtensorMap mapB;
    KStep ksteps[GEMM_MAX_KSTEPS];
    int num_ksteps;
    int bk;  // K elements per k-step (64 or 32)
    int ws;           // weight-stationary mode (set by gemm_build): W resident in shared memory, the ring carries activations only
    int lin_splits;   // > 0: weight-gradient mode (see gemm_build_wgrad): K runs over operand columns, split in lin_splits parts
    int lin_b_row0, lin_b_col0;
    int64_t lin_split_rows;
    int M, N;
    int m_tiles, n_tiles;
    Epilogue epi;
    // debug (PPV_GEMM_TRACE=<cta>, default 0): clock64 stamps of CTA trace_cta, [role][tile][event] with role 0 = producer,
    // 1 + g = MMA warpgroup g
    unsigned long long* trace;
    int trace_cta;
    int bn;  // n-tile width (64, 128 or 256): selects the kernel instance.  Last, so that no kernel parameter offset depends on it.
};
void gemm_trace_dump(const GemmParams& gp);

struct GemmSource {
    Planes t;
    int col0;     // first column
    int ncols;    // multiple of 64
    int row_off;  // tap offset in rows
};

// Precision of the tensor-core contraction.
//   PPV_PREC_BF16X3: A_hi*B_hi + A_lo*B_hi + A_hi*B_lo  (fp32-grade, ~2^-16 relative per product)
//   PPV_PREC_BF16  : A_hi*B_hi only
// BK = 0: 64, or 32 where a source's K slice is not a multiple of 64.
int gemm_build(GemmParams* gp, const GemmSource* srcs, int nsrc, const Planes& W, int M, int N, const Epilogue& epi,
               int BN, int BK = 0);
int gemm_build_wgrad(GemmParams* gp, const Planes& At, const Planes& Bt, int M, int N, int b_row0, int b_col0, int splits, float* out,
                     int64_t out_ld, int out_col0, int64_t split_rows, int BN);
int gemm_launch(const GemmParams& gp, int precision, int num_sms, cudaStream_t stream);
// The widest n-tile, up to max_bn, that divides N (64 at least).
inline int gemm_pick_bn(int N, int max_bn = 256) {
    for (int bn = max_bn; bn > 64; bn /= 2)
        if (N % bn == 0) return bn;
    return 64;
}

int encode_planes_map(CUtensorMap* m, const Planes& t, int box_rows);  // 3-D TMA map over split planes, box {64, box_rows, 1}, SWIZZLE_128B
int encode_planes_map_ex(CUtensorMap* m, const Planes& t, int box_cols, int box_rows, int swizzle_bytes);  // 0 / 64 / 128

// ---- Res2Net dilated conv, weight-stationary, one tall activation tile per source (res2conv.cu) ------
struct Res2Params {
    CUtensorMap mapA[2];  // source planes, box {64, 128 + 8, 1}
    CUtensorMap mapW;     // weight planes [2][64][nsrc*3*64], box {64, 64, 1}
    int a_col[2];
    int nsrc, dil;
    int l2_prefetch;
    int M, m_tiles;
    Epilogue epi;
};
int res2conv_build(Res2Params* rp, const GemmSource* srcs, int nsrc, const Planes& W, int M, int dil, const Epilogue& epi);
int res2conv_launch(const Res2Params& rp, int precision, int num_sms, cudaStream_t st);

// ---- 3x3 conv, 32 -> 32 channels, over zero-bordered image grids: weight-stationary, one image patch per work item (conv3x3.cu) ----
struct Conv3x3Params {
    CUtensorMap mapX;  // 5-D {C, Wp, Hp, B, plane}, box {32, 64, 8, 1, 1}, SWIZZLE_64B
    CUtensorMap mapW;  // weight planes [2][>= 32][9 x 32], box {32, 32, 1}, SWIZZLE_64B
    int x_col0;
    int B, H, W, Hp, Wp;
    int nph, npw, patches;
    Epilogue epi;
};
bool conv3x3_c32_supported(int Cin, int Cout, int H, int W);
int conv3x3_build(Conv3x3Params* cp, const Planes& x, int x_col0, const Planes& Wt, int B, int H, int W, int Hp, int Wp, const Epilogue& epi);
int conv3x3_launch(const Conv3x3Params& cp, int precision, int num_sms, cudaStream_t st);

// ---- the whole Res2Net chain of a block, operands resident in shared memory (res2chain.cu): two utterances per CTA up to
// Tp = 320 ("paired"), else one utterance per CTA up to Tp = 384 ----------
constexpr int RES2CHAIN_MAX = 7;
struct Res2ChainParams {
    CUtensorMap mapX;                  // tdnn1 output planes, box {64, 200 (one utterance per CTA) or 168 (paired), 1}: the resident tile of conv 1
    CUtensorMap mapXt, mapY, mapYtail; // one utterance per CTA only, 128-row staging tiles: next-chunk load, y store, y store of the utterance's last tile
    CUtensorMap mapW[RES2CHAIN_MAX];   // per-conv weight planes [2][>=64][>=192], box {64, 64, 1}
    const float* bias[RES2CHAIN_MAX];
    const float* bn_scale[RES2CHAIN_MAX];
    const float* bn_shift[RES2CHAIN_MAX];
    Planes x;  // tdnn1 output [rows][>= 8*64]: chunk j at columns 64 j
    Planes y;  // Res2Net output [rows][>= 8*64]: conv j (1-based) -> columns 64 j
    int nconv, width, B, T, P, Tp, dil, ntiles;
    int paired;                 // 1: res2chain_pair_kernel, 0: res2chain_kernel
    unsigned long long* trace;  // debug (PPV_RES2_TRACE): clock64 stamps of CTA 0's first utterance (pair), [role][conv][event]
};
int res2chain_build(Res2ChainParams* cp, const Planes& x, const Planes& y, const Planes* W, const float* const* bias, const float* const* bn_scale,
                    const float* const* bn_shift, int nconv, int B, int T, int P, int Tp, int dil, bool paired);
int res2chain_launch(const Res2ChainParams& cp, int precision, int num_sms, cudaStream_t st);
bool res2chain_fits(int T, int P);       // one utterance per CTA: Tp <= 384
bool res2chain_pair_fits(int T, int P);  // two utterances per CTA: Tp <= 320
void res2chain_trace_dump(const Res2ChainParams& cp);

// ---- 1x1 convs with K <= 64 on the CUDA cores, one thread per grid position (pointwise.cu) ----------------------------
int pointwise_launch(const GemmSource* srcs, int nsrc, const Planes& W, int64_t M, int N, const Epilogue& ep, int num_sms, cudaStream_t st);
struct PwStep {  // a planned pointwise conv (the model plans keep these next to their GemmParams)
    GemmSource srcs[2];
    int nsrc = 0, N = 0;
    int64_t M = 0;
    Planes W;
    Epilogue ep;
};
inline int pointwise_launch(const PwStep& s, int num_sms, cudaStream_t st) { return pointwise_launch(s.srcs, s.nsrc, s.W, s.M, s.N, s.ep, num_sms, st); }
// Plans a 1x1 conv over an image grid on the CUDA cores where pointwise_launch supports it; false: it takes the gather-GEMM.
// PPV_POINTWISE=0 keeps every such layer on the gather-GEMM (A-B timing).
bool pointwise_step_build(PwStep* s, const GemmSource* srcs, int nsrc, const Planes& W, int N, int64_t M, const Epilogue& ep);

// ---- skinny linear layers on the CUDA cores (skinny.cu): [B x K] x [K x N] with one row per utterance ----------------
bool skinny_linear_supported(int M, int N, int K, const Epilogue& ep);
int skinny_linear_launch(const Planes& x, int x_col0, const Planes& W, int M, int N, int K, const Epilogue& ep, cudaStream_t st);

// ---- fused attentive statistics pooling (asp_fused.cu) ----------------------------------------------
struct AspFusedParams {
    CUtensorMap mapW;    // planes [2][C][K]   box {64, 128, 1}
    CUtensorMap mapAtt;  // planes [2][rows][K] box {64, 64, 1}
    CUtensorMap mapX;    // planes [2][rows][C] box {128, 64, 1}, no swizzle
    Planes x;            // MFA output, padded time layout, ld = C
    const float* bn_scale;  // asp_bn folded, [2C]
    const float* bn_shift;
    Planes out;          // [B, 2C] (mean | std) after asp_bn -> fc GEMM operand
    float* out_raw;      // [B, 2C] fp32 before asp_bn (tap)
    int B, T, P, Tp, C, K;
    float eps;
    const int* nvalid;  // optional [B]: frames t >= nvalid[b] get attention weight 0 (`lengths`, pooling.py:112-115); set per launch
};

int asp_fused_build(AspFusedParams* p, const Planes& W, const Planes& att, const Planes& x, const float* bn_scale,
                    const float* bn_shift, const Planes& out, float* out_raw, int B, int T, int P, int Tp, int C, int K, float eps);
int asp_fused_launch(const AspFusedParams& p, int precision, int num_sms, cudaStream_t st);

// ---- other kernels (elementwise.cu) ---------------------------------------------------------------
int launch_pack_features(const float* feat, int B, int T, int F, const Planes& out, int P, int Tp, cudaStream_t st);
int launch_colstats(const Planes& x, int col0, int C, int B, int T, int P, int Tp, int mode, float eps, float* out_f32,
                    const Planes& out_pl, cudaStream_t st, float inv_count = 0.f, const int* nvalid = nullptr);
int launch_lengths_to_counts(const float* lengths, int B, int T, int* nvalid, cudaStream_t st);
int launch_se_scale_res(const Planes& z, const float* scale, const Planes& res, int rc0, const Planes& out, int oc0, int C,
                        int Tp, int64_t rows, int num_sms, cudaStream_t st, int relu = 0, float relu_max = 0.f);
int launch_asp_pool(const float* logits, int64_t lg_ld, const Planes& x, int C, int B, int T, int P, int Tp, float eps,
                    const float* bn_scale, const float* bn_shift, const Planes& out_pl, float* out_raw, cudaStream_t st);
int launch_planes_to_f32(const Planes& x, int col0, int C, int B, int T, int P, int Tp, float* out, cudaStream_t st);
int launch_f32_to_planes(const float* src, int64_t rows, int cols, const Planes& out, cudaStream_t st);

// ---- fbank.cu ---------------------------------------------------------------------------------------
struct Fbank;
int fbank_create(const ppv_fbank_cfg* cfg, Fbank** out);
void fbank_destroy(Fbank* h);
int fbank_num_frames(const Fbank* h, int L);
int fbank_n_mels(const Fbank* h);
int fbank_run(Fbank* h, const float* wav, const float* lens_ratio, int B, int L, float* raw, float* out_f32,
              const Planes& out_pl, int P, int Tp, cudaStream_t st, const int* valid_frames = nullptr);

// ---- audio_prep.cu ----------------------------------------------------------------------------------
size_t audio_prep_workspace_bytes(int B, int max_new_len);
int audio_prep(const float* wav, int64_t wav_ld, const int32_t* iparams, const float* fparams, const float* noise, int B, int max_new_len,
               float target_db, int normalize, int Lout, float* out, void* ws, size_t ws_bytes, cudaStream_t st);
size_t audio_prep_reverb_workspace_bytes(int B, int max_new_len, int max_rir_len);
int audio_prep_reverb(const float* wav, int64_t wav_ld, const int32_t* iparams, const float* fparams, const float* noise, const float* rir_bank,
                      int64_t rir_bank_len, const int32_t* rparams, int B, int max_new_len, int max_rir_len, float target_db, int normalize,
                      int Lout, float* out, void* ws, size_t ws_bytes, cudaStream_t st);

// ---- reverb.cu: the convolution stage of audio_prep_reverb (gains [B][2] in: signal / noise gains, out: normalisation gain of reverb items)
size_t reverb_workspace_bytes(int B, int max_new_len, int max_rir_len);
int reverb_run(const float* wav, int64_t wav_ld, const int32_t* iparams, const float* fparams, const float* noise, const float* rir_bank,
               int64_t rir_bank_len, const int32_t* rparams, int B, int max_new_len, int max_rir_len, float target_db, int normalize,
               int Lout, float* out, float* gains, void* ws, cudaStream_t st);

// ---- spectral.cu ------------------------------------------------------------------------------------
struct Spectral;
void spectral_default_cfg(ppv_spectral_cfg* c, int method);
int spectral_create(const ppv_spectral_cfg* cfg, Spectral** out);
void spectral_destroy(Spectral* h);
int spectral_num_frames(const Spectral* h, int L);
int spectral_feature_dim(const Spectral* h);
int spectral_run(Spectral* h, const float* wav, const float* lens_ratio, int B, int L, float* out, cudaStream_t st);
int spec_augment_run(float* feat, const int32_t* params, int B, int T, int F, int n_freq_masks, int n_time_masks, int fill_mode, cudaStream_t st);

// ---- model factories (ecapa.cu, resnet_se.cu, eres2net.cu, campplus.cu; the Model interface is in model_common.h) -------------
struct Model;
void ppv_ecapa_default_cfg_impl(ppv_ecapa_cfg* c);
int ecapa_create(const ppv_ecapa_cfg* cfg, Model** out);
// ECAPA-TDNN only (m must be one): waveform input through `fb`, `lengths`, and the launch-group profile
int ecapa_forward(Model* m, const float* feat, Fbank* fb, const float* wav, const float* lens_ratio, int B, int T, int L, float* emb,
                  void* ws, size_t ws_bytes, cudaStream_t st, const float* lengths = nullptr);
int ecapa_profile(Model* m, int enable);
int ecapa_profile_read(Model* m, double* gemm_ms, double* other_ms, int64_t* gemm_launches, int64_t* other_launches);
void ppv_resnetse_default_cfg_impl(ppv_resnetse_cfg* c);
int resnetse_create(const ppv_resnetse_cfg* cfg, Model** out);
void ppv_eres2net_default_cfg_impl(ppv_eres2net_cfg* c);
int eres2net_create(const ppv_eres2net_cfg* cfg, Model** out);
void ppv_campplus_default_cfg_impl(ppv_campplus_cfg* c);
int campplus_create(const ppv_campplus_cfg* cfg, Model** out);

// ---- conv2d models: zero-bordered NHWC image grids (image_plan.h / image_plan.cu) ------------------------
struct ImageGeo {
    int H = 0, W = 0, Hp = 0, Wp = 0;
    int64_t rows(int B) const { return int64_t(B) * Hp * Wp; }
};
// stem: 1 -> C0 channels, 3x3, padding 1, folded BN, ReLU, from feats [B,T,F] (image = feats transposed: H = F, W = T)
int launch_stem_conv(const float* feat, int B, int T, int F, const float* w9, const float* bias, int C0, const Planes& out, int Hp, int Wp,
                     cudaStream_t st);
// [B,Hp,Wp,C] image -> [B*W, C*H] time-major matrix (channel index c*H + h)
int launch_flatten_image(const Planes& in, int B, int H, int W, int Hp, int Wp, int C, const Planes& out, int num_sms, cudaStream_t st);
int launch_image_to_f32(const Planes& in, int B, int H, int W, int Hp, int Wp, int C, float* out, cudaStream_t st);
// xo = x * (1 + t) + y * (1 - t)  (AFF blend, eres2net.py:50-51 with t = tanh(att)); all rows
int launch_aff_combine(const Planes& x, int xc0, const Planes& y, int yc0, const Planes& t, const Planes& out, int C, int64_t rows, int num_sms,
                       cudaStream_t st);

// ---- ecapa_train.cu / train_kernels.cu ---------------------------------------------------------------
struct Trainer;
int trainer_create(const ppv_ecapa_cfg* cfg, int num_classes, Trainer** out);
void trainer_destroy(Trainer* t);
int64_t trainer_param_count(const Trainer* t);
int64_t trainer_stat_count(const Trainer* t);
int trainer_lookup(const Trainer* t, const char* name, int64_t* off, int64_t* numel, int* is_stat);
int trainer_bind(Trainer* t, float* params, float* grads, float* stats);
int trainer_set_precision(Trainer* t, int precision);
size_t trainer_workspace_bytes(const Trainer* t, int B, int T);
int trainer_forward_backward(Trainer* t, const float* feat, const int64_t* labels, int B, int T, float margin, float scale, int easy_margin,
                             float label_smoothing, float* loss_out, float* logits_out, void* ws, size_t ws_bytes, cudaStream_t st);
int trainer_read_tap(Trainer* t, const char* name, float* out, size_t out_elems, cudaStream_t st);
int adam_step(float* params, const float* grads, float* m, float* v, int64_t n, float lr, float beta1, float beta2, float eps, float weight_decay,
              int64_t step, float grad_scale, cudaStream_t st);

// ---- cosine.cu / aam.cu -----------------------------------------------------------------------------
size_t cosine_workspace_bytes(int M, int N, int D);
int cosine_matrix(const float* A, const float* Bm, int M, int N, int D, float* out, void* ws, size_t ws_bytes, int precision,
                  cudaStream_t st);
int cosine_pairlist(const float* E, const int32_t* idx, int64_t P, int n, int D, float* out, cudaStream_t st);
size_t aam_workspace_bytes(int B, int D, int S);
int aam_forward(const float* emb, const float* W, const int64_t* labels, int B, int D, int S, float margin, float scale,
                int easy_margin, float label_smoothing, float* logits, float* loss, void* ws, size_t ws_bytes, cudaStream_t st);
int aam_backward(const float* emb, const float* W, const int64_t* labels, const float* logits, int B, int D, int S, float margin,
                 float scale, int easy_margin, float label_smoothing, float* d_emb, float* d_W, void* ws, size_t ws_bytes,
                 cudaStream_t st);

// ---- metrics.cu -------------------------------------------------------------------------------------
size_t eer_workspace_bytes(int64_t n);
int eer_mindcf(const float* scores, const int32_t* labels, const int32_t* row_labels, const int32_t* col_labels, int ncols, int64_t n,
               double p_target, double c_miss, double c_fa, double* out, void* ws, size_t ws_bytes, cudaStream_t st);
int row_argmax(const float* sim, int rows, int cols, int32_t* idx, float* best, cudaStream_t st);

// ---- cluster.cu -------------------------------------------------------------------------------------
int cluster_prune(float* A, int N, double pval, cudaStream_t st);
int cluster_laplacian(const float* P, int N, double* L, cudaStream_t st);
size_t sym_eig_workspace_bytes(int N, int m);
int sym_eig_smallest(double* L, int N, int m, double* evals, double* evecs, void* ws, size_t ws_bytes, cudaStream_t st);
size_t kmeans_workspace_bytes(int N, int k);
int kmeans(const double* X, int ld, int N, int k, const double* uniforms, int n_uniforms, int max_iter, int32_t* labels, double* inertia, void* ws,
           size_t ws_bytes, cudaStream_t st);

int device_sm_count();

}  // namespace ppv
