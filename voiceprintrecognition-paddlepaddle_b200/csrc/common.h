// Shared host/device declarations for libppv_b200: status codes, error reporting, tensor views, workspace carving,
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
#include <vector>

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

// ---- caller-owned workspaces --------------------------------------------------------------------------
inline size_t align_up(size_t x, size_t a) { return (x + a - 1) / a * a; }

// Lays out a workspace: 256-byte aligned buffers in order from `base`.  Every call that takes a workspace has one carve function;
// run on a null base it measures the extent its size query returns, run on the workspace it yields the views, so the size and the
// layout cannot disagree.
struct WsCarver {
    uint8_t* base = nullptr;
    size_t off = 0;
    void* take(size_t bytes) {
        off = align_up(off, 256);
        void* p = base ? base + off : nullptr;
        off += bytes;
        return p;
    }
    Planes planes(int64_t rows, int ld) {
        Planes p;
        p.rows = int64_t(align_up(size_t(rows), 128));
        p.ld = ld;
        p.plane_stride = p.rows * ld;
        p.base = static_cast<__nv_bfloat16*>(take(size_t(2) * p.plane_stride * sizeof(__nv_bfloat16)));
        return p;
    }
};
// What a size query returns: the extent of `carve(WsCarver&)` run on a null base.
template <typename Carve>
size_t carve_extent(const Carve& carve) {
    WsCarver cv;
    carve(cv);
    return align_up(cv.off, 256);
}

// The check every call makes on its workspace before any launch: `ws` is non-null, 256-byte aligned and holds the `need` bytes the
// call's carve takes, which the size query `query` returns.
inline int check_workspace(const char* call, const void* ws, size_t ws_bytes, size_t need, const char* query) {
    if (ws && ws_bytes >= need && (reinterpret_cast<uintptr_t>(ws) & 255) == 0) return PPV_OK;
    return fail(PPV_EINVAL, std::string(call) + ": the workspace must be a non-null, 256-byte aligned buffer of at least " + std::to_string(need) +
                                " bytes (" + query + "); got " + std::to_string(ws_bytes) + " bytes at " +
                                std::to_string(reinterpret_cast<uintptr_t>(ws)));
}

// ---- GEMM -----------------------------------------------------------------------------------------
constexpr int GEMM_BM = 128;
constexpr int GEMM_BK = 64;
constexpr int GEMM_MAX_KSTEPS = 320;  // K up to 20480: the embedding layer of the 64-channel ERes2Net reads 2 x 10240 TSTP statistics
constexpr int GEMM_MAX_MAPS = 4;
constexpr int GEMM_WS_STAGES = 4;  // ring slots in weight-stationary mode (the rest of the ring's shared memory holds W)

// 4 bytes per k-step, so that the k-step table of GemmParams (a kernel parameter copied at every launch) stays small
struct KStep {
    int16_t row_off;   // row offset (conv tap * dilation)
    uint16_t map_col;  // bits 14-15: which A tensor map; bits 0-13: first column of the K slice in that A tensor, in units of 8
    __host__ __device__ int map() const { return map_col >> 14; }
    __host__ __device__ int a_col() const { return (map_col & 0x3fff) << 3; }
};
static_assert(GEMM_MAX_MAPS <= 4, "KStep holds the map index in two bits");

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
// per-utterance column statistics into the planes out_pl and / or fp32 out_f32 ([B][C] in mode 0, [B][2C] in modes 1-3)
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
              const Planes& out_pl, int P, int Tp, cudaStream_t st, const int* valid_frames = nullptr, const int* num_samples = nullptr);

// ---- audio_prep.cu ----------------------------------------------------------------------------------
size_t audio_prep_workspace_bytes(int B, int max_new_len);
int audio_prep(const float* wav, int64_t wav_ld, const int32_t* iparams, const float* fparams, const float* noise, int B, int max_new_len,
               float target_db, int normalize, int Lout, float* out, void* ws, size_t ws_bytes, cudaStream_t st);
size_t audio_prep_reverb_workspace_bytes(int B, int max_new_len, int max_rir_len);
int audio_prep_reverb(const float* wav, int64_t wav_ld, const int32_t* iparams, const float* fparams, const float* noise, const float* rir_bank,
                      int64_t rir_bank_len, const int32_t* rparams, int B, int max_new_len, int max_rir_len, float target_db, int normalize,
                      int Lout, float* out, void* ws, size_t ws_bytes, cudaStream_t st);

// ---- reverb.cu: the convolution stage of audio_prep_reverb (gains [B][2] in: signal / noise gains, out: normalisation gain of reverb items)
struct ReverbViews {  // per-output-block energies [B][nm], signal block spectra [B][nx][256], response partition spectra [B][nj][256]
    double* ypart;
    float2 *xspec, *hspec;
};
void carve_reverb(WsCarver& cv, int B, int max_new_len, int max_rir_len, ReverbViews* v);
int reverb_run(const float* wav, int64_t wav_ld, const int32_t* iparams, const float* fparams, const float* noise, const float* rir_bank,
               int64_t rir_bank_len, const int32_t* rparams, int B, int max_new_len, int max_rir_len, float target_db, int normalize,
               int Lout, float* out, float* gains, const ReverbViews& v, cudaStream_t st);

// ---- spectral.cu ------------------------------------------------------------------------------------
struct Spectral;
void spectral_default_cfg(ppv_spectral_cfg* c, int method);
int spectral_create(const ppv_spectral_cfg* cfg, Spectral** out);
void spectral_destroy(Spectral* h);
int spectral_num_frames(const Spectral* h, int L);
int spectral_feature_dim(const Spectral* h);
int spectral_run(Spectral* h, const float* wav, const float* lens_ratio, int B, int L, float* out, cudaStream_t st,
                 const int* valid_frames = nullptr, const int* num_samples = nullptr);
int spec_augment_run(float* feat, const int32_t* params, int B, int T, int F, int n_freq_masks, int n_time_masks, int fill_mode, cudaStream_t st);

// ---- model factories (ecapa.cu, resnet_se.cu, res2net.cu, eres2net.cu, campplus.cu; the Model interface is in model_common.h) -------------
struct Model;
void ppv_ecapa_default_cfg_impl(ppv_ecapa_cfg* c);
int ecapa_create(const ppv_ecapa_cfg* cfg, Model** out);
void ppv_resnetse_default_cfg_impl(ppv_resnetse_cfg* c);
int resnetse_create(const ppv_resnetse_cfg* cfg, Model** out);
void ppv_res2net_default_cfg_impl(ppv_res2net_cfg* c);
int res2net_create(const ppv_res2net_cfg* cfg, Model** out);
void ppv_eres2net_default_cfg_impl(ppv_eres2net_cfg* c);
int eres2net_create(const ppv_eres2net_cfg* cfg, Model** out);
void ppv_campplus_default_cfg_impl(ppv_campplus_cfg* c);
int campplus_create(const ppv_campplus_cfg* cfg, Model** out);
// CAM++'s context-mask MLP weights in the reference layout, w1 [64][128] and w2 [32][64], -> the transposed [128][64] and [64][32]
// the context kernel reads
void campplus_context_weights(const float* w1, const float* w2, std::vector<float>* w1t, std::vector<float>* w2t);
// The context mask of CAM++'s dense layers: h [B Tp, 128] planes (T frames from row P of each utterance) -> out [B nseg, 32] fp32,
// nseg = ceil(T / 100) <= 64
int campplus_context_launch(const Planes& h, int B, int T, int P, int Tp, const float* w1t, const float* b1, const float* w2t,
                            const float* b2, float* out, cudaStream_t st);

// ---- conv2d models: zero-bordered NHWC image grids (image_plan.h / image_plan.cu) ------------------------
struct ImageGeo {
    int H = 0, W = 0, Hp = 0, Wp = 0;
    int64_t rows(int B) const { return int64_t(B) * Hp * Wp; }
};
// stem: 1 -> C0 channels, 3x3, padding 1, folded BN, ReLU, from feats [B,T,F] (image = feats transposed: H = F, W = T)
int launch_stem_conv(const float* feat, int B, int T, int F, const float* w9, const float* bias, int C0, const Planes& out, int Hp, int Wp,
                     cudaStream_t st);
// Res2Net's stem (res2net.cu): 1 -> 32 channels, 7x7, stride 3, padding 1, folded BN (w [32][49]), ReLU, then MaxPool2D(3, 2, 1), from
// feats [B,T,F] into the pooled grid Hq x Wq (zero-bordered, ld out.ld); res2net_stem_grids gives the conv grid H1 x W1 and Hq x Wq
void res2net_stem_grids(int F, int T, int* H1, int* W1, int* Hq, int* Wq);
int launch_res2net_stem(const float* feat, int B, int T, int F, const float* w, const float* bias, int C0, const Planes& out, cudaStream_t st);
// AvgPool2D(3, stride 1 or 2, padding 1, exclusive): columns [in_col0, +ncols) of `in` on the H x W grid -> [out_col0, +ncols) of `out`
// on the ((H-1)/stride+1) x ((W-1)/stride+1) grid; ncols and both column offsets multiples of 8
int launch_avgpool3x3(const Planes& in, int in_col0, int B, int H, int W, int stride, int ncols, const Planes& out, int out_col0, int num_sms,
                      cudaStream_t st);
// [B,Hp,Wp,C] image -> [B*W, C*H] time-major matrix (channel index c*H + h)
int launch_flatten_image(const Planes& in, int B, int H, int W, int Hp, int Wp, int C, const Planes& out, int num_sms, cudaStream_t st);
int launch_image_to_f32(const Planes& in, int B, int H, int W, int Hp, int Wp, int C, float* out, cudaStream_t st);
// xo = x * (1 + t) + y * (1 - t)  (AFF blend, eres2net.py:50-51 with t = tanh(att)); all rows
int launch_aff_combine(const Planes& x, int xc0, const Planes& y, int yc0, const Planes& t, const Planes& out, int C, int64_t rows, int num_sms,
                       cudaStream_t st);

// ---- ecapa_train.cu / train_kernels.cu ---------------------------------------------------------------
struct Trainer;
int trainer_create(const ppv_ecapa_cfg* cfg, int num_classes, int classifier_type, int num_blocks, int inter_dim, Trainer** out);
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
int optimizer_state_count(int kind, int centered);
int optimizer_step(int kind, float* params, const float* grads, float* s0, float* s1, float* s2, int64_t n, const ppv_optim_args& args,
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
// The Linear output layer (fc.py:37-38, 50-51) in front of the same loss heads: logits = H W + b, H [B,D], W [D,S], b [S].  Takes
// the workspace of aam_forward / aam_backward (aam_workspace_bytes(B, D, S)).  Heads that take sqrt(1 - z^2) of the logits are refused.
int linear_head_forward(const float* H, const float* W, const float* bias, const int64_t* labels, int B, int D, int S, float margin, float scale,
                        int easy_margin, float label_smoothing, float* logits, float* loss, void* ws, size_t ws_bytes, cudaStream_t st);
int linear_head_backward(const float* H, const float* W, const int64_t* labels, const float* logits, int B, int D, int S, float margin, float scale,
                         int easy_margin, float label_smoothing, float* d_H, float* d_W, float* d_bias, void* ws, size_t ws_bytes, cudaStream_t st);

// ---- speaker_index.cu ---------------------------------------------------------------------------------
size_t speaker_index_bytes(int U, int D);
int speaker_index_build(const float* E, int n, int D, const int32_t* order, const int32_t* offsets, int U, float* means, void* index,
                        size_t index_bytes, cudaStream_t st);
size_t speaker_index_search_workspace_bytes(int Q, int U, int D, int k);
int speaker_index_search(const float* queries, int Q, int D, const void* index, size_t index_bytes, int U, int k, int32_t* idx, float* sim,
                         void* ws, size_t ws_bytes, cudaStream_t st);

// ---- score_norm.cu ------------------------------------------------------------------------------------
int topn_row_stats(const float* scores, int rows, int cols, int64_t ld, int top_n, float* mean, float* std, cudaStream_t st);
int as_norm_apply(float* scores, int M, int N, const float* trial_mean, const float* trial_std, const float* enroll_mean,
                  const float* enroll_std, cudaStream_t st);

// ---- vad.cu -----------------------------------------------------------------------------------------
int64_t vad_num_frames(const ppv_vad_cfg& cfg, int64_t L);
size_t vad_workspace_bytes(const ppv_vad_cfg& cfg, int R, int64_t total_samples);
int vad_energy(const ppv_vad_cfg& cfg, const float* wav, const int64_t* sample_offsets, int R, double* log_energy, uint8_t* voiced,
               int32_t* runs, int64_t run_cap, int32_t* n_runs, void* ws, size_t ws_bytes, cudaStream_t st);

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
