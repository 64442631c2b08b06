// Training-step building blocks shared by train_kernels.cu and ecapa_train.cu (SURVEY.md §8 row a11).
#pragma once
#include "common.h"

namespace ppv {

// One contribution to the gradient of an activation tensor [B * Tp rows][C] in the padded time layout:
//   value(b, t, c) = (t[row, col0 + c] (+ the halo rows mirroring frame t when `fold`)) * rowscale[b][c] * (1 - dtanh[row, c]^2)
//                    + rowbias[b][c]
// `fold` is the backward of the reflect padding (ppvector/models/utils.py:79-93): a data-gradient GEMM stores the gradient of
// the PADDED input on every row, and the halo rows belong to the frames they mirror.  t.base == nullptr: bias-only source.
struct GradSrc {
    Planes t;
    int col0 = 0;
    int fold = 0;
    const float* rowscale = nullptr;  // [B][row_ld]
    const float* rowbias = nullptr;   // [B][row_ld]
    int row_ld = 0;
    Planes dtanh;  // output of a tanh whose derivative multiplies this source
    int dtanh_col0 = 0;
};
struct GradSrcList {
    GradSrc s[3];
    int n = 0;
};

struct BnApplyArgs {
    Planes a, y, add, out2;  // y = a * scale + shift (+ tanh); out2 = y + add (optional, out2.base != nullptr)
    int a_col0 = 0, y_col0 = 0, add_col0 = 0, out2_col0 = 0;
    int C = 0, B = 0, T = 0, P = 0, Tp = 0;
    const float* scale = nullptr;
    const float* shift = nullptr;
    int tanh_ = 0;
};

// part: scratch of at least 3 * B * C floats
int tr_bn_forward(const Planes& a, int a_col0, int C, int B, int T, int P, int Tp, float eps, float momentum, const float* gamma, const float* beta,
                  float* mean, float* rstd, float* scale, float* shift, float* run_mean, float* run_var, float* part, const BnApplyArgs& apply_in,
                  int num_sms, cudaStream_t st);
// dz (valid frames) = d(conv output) through BatchNorm(train) and ReLU; dgamma / dbeta / dbias are [C] outputs.
// `part` holds part_elems floats; the launch needs 2 * B * tsplit * C of them and is refused if they do not fit.
int tr_bn_backward(const GradSrcList& gl, const Planes& a, int a_col0, int C, int B, int T, int P, int Tp, const float* mean, const float* rstd,
                   const float* gamma, float* dgamma, float* dbeta, const Planes& dz, int dz_col0, float* dbias, float* part, size_t part_elems,
                   cudaStream_t st, int tsplit = 1);  // tsplit > 1: `part` holds B * tsplit partial rows (no per-utterance sums)
// out (optional planes, valid frames) = summed sources; part [B][C] = per-utterance column sums; colsum (optional) [C]
int tr_grad_sum(const GradSrcList& gl, int C, int B, int T, int P, int Tp, const Planes& out, int out_col0, float* part, float* colsum, cudaStream_t st);
// out_bc [B][C] = sum_t grad(b,t,c) * y[b,t,c]
int tr_grad_dot(const GradSrcList& gl, const Planes& y, int y_col0, int C, int B, int T, int P, int Tp, float* out_bc, cudaStream_t st);
// out[c][r] = in[r + shift][col0 + c] (zero outside the input rows)
// ntaps > 1: tap z uses shift + z * shift_step and writes output rows [z * out_row_step, ...)  (one launch for all conv taps)
int tr_transpose(const Planes& in, int col0, int C, int64_t rows, const Planes& out, int shift, cudaStream_t st, int ntaps = 1, int shift_step = 0,
                 int64_t out_row_step = 0);
// w: reference conv weight, element (n, cin, tap) at w[n * w_ld + cin * taps + tap]
int tr_repack_conv(const float* w, int64_t w_ld, int Cout, int Cin, int Cinp, int taps, const Planes& wf, const Planes& wd, cudaStream_t st);
int tr_wgrad_unpack(const float* part, int splits, int64_t split_rows, int Cout, int Cin, int Cinp, int taps, float* grad, int64_t g_ld,
                    cudaStream_t st);
int tr_dense_fwd(const float* X, int64_t x_ld, const float* W, int64_t w_ld, const float* bias, int M, int N, int K, int act, float* Y, int64_t y_ld,
                 cudaStream_t st);
int tr_dense_bwd(const float* dY, int64_t dy_ld, const float* X, int64_t x_ld, const float* W, int64_t w_ld, int M, int N, int K, float* dX,
                 int64_t dx_ld, float* dW, int64_t dw_ld, float* db, cudaStream_t st);
int tr_act_bwd(float* dy, const float* y, int64_t n, int act, float alpha, cudaStream_t st);  // act 0: scale by alpha; 1 relu'; 2 sigmoid'
int tr_bn1d_fwd(const float* x, int B, int C, float eps, float momentum, const float* gamma, const float* beta, float* y, float* mean, float* rstd,
                float* run_mean, float* run_var, cudaStream_t st);
int tr_bn1d_bwd(const float* dy, const float* x, int B, int C, const float* gamma, const float* mean, const float* rstd, float* dx, float* dgamma,
                float* dbeta, cudaStream_t st);
int tr_asp_bwd(const float* logits, int64_t lg_ld, const Planes& x, int C, int B, int T, int P, int Tp, float eps, const float* pooled,
               const float* dpooled, const Planes& dlogits, const Planes& dx, cudaStream_t st);
// Backward of temporal average / statistics pooling (TAP / TSP) over x's first C columns: given pooled = [mean | var] and dpooled =
// [d mean | d var] as fp32 [B][var ? 2C : C], writes dx[b,t,c] = dmean[b,c] / T (+ dvar[b,c] * 2 (x[b,t,c] - mean[b,c]) / (T - 1) with
// `var`, the unbiased variance) on the T valid frames of each utterance; no other row of dx is written.
int tr_pool_stats_bwd(const Planes& x, int C, int B, int T, int P, int Tp, const float* pooled, const float* dpooled, bool var, const Planes& dx,
                      cudaStream_t st);
int tr_asp_global_bwd(const float* gstat, const float* dgstat, int B, int C, int T, float eps, float* rs, float* rb, cudaStream_t st);

}  // namespace ppv
