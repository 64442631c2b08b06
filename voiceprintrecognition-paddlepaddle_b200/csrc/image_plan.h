// How the 2-D models (ResNetSE, ERes2Net, CAM++) plan their convolutions, in one place (image_plan.cu).
//
// Layout: every activation is split-bf16 planes over rows (b, h+1, w+1) of a [B, H+2, W+2] grid whose border rows are zero and
// are never written (freq = H, time = W, channels last).  With that layout
//   * a 3x3 conv (padding 1) is the gather-GEMM with 9 taps at row offsets dh*(W+2)+dw -- the zero border IS the padding; a 32 ->
//     32 channel one runs on the weight-stationary patch kernel (conv3x3.cu) instead, unless PPV_CONV3X3=0;
//   * a strided conv is computed on the input grid and only the rows on the stride lattice are stored, straight into the output
//     grid (epilogue row remap: the strided 3x3 convs cost 4x their FLOPs in exchange for no strided-gather TMA path);
//   * BatchNorm(eval) directly after a conv is folded into the conv's weights and bias at finalize (ArenaBuilder::fold_conv);
//   * a 1x1 conv over a 32-column window may run on the CUDA cores (pointwise.cu), unless PPV_POINTWISE=0.
// A plan is a list of PlanSteps, each holding every argument of its launch; ImagePlanModel::run_steps launches them in order.
#pragma once
#include <string>
#include <vector>

#include "common.h"
#include "model_common.h"

namespace ppv {

// levels[0] = the stem grid H x W; each next level halves H, and W too if `halve_w` (a stride-2 conv's output grid)
void image_pyramid(ImageGeo* levels, int n, int H, int W, bool halve_w);
// Planes epilogue of a conv over grid `gin` whose outputs on the (stride_h, stride_w) lattice are stored into `out` on grid `gout`
Epilogue image_epilogue(const Planes& out, const ImageGeo& gin, const ImageGeo& gout, int stride_h, int stride_w);
// the nine K-sources of a 3x3 conv over columns [col0, col0 + ncols) of `p` on grid `g`, taps in (dh, dw) order
void image_taps(std::vector<GemmSource>* v, const Planes& p, int col0, int ncols, const ImageGeo& g);

struct PlanStep {
    enum Kind { GEMM, CONV3X3, POINTWISE, STEM, SCALE_RES, AFF_COMBINE, FLATTEN_IMAGE, COLSTATS, ASP_FUSED, MODEL } kind;
    int model_kind = 0;  // MODEL: a model's own step, launched by its run_model_step
    GemmParams gp;       // GEMM
    Conv3x3Params c3;    // CONV3X3
    PwStep pw;           // POINTWISE
    AspFusedParams ap;   // ASP_FUSED
    // STEM: feat -> out on grid g, weights vec[0] / vec[1], C0 = C;  SCALE_RES: out = relu(x * vec[0] + y) clipped at relu_max > 0
    // (vec[0] null: no scale) over grid g;  AFF_COMBINE: out = x (1 + t) + y (1 - t) over `rows`;  FLATTEN_IMAGE: x on grid g -> out;
    // COLSTATS: launch_colstats of x's first C columns into out;  MODEL: what the model puts here.
    Planes x, y, t, out;
    int xc0 = 0, yc0 = 0;
    const float* vec[4] = {};
    float* out_f32 = nullptr;
    ImageGeo g;
    int B = 0, C = 0, T = 0, P = 0, Tp = 0, mode = 0, n = 0;
    int64_t rows = 0;
    float eps = 0.f, inv_count = 0.f, relu_max = 0.f;
};

PlanStep stem_step(const float* w9, const float* bias, int C0, const Planes& out, const ImageGeo& g, int B);
PlanStep scale_res_step(const Planes& z, const float* scale, const Planes& res, const Planes& out, int C, const ImageGeo& g, int B,
                        float relu_max = 0.f);
PlanStep aff_combine_step(const Planes& x, int xc0, const Planes& y, int yc0, const Planes& t, const Planes& out, int C, int64_t rows);
PlanStep flatten_step(const Planes& in, const ImageGeo& g, int B, int C, const Planes& out);
PlanStep colstats_step(const Planes& x, int C, int B, int T, int P, int Tp, int mode, float eps, const Planes& out, float inv_count = 0.f);
PlanStep model_step(int model_kind);

// A model whose forward is a plan of PlanSteps.
struct ImagePlanModel : Model {
    std::vector<PlanStep> steps;

    using Model::Model;

  protected:
    int run_steps(const float* feat, cudaStream_t st) override;
    virtual int run_model_step(const PlanStep& s, cudaStream_t st);

    // Conv routing, one entry per kind of conv; each appends its step.  M = GEMM rows; ep.bias is set from gw.
    // gather-GEMM only
    int plan_gemm(const GemmWeights& gw, const std::vector<GemmSource>& srcs, int M, Epilogue ep);
    // the pointwise kernel where pointwise_step_build takes the conv (a 1x1 conv over a 32-column window), else the gather-GEMM
    int plan_conv(const GemmWeights& gw, const std::vector<GemmSource>& srcs, int M, Epilogue ep);
    // 3x3 conv over columns [col0, col0 + ncols) of x on grid g: the patch kernel for a 32 -> 32 channel conv, else nine taps
    int plan_conv3x3(const GemmWeights& gw, const Planes& x, int col0, int ncols, const ImageGeo& g, int B, Epilogue ep);

    // "<base><i>" with lo <= i <= hi (one digit) -> i, else 0
    static int name_index(const std::string& n, const char* base, int lo, int hi);
    // fp32 [B, H, W, C] copy of image planes, after checking out_elems
    int image_tap(const Planes& src, const ImageGeo& g, int C, float* out, size_t out_elems, cudaStream_t st) const;
};

}  // namespace ppv
