// The inference models' plans, in one place (plan.cu): ECAPA-TDNN, ResNetSE, ERes2Net(V2) and CAM++ each plan their forward as a
// list of PlanSteps, each holding every argument of its launch, and PlanModel::run_plan launches them in order.  The routing helpers
// choose a layer's kernel; what is about zero-bordered image grids (the 2-D models) is in image_plan.h.
#pragma once
#include <string>
#include <vector>

#include "common.h"
#include "model_common.h"

namespace ppv {

struct PlanStep {
    enum Kind { GEMM, SKINNY, RES2, RES2CHAIN, CONV3X3, POINTWISE, STEM, SCALE_RES, AFF_COMBINE, FLATTEN_IMAGE, COLSTATS, ASP_FUSED, MODEL } kind;
    int model_kind = 0;   // MODEL: a model's own step, launched by its run_model_step
    GemmParams gp;        // GEMM
    Res2Params rp;        // RES2
    Res2ChainParams cp;   // RES2CHAIN
    Conv3x3Params c3;     // CONV3X3
    PwStep pw;            // POINTWISE; SKINNY: srcs[0] is the input, its ncols the K
    AspFusedParams ap;    // ASP_FUSED; nvalid is set per launch
    // STEM: feat -> out on grid g, weights vec[0] / vec[1], C0 = C;
    // SCALE_RES: out[:, oc0 + c] = x[:, c] * vec[0][utterance][c] + y[:, yc0 + c] (vec[0] null: no scale), then, if relu, ReLU clipped
    // at relu_max > 0, over `rows` rows of utt_rows rows per utterance (Tp frames, or an image's Hp x Wp grid);
    // AFF_COMBINE: out = x (1 + t) + y (1 - t) over `rows`;  FLATTEN_IMAGE: x on grid g -> out;
    // COLSTATS: launch_colstats of x's first C columns into out, over each utterance's first nvalid frames if `masked` and the forward
    // has them;  MODEL: what the model puts here.
    Planes x, y, t, out;
    int xc0 = 0, yc0 = 0, oc0 = 0;
    const float* vec[4] = {};
    float* out_f32 = nullptr;
    ImageGeo g;
    int B = 0, C = 0, T = 0, P = 0, Tp = 0, mode = 0, n = 0;
    int64_t rows = 0;
    int utt_rows = 0;
    float eps = 0.f, inv_count = 0.f, relu_max = 0.f;
    bool relu = false, masked = false;
};

PlanStep stem_step(const float* w9, const float* bias, int C0, const Planes& out, const ImageGeo& g, int B);
PlanStep scale_res_step(const Planes& z, const float* scale, const Planes& res, int rc0, const Planes& out, int oc0, int C, int rows_per_utt,
                        int64_t rows, bool relu, float relu_max = 0.f);
PlanStep aff_combine_step(const Planes& x, int xc0, const Planes& y, int yc0, const Planes& t, const Planes& out, int C, int64_t rows);
PlanStep flatten_step(const Planes& in, const ImageGeo& g, int B, int C, const Planes& out);
PlanStep colstats_step(const Planes& x, int C, int B, int T, int P, int Tp, int mode, float eps, const Planes& out, float inv_count = 0.f,
                       bool masked = false);
PlanStep model_step(int model_kind);

// A model whose forward is a plan of PlanSteps.
struct PlanModel : Model {
    std::vector<PlanStep> steps;
    int max_bn = 256;  // widest gather-GEMM n-tile plan_gemm picks

    using Model::Model;
    ~PlanModel() override;

    // Launch profile (ppv_model_profile): with it on, run_plan records a CUDA event pair around each launch group; the launch counters
    // count every run.  Tensor-core steps (GEMM, CONV3X3, RES2, RES2CHAIN, ASP_FUSED) are one kind, every other launch the other.
    void profile(bool enable);
    // Sums the event-pair durations recorded since profile(true) by kind, synchronising on the last event, and resets the record.
    int profile_read(double* gemm_ms, double* other_ms, int64_t* gemm_launches, int64_t* other_launches);

  protected:
    int run_steps(const float* feat, cudaStream_t st) override { return run_plan(feat, nullptr, st); }
    // The executor: feat [plan_B, plan_T, input_size] for STEM steps, nvalid [plan_B] valid-frame counts for masked COLSTATS and
    // ASP_FUSED steps (null: every frame).
    int run_plan(const float* feat, const int* nvalid, cudaStream_t st);
    virtual int run_model_step(const PlanStep& s, cudaStream_t st);
    // an event pair around launches of kind 0 (tensor cores) or 1 (other), recorded while the profile is on
    void prof_begin(int kind, cudaStream_t st);
    void prof_end(cudaStream_t st);
    int64_t launches_gemm = 0, launches_other = 0;

    // Routing, one entry per kind of layer; each appends its step.  M = GEMM rows; ep.bias is set from gw.
    // gather-GEMM only, n-tile up to max_bn
    int plan_gemm(const GemmWeights& gw, const std::vector<GemmSource>& srcs, int M, Epilogue ep);
    // the pointwise kernel where pointwise_step_build takes the conv (a 1x1 conv over a 32-column window), else the gather-GEMM
    int plan_conv(const GemmWeights& gw, const std::vector<GemmSource>& srcs, int M, Epilogue ep);
    // A linear layer over one row per utterance (M = utterances) reading all of gw's K from `src`: the skinny kernel where it takes
    // the shape, else the gather-GEMM.  On the skinny kernel every SM takes a 16 x 16 output tile on the CUDA cores instead of 2-6
    // CTAs walking a latency-bound k-loop on the tensor cores.  The caller guarantees the one row per utterance: the skinny kernel
    // reads plain rows, with no padded time layout and no halo, so a per-frame layer goes to plan_gemm.
    int plan_row_linear(const GemmWeights& gw, const GemmSource& src, int M, Epilogue ep);

    // image-grid helpers (image_plan.cu)
    // 3x3 conv over columns [col0, col0 + ncols) of x on grid g: the patch kernel for a 32 -> 32 channel conv, else nine taps
    int plan_conv3x3(const GemmWeights& gw, const Planes& x, int col0, int ncols, const ImageGeo& g, int B, Epilogue ep);
    // "<base><i>" with lo <= i <= hi (one digit) -> i, else 0
    static int name_index(const std::string& n, const char* base, int lo, int hi);
    // fp32 [B, H, W, C] copy of image planes, after checking out_elems
    int image_tap(const Planes& src, const ImageGeo& g, int C, float* out, size_t out_elems, cudaStream_t st) const;

  private:
    bool prof_on = false;
    std::vector<cudaEvent_t> prof_ev;  // pairs
    std::vector<int> prof_kind;        // per pair: 0 = tensor cores, 1 = other
    size_t prof_used = 0;
};

}  // namespace ppv
