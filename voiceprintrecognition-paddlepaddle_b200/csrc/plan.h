// The plans, in one place (plan.cu): ECAPA-TDNN, ResNetSE, Res2Net, ERes2Net(V2) and CAM++ each plan their forward, and the ECAPA-TDNN
// trainer its training step, as a list of PlanSteps, each a launch with its arguments bound when the plan is built; PlanOwner::run_plan
// launches them in order.  The routing helpers choose a layer's kernel; what is about zero-bordered image grids (the 2-D models) is in
// image_plan.h.
#pragma once
#include <functional>
#include <string>
#include <vector>

#include "common.h"
#include "model_common.h"

namespace ppv {

// What a run of a plan reads besides the plan itself.
struct PlanInputs {
    const float* feat = nullptr;      // features [plan_B, plan_T, input_size]
    const int* nvalid = nullptr;      // inference: [plan_B] valid-frame counts for masked column statistics and fused ASP (null: every frame)
    const int64_t* labels = nullptr;  // training: [plan_B] class labels and the AAM-softmax settings
    float margin = 0.f, scale = 0.f, label_smoothing = 0.f;
    int easy_margin = 0;
};

// What a caller hands Model::forward: features, or waveforms through the fused Fbank front end; and, optionally, `lengths`.
struct ModelInput {
    const float* feat = nullptr;     // features [B, T, input_size]; null when wav is set
    Fbank* fb = nullptr;             // the front end of wav [B, L], with lens_ratio as ppv_fbank_forward takes it
    const float* wav = nullptr;
    const float* lens_ratio = nullptr;
    int L = 0;
    const float* lengths = nullptr;  // [B] relative lengths in (0, 1] (ppv_model_forward_lengths); null: every frame
};

// What only the run knows.  Precision is one of them: set_precision switches a live plan without rebuilding it.
struct StepRun {
    const PlanInputs& in;
    int precision, num_sms;
    cudaStream_t st;
};

// One launch of a plan.  `launch` owns copies of every argument the plan fixes (its closure captures values only: the builder's
// locals are gone when it runs) and takes the rest from the run.
struct PlanStep {
    const char* name;  // the launcher; named when a step fails under sync_each_step
    bool tensor;       // the launch profile's tensor-core class: GEMM, 3x3 conv, Res2Net conv / chain, fused ASP
    std::function<int(const StepRun&)> launch;
};

PlanStep gemm_step(const GemmParams& gp);  // a gather-GEMM built by gemm_build or gemm_build_wgrad
// feat -> out on grid g: the 1 -> C0 channel stem conv
PlanStep stem_step(const float* w9, const float* bias, int C0, const Planes& out, const ImageGeo& g, int B);
// out[:, oc0 + c] = z[:, c] * scale[utterance][c] + res[:, rc0 + c] (scale null: no scale), then, if relu, ReLU clipped at relu_max > 0,
// over `rows` rows of rows_per_utt rows per utterance (Tp frames, or an image's Hp x Wp grid)
PlanStep scale_res_step(const Planes& z, const float* scale, const Planes& res, int rc0, const Planes& out, int oc0, int C, int rows_per_utt,
                        int64_t rows, bool relu, float relu_max = 0.f);
// out = x (1 + t) + y (1 - t) over `rows`
PlanStep aff_combine_step(const Planes& x, int xc0, const Planes& y, int yc0, const Planes& t, const Planes& out, int C, int64_t rows);
// `in` on grid g -> time-major `out`
PlanStep flatten_step(const Planes& in, const ImageGeo& g, int B, int C, const Planes& out);
// launch_colstats of x's first C columns into the planes `out` or, if set, out_f32, over each utterance's first nvalid frames if
// `masked` and the run has them
PlanStep colstats_step(const Planes& x, int C, int B, int T, int P, int Tp, int mode, float eps, const Planes& out, float inv_count = 0.f,
                       bool masked = false, float* out_f32 = nullptr);

// A plan of launches over a caller-owned workspace, built for (workspace, B, T) and rebuilt whenever one of them changes: the
// inference models and the training step.
struct PlanOwner {
    const char* prefix;    // error-message prefix, e.g. "resnetse"
    const char* ws_query;  // the C ABI entry point that sizes the workspace, named in the "workspace too small" error
    int precision;
    int num_sms;
    void* plan_ws = nullptr;  // the plan's key (plan_ws, plan_B, plan_T); null and zeros when no plan is built
    int plan_B = 0, plan_T = 0;
    std::vector<PlanStep> steps;
    bool sync_each_step = false;  // run_plan synchronises after every step and names the one that failed (localises a faulting kernel)

    PlanOwner(const char* prefix, const char* ws_query, int precision)
        : prefix(prefix), ws_query(ws_query), precision(precision), num_sms(device_sm_count()) {}
    virtual ~PlanOwner();
    // Bytes of workspace a plan for B utterances of T frames carves; computed without touching the current plan.
    virtual size_t workspace_bytes(int B, int T) const = 0;

    // No plan: B > 0 in every run, so no key matches this one and the next run rebuilds.
    void invalidate_plan() {
        plan_ws = nullptr;
        plan_B = plan_T = 0;
    }
    int update_plan(int B, int T, void* ws, size_t ws_bytes, cudaStream_t st) {
        if (plan_ws == ws && plan_B == B && plan_T == T) return PPV_OK;
        int rc = build_plan(B, T, ws, ws_bytes, st);
        if (rc) {
            invalidate_plan();
            return rc;
        }
        plan_ws = ws;
        plan_B = B;
        plan_T = T;
        return PPV_OK;
    }

    // Launch profile (ppv_model_profile): with it on, run_plan records a CUDA event pair around each launch group; the launch counters
    // count every run.  Tensor-core steps (PlanStep::tensor) are one kind, every other launch the other.
    void profile(bool enable);
    // Sums the event-pair durations recorded since profile(true) by kind, synchronising on the last event, and resets the record.
    int profile_read(double* gemm_ms, double* other_ms, int64_t* gemm_launches, int64_t* other_launches);

  protected:
    // The opening of build_plan: `ws` must hold workspace_bytes(B, T) bytes at 256-byte alignment; it is zeroed on `st`, because the
    // plans rely on zero borders, zero padding rows and zero padding columns that no step writes.
    int claim_workspace(int B, int T, void* ws, size_t ws_bytes, cudaStream_t st) const {
        const size_t need = workspace_bytes(B, T);
        if (int rc = check_workspace(prefix, ws, ws_bytes, need, ws_query)) return rc;
        PPV_CUDA_OK(cudaMemsetAsync(ws, 0, need, st));
        return PPV_OK;
    }
    // Carves `ws` and plans the launches of a run over B utterances of T frames.
    virtual int build_plan(int B, int T, void* ws, size_t ws_bytes, cudaStream_t st) = 0;
    // The executor: launches the planned steps in order.
    int run_plan(const PlanInputs& in, cudaStream_t st);
    // an event pair around launches of kind 0 (tensor cores) or 1 (other), recorded while the profile is on
    void prof_begin(int kind, cudaStream_t st);
    void prof_end(cudaStream_t st);
    int64_t launches_gemm = 0, launches_other = 0;

  private:
    bool prof_on = false;
    std::vector<cudaEvent_t> prof_ev;  // pairs
    std::vector<int> prof_kind;        // per pair: 0 = tensor cores, 1 = other
    size_t prof_used = 0;
};

// An inference model behind ppv_model_*: weights are loaded by name, prepared into one device arena by finalize(), and each
// forward runs the plan.
struct Model : PlanOwner {
    WeightMap raw;
    bool finalized = false;
    void* arena = nullptr;
    float* emb_out = nullptr;  // workspace buffer the plan's last step writes the embeddings [B][embd_dim] to

    Model(const char* prefix, int precision) : PlanOwner(prefix, "ppv_model_workspace_bytes", precision) {}
    ~Model() override { cudaFree(arena); }
    virtual int embd_dim() const = 0;
    virtual int input_size() const = 0;
    // Which inputs forward() takes besides features: waveforms through the fused Fbank front end (the models ppv_model_profile takes
    // too), and `lengths`.
    virtual bool takes_wav() const { return false; }
    virtual bool takes_lengths() const { return false; }

    int load_weight(const char* name, const float* data, const int64_t* shape, int ndim) {
        if (finalized) return fail(PPV_ESTATE, std::string(prefix) + "_load_weight: model already finalized");
        return weight_map_load(&raw, name, data, shape, ndim);
    }
    int set_precision(int p) {
        PPV_REQUIRE(p == PPV_PREC_BF16X3 || p == PPV_PREC_BF16, "bad precision");
        precision = p;
        return PPV_OK;
    }
    int finalize() {
        if (finalized) return PPV_OK;
        ArenaBuilder ab;
        ab.wm = &raw;
        if (!prepare_weights(ab))
            return fail(PPV_EINVAL, std::string(prefix) + "_finalize: " + (ab.err.empty() ? std::string("bad weights") : ab.err));
        int rc = ab.upload(&arena);
        if (rc) return rc;
        raw.clear();
        finalized = true;
        return PPV_OK;
    }
    // B utterances -> emb [B, embd_dim]: T frames of in.feat, or as many as the front end makes of in.wav's L samples (T is then
    // ignored).  Plans for (ws, B, T) if the plan is not that one, stages the inputs, runs the plan and copies the embeddings out.
    int forward(const ModelInput& in, int B, int T, float* emb, void* ws, size_t ws_bytes, cudaStream_t st);
    int read_tap(const char* name, float* out, size_t out_elems, cudaStream_t st) {
        PPV_REQUIRE(name && out, std::string(prefix) + "_read_tap: null argument");
        if (!plan_ws) return fail(PPV_ESTATE, std::string(prefix) + "_read_tap: no forward has run");
        return tap(name, out, out_elems, st);
    }

  protected:
    // Puts the prepared weights into the arena image; false, with ab.err set where known, on a missing or misshapen weight.
    virtual bool prepare_weights(ArenaBuilder& ab) = 0;
    // Puts what the plan reads of `in` where it reads it and sets what else the run passes it in `pin` (pin->feat = in.feat on
    // entry); by default the plan reads in.feat as it is.
    virtual int stage_inputs(const ModelInput& in, PlanInputs* pin, cudaStream_t st) { return PPV_OK; }
    // The fused front end for stage_inputs: the Fbank of in.wav as fbank_run writes it (raw log-mel, then CMN into out_f32 or the
    // planes out_pl of the padded time layout), counted and timed as three other launches.
    int stage_fbank(const ModelInput& in, float* raw, float* out_f32, const Planes& out_pl, int P, int Tp, cudaStream_t st);
    virtual int tap(const std::string& name, float* out, size_t out_elems, cudaStream_t st) = 0;
};

struct AspHead;
struct AspHeadBuffers;

// An inference model with the layer routing helpers.
struct PlanModel : Model {
    int max_bn = 256;  // widest gather-GEMM n-tile plan_gemm picks

    using Model::Model;

  protected:
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
    // Attentive statistics pooling in one kernel (asp_fused_build's arguments); the run supplies the valid-frame counts.
    int plan_asp_fused(const Planes& W, const Planes& att, const Planes& x, const float* bn_scale, const float* bn_shift, const Planes& out,
                       float* out_raw, int B, int T, int P, int Tp, int C, int K, float eps);

    // image-grid helpers (image_plan.cu)
    // 3x3 conv over columns [col0, col0 + ncols) of x on grid g: the patch kernel for a 32 -> 32 channel conv, else nine taps
    int plan_conv3x3(const GemmWeights& gw, const Planes& x, int col0, int ncols, const ImageGeo& g, int B, Epilogue ep);
    // "<base><i>" with lo <= i <= hi (one digit) -> i, else 0
    static int name_index(const std::string& n, const char* base, int lo, int hi);
    // the ASP head of ResNetSE and Res2Net over hb.flat (B utterances of Tf frames) -> hb.emb_out
    int plan_asp_head(const AspHead& h, const AspHeadBuffers& hb, int B, int Tf);
    // fp32 [B, H, W, C] copy of image planes, after checking out_elems
    int image_tap(const Planes& src, const ImageGeo& g, int C, float* out, size_t out_elems, cudaStream_t st) const;
};

}  // namespace ppv
