// The plans (plan.h): step constructors, layer routing, the model forward, the step executor and its launch profile.
#include "plan.h"

namespace ppv {

// ------------------------------------------------------------------------------------------------ steps
PlanStep gemm_step(const GemmParams& gp) {
    return {"gemm_launch", true, [gp](const StepRun& r) { return gemm_launch(gp, r.precision, r.num_sms, r.st); }};
}
PlanStep stem_step(const float* w9, const float* bias, int C0, const Planes& out, const ImageGeo& g, int B) {
    return {"launch_stem_conv", false,
            [w9, bias, C0, out, g, B](const StepRun& r) { return launch_stem_conv(r.in.feat, B, g.W, g.H, w9, bias, C0, out, g.Hp, g.Wp, r.st); }};
}
PlanStep scale_res_step(const Planes& z, const float* scale, const Planes& res, int rc0, const Planes& out, int oc0, int C, int rows_per_utt,
                        int64_t rows, bool relu, float relu_max) {
    return {"launch_se_scale_res", false, [z, scale, res, rc0, out, oc0, C, rows_per_utt, rows, relu, relu_max](const StepRun& r) {
                return launch_se_scale_res(z, scale, res, rc0, out, oc0, C, rows_per_utt, rows, r.num_sms, r.st, relu ? 1 : 0, relu_max);
            }};
}
PlanStep aff_combine_step(const Planes& x, int xc0, const Planes& y, int yc0, const Planes& t, const Planes& out, int C, int64_t rows) {
    return {"launch_aff_combine", false, [x, xc0, y, yc0, t, out, C, rows](const StepRun& r) {
                return launch_aff_combine(x, xc0, y, yc0, t, out, C, rows, r.num_sms, r.st);
            }};
}
PlanStep flatten_step(const Planes& in, const ImageGeo& g, int B, int C, const Planes& out) {
    return {"launch_flatten_image", false,
            [in, g, B, C, out](const StepRun& r) { return launch_flatten_image(in, B, g.H, g.W, g.Hp, g.Wp, C, out, r.num_sms, r.st); }};
}
PlanStep colstats_step(const Planes& x, int C, int B, int T, int P, int Tp, int mode, float eps, const Planes& out, float inv_count, bool masked,
                       float* out_f32) {
    return {"launch_colstats", false, [x, C, B, T, P, Tp, mode, eps, out, inv_count, masked, out_f32](const StepRun& r) {
                return launch_colstats(x, 0, C, B, T, P, Tp, mode, eps, out_f32, out, r.st, inv_count, masked ? r.in.nvalid : nullptr);
            }};
}

// ------------------------------------------------------------------------------------------------ routing
int PlanModel::plan_gemm(const GemmWeights& gw, const std::vector<GemmSource>& srcs, int M, Epilogue ep) {
    ep.bias = gw.bias;
    GemmParams gp;
    int rc = gemm_build(&gp, srcs.data(), int(srcs.size()), gw.W, M, gw.N, ep, gemm_pick_bn(gw.N, max_bn));
    if (rc) return rc;
    steps.push_back(gemm_step(gp));
    return PPV_OK;
}

int PlanModel::plan_conv(const GemmWeights& gw, const std::vector<GemmSource>& srcs, int M, Epilogue ep) {
    ep.bias = gw.bias;
    PwStep pw;
    if (!pointwise_step_build(&pw, srcs.data(), int(srcs.size()), gw.W, gw.N, M, ep)) return plan_gemm(gw, srcs, M, ep);
    steps.push_back({"pointwise_launch", false, [pw](const StepRun& r) { return pointwise_launch(pw, r.num_sms, r.st); }});
    return PPV_OK;
}

int PlanModel::plan_row_linear(const GemmWeights& gw, const GemmSource& src, int M, Epilogue ep) {
    ep.bias = gw.bias;
    if (src.row_off != 0 || gw.Ktot != src.ncols || !skinny_linear_supported(M, gw.N, src.ncols, ep)) return plan_gemm(gw, {src}, M, ep);
    steps.push_back({"skinny_linear_launch", false, [x = src.t, col0 = src.col0, W = gw.W, M, N = gw.N, K = src.ncols, ep](const StepRun& r) {
                         return skinny_linear_launch(x, col0, W, M, N, K, ep, r.st);
                     }});
    return PPV_OK;
}

int PlanModel::plan_asp_fused(const Planes& W, const Planes& att, const Planes& x, const float* bn_scale, const float* bn_shift,
                              const Planes& out, float* out_raw, int B, int T, int P, int Tp, int C, int K, float eps) {
    AspFusedParams ap;
    int rc = asp_fused_build(&ap, W, att, x, bn_scale, bn_shift, out, out_raw, B, T, P, Tp, C, K, eps);
    if (rc) return rc;
    steps.push_back({"asp_fused_launch", true, [ap](const StepRun& r) {
                         AspFusedParams p = ap;
                         p.nvalid = r.in.nvalid;
                         return asp_fused_launch(p, r.precision, r.num_sms, r.st);
                     }});
    return PPV_OK;
}

// ------------------------------------------------------------------------------------------------ forward
int Model::forward(const ModelInput& in, int B, int T, float* emb, void* ws, size_t ws_bytes, cudaStream_t st) {
    const std::string fn = std::string(prefix) + "_forward";
    PPV_REQUIRE(emb && (in.feat != nullptr) != (in.wav != nullptr), fn + ": null argument, or not exactly one of feat / wav");
    if (in.wav && !takes_wav()) return fail(PPV_EUNSUPPORTED, fn + ": no fused waveform path; call ppv_fbank_forward + ppv_model_forward");
    if (in.lengths && !takes_lengths()) return fail(PPV_EUNSUPPORTED, fn + ": takes no lengths (only EcapaTdnn.forward does in the reference)");
    if (in.wav) {
        PPV_REQUIRE(in.fb, fn + ": wav input needs a fbank handle");
        PPV_REQUIRE(fbank_n_mels(in.fb) == input_size(), fn + ": fbank n_mels != model input_size");
        T = fbank_num_frames(in.fb, in.L);
        PPV_REQUIRE(T > 0, fn + ": waveform shorter than one frame");
    }
    if (!finalized) return fail(PPV_ESTATE, fn + ": call ppv_model_finalize first");
    PPV_REQUIRE(B > 0 && T > 0, fn + ": empty batch");
    PlanInputs pin{in.feat};
    int rc = update_plan(B, T, ws, ws_bytes, st);
    if (!rc) rc = stage_inputs(in, &pin, st);
    if (!rc) rc = run_plan(pin, st);
    if (rc) return rc;
    PPV_CUDA_OK(cudaMemcpyAsync(emb, emb_out, size_t(B) * embd_dim() * sizeof(float), cudaMemcpyDeviceToDevice, st));
    return PPV_OK;
}

int Model::stage_fbank(const ModelInput& in, float* raw, float* out_f32, const Planes& out_pl, int P, int Tp, cudaStream_t st) {
    prof_begin(1, st);
    const int rc = fbank_run(in.fb, in.wav, in.lens_ratio, plan_B, in.L, raw, out_f32, out_pl, P, Tp, st);
    launches_other += 3;
    prof_end(st);
    return rc;
}

// ------------------------------------------------------------------------------------------------ executor
int PlanOwner::run_plan(const PlanInputs& in, cudaStream_t st) {
    const StepRun run{in, precision, num_sms, st};
    for (size_t i = 0; i < steps.size(); ++i) {
        const PlanStep& s = steps[i];
        // (skinny and pointwise steps count as "other kernels": their FLOPs are not credited to the tensor-core roofline)
        prof_begin(s.tensor ? 0 : 1, st);
        if (s.tensor) launches_gemm += 1; else launches_other += 1;
        const int rc = s.launch(run);
        prof_end(st);
        if (rc) return rc;
        if (sync_each_step) {
            const cudaError_t e = cudaStreamSynchronize(st);
            if (e != cudaSuccess)
                return fail(PPV_ECUDA, std::string(prefix) + ": step " + std::to_string(i) + " (" + s.name + ") failed: " + cudaGetErrorString(e));
        }
    }
    return PPV_OK;
}

// ------------------------------------------------------------------------------------------------ profile
PlanOwner::~PlanOwner() {
    for (cudaEvent_t e : prof_ev) cudaEventDestroy(e);
}

void PlanOwner::profile(bool enable) {
    prof_on = enable;
    prof_used = 0;
    launches_gemm = launches_other = 0;
}

void PlanOwner::prof_begin(int kind, cudaStream_t st) {
    if (!prof_on) return;
    if (prof_used + 2 > prof_ev.size()) {
        cudaEvent_t a, b;
        cudaEventCreate(&a);
        cudaEventCreate(&b);
        prof_ev.push_back(a);
        prof_ev.push_back(b);
        prof_kind.push_back(kind);
    }
    prof_kind[prof_used / 2] = kind;
    cudaEventRecord(prof_ev[prof_used], st);
}

void PlanOwner::prof_end(cudaStream_t st) {
    if (!prof_on) return;
    cudaEventRecord(prof_ev[prof_used + 1], st);
    prof_used += 2;
}

int PlanOwner::profile_read(double* gemm_ms, double* other_ms, int64_t* gemm_launches, int64_t* other_launches) {
    double g = 0, o = 0;
    if (prof_used >= 2) PPV_CUDA_OK(cudaEventSynchronize(prof_ev[prof_used - 1]));
    for (size_t i = 0; i + 1 < prof_used; i += 2) {
        float ms = 0.f;
        PPV_CUDA_OK(cudaEventElapsedTime(&ms, prof_ev[i], prof_ev[i + 1]));
        (prof_kind[i / 2] == 0 ? g : o) += ms;
    }
    *gemm_ms = g;
    *other_ms = o;
    *gemm_launches = launches_gemm;
    *other_launches = launches_other;
    prof_used = 0;
    launches_gemm = launches_other = 0;
    return PPV_OK;
}

}  // namespace ppv
