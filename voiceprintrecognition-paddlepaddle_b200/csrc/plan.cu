// The plans (plan.h): step constructors, layer routing, the step executor and its launch profile.
#include "plan.h"

namespace ppv {

// ------------------------------------------------------------------------------------------------ steps
PlanStep stem_step(const float* w9, const float* bias, int C0, const Planes& out, const ImageGeo& g, int B) {
    PlanStep s;
    s.kind = PlanStep::STEM;
    s.vec[0] = w9;
    s.vec[1] = bias;
    s.C = C0;
    s.out = out;
    s.g = g;
    s.B = B;
    return s;
}
PlanStep scale_res_step(const Planes& z, const float* scale, const Planes& res, int rc0, const Planes& out, int oc0, int C, int rows_per_utt,
                        int64_t rows, bool relu, float relu_max) {
    PlanStep s;
    s.kind = PlanStep::SCALE_RES;
    s.x = z;
    s.vec[0] = scale;
    s.y = res;
    s.yc0 = rc0;
    s.out = out;
    s.oc0 = oc0;
    s.C = C;
    s.utt_rows = rows_per_utt;
    s.rows = rows;
    s.relu = relu;
    s.relu_max = relu_max;
    return s;
}
PlanStep aff_combine_step(const Planes& x, int xc0, const Planes& y, int yc0, const Planes& t, const Planes& out, int C, int64_t rows) {
    PlanStep s;
    s.kind = PlanStep::AFF_COMBINE;
    s.x = x;
    s.xc0 = xc0;
    s.y = y;
    s.yc0 = yc0;
    s.t = t;
    s.out = out;
    s.C = C;
    s.rows = rows;
    return s;
}
PlanStep flatten_step(const Planes& in, const ImageGeo& g, int B, int C, const Planes& out) {
    PlanStep s;
    s.kind = PlanStep::FLATTEN_IMAGE;
    s.x = in;
    s.g = g;
    s.B = B;
    s.C = C;
    s.out = out;
    return s;
}
PlanStep colstats_step(const Planes& x, int C, int B, int T, int P, int Tp, int mode, float eps, const Planes& out, float inv_count, bool masked) {
    PlanStep s;
    s.kind = PlanStep::COLSTATS;
    s.x = x;
    s.C = C;
    s.B = B;
    s.T = T;
    s.P = P;
    s.Tp = Tp;
    s.mode = mode;
    s.eps = eps;
    s.out = out;
    s.inv_count = inv_count;
    s.masked = masked;
    return s;
}
PlanStep model_step(int model_kind) {
    PlanStep s;
    s.kind = PlanStep::MODEL;
    s.model_kind = model_kind;
    return s;
}

// ------------------------------------------------------------------------------------------------ routing
int PlanModel::plan_gemm(const GemmWeights& gw, const std::vector<GemmSource>& srcs, int M, Epilogue ep) {
    ep.bias = gw.bias;
    PlanStep s;
    s.kind = PlanStep::GEMM;
    int rc = gemm_build(&s.gp, srcs.data(), int(srcs.size()), gw.W, M, gw.N, ep, gemm_pick_bn(gw.N, max_bn));
    if (rc) return rc;
    steps.push_back(s);
    return PPV_OK;
}

int PlanModel::plan_conv(const GemmWeights& gw, const std::vector<GemmSource>& srcs, int M, Epilogue ep) {
    ep.bias = gw.bias;
    PlanStep s;
    if (!pointwise_step_build(&s.pw, srcs.data(), int(srcs.size()), gw.W, gw.N, M, ep)) return plan_gemm(gw, srcs, M, ep);
    s.kind = PlanStep::POINTWISE;
    steps.push_back(s);
    return PPV_OK;
}

int PlanModel::plan_row_linear(const GemmWeights& gw, const GemmSource& src, int M, Epilogue ep) {
    ep.bias = gw.bias;
    if (src.row_off != 0 || gw.Ktot != src.ncols || !skinny_linear_supported(M, gw.N, src.ncols, ep)) return plan_gemm(gw, {src}, M, ep);
    PlanStep s;
    s.kind = PlanStep::SKINNY;
    s.pw.srcs[0] = src;
    s.pw.nsrc = 1;
    s.pw.W = gw.W;
    s.pw.M = M;
    s.pw.N = gw.N;
    s.pw.ep = ep;
    steps.push_back(s);
    return PPV_OK;
}

// ------------------------------------------------------------------------------------------------ executor
int PlanOwner::run_plan(const PlanInputs& in, cudaStream_t st) {
    for (size_t i = 0; i < steps.size(); ++i) {
        const PlanStep& s = steps[i];
        const bool tensor_step = s.kind == PlanStep::GEMM || s.kind == PlanStep::CONV3X3 || s.kind == PlanStep::RES2 ||
                                 s.kind == PlanStep::RES2CHAIN || s.kind == PlanStep::ASP_FUSED;
        // (SKINNY and POINTWISE steps count as "other kernels": their FLOPs are not credited to the tensor-core roofline)
        prof_begin(tensor_step ? 0 : 1, st);
        if (tensor_step) launches_gemm += 1; else launches_other += 1;
        int rc = PPV_OK;
        switch (s.kind) {
            case PlanStep::GEMM: rc = gemm_launch(s.gp, precision, num_sms, st); break;
            case PlanStep::SKINNY:
                rc = skinny_linear_launch(s.pw.srcs[0].t, s.pw.srcs[0].col0, s.pw.W, int(s.pw.M), s.pw.N, s.pw.srcs[0].ncols, s.pw.ep, st);
                break;
            case PlanStep::RES2: rc = res2conv_launch(s.rp, precision, num_sms, st); break;
            case PlanStep::RES2CHAIN:
                rc = res2chain_launch(s.cp, precision, num_sms, st);
                if (s.cp.trace) {
                    static int dumps = 0;
                    if (++dumps == 10) res2chain_trace_dump(s.cp);  // a warm launch of the first block
                }
                break;
            case PlanStep::CONV3X3: rc = conv3x3_launch(s.c3, precision, num_sms, st); break;
            case PlanStep::POINTWISE: rc = pointwise_launch(s.pw, num_sms, st); break;
            case PlanStep::STEM: rc = launch_stem_conv(in.feat, s.B, s.g.W, s.g.H, s.vec[0], s.vec[1], s.C, s.out, s.g.Hp, s.g.Wp, st); break;
            case PlanStep::SCALE_RES:
                rc = launch_se_scale_res(s.x, s.vec[0], s.y, s.yc0, s.out, s.oc0, s.C, s.utt_rows, s.rows, num_sms, st, s.relu ? 1 : 0, s.relu_max);
                break;
            case PlanStep::AFF_COMBINE: rc = launch_aff_combine(s.x, s.xc0, s.y, s.yc0, s.t, s.out, s.C, s.rows, num_sms, st); break;
            case PlanStep::FLATTEN_IMAGE: rc = launch_flatten_image(s.x, s.B, s.g.H, s.g.W, s.g.Hp, s.g.Wp, s.C, s.out, num_sms, st); break;
            case PlanStep::COLSTATS:
                rc = launch_colstats(s.x, 0, s.C, s.B, s.T, s.P, s.Tp, s.mode, s.eps, s.out_f32, s.out, st, s.inv_count, s.masked ? in.nvalid : nullptr);
                break;
            case PlanStep::ASP_FUSED: {
                AspFusedParams ap = s.ap;
                ap.nvalid = in.nvalid;
                rc = asp_fused_launch(ap, precision, num_sms, st);
                break;
            }
            case PlanStep::MODEL: rc = run_model_step(s, in, st); break;
        }
        prof_end(st);
        if (rc) return rc;
        if (sync_each_step) {
            const cudaError_t e = cudaStreamSynchronize(st);
            const std::string model = s.kind == PlanStep::MODEL ? ", model kind " + std::to_string(s.model_kind) : "";
            if (e != cudaSuccess)
                return fail(PPV_ECUDA, std::string(prefix) + ": step " + std::to_string(i) + " (kind " + std::to_string(int(s.kind)) + model + ") failed: " + cudaGetErrorString(e));
        }
    }
    return PPV_OK;
}

int PlanOwner::run_model_step(const PlanStep&, const PlanInputs&, cudaStream_t) { return fail(PPV_EINVAL, std::string(prefix) + ": plan step of unknown kind"); }

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
