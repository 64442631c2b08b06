// The 2-D models' shared plan pieces (image_plan.h): image-grid geometry and epilogues, conv routing, the plan step executor, and the
// kernels every 2-D model runs: the stem conv, the flatten of the last grid to a time-major matrix, and the fp32 image tap.
#include <stdlib.h>

#include "image_plan.h"
#include "ptx.cuh"

namespace ppv {

// ------------------------------------------------------------------------------------------------ kernels
// conv1: 1 -> C0 channels, 3x3, padding 1, BN folded, ReLU.  One thread per (output position, 8-channel group): the nine
// inputs are read once per thread and each thread stores 16 bytes per plane so that a warp writes whole 128-byte lines of
// consecutive positions.
__global__ void __launch_bounds__(256)
    rs_conv1_kernel(const float* __restrict__ feat, int B, int T, int F, const float* __restrict__ w9, const float* __restrict__ bias, int C0,
                    Planes out, int Hp, int Wp) {
    griddep_launch_dependents();
    // A thread owns one group of 8 output channels for the whole launch: its 72 weights and 8 biases live in registers, and it walks
    // the positions with a grid stride.  (Per-position weight reads from shared memory made the kernel LDS-bound: 72 LDS for 72 FMAs.)
    // Where the group count does not divide the block size, the spare threads recompute the first position of the next block's
    // range and store the same values.
    const int groups = C0 >> 3;
    const int g = threadIdx.x % groups;
    float wr[8][9], br[8];
#pragma unroll
    for (int c = 0; c < 8; ++c) {
        br[c] = __ldg(bias + g * 8 + c);
#pragma unroll
        for (int k = 0; k < 9; ++k) wr[c][k] = __ldg(w9 + (g * 8 + c) * 9 + k);
    }
    griddep_wait();
    const int64_t npos = int64_t(B) * F * T;
    const int64_t pstep = int64_t(gridDim.x) * (256 / groups);
    for (int64_t pos = int64_t(blockIdx.x) * (256 / groups) + threadIdx.x / groups; pos < npos; pos += pstep) {
        const int b = int(pos / (int64_t(F) * T));
        const int rem = int(pos - int64_t(b) * F * T);
        const int h = rem / T, w = rem % T;  // h = frequency bin, w = frame
        float x[9];
#pragma unroll
        for (int dh = -1; dh <= 1; ++dh)
#pragma unroll
            for (int dw = -1; dw <= 1; ++dw) {
                const int hh = h + dh, ww = w + dw;
                // input image is feats transposed: in[h][w] = feat[b][w][h]  (resnet_se.py:122-123)
                x[(dh + 1) * 3 + dw + 1] = (hh >= 0 && hh < F && ww >= 0 && ww < T) ? __ldg(feat + (int64_t(b) * T + ww) * F + hh) : 0.f;
            }
        const int64_t row = (int64_t(b) * Hp + h + 1) * Wp + w + 1;
        uint32_t hw[4], lw[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            float y[2];
#pragma unroll
            for (int e = 0; e < 2; ++e) {
                float acc = br[2 * j + e];
#pragma unroll
                for (int k = 0; k < 9; ++k) acc = fmaf(wr[2 * j + e][k], x[k], acc);
                y[e] = fmaxf(acc, 0.f);
            }
            split_pack_bf16x2(y[0], y[1], hw[j], lw[j]);
        }
        *reinterpret_cast<uint4*>(out.hi() + row * out.ld + g * 8) = make_uint4(hw[0], hw[1], hw[2], hw[3]);
        *reinterpret_cast<uint4*>(out.lo() + row * out.ld + g * 8) = make_uint4(lw[0], lw[1], lw[2], lw[3]);
    }
}

// [B, Hp, Wp, C] image -> [B * W, C * H] time-major matrix with channel index c * H + h  (x.reshape([B, -1, T']),
// resnet_se.py:133, then ASP treats axis 1 as channels)
__global__ void __launch_bounds__(256) rs_flatten_kernel(Planes in, int B, int H, int W, int Hp, int Wp, int C, Planes out) {
    griddep_launch_dependents();
    griddep_wait();
    const int64_t total = int64_t(B) * W * C * H;
    for (int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x; i < total; i += int64_t(gridDim.x) * blockDim.x) {
        const int col = int(i % (int64_t(C) * H));
        const int64_t bt = i / (int64_t(C) * H);
        const int c = col / H, h = col % H;
        const int b = int(bt / W), w = int(bt % W);
        const int64_t src = ((int64_t(b) * Hp + h + 1) * Wp + w + 1) * in.ld + c;
        out.hi()[bt * out.ld + col] = in.hi()[src];
        out.lo()[bt * out.ld + col] = in.lo()[src];
    }
}

// image planes -> fp32 [B, H, W, C] (taps)
__global__ void rs_image_to_f32_kernel(Planes in, int B, int H, int W, int Hp, int Wp, int C, float* __restrict__ out) {
    const int64_t total = int64_t(B) * H * W * C;
    for (int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x; i < total; i += int64_t(gridDim.x) * blockDim.x) {
        const int c = int(i % C);
        const int64_t p = i / C;
        const int w = int(p % W);
        const int h = int((p / W) % H);
        const int b = int(p / (int64_t(W) * H));
        const int64_t src = ((int64_t(b) * Hp + h + 1) * Wp + w + 1) * in.ld + c;
        out[i] = __bfloat162float(in.hi()[src]) + __bfloat162float(in.lo()[src]);
    }
}

int launch_stem_conv(const float* feat, int B, int T, int F, const float* w9, const float* bias, int C0, const Planes& out, int Hp, int Wp,
                     cudaStream_t st) {
    // every 8-channel group needs a thread of the 256-thread block
    PPV_REQUIRE(C0 % 8 == 0 && C0 >= 8 && C0 / 8 <= 256 && out.ld % 8 == 0, "stem conv: C0 must be a multiple of 8 up to 2048");
    const int64_t total = int64_t(B) * F * T * (C0 / 8);
    const unsigned grid = unsigned(std::min<int64_t>((total + 255) / 256, int64_t(device_sm_count()) * 8));
    PPV_PDL_OK(launch_pdl(rs_conv1_kernel, dim3(grid), dim3(256), 0, st, feat, B, T, F, w9, bias, C0, out, Hp, Wp), "rs_conv1_kernel");
    return PPV_OK;
}
int launch_flatten_image(const Planes& in, int B, int H, int W, int Hp, int Wp, int C, const Planes& out, int num_sms, cudaStream_t st) {
    const int64_t total = int64_t(B) * W * C * H;
    const int grid = int(std::min<int64_t>((total + 255) / 256, int64_t(num_sms) * 16));
    PPV_PDL_OK(launch_pdl(rs_flatten_kernel, dim3(grid), dim3(256), 0, st, in, B, H, W, Hp, Wp, C, out), "rs_flatten_kernel");
    return PPV_OK;
}
int launch_image_to_f32(const Planes& in, int B, int H, int W, int Hp, int Wp, int C, float* out, cudaStream_t st) {
    const int64_t total = int64_t(B) * H * W * C;
    rs_image_to_f32_kernel<<<int(std::min<int64_t>((total + 255) / 256, 132 * 32)), 256, 0, st>>>(in, B, H, W, Hp, Wp, C, out);
    PPV_LAUNCH_OK("rs_image_to_f32_kernel");
    return PPV_OK;
}

// ------------------------------------------------------------------------------------------------ geometry / epilogue / taps
void image_pyramid(ImageGeo* levels, int n, int H, int W, bool halve_w) {
    for (int l = 0; l < n; ++l) {
        if (l > 0) {
            H = (H - 1) / 2 + 1;
            if (halve_w) W = (W - 1) / 2 + 1;
        }
        levels[l].H = H;
        levels[l].W = W;
        levels[l].Hp = H + 2;
        levels[l].Wp = W + 2;
    }
}

Epilogue image_epilogue(const Planes& out, const ImageGeo& gin, const ImageGeo& gout, int stride_h, int stride_w) {
    Epilogue ep;
    ep.out_mode = OUT_PLANES;
    ep.out = out.base;
    ep.out_ld = out.ld;
    ep.out_plane_stride = out.plane_stride;
    ep.img_Hp = gin.Hp;
    ep.img_Wp = gin.Wp;
    ep.img_H = gin.H;
    ep.img_W = gin.W;
    ep.img_stride = stride_h;
    ep.img_stride_w = stride_w == stride_h ? 0 : stride_w;  // 0: the same stride on both axes
    ep.out_Hp = gout.Hp;
    ep.out_Wp = gout.Wp;
    return ep;
}

void image_taps(std::vector<GemmSource>* v, const Planes& p, int col0, int ncols, const ImageGeo& g) {
    for (int dh = -1; dh <= 1; ++dh)
        for (int dw = -1; dw <= 1; ++dw) v->push_back(GemmSource{p, col0, ncols, dh * g.Wp + dw});
}

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
PlanStep scale_res_step(const Planes& z, const float* scale, const Planes& res, const Planes& out, int C, const ImageGeo& g, int B, float relu_max) {
    PlanStep s;
    s.kind = PlanStep::SCALE_RES;
    s.x = z;
    s.vec[0] = scale;
    s.y = res;
    s.out = out;
    s.C = C;
    s.g = g;
    s.B = B;
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
PlanStep colstats_step(const Planes& x, int C, int B, int T, int P, int Tp, int mode, float eps, const Planes& out, float inv_count) {
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
    return s;
}
PlanStep model_step(int model_kind) {
    PlanStep s;
    s.kind = PlanStep::MODEL;
    s.model_kind = model_kind;
    return s;
}

// ------------------------------------------------------------------------------------------------ conv routing
int ImagePlanModel::plan_gemm(const GemmWeights& gw, const std::vector<GemmSource>& srcs, int M, Epilogue ep) {
    ep.bias = gw.bias;
    PlanStep s;
    s.kind = PlanStep::GEMM;
    int rc = gemm_build(&s.gp, srcs.data(), int(srcs.size()), gw.W, M, gw.N, ep, gemm_pick_bn(gw.N));
    if (rc) return rc;
    steps.push_back(s);
    return PPV_OK;
}

int ImagePlanModel::plan_conv(const GemmWeights& gw, const std::vector<GemmSource>& srcs, int M, Epilogue ep) {
    ep.bias = gw.bias;
    PlanStep s;
    if (!pointwise_step_build(&s.pw, srcs.data(), int(srcs.size()), gw.W, gw.N, M, ep)) return plan_gemm(gw, srcs, M, ep);
    s.kind = PlanStep::POINTWISE;
    steps.push_back(s);
    return PPV_OK;
}

int ImagePlanModel::plan_conv3x3(const GemmWeights& gw, const Planes& x, int col0, int ncols, const ImageGeo& g, int B, Epilogue ep) {
    const char* e = getenv("PPV_CONV3X3");  // 0 = every 3x3 conv on the gather-GEMM (debugging / A-B timing)
    const bool patch = !(e && e[0] == '0') && ncols == 32 && gw.N == 32 && gw.Ktot == 9 * 32 && conv3x3_c32_supported(ncols, gw.N, g.H, g.W);
    if (!patch) {
        std::vector<GemmSource> taps;
        image_taps(&taps, x, col0, ncols, g);
        return plan_gemm(gw, taps, int(g.rows(B)), ep);
    }
    ep.bias = gw.bias;
    PlanStep s;
    s.kind = PlanStep::CONV3X3;
    int rc = conv3x3_build(&s.c3, x, col0, gw.W, B, g.H, g.W, g.Hp, g.Wp, ep);
    if (rc) return rc;
    steps.push_back(s);
    return PPV_OK;
}

// ------------------------------------------------------------------------------------------------ executor
int ImagePlanModel::run_steps(const float* feat, cudaStream_t st) {
    for (const PlanStep& s : steps) {
        int rc = PPV_OK;
        switch (s.kind) {
            case PlanStep::GEMM: rc = gemm_launch(s.gp, precision, num_sms, st); break;
            case PlanStep::CONV3X3: rc = conv3x3_launch(s.c3, precision, num_sms, st); break;
            case PlanStep::POINTWISE: rc = pointwise_launch(s.pw, num_sms, st); break;
            case PlanStep::STEM: rc = launch_stem_conv(feat, s.B, s.g.W, s.g.H, s.vec[0], s.vec[1], s.C, s.out, s.g.Hp, s.g.Wp, st); break;
            case PlanStep::SCALE_RES:
                rc = launch_se_scale_res(s.x, s.vec[0], s.y, 0, s.out, 0, s.C, s.g.Hp * s.g.Wp, s.g.rows(s.B), num_sms, st, 1, s.relu_max);
                break;
            case PlanStep::AFF_COMBINE: rc = launch_aff_combine(s.x, s.xc0, s.y, s.yc0, s.t, s.out, s.C, s.rows, num_sms, st); break;
            case PlanStep::FLATTEN_IMAGE: rc = launch_flatten_image(s.x, s.B, s.g.H, s.g.W, s.g.Hp, s.g.Wp, s.C, s.out, num_sms, st); break;
            case PlanStep::COLSTATS:
                rc = launch_colstats(s.x, 0, s.C, s.B, s.T, s.P, s.Tp, s.mode, s.eps, nullptr, s.out, st, s.inv_count);
                break;
            case PlanStep::ASP_FUSED: rc = asp_fused_launch(s.ap, precision, num_sms, st); break;
            case PlanStep::MODEL: rc = run_model_step(s, st); break;
        }
        if (rc) return rc;
    }
    return PPV_OK;
}

int ImagePlanModel::run_model_step(const PlanStep&, cudaStream_t) { return fail(PPV_EINVAL, std::string(prefix) + ": plan step of unknown kind"); }

// ------------------------------------------------------------------------------------------------ taps
int ImagePlanModel::name_index(const std::string& n, const char* base, int lo, int hi) {
    const size_t len = strlen(base);
    if (n.size() != len + 1 || n.compare(0, len, base) != 0) return 0;
    const int i = n[len] - '0';
    return i >= lo && i <= hi ? i : 0;
}

int ImagePlanModel::image_tap(const Planes& src, const ImageGeo& g, int C, float* out, size_t out_elems, cudaStream_t st) const {
    PPV_REQUIRE(out_elems >= size_t(plan_B) * g.H * g.W * C, std::string(prefix) + "_read_tap: output too small");
    return launch_image_to_f32(src, plan_B, g.H, g.W, g.Hp, g.Wp, C, out, st);
}

}  // namespace ppv
