// The 2-D models' shared plan pieces (image_plan.h): image-grid geometry, epilogues and taps, 3x3 conv routing, the ASP head of ResNetSE
// and Res2Net, and the kernels every 2-D model runs: the stem conv, the flatten of the last grid to a time-major matrix, and the fp32
// image tap.
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
    Epilogue ep = planes_epilogue(out);
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

// ------------------------------------------------------------------------------------------------ 3x3 conv routing
int PlanModel::plan_conv3x3(const GemmWeights& gw, const Planes& x, int col0, int ncols, const ImageGeo& g, int B, Epilogue ep) {
    const char* e = getenv("PPV_CONV3X3");  // 0 = every 3x3 conv on the gather-GEMM (debugging / A-B timing)
    const bool patch = !(e && e[0] == '0') && ncols == 32 && gw.N == 32 && gw.Ktot == 9 * 32 && conv3x3_c32_supported(ncols, gw.N, g.H, g.W);
    if (!patch) {
        std::vector<GemmSource> taps;
        image_taps(&taps, x, col0, ncols, g);
        return plan_gemm(gw, taps, int(g.rows(B)), ep);
    }
    ep.bias = gw.bias;
    Conv3x3Params c3;
    int rc = conv3x3_build(&c3, x, col0, gw.W, B, g.H, g.W, g.Hp, g.Wp, ep);
    if (rc) return rc;
    steps.push_back({"conv3x3_launch", true, [c3](const StepRun& r) { return conv3x3_launch(c3, r.precision, r.num_sms, r.st); }});
    return PPV_OK;
}

// ------------------------------------------------------------------------------------------------ ASP head
bool prepare_asp_head(ArenaBuilder& ab, AspHead* h, int cat, int A, int E) {
    h->cat = cat;
    h->att = A;
    h->embd = E;
    const HostWeight* wt = ab.get("pooling.tdnn.conv.conv.weight", {A, 3 * cat, 1});
    const HostWeight* bt = ab.get("pooling.tdnn.conv.conv.bias", {A});
    const HostWeight* wc = ab.get("pooling.conv.conv.weight", {cat, A, 1});
    const HostWeight* wl = ab.get("linear.weight", {2 * cat, E});
    const HostWeight* bl = ab.get("linear.bias", {E});
    std::vector<double> s3, h3;
    const bool ok = wt && bt && wc && wl && bl && ab.put_bn(&h->att1_bn_scale, &h->att1_bn_shift, "pooling.tdnn.norm.norm", A, A) &&
                    ab.put_bn(&h->bn2_scale, &h->bn2_shift, "bn2.norm", 2 * cat, 2 * cat) && ab.bn_affine("bn3.norm", E, &s3, &h3);
    if (!ok) return false;
    std::vector<double> mx(size_t(A) * cat), mf(size_t(A) * 2 * cat), mc(size_t(cat) * A), ml(size_t(E) * 2 * cat);
    for (int a = 0; a < A; ++a) {
        for (int c = 0; c < cat; ++c) mx[size_t(a) * cat + c] = wt->v[size_t(a) * 3 * cat + c];
        for (int c = 0; c < 2 * cat; ++c) mf[size_t(a) * 2 * cat + c] = wt->v[size_t(a) * 3 * cat + cat + c];
    }
    for (size_t i = 0; i < mc.size(); ++i) mc[i] = wc->v[i];
    std::vector<float> bl2(E);
    for (int n = 0; n < E; ++n) {
        for (int k = 0; k < 2 * cat; ++k) ml[size_t(n) * 2 * cat + k] = double(wl->v[size_t(k) * E + n]) * s3[n];
        bl2[n] = float(double(bl->v[n]) * s3[n] + h3[n]);
    }
    ab.put_matrix(&h->att1, mx, A, cat);
    ab.put_f32(&h->att1.bias, bt->v);
    ab.put_matrix(&h->fold, mf, A, 2 * cat);
    ab.put_matrix(&h->att2, mc, cat, A);
    ab.put_matrix(&h->fc, ml, E, 2 * cat);
    ab.put_f32(&h->fc.bias, bl2);
    return true;
}

int PlanModel::plan_asp_head(const AspHead& h, const AspHeadBuffers& hb, int B, int Tf) {
    const int cat = h.cat;
    steps.push_back(colstats_step(hb.flat, cat, B, Tf, 0, Tf, 1, 1e-12f, hb.gstat));
    {
        Epilogue ep;
        ep.out_mode = OUT_F32;
        ep.out = hb.fold_out;
        ep.out_ld = h.att;
        int rc = plan_gemm(h.fold, {GemmSource{hb.gstat, 0, 2 * cat, 0}}, B, ep);
        if (rc) return rc;
    }
    {
        Epilogue ep = planes_epilogue(hb.attp);
        ep.relu = 1;
        ep.Tp = Tf;
        ep.P = 0;
        ep.T = Tf;
        ep.rowgrp_bias = hb.fold_out;
        ep.bn_scale = h.att1_bn_scale;
        ep.bn_shift = h.att1_bn_shift;
        ep.tanh_ = 1;
        int rc = plan_gemm(h.att1, {GemmSource{hb.flat, 0, cat, 0}}, B * Tf, ep);
        if (rc) return rc;
    }
    int rc = plan_asp_fused(h.att2.W, hb.attp, hb.flat, h.bn2_scale, h.bn2_shift, hb.pooled, hb.pooled_raw, B, Tf, 0, Tf, cat, h.att, 1e-12f);
    if (rc) return rc;
    Epilogue ep;
    ep.out_mode = OUT_F32;
    ep.out = hb.emb_out;
    ep.out_ld = h.embd;
    return plan_gemm(h.fc, {GemmSource{hb.pooled, 0, 2 * cat, 0}}, B, ep);
}

// ------------------------------------------------------------------------------------------------ taps
int PlanModel::name_index(const std::string& n, const char* base, int lo, int hi) {
    const size_t len = strlen(base);
    if (n.size() != len + 1 || n.compare(0, len, base) != 0) return 0;
    const int i = n[len] - '0';
    return i >= lo && i <= hi ? i : 0;
}

int PlanModel::image_tap(const Planes& src, const ImageGeo& g, int C, float* out, size_t out_elems, cudaStream_t st) const {
    PPV_REQUIRE(out_elems >= size_t(plan_B) * g.H * g.W * C, std::string(prefix) + "_read_tap: output too small");
    return launch_image_to_f32(src, plan_B, g.H, g.W, g.Hp, g.Wp, C, out, st);
}

}  // namespace ppv
