// ResNetSE forward as a plan of tensor-core gather-GEMMs over zero-bordered NHWC images.
// Reference graph: ppvector/models/resnet_se.py:121-139 (ResNetSE.forward), :24-45 (SEBottleneck.forward),
// :59-63 (SELayer.forward), :107-119 (_make_layer: 1x1 strided conv + BN shortcut), ppvector/models/pooling.py:86-125
// (ASP, shared with ECAPA-TDNN).  Eval mode.
//
// Layout: every activation is split-bf16 planes over rows (b, h+1, w+1) of a [B, H+2, W+2] grid whose border rows are
// zero and are never written (freq = H, time = W, channels last).  With that layout
//   * a 3x3 conv (padding 1) is the gather-GEMM with 9 taps at row offsets dh*(W+2)+dw -- the zero border IS the padding;
//   * a stride-2 conv is computed on the input grid and only the rows on the even (h, w) lattice are stored, straight
//     into the half-resolution grid (epilogue row remap; the 3 strided 3x3 convs cost 4x their FLOPs -- +36 % of the
//     model -- in exchange for not needing a strided-gather TMA path in round 1);
//   * BatchNorm(eval) directly after a conv is folded into the conv's weights and bias at finalize;
//   * SE: global average pool = column sums over the whole zero-bordered image; the two Linear layers are small
//     gather-GEMMs (ReLU / sigmoid epilogues); scale, residual add and ReLU are one elementwise pass.
// The tail (flatten to [B, T', 512*F'], ASP with the global-context fold, bn2, Linear, bn3) reuses the ECAPA kernels.
#include <stdlib.h>

#include "common.h"
#include "model_common.h"
#include "ptx.cuh"

namespace ppv {

namespace {

constexpr int RS_MAX_BLOCKS = 32;

using Geo = ImageGeo;  // one zero-bordered image grid

struct BlockW {
    GemmWeights conv1, conv2, conv3, down, se1, se2;
    bool has_down = false;
    int inplanes = 0, planes = 0, stride = 1, stage = 0;
};

struct RStep {
    enum Kind { CONV1, GEMM, CONV3, POOL, SCALE_RES, FLATTEN, ASP_GLOBAL, ASP_FUSED } kind;
    Conv3x3Params c3;  // CONV3: 3x3 conv with 32 -> 32 channels (layer1), conv3x3.cu
    GemmParams gp;
    AspFusedParams ap;
    // POOL / SCALE_RES operands
    Planes a, b, c;
    const float* scale = nullptr;
    int C = 0, img_rows = 0;
    float inv_count = 0.f;
    int64_t rows = 0;
};

}  // namespace

struct ResNetSEModel : Model {
    ppv_resnetse_cfg cfg;
    // weights
    float* conv1_w = nullptr;  // [32][9] BN folded
    float* conv1_b = nullptr;  // [32]
    std::vector<BlockW> blocks;
    GemmWeights fold, att1, att2, fc;
    float *att1_bn_scale = nullptr, *att1_bn_shift = nullptr, *bn2_scale = nullptr, *bn2_shift = nullptr;
    int att = 128, cat = 0, Hf = 0;
    // plan
    std::vector<RStep> steps;
    Geo geo[5];  // geo[l] = grid of stage l (1..4); geo[1] is also conv1's
    Planes conv1_out, flat, gstat, pooled, attp, se_mean, se_hid;
    std::vector<Planes> blk_out;  // per block
    float *se_scale = nullptr, *fold_out = nullptr, *pooled_raw = nullptr;
    int Tf = 0;

    explicit ResNetSEModel(const ppv_resnetse_cfg& c) : Model("resnetse", c.precision), cfg(c) {}
    int embd_dim() const override { return cfg.embd_dim; }
    size_t workspace_bytes(int B, int T) const override;

  protected:
    bool prepare_weights(ArenaBuilder& ab) override;
    int build_plan(int B, int T, void* ws, size_t ws_bytes, cudaStream_t st) override;
    int run_steps(const float* feat, cudaStream_t st) override;
    int tap(const std::string& n, float* out, size_t out_elems, cudaStream_t st) override;
};

// ------------------------------------------------------------------------------------------------ small kernels
// conv1: 1 -> C0 channels, 3x3, padding 1, BN folded, ReLU.  One thread per (output position, 8-channel group): the nine
// inputs are read once per thread and each thread stores 16 bytes per plane so that a warp writes whole 128-byte lines of
// consecutive positions.
__global__ void __launch_bounds__(256)
    rs_conv1_kernel(const float* __restrict__ feat, int B, int T, int F, const float* __restrict__ w9, const float* __restrict__ bias, int C0,
                    Planes out, int Hp, int Wp) {
    griddep_launch_dependents();
    // A thread owns one group of 8 output channels for the whole launch (the group count divides the block size): its 72 weights and 8
    // biases live in registers, and it walks the positions with a grid stride.  (Per-position weight reads from shared memory made the
    // kernel LDS-bound: 72 LDS for 72 FMAs.)
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
    PPV_REQUIRE((C0 == 32 || C0 == 64) && out.ld % 8 == 0, "stem conv: C0 must be 32 or 64");
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

// ------------------------------------------------------------------------------------------------ create / load
void ppv_resnetse_default_cfg_impl(ppv_resnetse_cfg* c) {
    c->input_size = 80;
    c->embd_dim = 192;
    const int l[4] = {3, 4, 6, 3}, f[4] = {32, 64, 128, 256};
    for (int i = 0; i < 4; ++i) {
        c->layers[i] = l[i];
        c->num_filters[i] = f[i];
    }
    c->attention_channels = 128;
    c->reduction = 8;
    c->precision = PPV_PREC_BF16X3;
}

int resnetse_create(const ppv_resnetse_cfg* cfg, Model** out) {
    PPV_REQUIRE(cfg && out, "resnetse_create: null argument");
    int nblocks = 0;
    for (int i = 0; i < 4; ++i) {
        if (cfg->layers[i] < 1 || cfg->num_filters[i] % 32 || cfg->num_filters[i] < 32)
            return fail(PPV_EUNSUPPORTED, "resnetse: layers >= 1 and num_filters multiples of 32 required");
        nblocks += cfg->layers[i];
    }
    if (nblocks > RS_MAX_BLOCKS) return fail(PPV_EUNSUPPORTED, "resnetse: too many blocks");
    if (cfg->input_size % 8 || cfg->attention_channels != 128 || cfg->embd_dim % 32 || cfg->reduction < 1)
        return fail(PPV_EUNSUPPORTED, "resnetse: input_size % 8, attention_channels == 128, embd_dim % 32 required");
    for (int i = 0; i < 4; ++i)
        if ((2 * cfg->num_filters[i]) / cfg->reduction > 64 || (2 * cfg->num_filters[i]) % cfg->reduction)
            return fail(PPV_EUNSUPPORTED, "resnetse: SE hidden width must be <= 64");
    if ((2 * cfg->num_filters[3] * (cfg->input_size / 8)) % 128) return fail(PPV_EUNSUPPORTED, "resnetse: pooled channels must be a multiple of 128");
    ResNetSEModel* m = new ResNetSEModel(*cfg);
    m->att = cfg->attention_channels;
    m->Hf = cfg->input_size / 8;
    m->cat = 2 * cfg->num_filters[3] * m->Hf;
    *out = m;
    return PPV_OK;
}

// ------------------------------------------------------------------------------------------------ finalize
bool ResNetSEModel::prepare_weights(ArenaBuilder& ab) {
    ResNetSEModel* const m = this;
    const ppv_resnetse_cfg& cf = m->cfg;
    bool ok = true;
    // conv (+ directly following BN) -> dense [N][taps*Cin] with BN folded; K order = (tap, cin)
    auto conv_bn = [&](GemmWeights* gw, const std::string& conv, const std::string& bn, int N, int Cin, int k) {
        const HostWeight* w = ab.get(conv + ".weight", {N, Cin, k, k});
        const HostWeight* b = ab.get(conv + ".bias", {N});
        std::vector<double> sc, sh;
        if (!w || !b || !ab.bn_affine(bn, N, &sc, &sh)) {
            ok = false;
            return;
        }
        const int taps = k * k;
        std::vector<double> mtx(size_t(N) * taps * Cin);
        std::vector<float> bias(std::max(N, 64), 0.f);
        for (int n = 0; n < N; ++n) {
            for (int t = 0; t < taps; ++t)
                for (int c = 0; c < Cin; ++c) mtx[(size_t(n) * taps + t) * Cin + c] = double(w->v[(size_t(n) * Cin + c) * taps + t]) * sc[n];
            bias[n] = float(double(b->v[n]) * sc[n] + sh[n]);
        }
        ab.put_matrix(gw, mtx, N, taps * Cin);
        ab.put_f32(&gw->bias, bias);
    };
    {  // stem
        const int C0 = cf.num_filters[0];
        const HostWeight* w = ab.get("conv1.weight", {C0, 1, 3, 3});
        const HostWeight* b = ab.get("conv1.bias", {C0});
        std::vector<double> sc, sh;
        if (w && b && ab.bn_affine("bn1", C0, &sc, &sh)) {
            std::vector<float> w9(size_t(C0) * 9), bb(C0);
            for (int c = 0; c < C0; ++c) {
                for (int k = 0; k < 9; ++k) w9[c * 9 + k] = float(double(w->v[c * 9 + k]) * sc[c]);
                bb[c] = float(double(b->v[c]) * sc[c] + sh[c]);
            }
            ab.put_f32(&m->conv1_w, w9);
            ab.put_f32(&m->conv1_b, bb);
        } else {
            ok = false;
        }
    }
    m->blocks.clear();
    m->blocks.reserve(RS_MAX_BLOCKS);  // the arena patches keep pointers into the elements: no reallocation allowed
    int inplanes = cf.num_filters[0];
    for (int li = 1; li <= 4 && ok; ++li) {
        const int planes = cf.num_filters[li - 1], C = 2 * planes, hid = C / cf.reduction;
        for (int bi = 0; bi < cf.layers[li - 1] && ok; ++bi) {
            m->blocks.emplace_back();
            BlockW& bw = m->blocks.back();
            bw.inplanes = inplanes;
            bw.planes = planes;
            bw.stage = li;
            bw.stride = (li > 1 && bi == 0) ? 2 : 1;
            const std::string p = "layer" + std::to_string(li) + "." + std::to_string(bi);
            conv_bn(&bw.conv1, p + ".conv1", p + ".bn1", planes, inplanes, 1);
            conv_bn(&bw.conv2, p + ".conv2", p + ".bn2", planes, planes, 3);
            conv_bn(&bw.conv3, p + ".conv3", p + ".bn3", C, planes, 1);
            bw.has_down = (bi == 0) && (bw.stride != 1 || inplanes != C);
            if (bw.has_down) conv_bn(&bw.down, p + ".downsample.0", p + ".downsample.1", C, inplanes, 1);
            // SE: Linear weights are [in, out] in Paddle (resnet_se.py:52-56); hidden width padded to 64
            const HostWeight *w0 = ab.get(p + ".se.fc.0.weight", {C, hid}), *b0 = ab.get(p + ".se.fc.0.bias", {hid}),
                             *w2 = ab.get(p + ".se.fc.2.weight", {hid, C}), *b2 = ab.get(p + ".se.fc.2.bias", {C});
            if (!w0 || !b0 || !w2 || !b2) {
                ok = false;
                break;
            }
            std::vector<double> m1(size_t(64) * C, 0.0), m2(size_t(C) * 64, 0.0);
            std::vector<float> bias1(64, 0.f);
            for (int j = 0; j < hid; ++j) {
                for (int c = 0; c < C; ++c) m1[size_t(j) * C + c] = w0->v[size_t(c) * hid + j];
                bias1[j] = b0->v[j];
            }
            for (int c = 0; c < C; ++c)
                for (int j = 0; j < hid; ++j) m2[size_t(c) * 64 + j] = w2->v[size_t(j) * C + c];
            ab.put_matrix(&bw.se1, m1, 64, C);
            ab.put_f32(&bw.se1.bias, bias1);
            ab.put_matrix(&bw.se2, m2, C, 64);
            ab.put_f32(&bw.se2.bias, b2->v);
            inplanes = C;
        }
    }
    if (ok) {  // ASP + head
        const int cat = m->cat, A = m->att, E = cf.embd_dim;
        const HostWeight* wt = ab.get("pooling.tdnn.conv.conv.weight", {A, 3 * cat, 1});
        const HostWeight* bt = ab.get("pooling.tdnn.conv.conv.bias", {A});
        const HostWeight* wc = ab.get("pooling.conv.conv.weight", {cat, A, 1});
        const HostWeight* wl = ab.get("linear.weight", {2 * cat, E});
        const HostWeight* bl = ab.get("linear.bias", {E});
        std::vector<double> s_t, h_t, s2, h2, s3, h3;
        ok = wt && bt && wc && wl && bl && ab.bn_affine("pooling.tdnn.norm.norm", A, &s_t, &h_t) && ab.bn_affine("bn2.norm", 2 * cat, &s2, &h2) &&
             ab.bn_affine("bn3.norm", E, &s3, &h3);
        if (ok) {
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
            ab.put_matrix(&m->att1, mx, A, cat);
            ab.put_f32(&m->att1.bias, bt->v);
            ab.put_matrix(&m->fold, mf, A, 2 * cat);
            ab.put_matrix(&m->att2, mc, cat, A);
            ab.put_matrix(&m->fc, ml, E, 2 * cat);
            ab.put_f32(&m->fc.bias, bl2);
            std::vector<float> f1(s_t.begin(), s_t.end()), f2(h_t.begin(), h_t.end()), f3(s2.begin(), s2.end()), f4(h2.begin(), h2.end());
            ab.put_f32(&m->att1_bn_scale, f1);
            ab.put_f32(&m->att1_bn_shift, f2);
            ab.put_f32(&m->bn2_scale, f3);
            ab.put_f32(&m->bn2_shift, f4);
        }
    }
    return ok;
}

// ------------------------------------------------------------------------------------------------ workspace / plan
namespace {

struct RsBuffers {
    Planes conv1_out, flat, gstat, pooled, attp, se_mean, se_hid;
    std::vector<Planes> out1, out2, out3, res, blk_out;
    float *se_scale, *fold_out, *pooled_raw, *emb_out;
};

void rs_geometry(const ResNetSEModel* m, int T, Geo* geo) {
    int H = m->cfg.input_size, W = T;
    for (int l = 1; l <= 4; ++l) {
        if (l > 1) {
            H = (H - 1) / 2 + 1;
            W = (W - 1) / 2 + 1;
        }
        geo[l].H = H;
        geo[l].W = W;
        geo[l].Hp = H + 2;
        geo[l].Wp = W + 2;
    }
}

void rs_carve(const ResNetSEModel* m, WsCarver& cv, int B, int T, Geo* geo, RsBuffers* rb) {
    rs_geometry(m, T, geo);
    rb->conv1_out = cv.planes(geo[1].rows(B), m->cfg.num_filters[0]);
    const size_t nb = m->blocks.size();
    rb->out1.resize(nb);
    rb->out2.resize(nb);
    rb->out3.resize(nb);
    rb->res.resize(nb);
    rb->blk_out.resize(nb);
    int maxC = 0;
    // Buffer liveness (round 2; every buffer used to be dedicated: 38 GB at batch 256).  One set of image buffers per STAGE: conv1 / conv2 /
    // conv3 outputs are dead once the block's SE pass has run, and the block output overwrites its own residual input in place
    // (out = s * z + res is elementwise).  The first block of a stage runs conv1 on the PREVIOUS stage's grid: that output aliases
    // the previous stage's conv3 buffer (same grid, same channel count, dead by then).  Zero borders survive because epilogues only
    // ever store interior positions and a buffer never changes its grid.
    Planes s_out1[5], s_out2[5], s_out3[5], s_act[5];
    for (size_t i = 0; i < nb; ++i) {
        const BlockW& bw = m->blocks[i];
        const int st = bw.stage;
        const Geo& gin = geo[bw.stride == 2 ? st - 1 : st];
        const Geo& gout = geo[st];
        if (!s_act[st].base && s_act[st].rows == 0) {  // first block of the stage: carve the stage's set
            s_out1[st] = cv.planes(gout.rows(B), bw.planes);
            s_out2[st] = cv.planes(gout.rows(B), bw.planes);
            s_out3[st] = cv.planes(gout.rows(B), 2 * bw.planes);
            s_act[st] = cv.planes(gout.rows(B), 2 * bw.planes);
        }
        if (bw.stride == 2) {
            const bool can_alias = st > 1 && s_out3[st - 1].rows > 0 && s_out3[st - 1].ld == bw.planes;
            rb->out1[i] = can_alias ? s_out3[st - 1] : cv.planes(gin.rows(B), bw.planes);
        } else {
            rb->out1[i] = s_out1[st];
        }
        rb->out2[i] = s_out2[st];
        rb->out3[i] = s_out3[st];
        if (bw.has_down) rb->res[i] = s_act[st];
        rb->blk_out[i] = s_act[st];
        maxC = std::max(maxC, 2 * bw.planes);
    }
    const int Tf = geo[4].W;
    rb->flat = cv.planes(int64_t(B) * Tf, m->cat);
    rb->gstat = cv.planes(B, 2 * m->cat);
    rb->pooled = cv.planes(B, 2 * m->cat);
    rb->attp = cv.planes(int64_t(B) * Tf, m->att);
    rb->se_mean = cv.planes(B, maxC);
    rb->se_hid = cv.planes(B, 64);
    rb->se_scale = static_cast<float*>(cv.take(size_t(B) * maxC * 4));
    rb->fold_out = static_cast<float*>(cv.take(mc_align_up(size_t(B), 128) * m->att * 4));
    rb->pooled_raw = static_cast<float*>(cv.take(size_t(B) * 2 * m->cat * 4));
    rb->emb_out = static_cast<float*>(cv.take(mc_align_up(size_t(B), 128) * m->cfg.embd_dim * 4));
}

}  // namespace

size_t ResNetSEModel::workspace_bytes(int B, int T) const {
    if (!finalized || B <= 0 || T <= 0) return 0;
    WsCarver cv;
    Geo g[5];
    RsBuffers rb;
    rs_carve(this, cv, B, T, g, &rb);
    return mc_align_up(cv.off, 256);
}

int ResNetSEModel::build_plan(int B, int T, void* ws, size_t ws_bytes, cudaStream_t st) {
    ResNetSEModel* const m = this;
    const size_t need = workspace_bytes(B, T);
    PPV_REQUIRE(ws && ws_bytes >= need, "resnetse: workspace too small (see ppv_model_workspace_bytes)");
    PPV_REQUIRE((reinterpret_cast<uintptr_t>(ws) & 255) == 0, "resnetse: workspace must be 256-byte aligned");
    PPV_REQUIRE(T >= 8, "resnetse: too few frames");
    WsCarver cv;
    cv.base = static_cast<uint8_t*>(ws);
    RsBuffers rb;
    rs_carve(m, cv, B, T, m->geo, &rb);
    PPV_REQUIRE(int64_t(m->geo[1].Hp) * m->geo[1].Wp * B < (int64_t(1) << 31), "resnetse: batch too large for 32-bit row indices");
    PPV_CUDA_OK(cudaMemsetAsync(ws, 0, need, st));  // zero borders
    m->steps.clear();

    auto img_epi = [&](const Planes& out, const Geo& gin, const Geo& gout, int stride, bool relu) {
        Epilogue ep;
        ep.out_mode = OUT_PLANES;
        ep.out = out.base;
        ep.out_ld = out.ld;
        ep.out_plane_stride = out.plane_stride;
        ep.relu = relu ? 1 : 0;
        ep.img_Hp = gin.Hp;
        ep.img_Wp = gin.Wp;
        ep.img_H = gin.H;
        ep.img_W = gin.W;
        ep.img_stride = stride;
        ep.out_Hp = gout.Hp;
        ep.out_Wp = gout.Wp;
        return ep;
    };
    auto add_gemm = [&](const GemmWeights& gw, const std::vector<GemmSource>& srcs, int M, Epilogue ep, int n_gemm) -> int {
        ep.bias = gw.bias;
        RStep s;
        s.kind = RStep::GEMM;
        int rc = gemm_build(&s.gp, srcs.data(), int(srcs.size()), gw.W, M, n_gemm, ep, gemm_pick_bn(n_gemm));
        if (rc) return rc;
        m->steps.push_back(s);
        return PPV_OK;
    };
    auto plain_planes = [&](const Planes& p, bool relu) {
        Epilogue ep;
        ep.out_mode = OUT_PLANES;
        ep.out = p.base;
        ep.out_ld = p.ld;
        ep.out_plane_stride = p.plane_stride;
        ep.relu = relu ? 1 : 0;
        return ep;
    };

    {
        RStep s;
        s.kind = RStep::CONV1;
        m->steps.push_back(s);
    }
    Planes x = rb.conv1_out;
    int rc;
    const char* c3env = getenv("PPV_CONV3X3");  // 0 = 3x3 convs through the generic gather-GEMM (debugging / A-B timing)
    const bool use_c3 = !(c3env && c3env[0] == '0');
    for (size_t i = 0; i < m->blocks.size(); ++i) {
        const BlockW& bw = m->blocks[i];
        const Geo& gin = m->geo[bw.stride == 2 ? bw.stage - 1 : bw.stage];
        const Geo& gout = m->geo[bw.stage];
        const int Min = int(gin.rows(B)), Mout = int(gout.rows(B)), C = 2 * bw.planes, p = bw.planes;
        // conv1 1x1 + BN + ReLU on the input grid
        rc = add_gemm(bw.conv1, {GemmSource{x, 0, bw.inplanes, 0}}, Min, img_epi(rb.out1[i], gin, gin, 1, true), std::max(p, 32));
        if (rc) return rc;
        // conv2 3x3 (stride) + BN + ReLU: 9 taps on the input grid, stored on the output grid
        if (use_c3 && p == 32 && conv3x3_c32_supported(p, p, gin.H, gin.W)) {  // weight-stationary patch kernel (conv3x3.cu)
            Epilogue ep = img_epi(rb.out2[i], gin, gout, bw.stride, true);
            ep.bias = bw.conv2.bias;
            RStep s3;
            s3.kind = RStep::CONV3;
            rc = conv3x3_build(&s3.c3, rb.out1[i], 0, bw.conv2.W, B, gin.H, gin.W, gin.Hp, gin.Wp, ep);
            if (rc) return rc;
            m->steps.push_back(s3);
        } else {
            std::vector<GemmSource> taps;
            for (int dh = -1; dh <= 1; ++dh)
                for (int dw = -1; dw <= 1; ++dw) taps.push_back(GemmSource{rb.out1[i], 0, p, dh * gin.Wp + dw});
            rc = add_gemm(bw.conv2, taps, Min, img_epi(rb.out2[i], gin, gout, bw.stride, true), std::max(p, 32));
            if (rc) return rc;
        }
        // conv3 1x1 + BN
        rc = add_gemm(bw.conv3, {GemmSource{rb.out2[i], 0, p, 0}}, Mout, img_epi(rb.out3[i], gout, gout, 1, false), C);
        if (rc) return rc;
        // shortcut
        Planes res = x;
        if (bw.has_down) {
            rc = add_gemm(bw.down, {GemmSource{x, 0, bw.inplanes, 0}}, Min, img_epi(rb.res[i], gin, gout, bw.stride, false), C);
            if (rc) return rc;
            res = rb.res[i];
        }
        // SE: pool -> fc -> fc -> scale
        RStep sp;
        sp.kind = RStep::POOL;
        sp.a = rb.out3[i];
        sp.b = rb.se_mean;
        sp.b.ld = C;  // view with the block's channel count
        sp.b.plane_stride = rb.se_mean.plane_stride;
        sp.C = C;
        sp.img_rows = gout.Hp * gout.Wp;
        sp.inv_count = 1.f / float(gout.H * gout.W);
        m->steps.push_back(sp);
        Planes mean_view = rb.se_mean;
        mean_view.ld = C;
        {
            Epilogue e1 = plain_planes(rb.se_hid, true);
            rc = add_gemm(bw.se1, {GemmSource{mean_view, 0, C, 0}}, B, e1, 64);
            if (rc) return rc;
            Epilogue e2;
            e2.out_mode = OUT_F32;
            e2.out = rb.se_scale;
            e2.out_ld = C;
            e2.sigmoid_ = 1;
            rc = add_gemm(bw.se2, {GemmSource{rb.se_hid, 0, 64, 0}}, B, e2, C);
            if (rc) return rc;
        }
        RStep sr;
        sr.kind = RStep::SCALE_RES;
        sr.a = rb.out3[i];
        sr.b = res;
        sr.c = rb.blk_out[i];
        sr.scale = rb.se_scale;
        sr.C = C;
        sr.img_rows = gout.Hp * gout.Wp;
        sr.rows = gout.rows(B);
        m->steps.push_back(sr);
        x = rb.blk_out[i];
    }
    // tail: flatten, ASP, bn2, linear, bn3
    const Geo& g4 = m->geo[4];
    const int Tf = g4.W, cat = m->cat;
    {
        RStep s;
        s.kind = RStep::FLATTEN;
        s.a = x;
        s.c = rb.flat;
        m->steps.push_back(s);
        s.kind = RStep::ASP_GLOBAL;
        m->steps.push_back(s);
    }
    {
        Epilogue ep;
        ep.out_mode = OUT_F32;
        ep.out = rb.fold_out;
        ep.out_ld = m->att;
        GemmWeights gw = m->fold;
        gw.bias = nullptr;
        rc = add_gemm(gw, {GemmSource{rb.gstat, 0, 2 * cat, 0}}, B, ep, m->att);
        if (rc) return rc;
    }
    {
        Epilogue ep = plain_planes(rb.attp, true);
        ep.Tp = Tf;
        ep.P = 0;
        ep.T = Tf;
        ep.rowgrp_bias = rb.fold_out;
        ep.bn_scale = m->att1_bn_scale;
        ep.bn_shift = m->att1_bn_shift;
        ep.tanh_ = 1;
        rc = add_gemm(m->att1, {GemmSource{rb.flat, 0, cat, 0}}, B * Tf, ep, m->att);
        if (rc) return rc;
    }
    {
        RStep s;
        s.kind = RStep::ASP_FUSED;
        rc = asp_fused_build(&s.ap, m->att2.W, rb.attp, rb.flat, rb.gstat, m->bn2_scale, m->bn2_shift, rb.pooled, rb.pooled_raw, B, Tf, 0, Tf, cat,
                             m->att, 1e-12f);
        if (rc) return rc;
        m->steps.push_back(s);
    }
    {
        Epilogue ep;
        ep.out_mode = OUT_F32;
        ep.out = rb.emb_out;
        ep.out_ld = m->cfg.embd_dim;
        rc = add_gemm(m->fc, {GemmSource{rb.pooled, 0, 2 * cat, 0}}, B, ep, m->cfg.embd_dim);
        if (rc) return rc;
    }
    m->conv1_out = rb.conv1_out;
    m->flat = rb.flat;
    m->gstat = rb.gstat;
    m->pooled = rb.pooled;
    m->attp = rb.attp;
    m->se_mean = rb.se_mean;
    m->se_hid = rb.se_hid;
    m->blk_out = rb.blk_out;
    m->se_scale = rb.se_scale;
    m->fold_out = rb.fold_out;
    m->pooled_raw = rb.pooled_raw;
    m->emb_out = rb.emb_out;
    m->Tf = Tf;
    return PPV_OK;
}

// ------------------------------------------------------------------------------------------------ forward
int ResNetSEModel::run_steps(const float* feat, cudaStream_t st) {
    ResNetSEModel* const m = this;
    const int B = m->plan_B, T = m->plan_T, F = m->cfg.input_size, cat = m->cat;
    int rc = PPV_OK;
    for (const RStep& s : m->steps) {
        switch (s.kind) {
            case RStep::CONV1: {
                const int64_t total = int64_t(B) * F * T;
                PPV_PDL_OK(launch_pdl(rs_conv1_kernel, dim3(unsigned((total + 7) / 8)), dim3(256), 0, st, feat, B, T, F, (const float*)m->conv1_w,
                                      (const float*)m->conv1_b, m->cfg.num_filters[0], m->conv1_out, m->geo[1].Hp, m->geo[1].Wp),
                           "rs_conv1_kernel");
                break;
            }
            case RStep::GEMM: rc = gemm_launch(s.gp, m->precision, m->num_sms, st); break;
            case RStep::CONV3: rc = conv3x3_launch(s.c3, m->precision, m->num_sms, st); break;
            case RStep::POOL:
                rc = launch_colstats(s.a, 0, s.C, B, s.img_rows, 0, s.img_rows, 0, 0.f, nullptr, s.b, st, s.inv_count);
                break;
            case RStep::SCALE_RES:
                rc = launch_se_scale_res(s.a, s.scale, s.b, 0, s.c, 0, s.C, s.img_rows, s.rows, m->num_sms, st, 1);
                break;
            case RStep::FLATTEN: {
                const Geo& g4 = m->geo[4];
                const int64_t total = int64_t(B) * g4.W * cat;
                const int grid = int(std::min<int64_t>((total + 255) / 256, int64_t(m->num_sms) * 16));
                PPV_PDL_OK(launch_pdl(rs_flatten_kernel, dim3(grid), dim3(256), 0, st, s.a, B, g4.H, g4.W, g4.Hp, g4.Wp, 2 * m->cfg.num_filters[3], s.c),
                           "rs_flatten_kernel");
                break;
            }
            case RStep::ASP_GLOBAL: rc = launch_colstats(m->flat, 0, cat, B, m->Tf, 0, m->Tf, 1, 1e-12f, nullptr, m->gstat, st); break;
            case RStep::ASP_FUSED: rc = asp_fused_launch(s.ap, m->precision, m->num_sms, st); break;
        }
        if (rc) return rc;
    }
    return PPV_OK;
}

// taps: "conv1", "layer1".."layer4" -> fp32 [B,H,W,C]; "flat" -> [B,T',cat]; "asp" -> [B, 2*cat]
int ResNetSEModel::tap(const std::string& n, float* out, size_t out_elems, cudaStream_t st) {
    ResNetSEModel* const m = this;
    const int B = m->plan_B;
    if (n == "asp") {
        PPV_REQUIRE(out_elems >= size_t(B) * 2 * m->cat, "resnetse_read_tap: output too small");
        PPV_CUDA_OK(cudaMemcpyAsync(out, m->pooled_raw, size_t(B) * 2 * m->cat * 4, cudaMemcpyDeviceToDevice, st));
        return PPV_OK;
    }
    if (n == "flat") {
        PPV_REQUIRE(out_elems >= size_t(B) * m->Tf * m->cat, "resnetse_read_tap: output too small");
        return launch_planes_to_f32(m->flat, 0, m->cat, B, m->Tf, 0, m->Tf, out, st);
    }
    Planes src;
    int stage = 0, C = 0;
    if (n == "conv1") {
        src = m->conv1_out;
        stage = 1;
        C = m->cfg.num_filters[0];
    } else if (n.rfind("layer", 0) == 0 && n.size() == 6 && n[5] >= '1' && n[5] <= '4') {
        stage = n[5] - '0';
        int last = -1;
        for (size_t i = 0; i < m->blocks.size(); ++i)
            if (m->blocks[i].stage == stage) last = int(i);
        src = m->blk_out[last];
        C = 2 * m->cfg.num_filters[stage - 1];
    } else {
        return fail(PPV_EINVAL, "resnetse_read_tap: unknown tap " + n);
    }
    const Geo& g = m->geo[stage];
    const int64_t total = int64_t(B) * g.H * g.W * C;
    PPV_REQUIRE(out_elems >= size_t(total), "resnetse_read_tap: output too small");
    rs_image_to_f32_kernel<<<int(std::min<int64_t>((total + 255) / 256, 132 * 32)), 256, 0, st>>>(src, B, g.H, g.W, g.Hp, g.Wp, C, out);
    PPV_LAUNCH_OK("rs_image_to_f32_kernel");
    return PPV_OK;
}

}  // namespace ppv
