// ResNetSE forward as a plan of tensor-core gather-GEMMs over zero-bordered NHWC images.
// Reference graph: ppvector/models/resnet_se.py:121-139 (ResNetSE.forward), :24-45 (SEBottleneck.forward),
// :59-63 (SELayer.forward), :107-119 (_make_layer: 1x1 strided conv + BN shortcut), ppvector/models/pooling.py:86-125
// (ASP, shared with ECAPA-TDNN).  Eval mode.
//
// Image layout and conv planning: image_plan.h.  What is specific here:
//   * every conv runs on the gather-GEMM or the patch kernel, none on the pointwise kernel;
//   * SE: global average pool = column sums over the whole zero-bordered image; the two Linear layers are small
//     gather-GEMMs (ReLU / sigmoid epilogues); scale, residual add and ReLU are one elementwise pass.
// The tail (flatten to [B, T', 512*F'], ASP with the global-context fold, bn2, Linear, bn3) reuses the ECAPA kernels.
#include "common.h"
#include "image_plan.h"
#include "model_common.h"

namespace ppv {

namespace {

constexpr int RS_MAX_BLOCKS = 32;

using Geo = ImageGeo;  // one zero-bordered image grid

struct BlockW {
    GemmWeights conv1, conv2, conv3, down, se1, se2;
    bool has_down = false;
    int inplanes = 0, planes = 0, stride = 1, stage = 0;
};

}  // namespace

struct ResNetSEModel : PlanModel {
    ppv_resnetse_cfg cfg;
    // weights
    float* conv1_w = nullptr;  // [32][9] BN folded
    float* conv1_b = nullptr;  // [32]
    std::vector<BlockW> blocks;
    GemmWeights fold, att1, att2, fc;
    float *att1_bn_scale = nullptr, *att1_bn_shift = nullptr, *bn2_scale = nullptr, *bn2_shift = nullptr;
    int att = 128, cat = 0, Hf = 0;
    // plan (what the taps read)
    Geo geo[5];  // geo[l] = grid of stage l (1..4); geo[1] is also conv1's
    Planes conv1_out, flat, stage_out[5];
    float* pooled_raw = nullptr;

    explicit ResNetSEModel(const ppv_resnetse_cfg& c) : PlanModel("resnetse", c.precision), cfg(c) {}
    int embd_dim() const override { return cfg.embd_dim; }
    size_t workspace_bytes(int B, int T) const override;

  protected:
    bool prepare_weights(ArenaBuilder& ab) override;
    int build_plan(int B, int T, void* ws, size_t ws_bytes, cudaStream_t st) override;
    int tap(const std::string& n, float* out, size_t out_elems, cudaStream_t st) override;
};

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
    bool ok = ab.fold_stem(&m->conv1_w, &m->conv1_b, "conv1", "bn1", cf.num_filters[0]);
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
            ok &= ab.fold_conv(&bw.conv1, p + ".conv1", p + ".bn1", planes, inplanes, 1, 2);
            ok &= ab.fold_conv(&bw.conv2, p + ".conv2", p + ".bn2", planes, planes, 3, 2);
            ok &= ab.fold_conv(&bw.conv3, p + ".conv3", p + ".bn3", C, planes, 1, 2);
            bw.has_down = (bi == 0) && (bw.stride != 1 || inplanes != C);
            if (bw.has_down) ok &= ab.fold_conv(&bw.down, p + ".downsample.0", p + ".downsample.1", C, inplanes, 1, 2);
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
        std::vector<double> s3, h3;
        ok = wt && bt && wc && wl && bl && ab.put_bn(&m->att1_bn_scale, &m->att1_bn_shift, "pooling.tdnn.norm.norm", A, A) &&
             ab.put_bn(&m->bn2_scale, &m->bn2_shift, "bn2.norm", 2 * cat, 2 * cat) && ab.bn_affine("bn3.norm", E, &s3, &h3);
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

void rs_carve(const ResNetSEModel* m, WsCarver& cv, int B, int T, Geo* geo, RsBuffers* rb) {
    image_pyramid(geo + 1, 4, m->cfg.input_size, T, true);
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
    PPV_REQUIRE(T >= 8, "resnetse: too few frames");
    image_pyramid(m->geo + 1, 4, m->cfg.input_size, T, true);
    PPV_REQUIRE(m->geo[1].rows(B) < (int64_t(1) << 31), "resnetse: batch too large for 32-bit row indices");
    int rc = claim_workspace(B, T, ws, ws_bytes, st);
    if (rc) return rc;
    WsCarver cv;
    cv.base = static_cast<uint8_t*>(ws);
    RsBuffers rb;
    rs_carve(m, cv, B, T, m->geo, &rb);
    m->steps.clear();

    auto plain_planes = [&](const Planes& p, bool relu) {
        Epilogue ep = planes_epilogue(p);
        ep.relu = relu ? 1 : 0;
        return ep;
    };
    auto img_relu = [](Epilogue ep) {
        ep.relu = 1;
        return ep;
    };

    m->steps.push_back(stem_step(m->conv1_w, m->conv1_b, m->cfg.num_filters[0], rb.conv1_out, m->geo[1], B));
    Planes x = rb.conv1_out;
    for (size_t i = 0; i < m->blocks.size(); ++i) {
        const BlockW& bw = m->blocks[i];
        const Geo& gin = m->geo[bw.stride == 2 ? bw.stage - 1 : bw.stage];
        const Geo& gout = m->geo[bw.stage];
        const int Min = int(gin.rows(B)), Mout = int(gout.rows(B)), C = 2 * bw.planes, p = bw.planes;
        // conv1 1x1 + BN + ReLU on the input grid
        rc = plan_gemm(bw.conv1, {GemmSource{x, 0, bw.inplanes, 0}}, Min, img_relu(image_epilogue(rb.out1[i], gin, gin, 1, 1)));
        if (rc) return rc;
        // conv2 3x3 (stride) + BN + ReLU on the input grid, stored on the output grid
        rc = plan_conv3x3(bw.conv2, rb.out1[i], 0, p, gin, B, img_relu(image_epilogue(rb.out2[i], gin, gout, bw.stride, bw.stride)));
        if (rc) return rc;
        // conv3 1x1 + BN
        rc = plan_gemm(bw.conv3, {GemmSource{rb.out2[i], 0, p, 0}}, Mout, image_epilogue(rb.out3[i], gout, gout, 1, 1));
        if (rc) return rc;
        // shortcut
        Planes res = x;
        if (bw.has_down) {
            rc = plan_gemm(bw.down, {GemmSource{x, 0, bw.inplanes, 0}}, Min, image_epilogue(rb.res[i], gin, gout, bw.stride, bw.stride));
            if (rc) return rc;
            res = rb.res[i];
        }
        // SE: pool -> fc -> fc -> scale
        Planes mean_view = rb.se_mean;  // view with the block's channel count
        mean_view.ld = C;
        const int img_rows = gout.Hp * gout.Wp;
        m->steps.push_back(colstats_step(rb.out3[i], C, B, img_rows, 0, img_rows, 0, 0.f, mean_view, 1.f / float(gout.H * gout.W)));
        rc = plan_gemm(bw.se1, {GemmSource{mean_view, 0, C, 0}}, B, plain_planes(rb.se_hid, true));
        if (rc) return rc;
        Epilogue e2;
        e2.out_mode = OUT_F32;
        e2.out = rb.se_scale;
        e2.out_ld = C;
        e2.sigmoid_ = 1;
        rc = plan_gemm(bw.se2, {GemmSource{rb.se_hid, 0, 64, 0}}, B, e2);
        if (rc) return rc;
        m->steps.push_back(scale_res_step(rb.out3[i], rb.se_scale, res, 0, rb.blk_out[i], 0, C, gout.Hp * gout.Wp, gout.rows(B), true));
        x = rb.blk_out[i];
        m->stage_out[bw.stage] = x;
    }
    // tail: flatten, ASP, bn2, linear, bn3
    const Geo& g4 = m->geo[4];
    const int Tf = g4.W, cat = m->cat;
    m->steps.push_back(flatten_step(x, g4, B, 2 * m->cfg.num_filters[3], rb.flat));
    m->steps.push_back(colstats_step(rb.flat, cat, B, Tf, 0, Tf, 1, 1e-12f, rb.gstat));
    {
        Epilogue ep;
        ep.out_mode = OUT_F32;
        ep.out = rb.fold_out;
        ep.out_ld = m->att;
        rc = plan_gemm(m->fold, {GemmSource{rb.gstat, 0, 2 * cat, 0}}, B, ep);
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
        rc = plan_gemm(m->att1, {GemmSource{rb.flat, 0, cat, 0}}, B * Tf, ep);
        if (rc) return rc;
    }
    {
        PlanStep s;
        s.kind = PlanStep::ASP_FUSED;
        rc = asp_fused_build(&s.ap, m->att2.W, rb.attp, rb.flat, m->bn2_scale, m->bn2_shift, rb.pooled, rb.pooled_raw, B, Tf, 0, Tf, cat,
                             m->att, 1e-12f);
        if (rc) return rc;
        m->steps.push_back(s);
    }
    {
        Epilogue ep;
        ep.out_mode = OUT_F32;
        ep.out = rb.emb_out;
        ep.out_ld = m->cfg.embd_dim;
        rc = plan_gemm(m->fc, {GemmSource{rb.pooled, 0, 2 * cat, 0}}, B, ep);
        if (rc) return rc;
    }
    m->conv1_out = rb.conv1_out;
    m->flat = rb.flat;
    m->pooled_raw = rb.pooled_raw;
    m->emb_out = rb.emb_out;
    return PPV_OK;
}

// taps: "conv1", "layer1".."layer4" -> fp32 [B,H,W,C]; "flat" -> [B,T',cat]; "asp" -> [B, 2*cat]
int ResNetSEModel::tap(const std::string& n, float* out, size_t out_elems, cudaStream_t st) {
    ResNetSEModel* const m = this;
    const int B = m->plan_B, Tf = m->geo[4].W;
    if (n == "asp") {
        PPV_REQUIRE(out_elems >= size_t(B) * 2 * m->cat, "resnetse_read_tap: output too small");
        PPV_CUDA_OK(cudaMemcpyAsync(out, m->pooled_raw, size_t(B) * 2 * m->cat * 4, cudaMemcpyDeviceToDevice, st));
        return PPV_OK;
    }
    if (n == "flat") {
        PPV_REQUIRE(out_elems >= size_t(B) * Tf * m->cat, "resnetse_read_tap: output too small");
        return launch_planes_to_f32(m->flat, 0, m->cat, B, Tf, 0, Tf, out, st);
    }
    if (n == "conv1") return image_tap(m->conv1_out, m->geo[1], m->cfg.num_filters[0], out, out_elems, st);
    if (const int stage = name_index(n, "layer", 1, 4)) return image_tap(m->stage_out[stage], m->geo[stage], 2 * m->cfg.num_filters[stage - 1], out, out_elems, st);
    return fail(PPV_EINVAL, "resnetse_read_tap: unknown tap " + n);
}

}  // namespace ppv
