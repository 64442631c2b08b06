// ERes2Net forward as a plan of tensor-core gather-GEMMs over zero-bordered NHWC images.
// Reference graph: ppvector/models/eres2net.py:239-263 (ERes2Net.forward), :85-108 (BasicBlockERes2Net.forward),
// :147-170 (BasicBlockERes2Net_diff_AFF.forward), :46-52 (AFF.forward), :12-19 (clipped ReLU = Hardtanh(0,20)),
// ppvector/models/pooling.py:138-146 (TSTP).  Eval mode, default configuration of configs/eres2net.yml
// (scale 2, expansion 2, base_width 32, one embedding layer).
//
// Image layout and conv planning: image_plan.h.  What is specific here:
//   * Res2Net split of scale 2: `sp + spx[1]` is two K-sources of the second 3x3 conv (conv is linear); `split` and
//     `concat` are column windows of the conv1 output / K-sources of conv3;
//   * layer1 works on 16-channel halves: the GEMM reads the whole 32-channel row and the weights of the other half are
//     zero (k-steps are 32 wide), outputs are padded to 32 columns of which 16 are zero;
//   * AFF (attentional feature fusion): concat -> 1x1 conv + BN + SiLU -> 1x1 conv + BN -> tanh are two small GEMMs
//     (two K-sources, SiLU / tanh epilogues), the blend x(1+t) + y(1-t) is one elementwise pass;
//   * TSTP = column mean and sqrt(unbiased variance + 1e-8) over time of the flattened [B, T', 512*F'] matrix.
#include "common.h"
#include "image_plan.h"
#include "model_common.h"

namespace ppv {

namespace {

constexpr int ER_MAX_BLOCKS = 32;
constexpr float ER_RELU_MAX = 20.f;

struct EBlockW {
    GemmWeights conv1, sc, conv_a, conv_b, conv3, aff_a, aff_b;
    bool has_sc = false, fuse = false;
    int in_planes = 0, planes = 0, width = 0, wpad = 0, stride = 1, stage = 0;
    // column plan of the conv1 output: chunk 0 at column 0, chunk 1 at column `c1_chunk1`; `c1_cols` columns in all.  Width 16 (ERes2Net
    // layer 1) packs both chunks into one 32-column window; every other width gives each chunk its own `wpad`-column window (zero padded:
    // ERes2NetV2's widths are 13 / 26 / 52 / 104).
    int c1_chunk1 = 0, c1_cols = 0;
    bool packed = false;
};
struct EFuseW {  // layerN_downsample + fuse_modeXYZ
    GemmWeights ds, aff_a, aff_b;
    int C = 0;  // channels of the finer stage output
};

}  // namespace

struct ERes2NetModel : PlanModel {
    ppv_eres2net_cfg cfg;
    float *stem_w = nullptr, *stem_b = nullptr;
    std::vector<EBlockW> blocks;
    EFuseW fuse[3];
    GemmWeights seg1;
    int fuse_first = 0;  // first bottom-up fusion stage in use (0: ERes2Net, 2: ERes2NetV2)
    int stats_ch = 0;  // 512 * F'
    // plan (what the taps read)
    ImageGeo geo[5];
    Planes stats, stage_out[5], fuse_out[3];

    explicit ERes2NetModel(const ppv_eres2net_cfg& c) : PlanModel("eres2net", c.precision), cfg(c) {}
    int embd_dim() const override { return cfg.embd_dim; }
    int input_size() const override { return cfg.input_size; }
    size_t workspace_bytes(int B, int T) const override;

  protected:
    bool prepare_weights(ArenaBuilder& ab) override;
    int build_plan(int B, int T, void* ws, size_t ws_bytes, cudaStream_t st) override;
    int tap(const std::string& n, float* out, size_t out_elems, cudaStream_t st) override;
};

void ppv_eres2net_default_cfg_impl(ppv_eres2net_cfg* c) {
    c->input_size = 80;
    c->embd_dim = 192;
    const int nb[4] = {3, 4, 6, 3};
    for (int i = 0; i < 4; ++i) c->num_blocks[i] = nb[i];
    c->m_channels = 32;
    c->precision = PPV_PREC_BF16X3;
    c->version = 1;
    c->base_width = 32;
}

int eres2net_create(const ppv_eres2net_cfg* cfg, Model** out) {
    PPV_REQUIRE(cfg && out, "eres2net_create: null argument");
    int nblocks = 0;
    for (int i = 0; i < 4; ++i) {
        if (cfg->num_blocks[i] < 1) return fail(PPV_EUNSUPPORTED, "eres2net: num_blocks >= 1 required");
        nblocks += cfg->num_blocks[i];
    }
    if (nblocks > ER_MAX_BLOCKS) return fail(PPV_EUNSUPPORTED, "eres2net: too many blocks");
    if (cfg->m_channels != 32 && cfg->m_channels != 64) return fail(PPV_EUNSUPPORTED, "eres2net: m_channels must be 32 or 64");
    if (cfg->input_size % 8 || cfg->embd_dim % 32) return fail(PPV_EUNSUPPORTED, "eres2net: input_size % 8, embd_dim % 32 required");
    if (cfg->version != 0 && cfg->version != 1 && cfg->version != 2) return fail(PPV_EUNSUPPORTED, "eres2net: version must be 1 (ERes2Net) or 2 (ERes2NetV2)");
    if (cfg->version != 2 && cfg->base_width != 0 && cfg->base_width != 32) return fail(PPV_EUNSUPPORTED, "eres2net: ERes2Net is built for base_width 32");
    if (cfg->version == 2 && cfg->base_width != 0 && (cfg->base_width < 8 || cfg->base_width > 32)) return fail(PPV_EUNSUPPORTED, "eres2net: ERes2NetV2 base_width must be in [8, 32]");
    ERes2NetModel* m = new ERes2NetModel(*cfg);
    m->stats_ch = (cfg->input_size / 8) * cfg->m_channels * 16;
    *out = m;
    return PPV_OK;
}

// ------------------------------------------------------------------------------------------------ finalize
bool ERes2NetModel::prepare_weights(ArenaBuilder& ab) {
    ERes2NetModel* const m = this;
    const ppv_eres2net_cfg& cf = m->cfg;
    auto aff_weights = [&](GemmWeights* ga, GemmWeights* gb, const std::string& p, int C, int src_cols) {
        // local_att.0: conv(2C -> C/4) over concat(x, y): two K groups of src_cols columns with C real channels each
        const int inter = C / 4, ipad = std::max((inter + 31) / 32 * 32, 32);
        const bool ok_a = ab.fold_conv(ga, p + ".local_att.0", p + ".local_att.1", inter, 2 * C, 1, 2, ipad, {{1, src_cols, 0, C, 0}, {1, src_cols, 0, C, C}});
        return ab.fold_conv(gb, p + ".local_att.3", p + ".local_att.4", C, inter, 1, 2, (C + 31) / 32 * 32, {{1, ipad, 0, inter, 0}}) && ok_a;
    };
    bool ok = ab.fold_stem(&m->stem_w, &m->stem_b, "conv1", "bn1", cf.m_channels);
    m->blocks.clear();
    m->blocks.reserve(ER_MAX_BLOCKS);  // arena patches point into the elements
    int in_planes = cf.m_channels;
    const bool v2 = cf.version == 2;
    const int base_width = v2 ? (cf.base_width > 0 ? cf.base_width : 26) : 32;
    for (int li = 1; li <= 4 && ok; ++li) {
        const int planes = cf.m_channels << (li - 1), width = planes * base_width / 64, wpad = std::max((width + 31) / 32 * 32, 32), C = 2 * planes;
        for (int bi = 0; bi < cf.num_blocks[li - 1] && ok; ++bi) {
            m->blocks.emplace_back();
            EBlockW& bw = m->blocks.back();
            bw.in_planes = in_planes;
            bw.planes = planes;
            bw.width = width;
            bw.wpad = wpad;
            bw.stage = li;
            bw.stride = (li > 1 && bi == 0) ? 2 : 1;
            bw.fuse = li >= 3;
            bw.packed = (width == 16);
            bw.c1_chunk1 = bw.packed ? width : wpad;
            bw.c1_cols = bw.packed ? 32 : 2 * wpad;
            const std::string p = "layer" + std::to_string(li) + "." + std::to_string(bi);
            ok &= ab.fold_conv(&bw.conv1, p + ".conv1", p + ".bn1", 2 * width, in_planes, 1, 2, bw.c1_cols, {}, width, bw.c1_chunk1);
            // first 3x3: reads chunk 0 of the conv1 output (for width 16 the 32-wide window with the upper half zero-weighted)
            ok &= ab.fold_conv(&bw.conv_a, p + ".convs.0", p + ".bns.0", width, width, 3, 2, wpad, {{9, wpad, 0, width, 0}});
            if (!bw.fuse) {
                // second 3x3 on sp + spx[1]: K sources (sp buffer, conv1-output window holding chunk 1)
                const int pos1 = bw.packed ? width : 0;  // where chunk 1 sits inside the 32-column-aligned window the GEMM reads
                ok &= ab.fold_conv(&bw.conv_b, p + ".convs.1", p + ".bns.1", width, width, 3, 2, wpad, {{9, wpad, 0, width, 0}, {9, wpad, pos1, width, 0}});
            } else {
                ok &= aff_weights(&bw.aff_a, &bw.aff_b, p + ".fuse_models.0", width, wpad);
                ok &= ab.fold_conv(&bw.conv_b, p + ".convs.1", p + ".bns.1", width, width, 3, 2, wpad, {{9, wpad, 0, width, 0}});
            }
            ok &= ab.fold_conv(&bw.conv3, p + ".conv3", p + ".bn3", C, 2 * width, 1, 2, C, {{1, wpad, 0, width, 0}, {1, wpad, 0, width, width}});
            bw.has_sc = (bw.stride != 1 || in_planes != C);
            if (bw.has_sc) ok &= ab.fold_conv(&bw.sc, p + ".shortcut.0", p + ".shortcut.1", C, in_planes, 1, 2);
            in_planes = C;
        }
    }
    // ERes2Net: three bottom-up fusions (eres2net.py:253-258); ERes2NetV2: only out3 -> out4 (layer3_ds + fuse34, eres2net.py:452-453)
    m->fuse_first = v2 ? 2 : 0;
    for (int i = m->fuse_first; i < 3 && ok; ++i) {
        const int Cin = cf.m_channels << (i + 1), Cout = 2 * Cin;  // layer(i+1)_downsample: 64->128, 128->256, 256->512
        EFuseW& fw = m->fuse[i];
        fw.C = Cout;
        ok &= ab.fold_conv(&fw.ds, v2 ? std::string("layer3_ds") : "layer" + std::to_string(i + 1) + "_downsample", "", Cout, Cin, 3, 2);
        static const char* names[3] = {"fuse_mode12", "fuse_mode123", "fuse_mode1234"};
        ok &= aff_weights(&fw.aff_a, &fw.aff_b, v2 ? "fuse34" : names[i], Cout, Cout);
    }
    if (ok) {
        const int K = 2 * m->stats_ch, E = cf.embd_dim;
        const HostWeight* w = ab.get("seg_1.weight", {K, E});
        const HostWeight* b = ab.get("seg_1.bias", {E});
        if (w && b) {
            std::vector<double> mtx(size_t(E) * K);
            for (int n = 0; n < E; ++n)
                for (int k = 0; k < K; ++k) mtx[size_t(n) * K + k] = w->v[size_t(k) * E + n];
            ab.put_matrix(&m->seg1, mtx, E, K);
            ab.put_f32(&m->seg1.bias, b->v);
        } else {
            ok = false;
        }
    }
    return ok;
}

// ------------------------------------------------------------------------------------------------ workspace / plan
namespace {

struct ErBuffers {
    Planes stem_out, flat, stats;
    std::vector<Planes> c1, s0, s1, a, t, xo, o3, sc, out;
    Planes ds[3], fa[3], ft[3], fout[3];
    float* emb_out;
};

void er_carve(const ERes2NetModel* m, WsCarver& cv, int B, int T, ImageGeo* geo, ErBuffers* eb) {
    image_pyramid(geo + 1, 4, m->cfg.input_size, T, true);
    eb->stem_out = cv.planes(geo[1].rows(B), m->cfg.m_channels);
    const size_t nb = m->blocks.size();
    for (auto* v : {&eb->c1, &eb->s0, &eb->s1, &eb->a, &eb->t, &eb->xo, &eb->o3, &eb->sc, &eb->out}) v->resize(nb);
    // Buffer liveness (round 2; every buffer used to be dedicated: 45 GB at batch 256).  All of a block's buffers live on its stage's
    // grid, and every one of them is dead when the block's add + ReLU has run: one set per STAGE, and the block output overwrites its
    // residual input in place (elementwise).  The per-stage activation buffer survives for the bottom-up fusion.  Zero borders and the
    // zero padding columns survive because a buffer never changes grid or column plan inside a stage.
    Planes s_c1[5], s_s0[5], s_s1[5], s_a[5], s_t[5], s_xo[5], s_o3[5], s_act[5];
    bool have[5] = {false, false, false, false, false};
    for (size_t i = 0; i < nb; ++i) {
        const EBlockW& bw = m->blocks[i];
        const int st = bw.stage;
        const int64_t R = geo[st].rows(B);
        if (!have[st]) {
            have[st] = true;
            s_c1[st] = cv.planes(R, bw.c1_cols);
            s_s0[st] = cv.planes(R, bw.wpad);
            s_s1[st] = cv.planes(R, bw.wpad);
            if (bw.fuse) {
                s_a[st] = cv.planes(R, std::max((bw.width / 4 + 31) / 32 * 32, 32));
                s_t[st] = cv.planes(R, bw.wpad);
                s_xo[st] = cv.planes(R, bw.wpad);
            }
            s_o3[st] = cv.planes(R, 2 * bw.planes);
            s_act[st] = cv.planes(R, 2 * bw.planes);
        }
        eb->c1[i] = s_c1[st];
        eb->s0[i] = s_s0[st];
        eb->s1[i] = s_s1[st];
        if (bw.fuse) {
            eb->a[i] = s_a[st];
            eb->t[i] = s_t[st];
            eb->xo[i] = s_xo[st];
        }
        eb->o3[i] = s_o3[st];
        if (bw.has_sc) eb->sc[i] = s_act[st];
        eb->out[i] = s_act[st];
    }
    for (int i = m->fuse_first; i < 3; ++i) {
        const int64_t R = geo[i + 2].rows(B);
        const int C = m->fuse[i].C;
        eb->ds[i] = cv.planes(R, C);
        eb->fa[i] = cv.planes(R, std::max(C / 4, 32));
        eb->ft[i] = cv.planes(R, C);
        eb->fout[i] = cv.planes(R, C);
    }
    const int Tf = geo[4].W;
    eb->flat = cv.planes(int64_t(B) * Tf, m->stats_ch);
    eb->stats = cv.planes(B, 2 * m->stats_ch);
    eb->emb_out = static_cast<float*>(cv.take(align_up(size_t(B), 128) * m->cfg.embd_dim * 4));
}

}  // namespace

size_t ERes2NetModel::workspace_bytes(int B, int T) const {
    if (!finalized || B <= 0 || T <= 0) return 0;
    WsCarver cv;
    ImageGeo g[5];
    ErBuffers eb;
    er_carve(this, cv, B, T, g, &eb);
    return align_up(cv.off, 256);
}

int ERes2NetModel::build_plan(int B, int T, void* ws, size_t ws_bytes, cudaStream_t st) {
    ERes2NetModel* const m = this;
    PPV_REQUIRE(T >= 16, "eres2net: too few frames (TSTP needs at least two pooled frames)");
    image_pyramid(m->geo + 1, 4, m->cfg.input_size, T, true);
    PPV_REQUIRE(m->geo[1].rows(B) < (int64_t(1) << 31), "eres2net: batch too large for 32-bit row indices");
    int rc = claim_workspace(B, T, ws, ws_bytes, st);
    if (rc) return rc;
    WsCarver cv;
    cv.base = static_cast<uint8_t*>(ws);
    ErBuffers eb;
    er_carve(m, cv, B, T, m->geo, &eb);
    m->steps.clear();

    auto relu20 = [](Epilogue ep) {
        ep.relu = 1;
        ep.relu_max = ER_RELU_MAX;
        return ep;
    };
    // AFF(x, y): a = SiLU(BN(conv(cat))), t = tanh(BN(conv(a))), out = x(1+t) + y(1-t)
    auto add_aff = [&](const GemmWeights& ga, const GemmWeights& gb, const Planes& x, int xc0, const Planes& y, int yc0, int C, const Planes& abuf,
                       const Planes& tbuf, const Planes& out, const ImageGeo& g) -> int {
        const int M = int(g.rows(B));
        Epilogue ea = image_epilogue(abuf, g, g, 1, 1);
        ea.silu_ = 1;
        int rc = plan_conv(ga, {GemmSource{x, xc0, C, 0}, GemmSource{y, yc0, C, 0}}, M, ea);
        if (rc) return rc;
        Epilogue et = image_epilogue(tbuf, g, g, 1, 1);
        et.tanh_ = 1;
        rc = plan_conv(gb, {GemmSource{abuf, 0, abuf.ld, 0}}, M, et);
        if (rc) return rc;
        m->steps.push_back(aff_combine_step(x, xc0, y, yc0, tbuf, out, C, g.rows(B)));
        return PPV_OK;
    };

    m->steps.push_back(stem_step(m->stem_w, m->stem_b, m->cfg.m_channels, eb.stem_out, m->geo[1], B));
    Planes x = eb.stem_out;
    for (size_t i = 0; i < m->blocks.size(); ++i) {
        const EBlockW& bw = m->blocks[i];
        const ImageGeo& gin = m->geo[bw.stride == 2 ? bw.stage - 1 : bw.stage];
        const ImageGeo& go = m->geo[bw.stage];
        const int Min = int(gin.rows(B)), Mo = int(go.rows(B)), wp = bw.wpad, C = 2 * bw.planes;
        // conv1 (1x1, stride) + bn1 + relu20 -> c1 on the output grid
        rc = plan_conv(bw.conv1, {GemmSource{x, 0, bw.in_planes, 0}}, Min, relu20(image_epilogue(eb.c1[i], gin, go, bw.stride, bw.stride)));
        if (rc) return rc;
        // first 3x3 on chunk 0
        rc = plan_conv3x3(bw.conv_a, eb.c1[i], 0, wp, go, B, relu20(image_epilogue(eb.s0[i], go, go, 1, 1)));
        if (rc) return rc;
        // second 3x3
        std::vector<GemmSource> tb;
        if (!bw.fuse) {
            image_taps(&tb, eb.s0[i], 0, wp, go);
            image_taps(&tb, eb.c1[i], bw.packed ? 0 : bw.c1_chunk1, wp, go);
        } else {
            rc = add_aff(bw.aff_a, bw.aff_b, eb.s0[i], 0, eb.c1[i], bw.c1_chunk1, wp, eb.a[i], eb.t[i], eb.xo[i], go);
            if (rc) return rc;
            image_taps(&tb, eb.xo[i], 0, wp, go);
        }
        rc = plan_conv(bw.conv_b, tb, Mo, relu20(image_epilogue(eb.s1[i], go, go, 1, 1)));
        if (rc) return rc;
        // conv3 (1x1) + bn3 over concat(s0, s1)
        rc = plan_conv(bw.conv3, {GemmSource{eb.s0[i], 0, wp, 0}, GemmSource{eb.s1[i], 0, wp, 0}}, Mo, image_epilogue(eb.o3[i], go, go, 1, 1));
        if (rc) return rc;
        Planes res = x;
        if (bw.has_sc) {
            rc = plan_conv(bw.sc, {GemmSource{x, 0, bw.in_planes, 0}}, Min, image_epilogue(eb.sc[i], gin, go, bw.stride, bw.stride));
            if (rc) return rc;
            res = eb.sc[i];
        }
        m->steps.push_back(scale_res_step(eb.o3[i], nullptr, res, 0, eb.out[i], 0, C, go.Hp * go.Wp, go.rows(B), true, ER_RELU_MAX));
        x = eb.out[i];
        m->stage_out[bw.stage] = x;
    }
    // bottom-up fusion: fuse12 = AFF(out2, ds(out1)); fuse123 = AFF(out3, ds(fuse12)); fuse1234 = AFF(out4, ds(fuse123))
    Planes prev = m->stage_out[m->fuse_first + 1];
    for (int i = m->fuse_first; i < 3; ++i) {
        const ImageGeo& gin = m->geo[i + 1];
        const ImageGeo& go = m->geo[i + 2];
        const EFuseW& fw = m->fuse[i];
        std::vector<GemmSource> td;
        image_taps(&td, prev, 0, fw.C / 2, gin);
        rc = plan_conv(fw.ds, td, int(gin.rows(B)), image_epilogue(eb.ds[i], gin, go, 2, 2));
        if (rc) return rc;
        rc = add_aff(fw.aff_a, fw.aff_b, m->stage_out[i + 2], 0, eb.ds[i], 0, fw.C, eb.fa[i], eb.ft[i], eb.fout[i], go);
        if (rc) return rc;
        prev = eb.fout[i];
        m->fuse_out[i] = prev;
    }
    const ImageGeo& g4 = m->geo[4];
    m->steps.push_back(flatten_step(prev, g4, B, m->cfg.m_channels * 16, eb.flat));
    m->steps.push_back(colstats_step(eb.flat, m->stats_ch, B, g4.W, 0, g4.W, 2, 1e-8f, eb.stats));
    {
        Epilogue ep;
        ep.out_mode = OUT_F32;
        ep.out = eb.emb_out;
        ep.out_ld = m->cfg.embd_dim;
        rc = plan_conv(m->seg1, {GemmSource{eb.stats, 0, 2 * m->stats_ch, 0}}, B, ep);
        if (rc) return rc;
    }
    m->stats = eb.stats;
    m->emb_out = eb.emb_out;
    return PPV_OK;
}

// taps: "layer1".."layer4", "fuse12", "fuse123", "fuse1234" -> fp32 [B,H,W,C]; "stats" -> [B, 2*512*F']
int ERes2NetModel::tap(const std::string& n, float* out, size_t out_elems, cudaStream_t st) {
    ERes2NetModel* const m = this;
    const int B = m->plan_B;
    if (n == "stats") {
        PPV_REQUIRE(out_elems >= size_t(B) * 2 * m->stats_ch, "eres2net_read_tap: output too small");
        return launch_planes_to_f32(m->stats, 0, 2 * m->stats_ch, B, 1, 0, 1, out, st);
    }
    if (const int stage = name_index(n, "layer", 1, 4)) return image_tap(m->stage_out[stage], m->geo[stage], 2 * (m->cfg.m_channels << (stage - 1)), out, out_elems, st);
    if (n == "fuse34" || n == "fuse12" || n == "fuse123" || n == "fuse1234") {
        const int i = (n == "fuse34") ? 2 : int(n.size()) - 6;
        PPV_REQUIRE(i >= m->fuse_first, "eres2net_read_tap: this fusion stage does not exist in ERes2NetV2");
        return image_tap(m->fuse_out[i], m->geo[i + 2], m->fuse[i].C, out, out_elems, st);
    }
    return fail(PPV_EINVAL, "eres2net_read_tap: unknown tap " + n);
}

}  // namespace ppv
