// ERes2Net forward as a plan of tensor-core gather-GEMMs over zero-bordered NHWC images.
// Reference graph: ppvector/models/eres2net.py:239-263 (ERes2Net.forward), :85-108 (BasicBlockERes2Net.forward),
// :147-170 (BasicBlockERes2Net_diff_AFF.forward), :46-52 (AFF.forward), :12-19 (clipped ReLU = Hardtanh(0,20)),
// ppvector/models/pooling.py:138-146 (TSTP).  Eval mode, default configuration of configs/eres2net.yml
// (scale 2, expansion 2, base_width 32, one embedding layer).
//
// Same image layout and conv2d-as-gather-GEMM scheme as resnet_se.cu.  What is specific here:
//   * Res2Net split of scale 2: `sp + spx[1]` is two K-sources of the second 3x3 conv (conv is linear); `split` and
//     `concat` are column windows of the conv1 output / K-sources of conv3;
//   * layer1 works on 16-channel halves: the GEMM reads the whole 32-channel row and the weights of the other half are
//     zero (k-steps are 32 wide), outputs are padded to 32 columns of which 16 are zero;
//   * AFF (attentional feature fusion): concat -> 1x1 conv + BN + SiLU -> 1x1 conv + BN -> tanh are two small GEMMs
//     (two K-sources, SiLU / tanh epilogues), the blend x(1+t) + y(1-t) is one elementwise pass;
//   * strided 1x1 / 3x3 convs are computed on the input grid and stored on the output grid (see resnet_se.cu);
//   * TSTP = column mean and sqrt(unbiased variance + 1e-8) over time of the flattened [B, T', 512*F'] matrix.
#include <math.h>

#include <stdlib.h>

#include "common.h"
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

struct EStep {
    enum Kind { STEM, GEMM, CONV3, PW, ADD_RELU, AFF_COMBINE, FLATTEN, TSTP } kind;
    PwStep pw;  // PW: 1x1 conv with K <= 64 on the CUDA cores (pointwise.cu)
    Conv3x3Params c3;  // CONV3: single-source 3x3 conv over a 32-channel (padded) chunk, conv3x3.cu
    GemmParams gp;
    Planes a, b, c, d;
    int ac0 = 0, bc0 = 0, C = 0, img_rows = 0;
    int64_t rows = 0;
};

}  // namespace

struct ERes2NetModel : Model {
    ppv_eres2net_cfg cfg;
    float *stem_w = nullptr, *stem_b = nullptr;
    std::vector<EBlockW> blocks;
    EFuseW fuse[3];
    GemmWeights seg1;
    int fuse_first = 0;  // first bottom-up fusion stage in use (0: ERes2Net, 2: ERes2NetV2)
    int stats_ch = 0;  // 512 * F'
    // plan
    std::vector<EStep> steps;
    ImageGeo geo[5];
    Planes stem_out, flat, stats;
    std::vector<Planes> blk_out;
    Planes fuse_out[3];
    int Tf = 0;

    explicit ERes2NetModel(const ppv_eres2net_cfg& c) : Model("eres2net", c.precision), cfg(c) {}
    int embd_dim() const override { return cfg.embd_dim; }
    size_t workspace_bytes(int B, int T) const override;

  protected:
    bool prepare_weights(ArenaBuilder& ab) override;
    int build_plan(int B, int T, void* ws, size_t ws_bytes, cudaStream_t st) override;
    int run_steps(const float* feat, cudaStream_t st) override;
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
    bool ok = true;
    // One K group of a dense weight matrix: `ncols` source columns per tap, of which columns [pos, pos+cnt) carry the conv's
    // input channels [cin0, cin0+cnt) and the rest are zero.
    struct KG {
        int taps, ncols, pos, cnt, cin0;
    };
    // conv [N, Cin, k, k] (+ optional BN folded) -> dense [Npad][sum taps*ncols]; output channel n lands in row n, or, with `chunk` > 0,
    // in row (n / chunk) * chunk_stride + n % chunk (zero-padded output chunks)
    auto conv_matrix = [&](GemmWeights* gw, const std::string& conv, const std::string& bn, int N, int Npad, int Cin, int k,
                           const std::vector<KG>& groups, int chunk = 0, int chunk_stride = 0) {
        const HostWeight* w = ab.get(conv + ".weight", {N, Cin, k, k});
        const HostWeight* b = ab.get(conv + ".bias", {N});
        std::vector<double> sc(N, 1.0), sh(N, 0.0);
        if (!w || !b || (!bn.empty() && !ab.bn_affine(bn, N, &sc, &sh))) {
            ok = false;
            return;
        }
        const int taps = k * k;
        int K = 0;
        for (const KG& g : groups) K += g.taps * g.ncols;
        std::vector<double> mtx(size_t(Npad) * K, 0.0);
        std::vector<float> bias(std::max(Npad, 64), 0.f);
        for (int n = 0; n < N; ++n) {
            const int row = chunk > 0 ? (n / chunk) * chunk_stride + n % chunk : n;
            int kpos = 0;
            for (const KG& g : groups) {
                for (int t = 0; t < g.taps; ++t) {
                    for (int c = 0; c < g.cnt; ++c)
                        mtx[size_t(row) * K + kpos + t * g.ncols + g.pos + c] = double(w->v[(size_t(n) * Cin + g.cin0 + c) * taps + t]) * sc[n];
                }
                kpos += g.taps * g.ncols;
            }
            bias[row] = float(double(b->v[n]) * sc[n] + sh[n]);
        }
        ab.put_matrix(gw, mtx, Npad, K);
        gw->N = Npad;
        ab.put_f32(&gw->bias, bias);
    };
    auto aff_weights = [&](GemmWeights* ga, GemmWeights* gb, const std::string& p, int C, int src_cols) {
        // local_att.0: conv(2C -> C/4) over concat(x, y): two K groups of src_cols columns with C real channels each
        const int inter = C / 4, ipad = std::max((inter + 31) / 32 * 32, 32);
        conv_matrix(ga, p + ".local_att.0", p + ".local_att.1", inter, ipad, 2 * C, 1, {{1, src_cols, 0, C, 0}, {1, src_cols, 0, C, C}});
        conv_matrix(gb, p + ".local_att.3", p + ".local_att.4", C, (C + 31) / 32 * 32, inter, 1, {{1, ipad, 0, inter, 0}});
    };
    {  // stem: conv1 + bn1 folded
        const int C0 = cf.m_channels;
        const HostWeight* w = ab.get("conv1.weight", {C0, 1, 3, 3});
        const HostWeight* b = ab.get("conv1.bias", {C0});
        std::vector<double> sc, sh;
        if (w && b && ab.bn_affine("bn1", C0, &sc, &sh)) {
            std::vector<float> w9(size_t(C0) * 9), bb(C0);
            for (int c = 0; c < C0; ++c) {
                for (int k = 0; k < 9; ++k) w9[c * 9 + k] = float(double(w->v[c * 9 + k]) * sc[c]);
                bb[c] = float(double(b->v[c]) * sc[c] + sh[c]);
            }
            ab.put_f32(&m->stem_w, w9);
            ab.put_f32(&m->stem_b, bb);
        } else {
            ok = false;
        }
    }
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
            conv_matrix(&bw.conv1, p + ".conv1", p + ".bn1", 2 * width, bw.c1_cols, in_planes, 1, {{1, in_planes, 0, in_planes, 0}}, width, bw.c1_chunk1);
            // first 3x3: reads chunk 0 of the conv1 output (for width 16 the 32-wide window with the upper half zero-weighted)
            conv_matrix(&bw.conv_a, p + ".convs.0", p + ".bns.0", width, wpad, width, 3, {{9, wpad, 0, width, 0}});
            if (!bw.fuse) {
                // second 3x3 on sp + spx[1]: K sources (sp buffer, conv1-output window holding chunk 1)
                const int pos1 = bw.packed ? width : 0;  // where chunk 1 sits inside the 32-column-aligned window the GEMM reads
                conv_matrix(&bw.conv_b, p + ".convs.1", p + ".bns.1", width, wpad, width, 3, {{9, wpad, 0, width, 0}, {9, wpad, pos1, width, 0}});
            } else {
                aff_weights(&bw.aff_a, &bw.aff_b, p + ".fuse_models.0", width, wpad);
                conv_matrix(&bw.conv_b, p + ".convs.1", p + ".bns.1", width, wpad, width, 3, {{9, wpad, 0, width, 0}});
            }
            conv_matrix(&bw.conv3, p + ".conv3", p + ".bn3", C, C, 2 * width, 1, {{1, wpad, 0, width, 0}, {1, wpad, 0, width, width}});
            bw.has_sc = (bw.stride != 1 || in_planes != C);
            if (bw.has_sc) conv_matrix(&bw.sc, p + ".shortcut.0", p + ".shortcut.1", C, C, in_planes, 1, {{1, in_planes, 0, in_planes, 0}});
            in_planes = C;
        }
    }
    // ERes2Net: three bottom-up fusions (eres2net.py:253-258); ERes2NetV2: only out3 -> out4 (layer3_ds + fuse34, eres2net.py:452-453)
    m->fuse_first = v2 ? 2 : 0;
    for (int i = m->fuse_first; i < 3 && ok; ++i) {
        const int Cin = cf.m_channels << (i + 1), Cout = 2 * Cin;  // layer(i+1)_downsample: 64->128, 128->256, 256->512
        EFuseW& fw = m->fuse[i];
        fw.C = Cout;
        conv_matrix(&fw.ds, v2 ? std::string("layer3_ds") : "layer" + std::to_string(i + 1) + "_downsample", "", Cout, Cout, Cin, 3, {{9, Cin, 0, Cin, 0}});
        static const char* names[3] = {"fuse_mode12", "fuse_mode123", "fuse_mode1234"};
        aff_weights(&fw.aff_a, &fw.aff_b, v2 ? "fuse34" : names[i], Cout, Cout);
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

void er_geometry(const ERes2NetModel* m, int T, ImageGeo* geo) {
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

void er_carve(const ERes2NetModel* m, WsCarver& cv, int B, int T, ImageGeo* geo, ErBuffers* eb) {
    er_geometry(m, T, geo);
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
    eb->emb_out = static_cast<float*>(cv.take(mc_align_up(size_t(B), 128) * m->cfg.embd_dim * 4));
}

}  // namespace

size_t ERes2NetModel::workspace_bytes(int B, int T) const {
    if (!finalized || B <= 0 || T <= 0) return 0;
    WsCarver cv;
    ImageGeo g[5];
    ErBuffers eb;
    er_carve(this, cv, B, T, g, &eb);
    return mc_align_up(cv.off, 256);
}

int ERes2NetModel::build_plan(int B, int T, void* ws, size_t ws_bytes, cudaStream_t st) {
    ERes2NetModel* const m = this;
    const size_t need = workspace_bytes(B, T);
    PPV_REQUIRE(ws && ws_bytes >= need, "eres2net: workspace too small (see ppv_model_workspace_bytes)");
    PPV_REQUIRE((reinterpret_cast<uintptr_t>(ws) & 255) == 0, "eres2net: workspace must be 256-byte aligned");
    PPV_REQUIRE(T >= 16, "eres2net: too few frames (TSTP needs at least two pooled frames)");
    WsCarver cv;
    cv.base = static_cast<uint8_t*>(ws);
    ErBuffers eb;
    er_carve(m, cv, B, T, m->geo, &eb);
    PPV_REQUIRE(m->geo[1].rows(B) < (int64_t(1) << 31), "eres2net: batch too large for 32-bit row indices");
    PPV_CUDA_OK(cudaMemsetAsync(ws, 0, need, st));  // zero borders, zero padded columns
    m->steps.clear();

    auto img_epi = [&](const Planes& out, const ImageGeo& gin, const ImageGeo& gout, int stride) {
        Epilogue ep;
        ep.out_mode = OUT_PLANES;
        ep.out = out.base;
        ep.out_ld = out.ld;
        ep.out_plane_stride = out.plane_stride;
        ep.img_Hp = gin.Hp;
        ep.img_Wp = gin.Wp;
        ep.img_H = gin.H;
        ep.img_W = gin.W;
        ep.img_stride = stride;
        ep.out_Hp = gout.Hp;
        ep.out_Wp = gout.Wp;
        return ep;
    };
    auto add_gemm = [&](const GemmWeights& gw, const std::vector<GemmSource>& srcs, int M, Epilogue ep) -> int {
        ep.bias = gw.bias;
        EStep s;
        if (pointwise_step_build(&s.pw, srcs.data(), int(srcs.size()), gw.W, gw.N, M, ep)) {
            s.kind = EStep::PW;
        } else {
            s.kind = EStep::GEMM;
            int rc = gemm_build(&s.gp, srcs.data(), int(srcs.size()), gw.W, M, gw.N, ep, gemm_pick_bn(gw.N));
            if (rc) return rc;
        }
        m->steps.push_back(s);
        return PPV_OK;
    };
    auto taps9 = [&](const Planes& p, int col0, int ncols, const ImageGeo& g, std::vector<GemmSource>* v) {
        for (int dh = -1; dh <= 1; ++dh)
            for (int dw = -1; dw <= 1; ++dw) v->push_back(GemmSource{p, col0, ncols, dh * g.Wp + dw});
    };
    auto relu20 = [](Epilogue ep) {
        ep.relu = 1;
        ep.relu_max = ER_RELU_MAX;
        return ep;
    };
    // AFF(x, y): a = SiLU(BN(conv(cat))), t = tanh(BN(conv(a))), out = x(1+t) + y(1-t)
    auto add_aff = [&](const GemmWeights& ga, const GemmWeights& gb, const Planes& x, int xc0, const Planes& y, int yc0, int C, const Planes& abuf,
                       const Planes& tbuf, const Planes& out, const ImageGeo& g) -> int {
        const int M = int(g.rows(B));
        Epilogue ea = img_epi(abuf, g, g, 1);
        ea.silu_ = 1;
        int rc = add_gemm(ga, {GemmSource{x, xc0, C, 0}, GemmSource{y, yc0, C, 0}}, M, ea);
        if (rc) return rc;
        Epilogue et = img_epi(tbuf, g, g, 1);
        et.tanh_ = 1;
        rc = add_gemm(gb, {GemmSource{abuf, 0, abuf.ld, 0}}, M, et);
        if (rc) return rc;
        EStep s;
        s.kind = EStep::AFF_COMBINE;
        s.a = x;
        s.ac0 = xc0;
        s.b = y;
        s.bc0 = yc0;
        s.c = tbuf;
        s.d = out;
        s.C = C;
        s.rows = g.rows(B);
        m->steps.push_back(s);
        return PPV_OK;
    };

    {
        EStep s;
        s.kind = EStep::STEM;
        m->steps.push_back(s);
    }
    Planes x = eb.stem_out;
    Planes stage_out[5];
    int rc;
    const char* c3env = getenv("PPV_CONV3X3");  // 0 = 3x3 convs through the generic gather-GEMM (debugging / A-B timing)
    const bool use_c3 = !(c3env && c3env[0] == '0');
    for (size_t i = 0; i < m->blocks.size(); ++i) {
        const EBlockW& bw = m->blocks[i];
        const ImageGeo& gin = m->geo[bw.stride == 2 ? bw.stage - 1 : bw.stage];
        const ImageGeo& go = m->geo[bw.stage];
        const int Min = int(gin.rows(B)), Mo = int(go.rows(B)), w = bw.width, wp = bw.wpad, C = 2 * bw.planes;
        // conv1 (1x1, stride) + bn1 + relu20 -> c1 on the output grid
        rc = add_gemm(bw.conv1, {GemmSource{x, 0, bw.in_planes, 0}}, Min, relu20(img_epi(eb.c1[i], gin, go, bw.stride)));
        if (rc) return rc;
        // first 3x3 on chunk 0
        if (use_c3 && wp == 32 && bw.conv_a.N == 32 && bw.conv_a.Ktot == 9 * 32) {  // weight-stationary patch kernel (conv3x3.cu)
            Epilogue ep = relu20(img_epi(eb.s0[i], go, go, 1));
            ep.bias = bw.conv_a.bias;
            EStep s3;
            s3.kind = EStep::CONV3;
            rc = conv3x3_build(&s3.c3, eb.c1[i], 0, bw.conv_a.W, B, go.H, go.W, go.Hp, go.Wp, ep);
            if (rc) return rc;
            m->steps.push_back(s3);
        } else {
            std::vector<GemmSource> ta;
            taps9(eb.c1[i], 0, wp, go, &ta);
            rc = add_gemm(bw.conv_a, ta, Mo, relu20(img_epi(eb.s0[i], go, go, 1)));
            if (rc) return rc;
        }
        // second 3x3
        std::vector<GemmSource> tb;
        if (!bw.fuse) {
            taps9(eb.s0[i], 0, wp, go, &tb);
            taps9(eb.c1[i], bw.packed ? 0 : bw.c1_chunk1, wp, go, &tb);
        } else {
            rc = add_aff(bw.aff_a, bw.aff_b, eb.s0[i], 0, eb.c1[i], bw.c1_chunk1, wp, eb.a[i], eb.t[i], eb.xo[i], go);
            if (rc) return rc;
            taps9(eb.xo[i], 0, wp, go, &tb);
        }
        rc = add_gemm(bw.conv_b, tb, Mo, relu20(img_epi(eb.s1[i], go, go, 1)));
        if (rc) return rc;
        // conv3 (1x1) + bn3 over concat(s0, s1)
        rc = add_gemm(bw.conv3, {GemmSource{eb.s0[i], 0, wp, 0}, GemmSource{eb.s1[i], 0, wp, 0}}, Mo, img_epi(eb.o3[i], go, go, 1));
        if (rc) return rc;
        Planes res = x;
        if (bw.has_sc) {
            rc = add_gemm(bw.sc, {GemmSource{x, 0, bw.in_planes, 0}}, Min, img_epi(eb.sc[i], gin, go, bw.stride));
            if (rc) return rc;
            res = eb.sc[i];
        }
        EStep s;
        s.kind = EStep::ADD_RELU;
        s.a = eb.o3[i];
        s.b = res;
        s.d = eb.out[i];
        s.C = C;
        s.img_rows = go.Hp * go.Wp;
        s.rows = go.rows(B);
        m->steps.push_back(s);
        x = eb.out[i];
        stage_out[bw.stage] = x;
    }
    // bottom-up fusion: fuse12 = AFF(out2, ds(out1)); fuse123 = AFF(out3, ds(fuse12)); fuse1234 = AFF(out4, ds(fuse123))
    Planes prev = stage_out[m->fuse_first + 1];
    for (int i = m->fuse_first; i < 3; ++i) {
        const ImageGeo& gin = m->geo[i + 1];
        const ImageGeo& go = m->geo[i + 2];
        const EFuseW& fw = m->fuse[i];
        std::vector<GemmSource> td;
        taps9(prev, 0, fw.C / 2, gin, &td);
        rc = add_gemm(fw.ds, td, int(gin.rows(B)), img_epi(eb.ds[i], gin, go, 2));
        if (rc) return rc;
        rc = add_aff(fw.aff_a, fw.aff_b, stage_out[i + 2], 0, eb.ds[i], 0, fw.C, eb.fa[i], eb.ft[i], eb.fout[i], go);
        if (rc) return rc;
        prev = eb.fout[i];
    }
    {
        EStep s;
        s.kind = EStep::FLATTEN;
        s.a = prev;
        s.d = eb.flat;
        m->steps.push_back(s);
        s.kind = EStep::TSTP;
        m->steps.push_back(s);
    }
    {
        Epilogue ep;
        ep.out_mode = OUT_F32;
        ep.out = eb.emb_out;
        ep.out_ld = m->cfg.embd_dim;
        rc = add_gemm(m->seg1, {GemmSource{eb.stats, 0, 2 * m->stats_ch, 0}}, B, ep);
        if (rc) return rc;
    }
    m->stem_out = eb.stem_out;
    m->flat = eb.flat;
    m->stats = eb.stats;
    m->blk_out = eb.out;
    for (int i = m->fuse_first; i < 3; ++i) m->fuse_out[i] = eb.fout[i];
    m->emb_out = eb.emb_out;
    m->Tf = m->geo[4].W;
    return PPV_OK;
}

// ------------------------------------------------------------------------------------------------ forward
int ERes2NetModel::run_steps(const float* feat, cudaStream_t st) {
    ERes2NetModel* const m = this;
    const int B = m->plan_B, T = m->plan_T;
    int rc = PPV_OK;
    for (const EStep& s : m->steps) {
        switch (s.kind) {
            case EStep::STEM:
                rc = launch_stem_conv(feat, B, T, m->cfg.input_size, m->stem_w, m->stem_b, m->cfg.m_channels, m->stem_out, m->geo[1].Hp, m->geo[1].Wp, st);
                break;
            case EStep::GEMM: rc = gemm_launch(s.gp, m->precision, m->num_sms, st); break;
            case EStep::CONV3: rc = conv3x3_launch(s.c3, m->precision, m->num_sms, st); break;
            case EStep::PW: rc = pointwise_launch(s.pw, m->num_sms, st); break;
            case EStep::ADD_RELU:
                rc = launch_se_scale_res(s.a, nullptr, s.b, 0, s.d, 0, s.C, s.img_rows, s.rows, m->num_sms, st, 1, ER_RELU_MAX);
                break;
            case EStep::AFF_COMBINE: rc = launch_aff_combine(s.a, s.ac0, s.b, s.bc0, s.c, s.d, s.C, s.rows, m->num_sms, st); break;
            case EStep::FLATTEN: {
                const ImageGeo& g4 = m->geo[4];
                rc = launch_flatten_image(s.a, B, g4.H, g4.W, g4.Hp, g4.Wp, m->cfg.m_channels * 16, s.d, m->num_sms, st);
                break;
            }
            case EStep::TSTP: rc = launch_colstats(m->flat, 0, m->stats_ch, B, m->Tf, 0, m->Tf, 2, 1e-8f, nullptr, m->stats, st); break;
        }
        if (rc) return rc;
    }
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
    Planes src;
    int stage = 0, C = 0;
    if (n.rfind("layer", 0) == 0 && n.size() == 6 && n[5] >= '1' && n[5] <= '4') {
        stage = n[5] - '0';
        int last = -1;
        for (size_t i = 0; i < m->blocks.size(); ++i)
            if (m->blocks[i].stage == stage) last = int(i);
        src = m->blk_out[last];
        C = 2 * (m->cfg.m_channels << (stage - 1));
    } else if (n == "fuse34" || n == "fuse12" || n == "fuse123" || n == "fuse1234") {
        const int i = (n == "fuse34") ? 2 : int(n.size()) - 6;
        PPV_REQUIRE(i >= m->fuse_first, "eres2net_read_tap: this fusion stage does not exist in ERes2NetV2");
        src = m->fuse_out[i];
        stage = i + 2;
        C = m->fuse[i].C;
    } else {
        return fail(PPV_EINVAL, "eres2net_read_tap: unknown tap " + n);
    }
    const ImageGeo& g = m->geo[stage];
    PPV_REQUIRE(out_elems >= size_t(B) * g.H * g.W * C, "eres2net_read_tap: output too small");
    return launch_image_to_f32(src, B, g.H, g.W, g.Hp, g.Wp, C, out, st);
}

}  // namespace ppv
