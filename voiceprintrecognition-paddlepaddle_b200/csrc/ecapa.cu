// ECAPA-TDNN forward as a fixed plan of tensor-core gather-GEMMs and HBM-bound reductions.
// Reference graph: ppvector/models/ecapa_tdnn.py:245-276 (EcapaTdnn.forward), :132-142 (SERes2NetBlock),
// :36-47 (Res2NetBlock), :69-82 (SEBlock); ppvector/models/pooling.py:86-125 (ASP, global_context);
// ppvector/models/utils.py:147 (TDNNBlock = BN(ReLU(conv))).  Eval mode, lengths = None (the only way the
// reference ever calls it: predict.py:232,266, trainer.py:210,392).
//
// What is restructured relative to the reference graph (results identical up to fp32 rounding):
//   * activations live channels-last in the padded time layout (common.h), so `transpose`, `F.pad(reflect)`,
//     `chunk` and `concat` cost nothing: they are column / row offsets of TMA tile loads;
//   * Res2Net's `x_i + y_{i-1}` is two K-sources of the same GEMM (conv is linear);
//   * BatchNorm(eval) is a per-channel FMA in the GEMM epilogue after the ReLU;
//   * ASP's tiled [mean;std] concat (K = 4608) becomes a per-utterance bias: W[:, C:3C] . [mean;std]
//     is one tiny GEMM, so the attention TDNN runs with K = 1536 (2.857 GFLOP / utterance executed
//     instead of 3.090).
#include <stdlib.h>
#include <string.h>

#include "common.h"
#include "model_common.h"

namespace ppv {

namespace {

struct ConvW : GemmWeights {  // + BatchNorm(eval) after the ReLU, as y = y * bn_scale + bn_shift
    float* bn_scale = nullptr;
    float* bn_shift = nullptr;
};

struct KSpec {  // one K group: `ncols` columns of a source at a row offset <- weight input channels
    int src;    // buffer id
    int col0, ncols, row_off;
    int w_cin0, w_cnt, w_tap;
};

enum Buf { B_FEAT, B_X0, B_H, B_Y, B_Z, B_CAT, B_MFA, B_ATT, B_GSTAT, B_POOL, B_SEM, B_SEH, B_COUNT };

struct Step {
    enum Kind { GEMM, SKINNY, RES2, RES2CHAIN, SE_SQUEEZE, SE_SCALE, ASP_GLOBAL, ASP_FUSED, POOL_STATS } kind;
    // SKINNY: one-row-per-utterance linear layer on the CUDA cores (skinny.cu)
    Planes sk_x, sk_w;
    int sk_col0 = 0, sk_M = 0, sk_N = 0, sk_K = 0;
    Epilogue sk_ep;
    GemmParams gp;
    AspFusedParams ap;
    Res2Params rp;
    Res2ChainParams cp;
    int blk = 0;  // block index for the SE steps
};

struct EcBuffers {  // the workspace of a plan
    Planes bufs[B_COUNT];
    float *se_mean = nullptr, *se_scale = nullptr, *fold_out = nullptr, *pooled_raw = nullptr, *raw_logmel = nullptr;
    int* nvalid = nullptr;  // [B] valid-frame counts of the current forward (`lengths`)
};

}  // namespace

struct EcapaModel : Model {
    ppv_ecapa_cfg cfg;
    int C = 0, C3 = 0, width = 0, scale = 0, Fp = 0, P = 0, att = 0, se = 0;
    // device weights
    ConvW conv0, tdnn1[3], res2[3][8], tdnn2[3], se1[3], se2[3], mfa, fold, att1, att2, fc;
    float *aspbn_scale = nullptr, *aspbn_shift = nullptr;
    // plan
    std::vector<Step> steps;
    EcBuffers buf;
    int Tp = 0;
    // profiling (bench.py roofline): CUDA events around every launch group of the forward
    bool prof_on = false;
    std::vector<cudaEvent_t> prof_ev;   // pairs
    std::vector<int> prof_kind;         // 0 = tensor-core GEMM, 1 = other kernels
    size_t prof_used = 0;
    int64_t launches_gemm = 0, launches_other = 0;

    explicit EcapaModel(const ppv_ecapa_cfg& c) : Model("ecapa", c.precision), cfg(c) {}
    ~EcapaModel() override {
        for (cudaEvent_t e : prof_ev) cudaEventDestroy(e);
    }
    int embd_dim() const override { return cfg.embd_dim; }
    size_t workspace_bytes(int B, int T) const override;
    int forward_ex(const float* feat, Fbank* fb, const float* wav, const float* lens_ratio, int B, int T, int L, float* emb, void* ws,
                   size_t ws_bytes, cudaStream_t st, const float* lengths);

  protected:
    bool prepare_weights(ArenaBuilder& ab) override;
    int build_plan(int B, int T, void* ws, size_t ws_bytes, cudaStream_t st) override;
    int run_steps(const float* feat, cudaStream_t st) override { return run(feat, nullptr, nullptr, nullptr, 0, nullptr, st); }
    int tap(const std::string& n, float* out, size_t out_elems, cudaStream_t st) override;
    int run(const float* feat, Fbank* fb, const float* wav, const float* lens_ratio, int L, const float* lengths, cudaStream_t st);
};

// ------------------------------------------------------------------------------------------------ create / load
void ppv_ecapa_default_cfg_impl(ppv_ecapa_cfg* c) {
    c->input_size = 80;
    c->embd_dim = 192;
    const int ch[5] = {512, 512, 512, 512, 1536}, ks[5] = {5, 3, 3, 3, 1}, dl[5] = {1, 2, 3, 4, 1};
    for (int i = 0; i < 5; ++i) {
        c->channels[i] = ch[i];
        c->kernel_sizes[i] = ks[i];
        c->dilations[i] = dl[i];
    }
    c->attention_channels = 128;
    c->res2net_scale = 8;
    c->se_channels = 128;
    c->precision = PPV_PREC_BF16X3;
    c->pooling = PPV_POOL_ASP;
    c->global_context = 1;
}

int ecapa_create(const ppv_ecapa_cfg* cfg, Model** out) {
    PPV_REQUIRE(cfg && out, "ecapa_create: null argument");
    const int C = cfg->channels[0];
    if (cfg->channels[1] != C || cfg->channels[2] != C || cfg->channels[3] != C)
        return fail(PPV_EUNSUPPORTED, "ecapa: channels[0..3] must be equal (no shortcut conv path)");
    if (cfg->channels[4] != 3 * C) return fail(PPV_EUNSUPPORTED, "ecapa: channels[4] must equal 3 * channels[0] (MFA concat)");
    if (cfg->res2net_scale < 2 || cfg->res2net_scale > 8 || C % cfg->res2net_scale)
        return fail(PPV_EUNSUPPORTED, "ecapa: res2net_scale must divide channels and be in [2,8]");
    const int width = C / cfg->res2net_scale;
    if (width % 64) return fail(PPV_EUNSUPPORTED, "ecapa: channels / res2net_scale must be a multiple of 64");
    if (cfg->kernel_sizes[1] != 3 || cfg->kernel_sizes[2] != 3 || cfg->kernel_sizes[3] != 3 || cfg->kernel_sizes[4] != 1 ||
        (cfg->kernel_sizes[0] % 2) == 0 || cfg->dilations[4] != 1)
        return fail(PPV_EUNSUPPORTED, "ecapa: kernel sizes must be [odd,3,3,3,1]");
    if (cfg->attention_channels % 64 || cfg->embd_dim % 32 || cfg->se_channels <= 0 || cfg->se_channels % 64)
        return fail(PPV_EUNSUPPORTED, "ecapa: attention_channels % 64, se_channels % 64, embd_dim % 32 required");
    if (cfg->pooling < PPV_POOL_ASP || cfg->pooling > PPV_POOL_TSP) return fail(PPV_EUNSUPPORTED, "ecapa: pooling must be PPV_POOL_ASP / SAP / TAP / TSP");
    EcapaModel* m = new EcapaModel(*cfg);
    m->C = C;
    m->C3 = 3 * C;
    m->width = width;
    m->scale = cfg->res2net_scale;
    m->Fp = int(mc_align_up(cfg->input_size, 64));
    m->att = cfg->attention_channels;
    m->se = cfg->se_channels;
    int P = (cfg->kernel_sizes[0] - 1) / 2 * cfg->dilations[0];
    for (int i = 1; i <= 3; ++i) P = std::max(P, cfg->dilations[i]);
    m->P = P;
    *out = m;
    return PPV_OK;
}

// ------------------------------------------------------------------------------------------------ finalize
namespace {

// conv weight [N, Cin, k] -> split planes [2][Npad][Ktot] following the K groups; rows padded to a multiple of 128
void put_conv(ArenaBuilder& ab, ConvW* cw, const std::vector<float>& w, int N, int Cin, int k, const std::vector<KSpec>& ks) {
    int Ktot = 0;
    for (const KSpec& s : ks) Ktot += s.ncols;
    std::vector<double> mtx(size_t(N) * Ktot, 0.0);
    for (int n = 0; n < N; ++n) {
        int kpos = 0;
        for (const KSpec& s : ks) {
            for (int c = 0; c < s.w_cnt; ++c) mtx[size_t(n) * Ktot + kpos + c] = w[(size_t(n) * Cin + s.w_cin0 + c) * k + s.w_tap];
            kpos += s.ncols;
        }
    }
    ab.put_matrix(cw, mtx, N, Ktot, 128);
}

// BatchNorm eval -> y = x * scale + shift  (ppvector/models/utils.py:96-119), rounded to fp32
bool bn_affine_f32(ArenaBuilder& ab, const std::string& prefix, int C, std::vector<float>* scale, std::vector<float>* shift) {
    std::vector<double> sc, sh;
    if (!ab.bn_affine(prefix, C, &sc, &sh)) return false;
    scale->assign(sc.begin(), sc.end());
    shift->assign(sh.begin(), sh.end());
    return true;
}

std::vector<KSpec> spec_conv0(const EcapaModel* m) {
    std::vector<KSpec> ks;
    const int k = m->cfg.kernel_sizes[0], d = m->cfg.dilations[0];
    for (int j = 0; j < k; ++j) ks.push_back({B_FEAT, 0, m->Fp, (j - (k - 1) / 2) * d, 0, m->cfg.input_size, j});
    return ks;
}
std::vector<KSpec> spec_res2(const EcapaModel* m, int blk, int j) {  // j = 1 .. scale-1
    std::vector<KSpec> ks;
    const int d = m->cfg.dilations[blk], w = m->width;
    for (int tap = 0; tap < 3; ++tap) ks.push_back({B_H, j * w, w, (tap - 1) * d, 0, w, tap});
    if (j >= 2)
        for (int tap = 0; tap < 3; ++tap) ks.push_back({B_Y, (j - 1) * w, w, (tap - 1) * d, 0, w, tap});
    return ks;
}

}  // namespace

bool EcapaModel::prepare_weights(ArenaBuilder& ab) {
    EcapaModel* const m = this;
    const int C = m->C, C3 = m->C3, w = m->width, F = m->cfg.input_size, A = m->att, S = m->se, E = m->cfg.embd_dim;
    const int k0 = m->cfg.kernel_sizes[0];
    auto conv_layer = [&](ConvW* cw, const std::string& wname, int N, int Cin, int k, const std::vector<KSpec>& ks,
                          const std::string& bn_prefix, bool has_bias) -> bool {
        const HostWeight* hw = ab.get(wname + ".weight", {N, Cin, k});
        if (!hw) return false;
        put_conv(ab, cw, hw->v, N, Cin, k, ks);
        if (has_bias) {
            const HostWeight* hb = ab.get(wname + ".bias", {N});
            if (!hb) return false;
            ab.put_f32(&cw->bias, hb->v);
        }
        if (!bn_prefix.empty()) {
            std::vector<float> sc, sh;
            if (!bn_affine_f32(ab, bn_prefix, N, &sc, &sh)) return false;
            ab.put_f32(&cw->bn_scale, sc);
            ab.put_f32(&cw->bn_shift, sh);
        }
        return true;
    };
    bool ok = conv_layer(&m->conv0, "blocks.0.conv.conv", C, F, k0, spec_conv0(m), "blocks.0.norm.norm", true);
    for (int b = 1; b <= 3 && ok; ++b) {
        const std::string p = "blocks." + std::to_string(b);
        ok = ok && conv_layer(&m->tdnn1[b - 1], p + ".tdnn1.conv.conv", C, C, 1, {{-1, 0, C, 0, 0, C, 0}}, p + ".tdnn1.norm.norm", true);
        for (int j = 1; j < m->scale && ok; ++j) {
            const std::string q = p + ".res2net_block.blocks." + std::to_string(j - 1);
            ok = ok && conv_layer(&m->res2[b - 1][j], q + ".conv.conv", w, w, 3, spec_res2(m, b, j), q + ".norm.norm", true);
        }
        ok = ok && conv_layer(&m->tdnn2[b - 1], p + ".tdnn2.conv.conv", C, C, 1, {{B_H, 0, w, 0, 0, w, 0}, {B_Y, w, C - w, 0, w, C - w, 0}},
                              p + ".tdnn2.norm.norm", true);
        // SE excitation as two small gather-GEMMs over the [B, C] squeeze (ecapa_tdnn.py:79-80)
        ok = ok && conv_layer(&m->se1[b - 1], p + ".se_block.conv1.conv", S, C, 1, {{B_SEM, 0, C, 0, 0, C, 0}}, "", true);
        ok = ok && conv_layer(&m->se2[b - 1], p + ".se_block.conv2.conv", C, S, 1, {{B_SEH, 0, S, 0, 0, S, 0}}, "", true);
    }
    ok = ok && conv_layer(&m->mfa, "mfa.conv.conv", C3, C3, 1, {{B_CAT, 0, C3, 0, 0, C3, 0}}, "mfa.norm.norm", true);
    const int pooling = m->cfg.pooling;
    // BatchNorm(eval) + Linear after a parameter-free or self-attentive pooling: fc(bn(p)) = (W diag(s)) p + (W t + b), folded here
    auto folded_fc = [&](int Kp) -> bool {
        const HostWeight* w = ab.get("fc.conv.weight", {E, Kp, 1});
        const HostWeight* b = ab.get("fc.conv.bias", {E});
        std::vector<float> sc, sh;
        if (!w || !b || !bn_affine_f32(ab, "asp_bn", Kp, &sc, &sh)) return false;  // paddle.nn.BatchNorm1D: keys asp_bn.weight / ._mean ...
        std::vector<float> wf(size_t(E) * Kp), bf(E);
        for (int n = 0; n < E; ++n) {
            double acc = b->v[n];
            for (int k = 0; k < Kp; ++k) {
                wf[size_t(n) * Kp + k] = w->v[size_t(n) * Kp + k] * sc[k];
                acc += double(w->v[size_t(n) * Kp + k]) * sh[k];
            }
            bf[n] = float(acc);
        }
        put_conv(ab, &m->fc, wf, E, Kp, 1, {{B_POOL, 0, Kp, 0, 0, Kp, 0}});
        ab.put_f32(&m->fc.bias, bf);
        return true;
    };
    if (pooling == PPV_POOL_ASP) {
    // ASP attention TDNN: weight [A, 3*C3, 1] split into the x part (cols 0..C3) and the [mean;std] part;
    // global_context = False (pooling.py:77-78, 108-109): the TDNN sees x alone, weight [A, C3, 1], no per-utterance bias
    const int ctx = m->cfg.global_context ? 3 : 1;
    ok = ok && conv_layer(&m->att1, "asp.tdnn.conv.conv", A, ctx * C3, 1, {{B_MFA, 0, C3, 0, 0, C3, 0}}, "asp.tdnn.norm.norm", true);
    if (ok && m->cfg.global_context) {
        const HostWeight* hw = ab.get("asp.tdnn.conv.conv.weight", {A, 3 * C3, 1});
        put_conv(ab, &m->fold, hw->v, A, 3 * C3, 1, {{B_GSTAT, 0, 2 * C3, 0, C3, 2 * C3, 0}});
    }
    ok = ok && conv_layer(&m->att2, "asp.conv.conv", C3, A, 1, {{B_ATT, 0, A, 0, 0, A, 0}}, "", true);
    ok = ok && conv_layer(&m->fc, "fc.conv", E, 2 * C3, 1, {{B_POOL, 0, 2 * C3, 0, 0, 2 * C3, 0}}, "", true);
    if (ok) {
        std::vector<float> sc, sh;
        ok = bn_affine_f32(ab, "asp_bn.norm", 2 * C3, &sc, &sh);
        if (ok) {
            ab.put_f32(&m->aspbn_scale, sc);
            ab.put_f32(&m->aspbn_shift, sh);
        }
    }
    } else if (pooling == PPV_POOL_SAP) {
        // SelfAttentivePooling (pooling.py:50-66): alpha = softmax_t(linear2(tanh(linear1(x)))); mean = sum alpha x.  The fused ASP
        // kernel computes exactly this weighted mean (its std half is ignored); linear2's bias cancels in the softmax.
        if (A != 128) {
            ab.err = "SAP pooling uses a 128-channel bottleneck (ecapa_tdnn.py:222): attention_channels must be 128";
            ok = false;
        }
        ok = ok && conv_layer(&m->att1, "asp.linear1", A, C3, 1, {{B_MFA, 0, C3, 0, 0, C3, 0}}, "", true);
        ok = ok && conv_layer(&m->att2, "asp.linear2", C3, A, 1, {{B_ATT, 0, A, 0, 0, A, 0}}, "", true);
        ok = ok && folded_fc(C3);
        if (ok) {
            ab.put_f32(&m->aspbn_scale, std::vector<float>(2 * C3, 1.f));
            ab.put_f32(&m->aspbn_shift, std::vector<float>(2 * C3, 0.f));
        }
    } else {
        ok = ok && folded_fc(pooling == PPV_POOL_TAP ? C3 : 2 * C3);
    }
    return ok;
}

// ------------------------------------------------------------------------------------------------ workspace
namespace {

void carve(const EcapaModel* m, WsCarver& cv, int B, int T, EcBuffers* eb, float** emb_out) {
    const int64_t R = int64_t(B) * (T + 2 * m->P);
    const int C = m->C, C3 = m->C3;
    eb->bufs[B_FEAT] = cv.planes(R, m->Fp);
    eb->bufs[B_X0] = cv.planes(R, C);
    eb->bufs[B_H] = cv.planes(R, C);
    eb->bufs[B_Y] = cv.planes(R, C);
    eb->bufs[B_Z] = cv.planes(R, C);
    eb->bufs[B_CAT] = cv.planes(R, C3);
    eb->bufs[B_MFA] = cv.planes(R, C3);
    eb->bufs[B_ATT] = cv.planes(R, m->att);
    eb->bufs[B_GSTAT] = cv.planes(B, 2 * C3);
    eb->bufs[B_POOL] = cv.planes(B, 2 * C3);
    eb->bufs[B_SEM] = cv.planes(B, C);
    eb->bufs[B_SEH] = cv.planes(B, m->se);
    eb->se_mean = static_cast<float*>(cv.take(size_t(B) * C * 4));
    eb->se_scale = static_cast<float*>(cv.take(size_t(B) * C * 4));
    eb->fold_out = static_cast<float*>(cv.take(mc_align_up(B, 128) * m->att * 4));
    eb->pooled_raw = static_cast<float*>(cv.take(size_t(B) * 2 * C3 * 4));
    eb->raw_logmel = static_cast<float*>(cv.take(size_t(B) * T * m->cfg.input_size * 4));
    *emb_out = static_cast<float*>(cv.take(mc_align_up(B, 128) * m->cfg.embd_dim * 4));
    eb->nvalid = static_cast<int*>(cv.take(size_t(B) * sizeof(int)));
}

// 128-wide n-tiles even where N allows 256: on an H100 SXM at 700 W (tools/gemm_bench.py, M = 78 336, profiles/gemm_bench_after.txt)
// BN = 128 with 64-wide k-steps takes 15-18 % less time than BN = 256 at every large layer of the model (N x K = 512 x 512 / 640,
// 1536 x 1536, split-bf16 x3), and no BN = 256 variant beats it by more than run-to-run noise.
constexpr int ECAPA_MAX_BN = 128;

}  // namespace

size_t EcapaModel::workspace_bytes(int B, int T) const {
    if (B <= 0 || T <= 0) return 0;
    WsCarver cv;
    EcBuffers eb;
    float* emb;
    carve(this, cv, B, T, &eb, &emb);
    return mc_align_up(cv.off, 256);
}

// ------------------------------------------------------------------------------------------------ plan
int EcapaModel::build_plan(int B, int T, void* ws, size_t ws_bytes, cudaStream_t st) {
    EcapaModel* const m = this;
    PPV_REQUIRE(T > m->P, "ecapa: too few frames for the reflect padding");
    int rc = claim_workspace(B, T, ws, ws_bytes, st);
    if (rc) return rc;
    WsCarver cv;
    cv.base = static_cast<uint8_t*>(ws);
    carve(m, cv, B, T, &m->buf, &m->emb_out);
    m->Tp = T + 2 * m->P;
    m->steps.clear();
    const int Tp = m->Tp, P = m->P, C = m->C, C3 = m->C3, w = m->width;
    const int64_t R = int64_t(B) * Tp;
    const char* r2env = getenv("PPV_RES2_GEMM");  // debugging aid: 1 = run the Res2Net convs through the generic gather-GEMM
    const bool use_res2_kernel = (w == 64) && !(r2env && r2env[0] == '1');
    // 0 = one launch per Res2Net conv (res2conv.cu) instead of the fused chain; single = the fused chain with one utterance per CTA
    // even where two fit (tests and A/B timing)
    const char* rcenv = getenv("PPV_RES2_CHAIN");
    const bool use_res2_chain = use_res2_kernel && m->scale == 8 && res2chain_fits(T, P) && !(rcenv && rcenv[0] == '0');
    const bool res2_paired = use_res2_chain && res2chain_pair_fits(T, P) && !(rcenv && strcmp(rcenv, "single") == 0);
    const char* skenv = getenv("PPV_SKINNY");  // 0 = the per-utterance linear layers through the tensor-core gather-GEMM (A-B timing)
    const bool use_skinny = !(skenv && skenv[0] == '0');

    auto add_gemm = [&](const ConvW& cw, const std::vector<KSpec>& ks, const Planes* src_override, int override_col0, int M,
                        Epilogue ep) -> int {
        std::vector<GemmSource> srcs;
        for (const KSpec& s : ks) {
            GemmSource g;
            if (s.src < 0) {
                g.t = *src_override;
                g.col0 = override_col0 + s.col0;
            } else {
                g.t = m->buf.bufs[s.src];
                g.col0 = s.col0;
            }
            g.ncols = s.ncols;
            g.row_off = s.row_off;
            srcs.push_back(g);
        }
        ep.bias = cw.bias;
        if (ep.relu) {
            ep.bn_scale = cw.bn_scale;
            ep.bn_shift = cw.bn_shift;
        }
        // one row per utterance (SE MLP, ASP context bias, fc): every SM takes a 16 x 16 output tile on the CUDA cores instead of 2-6
        // CTAs walking a latency-bound k-loop on the tensor cores
        if (use_skinny && M == B && srcs.size() == 1 && srcs[0].row_off == 0 && skinny_linear_supported(M, cw.N, srcs[0].ncols, ep) &&
            cw.Ktot == srcs[0].ncols) {
            Step sk;
            sk.kind = Step::SKINNY;
            sk.sk_x = srcs[0].t;
            sk.sk_col0 = srcs[0].col0;
            sk.sk_w = cw.W;
            sk.sk_M = M;
            sk.sk_N = cw.N;
            sk.sk_K = srcs[0].ncols;
            sk.sk_ep = ep;
            m->steps.push_back(sk);
            return PPV_OK;
        }
        Step stp;
        stp.kind = Step::GEMM;
        int rc = gemm_build(&stp.gp, srcs.data(), int(srcs.size()), cw.W, M, cw.N, ep, gemm_pick_bn(cw.N, ECAPA_MAX_BN));
        if (rc) return rc;
        m->steps.push_back(stp);
        return PPV_OK;
    };
    auto planes_out = [&](const Planes& p, int col0, bool halo) {
        Epilogue ep;
        ep.out_mode = OUT_PLANES;
        ep.out = p.base;
        ep.out_ld = p.ld;
        ep.out_plane_stride = p.plane_stride;
        ep.out_col0 = col0;
        ep.Tp = Tp;
        ep.P = P;
        ep.T = T;
        ep.halo = halo ? 1 : 0;
        ep.relu = 1;
        return ep;
    };
    rc = add_gemm(m->conv0, spec_conv0(m), nullptr, 0, int(R), planes_out(m->buf.bufs[B_X0], 0, false));
    if (rc) return rc;
    for (int b = 1; b <= 3; ++b) {
        const Planes& X = (b == 1) ? m->buf.bufs[B_X0] : m->buf.bufs[B_CAT];
        const int xcol = (b == 1) ? 0 : (b - 2) * C;
        // the fused Res2Net chain builds the reflect halo rows itself, so tdnn1 writes no halo rows (and gets the lean epilogue)
        rc = add_gemm(m->tdnn1[b - 1], {{-1, 0, C, 0, 0, C, 0}}, &X, xcol, int(R), planes_out(m->buf.bufs[B_H], 0, !use_res2_chain));
        if (rc) return rc;
        if (use_res2_chain) {  // all seven convs in one kernel, one or two utterances per CTA, operands resident in shared memory (res2chain.cu)
            Planes Wj[RES2CHAIN_MAX];
            const float *bj[RES2CHAIN_MAX], *sj[RES2CHAIN_MAX], *hj[RES2CHAIN_MAX];
            for (int j = 1; j < m->scale; ++j) {
                const ConvW& cw = m->res2[b - 1][j];
                Wj[j - 1] = cw.W;  // the first 3 x 64 columns are the taps of source 0; source 1 repeats the same weights
                bj[j - 1] = cw.bias;
                sj[j - 1] = cw.bn_scale;
                hj[j - 1] = cw.bn_shift;
            }
            Step stp;
            stp.kind = Step::RES2CHAIN;
            rc = res2chain_build(&stp.cp, m->buf.bufs[B_H], m->buf.bufs[B_Y], Wj, bj, sj, hj, m->scale - 1, B, T, P, Tp, m->cfg.dilations[b],
                                 res2_paired);
            if (rc) return rc;
            m->steps.push_back(stp);
        }
        for (int j = 1; j < m->scale && !use_res2_chain; ++j) {
            if (use_res2_kernel) {  // weight-stationary kernel, one tall tile per source (res2conv.cu)
                GemmSource srcs[2];
                srcs[0] = GemmSource{m->buf.bufs[B_H], j * w, w, 0};
                srcs[1] = GemmSource{m->buf.bufs[B_Y], (j - 1) * w, w, 0};
                Epilogue ep = planes_out(m->buf.bufs[B_Y], j * w, true);
                const ConvW& cw = m->res2[b - 1][j];
                ep.bias = cw.bias;
                ep.bn_scale = cw.bn_scale;
                ep.bn_shift = cw.bn_shift;
                Step stp;
                stp.kind = Step::RES2;
                rc = res2conv_build(&stp.rp, srcs, j >= 2 ? 2 : 1, cw.W, int(R), m->cfg.dilations[b], ep);
                if (rc) return rc;
                m->steps.push_back(stp);
            } else {
                rc = add_gemm(m->res2[b - 1][j], spec_res2(m, b, j), nullptr, 0, int(R), planes_out(m->buf.bufs[B_Y], j * w, true));
                if (rc) return rc;
            }
        }
        rc = add_gemm(m->tdnn2[b - 1], {{B_H, 0, w, 0, 0, w, 0}, {B_Y, w, C - w, 0, w, C - w, 0}}, nullptr, 0, int(R),
                      planes_out(m->buf.bufs[B_Z], 0, false));
        if (rc) return rc;
        Step s;
        s.blk = b;
        s.kind = Step::SE_SQUEEZE;
        m->steps.push_back(s);
        {  // s = sigmoid(W2 relu(W1 mean + b1) + b2): [B,C] -> [B,S] -> [B,C], plain (un-padded) row layout
            Epilogue e1;
            e1.out_mode = OUT_PLANES;
            e1.out = m->buf.bufs[B_SEH].base;
            e1.out_ld = m->buf.bufs[B_SEH].ld;
            e1.out_plane_stride = m->buf.bufs[B_SEH].plane_stride;
            e1.relu = 1;
            rc = add_gemm(m->se1[b - 1], {{B_SEM, 0, C, 0, 0, 0, 0}}, nullptr, 0, B, e1);
            if (rc) return rc;
            Epilogue e2;
            e2.out_mode = OUT_F32;
            e2.out = m->buf.se_scale;
            e2.out_ld = C;
            e2.sigmoid_ = 1;
            rc = add_gemm(m->se2[b - 1], {{B_SEH, 0, m->se, 0, 0, 0, 0}}, nullptr, 0, B, e2);
            if (rc) return rc;
        }
        s.kind = Step::SE_SCALE;
        m->steps.push_back(s);
    }
    rc = add_gemm(m->mfa, {{B_CAT, 0, C3, 0, 0, C3, 0}}, nullptr, 0, int(R), planes_out(m->buf.bufs[B_MFA], 0, false));
    if (rc) return rc;
    const int pooling = m->cfg.pooling;
    if (pooling == PPV_POOL_TAP || pooling == PPV_POOL_TSP) {
        Step s;  // mean (TAP) or mean | unbiased variance (TSP) over time, straight into the fc operand
        s.kind = Step::POOL_STATS;
        m->steps.push_back(s);
    } else {
        Step s;
        s.kind = Step::ASP_GLOBAL;
        m->steps.push_back(s);
    }
    if (pooling == PPV_POOL_ASP && m->cfg.global_context) {  // fold: [B, 2*C3] . W[:, C3:3*C3]^T -> per-utterance bias [B, att]  (no conv bias here)
        Epilogue ep;
        ep.out_mode = OUT_F32;
        ep.out = m->buf.fold_out;
        ep.out_ld = m->att;
        ConvW cw = m->fold;
        cw.bias = nullptr;
        rc = add_gemm(cw, {{B_GSTAT, 0, 2 * C3, 0, 0, 0, 0}}, nullptr, 0, B, ep);
        if (rc) return rc;
    }
    if (pooling == PPV_POOL_ASP || pooling == PPV_POOL_SAP) {
        {  // ASP: attention TDNN (K = C3) + per-utterance bias -> ReLU -> BN -> tanh;  SAP: tanh(linear1(x))
            Epilogue ep = planes_out(m->buf.bufs[B_ATT], 0, false);
            if (pooling == PPV_POOL_ASP) {
                if (m->cfg.global_context) ep.rowgrp_bias = m->buf.fold_out;
            } else {
                ep.relu = 0;
            }
            ep.tanh_ = 1;
            rc = add_gemm(m->att1, {{B_MFA, 0, C3, 0, 0, 0, 0}}, nullptr, 0, int(R), ep);
            if (rc) return rc;
        }
        {  // attention logits (transposed GEMM) + softmax over time + weighted mean / std + asp_bn, fused
            Step s;
            s.kind = Step::ASP_FUSED;
            rc = asp_fused_build(&s.ap, m->att2.W, m->buf.bufs[B_ATT], m->buf.bufs[B_MFA], m->buf.bufs[B_GSTAT], m->aspbn_scale, m->aspbn_shift,
                                 m->buf.bufs[B_POOL], m->buf.pooled_raw, B, T, P, Tp, C3, m->att, 1e-12f);
            if (rc) return rc;
            m->steps.push_back(s);
        }
    }
    {  // fc: pooled [B, Kp] -> [B, embd]
        Epilogue ep;
        ep.out_mode = OUT_F32;
        ep.out = m->emb_out;
        ep.out_ld = m->cfg.embd_dim;
        const int Kp = (pooling == PPV_POOL_ASP || pooling == PPV_POOL_TSP) ? 2 * C3 : C3;
        rc = add_gemm(m->fc, {{B_POOL, 0, Kp, 0, 0, 0, 0}}, nullptr, 0, B, ep);
        if (rc) return rc;
    }
    return PPV_OK;
}

// ------------------------------------------------------------------------------------------------ forward
int EcapaModel::forward_ex(const float* feat, Fbank* fb, const float* wav, const float* lens_ratio, int B, int T, int L, float* emb, void* ws,
                           size_t ws_bytes, cudaStream_t st, const float* lengths) {
    int rc = forward_begin(emb, B, T);
    if (rc) return rc;
    PPV_REQUIRE((feat != nullptr) != (wav != nullptr), "ecapa_forward: exactly one of feat / wav");
    if (wav) {
        PPV_REQUIRE(fb, "ecapa_forward: wav input needs a fbank handle");
        PPV_REQUIRE(fbank_n_mels(fb) == cfg.input_size, "ecapa_forward: fbank n_mels != model input_size");
        PPV_REQUIRE(fbank_num_frames(fb, L) == T, "ecapa_forward: frame count mismatch");
    }
    rc = update_plan(B, T, ws, ws_bytes, st);
    if (!rc) rc = run(feat, fb, wav, lens_ratio, L, lengths, st);
    return rc ? rc : copy_embeddings(emb, st);
}

int ecapa_forward(Model* m, const float* feat, Fbank* fb, const float* wav, const float* lens_ratio, int B, int T, int L, float* emb, void* ws,
                  size_t ws_bytes, cudaStream_t st, const float* lengths) {
    return static_cast<EcapaModel*>(m)->forward_ex(feat, fb, wav, lens_ratio, B, T, L, emb, ws, ws_bytes, st, lengths);
}

// Launches the plan's steps on features or, with `wav`, on the fbank of the waveforms.
int EcapaModel::run(const float* feat, Fbank* fb, const float* wav, const float* lens_ratio, int L, const float* lengths, cudaStream_t st) {
    EcapaModel* const m = this;
    const int B = m->plan_B, T = m->plan_T;
    const int Tp = m->Tp, P = m->P, C = m->C, C3 = m->C3;
    const int64_t R = int64_t(B) * Tp;
    int rc;
    auto prof_mark = [&](int kind, bool begin) {
        if (!m->prof_on) return;
        if (begin) {
            if (m->prof_used + 2 > m->prof_ev.size()) {
                cudaEvent_t a, b;
                cudaEventCreate(&a);
                cudaEventCreate(&b);
                m->prof_ev.push_back(a);
                m->prof_ev.push_back(b);
                m->prof_kind.push_back(kind);
            }
            m->prof_kind[m->prof_used / 2] = kind;
            cudaEventRecord(m->prof_ev[m->prof_used], st);
        } else {
            cudaEventRecord(m->prof_ev[m->prof_used + 1], st);
            m->prof_used += 2;
        }
    };
    // `lengths` (ecapa_tdnn.py:245, relative lengths in (0,1]): SEBlock squeezes and ASP pools over the first
    // #{t : t < lengths[b] * T} frames of each utterance (ecapa_tdnn.py:71-75, pooling.py:96-115); everything else sees all T frames.
    const int* nv = nullptr;
    if (lengths) {
        PPV_REQUIRE(m->cfg.pooling == PPV_POOL_ASP, "ecapa_forward: lengths is implemented for ASP pooling (the other heads ignore it in the reference)");
        rc = launch_lengths_to_counts(lengths, B, T, m->buf.nvalid, st);
        if (rc) return rc;
        nv = m->buf.nvalid;
    }
    prof_mark(1, true);
    if (wav) {
        rc = fbank_run(fb, wav, lens_ratio, B, L, m->buf.raw_logmel, nullptr, m->buf.bufs[B_FEAT], P, Tp, st);
        m->launches_other += 3;
    } else {
        rc = launch_pack_features(feat, B, T, m->cfg.input_size, m->buf.bufs[B_FEAT], P, Tp, st);
        m->launches_other += 1;
    }
    prof_mark(1, false);
    if (rc) return rc;
    for (const Step& s : m->steps) {
        const bool tensor_step = (s.kind == Step::GEMM || s.kind == Step::ASP_FUSED || s.kind == Step::RES2 || s.kind == Step::RES2CHAIN);
        // (SKINNY steps count as "other kernels": their FLOPs are not credited to the tensor-core roofline)
        prof_mark(tensor_step ? 0 : 1, true);
        if (tensor_step) m->launches_gemm += 1; else m->launches_other += 1;
        switch (s.kind) {
            case Step::GEMM: rc = gemm_launch(s.gp, m->precision, m->num_sms, st); break;
            case Step::SKINNY: rc = skinny_linear_launch(s.sk_x, s.sk_col0, s.sk_w, s.sk_M, s.sk_N, s.sk_K, s.sk_ep, st); break;
            case Step::RES2: rc = res2conv_launch(s.rp, m->precision, m->num_sms, st); break;
            case Step::RES2CHAIN:
                rc = res2chain_launch(s.cp, m->precision, m->num_sms, st);
                if (s.cp.trace) {
                    static int dumps = 0;
                    if (++dumps == 10) res2chain_trace_dump(s.cp);  // a warm launch of the first block
                }
                break;
            case Step::SE_SQUEEZE:
                rc = launch_colstats(m->buf.bufs[B_Z], 0, C, B, T, P, Tp, 0, 0.f, nullptr, m->buf.bufs[B_SEM], st, 0.f, nv);
                break;
            case Step::SE_SCALE: {
                const Planes& X = (s.blk == 1) ? m->buf.bufs[B_X0] : m->buf.bufs[B_CAT];
                const int xcol = (s.blk == 1) ? 0 : (s.blk - 2) * C;
                rc = launch_se_scale_res(m->buf.bufs[B_Z], m->buf.se_scale, X, xcol, m->buf.bufs[B_CAT], (s.blk - 1) * C, C, Tp, R, m->num_sms, st);
                break;
            }
            case Step::ASP_GLOBAL:
                rc = launch_colstats(m->buf.bufs[B_MFA], 0, C3, B, T, P, Tp, 1, 1e-12f, nullptr, m->buf.bufs[B_GSTAT], st, 0.f, nv);
                break;
            case Step::ASP_FUSED: {
                AspFusedParams ap = s.ap;
                ap.nvalid = nv;
                rc = asp_fused_launch(ap, m->precision, m->num_sms, st);
                break;
            }
            case Step::POOL_STATS:
                rc = launch_colstats(m->buf.bufs[B_MFA], 0, C3, B, T, P, Tp, m->cfg.pooling == PPV_POOL_TAP ? 0 : 3, 0.f, nullptr, m->buf.bufs[B_POOL], st);
                break;
        }
        prof_mark(0, false);
        if (rc) return rc;
    }
    return PPV_OK;
}

int ecapa_profile(Model* model, int enable) {
    EcapaModel* m = static_cast<EcapaModel*>(model);
    m->prof_on = enable != 0;
    m->prof_used = 0;
    m->launches_gemm = m->launches_other = 0;
    return PPV_OK;
}

// Sums the event-pair durations recorded since ecapa_profile(m, 1); synchronises on the last event.
int ecapa_profile_read(Model* model, double* gemm_ms, double* other_ms, int64_t* gemm_launches, int64_t* other_launches) {
    EcapaModel* m = static_cast<EcapaModel*>(model);
    PPV_REQUIRE(gemm_ms && other_ms && gemm_launches && other_launches, "ecapa_profile_read: null argument");
    double g = 0, o = 0;
    if (m->prof_used >= 2) PPV_CUDA_OK(cudaEventSynchronize(m->prof_ev[m->prof_used - 1]));
    for (size_t i = 0; i + 1 < m->prof_used; i += 2) {
        float ms = 0.f;
        PPV_CUDA_OK(cudaEventElapsedTime(&ms, m->prof_ev[i], m->prof_ev[i + 1]));
        (m->prof_kind[i / 2] == 0 ? g : o) += ms;
    }
    *gemm_ms = g;
    *other_ms = o;
    *gemm_launches = m->launches_gemm;
    *other_launches = m->launches_other;
    m->prof_used = 0;
    m->launches_gemm = m->launches_other = 0;
    return PPV_OK;
}

int EcapaModel::tap(const std::string& n, float* out, size_t out_elems, cudaStream_t st) {
    EcapaModel* const m = this;
    const int B = m->plan_B, T = m->plan_T, P = m->P, Tp = m->Tp, C = m->C, C3 = m->C3;
    const Planes* src = nullptr;
    int col0 = 0, cols = 0;
    if (n == "feat") {
        src = &m->buf.bufs[B_FEAT];
        cols = m->cfg.input_size;
    } else if (n == "blocks.0") {
        src = &m->buf.bufs[B_X0];
        cols = C;
    } else if (n == "blocks.1" || n == "blocks.2" || n == "blocks.3") {
        src = &m->buf.bufs[B_CAT];
        col0 = (n.back() - '1') * C;
        cols = C;
    } else if (n == "mfa") {
        src = &m->buf.bufs[B_MFA];
        cols = C3;
    } else if (n == "asp") {
        PPV_REQUIRE(out_elems >= size_t(B) * 2 * C3, "ecapa_read_tap: output too small");
        PPV_CUDA_OK(cudaMemcpyAsync(out, m->buf.pooled_raw, size_t(B) * 2 * C3 * 4, cudaMemcpyDeviceToDevice, st));
        return PPV_OK;
    } else {
        return fail(PPV_EINVAL, "ecapa_read_tap: unknown tap " + n);
    }
    PPV_REQUIRE(out_elems >= size_t(B) * T * cols, "ecapa_read_tap: output too small");
    return launch_planes_to_f32(*src, col0, cols, B, T, P, Tp, out, st);
}

}  // namespace ppv
