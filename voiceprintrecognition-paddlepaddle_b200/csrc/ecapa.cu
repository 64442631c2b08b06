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
#include "plan.h"

namespace ppv {

namespace {

struct ConvW : GemmWeights {  // + BatchNorm(eval) after the ReLU, as y = y * bn_scale + bn_shift
    float* bn_scale = nullptr;
    float* bn_shift = nullptr;
};

struct EcBuffers {  // the workspace of a plan
    Planes feat, x0, h, y, z, cat, mfa, att, gstat, pool, sem, seh;
    float *se_mean = nullptr, *se_scale = nullptr, *fold_out = nullptr, *pooled_raw = nullptr, *raw_logmel = nullptr;
    int* nvalid = nullptr;  // [B] valid-frame counts of the current forward (`lengths`)
};

}  // namespace

struct EcapaModel : PlanModel, EcapaGeometry {
    ppv_ecapa_cfg cfg;
    // device weights
    ConvW conv0, tdnn1[3], res2[3][8], tdnn2[3], se1[3], se2[3], mfa, fold, att1, att2, fc;
    float *aspbn_scale = nullptr, *aspbn_shift = nullptr;
    // plan
    EcBuffers buf;
    int Tp = 0;

    EcapaModel(const ppv_ecapa_cfg& c, const EcapaGeometry& g) : PlanModel("ecapa", c.precision), EcapaGeometry(g), cfg(c) {
        // 128-wide n-tiles even where N allows 256: on an H100 SXM at 700 W (tools/gemm_bench.py, M = 78 336,
        // profiles/gemm_bench_after.txt) BN = 128 with 64-wide k-steps takes 15-18 % less time than BN = 256 at every large layer of
        // the model (N x K = 512 x 512 / 640, 1536 x 1536, split-bf16 x3), and no BN = 256 variant beats it by more than run-to-run noise.
        max_bn = 128;
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
    EcapaGeometry g;
    int rc = ecapa_geometry(*cfg, &g);
    if (rc) return rc;
    if (cfg->dilations[4] != 1) return fail(PPV_EUNSUPPORTED, "ecapa: kernel sizes must be [odd,3,3,3,1]");
    if (cfg->attention_channels % 64 || cfg->embd_dim % 32 || cfg->se_channels <= 0 || cfg->se_channels % 64)
        return fail(PPV_EUNSUPPORTED, "ecapa: attention_channels % 64, se_channels % 64, embd_dim % 32 required");
    if (cfg->pooling < PPV_POOL_ASP || cfg->pooling > PPV_POOL_TSP) return fail(PPV_EUNSUPPORTED, "ecapa: pooling must be PPV_POOL_ASP / SAP / TAP / TSP");
    *out = new EcapaModel(*cfg, g);
    return PPV_OK;
}

// ------------------------------------------------------------------------------------------------ finalize
bool EcapaModel::prepare_weights(ArenaBuilder& ab) {
    const int w = width, F = cfg.input_size, A = att, S = se, E = cfg.embd_dim;
    const int k0 = cfg.kernel_sizes[0];
    // conv weight [N, Cin, k] -> split planes [2][N rounded up to 128][K], K in the order of `groups` (conv_weight_matrix)
    auto put_weights = [&](ConvW* cw, const float* wv, int N, int Cin, int k, const std::vector<ConvKGroup>& groups) {
        const std::vector<double> mtx = conv_weight_matrix(wv, N, Cin, k, N, groups);
        ab.put_matrix(cw, mtx, N, int(mtx.size() / N), 128);
    };
    // a conv with its bias and, unless `bn` is empty, the BatchNorm after its ReLU
    auto conv_layer = [&](ConvW* cw, const std::string& name, int N, int Cin, int k, const std::vector<ConvKGroup>& groups,
                          const std::string& bn) -> bool {
        const HostWeight* hw = ab.get(name + ".weight", {N, Cin, k});
        if (!hw) return false;
        put_weights(cw, hw->v.data(), N, Cin, k, groups);
        const HostWeight* hb = ab.get(name + ".bias", {N});
        if (!hb) return false;
        ab.put_f32(&cw->bias, hb->v);
        return bn.empty() || ab.put_bn(&cw->bn_scale, &cw->bn_shift, bn, N, N);
    };
    auto all_cols = [](int Cin) { return std::vector<ConvKGroup>{{1, Cin, 0, Cin, 0}}; };  // a 1x1 conv reading Cin columns
    bool ok = conv_layer(&conv0, "blocks.0.conv.conv", C, F, k0, {{k0, Fp, 0, F, 0}}, "blocks.0.norm.norm");
    for (int b = 1; b <= 3 && ok; ++b) {
        const std::string p = "blocks." + std::to_string(b);
        ok = ok && conv_layer(&tdnn1[b - 1], p + ".tdnn1.conv.conv", C, C, 1, all_cols(C), p + ".tdnn1.norm.norm");
        for (int j = 1; j < scale && ok; ++j) {
            // three taps of chunk j, then from j = 2 the same weights again for the three taps of conv j-1's output (x_j + y_{j-1})
            std::vector<ConvKGroup> groups = {{3, w, 0, w, 0}};
            if (j >= 2) groups.push_back({3, w, 0, w, 0});
            const std::string q = p + ".res2net_block.blocks." + std::to_string(j - 1);
            ok = ok && conv_layer(&res2[b - 1][j], q + ".conv.conv", w, w, 3, groups, q + ".norm.norm");
        }
        ok = ok && conv_layer(&tdnn2[b - 1], p + ".tdnn2.conv.conv", C, C, 1, {{1, w, 0, w, 0}, {1, C - w, 0, C - w, w}}, p + ".tdnn2.norm.norm");
        // SE excitation as two small linear layers over the [B, C] squeeze (ecapa_tdnn.py:79-80)
        ok = ok && conv_layer(&se1[b - 1], p + ".se_block.conv1.conv", S, C, 1, all_cols(C), "");
        ok = ok && conv_layer(&se2[b - 1], p + ".se_block.conv2.conv", C, S, 1, all_cols(S), "");
    }
    ok = ok && conv_layer(&mfa, "mfa.conv.conv", C3, C3, 1, all_cols(C3), "mfa.norm.norm");
    const int pooling = cfg.pooling;
    // BatchNorm(eval) + Linear after a parameter-free or self-attentive pooling: fc(bn(p)) = (W diag(s)) p + (W t + b), folded here
    auto folded_fc = [&](int Kp) -> bool {
        const HostWeight* wt = ab.get("fc.conv.weight", {E, Kp, 1});
        const HostWeight* bt = ab.get("fc.conv.bias", {E});
        std::vector<double> scd, shd;
        if (!wt || !bt || !ab.bn_affine("asp_bn", Kp, &scd, &shd)) return false;  // paddle.nn.BatchNorm1D: keys asp_bn.weight / ._mean ...
        const std::vector<float> sc(scd.begin(), scd.end()), sh(shd.begin(), shd.end());  // rounded to fp32 first
        std::vector<float> wf(size_t(E) * Kp), bf(E);
        for (int n = 0; n < E; ++n) {
            double acc = bt->v[n];
            for (int k = 0; k < Kp; ++k) {
                wf[size_t(n) * Kp + k] = wt->v[size_t(n) * Kp + k] * sc[k];
                acc += double(wt->v[size_t(n) * Kp + k]) * sh[k];
            }
            bf[n] = float(acc);
        }
        put_weights(&fc, wf.data(), E, Kp, 1, all_cols(Kp));
        ab.put_f32(&fc.bias, bf);
        return true;
    };
    if (pooling == PPV_POOL_ASP) {
        // ASP attention TDNN: weight [A, 3*C3, 1] split into the x part (cols 0..C3) and the [mean;std] part;
        // global_context = False (pooling.py:77-78, 108-109): the TDNN sees x alone, weight [A, C3, 1], no per-utterance bias
        const int ctx = cfg.global_context ? 3 : 1;
        ok = ok && conv_layer(&att1, "asp.tdnn.conv.conv", A, ctx * C3, 1, {{1, C3, 0, C3, 0}}, "asp.tdnn.norm.norm");
        if (ok && cfg.global_context) {
            const HostWeight* hw = ab.get("asp.tdnn.conv.conv.weight", {A, 3 * C3, 1});
            put_weights(&fold, hw->v.data(), A, 3 * C3, 1, {{1, 2 * C3, 0, 2 * C3, C3}});
        }
        ok = ok && conv_layer(&att2, "asp.conv.conv", C3, A, 1, all_cols(A), "");
        ok = ok && conv_layer(&fc, "fc.conv", E, 2 * C3, 1, all_cols(2 * C3), "");
        ok = ok && ab.put_bn(&aspbn_scale, &aspbn_shift, "asp_bn.norm", 2 * C3, 2 * C3);
    } else if (pooling == PPV_POOL_SAP) {
        // SelfAttentivePooling (pooling.py:50-66): alpha = softmax_t(linear2(tanh(linear1(x)))); mean = sum alpha x.  The fused ASP
        // kernel computes exactly this weighted mean (its std half is ignored); linear2's bias cancels in the softmax.
        if (A != 128) {
            ab.err = "SAP pooling uses a 128-channel bottleneck (ecapa_tdnn.py:222): attention_channels must be 128";
            ok = false;
        }
        ok = ok && conv_layer(&att1, "asp.linear1", A, C3, 1, all_cols(C3), "");
        ok = ok && conv_layer(&att2, "asp.linear2", C3, A, 1, all_cols(A), "");
        ok = ok && folded_fc(C3);
        if (ok) {
            ab.put_f32(&aspbn_scale, std::vector<float>(2 * C3, 1.f));
            ab.put_f32(&aspbn_shift, std::vector<float>(2 * C3, 0.f));
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
    eb->feat = cv.planes(R, m->Fp);
    eb->x0 = cv.planes(R, C);
    eb->h = cv.planes(R, C);
    eb->y = cv.planes(R, C);
    eb->z = cv.planes(R, C);
    eb->cat = cv.planes(R, C3);
    eb->mfa = cv.planes(R, C3);
    eb->att = cv.planes(R, m->att);
    eb->gstat = cv.planes(B, 2 * C3);
    eb->pool = cv.planes(B, 2 * C3);
    eb->sem = cv.planes(B, C);
    eb->seh = cv.planes(B, m->se);
    eb->se_mean = static_cast<float*>(cv.take(size_t(B) * C * 4));
    eb->se_scale = static_cast<float*>(cv.take(size_t(B) * C * 4));
    eb->fold_out = static_cast<float*>(cv.take(mc_align_up(B, 128) * m->att * 4));
    eb->pooled_raw = static_cast<float*>(cv.take(size_t(B) * 2 * C3 * 4));
    eb->raw_logmel = static_cast<float*>(cv.take(size_t(B) * T * m->cfg.input_size * 4));
    *emb_out = static_cast<float*>(cv.take(mc_align_up(B, 128) * m->cfg.embd_dim * 4));
    eb->nvalid = static_cast<int*>(cv.take(size_t(B) * sizeof(int)));
}

Epilogue f32_out(float* out, int ld) {
    Epilogue ep;
    ep.out_mode = OUT_F32;
    ep.out = out;
    ep.out_ld = ld;
    return ep;
}

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
    PPV_REQUIRE(T > P, "ecapa: too few frames for the reflect padding");
    int rc = claim_workspace(B, T, ws, ws_bytes, st);
    if (rc) return rc;
    WsCarver cv;
    cv.base = static_cast<uint8_t*>(ws);
    carve(this, cv, B, T, &buf, &emb_out);
    Tp = T + 2 * P;
    steps.clear();
    const int w = width, R = int(int64_t(B) * Tp);
    const bool use_res2_kernel = w == 64;
    // 0 = one launch per Res2Net conv (res2conv.cu) instead of the fused chain; single = the fused chain with one utterance per CTA
    // even where two fit (tests and A/B timing)
    const char* rcenv = getenv("PPV_RES2_CHAIN");
    const bool use_res2_chain = use_res2_kernel && scale == 8 && res2chain_fits(T, P) && !(rcenv && rcenv[0] == '0');
    const bool res2_paired = use_res2_chain && res2chain_pair_fits(T, P) && !(rcenv && strcmp(rcenv, "single") == 0);

    // planes output in the padded time layout: ReLU, then the layer's BatchNorm
    auto planes_out = [&](const Planes& p, int col0, bool halo, const ConvW& cw) {
        Epilogue ep = planes_epilogue(p, col0, Tp, P, T);
        ep.halo = halo ? 1 : 0;
        ep.relu = 1;
        ep.bn_scale = cw.bn_scale;
        ep.bn_shift = cw.bn_shift;
        return ep;
    };
    {
        std::vector<GemmSource> taps;
        const int k0 = cfg.kernel_sizes[0], d0 = cfg.dilations[0];
        for (int j = 0; j < k0; ++j) taps.push_back(GemmSource{buf.feat, 0, Fp, (j - (k0 - 1) / 2) * d0});
        rc = plan_gemm(conv0, taps, R, planes_out(buf.x0, 0, false, conv0));
        if (rc) return rc;
    }
    for (int b = 1; b <= 3; ++b) {
        const Planes& X = (b == 1) ? buf.x0 : buf.cat;
        const int xcol = (b == 1) ? 0 : (b - 2) * C, d = cfg.dilations[b];
        // the fused Res2Net chain builds the reflect halo rows itself, so tdnn1 writes no halo rows (and gets the lean epilogue)
        rc = plan_gemm(tdnn1[b - 1], {GemmSource{X, xcol, C, 0}}, R, planes_out(buf.h, 0, !use_res2_chain, tdnn1[b - 1]));
        if (rc) return rc;
        if (use_res2_chain) {  // all seven convs in one kernel, one or two utterances per CTA, operands resident in shared memory (res2chain.cu)
            Planes Wj[RES2CHAIN_MAX];
            const float *bj[RES2CHAIN_MAX], *sj[RES2CHAIN_MAX], *hj[RES2CHAIN_MAX];
            for (int j = 1; j < scale; ++j) {
                const ConvW& cw = res2[b - 1][j];
                Wj[j - 1] = cw.W;  // the first 3 x 64 columns are the taps of source 0; source 1 repeats the same weights
                bj[j - 1] = cw.bias;
                sj[j - 1] = cw.bn_scale;
                hj[j - 1] = cw.bn_shift;
            }
            PlanStep s;
            s.kind = PlanStep::RES2CHAIN;
            rc = res2chain_build(&s.cp, buf.h, buf.y, Wj, bj, sj, hj, scale - 1, B, T, P, Tp, d, res2_paired);
            if (rc) return rc;
            steps.push_back(s);
        }
        for (int j = 1; j < scale && !use_res2_chain; ++j) {
            const ConvW& cw = res2[b - 1][j];
            Epilogue ep = planes_out(buf.y, j * w, true, cw);
            if (use_res2_kernel) {  // weight-stationary kernel, one tall tile per source (res2conv.cu)
                const GemmSource srcs[2] = {GemmSource{buf.h, j * w, w, 0}, GemmSource{buf.y, (j - 1) * w, w, 0}};
                ep.bias = cw.bias;
                PlanStep s;
                s.kind = PlanStep::RES2;
                rc = res2conv_build(&s.rp, srcs, j >= 2 ? 2 : 1, cw.W, R, d, ep);
                if (rc) return rc;
                steps.push_back(s);
            } else {  // the gather-GEMM over the three taps of chunk j and, from j = 2, of conv j-1's output
                std::vector<GemmSource> srcs;
                for (int tap = 0; tap < 3; ++tap) srcs.push_back(GemmSource{buf.h, j * w, w, (tap - 1) * d});
                if (j >= 2)
                    for (int tap = 0; tap < 3; ++tap) srcs.push_back(GemmSource{buf.y, (j - 1) * w, w, (tap - 1) * d});
                rc = plan_gemm(cw, srcs, R, ep);
                if (rc) return rc;
            }
        }
        rc = plan_gemm(tdnn2[b - 1], {GemmSource{buf.h, 0, w, 0}, GemmSource{buf.y, w, C - w, 0}}, R, planes_out(buf.z, 0, false, tdnn2[b - 1]));
        if (rc) return rc;
        steps.push_back(colstats_step(buf.z, C, B, T, P, Tp, 0, 0.f, buf.sem, 0.f, true));
        {  // s = sigmoid(W2 relu(W1 mean + b1) + b2): [B,C] -> [B,S] -> [B,C], plain (un-padded) row layout
            Epilogue e1 = planes_epilogue(buf.seh);
            e1.relu = 1;
            rc = plan_row_linear(se1[b - 1], GemmSource{buf.sem, 0, C, 0}, B, e1);
            if (rc) return rc;
            Epilogue e2 = f32_out(buf.se_scale, C);
            e2.sigmoid_ = 1;
            rc = plan_row_linear(se2[b - 1], GemmSource{buf.seh, 0, se, 0}, B, e2);
            if (rc) return rc;
        }
        steps.push_back(scale_res_step(buf.z, buf.se_scale, X, xcol, buf.cat, (b - 1) * C, C, Tp, R, false));
    }
    rc = plan_gemm(mfa, {GemmSource{buf.cat, 0, C3, 0}}, R, planes_out(buf.mfa, 0, false, mfa));
    if (rc) return rc;
    const int pooling = cfg.pooling;
    if (pooling == PPV_POOL_TAP || pooling == PPV_POOL_TSP)  // mean (TAP) or mean | unbiased variance (TSP) over time, straight into the fc operand
        steps.push_back(colstats_step(buf.mfa, C3, B, T, P, Tp, pooling == PPV_POOL_TAP ? 0 : 3, 0.f, buf.pool));
    else  // global mean | std: ASP's context statistics
        steps.push_back(colstats_step(buf.mfa, C3, B, T, P, Tp, 1, 1e-12f, buf.gstat, 0.f, true));
    if (pooling == PPV_POOL_ASP && cfg.global_context) {  // fold: [B, 2*C3] . W[:, C3:3*C3]^T -> per-utterance bias [B, att]  (no conv bias here)
        rc = plan_row_linear(fold, GemmSource{buf.gstat, 0, 2 * C3, 0}, B, f32_out(buf.fold_out, att));
        if (rc) return rc;
    }
    if (pooling == PPV_POOL_ASP || pooling == PPV_POOL_SAP) {
        {  // ASP: attention TDNN (K = C3) + per-utterance bias -> ReLU -> BN -> tanh;  SAP: tanh(linear1(x))
            Epilogue ep = planes_out(buf.att, 0, false, att1);
            if (pooling == PPV_POOL_ASP) {
                if (cfg.global_context) ep.rowgrp_bias = buf.fold_out;
            } else {
                ep.relu = 0;
            }
            ep.tanh_ = 1;
            rc = plan_gemm(att1, {GemmSource{buf.mfa, 0, C3, 0}}, R, ep);
            if (rc) return rc;
        }
        {  // attention logits (transposed GEMM) + softmax over time + weighted mean / std + asp_bn, fused
            PlanStep s;
            s.kind = PlanStep::ASP_FUSED;
            rc = asp_fused_build(&s.ap, att2.W, buf.att, buf.mfa, aspbn_scale, aspbn_shift, buf.pool, buf.pooled_raw, B, T, P, Tp, C3,
                                 att, 1e-12f);
            if (rc) return rc;
            steps.push_back(s);
        }
    }
    // fc: pooled [B, Kp] -> [B, embd]
    const int Kp = (pooling == PPV_POOL_ASP || pooling == PPV_POOL_TSP) ? 2 * C3 : C3;
    return plan_row_linear(fc, GemmSource{buf.pool, 0, Kp, 0}, B, f32_out(emb_out, cfg.embd_dim));
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

// Packs the features or, with `wav`, computes the fbank of the waveforms into the first layer's operand, then runs the plan.
int EcapaModel::run(const float* feat, Fbank* fb, const float* wav, const float* lens_ratio, int L, const float* lengths, cudaStream_t st) {
    const int B = plan_B, T = plan_T;
    // `lengths` (ecapa_tdnn.py:245, relative lengths in (0,1]): SEBlock squeezes and ASP pools over the first
    // #{t : t < lengths[b] * T} frames of each utterance (ecapa_tdnn.py:71-75, pooling.py:96-115); everything else sees all T frames.
    const int* nv = nullptr;
    if (lengths) {
        PPV_REQUIRE(cfg.pooling == PPV_POOL_ASP, "ecapa_forward: lengths is implemented for ASP pooling (the other heads ignore it in the reference)");
        int rc = launch_lengths_to_counts(lengths, B, T, buf.nvalid, st);
        if (rc) return rc;
        nv = buf.nvalid;
    }
    int rc;
    prof_begin(1, st);
    if (wav) {
        rc = fbank_run(fb, wav, lens_ratio, B, L, buf.raw_logmel, nullptr, buf.feat, P, Tp, st);
        launches_other += 3;
    } else {
        rc = launch_pack_features(feat, B, T, cfg.input_size, buf.feat, P, Tp, st);
        launches_other += 1;
    }
    prof_end(st);
    return rc ? rc : run_plan(PlanInputs{feat, nv}, st);
}

int ecapa_profile(Model* model, int enable) {
    static_cast<EcapaModel*>(model)->profile(enable != 0);
    return PPV_OK;
}

int ecapa_profile_read(Model* model, double* gemm_ms, double* other_ms, int64_t* gemm_launches, int64_t* other_launches) {
    PPV_REQUIRE(gemm_ms && other_ms && gemm_launches && other_launches, "ecapa_profile_read: null argument");
    return static_cast<EcapaModel*>(model)->profile_read(gemm_ms, other_ms, gemm_launches, other_launches);
}

int EcapaModel::tap(const std::string& n, float* out, size_t out_elems, cudaStream_t st) {
    const int B = plan_B, T = plan_T;
    const Planes* src = nullptr;
    int col0 = 0, cols = 0;
    if (n == "feat") {
        src = &buf.feat;
        cols = cfg.input_size;
    } else if (n == "blocks.0") {
        src = &buf.x0;
        cols = C;
    } else if (n == "blocks.1" || n == "blocks.2" || n == "blocks.3") {
        src = &buf.cat;
        col0 = (n.back() - '1') * C;
        cols = C;
    } else if (n == "mfa") {
        src = &buf.mfa;
        cols = C3;
    } else if (n == "asp") {
        PPV_REQUIRE(out_elems >= size_t(B) * 2 * C3, "ecapa_read_tap: output too small");
        PPV_CUDA_OK(cudaMemcpyAsync(out, buf.pooled_raw, size_t(B) * 2 * C3 * 4, cudaMemcpyDeviceToDevice, st));
        return PPV_OK;
    } else {
        return fail(PPV_EINVAL, "ecapa_read_tap: unknown tap " + n);
    }
    PPV_REQUIRE(out_elems >= size_t(B) * T * cols, "ecapa_read_tap: output too small");
    return launch_planes_to_f32(*src, col0, cols, B, T, P, Tp, out, st);
}

}  // namespace ppv
