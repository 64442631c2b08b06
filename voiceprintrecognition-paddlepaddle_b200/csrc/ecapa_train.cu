// ECAPA-TDNN training step: train-mode forward, AAM-softmax loss, full backward into one flat gradient buffer.
// Reference: ppvector/trainer.py:206-229 (forward -> loss -> backward -> optimizer.step), ppvector/models/ecapa_tdnn.py:245-276,
// ppvector/models/utils.py:96-148 (TDNNBlock = BatchNorm(ReLU(conv)), BatchNorm in TRAIN mode: batch statistics over all
// B*T frames, momentum 0.9), ppvector/models/pooling.py:86-125, ppvector/models/fc.py:41-53, ppvector/loss/aamloss.py:28-53.
// lengths = None, as the reference trainer calls the model (trainer.py:210).
//
// Parameters, gradients and BatchNorm running statistics live in three caller-owned flat fp32 buffers (ppv_trainer_bind) laid
// out in the reference's state_dict order, so that the optimizer is one elementwise kernel (ppv_adam_step) and data-parallel
// training is ONE all-reduce over the gradient buffer (the reference's fleet.distributed_model, trainer.py:318-320).
//
// Every convolution is three tensor-core GEMMs on the wgmma kernel of gemm_wgmma.cu:
//   forward   A = input planes (taps = row offsets),      B = Wf [Cout][taps*Cin]
//   dgrad     A = dz planes (taps = negated row offsets),  B = Wd [Cin][taps*Cout]      -> gradient of the PADDED input
//   wgrad     A = dz^T [Cout][rows], B = x^T [Cin][rows] (tap = column offset), split-K partials summed in a fixed order
// Wf / Wd are re-derived from the flat fp32 parameters at the start of every step.  BatchNorm+ReLU backward, the reflect
// padding fold, SE, ASP and the small dense layers are in train_kernels.cu.
#include <math.h>
#include <stdlib.h>

#include <map>
#include <string>
#include <vector>

#include "common.h"
#include "model_common.h"
#include "train.h"

namespace ppv {

namespace {

constexpr float TR_BN_EPS = 1e-5f;
constexpr float TR_BN_MOMENTUM = 0.9f;  // paddle.nn.BatchNorm1D default
constexpr float TR_ASP_EPS = 1e-12f;

struct TConv {
    std::string name;  // e.g. "blocks.1.tdnn1.conv.conv" (weight [Cout, CinTotal, taps], bias [Cout])
    int Cout = 0, Cin = 0, CinTotal = 0, Cinp = 0, taps = 1, dil = 1;
    int64_t w_off = 0, b_off = 0;
    Planes wf, wd;
    bool dgrad = true;
};
struct TBN {
    std::string name;  // e.g. "blocks.1.tdnn1.norm.norm"
    int C = 0;
    int64_t g_off = 0, b_off = 0, rm_off = 0, rv_off = 0;
    float *mean = nullptr, *rstd = nullptr, *scale = nullptr, *shift = nullptr;  // workspace
};
struct TLayer {  // TDNNBlock
    TConv conv;
    TBN bn;
};

struct TStep {
    enum Kind {
        REPACK, PACK, GEMM, BN_FWD, SE_FWD, SCALE_RES, ASP_HEAD_FWD, ASP_TAIL_FWD, LOSS,
        HEAD_BWD, ASP_BWD, COLSUM, BN_BWD, WGRAD, ASP_CTX_BWD, GRAD_SUM, SE_BWD
    } kind;
    GemmParams gp;
    int a = 0, b = 0;  // small integer arguments (block index, split counts)
    GradSrcList gl;
    BnApplyArgs ap;
    Planes p0, p1;
    int c0 = 0, c1 = 0, C = 0;
    float* f0 = nullptr;
    // WGRAD
    std::vector<GemmParams> wg;
    struct Tr {
        Planes in;
        int col0, C, row0;  // row0: first row of the transposed buffer to write
        int which;          // 0 = TA, 1 = TB
        int shift = 0;      // row shift of the input (first conv tap)
        int ntaps = 1, shift_step = 0, row_step = 0;  // all taps of a conv in one launch
    };
    std::vector<Tr> trs;
    int layer = -1;
};

}  // namespace

struct Trainer {
    ppv_ecapa_cfg cfg;
    int S = 0;  // classes
    int C = 0, C3 = 0, width = 0, scale = 0, Fp = 0, P = 0, att = 0, se = 0, D = 0;
    int num_sms = 132;
    int precision = PPV_PREC_BF16X3;  // PPV_PREC_BF16: single-pass bf16 operands for every forward / data-gradient / weight-gradient GEMM (AMP mode)
    // flat layout
    std::map<std::string, std::pair<int64_t, int64_t>> pmap, smap;  // name -> (offset, numel)
    int64_t n_params = 0, n_stats = 0;
    float *params = nullptr, *grads = nullptr, *stats = nullptr;
    // layers: 0 conv0; per block b (1..3): tdnn1, res2 x7, tdnn2; mfa; att1; (att2 conv only)
    std::vector<TLayer> L;
    int l_conv0 = 0, l_tdnn1[3], l_res[3][8], l_tdnn2[3], l_mfa = 0, l_att1 = 0;
    TConv att2;
    int64_t se1_w[3], se1_b[3], se2_w[3], se2_b[3], aspbn_g = 0, aspbn_b = 0, aspbn_rm = 0, aspbn_rv = 0, fc_w = 0, fc_b = 0, cls_w = 0;
    // plan
    std::vector<TStep> steps;
    void* plan_ws = nullptr;
    int plan_B = 0, plan_T = 0, Tp = 0;
    int64_t R = 0, Rp = 0;
    // buffers
    Planes X0, A0, Y0, At1[3], Yt1[3], Ares[3], RC[3], IN[3], At2[3], Yt2[3], OUTCAT, Amfa, M, Aatt, A4, gstat_pl;
    Planes dlogits, dMd, dA4, dZatt, dMatt, dZmfa, dOUTCAT, Dbuf[3], dZt2[3], dRC[3], dZres[3], DIN[3], dZt1[3], dXt1[3], dZ0, TA, TB;  // per-block gradient buffers stay readable (taps)
    float *logits = nullptr, *se_s[3], *se_g1[3], *se_g2[3], *gstat = nullptr, *fold = nullptr, *pooled = nullptr, *pn = nullptr, *emb = nullptr,
          *cls_logits = nullptr, *loss = nullptr, *aspbn_mean = nullptr, *aspbn_rstd = nullptr;
    float *d_emb = nullptr, *dpn = nullptr, *dpooled = nullptr, *dgs = nullptr, *rs = nullptr, *rb = nullptr, *dg2 = nullptr, *dg1 = nullptr, *ds = nullptr,
          *part = nullptr, *wpart = nullptr;
    size_t part_elems = 0;
    void* aam_ws = nullptr;
    size_t aam_ws_bytes = 0;
};

// ------------------------------------------------------------------------------------------------ create: flat layout
static int64_t tr_add(std::map<std::string, std::pair<int64_t, int64_t>>& m, int64_t& total, const std::string& name, int64_t numel) {
    const int64_t off = total;
    m[name] = {off, numel};
    total += int64_t(mc_align_up(size_t(numel), 8));  // 32-byte aligned tensors (vector loads in the epilogues)
    return off;
}

int trainer_create(const ppv_ecapa_cfg* cfg, int num_classes, Trainer** out) {
    PPV_REQUIRE(cfg && out && num_classes > 1, "trainer_create: bad argument");
    const int C = cfg->channels[0];
    if (cfg->channels[1] != C || cfg->channels[2] != C || cfg->channels[3] != C || cfg->channels[4] != 3 * C)
        return fail(PPV_EUNSUPPORTED, "trainer: channels must be [C,C,C,C,3C]");
    if (cfg->res2net_scale != 8 || C % 512) return fail(PPV_EUNSUPPORTED, "trainer: res2net_scale 8 and channels % 512 == 0 required");
    if (cfg->kernel_sizes[1] != 3 || cfg->kernel_sizes[2] != 3 || cfg->kernel_sizes[3] != 3 || cfg->kernel_sizes[4] != 1 || (cfg->kernel_sizes[0] % 2) == 0)
        return fail(PPV_EUNSUPPORTED, "trainer: kernel sizes must be [odd,3,3,3,1]");
    if (cfg->attention_channels % 64 || cfg->se_channels % 8 || cfg->embd_dim % 8)
        return fail(PPV_EUNSUPPORTED, "trainer: attention_channels % 64, se_channels % 8, embd_dim % 8 required");
    if (cfg->pooling != PPV_POOL_ASP || !cfg->global_context)
        return fail(PPV_EUNSUPPORTED, "trainer: the training step implements pooling_type ASP with global_context");
    Trainer* t = new Trainer();
    t->cfg = *cfg;
    t->S = num_classes;
    t->C = C;
    t->C3 = 3 * C;
    t->scale = 8;
    t->width = C / 8;
    t->Fp = int(mc_align_up(size_t(cfg->input_size), 64));
    t->att = cfg->attention_channels;
    t->se = cfg->se_channels;
    t->D = cfg->embd_dim;
    int P = (cfg->kernel_sizes[0] - 1) / 2 * cfg->dilations[0];
    for (int i = 1; i <= 3; ++i) P = std::max(P, cfg->dilations[i]);
    t->P = P;
    t->num_sms = device_sm_count();

    auto add_layer = [&](const std::string& p, int cin, int cout, int k, int dil, bool dgrad) {
        TLayer l;
        l.conv.name = p + ".conv.conv";
        l.conv.Cout = cout;
        l.conv.Cin = l.conv.CinTotal = cin;
        l.conv.Cinp = int(mc_align_up(size_t(cin), 64));
        l.conv.taps = k;
        l.conv.dil = dil;
        l.conv.dgrad = dgrad;
        l.conv.w_off = tr_add(t->pmap, t->n_params, l.conv.name + ".weight", int64_t(cout) * cin * k);
        l.conv.b_off = tr_add(t->pmap, t->n_params, l.conv.name + ".bias", cout);
        l.bn.name = p + ".norm.norm";
        l.bn.C = cout;
        l.bn.g_off = tr_add(t->pmap, t->n_params, l.bn.name + ".weight", cout);
        l.bn.b_off = tr_add(t->pmap, t->n_params, l.bn.name + ".bias", cout);
        l.bn.rm_off = tr_add(t->smap, t->n_stats, l.bn.name + "._mean", cout);
        l.bn.rv_off = tr_add(t->smap, t->n_stats, l.bn.name + "._variance", cout);
        t->L.push_back(l);
        return int(t->L.size()) - 1;
    };
    // state_dict order of the reference model (ecapa_tdnn.py:145-243)
    t->l_conv0 = add_layer("blocks.0", cfg->input_size, C, cfg->kernel_sizes[0], cfg->dilations[0], false);
    for (int b = 0; b < 3; ++b) {
        const std::string p = "blocks." + std::to_string(b + 1);
        t->l_tdnn1[b] = add_layer(p + ".tdnn1", C, C, 1, 1, true);
        for (int j = 1; j < 8; ++j)
            t->l_res[b][j] = add_layer(p + ".res2net_block.blocks." + std::to_string(j - 1), t->width, t->width, 3, cfg->dilations[b + 1], true);
        t->l_tdnn2[b] = add_layer(p + ".tdnn2", C, C, 1, 1, true);
        t->se1_w[b] = tr_add(t->pmap, t->n_params, p + ".se_block.conv1.conv.weight", int64_t(t->se) * C);
        t->se1_b[b] = tr_add(t->pmap, t->n_params, p + ".se_block.conv1.conv.bias", t->se);
        t->se2_w[b] = tr_add(t->pmap, t->n_params, p + ".se_block.conv2.conv.weight", int64_t(C) * t->se);
        t->se2_b[b] = tr_add(t->pmap, t->n_params, p + ".se_block.conv2.conv.bias", C);
    }
    t->l_mfa = add_layer("mfa", t->C3, t->C3, 1, 1, true);
    t->l_att1 = add_layer("asp.tdnn", 3 * t->C3, t->att, 1, 1, true);
    {
        TConv& c1 = t->L[t->l_att1].conv;  // only the first C3 input channels go through the frame-level GEMM
        c1.Cin = t->C3;
        c1.Cinp = t->C3;
    }
    t->att2.name = "asp.conv.conv";
    t->att2.Cout = t->C3;
    t->att2.Cin = t->att2.CinTotal = t->att2.Cinp = t->att;
    t->att2.w_off = tr_add(t->pmap, t->n_params, "asp.conv.conv.weight", int64_t(t->C3) * t->att);
    t->att2.b_off = tr_add(t->pmap, t->n_params, "asp.conv.conv.bias", t->C3);
    t->aspbn_g = tr_add(t->pmap, t->n_params, "asp_bn.norm.weight", 2 * t->C3);
    t->aspbn_b = tr_add(t->pmap, t->n_params, "asp_bn.norm.bias", 2 * t->C3);
    t->aspbn_rm = tr_add(t->smap, t->n_stats, "asp_bn.norm._mean", 2 * t->C3);
    t->aspbn_rv = tr_add(t->smap, t->n_stats, "asp_bn.norm._variance", 2 * t->C3);
    t->fc_w = tr_add(t->pmap, t->n_params, "fc.conv.weight", int64_t(t->D) * 2 * t->C3);
    t->fc_b = tr_add(t->pmap, t->n_params, "fc.conv.bias", t->D);
    t->cls_w = tr_add(t->pmap, t->n_params, "classifier.weight", int64_t(t->D) * t->S);  // fc.py:30-36: [input_dim, num_speakers]
    *out = t;
    return PPV_OK;
}
void trainer_destroy(Trainer* t) { delete t; }
int64_t trainer_param_count(const Trainer* t) { return t ? t->n_params : 0; }
int64_t trainer_stat_count(const Trainer* t) { return t ? t->n_stats : 0; }
int trainer_lookup(const Trainer* t, const char* name, int64_t* off, int64_t* numel, int* is_stat) {
    PPV_REQUIRE(t && name && off && numel && is_stat, "trainer_lookup: null argument");
    auto it = t->pmap.find(name);
    if (it != t->pmap.end()) {
        *off = it->second.first;
        *numel = it->second.second;
        *is_stat = 0;
        return PPV_OK;
    }
    it = t->smap.find(name);
    if (it != t->smap.end()) {
        *off = it->second.first;
        *numel = it->second.second;
        *is_stat = 1;
        return PPV_OK;
    }
    return fail(PPV_EINVAL, std::string("trainer_lookup: unknown tensor ") + name);
}
int trainer_set_precision(Trainer* t, int precision) {
    PPV_REQUIRE(t, "trainer_set_precision: null handle");
    PPV_REQUIRE(precision == PPV_PREC_BF16X3 || precision == PPV_PREC_BF16, "trainer_set_precision: PPV_PREC_BF16X3 or PPV_PREC_BF16");
    t->precision = precision;
    return PPV_OK;
}

int trainer_bind(Trainer* t, float* params, float* grads, float* stats) {
    PPV_REQUIRE(t && params && grads && stats, "trainer_bind: null argument");
    PPV_REQUIRE(((reinterpret_cast<uintptr_t>(params) | reinterpret_cast<uintptr_t>(grads) | reinterpret_cast<uintptr_t>(stats)) & 31) == 0,
                "trainer_bind: buffers must be 32-byte aligned");
    t->params = params;
    t->grads = grads;
    t->stats = stats;
    t->plan_ws = nullptr;  // pointers are baked into the plan
    return PPV_OK;
}

// ------------------------------------------------------------------------------------------------ workspace
namespace {

struct TrCarve {
    WsCarver cv;
    Planes act(int64_t Rp, int C) { return cv.planes(Rp, C); }
    float* f32(size_t n) { return static_cast<float*>(cv.take(n * sizeof(float))); }
};

// Frame splits of a layer's BatchNorm backward: narrow layers split the frames of an utterance over several CTAs so the
// reduction fills the GPU.  The attention TDNN keeps per-utterance sums, which ASP_CTX_BWD reads back from `part`.
int tr_bn_bwd_tsplit(const Trainer* t, int layer, int B) {
    const int ctas = (t->L[layer].bn.C / 64) * B;
    return (layer == t->l_att1 || ctas >= 2 * t->num_sms) ? 1 : std::min(8, std::max(1, (2 * t->num_sms + ctas - 1) / ctas));
}

void tr_carve(Trainer* t, TrCarve& k, int B, int T) {
    const int Tp = T + 2 * t->P;
    const int64_t R = int64_t(B) * Tp, Rp = int64_t(mc_align_up(size_t(R), 128));
    const int C = t->C, C3 = t->C3;
    t->Tp = Tp;
    t->R = R;
    t->Rp = Rp;
    // weights in GEMM layouts
    auto wplanes = [&](TConv& c) {
        c.wf = k.cv.planes(int64_t(mc_align_up(size_t(c.Cout), 256)), c.taps * c.Cinp);
        if (c.dgrad) c.wd = k.cv.planes(int64_t(mc_align_up(size_t(c.Cinp), 256)), c.taps * c.Cout);
    };
    for (TLayer& l : t->L) {
        wplanes(l.conv);
        l.bn.mean = k.f32(l.bn.C);
        l.bn.rstd = k.f32(l.bn.C);
        l.bn.scale = k.f32(l.bn.C);
        l.bn.shift = k.f32(l.bn.C);
    }
    wplanes(t->att2);
    t->X0 = k.act(Rp, t->Fp);
    t->A0 = k.act(Rp, C);
    t->Y0 = k.act(Rp, C);
    for (int b = 0; b < 3; ++b) {
        t->At1[b] = k.act(Rp, C);
        t->Yt1[b] = k.act(Rp, C);
        t->Ares[b] = k.act(Rp, C);
        t->RC[b] = k.act(Rp, C);
        t->IN[b] = k.act(Rp, C);
        t->At2[b] = k.act(Rp, C);
        t->Yt2[b] = k.act(Rp, C);
        t->se_s[b] = k.f32(size_t(B) * C);
        t->se_g1[b] = k.f32(size_t(B) * t->se);
        t->se_g2[b] = k.f32(size_t(B) * C);
    }
    t->OUTCAT = k.act(Rp, C3);
    t->Amfa = k.act(Rp, C3);
    t->M = k.act(Rp, C3);
    t->Aatt = k.act(Rp, t->att);
    t->A4 = k.act(Rp, t->att);
    t->gstat_pl = k.cv.planes(B, 2 * C3);
    t->logits = k.f32(size_t(Rp) * C3);
    t->gstat = k.f32(size_t(B) * 2 * C3);
    t->fold = k.f32(size_t(B) * t->att);
    t->pooled = k.f32(size_t(B) * 2 * C3);
    t->pn = k.f32(size_t(B) * 2 * C3);
    t->emb = k.f32(size_t(B) * t->D);
    t->cls_logits = k.f32(size_t(B) * t->S);
    t->loss = k.f32(8);
    t->aspbn_mean = k.f32(2 * C3);
    t->aspbn_rstd = k.f32(2 * C3);
    // gradients
    t->dlogits = k.act(Rp, C3);
    t->dMd = k.act(Rp, C3);
    t->dA4 = k.act(Rp, t->att);
    t->dZatt = k.act(Rp, t->att);
    t->dMatt = k.act(Rp, C3);
    t->dZmfa = k.act(Rp, C3);
    t->dOUTCAT = k.act(Rp, C3);
    for (int b = 0; b < 3; ++b) {
        t->Dbuf[b] = k.act(Rp, C);
        t->dZt2[b] = k.act(Rp, C);
        t->dRC[b] = k.act(Rp, C);
        t->dZres[b] = k.act(Rp, C);
        t->DIN[b] = k.act(Rp, C);
        t->dZt1[b] = k.act(Rp, C);
        t->dXt1[b] = k.act(Rp, C);
    }
    t->dZ0 = k.act(Rp, C);
    t->TA = k.cv.planes(C3, int(Rp));
    t->TB = k.cv.planes(C3, int(Rp));
    t->d_emb = k.f32(size_t(B) * t->D);
    t->dpn = k.f32(size_t(B) * 2 * C3);
    t->dpooled = k.f32(size_t(B) * 2 * C3);
    t->dgs = k.f32(size_t(B) * 2 * C3);
    t->rs = k.f32(size_t(B) * C3);
    t->rb = k.f32(size_t(B) * C3);
    t->dg2 = k.f32(size_t(B) * C);
    t->dg1 = k.f32(size_t(B) * t->se);
    t->ds = k.f32(size_t(B) * C);
    // partial sums: BatchNorm forward statistics [B][3][C], per-utterance column sums [B][C], BatchNorm backward [B * tsplit][2][C]
    t->part_elems = size_t(3) * B * C3;
    for (int l = 0; l < int(t->L.size()); ++l)
        t->part_elems = std::max(t->part_elems, size_t(2) * B * tr_bn_bwd_tsplit(t, l, B) * t->L[l].bn.C);
    t->part = k.f32(t->part_elems);
    // weight-gradient partials: max over layers of splits * Mpad * Ktot; splits <= num_sms
    size_t wmax = 0;
    auto wsize = [&](const TConv& c) {
        const size_t N = size_t(c.taps) * c.Cinp, mt = (c.Cout + 127) / 128, bn = gemm_pick_bn(int(N)), nt = (N + bn - 1) / bn;
        const size_t splits = std::max<size_t>(1, std::min<size_t>((t->num_sms + mt * nt - 1) / (mt * nt), (Rp + 63) / 64));
        wmax = std::max(wmax, splits * mt * 128 * N);
    };
    for (const TLayer& l : t->L) wsize(l.conv);
    wsize(t->att2);
    t->wpart = k.f32(wmax);
    t->aam_ws_bytes = aam_workspace_bytes(B, t->D, t->S);
    t->aam_ws = k.cv.take(t->aam_ws_bytes);
}

}  // namespace

size_t trainer_workspace_bytes(Trainer* t, int B, int T) {
    if (!t || B <= 0 || T <= 0) return 0;
    TrCarve k;
    tr_carve(t, k, B, T);
    t->plan_ws = nullptr;  // carving overwrote the plan's buffer views
    return mc_align_up(k.cv.off, 256);
}

// ------------------------------------------------------------------------------------------------ plan
static int tr_build_plan(Trainer* t, int B, int T, void* ws, size_t ws_bytes, cudaStream_t st) {
    PPV_REQUIRE(t->params, "trainer: call ppv_trainer_bind first");
    PPV_REQUIRE(T > 2 * t->P, "trainer: too few frames for the reflect padding");
    TrCarve k;
    tr_carve(t, k, B, T);
    const size_t need = mc_align_up(k.cv.off, 256);
    PPV_REQUIRE(ws && ws_bytes >= need, "trainer: workspace too small (see ppv_trainer_workspace_bytes)");
    PPV_REQUIRE((reinterpret_cast<uintptr_t>(ws) & 255) == 0, "trainer: workspace must be 256-byte aligned");
    k = TrCarve();
    k.cv.base = static_cast<uint8_t*>(ws);
    tr_carve(t, k, B, T);
    PPV_CUDA_OK(cudaMemsetAsync(ws, 0, need, st));
    t->steps.clear();
    const int C = t->C, C3 = t->C3, W = t->width, P = t->P, Tp = t->Tp;
    const int M = int(t->R);
    float* const par = t->params;
    float* const grd = t->grads;
    int rc;

    auto push = [&](const TStep& s) { t->steps.push_back(s); };
    // forward conv: bias + ReLU -> post-activation planes (valid frames)
    auto fwd_gemm = [&](const TConv& c, const std::vector<GemmSource>& srcs, const Planes& out, int out_col0, bool relu, const float* rowgrp,
                        float* out_f32) -> int {
        Epilogue ep;
        ep.bias = par + c.b_off;
        ep.rowgrp_bias = rowgrp;
        ep.relu = relu ? 1 : 0;
        if (out_f32) {
            ep.out_mode = OUT_F32;
            ep.out = out_f32;
            ep.out_ld = c.Cout;
        } else {
            ep.out_mode = OUT_PLANES;
            ep.out = out.base;
            ep.out_ld = out.ld;
            ep.out_plane_stride = out.plane_stride;
            ep.out_col0 = out_col0;
        }
        ep.Tp = Tp;
        ep.P = P;
        ep.T = T;
        TStep s;
        s.kind = TStep::GEMM;
        int r = gemm_build(&s.gp, srcs.data(), int(srcs.size()), c.wf, M, c.Cout, ep, gemm_pick_bn(c.Cout));
        if (r) return r;
        push(s);
        return PPV_OK;
    };
    auto taps_of = [&](const TConv& c, const Planes& x, int col0, int sign) {
        std::vector<GemmSource> v;
        for (int tp = 0; tp < c.taps; ++tp) v.push_back(GemmSource{x, col0, sign > 0 ? c.Cinp : c.Cout, sign * (tp - (c.taps - 1) / 2) * c.dil});
        return v;
    };
    auto bn_fwd = [&](const TLayer& l, const Planes& a, int a_col0, const Planes& y, int y_col0, int tanh_, const Planes* add, int add_col0,
                      const Planes* out2, int out2_col0) {
        TStep s;
        s.kind = TStep::BN_FWD;
        s.layer = int(&l - t->L.data());
        s.p0 = a;
        s.c0 = a_col0;
        s.ap.y = y;
        s.ap.y_col0 = y_col0;
        s.ap.tanh_ = tanh_;
        if (out2) {
            s.ap.add = *add;
            s.ap.add_col0 = add_col0;
            s.ap.out2 = *out2;
            s.ap.out2_col0 = out2_col0;
        }
        push(s);
    };
    // data gradient: dx_pad[r, cin] = sum_tap dz[r - off_tap, :] . W[:, cin, tap]  -> planes on every row
    auto dgrad_gemm = [&](const TConv& c, const Planes& dz, int dz_col0, const Planes& out, int out_col0) -> int {
        Epilogue ep;
        ep.out_mode = OUT_PLANES;
        ep.out = out.base;
        ep.out_ld = out.ld;
        ep.out_plane_stride = out.plane_stride;
        ep.out_col0 = out_col0;
        TStep s;
        s.kind = TStep::GEMM;
        std::vector<GemmSource> srcs = taps_of(c, dz, dz_col0, -1);
        int r = gemm_build(&s.gp, srcs.data(), int(srcs.size()), c.wd, M, c.Cinp, ep, gemm_pick_bn(c.Cinp));
        if (r) return r;
        push(s);
        return PPV_OK;
    };
    // weight gradient: dz^T -> TA; one row-shifted transpose of the layer input per tap -> TB rows [tap * Cinp, ...); ONE GEMM
    // [Cout] x [taps * Cinp] over the frames (split-K partials); unpack into the flat gradient buffer
    auto wgrad = [&](int layer, const TConv& c, const Planes& dz, int dz_col0, const std::vector<TStep::Tr>& xs) -> int {
        TStep s;
        s.kind = TStep::WGRAD;
        s.layer = layer;
        s.trs.push_back(TStep::Tr{dz, dz_col0, c.Cout, 0, 0, 0});
        for (const TStep::Tr& x : xs) {
            TStep::Tr tr{x.in, x.col0, x.C, x.row0, 1, -((c.taps - 1) / 2) * c.dil};
            tr.ntaps = c.taps;
            tr.shift_step = c.dil;
            tr.row_step = c.Cinp;
            s.trs.push_back(tr);
        }
        const int N = c.taps * c.Cinp;
        const int BNw = gemm_pick_bn(N);
        const int mt = (c.Cout + 127) / 128, nt = (N + BNw - 1) / BNw;
        const int splits = std::max(1, std::min((t->num_sms + mt * nt - 1) / (mt * nt), int((t->Rp + 63) / 64)));
        GemmParams gp;
        int r = gemm_build_wgrad(&gp, t->TA, t->TB, c.Cout, N, 0, 0, splits, t->wpart, N, 0, int64_t(mt) * 128, BNw);
        if (r) return r;
        s.wg.push_back(gp);
        s.a = gp.lin_splits;
        s.b = mt * 128;
        push(s);
        return PPV_OK;
    };
    auto src1 = [](const Planes& p, int col0, int fold) {
        GradSrc g;
        g.t = p;
        g.col0 = col0;
        g.fold = fold;
        return g;
    };
    auto bn_bwd = [&](int layer, const GradSrcList& gl, const Planes& a, int a_col0, const Planes& dz, int dz_col0) {
        TStep s;
        s.kind = TStep::BN_BWD;
        s.layer = layer;
        s.gl = gl;
        s.p0 = a;
        s.c0 = a_col0;
        s.p1 = dz;
        s.c1 = dz_col0;
        s.a = tr_bn_bwd_tsplit(t, layer, B);
        push(s);
    };
    auto simple = [&](TStep::Kind kd, int a = 0) {
        TStep s;
        s.kind = kd;
        s.a = a;
        push(s);
    };

    // ================================================================= forward
    simple(TStep::REPACK);
    simple(TStep::PACK);
    {
        const TLayer& l = t->L[t->l_conv0];
        rc = fwd_gemm(l.conv, taps_of(l.conv, t->X0, 0, +1), t->A0, 0, true, nullptr, nullptr);
        if (rc) return rc;
        bn_fwd(l, t->A0, 0, t->Y0, 0, 0, nullptr, 0, nullptr, 0);
    }
    for (int b = 0; b < 3; ++b) {
        const Planes u = b == 0 ? t->Y0 : t->OUTCAT;
        const int uc = b == 0 ? 0 : C * (b - 1);
        {
            const TLayer& l = t->L[t->l_tdnn1[b]];
            rc = fwd_gemm(l.conv, {GemmSource{u, uc, C, 0}}, t->At1[b], 0, true, nullptr, nullptr);
            if (rc) return rc;
            bn_fwd(l, t->At1[b], 0, t->Yt1[b], 0, 0, nullptr, 0, nullptr, 0);
        }
        for (int j = 1; j < 8; ++j) {
            const TLayer& l = t->L[t->l_res[b][j]];
            const Planes& xin = j == 1 ? t->Yt1[b] : t->IN[b];
            rc = fwd_gemm(l.conv, taps_of(l.conv, xin, W * j, +1), t->Ares[b], W * j, true, nullptr, nullptr);
            if (rc) return rc;
            // r_j -> RC window j; in_{j+1} = r_j + chunk_{j+1}(tdnn1 output) -> IN window j+1   (ecapa_tdnn.py:41-45)
            if (j < 7)
                bn_fwd(l, t->Ares[b], W * j, t->RC[b], W * j, 0, &t->Yt1[b], W * (j + 1), &t->IN[b], W * (j + 1));
            else
                bn_fwd(l, t->Ares[b], W * j, t->RC[b], W * j, 0, nullptr, 0, nullptr, 0);
        }
        {
            const TLayer& l = t->L[t->l_tdnn2[b]];
            rc = fwd_gemm(l.conv, {GemmSource{t->Yt1[b], 0, W, 0}, GemmSource{t->RC[b], W, C - W, 0}}, t->At2[b], 0, true, nullptr, nullptr);
            if (rc) return rc;
            bn_fwd(l, t->At2[b], 0, t->Yt2[b], 0, 0, nullptr, 0, nullptr, 0);
        }
        simple(TStep::SE_FWD, b);
        {
            TStep s;
            s.kind = TStep::SCALE_RES;
            s.a = b;
            s.p0 = u;
            s.c0 = uc;
            push(s);
        }
    }
    {
        const TLayer& l = t->L[t->l_mfa];
        rc = fwd_gemm(l.conv, {GemmSource{t->OUTCAT, 0, C3, 0}}, t->Amfa, 0, true, nullptr, nullptr);
        if (rc) return rc;
        bn_fwd(l, t->Amfa, 0, t->M, 0, 0, nullptr, 0, nullptr, 0);
    }
    simple(TStep::ASP_HEAD_FWD);  // global stats -> per-utterance bias of the attention TDNN
    {
        const TLayer& l = t->L[t->l_att1];
        rc = fwd_gemm(l.conv, {GemmSource{t->M, 0, C3, 0}}, t->Aatt, 0, true, t->fold, nullptr);
        if (rc) return rc;
        bn_fwd(l, t->Aatt, 0, t->A4, 0, 1, nullptr, 0, nullptr, 0);
        rc = fwd_gemm(t->att2, {GemmSource{t->A4, 0, t->att, 0}}, Planes(), 0, false, nullptr, t->logits);
        if (rc) return rc;
    }
    simple(TStep::ASP_TAIL_FWD);  // softmax pooling, asp_bn (batch statistics), fc
    simple(TStep::LOSS);

    // ================================================================= backward
    simple(TStep::HEAD_BWD);  // AAM, fc, asp_bn -> dpooled
    simple(TStep::ASP_BWD);   // -> dlogits, dMd
    {
        // asp.conv: bias, weight, data gradients
        TStep s;
        s.kind = TStep::COLSUM;
        s.gl.n = 1;
        s.gl.s[0] = src1(t->dlogits, 0, 0);
        s.C = C3;
        s.f0 = grd + t->att2.b_off;
        push(s);
        rc = wgrad(-1, t->att2, t->dlogits, 0, {TStep::Tr{t->A4, 0, t->att, 0, 1}});
        if (rc) return rc;
        rc = dgrad_gemm(t->att2, t->dlogits, 0, t->dA4, 0);
        if (rc) return rc;
    }
    {
        // attention TDNN: tanh, BN, ReLU backward; frame-level weight / data gradients; per-utterance context gradients
        GradSrcList gl;
        gl.n = 1;
        gl.s[0] = src1(t->dA4, 0, 0);
        gl.s[0].dtanh = t->A4;
        bn_bwd(t->l_att1, gl, t->Aatt, 0, t->dZatt, 0);
        simple(TStep::ASP_CTX_BWD);
        const TConv& c = t->L[t->l_att1].conv;
        rc = wgrad(t->l_att1, c, t->dZatt, 0, {TStep::Tr{t->M, 0, C3, 0, 1}});
        if (rc) return rc;
        rc = dgrad_gemm(c, t->dZatt, 0, t->dMatt, 0);
        if (rc) return rc;
    }
    {
        // MFA: d(M) = ASP direct + attention path + global-context statistics (as row scale / bias on M itself)
        GradSrcList gl;
        gl.n = 3;
        gl.s[0] = src1(t->dMd, 0, 0);
        gl.s[1] = src1(t->dMatt, 0, 0);
        gl.s[2] = src1(t->M, 0, 0);
        gl.s[2].rowscale = t->rs;
        gl.s[2].rowbias = t->rb;
        gl.s[2].row_ld = C3;
        bn_bwd(t->l_mfa, gl, t->Amfa, 0, t->dZmfa, 0);
        const TConv& c = t->L[t->l_mfa].conv;
        rc = wgrad(t->l_mfa, c, t->dZmfa, 0, {TStep::Tr{t->OUTCAT, 0, C3, 0, 1}});
        if (rc) return rc;
        rc = dgrad_gemm(c, t->dZmfa, 0, t->dOUTCAT, 0);
        if (rc) return rc;
    }
    for (int b = 2; b >= 0; --b) {
        const Planes u = b == 0 ? t->Y0 : t->OUTCAT;
        const int uc = b == 0 ? 0 : C * (b - 1);
        const Planes& D = t->Dbuf[b];
        {
            // d(out_b) = MFA window + (next block: tdnn1 data gradient + its own residual gradient)
            TStep s;
            s.kind = TStep::GRAD_SUM;
            s.gl.n = 1;
            s.gl.s[0] = src1(t->dOUTCAT, C * b, 0);
            if (b < 2) {
                s.gl.n = 3;
                s.gl.s[1] = src1(t->dXt1[b + 1], 0, 0);
                s.gl.s[2] = src1(t->Dbuf[b + 1], 0, 0);
            }
            s.C = C;
            s.p0 = D;
            s.c0 = 0;
            push(s);
        }
        simple(TStep::SE_BWD, b);  // -> dg2 ... ds (scaled by 1/T), SE weight gradients
        {
            GradSrcList gl;
            gl.n = 1;
            gl.s[0] = src1(D, 0, 0);
            gl.s[0].rowscale = t->se_g2[b];
            gl.s[0].rowbias = t->ds;
            gl.s[0].row_ld = C;
            bn_bwd(t->l_tdnn2[b], gl, t->At2[b], 0, t->dZt2[b], 0);
            const TConv& c = t->L[t->l_tdnn2[b]].conv;
            rc = wgrad(t->l_tdnn2[b], c, t->dZt2[b], 0, {TStep::Tr{t->Yt1[b], 0, W, 0, 1}, TStep::Tr{t->RC[b], W, C - W, W, 1}});
            if (rc) return rc;
            rc = dgrad_gemm(c, t->dZt2[b], 0, t->dRC[b], 0);
            if (rc) return rc;
        }
        for (int j = 7; j >= 1; --j) {
            GradSrcList gl;
            gl.n = 1;
            gl.s[0] = src1(t->dRC[b], W * j, 0);
            if (j < 7) {
                gl.n = 2;
                gl.s[1] = src1(t->DIN[b], W * (j + 1), 1);
            }
            const int li = t->l_res[b][j];
            bn_bwd(li, gl, t->Ares[b], W * j, t->dZres[b], W * j);
            const TConv& c = t->L[li].conv;
            rc = wgrad(li, c, t->dZres[b], W * j, {TStep::Tr{j == 1 ? t->Yt1[b] : t->IN[b], W * j, W, 0, 1}});
            if (rc) return rc;
            rc = dgrad_gemm(c, t->dZres[b], W * j, t->DIN[b], W * j);
            if (rc) return rc;
        }
        {
            // chunk 0 of the tdnn1 output went straight into tdnn2: copy its gradient next to the others
            TStep s;
            s.kind = TStep::GRAD_SUM;
            s.gl.n = 1;
            s.gl.s[0] = src1(t->dRC[b], 0, 0);
            s.C = W;
            s.p0 = t->DIN[b];
            s.c0 = 0;
            push(s);
        }
        {
            GradSrcList gl;
            gl.n = 1;
            gl.s[0] = src1(t->DIN[b], 0, 1);
            bn_bwd(t->l_tdnn1[b], gl, t->At1[b], 0, t->dZt1[b], 0);
            const TConv& c = t->L[t->l_tdnn1[b]].conv;
            rc = wgrad(t->l_tdnn1[b], c, t->dZt1[b], 0, {TStep::Tr{u, uc, C, 0, 1}});
            if (rc) return rc;
            rc = dgrad_gemm(c, t->dZt1[b], 0, t->dXt1[b], 0);
            if (rc) return rc;
        }
    }
    {
        GradSrcList gl;
        gl.n = 2;
        gl.s[0] = src1(t->dXt1[0], 0, 0);
        gl.s[1] = src1(t->Dbuf[0], 0, 0);
        bn_bwd(t->l_conv0, gl, t->A0, 0, t->dZ0, 0);
        const TConv& c = t->L[t->l_conv0].conv;
        rc = wgrad(t->l_conv0, c, t->dZ0, 0, {TStep::Tr{t->X0, 0, t->Fp, 0, 1}});
        if (rc) return rc;
    }
    t->plan_ws = ws;
    t->plan_B = B;
    t->plan_T = T;
    return PPV_OK;
}

// ------------------------------------------------------------------------------------------------ step
int trainer_forward_backward(Trainer* t, const float* feat, const int64_t* labels, int B, int T, float margin, float scale, int easy_margin,
                             float label_smoothing, float* loss_out, float* logits_out, void* ws, size_t ws_bytes, cudaStream_t st) {
    PPV_REQUIRE(t && feat && labels, "trainer_forward_backward: null argument");
    PPV_REQUIRE(B > 1 && T > 0, "trainer_forward_backward: batch of at least 2 required (batch statistics)");
    if (t->plan_ws != ws || t->plan_B != B || t->plan_T != T) {
        int rc = tr_build_plan(t, B, T, ws, ws_bytes, st);
        if (rc) {
            t->plan_ws = nullptr;
            return rc;
        }
    }
    float* const par = t->params;
    float* const grd = t->grads;
    float* const sta = t->stats;
    const int C = t->C, C3 = t->C3, P = t->P, Tp = t->Tp, se = t->se, att = t->att, D = t->D;
    int rc = PPV_OK;
    static const bool debug_sync = getenv("PPV_TRAIN_DEBUG") != nullptr;  // localise a faulting kernel: sync after every step
    int step_idx = 0;
    for (const TStep& s : t->steps) {
        if (debug_sync) {
            cudaError_t e = cudaStreamSynchronize(st);
            if (e != cudaSuccess)
                return fail(PPV_ECUDA, "trainer: step " + std::to_string(step_idx - 1) + " (kind " + std::to_string(int(t->steps[std::max(step_idx - 1, 0)].kind)) +
                                           ", layer " + std::to_string(t->steps[std::max(step_idx - 1, 0)].layer) + ") failed: " + cudaGetErrorString(e));
        }
        ++step_idx;
        switch (s.kind) {
            case TStep::REPACK: {
                for (const TLayer& l : t->L) {
                    rc = tr_repack_conv(par + l.conv.w_off, int64_t(l.conv.CinTotal) * l.conv.taps, l.conv.Cout, l.conv.Cin, l.conv.Cinp, l.conv.taps,
                                        l.conv.wf, l.conv.dgrad ? l.conv.wd : Planes(), st);
                    if (rc) return rc;
                }
                rc = tr_repack_conv(par + t->att2.w_off, t->att2.CinTotal, t->att2.Cout, t->att2.Cin, t->att2.Cinp, 1, t->att2.wf, t->att2.wd, st);
                break;
            }
            case TStep::PACK: rc = launch_pack_features(feat, B, T, t->cfg.input_size, t->X0, P, Tp, st); break;
            case TStep::GEMM: rc = gemm_launch(s.gp, t->precision, t->num_sms, st); break;
            case TStep::BN_FWD: {
                const TBN& bn = t->L[s.layer].bn;
                rc = tr_bn_forward(s.p0, s.c0, bn.C, B, T, P, Tp, TR_BN_EPS, TR_BN_MOMENTUM, par + bn.g_off, par + bn.b_off, bn.mean, bn.rstd, bn.scale,
                                   bn.shift, sta + bn.rm_off, sta + bn.rv_off, t->part, s.ap, t->num_sms, st);
                break;
            }
            case TStep::SE_FWD: {
                const int b = s.a;
                rc = launch_colstats(t->Yt2[b], 0, C, B, T, P, Tp, 0, 0.f, t->se_s[b], Planes(), st);
                if (rc) return rc;
                rc = tr_dense_fwd(t->se_s[b], C, par + t->se1_w[b], C, par + t->se1_b[b], B, se, C, 1, t->se_g1[b], se, st);
                if (rc) return rc;
                rc = tr_dense_fwd(t->se_g1[b], se, par + t->se2_w[b], se, par + t->se2_b[b], B, C, se, 2, t->se_g2[b], C, st);
                break;
            }
            case TStep::SCALE_RES:
                rc = launch_se_scale_res(t->Yt2[s.a], t->se_g2[s.a], s.p0, s.c0, t->OUTCAT, C * s.a, C, Tp, t->R, t->num_sms, st);
                break;
            case TStep::ASP_HEAD_FWD: {
                rc = launch_colstats(t->M, 0, C3, B, T, P, Tp, 1, TR_ASP_EPS, nullptr, t->gstat_pl, st);
                if (rc) return rc;
                rc = launch_planes_to_f32(t->gstat_pl, 0, 2 * C3, B, 1, 0, 1, t->gstat, st);
                if (rc) return rc;
                const TConv& c = t->L[t->l_att1].conv;  // weight [att][3*C3]: columns C3.. multiply [mean | std]
                rc = tr_dense_fwd(t->gstat, 2 * C3, par + c.w_off + C3, 3 * C3, nullptr, B, att, 2 * C3, 0, t->fold, att, st);
                break;
            }
            case TStep::ASP_TAIL_FWD: {
                rc = launch_asp_pool(t->logits, C3, t->M, C3, B, T, P, Tp, TR_ASP_EPS, nullptr, nullptr, Planes(), t->pooled, st);
                if (rc) return rc;
                rc = tr_bn1d_fwd(t->pooled, B, 2 * C3, TR_BN_EPS, TR_BN_MOMENTUM, par + t->aspbn_g, par + t->aspbn_b, t->pn, t->aspbn_mean, t->aspbn_rstd,
                                 sta + t->aspbn_rm, sta + t->aspbn_rv, st);
                if (rc) return rc;
                rc = tr_dense_fwd(t->pn, 2 * C3, par + t->fc_w, 2 * C3, par + t->fc_b, B, D, 2 * C3, 0, t->emb, D, st);
                break;
            }
            case TStep::LOSS:
                rc = aam_forward(t->emb, par + t->cls_w, labels, B, D, t->S, margin, scale, easy_margin, label_smoothing, t->cls_logits, t->loss,
                                 t->aam_ws, t->aam_ws_bytes, st);
                break;
            case TStep::HEAD_BWD: {
                rc = aam_backward(t->emb, par + t->cls_w, labels, t->cls_logits, B, D, t->S, margin, scale, easy_margin, label_smoothing, t->d_emb,
                                  grd + t->cls_w, t->aam_ws, t->aam_ws_bytes, st);
                if (rc) return rc;
                rc = tr_dense_bwd(t->d_emb, D, t->pn, 2 * C3, par + t->fc_w, 2 * C3, B, D, 2 * C3, t->dpn, 2 * C3, grd + t->fc_w, 2 * C3, grd + t->fc_b, st);
                if (rc) return rc;
                rc = tr_bn1d_bwd(t->dpn, t->pooled, B, 2 * C3, par + t->aspbn_g, t->aspbn_mean, t->aspbn_rstd, t->dpooled, grd + t->aspbn_g,
                                 grd + t->aspbn_b, st);
                break;
            }
            case TStep::ASP_BWD:
                rc = tr_asp_bwd(t->logits, C3, t->M, C3, B, T, P, Tp, TR_ASP_EPS, t->pooled, t->dpooled, t->dlogits, t->dMd, st);
                break;
            case TStep::COLSUM: rc = tr_grad_sum(s.gl, s.C, B, T, P, Tp, Planes(), 0, t->part, s.f0, st); break;
            case TStep::GRAD_SUM: rc = tr_grad_sum(s.gl, s.C, B, T, P, Tp, s.p0, s.c0, t->part, nullptr, st); break;
            case TStep::BN_BWD: {
                const TLayer& l = t->L[s.layer];
                rc = tr_bn_backward(s.gl, s.p0, s.c0, l.bn.C, B, T, P, Tp, l.bn.mean, l.bn.rstd, par + l.bn.g_off, grd + l.bn.g_off, grd + l.bn.b_off,
                                    s.p1, s.c1, grd + l.conv.b_off, t->part, t->part_elems, st, s.a);
                break;
            }
            case TStep::ASP_CTX_BWD: {
                // t->part holds sum_t dz per utterance [B][att] (left by the BN backward of the attention TDNN)
                const TConv& c = t->L[t->l_att1].conv;
                rc = tr_dense_bwd(t->part, att, t->gstat, 2 * C3, par + c.w_off + C3, 3 * C3, B, att, 2 * C3, t->dgs, 2 * C3, grd + c.w_off + C3, 3 * C3,
                                  nullptr, st);
                if (rc) return rc;
                rc = tr_asp_global_bwd(t->gstat, t->dgs, B, C3, T, TR_ASP_EPS, t->rs, t->rb, st);
                break;
            }
            case TStep::SE_BWD: {
                const int b = s.a;
                GradSrcList gl;
                gl.n = 1;
                gl.s[0].t = t->Dbuf[b];
                rc = tr_grad_dot(gl, t->Yt2[b], 0, C, B, T, P, Tp, t->dg2, st);
                if (rc) return rc;
                rc = tr_act_bwd(t->dg2, t->se_g2[b], int64_t(B) * C, 2, 0.f, st);
                if (rc) return rc;
                rc = tr_dense_bwd(t->dg2, C, t->se_g1[b], se, par + t->se2_w[b], se, B, C, se, t->dg1, se, grd + t->se2_w[b], se, grd + t->se2_b[b], st);
                if (rc) return rc;
                rc = tr_act_bwd(t->dg1, t->se_g1[b], int64_t(B) * se, 1, 0.f, st);
                if (rc) return rc;
                rc = tr_dense_bwd(t->dg1, se, t->se_s[b], C, par + t->se1_w[b], C, B, se, C, t->ds, C, grd + t->se1_w[b], C, grd + t->se1_b[b], st);
                if (rc) return rc;
                rc = tr_act_bwd(t->ds, nullptr, int64_t(B) * C, 0, 1.f / float(T), st);
                break;
            }
            case TStep::WGRAD: {
                const TConv& c = s.layer >= 0 ? t->L[s.layer].conv : t->att2;
                for (const TStep::Tr& tr : s.trs) {
                    Planes dst = tr.which == 0 ? t->TA : t->TB;
                    dst.base += int64_t(tr.row0) * dst.ld;
                    dst.rows -= tr.row0;
                    rc = tr_transpose(tr.in, tr.col0, tr.C, t->R, dst, tr.shift, st, tr.ntaps, tr.shift_step, tr.row_step);
                    if (rc) return rc;
                }
                for (const GemmParams& gp : s.wg) {
                    rc = gemm_launch(gp, t->precision, t->num_sms, st);
                    if (rc) return rc;
                }
                rc = tr_wgrad_unpack(t->wpart, s.a, s.b, c.Cout, c.Cin, c.Cinp, c.taps, grd + c.w_off, int64_t(c.CinTotal) * c.taps, st);
                break;
            }
        }
        if (rc) return rc;
    }
    if (loss_out) PPV_CUDA_OK(cudaMemcpyAsync(loss_out, t->loss, sizeof(float), cudaMemcpyDeviceToDevice, st));
    if (logits_out) PPV_CUDA_OK(cudaMemcpyAsync(logits_out, t->cls_logits, size_t(B) * t->S * sizeof(float), cudaMemcpyDeviceToDevice, st));
    return PPV_OK;
}

// Taps for tests and debugging: every buffer of the step stays readable after it (tr_carve aliases none).
//   planes -> fp32 [B, T, C], valid frames; with the prefix "pad:" all Tp = T + 2P rows of every utterance, halo rows included
//     forward   "blocks.0".."blocks.3", "mfa" (block outputs); X0, A0, Y0, OUTCAT, Amfa, M, Aatt, A4; per block ("<name>:<0..2>")
//               At1, Yt1, Ares, RC, IN, At2, Yt2.  A* are the post-ReLU, pre-BatchNorm activations the BatchNorm backward reads.
//     gradients "g:<name>": dZ0, dOUTCAT, dMd, dMatt, dZmfa, dlogits, dZatt, dA4; per block D, dZt2, dRC, dZres, DIN, dZt1, dXt1
//   fp32 as stored: "asp" (pooled) [B, 2*C3], "emb" and "d_emb" [B, D], "logits" [B, Tp, C3] (every row), gstat, dgs, pn, dpn, dpooled
//     [B, 2*C3], rs, rb [B, C3]; per block se_s, se_g2 [B, C], se_g1 [B, se]; dg2, ds [B, C] and dg1 [B, se] are scratch that every
//     block's SE backward overwrites, so they hold block 0's values.
// A per-block name without a block suffix reads block 0.
int trainer_read_tap(Trainer* t, const char* name, float* out, size_t out_elems, cudaStream_t st) {
    PPV_REQUIRE(t && name && out, "trainer_read_tap: null argument");
    if (!t->plan_ws) return fail(PPV_ESTATE, "trainer_read_tap: no step has run");
    std::string n(name);
    const bool padded = n.rfind("pad:", 0) == 0;
    if (padded) n = n.substr(4);
    const int B = t->plan_B, T = t->plan_T, C = t->C, C3 = t->C3;
    int b = -1;  // block suffix
    const size_t colon = n.rfind(':');
    if (colon != std::string::npos && colon + 2 == n.size() && n.back() >= '0' && n.back() <= '9') {
        b = n.back() - '0';
        n.resize(colon);
        PPV_REQUIRE(b < 3, "trainer_read_tap: bad block");
    }
    const bool per_block = b >= 0;
    const int bk = per_block ? b : 0;
    auto unknown = [&]() { return fail(PPV_EINVAL, std::string("trainer_read_tap: unknown tap ") + name); };

    const float* vec = nullptr;
    size_t cnt = 0;
    bool vec_block = false;
    if (n == "asp") vec = t->pooled, cnt = size_t(B) * 2 * C3;
    else if (n == "emb") vec = t->emb, cnt = size_t(B) * t->D;
    else if (n == "d_emb") vec = t->d_emb, cnt = size_t(B) * t->D;
    else if (n == "logits") vec = t->logits, cnt = size_t(t->R) * C3;
    else if (n == "gstat") vec = t->gstat, cnt = size_t(B) * 2 * C3;
    else if (n == "dgs") vec = t->dgs, cnt = size_t(B) * 2 * C3;
    else if (n == "pn") vec = t->pn, cnt = size_t(B) * 2 * C3;
    else if (n == "dpn") vec = t->dpn, cnt = size_t(B) * 2 * C3;
    else if (n == "dpooled") vec = t->dpooled, cnt = size_t(B) * 2 * C3;
    else if (n == "rs") vec = t->rs, cnt = size_t(B) * C3;
    else if (n == "rb") vec = t->rb, cnt = size_t(B) * C3;
    else if (n == "dg2") vec = t->dg2, cnt = size_t(B) * C;
    else if (n == "dg1") vec = t->dg1, cnt = size_t(B) * t->se;
    else if (n == "ds") vec = t->ds, cnt = size_t(B) * C;
    else if (n == "se_s") vec = t->se_s[bk], cnt = size_t(B) * C, vec_block = true;
    else if (n == "se_g1") vec = t->se_g1[bk], cnt = size_t(B) * t->se, vec_block = true;
    else if (n == "se_g2") vec = t->se_g2[bk], cnt = size_t(B) * C, vec_block = true;
    if (vec) {
        if (padded || (per_block && !vec_block)) return unknown();
        PPV_REQUIRE(out_elems >= cnt, "trainer_read_tap: output too small");
        PPV_CUDA_OK(cudaMemcpyAsync(out, vec, cnt * sizeof(float), cudaMemcpyDeviceToDevice, st));
        return PPV_OK;
    }

    Planes src;
    int col0 = 0, cols = C;
    bool blocked = false;
    if (n.rfind("g:", 0) == 0) {
        const std::string g = n.substr(2);
        if (g == "D") src = t->Dbuf[bk], blocked = true;
        else if (g == "dZt2") src = t->dZt2[bk], blocked = true;
        else if (g == "dRC") src = t->dRC[bk], blocked = true;
        else if (g == "dZres") src = t->dZres[bk], blocked = true;
        else if (g == "DIN") src = t->DIN[bk], blocked = true;
        else if (g == "dZt1") src = t->dZt1[bk], blocked = true;
        else if (g == "dXt1") src = t->dXt1[bk], blocked = true;
        else if (g == "dZ0") src = t->dZ0;
        else if (g == "dOUTCAT") src = t->dOUTCAT, cols = C3;
        else if (g == "dMd") src = t->dMd, cols = C3;
        else if (g == "dMatt") src = t->dMatt, cols = C3;
        else if (g == "dZmfa") src = t->dZmfa, cols = C3;
        else if (g == "dlogits") src = t->dlogits, cols = C3;
        else if (g == "dZatt") src = t->dZatt, cols = t->att;
        else if (g == "dA4") src = t->dA4, cols = t->att;
        else return unknown();
    } else if (n == "blocks.0" || n == "Y0") {
        src = t->Y0;
    } else if (n == "blocks.1" || n == "blocks.2" || n == "blocks.3") {
        src = t->OUTCAT;
        col0 = C * (n[7] - '1');
    } else if (n == "mfa" || n == "M") {
        src = t->M, cols = C3;
    } else if (n == "X0") {
        src = t->X0, cols = t->cfg.input_size;
    } else if (n == "A0") {
        src = t->A0;
    } else if (n == "OUTCAT") {
        src = t->OUTCAT, cols = C3;
    } else if (n == "Amfa") {
        src = t->Amfa, cols = C3;
    } else if (n == "Aatt" || n == "A4") {
        src = n == "A4" ? t->A4 : t->Aatt, cols = t->att;
    } else {
        blocked = true;
        if (n == "At1") src = t->At1[bk];
        else if (n == "Yt1") src = t->Yt1[bk];
        else if (n == "Ares") src = t->Ares[bk];
        else if (n == "RC") src = t->RC[bk];
        else if (n == "IN") src = t->IN[bk];
        else if (n == "At2") src = t->At2[bk];
        else if (n == "Yt2") src = t->Yt2[bk];
        else return unknown();
    }
    if (per_block && !blocked) return unknown();
    const int rows = padded ? t->Tp : T;
    PPV_REQUIRE(out_elems >= size_t(B) * rows * cols, "trainer_read_tap: output too small");
    return launch_planes_to_f32(src, col0, cols, B, rows, padded ? 0 : t->P, t->Tp, out, st);
}

}  // namespace ppv
