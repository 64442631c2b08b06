// ECAPA-TDNN training step: train-mode forward, AAM-softmax loss, full backward into one flat gradient buffer.
// Reference: ppvector/trainer.py:206-229 (forward -> loss -> backward -> optimizer.step), ppvector/models/ecapa_tdnn.py:245-276,
// ppvector/models/utils.py:96-148 (TDNNBlock = BatchNorm(ReLU(conv)), BatchNorm in TRAIN mode: batch statistics over all
// B*T frames, momentum 0.9), ppvector/models/pooling.py:86-125, ppvector/models/fc.py:6-90 (DenseLayer blocks, Cosine or Linear output
// layer), ppvector/loss/aamloss.py:28-53.
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
#include "plan.h"
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
    bool dgrad = true;
};
struct TBN {
    std::string name;  // e.g. "blocks.1.tdnn1.norm.norm"
    int C = 0;
    int64_t g_off = 0, b_off = 0, rm_off = 0, rv_off = 0;
};
struct TLayer {  // TDNNBlock
    TConv conv;
    TBN bn;
};

// The workspace views of one plan (tr_carve).  `layer` is indexed like Trainer::conv: the TDNN layers, then the head's convs.
struct TrBuffers {
    int Tp = 0;          // rows per utterance: T + 2P
    int64_t R = 0, Rp = 0;  // rows of the padded time layout, B * Tp, and that rounded up to 128
    struct Layer {
        Planes wf, wd;  // weights in GEMM layouts
        float *mean = nullptr, *rstd = nullptr, *scale = nullptr, *shift = nullptr;  // BatchNorm (none for asp.conv)
    };
    std::vector<Layer> layer;
    Planes X0, A0, Y0, At1[3], Yt1[3], Ares[3], RC[3], IN[3], At2[3], Yt2[3], OUTCAT, Amfa, M, Aatt, A4, gstat_pl;
    Planes dlogits, dMd, dA4, dZatt, dMatt, dZmfa, dOUTCAT, Dbuf[3], dZt2[3], dRC[3], dZres[3], DIN[3], dZt1[3], dXt1[3], dZ0, TA, TB;
    float *logits = nullptr, *se_s[3], *se_g1[3], *se_g2[3], *gstat = nullptr, *fold = nullptr, *pooled = nullptr, *pn = nullptr, *emb = nullptr,
          *cls_logits = nullptr, *loss = nullptr, *aspbn_mean = nullptr, *aspbn_rstd = nullptr;
    float *d_emb = nullptr, *dpn = nullptr, *dpooled = nullptr, *dgs = nullptr, *rs = nullptr, *rb = nullptr, *dg2 = nullptr, *dg1 = nullptr, *ds = nullptr,
          *part = nullptr, *wpart = nullptr, *sap_stats = nullptr, *dsap_stats = nullptr;
    size_t part_elems = 0;
    float* aam_ws = nullptr;
    size_t aam_ws_bytes = 0;
    // classifier blocks (one entry per block, none without them): dense output z, BatchNorm output h (the block's output), its batch
    // mean / rstd, and dL/dh; dcls_z is the dL/dz scratch every block's backward reuses
    std::vector<float*> cls_z, cls_h, cls_mean, cls_rstd, dcls_h;
    float* dcls_z = nullptr;
};

// One readable tap (trainer_read_tap): planes read as fp32 [B, T, cols] from column col0, or `count` fp32 values as stored.  A
// per-block tap has one buffer per block; the others use index 0.
struct TrTap {
    bool per_block = false, fp32 = false;
    Planes pl[3];
    int col0 = 0, cols = 0;
    const float* vec[3] = {};
    size_t count = 0;
};

}  // namespace

struct Trainer : PlanOwner, EcapaGeometry {
    ppv_ecapa_cfg cfg;
    int S = 0;  // classes
    int D = 0;  // embedding size
    // (PlanOwner::precision PPV_PREC_BF16: single-pass bf16 operands for every forward / data-gradient / weight-gradient GEMM, AMP mode)
    // flat layout
    std::map<std::string, std::pair<int64_t, int64_t>> pmap, smap;  // name -> (offset, numel)
    int64_t n_params = 0, n_stats = 0;
    float *params = nullptr, *grads = nullptr, *stats = nullptr;
    // layers: 0 conv0; per block b (1..3): tdnn1, res2 x7, tdnn2; mfa; ASP: att1 (asp.tdnn)
    std::vector<TLayer> L;
    int l_conv0 = 0, l_tdnn1[3], l_res[3][8], l_tdnn2[3], l_mfa = 0, l_att1 = -1;
    // the pooling head's convs without a BatchNorm, numbered after L: ASP asp.conv.conv; SAP asp.linear1, asp.linear2; TAP / TSP none.
    // c_att2 is the conv that writes the softmax logits, c_lin1 SAP's linear1 (-1 where the head has none).
    std::vector<TConv> hconv;
    int c_lin1 = -1, c_att2 = -1;
    int Kp = 0;  // width of the pooled vector and of asp_bn: 2 * C3 (ASP, TSP) or C3 (SAP, TAP)
    int64_t se1_w[3], se1_b[3], se2_w[3], se2_b[3], aspbn_g = 0, aspbn_b = 0, aspbn_rm = 0, aspbn_rv = 0, fc_w = 0, fc_b = 0, cls_w = 0;
    // the classifier (fc.py:6-53): num_blocks DenseLayers (Conv1D 1x1 + BatchNorm1D, no ReLU), then the Cosine or Linear output layer
    struct ClsBlock {
        int in = 0;  // input width: embd_dim for block 0, inter_dim after it
        int64_t w = 0, b = 0, g = 0, beta = 0, rm = 0, rv = 0;
    };
    int cls_type = PPV_CLASSIFIER_COSINE, inter = 0;
    std::vector<ClsBlock> cls_blocks;
    int64_t cls_b = -1;  // Linear: classifier.output.bias
    int head_dim() const { return cls_blocks.empty() ? D : inter; }  // width of the output layer's input
    // plan
    TrBuffers buf;
    std::map<std::string, TrTap> taps;

    Trainer(const ppv_ecapa_cfg& c, const EcapaGeometry& g, int num_classes)
        : PlanOwner("trainer", "ppv_trainer_workspace_bytes", PPV_PREC_BF16X3), EcapaGeometry(g), cfg(c), S(num_classes), D(c.embd_dim) {
        sync_each_step = getenv("PPV_TRAIN_DEBUG") != nullptr;  // localise a faulting kernel
    }
    // convs by layer index: L's, then hconv
    int n_conv() const { return int(L.size() + hconv.size()); }
    const TConv& conv(int layer) const { return layer < int(L.size()) ? L[layer].conv : hconv[layer - L.size()]; }
    bool attentive() const { return cfg.pooling == PPV_POOL_ASP || cfg.pooling == PPV_POOL_SAP; }  // softmax pooling over logits
    bool context() const { return cfg.pooling == PPV_POOL_ASP && cfg.global_context; }
    size_t workspace_bytes(int B, int T) const override;
    using PlanOwner::run_plan;

  protected:
    int build_plan(int B, int T, void* ws, size_t ws_bytes, cudaStream_t st) override;
};

// ------------------------------------------------------------------------------------------------ create: flat layout
static int64_t tr_add(std::map<std::string, std::pair<int64_t, int64_t>>& m, int64_t& total, const std::string& name, int64_t numel) {
    const int64_t off = total;
    m[name] = {off, numel};
    total += int64_t(align_up(size_t(numel), 8));  // 32-byte aligned tensors (vector loads in the epilogues)
    return off;
}

int trainer_create(const ppv_ecapa_cfg* cfg, int num_classes, int classifier_type, int num_blocks, int inter_dim, Trainer** out) {
    PPV_REQUIRE(cfg && out && num_classes > 1, "trainer_create: bad argument");
    if (classifier_type != PPV_CLASSIFIER_COSINE && classifier_type != PPV_CLASSIFIER_LINEAR)
        return fail(PPV_EUNSUPPORTED, "trainer: classifier_type must be PPV_CLASSIFIER_COSINE or PPV_CLASSIFIER_LINEAR");  // fc.py:39-40
    PPV_REQUIRE(num_blocks >= 0 && (num_blocks == 0 || inter_dim > 0), "trainer: num_blocks >= 0 and inter_dim > 0 required");
    const int C = cfg->channels[0];
    if (cfg->channels[1] != C || cfg->channels[2] != C || cfg->channels[3] != C || cfg->channels[4] != 3 * C)
        return fail(PPV_EUNSUPPORTED, "trainer: channels must be [C,C,C,C,3C]");
    if (cfg->res2net_scale != 8 || C % 512) return fail(PPV_EUNSUPPORTED, "trainer: res2net_scale 8 and channels % 512 == 0 required");
    if (cfg->kernel_sizes[1] != 3 || cfg->kernel_sizes[2] != 3 || cfg->kernel_sizes[3] != 3 || cfg->kernel_sizes[4] != 1 || (cfg->kernel_sizes[0] % 2) == 0)
        return fail(PPV_EUNSUPPORTED, "trainer: kernel sizes must be [odd,3,3,3,1]");
    if (cfg->attention_channels % 64 || cfg->se_channels % 8 || cfg->embd_dim % 8)
        return fail(PPV_EUNSUPPORTED, "trainer: attention_channels % 64, se_channels % 8, embd_dim % 8 required");
    if (cfg->pooling < PPV_POOL_ASP || cfg->pooling > PPV_POOL_TSP) return fail(PPV_EUNSUPPORTED, "trainer: pooling must be PPV_POOL_ASP / SAP / TAP / TSP");
    if (cfg->pooling == PPV_POOL_SAP && cfg->attention_channels != 128)  // as the inference model refuses it, so a trained model can be evaluated
        return fail(PPV_EUNSUPPORTED, "trainer: SAP pooling uses a 128-channel bottleneck (ecapa_tdnn.py:222): attention_channels must be 128");
    EcapaGeometry g;  // its checks pass where the ones above do
    int rc = ecapa_geometry(*cfg, &g);
    if (rc) return rc;
    Trainer* t = new Trainer(*cfg, g, num_classes);

    auto add_layer = [&](const std::string& p, int cin, int cout, int k, int dil, bool dgrad) {
        TLayer l;
        l.conv.name = p + ".conv.conv";
        l.conv.Cout = cout;
        l.conv.Cin = l.conv.CinTotal = cin;
        l.conv.Cinp = int(align_up(size_t(cin), 64));
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
    // a 1x1 conv of the head without a BatchNorm after it ("<name>.weight" [Cout, Cin, 1], "<name>.bias" [Cout])
    auto add_head_conv = [&](const std::string& name, int cin, int cout) {
        TConv c;
        c.name = name;
        c.Cout = cout;
        c.Cin = c.CinTotal = c.Cinp = cin;
        c.w_off = tr_add(t->pmap, t->n_params, name + ".weight", int64_t(cout) * cin);
        c.b_off = tr_add(t->pmap, t->n_params, name + ".bias", cout);
        t->hconv.push_back(c);
        return int(t->L.size() + t->hconv.size()) - 1;
    };
    // the head and its asp_bn in the reference's state_dict order (ecapa_tdnn.py:212-241): ASP's BatchNorm1d wraps paddle's as `.norm`
    const int pool = cfg->pooling;
    t->Kp = (pool == PPV_POOL_ASP || pool == PPV_POOL_TSP) ? 2 * t->C3 : t->C3;
    if (pool == PPV_POOL_ASP) {
        t->l_att1 = add_layer("asp.tdnn", (cfg->global_context ? 3 : 1) * t->C3, t->att, 1, 1, true);
        TConv& c1 = t->L[t->l_att1].conv;  // only the first C3 input channels go through the frame-level GEMM
        c1.Cin = t->C3;
        c1.Cinp = t->C3;
        t->c_att2 = add_head_conv("asp.conv.conv", t->att, t->C3);
    } else if (pool == PPV_POOL_SAP) {
        t->c_lin1 = add_head_conv("asp.linear1", t->C3, t->att);
        t->c_att2 = add_head_conv("asp.linear2", t->att, t->C3);
    }
    const std::string bn = pool == PPV_POOL_ASP ? "asp_bn.norm" : "asp_bn";
    t->aspbn_g = tr_add(t->pmap, t->n_params, bn + ".weight", t->Kp);
    t->aspbn_b = tr_add(t->pmap, t->n_params, bn + ".bias", t->Kp);
    t->aspbn_rm = tr_add(t->smap, t->n_stats, bn + "._mean", t->Kp);
    t->aspbn_rv = tr_add(t->smap, t->n_stats, bn + "._variance", t->Kp);
    t->fc_w = tr_add(t->pmap, t->n_params, "fc.conv.weight", int64_t(t->D) * t->Kp);
    t->fc_b = tr_add(t->pmap, t->n_params, "fc.conv.bias", t->D);
    // the classifier in SpeakerIdentification's state_dict order (fc.py:25-38): the blocks, then the output layer
    t->cls_type = classifier_type;
    t->inter = num_blocks ? inter_dim : 0;
    for (int i = 0; i < num_blocks; ++i) {
        const std::string p = "classifier.blocks." + std::to_string(i);
        Trainer::ClsBlock k;
        k.in = i == 0 ? t->D : inter_dim;
        k.w = tr_add(t->pmap, t->n_params, p + ".linear.weight", int64_t(inter_dim) * k.in);  // Conv1D [inter, in, 1]
        k.b = tr_add(t->pmap, t->n_params, p + ".linear.bias", inter_dim);
        k.g = tr_add(t->pmap, t->n_params, p + ".nonlinear.batchnorm.weight", inter_dim);
        k.beta = tr_add(t->pmap, t->n_params, p + ".nonlinear.batchnorm.bias", inter_dim);
        k.rm = tr_add(t->smap, t->n_stats, p + ".nonlinear.batchnorm._mean", inter_dim);
        k.rv = tr_add(t->smap, t->n_stats, p + ".nonlinear.batchnorm._variance", inter_dim);
        t->cls_blocks.push_back(k);
    }
    if (classifier_type == PPV_CLASSIFIER_COSINE) {
        t->cls_w = tr_add(t->pmap, t->n_params, "classifier.weight", int64_t(t->head_dim()) * t->S);  // fc.py:30-36: [input_dim, num_speakers]
    } else {
        t->cls_w = tr_add(t->pmap, t->n_params, "classifier.output.weight", int64_t(t->head_dim()) * t->S);  // nn.Linear: [input_dim, num_speakers]
        t->cls_b = tr_add(t->pmap, t->n_params, "classifier.output.bias", t->S);
    }
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
    t->invalidate_plan();  // pointers are baked into the plan
    return PPV_OK;
}

// ------------------------------------------------------------------------------------------------ workspace
namespace {

// Frame splits of a layer's BatchNorm backward: narrow layers split the frames of an utterance over several CTAs so the
// reduction fills the GPU.  The attention TDNN keeps per-utterance sums, which ASP_CTX_BWD reads back from `part`.
int tr_bn_bwd_tsplit(const Trainer* t, int layer, int B) {
    const int ctas = (t->L[layer].bn.C / 64) * B;
    return (layer == t->l_att1 || ctas >= 2 * t->num_sms) ? 1 : std::min(8, std::max(1, (2 * t->num_sms + ctas - 1) / ctas));
}

// Split-K of a conv's weight-gradient GEMM [Cout] x [taps * Cinp] over the Rp frame rows: enough splits to fill the GPU, at most
// one per 64 rows.  Each split writes an [Mpad][taps * Cinp] partial to `wpart`.
struct WgradSplit {
    int splits, Mpad, BN;
};
WgradSplit tr_wgrad_split(const Trainer* t, const TConv& c, int64_t Rp) {
    const int N = c.taps * c.Cinp, BN = gemm_pick_bn(N);
    const int mt = (c.Cout + 127) / 128, nt = (N + BN - 1) / BN;
    return {std::max(1, std::min((t->num_sms + mt * nt - 1) / (mt * nt), int((Rp + 63) / 64))), mt * 128, BN};
}

void tr_carve(const Trainer* t, WsCarver& cv, int B, int T, TrBuffers* f) {
    f->Tp = T + 2 * t->P;
    f->R = int64_t(B) * f->Tp;
    f->Rp = int64_t(align_up(size_t(f->R), 128));
    const int64_t Rp = f->Rp;
    const int C = t->C, C3 = t->C3;
    auto f32 = [&](size_t n) { return static_cast<float*>(cv.take(n * sizeof(float))); };
    const int Kp = t->Kp;
    const bool attn = t->attentive(), ctx = t->context(), asp = t->cfg.pooling == PPV_POOL_ASP;
    f->layer.assign(t->n_conv(), TrBuffers::Layer());
    for (int l = 0; l < t->n_conv(); ++l) {
        const TConv& c = t->conv(l);
        TrBuffers::Layer& w = f->layer[l];
        w.wf = cv.planes(int64_t(align_up(size_t(c.Cout), 256)), c.taps * c.Cinp);
        if (c.dgrad) w.wd = cv.planes(int64_t(align_up(size_t(c.Cinp), 256)), c.taps * c.Cout);
        if (l >= int(t->L.size())) continue;
        const int Cb = t->L[l].bn.C;
        w.mean = f32(Cb);
        w.rstd = f32(Cb);
        w.scale = f32(Cb);
        w.shift = f32(Cb);
    }
    auto act = [&](std::initializer_list<Planes*> ps, int cols) {
        for (Planes* p : ps) *p = cv.planes(Rp, cols);
    };
    f->X0 = cv.planes(Rp, t->Fp);
    act({&f->A0, &f->Y0}, C);
    for (int b = 0; b < 3; ++b) {
        act({&f->At1[b], &f->Yt1[b], &f->Ares[b], &f->RC[b], &f->IN[b], &f->At2[b], &f->Yt2[b]}, C);
        f->se_s[b] = f32(size_t(B) * C);
        f->se_g1[b] = f32(size_t(B) * t->se);
        f->se_g2[b] = f32(size_t(B) * C);
    }
    act({&f->OUTCAT, &f->Amfa, &f->M}, C3);
    // the head's buffers, carved only for the heads that use them; the attention of SAP (tanh(linear1)) lands in A4 like ASP's
    if (asp) act({&f->Aatt}, t->att);
    if (attn) act({&f->A4}, t->att);
    if (ctx) f->gstat_pl = cv.planes(B, 2 * C3);
    if (attn) f->logits = f32(size_t(Rp) * C3);
    if (ctx) {
        f->gstat = f32(size_t(B) * 2 * C3);
        f->fold = f32(size_t(B) * t->att);
    }
    f->pooled = f32(size_t(B) * Kp);
    f->pn = f32(size_t(B) * Kp);
    f->emb = f32(size_t(B) * t->D);
    f->cls_logits = f32(size_t(B) * t->S);
    f->loss = f32(8);
    f->aspbn_mean = f32(Kp);
    f->aspbn_rstd = f32(Kp);
    // gradients
    if (attn) act({&f->dlogits}, C3);
    act({&f->dMd}, C3);
    if (attn) {
        act({&f->dA4, &f->dZatt}, t->att);
        act({&f->dMatt}, C3);
    }
    act({&f->dZmfa, &f->dOUTCAT}, C3);
    for (int b = 0; b < 3; ++b) act({&f->Dbuf[b], &f->dZt2[b], &f->dRC[b], &f->dZres[b], &f->DIN[b], &f->dZt1[b], &f->dXt1[b]}, C);
    act({&f->dZ0}, C);
    f->TA = cv.planes(C3, int(Rp));
    f->TB = cv.planes(C3, int(Rp));
    f->d_emb = f32(size_t(B) * t->D);
    f->dpn = f32(size_t(B) * Kp);
    f->dpooled = f32(size_t(B) * Kp);
    if (ctx) {
        f->dgs = f32(size_t(B) * 2 * C3);
        f->rs = f32(size_t(B) * C3);
        f->rb = f32(size_t(B) * C3);
    }
    f->dg2 = f32(size_t(B) * C);
    f->dg1 = f32(size_t(B) * t->se);
    f->ds = f32(size_t(B) * C);
    // partial sums: BatchNorm forward statistics [B][3][C], per-utterance column sums [B][C], BatchNorm backward [B * tsplit][2][C]
    f->part_elems = size_t(3) * B * C3;
    for (int l = 0; l < int(t->L.size()); ++l)
        f->part_elems = std::max(f->part_elems, size_t(2) * B * tr_bn_bwd_tsplit(t, l, B) * t->L[l].bn.C);
    f->part = f32(f->part_elems);
    // weight-gradient partials: the largest split-K output of any conv
    size_t wmax = 0;
    for (int l = 0; l < t->n_conv(); ++l) {
        const TConv& c = t->conv(l);
        const WgradSplit w = tr_wgrad_split(t, c, Rp);
        wmax = std::max(wmax, size_t(w.splits) * w.Mpad * c.taps * c.Cinp);
    }
    f->wpart = f32(wmax);
    f->aam_ws_bytes = aam_workspace_bytes(B, t->head_dim(), t->S);
    f->aam_ws = static_cast<float*>(cv.take(f->aam_ws_bytes));
    if (t->cfg.pooling == PPV_POOL_SAP) {  // the softmax pooling's [mean | std] and the gradient it reads back (std half: zero)
        f->sap_stats = f32(size_t(B) * 2 * C3);
        f->dsap_stats = f32(size_t(B) * 2 * C3);
    }
    const size_t nblk = t->cls_blocks.size();
    for (std::vector<float*>* v : {&f->cls_z, &f->cls_h, &f->cls_mean, &f->cls_rstd, &f->dcls_h}) v->assign(nblk, nullptr);
    for (size_t i = 0; i < nblk; ++i) {
        f->cls_z[i] = f32(size_t(B) * t->inter);
        f->cls_h[i] = f32(size_t(B) * t->inter);
        f->cls_mean[i] = f32(t->inter);
        f->cls_rstd[i] = f32(t->inter);
        f->dcls_h[i] = f32(size_t(B) * t->inter);
    }
    if (nblk) f->dcls_z = f32(size_t(B) * t->inter);
}

// The taps trainer_read_tap serves, by name without the "pad:" prefix and the block suffix.  A buffer the head does not carve
// has no tap.
std::map<std::string, TrTap> tr_tap_table(const Trainer* t, const TrBuffers& f, int B) {
    const int C = t->C, C3 = t->C3;
    std::map<std::string, TrTap> m;
    auto planes = [&](const std::string& name, const Planes* p, bool per_block, int cols, int col0 = 0) {
        if (!p[0].base) return;
        TrTap& e = m[name];
        e.per_block = per_block;
        for (int b = 0; b < (per_block ? 3 : 1); ++b) e.pl[b] = p[b];
        e.cols = cols;
        e.col0 = col0;
    };
    auto vec = [&](const std::string& name, float* const* p, bool per_block, size_t count) {
        if (!p[0]) return;
        TrTap& e = m[name];
        e.per_block = per_block;
        e.fp32 = true;
        for (int b = 0; b < (per_block ? 3 : 1); ++b) e.vec[b] = p[b];
        e.count = count;
    };
    using NamedPlanes = std::initializer_list<std::pair<const char*, const Planes*>>;
    using NamedVec = std::initializer_list<std::pair<const char*, float* const*>>;
    // forward planes
    planes("blocks.0", &f.Y0, false, C);
    for (int b = 1; b <= 3; ++b) planes("blocks." + std::to_string(b), &f.OUTCAT, false, C, C * (b - 1));
    planes("mfa", &f.M, false, C3);
    planes("X0", &f.X0, false, t->cfg.input_size);
    for (const auto& e : NamedPlanes{{"A0", &f.A0}, {"Y0", &f.Y0}}) planes(e.first, e.second, false, C);
    for (const auto& e : NamedPlanes{{"OUTCAT", &f.OUTCAT}, {"Amfa", &f.Amfa}, {"M", &f.M}}) planes(e.first, e.second, false, C3);
    for (const auto& e : NamedPlanes{{"Aatt", &f.Aatt}, {"A4", &f.A4}}) planes(e.first, e.second, false, t->att);
    for (const auto& e : NamedPlanes{{"At1", f.At1}, {"Yt1", f.Yt1}, {"Ares", f.Ares}, {"RC", f.RC}, {"IN", f.IN}, {"At2", f.At2}, {"Yt2", f.Yt2}})
        planes(e.first, e.second, true, C);
    // gradient planes
    planes("g:dZ0", &f.dZ0, false, C);
    for (const auto& e : NamedPlanes{{"g:dOUTCAT", &f.dOUTCAT}, {"g:dMd", &f.dMd}, {"g:dMatt", &f.dMatt}, {"g:dZmfa", &f.dZmfa}, {"g:dlogits", &f.dlogits}})
        planes(e.first, e.second, false, C3);
    for (const auto& e : NamedPlanes{{"g:dZatt", &f.dZatt}, {"g:dA4", &f.dA4}}) planes(e.first, e.second, false, t->att);
    for (const auto& e : NamedPlanes{{"g:D", f.Dbuf}, {"g:dZt2", f.dZt2}, {"g:dRC", f.dRC}, {"g:dZres", f.dZres}, {"g:DIN", f.DIN}, {"g:dZt1", f.dZt1},
                                     {"g:dXt1", f.dXt1}})
        planes(e.first, e.second, true, C);
    // fp32 as stored
    vec("asp", &f.pooled, false, size_t(B) * t->Kp);
    for (const auto& e : NamedVec{{"emb", &f.emb}, {"d_emb", &f.d_emb}}) vec(e.first, e.second, false, size_t(B) * t->D);
    vec("logits", &f.logits, false, size_t(f.R) * C3);
    for (const auto& e : NamedVec{{"gstat", &f.gstat}, {"dgs", &f.dgs}, {"sap_stats", &f.sap_stats}, {"dsap_stats", &f.dsap_stats}})
        vec(e.first, e.second, false, size_t(B) * 2 * C3);
    for (const auto& e : NamedVec{{"pn", &f.pn}, {"dpn", &f.dpn}, {"dpooled", &f.dpooled}}) vec(e.first, e.second, false, size_t(B) * t->Kp);
    for (const auto& e : NamedVec{{"rs", &f.rs}, {"rb", &f.rb}}) vec(e.first, e.second, false, size_t(B) * C3);
    for (const auto& e : NamedVec{{"dg2", &f.dg2}, {"ds", &f.ds}}) vec(e.first, e.second, false, size_t(B) * C);
    vec("dg1", &f.dg1, false, size_t(B) * t->se);
    for (const auto& e : NamedVec{{"se_s", f.se_s}, {"se_g2", f.se_g2}}) vec(e.first, e.second, true, size_t(B) * C);
    vec("se_g1", f.se_g1, true, size_t(B) * t->se);
    for (size_t i = 0; i < t->cls_blocks.size(); ++i) {  // classifier block outputs, their dense outputs and gradients [B, inter_dim]
        const std::string p = "classifier.blocks." + std::to_string(i);
        vec(p, &f.cls_h[i], false, size_t(B) * t->inter);
        vec(p + ".z", &f.cls_z[i], false, size_t(B) * t->inter);
        vec("g:" + p, &f.dcls_h[i], false, size_t(B) * t->inter);
    }
    vec("g:classifier.z", &f.dcls_z, false, size_t(B) * t->inter);
    return m;
}

}  // namespace

size_t Trainer::workspace_bytes(int B, int T) const {
    if (B <= 0 || T <= 0) return 0;
    WsCarver cv;
    TrBuffers f;
    tr_carve(this, cv, B, T, &f);
    return align_up(cv.off, 256);
}

size_t trainer_workspace_bytes(const Trainer* t, int B, int T) { return t ? t->workspace_bytes(B, T) : 0; }

// ------------------------------------------------------------------------------------------------ plan
int Trainer::build_plan(int B, int T, void* ws, size_t ws_bytes, cudaStream_t st) {
    Trainer* const t = this;
    PPV_REQUIRE(t->params, "trainer: call ppv_trainer_bind first");
    PPV_REQUIRE(T > 2 * t->P, "trainer: too few frames for the reflect padding");
    int rc = claim_workspace(B, T, ws, ws_bytes, st);
    if (rc) return rc;
    WsCarver cv;
    cv.base = static_cast<uint8_t*>(ws);
    TrBuffers& f = t->buf;
    tr_carve(t, cv, B, T, &f);
    t->taps = tr_tap_table(t, f, B);
    t->steps.clear();
    const int C = t->C, C3 = t->C3, W = t->width, P = t->P, Tp = f.Tp, se = t->se, att = t->att, D = t->D;
    const int M = int(f.R);
    float* const par = t->params;
    float* const grd = t->grads;
    float* const sta = t->stats;

    // the trainer's own steps: one launcher call each, none on the tensor cores
    auto push = [&](const char* name, std::function<int(const StepRun&)> launch) { t->steps.push_back({name, false, std::move(launch)}); };
    auto gemm = [&](const std::vector<GemmSource>& srcs, const Planes& w, int N, const Epilogue& ep) -> int {
        GemmParams gp;
        int err = gemm_build(&gp, srcs.data(), int(srcs.size()), w, M, N, ep, gemm_pick_bn(N));
        if (!err) t->steps.push_back(gemm_step(gp));
        return err;
    };
    // forward conv: bias + ReLU -> post-activation planes (valid frames), or fp32 rows
    auto fwd_gemm = [&](int li, const std::vector<GemmSource>& srcs, const Planes& out, int out_col0, bool relu, const float* rowgrp,
                        float* out_f32) -> int {
        const TConv& c = t->conv(li);
        Epilogue ep = planes_epilogue(out, out_col0, Tp, P, T);
        if (out_f32) {
            ep.out_mode = OUT_F32;
            ep.out = out_f32;
            ep.out_ld = c.Cout;
        }
        ep.bias = par + c.b_off;
        ep.rowgrp_bias = rowgrp;
        ep.relu = relu ? 1 : 0;
        return gemm(srcs, f.layer[li].wf, c.Cout, ep);
    };
    auto taps_of = [&](const TConv& c, const Planes& x, int col0, int sign) {
        std::vector<GemmSource> v;
        for (int tp = 0; tp < c.taps; ++tp) v.push_back(GemmSource{x, col0, sign > 0 ? c.Cinp : c.Cout, sign * (tp - (c.taps - 1) / 2) * c.dil});
        return v;
    };
    auto bn_fwd = [&](int li, const Planes& a, int a_col0, const Planes& y, int y_col0, int tanh_, const Planes* add, int add_col0,
                      const Planes* out2, int out2_col0) {
        const TBN& bn = t->L[li].bn;
        const TrBuffers::Layer& w = f.layer[li];
        BnApplyArgs apply;
        apply.y = y;
        apply.y_col0 = y_col0;
        apply.tanh_ = tanh_;
        if (out2) {
            apply.add = *add;
            apply.add_col0 = add_col0;
            apply.out2 = *out2;
            apply.out2_col0 = out2_col0;
        }
        push("tr_bn_forward", [a, a_col0, Cn = bn.C, B, T, P, Tp, gamma = par + bn.g_off, beta = par + bn.b_off, mean = w.mean, rstd = w.rstd,
                               scale = w.scale, shift = w.shift, run_mean = sta + bn.rm_off, run_var = sta + bn.rv_off, part = f.part,
                               apply](const StepRun& r) {
            return tr_bn_forward(a, a_col0, Cn, B, T, P, Tp, TR_BN_EPS, TR_BN_MOMENTUM, gamma, beta, mean, rstd, scale, shift, run_mean, run_var,
                                 part, apply, r.num_sms, r.st);
        });
    };
    auto dense_fwd = [&](const float* X, int x_ld, const float* Wt, int w_ld, const float* bias, int Mr, int N, int K, int act, float* Y, int y_ld) {
        push("tr_dense_fwd", [X, x_ld, Wt, w_ld, bias, Mr, N, K, act, Y, y_ld](const StepRun& r) {
            return tr_dense_fwd(X, x_ld, Wt, w_ld, bias, Mr, N, K, act, Y, y_ld, r.st);
        });
    };
    auto dense_bwd = [&](const float* dY, int dy_ld, const float* X, int x_ld, const float* Wt, int w_ld, int Mr, int N, int K, float* dX,
                         int dx_ld, float* dW, int dw_ld, float* db) {
        push("tr_dense_bwd", [dY, dy_ld, X, x_ld, Wt, w_ld, Mr, N, K, dX, dx_ld, dW, dw_ld, db](const StepRun& r) {
            return tr_dense_bwd(dY, dy_ld, X, x_ld, Wt, w_ld, Mr, N, K, dX, dx_ld, dW, dw_ld, db, r.st);
        });
    };
    auto act_bwd = [&](float* dy, const float* y, int64_t n, int act, float alpha) {
        push("tr_act_bwd", [dy, y, n, act, alpha](const StepRun& r) { return tr_act_bwd(dy, y, n, act, alpha, r.st); });
    };
    // data gradient: dx_pad[r, cin] = sum_tap dz[r - off_tap, :] . W[:, cin, tap]  -> planes on every row
    auto dgrad_gemm = [&](int li, const Planes& dz, int dz_col0, const Planes& out, int out_col0) -> int {
        const TConv& c = t->conv(li);
        return gemm(taps_of(c, dz, dz_col0, -1), f.layer[li].wd, c.Cinp, planes_epilogue(out, out_col0));
    };
    // out[c][row0 + r] = in[r + shift][col0 + c]; ntaps > 1: tap z shifted by z * shift_step into rows z * row_step on
    auto transpose = [&](const Planes& in, int col0, int Cn, Planes out, int row0, int shift, int ntaps, int shift_step, int row_step) {
        out.base += int64_t(row0) * out.ld;
        out.rows -= row0;
        push("tr_transpose", [in, col0, Cn, rows = f.R, out, shift, ntaps, shift_step, row_step](const StepRun& r) {
            return tr_transpose(in, col0, Cn, rows, out, shift, r.st, ntaps, shift_step, row_step);
        });
    };
    // weight gradient: dz^T -> TA; one row-shifted transpose of the layer input per tap -> TB rows [tap * Cinp, ...); ONE GEMM
    // [Cout] x [taps * Cinp] over the frames (split-K partials); unpack into the flat gradient buffer
    struct WgradInput {
        Planes x;
        int col0, C, row0;  // row0: first row of TB to write
    };
    auto wgrad = [&](int li, const Planes& dz, int dz_col0, const std::vector<WgradInput>& xs) -> int {
        const TConv& c = t->conv(li);
        transpose(dz, dz_col0, c.Cout, f.TA, 0, 0, 1, 0, 0);
        for (const WgradInput& x : xs) transpose(x.x, x.col0, x.C, f.TB, x.row0, -((c.taps - 1) / 2) * c.dil, c.taps, c.dil, c.Cinp);
        const int N = c.taps * c.Cinp;
        const WgradSplit sp = tr_wgrad_split(t, c, f.Rp);
        GemmParams gp;
        int err = gemm_build_wgrad(&gp, f.TA, f.TB, c.Cout, N, 0, 0, sp.splits, f.wpart, N, 0, sp.Mpad, sp.BN);
        if (err) return err;
        t->steps.push_back(gemm_step(gp));
        push("tr_wgrad_unpack", [part = f.wpart, splits = gp.lin_splits, split_rows = sp.Mpad, Cout = c.Cout, Cin = c.Cin, Cinp = c.Cinp, taps = c.taps,
                                 grad = grd + c.w_off, g_ld = int64_t(c.CinTotal) * c.taps](const StepRun& r) {
            return tr_wgrad_unpack(part, splits, split_rows, Cout, Cin, Cinp, taps, grad, g_ld, r.st);
        });
        return PPV_OK;
    };
    auto src1 = [](const Planes& p, int col0, int fold) {
        GradSrc g;
        g.t = p;
        g.col0 = col0;
        g.fold = fold;
        return g;
    };
    auto bn_bwd = [&](int li, const GradSrcList& gl, const Planes& a, int a_col0, const Planes& dz, int dz_col0) {
        const TLayer& l = t->L[li];
        const TrBuffers::Layer& w = f.layer[li];
        push("tr_bn_backward", [gl, a, a_col0, Cn = l.bn.C, B, T, P, Tp, mean = w.mean, rstd = w.rstd, gamma = par + l.bn.g_off,
                                dgamma = grd + l.bn.g_off, dbeta = grd + l.bn.b_off, dz, dz_col0, dbias = grd + l.conv.b_off, part = f.part,
                                part_elems = f.part_elems, tsplit = tr_bn_bwd_tsplit(t, li, B)](const StepRun& r) {
            return tr_bn_backward(gl, a, a_col0, Cn, B, T, P, Tp, mean, rstd, gamma, dgamma, dbeta, dz, dz_col0, dbias, part, part_elems, r.st,
                                  tsplit);
        });
    };
    // out (optional planes, valid frames) = summed sources, per-utterance column sums -> part, colsum (optional) [Cn]
    auto grad_sum = [&](const GradSrcList& gl, int Cn, const Planes& out, float* colsum) {
        push("tr_grad_sum", [gl, Cn, B, T, P, Tp, out, part = f.part, colsum](const StepRun& r) {
            return tr_grad_sum(gl, Cn, B, T, P, Tp, out, 0, part, colsum, r.st);
        });
    };

    // ================================================================= forward
    for (int l = 0; l < t->n_conv(); ++l) {
        const TConv& c = t->conv(l);
        push("tr_repack_conv", [w = par + c.w_off, w_ld = int64_t(c.CinTotal) * c.taps, Cout = c.Cout, Cin = c.Cin, Cinp = c.Cinp, taps = c.taps,
                                wf = f.layer[l].wf, wd = f.layer[l].wd](const StepRun& r) {
            return tr_repack_conv(w, w_ld, Cout, Cin, Cinp, taps, wf, wd, r.st);
        });
    }
    push("launch_pack_features", [B, T, F = t->cfg.input_size, X0 = f.X0, P, Tp](const StepRun& r) {
        return launch_pack_features(r.in.feat, B, T, F, X0, P, Tp, r.st);
    });
    {
        const int li = t->l_conv0;
        rc = fwd_gemm(li, taps_of(t->conv(li), f.X0, 0, +1), f.A0, 0, true, nullptr, nullptr);
        if (rc) return rc;
        bn_fwd(li, f.A0, 0, f.Y0, 0, 0, nullptr, 0, nullptr, 0);
    }
    for (int b = 0; b < 3; ++b) {
        const Planes u = b == 0 ? f.Y0 : f.OUTCAT;
        const int uc = b == 0 ? 0 : C * (b - 1);
        {
            const int li = t->l_tdnn1[b];
            rc = fwd_gemm(li, {GemmSource{u, uc, C, 0}}, f.At1[b], 0, true, nullptr, nullptr);
            if (rc) return rc;
            bn_fwd(li, f.At1[b], 0, f.Yt1[b], 0, 0, nullptr, 0, nullptr, 0);
        }
        for (int j = 1; j < 8; ++j) {
            const int li = t->l_res[b][j];
            const Planes& xin = j == 1 ? f.Yt1[b] : f.IN[b];
            rc = fwd_gemm(li, taps_of(t->conv(li), xin, W * j, +1), f.Ares[b], W * j, true, nullptr, nullptr);
            if (rc) return rc;
            // r_j -> RC window j; in_{j+1} = r_j + chunk_{j+1}(tdnn1 output) -> IN window j+1   (ecapa_tdnn.py:41-45)
            if (j < 7)
                bn_fwd(li, f.Ares[b], W * j, f.RC[b], W * j, 0, &f.Yt1[b], W * (j + 1), &f.IN[b], W * (j + 1));
            else
                bn_fwd(li, f.Ares[b], W * j, f.RC[b], W * j, 0, nullptr, 0, nullptr, 0);
        }
        {
            const int li = t->l_tdnn2[b];
            rc = fwd_gemm(li, {GemmSource{f.Yt1[b], 0, W, 0}, GemmSource{f.RC[b], W, C - W, 0}}, f.At2[b], 0, true, nullptr, nullptr);
            if (rc) return rc;
            bn_fwd(li, f.At2[b], 0, f.Yt2[b], 0, 0, nullptr, 0, nullptr, 0);
        }
        // SE: squeeze, excite, then scale + residual into OUTCAT's window b
        t->steps.push_back(colstats_step(f.Yt2[b], C, B, T, P, Tp, 0, 0.f, Planes(), 0.f, false, f.se_s[b]));
        dense_fwd(f.se_s[b], C, par + t->se1_w[b], C, par + t->se1_b[b], B, se, C, 1, f.se_g1[b], se);
        dense_fwd(f.se_g1[b], se, par + t->se2_w[b], se, par + t->se2_b[b], B, C, se, 2, f.se_g2[b], C);
        t->steps.push_back(scale_res_step(f.Yt2[b], f.se_g2[b], u, uc, f.OUTCAT, C * b, C, Tp, f.R, false));
    }
    {
        rc = fwd_gemm(t->l_mfa, {GemmSource{f.OUTCAT, 0, C3, 0}}, f.Amfa, 0, true, nullptr, nullptr);
        if (rc) return rc;
        bn_fwd(t->l_mfa, f.Amfa, 0, f.M, 0, 0, nullptr, 0, nullptr, 0);
    }
    const int pool = t->cfg.pooling, Kp = t->Kp;
    // copies the [B, C3] mean half of a [B, 2*C3] softmax-pooling row block to or from a plain [B, C3] matrix (SAP)
    auto mean_half = [&](float* dst, int dst_ld, const float* src, int src_ld) {
        push("cudaMemcpy2DAsync", [dst, dst_ld, src, src_ld, B, C3](const StepRun& r) {
            PPV_CUDA_OK(cudaMemcpy2DAsync(dst, size_t(dst_ld) * sizeof(float), src, size_t(src_ld) * sizeof(float), size_t(C3) * sizeof(float), B,
                                          cudaMemcpyDeviceToDevice, r.st));
            return PPV_OK;
        });
    };
    if (t->context()) {
        // global stats -> per-utterance bias of the attention TDNN: its weight [att][3*C3], columns C3.. multiply [mean | std]
        t->steps.push_back(colstats_step(f.M, C3, B, T, P, Tp, 1, TR_ASP_EPS, f.gstat_pl));
        push("launch_planes_to_f32", [x = f.gstat_pl, Cn = 2 * C3, B, out = f.gstat](const StepRun& r) {
            return launch_planes_to_f32(x, 0, Cn, B, 1, 0, 1, out, r.st);  // one row per utterance
        });
        dense_fwd(f.gstat, 2 * C3, par + t->L[t->l_att1].conv.w_off + C3, 3 * C3, nullptr, B, att, 2 * C3, 0, f.fold, att);
    }
    if (pool == PPV_POOL_ASP) {
        rc = fwd_gemm(t->l_att1, {GemmSource{f.M, 0, C3, 0}}, f.Aatt, 0, true, f.fold, nullptr);
        if (rc) return rc;
        bn_fwd(t->l_att1, f.Aatt, 0, f.A4, 0, 1, nullptr, 0, nullptr, 0);
    } else if (pool == PPV_POOL_SAP) {  // tanh(linear1(M)) (pooling.py:62): no ReLU, no BatchNorm
        const TConv& c = t->conv(t->c_lin1);
        Epilogue ep = planes_epilogue(f.A4, 0, Tp, P, T);
        ep.bias = par + c.b_off;
        ep.tanh_ = 1;
        rc = gemm({GemmSource{f.M, 0, C3, 0}}, f.layer[t->c_lin1].wf, c.Cout, ep);
        if (rc) return rc;
    }
    if (t->attentive()) {
        rc = fwd_gemm(t->c_att2, {GemmSource{f.A4, 0, t->att, 0}}, Planes(), 0, false, nullptr, f.logits);
        if (rc) return rc;
        // softmax pooling: ASP keeps [mean | std]; SAP pools the mean alone (pooling.py:63-65)
        float* const out = pool == PPV_POOL_SAP ? f.sap_stats : f.pooled;
        push("launch_asp_pool", [logits = f.logits, C3, x = f.M, B, T, P, Tp, out](const StepRun& r) {
            return launch_asp_pool(logits, C3, x, C3, B, T, P, Tp, TR_ASP_EPS, nullptr, nullptr, Planes(), out, r.st);
        });
        if (pool == PPV_POOL_SAP) mean_half(f.pooled, C3, f.sap_stats, 2 * C3);
    } else {  // TAP: mean over time; TSP: mean | unbiased variance (pooling.py:8-47)
        t->steps.push_back(colstats_step(f.M, C3, B, T, P, Tp, pool == PPV_POOL_TAP ? 0 : 3, 0.f, Planes(), 0.f, false, f.pooled));
    }
    {
        // asp_bn (batch statistics), fc, AAM-softmax loss
        push("tr_bn1d_fwd", [x = f.pooled, B, Cn = Kp, gamma = par + t->aspbn_g, beta = par + t->aspbn_b, y = f.pn, mean = f.aspbn_mean,
                             rstd = f.aspbn_rstd, run_mean = sta + t->aspbn_rm, run_var = sta + t->aspbn_rv](const StepRun& r) {
            return tr_bn1d_fwd(x, B, Cn, TR_BN_EPS, TR_BN_MOMENTUM, gamma, beta, y, mean, rstd, run_mean, run_var, r.st);
        });
        dense_fwd(f.pn, Kp, par + t->fc_w, Kp, par + t->fc_b, B, D, Kp, 0, f.emb, D);
    }
    // classifier blocks (fc.py:27-29, 44-45): h_i = BatchNorm1D(Conv1D_1x1(h_{i-1})) with batch statistics, h_{-1} = emb
    const int Hd = t->head_dim(), nblk = int(t->cls_blocks.size());
    const float* head_in = f.emb;
    for (int i = 0; i < nblk; ++i) {
        const Trainer::ClsBlock& k = t->cls_blocks[i];
        dense_fwd(head_in, k.in, par + k.w, k.in, par + k.b, B, t->inter, k.in, 0, f.cls_z[i], t->inter);
        push("tr_bn1d_fwd", [x = f.cls_z[i], B, Cn = t->inter, gamma = par + k.g, beta = par + k.beta, y = f.cls_h[i], mean = f.cls_mean[i],
                             rstd = f.cls_rstd[i], run_mean = sta + k.rm, run_var = sta + k.rv](const StepRun& r) {
            return tr_bn1d_fwd(x, B, Cn, TR_BN_EPS, TR_BN_MOMENTUM, gamma, beta, y, mean, rstd, run_mean, run_var, r.st);
        });
        head_in = f.cls_h[i];
    }
    // the output layer and the loss head: cosine logits (fc.py:48-49) or Linear logits (fc.py:50-51); the loss reads the logits alone
    if (t->cls_type == PPV_CLASSIFIER_COSINE) {
        push("aam_forward", [emb = head_in, cls_w = par + t->cls_w, B, D = Hd, S = t->S, logits = f.cls_logits, loss = f.loss, aam_ws = f.aam_ws,
                             aam_ws_bytes = f.aam_ws_bytes](const StepRun& r) {
            const PlanInputs& in = r.in;
            return aam_forward(emb, cls_w, in.labels, B, D, S, in.margin, in.scale, in.easy_margin, in.label_smoothing, logits, loss, aam_ws,
                               aam_ws_bytes, r.st);
        });
    } else {
        push("linear_head_forward", [h = head_in, w = par + t->cls_w, bias = par + t->cls_b, B, Hd, S = t->S, logits = f.cls_logits, loss = f.loss,
                                     aam_ws = f.aam_ws, aam_ws_bytes = f.aam_ws_bytes](const StepRun& r) {
            const PlanInputs& in = r.in;
            return linear_head_forward(h, w, bias, in.labels, B, Hd, S, in.margin, in.scale, in.easy_margin, in.label_smoothing, logits, loss, aam_ws,
                                       aam_ws_bytes, r.st);
        });
    }

    // ================================================================= backward
    {
        // loss head -> the last block's dL/dh (d_emb without blocks); blocks -> d_emb; fc, asp_bn -> dpooled; ASP -> dlogits, dMd
        float* const d_head = nblk ? f.dcls_h[nblk - 1] : f.d_emb;
        if (t->cls_type == PPV_CLASSIFIER_COSINE) {
            push("aam_backward", [emb = head_in, cls_w = par + t->cls_w, logits = f.cls_logits, B, D = Hd, S = t->S, d_emb = d_head,
                                  d_cls_w = grd + t->cls_w, aam_ws = f.aam_ws, aam_ws_bytes = f.aam_ws_bytes](const StepRun& r) {
                const PlanInputs& in = r.in;
                return aam_backward(emb, cls_w, in.labels, logits, B, D, S, in.margin, in.scale, in.easy_margin, in.label_smoothing, d_emb, d_cls_w,
                                    aam_ws, aam_ws_bytes, r.st);
            });
        } else {
            push("linear_head_backward", [h = head_in, w = par + t->cls_w, logits = f.cls_logits, B, Hd, S = t->S, d_h = d_head, d_w = grd + t->cls_w,
                                          d_b = grd + t->cls_b, aam_ws = f.aam_ws, aam_ws_bytes = f.aam_ws_bytes](const StepRun& r) {
                const PlanInputs& in = r.in;
                return linear_head_backward(h, w, in.labels, logits, B, Hd, S, in.margin, in.scale, in.easy_margin, in.label_smoothing, d_h, d_w, d_b,
                                            aam_ws, aam_ws_bytes, r.st);
            });
        }
        for (int i = nblk - 1; i >= 0; --i) {  // BatchNorm over the batch, then the 1x1 conv's dX / dW / db
            const Trainer::ClsBlock& k = t->cls_blocks[i];
            push("tr_bn1d_bwd", [dy = f.dcls_h[i], x = f.cls_z[i], B, Cn = t->inter, gamma = par + k.g, mean = f.cls_mean[i], rstd = f.cls_rstd[i],
                                 dx = f.dcls_z, dgamma = grd + k.g, dbeta = grd + k.beta](const StepRun& r) {
                return tr_bn1d_bwd(dy, x, B, Cn, gamma, mean, rstd, dx, dgamma, dbeta, r.st);
            });
            dense_bwd(f.dcls_z, t->inter, i ? f.cls_h[i - 1] : f.emb, k.in, par + k.w, k.in, B, t->inter, k.in, i ? f.dcls_h[i - 1] : f.d_emb, k.in,
                      grd + k.w, k.in, grd + k.b);
        }
        dense_bwd(f.d_emb, D, f.pn, Kp, par + t->fc_w, Kp, B, D, Kp, f.dpn, Kp, grd + t->fc_w, Kp, grd + t->fc_b);
        push("tr_bn1d_bwd", [dy = f.dpn, x = f.pooled, B, Cn = Kp, gamma = par + t->aspbn_g, mean = f.aspbn_mean, rstd = f.aspbn_rstd,
                             dx = f.dpooled, dgamma = grd + t->aspbn_g, dbeta = grd + t->aspbn_b](const StepRun& r) {
            return tr_bn1d_bwd(dy, x, B, Cn, gamma, mean, rstd, dx, dgamma, dbeta, r.st);
        });
        if (t->attentive()) {
            // SAP: the softmax pooling backward reads [d mean | d std] with the std half zero (never written since the workspace
            // was cleared), so its std terms add exactly zero
            const float* pooled = f.pooled;
            const float* dpooled = f.dpooled;
            if (pool == PPV_POOL_SAP) {
                mean_half(f.dsap_stats, 2 * C3, f.dpooled, C3);
                pooled = f.sap_stats;
                dpooled = f.dsap_stats;
            }
            push("tr_asp_bwd", [logits = f.logits, C3, x = f.M, B, T, P, Tp, pooled, dpooled, dlogits = f.dlogits, dx = f.dMd](const StepRun& r) {
                return tr_asp_bwd(logits, C3, x, C3, B, T, P, Tp, TR_ASP_EPS, pooled, dpooled, dlogits, dx, r.st);
            });
        } else {
            push("tr_pool_stats_bwd", [x = f.M, C3, B, T, P, Tp, pooled = f.pooled, dpooled = f.dpooled, var = pool == PPV_POOL_TSP,
                                       dx = f.dMd](const StepRun& r) { return tr_pool_stats_bwd(x, C3, B, T, P, Tp, pooled, dpooled, var, dx, r.st); });
        }
    }
    if (t->attentive()) {
        // asp.conv / asp.linear2: bias, weight, data gradients
        GradSrcList gl;
        gl.n = 1;
        gl.s[0] = src1(f.dlogits, 0, 0);
        grad_sum(gl, C3, Planes(), grd + t->conv(t->c_att2).b_off);
        rc = wgrad(t->c_att2, f.dlogits, 0, {{f.A4, 0, t->att, 0}});
        if (rc) return rc;
        rc = dgrad_gemm(t->c_att2, f.dlogits, 0, f.dA4, 0);
        if (rc) return rc;
    }
    if (pool == PPV_POOL_ASP) {
        // attention TDNN: tanh, BN, ReLU backward; per-utterance context gradients (from the sums the BN backward leaves in f.part
        // [B][att]); frame-level weight / data gradients
        GradSrcList gl;
        gl.n = 1;
        gl.s[0] = src1(f.dA4, 0, 0);
        gl.s[0].dtanh = f.A4;
        bn_bwd(t->l_att1, gl, f.Aatt, 0, f.dZatt, 0);
        if (t->context()) {
            const TConv& c = t->L[t->l_att1].conv;
            dense_bwd(f.part, att, f.gstat, 2 * C3, par + c.w_off + C3, 3 * C3, B, att, 2 * C3, f.dgs, 2 * C3, grd + c.w_off + C3, 3 * C3, nullptr);
            push("tr_asp_global_bwd", [gstat = f.gstat, dgs = f.dgs, B, C3, T, rs = f.rs, rb = f.rb](const StepRun& r) {
                return tr_asp_global_bwd(gstat, dgs, B, C3, T, TR_ASP_EPS, rs, rb, r.st);
            });
        }
        rc = wgrad(t->l_att1, f.dZatt, 0, {{f.M, 0, C3, 0}});
        if (rc) return rc;
        rc = dgrad_gemm(t->l_att1, f.dZatt, 0, f.dMatt, 0);
        if (rc) return rc;
    } else if (pool == PPV_POOL_SAP) {
        // linear1: tanh' straight after linear2's data gradient (no BatchNorm, no ReLU); the summed rows are linear1's bias gradient
        GradSrcList gl;
        gl.n = 1;
        gl.s[0] = src1(f.dA4, 0, 0);
        gl.s[0].dtanh = f.A4;
        grad_sum(gl, att, f.dZatt, grd + t->conv(t->c_lin1).b_off);
        rc = wgrad(t->c_lin1, f.dZatt, 0, {{f.M, 0, C3, 0}});
        if (rc) return rc;
        rc = dgrad_gemm(t->c_lin1, f.dZatt, 0, f.dMatt, 0);
        if (rc) return rc;
    }
    {
        // MFA: d(M) = pooling direct (+ attention path) (+ ASP's global-context statistics, as row scale / bias on M itself)
        GradSrcList gl;
        gl.n = 1;
        gl.s[0] = src1(f.dMd, 0, 0);
        if (t->attentive()) gl.s[gl.n++] = src1(f.dMatt, 0, 0);
        if (t->context()) {
            gl.s[gl.n] = src1(f.M, 0, 0);
            gl.s[gl.n].rowscale = f.rs;
            gl.s[gl.n].rowbias = f.rb;
            gl.s[gl.n].row_ld = C3;
            gl.n++;
        }
        bn_bwd(t->l_mfa, gl, f.Amfa, 0, f.dZmfa, 0);
        rc = wgrad(t->l_mfa, f.dZmfa, 0, {{f.OUTCAT, 0, C3, 0}});
        if (rc) return rc;
        rc = dgrad_gemm(t->l_mfa, f.dZmfa, 0, f.dOUTCAT, 0);
        if (rc) return rc;
    }
    for (int b = 2; b >= 0; --b) {
        const Planes u = b == 0 ? f.Y0 : f.OUTCAT;
        const int uc = b == 0 ? 0 : C * (b - 1);
        const Planes& Dg = f.Dbuf[b];
        {
            // d(out_b) = MFA window + (next block: tdnn1 data gradient + its own residual gradient)
            GradSrcList gl;
            gl.n = 1;
            gl.s[0] = src1(f.dOUTCAT, C * b, 0);
            if (b < 2) {
                gl.n = 3;
                gl.s[1] = src1(f.dXt1[b + 1], 0, 0);
                gl.s[2] = src1(f.Dbuf[b + 1], 0, 0);
            }
            grad_sum(gl, C, Dg, nullptr);
        }
        {
            // SE backward -> dg2 ... ds (scaled by 1/T), SE weight gradients
            GradSrcList gl;
            gl.n = 1;
            gl.s[0].t = Dg;
            push("tr_grad_dot", [gl, y = f.Yt2[b], C, B, T, P, Tp, out = f.dg2](const StepRun& r) {
                return tr_grad_dot(gl, y, 0, C, B, T, P, Tp, out, r.st);
            });
            act_bwd(f.dg2, f.se_g2[b], int64_t(B) * C, 2, 0.f);
            dense_bwd(f.dg2, C, f.se_g1[b], se, par + t->se2_w[b], se, B, C, se, f.dg1, se, grd + t->se2_w[b], se, grd + t->se2_b[b]);
            act_bwd(f.dg1, f.se_g1[b], int64_t(B) * se, 1, 0.f);
            dense_bwd(f.dg1, se, f.se_s[b], C, par + t->se1_w[b], C, B, se, C, f.ds, C, grd + t->se1_w[b], C, grd + t->se1_b[b]);
            act_bwd(f.ds, nullptr, int64_t(B) * C, 0, 1.f / float(T));
        }
        {
            GradSrcList gl;
            gl.n = 1;
            gl.s[0] = src1(Dg, 0, 0);
            gl.s[0].rowscale = f.se_g2[b];
            gl.s[0].rowbias = f.ds;
            gl.s[0].row_ld = C;
            bn_bwd(t->l_tdnn2[b], gl, f.At2[b], 0, f.dZt2[b], 0);
            rc = wgrad(t->l_tdnn2[b], f.dZt2[b], 0, {{f.Yt1[b], 0, W, 0}, {f.RC[b], W, C - W, W}});
            if (rc) return rc;
            rc = dgrad_gemm(t->l_tdnn2[b], f.dZt2[b], 0, f.dRC[b], 0);
            if (rc) return rc;
        }
        for (int j = 7; j >= 1; --j) {
            GradSrcList gl;
            gl.n = 1;
            gl.s[0] = src1(f.dRC[b], W * j, 0);
            if (j < 7) {
                gl.n = 2;
                gl.s[1] = src1(f.DIN[b], W * (j + 1), 1);
            }
            const int li = t->l_res[b][j];
            bn_bwd(li, gl, f.Ares[b], W * j, f.dZres[b], W * j);
            rc = wgrad(li, f.dZres[b], W * j, {{j == 1 ? f.Yt1[b] : f.IN[b], W * j, W, 0}});
            if (rc) return rc;
            rc = dgrad_gemm(li, f.dZres[b], W * j, f.DIN[b], W * j);
            if (rc) return rc;
        }
        {
            // chunk 0 of the tdnn1 output went straight into tdnn2: copy its gradient next to the others
            GradSrcList gl;
            gl.n = 1;
            gl.s[0] = src1(f.dRC[b], 0, 0);
            grad_sum(gl, W, f.DIN[b], nullptr);
        }
        {
            GradSrcList gl;
            gl.n = 1;
            gl.s[0] = src1(f.DIN[b], 0, 1);
            bn_bwd(t->l_tdnn1[b], gl, f.At1[b], 0, f.dZt1[b], 0);
            rc = wgrad(t->l_tdnn1[b], f.dZt1[b], 0, {{u, uc, C, 0}});
            if (rc) return rc;
            rc = dgrad_gemm(t->l_tdnn1[b], f.dZt1[b], 0, f.dXt1[b], 0);
            if (rc) return rc;
        }
    }
    {
        GradSrcList gl;
        gl.n = 2;
        gl.s[0] = src1(f.dXt1[0], 0, 0);
        gl.s[1] = src1(f.Dbuf[0], 0, 0);
        bn_bwd(t->l_conv0, gl, f.A0, 0, f.dZ0, 0);
        rc = wgrad(t->l_conv0, f.dZ0, 0, {{f.X0, 0, t->Fp, 0}});
        if (rc) return rc;
    }
    return PPV_OK;
}

int trainer_forward_backward(Trainer* t, const float* feat, const int64_t* labels, int B, int T, float margin, float scale, int easy_margin,
                             float label_smoothing, float* loss_out, float* logits_out, void* ws, size_t ws_bytes, cudaStream_t st) {
    PPV_REQUIRE(t && feat && labels, "trainer_forward_backward: null argument");
    PPV_REQUIRE(B > 1 && T > 0, "trainer_forward_backward: batch of at least 2 required (batch statistics)");
    int rc = t->update_plan(B, T, ws, ws_bytes, st);
    if (!rc) rc = t->run_plan(PlanInputs{feat, nullptr, labels, margin, scale, label_smoothing, easy_margin}, st);
    if (rc) return rc;
    if (loss_out) PPV_CUDA_OK(cudaMemcpyAsync(loss_out, t->buf.loss, sizeof(float), cudaMemcpyDeviceToDevice, st));
    if (logits_out) PPV_CUDA_OK(cudaMemcpyAsync(logits_out, t->buf.cls_logits, size_t(B) * t->S * sizeof(float), cudaMemcpyDeviceToDevice, st));
    return PPV_OK;
}

// Taps for tests and debugging: every buffer of the step stays readable after it (tr_carve aliases none).
//   planes -> fp32 [B, T, C], valid frames; with the prefix "pad:" all Tp = T + 2P rows of every utterance, halo rows included
//     forward   "blocks.0".."blocks.3", "mfa" (block outputs); X0, A0, Y0, OUTCAT, Amfa, M, Aatt, A4; per block ("<name>:<0..2>")
//               At1, Yt1, Ares, RC, IN, At2, Yt2.  A* are the post-ReLU, pre-BatchNorm activations the BatchNorm backward reads.
//     gradients "g:<name>": dZ0, dOUTCAT, dMd, dMatt, dZmfa, dlogits, dZatt, dA4; per block D, dZt2, dRC, dZres, DIN, dZt1, dXt1
//   fp32 as stored: "asp" (pooled) [B, Kp], "emb" and "d_emb" [B, D], "logits" [B, Tp, C3] (every row), gstat, dgs [B, 2*C3], pn, dpn,
//     dpooled [B, Kp], rs, rb [B, C3]; SAP: sap_stats (the softmax pooling's [mean | std]) and dsap_stats (the [d mean | 0] its backward
//     reads) [B, 2*C3]; per block se_s, se_g2 [B, C], se_g1 [B, se]; dg2, ds [B, C] and dg1 [B, se] are scratch that every block's SE
//     backward overwrites, so they hold block 0's values.  With classifier blocks: "classifier.blocks.<i>" (block i's output),
//     "classifier.blocks.<i>.z" (its dense output, the BatchNorm's input), "g:classifier.blocks.<i>" (dL/d output) and "g:classifier.z"
//     (the dL/dz scratch every block's BatchNorm backward overwrites, so it holds block 0's) [B, inter_dim].
// Kp = 2*C3 for ASP and TSP, C3 for SAP and TAP.  A head has the taps of the buffers it uses: Aatt, gstat, dgs, rs, rb are ASP's (the last
// four with global context), A4, logits and the attention gradients ASP's and SAP's.
// A per-block name without a block suffix reads block 0.
int trainer_read_tap(Trainer* t, const char* name, float* out, size_t out_elems, cudaStream_t st) {
    PPV_REQUIRE(t && name && out, "trainer_read_tap: null argument");
    if (!t->plan_ws) return fail(PPV_ESTATE, "trainer_read_tap: no step has run");
    std::string n(name);
    const bool padded = n.rfind("pad:", 0) == 0;
    if (padded) n = n.substr(4);
    int b = -1;  // block suffix
    const size_t colon = n.rfind(':');
    if (colon != std::string::npos && colon + 2 == n.size() && n.back() >= '0' && n.back() <= '9') {
        b = n.back() - '0';
        n.resize(colon);
        PPV_REQUIRE(b < 3, "trainer_read_tap: bad block");
    }
    const auto it = t->taps.find(n);
    if (it == t->taps.end() || (b >= 0 && !it->second.per_block) || (padded && it->second.fp32))
        return fail(PPV_EINVAL, std::string("trainer_read_tap: unknown tap ") + name);
    const TrTap& e = it->second;
    const int bk = std::max(b, 0);
    if (e.fp32) {
        PPV_REQUIRE(out_elems >= e.count, "trainer_read_tap: output too small");
        PPV_CUDA_OK(cudaMemcpyAsync(out, e.vec[bk], e.count * sizeof(float), cudaMemcpyDeviceToDevice, st));
        return PPV_OK;
    }
    const int B = t->plan_B, Tp = t->buf.Tp, rows = padded ? Tp : t->plan_T;
    PPV_REQUIRE(out_elems >= size_t(B) * rows * e.cols, "trainer_read_tap: output too small");
    return launch_planes_to_f32(e.pl[bk], e.col0, e.cols, B, rows, padded ? 0 : t->P, Tp, out, st);
}

}  // namespace ppv
