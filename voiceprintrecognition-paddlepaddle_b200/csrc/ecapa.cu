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

#include <map>
#include <string>
#include <vector>

#include "common.h"

namespace ppv {

namespace {

struct HostW {
    std::vector<float> v;
    std::vector<int64_t> shape;
};

struct ConvW {  // a conv / linear layer prepared for the gather-GEMM
    Planes W;   // [2][N][Ktot] split-bf16
    float* bias = nullptr;
    float* bn_scale = nullptr;
    float* bn_shift = nullptr;
    int N = 0, Ktot = 0;
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
    int BN = 0;
    int blk = 0;  // block index for the SE steps
};

inline size_t align_up(size_t x, size_t a) { return (x + a - 1) / a * a; }

}  // namespace

struct EcapaModel {
    ppv_ecapa_cfg cfg;
    std::map<std::string, HostW> raw;
    bool finalized = false;
    int precision = PPV_PREC_BF16X3;
    int num_sms = 132;
    int C = 0, C3 = 0, width = 0, scale = 0, Fp = 0, P = 0, att = 0, se = 0;
    // device weights
    void* arena = nullptr;
    size_t arena_bytes = 0, arena_used = 0;
    ConvW conv0, tdnn1[3], res2[3][8], tdnn2[3], se1[3], se2[3], mfa, fold, att1, att2, fc;
    float *aspbn_scale = nullptr, *aspbn_shift = nullptr;
    // plan
    std::vector<Step> steps;
    void* plan_ws = nullptr;
    int plan_B = 0, plan_T = 0, plan_prec = -1;
    Planes bufs[B_COUNT];
    float *se_mean = nullptr, *se_scale = nullptr, *fold_out = nullptr, *logits = nullptr, *pooled_raw = nullptr,
          *raw_logmel = nullptr, *emb_out = nullptr;
    int* nvalid = nullptr;  // [B] valid-frame counts of the current forward (`lengths`), workspace
    int Tp = 0;
    // profiling (bench.py roofline): CUDA events around every launch group of the forward
    bool prof_on = false;
    std::vector<cudaEvent_t> prof_ev;   // pairs
    std::vector<int> prof_kind;         // 0 = tensor-core GEMM, 1 = other kernels
    size_t prof_used = 0;
    int64_t launches_gemm = 0, launches_other = 0;
};

// ------------------------------------------------------------------------------------------------ create / load
int ecapa_create(const ppv_ecapa_cfg* cfg, EcapaModel** out) {
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
    EcapaModel* m = new EcapaModel();
    m->cfg = *cfg;
    m->precision = cfg->precision;
    m->C = C;
    m->C3 = 3 * C;
    m->width = width;
    m->scale = cfg->res2net_scale;
    m->Fp = int(align_up(cfg->input_size, 64));
    m->att = cfg->attention_channels;
    m->se = cfg->se_channels;
    int P = (cfg->kernel_sizes[0] - 1) / 2 * cfg->dilations[0];
    for (int i = 1; i <= 3; ++i) P = std::max(P, cfg->dilations[i]);
    m->P = P;
    m->num_sms = device_sm_count();
    *out = m;
    return PPV_OK;
}

void ecapa_destroy(EcapaModel* m) {
    if (!m) return;
    for (cudaEvent_t e : m->prof_ev) cudaEventDestroy(e);
    cudaFree(m->arena);
    delete m;
}

int ecapa_embd_dim(const EcapaModel* m) { return m->cfg.embd_dim; }

int ecapa_set_precision(EcapaModel* m, int precision) {
    PPV_REQUIRE(precision == PPV_PREC_BF16X3 || precision == PPV_PREC_BF16, "bad precision");
    m->precision = precision;
    return PPV_OK;
}

int ecapa_load_weight(EcapaModel* m, const char* name, const float* data, const int64_t* shape, int ndim) {
    PPV_REQUIRE(m && name && data && shape && ndim >= 1 && ndim <= 4, "ecapa_load_weight: bad argument");
    if (m->finalized) return fail(PPV_ESTATE, "ecapa_load_weight: model already finalized");
    HostW w;
    int64_t n = 1;
    for (int i = 0; i < ndim; ++i) {
        w.shape.push_back(shape[i]);
        n *= shape[i];
    }
    w.v.resize(size_t(n));
    cudaPointerAttributes attr;
    cudaError_t e = cudaPointerGetAttributes(&attr, data);
    if (e == cudaSuccess && (attr.type == cudaMemoryTypeDevice || attr.type == cudaMemoryTypeManaged)) {
        PPV_CUDA_OK(cudaMemcpy(w.v.data(), data, size_t(n) * sizeof(float), cudaMemcpyDeviceToHost));
    } else {
        cudaGetLastError();
        memcpy(w.v.data(), data, size_t(n) * sizeof(float));
    }
    m->raw[name] = std::move(w);
    return PPV_OK;
}

// ------------------------------------------------------------------------------------------------ finalize
namespace {

struct Finalizer {
    EcapaModel* m;
    std::vector<uint8_t> host;  // staged arena image
    std::string err;

    size_t reserve(size_t bytes) {
        const size_t off = align_up(host.size(), 256);
        host.resize(off + bytes, 0);
        return off;
    }
    const HostW* get(const std::string& name, std::initializer_list<int64_t> shape) {
        auto it = m->raw.find(name);
        if (it == m->raw.end()) {
            err = "missing weight " + name;
            return nullptr;
        }
        if (it->second.shape != std::vector<int64_t>(shape)) {
            err = "weight " + name + " has the wrong shape";
            return nullptr;
        }
        return &it->second;
    }
    // offsets are patched to pointers after upload
    size_t put_f32(const std::vector<float>& v) {
        const size_t off = reserve(v.size() * sizeof(float));
        memcpy(host.data() + off, v.data(), v.size() * sizeof(float));
        return off;
    }
    // conv weight [N, Cin, k] -> split planes [2][Npad][Ktot] following the K groups
    bool put_conv(ConvW* cw, const HostW* w, int N, int Cin, int k, const std::vector<KSpec>& ks, size_t* off_out) {
        int Ktot = 0;
        for (const KSpec& s : ks) Ktot += s.ncols;
        const int Npad = int(align_up(N, 128));
        const size_t plane = size_t(Npad) * Ktot;
        const size_t off = reserve(2 * plane * sizeof(__nv_bfloat16));
        __nv_bfloat16* hi = reinterpret_cast<__nv_bfloat16*>(host.data() + off);
        __nv_bfloat16* lo = hi + plane;
        for (size_t i = 0; i < 2 * plane; ++i) hi[i] = __float2bfloat16_rn(0.f);
        for (int n = 0; n < N; ++n) {
            int kpos = 0;
            for (const KSpec& s : ks) {
                for (int c = 0; c < s.w_cnt; ++c) {
                    const float x = w->v[(size_t(n) * Cin + s.w_cin0 + c) * k + s.w_tap];
                    const __nv_bfloat16 h = __float2bfloat16_rn(x);
                    hi[size_t(n) * Ktot + kpos + c] = h;
                    lo[size_t(n) * Ktot + kpos + c] = __float2bfloat16_rn(x - __bfloat162float(h));
                }
                kpos += s.ncols;
            }
        }
        cw->N = N;
        cw->Ktot = Ktot;
        cw->W.rows = Npad;
        cw->W.ld = Ktot;
        cw->W.plane_stride = int64_t(plane);
        *off_out = off;
        return true;
    }
    // BatchNorm eval -> y = x * scale + shift  (ppvector/models/utils.py:96-119, eps 1e-5)
    bool bn_affine(const std::string& prefix, int C, std::vector<float>* scale, std::vector<float>* shift) {
        const HostW *g = get(prefix + ".weight", {C}), *b = get(prefix + ".bias", {C}), *mu = get(prefix + "._mean", {C}),
                    *var = get(prefix + "._variance", {C});
        if (!g || !b || !mu || !var) return false;
        scale->resize(C);
        shift->resize(C);
        for (int i = 0; i < C; ++i) {
            const double s = double(g->v[i]) / sqrt(double(var->v[i]) + 1e-5);
            (*scale)[i] = float(s);
            (*shift)[i] = float(double(b->v[i]) - double(mu->v[i]) * s);
        }
        return true;
    }
};

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

int ecapa_finalize(EcapaModel* m) {
    PPV_REQUIRE(m, "ecapa_finalize: null model");
    if (m->finalized) return PPV_OK;
    Finalizer f{m, {}, ""};
    const int C = m->C, C3 = m->C3, w = m->width, F = m->cfg.input_size, A = m->att, S = m->se, E = m->cfg.embd_dim;
    const int k0 = m->cfg.kernel_sizes[0];
    struct Patch {
        void** dst;
        size_t off;
    };
    std::vector<Patch> patches;
    auto patch = [&](void* dst, size_t off) { patches.push_back({reinterpret_cast<void**>(dst), off}); };
    auto put_vec = [&](float** dst, const std::vector<float>& v) { patch(dst, f.put_f32(v)); };
    auto conv_layer = [&](ConvW* cw, const std::string& wname, int N, int Cin, int k, const std::vector<KSpec>& ks,
                          const std::string& bn_prefix, bool has_bias) -> bool {
        const HostW* hw = f.get(wname + ".weight", {N, Cin, k});
        if (!hw) return false;
        size_t off;
        f.put_conv(cw, hw, N, Cin, k, ks, &off);
        patch(&cw->W.base, off);
        if (has_bias) {
            const HostW* hb = f.get(wname + ".bias", {N});
            if (!hb) return false;
            put_vec(&cw->bias, hb->v);
        }
        if (!bn_prefix.empty()) {
            std::vector<float> sc, sh;
            if (!f.bn_affine(bn_prefix, N, &sc, &sh)) return false;
            put_vec(&cw->bn_scale, sc);
            put_vec(&cw->bn_shift, sh);
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
        const HostW* w = f.get("fc.conv.weight", {E, Kp, 1});
        const HostW* b = f.get("fc.conv.bias", {E});
        std::vector<float> sc, sh;
        if (!w || !b || !f.bn_affine("asp_bn", Kp, &sc, &sh)) return false;  // paddle.nn.BatchNorm1D: keys asp_bn.weight / ._mean ...
        HostW wf;
        wf.shape = {E, Kp, 1};
        wf.v.resize(size_t(E) * Kp);
        std::vector<float> bf(E);
        for (int n = 0; n < E; ++n) {
            double acc = b->v[n];
            for (int k = 0; k < Kp; ++k) {
                wf.v[size_t(n) * Kp + k] = w->v[size_t(n) * Kp + k] * sc[k];
                acc += double(w->v[size_t(n) * Kp + k]) * sh[k];
            }
            bf[n] = float(acc);
        }
        size_t off;
        f.put_conv(&m->fc, &wf, E, Kp, 1, {{B_POOL, 0, Kp, 0, 0, Kp, 0}}, &off);
        patch(&m->fc.W.base, off);
        put_vec(&m->fc.bias, bf);
        return true;
    };
    if (pooling == PPV_POOL_ASP) {
    // ASP attention TDNN: weight [A, 3*C3, 1] split into the x part (cols 0..C3) and the [mean;std] part;
    // global_context = False (pooling.py:77-78, 108-109): the TDNN sees x alone, weight [A, C3, 1], no per-utterance bias
    const int ctx = m->cfg.global_context ? 3 : 1;
    ok = ok && conv_layer(&m->att1, "asp.tdnn.conv.conv", A, ctx * C3, 1, {{B_MFA, 0, C3, 0, 0, C3, 0}}, "asp.tdnn.norm.norm", true);
    if (ok && m->cfg.global_context) {
        const HostW* hw = f.get("asp.tdnn.conv.conv.weight", {A, 3 * C3, 1});
        size_t off;
        f.put_conv(&m->fold, hw, A, 3 * C3, 1, {{B_GSTAT, 0, 2 * C3, 0, C3, 2 * C3, 0}}, &off);
        patch(&m->fold.W.base, off);
    }
    ok = ok && conv_layer(&m->att2, "asp.conv.conv", C3, A, 1, {{B_ATT, 0, A, 0, 0, A, 0}}, "", true);
    ok = ok && conv_layer(&m->fc, "fc.conv", E, 2 * C3, 1, {{B_POOL, 0, 2 * C3, 0, 0, 2 * C3, 0}}, "", true);
    if (ok) {
        std::vector<float> sc, sh;
        ok = f.bn_affine("asp_bn.norm", 2 * C3, &sc, &sh);
        if (ok) {
            put_vec(&m->aspbn_scale, sc);
            put_vec(&m->aspbn_shift, sh);
        }
    }
    } else if (pooling == PPV_POOL_SAP) {
        // SelfAttentivePooling (pooling.py:50-66): alpha = softmax_t(linear2(tanh(linear1(x)))); mean = sum alpha x.  The fused ASP
        // kernel computes exactly this weighted mean (its std half is ignored); linear2's bias cancels in the softmax.
        if (A != 128) {
            f.err = "SAP pooling uses a 128-channel bottleneck (ecapa_tdnn.py:222): attention_channels must be 128";
            ok = false;
        }
        ok = ok && conv_layer(&m->att1, "asp.linear1", A, C3, 1, {{B_MFA, 0, C3, 0, 0, C3, 0}}, "", true);
        ok = ok && conv_layer(&m->att2, "asp.linear2", C3, A, 1, {{B_ATT, 0, A, 0, 0, A, 0}}, "", true);
        ok = ok && folded_fc(C3);
        if (ok) {
            put_vec(&m->aspbn_scale, std::vector<float>(2 * C3, 1.f));
            put_vec(&m->aspbn_shift, std::vector<float>(2 * C3, 0.f));
        }
    } else {
        ok = ok && folded_fc(pooling == PPV_POOL_TAP ? C3 : 2 * C3);
    }
    if (!ok) return fail(PPV_EINVAL, "ecapa_finalize: " + f.err);
    PPV_CUDA_OK(cudaMalloc(&m->arena, f.host.size()));
    m->arena_bytes = f.host.size();
    PPV_CUDA_OK(cudaMemcpy(m->arena, f.host.data(), f.host.size(), cudaMemcpyHostToDevice));
    for (const Patch& p : patches) *p.dst = static_cast<uint8_t*>(m->arena) + p.off;
    m->raw.clear();
    m->finalized = true;
    return PPV_OK;
}

// ------------------------------------------------------------------------------------------------ workspace
namespace {

struct Carver {
    uint8_t* base;
    size_t off = 0;
    void* take(size_t bytes) {
        off = align_up(off, 256);
        void* p = base ? base + off : nullptr;
        off += bytes;
        return p;
    }
    Planes planes(int64_t rows, int ld) {
        Planes p;
        p.rows = int64_t(align_up(size_t(rows), 128));
        p.ld = ld;
        p.plane_stride = p.rows * ld;
        p.base = static_cast<__nv_bfloat16*>(take(size_t(2) * p.plane_stride * sizeof(__nv_bfloat16)));
        return p;
    }
};

void carve(EcapaModel* m, Carver& cv, int B, int T) {
    const int Tp = T + 2 * m->P;
    const int64_t R = int64_t(B) * Tp;
    const int C = m->C, C3 = m->C3;
    m->bufs[B_FEAT] = cv.planes(R, m->Fp);
    m->bufs[B_X0] = cv.planes(R, C);
    m->bufs[B_H] = cv.planes(R, C);
    m->bufs[B_Y] = cv.planes(R, C);
    m->bufs[B_Z] = cv.planes(R, C);
    m->bufs[B_CAT] = cv.planes(R, C3);
    m->bufs[B_MFA] = cv.planes(R, C3);
    m->bufs[B_ATT] = cv.planes(R, m->att);
    m->bufs[B_GSTAT] = cv.planes(B, 2 * C3);
    m->bufs[B_POOL] = cv.planes(B, 2 * C3);
    m->bufs[B_SEM] = cv.planes(B, C);
    m->bufs[B_SEH] = cv.planes(B, m->se);
    m->se_mean = static_cast<float*>(cv.take(size_t(B) * C * 4));
    m->se_scale = static_cast<float*>(cv.take(size_t(B) * C * 4));
    m->fold_out = static_cast<float*>(cv.take(size_t(align_up(B, 128)) * m->att * 4));
    m->pooled_raw = static_cast<float*>(cv.take(size_t(B) * 2 * C3 * 4));
    m->raw_logmel = static_cast<float*>(cv.take(size_t(B) * T * m->cfg.input_size * 4));
    m->emb_out = static_cast<float*>(cv.take(size_t(align_up(B, 128)) * m->cfg.embd_dim * 4));
    m->nvalid = static_cast<int*>(cv.take(size_t(B) * sizeof(int)));
    m->Tp = Tp;
}

// 128-wide n-tiles even where N allows 256: on an H100 SXM at 700 W (tools/gemm_bench.py, M = 78 336, profiles/gemm_bench_after.txt)
// BN = 128 with 64-wide k-steps takes 15-18 % less time than BN = 256 at every large layer of the model (N x K = 512 x 512 / 640,
// 1536 x 1536, split-bf16 x3), and no BN = 256 variant beats it by more than run-to-run noise.
inline int pick_bn(int N) { return (N % 128 == 0) ? 128 : 64; }

}  // namespace

size_t ecapa_workspace_bytes(const EcapaModel* m, int B, int T) {
    if (!m || B <= 0 || T <= 0) return 0;
    EcapaModel tmp = *m;  // carve on a copy with a null base
    tmp.raw.clear();
    tmp.steps.clear();
    Carver cv{nullptr};
    carve(&tmp, cv, B, T);
    return align_up(cv.off, 256);
}

// ------------------------------------------------------------------------------------------------ plan
static int build_plan(EcapaModel* m, int B, int T, void* ws, size_t ws_bytes, cudaStream_t st) {
    PPV_REQUIRE(T > m->P, "ecapa: too few frames for the reflect padding");
    const size_t need = ecapa_workspace_bytes(m, B, T);
    PPV_REQUIRE(ws && ws_bytes >= need, "ecapa: workspace too small (see ppv_model_workspace_bytes)");
    PPV_REQUIRE((reinterpret_cast<uintptr_t>(ws) & 255) == 0, "ecapa: workspace must be 256-byte aligned");
    Carver cv{static_cast<uint8_t*>(ws)};
    carve(m, cv, B, T);
    // garbage rows (halo of never-written buffers) must at least be finite
    PPV_CUDA_OK(cudaMemsetAsync(ws, 0, need, st));
    m->steps.clear();
    const int Tp = m->Tp, P = m->P, C = m->C, C3 = m->C3, w = m->width;
    const int64_t R = int64_t(B) * Tp;
    const char* r2env = getenv("PPV_RES2_GEMM");  // debugging aid: 1 = run the Res2Net convs through the generic gather-GEMM
    const bool use_res2_kernel = (w == 64) && !(r2env && r2env[0] == '1');
    const char* rcenv = getenv("PPV_RES2_CHAIN");  // 0 = one launch per Res2Net conv (res2conv.cu) instead of the fused chain
    const bool use_res2_chain = use_res2_kernel && m->scale == 8 && res2chain_fits(T, P) && !(rcenv && rcenv[0] == '0');
    const char* skenv = getenv("PPV_SKINNY");  // 0 = the per-utterance linear layers through the tensor-core gather-GEMM (A-B timing)
    const bool use_skinny = !(skenv && skenv[0] == '0');
    const char* bkenv = getenv("PPV_GEMM_BK32");  // experiment: 1 = 32-wide k-steps (SWIZZLE_64B) on the wide-N layers
    const bool bk32_enabled = (bkenv && bkenv[0] == '1');

    auto add_gemm = [&](const ConvW& cw, const std::vector<KSpec>& ks, const Planes* src_override, int override_col0, int M,
                        Epilogue ep) -> int {
        std::vector<GemmSource> srcs;
        for (const KSpec& s : ks) {
            GemmSource g;
            if (s.src < 0) {
                g.t = *src_override;
                g.col0 = override_col0 + s.col0;
            } else {
                g.t = m->bufs[s.src];
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
        stp.BN = pick_bn(cw.N);
        // 32-wide k-steps (twice the ring slots) for the wide-N layers whose K fits the k-step table
        const int bk = (cw.N >= 512 && cw.Ktot <= 32 * GEMM_MAX_KSTEPS && bk32_enabled) ? 32 : 64;
        int rc = gemm_build(&stp.gp, srcs.data(), int(srcs.size()), cw.W, M, cw.N, ep, stp.BN, bk);
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
    int rc = add_gemm(m->conv0, spec_conv0(m), nullptr, 0, int(R), planes_out(m->bufs[B_X0], 0, false));
    if (rc) return rc;
    for (int b = 1; b <= 3; ++b) {
        const Planes& X = (b == 1) ? m->bufs[B_X0] : m->bufs[B_CAT];
        const int xcol = (b == 1) ? 0 : (b - 2) * C;
        // the fused Res2Net chain builds the reflect halo rows itself, so tdnn1 writes no halo rows (and gets the lean epilogue)
        rc = add_gemm(m->tdnn1[b - 1], {{-1, 0, C, 0, 0, C, 0}}, &X, xcol, int(R), planes_out(m->bufs[B_H], 0, !use_res2_chain));
        if (rc) return rc;
        if (use_res2_chain) {  // all seven convs in one kernel, one utterance per CTA, operands resident in shared memory (res2chain.cu)
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
            rc = res2chain_build(&stp.cp, m->bufs[B_H], m->bufs[B_Y], Wj, bj, sj, hj, m->scale - 1, B, T, P, Tp, m->cfg.dilations[b]);
            if (rc) return rc;
            m->steps.push_back(stp);
        }
        for (int j = 1; j < m->scale && !use_res2_chain; ++j) {
            if (use_res2_kernel) {  // weight-stationary kernel, one tall tile per source (res2conv.cu)
                GemmSource srcs[2];
                srcs[0] = GemmSource{m->bufs[B_H], j * w, w, 0};
                srcs[1] = GemmSource{m->bufs[B_Y], (j - 1) * w, w, 0};
                Epilogue ep = planes_out(m->bufs[B_Y], j * w, true);
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
                rc = add_gemm(m->res2[b - 1][j], spec_res2(m, b, j), nullptr, 0, int(R), planes_out(m->bufs[B_Y], j * w, true));
                if (rc) return rc;
            }
        }
        rc = add_gemm(m->tdnn2[b - 1], {{B_H, 0, w, 0, 0, w, 0}, {B_Y, w, C - w, 0, w, C - w, 0}}, nullptr, 0, int(R),
                      planes_out(m->bufs[B_Z], 0, false));
        if (rc) return rc;
        Step s;
        s.blk = b;
        s.kind = Step::SE_SQUEEZE;
        m->steps.push_back(s);
        {  // s = sigmoid(W2 relu(W1 mean + b1) + b2): [B,C] -> [B,S] -> [B,C], plain (un-padded) row layout
            Epilogue e1;
            e1.out_mode = OUT_PLANES;
            e1.out = m->bufs[B_SEH].base;
            e1.out_ld = m->bufs[B_SEH].ld;
            e1.out_plane_stride = m->bufs[B_SEH].plane_stride;
            e1.relu = 1;
            rc = add_gemm(m->se1[b - 1], {{B_SEM, 0, C, 0, 0, 0, 0}}, nullptr, 0, B, e1);
            if (rc) return rc;
            Epilogue e2;
            e2.out_mode = OUT_F32;
            e2.out = m->se_scale;
            e2.out_ld = C;
            e2.sigmoid_ = 1;
            rc = add_gemm(m->se2[b - 1], {{B_SEH, 0, m->se, 0, 0, 0, 0}}, nullptr, 0, B, e2);
            if (rc) return rc;
        }
        s.kind = Step::SE_SCALE;
        m->steps.push_back(s);
    }
    rc = add_gemm(m->mfa, {{B_CAT, 0, C3, 0, 0, C3, 0}}, nullptr, 0, int(R), planes_out(m->bufs[B_MFA], 0, false));
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
        ep.out = m->fold_out;
        ep.out_ld = m->att;
        ConvW cw = m->fold;
        cw.bias = nullptr;
        rc = add_gemm(cw, {{B_GSTAT, 0, 2 * C3, 0, 0, 0, 0}}, nullptr, 0, B, ep);
        if (rc) return rc;
    }
    if (pooling == PPV_POOL_ASP || pooling == PPV_POOL_SAP) {
        {  // ASP: attention TDNN (K = C3) + per-utterance bias -> ReLU -> BN -> tanh;  SAP: tanh(linear1(x))
            Epilogue ep = planes_out(m->bufs[B_ATT], 0, false);
            if (pooling == PPV_POOL_ASP) {
                if (m->cfg.global_context) ep.rowgrp_bias = m->fold_out;
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
            rc = asp_fused_build(&s.ap, m->att2.W, m->bufs[B_ATT], m->bufs[B_MFA], m->bufs[B_GSTAT], m->aspbn_scale, m->aspbn_shift,
                                 m->bufs[B_POOL], m->pooled_raw, B, T, P, Tp, C3, m->att, 1e-12f);
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
    m->plan_ws = ws;
    m->plan_B = B;
    m->plan_T = T;
    return PPV_OK;
}

// ------------------------------------------------------------------------------------------------ forward
int ecapa_forward(EcapaModel* m, const float* feat, Fbank* fb, const float* wav, const float* lens_ratio, int B, int T, int L,
                  float* emb, void* ws, size_t ws_bytes, cudaStream_t st, const float* lengths) {
    PPV_REQUIRE(m && emb, "ecapa_forward: null argument");
    if (!m->finalized) return fail(PPV_ESTATE, "ecapa_forward: call ppv_model_finalize first");
    PPV_REQUIRE(B > 0 && T > 0, "ecapa_forward: empty batch");
    PPV_REQUIRE((feat != nullptr) != (wav != nullptr), "ecapa_forward: exactly one of feat / wav");
    if (wav) {
        PPV_REQUIRE(fb, "ecapa_forward: wav input needs a fbank handle");
        PPV_REQUIRE(fbank_n_mels(fb) == m->cfg.input_size, "ecapa_forward: fbank n_mels != model input_size");
        PPV_REQUIRE(fbank_num_frames(fb, L) == T, "ecapa_forward: frame count mismatch");
    }
    if (m->plan_ws != ws || m->plan_B != B || m->plan_T != T) {
        int rc = build_plan(m, B, T, ws, ws_bytes, st);
        if (rc) {
            m->plan_ws = nullptr;
            return rc;
        }
    }
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
        rc = launch_lengths_to_counts(lengths, B, T, m->nvalid, st);
        if (rc) return rc;
        nv = m->nvalid;
    }
    prof_mark(1, true);
    if (wav) {
        rc = fbank_run(fb, wav, lens_ratio, B, L, m->raw_logmel, nullptr, m->bufs[B_FEAT], P, Tp, st);
        m->launches_other += 3;
    } else {
        rc = launch_pack_features(feat, B, T, m->cfg.input_size, m->bufs[B_FEAT], P, Tp, st);
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
            case Step::GEMM: rc = gemm_launch(s.gp, s.BN, m->precision, m->num_sms, st); break;
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
                rc = launch_colstats(m->bufs[B_Z], 0, C, B, T, P, Tp, 0, 0.f, nullptr, m->bufs[B_SEM], st, 0.f, nv);
                break;
            case Step::SE_SCALE: {
                const Planes& X = (s.blk == 1) ? m->bufs[B_X0] : m->bufs[B_CAT];
                const int xcol = (s.blk == 1) ? 0 : (s.blk - 2) * C;
                rc = launch_se_scale_res(m->bufs[B_Z], m->se_scale, X, xcol, m->bufs[B_CAT], (s.blk - 1) * C, C, Tp, R, m->num_sms, st);
                break;
            }
            case Step::ASP_GLOBAL:
                rc = launch_colstats(m->bufs[B_MFA], 0, C3, B, T, P, Tp, 1, 1e-12f, nullptr, m->bufs[B_GSTAT], st, 0.f, nv);
                break;
            case Step::ASP_FUSED: {
                AspFusedParams ap = s.ap;
                ap.nvalid = nv;
                rc = asp_fused_launch(ap, m->precision, m->num_sms, st);
                break;
            }
            case Step::POOL_STATS:
                rc = launch_colstats(m->bufs[B_MFA], 0, C3, B, T, P, Tp, m->cfg.pooling == PPV_POOL_TAP ? 0 : 3, 0.f, nullptr, m->bufs[B_POOL], st);
                break;
        }
        prof_mark(0, false);
        if (rc) return rc;
    }
    PPV_CUDA_OK(cudaMemcpyAsync(emb, m->emb_out, size_t(B) * m->cfg.embd_dim * sizeof(float), cudaMemcpyDeviceToDevice, st));
    return PPV_OK;
}

int ecapa_profile(EcapaModel* m, int enable) {
    PPV_REQUIRE(m, "ecapa_profile: null model");
    m->prof_on = enable != 0;
    m->prof_used = 0;
    m->launches_gemm = m->launches_other = 0;
    return PPV_OK;
}

// Sums the event-pair durations recorded since ecapa_profile(m, 1); synchronises on the last event.
int ecapa_profile_read(EcapaModel* m, double* gemm_ms, double* other_ms, int64_t* gemm_launches, int64_t* other_launches) {
    PPV_REQUIRE(m && gemm_ms && other_ms && gemm_launches && other_launches, "ecapa_profile_read: null argument");
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

int ecapa_read_tap(EcapaModel* m, const char* name, float* out, size_t out_elems, cudaStream_t st) {
    PPV_REQUIRE(m && name && out, "ecapa_read_tap: null argument");
    if (!m->plan_ws) return fail(PPV_ESTATE, "ecapa_read_tap: no forward has run");
    const std::string n(name);
    const int B = m->plan_B, T = m->plan_T, P = m->P, Tp = m->Tp, C = m->C, C3 = m->C3;
    const Planes* src = nullptr;
    int col0 = 0, cols = 0;
    if (n == "feat") {
        src = &m->bufs[B_FEAT];
        cols = m->cfg.input_size;
    } else if (n == "blocks.0") {
        src = &m->bufs[B_X0];
        cols = C;
    } else if (n == "blocks.1" || n == "blocks.2" || n == "blocks.3") {
        src = &m->bufs[B_CAT];
        col0 = (n.back() - '1') * C;
        cols = C;
    } else if (n == "mfa") {
        src = &m->bufs[B_MFA];
        cols = C3;
    } else if (n == "asp") {
        PPV_REQUIRE(out_elems >= size_t(B) * 2 * C3, "ecapa_read_tap: output too small");
        PPV_CUDA_OK(cudaMemcpyAsync(out, m->pooled_raw, size_t(B) * 2 * C3 * 4, cudaMemcpyDeviceToDevice, st));
        return PPV_OK;
    } else {
        return fail(PPV_EINVAL, "ecapa_read_tap: unknown tap " + n);
    }
    PPV_REQUIRE(out_elems >= size_t(B) * T * cols, "ecapa_read_tap: output too small");
    return launch_planes_to_f32(*src, col0, cols, B, T, P, Tp, out, st);
}

}  // namespace ppv
