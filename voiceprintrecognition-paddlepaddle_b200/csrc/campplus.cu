// CAM++ (CAMPPlus) forward as a plan of tensor-core gather-GEMMs.
// Reference graph: ppvector/models/campplus.py:342-346 (CAMPPlus.forward), :278-289 (FCM head), :245-251 (BasicResBlock),
// :61-64 (TDNNLayer), :88-106 (CAMLayer + seg_pooling), :135-141 (CAMDenseTDNNLayer), :167-171 (dense concat),
// :183-186 (TransitLayer), :24-31 (statistics pooling), :196-204 (DenseLayer).  Eval mode, configs/cam++.yml defaults
// (growth 32, bn_size 4, init_channels 128, blocks 12/24/16 with dilations 1/2/2, 100-frame average segment pooling).
//
// Layouts:
//   * FCM head: zero-bordered NHWC images (H = frequency, W = time), planned as in image_plan.h; its convs stride the frequency
//     axis only, so a strided conv is computed on the input grid and stored on the (H/2, W) output grid;
//   * the head output [B, 32, F/8, T] is flattened to a time-major matrix that holds frame PAIRS: row (b, t') has the
//     320 channels of frame 2t' followed by those of frame 2t'+1.  The stride-2, kernel-5 TDNN conv is then five
//     K-sources (even|odd column windows at row offsets -1,-1,0,0,+1) and no output is computed and thrown away;
//   * D-TDNN part: padded time layout row = b*Tp + P + t with ZERO padding rows (Paddle's Conv1D pads with zeros).  One
//     buffer per dense block holds the growing concatenation; each layer's CAM output is stored into its 32-column window.
//
// Per dense layer (campplus.py:135-141):
//   relu(bn1(x))            one elementwise pass (the BN differs per layer, ReLU keeps it out of the weights)
//   linear1 + bn2 + relu    GEMM, BN folded into the weights, ReLU epilogue
//   context mask            one small kernel per utterance: segment sums -> mean + segment mean -> 128-64-32 MLP -> sigmoid
//   linear_local * mask     3-tap gather-GEMM whose epilogue multiplies by the mask of (utterance, segment)
#include <math.h>

#include "common.h"
#include "image_plan.h"
#include "model_common.h"
#include "ptx.cuh"

namespace ppv {

namespace {

constexpr int CP_P = 4;          // zero padding rows on each side of an utterance (>= max dilation)
constexpr int CP_SEG = 100;      // seg_pooling seg_len, campplus.py:95
constexpr int CP_MAX_SEG = 64;   // segments per utterance held in shared memory by the context kernel
constexpr int CP_MAX_LAYERS = 64;
constexpr int CP_NB = 3;
const int CP_LAYERS[CP_NB] = {12, 24, 16};
const int CP_DIL[CP_NB] = {1, 2, 2};

struct ResBlockW {
    GemmWeights conv1, conv2, sc;
    bool has_sc = false;
    int stride = 1, stage = 0;  // stage = index of the output geometry
};
struct DenseLayerW {
    float *bn1_scale = nullptr, *bn1_shift = nullptr;  // [Kp]
    GemmWeights linear1, local;
    float *w1t = nullptr, *b1 = nullptr, *w2t = nullptr, *b2 = nullptr;  // context MLP, transposed: [128][64], [64][32]
    int in_ch = 0, Kp = 0, block = 0, dil = 1;
};
struct TransitW {
    float *bn_scale = nullptr, *bn_shift = nullptr;
    GemmWeights linear;
    int C = 0;
};

// ------------------------------------------------------------------------------------------------ kernels
// out[r, c] = relu(x[r, c] * scale[c] + shift[c]) for c < C (C % 8 == 0), every row
__global__ void __launch_bounds__(256)
    cp_bn_relu_kernel(Planes x, const float* __restrict__ scale, const float* __restrict__ shift, Planes out, int C, int64_t rows) {
    griddep_launch_dependents();
    griddep_wait();
    const int groups = C >> 3;
    const int64_t total = rows * groups;
    for (int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x; i < total; i += int64_t(gridDim.x) * blockDim.x) {
        const int64_t r = i / groups;
        const int c = int(i - r * groups) * 8;
        const uint4 h = *reinterpret_cast<const uint4*>(x.hi() + r * x.ld + c);
        const uint4 l = *reinterpret_cast<const uint4*>(x.lo() + r * x.ld + c);
        const uint32_t hw[4] = {h.x, h.y, h.z, h.w}, lw[4] = {l.x, l.y, l.z, l.w};
        const float4 s0 = __ldg(reinterpret_cast<const float4*>(scale + c)), s1 = __ldg(reinterpret_cast<const float4*>(scale + c + 4));
        const float4 b0 = __ldg(reinterpret_cast<const float4*>(shift + c)), b1 = __ldg(reinterpret_cast<const float4*>(shift + c + 4));
        const float sv[8] = {s0.x, s0.y, s0.z, s0.w, s1.x, s1.y, s1.z, s1.w};
        const float bv[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
        uint32_t oh[4], ol[4];
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            const float2 hf = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&hw[k]));
            const float2 lf = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&lw[k]));
            const float y0 = fmaxf(fmaf(hf.x + lf.x, sv[2 * k], bv[2 * k]), 0.f);
            const float y1 = fmaxf(fmaf(hf.y + lf.y, sv[2 * k + 1], bv[2 * k + 1]), 0.f);
            __nv_bfloat16 h0, l0, h1, l1;
            split_bf16(y0, h0, l0);
            split_bf16(y1, h1, l1);
            oh[k] = pack_bf16x2(h0, h1);
            ol[k] = pack_bf16x2(l0, l1);
        }
        *reinterpret_cast<uint4*>(out.hi() + r * out.ld + c) = make_uint4(oh[0], oh[1], oh[2], oh[3]);
        *reinterpret_cast<uint4*>(out.lo() + r * out.ld + c) = make_uint4(ol[0], ol[1], ol[2], ol[3]);
    }
}

// Context mask of one utterance (campplus.py:88-93, :95-106): h [T, 128] ->
//   ctx[s] = mean_t h + mean_{t in segment s} h;  mask[s] = sigmoid(W2 relu(W1 ctx[s] + b1) + b2)   -> out [B * nseg, 32]
// Block = utterance, 256 threads: 16 channel groups of 8 x 16 frame lanes for the sums, then the tiny MLP in fp32.
__global__ void __launch_bounds__(256)
    cp_context_kernel(Planes h, int T, int P, int Tp, int nseg, const float* __restrict__ w1t, const float* __restrict__ b1,
                      const float* __restrict__ w2t, const float* __restrict__ b2, float* __restrict__ out) {
    __shared__ float s_part[16][128];
    __shared__ float s_seg[CP_MAX_SEG][128];  // segment sums, then ctx
    __shared__ float s_mean[128];
    __shared__ float s_hid[4][64];
    griddep_launch_dependents();
    griddep_wait();
    const int b = blockIdx.x;
    const int cg = threadIdx.x & 15, fl = threadIdx.x >> 4;
    const int64_t row0 = int64_t(b) * Tp + P;
    for (int s = 0; s < nseg; ++s) {
        const int t0 = s * CP_SEG, t1 = min(T, t0 + CP_SEG);
        float acc[8];
#pragma unroll
        for (int i = 0; i < 8; ++i) acc[i] = 0.f;
        for (int t = t0 + fl; t < t1; t += 16) {
            const uint4 hv = *reinterpret_cast<const uint4*>(h.hi() + (row0 + t) * h.ld + cg * 8);
            const uint4 lv = *reinterpret_cast<const uint4*>(h.lo() + (row0 + t) * h.ld + cg * 8);
            const uint32_t hw[4] = {hv.x, hv.y, hv.z, hv.w}, lw[4] = {lv.x, lv.y, lv.z, lv.w};
#pragma unroll
            for (int k = 0; k < 4; ++k) {
                const float2 hf = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&hw[k]));
                const float2 lf = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&lw[k]));
                acc[2 * k] += hf.x + lf.x;
                acc[2 * k + 1] += hf.y + lf.y;
            }
        }
#pragma unroll
        for (int i = 0; i < 8; ++i) s_part[fl][cg * 8 + i] = acc[i];
        __syncthreads();
        if (threadIdx.x < 128) {
            float v = 0.f;
#pragma unroll
            for (int k = 0; k < 16; ++k) v += s_part[k][threadIdx.x];
            s_seg[s][threadIdx.x] = v;
        }
        __syncthreads();
    }
    if (threadIdx.x < 128) {
        float tot = 0.f;
        for (int s = 0; s < nseg; ++s) tot += s_seg[s][threadIdx.x];
        s_mean[threadIdx.x] = tot / float(T);
    }
    __syncthreads();
    for (int i = threadIdx.x; i < nseg * 128; i += 256) {
        const int s = i >> 7, c = i & 127;
        const int cnt = min(T, (s + 1) * CP_SEG) - s * CP_SEG;
        s_seg[s][c] = s_mean[c] + s_seg[s][c] / float(cnt);
    }
    __syncthreads();
    // MLP: 4 segments at a time; thread (sl, j) computes hidden unit j of segment s0 + sl
    const int sl = threadIdx.x >> 6, j = threadIdx.x & 63;
    for (int s0 = 0; s0 < nseg; s0 += 4) {
        const int s = s0 + sl;
        if (s < nseg) {
            float a = __ldg(b1 + j);
#pragma unroll 8
            for (int c = 0; c < 128; ++c) a = fmaf(__ldg(w1t + c * 64 + j), s_seg[s][c], a);
            s_hid[sl][j] = fmaxf(a, 0.f);
        }
        __syncthreads();
        if (s < nseg && j < 32) {
            float a = __ldg(b2 + j);
#pragma unroll 8
            for (int k = 0; k < 64; ++k) a = fmaf(__ldg(w2t + k * 32 + j), s_hid[sl][k], a);
            out[(int64_t(b) * nseg + s) * 32 + j] = 1.f / (1.f + expf(-a));
        }
        __syncthreads();
    }
}

// [B, Hp, Wp, C] image -> frame-pair matrix: row b*Tp + P + (w >> 1), column (w & 1) * C*H + c*H + h
__global__ void __launch_bounds__(256) cp_flatten_pairs_kernel(Planes in, int B, int H, int W, int Hp, int Wp, int C, Planes out, int Tp, int P) {
    griddep_launch_dependents();
    griddep_wait();
    const int CH = C * H;
    const int64_t total = int64_t(B) * W * CH;
    for (int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x; i < total; i += int64_t(gridDim.x) * blockDim.x) {
        const int col = int(i % CH);
        const int64_t bt = i / CH;
        const int c = col / H, hh = col % H;
        const int b = int(bt / W), w = int(bt % W);
        const int64_t src = ((int64_t(b) * Hp + hh + 1) * Wp + w + 1) * in.ld + c;
        const int64_t dst = (int64_t(b) * Tp + P + (w >> 1)) * out.ld + (w & 1) * CH + col;
        out.hi()[dst] = in.hi()[src];
        out.lo()[dst] = in.lo()[src];
    }
}

int cp_segments(int T2, int* nseg) {
    *nseg = (T2 + CP_SEG - 1) / CP_SEG;
    PPV_REQUIRE(*nseg <= CP_MAX_SEG, "campplus: utterance too long (more than 64 context segments of 100 frames)");
    return PPV_OK;
}

}  // namespace

void campplus_context_weights(const float* w1, const float* w2, std::vector<float>* w1t, std::vector<float>* w2t) {
    constexpr int BC = 128, H = 64, G = 32;
    w1t->assign(size_t(BC) * H, 0.f);
    w2t->assign(size_t(H) * G, 0.f);
    for (int j = 0; j < H; ++j)
        for (int c = 0; c < BC; ++c) (*w1t)[size_t(c) * H + j] = w1[size_t(j) * BC + c];
    for (int n = 0; n < G; ++n)
        for (int k = 0; k < H; ++k) (*w2t)[size_t(k) * G + n] = w2[size_t(n) * H + k];
}

int campplus_context_launch(const Planes& h, int B, int T, int P, int Tp, const float* w1t, const float* b1, const float* w2t,
                            const float* b2, float* out, cudaStream_t st) {
    int nseg = 0;
    int rc = cp_segments(T, &nseg);
    if (rc) return rc;
    PPV_PDL_OK(launch_pdl(cp_context_kernel, dim3(B), dim3(256), 0, st, h, T, P, Tp, nseg, w1t, b1, w2t, b2, out), "cp_context_kernel");
    return PPV_OK;
}

struct CamppModel : PlanModel {
    ppv_campplus_cfg cfg;
    float *stem_w = nullptr, *stem_b = nullptr;
    std::vector<ResBlockW> res;
    GemmWeights head_conv2, tdnn, dense;
    std::vector<DenseLayerW> layers;
    TransitW transit[CP_NB];
    int block_in[CP_NB], block_out[CP_NB];  // channels entering / leaving each dense block
    int head_ch = 0, final_ch = 0;
    // plan (what the taps read)
    int T2 = 0, Tp = 0;
    ImageGeo geo[4];
    Planes stats, final_x;
    Planes stage_out[4];
    Planes xblk[CP_NB], tr_out[CP_NB];

    explicit CamppModel(const ppv_campplus_cfg& c) : PlanModel("campplus", c.precision), cfg(c) {}
    int embd_dim() const override { return cfg.embd_dim; }
    int input_size() const override { return cfg.input_size; }
    size_t workspace_bytes(int B, int T) const override;

  protected:
    bool prepare_weights(ArenaBuilder& ab) override;
    int build_plan(int B, int T, void* ws, size_t ws_bytes, cudaStream_t st) override;
    int tap(const std::string& n, float* out, size_t out_elems, cudaStream_t st) override;
};

void ppv_campplus_default_cfg_impl(ppv_campplus_cfg* c) {
    c->input_size = 80;
    c->embd_dim = 192;
    c->growth_rate = 32;
    c->bn_size = 4;
    c->init_channels = 128;
    c->precision = PPV_PREC_BF16X3;
}

int campplus_create(const ppv_campplus_cfg* cfg, Model** out) {
    PPV_REQUIRE(cfg && out, "campplus_create: null argument");
    if (cfg->growth_rate != 32 || cfg->bn_size != 4 || cfg->init_channels != 128)
        return fail(PPV_EUNSUPPORTED, "campplus: growth_rate 32, bn_size 4, init_channels 128 (configs/cam++.yml) are implemented");
    if (cfg->input_size % 8 || cfg->input_size < 8 || cfg->embd_dim % 32)
        return fail(PPV_EUNSUPPORTED, "campplus: input_size % 8 and embd_dim % 32 required");
    CamppModel* m = new CamppModel(*cfg);
    m->head_ch = 32 * (cfg->input_size / 8);
    *out = m;
    return PPV_OK;
}

// ------------------------------------------------------------------------------------------------ finalize
bool CamppModel::prepare_weights(ArenaBuilder& ab) {
    CamppModel* const m = this;
    const ppv_campplus_cfg& cf = m->cfg;
    const int G = cf.growth_rate, BC = cf.bn_size * cf.growth_rate;  // 32, 128

    bool ok = ab.fold_stem(&m->stem_w, &m->stem_b, "head.conv1", "head.bn1", 32);  // 1 -> 32 channels, CUDA-core stem
    m->res.clear();
    m->res.reserve(4);  // arena patches point into the elements
    for (int li = 1; li <= 2 && ok; ++li)
        for (int bi = 0; bi < 2 && ok; ++bi) {
            m->res.emplace_back();
            ResBlockW& rw = m->res.back();
            rw.stride = bi == 0 ? 2 : 1;
            rw.stage = li;
            rw.has_sc = bi == 0;
            const std::string p = "head.layer" + std::to_string(li) + "." + std::to_string(bi);
            ok &= ab.fold_conv(&rw.conv1, p + ".conv1", p + ".bn1", 32, 32, 3, 2);
            ok &= ab.fold_conv(&rw.conv2, p + ".conv2", p + ".bn2", 32, 32, 3, 2);
            if (rw.has_sc) ok &= ab.fold_conv(&rw.sc, p + ".shortcut.0", p + ".shortcut.1", 32, 32, 1, 2);
        }
    if (ok) ok = ab.fold_conv(&m->head_conv2, "head.conv2", "head.bn2", 32, 32, 3, 2);
    // TDNN: out[t'] = sum_k w_k x[2t' + k - 2]; K-sources in tap order over the frame-pair matrix
    if (ok) ok = ab.fold_conv(&m->tdnn, "xvector.tdnn.linear", "xvector.tdnn.nonlinear.batchnorm", cf.init_channels, m->head_ch, 5, 1);
    m->layers.clear();
    m->layers.reserve(CP_MAX_LAYERS);
    int channels = cf.init_channels;
    for (int bi = 0; bi < CP_NB && ok; ++bi) {
        m->block_in[bi] = channels;
        for (int li = 0; li < CP_LAYERS[bi] && ok; ++li) {
            m->layers.emplace_back();
            DenseLayerW& lw = m->layers.back();
            lw.block = bi;
            lw.dil = CP_DIL[bi];
            lw.in_ch = channels + li * G;
            lw.Kp = int(align_up(size_t(lw.in_ch), 64));
            const std::string p = "xvector.block" + std::to_string(bi + 1) + ".tdnnd" + std::to_string(li + 1);
            ok &= ab.put_bn(&lw.bn1_scale, &lw.bn1_shift, p + ".nonlinear1.batchnorm", lw.in_ch, lw.Kp);
            ok &= ab.fold_conv(&lw.linear1, p + ".linear1", p + ".nonlinear2.batchnorm", BC, lw.in_ch, 1, 1, 0, {{1, lw.Kp, 0, lw.in_ch, 0}});
            ok &= ab.fold_conv(&lw.local, p + ".cam_layer.linear_local", "", G, BC, 3, 1);
            const HostWeight* w1 = ab.get(p + ".cam_layer.linear1.weight", {BC / 2, BC, 1});
            const HostWeight* b1 = ab.get(p + ".cam_layer.linear1.bias", {BC / 2});
            const HostWeight* w2 = ab.get(p + ".cam_layer.linear2.weight", {G, BC / 2, 1});
            const HostWeight* b2 = ab.get(p + ".cam_layer.linear2.bias", {G});
            if (!w1 || !b1 || !w2 || !b2) {
                ok = false;
                break;
            }
            std::vector<float> w1t, w2t;
            campplus_context_weights(w1->v.data(), w2->v.data(), &w1t, &w2t);
            ab.put_f32(&lw.w1t, w1t);
            ab.put_f32(&lw.b1, b1->v);
            ab.put_f32(&lw.w2t, w2t);
            ab.put_f32(&lw.b2, b2->v);
        }
        channels += CP_LAYERS[bi] * G;
        m->block_out[bi] = channels;
        if (!ok) break;
        TransitW& tw = m->transit[bi];
        tw.C = channels;
        const std::string p = "xvector.transit" + std::to_string(bi + 1);
        ok &= ab.put_bn(&tw.bn_scale, &tw.bn_shift, p + ".nonlinear.batchnorm", channels, channels);
        // the last transit is followed directly by out_nonlinear (BN + ReLU): fold that BN into its weights
        ok &= ab.fold_conv(&tw.linear, p + ".linear", bi == CP_NB - 1 ? "xvector.out_nonlinear.batchnorm" : "", channels / 2, channels, 1, 1);
        channels /= 2;
    }
    m->final_ch = channels;
    if (ok) ok = ab.fold_conv(&m->dense, "xvector.dense.linear", "xvector.dense.nonlinear.batchnorm", cf.embd_dim, 2 * channels, 1, 1);
    return ok;
}

// ------------------------------------------------------------------------------------------------ workspace / plan
namespace {

struct CpBuffers {
    Planes stem_out, flat, tmp, hbuf, stats;
    Planes c1[4], c2[4], sc[4], out[4];
    Planes head_out;
    Planes xblk[CP_NB], final_x;
    float *mask, *emb_out;
};

void cp_carve(const CamppModel* m, WsCarver& cv, int B, int T, ImageGeo* geo, CpBuffers* cb) {
    image_pyramid(geo, 4, m->cfg.input_size, T, false);
    const int T2 = (T - 1) / 2 + 1, Tp = T2 + 2 * CP_P, nseg = (T2 + CP_SEG - 1) / CP_SEG;
    const int64_t R = int64_t(B) * Tp;
    cb->stem_out = cv.planes(geo[0].rows(B), 32);
    for (size_t i = 0; i < m->res.size(); ++i) {
        const int64_t Ro = geo[m->res[i].stage].rows(B);
        cb->c1[i] = cv.planes(Ro, 32);
        cb->c2[i] = cv.planes(Ro, 32);
        if (m->res[i].has_sc) cb->sc[i] = cv.planes(Ro, 32);
        cb->out[i] = cv.planes(Ro, 32);
    }
    cb->head_out = cv.planes(geo[3].rows(B), 32);
    cb->flat = cv.planes(R, 2 * m->head_ch);
    int maxc = 0;
    for (int bi = 0; bi < CP_NB; ++bi) {
        cb->xblk[bi] = cv.planes(R, m->block_out[bi]);
        maxc = std::max(maxc, m->block_out[bi]);
    }
    cb->tmp = cv.planes(R, maxc);
    cb->hbuf = cv.planes(R, m->cfg.bn_size * m->cfg.growth_rate);
    cb->final_x = cv.planes(R, m->final_ch);
    cb->stats = cv.planes(B, 2 * m->final_ch);
    cb->mask = static_cast<float*>(cv.take(size_t(B) * nseg * m->cfg.growth_rate * sizeof(float)));
    cb->emb_out = static_cast<float*>(cv.take(align_up(size_t(B), 128) * m->cfg.embd_dim * 4));
}

}  // namespace

size_t CamppModel::workspace_bytes(int B, int T) const {
    if (!finalized || B <= 0 || T <= 0) return 0;
    WsCarver cv;
    ImageGeo g[4];
    CpBuffers cb;
    cp_carve(this, cv, B, T, g, &cb);
    return align_up(cv.off, 256);
}

int CamppModel::build_plan(int B, int T, void* ws, size_t ws_bytes, cudaStream_t st) {
    CamppModel* const m = this;
    PPV_REQUIRE(T >= 3, "campplus: too few frames (the statistics pooling needs at least two frames after the stride-2 TDNN)");
    const int T2 = (T - 1) / 2 + 1, Tp = T2 + 2 * CP_P;
    int nseg = 0;
    int rc = cp_segments(T2, &nseg);
    if (rc) return rc;
    PPV_REQUIRE(T + 3 < 32768, "campplus: utterance too long for 16-bit tap offsets");
    image_pyramid(m->geo, 4, m->cfg.input_size, T, false);
    PPV_REQUIRE(m->geo[0].rows(B) < (int64_t(1) << 31), "campplus: batch too large for 32-bit row indices");
    rc = claim_workspace(B, T, ws, ws_bytes, st);
    if (rc) return rc;
    WsCarver cv;
    cv.base = static_cast<uint8_t*>(ws);
    CpBuffers cb;
    cp_carve(m, cv, B, T, m->geo, &cb);
    m->steps.clear();
    const int M2 = int(int64_t(B) * Tp);

    auto time_epi = [&](const Planes& out, int col0) {
        Epilogue ep = planes_epilogue(out, col0, Tp, CP_P, T2);
        ep.zero_invalid = 1;
        return ep;
    };
    auto relu = [](Epilogue ep) {
        ep.relu = 1;
        return ep;
    };
    // cb.tmp = relu(x * scale + shift) over C columns of every row
    auto bn_relu = [&](const Planes& x, const float* scale, const float* shift, int C) {
        m->steps.push_back({"cp_bn_relu_kernel", false, [x, scale, shift, out = cb.tmp, C, rows = int64_t(M2)](const StepRun& r) {
                                const int64_t total = rows * (C / 8);
                                const int grid = int(std::min<int64_t>((total + 255) / 256, int64_t(r.num_sms) * 16));
                                PPV_PDL_OK(launch_pdl(cp_bn_relu_kernel, dim3(grid), dim3(256), 0, r.st, x, scale, shift, out, C, rows),
                                           "cp_bn_relu_kernel");
                                return PPV_OK;
                            }});
    };
    // ---- FCM head: its convs stride the frequency axis only
    m->steps.push_back(stem_step(m->stem_w, m->stem_b, 32, cb.stem_out, m->geo[0], B));
    Planes x = cb.stem_out;
    for (size_t i = 0; i < m->res.size(); ++i) {
        const ResBlockW& rw = m->res[i];
        const ImageGeo& gin = m->geo[rw.stride == 2 ? rw.stage - 1 : rw.stage];
        const ImageGeo& go = m->geo[rw.stage];
        rc = plan_conv3x3(rw.conv1, x, 0, 32, gin, B, relu(image_epilogue(cb.c1[i], gin, go, rw.stride, 1)));
        if (rc) return rc;
        rc = plan_conv3x3(rw.conv2, cb.c1[i], 0, 32, go, B, image_epilogue(cb.c2[i], go, go, 1, 1));
        if (rc) return rc;
        Planes resid = x;
        if (rw.has_sc) {
            rc = plan_conv(rw.sc, {GemmSource{x, 0, 32, 0}}, int(gin.rows(B)), image_epilogue(cb.sc[i], gin, go, rw.stride, 1));
            if (rc) return rc;
            resid = cb.sc[i];
        }
        m->steps.push_back(scale_res_step(cb.c2[i], nullptr, resid, 0, cb.out[i], 0, 32, go.Hp * go.Wp, go.rows(B), true));
        x = cb.out[i];
        m->stage_out[rw.stage] = x;
    }
    {
        rc = plan_conv3x3(m->head_conv2, x, 0, 32, m->geo[2], B, relu(image_epilogue(cb.head_out, m->geo[2], m->geo[3], 2, 1)));
        if (rc) return rc;
        // head output on grid 3 -> frame-pair matrix
        m->steps.push_back({"cp_flatten_pairs_kernel", false, [in = cb.head_out, g = m->geo[3], B, C = 32, out = cb.flat, Tp](const StepRun& r) {
                                const int64_t total = int64_t(B) * g.W * C * g.H;
                                const int grid = int(std::min<int64_t>((total + 255) / 256, int64_t(r.num_sms) * 16));
                                PPV_PDL_OK(launch_pdl(cp_flatten_pairs_kernel, dim3(grid), dim3(256), 0, r.st, in, B, g.H, g.W, g.Hp, g.Wp, C, out,
                                                      Tp, CP_P),
                                           "cp_flatten_pairs_kernel");
                                return PPV_OK;
                            }});
    }
    // ---- TDNN (k5, stride 2) over the frame-pair matrix -> first 128 columns of block 1's buffer
    {
        const int HC = m->head_ch;
        std::vector<GemmSource> srcs = {GemmSource{cb.flat, 0, HC, -1}, GemmSource{cb.flat, HC, HC, -1}, GemmSource{cb.flat, 0, HC, 0},
                                        GemmSource{cb.flat, HC, HC, 0}, GemmSource{cb.flat, 0, HC, 1}};
        rc = plan_conv(m->tdnn, srcs, M2, relu(time_epi(cb.xblk[0], 0)));
        if (rc) return rc;
    }
    // ---- dense blocks
    size_t li = 0;
    for (int bi = 0; bi < CP_NB; ++bi) {
        const Planes& xb = cb.xblk[bi];
        for (int l = 0; l < CP_LAYERS[bi]; ++l, ++li) {
            const DenseLayerW& lw = m->layers[li];
            bn_relu(xb, lw.bn1_scale, lw.bn1_shift, lw.Kp);
            rc = plan_conv(lw.linear1, {GemmSource{cb.tmp, 0, lw.Kp, 0}}, M2, relu(time_epi(cb.hbuf, 0)));
            if (rc) return rc;
            m->steps.push_back({"campplus_context_launch", false,
                                [h = cb.hbuf, B, T2, Tp, w1t = lw.w1t, b1 = lw.b1, w2t = lw.w2t, b2 = lw.b2, mask = cb.mask](const StepRun& r) {
                                    return campplus_context_launch(h, B, T2, CP_P, Tp, w1t, b1, w2t, b2, mask, r.st);
                                }});
            Epilogue ep = time_epi(xb, lw.in_ch);
            ep.seg_scale = cb.mask;
            ep.seg_len = CP_SEG;
            ep.nseg = nseg;
            const int BCc = cb.hbuf.ld;
            rc = plan_conv(lw.local, {GemmSource{cb.hbuf, 0, BCc, -lw.dil}, GemmSource{cb.hbuf, 0, BCc, 0}, GemmSource{cb.hbuf, 0, BCc, lw.dil}}, M2, ep);
            if (rc) return rc;
        }
        const TransitW& tw = m->transit[bi];
        bn_relu(xb, tw.bn_scale, tw.bn_shift, tw.C);
        const bool last = bi == CP_NB - 1;
        Epilogue ep = time_epi(last ? cb.final_x : cb.xblk[bi + 1], 0);
        if (last) ep.relu = 1;  // out_nonlinear (BN folded into the transit weights) + ReLU
        rc = plan_conv(tw.linear, {GemmSource{cb.tmp, 0, tw.C, 0}}, M2, ep);
        if (rc) return rc;
        m->tr_out[bi] = last ? cb.final_x : cb.xblk[bi + 1];
    }
    {
        m->steps.push_back(colstats_step(cb.final_x, m->final_ch, B, T2, CP_P, Tp, 2, 0.f, cb.stats));
        Epilogue ep;
        ep.out_mode = OUT_F32;
        ep.out = cb.emb_out;
        ep.out_ld = m->cfg.embd_dim;
        rc = plan_conv(m->dense, {GemmSource{cb.stats, 0, 2 * m->final_ch, 0}}, B, ep);
        if (rc) return rc;
    }
    m->stats = cb.stats;
    m->final_x = cb.final_x;
    for (int bi = 0; bi < CP_NB; ++bi) m->xblk[bi] = cb.xblk[bi];
    m->emb_out = cb.emb_out;
    m->T2 = T2;
    m->Tp = Tp;
    return PPV_OK;
}

// taps: "head.layer1", "head.layer2" -> fp32 [B,H,W,32]; "tdnn" [B,T2,128]; "block1".."block3" [B,T2,C]; "transit1", "transit2"
// [B,T2,C/2]; "out_nonlinear" [B,T2,512] (transit3 + BN + ReLU); "stats" [B, 2*512]
int CamppModel::tap(const std::string& n, float* out, size_t out_elems, cudaStream_t st) {
    CamppModel* const m = this;
    const int B = m->plan_B;
    if (n == "stats") {
        PPV_REQUIRE(out_elems >= size_t(B) * 2 * m->final_ch, "campplus_read_tap: output too small");
        return launch_planes_to_f32(m->stats, 0, 2 * m->final_ch, B, 1, 0, 1, out, st);
    }
    if (const int stage = name_index(n, "head.layer", 1, 2)) return image_tap(m->stage_out[stage], m->geo[stage], 32, out, out_elems, st);
    Planes src;
    int C = 0;
    if (n == "tdnn") {
        src = m->xblk[0];
        C = m->cfg.init_channels;
    } else if (const int b = name_index(n, "block", 1, 3)) {
        src = m->xblk[b - 1];
        C = m->block_out[b - 1];
    } else if (const int t = name_index(n, "transit", 1, 2)) {
        src = m->tr_out[t - 1];
        C = m->block_out[t - 1] / 2;
    } else if (n == "out_nonlinear") {
        src = m->final_x;
        C = m->final_ch;
    } else {
        return fail(PPV_EINVAL, "campplus_read_tap: unknown tap " + n);
    }
    PPV_REQUIRE(out_elems >= size_t(B) * m->T2 * C, "campplus_read_tap: output too small");
    return launch_planes_to_f32(src, 0, C, B, m->T2, CP_P, m->Tp, out, st);
}

}  // namespace ppv
