// Res2Net forward as a plan over zero-bordered NHWC images (image_plan.h).
// Reference graph: ppvector/models/res2net.py:151-167 (Res2Net.forward), :11-87 (Bottle2neck), :132-147 (_make_layer: 1x1 strided
// conv + BN downsample), the ASP head of ResNetSE.  Eval mode, scale 2 (the reference's configs/res2net.yml: m_channels 32, layers [3,4,6,3],
// base_width 32, so nums = 1 and the chunk widths are 16 / 32 / 64 / 128).
//
// What is new here, on the CUDA cores:
//   * the stem: Conv2D(1 -> 32, 7x7, stride 3, padding 1) + BN + ReLU with the following MaxPool2D(3, stride 2, padding 1) fused in,
//     straight from the [B, T, F] fp32 features into the pooled grid's split-bf16 planes (res2net_stem_kernel);
//   * the stage block's AvgPool2D(3, stride, padding 1, exclusive) over the second half of conv1's output, written into its column
//     slot of conv3's operand (res2net_avgpool_kernel).
// Everything else is the image plan's: 1x1 convs on the gather-GEMM or the pointwise kernel, the 3x3 branch conv on the patch kernel or
// nine gather-GEMM taps with the strided-lattice epilogue, the residual add + ReLU pass, and ResNetSE's ASP head.
//
// Column plan of a block (width w, scale 2; wpad = max(w, 32)):
//   c1  [rows of the input grid][2w]  conv1 + BN + ReLU: chunk 0 in [0, w), chunk 1 in [w, 2w)
//   cat [rows of the output grid][max(2w, 32)]  conv3's operand: the branch conv in [0, wpad), the stage block's pooled chunk 1 in [w, 2w)
// For w = 16 the branch conv reads the 32-column window of c1 with chunk 1's weights zero and writes 32 columns of which the upper 16
// are zero; the stage block's pool runs after it and overwrites those 16.  A normal block's conv3 reads chunk 1 where it sits in c1
// (spx[1] unchanged): two K-sources, no concat copy.
#include "common.h"
#include "image_plan.h"
#include "model_common.h"
#include "ptx.cuh"

namespace ppv {

// ------------------------------------------------------------------------------------------------ kernels
namespace {

constexpr int STEM_C = 32;                        // stem output channels (m_channels)
constexpr int STEM_K = 7, STEM_S = 3;              // the stem conv's kernel and stride (padding 1)
constexpr int SP_H = 3, SP_W = 8;                  // pooled outputs per CTA
constexpr int SC_H = 2 * SP_H + 1, SC_W = 2 * SP_W + 1;                          // conv outputs the pooled tile's windows cover
constexpr int SI_H = STEM_S * (SC_H - 1) + STEM_K, SI_W = STEM_S * (SC_W - 1) + STEM_K;  // input patch those conv outputs read
constexpr int STEM_THREADS = 128;
static_assert(SC_H * SC_W <= STEM_THREADS && SP_H * SP_W * (STEM_C / 8) <= STEM_THREADS, "stem tile does not fit the CTA");

}  // namespace

// One CTA per (utterance, 3 x 8 tile of pooled positions).  Phase 1: each of the first 119 threads computes all 32 channels of one conv
// output of the 7 x 17 tile the pooled windows cover (49 taps from the input patch in shared memory, weights broadcast from shared
// memory as float4), BN folded, ReLU, into shared memory.  Phase 2: 96 threads take (pooled position, 8-channel group) and store the
// window maximum as split-bf16 planes.  Conv outputs shared by neighbouring tiles are computed by both (7 x 17 for 3 x 8 outputs).
//
// Why this is exact:
//   * padding: conv output row i reads input rows 3i-1 .. 3i+5.  The last row, i = (F-5)/3, reads at most row F: rows -1 and F are
//     the only out-of-range rows any output reads, and they are zeros here as the padding makes them.  The same holds for time.
//   * the fused max-pool: Paddle pads MaxPool2D with -inf.  The pooled values are taken after the ReLU, so every in-bounds element is
//     >= 0, and every window holds at least one in-bounds element (the centre, conv row 2p <= H1-1 for every pooled row p).  A window's
//     maximum over its in-bounds elements therefore equals its maximum with the out-of-bounds positions read as 0: the conv tile
//     stores 0 there, and the max starts from 0.
__global__ void __launch_bounds__(STEM_THREADS)
    res2net_stem_kernel(const float* __restrict__ feat, int T, int F, const float* __restrict__ w, const float* __restrict__ bias, Planes out,
                        int H1, int W1, int Hq, int Wq) {
    __shared__ __align__(16) float s_w[STEM_K * STEM_K][STEM_C];  // [tap][channel]
    __shared__ float s_b[STEM_C];
    __shared__ float s_in[SI_W * SI_H];                // [time][freq]
    __shared__ float s_conv[SC_H * SC_W][STEM_C + 1];  // post-ReLU conv tile, 0 outside the conv grid
    griddep_launch_dependents();
    for (int i = threadIdx.x; i < STEM_K * STEM_K * STEM_C; i += STEM_THREADS) {
        const int c = i / (STEM_K * STEM_K), t = i % (STEM_K * STEM_K);
        s_w[t][c] = __ldg(w + i);
    }
    if (threadIdx.x < STEM_C) s_b[threadIdx.x] = __ldg(bias + threadIdx.x);
    const int b = blockIdx.z, ph0 = blockIdx.y * SP_H, pw0 = blockIdx.x * SP_W;
    const int f0 = STEM_S * (2 * ph0 - 1) - 1, t0 = STEM_S * (2 * pw0 - 1) - 1;  // input position of the patch's first element
    griddep_wait();
    // the image is the features transposed (res2net.py:152-153): in[h = f][w = t] = feat[b][t][f]; loads run along f
    for (int i = threadIdx.x; i < SI_W * SI_H; i += STEM_THREADS) {
        const int r = i % SI_H, c = i / SI_H;
        const int f = f0 + r, t = t0 + c;
        s_in[i] = (f >= 0 && f < F && t >= 0 && t < T) ? __ldg(feat + (int64_t(b) * T + t) * F + f) : 0.f;
    }
    __syncthreads();
    if (threadIdx.x < SC_H * SC_W) {
        const int cr = threadIdx.x / SC_W, cc = threadIdx.x % SC_W;
        const int ch = 2 * ph0 - 1 + cr, cw = 2 * pw0 - 1 + cc;  // conv output position
        float acc[STEM_C];
#pragma unroll
        for (int c = 0; c < STEM_C; ++c) acc[c] = s_b[c];
#pragma unroll
        for (int kh = 0; kh < STEM_K; ++kh) {
#pragma unroll
            for (int kw = 0; kw < STEM_K; ++kw) {
                const float x = s_in[(STEM_S * cc + kw) * SI_H + STEM_S * cr + kh];
                const float4* wr = reinterpret_cast<const float4*>(s_w[kh * STEM_K + kw]);
#pragma unroll
                for (int q = 0; q < STEM_C / 4; ++q) {
                    const float4 wq = wr[q];
                    acc[4 * q + 0] = fmaf(wq.x, x, acc[4 * q + 0]);
                    acc[4 * q + 1] = fmaf(wq.y, x, acc[4 * q + 1]);
                    acc[4 * q + 2] = fmaf(wq.z, x, acc[4 * q + 2]);
                    acc[4 * q + 3] = fmaf(wq.w, x, acc[4 * q + 3]);
                }
            }
        }
        const bool inside = ch >= 0 && ch < H1 && cw >= 0 && cw < W1;
#pragma unroll
        for (int c = 0; c < STEM_C; ++c) s_conv[threadIdx.x][c] = inside ? fmaxf(acc[c], 0.f) : 0.f;
    }
    __syncthreads();
    if (threadIdx.x < SP_H * SP_W * (STEM_C / 8)) {
        const int g = threadIdx.x % (STEM_C / 8), p = threadIdx.x / (STEM_C / 8);
        const int pr = p / SP_W, pc = p % SP_W;
        const int ph = ph0 + pr, pw = pw0 + pc;
        if (ph < Hq && pw < Wq) {
            float m[8];
#pragma unroll
            for (int j = 0; j < 8; ++j) m[j] = 0.f;
#pragma unroll
            for (int dr = 0; dr < 3; ++dr)
#pragma unroll
                for (int dc = 0; dc < 3; ++dc) {
                    const float* v = s_conv[(2 * pr + dr) * SC_W + 2 * pc + dc] + g * 8;
#pragma unroll
                    for (int j = 0; j < 8; ++j) m[j] = fmaxf(m[j], v[j]);
                }
            uint32_t hw[4], lw[4];
#pragma unroll
            for (int j = 0; j < 4; ++j) split_pack_bf16x2(m[2 * j], m[2 * j + 1], hw[j], lw[j]);
            const int64_t row = (int64_t(b) * (Hq + 2) + ph + 1) * (Wq + 2) + pw + 1;
            *reinterpret_cast<uint4*>(out.hi() + row * out.ld + g * 8) = make_uint4(hw[0], hw[1], hw[2], hw[3]);
            *reinterpret_cast<uint4*>(out.lo() + row * out.ld + g * 8) = make_uint4(lw[0], lw[1], lw[2], lw[3]);
        }
    }
}

// AvgPool2D(3, stride, padding 1) with Paddle's default exclusive = True: each window's sum over its in-bounds elements divided by
// their number (4 at a corner, 6 on an edge, 9 inside).  Columns [in_col0, +ncols) of `in` on the H x W grid -> columns
// [out_col0, +ncols) of `out` on the Ho x Wo grid.  One thread per (output position, 8 channels): 16-byte loads of both planes.
__global__ void __launch_bounds__(256)
    res2net_avgpool_kernel(Planes in, int in_col0, int B, int H, int W, int stride, int ncols, Planes out, int out_col0, int Ho, int Wo) {
    griddep_launch_dependents();
    griddep_wait();
    const int groups = ncols / 8;
    const int64_t total = int64_t(B) * Ho * Wo * groups;
    for (int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x; i < total; i += int64_t(gridDim.x) * blockDim.x) {
        const int g = int(i % groups);
        const int64_t pos = i / groups;
        const int ow = int(pos % Wo), oh = int((pos / Wo) % Ho), b = int(pos / (int64_t(Wo) * Ho));
        float s[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) s[j] = 0.f;
        int cnt = 0;
#pragma unroll
        for (int dh = -1; dh <= 1; ++dh) {
            const int ih = oh * stride + dh;
            if (ih < 0 || ih >= H) continue;
#pragma unroll
            for (int dw = -1; dw <= 1; ++dw) {
                const int iw = ow * stride + dw;
                if (iw < 0 || iw >= W) continue;
                ++cnt;
                const int64_t off = ((int64_t(b) * (H + 2) + ih + 1) * (W + 2) + iw + 1) * in.ld + in_col0 + g * 8;
                const uint4 hv = *reinterpret_cast<const uint4*>(in.hi() + off);
                const uint4 lv = *reinterpret_cast<const uint4*>(in.lo() + off);
                const __nv_bfloat162* h2 = reinterpret_cast<const __nv_bfloat162*>(&hv);
                const __nv_bfloat162* l2 = reinterpret_cast<const __nv_bfloat162*>(&lv);
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                    const float2 a = __bfloat1622float2(h2[j]), c = __bfloat1622float2(l2[j]);
                    s[2 * j] += a.x + c.x;
                    s[2 * j + 1] += a.y + c.y;
                }
            }
        }
        const float n = float(cnt);
        uint32_t hw[4], lw[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) split_pack_bf16x2(s[2 * j] / n, s[2 * j + 1] / n, hw[j], lw[j]);
        const int64_t orow = (int64_t(b) * (Ho + 2) + oh + 1) * (Wo + 2) + ow + 1;
        *reinterpret_cast<uint4*>(out.hi() + orow * out.ld + out_col0 + g * 8) = make_uint4(hw[0], hw[1], hw[2], hw[3]);
        *reinterpret_cast<uint4*>(out.lo() + orow * out.ld + out_col0 + g * 8) = make_uint4(lw[0], lw[1], lw[2], lw[3]);
    }
}

void res2net_stem_grids(int F, int T, int* H1, int* W1, int* Hq, int* Wq) {
    *H1 = (F + 2 - STEM_K) / STEM_S + 1;
    *W1 = (T + 2 - STEM_K) / STEM_S + 1;
    *Hq = (*H1 - 1) / 2 + 1;
    *Wq = (*W1 - 1) / 2 + 1;
}

int launch_res2net_stem(const float* feat, int B, int T, int F, const float* w, const float* bias, int C0, const Planes& out, cudaStream_t st) {
    PPV_REQUIRE(C0 == STEM_C && out.ld % 8 == 0, "res2net stem: 32 output channels and 16-byte aligned rows required");
    PPV_REQUIRE(B > 0 && B <= 65535 && F >= STEM_K - 2 && T >= STEM_K - 2, "res2net stem: batch of 1..65535 utterances, F and T >= 5");
    int H1, W1, Hq, Wq;
    res2net_stem_grids(F, T, &H1, &W1, &Hq, &Wq);
    const dim3 grid((Wq + SP_W - 1) / SP_W, (Hq + SP_H - 1) / SP_H, B);
    PPV_PDL_OK(launch_pdl(res2net_stem_kernel, grid, dim3(STEM_THREADS), 0, st, feat, T, F, w, bias, out, H1, W1, Hq, Wq), "res2net_stem_kernel");
    return PPV_OK;
}

int launch_avgpool3x3(const Planes& in, int in_col0, int B, int H, int W, int stride, int ncols, const Planes& out, int out_col0, int num_sms,
                      cudaStream_t st) {
    PPV_REQUIRE(stride == 1 || stride == 2, "avgpool3x3: stride 1 or 2");
    PPV_REQUIRE(ncols > 0 && ncols % 8 == 0 && in_col0 % 8 == 0 && out_col0 % 8 == 0 && in.ld % 8 == 0 && out.ld % 8 == 0,
                "avgpool3x3: columns must come in 16-byte groups");
    const int Ho = (H - 1) / stride + 1, Wo = (W - 1) / stride + 1;
    const int64_t total = int64_t(B) * Ho * Wo * (ncols / 8);
    const int grid = int(std::min<int64_t>((total + 255) / 256, int64_t(num_sms) * 16));
    PPV_PDL_OK(launch_pdl(res2net_avgpool_kernel, dim3(grid), dim3(256), 0, st, in, in_col0, B, H, W, stride, ncols, out, out_col0, Ho, Wo),
               "res2net_avgpool_kernel");
    return PPV_OK;
}

// ------------------------------------------------------------------------------------------------ model
namespace {

constexpr int R2_MAX_BLOCKS = 32;

struct R2BlockW {
    GemmWeights conv1, conv, conv3, down;
    bool has_down = false, stage_block = false;
    int inplanes = 0, planes = 0, width = 0, wpad = 0, stride = 1, stage = 0;
};

}  // namespace

struct Res2NetModel : PlanModel {
    ppv_res2net_cfg cfg;
    float *stem_w = nullptr, *stem_b = nullptr;  // [32][49], [32], BN folded
    std::vector<R2BlockW> blocks;
    AspHead head;
    int cat = 0;
    // plan (what the taps read)
    ImageGeo geo[5];  // geo[1] = the pooled stem grid = layer1's grid
    Planes stem_out, flat, stage_out[5];
    float *pooled_raw = nullptr, *feat_buf = nullptr;

    explicit Res2NetModel(const ppv_res2net_cfg& c) : PlanModel("res2net", c.precision), cfg(c) {}
    int embd_dim() const override { return cfg.embd_dim; }
    int input_size() const override { return cfg.input_size; }
    bool takes_wav() const override { return true; }
    size_t workspace_bytes(int B, int T) const override;

  protected:
    bool prepare_weights(ArenaBuilder& ab) override;
    int build_plan(int B, int T, void* ws, size_t ws_bytes, cudaStream_t st) override;
    // The fused front end: the Fbank of the waveforms into the workspace's feature buffer, where the stem reads them.
    int stage_inputs(const ModelInput& in, PlanInputs* pin, cudaStream_t st) override {
        if (!in.wav) return PPV_OK;
        pin->feat = feat_buf;
        return stage_fbank(in, feat_buf, feat_buf, Planes{}, 0, 0, st);
    }
    int tap(const std::string& n, float* out, size_t out_elems, cudaStream_t st) override;
};

void ppv_res2net_default_cfg_impl(ppv_res2net_cfg* c) {
    c->input_size = 80;
    c->embd_dim = 192;
    const int l[4] = {3, 4, 6, 3};
    for (int i = 0; i < 4; ++i) c->layers[i] = l[i];
    c->m_channels = 32;
    c->base_width = 32;
    c->scale = 2;
    c->attention_channels = 128;
    c->precision = PPV_PREC_BF16X3;
}

// The final grid height of the stem + pool + three stride-2 stages: the reference sizes its head for input_size // base_width
// (res2net.py:115) and breaks where the two differ.
static int res2net_final_height(int F) {
    int H1, W1, Hq, Wq;
    res2net_stem_grids(F, 5, &H1, &W1, &Hq, &Wq);
    ImageGeo g[4];
    image_pyramid(g, 4, Hq, 1, false);
    return g[3].H;
}

int res2net_create(const ppv_res2net_cfg* cfg, Model** out) {
    PPV_REQUIRE(cfg && out, "res2net_create: null argument");
    if (cfg->scale != 2) return fail(PPV_EUNSUPPORTED, "res2net: scale 2 only (the sp = sp + spx[i] chain of scale > 2 is not implemented)");
    if (cfg->m_channels != STEM_C) return fail(PPV_EUNSUPPORTED, "res2net: m_channels must be 32");
    int nblocks = 0;
    for (int i = 0; i < 4; ++i) {
        if (cfg->layers[i] < 1) return fail(PPV_EUNSUPPORTED, "res2net: layers >= 1 required");
        nblocks += cfg->layers[i];
        const int width = (cfg->m_channels << i) * cfg->base_width / 64;
        if (width != 16 && (width < 32 || width % 32))
            return fail(PPV_EUNSUPPORTED, "res2net: every chunk width (planes * base_width / 64) must be 16 or a multiple of 32");
    }
    if (nblocks > R2_MAX_BLOCKS) return fail(PPV_EUNSUPPORTED, "res2net: too many blocks");
    if (cfg->input_size < STEM_K - 2 || cfg->base_width < 1 || res2net_final_height(cfg->input_size) != cfg->input_size / cfg->base_width)
        return fail(PPV_EUNSUPPORTED, "res2net: input_size must leave a final grid of input_size / base_width rows (the reference's head size)");
    const int cat = cfg->m_channels * 8 * 4 * (cfg->input_size / cfg->base_width);
    if (cfg->attention_channels != 128 || cfg->embd_dim % 32 || cat % 128)
        return fail(PPV_EUNSUPPORTED, "res2net: attention_channels == 128, embd_dim % 32 and pooled channels % 128 required");
    Res2NetModel* m = new Res2NetModel(*cfg);
    m->cat = cat;
    *out = m;
    return PPV_OK;
}

bool Res2NetModel::prepare_weights(ArenaBuilder& ab) {
    const ppv_res2net_cfg& cf = cfg;
    bool ok = ab.fold_stem(&stem_w, &stem_b, "conv1", "bn1", cf.m_channels, STEM_K);
    blocks.clear();
    blocks.reserve(R2_MAX_BLOCKS);  // the arena patches point into the elements: no reallocation allowed
    int inplanes = cf.m_channels;
    for (int li = 1; li <= 4 && ok; ++li) {
        const int planes = cf.m_channels << (li - 1), width = planes * cf.base_width / 64, wpad = std::max(width, 32), C = 4 * planes;
        for (int bi = 0; bi < cf.layers[li - 1] && ok; ++bi) {
            blocks.emplace_back();
            R2BlockW& bw = blocks.back();
            bw.inplanes = inplanes;
            bw.planes = planes;
            bw.width = width;
            bw.wpad = wpad;
            bw.stage = li;
            bw.stage_block = bi == 0;
            bw.stride = (li > 1 && bi == 0) ? 2 : 1;
            const std::string p = "layer" + std::to_string(li) + "." + std::to_string(bi);
            ok &= ab.fold_conv(&bw.conv1, p + ".conv1", p + ".bn1", 2 * width, inplanes, 1, 2);
            // branch conv on chunk 0: for w = 16 the GEMM reads c1's 32-column window, chunk 1's weights are zero
            ok &= ab.fold_conv(&bw.conv, p + ".convs.0", p + ".bns.0", width, width, 3, 2, wpad, {{9, wpad, 0, width, 0}});
            if (bw.stage_block) {  // cat holds [branch conv | pooled chunk 1] contiguously
                ok &= ab.fold_conv(&bw.conv3, p + ".conv3", p + ".bn3", C, 2 * width, 1, 2, C, {{1, std::max(2 * width, 32), 0, 2 * width, 0}});
            } else {  // K-sources: cat's branch-conv window, c1's chunk-1 window (for w = 16 the whole 32 columns, chunk 1 at 16)
                const int pos1 = width == 16 ? 16 : 0;
                ok &= ab.fold_conv(&bw.conv3, p + ".conv3", p + ".bn3", C, 2 * width, 1, 2, C, {{1, wpad, 0, width, 0}, {1, wpad, pos1, width, width}});
            }
            bw.has_down = bi == 0 && (bw.stride != 1 || inplanes != C);
            if (bw.has_down) ok &= ab.fold_conv(&bw.down, p + ".downsample.0", p + ".downsample.1", C, inplanes, 1, 2);
            inplanes = C;
        }
    }
    if (ok) ok = prepare_asp_head(ab, &head, cat, cf.attention_channels, cf.embd_dim);
    return ok;
}

// ------------------------------------------------------------------------------------------------ workspace / plan
namespace {

struct R2Buffers {
    float* feat;  // the fused front end's features [B, T, F]
    Planes stem_out;
    std::vector<Planes> c1, cat, o3, out;
    AspHeadBuffers head;
};

void r2_geometry(const ppv_res2net_cfg& cf, int T, ImageGeo* geo) {
    int H1, W1, Hq, Wq;
    res2net_stem_grids(cf.input_size, T, &H1, &W1, &Hq, &Wq);
    image_pyramid(geo + 1, 4, Hq, Wq, true);
}

void r2_carve(const Res2NetModel* m, WsCarver& cv, int B, int T, ImageGeo* geo, R2Buffers* rb) {
    r2_geometry(m->cfg, T, geo);
    rb->feat = static_cast<float*>(cv.take(size_t(B) * T * m->cfg.input_size * sizeof(float)));
    rb->stem_out = cv.planes(geo[1].rows(B), m->cfg.m_channels);
    const size_t nb = m->blocks.size();
    for (auto* v : {&rb->c1, &rb->cat, &rb->o3, &rb->out}) v->resize(nb);
    // Buffer liveness as in ResNetSE / ERes2Net: one set per stage, and a block's output overwrites its residual input in place (the
    // add is elementwise).  The stage block's conv1 runs on the previous stage's grid: it has its own c1 there.  Zero borders survive
    // because the epilogues store interior positions only and a buffer never changes its grid.
    Planes s_c1[5], s_cat[5], s_o3[5], s_act[5];
    for (size_t i = 0; i < nb; ++i) {
        const R2BlockW& bw = m->blocks[i];
        const int st = bw.stage;
        const int64_t R = geo[st].rows(B);
        if (bw.stage_block) {
            s_c1[st] = cv.planes(R, 2 * bw.width);
            s_cat[st] = cv.planes(R, std::max(2 * bw.width, 32));
            s_o3[st] = cv.planes(R, 4 * bw.planes);
            s_act[st] = cv.planes(R, 4 * bw.planes);
            rb->c1[i] = bw.stride == 2 ? cv.planes(geo[st - 1].rows(B), 2 * bw.width) : s_c1[st];
        } else {
            rb->c1[i] = s_c1[st];
        }
        rb->cat[i] = s_cat[st];
        rb->o3[i] = s_o3[st];
        rb->out[i] = s_act[st];
    }
    const int Tf = geo[4].W, cat = m->cat;
    rb->head.flat = cv.planes(int64_t(B) * Tf, cat);
    rb->head.gstat = cv.planes(B, 2 * cat);
    rb->head.pooled = cv.planes(B, 2 * cat);
    rb->head.attp = cv.planes(int64_t(B) * Tf, m->head.att);
    rb->head.fold_out = static_cast<float*>(cv.take(align_up(size_t(B), 128) * m->head.att * 4));
    rb->head.pooled_raw = static_cast<float*>(cv.take(size_t(B) * 2 * cat * 4));
    rb->head.emb_out = static_cast<float*>(cv.take(align_up(size_t(B), 128) * m->cfg.embd_dim * 4));
}

}  // namespace

size_t Res2NetModel::workspace_bytes(int B, int T) const {
    if (!finalized || B <= 0 || T <= 0) return 0;
    return carve_extent([&](WsCarver& cv) {
        ImageGeo g[5];
        R2Buffers rb;
        r2_carve(this, cv, B, T, g, &rb);
    });
}

int Res2NetModel::build_plan(int B, int T, void* ws, size_t ws_bytes, cudaStream_t st) {
    PPV_REQUIRE(T >= STEM_K - 2, "res2net: too few frames (the 7 x 7 stem needs at least 5)");
    PPV_REQUIRE(B <= 65535, "res2net: at most 65535 utterances per forward");
    r2_geometry(cfg, T, geo);
    PPV_REQUIRE(geo[1].rows(B) < (int64_t(1) << 31), "res2net: batch too large for 32-bit row indices");
    int rc = claim_workspace(B, T, ws, ws_bytes, st);
    if (rc) return rc;
    WsCarver cv;
    cv.base = static_cast<uint8_t*>(ws);
    R2Buffers rb;
    r2_carve(this, cv, B, T, geo, &rb);
    steps.clear();

    auto relu = [](Epilogue ep) {
        ep.relu = 1;
        return ep;
    };
    {
        const float *w = stem_w, *bias = stem_b;
        const int F = cfg.input_size, C0 = cfg.m_channels;
        const Planes o = rb.stem_out;
        steps.push_back({"launch_res2net_stem", false, [w, bias, F, C0, o, B, T](const StepRun& r) {
                             return launch_res2net_stem(r.in.feat, B, T, F, w, bias, C0, o, r.st);
                         }});
    }
    Planes x = rb.stem_out;
    for (size_t i = 0; i < blocks.size(); ++i) {
        const R2BlockW& bw = blocks[i];
        const ImageGeo& gin = geo[bw.stride == 2 ? bw.stage - 1 : bw.stage];
        const ImageGeo& go = geo[bw.stage];
        const int Min = int(gin.rows(B)), Mo = int(go.rows(B)), w = bw.width, C = 4 * bw.planes;
        const Planes& c1 = rb.c1[i];
        const Planes& cat = rb.cat[i];
        // conv1 (1x1) + bn1 + ReLU on the input grid
        rc = plan_conv(bw.conv1, {GemmSource{x, 0, bw.inplanes, 0}}, Min, relu(image_epilogue(c1, gin, gin, 1, 1)));
        if (rc) return rc;
        // convs[0] (3x3, stride) + bns[0] + ReLU on chunk 0, stored on the output grid's lattice into cat[:, 0:wpad)
        rc = plan_conv3x3(bw.conv, c1, 0, bw.wpad, gin, B, relu(image_epilogue(cat, gin, go, bw.stride, bw.stride)));
        if (rc) return rc;
        std::vector<GemmSource> k3;
        if (bw.stage_block) {  // pool(spx[1]) into cat[:, w:2w), after the branch conv (which, for w = 16, wrote zeros there)
            const Planes c1v = c1, catv = cat;
            const int H = gin.H, W = gin.W, s = bw.stride;
            steps.push_back({"launch_avgpool3x3", false, [c1v, catv, w, B, H, W, s](const StepRun& r) {
                                 return launch_avgpool3x3(c1v, w, B, H, W, s, w, catv, w, r.num_sms, r.st);
                             }});
            k3.push_back(GemmSource{cat, 0, cat.ld, 0});
        } else {  // concat(sp, spx[1]) as two K-sources
            k3.push_back(GemmSource{cat, 0, bw.wpad, 0});
            k3.push_back(GemmSource{c1, w == 16 ? 0 : w, bw.wpad, 0});
        }
        // conv3 (1x1) + bn3
        rc = plan_conv(bw.conv3, k3, Mo, image_epilogue(rb.o3[i], go, go, 1, 1));
        if (rc) return rc;
        Planes res = x;
        if (bw.has_down) {
            rc = plan_conv(bw.down, {GemmSource{x, 0, bw.inplanes, 0}}, Min, image_epilogue(rb.out[i], gin, go, bw.stride, bw.stride));
            if (rc) return rc;
            res = rb.out[i];
        }
        steps.push_back(scale_res_step(rb.o3[i], nullptr, res, 0, rb.out[i], 0, C, go.Hp * go.Wp, go.rows(B), true));
        x = rb.out[i];
        stage_out[bw.stage] = x;
    }
    // head: x.reshape([B, C*H, W]) -> ASP -> bn2 -> linear -> bn3 (res2net.py:161-167)
    const ImageGeo& g4 = geo[4];
    steps.push_back(flatten_step(x, g4, B, 32 * cfg.m_channels, rb.head.flat));
    rc = plan_asp_head(head, rb.head, B, g4.W);
    if (rc) return rc;
    stem_out = rb.stem_out;
    flat = rb.head.flat;
    pooled_raw = rb.head.pooled_raw;
    emb_out = rb.head.emb_out;
    feat_buf = rb.feat;
    return PPV_OK;
}

// taps: "stem" (after the max-pool), "layer1".."layer4" -> fp32 [B,H,W,C]; "flat" -> [B,T',cat]; "asp" -> [B, 2*cat]
int Res2NetModel::tap(const std::string& n, float* out, size_t out_elems, cudaStream_t st) {
    const int B = plan_B, Tf = geo[4].W;
    if (n == "asp") {
        PPV_REQUIRE(out_elems >= size_t(B) * 2 * cat, "res2net_read_tap: output too small");
        PPV_CUDA_OK(cudaMemcpyAsync(out, pooled_raw, size_t(B) * 2 * cat * 4, cudaMemcpyDeviceToDevice, st));
        return PPV_OK;
    }
    if (n == "flat") {
        PPV_REQUIRE(out_elems >= size_t(B) * Tf * cat, "res2net_read_tap: output too small");
        return launch_planes_to_f32(flat, 0, cat, B, Tf, 0, Tf, out, st);
    }
    if (n == "stem") return image_tap(stem_out, geo[1], cfg.m_channels, out, out_elems, st);
    if (const int stage = name_index(n, "layer", 1, 4)) return image_tap(stage_out[stage], geo[stage], 4 * (cfg.m_channels << (stage - 1)), out, out_elems, st);
    return fail(PPV_EINVAL, "res2net_read_tap: unknown tap " + n);
}

}  // namespace ppv
