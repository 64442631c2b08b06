// Host-side helpers shared by the model plans: named fp32 weights as loaded through the C ABI, an arena image that is
// built on the host (split-bf16 weight planes, fp32 vectors) and uploaded once, and the ECAPA-TDNN geometry.
#pragma once
#include <string.h>

#include <map>
#include <string>
#include <vector>

#include "common.h"

namespace ppv {

struct HostWeight {
    std::vector<float> v;
    std::vector<int64_t> shape;
};
using WeightMap = std::map<std::string, HostWeight>;

// Copies `data` (host or device fp32) into the map.
inline int weight_map_load(WeightMap* wm, const char* name, const float* data, const int64_t* shape, int ndim) {
    PPV_REQUIRE(wm && name && data && shape && ndim >= 1 && ndim <= 4, "load_weight: bad argument");
    HostWeight w;
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
    (*wm)[name] = std::move(w);
    return PPV_OK;
}

struct GemmWeights {  // one conv / linear layer prepared for the gather-GEMM
    Planes W;         // [2][Npad][Ktot] split-bf16
    float* bias = nullptr;
    int N = 0, Ktot = 0;
};

// One K group of a conv's dense weight matrix: `taps` taps of `ncols` source columns each, of which columns [pos, pos + cnt) carry
// the conv's input channels [cin0, cin0 + cnt) and the rest are zero.
struct ConvKGroup {
    int taps, ncols, pos, cnt, cin0;
};

// Conv weights w [N][Cin][taps] (Paddle's Conv1D / Conv2D order, taps in (kh, kw) order) -> dense [Npad][sum taps * ncols] in
// double, K order (group, tap, column), row n scaled by scale[n] (null: 1).  Output channel n lands in row n, or, with `chunk` > 0, in
// row (n / chunk) * chunk_stride + n % chunk (zero-padded output chunks).  Rows and columns that carry no weight are zero.
inline std::vector<double> conv_weight_matrix(const float* w, int N, int Cin, int taps, int Npad, const std::vector<ConvKGroup>& groups,
                                              const double* scale = nullptr, int chunk = 0, int chunk_stride = 0) {
    int K = 0;
    for (const ConvKGroup& g : groups) K += g.taps * g.ncols;
    std::vector<double> mtx(size_t(Npad) * K, 0.0);
    for (int n = 0; n < N; ++n) {
        const int row = chunk > 0 ? (n / chunk) * chunk_stride + n % chunk : n;
        const double s = scale ? scale[n] : 1.0;
        int kpos = 0;
        for (const ConvKGroup& g : groups) {
            for (int t = 0; t < g.taps; ++t)
                for (int c = 0; c < g.cnt; ++c) mtx[size_t(row) * K + kpos + t * g.ncols + g.pos + c] = double(w[(size_t(n) * Cin + g.cin0 + c) * taps + t]) * s;
            kpos += g.taps * g.ncols;
        }
    }
    return mtx;
}

struct ArenaBuilder {
    const WeightMap* wm = nullptr;
    std::vector<uint8_t> host;
    std::string err;
    struct Patch {
        void** dst;
        size_t off;
    };
    std::vector<Patch> patches;

    size_t reserve(size_t bytes) {
        const size_t off = align_up(host.size(), 256);
        host.resize(off + bytes, 0);
        return off;
    }
    const HostWeight* get(const std::string& name, const std::vector<int64_t>& shape) {
        auto it = wm->find(name);
        if (it == wm->end()) {
            if (err.empty()) err = "missing weight " + name;
            return nullptr;
        }
        if (it->second.shape != shape) {
            if (err.empty()) err = "weight " + name + " has the wrong shape";
            return nullptr;
        }
        return &it->second;
    }
    template <typename T>
    void put_f32(T** dst, const std::vector<float>& v) {
        const size_t off = reserve(v.size() * sizeof(float));
        memcpy(host.data() + off, v.data(), v.size() * sizeof(float));
        patches.push_back({reinterpret_cast<void**>(dst), off});
    }
    // dense fp32 [N][K] (row-major) -> split planes [2][Npad][K]; rows N..Npad stay zero
    void put_matrix(GemmWeights* gw, const std::vector<double>& m, int N, int K, int n_align = 256) {
        const int Npad = int(align_up(size_t(N), size_t(n_align)));
        const size_t plane = size_t(Npad) * K;
        const size_t off = reserve(2 * plane * sizeof(__nv_bfloat16));
        __nv_bfloat16* hi = reinterpret_cast<__nv_bfloat16*>(host.data() + off);
        __nv_bfloat16* lo = hi + plane;
        const __nv_bfloat16 z = __float2bfloat16_rn(0.f);
        for (size_t i = 0; i < 2 * plane; ++i) hi[i] = z;
        for (int n = 0; n < N; ++n)
            for (int k = 0; k < K; ++k) {
                const float x = float(m[size_t(n) * K + k]);
                const __nv_bfloat16 h = __float2bfloat16_rn(x);
                hi[size_t(n) * K + k] = h;
                lo[size_t(n) * K + k] = __float2bfloat16_rn(x - __bfloat162float(h));
            }
        gw->N = N;
        gw->Ktot = K;
        gw->W.rows = Npad;
        gw->W.ld = K;
        gw->W.plane_stride = int64_t(plane);
        patches.push_back({reinterpret_cast<void**>(&gw->W.base), off});
    }
    // BatchNorm(eval) as y = x * scale + shift (eps 1e-5), in double
    bool bn_affine(const std::string& prefix, int C, std::vector<double>* scale, std::vector<double>* shift) {
        const HostWeight *g = get(prefix + ".weight", {C}), *b = get(prefix + ".bias", {C}), *mu = get(prefix + "._mean", {C}),
                         *var = get(prefix + "._variance", {C});
        if (!g || !b || !mu || !var) return false;
        scale->resize(C);
        shift->resize(C);
        for (int i = 0; i < C; ++i) {
            const double s = double(g->v[i]) / sqrt(double(var->v[i]) + 1e-5);
            (*scale)[i] = s;
            (*shift)[i] = double(b->v[i]) - double(mu->v[i]) * s;
        }
        return true;
    }
    // Conv `conv` ([N][Cin][k] with dims 1, [N][Cin][k][k] with dims 2) with the BatchNorm `bn` folded in (none if empty) -> dense
    // [Npad][K] split-bf16 matrix (see conv_weight_matrix; no groups: one group of all taps x Cin) and bias [max(Npad, 64)].
    bool fold_conv(GemmWeights* gw, const std::string& conv, const std::string& bn, int N, int Cin, int k, int dims, int Npad = 0,
                   std::vector<ConvKGroup> groups = {}, int chunk = 0, int chunk_stride = 0) {
        const int taps = dims == 2 ? k * k : k;
        if (Npad == 0) Npad = N;
        if (groups.empty()) groups.push_back({taps, Cin, 0, Cin, 0});
        const HostWeight* w = get(conv + ".weight", dims == 2 ? std::vector<int64_t>{N, Cin, k, k} : std::vector<int64_t>{N, Cin, k});
        const HostWeight* b = get(conv + ".bias", {N});
        std::vector<double> sc(N, 1.0), sh(N, 0.0);
        if (!w || !b || (!bn.empty() && !bn_affine(bn, N, &sc, &sh))) return false;
        const std::vector<double> mtx = conv_weight_matrix(w->v.data(), N, Cin, taps, Npad, groups, sc.data(), chunk, chunk_stride);
        std::vector<float> bias(std::max(Npad, 64), 0.f);
        for (int n = 0; n < N; ++n) bias[chunk > 0 ? (n / chunk) * chunk_stride + n % chunk : n] = float(double(b->v[n]) * sc[n] + sh[n]);
        put_matrix(gw, mtx, Npad, int(mtx.size() / Npad));
        put_f32(&gw->bias, bias);
        return true;
    }
    // The 1 -> C0 channel k x k stem conv with its BatchNorm folded in: weights [C0][k k], bias [C0] (launch_stem_conv: k = 3;
    // Res2Net's 7 x 7 stem: launch_res2net_stem)
    bool fold_stem(float** w9, float** bias, const std::string& conv, const std::string& bn, int C0, int k = 3) {
        const HostWeight* w = get(conv + ".weight", {C0, 1, k, k});
        const HostWeight* b = get(conv + ".bias", {C0});
        std::vector<double> sc, sh;
        if (!w || !b || !bn_affine(bn, C0, &sc, &sh)) return false;
        const int kk = k * k;
        std::vector<float> wf(size_t(C0) * kk), bf(C0);
        for (int c = 0; c < C0; ++c) {
            for (int t = 0; t < kk; ++t) wf[c * kk + t] = float(double(w->v[c * kk + t]) * sc[c]);
            bf[c] = float(double(b->v[c]) * sc[c] + sh[c]);
        }
        put_f32(w9, wf);
        put_f32(bias, bf);
        return true;
    }
    // BatchNorm `bn` as fp32 scale / shift vectors of Cp >= C entries, zero beyond C
    bool put_bn(float** scale, float** shift, const std::string& bn, int C, int Cp) {
        std::vector<double> sc, sh;
        if (!bn_affine(bn, C, &sc, &sh)) return false;
        std::vector<float> s(Cp, 0.f), b(Cp, 0.f);
        for (int i = 0; i < C; ++i) {
            s[i] = float(sc[i]);
            b[i] = float(sh[i]);
        }
        put_f32(scale, s);
        put_f32(shift, b);
        return true;
    }
    int upload(void** arena) {
        PPV_CUDA_OK(cudaMalloc(arena, host.size()));
        PPV_CUDA_OK(cudaMemcpy(*arena, host.data(), host.size(), cudaMemcpyHostToDevice));
        for (const Patch& p : patches) *p.dst = static_cast<uint8_t*>(*arena) + p.off;
        return PPV_OK;
    }
};

// The geometry of an ECAPA-TDNN config, shared by the inference plan and the training step, after the checks both need:
// channels [C, C, C, C, 3C], res2net_scale in [2, 8] with chunks of a multiple of 64 channels, kernel sizes [odd, 3, 3, 3, 1].
struct EcapaGeometry {
    int C = 0, C3 = 0, width = 0, scale = 0, Fp = 0, P = 0, att = 0, se = 0;  // P: the reflect padding of the time axis
};
inline int ecapa_geometry(const ppv_ecapa_cfg& cfg, EcapaGeometry* g) {
    const int C = cfg.channels[0];
    if (cfg.channels[1] != C || cfg.channels[2] != C || cfg.channels[3] != C)
        return fail(PPV_EUNSUPPORTED, "ecapa: channels[0..3] must be equal (no shortcut conv path)");
    if (cfg.channels[4] != 3 * C) return fail(PPV_EUNSUPPORTED, "ecapa: channels[4] must equal 3 * channels[0] (MFA concat)");
    if (cfg.res2net_scale < 2 || cfg.res2net_scale > 8 || C % cfg.res2net_scale)
        return fail(PPV_EUNSUPPORTED, "ecapa: res2net_scale must divide channels and be in [2,8]");
    if ((C / cfg.res2net_scale) % 64) return fail(PPV_EUNSUPPORTED, "ecapa: channels / res2net_scale must be a multiple of 64");
    if (cfg.kernel_sizes[1] != 3 || cfg.kernel_sizes[2] != 3 || cfg.kernel_sizes[3] != 3 || cfg.kernel_sizes[4] != 1 || (cfg.kernel_sizes[0] % 2) == 0)
        return fail(PPV_EUNSUPPORTED, "ecapa: kernel sizes must be [odd,3,3,3,1]");
    g->C = C;
    g->C3 = 3 * C;
    g->scale = cfg.res2net_scale;
    g->width = C / cfg.res2net_scale;
    g->Fp = int(align_up(size_t(cfg.input_size), 64));
    g->att = cfg.attention_channels;
    g->se = cfg.se_channels;
    g->P = (cfg.kernel_sizes[0] - 1) / 2 * cfg.dilations[0];
    for (int i = 1; i <= 3; ++i) g->P = std::max(g->P, cfg.dilations[i]);
    return PPV_OK;
}

}  // namespace ppv
