// Verification metrics on the GPU: EER (+ its threshold) and minDCF of a score set, and enrol-DB retrieval (row arg-max).
// Reference: ppvector/metric/metrics.py:4-37 (compute_fnr_fpr / compute_eer / compute_dcf over the SORTED scores) as called by
// ppvector/trainer.py:424-431, and ppvector/predict.py:173-187 (__retrieval: arg-max of the cosine row, threshold test).
//
// The reference sorts ~1e6 scores with numpy and walks cumulative sums on the host.  Here, all on the device and deterministic:
//   1. pack     key = (order-preserving bits of the score) << 1 | label      (label = 1 for a target trial; may come from two
//                                                                              label vectors of a trial x enrol score matrix)
//   2. sort     least-significant-digit radix sort of the 33-bit keys, 8 bits per pass (histogram / scan / stable scatter);
//               equal scores order impostors before targets (numpy's order among ties is unspecified)
//   3. sweep    one pass over the sorted keys: cumulative target count -> FNR[i], FPR[i] in fp64 exactly as metrics.py:15-17,
//               reduced on the fly to  x1 = first i with FNR >= FPR,  x2 = last i with FNR < FPR,  min_i DCF cost
//   4. finish   EER by the reference's linear interpolation between x1 and x2, threshold = sorted score at x1, minDCF normalised.
// HBM-bound integer work: 5 sort passes x 16 B per element + one sweep.
#include <math.h>

#include "common.h"
#include "ptx.cuh"

namespace ppv {

namespace {

constexpr int RS_THREADS = 256;
constexpr int RS_ITEMS = 8;
constexpr int RS_TILE = RS_THREADS * RS_ITEMS;  // 2048 keys per block
constexpr int RS_PASSES = 5;                    // 33 significant bits

__device__ __forceinline__ uint32_t float_to_ordered(float f) {
    const uint32_t u = __float_as_uint(f);
    return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ float ordered_to_float(uint32_t k) {
    return __uint_as_float((k & 0x80000000u) ? (k & 0x7fffffffu) : ~k);
}

// labels != nullptr: label[i] = (labels[i] == 1).  Else a [M, N] score matrix: label = (row_labels[i / N] == col_labels[i % N]).
__global__ void __launch_bounds__(256) eer_pack_kernel(const float* __restrict__ scores, const int32_t* __restrict__ labels,
                                                       const int32_t* __restrict__ row_labels, const int32_t* __restrict__ col_labels, int ncols,
                                                       int64_t n, unsigned long long* __restrict__ keys) {
    for (int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x; i < n; i += int64_t(gridDim.x) * blockDim.x) {
        uint32_t lab;
        if (labels) {
            lab = labels[i] == 1 ? 1u : 0u;
        } else {
            const int64_t r = i / ncols;
            lab = row_labels[r] == col_labels[i - r * ncols] ? 1u : 0u;
        }
        keys[i] = (static_cast<unsigned long long>(float_to_ordered(scores[i])) << 1) | lab;
    }
}

__global__ void __launch_bounds__(RS_THREADS) rs_hist_kernel(const unsigned long long* __restrict__ keys, int64_t n, int shift, int nb,
                                                             uint32_t* __restrict__ hist) {
    __shared__ uint32_t h[256];
    h[threadIdx.x] = 0;
    __syncthreads();
    const int64_t base = int64_t(blockIdx.x) * RS_TILE;
#pragma unroll
    for (int r = 0; r < RS_ITEMS; ++r) {
        const int64_t i = base + r * RS_THREADS + threadIdx.x;
        if (i < n) atomicAdd(&h[(keys[i] >> shift) & 255u], 1u);
    }
    __syncthreads();
    hist[size_t(threadIdx.x) * nb + blockIdx.x] = h[threadIdx.x];  // digit-major: a scan over this array is the scatter base
}

// exclusive scan of `total` counters in place, one block (total = 256 * nb <= a few hundred thousand)
__global__ void __launch_bounds__(1024) rs_scan_kernel(uint32_t* __restrict__ a, int total) {
    __shared__ uint32_t warp_sums[32];
    __shared__ uint32_t carry;
    const int per = (total + 1023) / 1024;
    const int beg = min(total, int(threadIdx.x) * per), end = min(total, beg + per);
    uint32_t s = 0;
    for (int i = beg; i < end; ++i) s += a[i];
    // block exclusive scan of the per-thread sums
    uint32_t v = s;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const uint32_t t = __shfl_up_sync(0xffffffffu, v, o);
        if (lane >= o) v += t;
    }
    if (lane == 31) warp_sums[warp] = v;
    __syncthreads();
    if (warp == 0) {
        uint32_t w = warp_sums[lane];
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const uint32_t t = __shfl_up_sync(0xffffffffu, w, o);
            if (lane >= o) w += t;
        }
        warp_sums[lane] = w;
        if (lane == 31) carry = w;
    }
    __syncthreads();
    uint32_t run = v - s + (warp > 0 ? warp_sums[warp - 1] : 0u);  // exclusive prefix of this thread's chunk
    for (int i = beg; i < end; ++i) {
        const uint32_t t = a[i];
        a[i] = run;
        run += t;
    }
}

// stable scatter of one tile: rounds of 256 keys in tile order; rank inside a round = warp-level match + per-warp digit counters
__global__ void __launch_bounds__(RS_THREADS) rs_scatter_kernel(const unsigned long long* __restrict__ in, unsigned long long* __restrict__ out,
                                                                int64_t n, int shift, int nb, const uint32_t* __restrict__ hist) {
    __shared__ uint32_t base[256];
    __shared__ uint32_t cnt[RS_THREADS / 32][256];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    base[tid] = hist[size_t(tid) * nb + blockIdx.x];
    const int64_t tile0 = int64_t(blockIdx.x) * RS_TILE;
    for (int r = 0; r < RS_ITEMS; ++r) {
#pragma unroll
        for (int w = 0; w < RS_THREADS / 32; ++w) cnt[w][tid] = 0;
        __syncthreads();
        const int64_t i = tile0 + r * RS_THREADS + tid;
        const bool valid = i < n;
        unsigned long long key = 0;
        uint32_t d = 256u + uint32_t(lane);  // invalid lanes: a digit nobody shares
        if (valid) {
            key = in[i];
            d = uint32_t(key >> shift) & 255u;
        }
        const uint32_t peers = __match_any_sync(0xffffffffu, d);
        const uint32_t rank_w = __popc(peers & ((1u << lane) - 1u));
        if (valid && rank_w == 0) cnt[warp][d] = __popc(peers);
        __syncthreads();
        {  // thread `tid` owns digit `tid`: turn the per-warp counts into start offsets, advance the running base
            uint32_t off = base[tid];
#pragma unroll
            for (int w = 0; w < RS_THREADS / 32; ++w) {
                const uint32_t t = cnt[w][tid];
                cnt[w][tid] = off;
                off += t;
            }
            base[tid] = off;
        }
        __syncthreads();
        if (valid) out[cnt[warp][d] + rank_w] = key;
        __syncthreads();
    }
}

struct EerAcc {                    // device scratch of the sweep
    unsigned long long x1;         // min index with FNR >= FPR
    unsigned long long x2p1;       // 1 + max index with FNR <  FPR (0: none)
    unsigned long long min_cost;   // bits of the smallest detection cost (non-negative doubles order like their bit patterns)
    unsigned long long n_target;
};

__global__ void __launch_bounds__(256) eer_count_kernel(const unsigned long long* __restrict__ keys, int64_t n, uint32_t* __restrict__ tile_sums) {
    __shared__ uint32_t ws[8];
    const int64_t base = int64_t(blockIdx.x) * RS_TILE;
    uint32_t s = 0;
#pragma unroll
    for (int r = 0; r < RS_ITEMS; ++r) {
        const int64_t i = base + r * RS_THREADS + threadIdx.x;
        if (i < n) s += uint32_t(keys[i] & 1ull);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if ((threadIdx.x & 31) == 0) ws[threadIdx.x >> 5] = s;
    __syncthreads();
    if (threadIdx.x == 0) {
        uint32_t t = 0;
        for (int w = 0; w < 8; ++w) t += ws[w];
        tile_sums[blockIdx.x] = t;
    }
}

__global__ void eer_init_kernel(EerAcc* acc, const uint32_t* tile_sums_scanned, const uint32_t* last_tile_sum_src, int nb) {
    // tile_sums was scanned in place (exclusive); the total is the last exclusive prefix + the last tile's own count
    acc->x1 = ~0ull;
    acc->x2p1 = 0ull;
    acc->min_cost = ~0ull;
    acc->n_target = static_cast<unsigned long long>(tile_sums_scanned[nb - 1]) + *last_tile_sum_src;
}

// One tile per block, thread t owns RS_ITEMS CONSECUTIVE keys (so that the in-tile scan is a thread-local walk + a block scan).
__global__ void __launch_bounds__(RS_THREADS) eer_sweep_kernel(const unsigned long long* __restrict__ keys, int64_t n,
                                                               const uint32_t* __restrict__ tile_prefix, double p_target, double c_miss, double c_fa,
                                                               EerAcc* acc) {
    __shared__ uint32_t warp_sums[RS_THREADS / 32];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int64_t first = int64_t(blockIdx.x) * RS_TILE + int64_t(tid) * RS_ITEMS;
    uint32_t lab[RS_ITEMS], s = 0;
#pragma unroll
    for (int k = 0; k < RS_ITEMS; ++k) {
        lab[k] = (first + k < n) ? uint32_t(keys[first + k] & 1ull) : 0u;
        s += lab[k];
    }
    uint32_t v = s;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const uint32_t t = __shfl_up_sync(0xffffffffu, v, o);
        if (lane >= o) v += t;
    }
    if (lane == 31) warp_sums[warp] = v;
    __syncthreads();
    uint32_t wpre = 0;
    for (int w = 0; w < warp; ++w) wpre += warp_sums[w];
    unsigned long long tcount = static_cast<unsigned long long>(tile_prefix[blockIdx.x]) + wpre + (v - s);  // targets before this thread's keys
    const double nt = double(acc->n_target), ni = double(static_cast<unsigned long long>(n) - acc->n_target);
    unsigned long long x1 = ~0ull, x2p1 = 0ull, mc = ~0ull;
#pragma unroll
    for (int k = 0; k < RS_ITEMS; ++k) {
        const int64_t i = first + k;
        if (i >= n) break;
        tcount += lab[k];
        const double fnr = double(tcount) / nt;                                            // metrics.py:15
        const double fpr = 1.0 - double(static_cast<unsigned long long>(i + 1) - tcount) / ni;  // metrics.py:16
        if (fnr - fpr >= 0.0) {
            if (x1 == ~0ull) x1 = static_cast<unsigned long long>(i);
        } else {
            x2p1 = static_cast<unsigned long long>(i) + 1ull;
        }
        const double cost = c_miss * fnr * p_target + c_fa * fpr * (1.0 - p_target);       // metrics.py:34
        const unsigned long long cb = static_cast<unsigned long long>(__double_as_longlong(cost < 0.0 ? 0.0 : cost));
        mc = cb < mc ? cb : mc;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        const unsigned long long a = __shfl_xor_sync(0xffffffffu, x1, o), b = __shfl_xor_sync(0xffffffffu, x2p1, o),
                                 c = __shfl_xor_sync(0xffffffffu, mc, o);
        x1 = a < x1 ? a : x1;
        x2p1 = b > x2p1 ? b : x2p1;
        mc = c < mc ? c : mc;
    }
    if (lane == 0) {
        if (x1 != ~0ull) atomicMin(&acc->x1, x1);
        if (x2p1 != 0ull) atomicMax(&acc->x2p1, x2p1);
        atomicMin(&acc->min_cost, mc);
    }
}

// target count before index i (inclusive of i): a short serial walk is enough for the two indices the finish step needs
__device__ double fnr_at(const unsigned long long* keys, const uint32_t* tile_prefix, int64_t i, double nt, double* fpr, double ni) {
    const int64_t tile = i / RS_TILE;
    unsigned long long t = tile_prefix[tile];
    for (int64_t j = tile * RS_TILE; j <= i; ++j) t += keys[j] & 1ull;
    *fpr = 1.0 - double(static_cast<unsigned long long>(i + 1) - t) / ni;
    return double(t) / nt;
}

__global__ void eer_finish_kernel(const unsigned long long* __restrict__ keys, int64_t n, const uint32_t* __restrict__ tile_prefix, const EerAcc* acc,
                                  double p_target, double c_miss, double c_fa, double* __restrict__ out) {
    const double nt = double(acc->n_target), ni = double(static_cast<unsigned long long>(n) - acc->n_target);
    const double nan = __longlong_as_double(0x7ff8000000000000ll);
    double eer = nan, thr = nan;
    if (acc->x1 != ~0ull && acc->x2p1 != 0ull && nt > 0.0 && ni > 0.0) {  // metrics.py:21-30
        const int64_t x1 = int64_t(acc->x1), x2 = int64_t(acc->x2p1) - 1;
        double fpr1, fpr2;
        const double fnr1 = fnr_at(keys, tile_prefix, x1, nt, &fpr1, ni);
        const double fnr2 = fnr_at(keys, tile_prefix, x2, nt, &fpr2, ni);
        const double a = (fnr1 - fpr1) / (fpr2 - fpr1 - (fnr2 - fnr1));
        eer = fnr1 + a * (fnr2 - fnr1);
        thr = double(ordered_to_float(uint32_t(keys[x1] >> 1)));
    }
    const double c_def = fmin(c_miss * p_target, c_fa * (1.0 - p_target));
    out[0] = eer;
    out[1] = thr;
    out[2] = __longlong_as_double(static_cast<long long>(acc->min_cost)) / c_def;
    out[3] = nt;
}

__global__ void __launch_bounds__(256) row_argmax_kernel(const float* __restrict__ sim, int rows, int cols, int32_t* __restrict__ idx,
                                                         float* __restrict__ best) {
    __shared__ float sv[8];
    __shared__ int si[8];
    const int r = blockIdx.x;
    float bv = -INFINITY;
    int bi = 0x7fffffff;
    for (int c = threadIdx.x; c < cols; c += blockDim.x) {
        const float v = sim[int64_t(r) * cols + c];
        if (v > bv || (v == bv && c < bi)) {  // first maximum, like numpy.argmax
            bv = v;
            bi = c;
        }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        const float ov = __shfl_xor_sync(0xffffffffu, bv, o);
        const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
        if (ov > bv || (ov == bv && oi < bi)) {
            bv = ov;
            bi = oi;
        }
    }
    if ((threadIdx.x & 31) == 0) {
        sv[threadIdx.x >> 5] = bv;
        si[threadIdx.x >> 5] = bi;
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        for (int w = 1; w < 8; ++w)
            if (sv[w] > bv || (sv[w] == bv && si[w] < bi)) {
                bv = sv[w];
                bi = si[w];
            }
        idx[r] = bi;
        best[r] = bv;
    }
}

struct EerWs {
    unsigned long long *ka, *kb;  // [n] sort keys, ping-pong
    uint32_t *hist, *tsum, *tsum_raw;  // [256][nb] digit counts; [nb] per-tile target counts, scanned and raw
    EerAcc* acc;
};
void carve_eer(WsCarver& cv, int64_t n, EerWs* w) {
    const size_t nb = size_t((n + RS_TILE - 1) / RS_TILE);
    w->ka = static_cast<unsigned long long*>(cv.take(size_t(n) * 8));
    w->kb = static_cast<unsigned long long*>(cv.take(size_t(n) * 8));
    w->hist = static_cast<uint32_t*>(cv.take(256 * nb * 4));
    w->tsum = static_cast<uint32_t*>(cv.take(nb * 4));
    w->tsum_raw = static_cast<uint32_t*>(cv.take(nb * 4));
    w->acc = static_cast<EerAcc*>(cv.take(sizeof(EerAcc)));
}

}  // namespace

size_t eer_workspace_bytes(int64_t n) {
    if (n <= 0) return 0;
    return carve_extent([&](WsCarver& cv) { EerWs w; carve_eer(cv, n, &w); });
}

// Exactly one of `labels` [n] or (`row_labels` [n / ncols], `col_labels` [ncols]).  out: device double[4] = {eer, threshold, min_dcf, n_target}.
int eer_mindcf(const float* scores, const int32_t* labels, const int32_t* row_labels, const int32_t* col_labels, int ncols, int64_t n,
               double p_target, double c_miss, double c_fa, double* out, void* ws, size_t ws_bytes, cudaStream_t st) {
    PPV_REQUIRE(scores && out, "eer_mindcf: null argument");
    PPV_REQUIRE(n >= 2 && n < (int64_t(1) << 32), "eer_mindcf: need 2 <= n < 2^32 scores");
    PPV_REQUIRE((labels != nullptr) != (row_labels != nullptr && col_labels != nullptr), "eer_mindcf: labels XOR (row_labels, col_labels)");
    if (!labels) PPV_REQUIRE(ncols > 0 && n % ncols == 0, "eer_mindcf: n must be rows x ncols");
    if (int rc = check_workspace("eer_mindcf", ws, ws_bytes, eer_workspace_bytes(n), "ppv_eer_workspace_bytes")) return rc;
    const int nb = int((n + RS_TILE - 1) / RS_TILE);
    WsCarver cv{static_cast<uint8_t*>(ws)};
    EerWs w;
    carve_eer(cv, n, &w);
    const int pack_grid = int(std::min<int64_t>((n + 255) / 256, 132 * 8));
    eer_pack_kernel<<<pack_grid, 256, 0, st>>>(scores, labels, row_labels, col_labels, ncols, n, w.ka);
    PPV_LAUNCH_OK("eer_pack_kernel");
    for (int pass = 0; pass < RS_PASSES; ++pass) {
        const int shift = 8 * pass;
        rs_hist_kernel<<<nb, RS_THREADS, 0, st>>>(w.ka, n, shift, nb, w.hist);
        rs_scan_kernel<<<1, 1024, 0, st>>>(w.hist, 256 * nb);
        rs_scatter_kernel<<<nb, RS_THREADS, 0, st>>>(w.ka, w.kb, n, shift, nb, w.hist);
        PPV_LAUNCH_OK("radix sort pass");
        std::swap(w.ka, w.kb);
    }
    eer_count_kernel<<<nb, RS_THREADS, 0, st>>>(w.ka, n, w.tsum);
    PPV_CUDA_OK(cudaMemcpyAsync(w.tsum_raw, w.tsum, size_t(nb) * 4, cudaMemcpyDeviceToDevice, st));
    rs_scan_kernel<<<1, 1024, 0, st>>>(w.tsum, nb);
    eer_init_kernel<<<1, 1, 0, st>>>(w.acc, w.tsum, w.tsum_raw + (nb - 1), nb);
    eer_sweep_kernel<<<nb, RS_THREADS, 0, st>>>(w.ka, n, w.tsum, p_target, c_miss, c_fa, w.acc);
    eer_finish_kernel<<<1, 1, 0, st>>>(w.ka, n, w.tsum, w.acc, p_target, c_miss, c_fa, out);
    PPV_LAUNCH_OK("eer sweep");
    return PPV_OK;
}

int row_argmax(const float* sim, int rows, int cols, int32_t* idx, float* best, cudaStream_t st) {
    PPV_REQUIRE(sim && idx && best && rows > 0 && cols > 0, "row_argmax: bad argument");
    row_argmax_kernel<<<rows, 256, 0, st>>>(sim, rows, cols, idx, best);
    PPV_LAUNCH_OK("row_argmax_kernel");
    return PPV_OK;
}

}  // namespace ppv
