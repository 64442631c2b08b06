// Adaptive score normalisation (AS-norm) against a cohort: per-row statistics of the top_n largest scores, and the normalisation of
// the trial x enrolment matrix from them.  There is no counterpart in the reference (it scores raw cosines only).
//   row stats: scores [rows, cols] (leading dimension ld) -> mean / std of each row's top_n largest values.  One CTA per row.  An exact
//              radix select over the order-preserving uint32 image of the floats (three digit passes of 11 / 11 / 10 bits, a per-CTA
//              histogram in shared memory each) finds the top_n-th largest value tau and how many values lie strictly above it; a
//              fourth pass accumulates sum(x - tau) and sum((x - tau)^2) over those in fp64, and the (top_n - above) copies of tau add
//              zero to both.  Shifting by tau keeps the variance free of the cancellation a raw sum(x^2) has for scores near 1.0.
//              Every thread takes the same columns in the same order whatever the number of rows, and the partial sums are reduced in
//              a fixed tree: the output is bitwise reproducible and independent of how rows are batched.  Rows of up to
//              TN_SMEM_COLS columns are staged in shared memory and read from HBM once; wider rows take the four passes over global
//              memory.  Both run the same code on a different source pointer, so the two sides of the cut agree bit for bit.
//   apply    : s'(t, e) = 0.5 * ((s - mean_e) / std_e + (s - mean_t) / std_t), in place, one pass.
#include "common.h"

namespace ppv {

namespace {

constexpr int TN_THREADS = 256;
constexpr int TN_WARPS = TN_THREADS / 32;
constexpr int TN_BINS = 2048;                        // 11-bit digits
constexpr int TN_BINS_PER_THREAD = TN_BINS / TN_THREADS;
constexpr int TN_SMEM_COLS = 10240;                  // 40 KB row + 8 KB histogram: four CTAs per SM
constexpr int TN_UNROLL = 8;                         // loads in flight per thread on the global path
constexpr double TN_STD_FLOOR = 1e-6;

// Order-preserving image of a float: a < b (as finite floats, -0 < +0) iff key(a) < key(b).
__device__ __forceinline__ uint32_t order_key(float x) {
    const uint32_t u = __float_as_uint(x);
    return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ float key_value(uint32_t k) { return __uint_as_float((k & 0x80000000u) ? (k & 0x7fffffffu) : ~k); }

// f(x) on every value of the row; thread t visits columns t, t + T, t + 2T, ... in that order (the order the fp64 sums depend on).
template <typename F>
__device__ __forceinline__ void for_each_col(const float* row, int cols, F&& f) {
    int i = threadIdx.x;
    for (; i + (TN_UNROLL - 1) * TN_THREADS < cols; i += TN_UNROLL * TN_THREADS) {
        float v[TN_UNROLL];
#pragma unroll
        for (int u = 0; u < TN_UNROLL; ++u) v[u] = row[i + u * TN_THREADS];
#pragma unroll
        for (int u = 0; u < TN_UNROLL; ++u) f(v[u]);
    }
    for (; i < cols; i += TN_THREADS) f(row[i]);
}

__global__ void __launch_bounds__(TN_THREADS) topn_row_stats_kernel(const float* __restrict__ scores, int cols, int64_t ld, int top_n,
                                                                     bool staged, float* __restrict__ mean_out, float* __restrict__ std_out) {
    extern __shared__ float srow[];
    __shared__ uint32_t hist[TN_BINS];
    __shared__ uint32_t warp_tot[TN_WARPS];
    __shared__ double warp_s1[TN_WARPS], warp_s2[TN_WARPS];
    __shared__ uint32_t sel_bin, sel_above;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const float* row = scores + int64_t(blockIdx.x) * ld;
    if (staged) {
        for (int i = tid; i < cols; i += TN_THREADS) srow[i] = row[i];
        row = srow;  // made visible by the first barrier below
    }

    // Radix select, most significant digit first.  Invariant: the values whose key matches `prefix` under `mask` hold the
    // `need`-th largest of the top_n; `above` values lie strictly above all of them.
    uint32_t prefix = 0, mask = 0;
    int need = top_n, above = 0;
#pragma unroll 1
    for (int pass = 0; pass < 3; ++pass) {
        const int shift = pass == 0 ? 21 : pass == 1 ? 10 : 0;
        const uint32_t digit_mask = pass == 2 ? 0x3ffu : 0x7ffu;
        for (int b = tid; b < TN_BINS; b += TN_THREADS) hist[b] = 0;
        __syncthreads();
        for_each_col(row, cols, [&](float x) {
            const uint32_t k = order_key(x);
            if ((k & mask) == prefix) atomicAdd(&hist[(k >> shift) & digit_mask], 1u);
        });
        __syncthreads();
        // thread t owns bins TN_BINS-1-8t down to TN_BINS-8-8t: an exclusive scan over threads counts the values above its bins
        uint32_t own = 0;
#pragma unroll
        for (int j = 0; j < TN_BINS_PER_THREAD; ++j) own += hist[TN_BINS - 1 - (tid * TN_BINS_PER_THREAD + j)];
        uint32_t inc = own;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const uint32_t v = __shfl_up_sync(0xffffffffu, inc, o);
            if (lane >= o) inc += v;
        }
        if (lane == 31) warp_tot[warp] = inc;
        __syncthreads();
        uint32_t run = inc - own;
        for (int w = 0; w < warp; ++w) run += warp_tot[w];
        if (run < uint32_t(need) && run + own >= uint32_t(need)) {  // exactly one thread: the one holding the need-th value
#pragma unroll 1
            for (int j = 0; j < TN_BINS_PER_THREAD; ++j) {
                const int b = TN_BINS - 1 - (tid * TN_BINS_PER_THREAD + j);
                const uint32_t h = hist[b];
                if (run + h >= uint32_t(need)) {
                    sel_bin = uint32_t(b);
                    sel_above = run;
                    break;
                }
                run += h;
            }
        }
        __syncthreads();
        prefix |= sel_bin << shift;
        mask |= digit_mask << shift;
        need -= int(sel_above);
        above += int(sel_above);
        __syncthreads();  // sel_* and hist are rewritten by the next pass
    }
    // prefix is now the key of tau; `above` values are strictly greater, `need` >= 1 copies of tau complete the top_n
    const float tau = key_value(prefix);
    const double t = double(tau);
    double s1 = 0.0, s2 = 0.0;
    for_each_col(row, cols, [&](float x) {
        if (order_key(x) > prefix) {
            const double d = double(x) - t;
            s1 += d;
            s2 += d * d;
        }
    });
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        s1 += __shfl_xor_sync(0xffffffffu, s1, o);
        s2 += __shfl_xor_sync(0xffffffffu, s2, o);
    }
    if (lane == 0) {
        warp_s1[warp] = s1;
        warp_s2[warp] = s2;
    }
    __syncthreads();
    if (tid == 0) {
        double S1 = 0.0, S2 = 0.0;
        for (int w = 0; w < TN_WARPS; ++w) {
            S1 += warp_s1[w];
            S2 += warp_s2[w];
        }
        const double n = double(top_n);
        const double var = fmax(S2 - S1 * S1 / n, 0.0) / (n - 1.0);
        mean_out[blockIdx.x] = float(t + S1 / n);
        std_out[blockIdx.x] = float(fmax(sqrt(var), TN_STD_FLOOR));
    }
}

__global__ void __launch_bounds__(256) as_norm_apply_kernel(float* __restrict__ S, int M, int N, const float* __restrict__ trial_mean,
                                                            const float* __restrict__ trial_std, const float* __restrict__ enroll_mean,
                                                            const float* __restrict__ enroll_std) {
    const float floor = float(TN_STD_FLOOR);
    for (int r = blockIdx.y; r < M; r += gridDim.y) {
        const float mt = trial_mean[r], st = fmaxf(trial_std[r], floor);
        float* row = S + int64_t(r) * N;
        for (int c = blockIdx.x * blockDim.x + threadIdx.x; c < N; c += gridDim.x * blockDim.x) {
            const float s = row[c];
            row[c] = 0.5f * ((s - enroll_mean[c]) / fmaxf(enroll_std[c], floor) + (s - mt) / st);
        }
    }
}

}  // namespace

int topn_row_stats(const float* scores, int rows, int cols, int64_t ld, int top_n, float* mean, float* std, cudaStream_t st) {
    PPV_REQUIRE(scores && mean && std, "topn_row_stats: null argument");
    PPV_REQUIRE(rows > 0 && cols > 0, "topn_row_stats: rows and cols must be positive (got " + std::to_string(rows) + ", " +
                                          std::to_string(cols) + ")");
    PPV_REQUIRE(ld >= cols, "topn_row_stats: ld " + std::to_string(ld) + " < cols " + std::to_string(cols));
    PPV_REQUIRE(top_n >= 2 && top_n <= cols,
                "topn_row_stats: top_n must satisfy 2 <= top_n <= cols (got top_n " + std::to_string(top_n) + ", cols " + std::to_string(cols) + ")");
    const bool staged = cols <= TN_SMEM_COLS;
    const size_t smem = staged ? size_t(cols) * sizeof(float) : 0;
    PPV_ONCE_PER_DEVICE(PPV_CUDA_OK(cudaFuncSetAttribute(topn_row_stats_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                                         int(TN_SMEM_COLS * sizeof(float)))));
    topn_row_stats_kernel<<<rows, TN_THREADS, smem, st>>>(scores, cols, ld, top_n, staged, mean, std);
    PPV_LAUNCH_OK("topn_row_stats_kernel");
    return PPV_OK;
}

int as_norm_apply(float* scores, int M, int N, const float* trial_mean, const float* trial_std, const float* enroll_mean,
                  const float* enroll_std, cudaStream_t st) {
    PPV_REQUIRE(scores && trial_mean && trial_std && enroll_mean && enroll_std, "as_norm_apply: null argument");
    PPV_REQUIRE(M > 0 && N > 0, "as_norm_apply: M and N must be positive (got " + std::to_string(M) + ", " + std::to_string(N) + ")");
    const dim3 grid(unsigned(std::min((N + 255) / 256, 1024)), unsigned(std::min(M, 65535)));
    as_norm_apply_kernel<<<grid, 256, 0, st>>>(scores, M, N, trial_mean, trial_std, enroll_mean, enroll_std);
    PPV_LAUNCH_OK("as_norm_apply_kernel");
    return PPV_OK;
}

}  // namespace ppv
