// Spectral clustering of the diarization chunk embeddings on the GPU.
// Reference: ppvector/infer_utils/speaker_diarization.py:219-310 (SpectralCluster): cosine affinity, per-row pruning (:260-275),
// symmetrised Laplacian (:242-244, :277-283), scipy.linalg.eigh (:285-296) and sklearn's k_means (:299-302).
//
//   prune      one block per row: radix select (4 x 8-bit passes over order-preserving fp32 keys) of the n_elems-th smallest entry,
//              then every entry below it and the first (in column order) of the entries equal to it are zeroed.  numpy's argsort
//              leaves the order of exact ties unspecified; here the lower column index goes first.
//   laplacian  one block per row: M = (P + P^T) / 2 with a zero diagonal, D_i = sum_j |M_ij| in a fixed order, L = diag(D) - M (fp64).
//   eig        the m smallest eigenpairs of L, all fp64, the classic LAPACK chain:
//                sytrd  unblocked Householder tridiagonalisation; per column one single-block "house" launch (finishes w of the
//                       previous column, applies its pending rank-2 update to row k and forms the reflector) and one fused launch
//                       that applies the pending rank-2 update to the trailing matrix and computes p = tau A v in the same pass.
//                       The full symmetric trailing matrix is kept (both triangles), so every pass reads rows contiguously; the
//                       reflector v_k is stored in row k (the lower triangle of LAPACK's column-major view).  The trailing matrix
//                       is read and written once per column: ~N^3/3 x 16 B, HBM-bound above the L2-resident sizes.
//                stebz  bisection on Sturm counts, one warp per eigenvalue, 32 points per step (multisection).
//                stein  inverse iteration on the tridiagonal (LU with partial pivoting), modified Gram-Schmidt (twice) against the
//                       earlier vectors of a cluster of close eigenvalues (gap < 1e-3 |T|_1), like LAPACK's dstein.
//                ormtr  back-transformation Q z, one block per vector, the vector in registers.
//   kmeans     sklearn's KMeans(n_init=1, init="k-means++", algorithm="lloyd") in one block: greedy k-means++ with 2 + int(log k)
//              local trials on caller-supplied uniforms, Lloyd iterations, the final E-step, inertia.
// Every sum runs in a fixed order (no floating-point atomics), so results are bitwise reproducible; sequential stages are
// sequences of launches (no grid-wide barriers).
#include <float.h>
#include <math.h>

#include "common.h"

namespace ppv {

namespace {

constexpr int CL_MAX_N = 8192;
constexpr int CL_MAX_K = 32;  // eigenpairs / clusters
constexpr int CL_MAX_TRIALS = 2 + 3;  // 2 + int(log 32)

__device__ __forceinline__ uint32_t ordered_key(float f) {
    const uint32_t u = __float_as_uint(f);
    return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}

// Block-wide sum of one double per thread, in a fixed order.  red: >= 32 doubles of shared memory.  All threads get the result.
__device__ double block_sum(double v, double* red) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = (blockDim.x + 31) >> 5;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    __syncthreads();  // red may still be read by a previous call
    if (lane == 0) red[warp] = v;
    __syncthreads();
    double s = 0.0;
    for (int w = 0; w < nw; ++w) s += red[w];
    return s;
}

// ---------------------------------------------------------------- pruning
__global__ void __launch_bounds__(256) prune_kernel(float* __restrict__ A, int N, int n_elems) {
    extern __shared__ uint32_t keys[];
    __shared__ uint32_t hist[256];
    __shared__ uint32_t sel[2];
    __shared__ uint32_t wcnt[8];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    float* row = A + int64_t(blockIdx.x) * N;
    for (int j = tid; j < N; j += 256) keys[j] = ordered_key(row[j]);
    uint32_t prefix = 0, mask = 0, r = uint32_t(n_elems - 1);
    for (int pass = 0; pass < 4; ++pass) {
        const int shift = 24 - 8 * pass;
        hist[tid] = 0;
        __syncthreads();
        for (int j = tid; j < N; j += 256) {
            const uint32_t k = keys[j];
            if ((k & mask) == prefix) atomicAdd(&hist[(k >> shift) & 255u], 1u);
        }
        __syncthreads();
        if (tid == 0) {
            uint32_t cum = 0, d = 255;
            for (uint32_t q = 0; q < 256; ++q) {
                if (cum + hist[q] > r) {
                    d = q;
                    break;
                }
                cum += hist[q];
            }
            sel[0] = d;
            sel[1] = r - cum;
        }
        __syncthreads();
        prefix |= sel[0] << shift;
        mask |= 255u << shift;
        r = sel[1];
        __syncthreads();
    }
    const uint32_t thr = prefix, ties = r + 1;  // entries equal to thr that are pruned: the first `ties` in column order
    uint32_t seen = 0;
    for (int c0 = 0; c0 < N; c0 += 256) {
        const int j = c0 + tid;
        const uint32_t k = j < N ? keys[j] : 0xffffffffu;
        const bool eq = j < N && k == thr;
        const uint32_t ball = __ballot_sync(0xffffffffu, eq);
        if (lane == 0) wcnt[warp] = __popc(ball);
        __syncthreads();
        uint32_t before = seen, total = 0;
        for (int w = 0; w < 8; ++w) {
            if (w < warp) before += wcnt[w];
            total += wcnt[w];
        }
        before += __popc(ball & ((1u << lane) - 1u));
        if (j < N && (k < thr || (eq && before < ties))) row[j] = 0.f;
        seen += total;
        __syncthreads();
    }
}

// ---------------------------------------------------------------- Laplacian
__global__ void __launch_bounds__(256) laplacian_kernel(const float* __restrict__ P, int N, double* __restrict__ L) {
    __shared__ double red[32];
    const int i = blockIdx.x;
    double acc = 0.0;
    for (int j = threadIdx.x; j < N; j += 256) {
        const double m = (i == j) ? 0.0 : 0.5 * (double(P[int64_t(i) * N + j]) + double(P[int64_t(j) * N + i]));
        L[int64_t(i) * N + j] = 0.0 - m;
        acc += fabs(m);
    }
    const double d = block_sum(acc, red);
    if (threadIdx.x == 0) L[int64_t(i) * N + i] = d;
}

// ---------------------------------------------------------------- sytrd
struct EigWs {
    double *d, *e, *e2, *tau, *p, *w, *scal;  // scal: {gl, gu, onenrm, pivmin}
    double *u0, *u1, *u2, *mult, *x;
    int* piv;
    double* Z;  // [m][N] tridiagonal eigenvectors
};

// symmetric rank-2 term v_i w_j + w_i v_j, rounded the same way for (i, j) and (j, i)
__device__ __forceinline__ double r2(double vi, double wi, double vj, double wj) { return __dadd_rn(__dmul_rn(vi, wj), __dmul_rn(wi, vj)); }

// Column k: w_{k-1} = p - (tau_{k-1} / 2)(p . v_{k-1}) v_{k-1}; row k of A += pending update k-1; reflector of A[k, k+1:].
__global__ void __launch_bounds__(1024) house_kernel(double* __restrict__ A, int N, int k, EigWs ws) {
    __shared__ double red[32];
    const int tid = threadIdx.x;
    const double* vp = A + int64_t(k > 0 ? k - 1 : 0) * N;  // v_{k-1}, valid at columns >= k
    double* row = A + int64_t(k) * N;
    if (k > 0) {
        double s = 0.0;
        for (int j = k + tid; j < N; j += 1024) s += ws.p[j] * vp[j];
        const double alpha = -0.5 * ws.tau[k - 1] * block_sum(s, red);
        for (int j = k + tid; j < N; j += 1024) ws.w[j] = ws.p[j] + alpha * vp[j];
        __syncthreads();
        const double vk = vp[k], wk = ws.w[k];
        for (int j = k + tid; j < N; j += 1024) row[j] = __dsub_rn(row[j], r2(vk, wk, vp[j], ws.w[j]));
        __syncthreads();
    }
    if (tid == 0) ws.d[k] = row[k];
    if (k == N - 1) return;
    const double alpha = row[k + 1];  // read before block_sum's barrier: thread 0 overwrites it with 1 below
    double s = 0.0;
    for (int j = k + 2 + tid; j < N; j += 1024) s += row[j] * row[j];
    const double xnorm = sqrt(block_sum(s, red));
    double tau = 0.0, beta = alpha, scale = 0.0;
    if (xnorm != 0.0) {
        beta = -copysign(hypot(alpha, xnorm), alpha);
        tau = (beta - alpha) / beta;
        scale = 1.0 / (alpha - beta);
    }
    for (int j = k + 2 + tid; j < N; j += 1024) row[j] *= scale;
    if (tid == 0) {
        row[k + 1] = 1.0;
        ws.e[k] = beta;
        ws.tau[k] = tau;
    }
}

constexpr int TR_ROWS = 8;
// Rows [k+1, N) x columns [k+1, N): A -= (v_{k-1} w_{k-1}^T + w_{k-1} v_{k-1}^T) (k > 0), then p = tau_k A v_k.
__global__ void __launch_bounds__(256) trail_update_symv_kernel(double* __restrict__ A, int N, int k, EigWs ws) {
    __shared__ double part[8][TR_ROWS];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int i0 = k + 1 + blockIdx.x * TR_ROWS;
    const double* vk = A + int64_t(k) * N;
    const double* vp = A + int64_t(k > 0 ? k - 1 : 0) * N;
    double acc[TR_ROWS], vpi[TR_ROWS], wpi[TR_ROWS];
#pragma unroll
    for (int r = 0; r < TR_ROWS; ++r) {
        acc[r] = 0.0;
        const int i = min(i0 + r, N - 1);
        vpi[r] = k > 0 ? vp[i] : 0.0;
        wpi[r] = k > 0 ? ws.w[i] : 0.0;
    }
    for (int j = k + 1 + tid; j < N; j += 256) {
        const double vj = vk[j];
        const double vpj = k > 0 ? vp[j] : 0.0, wpj = k > 0 ? ws.w[j] : 0.0;
#pragma unroll
        for (int r = 0; r < TR_ROWS; ++r) {
            const int i = i0 + r;
            if (i < N) {
                double* a = A + int64_t(i) * N + j;
                double v = *a;
                if (k > 0) {
                    v = __dsub_rn(v, r2(vpi[r], wpi[r], vpj, wpj));
                    *a = v;
                }
                acc[r] = fma(v, vj, acc[r]);
            }
        }
    }
#pragma unroll
    for (int r = 0; r < TR_ROWS; ++r) {
        double v = acc[r];
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
        if (lane == 0) part[warp][r] = v;
    }
    __syncthreads();
    if (tid < TR_ROWS && i0 + tid < N) {
        double s = 0.0;
        for (int w = 0; w < 8; ++w) s += part[w][tid];
        ws.p[i0 + tid] = ws.tau[k] * s;
    }
}

// ---------------------------------------------------------------- stebz
// Gershgorin interval, |T|_1, pivmin and e^2 (one block).
__global__ void __launch_bounds__(1024) tridiag_prep_kernel(int N, EigWs ws) {
    __shared__ double red[32];
    double gl = INFINITY, gu = -INFINITY, nrm = 0.0, e2max = 0.0;
    for (int i = threadIdx.x; i < N; i += 1024) {
        const double em = i > 0 ? fabs(ws.e[i - 1]) : 0.0, ep = i < N - 1 ? fabs(ws.e[i]) : 0.0;
        gl = fmin(gl, ws.d[i] - em - ep);
        gu = fmax(gu, ws.d[i] + em + ep);
        nrm = fmax(nrm, fabs(ws.d[i]) + em + ep);
        if (i < N - 1) {
            ws.e2[i] = ws.e[i] * ws.e[i];
            e2max = fmax(e2max, ws.e2[i]);
        }
    }
    // min / max do not depend on the order
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        gl = fmin(gl, __shfl_xor_sync(0xffffffffu, gl, o));
        gu = fmax(gu, __shfl_xor_sync(0xffffffffu, gu, o));
        nrm = fmax(nrm, __shfl_xor_sync(0xffffffffu, nrm, o));
        e2max = fmax(e2max, __shfl_xor_sync(0xffffffffu, e2max, o));
    }
    __shared__ double s4[4][32];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    if (lane == 0) {
        s4[0][warp] = gl;
        s4[1][warp] = gu;
        s4[2][warp] = nrm;
        s4[3][warp] = e2max;
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        for (int w = 1; w < 32; ++w) {
            gl = fmin(gl, s4[0][w]);
            gu = fmax(gu, s4[1][w]);
            nrm = fmax(nrm, s4[2][w]);
            e2max = fmax(e2max, s4[3][w]);
        }
        const double pad = 2.0 * DBL_EPSILON * fmax(fabs(gl), fabs(gu)) + DBL_MIN;
        ws.scal[0] = gl - pad;
        ws.scal[1] = gu + pad;
        ws.scal[2] = nrm;
        ws.scal[3] = DBL_MIN * fmax(1.0, e2max);
    }
    (void)red;
}

// number of eigenvalues <= x (LAPACK dlaebz's Sturm count)
__device__ int sturm_count(const double* __restrict__ d, const double* __restrict__ e2, int N, double x, double pivmin) {
    double q = d[0] - x;
    if (fabs(q) < pivmin) q = -pivmin;
    int c = q <= 0.0;
#pragma unroll 1
    for (int i = 1; i < N; ++i) {
        q = d[i] - e2[i - 1] / q - x;
        if (fabs(q) < pivmin) q = -pivmin;
        c += q <= 0.0;
    }
    return c;
}

// one warp per eigenvalue j (0-based, ascending): 32-point multisection keeping count(lo) <= j < count(hi)
__global__ void __launch_bounds__(128) stebz_kernel(int N, int m, EigWs ws, double* __restrict__ evals) {
    const int lane = threadIdx.x & 31;
    const int j = blockIdx.x * 4 + (threadIdx.x >> 5);
    if (j >= m) return;
    double lo = ws.scal[0], hi = ws.scal[1];
    const double nrm = ws.scal[2], pivmin = ws.scal[3];
    for (int it = 0; it < 64; ++it) {  // 33x narrower per step: ~11 steps from the Gershgorin interval to eps |T|
        if (hi - lo <= 2.0 * DBL_EPSILON * fmax(fabs(lo), fabs(hi)) + DBL_EPSILON * nrm + 2.0 * pivmin) break;
        const double x = lo + (hi - lo) * double(lane + 1) / 33.0;
        const int c = sturm_count(ws.d, ws.e2, N, x, pivmin);
        const uint32_t above = __ballot_sync(0xffffffffu, c > j);
        const double xprev = __shfl_up_sync(0xffffffffu, x, 1);
        if (above == 0u) {
            lo = __shfl_sync(0xffffffffu, x, 31);
        } else {
            const int l = __ffs(above) - 1;
            const double nhi = __shfl_sync(0xffffffffu, x, l);
            const double nlo = __shfl_sync(0xffffffffu, xprev, l);
            if (l > 0) lo = nlo;
            hi = nhi;
        }
    }
    if (lane == 0) evals[j] = 0.5 * (lo + hi);
}

// ---------------------------------------------------------------- stein
__device__ __forceinline__ double unit_rand(uint64_t s) {  // splitmix64 -> uniform(-1, 1)
    s += 0x9E3779B97F4A7C15ull;
    s = (s ^ (s >> 30)) * 0xBF58476D1CE4E5B9ull;
    s = (s ^ (s >> 27)) * 0x94D049BB133111EBull;
    s ^= s >> 31;
    return double(s >> 11) * (2.0 / 9007199254740992.0) - 1.0;
}

// LU with partial pivoting of T - sigma I (rows i, i+1 swapped where |sub| > |pivot|); tiny pivots replaced by +-tiny.
__device__ void tri_factor(int N, const EigWs& ws, double sigma, double tiny) {
    double a = ws.d[0] - sigma, c = N > 1 ? ws.e[0] : 0.0;
    for (int i = 0; i < N - 1; ++i) {
        const double b = ws.e[i], an = ws.d[i + 1] - sigma, cn = i + 1 < N - 1 ? ws.e[i + 1] : 0.0;
        if (fabs(a) >= fabs(b)) {
            const double mu = b == 0.0 ? 0.0 : b / a;
            ws.u0[i] = a;
            ws.u1[i] = c;
            ws.u2[i] = 0.0;
            ws.mult[i] = mu;
            ws.piv[i] = 0;
            a = an - mu * c;
            c = cn;
        } else {
            const double mu = a / b;
            ws.u0[i] = b;
            ws.u1[i] = an;
            ws.u2[i] = cn;
            ws.mult[i] = mu;
            ws.piv[i] = 1;
            a = c - mu * an;
            c = -mu * cn;
        }
    }
    ws.u0[N - 1] = a;
    for (int i = 0; i < N; ++i)
        if (fabs(ws.u0[i]) < tiny) ws.u0[i] = ws.u0[i] < 0.0 ? -tiny : tiny;
}

__device__ void tri_solve(int N, const EigWs& ws, double* __restrict__ x) {
    for (int i = 0; i < N - 1; ++i) {
        if (ws.piv[i]) {
            const double t = x[i];
            x[i] = x[i + 1];
            x[i + 1] = t;
        }
        x[i + 1] -= ws.mult[i] * x[i];
    }
    x[N - 1] /= ws.u0[N - 1];
    if (N > 1) x[N - 2] = (x[N - 2] - ws.u1[N - 2] * x[N - 1]) / ws.u0[N - 2];
    for (int i = N - 3; i >= 0; --i) x[i] = (x[i] - ws.u1[i] * x[i + 1] - ws.u2[i] * x[i + 2]) / ws.u0[i];
}

constexpr int STEIN_ITERS = 5;
// One block, the m vectors in order (a vector is orthogonalised against the earlier ones of its cluster).
__global__ void __launch_bounds__(256) stein_kernel(int N, int m, EigWs ws, const double* __restrict__ evals) {
    __shared__ double red[32];
    const int tid = threadIdx.x;
    const double onenrm = ws.scal[2];
    const double ortol = 1e-3 * onenrm, tiny = DBL_EPSILON * fmax(onenrm, DBL_MIN);
    double* x = ws.x;
    double sigma_prev = 0.0;
    int first = 0;
    for (int j = 0; j < m; ++j) {
        double sigma = evals[j];
        if (j > 0) {
            if (sigma - evals[j - 1] > ortol) first = j;
            const double pertol = 10.0 * fabs(DBL_EPSILON * sigma);
            if (sigma - sigma_prev < pertol) sigma = sigma_prev + pertol;
        }
        sigma_prev = sigma;
        if (tid == 0) tri_factor(N, ws, sigma, tiny);
        double s = 0.0;
        for (int i = tid; i < N; i += 256) {
            x[i] = unit_rand(uint64_t(j) * uint64_t(CL_MAX_N) + uint64_t(i));
            s += x[i] * x[i];
        }
        double nrm = sqrt(block_sum(s, red));
        for (int i = tid; i < N; i += 256) x[i] /= nrm;
        __syncthreads();
        for (int it = 0; it < STEIN_ITERS; ++it) {
            if (tid == 0) tri_solve(N, ws, x);
            __syncthreads();
            for (int pass = 0; pass < 2; ++pass) {
                for (int q = first; q < j; ++q) {
                    const double* zq = ws.Z + int64_t(q) * N;
                    double dq = 0.0;
                    for (int i = tid; i < N; i += 256) dq += zq[i] * x[i];
                    dq = block_sum(dq, red);
                    for (int i = tid; i < N; i += 256) x[i] -= dq * zq[i];
                    __syncthreads();
                }
            }
            s = 0.0;
            for (int i = tid; i < N; i += 256) s += x[i] * x[i];
            nrm = sqrt(block_sum(s, red));
            for (int i = tid; i < N; i += 256) x[i] /= nrm;
            __syncthreads();
        }
        double* zj = ws.Z + int64_t(j) * N;
        for (int i = tid; i < N; i += 256) zj[i] = x[i];
        __syncthreads();
    }
}

// ---------------------------------------------------------------- ormtr
constexpr int OR_THREADS = 512;
constexpr int OR_PER = CL_MAX_N / OR_THREADS;
// evecs[:, j] = H_0 H_1 ... H_{N-2} z_j, H_k = I - tau_k v_k v_k^T with v_k in row k of A (columns k+1..N-1)
__global__ void __launch_bounds__(OR_THREADS) ormtr_kernel(const double* __restrict__ A, int N, int m, EigWs ws, double* __restrict__ evecs) {
    __shared__ double part[2][OR_THREADS / 32];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int j = blockIdx.x;
    double z[OR_PER];
#pragma unroll
    for (int r = 0; r < OR_PER; ++r) {
        const int i = tid + r * OR_THREADS;
        z[r] = i < N ? ws.Z[int64_t(j) * N + i] : 0.0;
    }
    int buf = 0;  // partials double-buffered over the reflectors actually applied: one barrier per reflector
    for (int k = N - 2; k >= 0; --k) {
        const double tau = ws.tau[k];
        if (tau == 0.0) continue;
        buf ^= 1;
        const double* v = A + int64_t(k) * N;
        double s = 0.0;
#pragma unroll
        for (int r = 0; r < OR_PER; ++r) {
            const int i = tid + r * OR_THREADS;
            if (i > k && i < N) s = fma(v[i], z[r], s);
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
        if (lane == 0) part[buf][warp] = s;
        __syncthreads();
        s = 0.0;
#pragma unroll
        for (int w = 0; w < OR_THREADS / 32; ++w) s += part[buf][w];
        const double f = tau * s;
#pragma unroll
        for (int r = 0; r < OR_PER; ++r) {
            const int i = tid + r * OR_THREADS;
            if (i > k && i < N) z[r] -= f * v[i];
        }
    }
#pragma unroll
    for (int r = 0; r < OR_PER; ++r) {
        const int i = tid + r * OR_THREADS;
        if (i < N) evecs[int64_t(i) * m + j] = z[r];
    }
}

// ---------------------------------------------------------------- k-means
struct KmWs {
    double *X, *xsq, *closest, *cum, *dcand;  // X: centred copy [N][k]
    int* labels_old;
};

constexpr int KM_THREADS = 512;

// sklearn E-step distance ||c||^2 - 2 x.c  (the ||x||^2 term does not change the arg-min); first minimum wins
__device__ __forceinline__ int nearest(const double* __restrict__ x, const double* C, const double* cc, int k) {
    int best = 0;
    double bd = 0.0;
    for (int c = 0; c < k; ++c) {
        double dot = 0.0;
        for (int f = 0; f < k; ++f) dot = fma(x[f], C[c * k + f], dot);
        const double dist = cc[c] - 2.0 * dot;
        if (c == 0 || dist < bd) {
            bd = dist;
            best = c;
        }
    }
    return best;
}

// sklearn _euclidean_distances(c, x, Y_norm_squared=||x||^2, squared=True): max(-2 x.c + ||c||^2 + ||x||^2, 0)
__device__ __forceinline__ double sqdist(const double* __restrict__ x, double xx, const double* c, double ccn, int k) {
    double dot = 0.0;
    for (int f = 0; f < k; ++f) dot = fma(c[f], x[f], dot);
    return fmax(-2.0 * dot + ccn + xx, 0.0);
}

__global__ void __launch_bounds__(KM_THREADS) kmeans_kernel(const double* __restrict__ Xin, int ld, int N, int k, const double* __restrict__ u,
                                                            int max_iter, int32_t* __restrict__ labels, double* __restrict__ inertia, KmWs ws) {
    __shared__ double C[CL_MAX_K * CL_MAX_K], Cn[CL_MAX_K * CL_MAX_K], cc[CL_MAX_K], wgt[CL_MAX_K], mean[CL_MAX_K];
    __shared__ double red[32];
    __shared__ double cpot[CL_MAX_TRIALS];
    __shared__ int cand[CL_MAX_TRIALS];
    __shared__ double sh_tol, sh_pot;
    __shared__ int sh_best;
    __shared__ int taken[CL_MAX_K];  // points already moved into an empty cluster in this iteration
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    double* X = ws.X;
    // centre X (KMeans.fit subtracts the column means) and the tolerance 1e-4 * mean(var(X, axis=0)) of the uncentred data
    if (tid < k) {
        double s = 0.0;
        for (int i = 0; i < N; ++i) s += Xin[int64_t(i) * ld + tid];
        const double mu = s / double(N);
        double v = 0.0;
        for (int i = 0; i < N; ++i) {
            const double t = Xin[int64_t(i) * ld + tid] - mu;
            v += t * t;
        }
        mean[tid] = mu;
        cc[tid] = v / double(N);
    }
    __syncthreads();
    if (tid == 0) {
        double s = 0.0;
        for (int f = 0; f < k; ++f) s += cc[f];
        sh_tol = s / double(k) * 1e-4;
    }
    for (int i = tid; i < N; i += KM_THREADS) {
        double s = 0.0;
        for (int f = 0; f < k; ++f) {
            const double t = Xin[int64_t(i) * ld + f] - mean[f];
            X[int64_t(i) * k + f] = t;
            s += t * t;
        }
        ws.xsq[i] = s;
        ws.labels_old[i] = -1;
    }
    __syncthreads();

    // ---- k-means++ (sklearn _kmeans_plusplus) ----
    const int n_trials = 2 + int(log(double(k)));
    if (tid == 0) {  // random_state.choice(N, p=1/N): searchsorted(cumsum(p) / cumsum(p)[-1], u, side="right")
        const double p = 1.0 / double(N);
        double s = 0.0;
        for (int i = 0; i < N; ++i) {
            s += p;
            ws.cum[i] = s;
        }
        const double last = ws.cum[N - 1];
        int id = N;
        for (int i = 0; i < N; ++i)
            if (ws.cum[i] / last > u[0]) {
                id = i;
                break;
            }
        sh_best = min(id, N - 1);
    }
    __syncthreads();
    {
        const int c0 = sh_best;
        if (tid < k) C[tid] = X[int64_t(c0) * k + tid];
        __syncthreads();
        double ccn = 0.0;
        for (int f = 0; f < k; ++f) ccn += C[f] * C[f];
        double s = 0.0;
        for (int i = tid; i < N; i += KM_THREADS) {
            const double dd = sqdist(X + int64_t(i) * k, ws.xsq[i], C, ccn, k);
            ws.closest[i] = dd;
        }
        __syncthreads();
        for (int i = tid; i < N; i += KM_THREADS) s += ws.closest[i];
        const double pot = block_sum(s, red);
        if (tid == 0) sh_pot = pot;
        __syncthreads();
    }
    for (int c = 1; c < k; ++c) {
        if (tid == 0) {
            double s = 0.0;
            for (int i = 0; i < N; ++i) {
                s += ws.closest[i];
                ws.cum[i] = s;
            }
            for (int t = 0; t < n_trials; ++t) {  // searchsorted (side="left"), clipped to N - 1
                const double val = u[1 + (c - 1) * n_trials + t] * sh_pot;
                int lo = 0, hi = N;
                while (lo < hi) {
                    const int mid = (lo + hi) >> 1;
                    if (ws.cum[mid] < val) lo = mid + 1;
                    else hi = mid;
                }
                cand[t] = min(lo, N - 1);
            }
        }
        __syncthreads();
        for (int t = 0; t < n_trials; ++t) {
            const double* xc = X + int64_t(cand[t]) * k;
            double ccn = 0.0;
            for (int f = 0; f < k; ++f) ccn += xc[f] * xc[f];
            double s = 0.0;
            for (int i = tid; i < N; i += KM_THREADS) {
                const double dd = fmin(ws.closest[i], sqdist(X + int64_t(i) * k, ws.xsq[i], xc, ccn, k));
                ws.dcand[int64_t(t) * N + i] = dd;
                s += dd;
            }
            const double pot = block_sum(s, red);
            if (tid == 0) cpot[t] = pot;
        }
        __syncthreads();
        if (tid == 0) {
            int b = 0;
            for (int t = 1; t < n_trials; ++t)
                if (cpot[t] < cpot[b]) b = t;
            sh_best = b;
            sh_pot = cpot[b];
        }
        __syncthreads();
        const int b = sh_best;
        for (int i = tid; i < N; i += KM_THREADS) ws.closest[i] = ws.dcand[int64_t(b) * N + i];
        if (tid < k) C[c * k + tid] = X[int64_t(cand[b]) * k + tid];
        __syncthreads();
    }

    // ---- Lloyd (sklearn _kmeans_single_lloyd) ----
    bool strict = false;
    const int npair = k * (k + 1);  // (cluster, feature) sums and, at feature k, the cluster weight
    for (int iter = 0; iter < max_iter; ++iter) {
        if (tid < k) {
            double s = 0.0;
            for (int f = 0; f < k; ++f) s += C[tid * k + f] * C[tid * k + f];
            cc[tid] = s;
        }
        __syncthreads();
        int changed = 0;
        for (int i = tid; i < N; i += KM_THREADS) {
            const int l = nearest(X + int64_t(i) * k, C, cc, k);
            labels[i] = l;
            changed |= l != ws.labels_old[i];
        }
        changed = __syncthreads_or(changed);
        for (int pr = warp; pr < npair; pr += KM_THREADS / 32) {
            const int c = pr / (k + 1), f = pr % (k + 1);
            double s = 0.0;
            for (int i = lane; i < N; i += 32)
                if (labels[i] == c) s += f < k ? X[int64_t(i) * k + f] : 1.0;
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
            if (lane == 0) {
                if (f < k) Cn[c * k + f] = s;
                else wgt[c] = s;
            }
        }
        __syncthreads();
        if (tid == 0) {
            // _relocate_empty_clusters_dense: an empty cluster takes the point farthest from its (old) centre; several empty
            // clusters take the farthest points in decreasing distance, ties to the lower index
            int ntaken = 0;
            for (int c = 0; c < k; ++c) {
                if (wgt[c] != 0.0) continue;
                int far = -1;
                double fd = -1.0;
                for (int i = 0; i < N; ++i) {
                    bool used = false;
                    for (int t = 0; t < ntaken; ++t) used |= taken[t] == i;
                    if (used) continue;
                    const int l = labels[i];
                    double dd = 0.0;
                    for (int f = 0; f < k; ++f) {
                        const double t = X[int64_t(i) * k + f] - C[l * k + f];
                        dd += t * t;
                    }
                    if (dd > fd) {
                        fd = dd;
                        far = i;
                    }
                }
                const int old = labels[far];
                for (int f = 0; f < k; ++f) {
                    Cn[old * k + f] -= X[int64_t(far) * k + f];
                    Cn[c * k + f] = X[int64_t(far) * k + f];
                }
                wgt[c] = 1.0;
                wgt[old] -= 1.0;
                taken[ntaken++] = far;
            }
            double tot = 0.0;
            for (int c = 0; c < k; ++c) {
                if (wgt[c] > 0.0) {
                    const double a = 1.0 / wgt[c];
                    for (int f = 0; f < k; ++f) Cn[c * k + f] *= a;
                }
                double s = 0.0;
                for (int f = 0; f < k; ++f) {
                    const double t = Cn[c * k + f] - C[c * k + f];
                    s += t * t;
                }
                const double sh = sqrt(s);
                tot += sh * sh;
            }
            red[0] = tot;
        }
        __syncthreads();
        const double tot = red[0];
        for (int q = tid; q < k * k; q += KM_THREADS) C[q] = Cn[q];
        __syncthreads();
        if (!changed) {
            strict = true;
            break;
        }
        if (tot <= sh_tol) break;
        for (int i = tid; i < N; i += KM_THREADS) ws.labels_old[i] = labels[i];
        __syncthreads();
    }
    if (!strict) {  // the final E-step: labels of the final centres
        if (tid < k) {
            double s = 0.0;
            for (int f = 0; f < k; ++f) s += C[tid * k + f] * C[tid * k + f];
            cc[tid] = s;
        }
        __syncthreads();
        for (int i = tid; i < N; i += KM_THREADS) labels[i] = nearest(X + int64_t(i) * k, C, cc, k);
        __syncthreads();
    }
    double s = 0.0;
    for (int i = tid; i < N; i += KM_THREADS) {
        const int l = labels[i];
        double dd = 0.0;
        for (int f = 0; f < k; ++f) {
            const double t = X[int64_t(i) * k + f] - C[l * k + f];
            dd += t * t;
        }
        s += dd;
    }
    const double in = block_sum(s, red);
    if (tid == 0) *inertia = in;
}

void carve_eig(WsCarver& cv, int N, int m, EigWs* w) {
    auto vec = [&] { return static_cast<double*>(cv.take(size_t(N) * 8)); };
    w->d = vec();
    w->e = vec();
    w->e2 = vec();
    w->tau = vec();
    w->p = vec();
    w->w = vec();
    w->scal = static_cast<double*>(cv.take(8 * 8));
    w->u0 = vec();
    w->u1 = vec();
    w->u2 = vec();
    w->mult = vec();
    w->x = vec();
    w->piv = static_cast<int*>(cv.take(size_t(N) * 4));
    w->Z = static_cast<double*>(cv.take(size_t(N) * m * 8));
}

void carve_km(WsCarver& cv, int N, int k, KmWs* w) {
    w->X = static_cast<double*>(cv.take(size_t(N) * k * 8));
    w->xsq = static_cast<double*>(cv.take(size_t(N) * 8));
    w->closest = static_cast<double*>(cv.take(size_t(N) * 8));
    w->cum = static_cast<double*>(cv.take(size_t(N) * 8));
    w->dcand = static_cast<double*>(cv.take(size_t(N) * CL_MAX_TRIALS * 8));
    w->labels_old = static_cast<int*>(cv.take(size_t(N) * 4));
}

int check_n(int N, const char* what) {
    if (N < 1 || N > CL_MAX_N)
        return fail(PPV_EINVAL, std::string(what) + ": N = " + std::to_string(N) + " windows; speaker diarization supports 1 <= N <= " +
                                    std::to_string(CL_MAX_N) + " (about 1.7 h of speech at the 0.75 s window shift)");
    return PPV_OK;
}

}  // namespace

int cluster_prune(float* A, int N, double pval, cudaStream_t st) {
    if (int rc = check_n(N, "ppv_cluster_prune")) return rc;
    PPV_REQUIRE(A && pval >= 0.0 && pval <= 1.0, "ppv_cluster_prune: null matrix or pval outside [0, 1]");
    if (double(N) * pval < 6.0) pval = 6.0 / double(N);  // speaker_diarization.py:261-264
    const int n_elems = int((1.0 - pval) * double(N));
    if (n_elems <= 0) return PPV_OK;
    prune_kernel<<<N, 256, size_t(N) * 4, st>>>(A, N, n_elems);
    PPV_LAUNCH_OK("prune_kernel");
    return PPV_OK;
}

int cluster_laplacian(const float* P, int N, double* L, cudaStream_t st) {
    if (int rc = check_n(N, "ppv_cluster_laplacian")) return rc;
    PPV_REQUIRE(P && L, "ppv_cluster_laplacian: null argument");
    laplacian_kernel<<<N, 256, 0, st>>>(P, N, L);
    PPV_LAUNCH_OK("laplacian_kernel");
    return PPV_OK;
}

size_t sym_eig_workspace_bytes(int N, int m) {
    if (N < 1 || m < 1) return 0;
    return carve_extent([&](WsCarver& cv) { EigWs w; carve_eig(cv, N, m, &w); });
}

int sym_eig_smallest(double* L, int N, int m, double* evals, double* evecs, void* ws, size_t ws_bytes, cudaStream_t st) {
    if (int rc = check_n(N, "ppv_sym_eig_smallest")) return rc;
    PPV_REQUIRE(L && evals && evecs, "ppv_sym_eig_smallest: null argument");
    PPV_REQUIRE(m >= 1 && m <= std::min(N, CL_MAX_K), "ppv_sym_eig_smallest: need 1 <= m <= min(N, 32)");
    if (int rc = check_workspace("ppv_sym_eig_smallest", ws, ws_bytes, sym_eig_workspace_bytes(N, m), "ppv_sym_eig_workspace_bytes")) return rc;
    WsCarver cv{static_cast<uint8_t*>(ws)};
    EigWs w;
    carve_eig(cv, N, m, &w);
    for (int k = 0; k < N; ++k) {
        house_kernel<<<1, 1024, 0, st>>>(L, N, k, w);
        if (k < N - 1) trail_update_symv_kernel<<<(N - k - 1 + TR_ROWS - 1) / TR_ROWS, 256, 0, st>>>(L, N, k, w);
    }
    PPV_LAUNCH_OK("sytrd");
    if (N == 1) PPV_CUDA_OK(cudaMemsetAsync(w.tau, 0, 8, st));
    tridiag_prep_kernel<<<1, 1024, 0, st>>>(N, w);
    stebz_kernel<<<(m + 3) / 4, 128, 0, st>>>(N, m, w, evals);
    stein_kernel<<<1, 256, 0, st>>>(N, m, w, evals);
    ormtr_kernel<<<m, OR_THREADS, 0, st>>>(L, N, m, w, evecs);
    PPV_LAUNCH_OK("stebz / stein / ormtr");
    return PPV_OK;
}

size_t kmeans_workspace_bytes(int N, int k) {
    if (N < 1 || k < 1) return 0;
    return carve_extent([&](WsCarver& cv) { KmWs w; carve_km(cv, N, k, &w); });
}

int kmeans(const double* X, int ld, int N, int k, const double* uniforms, int n_uniforms, int max_iter, int32_t* labels, double* inertia, void* ws,
           size_t ws_bytes, cudaStream_t st) {
    if (int rc = check_n(N, "ppv_kmeans")) return rc;
    PPV_REQUIRE(X && uniforms && labels && inertia, "ppv_kmeans: null argument");
    PPV_REQUIRE(k >= 1 && k <= std::min(N, CL_MAX_K) && ld >= k && max_iter >= 1, "ppv_kmeans: need 1 <= k <= min(N, 32), ld >= k, max_iter >= 1");
    const int n_trials = 2 + int(log(double(k)));
    PPV_REQUIRE(n_uniforms >= 1 + (k - 1) * n_trials, "ppv_kmeans: need 1 + (k - 1) * (2 + int(log k)) uniforms");
    if (int rc = check_workspace("ppv_kmeans", ws, ws_bytes, kmeans_workspace_bytes(N, k), "ppv_kmeans_workspace_bytes")) return rc;
    WsCarver cv{static_cast<uint8_t*>(ws)};
    KmWs w;
    carve_km(cv, N, k, &w);
    kmeans_kernel<<<1, KM_THREADS, 0, st>>>(X, ld, N, k, uniforms, max_iter, labels, inertia, w);
    PPV_LAUNCH_OK("kmeans_kernel");
    return PPV_OK;
}

}  // namespace ppv
