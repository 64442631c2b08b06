// Speaker index: per-user mean embeddings of an enrolment database, and a fused cosine top-k search over them.
// Reference: ppvector/predict.py:154-163 (per-user means in __load_audio_db), :173-187 (__retrieval: sklearn cosine_similarity + argmax),
// :285-322 / :344-364 (register / remove_user update the means).
//   build : E [n, D] rows grouped by user (CSR order / offsets) -> means [U, D] fp32, summed in enrolment order (numpy's
//           a[idx].mean(axis=0), bit for bit), and the L2-normalised means as split-bf16 planes [2][Up][Dp], Up = U rounded up to 64.
//   search: queries [Q, D] -> the k best users per query.  Each CTA keeps a 64-query block resident in shared memory and streams its
//           split of the index through a TMA / mbarrier ring; one warpgroup runs the split-bf16 products on the tensor cores
//           (hi.hi + lo.hi + hi.lo, as PPV_PREC_BF16X3) and keeps a per-query top-k in registers, so the [Q, U] score matrix is never
//           written.  A second kernel merges the per-split candidates in split order.
#include <climits>
#include <cstring>

#include "common.h"
#include "normalize_rows.cuh"
#include "ptx.cuh"

namespace ppv {

namespace {

constexpr int SI_ROWS = 64;                 // index rows per ring tile, query rows per CTA
constexpr int SI_CHUNK = SI_ROWS * 64 * 2;  // one TMA box: 64 rows x 64 bf16 (128 B, SWIZZLE_128B)
constexpr int SI_MAX_STAGES = 4;
constexpr int SI_SMEM_MAX = 227 * 1024;
constexpr int SI_THREADS = 160;  // warps 0-3: MMA + top-k warpgroup, warp 4: TMA producer
constexpr int SI_MAX_D = 256;
constexpr int SI_MAX_K = 8;

inline int padded_dim(int D) { return int(align_up(size_t(D), 64)); }
inline int64_t padded_users(int U) { return int64_t(align_up(size_t(U), SI_ROWS)); }

Planes index_planes(void* base, int U, int D) {
    Planes p;
    p.base = static_cast<__nv_bfloat16*>(base);
    p.rows = padded_users(U);
    p.ld = padded_dim(D);
    p.plane_stride = p.rows * p.ld;
    return p;
}

// Total order of candidates: higher similarity first, equal similarities lowest index first (numpy.argmax's first maximum).
__device__ __forceinline__ bool better(float v, int i, float w, int j) { return v > w || (v == w && i < j); }

// Sorted top-K list in registers; insertion of one candidate (no-op unless it beats the current K-th).
template <int K>
__device__ __forceinline__ void topk_insert(float (&val)[K], int (&idx)[K], float v, int i) {
    if (!better(v, i, val[K - 1], idx[K - 1])) return;
    val[K - 1] = v;
    idx[K - 1] = i;
#pragma unroll
    for (int j = K - 1; j > 0; --j) {
        if (better(val[j], idx[j], val[j - 1], idx[j - 1])) {
            const float tv = val[j];
            val[j] = val[j - 1];
            val[j - 1] = tv;
            const int ti = idx[j];
            idx[j] = idx[j - 1];
            idx[j - 1] = ti;
        }
    }
}

// Merge the sorted lists of the lanes in `width`-lane groups (xor masks < width): round r takes the best head of the group and
// its owner pops it.  Every lane of the group ends with the merged list in out_val / out_idx.
template <int K, int WIDTH>
__device__ __forceinline__ void topk_merge_lanes(float (&val)[K], int (&idx)[K], float (&ov)[K], int (&oi)[K]) {
#pragma unroll
    for (int r = 0; r < K; ++r) {
        float bv = val[0];
        int bi = idx[0];
#pragma unroll
        for (int o = 1; o < WIDTH; o <<= 1) {
            const float v = __shfl_xor_sync(0xffffffffu, bv, o);
            const int i = __shfl_xor_sync(0xffffffffu, bi, o);
            if (better(v, i, bv, bi)) {
                bv = v;
                bi = i;
            }
        }
        ov[r] = bv;
        oi[r] = bi;
        if (idx[0] == bi && val[0] == bv) {  // indices are distinct across lanes: only the owner pops
#pragma unroll
            for (int j = 0; j < K - 1; ++j) {
                val[j] = val[j + 1];
                idx[j] = idx[j + 1];
            }
            val[K - 1] = -INFINITY;
            idx[K - 1] = INT_MAX;
        }
    }
}

// ---------------------------------------------------------------- build
// One warp per padded user row.  User u's rows are E[order[offsets[u] .. offsets[u+1])], summed in that order starting from the
// first row (as numpy's add.reduce over axis 0 does), then divided by the count with IEEE division.
__global__ void __launch_bounds__(256) speaker_index_build_kernel(const float* __restrict__ E, int D, const int32_t* __restrict__ order,
                                                                  const int32_t* __restrict__ offsets, int U, float* __restrict__ means,
                                                                  Planes out) {
    const int u = blockIdx.x * 8 + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    if (u >= out.rows) return;
    if (u >= U) {  // padding rows of the last tile: zero, so that they score 0 (they are masked in the search as well)
        for (int i = lane; i < out.ld; i += 32) {
            out.hi()[int64_t(u) * out.ld + i] = __float2bfloat16_rn(0.f);
            out.lo()[int64_t(u) * out.ld + i] = __float2bfloat16_rn(0.f);
        }
        return;
    }
    const int beg = offsets[u], end = offsets[u + 1];
    float acc[SI_MAX_D / 32];
    {
        const float* x = E + int64_t(order[beg]) * D;
#pragma unroll
        for (int c = 0; c < SI_MAX_D / 32; ++c) acc[c] = (lane + 32 * c < D) ? x[lane + 32 * c] : 0.f;
    }
    for (int j = beg + 1; j < end; ++j) {
        const float* x = E + int64_t(order[j]) * D;
#pragma unroll
        for (int c = 0; c < SI_MAX_D / 32; ++c)
            if (lane + 32 * c < D) acc[c] = __fadd_rn(acc[c], x[lane + 32 * c]);
    }
    const float cnt = float(end - beg);
    float* m = means + int64_t(u) * D;
#pragma unroll
    for (int c = 0; c < SI_MAX_D / 32; ++c)
        if (lane + 32 * c < D) m[lane + 32 * c] = __fdiv_rn(acc[c], cnt);
    __syncwarp();
    normalize_row_to_planes(m, D, out, u, lane);
}

// ---------------------------------------------------------------- search
struct SearchParams {
    CUtensorMap mapQ;  // query planes [2][Qp][Dp], box {64, 64, 1}, SWIZZLE_128B
    CUtensorMap mapX;  // index planes [2][Up][Dp], same box
    int Q, U, nchunks, ntiles, splits, stages;
    float* cand_val;  // [Q][splits][KMAX]
    int32_t* cand_idx;
};

struct SearchPlan {
    int Dp, nchunks, qblocks, ntiles, splits, stages;
    size_t q_bytes, tile_bytes, smem;
};

SearchPlan plan_search(int Q, int U, int D, int kmax, int num_sms) {
    SearchPlan p;
    p.Dp = padded_dim(D);
    p.nchunks = p.Dp / 64;
    p.qblocks = (Q + SI_ROWS - 1) / SI_ROWS;
    p.ntiles = int(padded_users(U) / SI_ROWS);
    p.q_bytes = size_t(2) * p.nchunks * SI_CHUNK;
    p.tile_bytes = p.q_bytes;
    // The one consumer takes the tiles in order, so a slot's previous fill has always completed before the consumer waits on it again
    // (a parity wait cannot tell fill n from fill n + 2).  Dp = 256: 2 stages, 192: 3, <= 128: 4.
    const size_t room = SI_SMEM_MAX - 1024 - 256 - p.q_bytes;
    p.stages = int(std::min<size_t>(SI_MAX_STAGES, room / p.tile_bytes));
    p.smem = 1024 + p.q_bytes + size_t(p.stages) * p.tile_bytes + 256;
    // Splits of the index: the fewest tile-times on the busiest SM, counting one CTA's set-up (query block load, drain, candidate
    // store) as about two tiles.  One CTA per SM fits (shared memory).
    int best = 1;
    double best_cost = 1e300;
    const int max_splits = std::max(1, std::min(p.ntiles, std::min(1024, (16 * num_sms + p.qblocks - 1) / p.qblocks)));
    for (int s = 1; s <= max_splits; ++s) {
        const double waves = double((int64_t(p.qblocks) * s + num_sms - 1) / num_sms);
        const double cost = waves * ((p.ntiles + s - 1) / s + 2.0);
        if (cost < best_cost) {
            best_cost = cost;
            best = s;
        }
    }
    p.splits = best;
    return p;
}

// The search workspace: the normalised queries as split-bf16 planes [2][qblocks * 64][Dp], then the per-split candidates
// [Q][splits][kmax] (similarities, then indices).
struct SearchWs {
    Planes q;
    float* cand_val;
    int32_t* cand_idx;
};
void carve_search(WsCarver& cv, const SearchPlan& pl, int Q, int kmax, SearchWs* w) {
    const int64_t rows = int64_t(pl.qblocks) * SI_ROWS;
    w->q = Planes{static_cast<__nv_bfloat16*>(cv.take(size_t(2 * rows * pl.Dp) * sizeof(__nv_bfloat16))), rows, pl.Dp, rows * pl.Dp};
    const size_t cand = size_t(Q) * pl.splits * kmax;
    w->cand_val = static_cast<float*>(cv.take(cand * sizeof(float)));
    w->cand_idx = static_cast<int32_t*>(cv.take(cand * sizeof(int32_t)));
}

// The three split-bf16 products of one 64 x 64 tile over the whole (padded) D: A = query block, B = index tile.
__device__ __forceinline__ void tile_mma(float (&acc)[32], uint32_t q_smem, uint32_t x_smem, int nchunks) {
    wgmma_fence();
    uint32_t scale_d = 0;
    for (int c = 0; c < nchunks; ++c) {
        const uint64_t qh = make_sw128_kmajor_desc(q_smem + c * SI_CHUNK);
        const uint64_t ql = make_sw128_kmajor_desc(q_smem + (nchunks + c) * SI_CHUNK);
        const uint64_t xh = make_sw128_kmajor_desc(x_smem + c * SI_CHUNK);
        const uint64_t xl = make_sw128_kmajor_desc(x_smem + (nchunks + c) * SI_CHUNK);
#pragma unroll
        for (int k = 0; k < 4; ++k) {  // +32 B (16 bf16) along K inside the swizzle atom = +2 in the descriptor
            wgmma_m64n64k16(acc, qh + 2 * k, xh + 2 * k, scale_d);
            scale_d = 1;
            wgmma_m64n64k16(acc, ql + 2 * k, xh + 2 * k, 1);
            wgmma_m64n64k16(acc, qh + 2 * k, xl + 2 * k, 1);
        }
    }
    wgmma_commit();
}

// Fold one tile's accumulator (rows r0 = 16 w + l / 4 and r0 + 8, columns 8 i + 2 (l % 4) + {0, 1}) into the two rows' lists.
template <int K>
__device__ __forceinline__ void tile_topk(const float (&acc)[32], int u0, int U, int lane, float (&v0)[K], int (&i0)[K], float (&v1)[K],
                                          int (&i1)[K]) {
#pragma unroll
    for (int i = 0; i < 8; ++i) {
#pragma unroll
        for (int e = 0; e < 2; ++e) {
            const int u = u0 + 8 * i + 2 * (lane & 3) + e;
            if (u < U) {
                topk_insert<K>(v0, i0, acc[4 * i + e], u);
                topk_insert<K>(v1, i1, acc[4 * i + 2 + e], u);
            }
        }
    }
}

template <int K>
__global__ void __launch_bounds__(SI_THREADS, 1) speaker_index_search_kernel(const __grid_constant__ SearchParams p) {
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    const int tile_bytes = 2 * p.nchunks * SI_CHUNK;
    const uint32_t q_smem = smem_u32(smem);
    const uint32_t ring = q_smem + tile_bytes;
    uint64_t* bars = reinterpret_cast<uint64_t*>(smem + size_t(tile_bytes) * (1 + p.stages));
    const uint32_t q_bar = smem_u32(bars);
    auto full_bar = [&](int s) { return smem_u32(bars + 1 + s); };
    auto empty_bar = [&](int s) { return smem_u32(bars + 1 + SI_MAX_STAGES + s); };

    const int qb = blockIdx.x, split = blockIdx.y;
    const int t_beg = int(int64_t(split) * p.ntiles / p.splits);
    const int t_end = int(int64_t(split + 1) * p.ntiles / p.splits);
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    if (threadIdx.x == 0) {
        mbar_init(q_bar, 1);
        for (int s = 0; s < p.stages; ++s) {
            mbar_init(full_bar(s), 1);
            mbar_init(empty_bar(s), 4);  // one arrival per consumer warp
        }
        fence_mbar_init();
    }
    __syncthreads();

    if (warp == 4) {
        // ===================== TMA producer =====================
        if (lane == 0) {
            prefetch_tmap(&p.mapQ);
            prefetch_tmap(&p.mapX);
            mbar_arrive_expect_tx(q_bar, tile_bytes);
            for (int pl = 0; pl < 2; ++pl)
                for (int c = 0; c < p.nchunks; ++c) tma_load_3d(q_smem + (pl * p.nchunks + c) * SI_CHUNK, &p.mapQ, q_bar, 64 * c, SI_ROWS * qb, pl);
            for (int t = t_beg; t < t_end; ++t) {
                const int n = t - t_beg, s = n % p.stages, use = n / p.stages;
                if (use > 0) mbar_wait(empty_bar(s), (use - 1) & 1);
                const uint32_t dst = ring + s * tile_bytes;
                mbar_arrive_expect_tx(full_bar(s), tile_bytes);
                for (int pl = 0; pl < 2; ++pl)
                    for (int c = 0; c < p.nchunks; ++c) tma_load_3d(dst + (pl * p.nchunks + c) * SI_CHUNK, &p.mapX, full_bar(s), 64 * c, SI_ROWS * t, pl);
            }
        }
        return;
    }

    // ===================== MMA + top-k warpgroup =====================
    // The top-k fold reads the accumulator in data-dependent branches, so it runs after the tile's MMAs have completed (a wgmma in flight
    // across a divergent path makes ptxas serialise every wgmma of the kernel); the producer keeps the next tiles loading meanwhile.
    float v0[K], v1[K];
    int i0[K], i1[K];
#pragma unroll
    for (int j = 0; j < K; ++j) {
        v0[j] = v1[j] = -INFINITY;
        i0[j] = i1[j] = INT_MAX;
    }
    float acc[32];
    mbar_wait(q_bar, 0);
    for (int n = 0; n < t_end - t_beg; ++n) {
        const int s = n % p.stages;
        mbar_wait(full_bar(s), (n / p.stages) & 1);
        tile_mma(acc, q_smem, ring + s * tile_bytes, p.nchunks);
        wgmma_wait<0>();
        wgmma_fence_acc(acc);
        if (lane == 0) mbar_arrive(empty_bar(s));
        tile_topk<K>(acc, SI_ROWS * (t_beg + n), p.U, lane, v0, i0, v1, i1);
    }
    // the four lanes of a quad hold disjoint column sets of the same two rows: merge them, lane 0 of the quad stores
    float m_v[K];
    int m_i[K];
    const int r0 = SI_ROWS * qb + 16 * warp + (lane >> 2);
#pragma unroll
    for (int h = 0; h < 2; ++h) {
        if (h == 0) topk_merge_lanes<K, 4>(v0, i0, m_v, m_i);
        else topk_merge_lanes<K, 4>(v1, i1, m_v, m_i);
        const int q = r0 + 8 * h;
        if ((lane & 3) == 0 && q < p.Q) {
            const int64_t o = (int64_t(q) * p.splits + split) * K;
#pragma unroll
            for (int j = 0; j < K; ++j) {
                p.cand_val[o + j] = m_v[j];
                p.cand_idx[o + j] = m_i[j];
            }
        }
    }
}

// One warp per query: each lane folds splits lane, lane + 32, ... into its list, then the warp merges the 32 lists.
template <int K>
__global__ void __launch_bounds__(256) speaker_index_merge_kernel(const float* __restrict__ cand_val, const int32_t* __restrict__ cand_idx,
                                                                  int Q, int splits, int k, int32_t* __restrict__ out_idx,
                                                                  float* __restrict__ out_sim) {
    const int q = blockIdx.x * 8 + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    if (q >= Q) return;
    float v[K];
    int ix[K];
#pragma unroll
    for (int j = 0; j < K; ++j) {
        v[j] = -INFINITY;
        ix[j] = INT_MAX;
    }
    for (int s = lane; s < splits; s += 32) {
        const int64_t o = (int64_t(q) * splits + s) * K;
#pragma unroll
        for (int j = 0; j < K; ++j) topk_insert<K>(v, ix, cand_val[o + j], cand_idx[o + j]);
    }
    float mv[K];
    int mi[K];
    topk_merge_lanes<K, 32>(v, ix, mv, mi);
    if (lane == 0) {
#pragma unroll
        for (int j = 0; j < K; ++j)
            if (j < k) {
                out_idx[int64_t(q) * k + j] = mi[j];
                out_sim[int64_t(q) * k + j] = mv[j];
            }
    }
}

template <int K>
int search_launch(const float* queries, int Q, int D, const void* index, int U, int k, int32_t* idx, float* sim, void* ws, cudaStream_t st) {
    const SearchPlan pl = plan_search(Q, U, D, K, device_sm_count());
    WsCarver cv{static_cast<uint8_t*>(ws)};
    SearchWs w;
    carve_search(cv, pl, Q, K, &w);
    SearchParams p;
    memset(&p, 0, sizeof(p));
    int rc = encode_planes_map_ex(&p.mapQ, w.q, 64, SI_ROWS, 128);
    if (rc) return rc;
    rc = encode_planes_map_ex(&p.mapX, index_planes(const_cast<void*>(index), U, D), 64, SI_ROWS, 128);
    if (rc) return rc;
    p.Q = Q;
    p.U = U;
    p.nchunks = pl.nchunks;
    p.ntiles = pl.ntiles;
    p.splits = pl.splits;
    p.stages = pl.stages;
    p.cand_val = w.cand_val;
    p.cand_idx = w.cand_idx;
    // query rows past Q feed only rows that are never stored; keep them zero all the same
    if (w.q.rows > Q) {
        PPV_CUDA_OK(cudaMemsetAsync(w.q.hi() + int64_t(Q) * w.q.ld, 0, size_t(w.q.rows - Q) * w.q.ld * sizeof(__nv_bfloat16), st));
        PPV_CUDA_OK(cudaMemsetAsync(w.q.lo() + int64_t(Q) * w.q.ld, 0, size_t(w.q.rows - Q) * w.q.ld * sizeof(__nv_bfloat16), st));
    }
    normalize_rows_kernel<<<(Q + 7) / 8, 256, 0, st>>>(queries, Q, D, w.q);
    PPV_LAUNCH_OK("normalize_rows_kernel(queries)");
    PPV_ONCE_PER_DEVICE(PPV_CUDA_OK(cudaFuncSetAttribute(speaker_index_search_kernel<K>, cudaFuncAttributeMaxDynamicSharedMemorySize, SI_SMEM_MAX)));
    speaker_index_search_kernel<K><<<dim3(pl.qblocks, pl.splits), SI_THREADS, pl.smem, st>>>(p);
    PPV_LAUNCH_OK("speaker_index_search_kernel");
    speaker_index_merge_kernel<K><<<(Q + 7) / 8, 256, 0, st>>>(w.cand_val, w.cand_idx, Q, pl.splits, k, idx, sim);
    PPV_LAUNCH_OK("speaker_index_merge_kernel");
    return PPV_OK;
}

int check_search_shape(int Q, int U, int D, int k) {
    PPV_REQUIRE(Q >= 1, "speaker_index_search: Q must be >= 1 (got " + std::to_string(Q) + ")");
    PPV_REQUIRE(U >= 1, "speaker_index_search: U must be >= 1 (got " + std::to_string(U) + ")");
    PPV_REQUIRE(D >= 1 && D <= SI_MAX_D, "speaker_index_search: D must be in [1, 256] (got " + std::to_string(D) + ")");
    PPV_REQUIRE(k >= 1 && k <= SI_MAX_K && k <= U,
                "speaker_index_search: k must be in [1, min(8, U)] (got k = " + std::to_string(k) + ", U = " + std::to_string(U) + ")");
    return PPV_OK;
}

}  // namespace

size_t speaker_index_bytes(int U, int D) {
    if (U < 1 || D < 1 || D > SI_MAX_D) return 0;
    return size_t(padded_users(U)) * padded_dim(D) * 2 * sizeof(__nv_bfloat16);
}

int speaker_index_build(const float* E, int n, int D, const int32_t* order, const int32_t* offsets, int U, float* means, void* index,
                        size_t index_bytes, cudaStream_t st) {
    PPV_REQUIRE(E && order && offsets && means && index, "speaker_index_build: null argument");
    PPV_REQUIRE(n >= U && U >= 1, "speaker_index_build: need 1 <= U <= n (every user has a row)");
    PPV_REQUIRE(D >= 1 && D <= SI_MAX_D, "speaker_index_build: D must be in [1, 256] (got " + std::to_string(D) + ")");
    PPV_REQUIRE(index_bytes >= speaker_index_bytes(U, D), "speaker_index_build: index buffer too small");
    PPV_REQUIRE((reinterpret_cast<uintptr_t>(index) & 255) == 0, "speaker_index_build: index must be 256-byte aligned");
    const Planes out = index_planes(index, U, D);
    speaker_index_build_kernel<<<unsigned((out.rows + 7) / 8), 256, 0, st>>>(E, D, order, offsets, U, means, out);
    PPV_LAUNCH_OK("speaker_index_build_kernel");
    return PPV_OK;
}

size_t speaker_index_search_workspace_bytes(int Q, int U, int D, int k) {
    if (Q < 1 || U < 1 || D < 1 || D > SI_MAX_D || k < 1 || k > SI_MAX_K) return 0;
    const int kmax = k == 1 ? 1 : SI_MAX_K;
    const SearchPlan pl = plan_search(Q, U, D, kmax, device_sm_count());
    return carve_extent([&](WsCarver& cv) { SearchWs w; carve_search(cv, pl, Q, kmax, &w); });
}

int speaker_index_search(const float* queries, int Q, int D, const void* index, size_t index_bytes, int U, int k, int32_t* idx, float* sim,
                         void* ws, size_t ws_bytes, cudaStream_t st) {
    int rc = check_search_shape(Q, U, D, k);
    if (rc) return rc;
    PPV_REQUIRE(queries && index && idx && sim, "speaker_index_search: null argument");
    PPV_REQUIRE(index_bytes >= speaker_index_bytes(U, D), "speaker_index_search: index buffer smaller than ppv_speaker_index_bytes(U, D)");
    PPV_REQUIRE((reinterpret_cast<uintptr_t>(index) & 255) == 0, "speaker_index_search: index must be 256-byte aligned");
    if (int rc = check_workspace("speaker_index_search", ws, ws_bytes, speaker_index_search_workspace_bytes(Q, U, D, k),
                                 "ppv_speaker_index_search_workspace_bytes")) return rc;
    return k == 1 ? search_launch<1>(queries, Q, D, index, U, k, idx, sim, ws, st) : search_launch<SI_MAX_K>(queries, Q, D, index, U, k, idx, sim, ws, st);
}

}  // namespace ppv
