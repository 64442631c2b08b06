// Batched cosine scoring (K11).
// Reference: ppvector/predict.py:279-283 (contrast: dot / (|a||b|)), predict.py:173-187 (retrieval through
// sklearn cosine_similarity), ppvector/trainer.py:416-423 (eval: one 1-vs-all-enrol cosine row per trial in a
// Python loop).  Two forms:
//   all-pairs  [M,D] x [N,D] -> [M,N] : rows are L2-normalised into split-bf16 planes, then the same wgmma
//              gather-GEMM as the model (K = D, fp32 out).  Tensor-core bound, 384 FLOP / pair.
//   pair-list  idx[P,2] -> [P]        : 8 lanes per pair, gather both rows (1536 B / pair), HBM/L2-bound.
#include "common.h"
#include "normalize_rows.cuh"
#include "ptx.cuh"

namespace ppv {

// The all-pairs workspace: the normalised rows of A and of B as split-bf16 planes [2][pad128(rows)][pad64(D)].
static void carve_cosine(WsCarver& cv, int M, int N, int D, Planes* pa, Planes* pb) {
    const int Dp = int(align_up(size_t(D), 64));
    *pa = cv.planes(M, Dp);
    *pb = cv.planes(N, Dp);
}
size_t cosine_workspace_bytes(int M, int N, int D) {
    return carve_extent([&](WsCarver& cv) { Planes pa, pb; carve_cosine(cv, M, N, D, &pa, &pb); });
}

int cosine_matrix(const float* A, const float* Bm, int M, int N, int D, float* out, void* ws, size_t ws_bytes, int precision,
                  cudaStream_t st) {
    PPV_REQUIRE(A && Bm && out, "cosine_matrix: null argument");
    PPV_REQUIRE(M > 0 && N > 0 && D > 0, "cosine_matrix: empty input");
    const size_t need = cosine_workspace_bytes(M, N, D);
    if (int rc = check_workspace("cosine_matrix", ws, ws_bytes, need, "ppv_cosine_workspace_bytes")) return rc;
    WsCarver cv{static_cast<uint8_t*>(ws)};
    Planes pa, pb;
    carve_cosine(cv, M, N, D, &pa, &pb);
    // rows beyond M / N must be finite (they only feed masked outputs, but keep them zero)
    PPV_CUDA_OK(cudaMemsetAsync(ws, 0, need, st));
    normalize_rows_kernel<<<(M + 7) / 8, 256, 0, st>>>(A, M, D, pa);
    PPV_LAUNCH_OK("normalize_rows_kernel(A)");
    normalize_rows_kernel<<<(N + 7) / 8, 256, 0, st>>>(Bm, N, D, pb);
    PPV_LAUNCH_OK("normalize_rows_kernel(B)");
    GemmSource src{pa, 0, pa.ld, 0};
    Epilogue ep;
    ep.out_mode = OUT_F32;
    ep.out = out;
    ep.out_ld = N;
    GemmParams gp;
    int rc = gemm_build(&gp, &src, 1, pb, M, N, ep, 128);
    if (rc) return rc;
    return gemm_launch(gp, precision, device_sm_count(), st);
}

// pair list: 8 lanes per pair, float4 loads
__global__ void __launch_bounds__(256)
    cosine_pairlist_kernel(const float* __restrict__ E, const int32_t* __restrict__ idx, int64_t P, int n, int D, float* __restrict__ out) {
    const int64_t gid = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
    const int64_t pair = gid >> 3;
    const int sub = int(gid & 7);
    float dot = 0.f, na = 0.f, nb = 0.f;
    const bool ok = pair < P;
    if (ok) {
        const int ia = idx[2 * pair], ib = idx[2 * pair + 1];
        if (ia >= 0 && ia < n && ib >= 0 && ib < n) {
            const float* a = E + int64_t(ia) * D;
            const float* b = E + int64_t(ib) * D;
            if ((D & 3) == 0) {
                const float4* a4 = reinterpret_cast<const float4*>(a);
                const float4* b4 = reinterpret_cast<const float4*>(b);
                for (int i = sub; i < D / 4; i += 8) {
                    const float4 x = __ldg(a4 + i), y = __ldg(b4 + i);
                    dot += x.x * y.x + x.y * y.y + x.z * y.z + x.w * y.w;
                    na += x.x * x.x + x.y * x.y + x.z * x.z + x.w * x.w;
                    nb += y.x * y.x + y.y * y.y + y.z * y.z + y.w * y.w;
                }
            } else {
                for (int i = sub; i < D; i += 8) {
                    const float x = a[i], y = b[i];
                    dot += x * y;
                    na += x * x;
                    nb += y * y;
                }
            }
        } else {
            dot = NAN;
        }
    }
#pragma unroll
    for (int o = 4; o > 0; o >>= 1) {
        dot += __shfl_xor_sync(0xffffffffu, dot, o);
        na += __shfl_xor_sync(0xffffffffu, na, o);
        nb += __shfl_xor_sync(0xffffffffu, nb, o);
    }
    if (ok && sub == 0) out[pair] = dot / (sqrtf(na) * sqrtf(nb));
}

int cosine_pairlist(const float* E, const int32_t* idx, int64_t P, int n, int D, float* out, cudaStream_t st) {
    if (P == 0) return PPV_OK;
    PPV_REQUIRE(E && idx && out, "cosine_pairlist: null argument");
    PPV_REQUIRE(P > 0 && n > 0 && D > 0, "cosine_pairlist: bad sizes");
    const int64_t threads = P * 8;
    cosine_pairlist_kernel<<<unsigned((threads + 255) / 256), 256, 0, st>>>(E, idx, P, n, D, out);
    PPV_LAUNCH_OK("cosine_pairlist_kernel");
    return PPV_OK;
}

}  // namespace ppv
