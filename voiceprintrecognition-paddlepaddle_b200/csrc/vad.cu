// Energy voice-activity detection (Kaldi's compute-vad, src/ivector/voice-activity-detection.cc) for a batch of recordings that
// arrive as one concatenated sample buffer.  The definition is DESIGN.md §1 (f8); in short, per recording:
//   e_t  = ln(max(32768^2 * sum_n (x[t*shift + n] - mean_t)^2, FLT_EPSILON))       n < win, mean_t the frame's own mean, fp64
//   thr  = energy_threshold + energy_mean_scale * (sum_t e_t) / T                 fp64
//   voiced_t = num >= den * proportion_threshold (fp32 product), over the frames t2 in [t - c, t + c] ∩ [0, T): den of them, num with
//              e_t2 > thr
// and the maximal runs of voiced frames are listed as (recording, first_frame, end_frame) triples in recording and frame order.
// Five launches, all sums in a fixed order (bitwise reproducible, independent of how recordings are batched):
//   energy   : one CTA per tile of up to VAD_TILE_FRAMES frames of one recording.  The tile's samples ((nf - 1) * shift + win of them)
//              are staged in shared memory by one 1-D bulk copy on an mbarrier, so the 2.5x frame overlap is read from HBM once; each
//              warp takes frames warp, warp + 8, ... and reduces each frame's two fp64 passes across its lanes.  Writes e_t (fp64) and
//              the tile's sum of e_t.
//   threshold: one CTA per recording reduces its tiles' sums in a fixed tree -> thr.
//   decide   : one CTA per tile: voiced_t, and the tile's counts of run starts and run ends.
//   scan     : one CTA: exclusive scan of the per-tile counts over all tiles -> each tile's first run slot, and the run count.
//   emit     : one CTA per tile writes its starts and ends into their slots (ranks from warp ballots; no atomics).
#include <float.h>
#include <math.h>

#include <cmath>

#include "common.h"
#include "ptx.cuh"

namespace ppv {

namespace {

constexpr int VAD_THREADS = 256;  // energy kernel
constexpr int VAD_WARPS = VAD_THREADS / 32;
constexpr int VAD_TILE_FRAMES = 64;
constexpr int VAD_TILE_THREADS = 128;      // decide / emit: one thread per frame of the tile, two more for its neighbours
constexpr int VAD_STAGE_FLOATS = 12288;    // 48 KB of staged samples per tile at most (41 KB at 16 kHz: 63 * 160 + 400 + 3)
constexpr int VAD_MAX_WIN = 2048;
constexpr int VAD_SCAN_THREADS = 1024;
constexpr double VAD_SCALE2 = 1073741824.0;  // 32768^2: Kaldi's energies are of 16-bit integer samples

struct VadGeom {
    const int64_t* sample_off;  // [R + 1] into the concatenated samples
    const int64_t* frame_off;   // [R + 1] into the concatenated frames
    const int64_t* tile_off;    // [R + 1] into the tiles
    int R, win, shift, tile_frames;
};

// The recording a tile belongs to: the largest r with tile_off[r] <= tile (recordings without frames own no tile).
__device__ __forceinline__ int tile_recording(const int64_t* tile_off, int R, int64_t tile) {
    int lo = 0, hi = R;
    while (hi - lo > 1) {
        const int mid = (lo + hi) >> 1;
        if (tile_off[mid] <= tile) lo = mid;
        else hi = mid;
    }
    return lo;
}

struct TileFrames {
    int r, nf;
    int64_t f0, T, base;  // first frame of the tile, frames of its recording, the recording's first frame in the concatenation
};
__device__ __forceinline__ TileFrames tile_of(const VadGeom& g) {
    TileFrames t;
    t.r = tile_recording(g.tile_off, g.R, blockIdx.x);
    t.f0 = (int64_t(blockIdx.x) - g.tile_off[t.r]) * g.tile_frames;
    t.base = g.frame_off[t.r];
    t.T = g.frame_off[t.r + 1] - t.base;
    t.nf = int(std::min<int64_t>(g.tile_frames, t.T - t.f0));
    return t;
}

__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);  // every lane ends with the same bits (a + b == b + a)
    return v;
}

__global__ void __launch_bounds__(VAD_THREADS) vad_energy_kernel(const float* __restrict__ wav, VadGeom g, double* __restrict__ energy,
                                                                 double* __restrict__ tile_sum) {
    extern __shared__ __align__(16) float s_stage[];
    __shared__ __align__(8) uint64_t s_bar;
    __shared__ double s_warp[VAD_WARPS];
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const TileFrames tf = tile_of(g);
    const int nf = tf.nf;
    const float* src = wav + g.sample_off[tf.r] + tf.f0 * g.shift;
    const int len = (nf - 1) * g.shift + g.win;
    // samples before the first 16-byte boundary (head) and after the last (tail) are plain loads; the body is one bulk copy into a
    // 16-byte aligned destination: sample i of the tile sits at stage[pad + i] with (pad + head) % 4 == 0
    const int head = min(int((16u - (reinterpret_cast<uintptr_t>(src) & 15u)) & 15u) >> 2, len);
    const int body = (len - head) & ~3;
    float* s = s_stage + ((4 - head) & 3);
    const uint32_t bar = smem_u32(&s_bar);
    if (tid == 0) {
        mbar_init(bar, 1);
        fence_mbar_init();
    }
    __syncthreads();
    if (tid == 0 && body > 0) {
        mbar_arrive_expect_tx(bar, uint32_t(body) * 4u);
        bulk_load_1d(smem_u32(s + head), src + head, uint32_t(body) * 4u, bar);
    }
    if (tid < head) s[tid] = __ldg(src + tid);
    if (tid < len - head - body) s[head + body + tid] = __ldg(src + head + body + tid);
    __syncthreads();
    if (body > 0) mbar_wait(bar, 0);

    double acc = 0.0;  // this warp's frames, in frame order
    const double inv_win = 1.0 / double(g.win);
    for (int j = warp; j < nf; j += VAD_WARPS) {
        const float* x = s + j * g.shift;
        double s1 = 0.0;
        for (int i = lane; i < g.win; i += 32) s1 += double(x[i]);
        const double mean = warp_sum(s1) * inv_win;
        double s2 = 0.0;
        for (int i = lane; i < g.win; i += 32) {
            const double d = double(x[i]) - mean;
            s2 = fma(d, d, s2);
        }
        const double e = log(fmax(warp_sum(s2) * VAD_SCALE2, double(FLT_EPSILON)));
        if (lane == 0) energy[tf.base + tf.f0 + j] = e;
        acc += e;
    }
    if (lane == 0) s_warp[warp] = acc;
    __syncthreads();
    if (tid == 0) {
        double t = 0.0;
        for (int w = 0; w < VAD_WARPS; ++w) t += s_warp[w];
        tile_sum[blockIdx.x] = t;
    }
}

__global__ void __launch_bounds__(VAD_THREADS) vad_threshold_kernel(VadGeom g, const double* __restrict__ tile_sum, float energy_threshold,
                                                                    float energy_mean_scale, double* __restrict__ thr) {
    __shared__ double s_part[VAD_THREADS];
    const int r = blockIdx.x, tid = threadIdx.x;
    const int64_t t0 = g.tile_off[r], t1 = g.tile_off[r + 1];
    const int64_t T = g.frame_off[r + 1] - g.frame_off[r];
    if (T == 0) return;
    double acc = 0.0;
    for (int64_t i = t0 + tid; i < t1; i += VAD_THREADS) acc += tile_sum[i];
    s_part[tid] = acc;
    __syncthreads();
    for (int h = VAD_THREADS / 2; h > 0; h >>= 1) {
        if (tid < h) s_part[tid] += s_part[tid + h];
        __syncthreads();
    }
    if (tid == 0) thr[r] = double(energy_threshold) + double(energy_mean_scale) * s_part[0] / double(T);
}

// Kaldi's ComputeVadEnergy decision for frame t of a recording with T frames.
__device__ __forceinline__ uint8_t voiced_at(const double* __restrict__ e, int64_t T, int64_t t, int context, double thr, float proportion) {
    const int64_t lo = std::max<int64_t>(t - context, 0), hi = std::min<int64_t>(t + context, T - 1);
    int num = 0;
    for (int64_t u = lo; u <= hi; ++u) num += e[u] > thr;
    return float(num) >= __fmul_rn(float(hi - lo + 1), proportion) ? 1 : 0;
}

__global__ void __launch_bounds__(VAD_TILE_THREADS) vad_decide_kernel(VadGeom g, const double* __restrict__ energy, const double* __restrict__ thr,
                                                                      int context, float proportion, uint8_t* __restrict__ voiced,
                                                                      int2* __restrict__ tile_count) {
    __shared__ uint8_t v[VAD_TILE_FRAMES + 2];  // v[1 + j] = voiced(f0 + j); v[0], v[nf + 1]: the neighbours, 0 past the recording's ends
    const int tid = threadIdx.x;
    const TileFrames tf = tile_of(g);
    const double th = thr[tf.r];
    const double* e = energy + tf.base;
    if (tid < tf.nf) {
        v[1 + tid] = voiced_at(e, tf.T, tf.f0 + tid, context, th, proportion);
        voiced[tf.base + tf.f0 + tid] = v[1 + tid];
    } else if (tid == VAD_TILE_THREADS - 2) {
        v[0] = tf.f0 > 0 ? voiced_at(e, tf.T, tf.f0 - 1, context, th, proportion) : 0;
    } else if (tid == VAD_TILE_THREADS - 1) {
        v[tf.nf + 1] = tf.f0 + tf.nf < tf.T ? voiced_at(e, tf.T, tf.f0 + tf.nf, context, th, proportion) : 0;
    }
    __syncthreads();
    const bool in = tid < tf.nf && v[1 + tid];
    const int starts = __syncthreads_count(in && !v[tid]);
    const int ends = __syncthreads_count(in && !v[tid + 2]);
    if (tid == 0) tile_count[blockIdx.x] = make_int2(starts, ends);
}

// Exclusive scan of the per-tile (starts, ends) over all tiles, in tile order.  Thread i takes a contiguous chunk of tiles.
__global__ void __launch_bounds__(VAD_SCAN_THREADS) vad_scan_kernel(const int2* __restrict__ tile_count, int64_t ntiles, int2* __restrict__ tile_base,
                                                                    int32_t* __restrict__ n_runs) {
    __shared__ int2 s_tot[VAD_SCAN_THREADS / 32];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int64_t per = (ntiles + VAD_SCAN_THREADS - 1) / VAD_SCAN_THREADS;
    const int64_t i0 = std::min<int64_t>(tid * per, ntiles), i1 = std::min<int64_t>(i0 + per, ntiles);
    int2 own = make_int2(0, 0);
    for (int64_t i = i0; i < i1; ++i) {
        const int2 c = tile_count[i];
        own.x += c.x;
        own.y += c.y;
    }
    int2 inc = own;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const int x = __shfl_up_sync(0xffffffffu, inc.x, o), y = __shfl_up_sync(0xffffffffu, inc.y, o);
        if (lane >= o) {
            inc.x += x;
            inc.y += y;
        }
    }
    if (lane == 31) s_tot[warp] = inc;
    __syncthreads();
    int2 run = make_int2(inc.x - own.x, inc.y - own.y);
    for (int w = 0; w < warp; ++w) {
        run.x += s_tot[w].x;
        run.y += s_tot[w].y;
    }
    for (int64_t i = i0; i < i1; ++i) {
        tile_base[i] = run;
        const int2 c = tile_count[i];
        run.x += c.x;
        run.y += c.y;
    }
    if (tid == VAD_SCAN_THREADS - 1) *n_runs = run.x;
}

__global__ void __launch_bounds__(VAD_TILE_THREADS) vad_emit_kernel(VadGeom g, const uint8_t* __restrict__ voiced, const int2* __restrict__ tile_base,
                                                                    int32_t* __restrict__ runs) {
    __shared__ int s_warp_starts[VAD_TILE_THREADS / 32], s_warp_ends[VAD_TILE_THREADS / 32];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const TileFrames tf = tile_of(g);
    const uint8_t* v = voiced + tf.base;
    const int64_t t = tf.f0 + tid;
    const bool in = tid < tf.nf && v[t];
    const bool start = in && (t == 0 || !v[t - 1]);
    const bool end = in && (t + 1 == tf.T || !v[t + 1]);
    const uint32_t bs = __ballot_sync(0xffffffffu, start), be = __ballot_sync(0xffffffffu, end);
    if (lane == 0) {
        s_warp_starts[warp] = __popc(bs);
        s_warp_ends[warp] = __popc(be);
    }
    __syncthreads();
    const uint32_t below = (1u << lane) - 1u;
    int2 slot = tile_base[blockIdx.x];
    slot.x += __popc(bs & below);
    slot.y += __popc(be & below);
    for (int w = 0; w < warp; ++w) {
        slot.x += s_warp_starts[w];
        slot.y += s_warp_ends[w];
    }
    if (start) {
        runs[3 * int64_t(slot.x) + 0] = tf.r;
        runs[3 * int64_t(slot.x) + 1] = int32_t(t);
    }
    if (end) runs[3 * int64_t(slot.y) + 2] = int32_t(t + 1);
}

bool vad_cfg_ok(const ppv_vad_cfg& c, std::string* why) {
    std::string w;
    if (c.window < 1 || c.window > VAD_MAX_WIN) w = "window must be in [1, 2048] samples (got " + std::to_string(c.window) + ")";
    else if (c.shift < 1 || c.shift > c.window) w = "shift must be in [1, window] (got " + std::to_string(c.shift) + ")";
    else if (!std::isfinite(c.energy_threshold)) w = "energy_threshold must be finite";
    else if (!(c.energy_mean_scale >= 0.f) || !std::isfinite(c.energy_mean_scale)) w = "energy_mean_scale must be >= 0";
    else if (c.frames_context < 0) w = "frames_context must be >= 0 (got " + std::to_string(c.frames_context) + ")";
    else if (!(c.proportion_threshold > 0.f && c.proportion_threshold < 1.f)) w = "proportion_threshold must lie in (0, 1)";
    if (why) *why = w;
    return w.empty();
}

int tile_frames_for(const ppv_vad_cfg& c) {
    return std::max(1, std::min(VAD_TILE_FRAMES, (VAD_STAGE_FLOATS - 3 - c.window) / c.shift + 1));
}

struct VadWs {
    int64_t* meta;  // [3][R + 1] sample, frame and tile offsets
    double *energy, *tile_sum, *thr;
    int2 *count, *base;
};
// Sized from R and the sample total alone: T_r <= L_r / shift (window >= shift), tiles <= frames / tile_frames + R.
void carve_vad(WsCarver& cv, const ppv_vad_cfg& c, int R, int64_t total_samples, VadWs* w) {
    const int64_t frames = total_samples / c.shift;
    const int64_t tiles = frames / tile_frames_for(c) + R;
    w->meta = static_cast<int64_t*>(cv.take(size_t(3) * (R + 1) * sizeof(int64_t)));
    w->energy = static_cast<double*>(cv.take(size_t(frames) * sizeof(double)));
    w->tile_sum = static_cast<double*>(cv.take(size_t(tiles) * sizeof(double)));
    w->thr = static_cast<double*>(cv.take(size_t(R) * sizeof(double)));
    w->count = static_cast<int2*>(cv.take(size_t(tiles) * sizeof(int2)));
    w->base = static_cast<int2*>(cv.take(size_t(tiles) * sizeof(int2)));
}

}  // namespace

int64_t vad_num_frames(const ppv_vad_cfg& c, int64_t L) {
    if (!vad_cfg_ok(c, nullptr) || L < 0) return -1;
    return L < c.window ? 0 : 1 + (L - c.window) / c.shift;
}

size_t vad_workspace_bytes(const ppv_vad_cfg& c, int R, int64_t total_samples) {
    if (!vad_cfg_ok(c, nullptr) || R < 1 || total_samples < 0) return 0;
    return carve_extent([&](WsCarver& cv) { VadWs w; carve_vad(cv, c, R, total_samples, &w); });
}

int vad_energy(const ppv_vad_cfg& c, const float* wav, const int64_t* sample_offsets, int R, double* log_energy, uint8_t* voiced,
               int32_t* runs, int64_t run_cap, int32_t* n_runs, void* ws, size_t ws_bytes, cudaStream_t st) {
    std::string why;
    PPV_REQUIRE(vad_cfg_ok(c, &why), "vad_energy: " + why);
    PPV_REQUIRE(wav && sample_offsets && voiced && runs && n_runs, "vad_energy: null argument");
    PPV_REQUIRE(R >= 1, "vad_energy: R must be >= 1 (got " + std::to_string(R) + ")");
    PPV_REQUIRE(reinterpret_cast<uintptr_t>(wav) % 4 == 0, "vad_energy: wav must be 4-byte aligned");
    PPV_REQUIRE(sample_offsets[0] >= 0, "vad_energy: sample_offsets[0] must be >= 0");
    const int tf = tile_frames_for(c);
    std::vector<int64_t> meta(size_t(3) * (R + 1));
    int64_t *so = meta.data(), *fo = so + (R + 1), *to = fo + (R + 1);
    int64_t need_runs = 0;
    fo[0] = to[0] = 0;
    for (int r = 0; r < R; ++r) {
        const int64_t L = sample_offsets[r + 1] - sample_offsets[r];
        PPV_REQUIRE(L >= 0, "vad_energy: sample offsets decrease at recording " + std::to_string(r));
        const int64_t T = vad_num_frames(c, L);
        PPV_REQUIRE(T < (int64_t(1) << 31) - 1, "vad_energy: recording " + std::to_string(r) + " has more than 2^31 - 2 frames");
        so[r] = sample_offsets[r];
        fo[r + 1] = fo[r] + T;
        to[r + 1] = to[r] + (T + tf - 1) / tf;
        need_runs += (T + 1) / 2;
    }
    so[R] = sample_offsets[R];
    const int64_t frames = fo[R], tiles = to[R];
    PPV_REQUIRE(frames < (int64_t(1) << 31), "vad_energy: more than 2^31 - 1 frames in the batch");
    PPV_REQUIRE(run_cap >= need_runs, "vad_energy: run capacity " + std::to_string(run_cap) + " < " + std::to_string(need_runs) +
                                          " (sum over recordings of ceil(T / 2))");
    if (int rc = check_workspace("vad_energy", ws, ws_bytes, vad_workspace_bytes(c, R, so[R]), "ppv_vad_workspace_bytes")) return rc;
    WsCarver cv{static_cast<uint8_t*>(ws)};
    VadWs w;
    carve_vad(cv, c, R, so[R], &w);
    double* energy = log_energy ? log_energy : w.energy;
    if (tiles == 0) {
        PPV_CUDA_OK(cudaMemsetAsync(n_runs, 0, sizeof(int32_t), st));
        return PPV_OK;
    }
    PPV_CUDA_OK(cudaMemcpyAsync(w.meta, meta.data(), meta.size() * sizeof(int64_t), cudaMemcpyHostToDevice, st));
    const VadGeom g{w.meta, w.meta + (R + 1), w.meta + 2 * (R + 1), R, c.window, c.shift, tf};
    const size_t smem = size_t((tf - 1) * c.shift + c.window + 3) * sizeof(float);
    PPV_ONCE_PER_DEVICE(PPV_CUDA_OK(cudaFuncSetAttribute(vad_energy_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                                         int(VAD_STAGE_FLOATS * sizeof(float)))));
    vad_energy_kernel<<<unsigned(tiles), VAD_THREADS, smem, st>>>(wav, g, energy, w.tile_sum);
    PPV_LAUNCH_OK("vad_energy_kernel");
    vad_threshold_kernel<<<R, VAD_THREADS, 0, st>>>(g, w.tile_sum, c.energy_threshold, c.energy_mean_scale, w.thr);
    PPV_LAUNCH_OK("vad_threshold_kernel");
    vad_decide_kernel<<<unsigned(tiles), VAD_TILE_THREADS, 0, st>>>(g, energy, w.thr, c.frames_context, c.proportion_threshold, voiced, w.count);
    PPV_LAUNCH_OK("vad_decide_kernel");
    vad_scan_kernel<<<1, VAD_SCAN_THREADS, 0, st>>>(w.count, tiles, w.base, n_runs);
    PPV_LAUNCH_OK("vad_scan_kernel");
    vad_emit_kernel<<<unsigned(tiles), VAD_TILE_THREADS, 0, st>>>(g, voiced, w.base, runs);
    PPV_LAUNCH_OK("vad_emit_kernel");
    return PPV_OK;
}

}  // namespace ppv
