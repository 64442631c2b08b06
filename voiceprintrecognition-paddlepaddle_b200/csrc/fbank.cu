// Fused Kaldi Fbank front end (K1): framing -> DC removal -> pre-emphasis -> povey window -> zero-pad ->
// 512-point real FFT (one 256-point complex FFT) -> power -> sparse mel (501 non-zeros for 80 bins) -> log,
// then CMN over time (+ optional tail mask).
// Reference: ppvector/data_utils/featurizer.py:88-101 (KaldiFbank -> paddleaudio.compliance.kaldi.fbank,
// algorithm as torchaudio/compliance/kaldi.py:_get_window / fbank) and featurizer.py:43-59.
//
// fbank_logmel_kernel (round 2).  Persistent CTAs walk work items of 16 consecutive frames of one utterance.
//   * The item's waveform segment (15 * shift + win samples, 11 KB) arrives by ONE cp.async.bulk (TMA 1-D) on an mbarrier,
//     double-buffered: the copy of item i+2 is in flight while item i is in the butterflies.  HBM sees each sample ~1.09 times
//     (frames overlap 2.5x inside an item; only the item seams are re-read, from L2).
//   * 16 lanes own one frame (a warp = 2 frames): the 256-point complex FFT is two radix-16 passes held ENTIRELY in registers
//     (16 complex values per lane, radix-4 x radix-4 with constant twiddles) with one transpose through padded shared memory in
//     between -- no shuffle butterflies, no bit-reversal pass.  (Round 1 put one warp on one frame: 80 shuffles per lane
//     per frame plus a bank-conflicting bit-reversed round trip made it shuffle / LSU-issue bound at 4.6 % of the HBM roofline.)
//   * log-mel rows of the item are staged in shared memory and leave as 16-byte coalesced stores, together with the item's
//     column sums, so the separate mean pass over [B,T,F] is gone: fbank_finalize reads the partial sums.
//
// fbank_frame_kernel (every other configuration: FFT sizes 128..4096, snip_edges off, no DC removal, magnitude or linear output).
//   One CTA per work item of 16 frames, the same items and the same output contract (raw rows + per-item column sums) as
//   fbank_logmel_kernel, so fbank_finalize and the models' fused waveform path are shared.  The frames of an item go through the
//   radix-2 shared-memory FFT of fft_radix2.cuh 4096 / n_fft at a time (one frame per pass at 4096 points, all 16 at <= 256).
//   fbank_create chooses the kernel from the config; nothing else selects it.
#include <math.h>

#include <vector>

#include "common.h"
#include "fft512.cuh"
#include "fft_radix2.cuh"
#include "ptx.cuh"

namespace ppv {

constexpr int FB_NFFT = 512;          // padded window (round_to_power_of_two)
constexpr int FB_HALF = FB_NFFT / 2;  // complex FFT length
constexpr int FB_ITEM = 16;           // frames per work item
constexpr int FB_THREADS = 256;       // 8 warps x 2 frames
constexpr int FB_SCR = 17 * 16;       // float2 scratch per frame: [k1][n2] padded to 17 columns
constexpr int FB_SCR_PAIR = 2 * FB_SCR + 8;  // the two frames of a warp: the odd one starts 64 B (16 banks) past the even one's end
constexpr int FB_MAX_MELS = 128;
constexpr int FB_PART_ROWS = 32768;   // handle-owned partial-sum rows ([row][FB_MAX_MELS]): utterances x items per launch group
constexpr int FB_FIN_FRAMES = 32;     // frames per finalize block
constexpr int FB_TW512 = 144;         // e^{-2 pi i k / 512} is needed for k <= 143 only (bins k and 256 - k share a pair)
constexpr int FB_MIN_NFFT = 128, FB_MAX_NFFT = 4096;
constexpr int FG_POINTS = 4096;       // complex points per FFT pass of fbank_frame_kernel
constexpr int FG_THREADS = 256;

struct FbankTables {
    float* window = nullptr;    // [n_fft] zero-padded
    float2* tw = nullptr;       // [16][16]  exp(-2 pi i k1 n2 / 256) at [k1*16 + n2]
    float2* tw512 = nullptr;    // [256]  exp(-2 pi i k / 512)
    float* mel_w = nullptr;     // [nnz]  (x 0.25 for fbank_logmel_kernel: its spectrum is 2 X)
    int* mel_start = nullptr;   // [n_mels] first FFT bin
    int* mel_len = nullptr;     // [n_mels]
    int* mel_off = nullptr;     // [n_mels] offset into mel_w
    int nnz = 0;
};

struct Fbank {
    ppv_fbank_cfg cfg;
    int win = 0, shift = 0, nfft = 0, log2n = 0;
    bool general = false;         // fbank_frame_kernel; otherwise fbank_logmel_kernel
    FbankTables tb;
    float2* twiddle = nullptr;    // [n_fft / 2] exp(-2 pi i k / n_fft), fbank_frame_kernel only
    float* part = nullptr;   // [FB_PART_ROWS, FB_MAX_MELS] per-item column sums
    float* part2 = nullptr;  // [FB_PART_ROWS / 64, FB_MAX_MELS] per-utterance sums (long utterances)
};

struct FbankSmem {  // byte offsets of the dynamic shared-memory carve-up (host and device agree through this struct)
    int tw, tw512, win, melw, mstart, mlen, moff, scr, out, seg, bar, total, seg_stride;
};
__host__ __device__ inline FbankSmem fbank_smem_layout(int nnz, int n_mels, int win, int shift) {
    FbankSmem L;
    int o = 0;
    auto take = [&](int bytes) { const int at = o; o += (bytes + 15) & ~15; return at; };
    L.tw = take(256 * 8);
    L.tw512 = take(FB_TW512 * 8);
    L.win = take(FB_NFFT * 4);
    L.melw = take(nnz * 4);
    L.mstart = take(n_mels * 4);
    L.mlen = take(n_mels * 4);
    L.moff = take(n_mels * 4);
    L.scr = take((FB_ITEM / 2) * FB_SCR_PAIR * 8);
    L.out = take(2 * FB_ITEM * n_mels * 4);
    L.seg_stride = (((FB_ITEM - 1) * shift + win) * 4 + 127) & ~127;
    L.seg = take(2 * L.seg_stride);
    L.bar = take(2 * 8);
    L.total = o;
    return L;
}

// raw log-mel out_raw [B, T, n_mels] + per-item column sums part[(b * nitem + item) * FB_MAX_MELS + m]
// WIN > 0: the window length is a compile-time constant (400 for 16 kHz / 25 ms): the bounds tests of the frame load disappear.
template <bool VEC, int WIN>
__global__ void __launch_bounds__(FB_THREADS, 3)
    fbank_logmel_kernel(const float* __restrict__ wav, int B, int L, int T, int win_rt, int shift, int n_mels, float preemph,
                        float log_floor, FbankTables tb, int use_tma, float* __restrict__ out_raw, float* __restrict__ part,
                        const int* __restrict__ valid_frames) {
    extern __shared__ __align__(128) uint8_t fb_smem[];
    const int win = WIN > 0 ? WIN : win_rt;
    const FbankSmem lay = fbank_smem_layout(tb.nnz, n_mels, win, shift);
    float2* s_tw = reinterpret_cast<float2*>(fb_smem + lay.tw);
    float2* s_tw512 = reinterpret_cast<float2*>(fb_smem + lay.tw512);
    float* s_win = reinterpret_cast<float*>(fb_smem + lay.win);
    float* s_melw = reinterpret_cast<float*>(fb_smem + lay.melw);
    int* s_mstart = reinterpret_cast<int*>(fb_smem + lay.mstart);
    int* s_mlen = reinterpret_cast<int*>(fb_smem + lay.mlen);
    int* s_moff = reinterpret_cast<int*>(fb_smem + lay.moff);
    float2* s_scr = reinterpret_cast<float2*>(fb_smem + lay.scr);
    float* s_out = reinterpret_cast<float*>(fb_smem + lay.out);
    const uint32_t bar0 = smem_u32(fb_smem + lay.bar);

    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, q = lane & 15;
    const int fl = warp * 2 + (lane >> 4);  // frame slot inside the item
    const int nitem = (T + FB_ITEM - 1) / FB_ITEM;
    const int total = B * nitem;

    for (int i = tid; i < 256; i += FB_THREADS) s_tw[i] = tb.tw[i];
    for (int i = tid; i < FB_TW512; i += FB_THREADS) s_tw512[i] = tb.tw512[i];
    for (int i = tid; i < FB_NFFT; i += FB_THREADS) s_win[i] = tb.window[i];
    for (int i = tid; i < tb.nnz; i += FB_THREADS) s_melw[i] = tb.mel_w[i];
    for (int i = tid; i < n_mels; i += FB_THREADS) {
        s_mstart[i] = tb.mel_start[i];
        s_mlen[i] = tb.mel_len[i];
        s_moff[i] = tb.mel_off[i];
    }
    if (tid == 0) {
        mbar_init(bar0, 1);
        mbar_init(bar0 + 8, 1);
        fence_mbar_init();
    }
    griddep_launch_dependents();
    griddep_wait();  // the tables above are constants; the waveform / output buffers may belong to the previous step
    __syncthreads();

    auto item_geom = [&](int it, int& b, int& f0, int& nf) {
        b = it / nitem;
        f0 = (it - b * nitem) * FB_ITEM;
        nf = min(FB_ITEM, T - f0);
    };
    auto issue = [&](int it, int buf) {  // one elected thread: TMA 1-D bulk copy of the item's waveform segment
        int b, f0, nf;
        item_geom(it, b, f0, nf);
        const uint32_t bytes = uint32_t((nf - 1) * shift + win) * 4u;
        mbar_arrive_expect_tx(bar0 + 8 * buf, bytes);
        bulk_load_1d(smem_u32(fb_smem + lay.seg + buf * lay.seg_stride), wav + int64_t(b) * L + int64_t(f0) * shift, bytes, bar0 + 8 * buf);
    };
    if (use_tma && tid == 0) {
        if (int(blockIdx.x) < total) issue(blockIdx.x, 0);
        if (int(blockIdx.x + gridDim.x) < total) issue(blockIdx.x + gridDim.x, 1);
    }

    const float inv_win = 1.f / float(win);
    // the two frames of a warp sit 16 banks apart (odd slot = even slot + FB_SCR + 8 float2): their 4-byte power stores / mel reads do not
    // collide; every pair owns its own 64 B of slack, no slot overlaps another
    float2* scr = s_scr + (fl >> 1) * FB_SCR_PAIR + (fl & 1) * (FB_SCR + 8);
    int n = 0;
    for (int it = blockIdx.x; it < total; it += gridDim.x, ++n) {
        const int buf = n & 1;
        int b, f0, nf;
        item_geom(it, b, f0, nf);
        const float* seg = reinterpret_cast<const float*>(fb_smem + lay.seg + buf * lay.seg_stride);
        if (use_tma) {
            mbar_wait(bar0 + 8 * buf, (n >> 1) & 1);
        } else {  // unaligned waveforms: plain loads (a [B, L] batch with L % 4 != 0)
            const int len = (nf - 1) * shift + win;
            const float* src = wav + int64_t(b) * L + int64_t(f0) * shift;
            float* dst = const_cast<float*>(seg);
            for (int i = tid; i < len; i += FB_THREADS) dst[i] = __ldg(src + i);
            __syncthreads();
        }
        const float* s = seg + min(fl, nf - 1) * shift;  // idle slots of a short last item recompute its last frame, unseen

        // ---- load: lane q holds z[16 n1 + q] = (y[32 n1 + 2q], y[32 n1 + 2q + 1]) for n1 = 0..15 ----
        float2 v[16];
        float prev[16];
        float acc = 0.f;
#pragma unroll
        for (int n1 = 0; n1 < 16; ++n1) {
            const int j = 32 * n1 + 2 * q;
            float a0 = 0.f, a1 = 0.f, ap = 0.f;
            if (WIN > 0 && 32 * n1 + 32 <= WIN) {  // whole row inside the window: no test at all
                if constexpr (VEC) {
                    const float2 t = *reinterpret_cast<const float2*>(s + j);
                    a0 = t.x;
                    a1 = t.y;
                } else {
                    a0 = s[j];
                    a1 = s[j + 1];
                }
                ap = s[n1 == 0 ? max(j - 1, 0) : j - 1];
            } else if (WIN > 0 && 32 * n1 >= WIN) {
                // zero padding
            } else if (j + 1 < win) {
                if constexpr (VEC) {
                    const float2 t = *reinterpret_cast<const float2*>(s + j);
                    a0 = t.x;
                    a1 = t.y;
                } else {
                    a0 = s[j];
                    a1 = s[j + 1];
                }
                ap = s[j > 0 ? j - 1 : 0];
            } else if (j < win) {
                a0 = s[j];
                ap = s[j > 0 ? j - 1 : 0];
            }
            v[n1] = make_float2(a0, a1);
            prev[n1] = ap;
            acc += a0 + a1;
        }
        // DC offset over the frame's win samples (torchaudio kaldi.py:_get_window remove_dc_offset): 16-lane sum
        acc += __shfl_xor_sync(0xffffffffu, acc, 8);
        acc += __shfl_xor_sync(0xffffffffu, acc, 4);
        acc += __shfl_xor_sync(0xffffffffu, acc, 2);
        acc += __shfl_xor_sync(0xffffffffu, acc, 1);
        const float cdc = (1.f - preemph) * (acc * inv_win);
        // pre-emphasis + povey window: ((s_j - mu) - p (s_{j-1} - mu)) w_j = (s_j - p s_{j-1} - (1 - p) mu) w_j; s_{-1} := s_0
#pragma unroll
        for (int n1 = 0; n1 < 16; ++n1) {
            if (WIN > 0 && 32 * n1 >= WIN) continue;  // v[n1] is already (0, 0)
            const float2 w = *reinterpret_cast<const float2*>(s_win + 32 * n1 + 2 * q);  // zero beyond win
            const float y0 = (fmaf(-preemph, prev[n1], v[n1].x) - cdc) * w.x;
            const float y1 = (fmaf(-preemph, v[n1].x, v[n1].y) - cdc) * w.y;
            v[n1] = make_float2(y0, y1);
        }
        // ---- pass 1: 16-point DFT over n1 (lane = n2), twiddle W256^{n2 k1}, transpose through shared memory ----
        fft16(v);
#pragma unroll
        for (int r = 0; r < 16; ++r) {
            const int k1 = fb_k_of_slot(r);
            scr[k1 * 17 + q] = k1 == 0 ? v[r] : cmul(v[r], s_tw[k1 * 16 + q]);
        }
        __syncwarp();
#pragma unroll
        for (int n2 = 0; n2 < 16; ++n2) v[n2] = scr[q * 17 + n2];
        // ---- pass 2: 16-point DFT over n2 (lane = k1): slot r holds Z[q + 16 k2(r)] ----
        fft16(v);
        __syncwarp();
#pragma unroll
        for (int r = 0; r < 16; ++r) scr[q + 16 * fb_k_of_slot(r)] = v[r];
        __syncwarp();
        // ---- real-FFT untangling, bins k and 256-k from the same pair: with 2F = Zk + conj Z[256-k], 2G = -i (Zk - conj Z[256-k]),
        //      2 X[k] = 2F + W^k 2G and 2 X[256-k] = conj(2F - W^k 2G), W = e^{-2 pi i / 512}.  Lane q takes k = q + 16 i, i = 0..8
        //      (i = 8 is k = 128, lane 0 only). ----
        float pk[9], pn[9];
#pragma unroll
        for (int i = 0; i < 9; ++i) {
            const int k = q + 16 * i;  // <= 143
            const float2 zk = scr[k];
            const float2 zn = scr[(FB_HALF - k) & (FB_HALF - 1)];
            const float2 f = make_float2(zk.x + zn.x, zk.y - zn.y);
            const float2 g = make_float2(zk.y + zn.y, zn.x - zk.x);  // -i (zk - conj zn)
            const float2 wg = cmul(s_tw512[k], g);
            const float ar = f.x + wg.x, ai = f.y + wg.y, br = f.x - wg.x, bi = f.y - wg.y;
            pk[i] = fmaf(ar, ar, ai * ai);
            pn[i] = fmaf(br, br, bi * bi);
        }
        __syncwarp();
        float* ps = reinterpret_cast<float*>(scr);
#pragma unroll
        for (int i = 0; i < 9; ++i) {
            const int k = q + 16 * i;
            if (i < 8 || q == 0) {  // i = 8: only k = 128 is new (the pairs (128 + q, 128 - q) belong to lane 16 - q at i = 7)
                ps[k] = pk[i];
                if (k > 0 && k < FB_HALF / 2) ps[FB_HALF - k] = pn[i];  // k = 0: the partner is the Nyquist bin, unused by the mel banks
            }
        }
        __syncwarp();
        // ---- sparse mel + log into the staging tile ----
        float* so = s_out + buf * (FB_ITEM * n_mels);
        if (fl < nf) {
            for (int m = q; m < n_mels; m += 16) {
                const float* w = s_melw + s_moff[m];
                const float* p = ps + s_mstart[m];
                const int len = s_mlen[m];  // a multiple of 4 (rows are padded with zero weights)
                float e0 = 0.f, e1 = 0.f;
                for (int j = 0; j < len; j += 4) {
                    e0 = fmaf(w[j], p[j], e0);
                    e1 = fmaf(w[j + 1], p[j + 1], e1);
                    e0 = fmaf(w[j + 2], p[j + 2], e0);
                    e1 = fmaf(w[j + 3], p[j + 3], e1);
                }
                so[fl * n_mels + m] = logf(fmaxf(e0 + e1, log_floor));
            }
        }
        __syncthreads();  // staging tile complete; every warp is done with this item's waveform segment and scratch
        if (use_tma && tid == 0) {
            const int nxt = it + 2 * int(gridDim.x);
            if (nxt < total) issue(nxt, buf);
        }
        // ---- coalesced store of the item's rows + its column sums ----
        float* dst = out_raw + (int64_t(b) * T + f0) * n_mels;
        const int cnt = nf * n_mels;
        if (((reinterpret_cast<uintptr_t>(dst) | uintptr_t(cnt * 4)) & 15) == 0) {
            for (int i = tid; i < cnt / 4; i += FB_THREADS) reinterpret_cast<float4*>(dst)[i] = reinterpret_cast<const float4*>(so)[i];
        } else {
            for (int i = tid; i < cnt; i += FB_THREADS) dst[i] = so[i];
        }
        if (tid < n_mels) {
            // ragged batches: frames beyond the utterance's own count are padding and stay out of its time mean
            const int nsum = valid_frames ? max(0, min(nf, valid_frames[b] - f0)) : nf;
            float sum = 0.f;
            for (int f = 0; f < nsum; ++f) sum += so[f * n_mels + tid];
            part[int64_t(it) * FB_MAX_MELS + tid] = sum;
        }
    }
}

// Where frame 0 starts in the waveform.  snip_edges: at sample 0.  Otherwise torchaudio's _get_strided frames the waveform with
// min(pad, L) of its first samples prepended in reverse (pad = win / 2 - shift / 2 > 0; the edge sample repeats, unlike numpy's
// 'reflect') or with its first min(-pad, L) samples dropped (pad <= 0), and the whole reversed waveform appended on the right.
// Sample n of frame t is then index g = t * shift + n + origin of the waveform, mirrored as -1 - g below 0 and 2L - 1 - g from L on.
__host__ __device__ inline int fbank_frame_origin(int L, int win, int shift, int snip_edges) {
    if (snip_edges) return 0;
    const int pad = win / 2 - shift / 2;
    return pad > 0 ? -min(pad, L) : min(-pad, L);
}

struct FbankFrameArgs {
    const float* window;    // [n_fft], zero beyond win
    const float2* twiddle;  // [n_fft / 2]
    const float* mel_w;
    const int* mel_start;
    const int* mel_len;
    const int* mel_off;
    int win, shift, log2n, n_mels, snip_edges, remove_dc, use_power, use_log;
    float preemph, log_floor;
};

__host__ __device__ inline int fbank_frame_smem_bytes(int n_mels) {
    return FG_POINTS * 8 + (FG_POINTS / 2) * 4 + FB_ITEM * n_mels * 4 + FB_ITEM * 4;
}

// The general Kaldi frame: framing (either snip_edges) -> DC removal (optional) -> pre-emphasis -> window -> zero-pad to n_fft ->
// radix-2 FFT -> power or magnitude -> sparse mel -> log (optional).  Same output contract as fbank_logmel_kernel: raw rows
// out_raw [B, T, n_mels] and per-item column sums part[(b * nitem + item) * FB_MAX_MELS + m].  num_samples (optional): utterance b's
// own length, where its right edge is reflected (ragged batches); frames past an utterance's own count are computed from clamped
// indices and only ever read as padding.
__global__ void __launch_bounds__(FG_THREADS, 2)
    fbank_frame_kernel(const float* __restrict__ wav, int L, int T, FbankFrameArgs a, const int* __restrict__ num_samples,
                       float* __restrict__ out_raw, float* __restrict__ part, const int* __restrict__ valid_frames) {
    extern __shared__ __align__(16) uint8_t fg_smem[];
    float2* z = reinterpret_cast<float2*>(fg_smem);       // [FG_POINTS] the transforms of one pass, back to back
    float* pw = reinterpret_cast<float*>(z + FG_POINTS);  // [FG_POINTS / 2] their spectra, bins 0 .. n_fft / 2 - 1
    float* s_out = pw + FG_POINTS / 2;                    // [FB_ITEM][n_mels]
    float* s_mu = s_out + FB_ITEM * a.n_mels;             // [FB_ITEM] frame means of the pass
    griddep_launch_dependents();
    griddep_wait();
    const int N = 1 << a.log2n, half = N >> 1;
    const int nitem = (T + FB_ITEM - 1) / FB_ITEM;
    const int it = blockIdx.x, b = it / nitem, f0 = (it - b * nitem) * FB_ITEM, nf = min(FB_ITEM, T - f0);
    const int Lb = num_samples ? min(max(num_samples[b], 1), L) : L;
    const int origin = fbank_frame_origin(Lb, a.win, a.shift, a.snip_edges);
    const float* x = wav + int64_t(b) * L;
    const int shift = a.shift;
    auto sample = [=](int t, int n) {
        int g = t * shift + n + origin;
        if (g < 0) g = -1 - g;
        if (g >= Lb) g = 2 * Lb - 1 - g;
        return __ldg(x + min(max(g, 0), Lb - 1));
    };
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int fpp = min(FB_ITEM, FG_POINTS >> a.log2n);  // frames per pass
    for (int p0 = 0; p0 < nf; p0 += fpp) {
        const int np = min(fpp, nf - p0);
        for (int fr = warp; fr < np; fr += FG_THREADS / 32) {
            float s = 0.f;
            if (a.remove_dc)
                for (int n = lane; n < a.win; n += 32) s += sample(f0 + p0 + fr, n);
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
            if (lane == 0) s_mu[fr] = s / float(a.win);
        }
        __syncthreads();
        // ((x_n - mu) - p (x_{n-1} - mu)) w_n with x_{-1} := x_0, zero from win on; stored bit-reversed for the FFT
        for (int i = threadIdx.x; i < np * N; i += FG_THREADS) {
            const int fr = i >> a.log2n, n = i & (N - 1);
            float y = 0.f;
            if (n < a.win) {
                const int t = f0 + p0 + fr;
                const float mu = s_mu[fr];
                const float cur = sample(t, n) - mu, prev = sample(t, n > 0 ? n - 1 : 0) - mu;
                y = fmaf(-a.preemph, prev, cur) * __ldg(a.window + n);
            }
            z[(fr << a.log2n) + fft_bitrev(n, a.log2n)] = make_float2(y, 0.f);
        }
        __syncthreads();
        fft_radix2(z, a.log2n, np, a.twiddle);
        for (int i = threadIdx.x; i < np * half; i += FG_THREADS) {
            const float2 c = z[((i >> (a.log2n - 1)) << a.log2n) + (i & (half - 1))];
            const float p = fmaf(c.x, c.x, c.y * c.y);
            pw[i] = a.use_power ? p : sqrtf(p);
        }
        __syncthreads();
        for (int i = threadIdx.x; i < np * a.n_mels; i += FG_THREADS) {
            const int fr = i / a.n_mels, m = i - fr * a.n_mels;
            const float* w = a.mel_w + __ldg(a.mel_off + m);
            const float* p = pw + fr * half + __ldg(a.mel_start + m);
            const int len = __ldg(a.mel_len + m);
            float e = 0.f;
            for (int j = 0; j < len; ++j) e = fmaf(__ldg(w + j), p[j], e);
            s_out[(p0 + fr) * a.n_mels + m] = a.use_log ? logf(fmaxf(e, a.log_floor)) : e;
        }
        __syncthreads();
    }
    float* dst = out_raw + (int64_t(b) * T + f0) * a.n_mels;
    for (int i = threadIdx.x; i < nf * a.n_mels; i += FG_THREADS) dst[i] = s_out[i];
    if (int(threadIdx.x) < a.n_mels) {
        // ragged batches: frames beyond the utterance's own count are padding and stay out of its time mean
        const int nsum = valid_frames ? max(0, min(nf, valid_frames[b] - f0)) : nf;
        float sum = 0.f;
        for (int f = 0; f < nsum; ++f) sum += s_out[f * a.n_mels + threadIdx.x];
        part[int64_t(it) * FB_MAX_MELS + threadIdx.x] = sum;
    }
}

// long utterances: fold the per-item sums of each utterance into one row (nitem -> 1)
__global__ void __launch_bounds__(128) fbank_part_reduce_kernel(const float* __restrict__ part, int nitem, float* __restrict__ out) {
    griddep_launch_dependents();
    griddep_wait();
    const int b = blockIdx.x, f = threadIdx.x;
    float s = 0.f;
    for (int i = 0; i < nitem; ++i) s += part[(int64_t(b) * nitem + i) * FB_MAX_MELS + f];
    out[int64_t(b) * FB_MAX_MELS + f] = s;
}

// CMN + tail mask; writes fp32 [B,T,F] (out_f32, may alias raw) and/or split planes in the padded layout.
// mean[b][f] = (sum over the utterance's nsum partial rows) / T.
__global__ void __launch_bounds__(256)
    fbank_finalize_kernel(const float* __restrict__ raw, const float* __restrict__ part, int nsum, const float* __restrict__ lens_ratio,
                          const int* __restrict__ valid_frames, int B, int T, int F, float* out_f32, Planes out_pl, int P, int Tp) {
    __shared__ float s_mu[FB_MAX_MELS];
    griddep_launch_dependents();
    griddep_wait();
    const int b = blockIdx.y;
    if (threadIdx.x < FB_MAX_MELS) {
        float s = 0.f;
        if (int(threadIdx.x) < F)
            for (int i = 0; i < nsum; ++i) s += part[(int64_t(b) * nsum + i) * FB_MAX_MELS + threadIdx.x];
        s_mu[threadIdx.x] = s / float(valid_frames ? max(1, min(T, valid_frames[b])) : T);
    }
    __syncthreads();
    const int lane = threadIdx.x & 31;
    int keep_n = T;
    if (lens_ratio) keep_n = int(lens_ratio[b] * float(T));  // featurizer.py:51: (ratio * T).astype(int32)
    if (valid_frames) keep_n = min(keep_n, valid_frames[b]);
    for (int t = blockIdx.x * FB_FIN_FRAMES + (threadIdx.x >> 5); t < min(T, (int(blockIdx.x) + 1) * FB_FIN_FRAMES); t += 8) {
        const int64_t frame = int64_t(b) * T + t;
        const bool keep = t < keep_n;
        const float* src = raw + frame * F;
        if (out_f32) {
            for (int f = lane; f < F; f += 32) out_f32[frame * F + f] = keep ? src[f] - s_mu[f] : 0.f;
        }
        if (out_pl.base) {
            const int64_t row = int64_t(b) * Tp + P + t;
            int64_t rows[3] = {row, -1, -1};
            if (t >= 1 && t <= P) rows[1] = row - 2 * t;
            const int u = T - 1 - t;
            if (u >= 1 && u <= P) rows[2] = row + 2 * u;
            for (int c = 2 * lane; c < out_pl.ld; c += 64) {
                const float a = (c < F && keep) ? src[c] - s_mu[c] : 0.f;
                const float bb = (c + 1 < F && keep) ? src[c + 1] - s_mu[c + 1] : 0.f;
                uint32_t hi, lo;
                split_pack_bf16x2(a, bb, hi, lo);
#pragma unroll
                for (int k = 0; k < 3; ++k)
                    if (rows[k] >= 0) {
                        *reinterpret_cast<uint32_t*>(out_pl.hi() + rows[k] * out_pl.ld + c) = hi;
                        *reinterpret_cast<uint32_t*>(out_pl.lo() + rows[k] * out_pl.ld + c) = lo;
                    }
            }
        }
    }
}

// ------------------------------------------------------------------------------------------------ host
static int next_pow2(int x) {
    int p = 1;
    while (p < x) p <<= 1;
    return p;
}

template <typename T>
static int upload(T** dst, const std::vector<T>& v) {
    PPV_CUDA_OK(cudaMalloc(reinterpret_cast<void**>(dst), v.size() * sizeof(T)));
    PPV_CUDA_OK(cudaMemcpy(*dst, v.data(), v.size() * sizeof(T), cudaMemcpyHostToDevice));
    return PPV_OK;
}

// torchaudio kaldi.py:_feature_window_function, in double, rounded once
static float fbank_window_value(int type, int i, int win, double blackman_coeff) {
    const double c = cos(2.0 * M_PI * i / (win - 1));
    switch (type) {
        case PPV_FBANK_WIN_HANNING: return float(0.5 - 0.5 * c);
        case PPV_FBANK_WIN_HAMMING: return float(0.54 - 0.46 * c);
        case PPV_FBANK_WIN_RECTANGULAR: return 1.f;
        case PPV_FBANK_WIN_BLACKMAN: {
            const double a = 2.0 * M_PI / (win - 1);
            return float(blackman_coeff - 0.5 * cos(a * i) + (0.5 - blackman_coeff) * cos(2.0 * a * i));
        }
        default: {  // povey: hann(periodic=False)^0.85
            const double hann = 0.5 - 0.5 * cos(2.0 * M_PI * i / (win - 1));
            return float(pow(hann, 0.85));
        }
    }
}

int fbank_create(const ppv_fbank_cfg* cfg, Fbank** out) {
    PPV_REQUIRE(cfg && out, "fbank_create: null argument");
    Fbank* h = new Fbank();
    h->cfg = *cfg;
    h->win = int(cfg->sample_rate * cfg->frame_length_ms * 0.001f);
    h->shift = int(cfg->sample_rate * cfg->frame_shift_ms * 0.001f);
    if (cfg->sample_rate <= 0 || h->shift <= 0 || h->win < 2) {
        delete h;
        return fail(PPV_EINVAL, "fbank: sample_rate, frame_length_ms and frame_shift_ms must give a window of >= 2 samples and a shift of >= 1");
    }
    h->nfft = next_pow2(h->win);  // round_to_power_of_two
    if (h->nfft < FB_MIN_NFFT || h->nfft > FB_MAX_NFFT) {
        const int nfft = h->nfft, win = h->win;
        delete h;
        return fail(PPV_EUNSUPPORTED, "fbank: a " + std::to_string(win) + "-sample window pads to a " + std::to_string(nfft) +
                                          "-point FFT; the FFT size must be a power of two in [128, 4096]");
    }
    while ((1 << h->log2n) < h->nfft) ++h->log2n;
    if (cfg->n_mels < 4 || cfg->n_mels > FB_MAX_MELS) {
        delete h;
        return fail(PPV_EUNSUPPORTED, "fbank: n_mels must be in [4,128]");
    }
    if (cfg->window_type < PPV_FBANK_WIN_POVEY || cfg->window_type > PPV_FBANK_WIN_BLACKMAN) {
        delete h;
        return fail(PPV_EINVAL, "fbank: unknown window_type");
    }
    h->general = !(h->nfft == FB_NFFT && cfg->snip_edges && cfg->remove_dc_offset && cfg->use_power && cfg->use_log_fbank);
    const int win = h->win, nfft = h->nfft, half = nfft / 2;
    std::vector<float> window(nfft, 0.f);  // zero beyond win: the kernels multiply all n_fft slots
    for (int i = 0; i < win; ++i) window[i] = fbank_window_value(cfg->window_type, i, win, double(cfg->blackman_coeff));
    // mel banks, evaluated in float32 like torchaudio kaldi.py:get_mel_banks
    const int nb = cfg->n_mels;
    const float sr = float(cfg->sample_rate);
    const float nyq = 0.5f * sr;
    float high = cfg->high_freq;
    if (high <= 0.f) high += nyq;
    const float low = cfg->low_freq;
    if (!(low >= 0.f && low < nyq && high > 0.f && high <= nyq && low < high)) {
        delete h;
        return fail(PPV_EINVAL, "fbank: bad low_freq / high_freq");
    }
    const bool warp = cfg->vtln_warp != 1.f;
    float vtln_high = cfg->vtln_high;
    if (vtln_high < 0.f) vtln_high += nyq;
    // the piecewise-linear VTLN warp of kaldi.py:vtln_warp_freq, inflection points l and h, slopes in double, applied in float32
    const double wf = cfg->vtln_warp;
    const double vl = double(cfg->vtln_low) * std::max(1.0, wf), vh = double(vtln_high) * std::min(1.0, wf);
    if (warp && !(wf > 0.0 && low < cfg->vtln_low && cfg->vtln_low < high && 0.f < vtln_high && vtln_high < high &&
                  cfg->vtln_low < vtln_high && vl > low && vh < high)) {
        delete h;
        return fail(PPV_EINVAL, "fbank: bad vtln_warp / vtln_low / vtln_high (need low_freq < vtln_low < vtln_high < high_freq)");
    }
    const double sd = 1.0 / wf;
    const float scale = float(sd), scale_left = float((sd * vl - low) / (vl - low)), scale_right = float((high - sd * vh) / (high - vh));
    auto warp_mel = [&](float mel) {
        const float f = 700.0f * (expf(mel / 1127.0f) - 1.0f);
        float r;
        if (f < low || f > high) r = f;
        else if (f < float(vl)) r = low + scale_left * (f - low);
        else if (f < float(vh)) r = scale * f;
        else r = high + scale_right * (f - high);
        return 1127.0f * logf(1.0f + r / 700.0f);
    };
    const double mel_low = 1127.0 * log(1.0 + double(low) / 700.0);
    const double mel_high = 1127.0 * log(1.0 + double(high) / 700.0);
    const double delta = (mel_high - mel_low) / (nb + 1);
    const float bin_width = sr / float(nfft);
    // fbank_logmel_kernel's power spectrum is |2X|^2, so its weights carry the 1/4; the general kernel's spectrum is X itself
    const float mel_scale = h->general ? 1.f : 0.25f;
    std::vector<float> melw;
    std::vector<int> mstart(nb), mlen(nb), moff(nb);
    for (int m = 0; m < nb; ++m) {
        float left = float(mel_low) + float(m) * float(delta);
        float center = float(mel_low) + (float(m) + 1.0f) * float(delta);
        float right = float(mel_low) + (float(m) + 2.0f) * float(delta);
        if (warp) {
            left = warp_mel(left);
            center = warp_mel(center);
            right = warp_mel(right);
        }
        int first = -1, last = -1;
        std::vector<float> row(half, 0.f);
        for (int k = 0; k < half; ++k) {
            const float mel = 1127.0f * logf(1.0f + (bin_width * float(k)) / 700.0f);
            const float up = (mel - left) / (center - left);
            const float down = (right - mel) / (right - center);
            // warped edges may come in any order: only the rising and falling flanks count (get_mel_banks, vtln_warp != 1)
            const float w = !warp ? fmaxf(0.f, fminf(up, down)) : (mel > left && mel <= center) ? up : (mel > center && mel < right) ? down : 0.f;
            row[k] = w;
            if (w != 0.f) {
                if (first < 0) first = k;
                last = k;
            }
        }
        mstart[m] = first < 0 ? 0 : first;
        int len = first < 0 ? 0 : last - first + 1;
        len = (len + 3) & ~3;  // fbank_logmel_kernel's mel loop is unrolled by 4: pad with zero weights over valid power bins
        if (mstart[m] + len > half) mstart[m] = half - len;
        mlen[m] = len;
        moff[m] = int(melw.size());
        for (int k = 0; k < len; ++k) melw.push_back(mel_scale * row[mstart[m] + k]);
    }
    if (melw.empty()) melw.push_back(0.f);
    h->tb.nnz = int(melw.size());
    int rc = upload(&h->tb.window, window);
    if (!rc && !h->general) {
        std::vector<float2> tw(256), tw512(256);
        for (int k1 = 0; k1 < 16; ++k1)
            for (int n2 = 0; n2 < 16; ++n2)
                tw[k1 * 16 + n2] = fft_twiddle(k1 * n2, 256);
        for (int k = 0; k < 256; ++k) tw512[k] = fft_twiddle(k, 512);
        rc = upload(&h->tb.tw, tw);
        if (!rc) rc = upload(&h->tb.tw512, tw512);
    }
    if (!rc && h->general) {
        std::vector<float2> tw(half);
        for (int k = 0; k < half; ++k) tw[k] = fft_twiddle(k, nfft);
        rc = upload(&h->twiddle, tw);
    }
    if (!rc) rc = upload(&h->tb.mel_w, melw);
    if (!rc) rc = upload(&h->tb.mel_start, mstart);
    if (!rc) rc = upload(&h->tb.mel_len, mlen);
    if (!rc) rc = upload(&h->tb.mel_off, moff);
    if (!rc && (cudaMalloc(reinterpret_cast<void**>(&h->part), size_t(FB_PART_ROWS) * FB_MAX_MELS * sizeof(float)) != cudaSuccess ||
                cudaMalloc(reinterpret_cast<void**>(&h->part2), size_t(FB_PART_ROWS / 64) * FB_MAX_MELS * sizeof(float)) != cudaSuccess))
        rc = fail(PPV_ECUDA, "fbank: cudaMalloc(partial sums) failed");
    if (rc) {
        fbank_destroy(h);
        return rc;
    }
    *out = h;
    return PPV_OK;
}

void fbank_destroy(Fbank* h) {
    if (!h) return;
    cudaFree(h->tb.window);
    cudaFree(h->tb.tw);
    cudaFree(h->tb.tw512);
    cudaFree(h->tb.mel_w);
    cudaFree(h->tb.mel_start);
    cudaFree(h->tb.mel_len);
    cudaFree(h->tb.mel_off);
    cudaFree(h->twiddle);
    cudaFree(h->part);
    cudaFree(h->part2);
    delete h;
}

int fbank_num_frames(const Fbank* h, int L) {
    if (!h->cfg.snip_edges) {
        if (L <= 0) return 0;
        const int m = int((int64_t(L) + h->shift / 2) / h->shift);
        // the last frame must end inside the reflected waveform (2L samples from the origin on), as _get_strided's view must
        const int64_t end = int64_t(m - 1) * h->shift + h->win + fbank_frame_origin(L, h->win, h->shift, 0);
        return m > 0 && end <= 2 * int64_t(L) ? m : 0;
    }
    if (L < h->win) return 0;
    return 1 + (L - h->win) / h->shift;
}
int fbank_n_mels(const Fbank* h) { return h->cfg.n_mels; }

// raw: scratch [B,T,F] (may equal out_f32).  Exactly one or both of out_f32 / out_pl.
int fbank_run(Fbank* h, const float* wav, const float* lens_ratio, int B, int L, float* raw, float* out_f32,
              const Planes& out_pl, int P, int Tp, cudaStream_t st, const int* valid_frames, const int* num_samples) {
    PPV_REQUIRE(h && wav && raw, "fbank_run: null argument");
    PPV_REQUIRE(B > 0, "fbank_run: empty batch");
    const int T = fbank_num_frames(h, L);
    PPV_REQUIRE(T > 0, "fbank_run: waveform shorter than one frame");
    const int F = h->cfg.n_mels;
    const int nitem = (T + FB_ITEM - 1) / FB_ITEM;
    PPV_REQUIRE(nitem <= FB_PART_ROWS, "fbank_run: utterance too long (more than 524288 frames)");
    const int group = std::max(1, std::min(B, FB_PART_ROWS / nitem));  // utterances per launch group (partial-sum rows)
    const int sms = device_sm_count();
    FbankSmem lay{};
    void (*kern)(const float*, int, int, int, int, int, int, float, float, FbankTables, int, float*, float*, const int*) = nullptr;
    int use_tma = 0, smem = 0;
    FbankFrameArgs fa{};
    if (h->general) {
        smem = fbank_frame_smem_bytes(F);
        PPV_CUDA_OK(cudaFuncSetAttribute(fbank_frame_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
        fa = FbankFrameArgs{h->tb.window, h->twiddle, h->tb.mel_w, h->tb.mel_start, h->tb.mel_len, h->tb.mel_off, h->win, h->shift, h->log2n, F,
                            h->cfg.snip_edges, h->cfg.remove_dc_offset, h->cfg.use_power, h->cfg.use_log_fbank, h->cfg.preemph, h->cfg.log_floor};
    } else {
        lay = fbank_smem_layout(h->tb.nnz, F, h->win, h->shift);
        PPV_REQUIRE(lay.total <= 200 * 1024, "fbank_run: shared memory budget exceeded (frame shift too large)");
        // three CTAs per SM need <= 76 800 B each (228 KB - 1 KB reserved per CTA): 76 784 B for 16 kHz / 25 ms / 10 ms / 80 bins
        const bool vec = (h->shift % 2) == 0;
        kern = (h->win == 400) ? (vec ? fbank_logmel_kernel<true, 400> : fbank_logmel_kernel<false, 400>)
                               : (vec ? fbank_logmel_kernel<true, 0> : fbank_logmel_kernel<false, 0>);
        PPV_CUDA_OK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, lay.total));  // per device: cheap, set every call
        // TMA 1-D bulk copies need 16-byte aligned sources and sizes: every item starts at b * L + 16 k * shift samples
        use_tma = (reinterpret_cast<uintptr_t>(wav) % 16 == 0) && (L % 4 == 0) && ((FB_ITEM * h->shift) % 4 == 0) && (h->shift % 4 == 0) &&
                  (h->win % 4 == 0);
    }
    for (int b0 = 0; b0 < B; b0 += group) {
        const int nb = std::min(group, B - b0);
        const float* w = wav + int64_t(b0) * L;
        float* r = raw + int64_t(b0) * T * F;
        const int* vf = valid_frames ? valid_frames + b0 : (const int*)nullptr;
        if (h->general) {
            PPV_PDL_OK(launch_pdl(fbank_frame_kernel, dim3(nb * nitem), dim3(FG_THREADS), size_t(smem), st, w, L, T, fa,
                                  num_samples ? num_samples + b0 : (const int*)nullptr, r, h->part, vf),
                       "fbank_frame_kernel");
        } else {
            const int grid = std::min(nb * nitem, 3 * sms);
            PPV_PDL_OK(launch_pdl(kern, dim3(grid), dim3(FB_THREADS), size_t(lay.total), st, w, nb, L, T, h->win, h->shift, F, h->cfg.preemph,
                                  h->cfg.log_floor, h->tb, use_tma, r, h->part, vf),
                       "fbank_logmel_kernel");
        }
        const float* sums = h->part;
        int nsum = nitem;
        if (nitem > 64 && nb <= FB_PART_ROWS / 64) {  // long utterances: one row of sums per utterance instead of nitem per finalize block
            PPV_PDL_OK(launch_pdl(fbank_part_reduce_kernel, dim3(nb), dim3(FB_MAX_MELS), 0, st, (const float*)h->part, nitem, h->part2),
                       "fbank_part_reduce_kernel");
            sums = h->part2;
            nsum = 1;
        }
        Planes pl = out_pl;
        if (pl.base) {  // rows of this group start at b0 * Tp
            pl.base += int64_t(b0) * Tp * pl.ld;
        }
        PPV_PDL_OK(launch_pdl(fbank_finalize_kernel, dim3((T + FB_FIN_FRAMES - 1) / FB_FIN_FRAMES, nb), dim3(256), 0, st, (const float*)r, sums,
                              nsum, lens_ratio ? lens_ratio + b0 : (const float*)nullptr, vf, nb, T, F,
                              out_f32 ? out_f32 + int64_t(b0) * T * F : (float*)nullptr, pl, P, Tp),
                   "fbank_finalize_kernel");
    }
    return PPV_OK;
}

}  // namespace ppv
