"""fp64 numpy statement of the energy voice-activity detection (DESIGN.md §1, f8) that csrc/vad.cu and ppvector/infer_utils/vad.py
follow: Kaldi's compute-vad (ComputeVadEnergy) on the raw log energy of each snip_edges frame, then the runs of voiced frames turned
into segments in integer samples."""
import numpy as np

FLT_EPSILON = float(np.finfo(np.float32).eps)
DEFAULTS = dict(energy_threshold=5.5, energy_mean_scale=0.5, frames_context=2, proportion_threshold=0.12,
                min_speech_ms=250, min_silence_ms=100, speech_pad_ms=30)


def geometry(sample_rate):
    """(win, shift) = (int(sample_rate * 0.025), int(sample_rate * 0.010)) in samples."""
    return int(sample_rate) * 25 // 1000, int(sample_rate) * 10 // 1000


def num_frames(L, win, shift):
    return 0 if L < win else 1 + (L - win) // shift


def log_energy(x, win, shift, block=8192):
    """e_t = ln(max(32768^2 * sum_{n < win} (x[t*shift + n] - mean_t)^2, FLT_EPSILON)) in fp64, mean_t the frame's own mean."""
    x = np.asarray(x, dtype=np.float64).reshape(-1)
    T = num_frames(x.size, win, shift)
    e = np.empty(T, dtype=np.float64)
    for t0 in range(0, T, block):  # in blocks of frames, so an hour of audio does not need [T, win] at once
        t = np.arange(t0, min(T, t0 + block))
        fr = x[t[:, None] * shift + np.arange(win)[None, :]]
        fr = fr - fr.mean(axis=1, keepdims=True)
        e[t] = np.log(np.maximum(32768.0 ** 2 * (fr * fr).sum(axis=1), FLT_EPSILON))
    return e


def threshold(e, energy_threshold=5.5, energy_mean_scale=0.5):
    """thr = energy_threshold + energy_mean_scale * (sum_t e_t) / T; the options are fp32 (as the C ABI holds them), the sum fp64."""
    total = float(np.cumsum(e)[-1]) if len(e) else 0.0  # frame order
    return float(np.float32(energy_threshold)) + float(np.float32(energy_mean_scale)) * total / max(len(e), 1)


def decide(e, thr, frames_context=2, proportion_threshold=0.12):
    """voiced_t iff num >= den * proportion_threshold, the product in fp32; den counts the frames within frames_context of t inside
    [0, T), num those of them with e > thr."""
    T = len(e)
    above = np.concatenate([[0], np.cumsum(np.asarray(e) > thr)])
    t = np.arange(T)
    lo, hi = np.maximum(t - frames_context, 0), np.minimum(t + frames_context, T - 1)
    num, den = above[hi + 1] - above[lo], hi - lo + 1
    return num.astype(np.float32) >= den.astype(np.float32) * np.float32(proportion_threshold)


def runs(voiced):
    """Maximal runs of voiced frames -> [(first_frame, end_frame), ...]."""
    d = np.diff(np.concatenate([[0], np.asarray(voiced, dtype=np.int8), [0]]))
    return list(zip(np.flatnonzero(d == 1).tolist(), np.flatnonzero(d == -1).tolist()))


def segments(run_list, L, sample_rate, min_speech_ms=250, min_silence_ms=100, speech_pad_ms=30):
    """Run [a, b) -> samples [a*shift, (b-1)*shift + win); merge gaps < min_silence, drop runs < min_speech, pad (gap // 2 each where the
    gap is under two pads), clamp to [0, L].  Durations in samples are sample_rate * ms // 1000."""
    win, shift = geometry(sample_rate)
    ms = lambda v: int(sample_rate * v // 1000)  # noqa: E731
    spans = [[a * shift, (b - 1) * shift + win] for a, b in run_list]
    merged = spans[:1]
    for s in spans[1:]:
        if s[0] - merged[-1][1] < ms(min_silence_ms):
            merged[-1] = [merged[-1][0], max(merged[-1][1], s[1])]
        else:
            merged.append(s)
    kept = [s for s in merged if s[1] - s[0] >= ms(min_speech_ms)]
    pad = ms(speech_pad_ms)
    out = [list(s) for s in kept]
    for i in range(len(kept) - 1):
        gap = kept[i + 1][0] - kept[i][1]
        move = pad if gap >= 2 * pad else gap // 2
        out[i][1] += move
        out[i + 1][0] -= move
    if out:
        out[0][0] -= pad
        out[-1][1] += pad
    return [{'start': max(0, s), 'end': min(L, e)} for s, e in out]


def vad(x, sample_rate=16000, **opts):
    """-> dict(e, thr, voiced, runs, segments) of one recording (segments in samples)."""
    o = {**DEFAULTS, **opts}
    win, shift = geometry(sample_rate)
    e = log_energy(x, win, shift)
    thr = threshold(e, o['energy_threshold'], o['energy_mean_scale'])
    v = decide(e, thr, o['frames_context'], o['proportion_threshold'])
    r = runs(v)
    seg = segments(r, len(x), sample_rate, o['min_speech_ms'], o['min_silence_ms'], o['speech_pad_ms'])
    return dict(e=e, thr=thr, voiced=v, runs=r, segments=seg)
