"""Energy voice-activity detection in front of speaker diarization (DESIGN.md §1, f8).

The reference finds the speech with silero-vad (``AudioSegment.vad`` of yeaudio, a neural network whose weights ship inside that
package).  This build runs the classical energy VAD of Kaldi instead (``compute-vad``, the VAD of Kaldi's x-vector recipes):
  * per 25 ms / 10 ms snip_edges frame, the raw log energy on Kaldi's 16-bit scale, ln(max(32768^2 * sum (x - mean)^2, FLT_EPSILON));
  * a frame is voiced when at least ``proportion_threshold`` of the frames within ``frames_context`` of it have an energy above
    ``energy_threshold + energy_mean_scale * mean(log energy)``.
Both run on the GPU for a whole batch of recordings in one launch sequence (csrc/vad.cu, ``ppv_vad_energy``).  The runs of voiced
frames then become segments on the host, in integer samples: neighbours closer than ``min_silence_ms`` are merged, runs shorter
than ``min_speech_ms`` dropped, and the rest padded by ``speech_pad_ms`` (half the gap where two runs are closer than two pads).  Those
three knobs borrow the names and defaults of silero-vad's ``get_speech_timestamps``.
"""
import ctypes as C
import math

import numpy as np
import torch

from ppvector import _lib

__all__ = ['DECISION_DEFAULTS', 'SEGMENT_DEFAULTS', 'energy_vad', 'frame_geometry', 'speech_segments', 'vad_options', 'voiced_runs']

# Kaldi's VoxCeleb / SRE16 x-vector recipes, conf/vad.conf
DECISION_DEFAULTS = {'energy_threshold': 5.5, 'energy_mean_scale': 0.5, 'frames_context': 2, 'proportion_threshold': 0.12}
# silero-vad's get_speech_timestamps
SEGMENT_DEFAULTS = {'min_speech_ms': 250, 'min_silence_ms': 100, 'speech_pad_ms': 30}


def vad_options(**opts) -> dict:
    """The VAD options with their defaults filled in; unknown names raise TypeError, values out of range ValueError."""
    unknown = sorted(set(opts) - set(DECISION_DEFAULTS) - set(SEGMENT_DEFAULTS))
    if unknown:
        raise TypeError(f'unknown VAD option(s) {unknown}; known: {sorted(DECISION_DEFAULTS) + sorted(SEGMENT_DEFAULTS)}')
    o = {**DECISION_DEFAULTS, **SEGMENT_DEFAULTS, **opts}
    if not math.isfinite(o['energy_threshold']):
        raise ValueError(f"energy_threshold must be finite, got {o['energy_threshold']}")
    if not (o['energy_mean_scale'] >= 0 and math.isfinite(o['energy_mean_scale'])):
        raise ValueError(f"energy_mean_scale must be >= 0, got {o['energy_mean_scale']}")
    if int(o['frames_context']) != o['frames_context'] or o['frames_context'] < 0:
        raise ValueError(f"frames_context must be an integer >= 0, got {o['frames_context']}")
    if not 0 < o['proportion_threshold'] < 1:
        raise ValueError(f"proportion_threshold must lie in (0, 1), got {o['proportion_threshold']}")
    for k in SEGMENT_DEFAULTS:
        if not o[k] >= 0:
            raise ValueError(f'{k} must be >= 0, got {o[k]}')
    o['frames_context'] = int(o['frames_context'])
    return o


def frame_geometry(sample_rate):
    """(window, shift) in samples: 25 ms and 10 ms frames, rounded down (400 / 160 at 16 kHz)."""
    return int(sample_rate) * 25 // 1000, int(sample_rate) * 10 // 1000


def _ms_to_samples(ms, sample_rate):
    return int(sample_rate * ms // 1000)


def speech_segments(runs, n_samples, sample_rate, min_speech_ms=250, min_silence_ms=100, speech_pad_ms=30):
    """Runs of voiced frames [(first_frame, end_frame), ...] of one recording of ``n_samples`` samples -> [{'start', 'end'}, ...] in samples.
    Run [a, b) covers samples [a * shift, (b - 1) * shift + window); then, in this order: merge neighbours whose gap is shorter than
    min_silence_ms, drop runs shorter than min_speech_ms, pad each side by speech_pad_ms (by gap // 2 where the gap to the neighbour
    is shorter than two pads), clamped to [0, n_samples]."""
    window, shift = frame_geometry(sample_rate)
    min_silence, min_speech = _ms_to_samples(min_silence_ms, sample_rate), _ms_to_samples(min_speech_ms, sample_rate)
    pad = _ms_to_samples(speech_pad_ms, sample_rate)
    merged = []
    for a, b in runs:
        s, e = int(a) * shift, (int(b) - 1) * shift + window
        if merged and s - merged[-1][1] < min_silence:
            merged[-1][1] = max(merged[-1][1], e)
        else:
            merged.append([s, e])
    kept = [m for m in merged if m[1] - m[0] >= min_speech]
    out = []
    for i, (s, e) in enumerate(kept):
        left = pad if i == 0 else min(pad, (s - kept[i - 1][1]) // 2)
        right = pad if i == len(kept) - 1 else min(pad, (kept[i + 1][0] - e) // 2)
        out.append({'start': max(0, s - left), 'end': min(int(n_samples), e + right)})
    return out


def _host_f32(x):
    if torch.is_tensor(x):
        x = x.detach().cpu().numpy()
    return np.ascontiguousarray(np.asarray(x, dtype=np.float32).reshape(-1))


def _launch(recordings, sample_rate, o, frames):
    """One H2D copy of the concatenated batch and one ppv_vad_energy call -> (lengths, per-recording results): the
    (log_energy fp64, voiced bool) frame arrays with frames=True, else the lists of voiced runs (first_frame, end_frame)."""
    lib = _lib.load()
    cfg = _lib.VadCfg()
    lib.ppv_vad_default_cfg(C.byref(cfg), int(sample_rate))
    for k in DECISION_DEFAULTS:
        setattr(cfg, k, o[k])
    xs = [_host_f32(x) for x in recordings]
    R = len(xs)
    lengths = np.array([x.size for x in xs], dtype=np.int64)
    if R == 0:
        return lengths, []
    offsets = np.zeros(R + 1, dtype=np.int64)
    np.cumsum(lengths, out=offsets[1:])
    T = np.array([lib.ppv_vad_num_frames(C.byref(cfg), int(n)) for n in lengths], dtype=np.int64)
    if (T < 0).any():
        raise _lib.PPVError(f'ppv_vad_num_frames: frame geometry out of range at sample_rate {sample_rate}')
    frame_off = np.zeros(R + 1, dtype=np.int64)
    np.cumsum(T, out=frame_off[1:])
    run_cap = int(((T + 1) // 2).sum())
    dev = torch.device('cuda', torch.cuda.current_device())
    host = np.zeros(max(int(offsets[-1]), 4), dtype=np.float32)  # never an empty (null) buffer
    if offsets[-1]:
        np.concatenate(xs, out=host[:offsets[-1]])
    wav = torch.from_numpy(host).to(dev)
    voiced = torch.empty(max(int(frame_off[-1]), 1), dtype=torch.uint8, device=dev)
    energy = torch.empty(max(int(frame_off[-1]), 1), dtype=torch.float64, device=dev) if frames else None
    runs = torch.empty((max(run_cap, 1), 3), dtype=torch.int32, device=dev)
    n_runs = torch.zeros(1, dtype=torch.int32, device=dev)
    nbytes = lib.ppv_vad_workspace_bytes(C.byref(cfg), R, int(offsets[-1]))
    ws = torch.empty(max(int(nbytes), 1), dtype=torch.uint8, device=dev)
    with torch.cuda.device(dev):
        _lib.check(lib.ppv_vad_energy(C.byref(cfg), _lib.ptr(wav), offsets.ctypes.data_as(C.POINTER(C.c_int64)), R, _lib.ptr(energy),
                                      _lib.ptr(voiced), _lib.ptr(runs), run_cap, _lib.ptr(n_runs), C.c_void_p(ws.data_ptr()), nbytes,
                                      _lib.current_stream()), 'ppv_vad_energy')
    if frames:
        e, v = energy.cpu().numpy(), voiced.cpu().numpy().astype(bool)
        return lengths, [(e[frame_off[r]:frame_off[r + 1]], v[frame_off[r]:frame_off[r + 1]]) for r in range(R)]
    per = [[] for _ in range(R)]
    for r, a, b in runs[:int(n_runs.item())].cpu().numpy().tolist():
        per[r].append((a, b))
    return lengths, per


def voiced_runs(recordings, sample_rate=16000, **opts):
    """Per recording, the maximal runs of voiced frames [(first_frame, end_frame), ...] (before any post-processing)."""
    return _launch(recordings, sample_rate, vad_options(**opts), frames=False)[1]


def energy_vad(recordings, sample_rate=16000, frames=False, return_seconds=False, **opts):
    """A list of 1-D float32 recordings (numpy arrays or tensors, as ``_load_audio`` leaves them) -> one list of {'start', 'end'} per
    recording, in samples (or seconds, ``sample / sample_rate``, with return_seconds=True).  The whole batch goes to the device in one
    copy and through one ``ppv_vad_energy`` call; the run list comes back and is turned into segments on the host (speech_segments).
    frames=True returns (log_energy fp64 [T], voiced bool [T]) per recording instead.  Options: vad_options."""
    o = vad_options(**opts)
    lengths, res = _launch(recordings, sample_rate, o, frames)
    if frames:
        return res
    out = []
    for n, runs in zip(lengths.tolist(), res):
        segs = speech_segments(runs, n, sample_rate, o['min_speech_ms'], o['min_silence_ms'], o['speech_pad_ms'])
        if return_seconds:
            segs = [{'start': s['start'] / sample_rate, 'end': s['end'] / sample_rate} for s in segs]
        out.append(segs)
    return out
