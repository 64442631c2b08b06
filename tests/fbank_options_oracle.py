"""fp64 numpy statement of the Fbank front end with every option AudioFeaturizer('Fbank') accepts, which csrc/fbank.cu follows:
torchaudio kaldi.py:fbank (the code paddleaudio's kaldi module was ported from) with dither 0, use_energy False and
round_to_power_of_two, over any sample rate and frame length, the five window types and blackman_coeff, snip_edges, remove_dc_offset,
use_power, use_log_fbank, VTLN and subtract_mean.  Keyword names are torchaudio's, which are paddleaudio's except sr (sample_frequency)
and n_mels (num_mel_bins).  It extends oracle/fbank.py (the default configuration) to the other options; tests/test_fbank_options_cpu.py
pins it to torchaudio.compliance.kaldi.fbank in fp64."""
import math

import numpy as np

from oracle.fbank import FLT_EPS, next_pow2, povey_window


def num_frames(num_samples: int, window_size: int = 400, window_shift: int = 160, snip_edges: bool = True) -> int:
    """Frame count of torchaudio kaldi.py:_get_strided.  snip_edges=False: (L + shift // 2) // shift, or 0 when the reflected
    waveform is too short to hold the last frame (where _get_strided's as_strided view fails)."""
    if snip_edges:
        if num_samples < window_size:
            return 0
        return 1 + (num_samples - window_size) // window_shift
    m = (num_samples + window_shift // 2) // window_shift
    if num_samples <= 0 or m <= 0:
        return 0
    return m if (m - 1) * window_shift + window_size <= len(_reflected(num_samples, window_size, window_shift)) else 0


def _reflected(L: int, window_size: int, window_shift: int) -> np.ndarray:
    """snip_edges=False: the sample indices _get_strided frames, as torchaudio builds them: the first min(pad, L) samples reversed
    (edge sample repeated) in front, or the first min(-pad, L) samples dropped, and the whole reversed waveform appended."""
    idx = np.arange(L)
    rev = idx[::-1]
    pad = window_size // 2 - window_shift // 2
    if pad > 0:
        return np.concatenate([rev[-pad:], idx, rev])  # rev[-pad:] is all of rev when pad > L, as in torch
    return np.concatenate([idx[-pad:], rev])


def frame_signal(x: np.ndarray, window_size: int, window_shift: int, snip_edges: bool = True) -> np.ndarray:
    """[L] -> [T, window_size] frames (torchaudio kaldi.py:_get_strided)."""
    T = num_frames(x.shape[0], window_size, window_shift, snip_edges)
    src = np.arange(x.shape[0]) if snip_edges else _reflected(x.shape[0], window_size, window_shift)
    return x[src[np.arange(T)[:, None] * window_shift + np.arange(window_size)[None, :]]]


WINDOW_TYPES = ("povey", "hanning", "hamming", "rectangular", "blackman")


def feature_window(window_type: str, window_size: int, blackman_coeff: float = 0.42, dtype=np.float64) -> np.ndarray:
    """torchaudio kaldi.py:_feature_window_function"""
    n = np.arange(window_size, dtype=np.float64)
    a = 2.0 * math.pi / (window_size - 1)
    if window_type == "povey":
        return povey_window(window_size, dtype)
    if window_type == "hanning":
        w = 0.5 - 0.5 * np.cos(a * n)
    elif window_type == "hamming":
        w = 0.54 - 0.46 * np.cos(a * n)
    elif window_type == "rectangular":
        w = np.ones(window_size)
    elif window_type == "blackman":
        w = blackman_coeff - 0.5 * np.cos(a * n) + (0.5 - blackman_coeff) * np.cos(2 * a * n)
    else:
        raise ValueError(f"unknown window_type {window_type!r}")
    return w.astype(dtype)


def _f32_log(x):
    """float32 log as torch evaluates it: its vectorised log and numpy's differ by an ulp on some inputs, which moves a mel
    weight by up to ~1e-5, so the float32 mel-scale transcendentals go through the same kernels as torchaudio's."""
    import torch
    return torch.from_numpy(np.ascontiguousarray(x, dtype=np.float32)).log().numpy()


def _f32_exp(x):
    import torch
    return torch.from_numpy(np.ascontiguousarray(x, dtype=np.float32)).exp().numpy()


def _vtln_warp_mel(mel, vtln_low, vtln_high, low_freq, high_freq, warp):
    """kaldi.py:vtln_warp_mel_freq in float32 (torch evaluates the tensor side in float32, scalars rounded to it)."""
    f32 = np.float32
    freq = (f32(700.0) * (_f32_exp(mel / f32(1127.0)) - f32(1.0))).astype(f32)
    l_ = vtln_low * max(1.0, warp)
    h_ = vtln_high * min(1.0, warp)
    scale = 1.0 / warp
    scale_left = (scale * l_ - low_freq) / (l_ - low_freq)
    scale_right = (high_freq - scale * h_) / (high_freq - h_)
    res = np.where(freq >= f32(h_), f32(high_freq) + f32(scale_right) * (freq - f32(high_freq)), freq)
    res = np.where(freq < f32(h_), f32(scale) * freq, res)
    res = np.where(freq < f32(l_), f32(low_freq) + f32(scale_left) * (freq - f32(low_freq)), res)
    res = np.where((freq < f32(low_freq)) | (freq > f32(high_freq)), freq, res).astype(f32)
    return (f32(1127.0) * _f32_log(f32(1.0) + res / f32(700.0))).astype(f32)


def mel_banks(num_bins: int, padded_window: int, sample_freq: float,
              low_freq: float = 20.0, high_freq: float = 0.0, dtype=np.float32,
              vtln_low: float = 100.0, vtln_high: float = -500.0, vtln_warp: float = 1.0) -> np.ndarray:
    """Triangular mel filters, [num_bins, padded_window//2 + 1] (last column zero).

    torchaudio kaldi.py:get_mel_banks, VTLN included.  torchaudio evaluates this in float32; we evaluate in float32 as well, with
    its log and exp, so the weights agree bit for bit.
    """
    num_fft_bins = padded_window // 2
    nyquist = 0.5 * sample_freq
    if high_freq <= 0.0:
        high_freq += nyquist
    f32 = np.float32
    fft_bin_width = sample_freq / padded_window
    mel_low = 1127.0 * math.log(1.0 + low_freq / 700.0)
    mel_high = 1127.0 * math.log(1.0 + high_freq / 700.0)
    delta = (mel_high - mel_low) / (num_bins + 1)
    if vtln_high < 0.0:
        vtln_high += nyquist
    b = np.arange(num_bins, dtype=f32)[:, None]
    left = (f32(mel_low) + b * f32(delta)).astype(f32)
    center = (f32(mel_low) + (b + f32(1.0)) * f32(delta)).astype(f32)
    right = (f32(mel_low) + (b + f32(2.0)) * f32(delta)).astype(f32)
    if vtln_warp != 1.0:
        assert low_freq < vtln_low < high_freq and 0.0 < vtln_high < high_freq and vtln_low < vtln_high
        left, center, right = (_vtln_warp_mel(v, vtln_low, vtln_high, low_freq, high_freq, vtln_warp) for v in (left, center, right))
    freqs = (f32(fft_bin_width) * np.arange(num_fft_bins, dtype=f32)).astype(f32)
    mel = (f32(1127.0) * _f32_log(f32(1.0) + freqs / f32(700.0))).astype(f32)[None, :]
    up = (mel - left) / (center - left)
    down = (right - mel) / (right - center)
    if vtln_warp == 1.0:
        bins = np.maximum(f32(0.0), np.minimum(up, down))
    else:
        bins = np.where((mel > left) & (mel <= center), up, np.where((mel > center) & (mel < right), down, f32(0.0)))
    return np.pad(bins.astype(dtype), ((0, 0), (0, 1)))


def kaldi_fbank(waveform: np.ndarray, sr: int = 16000, n_mels: int = 80,
                frame_length_ms: float = 25.0, frame_shift_ms: float = 10.0,
                preemph: float = 0.97, low_freq: float = 20.0, high_freq: float = 0.0,
                log_floor: float = FLT_EPS, dtype=np.float32, window_type: str = "povey",
                blackman_coeff: float = 0.42, remove_dc_offset: bool = True, snip_edges: bool = True,
                use_power: bool = True, use_log_fbank: bool = True, vtln_warp: float = 1.0,
                vtln_low: float = 100.0, vtln_high: float = -500.0, subtract_mean: bool = False) -> np.ndarray:
    """One utterance: waveform [L] -> log-mel [T, n_mels].

    Mirrors torchaudio kaldi.py:fbank (:591-647) / _get_window (:154-217) with dither 0, use_energy False and
    round_to_power_of_two (the reference's defaults, featurizer.py:97, are the keyword defaults here).  ``dtype`` selects the
    arithmetic precision (float32 = what the reference computes in; float64 = "truth").
    """
    x = np.asarray(waveform, dtype=dtype).reshape(-1)
    win = int(sr * frame_length_ms * 0.001)
    shift = int(sr * frame_shift_ms * 0.001)
    padded = next_pow2(win)
    frames = frame_signal(x, win, shift, snip_edges)             # as_strided framing
    if frames.shape[0] == 0:
        return np.zeros((0, n_mels), dtype=dtype)
    if remove_dc_offset:
        frames = frames - frames.mean(axis=1, keepdims=True)
    prev = np.concatenate([frames[:, :1], frames[:, :-1]], axis=1)  # replicate-pad left
    frames = frames - dtype(preemph) * prev                      # pre-emphasis
    frames = frames * feature_window(window_type, win, blackman_coeff, dtype)[None, :]
    frames = np.pad(frames, ((0, 0), (0, padded - win)))         # zero-pad to the FFT size
    spec = np.fft.rfft(frames.astype(np.float64 if dtype == np.float64 else np.float32), axis=1)
    power = (spec.real.astype(dtype) ** 2 + spec.imag.astype(dtype) ** 2).astype(dtype)
    if not use_power:
        power = np.sqrt(power)
    banks = mel_banks(n_mels, padded, float(sr), low_freq, high_freq, np.float32, vtln_low, vtln_high, vtln_warp).astype(dtype)
    mel = power @ banks.T
    if use_log_fbank:
        mel = np.log(np.maximum(mel, dtype(log_floor)))
    if subtract_mean:
        mel = mel - mel.mean(axis=0, keepdims=True)
    return mel.astype(dtype)


def audio_featurizer_fbank(waveforms: np.ndarray, input_lens_ratio=None, dtype=np.float32,
                           **fbank_args) -> np.ndarray:
    """AudioFeaturizer('Fbank').forward  (featurizer.py:33-60): [B,L] -> [B,T,F].

    CMN takes the mean over ALL T frames, including frames that came from zero padding
    (quirk kept, SURVEY.md quirks register); the tail mask (frames t >= int(ratio*T) -> 0)
    is applied AFTER the mean subtraction (featurizer.py:48-59).
    """
    w = np.asarray(waveforms)
    if w.ndim == 1:
        w = w[None, :]
    feats = np.stack([kaldi_fbank(u, dtype=dtype, **fbank_args) for u in w])   # [B,T,F]
    feats = feats - feats.mean(axis=1, keepdims=True)
    if input_lens_ratio is not None:
        T = feats.shape[1]
        # paddle: (ratio * T).astype(int32) -- float32 multiply then truncate
        lens = (np.asarray(input_lens_ratio, dtype=np.float32) * np.float32(T)).astype(np.int32)
        mask = np.arange(T)[None, :] < lens[:, None]
        feats = np.where(mask[:, :, None], feats, 0).astype(dtype)
    return feats.astype(dtype)
