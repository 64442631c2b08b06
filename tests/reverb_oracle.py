"""Oracle of the reverb step of the training data path (numpy / scipy, fp64), used by tests/test_reverb_prep.py and
tests/test_gpu_reverb.py.

PARITY UNPINNED, like oracle/audio_prep.py: yeaudio is not vendored, and what is restated here is its RECALLED
ReverbPerturbAugmentor(reverb_dir, prob), the fourth step of reader.py:153-163's augment_audio (speed -> volume -> noise -> reverb),
followed by normalize(target_db) and the crop (reader.py:96-101):

  files     every file in reverb_dir; a missing or empty directory disables the augmentor
  draw      random.random() < prob applies it; random.choice(files) picks the response
  resample  the response is resampled to the utterance's rate when its rate differs
  convolve  samples = scipy.signal.fftconvolve(samples, rir, "full"): NOT truncated, the utterance grows by len(rir) - 1 samples;
            neither the response nor the result is normalised beyond the usual normalize(target_db) afterwards

So with dB normalisation on only the response's shape and length matter; with it off the raw convolution is the output.
``prepare_reverb`` is oracle/audio_prep.prepare with the convolution inserted after the noise.
"""
import numpy as np
import scipy.signal

from oracle.audio_prep import change_speed, rms_db

DIRECT_MAX_MACS = 2e7  # below this many multiply-adds the full convolution is summed directly (np.convolve), above it through fp64 FFTs


def reverb_convolve(y, rir):
    y = np.asarray(y, dtype=np.float64)
    h = np.asarray(rir, dtype=np.float64)
    if y.shape[0] * h.shape[0] <= DIRECT_MAX_MACS:
        return np.convolve(y, h, mode="full")
    return scipy.signal.fftconvolve(y, h, mode="full")


def prepare_reverb(x, speed_rate=1.0, vol_gain_db=0.0, noise=None, noise_off=0, snr_db=None, rir=None, target_db=-20.0, normalize=True,
                   crop_start=0, crop_len=None, out_len=None):
    """One utterance through speed -> volume -> noise -> reverb -> dB normalise -> crop -> zero-pad; float64 inside, float32 out.
    ``noise`` is the clip segment the draw selected (tiled from ``noise_off``); ``rir`` None = no reverb."""
    y = change_speed(np.asarray(x, dtype=np.float32), speed_rate).astype(np.float64)
    y = y * 10.0 ** (vol_gain_db / 20.0)
    if noise is not None:
        n = np.asarray(noise, dtype=np.float64)
        seg = n[(noise_off + np.arange(y.shape[0])) % n.shape[0]]
        g = min(rms_db(y) - rms_db(seg) - snr_db, 300.0)
        y = y + seg * 10.0 ** (g / 20.0)
    if rir is not None:
        y = reverb_convolve(y, rir)
    if normalize:
        y = y * 10.0 ** (min(target_db - rms_db(y), 300.0) / 20.0)
    crop_len = y.shape[0] - crop_start if crop_len is None else crop_len
    y = y[crop_start:crop_start + crop_len]
    out_len = y.shape[0] if out_len is None else out_len
    out = np.zeros(out_len, dtype=np.float32)
    out[:y.shape[0]] = y.astype(np.float32)
    return out
