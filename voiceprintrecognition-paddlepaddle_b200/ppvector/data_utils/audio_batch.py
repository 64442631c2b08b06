"""Batched waveform preparation / augmentation on the GPU (libppv_b200 ``ppv_audio_prep`` / ``ppv_audio_prep_reverb``, csrc/audio_prep.cu,
csrc/reverb.cu).

The reference prepares training audio one utterance at a time on the CPU inside DataLoader workers (ppvector/data_utils/reader.py:85-104,
augmentation :143-163 through yeaudio; configs/augmentation.yml).  Here the host only decodes the files and draws the random numbers --
in the reference's order, with Python's ``random`` -- and ONE launch sequence per batch does speed perturbation (linear-interpolation
resampling), volume gain, additive noise at the drawn SNR, reverberation (the full convolution with a drawn room impulse response,
partitioned overlap-save FFT), dB normalisation and the crop.  A batch in which no item drew a response takes ``ppv_audio_prep``
unchanged.  yeaudio is not vendored: the semantics are recalled (SURVEY.md §8c-6) and restated in oracle/audio_prep.py and, for the
reverb, tests/reverb_oracle.py.
"""
import ctypes as C
import os
import random

import numpy as np
import torch

from ppvector import _lib
from ppvector.data_utils.audio import AudioSegment

SPEEDS = (1.0, 0.9, 1.1)


def _conf(sub):
    if sub is None:
        return None
    return dict(sub) if isinstance(sub, dict) else dict(vars(sub))


def load_bank(d, sample_rate, device):
    """Every decodable, non-empty audio file of directory ``d`` in sorted order, resampled to ``sample_rate`` and concatenated into one
    float32 tensor on ``device`` -> (bank or None, [(offset, length)] per clip).  A missing or empty directory gives (None, [])."""
    d = str(d or '')
    files = sorted(os.path.join(d, f) for f in os.listdir(d)) if os.path.isdir(d) else []
    clips, index, off = [], [], 0
    for f in files:
        try:
            seg = AudioSegment.from_file(f)
        except Exception:
            continue
        if seg.sample_rate != sample_rate:
            seg.resample(sample_rate)
        if seg.samples.shape[0] == 0:
            continue
        clips.append(seg.samples)
        index.append((off, seg.samples.shape[0]))
        off += seg.samples.shape[0]
    if not clips:
        return None, []
    return torch.from_numpy(np.concatenate(clips)).to(device), index


class WaveAugmentor:
    """Holds the augmentation configuration (configs/augmentation.yml: speed / volume / noise / reverb), the noise bank and the room
    impulse response bank; ``draw`` makes one utterance's random decisions in the order the reference's augment_audio makes them
    (reader.py:153-163).  Like yeaudio's augmentors, a missing or empty noise_dir / reverb_dir disables that augmentor."""

    def __init__(self, aug_conf=None, num_speakers=None, sample_rate=16000, device='cuda'):
        conf = _conf(aug_conf) or {}
        self.speed, self.volume, self.noise = _conf(conf.get('speed')), _conf(conf.get('volume')), _conf(conf.get('noise'))
        self.reverb = _conf(conf.get('reverb'))
        self.num_speakers = num_speakers
        self.device = torch.device(device)
        self.noise_bank, self.noise_clips = None, []
        if self.noise and self.noise.get('prob', 0) > 0:
            self.noise_bank, self.noise_clips = load_bank(self.noise.get('noise_dir'), sample_rate, self.device)
        self.rir_bank, self.rir_clips = None, []
        if self.reverb and self.reverb.get('prob', 0) > 0:
            self.rir_bank, self.rir_clips = load_bank(self.reverb.get('reverb_dir'), sample_rate, self.device)

    def draw(self, raw_len, spk_id, rng=random):
        """-> dict(speed_rate, spk_id, vol_gain_db, noise=(off, len) or None, snr_db), plus reverb=(off, len) or None when a response
        bank is loaded (without one the dict has no ``reverb`` key and the draw consumes no random numbers for it)."""
        d = dict(speed_rate=1.0, spk_id=spk_id, vol_gain_db=0.0, noise=None, snr_db=0.0)
        if self.speed and rng.random() < self.speed.get('prob', 0.0):
            k = rng.randint(0, 2)
            d['speed_rate'] = SPEEDS[k]
            if self.speed.get('speed_perturb_3_class', False) and self.num_speakers:
                d['spk_id'] = spk_id + self.num_speakers * k
        if self.volume and rng.random() < self.volume.get('prob', 0.0):
            d['vol_gain_db'] = rng.uniform(self.volume.get('min_gain_dBFS', -15), self.volume.get('max_gain_dBFS', 15))
        if self.noise_bank is not None and rng.random() < self.noise.get('prob', 0.0):
            off, n = self.noise_clips[rng.randint(0, len(self.noise_clips) - 1)]
            new_len = raw_len if d['speed_rate'] == 1.0 else int(raw_len / d['speed_rate'])
            start = rng.randint(0, n - new_len) if n > new_len else 0  # a longer clip contributes a random sub-segment, a shorter one is tiled
            d['noise'] = (off + start, n - start if n > new_len else n)
            d['snr_db'] = rng.uniform(self.noise.get('min_snr_dB', 10), self.noise.get('max_snr_dB', 50))
        if self.rir_bank is not None:
            d['reverb'] = rng.choice(self.rir_clips) if rng.random() < self.reverb.get('prob', 0.0) else None
        return d


def augmented_len(raw_len, draw):
    """Length of the augmented utterance before the crop: speed changes it to int(raw_len / rate), a room response of R taps adds R - 1."""
    d = draw or {}
    rate = d.get('speed_rate', 1.0)
    n = raw_len if rate == 1.0 else int(raw_len / rate)
    if d.get('reverb') is not None:
        n += d['reverb'][1] - 1
    return n


def prepare_batch(waves, draws, crops, target_db=-20.0, normalize=True, noise_bank=None, device='cuda', rir_bank=None):
    """waves: list of float32 numpy arrays (already at the target rate); draws: list of WaveAugmentor.draw dicts (or None);
    crops: list of (start, length) on the augmented (speed-changed, reverberant) utterance, length None = to the end; rir_bank: the
    WaveAugmentor's response bank, needed when a draw has a ``reverb`` entry.  Returns (out [B, Lout] CUDA float32, lengths list).
    One H2D copy of the padded batch + three kernels, or six when some item drew a room response."""
    dev = torch.device(device)
    B = len(waves)
    raw_max = max(w.shape[0] for w in waves)
    host = torch.zeros((B, raw_max), dtype=torch.float32).pin_memory()
    ip = np.zeros((B, _lib.PPV_PREP_NI), dtype=np.int32)
    fp = np.zeros((B, _lib.PPV_PREP_NF), dtype=np.float32)
    rp = np.zeros((B, 2), dtype=np.int32)
    out_lens = []
    for b, w in enumerate(waves):
        host[b, :w.shape[0]] = torch.from_numpy(np.ascontiguousarray(w, dtype=np.float32))
        d = draws[b] or {}
        rate = d.get('speed_rate', 1.0)
        raw = w.shape[0]
        new = raw if rate == 1.0 else int(raw / rate)
        if d.get('reverb') is not None:
            off, n = (int(v) for v in d['reverb'])
            if rir_bank is None or n < 1 or off < 0 or off + n > rir_bank.numel():
                raise ValueError(f'prepare_batch: item {b} draws room response {(off, n)} outside the response bank')
            rp[b] = (off, n)
        start, length = crops[b]
        full = augmented_len(raw, d)
        length = full - start if length is None else min(length, full - start)
        ip[b, :4] = (raw, new, start, length)
        if d.get('noise') is not None:
            ip[b, 4:7] = (d['noise'][0], d['noise'][1], 1)
        fp[b, 1], fp[b, 2] = d.get('vol_gain_db', 0.0), d.get('snr_db', 0.0)
        out_lens.append(int(length))
    Lout = max(out_lens)
    new_max = int(ip[:, 1].max())
    rir_max = int(rp[:, 1].max())
    lib = _lib.load()
    with torch.cuda.device(dev):
        wav = host.to(dev, non_blocking=True)
        ipd, fpd = torch.from_numpy(ip).to(dev), torch.from_numpy(fp).to(dev)
        out = torch.empty((B, Lout), dtype=torch.float32, device=dev)
        if rir_max == 0:
            nbytes = lib.ppv_audio_prep_workspace_bytes(B, new_max)
            ws = torch.empty(nbytes, dtype=torch.uint8, device=dev)
            _lib.check(lib.ppv_audio_prep(_lib.ptr(wav), raw_max, _lib.ptr(ipd), _lib.ptr(fpd), _lib.ptr(noise_bank), B, new_max,
                                          float(target_db), 1 if normalize else 0, Lout, _lib.ptr(out), C.c_void_p(ws.data_ptr()), nbytes,
                                          _lib.current_stream()), 'ppv_audio_prep')
        else:
            _lib.require_cuda(rir_bank, 'rir_bank')
            rpd = torch.from_numpy(rp).to(dev)
            nbytes = lib.ppv_audio_prep_reverb_workspace_bytes(B, new_max, rir_max)
            ws = torch.empty(nbytes, dtype=torch.uint8, device=dev)
            _lib.check(lib.ppv_audio_prep_reverb(_lib.ptr(wav), raw_max, _lib.ptr(ipd), _lib.ptr(fpd), _lib.ptr(noise_bank), _lib.ptr(rir_bank),
                                                 rir_bank.numel(), _lib.ptr(rpd), B, new_max, rir_max, float(target_db), 1 if normalize else 0,
                                                 Lout, _lib.ptr(out), C.c_void_p(ws.data_ptr()), nbytes, _lib.current_stream()),
                       'ppv_audio_prep_reverb')
    return out, out_lens
