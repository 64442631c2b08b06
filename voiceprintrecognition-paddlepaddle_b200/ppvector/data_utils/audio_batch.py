"""Batched waveform preparation / augmentation on the GPU (libppv_b200 ``ppv_audio_prep``, csrc/audio_prep.cu).

The reference prepares training audio one utterance at a time on the CPU inside DataLoader workers (ppvector/data_utils/reader.py:85-104,
augmentation :143-163 through yeaudio; configs/augmentation.yml).  Here the host only decodes the files and draws the random numbers --
in the reference's order, with Python's ``random`` -- and ONE launch sequence per batch does speed perturbation (linear-interpolation
resampling), volume gain, additive noise at the drawn SNR, dB normalisation and the crop.  Reverberation (an FIR convolution with a room
response, ``reverb`` in augmentation.yml) is not implemented: a config that enables it raises.  yeaudio is not vendored: the semantics are
recalled (SURVEY.md §8c-6) and restated in oracle/audio_prep.py.
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


class WaveAugmentor:
    """Holds the augmentation configuration (configs/augmentation.yml: speed / volume / noise) and the noise bank; ``draw`` makes one
    utterance's random decisions in the order the reference's augment_audio makes them (reader.py:153-163)."""

    def __init__(self, aug_conf=None, num_speakers=None, sample_rate=16000, device='cuda'):
        conf = _conf(aug_conf) or {}
        self.speed, self.volume, self.noise = _conf(conf.get('speed')), _conf(conf.get('volume')), _conf(conf.get('noise'))
        reverb = _conf(conf.get('reverb'))
        if reverb and reverb.get('prob', 0) > 0 and os.path.isdir(str(reverb.get('reverb_dir', ''))) and os.listdir(reverb['reverb_dir']):
            raise NotImplementedError('reverb augmentation is not implemented on the H100 path; set reverb.prob to 0')
        self.num_speakers = num_speakers
        self.device = torch.device(device)
        self.noise_bank, self.noise_clips = None, []
        if self.noise and self.noise.get('prob', 0) > 0:
            d = str(self.noise.get('noise_dir', ''))
            files = sorted(os.path.join(d, f) for f in os.listdir(d)) if os.path.isdir(d) else []
            clips, off = [], 0
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
                self.noise_clips.append((off, seg.samples.shape[0]))
                off += seg.samples.shape[0]
            if clips:  # like yeaudio: an empty / missing noise_dir disables the augmentor
                self.noise_bank = torch.from_numpy(np.concatenate(clips)).to(self.device)

    def draw(self, raw_len, spk_id, rng=random):
        """-> dict(speed_rate, spk_id, vol_gain_db, noise=(off, len) or None, snr_db)"""
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
        return d


def prepare_batch(waves, draws, crops, target_db=-20.0, normalize=True, noise_bank=None, device='cuda'):
    """waves: list of float32 numpy arrays (already at the target rate); draws: list of WaveAugmentor.draw dicts (or None);
    crops: list of (start, length) on the augmented utterance, length None = to the end.  Returns (out [B, Lout] CUDA float32,
    lengths list).  One H2D copy of the padded batch + three kernels."""
    dev = torch.device(device)
    B = len(waves)
    raw_max = max(w.shape[0] for w in waves)
    host = torch.zeros((B, raw_max), dtype=torch.float32).pin_memory()
    ip = np.zeros((B, _lib.PPV_PREP_NI), dtype=np.int32)
    fp = np.zeros((B, _lib.PPV_PREP_NF), dtype=np.float32)
    out_lens = []
    for b, w in enumerate(waves):
        host[b, :w.shape[0]] = torch.from_numpy(np.ascontiguousarray(w, dtype=np.float32))
        d = draws[b] or {}
        rate = d.get('speed_rate', 1.0)
        raw = w.shape[0]
        new = raw if rate == 1.0 else int(raw / rate)
        start, length = crops[b]
        length = new - start if length is None else min(length, new - start)
        ip[b, :4] = (raw, new, start, length)
        if d.get('noise') is not None:
            ip[b, 4:7] = (d['noise'][0], d['noise'][1], 1)
        fp[b, 1], fp[b, 2] = d.get('vol_gain_db', 0.0), d.get('snr_db', 0.0)
        out_lens.append(int(length))
    Lout = max(out_lens)
    new_max = int(ip[:, 1].max())
    lib = _lib.load()
    with torch.cuda.device(dev):
        wav = host.to(dev, non_blocking=True)
        ipd, fpd = torch.from_numpy(ip).to(dev), torch.from_numpy(fp).to(dev)
        out = torch.empty((B, Lout), dtype=torch.float32, device=dev)
        nbytes = lib.ppv_audio_prep_workspace_bytes(B, new_max)
        ws = torch.empty(nbytes, dtype=torch.uint8, device=dev)
        _lib.check(lib.ppv_audio_prep(_lib.ptr(wav), raw_max, _lib.ptr(ipd), _lib.ptr(fpd), _lib.ptr(noise_bank), B, new_max, float(target_db),
                                      1 if normalize else 0, Lout, _lib.ptr(out), C.c_void_p(ws.data_ptr()), nbytes, _lib.current_stream()),
                   'ppv_audio_prep')
    return out, out_lens
