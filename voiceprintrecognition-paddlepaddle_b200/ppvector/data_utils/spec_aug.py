"""SpecAugmentor -- the masking the reference applies to training features (ppvector/data_utils/reader.py:105-107,
``yeaudio.augmentation.SpecAugmentor(**aug_conf.spec_aug)``, parameters configs/augmentation.yml:36-48), batched on the GPU.

The reference masks one [T, F] numpy feature at a time on the CPU inside the DataLoader worker.  Here the random draws stay on
the host, made per utterance in the same order with Python's ``random`` (apply?, frequency-mask widths/starts, time-mask
widths/starts), and one kernel (``ppv_spec_augment``, csrc/spectral.cu) writes all bands of the whole [B, T, F] batch in place.
yeaudio is not vendored: the band semantics (width ~ U[0, ratio * size], start ~ U[0, size - width], zero fill unless
``replace_with_zero=False`` -> utterance mean) are recalled, SURVEY.md §8c(6).  ``max_time_warp`` must be 0
(the shipped configuration); time warping is not implemented.
"""
import random

import torch

from ppvector import _lib


class SpecAugmentor:
    def __init__(self, prob=0.5, freq_mask_ratio=0.15, n_freq_masks=2, time_mask_ratio=0.05, n_time_masks=2, inplace=True,
                 max_time_warp=0, replace_with_zero=True):
        if max_time_warp:
            raise NotImplementedError('SpecAugmentor on the H100 path: max_time_warp must be 0 (configs/augmentation.yml:48)')
        if 2 + 2 * (n_freq_masks + n_time_masks) > _lib.PPV_SPECAUG_NPARAM:
            raise ValueError('too many masks')
        self.prob, self.freq_mask_ratio, self.n_freq_masks = prob, freq_mask_ratio, n_freq_masks
        self.time_mask_ratio, self.n_time_masks = time_mask_ratio, n_time_masks
        self.inplace, self.replace_with_zero = inplace, replace_with_zero

    def draw(self, num_frames, num_bins, rng=random):
        """One utterance's parameter row: [apply, T_b, (f0, fw) * n_freq, (t0, tw) * n_time], zero padded."""
        row = [0] * _lib.PPV_SPECAUG_NPARAM
        row[1] = int(num_frames)
        if rng.random() >= self.prob:
            return row
        row[0] = 1
        k = 2
        for _ in range(self.n_freq_masks):
            w = int(rng.uniform(0, num_bins * self.freq_mask_ratio))
            row[k], row[k + 1] = rng.randint(0, num_bins - w), w
            k += 2
        for _ in range(self.n_time_masks):
            w = int(rng.uniform(0, num_frames * self.time_mask_ratio))
            row[k], row[k + 1] = rng.randint(0, max(num_frames - w, 0)), w
            k += 2
        return row

    def apply(self, features, params):
        """features [B,T,F] float32 CUDA, params int32 [B, PPV_SPECAUG_NPARAM] (host or device) -> masked features"""
        _lib.require_cuda(features, 'features')
        x = features if self.inplace else features.clone()
        x = x.contiguous()
        B, T, F = x.shape
        p = torch.as_tensor(params, dtype=torch.int32).to(x.device).contiguous()
        assert p.shape == (B, _lib.PPV_SPECAUG_NPARAM)
        with torch.cuda.device(x.device):
            _lib.check(_lib.load().ppv_spec_augment(_lib.ptr(x), _lib.ptr(p), B, T, F, self.n_freq_masks, self.n_time_masks,
                                                    0 if self.replace_with_zero else 1, _lib.current_stream()), 'ppv_spec_augment')
        return x

    def __call__(self, features, num_frames=None, rng=random):
        """Mask a batch [B,T,F] (or one [T,F] feature); ``num_frames`` = true frame count per utterance (default T)."""
        single = features.dim() == 2
        x = features.unsqueeze(0) if single else features
        B, T, F = x.shape
        nf = [T] * B if num_frames is None else [int(n) for n in num_frames]
        y = self.apply(x, [self.draw(nf[b], F, rng) for b in range(B)])
        return y.squeeze(0) if single else y
