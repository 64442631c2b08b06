"""AudioFeaturizer -- drop-in for ppvector/data_utils/featurizer.py:7-80 of the reference.

Same constructor (``feature_method``, ``method_args``), same ``forward(waveforms, input_lens_ratio=None)``
contract ([B,L] or [L] float32 in [-1,1] -> [B,T,F] float32, per-utterance time mean subtracted, optional
tail mask applied after the mean subtraction), same ``feature_dim`` property.  The arithmetic runs in one
fused CUDA kernel family behind the C ABI: ``csrc/fbank.cu`` (``ppv_fbank_forward``) for ``Fbank``, ``csrc/spectral.cu``
(``ppv_spectral_forward``) for the ``paddle.audio.features`` methods (Spectrogram, MelSpectrogram, LogMelSpectrogram, MFCC).
"""
import ctypes as C

import torch

from ppvector import _lib


class AudioFeaturizer(torch.nn.Module):
    """reference: featurizer.py:16-31 (constructor dispatch on feature_method)"""

    def __init__(self, feature_method='MelSpectrogram', method_args={}):
        super().__init__()
        self._method_args = dict(method_args or {})
        self._feature_method = feature_method
        self._handle = None
        if feature_method == 'Fbank':
            self._cfg = self._fbank_cfg(self._method_args)
        elif feature_method in self._SPECTRAL:
            self._cfg = self._spectral_cfg(feature_method, self._method_args)
        else:
            raise Exception(f'预处理方法 {self._feature_method} 不存在!')  # featurizer.py:31

    _SPECTRAL = {'Spectrogram': _lib.PPV_SPEC_SPECTROGRAM, 'MelSpectrogram': _lib.PPV_SPEC_MEL,
                 'LogMelSpectrogram': _lib.PPV_SPEC_LOGMEL, 'MFCC': _lib.PPV_SPEC_MFCC}

    @classmethod
    def _spectral_cfg(cls, method, args):
        """paddle.audio.features.<method>(**method_args) keyword names -> ppv_spectral_cfg"""
        lib = _lib.load()
        cfg = _lib.SpectralCfg()
        lib.ppv_spectral_default_cfg(C.byref(cfg), cls._SPECTRAL[method])
        direct = {'sr': 'sample_rate', 'n_fft': 'n_fft', 'hop_length': 'hop_length', 'power': 'power', 'n_mels': 'n_mels',
                  'f_min': 'f_min', 'ref_value': 'ref_value', 'amin': 'amin', 'n_mfcc': 'n_mfcc'}
        for k, v in args.items():
            if k in direct:
                setattr(cfg, direct[k], type(getattr(cfg, direct[k]))(v))
            elif k == 'win_length':
                cfg.win_length = 0 if v is None else int(v)
            elif k == 'f_max':
                cfg.f_max = 0.0 if v is None else float(v)
            elif k == 'htk':
                cfg.htk = int(bool(v))
            elif k == 'norm':
                if v not in ('slaney', None):
                    raise _lib.PPVError(f'{method}: norm={v!r} is not supported by the CUDA kernel (slaney or None)')
                cfg.norm_slaney = int(v == 'slaney')
            elif k == 'center':
                cfg.center = int(bool(v))
            elif k == 'window' and v == 'hann' or k == 'pad_mode' and v == 'reflect' or k == 'dtype' and v == 'float32' \
                    or k == 'top_db' and v is None:
                pass
            else:
                raise _lib.PPVError(f'{method} argument {k}={v!r} is not supported by the CUDA kernel')
        return cfg

    # paddleaudio.compliance.kaldi.fbank keyword names (featurizer.py:97: Kaldi.fbank(waveform, **kwargs)); they are torchaudio's
    # except sr (sample_frequency) and n_mels (num_mel_bins)
    _FBANK_DIRECT = {'sr': 'sample_rate', 'n_mels': 'n_mels', 'frame_length': 'frame_length_ms', 'frame_shift': 'frame_shift_ms',
                     'preemphasis_coefficient': 'preemph', 'low_freq': 'low_freq', 'high_freq': 'high_freq',
                     'blackman_coeff': 'blackman_coeff', 'vtln_warp': 'vtln_warp', 'vtln_low': 'vtln_low', 'vtln_high': 'vtln_high'}
    _FBANK_FLAGS = ('remove_dc_offset', 'snip_edges', 'use_power', 'use_log_fbank')
    _FBANK_WINDOWS = {'povey': _lib.PPV_FBANK_WIN_POVEY, 'hanning': _lib.PPV_FBANK_WIN_HANNING, 'hamming': _lib.PPV_FBANK_WIN_HAMMING,
                      'rectangular': _lib.PPV_FBANK_WIN_RECTANGULAR, 'blackman': _lib.PPV_FBANK_WIN_BLACKMAN}
    # these only shape the energy column (use_energy) or repeat the time-mean subtraction forward() applies anyway
    _FBANK_NO_EFFECT = ('htk_compat', 'raw_energy', 'energy_floor', 'subtract_mean')

    @classmethod
    def _fbank_cfg(cls, args):
        lib = _lib.load()
        cfg = _lib.FbankCfg()
        lib.ppv_fbank_default_cfg(C.byref(cfg))
        cfg.n_mels = 23  # paddleaudio kaldi.fbank default when n_mels is not given (cf. feature_dim, featurizer.py:77)
        for k, v in args.items():
            if k in cls._FBANK_DIRECT:
                setattr(cfg, cls._FBANK_DIRECT[k], type(getattr(cfg, cls._FBANK_DIRECT[k]))(v))
            elif k in cls._FBANK_FLAGS:
                setattr(cfg, k, int(bool(v)))
            elif k == 'window_type':
                if v not in cls._FBANK_WINDOWS:
                    raise _lib.PPVError(f'Fbank: unknown window_type {v!r} (one of {", ".join(cls._FBANK_WINDOWS)})')
                cfg.window_type = cls._FBANK_WINDOWS[v]
            elif k in cls._FBANK_NO_EFFECT:
                pass
            elif k == 'dither':
                if v != 0:
                    raise _lib.PPVError('Fbank: dither != 0 is not supported: its noise comes from Paddle\'s random generator and cannot '
                                        'be reproduced')
            elif k == 'use_energy':
                if v:
                    raise _lib.PPVError('Fbank: use_energy=True is not supported: kaldi emits n_mels + 1 columns while feature_dim reports '
                                        'n_mels, so the model\'s first layer would reject the features (the reference fails the same way)')
            elif k == 'round_to_power_of_two':
                if not v:
                    raise _lib.PPVError('Fbank: round_to_power_of_two=False is not supported: the FFT size must be a power of two')
            else:
                raise _lib.PPVError(f'Fbank argument {k!r} is not supported by the CUDA kernel')
        return cfg

    def _get_handle(self):
        if self._handle is None:
            lib = _lib.load()
            h = C.c_void_p()
            if self._feature_method == 'Fbank':
                _lib.check(lib.ppv_fbank_create(C.byref(self._cfg), C.byref(h)), 'ppv_fbank_create')
            else:
                _lib.check(lib.ppv_spectral_create(C.byref(self._cfg), C.byref(h)), 'ppv_spectral_create')
            self._handle = h
        return self._handle

    def __del__(self):
        try:
            if self._handle is not None:
                lib = _lib.load()
                (lib.ppv_fbank_destroy if self._feature_method == 'Fbank' else lib.ppv_spectral_destroy)(self._handle)
                self._handle = None
        except Exception:
            pass

    def num_frames(self, num_samples: int) -> int:
        lib = _lib.load()
        fn = lib.ppv_fbank_num_frames if self._feature_method == 'Fbank' else lib.ppv_spectral_num_frames
        return fn(self._get_handle(), int(num_samples))

    def forward(self, waveforms, input_lens_ratio=None):
        """reference: featurizer.py:33-60"""
        if not torch.is_tensor(waveforms):
            waveforms = torch.as_tensor(waveforms)
        if waveforms.dim() == 1:
            waveforms = waveforms.unsqueeze(0)
        _lib.require_cuda(waveforms, 'waveforms')
        wav = waveforms.to(torch.float32).contiguous()
        B, L = wav.shape
        lib = _lib.load()
        h = self._get_handle()
        fbank = self._feature_method == 'Fbank'
        T = (lib.ppv_fbank_num_frames if fbank else lib.ppv_spectral_num_frames)(h, L)
        if T <= 0:
            raise _lib.PPVError(f'waveform of {L} samples is shorter than one frame')
        ratio = None
        if input_lens_ratio is not None:
            ratio = torch.as_tensor(input_lens_ratio, dtype=torch.float32, device=wav.device).contiguous()
            assert ratio.numel() == B
        F = self._cfg.n_mels if fbank else lib.ppv_spectral_feature_dim(h)
        out = torch.empty((B, T, F), dtype=torch.float32, device=wav.device)
        with torch.cuda.device(wav.device):
            if fbank:
                _lib.check(lib.ppv_fbank_forward(h, _lib.ptr(wav), _lib.ptr(ratio), B, L, _lib.ptr(out),
                                                 _lib.current_stream()), 'ppv_fbank_forward')
            else:
                _lib.check(lib.ppv_spectral_forward(h, _lib.ptr(wav), _lib.ptr(ratio), B, L, _lib.ptr(out),
                                                    _lib.current_stream()), 'ppv_spectral_forward')
        return out

    def forward_ragged(self, waveforms, lengths):
        """A zero-padded batch of utterances of different lengths, each featurised as if alone (what the reference's training path
        computes sample by sample, reader.py:101-104, before collate_fn zero-pads the features): waveforms [B,L] CUDA, lengths [B]
        samples -> (features [B,Tmax,F] with per-utterance CMN over its own frames and zeros beyond them, frames per utterance).
        One launch sequence for the whole batch, whatever the front end (``ppv_fbank_forward_ragged_samples`` /
        ``ppv_spectral_forward_ragged_samples``)."""
        _lib.require_cuda(waveforms, 'waveforms')
        wav = waveforms.to(torch.float32).contiguous()
        B, L = wav.shape
        frames = [self.num_frames(int(n)) for n in lengths]
        if min(frames) <= 0:
            raise _lib.PPVError('an utterance is shorter than one frame')
        lib, h = _lib.load(), self._get_handle()
        fbank = self._feature_method == 'Fbank'
        T = (lib.ppv_fbank_num_frames if fbank else lib.ppv_spectral_num_frames)(h, L)
        vf = torch.tensor(frames, dtype=torch.int32, device=wav.device)
        # where snip_edges=False (Fbank) or center=True (the STFT front ends) reflects each utterance at its own end
        ns = torch.tensor([int(n) for n in lengths], dtype=torch.int32, device=wav.device)
        F = self._cfg.n_mels if fbank else lib.ppv_spectral_feature_dim(h)
        out = torch.empty((B, T, F), dtype=torch.float32, device=wav.device)
        name = 'ppv_fbank_forward_ragged_samples' if fbank else 'ppv_spectral_forward_ragged_samples'
        with torch.cuda.device(wav.device):
            _lib.check(getattr(lib, name)(h, _lib.ptr(wav), _lib.ptr(vf), _lib.ptr(ns), B, L, _lib.ptr(out), _lib.current_stream()), name)
        return out[:, :max(frames)], frames

    @property
    def feature_dim(self):
        """reference: featurizer.py:62-80"""
        if self._feature_method == 'LogMelSpectrogram':
            return self._method_args.get('n_mels', 128)
        elif self._feature_method == 'MelSpectrogram':
            return self._method_args.get('n_mels', 64)
        elif self._feature_method == 'Spectrogram':
            return self._method_args.get('n_fft', 512) // 2 + 1
        elif self._feature_method == 'MFCC':
            return self._method_args.get('n_mfcc', 40)
        elif self._feature_method == 'Fbank':
            return self._method_args.get('n_mels', 23)
        else:
            raise Exception('没有{}预处理方法'.format(self._feature_method))
