"""Shared plumbing of the backbone mirrors: a torch ``nn.Module`` that only HOLDS parameters (named like the reference's
Paddle state_dict) and whose ``forward`` is one call into libppv_b200 (``ppv_model_forward``).  No torch compute, no
fallback: without the library or a GPU these modules raise."""
import ctypes as C

import torch
from torch import nn

from ppvector import _lib


class NativeBackbone(nn.Module):
    """Subclasses implement ``_native_cfg() -> (kind, ctypes cfg struct)`` and set ``embd_dim`` / ``input_size``."""

    # True: the library takes this model's waveforms through the Fbank front end in the same call (ppv_model_forward_wav)
    _fused_wav = False

    def __init__(self, precision='bf16x3'):
        super().__init__()
        self.precision = precision
        self._handle = None
        self._ws = None

    def _native_cfg(self):
        raise NotImplementedError

    def _prec_code(self):
        return {'bf16x3': _lib.PPV_PREC_BF16X3, 'bf16': _lib.PPV_PREC_BF16}[self.precision]

    def invalidate(self):
        """Drop the device-side copy of the weights (call after changing parameters / load_state_dict)."""
        if self._handle is not None:
            _lib.load().ppv_model_destroy(self._handle)
            self._handle = None

    def load_state_dict(self, *a, **k):
        r = super().load_state_dict(*a, **k)
        self.invalidate()
        return r

    def _get_handle(self):
        if self._handle is not None:
            return self._handle
        lib = _lib.load()
        kind, cfg = self._native_cfg()
        cfg.precision = self._prec_code()
        h = C.c_void_p()
        _lib.check(lib.ppv_model_create(kind, C.byref(cfg), C.byref(h)), 'ppv_model_create')
        for name, t in self.state_dict().items():
            t = t.detach().to(torch.float32).contiguous()
            shape = (C.c_int64 * t.dim())(*t.shape)
            _lib.check(lib.ppv_model_load_weight(h, name.encode(), C.c_void_p(t.data_ptr()), shape, t.dim()),
                       f'ppv_model_load_weight({name})')
        _lib.check(lib.ppv_model_finalize(h), 'ppv_model_finalize')
        self._handle = h
        return h

    def set_precision(self, precision: str):
        self.precision = precision
        if self._handle is not None:
            _lib.check(_lib.load().ppv_model_set_precision(self._handle, self._prec_code()), 'ppv_model_set_precision')

    def _workspace(self, B, T, device):
        need = _lib.load().ppv_model_workspace_bytes(self._get_handle(), B, T)
        if self._ws is None or self._ws.numel() < need or self._ws.device != device:
            self._ws = None
            self._ws = torch.empty(need, dtype=torch.uint8, device=device)
        return self._ws

    def __del__(self):
        try:
            self.invalidate()
        except Exception:
            pass

    def _lengths_refusal(self):
        """Why ``forward`` cannot take ``lengths``, or None where it can (ppv_model_forward_lengths)."""
        return 'lengths masking is never used by the reference callers and is not implemented'

    def _check_eval(self):
        if self.training:
            raise _lib.PPVError(f'{type(self).__name__} on the H100 path implements the eval-mode forward only; call .eval()')

    def _embed(self, entry, args, device, B, T):
        """[B, embd_dim] from the library call ``entry(handle, *args, emb, workspace, workspace_bytes, stream)``, on a workspace
        sized for B utterances of T frames."""
        with torch.cuda.device(device):
            h = self._get_handle()
            ws = self._workspace(B, T, device)
            emb = torch.empty((B, self.embd_dim), dtype=torch.float32, device=device)
            _lib.check(getattr(_lib.load(), entry)(h, *args, _lib.ptr(emb), C.c_void_p(ws.data_ptr()), ws.numel(),
                                                    _lib.current_stream()), entry)
        return emb

    def forward(self, x, lengths=None):
        """x [N, time, freq] float32 CUDA -> [N, embd_dim].  ``lengths`` [N], where the model takes it: relative lengths in (0, 1]."""
        refusal = lengths is not None and self._lengths_refusal()
        if refusal:
            raise NotImplementedError(refusal)
        self._check_eval()
        _lib.require_cuda(x, 'x')
        x = x.to(torch.float32).contiguous()
        B, T, F = x.shape
        assert F == self.input_size
        if lengths is None:
            return self._embed('ppv_model_forward', (_lib.ptr(x), B, T), x.device, B, T)
        lengths = torch.as_tensor(lengths, dtype=torch.float32, device=x.device).contiguous()
        assert lengths.shape == (B,)
        return self._embed('ppv_model_forward_lengths', (_lib.ptr(x), _lib.ptr(lengths), B, T), x.device, B, T)

    def forward_wav(self, featurizer, waveforms, input_lens_ratio=None):
        """waveforms [N, samples] -> [N, embd_dim], equal to ``self(featurizer(waveforms, input_lens_ratio))``.  Models with
        ``_fused_wav`` and an Fbank front end take one library call (``ppv_model_forward_wav``) that never materialises the
        [N, time, freq] features; every other pairing featurises, then embeds (two calls)."""
        if not self._fused_wav or getattr(featurizer, '_feature_method', 'Fbank') != 'Fbank':
            return self(featurizer(waveforms, input_lens_ratio))
        self._check_eval()
        _lib.require_cuda(waveforms, 'waveforms')
        if waveforms.dim() == 1:
            waveforms = waveforms.unsqueeze(0)
        wav = waveforms.to(torch.float32).contiguous()
        B, L = wav.shape
        ratio = None
        if input_lens_ratio is not None:
            ratio = torch.as_tensor(input_lens_ratio, dtype=torch.float32, device=wav.device).contiguous()
        return self._embed('ppv_model_forward_wav', (featurizer._get_handle(), _lib.ptr(wav), _lib.ptr(ratio), B, L), wav.device,
                           B, featurizer.num_frames(L))

    def _read_tap(self, name, shape):
        out = torch.empty(shape, dtype=torch.float32, device=self._ws.device)
        _lib.check(_lib.load().ppv_model_read_tap(self._get_handle(), name.encode(), _lib.ptr(out), out.numel(),
                                                   _lib.current_stream()), 'ppv_model_read_tap')
        return out


class ConvParams(nn.Module):
    """Parameter holder named like paddle.nn.Conv1D / Conv2D (weight [Cout,Cin,*k], bias [Cout])."""

    def __init__(self, cin, cout, *k):
        super().__init__()
        fan_in = cin
        for d in k:
            fan_in *= d
        # paddle.nn.Conv1D / Conv2D default initializer: Normal(0, sqrt(2 / fan_in)), bias 0
        self.weight = nn.Parameter(torch.empty(cout, cin, *k).normal_(0.0, (2.0 / fan_in) ** 0.5))
        self.bias = nn.Parameter(torch.zeros(cout))


class BNParams(nn.Module):
    """Parameter holder named like paddle.nn.BatchNorm (weight, bias, _mean, _variance)."""

    def __init__(self, c):
        super().__init__()
        self.weight = nn.Parameter(torch.ones(c))
        self.bias = nn.Parameter(torch.zeros(c))
        self.register_buffer('_mean', torch.zeros(c))
        self.register_buffer('_variance', torch.ones(c))


class LinearParams(nn.Module):
    """Parameter holder named like paddle.nn.Linear: weight is [in, out] (Paddle layout), bias [out]."""

    def __init__(self, cin, cout):
        super().__init__()
        bound = (6.0 / (cin + cout)) ** 0.5  # paddle.nn.Linear default: Xavier uniform, bias 0
        self.weight = nn.Parameter(torch.empty(cin, cout).uniform_(-bound, bound))
        self.bias = nn.Parameter(torch.zeros(cout))


class Empty(nn.Module):
    """Placeholder for parameter-free layers inside a Sequential (keeps the reference's index-based key names)."""
