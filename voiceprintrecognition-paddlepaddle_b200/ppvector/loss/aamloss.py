"""AAMLoss -- drop-in for ppvector/loss/aamloss.py:8-53 (ArcFace margin + softmax cross-entropy).

``forward(inputs, labels)`` takes the dict returned by SpeakerIdentification.  The fused CUDA head
(``ppv_aam_forward`` / ``ppv_aam_backward``, csrc/aam.cu) recomputes the cosines from ``features`` and the
classifier weight, applies the margin to the target class, and does the online-softmax CE without one_hot
or [B,S] temporaries; the backward returns d(features) and d(weight) in one pass.
"""
import ctypes as C
import math

import torch
from torch import nn

from ppvector import _lib


def aam_forward_raw(emb, weight, labels, margin, scale, easy_margin, label_smoothing):
    """``easy_margin`` doubles as the head selector of the C ABI: False / True = AAMLoss, _lib.PPV_HEAD_AM / ARM / CE = the other heads."""
    _lib.require_cuda(emb, 'features')
    lib = _lib.load()
    emb = emb.to(torch.float32).contiguous()
    weight = weight.to(torch.float32).contiguous()
    labels = labels.to(device=emb.device, dtype=torch.int64).contiguous()
    B, D = emb.shape
    D2, S = weight.shape
    assert D == D2
    logits = torch.empty((B, S), dtype=torch.float32, device=emb.device)
    loss = torch.empty((), dtype=torch.float32, device=emb.device)
    nbytes = lib.ppv_aam_workspace_bytes(B, D, S)
    ws = torch.empty(nbytes, dtype=torch.uint8, device=emb.device)
    with torch.cuda.device(emb.device):
        _lib.check(lib.ppv_aam_forward(_lib.ptr(emb), _lib.ptr(weight), _lib.ptr(labels), B, D, S, float(margin), float(scale),
                                       int(easy_margin), float(label_smoothing), _lib.ptr(logits), _lib.ptr(loss),
                                       C.c_void_p(ws.data_ptr()), nbytes, _lib.current_stream()), 'ppv_aam_forward')
    return logits, loss, ws


class _AAMFunction(torch.autograd.Function):
    @staticmethod
    def forward(ctx, emb, weight, labels, margin, scale, easy_margin, label_smoothing):
        logits, loss, ws = aam_forward_raw(emb, weight, labels, margin, scale, easy_margin, label_smoothing)
        ctx.save_for_backward(emb.detach(), weight.detach(), labels, logits)
        ctx.ws = ws
        ctx.args = (margin, scale, easy_margin, label_smoothing)
        return loss

    @staticmethod
    def backward(ctx, grad_out):
        emb, weight, labels, logits = ctx.saved_tensors
        margin, scale, easy_margin, label_smoothing = ctx.args
        lib = _lib.load()
        emb = emb.to(torch.float32).contiguous()
        weight = weight.to(torch.float32).contiguous()
        labels = labels.to(torch.int64).contiguous()
        B, D = emb.shape
        S = weight.shape[1]
        d_emb = torch.empty_like(emb)
        d_w = torch.empty_like(weight)
        ws = ctx.ws
        with torch.cuda.device(emb.device):
            _lib.check(lib.ppv_aam_backward(_lib.ptr(emb), _lib.ptr(weight), _lib.ptr(labels), _lib.ptr(logits), B, D, S,
                                            float(margin), float(scale), int(easy_margin), float(label_smoothing),
                                            _lib.ptr(d_emb), _lib.ptr(d_w), C.c_void_p(ws.data_ptr()), ws.numel(),
                                            _lib.current_stream()), 'ppv_aam_backward')
        return d_emb * grad_out, d_w * grad_out, None, None, None, None, None


class AAMLoss(nn.Module):
    def __init__(self, margin=0.2, scale=32, easy_margin=False, label_smoothing=0.0):
        super().__init__()
        self.scale = scale
        self.easy_margin = easy_margin
        self.label_smoothing = label_smoothing
        self.update(margin)

    def forward(self, inputs, labels):
        """reference: aamloss.py:28-46.  inputs: dict with 'features' [B,D] and the classifier weight."""
        features = inputs['features']
        weight = inputs.get('_weight')
        if weight is None:
            raise _lib.PPVError("AAMLoss on the H100 path needs the classifier weight: pass SpeakerIdentification's output dict")
        return _AAMFunction.apply(features, weight, labels, self.margin, self.scale, self.easy_margin, self.label_smoothing)

    def update(self, margin=0.2):
        """reference: aamloss.py:48-53 (called each step by MarginScheduler)"""
        self.margin = margin
        self.cos_m = math.cos(margin)
        self.sin_m = math.sin(margin)
        self.th = math.cos(math.pi - margin)
        self.mmm = 1.0 + math.cos(math.pi - margin)
