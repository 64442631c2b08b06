"""SpeakerIdentification -- drop-in for ppvector/models/fc.py:6-53 (Cosine classifier, num_blocks=0).

The cosine logits are produced together with the loss by ``ppv_aam_forward`` (see ppvector/loss/aamloss.py);
``forward`` returns the same ``{"features", "logits"}`` dict as the reference.
"""
import ctypes as C
import math

import torch
from torch import nn

from ppvector import _lib


class _CosineLogits(torch.autograd.Function):
    """logits = normalize(x) @ normalize(W, axis=0) via libppv_b200 (fc.py:49)."""

    @staticmethod
    def forward(ctx, x, weight):
        from ppvector.loss.aamloss import aam_forward_raw
        B = x.shape[0]
        labels = torch.zeros(B, dtype=torch.int64, device=x.device)
        logits, _, _ = aam_forward_raw(x, weight, labels, 0.0, 1.0, False, 0.0)
        ctx.save_for_backward(x, weight)
        return logits

    @staticmethod
    def backward(ctx, g):  # pragma: no cover - training path goes through AAMLoss' fused backward
        raise NotImplementedError('gradients flow through ppvector.loss.AAMLoss (fused head), not through the raw logits')


class SpeakerIdentification(nn.Module):
    def __init__(self, input_dim, num_speakers, classifier_type='Cosine', K=1, num_blocks=0, inter_dim=512):
        super().__init__()
        if classifier_type != 'Cosine' or num_blocks != 0:
            raise NotImplementedError('only classifier_type="Cosine" with num_blocks=0 is implemented on the H100 path')
        self.classifier_type = classifier_type
        # XavierUniform on a [input_dim, num_speakers*K] tensor (fc.py:31-33)
        bound = math.sqrt(6.0 / (input_dim + num_speakers * K))
        self.weight = nn.Parameter(torch.empty(input_dim, num_speakers * K).uniform_(-bound, bound))

    def forward(self, features):
        logits = _CosineLogits.apply(features, self.weight)
        return {"features": features, "logits": logits, "_weight": self.weight}
