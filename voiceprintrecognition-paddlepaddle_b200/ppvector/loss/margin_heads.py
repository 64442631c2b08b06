"""AMLoss, ARMLoss, CELoss -- drop-ins for ppvector/loss/amloss.py:5-28, armloss.py:5-35, celoss.py:5-22: the other softmax heads over
the cosine logits of ``SpeakerIdentification``.  They run on the same fused CUDA head as AAMLoss (``ppv_aam_forward`` /
``ppv_aam_backward`` with a head selector, csrc/aam.cu): cosines from ``features`` and the classifier weight, the head's margin rule on
the fly, online-softmax cross-entropy (``reduction='sum'`` / batch size = mean), label smoothing; backward in one pass.

  AMLoss   z = scale * (cos - margin * onehot)
  ARMLoss  z as AMLoss, then every entry whose z is below its row's target z is replaced by 0
  CELoss   z = the logits as they are (no scale)
  SphereFace2 (sphereface2.py:9-77)  not a softmax: lanbuda * softplus(-z_p) on the target entry, (1 - lanbuda) * softplus(z_n) on the others,
           z over g(c) = 2 ((c + 1) / 2)^t - 1 with an additive ('C') or angular ('A') margin, summed over classes, mean over the batch
  SubCenterLoss (subcenterloss.py:8-61)  the classifier has K sub-centres per class (fc.py:33: columns c*K .. c*K+K-1); a class's cosine
           is the maximum over its K columns, then AAMLoss's margin rule; only the winning sub-centre receives the class's gradient
"""
from torch import nn

from ppvector import _lib
from ppvector.loss.aamloss import _AAMFunction


class _MarginHead(nn.Module):
    head = None

    def __init__(self, margin=0.2, scale=30, label_smoothing=0.0):
        super().__init__()
        self.margin, self.scale, self.label_smoothing = margin, scale, label_smoothing
        self.easy_margin = self.head  # what the training loop forwards to the C ABI as the head selector

    def forward(self, inputs, labels):
        weight = inputs.get('_weight')
        if weight is None:
            raise _lib.PPVError(f"{type(self).__name__} on the H100 path needs the classifier weight: pass SpeakerIdentification's output dict")
        return _AAMFunction.apply(inputs['features'], weight, labels, self.margin, self.scale, self.head, self.label_smoothing)

    def update(self, margin=0.2):
        self.margin = margin


class AMLoss(_MarginHead):
    head = _lib.PPV_HEAD_AM


class ARMLoss(_MarginHead):
    head = _lib.PPV_HEAD_ARM


class SubCenterLoss(_MarginHead):
    def __init__(self, margin=0.2, scale=32, easy_margin=False, K=3, label_smoothing=0.0):
        super().__init__(margin=margin, scale=scale, label_smoothing=label_smoothing)
        self.K = int(K)
        self.head = _lib.PPV_HEAD_SUBCENTER | (self.K << 5) | int(bool(easy_margin))
        self.easy_margin = self.head


class SphereFace2(_MarginHead):
    """sphereface2.py:9-77: per-entry binary logistic loss over g(z) = 2 ((z + 1) / 2)^t - 1; ``lanbuda`` weighs positives against negatives.
    The reference creates a bias parameter at 0 and never hands it to the optimizer (trainer.py passes model.parameters() only): it is 0 here."""

    def __init__(self, margin=0.2, scale=32.0, lanbuda=0.7, t=3, margin_type='C'):
        super().__init__(margin=margin, scale=scale, label_smoothing=float(lanbuda))  # the ABI's label_smoothing slot carries lanbuda
        assert margin_type in ('A', 'C') and 1 <= int(t) <= 16
        self.lanbuda, self.t, self.margin_type = float(lanbuda), int(t), margin_type
        self.head = _lib.PPV_HEAD_SPHEREFACE2 | (self.t << 5) | int(margin_type == 'A')
        self.easy_margin = self.head


class CELoss(_MarginHead):
    head = _lib.PPV_HEAD_CE

    def __init__(self, label_smoothing=0.0):
        super().__init__(margin=0.0, scale=1.0, label_smoothing=label_smoothing)

    def update(self, margin=0.2):  # celoss.py:21-22
        pass
