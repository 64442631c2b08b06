"""Test helper: oracle/train.py's fp64 ECAPA-TDNN training step with the classifier of ppvector/models/fc.py:6-90 in front of the loss.

The backbone is oracle.ecapa.ecapa_forward (ASP with the global context) with oracle.train.make_bn_train.  The classifier follows
SpeakerIdentification and DenseLayer(config_str='batchnorm'):
  * block i: z = Conv1D(in_i, inter_dim, 1)(h) with bias (a matrix product on the [B, in] embedding), h = BatchNorm1D(z) with batch
    statistics (make_bn_train: biased variance, running = 0.9 running + 0.1 batch), no ReLU;
  * 'Cosine': logits = normalize(h) @ normalize(W, axis=0) (oracle.head.cosine_logits), W [in, S];
  * 'Linear': logits = h @ W + b, W [in, S] (Paddle's Linear layout), b [S].
The loss reads the logits (oracle.head.aam_loss / margin_head_loss).  Torch autograd gives the gradients.  Pinned to the reference's
own training step by tests/test_train_classifier_cpu.py."""
import math

import torch

from oracle import ecapa, head
from oracle.train import is_stat, make_bn_train


def classifier_names(classifier_type, num_blocks):
    """The classifier's state_dict names under 'classifier.' (fc.py:25-38), running statistics included."""
    out = []
    for i in range(num_blocks):
        p = f"classifier.blocks.{i}."
        out += [p + "linear.weight", p + "linear.bias"] + [p + "nonlinear.batchnorm." + n for n in ("weight", "bias", "_mean", "_variance")]
    return out + (["classifier.weight"] if classifier_type == "Cosine" else ["classifier.output.weight", "classifier.output.bias"])


def make_classifier_weights(seed, S, classifier_type, num_blocks, inter_dim=512, embd_dim=192, gain=1.0, dtype=torch.float64):
    """Seeded classifier tensors: conv weight N(0, 2 / fan_in) (Paddle's default), conv bias ~ U(+-0.1), BatchNorm gamma ~ U(0.5, 1.5),
    beta ~ N(0, 0.1), running mean ~ N(0, 0.1), running variance ~ U(0.5, 1.5) (perturbed so BatchNorm bugs show), output weight
    Xavier uniform times `gain`, Linear bias ~ N(0, 0.1)."""
    g = torch.Generator().manual_seed(seed)
    W, d = {}, embd_dim
    for i in range(num_blocks):
        p = f"classifier.blocks.{i}."
        W[p + "linear.weight"] = torch.randn(inter_dim, d, 1, generator=g, dtype=torch.float64) * math.sqrt(2.0 / d)
        W[p + "linear.bias"] = (torch.rand(inter_dim, generator=g, dtype=torch.float64) * 2 - 1) * 0.1
        W[p + "nonlinear.batchnorm.weight"] = torch.rand(inter_dim, generator=g, dtype=torch.float64) + 0.5
        W[p + "nonlinear.batchnorm.bias"] = torch.randn(inter_dim, generator=g, dtype=torch.float64) * 0.1
        W[p + "nonlinear.batchnorm._mean"] = torch.randn(inter_dim, generator=g, dtype=torch.float64) * 0.1
        W[p + "nonlinear.batchnorm._variance"] = torch.rand(inter_dim, generator=g, dtype=torch.float64) + 0.5
        d = inter_dim
    wout = (torch.rand(d, S, generator=g, dtype=torch.float64) * 2 - 1) * math.sqrt(6.0 / (d + S)) * gain
    if classifier_type == "Cosine":
        W["classifier.weight"] = wout
    else:
        W["classifier.output.weight"] = wout
        W["classifier.output.bias"] = torch.randn(S, generator=g, dtype=torch.float64) * 0.1
    return {k: v.to(dtype) for k, v in W.items()}


def classifier_forward(emb, P, classifier_type, num_blocks, bn, taps=None):
    """fc.py:41-53: -> logits [B, S]; taps (optional dict) gets each block's output as 'classifier.blocks.<i>'."""
    x = emb
    for i in range(num_blocks):
        p = f"classifier.blocks.{i}."
        x = bn(x @ P[p + "linear.weight"][:, :, 0].T + P[p + "linear.bias"], P, p + "nonlinear.batchnorm")
        if taps is not None:
            taps[f"classifier.blocks.{i}"] = x
    if classifier_type == "Cosine":
        return head.cosine_logits(x, P["classifier.weight"])
    if classifier_type == "Linear":
        return x @ P["classifier.output.weight"] + P["classifier.output.bias"]
    raise ValueError(f"不支持该输出层：{classifier_type}")


# loss -> (oracle kind, default margin, default scale) of the reference's constructors; SphereFace2 C with t = 3, lanbuda = 0.7
LOSSES = {"AAMLoss": ("AAM", 0.2, 32.0), "CELoss": ("CE", 0.0, 1.0), "AMLoss": ("AM", 0.2, 30.0), "ARMLoss": ("ARM", 0.2, 30.0),
          "SphereFace2": ("SF2C3", 0.2, 32.0)}


def loss_of(logits, labels, loss):
    kind, margin, scale = LOSSES[loss]
    if kind == "AAM":
        return head.aam_loss(logits, labels, margin=margin, scale=scale)
    return head.margin_head_loss(logits, labels, kind, margin=margin, scale=scale, label_smoothing=0.7 if kind.startswith("SF2") else 0.0)


def train_step_grads(feats, labels, W, classifier_type, num_blocks, loss="AAMLoss", taps=None):
    """-> (loss, grads of every parameter, new running statistics, logits, emb); W holds the backbone's and the classifier's tensors.
    taps (optional dict) gets the block outputs with their .grad kept."""
    P = {k: v.clone().requires_grad_(not is_stat(k)) for k, v in W.items()}
    new_stats = {}
    bn = make_bn_train(new_stats)
    emb = ecapa.ecapa_forward(feats, P, bn=bn)
    emb.retain_grad()
    logits = classifier_forward(emb, P, classifier_type, num_blocks, bn, taps=taps)
    if taps is not None:
        for v in taps.values():
            v.retain_grad()
    out = loss_of(logits, labels, loss)
    out.backward()
    grads = {k: v.grad for k, v in P.items() if not is_stat(k)}
    grads["emb"] = emb.grad
    return out.detach(), grads, new_stats, logits.detach(), emb.detach()
