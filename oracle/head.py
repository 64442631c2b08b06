"""Oracle: cosine classifier, AAMLoss (ArcFace), margin scheduler and cosine scoring (CPU).

TEST INFRASTRUCTURE -- see oracle/__init__.py.

Follows
  * ppvector/models/fc.py:41-53        SpeakerIdentification.forward (Cosine, num_blocks=0)
  * ppvector/loss/aamloss.py:28-53     AAMLoss.forward / update
  * ppvector/optimizer/scheduler.py:43-102  MarginScheduler
  * ppvector/predict.py:279-283        contrast: dot / (|a||b|)
  * ppvector/predict.py:168-187        normalize_features + sklearn cosine_similarity + argmax
  * ppvector/trainer.py:416-423        eval scoring: cosine_similarity(trial[1,D], enroll[N,D]) per trial
"""
import math

import numpy as np
import torch
import torch.nn.functional as F


def cosine_logits(x: torch.Tensor, weight: torch.Tensor) -> torch.Tensor:
    """fc.py:49  F.linear(F.normalize(x), F.normalize(weight, axis=0)); weight is [D, S]
    (Paddle Linear layout), normalize eps 1e-12."""
    xn = x / x.norm(dim=1, keepdim=True).clamp_min(1e-12)
    wn = weight / weight.norm(dim=0, keepdim=True).clamp_min(1e-12)
    return xn @ wn


def aam_params(margin: float):
    """aamloss.py:21-26 / 48-53"""
    return dict(cos_m=math.cos(margin), sin_m=math.sin(margin),
                th=math.cos(math.pi - margin), mmm=1.0 + math.cos(math.pi - margin))


def aam_loss(logits: torch.Tensor, labels: torch.Tensor, margin=0.2, scale=32.0,
             easy_margin=False, label_smoothing=0.0) -> torch.Tensor:
    """aamloss.py:34-46.  The reference leaves sqrt(1 - c^2) unclamped (NaN if |c|>1 by
    rounding); the CUDA kernel clamps at 0 -- identical whenever |c| <= 1, which
    cosine_logits guarantees up to rounding.  The oracle clamps too and says so."""
    p = aam_params(margin)
    sine = torch.sqrt((1.0 - logits.pow(2)).clamp_min(0.0))
    phi = logits * p["cos_m"] - sine * p["sin_m"]
    if easy_margin:
        phi = torch.where(logits > 0, phi, logits)
    else:
        phi = torch.where(logits > p["th"], phi, logits - p["mmm"])
    one_hot = F.one_hot(labels, logits.shape[1]).to(logits.dtype)
    output = (one_hot * phi + (1.0 - one_hot) * logits) * scale
    return F.cross_entropy(output, labels, label_smoothing=label_smoothing)


def margin_schedule(step: int, epochs: int, steps_per_epoch: int, initial_margin=0.0, final_margin=0.3,
                    increase_start_epoch=None, fix_epoch=None) -> float:
    """scheduler.py:43-102 MarginScheduler.get_margin: exponential ramp between
    increase_start_epoch (30 % of epochs) and fix_epoch (70 %)."""
    if increase_start_epoch is None:
        increase_start_epoch = int(epochs * 0.3)
    if fix_epoch is None:
        fix_epoch = int(epochs * 0.7)
    start_iter = increase_start_epoch * steps_per_epoch
    fix_iter = fix_epoch * steps_per_epoch
    if step >= fix_iter:
        return final_margin
    if step < start_iter:
        return initial_margin
    a, b = 1.0, 1e-3
    cur = step - start_iter
    total = fix_iter - start_iter
    ratio = 1.0 - math.exp((cur / total) * math.log(b / (a + 1e-6))) * a
    return initial_margin + (final_margin - initial_margin) * ratio


def cosine_pair(a: np.ndarray, b: np.ndarray) -> float:
    """predict.py:282"""
    a = np.asarray(a, dtype=np.float64)
    b = np.asarray(b, dtype=np.float64)
    return float(np.dot(a, b) / (np.linalg.norm(a) * np.linalg.norm(b)))


def cosine_matrix(A: np.ndarray, B: np.ndarray) -> np.ndarray:
    """trainer.py:416-423 / sklearn cosine_similarity: [M,D],[N,D] -> [M,N]."""
    A = np.asarray(A, dtype=np.float64)
    B = np.asarray(B, dtype=np.float64)
    An = A / np.linalg.norm(A, axis=1, keepdims=True)
    Bn = B / np.linalg.norm(B, axis=1, keepdims=True)
    return An @ Bn.T


def cosine_pairlist(E: np.ndarray, idx: np.ndarray) -> np.ndarray:
    """Pair-list form: score[p] = cos(E[idx[p,0]], E[idx[p,1]])."""
    E = np.asarray(E, dtype=np.float64)
    En = E / np.linalg.norm(E, axis=1, keepdims=True)
    return np.einsum("pd,pd->p", En[idx[:, 0]], En[idx[:, 1]])


def margin_head_loss(logits: torch.Tensor, labels: torch.Tensor, kind: str, margin=0.2, scale=30.0, label_smoothing=0.0) -> torch.Tensor:
    """The reference's other softmax heads over the cosine logits:
      'AM'  ppvector/loss/amloss.py:18-24    predictions = scale * (logits - margin * onehot)
      'ARM' ppvector/loss/armloss.py:18-31   as AM, then entries below their row's target value are replaced by 0
      'CE'  ppvector/loss/celoss.py:16-18    predictions = logits
      'SF2C<t>' / 'SF2A<t>'  ppvector/loss/sphereface2.py:44-70 (label_smoothing = lanbuda)
      'SUB<K>' / 'SUB<K>e'  ppvector/loss/subcenterloss.py:33-54 with K sub-centres (e: easy_margin)
    all with CrossEntropyLoss(reduction='sum', label_smoothing) / batch size."""
    B = logits.shape[0]
    if kind.startswith("SUB"):  # "SUB<K>[e]": SubCenterLoss (subcenterloss.py:40-54): max over the K adjacent sub-centre columns, then AAMLoss
        K = int(kind[3:].rstrip("e"))
        cosine = logits.reshape(B, logits.shape[1] // K, K).max(dim=2).values
        return aam_loss(cosine, labels, margin=margin, scale=scale, easy_margin=kind.endswith("e"), label_smoothing=label_smoothing)
    if kind.startswith("SF2"):  # "SF2C<t>" / "SF2A<t>": SphereFace2 (sphereface2.py:44-70); label_smoothing carries lanbuda; bias = 0
        t, lam = int(kind[4:]), label_smoothing
        g = lambda z: 2 * ((z + 1) / 2) ** t - 1  # noqa: E731
        if kind[3] == "A":
            p = aam_params(margin)
            sin = torch.sqrt((1.0 - logits ** 2).clamp_min(0))
            zp = scale * g(torch.where(logits > p["th"], logits * p["cos_m"] - sin * p["sin_m"], logits - p["mmm"]))
            zn = scale * g(logits * p["cos_m"] + sin * p["sin_m"])
        else:
            zp, zn = scale * (g(logits) - margin), scale * (g(logits) + margin)
        tm = F.one_hot(labels, logits.shape[1]).to(logits.dtype)
        # the reference's log(1 + exp(x)): torch's default softplus is x itself past 20, exp(-x) (2e-9 at 20) away in value and slope;
        # past 50 that gap is below fp64's resolution of x
        sp = lambda x: F.softplus(x, threshold=50.0)  # noqa: E731
        return (tm * lam * sp(-zp) + (1 - tm) * (1 - lam) * sp(zn)).sum(1).mean()
    if kind == "CE":
        pred = logits
    else:
        one_hot = F.one_hot(labels, logits.shape[1]).to(logits.dtype)
        pred = scale * (logits - margin * one_hot)
        if kind == "ARM":
            tgt = pred.gather(1, labels.view(-1, 1))
            pred = torch.where(pred - tgt < 0.0, torch.zeros_like(pred), pred)
    return F.cross_entropy(pred, labels, label_smoothing=label_smoothing, reduction="sum") / B
