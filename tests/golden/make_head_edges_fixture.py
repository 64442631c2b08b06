"""Mint tests/golden/ref_head_edges.npz: the reference's OWN loss classes (AAMLoss, SubCenterLoss, SphereFace2, ARMLoss; imported unmodified
from /root/reference under tests/paddle_shim, with the set-up of make_ref_fixtures.py) on constructed logits that reach the branches random
embeddings never reach: target cosines on both sides of the hard-margin threshold th = cos(pi - m) and of 0 (easy_margin), at +-(1 - 1e-3)
where d phi / dc is badly conditioned, a SubCenterLoss class whose winning sub-centre is below th, SphereFace2 targets below th (where
type A's fallback c - mmm takes the polynomial's base below 0) for t in {1, 2, 3, 5}, and an ARMLoss entry exactly equal to its row's
target value (kept, not zeroed).  Forward and backward through torch autograd in fp64.  Consumed by tests/test_head_edges_cpu.py on any
machine; the file holds the constructed logits and labels, each case's parameters, and what the reference computed: the loss and
dL/dlogits.

Runs only in the authoring container (needs /root/reference).
Usage:  python tests/golden/make_head_edges_fixture.py            (rewrites ref_head_edges.npz)
        python tests/golden/make_head_edges_fixture.py --check    (recomputes and compares with the committed file)
"""
import math
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))
from make_ref_fixtures import paddle  # noqa: E402  (sets up the shim and the reference's package path)

from ppvector.loss.aamloss import AAMLoss  # noqa: E402  (the REFERENCE's files)
from ppvector.loss.armloss import ARMLoss  # noqa: E402
from ppvector.loss.sphereface2 import SphereFace2  # noqa: E402
from ppvector.loss.subcenterloss import SubCenterLoss  # noqa: E402

OUT = os.path.join(HERE, "ref_head_edges.npz")
S = 8  # classes of the plain heads
EDGE = 1.0 - 1e-3


def target_cosines(margin):
    """One row per branch: halfway between -1 and th, just below / above th, just below / above 0, +-(1 - 1e-3), and an ordinary value."""
    th = math.cos(math.pi - margin)
    return [0.5 * (th - 1.0), th - 0.005, th + 0.005, -0.01, 0.01, -EDGE, EDGE, 0.3]


def plain_logits(margin, seed):
    g = torch.Generator().manual_seed(seed)
    c = target_cosines(margin)
    B = len(c)
    logits = torch.rand(B, S, generator=g, dtype=torch.float64) - 0.5
    labels = torch.randint(0, S, (B,), generator=g)
    logits[torch.arange(B), labels] = torch.tensor(c, dtype=torch.float64)
    return logits, labels


def subcenter_logits(margin, K, seed):
    """K sub-centre columns per class; the target class's best sub-centre sits in the fallback region on the first rows, above th on the
    others.  Rows 0-1 are the ones that matter: every sub-centre of the target class is below th."""
    g = torch.Generator().manual_seed(seed)
    th = math.cos(math.pi - margin)
    best = [0.5 * (th - 1.0), th - 0.005, th + 0.005, -0.01, 0.01, EDGE, 0.3]
    B, C = len(best), 5
    logits = torch.rand(B, C * K, generator=g, dtype=torch.float64) - 0.5
    labels = torch.randint(0, C, (B,), generator=g)
    for b in range(B):
        base = int(labels[b]) * K
        for k in range(K):  # the losers strictly below the winner, the winner in slot b % K
            logits[b, base + k] = best[b] - 0.001 * (k + 1)
        logits[b, base + (b % K)] = best[b]
    return logits, labels


def arm_tie_logits():
    """ARMLoss (armloss.py:28-29) keeps an entry whose scaled value equals the target's: target 0.75, margin 0.25, so the target's value is
    scale * 0.5 and the non-target 0.5 ties it exactly (0.75 - 0.25 is exact in binary).  Row 1 has no tie; row 2 two ties."""
    logits = torch.tensor([[0.75, 0.5, 0.1, -0.2, 0.6, 0.3],
                           [0.2, -0.1, 0.9, 0.45, 0.5, -0.6],
                           [0.5, 0.5, -0.3, 0.75, 0.49, 0.51]], dtype=torch.float64)
    labels = torch.tensor([0, 2, 3])
    return logits, labels


def cases():
    """tag -> (kind, margin, scale, ls-or-lanbuda, logits, labels).  kind is oracle.head's name for the head ('AAM', 'AAMe', 'SUB<K>[e]',
    'SF2{A,C}<t>', 'ARM')."""
    out = {}
    for mi, margin in enumerate((0.2, 0.5)):
        logits, labels = plain_logits(margin, 100 + mi)
        for easy in (False, True):
            for ls in (0.0, 0.1):
                out[f"AAM{'e' if easy else ''}_m{margin}_ls{ls}"] = ("AAMe" if easy else "AAM", margin, 32.0, ls, logits, labels)
        for mt in ("A", "C"):
            for t in (1, 2, 3, 5):
                out[f"SF2{mt}{t}_m{margin}_l0.7"] = (f"SF2{mt}{t}", margin, 32.0, 0.7, logits, labels)
    for K, margin, easy, ls, seed in ((3, 0.2, False, 0.0, 200), (3, 0.5, False, 0.1, 201), (3, 0.5, True, 0.0, 202), (2, 0.5, False, 0.0, 203)):
        logits, labels = subcenter_logits(margin, K, seed)
        out[f"SUB{K}{'e' if easy else ''}_m{margin}_ls{ls}"] = (f"SUB{K}{'e' if easy else ''}", margin, 32.0, ls, logits, labels)
    logits, labels = arm_tie_logits()
    for ls in (0.0, 0.1):
        out[f"ARM_m0.25_ls{ls}"] = ("ARM", 0.25, 30.0, ls, logits, labels)
    return out


def reference_loss(kind, margin, scale, ls):
    if kind.startswith("AAM"):
        return AAMLoss(margin=margin, scale=scale, easy_margin=kind.endswith("e"), label_smoothing=ls)
    if kind.startswith("SUB"):
        return SubCenterLoss(margin=margin, scale=scale, easy_margin=kind.endswith("e"), K=int(kind[3:].rstrip("e")), label_smoothing=ls)
    if kind.startswith("SF2"):
        return SphereFace2(margin=margin, scale=scale, lanbuda=ls, t=int(kind[4:]), margin_type=kind[3])
    assert kind == "ARM", kind
    return ARMLoss(margin=margin, scale=scale, label_smoothing=ls)


def make():
    d = {}
    for tag, (kind, margin, scale, ls, logits, labels) in cases().items():
        x = paddle.to_tensor(logits)
        x.requires_grad_(True)
        loss = reference_loss(kind, margin, scale, ls)({"features": None, "logits": x}, paddle.to_tensor(labels))
        loss.backward()
        assert torch.isfinite(loss) and torch.isfinite(x.grad).all(), tag
        d[f"{tag}_logits"] = logits.numpy()
        d[f"{tag}_labels"] = labels.numpy()
        d[f"{tag}_params"] = np.array([margin, scale, ls])
        d[f"{tag}_loss"] = np.array(float(loss.detach()))
        d[f"{tag}_dlogits"] = x.grad.detach().numpy().copy()
    return d


def main():
    d = make()
    if "--check" in sys.argv:
        old = np.load(OUT)
        assert sorted(old.files) == sorted(d), set(old.files) ^ set(d)
        err = max(float(np.abs(old[k] - d[k]).max()) for k in d)
        print(f"{os.path.basename(OUT)}: {len(d)} arrays, max |committed - recomputed| = {err:.3e}")
        sys.exit(1 if err > 1e-12 else 0)
    np.savez_compressed(OUT, **d)
    print(f"wrote {os.path.basename(OUT)}: {len(d)} arrays, {os.path.getsize(OUT)} bytes")


if __name__ == "__main__":
    main()
