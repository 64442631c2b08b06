"""CPU: the fp64 training oracle -- oracle/train.py's train-mode step run with the head (tests/train_pooling_oracle.py) -- pinned to the
reference's own training step for every pooling head besides ASP with global context (that one is pinned by
test_oracle_vs_reference.py::test_train_step_matches_reference_code): ASP without global context, SAP, TAP and TSP.
tests/golden/ref_train_pooling.npz holds what the reference's EcapaTdnn, SpeakerIdentification and AAMLoss computed for one train-mode
step on seeded inputs (tests/golden/make_train_pooling_fixture.py): the loss, the logits, the gradients of the head's parameters, of mfa
and of the classifier, and the updated running statistics.  Agreement is to 1e-10."""
import numpy as np
import pytest
import torch

from oracle import ecapa as oe
from train_pooling_oracle import train_step_grads

HEADS = {"ASP_noctx": ("ASP", False), "SAP": ("SAP", True), "TAP": ("TAP", True), "TSP": ("TSP", True)}
B, T, S, SEED = 4, 61, 37, 78
TOL = 1e-10


def problem():
    g = torch.Generator().manual_seed(SEED)
    f = torch.randn(B, T, 80, generator=g, dtype=torch.float64)
    f = f - f.mean(1, keepdim=True)
    labels = torch.randint(0, S, (B,), generator=g)
    Wc = (torch.rand(192, S, generator=g, dtype=torch.float64) * 2 - 1) * (6.0 / (192 + S)) ** 0.5
    return f, labels, Wc


def tap_slice(t):
    idx = tuple(slice(0, min(n, 6)) for n in t.shape)
    return np.concatenate([t[idx].reshape(-1).numpy(), [float(t.abs().mean()), float(t.sum())]])


def close(a, b, tol=TOL):
    a, b = np.asarray(a, dtype=np.float64), np.asarray(b, dtype=np.float64)
    assert a.shape == b.shape, (a.shape, b.shape)
    err = np.abs(a - b).max() / max(1.0, np.abs(b).max())
    assert err <= tol, err


@pytest.fixture(scope="module")
def ref(golden_dir):
    return np.load(f"{golden_dir}/ref_train_pooling.npz")


@pytest.mark.parametrize("tag", list(HEADS))
def test_train_step_matches_reference_code(ref, tag):
    pt, gc = HEADS[tag]
    f, labels, Wc = problem()
    W = oe.make_ecapa_weights(seed=1000, dtype=torch.float64, pooling_type=pt, global_context=gc)
    loss, grads, new_stats, logits = train_step_grads(f, labels, W, Wc, pt, gc, margin=0.2, scale=32.0)
    assert abs(loss.item() - float(ref[f"{tag}_loss"])) < TOL
    close(logits.numpy(), ref[f"{tag}_logits"])
    close(grads["classifier.weight"].numpy(), ref[f"{tag}_grad_classifier.weight"])
    names = [k[len(tag) + 6:] for k in ref.files if k.startswith(f"{tag}_grad_") and not k.endswith("classifier.weight")]
    stats = [k[len(tag) + 6:] for k in ref.files if k.startswith(f"{tag}_stat_")]
    # every head tensor is in the fixture: the oracle's parameter table of the head equals the reference's
    assert sorted(names + stats) == sorted(k for k in W if k.startswith(("mfa.", "asp.", "asp_bn.", "fc.")))
    for name in names:
        g = grads[name]
        close(g.numpy() if g.dim() == 1 else tap_slice(g), ref[f"{tag}_grad_{name}"])
        want = float(ref[f"{tag}_gradnorm_{name}"])
        assert abs(float(g.norm()) - want) <= TOL * max(1.0, want), name
    for name in stats:
        close(new_stats[name].numpy(), ref[f"{tag}_stat_{name}"])
