"""CPU: oracle/head.py pinned to the reference's own loss classes on the branches random embeddings never reach (tests/golden/ref_head_edges.npz,
made by tests/golden/make_head_edges_fixture.py): AAMLoss normal and easy with target cosines on both sides of th and of 0 and at
+-(1 - 1e-3), SubCenterLoss with the winning sub-centre below th, SphereFace2 types A and C with t in {1, 2, 3, 5} and targets below th (type
A's polynomial then has a negative base), and ARMLoss with an entry exactly equal to its row's target value.  Loss and dL/dlogits in fp64 to
1e-10.  The GPU tests of the loss heads (test_gpu_loss_heads.py) take this oracle as their reference."""
import numpy as np
import pytest
import torch

from oracle import head as oh

TOL = 1e-10


@pytest.fixture(scope="module")
def ref(golden_dir):
    return np.load(f"{golden_dir}/ref_head_edges.npz")


def tags(ref):
    return sorted(k[:-len("_loss")] for k in ref.files if k.endswith("_loss"))


def oracle_loss(kind, logits, labels, margin, scale, ls):
    if kind in ("AAM", "AAMe"):
        return oh.aam_loss(logits, labels, margin=margin, scale=scale, easy_margin=kind == "AAMe", label_smoothing=ls)
    return oh.margin_head_loss(logits, labels, kind, margin=margin, scale=scale, label_smoothing=ls)


def test_fixture_reaches_every_branch(ref):
    """The cases are what they claim: targets below th for every margin, the ARM tie exact, the sub-centre winner below th."""
    for tag in tags(ref):
        margin = float(ref[f"{tag}_params"][0])
        th = oh.aam_params(margin)["th"]
        c, y = ref[f"{tag}_logits"], ref[f"{tag}_labels"]
        if tag.startswith(("AAM", "SF2")):
            tc = c[np.arange(len(y)), y]
            assert (tc < th).sum() >= 2 and (tc > th).any() and (np.abs(tc) > 0.998).sum() == 2, tag
        if tag.startswith("SUB"):
            K = int(tag[3])
            best = c.reshape(len(y), -1, K).max(2)[np.arange(len(y)), y]
            assert (best < th).sum() >= 2, tag
        if tag.startswith("ARM"):
            assert c[0, 1] * 30.0 == (c[0, 0] - 0.25) * 30.0


@pytest.mark.parametrize("kind", ["AAM_", "AAMe_", "SUB", "SF2A", "SF2C", "ARM"])
def test_oracle_matches_reference_at_the_margin_branches(ref, kind):
    seen = 0
    for tag in tags(ref):
        if not tag.startswith(kind):
            continue
        name = tag.split("_")[0]
        margin, scale, ls = (float(v) for v in ref[f"{tag}_params"])
        logits = torch.from_numpy(ref[f"{tag}_logits"]).requires_grad_(True)
        labels = torch.from_numpy(ref[f"{tag}_labels"])
        loss = oracle_loss(name, logits, labels, margin, scale, ls)
        loss.backward()
        want = float(ref[f"{tag}_loss"])
        assert abs(loss.item() - want) <= TOL * max(1.0, abs(want)), (tag, loss.item(), want)
        dl, dw = logits.grad.numpy(), ref[f"{tag}_dlogits"]
        err = np.abs(dl - dw).max() / max(1.0, np.abs(dw).max())
        assert err <= TOL, (tag, err)
        seen += 1
    assert seen >= 2, kind
