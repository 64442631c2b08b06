"""CPU: the fp64 training oracle with the classifier of fc.py (tests/classifier_oracle.py) pinned to the reference's own training step:
Cosine + AAMLoss with one and two DenseLayer blocks, Linear + CELoss / AMLoss / SphereFace2 (margin_type C) with none and two blocks, and
a 96-wide block.  tests/golden/ref_classifier.npz holds what the reference's EcapaTdnn, SpeakerIdentification and loss classes computed for
one train-mode step on seeded inputs (tests/golden/make_classifier_fixture.py): the loss, the logits, the gradients of every classifier
tensor and of fc, and the blocks' updated running statistics.  Agreement is to 1e-10.  Also the trainer's classifier initialisation and
its checkpoint-key check, which need no GPU."""
import numpy as np
import pytest
import torch

from classifier_oracle import classifier_names, make_classifier_weights, train_step_grads
from oracle import ecapa as oe

CASES = {"cos_b1_AAM": ("Cosine", 1, 512, "AAMLoss", 1.0), "cos_b2_AAM": ("Cosine", 2, 512, "AAMLoss", 1.0),
         "lin_b0_CE": ("Linear", 0, 512, "CELoss", 1.0), "lin_b2_CE": ("Linear", 2, 512, "CELoss", 1.0),
         "lin_b0_AM": ("Linear", 0, 512, "AMLoss", 1.0), "lin_b2_AM": ("Linear", 2, 512, "AMLoss", 1.0),
         "lin_b0_SF2C": ("Linear", 0, 512, "SphereFace2", 0.3), "lin_b2_SF2C": ("Linear", 2, 512, "SphereFace2", 0.3),
         "cos_b2_i96_AAM": ("Cosine", 2, 96, "AAMLoss", 1.0)}
B, T, S, SEED, CLS_SEED = 4, 61, 37, 78, 79
TOL = 1e-10


def problem():
    g = torch.Generator().manual_seed(SEED)
    f = torch.randn(B, T, 80, generator=g, dtype=torch.float64)
    f = f - f.mean(1, keepdim=True)
    labels = torch.randint(0, S, (B,), generator=g)
    return f, labels


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
    return np.load(f"{golden_dir}/ref_classifier.npz")


@pytest.mark.parametrize("tag", list(CASES))
def test_train_step_matches_reference_code(ref, tag):
    ct, nb, inter, loss_name, gain = CASES[tag]
    f, labels = problem()
    Wc = make_classifier_weights(CLS_SEED, S, ct, nb, inter, gain=gain)
    W = dict(oe.make_ecapa_weights(seed=1000, dtype=torch.float64), **Wc)
    loss, grads, new_stats, logits, _ = train_step_grads(f, labels, W, ct, nb, loss=loss_name)
    assert abs(loss.item() - float(ref[f"{tag}_loss"])) < TOL * max(1.0, abs(float(ref[f"{tag}_loss"])))
    close(logits.numpy(), ref[f"{tag}_logits"])
    # every classifier tensor is in the fixture: the oracle's classifier table equals the reference's state_dict
    names = sorted(k[len(tag) + 6:] for k in ref.files if k.startswith(f"{tag}_grad_") and not k.endswith(("fc.conv.weight", "fc.conv.bias")))
    stats = sorted(k[len(tag) + 6:] for k in ref.files if k.startswith(f"{tag}_stat_"))
    assert sorted(names + stats) == sorted(classifier_names(ct, nb)) == sorted(Wc)
    for name in names + ["fc.conv.weight", "fc.conv.bias"]:
        g = grads[name]
        close(g.numpy() if g.dim() == 1 else tap_slice(g), ref[f"{tag}_grad_{name}"])
        if g.dim() > 1:
            want = float(ref[f"{tag}_gradnorm_{name}"])
            assert abs(float(g.norm()) - want) <= TOL * max(1.0, want), name
    for name in stats:
        close(new_stats[name].numpy(), ref[f"{tag}_stat_{name}"])


def test_classifier_init_follows_paddle_defaults():
    from ppvector.train_engine import classifier_shapes
    from ppvector.trainer import init_classifier
    shapes = classifier_shapes(192, 300, "Linear", 2, 256)
    assert list(shapes) == classifier_names("Linear", 2)
    assert shapes["classifier.blocks.0.linear.weight"] == (256, 192, 1) and shapes["classifier.blocks.1.linear.weight"] == (256, 256, 1)
    assert shapes["classifier.output.weight"] == (256, 300) and shapes["classifier.output.bias"] == (300,)
    torch.manual_seed(0)
    W = init_classifier(shapes)
    for i, fan_in in ((0, 192), (1, 256)):
        p = f"classifier.blocks.{i}."
        assert abs(float(W[p + "linear.weight"].std()) - (2.0 / fan_in) ** 0.5) < 0.05 * (2.0 / fan_in) ** 0.5
        assert not W[p + "linear.bias"].any() and not W[p + "nonlinear.batchnorm.bias"].any() and not W[p + "nonlinear.batchnorm._mean"].any()
        assert (W[p + "nonlinear.batchnorm.weight"] == 1).all() and (W[p + "nonlinear.batchnorm._variance"] == 1).all()
    bound = (6.0 / (256 + 300)) ** 0.5
    assert float(W["classifier.output.weight"].abs().max()) <= bound and float(W["classifier.output.weight"].abs().max()) > 0.9 * bound
    assert not W["classifier.output.bias"].any()
    # the default classifier draws exactly what the Cosine-only trainer drew: one Xavier-uniform [embd_dim, S] weight
    torch.manual_seed(0)
    W = init_classifier(classifier_shapes(192, 300))
    torch.manual_seed(0)
    assert list(W) == ["classifier.weight"] and torch.equal(W["classifier.weight"], torch.nn.init.xavier_uniform_(torch.empty(192, 300)))


def test_checkpoint_classifier_keys_must_match():
    from ppvector.train_engine import classifier_shapes
    from ppvector.trainer import check_classifier_keys
    shapes = classifier_shapes(192, 30, "Cosine", 1, 64)
    good = {k: np.zeros(s) for k, s in shapes.items()}
    check_classifier_keys(good, shapes, "ckpt")
    check_classifier_keys({}, shapes, "ckpt")  # a backbone-only checkpoint leaves the classifier as initialised
    with pytest.raises(ValueError, match=r"missing keys \['1.blocks.0..*unexpected keys \['1.output.weight'"):
        check_classifier_keys({"classifier.output.weight": np.zeros((192, 30)), "classifier.weight": np.zeros((64, 30))}, shapes, "ckpt")
    with pytest.raises(ValueError, match=r"another shape \['1.weight'\]"):
        check_classifier_keys(dict(good, **{"classifier.weight": np.zeros((192, 30))}), shapes, "ckpt")
