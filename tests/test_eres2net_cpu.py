"""CPU: the ERes2Net configurations the GPU tests rely on, checked on the fp64 oracle and the model's parameter holders.

* The clipped-ReLU case (eres2net_clip_case.py): every Hardtanh(0, 20) of ERes2Net and ERes2NetV2 clips at least 1 % of its inputs, so
  the GPU test on these inputs cannot silently stop exercising the clip if the weight generator changes; and the case stays well
  conditioned, so that the GPU test's fp64 bounds measure the kernels and not the network's sensitivity to rounding.
* ERes2Net with m_channels = 64: the state dict's names and shapes equal the oracle's shape table."""
import pytest
import torch

import eres2net_clip_case as case
from oracle import eres2net as oe

MIN_CLIPPED = 0.01


@pytest.mark.parametrize("T", case.T_VALUES)
@pytest.mark.parametrize("variant", list(case.VARIANTS))
def test_every_clipped_relu_clips(monkeypatch, variant, T):
    fractions = []
    relu20 = oe.relu20

    def counting_relu20(x):
        fractions.append((x > 20.0).double().mean().item())
        return relu20(x)

    monkeypatch.setattr(oe, "relu20", counting_relu20)
    emb = case.forward(variant, case.feats(T))
    assert torch.isfinite(emb).all()
    assert len(fractions) == 4 * sum((3, 4, 6, 3))  # bn1, bns.0, bns.1 and the residual add of each of the 16 blocks
    assert min(fractions) >= MIN_CLIPPED, sorted(fractions)[:4]
    assert max(fractions) < 0.9  # and each keeps a share of unclipped values
    print(f"\n{variant} T={T}: clipped share per Hardtanh {min(fractions):.3f} - {max(fractions):.3f}")


def split_bf16(x):
    """x rounded to the hi + lo bf16 pair the device stores, in fp64"""
    xf = x.float()
    hi = xf.bfloat16().float()
    return hi.double() + (xf - hi).bfloat16().double()


@pytest.mark.parametrize("variant", list(case.VARIANTS))
def test_clip_case_is_well_conditioned(monkeypatch, variant):
    """The oracle with the features, the weights and every Hardtanh output rounded to split-bf16 stays within 3e-5 of the exact oracle at
    every tap (measured 1.0e-5 - 1.6e-5), well inside the GPU test's 5e-5; gain 6 without the shift gives 0.5 at layer3."""
    f, W = case.feats(64), case.weights(variant)
    taps, rounded = {}, {}
    case.forward(variant, f, W, taps)
    relu20 = oe.relu20
    monkeypatch.setattr(oe, "relu20", lambda x: split_bf16(relu20(x)))
    case.forward(variant, split_bf16(f), {k: split_bf16(v) for k, v in W.items()}, rounded)
    for name, want in taps.items():
        rel = ((rounded[name] - want).norm() / want.norm()).item()
        assert rel < 3e-5, (name, rel)


def test_push_into_clip_changes_the_backbone_batchnorms_only():
    W = oe.make_eres2net_weights(seed=1000, dtype=torch.float64)
    gains = sorted(k for k in W if oe.is_backbone_bn_gain(k))
    assert len(gains) == 1 + 4 * 16  # the stem's bn1; bn1, bns.0, bns.1, bn3 of each block
    assert all(W[k].dim() == 1 for k in gains)
    assert not any("shortcut" in k or "local_att" in k for k in gains)
    P = oe.push_into_clip(W, case.GAIN, case.SHIFT)
    changed = sorted(k for k in W if not torch.equal(W[k], P[k]))
    assert changed == sorted(gains + [k[:-len("weight")] + "bias" for k in gains])


def test_m_channels_64_names_and_shapes():
    from ppvector.models.eres2net import ERes2Net
    sd = ERes2Net(input_size=80, m_channels=64).state_dict()
    S = oe.eres2net_param_shapes(m_channels=64)
    assert sorted(sd) == sorted(S)
    for k, v in sd.items():
        assert tuple(v.shape) == tuple(S[k]), k
    assert sd["conv1.weight"].shape == (64, 1, 3, 3) and sd["layer1.0.conv1.weight"].shape == (64, 64, 1, 1)
    assert sd["seg_1.weight"].shape == (2 * 10240, 192)  # TSTP over 1024 channels x 10 frequency rows
