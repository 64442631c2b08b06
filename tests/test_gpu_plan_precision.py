"""GPU: precision is an input of each run, not part of the plan.

``ppv_model_set_precision`` and ``ppv_trainer_set_precision`` switch a live handle without rebuilding its plan (the predictor switches
the backbones it already holds), so every tensor-core step has to read the precision when it launches.  A handle that ran at bf16x3,
then at bf16 on the same plan, then at bf16x3 again, must give bitwise what a fresh handle at each precision gives: ECAPA-TDNN and
CAM++ forwards, and the ECAPA-TDNN training step's loss, logits and gradients."""
import pytest
import torch

pytestmark = pytest.mark.gpu

PRECISIONS = ["bf16x3", "bf16"]
SWITCHES = ["bf16", "bf16x3"]  # after the first run at bf16x3
S = 37


def backbone(cuda, name, precision):
    from ppvector.models.campplus import CAMPPlus
    from ppvector.models.ecapa_tdnn import EcapaTdnn
    from ppvector.utils.init import seeded_state_dict
    m = {"EcapaTdnn": EcapaTdnn, "CAMPPlus": CAMPPlus}[name](input_size=80, precision=precision).eval()
    m.load_state_dict(seeded_state_dict(m, seed=3))
    return m.to(cuda)


@pytest.mark.parametrize("name", ["EcapaTdnn", "CAMPPlus"])
def test_model_precision_switch_on_a_live_plan(cuda, name):
    x = torch.randn(2, 98, 80, generator=torch.Generator().manual_seed(0)).to(cuda)
    fresh = {p: backbone(cuda, name, p)(x) for p in PRECISIONS}
    assert not torch.equal(fresh["bf16x3"], fresh["bf16"])  # the two precisions run different kernels
    m = backbone(cuda, name, "bf16x3")
    assert torch.equal(m(x), fresh["bf16x3"])
    for p in SWITCHES:
        m.set_precision(p)
        assert torch.equal(m(x), fresh[p]), p


def engine(cuda, precision):
    from oracle import ecapa as oe
    from ppvector.train_engine import TrainEngine
    eng = TrainEngine(input_size=80, num_speakers=S, device=cuda)
    eng.set_precision(precision)
    g = torch.Generator().manual_seed(7)
    eng.load_state_dict(oe.make_ecapa_weights(seed=1000, dtype=torch.float64), (torch.rand(192, S, generator=g, dtype=torch.float64) * 2 - 1) * 0.15)
    return eng


def train_step(eng, x, y):
    """(loss, logits, gradients) of one step; the gradient buffer is cleared first, so the result does not depend on whether the step
    overwrites or accumulates it"""
    eng.grads.zero_()
    loss, logits = eng.forward_backward(x, y, return_logits=True)
    return loss.clone(), logits.clone(), eng.grads.clone()


def test_trainer_precision_switch_on_a_live_plan(cuda):
    g = torch.Generator().manual_seed(11)
    x = torch.randn(3, 35, 80, generator=g).to(cuda)
    y = torch.randint(0, S, (3,), generator=g).to(cuda)
    fresh = {p: train_step(engine(cuda, p), x, y) for p in PRECISIONS}
    assert not torch.equal(fresh["bf16x3"][2], fresh["bf16"][2])  # the two precisions run different kernels
    eng = engine(cuda, "bf16x3")
    runs = [("bf16x3", train_step(eng, x, y))]
    for p in SWITCHES:
        eng.set_precision(p)
        runs.append((p, train_step(eng, x, y)))
    for p, got in runs:
        for what, a, b in zip(("loss", "logits", "gradients"), got, fresh[p]):
            assert torch.equal(a, b), (p, what)
