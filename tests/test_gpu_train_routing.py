"""GPU: the kernels one warm ECAPA-TDNN training step launches.

The ordered kernel names, template arguments included, that torch.profiler records for one ``ppv_trainer_forward_backward`` at a
small and at the training configuration's batch shape, in both precisions.  A plan change that swaps a kernel, a template instance
or the launch order fails here even when the loss and gradients stay within tolerance.  tests/golden/train_routing.json holds the
expected sequences."""
import functools
import json
import os

import pytest
import torch

from launch_check import check_launches

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "train_routing.json")
S = 37


@functools.lru_cache(maxsize=None)
def golden():
    with open(GOLDEN) as f:
        return json.load(f)


@pytest.mark.parametrize("precision", ["bf16x3", "bf16"])
@pytest.mark.parametrize("B,T", [(3, 35), (64, 298)])
def test_train_step_launch_sequence(cuda, B, T, precision):
    from oracle import ecapa as oe
    from ppvector.train_engine import TrainEngine
    eng = TrainEngine(input_size=80, num_speakers=S, device=cuda)
    eng.set_precision(precision)
    g = torch.Generator().manual_seed(7)
    eng.load_state_dict(oe.make_ecapa_weights(seed=1000, dtype=torch.float64), (torch.rand(192, S, generator=g, dtype=torch.float64) * 2 - 1) * 0.15)
    x = torch.randn(B, T, 80, generator=g).to(cuda)
    y = torch.randint(0, S, (B,), generator=g).to(cuda)
    check_launches(lambda: eng.forward_backward(x, y), golden()[f"{B}x{T}/{precision}"])
