"""The ERes2Net / ERes2NetV2 inputs under which the clipped ReLU acts, shared by the GPU test that runs them (test_gpu_eres2net_clip.py)
and the CPU tests that check them on the oracle (test_eres2net_cpu.py).

The seed-1000 test weights keep every value that reaches Hardtanh(0, 20) below 3.1 at these features.  With every backbone BatchNorm
gain doubled and 10 added to its bias (oracle.eres2net.push_into_clip), each of the 64 Hardtanh calls clips between ~14 % and ~75 % of
its inputs.  Larger gains clip as much without the shift, but leave the network chaotic: at gain 6 (no shift), rounding each stored
activation to split-bf16 (~2^-17) moves layer3 by 50 %, so no kernel could be compared with fp64 there.  At gain 2 and shift 10 the same
rounding moves every tap by ~1.6e-5 (5e-6 at the unscaled weights)."""
import torch

from oracle import eres2net as oe

GAIN, SHIFT = 2.0, 10.0
B = 2
T_VALUES = [64, 149]
VARIANTS = {"ERes2Net": {}, "ERes2NetV2": {"base_width": 26, "version": 2}}


def weights(variant):
    """fp64 seed-1000 weights of `variant` with the backbone BatchNorms raised into the clip"""
    return oe.push_into_clip(oe.make_eres2net_weights(seed=1000, dtype=torch.float64, **VARIANTS[variant]), GAIN, SHIFT)


def feats(T):
    """[B, T, 80] fp64 features, mean-normalised over time (the features of test_gpu_eres2net.py at this T)"""
    f = torch.randn(B, T, 80, generator=torch.Generator().manual_seed(3000 + T), dtype=torch.float64)
    return f - f.mean(1, keepdim=True)


def forward(variant, f, W=None, taps=None):
    return oe.eres2net_forward(f, weights(variant) if W is None else W, taps=taps, **VARIANTS[variant])
