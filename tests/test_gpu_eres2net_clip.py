"""GPU: ERes2Net and ERes2NetV2 where their clipped ReLU acts, against the fp64 oracle.

With the seed-1000 test weights no value that reaches Hardtanh(0, 20) exceeds ~3, so the other model tests pass whether or not the
kernels clip.  Here every backbone BatchNorm gain is doubled and its bias raised by 10 (eres2net_clip_case.py; test_eres2net_cpu.py
checks on the oracle that each of the 64 Hardtanh calls then clips at least 1 % of its inputs, and that the case is well conditioned).
The clip runs in the wgmma epilogue (gather-GEMM and 3x3 patch kernel), the pointwise kernel and the residual add
(se_scale_res_kernel); the model runs three ways:
  default        the 3x3 32 -> 32 convs on the patch kernel, the 32-channel 1x1 convs on the pointwise kernel;
  PPV_CONV3X3=0  the 3x3 convs on the gather-GEMM;
  PPV_POINTWISE=0  the 1x1 convs on the gather-GEMM.
Bounds: those of test_gpu_eres2net.py / test_gpu_eres2netv2.py (stage taps 5e-5 relative in norm, embedding 1 - cos < 1e-8 and
1e-4 relative).  Every stage output ends in a clipped residual add: its largest value must be exactly 20.0."""
import functools

import pytest
import torch

import eres2net_clip_case as case
from ppvector.models.eres2net import ERes2Net, ERes2NetV2

pytestmark = pytest.mark.gpu

CLASSES = {"ERes2Net": ERes2Net, "ERes2NetV2": ERes2NetV2}
TAPS = {"ERes2Net": ["fuse12", "fuse123", "fuse1234"], "ERes2NetV2": ["fuse34"]}
ROUTES = {"default": {}, "conv3x3_off": {"PPV_CONV3X3": "0"}, "pointwise_off": {"PPV_POINTWISE": "0"}}
# the kernel each route must (True) or must not (False) run
ROUTE_KERNELS = {"default": {"conv3x3_c32_kernel": True, "pw_conv_kernel": True}, "conv3x3_off": {"conv3x3_c32_kernel": False},
                 "pointwise_off": {"pw_conv_kernel": False}}
TAP_TOL = 5e-5
EMB_REL_TOL = 1e-4
COS_TOL = 1e-8


@functools.lru_cache(maxsize=None)
def oracle(variant, T):
    taps = {}
    emb = case.forward(variant, case.feats(T), taps=taps)
    return emb, taps


@pytest.mark.parametrize("T", case.T_VALUES)
@pytest.mark.parametrize("route", list(ROUTES))
@pytest.mark.parametrize("variant", list(case.VARIANTS))
def test_clipped_model_against_fp64(cuda, monkeypatch, variant, route, T):
    from torch.profiler import ProfilerActivity, profile
    for var in ("PPV_CONV3X3", "PPV_POINTWISE"):
        monkeypatch.delenv(var, raising=False)
    for var, val in ROUTES[route].items():
        monkeypatch.setenv(var, val)
    m = CLASSES[variant](input_size=80).eval()
    m.load_state_dict({k: v.float() for k, v in case.weights(variant).items()}, strict=True)
    m = m.to(cuda)
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        emb = m(case.feats(T).float().to(cuda))
        torch.cuda.synchronize()
    names = {e.key for e in prof.key_averages()}
    for kernel, ran in ROUTE_KERNELS[route].items():
        assert any(kernel in n for n in names) == ran, (route, kernel)

    ref, taps = oracle(variant, T)
    worst = 0.0
    for name in ["layer1", "layer2", "layer3", "layer4"] + TAPS[variant] + ["stats"]:
        got = m.read_tap(name, case.B, T).double().cpu()
        want = taps[name] if name == "stats" else taps[name].permute(0, 2, 3, 1)
        assert got.shape == want.shape, (name, got.shape, want.shape)
        rel = ((got - want).norm() / want.norm()).item()
        worst = max(worst, rel)
        assert rel < TAP_TOL, (name, rel)
        if name.startswith("layer"):
            assert got.max().item() == 20.0, (name, got.max().item())  # clipped: exactly 20, never above
            assert (got == 20.0).double().mean() >= 0.5 * (want == 20.0).double().mean(), name
    emb = emb.double().cpu()
    rel = ((emb - ref).norm(dim=1) / ref.norm(dim=1)).max().item()
    one_minus_cos = (1 - torch.nn.functional.cosine_similarity(emb, ref)).max().item()
    print(f"\n{variant} {route} T={T}: taps worst rel {worst:.1e} (bound {TAP_TOL:.0e}); embedding rel {rel:.1e} (bound {EMB_REL_TOL:.0e}), "
          f"1 - cos {one_minus_cos:.1e} (bound {COS_TOL:.0e})")
    assert rel < EMB_REL_TOL and one_minus_cos < COS_TOL
