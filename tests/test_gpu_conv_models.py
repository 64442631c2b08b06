"""GPU: the four 2-D models (ResNetSE, ERes2Net, ERes2NetV2, CAM++) around their conv kernels, against the fp64 oracle.

* The kernel switches: PPV_CONV3X3=0 moves the 3x3 32 -> 32 convs from the patch kernel to the gather-GEMM, PPV_POINTWISE=0 the
  32-channel 1x1 convs from the pointwise kernel to the gather-GEMM.  Both runs must agree with each other and with the oracle, and
  the profiler's kernel names show that the two runs took different kernels.  T = 62, 63, 125 and 298 put the image width (time) at
  one whole patch of 62 outputs, one more column, two patches and one, and the 3 s utterance.
* The bf16 precision, which no other test compares with the oracle.
* The full batch of tools/model_bench.py (256 x 298 frames), rows spread over the batch.
* Plan reuse: a plan zeroes its workspace once; every later forward relies on the zero borders staying zero."""
import functools

import pytest
import torch

from oracle import campplus as oc
from oracle import eres2net as oe
from oracle import resnet_se as orr
from ppvector import _lib
from ppvector.models.campplus import CAMPPlus
from ppvector.models.eres2net import ERes2Net, ERes2NetV2
from ppvector.models.resnet_se import ResNetSE

pytestmark = pytest.mark.gpu

# name -> (model class, seed-1000 fp64 weights, fp64 oracle forward)
MODELS = {
    "ResNetSE": (ResNetSE, lambda: orr.make_resnet_se_weights(seed=1000, dtype=torch.float64), orr.resnet_se_forward),
    "ERes2Net": (ERes2Net, lambda: oe.make_eres2net_weights(seed=1000, dtype=torch.float64), oe.eres2net_forward),
    "ERes2NetV2": (ERes2NetV2, lambda: oe.make_eres2net_weights(seed=1000, dtype=torch.float64, base_width=26, version=2),
                   functools.partial(oe.eres2net_forward, base_width=26, version=2)),
    "CAMPPlus": (CAMPPlus, lambda: oc.make_campplus_weights(seed=1000, dtype=torch.float64), oc.campplus_forward),
}
# the models that plan a pointwise step (a 1x1 conv over the 32-channel stem / FCM grid); ResNetSE runs its 1x1 convs on the gather-GEMM
POINTWISE_MODELS = ["ERes2Net", "ERes2NetV2", "CAMPPlus"]
EDGE_T = [62, 63, 125, 298]
B_SMALL = 3
ORACLE_ROWS = [0, B_SMALL - 1]
# Bounds, with what an H100 SXM (700 W) measured at these inputs:
REL_TOL = 1e-4  # the per-model test files' embedding bound (~50 stacked convolutions at ~2^-17 per product); measured 6.3e-6 - 5.0e-5
SWITCH_TOL = 2e-5  # two kernels at the same precision; measured: patch kernel == gather-GEMM bitwise, pointwise vs gather-GEMM 1.5e-6 - 4.8e-6
BF16_COS_TOL = 2e-5  # 1 - cos of the bf16 embeddings vs the oracle; measured 1.7e-6 - 4.0e-6


@functools.lru_cache(maxsize=None)
def weights(name):
    return MODELS[name][1]()


def feats(B, T, seed):
    return torch.randn(B, T, 80, generator=torch.Generator().manual_seed(seed))


@functools.lru_cache(maxsize=None)
def oracle(name, B, T, seed, rows):
    return MODELS[name][2](feats(B, T, seed)[list(rows)].double(), weights(name))


def make_model(cuda, name, precision="bf16x3"):
    m = MODELS[name][0](input_size=80, precision=precision).eval()
    m.load_state_dict({k: v.float() for k, v in weights(name).items()}, strict=True)
    return m.to(cuda)


def run(cuda, monkeypatch, name, f, env=None, precision="bf16x3"):
    """a fresh model (so a fresh plan) under `env`: (embeddings on the CPU, names of the CUDA kernels the forward ran)"""
    from torch.profiler import ProfilerActivity, profile
    for var in ("PPV_CONV3X3", "PPV_POINTWISE"):
        monkeypatch.delenv(var, raising=False)
    for var, val in (env or {}).items():
        monkeypatch.setenv(var, val)
    m = make_model(cuda, name, precision)
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        emb = m(f.to(cuda))
        torch.cuda.synchronize()
    return emb.double().cpu(), {e.key for e in prof.key_averages()}


def rel_err(a, b):
    return ((a - b).norm(dim=1) / b.norm(dim=1)).max().item()


def check_oracle(name, emb, B, T, seed, rows, what):
    ref = oracle(name, B, T, seed, tuple(rows))
    got = emb[rows]
    rel = rel_err(got, ref)
    assert rel < REL_TOL, (what, rel)
    assert (1 - torch.nn.functional.cosine_similarity(got, ref)).max() < 1e-8, what
    return rel


_default_runs = {}


def default_run(cuda, monkeypatch, name, T):
    """the default plan's embeddings and kernels at (B_SMALL, T), shared by the two switch tests"""
    if (name, T) not in _default_runs:
        _default_runs[(name, T)] = run(cuda, monkeypatch, name, feats(B_SMALL, T, T))
    return _default_runs[(name, T)]


def has_kernel(names, kernel):
    return any(kernel in n for n in names)


@pytest.mark.parametrize("T", EDGE_T)
@pytest.mark.parametrize("name", list(MODELS))
def test_conv3x3_switch(cuda, monkeypatch, name, T):
    emb, names = default_run(cuda, monkeypatch, name, T)
    emb_g, names_g = run(cuda, monkeypatch, name, feats(B_SMALL, T, T), {"PPV_CONV3X3": "0"})
    assert has_kernel(names, "conv3x3_c32_kernel") and not has_kernel(names_g, "conv3x3_c32_kernel")
    rel = rel_err(emb, emb_g)
    r0 = check_oracle(name, emb, B_SMALL, T, T, ORACLE_ROWS, "patch kernel")
    r1 = check_oracle(name, emb_g, B_SMALL, T, T, ORACLE_ROWS, "PPV_CONV3X3=0")
    print(f"\n{name} T={T}: patch kernel vs gather-GEMM rel {rel:.1e} (bound {SWITCH_TOL:.0e}); vs oracle {r0:.1e} / {r1:.1e} "
          f"(bound {REL_TOL:.0e})")
    assert rel < SWITCH_TOL, rel


@pytest.mark.parametrize("T", EDGE_T)
@pytest.mark.parametrize("name", POINTWISE_MODELS)
def test_pointwise_switch(cuda, monkeypatch, name, T):
    emb, names = default_run(cuda, monkeypatch, name, T)
    emb_g, names_g = run(cuda, monkeypatch, name, feats(B_SMALL, T, T), {"PPV_POINTWISE": "0"})
    assert has_kernel(names, "pw_conv_kernel") and not has_kernel(names_g, "pw_conv_kernel")
    rel = rel_err(emb, emb_g)
    r0 = check_oracle(name, emb, B_SMALL, T, T, ORACLE_ROWS, "pointwise kernel")
    r1 = check_oracle(name, emb_g, B_SMALL, T, T, ORACLE_ROWS, "PPV_POINTWISE=0")
    print(f"\n{name} T={T}: pointwise kernel vs gather-GEMM rel {rel:.1e} (bound {SWITCH_TOL:.0e}); vs oracle {r0:.1e} / {r1:.1e} "
          f"(bound {REL_TOL:.0e})")
    assert rel < SWITCH_TOL, rel


@pytest.mark.parametrize("name", list(MODELS))
def test_bf16_precision_is_close_but_different(cuda, monkeypatch, name):
    T = 298
    emb, _ = run(cuda, monkeypatch, name, feats(B_SMALL, T, T), precision="bf16")
    ref = oracle(name, B_SMALL, T, T, tuple(ORACLE_ROWS))
    one_minus_cos = (1 - torch.nn.functional.cosine_similarity(emb[ORACLE_ROWS], ref)).max().item()
    print(f"\n{name} bf16: 1 - cos vs oracle {one_minus_cos:.1e} (bound {BF16_COS_TOL:.0e})")
    assert one_minus_cos < BF16_COS_TOL
    emb_x3, _ = default_run(cuda, monkeypatch, name, T)
    assert not torch.equal(emb, emb_x3)  # the bf16 plan ran the one-MMA kernels, not the bf16x3 ones


@pytest.mark.parametrize("name", list(MODELS))
def test_full_batch(cuda, monkeypatch, name):
    """256 x 298 frames.  Rows: both ends of the batch; image 1, which holds the patch that starts the patch kernel's second pass over
    the SMs (70 patches per 80 x 298 image); images SMs - 1 and SMs, either side of the SM count for the kernels that give each utterance
    its own CTAs (CAM++'s context pooling, the column statistics)."""
    B, T, seed = 256, 298, 256
    S = _lib.load().ppv_device_sm_count()
    rows = sorted({0, S // 70, S - 1, S, B - 2, B - 1})
    emb, _ = run(cuda, monkeypatch, name, feats(B, T, seed))
    assert emb.shape == (B, 192) and torch.isfinite(emb).all()
    rel = check_oracle(name, emb, B, T, seed, rows, "full batch")
    print(f"\n{name} B={B}: rows {rows} vs oracle rel {rel:.1e} (bound {REL_TOL:.0e})")


@pytest.mark.parametrize("name", list(MODELS))
def test_plan_reuse(cuda, monkeypatch, name):
    """a, then b, then a through one plan; a on a fresh model: all bitwise equal"""
    T = 63  # one output column in the second patch of each row
    a, b = feats(B_SMALL, T, 1).to(cuda), (4 * feats(B_SMALL, T, 2)).to(cuda)
    monkeypatch.delenv("PPV_CONV3X3", raising=False)
    monkeypatch.delenv("PPV_POINTWISE", raising=False)
    m = make_model(cuda, name)
    e1 = m(a).clone()
    eb = m(b).clone()
    e2 = m(a).clone()
    assert torch.isfinite(e1).all() and not torch.equal(e1, eb)
    assert torch.equal(e1, e2)
    assert torch.equal(make_model(cuda, name)(a), e1)
