"""GPU: the kernels each inference model's plan launches, and what the ECAPA-TDNN launch profile counts.

* Launch sequences: the ordered kernel names, template arguments included, that torch.profiler records for one warm forward of
  ECAPA-TDNN in every routing configuration (the paired, single-utterance and per-conv Res2Net paths, each pooling head, no global
  context, `lengths`, the waveform input, and width 128, which takes the gather-GEMM Res2Net path), and of each 2-D model.  A plan
  change that swaps a kernel, a template instance or the launch order fails here even when the outputs stay within tolerance.
  tests/golden/plan_routing.json holds the expected sequences and profile counts.
* Profile counters: ppv_model_profile's tensor-core / other launch counts for a feature, a waveform and a `lengths` forward; a
  ResNetSE handle is refused.
* Plan reuse with and without `lengths`: the valid-frame counts are a per-forward input of a plan built once.
* Width 128 (res2net_scale = 4) against the fp64 oracle."""
import ctypes as C
import functools
import json
import os

import pytest
import torch

from launch_check import check_launches

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "plan_routing.json")
B = 2
# ECAPA-TDNN configurations: name -> (constructor kwargs, T, PPV_RES2_CHAIN value or None, input: "feat" | "lengths" | "wav")
ECAPA_CASES = {
    "default_T98": ({}, 98, None, "feat"),  # paired Res2Net chain
    "T330": ({}, 330, None, "feat"),  # one utterance per chain CTA
    "T400": ({}, 400, None, "feat"),  # per-conv res2conv
    "chain0": ({}, 98, "0", "feat"),
    "chain_single": ({}, 98, "single", "feat"),
    "SAP": ({"pooling_type": "SAP"}, 98, None, "feat"),
    "TAP": ({"pooling_type": "TAP"}, 98, None, "feat"),
    "TSP": ({"pooling_type": "TSP"}, 98, None, "feat"),
    "no_global_context": ({"global_context": False}, 98, None, "feat"),
    "lengths": ({}, 98, None, "lengths"),
    "wav": ({}, 98, None, "wav"),
    "scale4": ({"res2net_scale": 4}, 98, None, "feat"),  # width 128: Res2Net convs on the gather-GEMM
}
IMAGE_MODELS = ["ResNetSE", "ERes2Net", "ERes2NetV2", "CAMPPlus"]
IMAGE_T = 63
WAV_SAMPLES = 16000  # 98 frames of the 25 ms / 10 ms fbank
LENGTHS = [1.0, 0.6]


@functools.lru_cache(maxsize=None)
def golden():
    with open(GOLDEN) as f:
        return json.load(f)


def ecapa(cuda, seed=3, **kw):
    from ppvector.models.ecapa_tdnn import EcapaTdnn
    from ppvector.utils.init import seeded_state_dict
    m = EcapaTdnn(input_size=80, **kw).eval()
    m.load_state_dict(seeded_state_dict(m, seed=seed))
    return m.to(cuda)


def image_model(cuda, name):
    from ppvector.models.campplus import CAMPPlus
    from ppvector.models.eres2net import ERes2Net, ERes2NetV2
    from ppvector.models.resnet_se import ResNetSE
    from ppvector.utils.init import seeded_state_dict
    m = {"ResNetSE": ResNetSE, "ERes2Net": ERes2Net, "ERes2NetV2": ERes2NetV2, "CAMPPlus": CAMPPlus}[name](input_size=80).eval()
    m.load_state_dict(seeded_state_dict(m, seed=3))
    return m.to(cuda)


def feats(T, seed=0):
    return torch.randn(B, T, 80, generator=torch.Generator().manual_seed(seed))


def ecapa_call(cuda, case):
    """(model, a function running one forward of the case) under the case's PPV_RES2_CHAIN; the caller restores the environment"""
    from ppvector.data_utils.featurizer import AudioFeaturizer
    kw, T, chain, inp = ECAPA_CASES[case]
    m = ecapa(cuda, **kw)
    if inp == "wav":
        fz = AudioFeaturizer("Fbank", {"sr": 16000, "n_mels": 80})
        wav = (0.1 * torch.randn(B, WAV_SAMPLES, generator=torch.Generator().manual_seed(1))).clamp(-1, 1).to(cuda)
        return m, lambda: m.forward_wav(fz, wav)
    x = feats(T).to(cuda)
    if inp == "lengths":
        lens = torch.tensor(LENGTHS, device=cuda)
        return m, lambda: m(x, lens)
    return m, lambda: m(x)


def set_chain(monkeypatch, chain):
    if chain is None:
        monkeypatch.delenv("PPV_RES2_CHAIN", raising=False)
    else:
        monkeypatch.setenv("PPV_RES2_CHAIN", chain)


@pytest.fixture(autouse=True)
def default_routing(monkeypatch):
    for var in ("PPV_RES2_CHAIN", "PPV_CONV3X3", "PPV_POINTWISE"):
        monkeypatch.delenv(var, raising=False)


@pytest.mark.parametrize("case", list(ECAPA_CASES))
def test_ecapa_launch_sequence(cuda, monkeypatch, case):
    set_chain(monkeypatch, ECAPA_CASES[case][2])
    _, fn = ecapa_call(cuda, case)
    check_launches(fn, golden()["sequences"]["ecapa/" + case])


@pytest.mark.parametrize("name", IMAGE_MODELS)
def test_image_model_launch_sequence(cuda, name):
    m = image_model(cuda, name)
    x = feats(IMAGE_T).to(cuda)
    check_launches(lambda: m(x), golden()["sequences"][name])


def profile_counts(cuda, case):
    """(tensor-core launches, other launches) that ppv_model_profile counts over one warm forward of the case"""
    from ppvector import _lib
    lib = _lib.load()
    m, fn = ecapa_call(cuda, case)
    fn()
    h = m._get_handle()
    _lib.check(lib.ppv_model_profile(h, 1), "ppv_model_profile")
    fn()
    g_ms, o_ms, g_n, o_n = C.c_double(), C.c_double(), C.c_int64(), C.c_int64()
    _lib.check(lib.ppv_model_profile_read(h, C.byref(g_ms), C.byref(o_ms), C.byref(g_n), C.byref(o_n)), "ppv_model_profile_read")
    _lib.check(lib.ppv_model_profile(h, 0), "ppv_model_profile")
    assert g_ms.value > 0 and o_ms.value > 0
    return [g_n.value, o_n.value]


@pytest.mark.parametrize("case", ["default_T98", "wav", "lengths"])
def test_profile_counts(cuda, case):
    assert profile_counts(cuda, case) == golden()["profile_counts"][case]


def test_profile_refuses_other_models(cuda):
    from ppvector import _lib
    m = image_model(cuda, "ResNetSE")
    m(feats(IMAGE_T).to(cuda))
    assert _lib.load().ppv_model_profile(m._get_handle(), 1) == golden()["profile_refusal_status"] != 0


def test_plan_reuse_with_and_without_lengths(cuda):
    """lengths, no lengths, other lengths through one plan: each bitwise equal to the same call on a fresh model"""
    x = feats(98).to(cuda)
    calls = [lambda m: m(x, torch.tensor(LENGTHS, device=cuda)), lambda m: m(x), lambda m: m(x, torch.tensor([0.3, 0.9], device=cuda))]
    m = ecapa(cuda)
    got = [call(m).clone() for call in calls]
    assert not torch.equal(got[0], got[1]) and not torch.equal(got[1], got[2])
    for call, e in zip(calls, got):
        assert torch.equal(call(ecapa(cuda)), e)


@pytest.mark.parametrize("Bw,T", [(1, 28), (5, 150), (3, 298)])
def test_width128_against_oracle(cuda, Bw, T):
    """res2net_scale = 4 at 512 channels: 128-wide Res2Net convs, on the gather-GEMM; test_gpu_ecapa.py::test_shapes's bound"""
    from oracle import ecapa as oe
    W64 = oe.make_ecapa_weights(seed=1000, dtype=torch.float64, res2net_scale=4)
    from ppvector.models.ecapa_tdnn import EcapaTdnn
    m = EcapaTdnn(input_size=80, res2net_scale=4).eval()
    m.load_state_dict({k: v.float() for k, v in W64.items()}, strict=True)
    m.to(cuda)
    f = torch.randn(Bw, T, 80, generator=torch.Generator().manual_seed(Bw * 1000 + T))
    ref = oe.ecapa_forward(f[: min(Bw, 4)].double(), W64, res2net_scale=4)
    emb = m(f.to(cuda)).double().cpu()
    assert emb.shape == (Bw, 192)
    rel = (emb[: min(Bw, 4)] - ref).norm(dim=1) / ref.norm(dim=1)
    assert rel.max() < 2e-5, rel
