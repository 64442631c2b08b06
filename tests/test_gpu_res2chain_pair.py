"""GPU: the paired Res2Net chain (csrc/res2chain.cu, two utterances per CTA, padded lengths up to 320) against the one-utterance
chain (PPV_RES2_CHAIN=single).  Both run the same MMAs in the same order per row and the same epilogue arithmetic, so the block
outputs and the embeddings must be bitwise equal."""
import pytest
import torch

pytestmark = pytest.mark.gpu

TAPS = ["blocks.1", "blocks.2", "blocks.3"]


@pytest.fixture(scope="module")
def state_dict():
    from ppvector.models.ecapa_tdnn import EcapaTdnn
    from ppvector.utils.init import seeded_state_dict
    return seeded_state_dict(EcapaTdnn(input_size=80), seed=3)


def run(cuda, monkeypatch, sd, x, precision, flag):
    from ppvector.models.ecapa_tdnn import EcapaTdnn
    if flag is None:
        monkeypatch.delenv("PPV_RES2_CHAIN", raising=False)
    else:
        monkeypatch.setenv("PPV_RES2_CHAIN", flag)
    m = EcapaTdnn(input_size=80, precision=precision).eval()
    m.load_state_dict(sd)
    m.to(cuda)
    emb = m(x).cpu()
    B, T = x.shape[0], x.shape[1]
    return emb, [m.read_tap(name, B, T).cpu() for name in TAPS]


# T = 312 is the longest utterance the paired kernel takes (Tp = 320); T = 313 takes the one-utterance kernel either way.
# B = 1 and 3 leave a CTA with a lone utterance, 133 and 265 give more pairs than the H100 has SMs.
@pytest.mark.parametrize("precision", ["bf16x3", "bf16"])
@pytest.mark.parametrize("B", [1, 3, 133, 265])
@pytest.mark.parametrize("T", [9, 121, 250, 298, 312, 313])
def test_paired_chain_bitwise_equals_single(cuda, monkeypatch, state_dict, T, B, precision):
    g = torch.Generator().manual_seed(T * 1000 + B)
    x = torch.randn(B, T, 80, generator=g).to(cuda)
    emb_p, taps_p = run(cuda, monkeypatch, state_dict, x, precision, None)
    emb_s, taps_s = run(cuda, monkeypatch, state_dict, x, precision, "single")
    assert torch.isfinite(emb_p).all()
    for name, a, b in zip(TAPS, taps_p, taps_s):
        assert torch.equal(a, b), name
    assert torch.equal(emb_p, emb_s)


# Which chain kernel ran, read from the profiler's kernel names: the comparison above means nothing if both runs took the same one.
@pytest.mark.parametrize("T, flag, want", [(298, None, "res2chain_pair_kernel"), (312, None, "res2chain_pair_kernel"),
                                           (298, "single", "res2chain_kernel"), (313, None, "res2chain_kernel"),
                                           (313, "single", "res2chain_kernel")])
def test_chain_variant_taken(cuda, monkeypatch, state_dict, T, flag, want):
    from torch.profiler import ProfilerActivity, profile
    x = torch.randn(3, T, 80, generator=torch.Generator().manual_seed(T)).to(cuda)
    run(cuda, monkeypatch, state_dict, x, "bf16x3", flag)  # plan and warm up outside the profiled region
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        run(cuda, monkeypatch, state_dict, x, "bf16x3", flag)
        torch.cuda.synchronize()
    names = {e.key for e in prof.key_averages()}
    chain = {n for n in names if "res2chain" in n}
    assert chain and all(want + "<" in n for n in chain), chain
