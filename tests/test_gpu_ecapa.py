"""GPU: ECAPA-TDNN forward (ppv_model_forward / ppv_model_forward_wav) vs the fp64 oracle and the golden
embeddings.  Tolerance (BASELINE.json north_star): cosine scores within 1e-4 of the reference path."""
import numpy as np
import pytest
import torch

from oracle import ecapa as oe
from oracle import fbank as ofb
from oracle import head as oh
from ppvector._lib import PPVError
from ppvector.data_utils.featurizer import AudioFeaturizer
from ppvector.models.ecapa_tdnn import EcapaTdnn

pytestmark = pytest.mark.gpu

COS_TOL = 1e-4


def make_model(cuda, W, precision="bf16x3"):
    m = EcapaTdnn(input_size=80, precision=precision).eval()
    missing, unexpected = m.load_state_dict({k: v.float() for k, v in W.items()}, strict=True)
    return m.to(cuda)


@pytest.fixture(scope="module")
def W64():
    return oe.make_ecapa_weights(seed=1000, dtype=torch.float64)


@pytest.fixture(scope="module")
def model(cuda, W64):
    return make_model(cuda, W64)


def test_state_dict_names_match_reference(W64):
    m = EcapaTdnn(input_size=80)
    assert sorted(m.state_dict().keys()) == sorted(W64.keys())
    for k, v in m.state_dict().items():
        assert tuple(v.shape) == tuple(W64[k].shape), k


@pytest.mark.parametrize("T", [98, 298])
def test_layerwise_taps_and_embedding(cuda, model, W64, golden_dir, T):
    g = np.load(f"{golden_dir}/ecapa_seed1000.npz")
    gi = torch.Generator().manual_seed(1000 + T)
    f = torch.randn(3, T, 80, generator=gi, dtype=torch.float64)
    f = f - f.mean(1, keepdim=True)
    taps = {}
    ref = oe.ecapa_forward(f, W64, taps=taps)
    emb = model(f.float().to(cuda))
    torch.cuda.synchronize()
    # per-layer parity first: localises a broken kernel
    for name in ["feat", "blocks.0", "blocks.1", "blocks.2", "blocks.3", "mfa", "asp"]:
        got = model.read_tap(name, 3, T).double().cpu()
        want = f if name == "feat" else taps[name]
        if name not in ("feat", "asp"):
            want = want.transpose(1, 2)  # oracle is [B,C,T]
        rel = (got - want).norm() / want.norm()
        assert rel < 2e-5, (name, rel.item())
    emb = emb.double().cpu()
    assert np.abs(emb.numpy() - g[f"emb_T{T}"]).max() < 2e-5
    cos = torch.nn.functional.cosine_similarity(emb, ref)
    assert (1 - cos).max() < 1e-8
    # score parity: all-pairs cosine between the 3 embeddings
    assert np.abs(oh.cosine_matrix(emb.numpy(), emb.numpy()) - oh.cosine_matrix(ref.numpy(), ref.numpy())).max() < COS_TOL


@pytest.mark.parametrize("B,T", [(1, 28), (2, 33), (5, 150), (32, 298), (3, 1998)])
def test_shapes(cuda, model, W64, B, T):
    gi = torch.Generator().manual_seed(B * 1000 + T)
    f = torch.randn(B, T, 80, generator=gi)
    ref = oe.ecapa_forward(f[: min(B, 4)].double(), W64)
    emb = model(f.to(cuda)).double().cpu()
    assert emb.shape == (B, 192)
    rel = (emb[: min(B, 4)] - ref).norm(dim=1) / ref.norm(dim=1)
    assert rel.max() < 2e-5, rel


def test_waveform_to_embedding_and_scores(cuda, model, W64, golden_dir):
    """End to end on the reference's own wavs (a_*, b_* from dataset/): waveform -> Fbank -> ECAPA -> cosine
    score matrix; scores within 1e-4 of the oracle path."""
    g = np.load(f"{golden_dir}/fbank_wavs.npz")
    fz = AudioFeaturizer("Fbank", {"sr": 16000, "n_mels": 80})
    embs, refs = [], []
    for name in ["a_1", "a_2", "b_1", "b_2"]:
        x = ofb.db_normalize(g[name + "_pcm"].astype(np.float32) / 32768.0, -20.0)
        ref_feat = torch.from_numpy(ofb.audio_featurizer_fbank(x, None, dtype=np.float64, n_mels=80))
        refs.append(oe.ecapa_forward(ref_feat, W64)[0])
        xt = torch.from_numpy(x).to(cuda)
        e1 = model(fz(xt))
        e2 = model.forward_wav(fz, xt)
        assert (e1 - e2).abs().max().item() < 1e-5  # fused path == two-call path
        embs.append(e2[0].double().cpu())
    E, R = torch.stack(embs).numpy(), torch.stack(refs).numpy()
    assert np.abs(oh.cosine_matrix(E, E) - oh.cosine_matrix(R, R)).max() < COS_TOL


def test_batch_padding_semantics(cuda, model, W64):
    """predict_batch (predict.py:247-266): zero-padded waveforms + lens ratio; the mean is taken over padded
    frames and the tail is masked after it (featurizer.py:48-59) -- replicate, then compare with the oracle."""
    gen = torch.Generator().manual_seed(7)
    lens = [48000, 30000, 20000]
    x = torch.zeros(3, 48000)
    for i, n in enumerate(lens):
        x[i, :n] = (0.1 * torch.randn(n, generator=gen)).clamp(-1, 1)
    ratio = torch.tensor([n / 48000 for n in lens])
    fz = AudioFeaturizer("Fbank", {"sr": 16000, "n_mels": 80})
    emb = model.forward_wav(fz, x.to(cuda), ratio).double().cpu()
    feat = torch.from_numpy(ofb.audio_featurizer_fbank(x.numpy(), ratio.numpy(), dtype=np.float64, n_mels=80))
    ref = oe.ecapa_forward(feat, W64)
    rel = (emb - ref).norm(dim=1) / ref.norm(dim=1)
    assert rel.max() < 5e-5, rel


def test_forward_wav_refuses_training_mode(cuda, model):
    """forward_wav is the eval-mode forward, as forward is: a model in training mode raises instead of embedding in eval mode"""
    fz = AudioFeaturizer("Fbank", {"sr": 16000, "n_mels": 80})
    model.train()
    try:
        with pytest.raises(PPVError, match=r"call \.eval\(\)"):
            model.forward_wav(fz, torch.zeros(1, 16000, device=cuda))
    finally:
        model.eval()


def test_bf16_fast_mode_is_close_but_flagged(cuda, W64):
    m = make_model(cuda, W64, precision="bf16")
    gi = torch.Generator().manual_seed(3)
    f = torch.randn(4, 298, 80, generator=gi)
    ref = oe.ecapa_forward(f.double(), W64)
    emb = m(f.to(cuda)).double().cpu()
    cos = torch.nn.functional.cosine_similarity(emb, ref)
    assert (1 - cos).max() < 1e-3  # fast mode: NOT within the 1e-4 score tolerance, hence not the default


def test_full_size_properties(cuda, model, W64):
    """BASELINE config 2 (256 x 298 frames): utterances are independent -- a row of the big batch equals the
    same utterance run alone (bit-exact: same kernels, same per-row arithmetic); embeddings finite; and a DIRECT comparison of
    8 rows of the full-size batch with the fp64 oracle (both ends of the batch, both waves of the one-CTA-per-utterance kernels)."""
    gi = torch.Generator().manual_seed(1000)
    f = torch.randn(256, 298, 80, generator=gi).to(cuda)
    emb = model(f)
    assert emb.shape == (256, 192) and torch.isfinite(emb).all()
    for b in (0, 100, 255):
        single = model(f[b:b + 1])
        assert torch.equal(single, emb[b:b + 1])
    rows = [0, 1, 100, 147, 148, 200, 254, 255]
    ref = oe.ecapa_forward(f[rows].double().cpu(), W64)
    got = emb[rows].double().cpu()
    rel = (got - ref).norm(dim=1) / ref.norm(dim=1)
    assert rel.max() < 1e-4, rel
    assert (1 - torch.nn.functional.cosine_similarity(got, ref)).max() < 1e-8
    s_ref = oh.cosine_matrix(ref.numpy(), ref.numpy())
    s_got = oh.cosine_matrix(got.numpy(), got.numpy())
    assert np.abs(s_ref - s_got).max() < COS_TOL


@pytest.mark.parametrize("pooling_type", ["SAP", "TAP", "TSP"])
@pytest.mark.parametrize("T", [98, 298])
def test_other_pooling_types(cuda, pooling_type, T):
    """EcapaTdnn(pooling_type=...) of the reference (ecapa_tdnn.py:212-243, pooling.py:8-66): self-attentive, average and
    mean | unbiased-variance pooling, each followed by paddle.nn.BatchNorm1D and the fc conv."""
    from oracle import ecapa as oe_
    from ppvector.models.ecapa_tdnn import EcapaTdnn as Model
    W = oe_.make_ecapa_weights(seed=1000, dtype=torch.float64, pooling_type=pooling_type)
    m = Model(input_size=80, pooling_type=pooling_type).eval()
    m.load_state_dict({k: v.float() for k, v in W.items()}, strict=True)
    m.to(cuda)
    gi = torch.Generator().manual_seed(77 + T)
    f = torch.randn(3, T, 80, generator=gi, dtype=torch.float64)
    f = f - f.mean(1, keepdim=True)
    ref = oe_.ecapa_forward(f, W, pooling_type=pooling_type)
    emb = m(f.float().to(cuda)).double().cpu()
    rel = (emb - ref).norm(dim=1) / ref.norm(dim=1)
    assert rel.max() < 1e-4, (pooling_type, rel)
    cos = torch.nn.functional.cosine_similarity(emb, ref)
    assert (1 - cos).max() < 1e-8
    with pytest.raises(Exception):
        Model(input_size=80, pooling_type="XYZ")


@pytest.mark.parametrize("T", [9, 121, 249, 250, 376, 377])
def test_fused_res2net_chain_equals_per_conv_path(cuda, monkeypatch, T):
    """csrc/res2chain.cu (one utterance per CTA, operand resident in shared memory) against csrc/res2conv.cu (one launch per conv) on
    awkward lengths: padded lengths 17, 129, 257, 258 (a last tile of one or two rows), 384 (the largest the chain takes) and 385
    (falls back).  The two paths round x_{j+1} + y_j at different places, hence ~1e-6 and not bitwise."""
    from ppvector.models.ecapa_tdnn import EcapaTdnn as Model
    from ppvector.utils.init import seeded_state_dict
    sd = seeded_state_dict(Model(input_size=80), seed=1)
    g = torch.Generator().manual_seed(1)
    x = torch.randn(5, T, 80, generator=g).to(cuda)
    outs = []
    for flag in ("1", "0"):
        monkeypatch.setenv("PPV_RES2_CHAIN", flag)
        m = Model(input_size=80).eval()
        m.load_state_dict(sd)
        m.to(cuda)
        outs.append(m(x).double().cpu())
    assert torch.isfinite(outs[0]).all()
    assert (outs[0] - outs[1]).norm() / outs[1].norm() < 1e-5


@pytest.mark.parametrize("T", [98, 298])
def test_lengths_masking_matches_reference_fixture(cuda, model, W64, golden_dir, T):
    """`lengths` (ecapa_tdnn.py:245; SEBlock :71-75, ASP pooling.py:96-115): the CUDA path against the oracle, and at T = 98 against
    the embedding the REFERENCE's own code produced (tests/golden/ref_models.npz, lengths = [1.0, 0.6])."""
    gi = torch.Generator().manual_seed(1000 + T)
    f = torch.randn(2, T, 80, generator=gi, dtype=torch.float64)
    f = f - f.mean(1, keepdim=True)
    lens = torch.tensor([1.0, 0.6], dtype=torch.float64)
    ref = oe.ecapa_forward(f, W64, lengths=lens)
    emb = model(f.float().to(cuda), lengths=lens.float().to(cuda)).double().cpu()
    rel = (emb - ref).norm(dim=1) / ref.norm(dim=1)
    assert rel.max() < 1e-4, rel
    assert (1 - torch.nn.functional.cosine_similarity(emb, ref)).max() < 1e-8
    if T == 98:
        g = np.load(f"{golden_dir}/ref_models.npz")
        want = torch.from_numpy(g["ecapa_T98_lengths_emb"])
        assert ((emb - want).norm(dim=1) / want.norm(dim=1)).max() < 1e-4
    # row 0 has lengths 1.0: identical to the un-masked forward; row 1 differs
    plain = model(f.float().to(cuda)).double().cpu()
    assert torch.allclose(plain[0], emb[0], rtol=0, atol=1e-6)
    assert (plain[1] - emb[1]).abs().max() > 1e-3
    # odd ratios: the count is #{t : t < ratio * T} (float compare, utils.py:8-19)
    for r in (0.013, 0.5, 0.999):
        lens = torch.tensor([r, 1.0], dtype=torch.float64)
        ref = oe.ecapa_forward(f, W64, lengths=lens)
        emb = model(f.float().to(cuda), lengths=lens.float().to(cuda)).double().cpu()
        assert ((emb - ref).norm(dim=1) / ref.norm(dim=1)).max() < 1e-4, r


def test_asp_without_global_context(cuda, golden_dir):
    """AttentiveStatisticsPooling(global_context=False) (pooling.py:77-78, 108-109) against the oracle and the reference-code fixture."""
    Wg = oe.make_ecapa_weights(seed=1000, dtype=torch.float64, global_context=False)
    m = EcapaTdnn(input_size=80, global_context=False).eval()
    m.load_state_dict({k: v.float() for k, v in Wg.items()}, strict=True)
    m.to(cuda)
    gi = torch.Generator().manual_seed(1000 + 98)
    f = torch.randn(2, 98, 80, generator=gi, dtype=torch.float64)
    f = f - f.mean(1, keepdim=True)
    ref = oe.ecapa_forward(f, Wg, global_context=False)
    emb = m(f.float().to(cuda)).double().cpu()
    assert ((emb - ref).norm(dim=1) / ref.norm(dim=1)).max() < 1e-4
    want = torch.from_numpy(np.load(f"{golden_dir}/ref_models.npz")["ecapa_T98_noctx_emb"])
    assert ((emb - want).norm(dim=1) / want.norm(dim=1)).max() < 1e-4
