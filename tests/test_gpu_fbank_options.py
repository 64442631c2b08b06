"""GPU: the Fbank front end at any sample rate and frame length, with kaldi.fbank's framing, window and spectrum options.  Both
kernels (the 512-point register-resident one and the general per-frame one) against the fp64 oracle over the option grid of
tests/fbank_options_cases.py, ragged batches against per-utterance calls for either snip_edges setting, the refused FFT sizes, and an
8 kHz model through the fused waveform path and through PPVectorPredictor."""
import copy
import os

import numpy as np
import pytest
import torch
import yaml

import fbank_options_oracle as ofb
from fbank_options_cases import CASES, frame_geometry, oracle_kwargs
from oracle import ecapa as oe
from oracle import head as oh
from oracle.fbank import db_normalize
from ppvector._lib import PPVError
from ppvector.data_utils.featurizer import AudioFeaturizer

pytestmark = pytest.mark.gpu

TOL_MAX = 2e-3  # the bounds of tests/test_gpu_fbank.py
TOL_MEAN = 5e-5
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _waves(lengths, seed):
    g = torch.Generator().manual_seed(seed)
    return [(0.1 * torch.randn(n, generator=g)).clamp(-1, 1) for n in lengths]


def _check(out, ref, what):
    """log domain: absolute bounds; linear mel energies: the same bounds relative to the largest energy"""
    d = np.abs(np.asarray(out, np.float64) - ref) / max(1.0, float(np.abs(ref).max()))
    assert d.max() < TOL_MAX and d.mean() < TOL_MEAN, (what, d.max(), d.mean())


@pytest.mark.parametrize("case", sorted(CASES))
def test_batch_with_tail_mask_vs_oracle(cuda, case):
    args = CASES[case]
    sr = args["sr"]
    L = int(1.5 * sr) + 7
    x = torch.stack(_waves([L] * 3, seed=len(case)))
    ratio = np.array([1.0, 0.71, 0.4], np.float32)
    fz = AudioFeaturizer("Fbank", args)
    out = fz(x.to(cuda), torch.from_numpy(ratio)).cpu().numpy()
    win, shift, snip = frame_geometry(args)
    assert out.shape == (3, ofb.num_frames(L, win, shift, snip), args["n_mels"]) == (3, fz.num_frames(L), fz.feature_dim)
    ref = ofb.audio_featurizer_fbank(x.numpy(), ratio, dtype=np.float64, **oracle_kwargs(args))
    _check(out, ref, case)


@pytest.mark.parametrize("case", sorted(CASES))
def test_ragged_mixed_lengths_vs_oracle(cuda, case):
    """utterances of different lengths in one zero-padded batch, each featurised as if alone (its own frames, its own mean, its own
    right edge with snip_edges=False), against the oracle on each utterance alone"""
    args = CASES[case]
    sr = args["sr"]
    win, shift, snip = frame_geometry(args)
    lens = [int(1.2 * sr), win + 3 * shift + 1, int(0.5 * sr) + 5, win]
    ws = _waves(lens, seed=7 + len(case))
    batch = torch.zeros(len(lens), max(lens))
    for b, w in enumerate(ws):
        batch[b, :len(w)] = w
    fz = AudioFeaturizer("Fbank", args)
    feats, frames = fz.forward_ragged(batch.to(cuda), lens)
    assert frames == [ofb.num_frames(n, win, shift, snip) for n in lens]
    feats = feats.cpu().numpy()
    for b, w in enumerate(ws):
        ref = ofb.audio_featurizer_fbank(w.numpy(), None, dtype=np.float64, **oracle_kwargs(args))[0]
        _check(feats[b, :frames[b]], ref, (case, lens[b]))
        assert (feats[b, frames[b]:] == 0).all()


@pytest.mark.parametrize("snip", [True, False])
@pytest.mark.parametrize("sr", [8000, 16000])
def test_ragged_equals_per_utterance(cuda, snip, sr):
    fz = AudioFeaturizer("Fbank", {"sr": sr, "n_mels": 80, "snip_edges": snip})
    lens = [3 * sr, sr, int(0.025 * sr), 30011 * sr // 16000, 3 * sr - 1]
    ws = _waves(lens, seed=sr + snip)
    batch = torch.zeros(len(lens), max(lens))
    for b, w in enumerate(ws):
        batch[b, :len(w)] = w
    feats, frames = fz.forward_ragged(batch.to(cuda), lens)
    assert frames == [fz.num_frames(n) for n in lens] and feats.shape == (5, max(frames), 80)
    for b, w in enumerate(ws):
        alone = fz(w.to(cuda))[0]
        assert torch.equal(feats[b, :frames[b]], alone), b  # same kernels, same per-utterance arithmetic: bit-exact
        assert (feats[b, frames[b]:] == 0).all()


def test_short_inputs_without_snip_edges(cuda):
    """snip_edges=False on inputs shorter than the window and than the reflection pad (16 kHz, 25 ms / 2.5 ms: pad = 180), against
    the oracle's _get_strided framing; lengths that leave no frame, or whose reflection cannot hold the last one, are refused"""
    args = {"sr": 16000, "n_mels": 40, "frame_shift": 2.5, "snip_edges": False}
    fz = AudioFeaturizer("Fbank", args)
    for L in (179, 200, 250, 399, 400, 401, 560):
        T = ofb.num_frames(L, 400, 40, snip_edges=False)
        assert fz.num_frames(L) == T, L
        x = _waves([L], seed=L)[0]
        if T == 0:
            with pytest.raises(PPVError):
                fz(x.to(cuda))
            continue
        ref = ofb.audio_featurizer_fbank(x.numpy(), None, dtype=np.float64, **oracle_kwargs(args))
        _check(fz(x.to(cuda)).cpu().numpy(), ref, L)
    assert fz.num_frames(170) == 0 and fz.num_frames(19) == 0
    with pytest.raises(PPVError):
        fz(torch.zeros(1, 19, device=cuda))  # (19 + 20) // 40 = 0 frames


@pytest.mark.parametrize("args,nfft", [({"sr": 16000, "frame_length": 3.0}, 64), ({"sr": 16000, "frame_length": 300.0}, 8192),
                                       ({"sr": 48000, "frame_length": 100.0}, 8192)])
def test_out_of_range_fft_sizes_are_refused(cuda, args, nfft):
    fz = AudioFeaturizer("Fbank", dict(args, n_mels=40))
    with pytest.raises(PPVError, match=f"{nfft}-point FFT"):
        fz(torch.zeros(1, 48000, device=cuda))


def test_bad_vtln_is_refused(cuda):
    fz = AudioFeaturizer("Fbank", {"sr": 8000, "n_mels": 40, "vtln_warp": 0.9, "vtln_low": 10.0})  # vtln_low below low_freq
    with pytest.raises(PPVError, match="vtln"):
        fz(torch.zeros(1, 8000, device=cuda))


def test_long_utterances_fold_their_partial_sums(cuda):
    """more than 64 items per utterance: the general kernel's per-item sums go through the same fold as the specialised kernel's"""
    args = {"sr": 8000, "n_mels": 80, "snip_edges": False}
    x = torch.stack(_waves([8000 * 20] * 2, seed=3))
    out = AudioFeaturizer("Fbank", args)(x.to(cuda)).cpu().numpy()
    ref = ofb.audio_featurizer_fbank(x.numpy(), None, dtype=np.float64, **oracle_kwargs(args))
    _check(out, ref, "20 s")


@pytest.fixture(scope="module")
def W64():
    return oe.make_ecapa_weights(seed=1000, dtype=torch.float64)


def test_8k_ecapa_forward_wav_equals_model_of_featurizer(cuda, W64):
    from ppvector.models.ecapa_tdnn import EcapaTdnn
    model = EcapaTdnn(input_size=80).eval()
    model.load_state_dict({k: v.float() for k, v in W64.items()})
    model.to(cuda)
    for args in ({"sr": 8000, "n_mels": 80}, {"sr": 8000, "n_mels": 80, "snip_edges": False, "window_type": "hamming"}):
        fz = AudioFeaturizer("Fbank", args)
        x = torch.stack(_waves([24000] * 4, seed=11)).to(cuda)
        ratio = torch.tensor([1.0, 0.8, 0.6, 0.5])
        fused = model.forward_wav(fz, x, ratio)
        two_calls = model(fz(x, ratio))
        assert torch.allclose(fused, two_calls, rtol=0, atol=1e-5), (fused - two_calls).abs().max()
        feat = torch.from_numpy(ofb.audio_featurizer_fbank(x.cpu().numpy(), ratio.numpy(), dtype=np.float64, **oracle_kwargs(args)))
        ref = oe.ecapa_forward(feat, W64)
        rel = (fused.double().cpu() - ref).norm(dim=1) / ref.norm(dim=1)
        assert rel.max() < 5e-5, rel


def test_predictor_at_8k(cuda, W64, golden_dir):
    from ppvector.predict import PPVectorPredictor
    cfg = copy.deepcopy(yaml.load(open(os.path.join(ROOT, "configs", "ecapa_tdnn.yml")), Loader=yaml.FullLoader))
    cfg["dataset_conf"]["dataset"]["sample_rate"] = 8000
    cfg["preprocess_conf"]["method_args"]["sr"] = 8000
    pred = PPVectorPredictor(cfg, model_path=None, use_gpu=True, state_dict={k: v.float().numpy() for k, v in W64.items()})
    g = np.load(f"{golden_dir}/fbank_wavs.npz")
    pcm = g["a_1_pcm"][::2]  # 8 kHz audio: no resampling on the way in
    e = pred.predict(pcm, sample_rate=8000)
    assert e.shape == (192,) and np.isfinite(e).all()
    x = db_normalize(pcm.astype(np.float32) / 32768.0, -20.0)
    feat = torch.from_numpy(ofb.audio_featurizer_fbank(x, None, dtype=np.float64, n_mels=80, sr=8000))
    ref = oe.ecapa_forward(feat, W64)[0].numpy()
    assert 1 - oh.cosine_pair(e, ref) < 1e-8
