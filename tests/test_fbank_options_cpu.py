"""CPU: the Fbank front end's options -- the fp64 oracle against torchaudio.compliance.kaldi.fbank over sample rates, FFT sizes
128..4096, window types, snip_edges framing of short inputs, DC / power / log switches, VTLN and subtract_mean; and
AudioFeaturizer's mapping of paddleaudio's keyword names onto ppv_fbank_cfg, with the three refusals."""
import numpy as np
import pytest
import torch
import torchaudio

import fbank_options_oracle as ofb
from fbank_options_cases import CASES, frame_geometry, oracle_kwargs, torchaudio_kwargs
from ppvector import _lib
from ppvector.data_utils.featurizer import AudioFeaturizer

# fp64 on both sides; the mel weights are float32 on both sides (get_mel_banks), so what is left is fp64 rounding
TOL = 1e-9


def _wave(n, seed):
    g = np.random.default_rng(seed)
    t = np.arange(n) / 16000.0
    return 0.3 * np.sin(2 * np.pi * 440.0 * t) + 0.05 * g.standard_normal(n)


def _torchaudio(x, args):
    return torchaudio.compliance.kaldi.fbank(torch.from_numpy(x)[None], **torchaudio_kwargs(args)).numpy()


@pytest.mark.parametrize("case", sorted(CASES))
def test_oracle_matches_torchaudio(case):
    args = CASES[case]
    x = _wave(int(args["sr"] * 0.7) + 13, seed=len(case))
    want = _torchaudio(x, args)
    got = ofb.kaldi_fbank(x, dtype=np.float64, **oracle_kwargs(args))
    assert got.shape == want.shape and got.shape[0] > 0
    d = np.abs(got - want).max() / max(1.0, np.abs(want).max())
    assert d < TOL, (case, d)


# snip_edges=False at 16 kHz / 25 ms / 10 ms (pad = 120) and at 16 kHz / 25 ms / 2.5 ms (pad = 180); torchaudio's fbank refuses
# L < window, so the framing is pinned against its _get_strided directly there
SHORT = [(400, 160, L) for L in (81, 200, 250, 399, 400, 401, 559, 560)] + [(400, 40, L) for L in (150, 170, 179, 200, 399)]


@pytest.mark.parametrize("win,shift,L", SHORT)
def test_short_input_framing_matches_torchaudio(win, shift, L):
    x = np.arange(L, dtype=np.float64) + 1.0
    T = ofb.num_frames(L, win, shift, snip_edges=False)
    assert T == 0 or T == (L + shift // 2) // shift
    try:
        want = torchaudio.compliance.kaldi._get_strided(torch.from_numpy(x), win, shift, False).numpy()
    except RuntimeError:  # the reflected waveform cannot hold the last frame: as_strided refuses the view
        want = None
    if T == 0:
        assert want is None, (win, shift, L)
        assert ofb.frame_signal(x, win, shift, snip_edges=False).shape == (0, win)
        return
    np.testing.assert_array_equal(ofb.frame_signal(x, win, shift, snip_edges=False), want)
    assert ofb.num_frames(L, win, shift, snip_edges=True) == (0 if L < win else 1 + (L - win) // shift)


def test_short_utterances_through_the_whole_oracle():
    """snip_edges=False on inputs down to L = window (torchaudio's fbank floor), and the one-frame snip_edges case"""
    for L in (400, 401, 559, 560, 800):
        x = _wave(L, seed=L)
        args = dict(sr=16000, n_mels=80, snip_edges=False)
        want, got = _torchaudio(x, args), ofb.kaldi_fbank(x, dtype=np.float64, **oracle_kwargs(args))
        assert got.shape == want.shape == ((L + 80) // 160, 80)
        assert np.abs(got - want).max() < TOL * 100
    x = _wave(400, seed=1)
    assert ofb.kaldi_fbank(x, dtype=np.float64).shape == (1, 80)
    assert ofb.kaldi_fbank(x[:399], dtype=np.float64).shape == (0, 80)


def test_vtln_banks_match_torchaudio():
    for warp, sr, lo, hi in ((0.9, 16000, 100.0, -500.0), (1.1, 16000, 100.0, -500.0), (0.85, 8000, 300.0, 3000.0)):
        want, _ = torchaudio.compliance.kaldi.get_mel_banks(80, 512, float(sr), 20.0, 0.0, lo, hi, warp)
        got = ofb.mel_banks(80, 512, float(sr), 20.0, 0.0, np.float32, lo, hi, warp)[:, :-1]
        assert np.abs(got - want.numpy()).max() < 1e-6, warp
        assert not np.array_equal(got, ofb.mel_banks(80, 512, float(sr))[:, :-1])


def test_keyword_mapping():
    cfg = AudioFeaturizer._fbank_cfg(dict(sr=8000, n_mels=64, frame_length=50.0, frame_shift=12.5, preemphasis_coefficient=0.9,
                                          low_freq=40.0, high_freq=-200.0, window_type="blackman", blackman_coeff=0.4,
                                          remove_dc_offset=False, snip_edges=False, use_power=False, use_log_fbank=False,
                                          vtln_warp=1.1, vtln_low=150.0, vtln_high=-600.0, htk_compat=True, raw_energy=False,
                                          energy_floor=1.0, subtract_mean=True, dither=0.0, use_energy=False,
                                          round_to_power_of_two=True))
    assert (cfg.sample_rate, cfg.n_mels, cfg.frame_length_ms, cfg.frame_shift_ms) == (8000, 64, 50.0, 12.5)
    assert abs(cfg.preemph - 0.9) < 1e-7 and (cfg.low_freq, cfg.high_freq) == (40.0, -200.0)
    assert cfg.window_type == _lib.PPV_FBANK_WIN_BLACKMAN and abs(cfg.blackman_coeff - 0.4) < 1e-7
    assert (cfg.remove_dc_offset, cfg.snip_edges, cfg.use_power, cfg.use_log_fbank) == (0, 0, 0, 0)
    assert abs(cfg.vtln_warp - 1.1) < 1e-7 and (cfg.vtln_low, cfg.vtln_high) == (150.0, -600.0)
    d = AudioFeaturizer._fbank_cfg({})
    assert (d.window_type, d.remove_dc_offset, d.snip_edges, d.use_power, d.use_log_fbank) == (_lib.PPV_FBANK_WIN_POVEY, 1, 1, 1, 1)
    assert (d.vtln_warp, d.vtln_low, d.vtln_high, d.n_mels) == (1.0, 100.0, -500.0, 23)
    assert abs(d.blackman_coeff - 0.42) < 1e-7
    for name, code in (("povey", 0), ("hanning", 1), ("hamming", 2), ("rectangular", 3), ("blackman", 4)):
        assert AudioFeaturizer._fbank_cfg({"window_type": name}).window_type == code
    assert AudioFeaturizer("Fbank", {"sr": 8000, "n_mels": 80, "snip_edges": False}).feature_dim == 80


@pytest.mark.parametrize("args,match", [({"dither": 1.0}, "random generator"), ({"use_energy": True}, "n_mels \\+ 1"),
                                        ({"round_to_power_of_two": False}, "power of two"), ({"window_type": "kaiser"}, "window_type"),
                                        ({"channel": 0}, "not supported"), ({"min_duration": 0.1}, "not supported")])
def test_refusals(args, match):
    with pytest.raises(_lib.PPVError, match=match):
        AudioFeaturizer("Fbank", args)


def test_case_grid_covers_every_fft_size():
    from oracle.fbank import next_pow2
    sizes = {next_pow2(frame_geometry(a)[0]) for a in CASES.values()}
    assert sizes == {128, 256, 512, 1024, 2048, 4096}
