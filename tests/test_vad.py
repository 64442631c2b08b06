"""CPU: the energy voice-activity detection (DESIGN.md §1, f8) -- the fp64 oracle's log energy against torchaudio's Kaldi fbank energy
column, hand-worked decision and post-processing cases, and the host plumbing (AudioSegment.vad, SpeakerDiarization.segments_audio,
the predictor's vad / vad_segments options, the command line) with the GPU call stubbed."""
import numpy as np
import pytest
import torch

import vad_oracle as vo
from ppvector.data_utils.audio import AudioSegment
from ppvector.infer_utils import vad as pvad


def kaldi_energy(x, sample_rate=16000):
    """Column 0 of torchaudio's Kaldi fbank on the 16-bit scale: raw energy, no dither, no energy floor (fp32)."""
    import torchaudio
    feats = torchaudio.compliance.kaldi.fbank(torch.from_numpy(np.asarray(x, dtype=np.float32) * 32768.0)[None], use_energy=True,
                                              raw_energy=True, dither=0.0, energy_floor=0.0, sample_frequency=sample_rate)
    return feats[:, 0].double().numpy()


def bursts(seed, sr=16000, seconds=6.0):
    """Tonal and noise bursts separated by quiet pauses."""
    rng = np.random.default_rng(seed)
    x = 1e-3 * rng.standard_normal(int(sr * seconds))
    t = 0
    while t < x.size:
        n = int(sr * rng.uniform(0.2, 0.8))
        if rng.random() < 0.6:
            k = np.arange(min(n, x.size - t))
            x[t:t + k.size] += (0.3 * np.sin(2 * np.pi * rng.uniform(100, 900) * k / sr) if rng.random() < 0.5
                                else 0.2 * rng.standard_normal(k.size))
        t += n
    return x.astype(np.float32)


@pytest.mark.parametrize("seed", [0, 1, 2])
@pytest.mark.parametrize("sr", [8000, 16000])
def test_oracle_energy_matches_torchaudio(seed, sr):
    x = bursts(seed, sr)
    win, shift = vo.geometry(sr)
    e = vo.log_energy(x, win, shift)
    ref = kaldi_energy(x, sr)
    assert e.shape == ref.shape and np.abs(e - ref).max() <= 1e-4


def test_oracle_energy_on_the_reference_wavs(golden_dir):
    """The reference project's bundled recordings (16-bit PCM, kept in tests/golden/fbank_wavs.npz)."""
    g = np.load(f"{golden_dir}/fbank_wavs.npz")
    for name in ("a_1", "a_2", "b_1", "b_2", "long3s"):
        x = g[f"{name}_pcm"].astype(np.float32) / 32768.0
        e = vo.log_energy(x, 400, 160)
        assert np.abs(e - kaldi_energy(x)).max() <= 1e-4, name


def test_frame_counts_at_the_edges():
    win, shift = 400, 160
    assert vo.num_frames(win - 1, win, shift) == 0 and vo.log_energy(np.zeros(win - 1), win, shift).shape == (0,)
    assert vo.num_frames(win, win, shift) == 1
    for k in (1, 5, 37):
        assert vo.num_frames(win + k * shift - 1, win, shift) == k
        assert vo.num_frames(win + k * shift, win, shift) == k + 1
        assert vo.num_frames(win + k * shift + 1, win, shift) == k + 1
    r = vo.vad(np.ones(win - 1, dtype=np.float32))
    assert r['runs'] == [] and r['segments'] == []


def test_context_window_shrinks_at_both_ends():
    e = np.array([10.0, 0, 0, 0, 0, 0, 10.0])
    # den = 3, 4, 5, 5, 5, 4, 3; only the end frames have num / den >= 0.3
    assert vo.decide(e, 5.0, frames_context=2, proportion_threshold=0.3).tolist() == [1, 0, 0, 0, 0, 0, 1]
    assert vo.decide(e, 5.0, frames_context=0, proportion_threshold=0.3).tolist() == [1, 0, 0, 0, 0, 0, 1]
    assert vo.decide(e, 5.0, frames_context=6, proportion_threshold=0.25).tolist() == [1] * 7  # 2 of 7 everywhere


def test_decision_at_equality_and_in_fp32():
    # num == den * p exactly: voiced
    assert vo.decide(np.array([0.0, 10.0, 0.0, 0.0]), 5.0, frames_context=1, proportion_threshold=0.5).tolist() == [1, 0, 0, 0]
    # 15 of 25 frames at Kaldi's default p = 0.6: float32(25) * float32(0.6) = 15.000001 > 15, so the frame is unvoiced; in fp64 with
    # the decimal 0.6 the product is 15.0 and it would be voiced.  The product is fp32, as in Kaldi.
    e = np.zeros(25)
    e[:15] = 10.0
    assert not vo.decide(e, 5.0, frames_context=12, proportion_threshold=0.6)[12]
    assert 15 >= 25 * 0.6


def test_threshold_and_mean_scale_zero():
    e = np.array([1.0, 2.0, 3.0, 6.0])
    assert vo.threshold(e, 5.5, 0.0) == 5.5
    assert vo.threshold(e, 5.5, 0.5) == 5.5 + 0.5 * 12.0 / 4
    assert vo.decide(e, vo.threshold(e, 5.5, 0.0), 0, 0.5).tolist() == [0, 0, 0, 1]


@pytest.mark.parametrize("value", [0.0, 0.3])
def test_silent_and_constant_recordings_have_no_speech(value):
    x = np.full(16000, value, dtype=np.float32)
    r = vo.vad(x)
    assert np.all(r['e'] == np.log(np.float32(np.finfo(np.float32).eps).astype(np.float64)))
    assert abs(r['thr'] - (5.5 + 0.5 * r['e'][0])) < 1e-12 and not r['voiced'].any() and r['segments'] == []


# ---- post-processing, at 1 kHz (window 25, shift 10, one sample per millisecond) -----------------------------------------------------
SR = 1000


@pytest.mark.parametrize("segments", [vo.segments, lambda runs, L, sr, *a: pvad.speech_segments(runs, L, sr, *a)])
def test_post_processing_by_hand(segments):
    assert pvad.frame_geometry(SR) == vo.geometry(SR) == (25, 10)
    two = [(0, 10), (13, 40)]  # samples [0, 115) and [130, 415): gap 15
    assert segments(two, 1000, SR, 0, 16, 0) == [{'start': 0, 'end': 415}]  # gap = min_silence - 1: merged
    assert segments(two, 1000, SR, 0, 15, 0) == [{'start': 0, 'end': 115}, {'start': 130, 'end': 415}]  # gap = min_silence: kept apart
    assert segments([(0, 10)], 1000, SR, 115, 0, 0) == [{'start': 0, 'end': 115}]  # exactly min_speech: kept
    assert segments([(0, 10)], 1000, SR, 116, 0, 0) == []  # one sample short: dropped
    # drop after merge: the merged run is long enough even though each part alone is not
    assert segments(two, 1000, SR, 400, 16, 0) == [{'start': 0, 'end': 415}]
    # pads of 10 around a gap of 15 < 20: each side moves by 7; the outer sides are clamped to [0, L]
    assert segments(two, 420, SR, 0, 0, 10) == [{'start': 0, 'end': 122}, {'start': 123, 'end': 420}]
    assert segments([(3, 10)], 1000, SR, 0, 0, 10) == [{'start': 20, 'end': 125}]
    # overlapping frame spans (gap < 0) merge even at min_silence 0
    assert segments([(0, 10), (11, 20)], 1000, SR, 0, 0, 0) == [{'start': 0, 'end': 215}]
    assert segments([], 1000, SR, 0, 0, 10) == []


def test_product_post_processing_equals_the_oracle_on_random_runs():
    rng = np.random.default_rng(0)
    for trial in range(200):
        v = rng.random(400) < rng.uniform(0.05, 0.95)
        runs = vo.runs(v)
        L = 16000 * 4 + int(rng.integers(0, 160))
        opts = [int(rng.integers(0, 400)), int(rng.integers(0, 200)), int(rng.integers(0, 60))]
        assert pvad.speech_segments(runs, L, 16000, *opts) == vo.segments(runs, L, 16000, *opts), trial


def test_vad_options():
    assert pvad.vad_options() == {**pvad.DECISION_DEFAULTS, **pvad.SEGMENT_DEFAULTS} == vo.DEFAULTS
    assert pvad.vad_options(frames_context=0)['frames_context'] == 0
    with pytest.raises(TypeError, match="threshold_db"):
        pvad.vad_options(threshold_db=3)
    for bad in (dict(frames_context=-1), dict(frames_context=1.5), dict(energy_mean_scale=-0.1), dict(proportion_threshold=0.0),
                dict(proportion_threshold=1.0), dict(energy_threshold=float("nan")), dict(min_speech_ms=-1), dict(speech_pad_ms=-5)):
        with pytest.raises(ValueError):
            pvad.vad_options(**bad)


# ---- host plumbing with the GPU call stubbed --------------------------------------------------------------------------------------------
def test_audio_segment_vad_plumbing(monkeypatch):
    calls = []

    def stub(recs, sr, return_seconds=False, **opts):
        calls.append((len(recs), recs[0].shape, sr, return_seconds, opts))
        return [[{'start': 8000 / sr if return_seconds else 8000, 'end': 24000 / sr if return_seconds else 24000}]]

    monkeypatch.setattr(pvad, "energy_vad", stub)
    seg = AudioSegment(np.zeros(32000, dtype=np.float32), 16000)
    assert seg.vad() == [{'start': 8000, 'end': 24000}]
    assert seg.vad(return_seconds=True, frames_context=0) == [{'start': 0.5, 'end': 1.5}]
    assert calls == [(1, (32000,), 16000, False, {}), (1, (32000,), 16000, True, {'frames_context': 0})]


def test_segments_audio_plumbing(monkeypatch):
    from ppvector.infer_utils.speaker_diarization import SpeakerDiarization
    spans = [{'start': 0.12345, 'end': 3.30071}, {'start': 4.0, 'end': 7.6}]
    monkeypatch.setattr(pvad, "energy_vad", lambda recs, sr, return_seconds=False, **o: [spans])
    x = np.random.default_rng(1).standard_normal(8 * 8000).astype(np.float32)
    sd = SpeakerDiarization()
    chunks = sd.segments_audio(AudioSegment(x, 8000))
    assert sd.sample_rate == 8000
    vad_segments = [[0.123, 3.301, x[984:26408]], [4.0, 7.6, x[32000:60800]]]
    expect = sd._chunk(vad_segments)
    assert len(chunks) == len(expect) > 0
    for c, e in zip(chunks, expect):
        assert c[0] == e[0] and c[1] == e[1] and np.array_equal(c[2], e[2])
    monkeypatch.setattr(pvad, "energy_vad", lambda recs, sr, return_seconds=False, **o: [[{'start': 0.0, 'end': 4.0}]])
    with pytest.raises(AssertionError):  # not more than 5 s of speech
        sd.segments_audio(AudioSegment(x, 8000))


def _bare_predictor():
    import os

    import yaml

    from ppvector.predict import PPVectorPredictor
    from ppvector.utils.utils import dict_to_object
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    p = PPVectorPredictor.__new__(PPVectorPredictor)  # no CUDA in this test: skip __init__
    p.configs = dict_to_object(yaml.load(open(os.path.join(root, "configs", "ecapa_tdnn.yml")), Loader=yaml.FullLoader))
    p.extract_embeddings = lambda w, ratio=None: np.stack([w.mean(1), w.std(1)], 1).astype(np.float32)
    return p


def test_predictor_vad_option(monkeypatch):
    p = _bare_predictor()
    x = (0.1 * np.random.default_rng(5).standard_normal(80000)).astype(np.float32)
    seen = []

    def stub(recs, sr, return_seconds=False, **o):
        seen.append(recs[0].copy())
        return [[{'start': 0.5, 'end': 2.6}, {'start': 3.0, 'end': 3.4}]]

    monkeypatch.setattr(pvad, "energy_vad", stub)
    t, e = p.diarization_embeddings(x, sample_rate=16000, vad=True)
    t2, e2 = p.diarization_embeddings(x, sample_rate=16000, vad_segments=[(0.5, 2.6), (3.0, 3.4)])
    assert np.array_equal(t, t2) and np.array_equal(e, e2)
    assert np.array_equal(seen[0], p._load_audio(x, 16000).samples)  # the VAD sees the loaded (dB-normalised) audio
    for call in (p.diarization_embeddings, p.speaker_diarization):
        with pytest.raises(ValueError, match="not both"):
            call(x, sample_rate=16000, vad=True, vad_segments=[(0.5, 2.6)])
    assert len(seen) == 1


def test_cli_vad_option(capsys):
    import importlib
    import os
    import sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    sys.path.insert(0, root)
    import cli_common
    mod = importlib.import_module("infer_speaker_diarization")
    assert "vad" not in {r[0] for r in mod.OPTIONS}  # the reference's option table stays as it is
    row = [r for r in mod.EXTENSION_OPTIONS if r[0] == "vad"]
    assert len(row) == 1 and row[0][1] is bool and row[0][2] is False
    table = mod.OPTIONS + mod.EXTENSION_OPTIONS
    assert cli_common.parse_options("x", table, ["--vad", "true"]).vad is True
    assert cli_common.parse_options("x", table, []).vad is False
