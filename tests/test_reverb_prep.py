"""CPU: the reverb step of the training data path -- the oracle (tests/reverb_oracle.py) against direct and FFT convolution, the order
of the random draws (speed -> volume -> noise -> reverb -> crop), the crop planned on the reverberant length, and the response bank
(sorted, undecodable files skipped, resampled, a missing / empty directory disables it).  No GPU: the augmentor runs on device='cpu'."""
import random
import types
import wave

import numpy as np
import pytest
import scipy.signal

from oracle import audio_prep as oap
from ppvector.data_utils.audio_batch import WaveAugmentor, augmented_len
from ppvector.data_utils.reader import PPVectorDataset
from reverb_oracle import prepare_reverb, reverb_convolve


def write_wav(path, x, sr=16000):
    with wave.open(str(path), "wb") as w:
        w.setnchannels(1)
        w.setsampwidth(2)
        w.setframerate(sr)
        w.writeframes((np.clip(x, -1, 1) * 32767).astype("<i2").tobytes())


def test_oracle_convolution_direct_and_fft():
    rng = np.random.default_rng(0)
    x = rng.standard_normal(5000)
    for R in (1, 37, 256, 257, 1000):
        h = rng.standard_normal(R)
        y = reverb_convolve(x, h)
        assert y.shape == (5000 + R - 1,)
        direct = np.array([sum(x[n - t] * h[t] for t in range(max(0, n - 4999), min(R, n + 1))) for n in (0, 1, R - 1, 2500, 5000 + R - 2)])
        assert np.allclose(y[[0, 1, R - 1, 2500, 5000 + R - 2]], direct, rtol=1e-12, atol=1e-12)
        assert np.array_equal(y, np.convolve(x, h))
    x = rng.standard_normal(60000)
    h = rng.standard_normal(70000) * np.exp(-np.arange(70000) / 8000.0)  # longer than the utterance
    y = reverb_convolve(x, h)
    ref = scipy.signal.fftconvolve(x, h, "full")
    assert y.shape == (60000 + 70000 - 1,)
    assert np.abs(y - ref).max() <= 1e-9 * np.abs(ref).max()
    # spot check the FFT path against the direct sum
    for n in (0, 59999, 69999, 129998):
        t = np.arange(max(0, n - 59999), min(70000, n + 1))
        assert abs(y[n] - np.dot(x[n - t], h[t])) <= 1e-9 * np.abs(ref).max()


def test_oracle_pipeline_order_and_normalisation():
    rng = np.random.default_rng(1)
    x = (0.1 * rng.standard_normal(3000)).astype(np.float32)
    noise = (0.05 * rng.standard_normal(700)).astype(np.float32)
    h = rng.standard_normal(400) * np.exp(-np.arange(400) / 80.0)
    # un-normalised: exactly the convolution of the noisy, volume-scaled, speed-changed signal; not truncated
    y = oap.change_speed(x, 0.9).astype(np.float64) * 10 ** (3.0 / 20)
    seg = noise.astype(np.float64)[(5 + np.arange(y.shape[0])) % 700]
    y = y + seg * 10 ** (min(oap.rms_db(y) - oap.rms_db(seg) - 20.0, 300.0) / 20)
    want = np.convolve(y, h)
    got = prepare_reverb(x, 0.9, 3.0, noise, 5, 20.0, h, normalize=False)
    assert got.shape == (int(3000 / 0.9) + 399,)
    assert np.abs(got - want).max() <= 1e-6 * np.abs(want).max()
    # normalised: the response's scale cancels, the -20 dB target holds on the whole reverberant utterance
    a = prepare_reverb(x, 1.0, 0.0, rir=h)
    b = prepare_reverb(x, 1.0, 0.0, rir=37.0 * h)
    assert np.abs(a - b).max() < 1e-6 and abs(oap.rms_db(a) + 20.0) < 1e-4
    # no response: the same as the reference oracle
    assert np.array_equal(prepare_reverb(x, 1.1, -4.0, noise, 0, 15.0, None, crop_start=100, crop_len=2000),
                          oap.prepare(x, 1.1, -4.0, noise, 0, 15.0, -20.0, True, 100, 2000))


def make_augmentor(tmp_path, prob=1.0, rir_lens=(800, 3000), noise=True):
    nd, rd = tmp_path / "noise", tmp_path / "rir"
    nd.mkdir(exist_ok=True)
    rd.mkdir(exist_ok=True)
    rng = np.random.default_rng(7)
    if noise:
        write_wav(nd / "n0.wav", 0.1 * rng.standard_normal(8000))
        write_wav(nd / "n1.wav", 0.1 * rng.standard_normal(64000))
    for i, n in enumerate(rir_lens):
        write_wav(rd / f"r{i}.wav", 0.5 * rng.standard_normal(n) * np.exp(-np.arange(n) / 400.0))
    conf = {"speed": {"prob": 0.5, "speed_perturb_3_class": True}, "volume": {"prob": 0.5, "min_gain_dBFS": -15, "max_gain_dBFS": 15},
            "noise": {"prob": 0.5, "noise_dir": str(nd), "min_snr_dB": 10, "max_snr_dB": 50},
            "reverb": {"prob": prob, "reverb_dir": str(rd)}}
    return WaveAugmentor(conf, num_speakers=10, device="cpu"), conf


def hand_sequence(rng, raw_len, spk, noise_clips, rir_clips, max_len):
    """The reference's draws written out: speed, volume, noise, reverb (augment_audio), then the crop start (reader.py:100-101)."""
    rate, spk_out, gain, nz, snr, rv = 1.0, spk, 0.0, None, 0.0, None
    if rng.random() < 0.5:
        k = rng.randint(0, 2)
        rate, spk_out = (1.0, 0.9, 1.1)[k], spk + 10 * k
    if rng.random() < 0.5:
        gain = rng.uniform(-15, 15)
    new_len = raw_len if rate == 1.0 else int(raw_len / rate)
    if rng.random() < 0.5:
        off, n = noise_clips[rng.randint(0, len(noise_clips) - 1)]
        start = rng.randint(0, n - new_len) if n > new_len else 0
        nz = (off + start, n - start if n > new_len else n)
        snr = rng.uniform(10, 50)
    if rng.random() < 0.5:
        rv = rir_clips[rng.randrange(len(rir_clips))]
    full = new_len + (rv[1] - 1 if rv else 0)
    crop = (rng.randint(0, full - max_len), max_len) if full > max_len else (0, None)
    return dict(speed_rate=rate, spk_id=spk_out, vol_gain_db=gain, noise=nz, snr_db=snr, reverb=rv), crop


def test_draw_order_speed_volume_noise_reverb_crop(tmp_path):
    aug, _ = make_augmentor(tmp_path, prob=0.5)
    assert aug.rir_clips == [(0, 800), (800, 3000)] and aug.rir_bank.device.type == "cpu" and aug.rir_bank.numel() == 3800
    ds = types.SimpleNamespace(wave_augment=aug, mode="train", max_duration=3, _target_sample_rate=16000)
    seen = set()
    for seed in range(40):
        raw = 46000 + 37 * seed
        random.seed(seed)
        draw, crop, label = PPVectorDataset._plan(ds, np.zeros(raw, np.float32), 3)
        want_draw, want_crop = hand_sequence(random.Random(seed), raw, 3, aug.noise_clips, aug.rir_clips, 48000)
        assert draw == want_draw and crop == want_crop and label == want_draw["spk_id"], seed
        seen.add(draw["reverb"])
    assert seen == {None, (0, 800), (800, 3000)}


def test_plan_crops_on_the_reverberant_length():
    n = 48000

    class Fixed:
        def __init__(self, d):
            self.d = d

        def draw(self, raw_len, spk_id, rng=random):
            return dict(self.d, spk_id=spk_id)

    base = dict(speed_rate=1.0, vol_gain_db=0.0, noise=None, snr_db=0.0)
    calls = []
    real_randint = random.randint
    random.randint = lambda a, b: calls.append((a, b)) or a
    try:
        for raw, rv, rate, want in [(46400, (0, 8000), 1.0, (0, 46400 + 7999 - n)),  # 2.9 s + 0.5 s response: cropped
                                    (46400, None, 1.0, None),                       # 2.9 s without: kept whole
                                    (40002, (5, 8000), 1.0, (0, 1)),                # one sample over 3 s: two starts
                                    (40001, (5, 8000), 1.0, None),                  # exactly 3 s: kept whole
                                    (44000, (0, 1), 0.9, None),                     # 1-tap response: no growth, int(44000 / 0.9) = 48888
                                    ]:
            calls.clear()
            d = dict(base, speed_rate=rate, reverb=rv)
            ds = types.SimpleNamespace(wave_augment=Fixed(d), mode="train", max_duration=3, _target_sample_rate=16000)
            _, crop, _ = PPVectorDataset._plan(ds, np.zeros(raw, np.float32), 0)
            full = augmented_len(raw, d)
            assert full == (raw if rate == 1.0 else int(raw / rate)) + (rv[1] - 1 if rv else 0)
            if want is None and full <= n:
                assert crop == (0, None) and calls == []
            elif want is None:
                assert crop == (0, n) and calls == [(0, full - n)]
            else:
                assert crop == (0, n) and calls == [want]
        ds = types.SimpleNamespace(wave_augment=Fixed(dict(base, reverb=(0, 8000))), mode="eval", max_duration=3, _target_sample_rate=16000)
        calls.clear()
        assert PPVectorDataset._plan(ds, np.zeros(46400, np.float32), 0)[1] == (0, n) and calls == []  # eval: from 0
    finally:
        random.randint = real_randint


def test_bank_resamples_skips_undecodable_and_sorts(tmp_path):
    rd = tmp_path / "rir"
    rd.mkdir()
    rng = np.random.default_rng(3)
    h44 = 0.5 * rng.standard_normal(4410) * np.exp(-np.arange(4410) / 500.0)
    write_wav(rd / "b_44k.wav", h44, sr=44100)
    write_wav(rd / "c_16k.wav", 0.3 * rng.standard_normal(1600))
    (rd / "a_broken.wav").write_bytes(b"not audio at all")
    (rd / "d_empty.wav").write_bytes(b"")
    aug = WaveAugmentor({"reverb": {"prob": 1.0, "reverb_dir": str(rd)}}, device="cpu")
    want44 = scipy.signal.resample_poly((np.clip(h44, -1, 1) * 32767).astype("<i2").astype(np.float32) / 32768.0, 160, 441)
    assert aug.rir_clips == [(0, want44.shape[0]), (want44.shape[0], 1600)]
    assert want44.shape[0] == 1600
    assert np.allclose(aug.rir_bank[:1600].numpy(), want44.astype(np.float32), atol=1e-7)


@pytest.mark.parametrize("where", ["missing", "empty", "prob0"])
def test_missing_or_empty_dir_disables_reverb(tmp_path, where):
    rd = tmp_path / "rir"
    if where != "missing":
        rd.mkdir()
    if where == "prob0":
        write_wav(rd / "r.wav", np.ones(100) * 0.1)
    conf = {"speed": {"prob": 1.0}, "volume": {"prob": 1.0, "min_gain_dBFS": -15, "max_gain_dBFS": 15},
            "reverb": {"prob": 0.0 if where == "prob0" else 1.0, "reverb_dir": str(rd)}}
    aug = WaveAugmentor(conf, device="cpu")
    assert aug.rir_bank is None and aug.rir_clips == []
    plain = WaveAugmentor({k: v for k, v in conf.items() if k != "reverb"}, device="cpu")
    r1, r2 = random.Random(11), random.Random(11)
    for _ in range(5):
        d = aug.draw(16000, 2, r1)
        assert "reverb" not in d and d == plain.draw(16000, 2, r2)
    assert r1.getstate() == r2.getstate()  # no random numbers drawn for the disabled augmentor
