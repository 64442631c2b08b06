"""GPU: reverberation in the batched audio preparation (csrc/reverb.cu through ppv_audio_prep_reverb) against the fp64 oracle
(tests/reverb_oracle.py, recalled yeaudio semantics), a shifted delta response, bit-identity with ppv_audio_prep where no item drew a
response, run-to-run determinism, the batched dataset path against the per-item path, and the shipped augmentation config."""
import random
import wave

import numpy as np
import pytest
import torch

from oracle import audio_prep as oap
from ppvector.data_utils.audio_batch import prepare_batch
from reverb_oracle import prepare_reverb

pytestmark = pytest.mark.gpu

RIR_LENS = [1, 37, 256, 257, 8000, 70000]


def waves(seed, lens):
    rng = np.random.default_rng(seed)
    return [(0.1 * rng.standard_normal(n) * (1 + 0.5 * np.sin(np.arange(n) / 700.0))).astype(np.float32) for n in lens]


def rir_bank(seed=4):
    rng = np.random.default_rng(seed)
    clips = [(rng.standard_normal(n) * np.exp(-np.arange(n) / max(1.0, n / 6.0))).astype(np.float32) for n in RIR_LENS]
    offs = np.cumsum([0] + RIR_LENS[:-1])
    return np.concatenate(clips), [(int(o), n) for o, n in zip(offs, RIR_LENS)]


def mixed_batch():
    """Speed 0.9 / 1.1, noise, every response length (the 70000-tap one longer than its utterance), a 200-sample utterance, one item
    without reverb; crops inside, across and beyond the reverberant length."""
    ws = waves(1, [48000, 30011, 20000, 200, 52345, 40000, 16000])
    noise = (0.05 * np.random.default_rng(2).standard_normal(20000)).astype(np.float32)
    bank, clips = rir_bank()
    base = dict(speed_rate=1.0, vol_gain_db=0.0, noise=None, snr_db=0.0)
    draws = [dict(base, reverb=clips[0]),
             dict(base, speed_rate=0.9, vol_gain_db=-7.5, noise=(1234, 20000 - 1234), snr_db=15.0, reverb=clips[1]),
             dict(base, speed_rate=1.1, vol_gain_db=4.0, reverb=clips[2]),
             dict(base, reverb=clips[3]),
             dict(base, noise=(0, 20000), snr_db=30.0, reverb=clips[4]),
             dict(base, speed_rate=0.9, reverb=clips[5]),
             dict(base, noise=(500, 19500), snr_db=20.0, reverb=None)]
    crops = [(0, None), (100, 30000), (5000, 48000), (0, None), (4345, 48000), (70000, 48000), (0, None)]
    return ws, noise, bank, draws, crops


def oracle_rows(ws, noise, bank, draws, crops, Lout, normalize):
    rows = []
    for w, d, (cs, cl) in zip(ws, draws, crops):
        nz = None if d["noise"] is None else noise[d["noise"][0]:d["noise"][0] + d["noise"][1]]
        rir = None if d["reverb"] is None else bank[d["reverb"][0]:d["reverb"][0] + d["reverb"][1]]
        rows.append(prepare_reverb(w, d["speed_rate"], d["vol_gain_db"], nz, 0, d["snr_db"], rir, -20.0, normalize, cs, cl, out_len=Lout))
    return np.stack(rows)


@pytest.mark.parametrize("normalize", [True, False])
def test_reverb_matches_oracle(cuda, normalize):
    ws, noise, bank, draws, crops = mixed_batch()
    out, lens = prepare_batch(ws, draws, crops, normalize=normalize, noise_bank=torch.from_numpy(noise).to(cuda), device=cuda,
                              rir_bank=torch.from_numpy(bank).to(cuda))
    got = out.cpu().numpy()
    want = oracle_rows(ws, noise, bank, draws, crops, out.shape[1], normalize)
    for b in range(len(ws)):
        full = len(oap.change_speed(ws[b], draws[b]["speed_rate"])) + (draws[b]["reverb"][1] - 1 if draws[b]["reverb"] else 0)
        cs, cl = crops[b]
        assert lens[b] == (min(cl, full - cs) if cl is not None else full - cs), b
        assert np.all(got[b, lens[b]:] == 0), b
        err = float(np.abs(got[b] - want[b]).max())
        # -20 dB rows have an RMS of 0.1: 1e-5 is 1e-4 of it.  Un-normalised rows are held to the same bound relative to their RMS.
        scale = 1.0 if normalize else max(1.0, 10.0 * float(np.sqrt(np.mean(want[b][:lens[b]].astype(np.float64) ** 2))))
        assert err <= 1e-5 * scale, (b, err, scale)
    if normalize:  # the un-cropped rows meet the -20 dB target over the whole reverberant utterance
        for b in (0, 3):
            assert abs(oap.rms_db(got[b][:lens[b]]) + 20.0) < 1e-3


@pytest.mark.parametrize("normalize", [False, True])
def test_shifted_delta(cuda, normalize):
    """h = [0]*d + [1]: the no-reverb output shifted by d with d more samples.  dB normalisation averages over the d extra (silent) samples
    too, so with it on the shifted rows are scaled by sqrt((n + d) / n)."""
    ws = waves(6, [30011, 150])
    for d in (1, 255, 256, 300, 1000):
        h = np.zeros(d + 1, np.float32)
        h[d] = 1.0
        bank = torch.from_numpy(h).to(cuda)
        draws = [dict(speed_rate=0.9, vol_gain_db=3.0, noise=None, snr_db=0.0, reverb=(0, d + 1)),
                 dict(speed_rate=1.0, vol_gain_db=0.0, noise=None, snr_db=0.0, reverb=(0, d + 1))]
        plain, plens = prepare_batch(ws, [dict(x, reverb=None) for x in draws], [(0, None)] * 2, normalize=normalize, device=cuda)
        rev, rlens = prepare_batch(ws, draws, [(0, None)] * 2, normalize=normalize, device=cuda, rir_bank=bank)
        for b in range(2):
            n = plens[b]
            assert rlens[b] == n + d
            r, p = rev[b, :rlens[b]].cpu().numpy(), plain[b, :n].cpu().numpy().astype(np.float64)
            if normalize:
                p = p * np.sqrt((n + d) / n)
            assert np.abs(r[:d]).max() <= 1e-6 and np.abs(r[d:] - p).max() <= 1e-6, (d, b, np.abs(r[d:] - p).max())


def test_no_item_drew_reverb_is_bit_identical(cuda):
    ws, noise, bank, draws, crops = mixed_batch()
    nb, rb = torch.from_numpy(noise).to(cuda), torch.from_numpy(bank).to(cuda)
    none = [dict(d, reverb=None) for d in draws]
    crops = [(0, None), (100, 30000), (5000, 15000), (0, None), (4345, 48000), (7000, 20000), (0, None)]
    a, la = prepare_batch(ws, none, crops, noise_bank=nb, device=cuda, rir_bank=rb)
    b, lb = prepare_batch(ws, [{k: v for k, v in d.items() if k != "reverb"} for d in draws], crops, noise_bank=nb, device=cuda)
    assert la == lb and torch.equal(a, b)
    # in a mixed batch, the item without reverb still comes out exactly as from ppv_audio_prep
    ws, noise, bank, draws, crops = mixed_batch()
    mixed, lm = prepare_batch(ws, draws, crops, noise_bank=nb, device=cuda, rir_bank=rb)
    alone, la = prepare_batch(ws[6:], draws[6:], crops[6:], noise_bank=nb, device=cuda)
    assert torch.equal(mixed[6, :la[0]], alone[0]) and (mixed[6, la[0]:] == 0).all()


def test_deterministic(cuda):
    ws, noise, bank, draws, crops = mixed_batch()
    nb, rb = torch.from_numpy(noise).to(cuda), torch.from_numpy(bank).to(cuda)
    a, _ = prepare_batch(ws, draws, crops, noise_bank=nb, device=cuda, rir_bank=rb)
    b, _ = prepare_batch(ws, draws, crops, noise_bank=nb, device=cuda, rir_bank=rb)
    assert torch.equal(a, b)


def write_wav(path, x, sr=16000):
    with wave.open(str(path), "wb") as f:
        f.setnchannels(1)
        f.setsampwidth(2)
        f.setframerate(sr)
        f.writeframes((np.clip(x, -1, 1) * 32767).astype("<i2").tobytes())


def make_list(tmp_path, lens):
    lines = []
    for i, w in enumerate(waves(9, lens)):
        p = tmp_path / f"u{i}.wav"
        write_wav(p, w)
        lines.append(f"{p}\t{i}\n")
    lst = tmp_path / "list.txt"
    lst.write_text("".join(lines))
    return lst


def make_rir_dir(tmp_path, lens=(8000, 300, 16000)):
    rd = tmp_path / "reverb"
    rd.mkdir()
    rng = np.random.default_rng(12)
    for i, n in enumerate(lens):
        write_wav(rd / f"r{i}.wav", 0.8 * rng.standard_normal(n) * np.exp(-np.arange(n) / (n / 5.0)))
    return rd


def test_dataset_batch_path_equals_per_item_path_with_reverb(cuda, tmp_path):
    from ppvector.data_utils.collate_fn import collate_fn
    from ppvector.data_utils.featurizer import AudioFeaturizer
    from ppvector.data_utils.reader import PPVectorDataset
    lst = make_list(tmp_path, [20000, 70000, 48000, 9000, 40000])
    conf = {"speed": {"prob": 0.5}, "volume": {"prob": 0.5, "min_gain_dBFS": -15, "max_gain_dBFS": 15},
            "reverb": {"prob": 0.7, "reverb_dir": str(make_rir_dir(tmp_path))}}
    fz = AudioFeaturizer("Fbank", {"sr": 16000, "n_mels": 80})
    ds = PPVectorDataset(str(lst), fz, mode="train", aug_conf=conf, device=cuda)
    assert ds.wave_augment.rir_bank is not None and len(ds.wave_augment.rir_clips) == 3
    random.seed(5)
    f1, l1, n1 = ds.load_batch(range(5))
    random.seed(5)
    f2, l2, n2 = collate_fn([ds[i] for i in range(5)])
    assert torch.equal(l1, l2) and torch.equal(n1, n2)
    assert torch.allclose(f1, f2, atol=2e-5), (f1 - f2).abs().max()
    random.seed(5)
    plans = [ds._plan(ds.decode(i)[0], 0) for i in range(5)]
    assert any(p[0]["reverb"] is not None for p in plans) and any(p[0]["reverb"] is None for p in plans)


def test_shipped_augmentation_config_trains(cuda, tmp_path):
    import os

    import yaml

    from ppvector.data_utils.featurizer import AudioFeaturizer
    from ppvector.data_utils.reader import PPVectorDataset
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    conf = yaml.safe_load(open(os.path.join(root, "configs", "augmentation.yml")))
    assert conf["reverb"]["prob"] == 0.5
    conf["reverb"]["reverb_dir"] = str(make_rir_dir(tmp_path))
    nd = tmp_path / "noise"
    nd.mkdir()
    write_wav(nd / "n.wav", 0.05 * np.random.default_rng(1).standard_normal(32000))
    conf["noise"]["noise_dir"] = str(nd)
    lst = make_list(tmp_path, [20000, 70000, 48000, 9000, 40000, 52000, 33000, 47000])
    fz = AudioFeaturizer("Fbank", {"sr": 16000, "n_mels": 80})
    ds = PPVectorDataset(str(lst), fz, mode="train", aug_conf=conf, device=cuda)
    random.seed(0)
    feats, labels, frames = ds.load_batch(range(8))
    assert feats.shape[0] == 8 and feats.shape[2] == 80 and int(frames.max()) <= 298
    assert torch.isfinite(feats).all()
