"""GPU: the STFT front ends (Spectrogram / MelSpectrogram / LogMelSpectrogram / MFCC) on a ragged batch in one launch sequence
(AudioFeaturizer.forward_ragged -> ppv_spectral_forward_ragged_samples):
  * every row equals the same utterance featurised alone, bitwise, with zeros beyond its frames, and matches the fp64 oracle;
  * samples past an utterance's own length are never read (1e4 or NaN there changes nothing);
  * two launches whatever B: the frame kernel, then the CMN kernel;
  * PPVectorDataset.load_batch and PPVectorTrainer.train run on it with MelSpectrogram features;
  * the C entry refuses null pointers, an empty or oversized batch and too short a waveform."""
import os
import wave

import numpy as np
import pytest
import torch
import yaml
from launch_check import check_launches

from oracle import spectral as osp
from ppvector import _lib
from ppvector.data_utils.featurizer import AudioFeaturizer

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PPV_EINVAL = -1
MEL64 = dict(sr=16000, n_fft=1024, hop_length=160, n_mels=64)
CASES = {"Spectrogram-win400-power1": ("Spectrogram", dict(n_fft=512, hop_length=128, win_length=400, power=1.0)),
         "MelSpectrogram-64": ("MelSpectrogram", MEL64),
         "MelSpectrogram-htk-nonorm-power1": ("MelSpectrogram", dict(sr=16000, n_fft=256, hop_length=64, n_mels=40, htk=True, norm=None,
                                                                     power=1.0)),
         "LogMelSpectrogram-win400": ("LogMelSpectrogram", dict(sr=16000, n_fft=512, hop_length=160, win_length=400, n_mels=80, f_min=20.0)),
         "MFCC-13": ("MFCC", dict(sr=16000, n_fft=512, hop_length=160, n_mels=40, n_mfcc=13, f_min=0.0, f_max=7600.0))}
KERNELS = ["ppv::spectral_frame_kernel(float const*, int, int, int, ppv::SpecKernelArgs, int const*, int const*, float*)",
           "ppv::spectral_cmn_kernel(float*, float const*, int const*, int, int)"]


def waves(seed, lens):
    rng = np.random.default_rng(seed)
    return [(0.1 * rng.standard_normal(n) * (1 + 0.5 * np.sin(np.arange(n) / 700.0))).astype(np.float32) for n in lens]


def padded(ws, L, fill=0.0):
    batch = torch.full((len(ws), L), fill, dtype=torch.float32)
    for b, w in enumerate(ws):
        batch[b, :len(w)] = torch.from_numpy(w)
    return batch


def lengths(kw, center):
    """the padded maximum, the shortest utterance the front end frames, lengths that are not multiples of hop"""
    n_fft, hop = kw.get("n_fft", 2048), kw.get("hop_length", 512)
    shortest = n_fft // 2 + 1 if center else n_fft
    return [20000, shortest, 20000 - 37, n_fft + 3 * hop + 7, 12345]


def featurizer(case, center):
    method, kw = CASES[case]
    return method, dict(kw, center=center), AudioFeaturizer(method, dict(kw, center=center))


@pytest.mark.parametrize("center", [True, False], ids=["center", "no-center"])
@pytest.mark.parametrize("case", list(CASES))
def test_ragged_rows_equal_utterances_alone(cuda, case, center):
    method, kw, fz = featurizer(case, center)
    lens = lengths(kw, center)
    ws = waves(len(case), lens)
    for rows in (range(len(lens)), [4]):  # the mixed batch, and B = 1 with padding past its utterance
        sub = [ws[b] for b in rows]
        n = [lens[b] for b in rows]
        feats, frames = fz.forward_ragged(padded(sub, max(lens)).to(cuda), n)
        assert frames == [fz.num_frames(k) for k in n] and min(frames) >= 1
        assert feats.shape == (len(sub), max(frames), fz.feature_dim)
        for b, w in enumerate(sub):
            alone = fz(torch.from_numpy(w).to(cuda))[0]
            assert torch.equal(feats[b, :frames[b]], alone), (b, n[b])  # same kernels, same per-utterance arithmetic
            assert (feats[b, frames[b]:] == 0).all(), b
        if len(sub) == len(lens):
            got = feats.double().cpu()
    for b, w in enumerate(ws):
        want = osp.featurize(torch.from_numpy(w).double()[None], method, **kw)[0]
        tol = 2e-5 * want.abs().max() if method != "MFCC" else 2e-2  # test_gpu_spectral.py's tolerances
        assert want.shape[0] == fz.num_frames(lens[b])
        assert float((got[b, :want.shape[0]] - want).abs().max()) <= tol, (b, lens[b])


@pytest.mark.parametrize("center", [True, False], ids=["center", "no-center"])
@pytest.mark.parametrize("case", list(CASES))
def test_padding_samples_are_never_read(cuda, case, center):
    _, kw, fz = featurizer(case, center)
    lens = lengths(kw, center)
    ws = waves(7, lens)
    clean, frames = fz.forward_ragged(padded(ws, max(lens)).to(cuda), lens)
    for fill in (1e4, float("nan")):
        out, f2 = fz.forward_ragged(padded(ws, max(lens), fill).to(cuda), lens)
        assert f2 == frames and torch.isfinite(out).all(), fill
        assert torch.equal(out, clean), fill


@pytest.mark.parametrize("B", [3, 64])
def test_two_launches_whatever_the_batch(cuda, B):
    fz = AudioFeaturizer("MelSpectrogram", MEL64)
    lens = [int(n) for n in np.random.default_rng(B).integers(8000, 48001, size=B)]
    wav = padded(waves(B, lens), max(lens)).to(cuda)
    check_launches(lambda: fz.forward_ragged(wav, lens), KERNELS)


def write_wavs(tmp_path, lens, seed):
    paths = []
    for i, w in enumerate(waves(seed, lens)):
        p = tmp_path / f"u{i}.wav"
        with wave.open(str(p), "wb") as f:
            f.setnchannels(1)
            f.setsampwidth(2)
            f.setframerate(16000)
            f.writeframes((w * 32767).astype("<i2").tobytes())
        paths.append(str(p))
    return paths


def test_dataset_batch_path_equals_per_item_path(cuda, tmp_path):
    from ppvector.data_utils.collate_fn import collate_fn
    from ppvector.data_utils.reader import PPVectorDataset
    paths = write_wavs(tmp_path, [20000, 70000, 48000, 9000, 8001], seed=9)
    lst = tmp_path / "list.txt"
    lst.write_text("".join(f"{p}\t{i}\n" for i, p in enumerate(paths)))
    fz = AudioFeaturizer("MelSpectrogram", MEL64)
    ds = PPVectorDataset(str(lst), fz, mode="eval", device=cuda)  # eval: crop from 0, no augmentation -> deterministic
    f1, l1, n1 = ds.load_batch(range(5))
    f2, l2, n2 = collate_fn([ds[i] for i in range(5)])
    assert torch.equal(l1, l2) and torch.equal(n1, n2)
    assert torch.equal(f1, f2)
    assert f1.shape == (5, fz.num_frames(48000), 64)  # the 70000-sample utterance is cropped to max_duration 3 s


def test_trainer_runs_on_mel_spectrogram_features(cuda, tmp_path):
    from ppvector.trainer import PPVectorTrainer
    paths = write_wavs(tmp_path, [48000, 30011, 20000, 40000, 16000, 36000, 26000, 44000], seed=11)
    lst = tmp_path / "list.txt"
    lst.write_text("".join(f"{p}\t{i % 2}\n" for i, p in enumerate(paths)))
    cfg = yaml.load(open(os.path.join(ROOT, "configs", "ecapa_tdnn.yml")), Loader=yaml.FullLoader)
    for k in ("train_list", "enroll_list", "trials_list"):
        cfg["dataset_conf"][k] = str(lst)
    cfg["dataset_conf"]["sampler"]["batch_size"] = 4
    cfg["model_conf"]["classifier"]["num_speakers"] = 2
    cfg["preprocess_conf"] = {"feature_method": "MelSpectrogram", "method_args": dict(MEL64)}
    history = PPVectorTrainer(cfg, use_gpu=True).train(save_model_path=str(tmp_path / "models"), do_eval=False, max_steps=2)
    assert len(history) == 2 and all(np.isfinite(history))


def test_refusals(cuda):
    lib = _lib.load()
    fz = AudioFeaturizer("MelSpectrogram", MEL64)
    h = fz._get_handle()
    L, B = 4000, 2
    wav = torch.zeros(B, L, device=cuda)
    vf = torch.full((B,), fz.num_frames(L), dtype=torch.int32, device=cuda)
    ns = torch.full((B,), L, dtype=torch.int32, device=cuda)
    out = torch.empty(B, fz.num_frames(L), 64, device=cuda)

    def call(h=h, wav=wav, vf=vf, ns=ns, B=B, L=L, out=out):
        rc = lib.ppv_spectral_forward_ragged_samples(h, _lib.ptr(wav), _lib.ptr(vf), _lib.ptr(ns), B, L, _lib.ptr(out),
                                                     _lib.current_stream())
        return rc, _lib.last_error()

    assert call()[0] == 0
    for kwargs, msg in [(dict(h=None), "null argument"), (dict(wav=None), "null argument"), (dict(vf=None), "null argument"),
                        (dict(ns=None), "null argument"), (dict(out=None), "null argument"), (dict(B=0), "empty input"),
                        (dict(B=65536), "batch must be in [1, 65535]"), (dict(L=MEL64["n_fft"] // 2), "too short for one frame")]:
        rc, err = call(**kwargs)
        assert rc == PPV_EINVAL and msg in err, (kwargs, rc, err)
    torch.cuda.synchronize()
