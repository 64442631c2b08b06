"""GPU: the energy voice-activity detection kernels (csrc/vad.cu, ppv_vad_energy) against the fp64 oracle (tests/vad_oracle.py) on
seeded recordings, ragged batches against one call per recording, the run buffer's worst case, every PPV_EINVAL path, and the
diarization path with vad=True end to end."""
import ctypes as C

import numpy as np
import pytest
import torch

import vad_oracle as vo

pytestmark = pytest.mark.gpu


def bursts(seed, sr=16000, seconds=6.0, snr_db=20.0):
    """Tonal and noise bursts separated by pauses of background noise snr_db below the bursts."""
    rng = np.random.default_rng(seed)
    x = 0.2 * 10 ** (-snr_db / 20) * rng.standard_normal(int(sr * seconds))
    t = 0
    while t < x.size:
        n = int(sr * rng.uniform(0.2, 0.8))
        if rng.random() < 0.6:
            k = np.arange(min(n, x.size - t))
            x[t:t + k.size] += (0.3 * np.sin(2 * np.pi * rng.uniform(100, 900) * k / sr) if rng.random() < 0.5
                                else 0.2 * rng.standard_normal(k.size))
        t += n
    return x.astype(np.float32)


def check_against_oracle(x, sr, got_e, got_v, got_runs=None, got_segments=None):
    r = vo.vad(x, sr)
    # exact equality of the decisions is a fair demand only where no frame sits within 1e-9 of the threshold
    assert len(r['e']) == 0 or np.abs(r['e'] - r['thr']).min() > 1e-9
    assert got_e.shape == r['e'].shape
    assert np.all(np.abs(got_e - r['e']) <= 1e-9 * np.abs(r['e']))
    assert np.array_equal(got_v, r['voiced'])
    if got_runs is not None:
        assert got_runs == r['runs']
    if got_segments is not None:
        assert got_segments == r['segments']
    return r


@pytest.mark.parametrize("sr", [8000, 16000])
@pytest.mark.parametrize("snr_db", [20.0, 40.0, 50.0, 60.0])
@pytest.mark.parametrize("seed", [0, 1])
def test_matches_the_oracle(cuda, seed, snr_db, sr):
    from ppvector.infer_utils import vad
    x = bursts(seed, sr, 8.0, snr_db)
    (e, v), = vad.energy_vad([x], sr, frames=True)
    r = check_against_oracle(x, sr, e, v, vad.voiced_runs([x], sr)[0], vad.energy_vad([x], sr)[0])
    # the threshold sits 5.5 nepers above half the mean log energy: pauses 20 dB down are still "voiced", 40 dB down they are not
    assert r['voiced'].any() and (snr_db < 40 or (len(r['runs']) >= 2 and not r['voiced'].all()))


def test_reference_wavs_match_the_oracle(cuda, golden_dir):
    from ppvector.infer_utils import vad
    g = np.load(f"{golden_dir}/fbank_wavs.npz")
    xs = [g[f"{n}_pcm"].astype(np.float32) / 32768.0 for n in ("a_1", "a_2", "b_1", "b_2", "long3s")]
    for x, (e, v), runs in zip(xs, vad.energy_vad(xs, 16000, frames=True), vad.voiced_runs(xs, 16000)):
        check_against_oracle(x, 16000, e, v, runs)


def test_ragged_batches_equal_separate_calls(cuda):
    from ppvector.infer_utils import vad
    rng = np.random.default_rng(3)
    edge = [0, 1, 399, 400, 401, 559, 560, 561, 160 * 64 + 400, 160 * 64 + 399]
    lengths = edge + np.exp(rng.uniform(np.log(160), np.log(16000 * 60), 290)).astype(int).tolist()
    xs = [bursts(100 + i, 16000, n / 16000 + 1e-3)[:n] for i, n in enumerate(lengths)]
    for R in (1, 2, 7, 64, 300):
        batch = xs[:R]
        frames = vad.energy_vad(batch, 16000, frames=True)
        runs = vad.voiced_runs(batch, 16000)
        segs = vad.energy_vad(batch, 16000)
        for i, x in enumerate(batch):
            (e1, v1), = vad.energy_vad([x], 16000, frames=True)
            assert np.array_equal(frames[i][0], e1) and np.array_equal(frames[i][1], v1), (R, i)
            assert runs[i] == vad.voiced_runs([x], 16000)[0] and segs[i] == vad.energy_vad([x], 16000)[0], (R, i)
    again = vad.energy_vad(xs, 16000, frames=True)
    assert all(np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1]) for a, b in zip(again, frames))


def test_one_hour_recording(cuda):
    from ppvector.infer_utils import vad
    sr = 16000
    x = np.concatenate([bursts(1000 + i, sr, 60.0, 10.0 + i % 30) for i in range(60)])
    assert x.size == 57_600_000
    (e, v), = vad.energy_vad([x], sr, frames=True)
    assert e.size == 359_998
    runs = vad.voiced_runs([x], sr)[0]
    check_against_oracle(x, sr, e, v, runs, vad.energy_vad([x], sr)[0])
    short = bursts(7, sr, 3.0)
    both = vad.energy_vad([short, x, short], sr, frames=True)
    assert np.array_equal(both[1][0], e) and np.array_equal(both[1][1], v)
    (e2, v2), = vad.energy_vad([x], sr, frames=True)
    assert np.array_equal(e2, e) and np.array_equal(v2, v)


# ---- the C ABI directly ------------------------------------------------------------------------------------------------------------------
def abi_call(xs, cfg=None, run_cap=None, ws_bytes=None, offsets=None, R=None, null=(), ws_offset=0, wav_offset=0, lib=None):
    """-> (status, n_runs, runs [n, 3]) of one ppv_vad_energy call; null names the pointer arguments to pass as NULL."""
    from ppvector import _lib
    lib = lib or _lib.load()
    if cfg is None:
        cfg = _lib.VadCfg()
        lib.ppv_vad_default_cfg(C.byref(cfg), 16000)
    lengths = [len(x) for x in xs]
    off = np.concatenate([[0], np.cumsum(lengths)]).astype(np.int64) if offsets is None else np.asarray(offsets, dtype=np.int64)
    T = [max(lib.ppv_vad_num_frames(C.byref(cfg), int(n)), 0) for n in lengths]
    n_total = sum(lengths)
    wav = torch.zeros(max(int(off[-1]), n_total) + 8, dtype=torch.float32, device='cuda')
    if n_total:
        wav[:n_total] = torch.from_numpy(np.concatenate(xs).astype(np.float32))
    voiced = torch.zeros(max(sum(T), 1), dtype=torch.uint8, device='cuda')
    cap = sum((t + 1) // 2 for t in T) if run_cap is None else run_cap
    runs = torch.full((max(cap, 1), 3), -1, dtype=torch.int32, device='cuda')
    n_runs = torch.full((1,), -1, dtype=torch.int32, device='cuda')
    need = lib.ppv_vad_workspace_bytes(C.byref(cfg), len(xs), int(off[-1]))
    nb = need if ws_bytes is None else ws_bytes
    ws = torch.empty(max(need, 1) + 512, dtype=torch.uint8, device='cuda')
    ptr = {'cfg': C.byref(cfg), 'wav': C.c_void_p(wav.data_ptr() + wav_offset), 'offsets': off.ctypes.data_as(C.POINTER(C.c_int64)),
           'voiced': C.c_void_p(voiced.data_ptr()), 'runs': C.c_void_p(runs.data_ptr()), 'n_runs': C.c_void_p(n_runs.data_ptr()),
           'ws': C.c_void_p(ws.data_ptr() + ws_offset)}
    for k in null:
        ptr[k] = None
    rc = lib.ppv_vad_energy(ptr['cfg'], ptr['wav'], ptr['offsets'], len(xs) if R is None else R, None, ptr['voiced'], ptr['runs'], cap,
                            ptr['n_runs'], ptr['ws'], nb, _lib.current_stream())
    torch.cuda.synchronize()
    n = int(n_runs.item())
    return rc, n, runs[:max(n, 0)].cpu().numpy()


def test_alternating_frames_fill_the_run_buffer(cuda):
    """window = shift = 160, no context, a fixed threshold: frames alternate loud / silent, so every other frame is a run of one and the
    run buffer of sum ceil(T / 2) entries is exactly full."""
    from ppvector import _lib
    lib = _lib.load()
    cfg = _lib.VadCfg()
    lib.ppv_vad_default_cfg(C.byref(cfg), 16000)
    cfg.window, cfg.shift, cfg.frames_context, cfg.energy_mean_scale, cfg.energy_threshold = 160, 160, 0, 0.0, 10.0
    rng = np.random.default_rng(9)
    xs = []
    for T in (1, 2, 7, 1000, 64 * 3 + 1):
        blocks = [(0.3 if t % 2 == 0 else 0.0) * rng.standard_normal(160) for t in range(T)]
        xs.append(np.concatenate(blocks).astype(np.float32))
    rc, n, runs = abi_call(xs, cfg)
    assert rc == 0
    cap = sum((len(x) // 160 + 1) // 2 for x in xs)
    assert n == cap
    expect = [(r, 2 * k, 2 * k + 1) for r, x in enumerate(xs) for k in range((len(x) // 160 + 1) // 2)]
    assert [tuple(row) for row in runs.tolist()] == expect
    assert abi_call(xs, cfg, run_cap=cap - 1)[0] == -1  # PPV_EINVAL


def test_einval_paths(cuda):
    from ppvector import _lib
    lib = _lib.load()
    EINVAL = -1
    xs = [bursts(5, 16000, 1.0), bursts(6, 16000, 0.5)]
    assert abi_call(xs)[0] == 0
    for k in ('cfg', 'wav', 'offsets', 'voiced', 'runs', 'n_runs', 'ws'):
        assert abi_call(xs, null=(k,))[0] == EINVAL, k
    assert abi_call(xs, R=0)[0] == EINVAL
    assert abi_call(xs, offsets=[0, 16000, 15000])[0] == EINVAL  # decreasing
    assert abi_call(xs, offsets=[-1, 16000, 24000])[0] == EINVAL
    assert abi_call(xs, ws_bytes=lib.ppv_vad_workspace_bytes(C.byref(_cfg(lib)), 2, 24000) - 1)[0] == EINVAL
    assert abi_call(xs, ws_offset=16)[0] == EINVAL  # workspace not 256-byte aligned
    assert abi_call(xs, wav_offset=2)[0] == EINVAL  # samples not 4-byte aligned
    assert abi_call(xs, run_cap=0)[0] == EINVAL
    for field, value in (('window', 0), ('window', 2049), ('shift', 0), ('shift', 401), ('frames_context', -1),
                         ('energy_mean_scale', -0.5), ('proportion_threshold', 0.0), ('proportion_threshold', 1.0),
                         ('energy_threshold', float('nan'))):
        cfg = _cfg(lib)
        setattr(cfg, field, value)
        assert abi_call(xs, cfg)[0] == EINVAL, field
        assert lib.ppv_vad_num_frames(C.byref(cfg), 16000) == -1 and lib.ppv_vad_workspace_bytes(C.byref(cfg), 2, 24000) == 0, field
    assert "energy_threshold must be finite" in _lib.last_error()
    # unaligned samples that are still floats, and recordings without frames, are not errors
    rc, n, _ = abi_call([np.zeros(0, np.float32), bursts(8, 16000, 2.0), np.zeros(100, np.float32)], wav_offset=4)
    assert rc == 0 and n >= 0
    rc, n, _ = abi_call([np.zeros(399, np.float32)], run_cap=0)
    assert rc == 0 and n == 0


def _cfg(lib):
    from ppvector import _lib
    cfg = _lib.VadCfg()
    lib.ppv_vad_default_cfg(C.byref(cfg), 16000)
    return cfg


# ---- diarization end to end ------------------------------------------------------------------------------------------------------------
def speakers_with_pauses(sr=16000):
    rng = np.random.default_rng(7)
    parts = []
    for f, speech, pause in ((180, 4.0, 0.8), (420, 4.0, 1.1), (180, 4.0, 0.6), (420, 3.0, 0.0)):
        t = np.arange(int(sr * speech)) / sr
        parts.append(0.3 * np.sin(2 * np.pi * f * t) * (1 + 0.1 * rng.normal(size=t.size)))
        parts.append(1e-3 * rng.normal(size=int(sr * pause)))
    return np.concatenate(parts).astype(np.float32)


def test_speaker_diarization_with_vad(cuda):
    import os

    import yaml

    from oracle import ecapa as oe
    from ppvector.data_utils.audio import AudioSegment
    from ppvector.infer_utils.speaker_diarization import SpeakerDiarization
    from ppvector.predict import PPVectorPredictor
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    cfg = yaml.load(open(os.path.join(root, 'configs', 'ecapa_tdnn.yml')), Loader=yaml.FullLoader)
    pred = PPVectorPredictor(cfg, state_dict={k: v.float().numpy() for k, v in oe.make_ecapa_weights(seed=1000, dtype=torch.float64).items()})
    sr = 16000
    wav = speakers_with_pauses(sr)
    loaded = pred._load_audio(wav.copy(), sr).samples
    r = vo.vad(loaded, sr)
    assert np.abs(r['e'] - r['thr']).min() > 1e-9
    spans = [(s['start'] / sr, s['end'] / sr) for s in r['segments']]
    assert len(spans) >= 3
    np.random.seed(3)
    out = pred.speaker_diarization(wav.copy(), sample_rate=sr, vad=True)
    np.random.seed(3)
    ref = pred.speaker_diarization(wav.copy(), sample_rate=sr, vad_segments=spans)
    assert out == ref and len(out) >= 1
    t1, e1 = pred.diarization_embeddings(wav.copy(), sample_rate=sr, vad=True)
    t2, e2 = pred.diarization_embeddings(wav.copy(), sample_rate=sr, vad_segments=spans)
    assert np.array_equal(t1, t2) and np.array_equal(e1, e2)
    sd = SpeakerDiarization()
    chunks = sd.segments_audio(AudioSegment(wav, sr))
    x = wav
    r = vo.vad(x, sr)
    assert np.abs(r['e'] - r['thr']).min() > 1e-9
    vad_segments = []
    for s in r['segments']:
        st, ed = round(s['start'] / sr, 3), round(s['end'] / sr, 3)
        vad_segments.append([st, ed, x[int(st * sr):int(ed * sr)]])
    expect = sd._chunk(vad_segments)
    assert len(chunks) == len(expect) > 0
    for c, e in zip(chunks, expect):
        assert c[0] == e[0] and c[1] == e[1] and np.array_equal(c[2], e[2])
