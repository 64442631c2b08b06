"""GPU: AS-norm (csrc/score_norm.cu, ppvector/metric/score_norm.py) against the fp64 oracle (tests/score_norm_oracle.py) -- the exact
top-N selection of ppv_topn_row_stats on both sides of its shared-memory cut with ties, constant rows, exact 1.0 and 1-ulp neighbours at
the cut; cohort_stats from embeddings in both cohort modes with several chunks; as_norm and the EER of its output; and
PPVectorTrainer.evaluate with and without the score_norm key."""
import copy
import ctypes as C
import os
import wave

import numpy as np
import pytest
import torch
import yaml

import score_norm_oracle as so
from ppvector import _lib
from ppvector.metric.cosine import cosine_matrix
from ppvector.metric.metrics import compute_dcf, compute_eer, compute_fnr_fpr, eer_mindcf_from_matrix_gpu
from ppvector.metric.score_norm import as_norm, cohort_stats, speaker_cohort, topn_row_stats

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SMEM_COLS = 10240  # rows up to this width are staged in shared memory (TN_SMEM_COLS in csrc/score_norm.cu)
PAD = 3            # ld = cols + PAD: rows start unaligned


def special_rows(rng, rows, cols, top_n):
    """Cosine-like rows; row r % 4 == 0: a run of equal values straddling the cut, 1: constant, 2: exact 1.0 (several), 3: 1-ulp
    neighbours around the cut."""
    x = (rng.uniform(-1, 1, size=(rows, cols)) * rng.uniform(0.05, 1, size=(rows, 1))).astype(np.float32)
    lo, hi = max(0, top_n - 3), min(cols, top_n + 3)
    for r in range(rows):
        kind = r % 4
        order = np.argpartition(-x[r], hi - 1)[:hi]  # the hi largest, then in descending order
        order = order[np.argsort(-x[r, order], kind='stable')]
        if kind == 0:
            x[r, order[lo:hi]] = x[r, order[top_n - 1]]
        elif kind == 1:
            x[r] = np.float32(0.37)
        elif kind == 2:
            x[r, order[:min(cols, 3)]] = 1.0
        else:
            v = x[r, order[top_n - 1]]
            for j, c in enumerate(order[lo:hi]):
                x[r, c] = np.nextafter(v, np.float32(np.inf if j % 2 else -np.inf), dtype=np.float32) if j % 3 else v
    return x


def run_stats(dev_rows):
    return [t.cpu().numpy() for t in topn_row_stats(dev_rows[0], dev_rows[1])]


CASES = [(2, 1), (2, 63), (2, 64), (2, 65), (2, 4097), (300, 1), (300, 65), (300, 4097), (301, 64), (301, 4097),
         (SMEM_COLS, 1), (SMEM_COLS, 63), (SMEM_COLS, 4097), (SMEM_COLS + 1, 1), (SMEM_COLS + 1, 65), (SMEM_COLS + 1, 4097),
         (10**5, 1), (10**5, 64), (10**5, 65), (10**6, 1), (10**6, 65)]


@pytest.mark.parametrize("cols,rows", CASES)
def test_topn_row_stats_exact(cuda, cols, rows):
    rng = np.random.default_rng(cols * 7 + rows)
    for top_n in sorted({2, min(300, cols), cols}):
        x = special_rows(rng, rows, cols, top_n)
        buf = torch.zeros((rows, cols + PAD), dtype=torch.float32, device=cuda)
        buf[:, cols:] = 2.0  # padding that would be the row maximum if it were read
        buf[:, :cols] = torch.from_numpy(x).to(cuda)
        view = buf[:, :cols]
        mean, std = run_stats((view, top_n))
        ref_mean, ref_std = so.topn_stats(x, top_n)
        assert np.abs(mean - ref_mean).max() <= 1e-6, (top_n, np.abs(mean - ref_mean).max())
        assert np.abs(std - ref_std).max() <= 1e-6, (top_n, np.abs(std - ref_std).max())
        if rows > 1:
            assert std[1] == np.float32(1e-6) and mean[1] == np.float32(0.37)
        again = run_stats((view, top_n))
        assert mean.tobytes() == again[0].tobytes() and std.tobytes() == again[1].tobytes()
        cut = sorted({0, 1, rows // 3, rows})
        parts = [run_stats((view[a:b], top_n)) for a, b in zip(cut, cut[1:]) if b > a]
        assert np.concatenate([p[0] for p in parts]).tobytes() == mean.tobytes()
        assert np.concatenate([p[1] for p in parts]).tobytes() == std.tobytes()
        del buf, view


def embeddings(rng, n, D, n_spk):
    centres = rng.normal(size=(n_spk, D))
    labels = rng.integers(0, n_spk, size=n)
    return (centres[labels] + 1.5 * rng.normal(size=(n, D))).astype(np.float32), labels


@pytest.mark.parametrize("D", [80, 192, 256])
@pytest.mark.parametrize("mode", ["speaker", "utterance"])
def test_cohort_stats_from_embeddings(cuda, D, mode):
    rng = np.random.default_rng(D)
    cohort_emb, cohort_lab = embeddings(rng, 3000, D, 500)
    q, _ = embeddings(rng, 301, D, 500)
    if mode == "speaker":
        cohort = speaker_cohort(torch.from_numpy(cohort_emb).to(cuda), cohort_lab)
        ref_cohort = so.speaker_cohort(cohort_emb, cohort_lab)
        assert cohort.cpu().numpy().tobytes() == ref_cohort.tobytes()
    else:
        cohort, ref_cohort = torch.from_numpy(cohort_emb).to(cuda), cohort_emb
    Nc = ref_cohort.shape[0]
    for top_n in (2, 300):
        mean, std = cohort_stats(torch.from_numpy(q).to(cuda), cohort, top_n, max_ws_bytes=4 * Nc * 70)  # 5 chunks
        ref_mean, ref_std = so.cohort_stats(q, ref_cohort, top_n)
        assert np.abs(mean.cpu().numpy() - ref_mean).max() <= 2e-6
        assert np.abs(std.cpu().numpy() - ref_std).max() <= 2e-6
        whole = cohort_stats(torch.from_numpy(q).to(cuda), cohort, top_n)
        assert whole[0].cpu().numpy().tobytes() == mean.cpu().numpy().tobytes()


def test_as_norm_and_eer(cuda):
    rng = np.random.default_rng(5)
    M, N = 257, 131
    s = rng.uniform(-0.3, 0.9, size=(M, N)).astype(np.float32)
    t_stats = (rng.uniform(0, 0.5, M).astype(np.float32), rng.uniform(0.02, 0.2, M).astype(np.float32))
    e_stats = (rng.uniform(0, 0.5, N).astype(np.float32), rng.uniform(0.02, 0.2, N).astype(np.float32))
    t_stats[1][3] = 0.0  # floored at 1e-6
    got = as_norm(torch.from_numpy(s).to(cuda), t_stats, e_stats)
    ref = so.as_norm(s, t_stats, e_stats)
    g = got.cpu().numpy()
    assert np.all(np.abs(g - ref) <= 1e-6 * np.maximum(1.0, np.abs(ref)))
    tl, el = rng.integers(0, 20, M).astype(np.int32), rng.integers(0, 20, N).astype(np.int32)
    eer, dcf, thr = eer_mindcf_from_matrix_gpu(got, tl, el)
    flat = g.reshape(-1)
    lab = (tl[:, None] == el[None, :]).astype(np.int32).reshape(-1)
    fnr, fpr, _ = compute_fnr_fpr(flat, lab)
    eer_ref, thr_ref = compute_eer(fnr, fpr, flat)
    assert abs(eer - float(eer_ref)) < 1e-9 and abs(dcf - compute_dcf(fnr, fpr)) < 1e-9 and thr == pytest.approx(float(thr_ref), abs=1e-6)


def test_errors(cuda):
    lib = _lib.load()
    x = torch.zeros((4, 10), device=cuda)
    m = torch.empty(4, device=cuda)
    st = _lib.current_stream()
    p = C.c_void_p(x.data_ptr())
    for rows, cols, ld, top_n, ptr in ((4, 10, 10, 1, p), (4, 10, 10, 11, p), (4, 10, 9, 2, p), (4, 10, 10, 2, None), (0, 10, 10, 2, p)):
        assert lib.ppv_topn_row_stats(ptr, rows, cols, ld, top_n, _lib.ptr(m), _lib.ptr(m), st) == -1
        assert _lib.last_error()
    assert lib.ppv_as_norm_apply(p, 4, 10, None, _lib.ptr(m), _lib.ptr(m), _lib.ptr(m), st) == -1
    rng = np.random.default_rng(0)
    q, c = torch.from_numpy(rng.normal(size=(5, 192)).astype(np.float32)).to(cuda), torch.from_numpy(rng.normal(size=(20, 192)).astype(np.float32)).to(cuda)
    with pytest.raises(_lib.PPVError):
        cohort_stats(q, c, top_n=21)
    with pytest.raises(_lib.PPVError):
        cohort_stats(q, c[:, :80], top_n=2)
    with pytest.raises(_lib.PPVError):
        as_norm(torch.zeros((5, 20), device=cuda), (m, m), (m, m))


NAMES = ["a_1", "a_2", "b_1", "b_2", "long3s"]
SPK = {"a_1": 0, "a_2": 0, "b_1": 1, "b_2": 1, "long3s": 2}


@pytest.fixture(scope="module")
def lists(tmp_path_factory, golden_dir):
    d = tmp_path_factory.mktemp("asnorm")
    g = np.load(f"{golden_dir}/fbank_wavs.npz")
    paths = {}
    for n in NAMES:
        p = str(d / f"{n}.wav")
        with wave.open(p, "wb") as w:
            w.setnchannels(1)
            w.setsampwidth(2)
            w.setframerate(16000)
            w.writeframes(g[n + "_pcm"].astype("<i2").tobytes())
        paths[n] = p
    out = {}
    for name, members in {"enroll": ["a_1", "b_1", "long3s"], "trials": ["a_2", "b_2", "long3s"], "cohort": NAMES + ["a_1", "b_2"]}.items():
        out[name] = str(d / f"{name}_list.txt")
        with open(out[name], "w") as f:
            for n in members:
                f.write(f"{paths[n]}\t{SPK[n]}\n")
    return out


@pytest.mark.parametrize("mode,top_n", [("speaker", 3), ("utterance", 4)])
def test_evaluate_end_to_end(cuda, lists, mode, top_n):
    from oracle import ecapa as oe
    from ppvector.trainer import PPVectorTrainer
    cfg = yaml.load(open(os.path.join(ROOT, "configs", "ecapa_tdnn.yml")), Loader=yaml.FullLoader)
    cfg["dataset_conf"]["enroll_list"], cfg["dataset_conf"]["trials_list"] = lists["enroll"], lists["trials"]
    sd = {k: v.float().numpy() for k, v in oe.make_ecapa_weights(seed=1000, dtype=torch.float64).items()}
    plain = PPVectorTrainer(copy.deepcopy(cfg), use_gpu=True, state_dict=sd)
    raw = plain.evaluate()
    # without the key: exactly the raw cosine path
    with torch.no_grad():
        E, e_lab = plain._embed_list(lists["enroll"], "e")
        T, t_lab = plain._embed_list(lists["trials"], "t")
        Cm, c_lab = plain._embed_list(lists["cohort"], "c")
    assert raw == eer_mindcf_from_matrix_gpu(cosine_matrix(T, E), t_lab, e_lab)
    cfg["dataset_conf"]["eval_conf"]["score_norm"] = {"cohort_list": lists["cohort"], "top_n": top_n, "cohort": mode}
    eer, dcf, thr = PPVectorTrainer(cfg, use_gpu=True, state_dict=sd).evaluate()
    # the oracle pipeline on the model's own embeddings
    E, T, Cm = (x.cpu().numpy() for x in (E, T, Cm))
    cohort = so.speaker_cohort(Cm, c_lab) if mode == "speaker" else Cm
    ref = so.as_norm(so.cosine(T, E), so.cohort_stats(T, cohort, top_n), so.cohort_stats(E, cohort, top_n)).reshape(-1)
    lab = (t_lab[:, None] == e_lab[None, :]).astype(np.int32).reshape(-1)
    fnr, fpr, _ = compute_fnr_fpr(ref, lab)
    eer_ref, thr_ref = compute_eer(fnr, fpr, ref)
    assert abs(eer - float(eer_ref)) < 1e-6 and abs(dcf - compute_dcf(fnr, fpr)) < 1e-6
    assert abs(thr - float(thr_ref)) < 1e-3 * max(1.0, abs(float(thr_ref)))
