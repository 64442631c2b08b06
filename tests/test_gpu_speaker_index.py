"""GPU: the speaker index (ppv_speaker_index_build / ppv_speaker_index_search) against numpy -- means bitwise equal to float32
a[rows].mean(axis=0), the fused top-k search against fp64 cosine -- and PPVectorPredictor's register / remove_user / recognition
round trip on a temporary database against the enrolment oracle (tests/enrol_oracle.py)."""
import ctypes as C
import os
import pickle

import numpy as np
import pytest
import torch

from enrol_oracle import EnrolDB, topk
from ppvector import _lib
from ppvector.infer_utils.speaker_index import SpeakerIndex

pytestmark = pytest.mark.gpu


def planes_bytes(index):
    return index._index.cpu().numpy().tobytes()


def test_build_means_bitwise(cuda):
    rng = np.random.default_rng(1)
    counts = [1, 2, 7, 300, 1, 2]
    uid = np.concatenate([np.full(c, u) for u, c in enumerate(counts)])
    rng.shuffle(uid)  # users' rows interleaved: enrolment order within a user is row order
    E = (rng.normal(size=(uid.size, 192)) * rng.uniform(0.01, 100, size=(uid.size, 1))).astype(np.float32)
    E[0, :3] = -0.0
    ix = SpeakerIndex(E, uid, len(counts), cuda)
    means = ix.means.cpu().numpy()
    for u in range(len(counts)):
        ref = E[np.flatnonzero(uid == u)].mean(axis=0)
        assert means[u].tobytes() == ref.tobytes(), u
    first = planes_bytes(ix)
    ix.rebuild()
    assert planes_bytes(ix) == first and ix.means.cpu().numpy().tobytes() == means.tobytes()


def fp64_sim(q, db):
    q = q.astype(np.float64)
    db = db.astype(np.float64)
    qn = np.linalg.norm(q, axis=1, keepdims=True)
    dn = np.linalg.norm(db, axis=1, keepdims=True)
    return (q / np.where(qn > 0, qn, 1)) @ (db / np.where(dn > 0, dn, 1)).T


@pytest.mark.parametrize("U", [1, 63, 64, 65, 100000])
@pytest.mark.parametrize("Q", [1, 64, 65, 300])
@pytest.mark.parametrize("k", [1, 8])
def test_search_against_fp64(cuda, U, Q, k):
    if k > U:
        pytest.skip("k > U is rejected (test_search_rejects_bad_shapes)")
    rng = np.random.default_rng(U * 1000 + Q * 10 + k)
    D = 192
    db = rng.normal(size=(U, D)).astype(np.float32)
    if U >= 65:
        db[40] = db[7]  # exact duplicates: equal similarities, lowest index first
        db[64] = db[7]
        db[3] = 0.0  # zero-norm mean scores 0
    q = rng.normal(size=(Q, D)).astype(np.float32)
    q[0] = db[min(7, U - 1)] * 2.5 + 0.01 * rng.normal(size=D).astype(np.float32)
    if Q > 1:
        q[-1] = 0.0  # zero-norm query scores 0 everywhere
    ix = SpeakerIndex(db, np.arange(U), U, cuda)
    idx, sim = ix.search(q, k)
    idx, sim = idx.cpu().numpy(), sim.cpu().numpy()
    ref = fp64_sim(q, db)
    kth = np.sort(ref, axis=1)[:, ::-1][:, k - 1]
    assert idx.shape == (Q, k) and sim.shape == (Q, k)
    assert ((idx >= 0) & (idx < U)).all()
    got_ref = np.take_along_axis(ref, idx.astype(np.int64), axis=1)
    assert np.abs(sim - got_ref).max() <= 1e-5
    assert (sim >= kth[:, None] - 2e-5).all()
    for r in range(Q):
        assert len(set(idx[r].tolist())) == k
        for j in range(k - 1):
            assert sim[r, j] > sim[r, j + 1] or (sim[r, j] == sim[r, j + 1] and idx[r, j] < idx[r, j + 1])
    if U >= 65 and k == 8:
        assert idx[0, :3].tolist() == [7, 40, 64] and sim[0, 0] == sim[0, 1] == sim[0, 2]
    if Q > 1:
        assert (sim[-1] == 0).all() and idx[-1].tolist() == list(range(k))  # all zero: lowest indices first
    if k == 1:
        ref_idx, _ = topk(ref, 1)
        near_tie = np.sort(ref, axis=1)[:, ::-1]
        clear = (near_tie[:, 0] - near_tie[:, 1] > 1e-4) if U > 1 else np.ones(Q, bool)
        assert (idx[clear, 0] == ref_idx[clear, 0]).all()


def test_search_rejects_bad_shapes(cuda):
    lib = _lib.load()
    ix = SpeakerIndex(np.eye(4, 16, dtype=np.float32), np.arange(4), 4, cuda)
    q = torch.ones((2, 16), device=cuda)
    out_i = torch.empty(64, dtype=torch.int32, device=cuda)
    out_s = torch.empty(64, dtype=torch.float32, device=cuda)
    ws = torch.empty(1 << 20, dtype=torch.uint8, device=cuda)
    for Q, U, D, k in [(2, 4, 16, 0), (2, 4, 16, 9), (2, 4, 16, 5), (0, 4, 16, 1), (2, 0, 16, 1), (2, 4, 0, 1), (2, 4, 257, 1)]:
        rc = lib.ppv_speaker_index_search(_lib.ptr(q), Q, D, C.c_void_p(ix._index.data_ptr()), ix._index.numel(), U, k, _lib.ptr(out_i),
                                          _lib.ptr(out_s), C.c_void_p(ws.data_ptr()), ws.numel(), _lib.current_stream())
        assert rc == -1, (Q, U, D, k)
        assert 'speaker_index_search' in _lib.last_error()
    assert lib.ppv_speaker_index_bytes(4, 257) == 0 and lib.ppv_speaker_index_search_workspace_bytes(2, 4, 16, 9) == 0
    with pytest.raises(_lib.PPVError):
        ix.search(q, 9)
    torch.cuda.synchronize()


# ---- predictor round trip -------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def predictor_parts():
    import yaml
    from oracle import ecapa as oe
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    cfg = yaml.load(open(os.path.join(root, 'configs', 'ecapa_tdnn.yml')), Loader=yaml.FullLoader)
    sd = {k: v.float().numpy() for k, v in oe.make_ecapa_weights(seed=1000, dtype=torch.float64).items()}
    sr = 16000
    t = np.arange(sr * 3) / sr
    rng = np.random.default_rng(21)
    tones = [(0.3 * np.sin(2 * np.pi * f * t) * (1 + 0.1 * rng.normal(size=t.size))).astype(np.float32) for f in (180, 190, 420, 700)]
    return cfg, sd, tones


def read_index(db):
    with open(os.path.join(db, 'audio_indexes.bin'), 'rb') as f:
        return pickle.load(f)


def check_state(pred, ora, db):
    idx = read_index(db)
    assert idx['users_name'] == ora.users_name and idx['users_image_path'] == ora.users_audio_path
    assert np.asarray(idx['faces_feature']).tobytes() == ora.audio_feature.tobytes()
    assert pred.users_name == ora.users_name and pred.users_audio_path == ora.users_audio_path
    assert pred.users_name_mean == ora.users_name_mean
    assert pred.audio_feature_mean.tobytes() == ora.audio_feature_mean.tobytes()
    on_disk = sorted(f'{db}/{u}/{f}' for u in os.listdir(db) if os.path.isdir(os.path.join(db, u)) for f in os.listdir(os.path.join(db, u)))
    assert on_disk == sorted(ora.users_audio_path)


def check_recognition(pred, ora, tones):
    feats = np.stack([pred.predict(x) for x in tones])
    expect = ora.retrieval(feats, pred.threshold)
    single = [pred.recognition(x) for x in tones]
    batch = pred.recognition_batch(tones, top_k=1)
    sims = ora.similarities(feats)
    for s, b, e, row in zip(single, batch, expect, sims):
        assert (b[0] if b else [None, None]) == s
        top = np.sort(row)[::-1]
        if len(top) == 1 or top[0] - top[1] > 1e-4:
            assert s[0] == e[0]
        if s[0] is not None:
            assert abs(s[1] - row[ora.users_name_mean.index(s[0])]) <= 2e-5


def test_register_remove_recognize_round_trip(cuda, tmp_path, predictor_parts):
    from ppvector.predict import PPVectorPredictor
    cfg, sd, tones = predictor_parts
    db = str(tmp_path / 'db')
    pred = PPVectorPredictor(cfg, state_dict=sd, audio_db_path=db, threshold=0.5)
    with pytest.raises(AssertionError):
        pred.recognition(tones[0])
    ora = EnrolDB()
    for x, name in [(tones[0], 'alice'), (tones[2], 'bob'), (tones[1], 'alice')]:
        path = EnrolDB.next_path(db, name)
        assert pred.register(x, name) == (True, "注册成功")
        ora.register(name, pred.audio_feature[-1], path)
        check_state(pred, ora, db)
        check_recognition(pred, ora, tones)
        fresh = PPVectorPredictor(cfg, state_dict=sd, audio_db_path=db, threshold=0.5)
        assert sorted(fresh.users_name_mean) == sorted(ora.users_name_mean)
        assert fresh.users_name == ora.users_name and np.asarray(fresh.audio_feature).tobytes() == ora.audio_feature.tobytes()
        for name_ in ora.users_name_mean:
            i, j = fresh.users_name_mean.index(name_), ora.users_name_mean.index(name_)
            assert fresh.audio_feature_mean[i].tobytes() == ora.audio_feature_mean[j].tobytes()
    top2 = pred.recognition_batch(tones, threshold=-1.0, top_k=5)
    assert all(len(r) == 2 for r in top2)  # capped at the number of users
    assert pred.remove_user('carol') is False
    assert pred.remove_user('alice') is True
    assert ora.remove_user('alice')
    assert not os.path.exists(os.path.join(db, 'alice'))
    check_state(pred, ora, db)
    check_recognition(pred, ora, tones)
    fresh = PPVectorPredictor(cfg, state_dict=sd, audio_db_path=db, threshold=0.5)
    assert fresh.users_name_mean == ['bob'] and fresh.audio_feature_mean.tobytes() == ora.audio_feature_mean.tobytes()
    with pytest.raises(ValueError):
        PPVectorPredictor(cfg, state_dict=sd).register(tones[0], 'x')
