"""CPU: the diarization oracle (oracle/diarization.py) against what the reference's own speaker_diarization.py computed
(tests/golden/ref_diarization.npz, minted by tests/golden/make_diarization_fixture.py), the CLI's option table, and the enrolment
index format."""
import hashlib
import os
import pickle

import numpy as np
import pytest
import scipy.linalg

from oracle import diarization as od

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ref_diarization.npz")
SETS = ["n12", "n40", "n200", "n801", "tie"]


def sha(a):
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


@pytest.mark.parametrize("name", SETS)
def test_oracle_equals_reference(name):
    d = np.load(GOLDEN)
    g = {k.split("/", 1)[1]: d[k] for k in d.files if k.startswith(name + "/")}
    X = g["Xi"].astype(np.float32)
    A = od.integer_affinity(g["Xi"])
    if "tie_vals" in g:
        A[3] = g["tie_vals"]
    N = A.shape[0]
    P = od.prune(A)
    assert np.array_equal(np.packbits(P != 0), g["pruned_mask"])
    assert sha(P) == str(g["pruned_sha"])
    L = od.laplacian(P)  # the reference's float32 path, op for op
    assert L.dtype == np.float32 and np.array_equal(np.diag(L), g["laplacian_diag"]) and sha(L) == str(g["laplacian_sha"])
    L64 = od.laplacian(P, np.float64)
    lam64 = scipy.linalg.eigvalsh(L64)[:16]
    nrm = np.linalg.norm(L64, 2)
    assert np.abs(lam64 - g["lambdas"].astype(np.float64)).max() <= 1e-5 * nrm  # the reference's float32 eigh
    assert od.eigengap_k(g["lambdas"]) == int(g["k_auto"]) == od.eigengap_k(lam64)
    # the reference's labels: sklearn k_means after np.random.seed(seed); the oracle takes the same draws
    for tag in ("auto", "oracle"):
        k = int(g["k_" + tag])
        V = scipy.linalg.eigh(L64)[1][:, :k]
        rs = np.random.RandomState(int(g["seed"]))
        lab, _, _ = od.kmeans(V, k, rs.random_sample(od.n_uniforms(k)))
        assert np.array_equal(od.correct_labels(lab), g["labels_" + tag]), tag
    lab = g["labels_auto"]
    assert np.array_equal(od.cluster_centres(X, lab), g["centres"])
    merged = od.merge_by_cos(lab, list(g["centres"]), float(g["merge_threshold"]))
    assert np.array_equal(merged, g["merged"])
    times = np.stack([np.arange(N) * 0.75, np.arange(N) * 0.75 + 1.5], axis=1)
    out = od.postprocess(times, merged)
    assert [[o["speaker"], o["start"], o["end"]] for o in out] == g["post"].tolist()


def test_integer_affinity_is_exact():
    """The fixture's affinity recipe: exact integer Gram matrix, so the float32 result does not depend on the BLAS summation order."""
    rng = np.random.default_rng(0)
    Xi = rng.integers(-1024, 1025, size=(50, 32))
    A = od.integer_affinity(Xi)
    G = [[sum(int(a) * int(b) for a, b in zip(x, y)) for y in Xi] for x in Xi]
    n = np.sqrt(np.array([G[i][i] for i in range(50)], dtype=np.float64))
    ref = (np.array(G, dtype=np.float64) / (n[:, None] * n[None, :])).astype(np.float32)
    assert np.array_equal(A, ref)


def test_merge_by_cos_quirk():
    """After a merge the reference keeps indexing its original centre list: with centres a, a', b (a ~ a'), merging 0 and 1 leaves
    labels {0, 1} compared against centres [a, a'] -- so b's centre drops out and the a/b labels merge too."""
    a = np.array([1.0, 0.0, 0.0])
    c = [a, a + [0, 0.05, 0], np.array([0.0, 1.0, 0.0])]
    lab = np.array([0, 1, 2, 2, 0])
    assert od.merge_by_cos(lab, c, 0.78).tolist() == [0, 0, 0, 0, 0]
    from ppvector.infer_utils.speaker_diarization import SpeakerDiarization
    assert SpeakerDiarization._merge_by_cos(lab.copy(), c, 0.78).tolist() == [0, 0, 0, 0, 0]


def test_host_postprocess_equals_oracle():
    from ppvector.infer_utils.speaker_diarization import SpeakerDiarization
    rng = np.random.default_rng(3)
    times = np.stack([np.arange(40) * 0.75, np.arange(40) * 0.75 + 1.5], axis=1)
    labels = np.repeat(rng.integers(0, 3, 10), 4)
    labels[17] = (labels[17] + 1) % 3  # a short turn that _smooth absorbs
    host = SpeakerDiarization().postprocess([list(t) for t in times.tolist()], labels)
    assert host == od.postprocess(times, labels)
    with pytest.raises(IndexError):  # the reference's _smooth on a single too-short segment
        SpeakerDiarization()._smooth([[0.0, 0.5, 0]])


def test_cli_options_match_reference():
    import infer_speaker_diarization as cli
    assert [(n, t, d) for n, t, d, _ in cli.OPTIONS] == [
        ('configs', str, 'configs/cam++.yml'), ('audio_path', str, 'dataset/test_long.wav'), ('audio_db_path', str, 'audio_db/'),
        ('speaker_num', int, None), ('use_gpu', bool, True), ('show_plot', bool, True), ('search_audio_db', bool, True),
        ('threshold', float, 0.6), ('model_path', str, 'models/CAMPPlus_Fbank/best_model/')]


def test_audio_index_round_trip(tmp_path):
    """audio_indexes.bin: the reference's pickle layout, read back by the predictor's loader (files that are gone are dropped)."""
    from ppvector.predict import PPVectorPredictor
    (tmp_path / "a.wav").write_bytes(b"")
    feats = np.arange(6, dtype=np.float32).reshape(2, 3)
    with open(tmp_path / "audio_indexes.bin", "wb") as f:
        pickle.dump({"users_name": ["u", "v"], "faces_feature": feats,
                     "users_image_path": [str(tmp_path / "a.wav"), str(tmp_path / "gone.wav")]}, f)
    p = PPVectorPredictor.__new__(PPVectorPredictor)
    p.users_name, p.users_audio_path, p.audio_feature = [], [], None
    p.audio_indexes_path = str(tmp_path / "audio_indexes.bin")
    p._load_audio_indexes()
    assert p.users_name == ["u"] and p.users_audio_path == [str(tmp_path / "a.wav")]
    assert np.array_equal(p.audio_feature, feats[:1])
    p._write_index()
    with open(tmp_path / "audio_indexes.bin", "rb") as f:
        back = pickle.load(f)
    assert back["users_name"] == ["u"] and np.array_equal(back["faces_feature"], feats[:1])
