"""GPU: the spectral-clustering kernels of speaker diarization (csrc/cluster.cu), each stage on its own stored inputs, against
the fp64 oracle (oracle/diarization.py) and scipy; then SpectralCluster and PPVectorPredictor.speaker_diarization end to end."""
import numpy as np
import pytest
import scipy.linalg
import torch

from oracle import diarization as od

pytestmark = pytest.mark.gpu

SIZES = [7, 16, 40, 257, 1000, 3001]


def mixture(N, k, seed, dim=192, noise=0.5):
    """Synthetic speaker mixture: k centroids on the sphere plus noise, contiguous speaker turns."""
    rng = np.random.default_rng(seed)
    cent = rng.normal(size=(k, dim))
    cent /= np.linalg.norm(cent, axis=1, keepdims=True)
    turns = np.sort(rng.integers(0, N, size=3 * k))
    lab = np.zeros(N, dtype=np.int64)
    for t, s in enumerate(turns):
        lab[s:] = t % k
    return (cent[lab] + noise / np.sqrt(dim) * rng.normal(size=(N, dim))).astype(np.float32)


def gpu_affinity(X, cuda):
    from ppvector.metric.cosine import cosine_matrix
    return cosine_matrix(torch.from_numpy(X).to(cuda), torch.from_numpy(X).to(cuda))


@pytest.mark.parametrize("N", SIZES)
def test_prune_and_laplacian(cuda, N):
    from ppvector.infer_utils.speaker_diarization import SpectralCluster
    X = mixture(N, 3, N)
    A = gpu_affinity(X, cuda)
    if N == 40:  # a row of exact ties at the threshold: the lower column index is pruned first
        A[5] = 0.25
        A[5, :3] = 0.5
    A_host = A.cpu().numpy()
    L = SpectralCluster.laplacian(A, 0.022).cpu().numpy()
    P_ref = od.prune(A_host)
    assert np.array_equal(A.cpu().numpy() == 0, P_ref == 0)
    assert np.array_equal(A.cpu().numpy(), P_ref)
    L_ref = od.laplacian(P_ref, np.float64)
    assert np.abs(L - L_ref).max() <= 1e-12 * np.abs(L_ref).max()


@pytest.mark.parametrize("N", SIZES)
def test_smallest_eigenpairs(cuda, N):
    from ppvector.infer_utils.speaker_diarization import SpectralCluster
    k = min(4, N)
    X = mixture(N, k, 100 + N)
    L_ref = od.laplacian(od.prune(gpu_affinity(X, cuda).cpu().numpy()), np.float64)
    m = min(16, N)
    lam_ref, V_ref = scipy.linalg.eigh(L_ref)
    evals, V = SpectralCluster.smallest_eigs(torch.from_numpy(L_ref.copy()).to(cuda), m)
    V = V.cpu().numpy()
    nrm = np.linalg.norm(L_ref, 2)
    assert np.abs(evals - lam_ref[:m]).max() <= 1e-10 * nrm
    assert np.abs(V.T @ V - np.eye(m)).max() <= 1e-10
    assert np.abs(L_ref @ V - V * evals[None, :]).max() <= 1e-9 * nrm
    # the k-subspace where the gap after lambda_k is clear: principal angles against scipy's
    for kk in range(1, m):
        gap = lam_ref[kk] - lam_ref[kk - 1]
        if gap > 1e-3 * nrm:
            assert scipy.linalg.subspace_angles(V_ref[:, :kk], V[:, :kk]).max() <= 1e-8, kk


@pytest.mark.parametrize("N", SIZES)
def test_kmeans_matches_oracle(cuda, N):
    from ppvector.infer_utils.speaker_diarization import SpectralCluster
    k = min(5, N)
    X = mixture(N, k, 200 + N)
    L_ref = od.laplacian(od.prune(od.cosine_affinity(X.astype(np.float64)).astype(np.float32)), np.float64)
    m = min(16, N)
    V = scipy.linalg.eigh(L_ref)[1][:, :m]
    rng = np.random.RandomState(N)
    for kk in sorted({1, 2, k}):
        u = rng.random_sample(od.n_uniforms(kk))
        lab, inertia = SpectralCluster.kmeans(torch.from_numpy(np.ascontiguousarray(V)).to(cuda), kk, u)
        lab_ref, in_ref, _ = od.kmeans(V[:, :kk], kk, u)
        assert np.array_equal(lab, lab_ref), kk
        # relative to the inertia, or to the total spread where the clusters collapse to points (inertia ~ 0)
        spread = float(((V[:, :kk] - V[:, :kk].mean(0)) ** 2).sum())
        assert abs(inertia - in_ref) <= 1e-9 * max(abs(in_ref), spread), kk


@pytest.mark.parametrize("N,k", [(60, 2), (400, 3), (1200, 5), (3000, 9)])
def test_spectral_cluster_end_to_end(cuda, N, k):
    from ppvector.infer_utils.speaker_diarization import SpectralCluster
    X = mixture(N, k, 300 + N, noise=0.3)
    A = gpu_affinity(X, cuda).cpu().numpy()
    for oracle_num in (None, k):
        np.random.seed(N)
        labels = SpectralCluster()(X, oracle_num=oracle_num)
        np.random.seed(N)
        ref, k_ref, _ = od.spectral_cluster(X, np.random.random_sample, oracle_num=oracle_num, affinity=A)
        assert labels.max() + 1 == k_ref
        assert np.array_equal(od.correct_labels(labels), od.correct_labels(ref))


def test_too_many_windows_raise(cuda):
    from ppvector import _lib
    from ppvector.infer_utils.speaker_diarization import SpectralCluster
    A = torch.zeros((8193, 8193), dtype=torch.float32, device=cuda)
    with pytest.raises(_lib.PPVError, match="8192"):
        SpectralCluster.laplacian(A)


def test_speaker_diarization_predictor(cuda):
    """A seeded multi-segment recording: the predictor's result equals the oracle run on the embeddings diarization_embeddings
    returns (same k-means draws)."""
    from oracle import ecapa as oe
    from ppvector.infer_utils.speaker_diarization import SpeakerDiarization
    from ppvector.predict import PPVectorPredictor
    import yaml
    import os
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    cfg = yaml.load(open(os.path.join(root, 'configs', 'ecapa_tdnn.yml')), Loader=yaml.FullLoader)
    W = oe.make_ecapa_weights(seed=1000, dtype=torch.float64)
    pred = PPVectorPredictor(cfg, state_dict={k: v.float().numpy() for k, v in W.items()})
    rng = np.random.default_rng(7)
    sr = 16000
    t = np.arange(sr * 12) / sr
    wav = np.concatenate([0.3 * np.sin(2 * np.pi * f * t[:sr * 4]) * (1 + 0.1 * rng.normal(size=sr * 4)) for f in (180, 420, 180)])
    wav = wav.astype(np.float32)
    vad = [(0.0, 5.2), (5.5, 12.0)]
    np.random.seed(3)
    out = pred.speaker_diarization(wav, sample_rate=sr, vad_segments=vad)
    times, emb = pred.diarization_embeddings(wav, sample_rate=sr, vad_segments=vad)
    np.random.seed(3)
    lab, _, _ = od.spectral_cluster(emb, np.random.random_sample, affinity=gpu_affinity(emb, cuda).cpu().numpy())
    lab = od.correct_labels(lab)
    lab = od.merge_by_cos(lab, od.cluster_centres(emb, lab), SpeakerDiarization().merge_threshold)
    assert out == od.postprocess(times, lab)
    assert len(out) >= 1 and out[0]['start'] == 0.0


def test_search_audio_db_names(cuda, tmp_path):
    """With an enrolment database, search_audio_db=True names each speaker like a numpy cosine arg-max with the threshold applied
    (the reference indexes the pre-merge centres with the post-merge labels; that is what this reproduces)."""
    import os
    import pickle

    import scipy.io.wavfile
    import yaml

    from oracle import ecapa as oe
    from ppvector.infer_utils.speaker_diarization import SpeakerDiarization
    from ppvector.predict import PPVectorPredictor
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    cfg = yaml.load(open(os.path.join(root, 'configs', 'ecapa_tdnn.yml')), Loader=yaml.FullLoader)
    sd = {k: v.float().numpy() for k, v in oe.make_ecapa_weights(seed=1000, dtype=torch.float64).items()}
    sr = 16000
    t = np.arange(sr * 4) / sr
    rng = np.random.default_rng(11)
    tone = {name: (0.3 * np.sin(2 * np.pi * f * t) * (1 + 0.1 * rng.normal(size=t.size))).astype(np.float32)
            for name, f in (('alice', 180), ('bob', 420))}
    for name, x in tone.items():
        os.makedirs(tmp_path / name)
        scipy.io.wavfile.write(str(tmp_path / name / '0.wav'), sr, x)
    pred = PPVectorPredictor(cfg, state_dict=sd, audio_db_path=str(tmp_path), threshold=0.5)
    assert sorted(pred.get_users()) == ['alice', 'bob'] and os.path.exists(tmp_path / 'audio_indexes.bin')
    with open(tmp_path / 'audio_indexes.bin', 'rb') as f:
        idx = pickle.load(f)
    assert set(idx) == {'users_name', 'faces_feature', 'users_image_path'} and idx['faces_feature'].shape[0] == 2
    wav = np.concatenate([tone['alice'], tone['bob'], tone['alice']])
    np.random.seed(5)
    out = pred.speaker_diarization(wav, sample_rate=sr, search_audio_db=True)
    np.random.seed(5)
    plain = pred.speaker_diarization(wav, sample_rate=sr)
    times, emb = pred.diarization_embeddings(wav, sample_rate=sr)
    np.random.seed(5)
    lab = od.correct_labels(SpeakerDiarization().spectral_cluster(emb))
    centres = od.cluster_centres(emb, lab)
    q = centres / np.linalg.norm(centres, axis=1, keepdims=True)
    db = pred.audio_feature_mean / np.linalg.norm(pred.audio_feature_mean, axis=1, keepdims=True)
    sim = q @ db.T
    names = [pred.users_name_mean[int(np.argmax(s))] if s.max() >= 0.5 else None for s in sim]
    assert [o['speaker'] for o in out] == [names[p['speaker']] or f"陌生人{p['speaker']}" for p in plain]
    assert [(o['start'], o['end']) for o in out] == [(p['start'], p['end']) for p in plain]
