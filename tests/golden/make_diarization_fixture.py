"""Mint tests/golden/ref_diarization.npz: run the reference's own SpectralCluster / SpeakerDiarization
(ppvector/infer_utils/speaker_diarization.py, imported unmodified; sklearn and scipy are the real ones) stage by stage on seeded
synthetic speaker mixtures and record what it computes.  Consumed by tests/test_oracle_diarization.py on any machine.

yeaudio is not installed: the reference module imports its AudioSegment only for the silero-VAD step (segments_audio), which is not
called here, so an empty stand-in module is registered under that name before the import.

The embeddings are small integers and the affinity is oracle.diarization.integer_affinity of them, which is bitwise the same on
every machine; so the file carries the embeddings (int16) instead of the N x N affinity, the pruned matrix as a packed keep-mask
plus a SHA-256 of its bytes, and the Laplacian as a SHA-256 of its bytes plus its diagonal.

Runs only where the reference checkout is (PPV_REFERENCE, default /root/reference).
Usage:  python tests/golden/make_diarization_fixture.py            (rewrites the fixture)
        python tests/golden/make_diarization_fixture.py --check    (recomputes and compares with the committed file)
"""
import hashlib
import os
import sys
import types

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
REF = os.environ.get("PPV_REFERENCE", "/root/reference")
OUT = os.path.join(HERE, "ref_diarization.npz")
DIM = 32

# name: (N, speakers, seed); n12 / n40 / n200 have N * pval < 6 (pval -> 6 / N); "tie" has a row whose kept / pruned split falls
# between two values one ulp apart
SETS = {"n12": (12, 1, 11), "n40": (40, 2, 12), "n200": (200, 4, 13), "n801": (801, 7, 14), "tie": (40, 3, 15)}
TIE_ROW = 3


def sha(a):
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


def embeddings(N, k, seed):
    """Integer embeddings [N, DIM]: k directions on the sphere, speaker turns in runs, noise; scaled to |x| <= 1024."""
    rng = np.random.default_rng(seed)
    cent = rng.normal(size=(k, DIM))
    cent /= np.linalg.norm(cent, axis=1, keepdims=True)
    lab = np.roll(np.repeat(np.arange(k), -(-N // k))[:N], N // (3 * k))
    X = cent[lab] + 0.3 / np.sqrt(DIM) * rng.normal(size=(N, DIM))
    return np.clip(np.round(400 * X), -1024, 1024).astype(np.int16)


def tie_row(N):
    """0.1 everywhere, then 0.5 plus 0, 1, 2, ... ulps from column 10 on: the 6 kept entries and the largest pruned one are adjacent floats."""
    v = np.full(N, 0.1, dtype=np.float32)
    x = np.float32(0.5)
    for j in range(10, N):
        v[j] = x
        x = np.nextafter(x, np.float32(1))
    return v


def make():
    sys.path[:0] = [REF, ROOT]
    sys.modules.setdefault("yeaudio", types.ModuleType("yeaudio"))
    audio = types.ModuleType("yeaudio.audio")
    audio.AudioSegment = type("AudioSegment", (), {})
    sys.modules.setdefault("yeaudio.audio", audio)
    import scipy.linalg
    from ppvector.infer_utils.speaker_diarization import SpeakerDiarization, SpectralCluster

    import ppvector
    assert os.path.realpath(ppvector.__file__).startswith(os.path.realpath(REF)), ppvector.__file__
    from oracle.diarization import integer_affinity

    d = {}
    for name, (N, k, seed) in SETS.items():
        Xi = embeddings(N, k, seed)
        X = Xi.astype(np.float32)
        sc = SpectralCluster()
        A = integer_affinity(Xi)
        out = {"Xi": Xi}
        if name == "tie":
            A[TIE_ROW] = out["tie_vals"] = tie_row(N)
        pval = 6. / N if N * sc.pval < 6 else sc.pval
        n_elems = int((1 - pval) * N)
        srt = np.sort(A, axis=1)
        # no exact tie straddles the threshold: numpy's argsort (what the reference uses) leaves the order of equal values unspecified
        assert np.all(srt[:, n_elems - 1] < srt[:, n_elems]), name
        P = sc.p_pruning(A.copy())
        L = sc.get_laplacian(0.5 * (P + P.T))
        lam = scipy.linalg.eigh(L)[0]
        _, k_auto = sc.get_spec_embs(L)
        out.update(pruned_mask=np.packbits(P != 0), pruned_sha=np.array(sha(P)), laplacian_sha=np.array(sha(L)),
                   laplacian_diag=np.diag(L).copy(), lambdas=lam[:16], seed=np.array(seed), k_auto=np.array(k_auto), k_oracle=np.array(k))
        for tag, kk in (("auto", None), ("oracle", k)):
            emb, num = sc.get_spec_embs(L, kk)
            np.random.seed(seed)
            out["labels_" + tag] = SpeakerDiarization._correct_labels(sc.cluster_embs(emb, num))
        sd = SpeakerDiarization()
        labels = out["labels_auto"]
        centres = np.stack([X[labels == i].mean(0) for i in range(labels.max() + 1)], axis=0)
        merged = sd._merge_by_cos(labels.copy(), list(centres), sd.merge_threshold)
        times = np.stack([np.arange(N) * 0.75, np.arange(N) * 0.75 + 1.5], axis=1)
        post = sd.postprocess([[t[0], t[1], None] for t in times.tolist()], merged)
        out.update(centres=centres, merged=merged, merge_threshold=np.array(sd.merge_threshold),
                   post=np.array([[r["speaker"], r["start"], r["end"]] for r in post], dtype=np.float64))
        d.update({f"{name}/{key}": np.asarray(v) for key, v in out.items()})
    return d


def main():
    d = make()
    if "--check" in sys.argv:
        old = np.load(OUT)
        assert sorted(old.files) == sorted(d), set(old.files) ^ set(d)
        bad = [k for k in d if not np.array_equal(old[k], d[k])]
        print(f"{os.path.basename(OUT)}: {len(d)} arrays, {len(bad)} differ {bad}")
        sys.exit(1 if bad else 0)
    np.savez_compressed(OUT, **d)
    print(f"wrote {os.path.basename(OUT)}: {len(d)} arrays, {os.path.getsize(OUT)} bytes")


if __name__ == "__main__":
    main()
