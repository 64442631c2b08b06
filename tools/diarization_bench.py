"""Time the speaker-diarization clustering chain stage by stage on the GPU (CUDA events) at N = 800, 3200, 8000 windows, and the
reference's CPU chain (numpy pruning loop, scipy.linalg.eigh, sklearn k_means) on the same data in the same run.

    python tools/diarization_bench.py [--sizes 800,3200,8000] [--out profiles/diarization_bench.txt]
"""
import argparse
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "voiceprintrecognition-paddlepaddle_b200")]


def mixture(N, k, seed, dim=192):
    rng = np.random.default_rng(seed)
    cent = rng.normal(size=(k, dim))
    cent /= np.linalg.norm(cent, axis=1, keepdims=True)
    lab = np.sort(rng.integers(0, k, N))
    return (cent[lab] + 0.4 / np.sqrt(dim) * rng.normal(size=(N, dim))).astype(np.float32)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="800,3200,8000")
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "diarization_bench.txt"))
    ap.add_argument("--skip-cpu-above", type=int, default=8192)
    a = ap.parse_args()
    import scipy.linalg
    import torch
    from sklearn.cluster import k_means

    from ppvector.infer_utils.speaker_diarization import SpectralCluster
    from ppvector.metric.cosine import cosine_matrix
    assert torch.cuda.is_available(), "diarization_bench needs a GPU"
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    lines = [f"# GPU: {q.stdout.strip() or torch.cuda.get_device_name()}",
             f"# CPU chain: {os.cpu_count()} host cores (numpy / scipy / sklearn threads as configured)",
             "# N, k, stage times in ms: cosine, prune+laplacian, eig (m=16), kmeans, GPU total | CPU prune+laplacian, eigh, kmeans, CPU total"]
    sc = SpectralCluster()
    for N in [int(s) for s in a.sizes.split(",")]:
        k = 6
        X = torch.from_numpy(mixture(N, k, N)).cuda()
        for rep in range(2):  # the first pass warms up
            ev = [torch.cuda.Event(enable_timing=True) for _ in range(5)]
            ev[0].record()
            A = cosine_matrix(X, X)
            ev[1].record()
            L = sc.laplacian(A, sc.pval)
            ev[2].record()
            lam, V = sc.smallest_eigs(L, 16)
            ev[3].record()
            np.random.seed(0)
            sc.kmeans(V, k, np.random.random_sample(1 + (k - 1) * (2 + int(np.log(k)))))
            ev[4].record()
            torch.cuda.synchronize()
        g = [ev[i].elapsed_time(ev[i + 1]) for i in range(4)]
        row = f"{N:5d} {k:2d}  " + " ".join(f"{t:9.2f}" for t in g) + f" {sum(g):9.2f} |"
        if N <= a.skip_cpu_above:
            A_h = A.cpu().numpy()
            t0 = time.perf_counter()
            P = sc_ref_prune(A_h, sc.pval)
            M = 0.5 * (P + P.T)
            M[np.diag_indices(N)] = 0
            Lh = np.diag(np.abs(M).sum(1)) - M
            t1 = time.perf_counter()
            _, vecs = scipy.linalg.eigh(Lh)
            t2 = time.perf_counter()
            np.random.seed(0)
            k_means(vecs[:, :k], k, n_init="auto")
            t3 = time.perf_counter()
            c = [1e3 * (t1 - t0), 1e3 * (t2 - t1), 1e3 * (t3 - t2)]
            row += " " + " ".join(f"{t:9.2f}" for t in c) + f" {sum(c):9.2f}"
        lines.append(row)
        print(row, flush=True)
    os.makedirs(os.path.dirname(a.out), exist_ok=True)
    with open(a.out, "w") as f:
        f.write("\n".join(lines) + "\n")
    print("\n".join(lines[:3]))


def sc_ref_prune(A, pval):
    """The reference's p_pruning loop (argsort per row) on a copy."""
    A = A.copy()
    N = A.shape[0]
    if N * pval < 6:
        pval = 6. / N
    n = int((1 - pval) * N)
    for i in range(N):
        A[i, np.argsort(A[i, :])[:n]] = 0
    return A


if __name__ == "__main__":
    main()
