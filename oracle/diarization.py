"""numpy / scipy restatement of the reference's spectral clustering and diarization post-processing
(ppvector/infer_utils/speaker_diarization.py of the reference checkout), the yardstick of csrc/cluster.cu and
ppvector/infer_utils/speaker_diarization.py.

Every function computes in the dtype it is given (float32 reproduces the reference's own float32 path; float64 is the
fp64 yardstick of the kernels).  k-means restates sklearn's ``k_means(X, k, n_init="auto")`` (sklearn/cluster/_kmeans.py:
``KMeans.fit`` centring, ``_tolerance``, ``_kmeans_plusplus``, ``_kmeans_single_lloyd``; the E-step / M-step of
``_k_means_lloyd.pyx`` and ``_relocate_empty_clusters_dense`` / ``_average_centers`` / ``_center_shift`` / ``_inertia_dense`` of
``_k_means_common.pyx``) on caller-supplied uniforms, drawn in numpy's order: one for the first centre
(``RandomState.choice(n, p=w)``), then ``2 + int(log k)`` per further centre (``RandomState.uniform``).
"""
import numpy as np
import scipy.linalg

__all__ = ['cosine_affinity', 'integer_affinity', 'prune', 'laplacian', 'eigengap_k', 'kmeans', 'n_uniforms', 'spectral_cluster', 'correct_labels',
           'merge_by_cos', 'merge_seque', 'smooth', 'postprocess', 'cluster_centres']


def cosine_affinity(X):
    """sklearn cosine_similarity (speaker_diarization.py:253-257)."""
    X = np.asarray(X)
    n = np.linalg.norm(X, axis=1, keepdims=True)
    n[n == 0] = 1
    Xn = X / n
    return Xn @ Xn.T


def integer_affinity(Xi):
    """float32 cosine affinity of integer-valued embeddings Xi (|x| <= 2^10, D <= 64), bitwise the same on every machine: the dot
    products are exact integers in fp64 whatever the BLAS summation order, and sqrt, product, quotient and the cast to float32 are
    each correctly rounded.  The reference fixture is built on it, so the fixture carries the embeddings, not the N x N affinity."""
    X = np.asarray(Xi, dtype=np.float64)
    assert np.all(X == np.round(X)) and np.abs(X).max() <= 1024 and X.shape[1] <= 64
    G = X @ X.T
    n = np.sqrt(np.diag(G))
    return (G / (n[:, None] * n[None, :])).astype(np.float32)


def prune(A, pval=0.022):
    """p_pruning (:260-275), on a copy.  Exact ties at the threshold: the lower column index is pruned first (a stable sort);
    numpy's default argsort, which the reference uses, leaves that order unspecified."""
    A = np.array(A, copy=True)
    N = A.shape[0]
    if N * pval < 6:
        pval = 6. / N
    n_elems = int((1 - pval) * N)
    for i in range(N):
        low = np.argsort(A[i, :], kind='stable')[:n_elems]
        A[i, low] = 0
    return A


def laplacian(P, dtype=None):
    """:246 (symmetrise) and get_laplacian (:277-283) in ``dtype`` (default: P's)."""
    P = np.asarray(P, dtype=dtype or np.asarray(P).dtype)
    M = 0.5 * (P + P.T)
    M[np.diag_indices(M.shape[0])] = 0
    D = np.sum(np.abs(M), axis=1)
    return np.diag(D) - M


def eigengap_k(lambdas, min_num_spks=1, max_num_spks=15):
    """get_spec_embs without oracle_num (:291-292) and get_eigen_gaps (:305-310)."""
    vals = lambdas[min_num_spks - 1:max_num_spks + 1]
    gaps = [float(vals[i + 1]) - float(vals[i]) for i in range(len(vals) - 1)]
    return int(np.argmax(gaps)) + min_num_spks


def n_uniforms(k):
    return 1 + (k - 1) * (2 + int(np.log(k)))


def kmeans(X, k, uniforms, max_iter=300, tol=1e-4):
    """sklearn k_means(X, k, n_init="auto") with the given uniforms -> (labels int32, inertia, centres)."""
    X = np.array(X, dtype=np.float64, copy=True)
    N = X.shape[0]
    u = np.asarray(uniforms, dtype=np.float64)
    assert u.size >= n_uniforms(k)
    tol = np.mean(np.var(X, axis=0)) * tol                  # _tolerance, on the uncentred data
    X -= X.mean(axis=0)                                     # KMeans.fit
    xsq = np.einsum('ij,ij->i', X, X)
    w = np.ones(N)
    # _kmeans_plusplus
    n_trials = 2 + int(np.log(k))
    cdf = np.cumsum(w / w.sum())
    cdf /= cdf[-1]
    cid = min(int(np.searchsorted(cdf, u[0], side='right')), N - 1)
    centres = np.empty((k, X.shape[1]))
    centres[0] = X[cid]

    def sqd(C):  # _euclidean_distances(C, X, Y_norm_squared=xsq, squared=True)
        d = -2 * (C @ X.T)
        d += np.einsum('ij,ij->i', C, C)[:, None]
        d += xsq[None, :]
        return np.maximum(d, 0)

    closest = sqd(centres[:1])[0]
    pot = closest.sum()
    for c in range(1, k):
        vals = u[1 + (c - 1) * n_trials:1 + c * n_trials] * pot
        cand = np.minimum(np.searchsorted(np.cumsum(closest), vals), N - 1)
        dc = np.minimum(closest[None, :], sqd(X[cand]))
        pots = dc.sum(axis=1)
        b = int(np.argmin(pots))
        pot, closest = pots[b], dc[b]
        centres[c] = X[cand[b]]
    # _kmeans_single_lloyd
    labels_old = np.full(N, -1)
    strict = False
    for _ in range(max_iter):
        labels = np.argmin(np.einsum('ij,ij->i', centres, centres)[None, :] - 2 * (X @ centres.T), axis=1)
        sums = np.zeros_like(centres)
        np.add.at(sums, labels, X)
        wk = np.bincount(labels, minlength=k).astype(np.float64)
        empty = np.where(wk == 0)[0]
        if len(empty):  # _relocate_empty_clusters_dense: farthest points from their (old) centre, ties to the lower index
            dist = ((X - centres[labels]) ** 2).sum(axis=1)
            far = np.argsort(-dist, kind='stable')[:len(empty)]
            for new, fi in zip(empty, far):
                old = labels[fi]
                sums[old] -= X[fi]
                sums[new] = X[fi]
                wk[new] = 1
                wk[old] -= 1
        new_c = sums * (1.0 / np.where(wk > 0, wk, 1))[:, None]
        shift_tot = (np.sqrt(((new_c - centres) ** 2).sum(axis=1)) ** 2).sum()
        centres = new_c
        if np.array_equal(labels, labels_old):
            strict = True
            break
        if shift_tot <= tol:
            break
        labels_old = labels
    if not strict:
        labels = np.argmin(np.einsum('ij,ij->i', centres, centres)[None, :] - 2 * (X @ centres.T), axis=1)
    inertia = float(((X - centres[labels]) ** 2).sum())
    return labels.astype(np.int32), inertia, centres


def spectral_cluster(X, uniforms_fn, oracle_num=None, pval=0.022, min_num_spks=1, max_num_spks=15, affinity=None):
    """SpectralCluster.__call__ (:235-250) in fp64 -> (labels, k, the 16 smallest eigenvalues).  ``uniforms_fn(n)`` supplies the
    k-means draws; ``affinity`` replaces the cosine affinity (e.g. the GPU's fp32 one)."""
    A = cosine_affinity(X) if affinity is None else affinity
    L = laplacian(prune(A, pval), np.float64)
    lam, V = scipy.linalg.eigh(L)
    k = oracle_num if oracle_num is not None else eigengap_k(lam, min_num_spks, max_num_spks)
    labels, _, _ = kmeans(V[:, :k], k, uniforms_fn(n_uniforms(k)))
    return labels, k, lam[:16]


# ---- SpeakerDiarization (:9-216): label and segment post-processing ---------------------------------------------------
def correct_labels(labels):
    """_correct_labels (:177-187): renumber in order of first appearance."""
    id2id, out = {}, []
    for i in labels:
        if i not in id2id:
            id2id[i] = len(id2id)
        out.append(id2id[i])
    return np.array(out)


def cluster_centres(embeddings, labels):
    """clustering (:100-107): mean embedding of every label."""
    return np.stack([embeddings[labels == i].mean(0) for i in range(labels.max() + 1)], axis=0)


def merge_by_cos(labels, spk_center_emb, cos_thr):
    """_merge_by_cos (:113-136), quirk included: after a merge the label count drops but the centre list is not updated, so
    the next round compares the first (count) centres of the ORIGINAL list -- the last centre drops out, not the merged one."""
    labels = np.array(labels, copy=True)
    assert 0 < cos_thr <= 1
    while True:
        spk_num = labels.max() + 1
        if spk_num == 1:
            break
        c = np.stack([spk_center_emb[i] for i in range(spk_num)], axis=0)
        c = c / np.linalg.norm(c, axis=1, keepdims=True)
        aff = np.triu(c @ c.T, 1)
        spks = np.unravel_index(np.argmax(aff), aff.shape)
        if aff[spks] < cos_thr:
            break
        for i in range(len(labels)):
            if labels[i] == spks[1]:
                labels[i] = spks[0]
            elif labels[i] > spks[1]:
                labels[i] -= 1
    return labels


def merge_seque(res):
    """_merge_seque (:190-198)."""
    out = [res[0]]
    for r in res[1:]:
        if r[2] != out[-1][2] or r[0] > out[-1][1]:
            out.append(r)
        else:
            out[-1][1] = r[1]
    return out


def smooth(res, min_duration=1):
    """_smooth (:201-216); like the reference it raises IndexError for a single too-short segment."""
    for i in range(len(res)):
        res[i][0] = round(res[i][0], 2)
        res[i][1] = round(res[i][1], 2)
        if res[i][1] - res[i][0] < min_duration:
            if i == 0:
                res[i][2] = res[i + 1][2]
            elif i == len(res) - 1:
                res[i][2] = res[i - 1][2]
            elif res[i][0] - res[i - 1][1] <= res[i + 1][0] - res[i][1]:
                res[i][2] = res[i - 1][2]
            else:
                res[i][2] = res[i + 1][2]
    return merge_seque(res)


def postprocess(times, labels):
    """postprocess (:138-174): times [n, 2] seconds, labels [n] -> [{'speaker', 'start', 'end'}]."""
    assert len(times) == len(labels)
    res = merge_seque([[times[i][0], times[i][1], labels[i]] for i in range(len(times))])
    for i in range(1, len(res)):
        if res[i - 1][1] > res[i][0] + 1e-4:
            p = (res[i][0] + res[i - 1][1]) / 2
            res[i][0] = p
            res[i - 1][1] = p
    res = smooth(res)
    return [dict(speaker=r[2], start=round(r[0], 3), end=round(r[1], 3)) for r in res]
