"""fp64 numpy statement of adaptive symmetric score normalisation (AS-norm), the definition ppvector/metric/score_norm.py and
csrc/score_norm.cu follow: for each query row the multiset of its top_n largest cohort scores (ties by value, counted with
multiplicity), its mean and its standard deviation with the (top_n - 1) divisor floored at 1e-6, and
s'(t, e) = ((s - mean_e) / std_e + (s - mean_t) / std_t) / 2."""
import numpy as np

STD_FLOOR = 1e-6


def cosine(a, b):
    """fp64 cosine [len(a), len(b)] (a zero-norm row scores 0)."""
    a = np.asarray(a, dtype=np.float64)
    b = np.asarray(b, dtype=np.float64)
    an = np.linalg.norm(a, axis=1, keepdims=True)
    bn = np.linalg.norm(b, axis=1, keepdims=True)
    return (a / np.where(an > 0, an, 1.0)) @ (b / np.where(bn > 0, bn, 1.0)).T


def top_n_values(scores, top_n):
    """[rows, top_n] fp64: each row's top_n largest values, descending."""
    s = np.asarray(scores, dtype=np.float64)
    part = -np.partition(-s, top_n - 1, axis=1)[:, :top_n]
    return -np.sort(-part, axis=1)


def topn_stats(scores, top_n):
    """scores [rows, cols] -> (mean [rows], std [rows]) fp64 of each row's top_n largest values."""
    top = top_n_values(scores, top_n)
    mean = top.mean(axis=1)
    std = np.sqrt(((top - mean[:, None]) ** 2).sum(axis=1) / (top_n - 1))
    return mean, np.maximum(std, STD_FLOOR)


def speaker_cohort(emb, labels):
    """One float32 row per distinct label (ascending): the mean of that label's rows in list order."""
    emb = np.asarray(emb, dtype=np.float32)
    labels = np.asarray(labels)
    return np.stack([emb[labels == u].mean(axis=0) for u in np.unique(labels)])


def cohort_stats(emb, cohort, top_n):
    return topn_stats(cosine(emb, cohort), top_n)


def as_norm(scores, trial_stats, enroll_stats):
    """fp64 normalised [M, N] scores from (mean, std) of the trials [M] and the enrolments [N]."""
    s = np.asarray(scores, dtype=np.float64)
    mt, st = (np.asarray(x, dtype=np.float64) for x in trial_stats)
    me, se = (np.asarray(x, dtype=np.float64) for x in enroll_stats)
    st, se = np.maximum(st, STD_FLOOR), np.maximum(se, STD_FLOOR)
    return 0.5 * ((s - me[None, :]) / se[None, :] + (s - mt[:, None]) / st[:, None])
