"""Brute-force diarization error rate on a 1 ms grid, independent of ppvector.metric.der: annotations are [(start_ms, end_ms, label)]
with integer milliseconds, every grid cell counts its reference and hypothesis turns per label, the collar and overlap masks are
cells, and the speaker mapping is searched over every injective assignment of hypothesis labels to reference labels.

Returns every distinct component set that an optimal assignment gives (one, unless tied assignments score differently: that can
only happen where a label's turns overlap each other)."""
import itertools

import numpy as np


def _counts(turns, labels, lo, n):
    c = np.zeros((len(labels), n), np.int64)
    for a, b, lab in turns:
        c[labels.index(lab), a - lo:b - lo] += 1
    return c


def der_components_ms(reference, hypothesis, collar_ms=0, skip_overlap=False):
    """-> list of {component: seconds} dicts, one per distinct result of the optimal assignments."""
    turns = [t for t in reference + hypothesis if t[1] > t[0]]
    zero = dict.fromkeys(('false alarm', 'missed detection', 'confusion', 'correct', 'total'), 0.0)
    if not turns:
        return [zero]
    lo, hi = min(t[0] for t in turns), max(t[1] for t in turns)
    pad = collar_ms
    lo, hi, n = lo - pad, hi + pad, hi - lo + 2 * pad
    rl = sorted({t[2] for t in reference}, key=str)
    hl = sorted({t[2] for t in hypothesis}, key=str)
    rc, hc = _counts(reference, rl, lo, n), _counts(hypothesis, hl, lo, n)
    keep = np.zeros(n, bool)
    keep[pad:n - pad] = True  # the union extent
    half = collar_ms // 2
    for a, b, _ in reference:
        for t in (a, b):
            keep[t - half - lo:t + half - lo] = False
    if skip_overlap:
        keep &= rc.sum(axis=0) < 2
    rc, hc = rc[:, keep], hc[:, keep]
    cooc = rc @ hc.T
    best, results = -1, []
    small, large = (hl, rl) if len(hl) <= len(rl) else (rl, hl)
    for perm in itertools.permutations(range(len(large)), len(small)):
        pairs = [(i, p) if small is rl else (p, i) for i, p in enumerate(perm)]  # (reference index, hypothesis index)
        score = sum(int(cooc[r, h]) for r, h in pairs)
        if score < best:
            continue
        matched = sum((np.minimum(rc[r], hc[h]) for r, h in pairs if cooc[r, h] > 0), np.zeros(rc.shape[1], np.int64))
        if score > best:
            best, results = score, []
        results.append(matched)
    if not results:
        results = [np.zeros(rc.shape[1], np.int64)]
    nr, nh = rc.sum(axis=0), hc.sum(axis=0)
    out = []
    for matched in results:
        c = {'total': nr.sum() / 1000, 'correct': matched.sum() / 1000, 'confusion': (np.minimum(nr, nh) - matched).sum() / 1000,
             'missed detection': np.maximum(0, nr - nh).sum() / 1000, 'false alarm': np.maximum(0, nh - nr).sum() / 1000}
        c = {k: float(v) for k, v in c.items()}
        if c not in out:
            out.append(c)
    return out
