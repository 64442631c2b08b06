"""Diarization error rate and RTTM I/O on the host -- the part of pyannote.metrics / pyannote.database that the reference's
tools/eval_speaker_diarization scores with, restated without pyannote (DESIGN.md §7, "Diarization error rate").

An annotation is a list of speaker turns ``[(start_s, end_s, label), ...]``.  Turns may overlap, also under the same label; they are
never merged.  Scoring one session is arithmetic over a few thousand turn boundaries, so it stays in numpy / scipy."""
import math

import numpy as np
from scipy.optimize import linear_sum_assignment

__all__ = ['load_rttm', 'write_rttm', 'DiarizationErrorRate']


def load_rttm(path):
    """-> {uri: [(start, end, label), ...]} in file order, as pyannote.database.util.load_rttm reads it: the whitespace-separated
    ``SPEAKER`` lines, field 1 the uri, field 3 the start, field 4 the duration, field 7 the label (further fields are ignored).
    Other record types and blank lines are skipped; turns of zero duration are dropped (pyannote's Annotation skips empty segments),
    but their uri is still listed.  A malformed SPEAKER line or a negative duration raises ValueError with the line number."""
    out = {}
    with open(path, 'r', encoding='utf-8') as f:
        for n, line in enumerate(f, 1):
            fields = line.split()
            if not fields or fields[0] != 'SPEAKER':
                continue
            if len(fields) < 8:
                raise ValueError(f'{path}:{n}: a SPEAKER line needs at least 8 fields (type uri channel start duration ortho stype '
                                 f'label), got {len(fields)}')
            try:
                start, duration = float(fields[3]), float(fields[4])
            except ValueError:
                raise ValueError(f'{path}:{n}: start {fields[3]!r} or duration {fields[4]!r} is not a number') from None
            if not (math.isfinite(start) and math.isfinite(duration)):
                raise ValueError(f'{path}:{n}: start {fields[3]!r} and duration {fields[4]!r} must be finite')
            if duration < 0:
                raise ValueError(f'{path}:{n}: negative duration {fields[4]!r}')
            turns = out.setdefault(fields[1], [])
            if duration > 0:
                turns.append((start, start + duration, fields[7]))
    return out


def _check_token(kind, value):
    text = str(value)
    if not text or any(c.isspace() for c in text):
        raise ValueError(f'RTTM {kind} {text!r} is empty or contains whitespace: the line could not be read back')
    return text


def write_rttm(f, uri, segments):
    """Writes one session to the text file ``f`` in pyannote's ``Annotation.to_rttm()`` format, one line per turn sorted by
    (start, end): ``SPEAKER {uri} 1 {start:.3f} {duration:.3f} <NA> <NA> {label} <NA> <NA>``.  Turns of zero duration are skipped
    (an Annotation cannot hold them); a uri or label that is empty or contains whitespace is refused."""
    uri = _check_token('uri', uri)
    rows = []
    for start, end, label in segments:
        start, end = float(start), float(end)
        if not end >= start:
            raise ValueError(f'turn ({start}, {end}, {label!r}) ends before it starts')
        rows.append((start, end, _check_token('label', label)))
    rows.sort(key=lambda r: (r[0], r[1]))
    for start, end, label in rows:
        if end > start:
            f.write(f'SPEAKER {uri} 1 {start:.3f} {end - start:.3f} <NA> <NA> {label} <NA> <NA>\n')


def _turns(annotation, name):
    """-> (starts, ends, label ids, label list) of the non-empty turns."""
    starts, ends, ids, labels, index = [], [], [], [], {}
    for start, end, label in annotation:
        start, end = float(start), float(end)
        if not (math.isfinite(start) and math.isfinite(end)) or end < start:
            raise ValueError(f'{name} turn ({start}, {end}, {label!r}) is not a finite interval')
        if end == start:
            continue
        if label not in index:
            index[label] = len(labels)
            labels.append(label)
        starts.append(start)
        ends.append(end)
        ids.append(index[label])
    return np.array(starts, np.float64), np.array(ends, np.float64), np.array(ids, np.int64), labels


def _union(starts, ends):
    """Disjoint sorted [(a, b), ...] covering the union of the intervals."""
    out = []
    for a, b in sorted(zip(starts.tolist(), ends.tolist())):
        if b <= a:
            continue
        if out and a <= out[-1][1]:
            out[-1][1] = max(out[-1][1], b)
        else:
            out.append([a, b])
    return out


def _overlap_regions(starts, ends):
    """[(a, b), ...] where two or more of the intervals overlap (a sweep over the sorted boundaries)."""
    events = sorted([(t, 1) for t in starts.tolist()] + [(t, -1) for t in ends.tolist()], key=lambda e: (e[0], e[1]))
    out, depth, open_at = [], 0, None
    for t, step in events:  # ends sort before starts at equal times: touching turns do not overlap
        depth += step
        if depth >= 2 and open_at is None:
            open_at = t
        elif depth < 2 and open_at is not None:
            if t > open_at:
                out.append((open_at, t))
            open_at = None
    return out


def _evaluated_region(ref, hyp, collar, skip_overlap):
    """The union extent of both annotations, less [b - collar/2, b + collar/2] around every reference boundary b and, with
    skip_overlap, the reference's overlap regions -> disjoint sorted [(a, b), ...]."""
    starts = np.concatenate([ref[0], hyp[0]])
    ends = np.concatenate([ref[1], hyp[1]])
    if starts.size == 0:
        return []
    lo, hi = float(starts.min()), float(ends.max())
    removed_a, removed_b = [], []
    if collar > 0:
        bounds = np.unique(np.concatenate([ref[0], ref[1]]))
        removed_a.append(bounds - 0.5 * collar)
        removed_b.append(bounds + 0.5 * collar)
    if skip_overlap:
        regions = _overlap_regions(ref[0], ref[1])
        removed_a.append(np.array([a for a, _ in regions], np.float64))
        removed_b.append(np.array([b for _, b in regions], np.float64))
    region, t = [], lo
    if removed_a:
        for a, b in _union(np.concatenate(removed_a), np.concatenate(removed_b)):
            if a > t:
                region.append((t, min(a, hi)))
            t = max(t, b)
            if t >= hi:
                break
    if t < hi:
        region.append((t, hi))
    return [(a, b) for a, b in region if b > a]


def _crop(turns, region):
    """The turns intersected with each interval of the region (a turn cut by a removed stretch becomes several pieces)."""
    starts, ends, ids, labels = turns
    if not region or starts.size == 0:
        return np.zeros(0), np.zeros(0), np.zeros(0, np.int64), labels
    ra = np.array([a for a, _ in region])
    rb = np.array([b for _, b in region])
    s = np.maximum(starts[:, None], ra[None, :])
    e = np.minimum(ends[:, None], rb[None, :])
    keep = e > s
    return s[keep], e[keep], np.broadcast_to(ids[:, None], keep.shape)[keep], labels


def _counts(turns, bounds):
    """[labels, segments] number of turns of each label covering each elementary segment [bounds[i], bounds[i + 1])."""
    starts, ends, ids, labels = turns
    diff = np.zeros((len(labels), bounds.size), np.int64)
    np.add.at(diff, (ids, np.searchsorted(bounds, starts)), 1)
    np.add.at(diff, (ids, np.searchsorted(bounds, ends)), -1)
    return np.cumsum(diff, axis=1)[:, :-1]


class DiarizationErrorRate:
    """Diarization error rate after pyannote.metrics 3.x's ``DiarizationErrorRate(collar, skip_overlap)`` with no UEM.

    Per call, on reference and hypothesis annotations ``[(start_s, end_s, label), ...]``:
      * evaluated region: the extent of the union of both annotations (pyannote's approximation when no UEM is given), less
        ``[b - collar/2, b + collar/2]`` around every reference boundary ``b`` (collar > 0) and, with ``skip_overlap``, less every
        region where two or more reference turns overlap; both annotations are cropped to it;
      * speaker mapping: the co-occurrence matrix of total overlap per (reference label, hypothesis label), summed over pairs of turns,
        is solved by ``scipy.optimize.linear_sum_assignment`` (maximising); only pairs with co-occurrence > 0 are mapped, and an
        unmapped hypothesis label never matches;
      * on each elementary segment of the union of both boundary sets, of duration ``dur``, with ``r`` / ``h`` the multisets of
        reference / mapped hypothesis labels active there (turns are not merged, so two overlapping turns of one label count twice):
        total += dur·|r|, correct += dur·|r ∩ h|, confusion += dur·(min(|r|, |h|) − |r ∩ h|), missed detection += dur·max(0, |r| − |h|),
        false alarm += dur·max(0, |h| − |r|);
      * rate = (false alarm + missed detection + confusion) / total, and when total is 0: 0 if the numerator is 0, else 1.  That last
        rule is recalled from pyannote's ``compute_metric``, not checked against it.

    Ties: where no label's turns overlap each other in either annotation, correct = Σ co-occurrence of the mapped pairs, so every
    optimal assignment gives the same correct duration -- and total, false alarm and missed detection do not depend on the mapping
    at all -- hence the same rate, however ``linear_sum_assignment`` breaks ties.  Where a label overlaps itself, |r ∩ h| counts
    min(#r, #h) while the co-occurrence counts #r·#h, and tied assignments may then score differently, as in pyannote.

    ``metric(reference, hypothesis, detailed=False)`` returns the rate, or with ``detailed=True`` a dict with pyannote's keys
    ('diarization error rate', 'false alarm', 'missed detection', 'confusion', 'correct', 'total'; durations in seconds).  Every call
    also accumulates its components: ``abs(metric)`` is the corpus rate Σ errors / Σ total, and ``reset()`` clears it."""

    COMPONENTS = ('false alarm', 'missed detection', 'confusion', 'correct', 'total')
    NAME = 'diarization error rate'

    def __init__(self, collar=0.0, skip_overlap=False):
        if not collar >= 0:
            raise ValueError(f'collar must be >= 0 seconds, got {collar}')
        self.collar = float(collar)
        self.skip_overlap = bool(skip_overlap)
        self.reset()

    def reset(self):
        self.accumulated_ = dict.fromkeys(self.COMPONENTS, 0.0)

    @staticmethod
    def rate(components):
        errors = components['false alarm'] + components['missed detection'] + components['confusion']
        if components['total'] == 0:
            return 0.0 if errors == 0 else 1.0
        return errors / components['total']

    def compute_components(self, reference, hypothesis):
        """-> {component: seconds} of one session (nothing is accumulated)."""
        ref, hyp = _turns(reference, 'reference'), _turns(hypothesis, 'hypothesis')
        region = _evaluated_region(ref, hyp, self.collar, self.skip_overlap)
        ref, hyp = _crop(ref, region), _crop(hyp, region)
        bounds = np.unique(np.concatenate([ref[0], ref[1], hyp[0], hyp[1]]))
        out = dict.fromkeys(self.COMPONENTS, 0.0)
        if bounds.size < 2:
            return out
        dur = np.diff(bounds)
        rc, hc = _counts(ref, bounds), _counts(hyp, bounds)
        matched = np.zeros(dur.size, np.int64)
        if rc.shape[0] and hc.shape[0]:
            cooccurrence = (rc * dur) @ hc.T.astype(np.float64)
            rows, cols = linear_sum_assignment(cooccurrence, maximize=True)
            for r, h in zip(rows, cols):
                if cooccurrence[r, h] > 0:
                    matched += np.minimum(rc[r], hc[h])
        nr, nh = rc.sum(axis=0), hc.sum(axis=0)
        out['total'] = float(dur @ nr)
        out['correct'] = float(dur @ matched)
        out['confusion'] = float(dur @ (np.minimum(nr, nh) - matched))
        out['missed detection'] = float(dur @ np.maximum(0, nr - nh))
        out['false alarm'] = float(dur @ np.maximum(0, nh - nr))
        return out

    def __call__(self, reference, hypothesis, detailed=False):
        components = self.compute_components(reference, hypothesis)
        for k in self.COMPONENTS:
            self.accumulated_[k] += components[k]
        components[self.NAME] = self.rate(components)
        return components if detailed else components[self.NAME]

    def __abs__(self):
        return self.rate(self.accumulated_)
