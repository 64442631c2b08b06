"""Diarization error rate and RTTM I/O (ppvector/metric/der.py) on the host: seeded random annotations against the brute-force 1 ms
grid oracle (tests/der_oracle.py) at every collar / skip_overlap setting, hand cases with known answers, tie-breaking, corpus
accumulation, compute_metrics.py's averages, RTTM round trips and refusals, and the --rttm_path option of the diarization CLI."""
import io
import os
import re
import subprocess
import sys

import numpy as np
import pytest

from der_oracle import der_components_ms
from ppvector.metric import der
from ppvector.metric.der import DiarizationErrorRate, load_rttm, write_rttm

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
KEYS = ('false alarm', 'missed detection', 'confusion', 'correct', 'total')


def random_annotation_ms(rng, labels, span_ms, n_turns):
    """Turns on a 1 ms grid; some labels get a second turn overlapping one of their own."""
    turns = []
    for _ in range(n_turns):
        a = int(rng.integers(0, span_ms))
        turns.append((a, a + int(rng.integers(1, 3000)), labels[int(rng.integers(len(labels)))]))
    for _ in range(int(rng.integers(0, 3)) if turns else 0):
        a, b, lab = turns[int(rng.integers(len(turns)))]
        c = int(rng.integers(a, b))
        turns.append((c, c + int(rng.integers(1, 1500)), lab))
    return turns


def random_case(seed):
    """A reference of up to 5 speakers and a hypothesis of up to 6: either independent turns, or the reference's turns with moved
    boundaries, relabelled, with some dropped and some spurious ones; the hypothesis may run past the reference."""
    rng = np.random.default_rng(seed)
    rl = [f'spk{i}' for i in range(int(rng.integers(1, 6)))]
    hl = list(range(int(rng.integers(1, 7))))
    ref = random_annotation_ms(rng, rl, 15000, int(rng.integers(1, 12)))
    if seed % 2:
        hyp = random_annotation_ms(rng, hl, 18000, int(rng.integers(1, 12)))
    else:
        rename = {lab: hl[i % len(hl)] for i, lab in enumerate(rng.permutation(rl))}
        hyp = []
        for a, b, lab in ref:
            if rng.random() < 0.15:
                continue
            a2, b2 = a + int(rng.integers(-300, 301)), b + int(rng.integers(-300, 301))
            if b2 > a2:
                hyp.append((a2, b2, rename[lab] if rng.random() < 0.85 else hl[int(rng.integers(len(hl)))]))
        hyp += random_annotation_ms(rng, hl, 20000, int(rng.integers(0, 3)))
    return ref, hyp


def seconds(turns):
    return [(a / 1000, b / 1000, lab) for a, b, lab in turns]


@pytest.mark.parametrize("skip_overlap", [False, True])
@pytest.mark.parametrize("collar", [0.0, 0.25, 0.5])
def test_random_against_oracle(collar, skip_overlap):
    metric = DiarizationErrorRate(collar=collar, skip_overlap=skip_overlap)
    for seed in range(60):
        ref, hyp = random_case(seed)
        got = metric.compute_components(seconds(ref), seconds(hyp))
        want = der_components_ms(ref, hyp, int(round(collar * 1000)), skip_overlap)
        assert any(all(abs(got[k] - w[k]) <= 1e-9 for k in KEYS) for w in want), (seed, got, want)
        assert got['correct'] + got['confusion'] + got['missed detection'] == pytest.approx(got['total'], abs=1e-9)


def test_oracle_cases_are_not_trivial():
    """The random cases reach overlaps, same-label overlaps, partial matches and a hypothesis past the reference."""
    hits = dict.fromkeys(('same-label overlap', 'confusion', 'false alarm', 'missed', 'past the end'), 0)
    for seed in range(60):
        ref, hyp = random_case(seed)
        c = der_components_ms(ref, hyp)[0]
        hits['confusion'] += c['confusion'] > 0
        hits['false alarm'] += c['false alarm'] > 0
        hits['missed'] += c['missed detection'] > 0
        hits['past the end'] += max(b for _, b, _ in hyp) > max(b for _, b, _ in ref)
        hits['same-label overlap'] += any(l1 == l2 and a1 < b2 and a2 < b1 for i, (a1, b1, l1) in enumerate(ref)
                                          for (a2, b2, l2) in ref[i + 1:])
    assert all(v >= 10 for v in hits.values()), hits


def test_permuted_perfect_hypothesis_scores_zero():
    ref = [(0.0, 2.0, 'A'), (2.0, 5.5, 'B'), (5.5, 6.0, 'A'), (7.0, 9.0, 'C'), (8.0, 9.5, 'A')]
    hyp = [(a, b, {'A': 'x', 'B': 'y', 'C': 'z'}[lab]) for a, b, lab in ref[::-1]]
    for collar in (0.0, 0.5):
        for skip in (False, True):
            d = DiarizationErrorRate(collar, skip)(ref, hyp, detailed=True)
            assert d['diarization error rate'] == 0.0 and d['correct'] == pytest.approx(d['total']) and d['total'] > 0


def test_empty_cases():
    ref = [(0.0, 2.0, 'A'), (3.0, 4.0, 'B')]
    d = DiarizationErrorRate()(ref, [], detailed=True)
    assert d['diarization error rate'] == 1.0 and d['missed detection'] == pytest.approx(3.0) and d['total'] == pytest.approx(3.0)
    d = DiarizationErrorRate()([], [], detailed=True)
    assert d == {**dict.fromkeys(KEYS, 0.0), 'diarization error rate': 0.0}
    d = DiarizationErrorRate()([], [(1.0, 2.5, 0)], detailed=True)
    assert d['diarization error rate'] == 1.0 and d['false alarm'] == pytest.approx(1.5) and d['total'] == 0.0


def test_split_speaker_confusion_is_the_shorter_part():
    d = DiarizationErrorRate()([(0.0, 10.0, 'A')], [(0.0, 7.0, 0), (7.0, 10.0, 1)], detailed=True)
    assert d['confusion'] == pytest.approx(3.0) and d['correct'] == pytest.approx(7.0)
    assert d['missed detection'] == 0.0 and d['false alarm'] == 0.0 and d['diarization error rate'] == pytest.approx(0.3)


def test_reference_overlap_under_one_speaker_is_missed():
    d = DiarizationErrorRate()([(0.0, 7.0, 'A'), (5.0, 10.0, 'B')], [(0.0, 10.0, 0)], detailed=True)
    assert d['missed detection'] == pytest.approx(2.0) and d['total'] == pytest.approx(12.0)
    assert d['confusion'] == pytest.approx(3.0) and d['correct'] == pytest.approx(7.0)
    # skip_overlap leaves the overlap out: nothing is missed
    d = DiarizationErrorRate(skip_overlap=True)([(0.0, 7.0, 'A'), (5.0, 10.0, 'B')], [(0.0, 10.0, 0)], detailed=True)
    assert d['missed detection'] == 0.0 and d['total'] == pytest.approx(8.0)


def test_collar_removes_boundary_neighbourhoods():
    # every boundary error is within 0.1 s of a reference boundary: a 0.25 s collar forgives them all
    ref = [(1.0, 4.0, 'A'), (4.0, 6.0, 'B')]
    hyp = [(0.9, 4.1, 0), (4.1, 6.05, 1)]
    assert DiarizationErrorRate()(ref, hyp) > 0
    d = DiarizationErrorRate(collar=0.25)(ref, hyp, detailed=True)
    assert d['diarization error rate'] == 0.0 and d['total'] == pytest.approx(5.0 - 2 * 0.25)


def _forced_assignment(monkeypatch, pick):
    """Make der's linear_sum_assignment return pick(matrix) instead of scipy's choice."""
    monkeypatch.setattr(der, 'linear_sum_assignment', lambda m, maximize: pick(np.asarray(m)))


def test_tied_cooccurrence_gives_the_same_rate(monkeypatch):
    """A co-occurrence matrix of equal entries: both assignments are optimal and score the same."""
    ref = [(0.0, 2.0, 'A'), (2.0, 4.0, 'B'), (6.0, 7.0, 'C')]
    hyp = [(0.0, 1.0, 'x'), (2.0, 3.0, 'x'), (1.0, 2.0, 'y'), (3.0, 4.0, 'y')]
    results = []
    for pick in (lambda m: (np.array([0, 1]), np.array([0, 1])), lambda m: (np.array([0, 1]), np.array([1, 0]))):
        with monkeypatch.context() as mp:
            _forced_assignment(mp, pick)
            results.append(DiarizationErrorRate()(ref, hyp, detailed=True))
    assert results[0] == results[1]
    assert results[0]['correct'] == pytest.approx(2.0) and results[0]['confusion'] == pytest.approx(2.0)
    assert results[0]['missed detection'] == pytest.approx(1.0)


def test_ties_matter_only_where_a_label_overlaps_itself(monkeypatch):
    """Where a label's turns overlap each other, |r ∩ h| counts min(#r, #h) but the co-occurrence #r·#h, so tied assignments can
    score differently (as in pyannote): the oracle finds both results, and either assignment gives one of them."""
    ref = [(0.0, 1.0, 'A'), (0.0, 1.0, 'A'), (5.0, 7.0, 'A'), (1.0, 3.0, 'B'), (8.0, 10.0, 'B')]
    hyp = [(0.0, 1.0, 'x'), (8.0, 10.0, 'x'), (1.0, 3.0, 'y'), (5.0, 7.0, 'y')]
    ms = [(int(a * 1000), int(b * 1000), lab) for a, b, lab in ref], [(int(a * 1000), int(b * 1000), lab) for a, b, lab in hyp]
    want = der_components_ms(*ms)
    assert sorted(w['correct'] for w in want) == [3.0, 4.0]
    for pick in (lambda m: (np.array([0, 1]), np.array([0, 1])), lambda m: (np.array([0, 1]), np.array([1, 0]))):
        with monkeypatch.context() as mp:
            _forced_assignment(mp, pick)
            got = DiarizationErrorRate().compute_components(ref, hyp)
        assert any(all(abs(got[k] - w[k]) <= 1e-9 for k in KEYS) for w in want)


def test_accumulation_is_the_corpus_rate():
    metric = DiarizationErrorRate(collar=0.25)
    errors = total = 0.0
    for seed in range(5):
        ref, hyp = random_case(100 + seed)
        d = metric(seconds(ref), seconds(hyp), detailed=True)
        errors += d['false alarm'] + d['missed detection'] + d['confusion']
        total += d['total']
    assert abs(metric) == pytest.approx(errors / total, rel=1e-12)
    for k in KEYS:
        assert metric.accumulated_[k] > 0
    metric.reset()
    assert abs(metric) == 0.0 and all(v == 0.0 for v in metric.accumulated_.values())


def test_refuses_bad_input():
    with pytest.raises(ValueError, match='collar'):
        DiarizationErrorRate(collar=-0.1)
    with pytest.raises(ValueError, match='not a finite interval'):
        DiarizationErrorRate()([(2.0, 1.0, 'A')], [])


# ---- RTTM --------------------------------------------------------------------------------------------------------------------------
def test_rttm_round_trip(tmp_path):
    rng = np.random.default_rng(5)
    sessions = {}
    for uri in ('sess_a', 'S02-meeting'):
        starts = rng.uniform(0, 600, size=200)
        sessions[uri] = [(float(a), float(a + d), f'spk{int(k)}') for a, d, k in
                         zip(starts, rng.uniform(0.01, 20, size=200), rng.integers(0, 7, size=200))]
    path = tmp_path / 'x.rttm'
    with open(path, 'w') as f:
        for uri, segs in sessions.items():
            write_rttm(f, uri, segs)
    lines = path.read_text().splitlines()
    assert len(lines) == 400 and re.fullmatch(r'SPEAKER sess_a 1 \d+\.\d{3} \d+\.\d{3} <NA> <NA> spk\d <NA> <NA>', lines[0])
    back = load_rttm(path)
    assert list(back) == list(sessions)
    for uri, segs in sessions.items():
        want = sorted(segs, key=lambda s: (s[0], s[1]))
        assert [s[2] for s in back[uri]] == [s[2] for s in want]
        assert np.abs(np.array([s[:2] for s in back[uri]]) - np.array([s[:2] for s in want])).max() <= 1e-3 + 1e-9
        assert [s[0] for s in back[uri]] == sorted(s[0] for s in back[uri])


def test_write_rttm_format():
    f = io.StringIO()
    write_rttm(f, 'rec', [(2.0, 3.25, 1), (0.5, 1.0, 'spk0'), (0.5, 0.75, 'spk1'), (4.0, 4.0, 'empty')])
    assert f.getvalue() == ('SPEAKER rec 1 0.500 0.250 <NA> <NA> spk1 <NA> <NA>\n'
                            'SPEAKER rec 1 0.500 0.500 <NA> <NA> spk0 <NA> <NA>\n'
                            'SPEAKER rec 1 2.000 1.250 <NA> <NA> 1 <NA> <NA>\n')


def test_load_rttm_pyannote_lines(tmp_path):
    path = tmp_path / 'refs.rttm'
    path.write_text(
        ';; a comment\n'
        'SPKR-INFO L_R003S01C02 1 <NA> <NA> <NA> unknown 004 <NA>\n'
        '\n'
        'SPEAKER L_R003S01C02 1 12.01 3.5 <NA> <NA> 004 <NA> <NA>\n'
        'SPEAKER L_R003S01C02 1 0.120 1.000 <NA> <NA> 003 0.97 <NA> extra-column\n'
        '  SPEAKER\tL_R003S01C02  1  20  0  <NA>  <NA>  005  <NA>  <NA>  \n'
        'SPEAKER other 1 1 0 <NA> <NA> A <NA> <NA>\n'
        'NON-SPEECH L_R003S01C02 1 5.0 1.0 <NA> <NA> <NA> <NA> <NA>\n')
    back = load_rttm(path)
    assert back == {'L_R003S01C02': [(12.01, 15.51, '004'), (0.12, 1.12, '003')], 'other': []}


@pytest.mark.parametrize("line,match", [
    ('SPEAKER rec 1 0.5 1.0 <NA> <NA>', 'line|:2:'),
    ('SPEAKER rec 1 zero 1.0 <NA> <NA> A <NA> <NA>', 'not a number'),
    ('SPEAKER rec 1 0.5 nan <NA> <NA> A <NA> <NA>', 'finite'),
    ('SPEAKER rec 1 0.5 -0.1 <NA> <NA> A <NA> <NA>', 'negative duration'),
])
def test_load_rttm_refuses(tmp_path, line, match):
    path = tmp_path / 'bad.rttm'
    path.write_text('SPEAKER rec 1 0.0 0.5 <NA> <NA> A <NA> <NA>\n' + line + '\n')
    with pytest.raises(ValueError, match=match) as e:
        load_rttm(path)
    assert ':2:' in str(e.value)


@pytest.mark.parametrize("uri,label", [('my rec', 'A'), ('rec', 'spk 1'), ('rec', 'a\tb'), ('', 'A'), ('rec', '')])
def test_write_rttm_refuses_whitespace(uri, label):
    with pytest.raises(ValueError, match='whitespace'):
        write_rttm(io.StringIO(), uri, [(0.0, 1.0, label)])


def test_write_rttm_refuses_reversed_turn():
    with pytest.raises(ValueError, match='ends before'):
        write_rttm(io.StringIO(), 'rec', [(1.0, 0.5, 'A')])


# ---- tools/eval_speaker_diarization/compute_metrics.py -----------------------------------------------------------------------------
def test_compute_metrics_averages(tmp_path):
    """Two sessions (one missing from the hypotheses): the printed averages are the reference's mean-over-files formulas and the last
    line is the corpus rate."""
    refs = {'s1': [(0.0, 4.0, 'A'), (4.0, 9.0, 'B'), (8.5, 10.0, 'A')], 's2': [(0.5, 3.0, 'C'), (3.0, 6.0, 'D')], 's3': [(0.0, 2.0, 'E')]}
    hyps = {'s1': [(0.0, 4.2, 0), (4.2, 10.0, 1)], 's2': [(0.0, 2.0, 0), (2.0, 6.5, 0), (6.5, 7.0, 1)]}
    os.makedirs(tmp_path / 'dataset')  # the tool's default paths, relative to where it runs
    for name, sessions in (('references.rttm', refs), ('hypotheses.rttm', hyps)):
        with open(tmp_path / 'dataset' / name, 'w') as f:
            for uri, segs in sessions.items():
                write_rttm(f, uri, segs)
    r = subprocess.run([sys.executable, os.path.join(ROOT, 'tools', 'eval_speaker_diarization', 'compute_metrics.py')],
                       capture_output=True, text=True, cwd=tmp_path, timeout=120)
    assert r.returncode == 0, r.stdout + r.stderr
    printed = dict(re.findall(r'^([A-Za-z ]+): (\S+)$', r.stdout, flags=re.M))
    metric = DiarizationErrorRate()
    per_file = [metric(refs[u], hyps.get(u, []), detailed=True) for u in refs]
    for label, key in (('False alarm', 'false alarm'), ('Confusion', 'confusion'), ('Missed detection', 'missed detection'),
                       ('Diarization error rate', 'diarization error rate')):
        assert float(printed[label]) == round(sum(d[key] for d in per_file) / 3, 5), label
    errors = sum(d['false alarm'] + d['missed detection'] + d['confusion'] for d in per_file)
    assert float(printed['Corpus diarization error rate']) == round(errors / sum(d['total'] for d in per_file), 5)
    assert per_file[2]['diarization error rate'] == 1.0  # s3 has no hypothesis: all of it is missed
    for uri in refs:
        assert re.search(rf'^{uri} : \{{', r.stdout, flags=re.M)


# ---- infer_speaker_diarization.py --rttm_path ----------------------------------------------------------------------------------------
def test_cli_rttm_path_option():
    import cli_common
    import infer_speaker_diarization as cli
    assert 'rttm_path' not in {r[0] for r in cli.OPTIONS}
    row = [r for r in cli.EXTENSION_OPTIONS if r[0] == 'rttm_path']
    assert len(row) == 1 and row[0][1] is str and row[0][2] is None
    table = cli.OPTIONS + cli.EXTENSION_OPTIONS
    assert cli_common.parse_options('x', table, ['--rttm_path', 'out/h.rttm']).rttm_path == 'out/h.rttm'
    assert cli_common.parse_options('x', table, []).rttm_path is None
