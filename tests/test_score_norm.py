"""CPU: the AS-norm oracle (tests/score_norm_oracle.py) on a hand-worked example with ties at the cut, against the S-norm closed form
at top_n == cohort size, under permutation of the cohort, and the parsing of the ``dataset_conf.eval_conf.score_norm`` key."""
import numpy as np
import pytest

import score_norm_oracle as so
from ppvector.metric.score_norm import score_norm_config


def test_hand_worked_ties_at_the_cut():
    # top 3 of the row: 0.9 and two of the three 0.7s -- the tie at the cut counts with multiplicity
    row = np.array([[0.5, 0.9, 0.7, 0.7, 0.7, 0.1]])
    mean, std = so.topn_stats(row, 3)
    assert mean[0] == pytest.approx(2.3 / 3, abs=1e-15)
    # deviations 2/15, -1/15, -1/15: sum of squares 6/225, over top_n - 1 = 2
    assert std[0] == pytest.approx(np.sqrt(1 / 75), abs=1e-15)
    # top 4 takes all three 0.7s: mean 3.0 / 4, deviations 0.15, -0.05 x 3
    mean, std = so.topn_stats(row, 4)
    assert mean[0] == pytest.approx(0.75, abs=1e-15)
    assert std[0] == pytest.approx(np.sqrt((0.15 ** 2 + 3 * 0.05 ** 2) / 3), abs=1e-15)
    # a constant top set: the spread floors at 1e-6
    mean, std = so.topn_stats(np.array([[0.3, 0.7, 0.7, 0.7]]), 3)
    assert mean[0] == pytest.approx(0.7, abs=1e-15) and std[0] == so.STD_FLOOR


def test_full_cohort_is_s_norm():
    rng = np.random.default_rng(0)
    T, E, C = rng.normal(size=(7, 16)), rng.normal(size=(5, 16)), rng.normal(size=(40, 16))
    ct, ce = so.cosine(T, C), so.cosine(E, C)
    t_stats, e_stats = so.topn_stats(ct, 40), so.topn_stats(ce, 40)
    np.testing.assert_allclose(t_stats[0], ct.mean(axis=1), rtol=0, atol=1e-15)
    np.testing.assert_allclose(t_stats[1], ct.std(axis=1, ddof=1), rtol=1e-13)
    np.testing.assert_allclose(e_stats[1], ce.std(axis=1, ddof=1), rtol=1e-13)
    s = so.cosine(T, E)
    snorm = 0.5 * ((s - ce.mean(1)[None]) / ce.std(1, ddof=1)[None] + (s - ct.mean(1)[:, None]) / ct.std(1, ddof=1)[:, None])
    np.testing.assert_allclose(so.as_norm(s, t_stats, e_stats), snorm, rtol=1e-12, atol=1e-12)


def test_cohort_permutation_invariance():
    rng = np.random.default_rng(1)
    Q, C = rng.normal(size=(9, 32)), rng.normal(size=(200, 32))
    C[17] = C[3]  # duplicated cohort rows: equal scores
    perm = rng.permutation(200)
    a = so.cohort_stats(Q, C, 50)
    b = so.cohort_stats(Q, C[perm], 50)
    np.testing.assert_allclose(a[0], b[0], rtol=0, atol=1e-14)
    np.testing.assert_allclose(a[1], b[1], rtol=0, atol=1e-14)
    labels = rng.integers(0, 20, size=200)
    np.testing.assert_allclose(so.speaker_cohort(C, labels), so.speaker_cohort(C[perm], labels[perm]), rtol=1e-6, atol=1e-7)


def test_config_parsing():
    assert score_norm_config(None) is None
    assert score_norm_config({'cohort_list': 'c.txt'}) == {'cohort_list': 'c.txt', 'top_n': 300, 'cohort': 'speaker'}
    assert score_norm_config({'cohort_list': 'c.txt', 'top_n': 2, 'cohort': 'utterance'}) == \
        {'cohort_list': 'c.txt', 'top_n': 2, 'cohort': 'utterance'}
    for bad in ('c.txt', {}, {'cohort_list': ''}, {'cohort_list': None}, {'cohort_list': 'c.txt', 'top_n': 1},
                {'cohort_list': 'c.txt', 'top_n': 2.5}, {'cohort_list': 'c.txt', 'top_n': True}, {'cohort_list': 'c.txt', 'top_n': '300'},
                {'cohort_list': 'c.txt', 'cohort': 'speakers'}, {'cohort_list': 'c.txt', 'topn': 300}):
        with pytest.raises(ValueError):
            score_norm_config(bad)
