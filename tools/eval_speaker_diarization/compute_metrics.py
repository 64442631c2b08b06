"""Step 3 of the diarization evaluation: score the hypothesis RTTM (infer_data.py) against the reference RTTM
(create_test_rttm.py) with the diarization error rate of ppvector.metric.der.

Prints each session's result, then the reference's four averages over sessions (mean false-alarm, confusion and missed-detection
seconds, and the mean of the per-session rates), then the corpus rate: all sessions' errors over all their reference speech.  A
session missing from the hypotheses is scored against an empty hypothesis.  Run from this directory; the default paths are the
reference's.

    python compute_metrics.py [--references dataset/references.rttm] [--hypotheses dataset/hypotheses.rttm]
"""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path[:0] = [ROOT, os.path.join(ROOT, 'voiceprintrecognition-paddlepaddle_b200')]

from cli_common import parse_options  # noqa: E402

OPTIONS = [
    ('references', str, 'dataset/references.rttm', 'reference RTTM'),
    ('hypotheses', str, 'dataset/hypotheses.rttm', 'hypothesis RTTM'),
]


def evaluate(references_path, hypotheses_path):
    """-> ([(uri, detailed result), ...] in reference order, the four averages over sessions, corpus rate)."""
    from ppvector.metric.der import DiarizationErrorRate, load_rttm
    metric = DiarizationErrorRate()
    references, hypotheses = load_rttm(references_path), load_rttm(hypotheses_path)
    results = [(uri, metric(reference, hypotheses.get(uri, []), detailed=True)) for uri, reference in references.items()]
    averages = {key: sum(r[key] for _, r in results) / len(results) if results else 0.0
                for key in ('false alarm', 'confusion', 'missed detection', 'diarization error rate')}
    return results, averages, abs(metric)


def main(opt):
    results, averages, corpus = evaluate(opt.references, opt.hypotheses)
    for uri, result in results:
        print(uri, ':', result)
    print('False alarm:', round(averages['false alarm'], 5))
    print('Confusion:', round(averages['confusion'], 5))
    print('Missed detection:', round(averages['missed detection'], 5))
    print('Diarization error rate:', round(averages['diarization error rate'], 5))
    print('Corpus diarization error rate:', round(corpus, 5))


if __name__ == '__main__':
    main(parse_options(__doc__, OPTIONS))
