"""Scoring and verification metrics: cosine scoring on the GPU (cosine.py), EER / minDCF on the host (metrics.py), and the
diarization error rate with RTTM I/O on the host (der.py)."""
