"""Adaptive symmetric score normalisation (AS-norm) of verification scores against a cohort, on the GPU (libppv_b200:
ppv_topn_row_stats / ppv_as_norm_apply).  The reference has no score normalisation; the definition follows the usual AS-norm of
speaker-verification evaluations:

- for a query row q (a trial or an enrolment) S_q is the multiset of its ``top_n`` largest cosines against the cohort rows (ties by
  value: equal scores at the cut count with multiplicity); mean_q = mean(S_q), std_q = sqrt(sum((x - mean_q)^2) / (top_n - 1)),
  floored at 1e-6;
- s'(t, e) = ((s - mean_e) / std_e + (s - mean_t) / std_t) / 2.  With ``top_n`` equal to the cohort size this is plain S-norm.

``cohort_stats`` scores the queries chunk by chunk against the cohort (``ppv_cosine_matrix``) into a buffer of at most ``max_ws_bytes``
and takes each chunk's statistics before the next, so the [queries x cohort] matrix is never held whole.  ``score_norm_config`` reads
the optional ``dataset_conf.eval_conf.score_norm`` key of ``PPVectorTrainer.evaluate``.
"""
import ctypes as C

import numpy as np

from ppvector import _lib

COHORT_MODES = ('speaker', 'utterance')
DEFAULT_TOP_N = 300
DEFAULT_MAX_WS_BYTES = 1 << 30


def score_norm_config(conf):
    """``eval_conf.score_norm`` -> None when absent, else a dict {cohort_list, top_n, cohort} with the defaults filled in.  Raises
    ValueError on an unknown key, a missing or empty ``cohort_list``, ``top_n`` that is not an integer >= 2, or an unknown cohort."""
    if conf is None:
        return None
    if not isinstance(conf, dict):
        raise ValueError(f'score_norm: expected a mapping {{cohort_list, top_n, cohort}}, got {conf!r}')
    unknown = set(conf) - {'cohort_list', 'top_n', 'cohort'}
    if unknown:
        raise ValueError(f'score_norm: unknown key(s) {sorted(unknown)}; allowed: cohort_list, top_n, cohort')
    cohort_list = conf.get('cohort_list')
    if not isinstance(cohort_list, str) or not cohort_list:
        raise ValueError(f'score_norm.cohort_list: a list file path is required, got {cohort_list!r}')
    top_n = conf.get('top_n', DEFAULT_TOP_N)
    if isinstance(top_n, bool) or not isinstance(top_n, (int, np.integer)) or top_n < 2:
        raise ValueError(f'score_norm.top_n: an integer >= 2 is required, got {top_n!r}')
    cohort = conf.get('cohort', 'speaker')
    if cohort not in COHORT_MODES:
        raise ValueError(f'score_norm.cohort: one of {COHORT_MODES}, got {cohort!r}')
    return {'cohort_list': cohort_list, 'top_n': int(top_n), 'cohort': cohort}


def speaker_cohort(emb, labels):
    """emb [n, D], labels [n] -> [U, D] float32 CUDA tensor: one row per distinct label (ascending), the mean of that label's
    embeddings in list order (the speaker index's means: bitwise numpy's emb[rows].mean(axis=0))."""
    import torch

    from ppvector.infer_utils.speaker_index import SpeakerIndex
    labels = labels.cpu().numpy() if torch.is_tensor(labels) else np.asarray(labels)
    _, uid = np.unique(labels, return_inverse=True)
    num = int(uid.max()) + 1 if uid.size else 0
    device = emb.device if torch.is_tensor(emb) and emb.is_cuda else torch.device('cuda', torch.cuda.current_device())
    return SpeakerIndex(emb, uid.reshape(-1), num, device=device).means


def topn_row_stats(scores, top_n, mean=None, std=None):
    """scores [rows, cols] float32 CUDA tensor (rows may be strided: unit column stride, any row stride >= cols) -> (mean [rows],
    std [rows]) of each row's ``top_n`` largest values."""
    import torch
    _lib.require_cuda(scores, 'scores')
    if scores.dtype != torch.float32 or scores.dim() != 2 or scores.stride(1) != 1:
        raise _lib.PPVError(f'topn_row_stats: scores must be a 2-D float32 tensor with unit column stride, got {scores.dtype} '
                            f'{tuple(scores.shape)} strides {scores.stride()}')
    rows, cols = scores.shape
    mean = torch.empty(rows, dtype=torch.float32, device=scores.device) if mean is None else mean
    std = torch.empty(rows, dtype=torch.float32, device=scores.device) if std is None else std
    with torch.cuda.device(scores.device):
        _lib.check(_lib.load().ppv_topn_row_stats(C.c_void_p(scores.data_ptr()), rows, cols, max(scores.stride(0), cols), int(top_n),
                                                  _lib.ptr(mean), _lib.ptr(std), _lib.current_stream()), 'ppv_topn_row_stats')
    return mean, std


def cohort_stats(emb, cohort, top_n=DEFAULT_TOP_N, max_ws_bytes=DEFAULT_MAX_WS_BYTES):
    """emb [Q, D] query embeddings, cohort [Nc, D] cohort rows -> (mean [Q], std [Q]) float32 CUDA tensors: the statistics of each
    query's ``top_n`` highest cosines against the cohort.  Queries are scored in chunks whose [chunk, Nc] fp32 score buffer takes at
    most ``max_ws_bytes`` (at least one row); the cosine planes of the chunk and the cohort come on top, O((chunk + Nc) * D)."""
    import torch

    from ppvector.metric.cosine import _prep
    emb = _prep(emb)
    cohort = _prep(cohort, emb.device)
    if emb.dim() != 2 or cohort.dim() != 2 or emb.shape[1] != cohort.shape[1]:
        raise _lib.PPVError(f'cohort_stats: embeddings {tuple(emb.shape)} and cohort {tuple(cohort.shape)} must be [*, D] with the same D')
    Q, D = emb.shape
    Nc = cohort.shape[0]
    chunk = int(max(1, min(Q, int(max_ws_bytes) // (4 * Nc))))
    lib = _lib.load()
    mean = torch.empty(Q, dtype=torch.float32, device=emb.device)
    std = torch.empty(Q, dtype=torch.float32, device=emb.device)
    buf = torch.empty((chunk, Nc), dtype=torch.float32, device=emb.device)
    ws_bytes = lib.ppv_cosine_workspace_bytes(chunk, Nc, D)
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device=emb.device)
    with torch.cuda.device(emb.device):
        for q0 in range(0, Q, chunk):
            q = min(chunk, Q - q0)
            part = emb[q0:q0 + q]
            _lib.check(lib.ppv_cosine_matrix(_lib.ptr(part), _lib.ptr(cohort), q, Nc, D, _lib.ptr(buf), C.c_void_p(ws.data_ptr()), ws_bytes,
                                             _lib.current_stream()), 'ppv_cosine_matrix')
            topn_row_stats(buf[:q], top_n, mean[q0:q0 + q], std[q0:q0 + q])
    return mean, std


def as_norm(scores, trial_stats, enroll_stats):
    """In place on scores [M, N] (float32, contiguous CUDA tensor of trials x enrolments) from (mean, std) of the trials [M] and of the
    enrolments [N]; returns ``scores``."""
    import torch
    _lib.require_cuda(scores, 'scores')
    if scores.dtype != torch.float32 or scores.dim() != 2 or not scores.is_contiguous():
        raise _lib.PPVError(f'as_norm: scores must be a contiguous 2-D float32 tensor, got {scores.dtype} {tuple(scores.shape)}')
    M, N = scores.shape
    stats = []
    for name, (m, s), n in (('trial', trial_stats, M), ('enrolment', enroll_stats, N)):
        m = torch.as_tensor(m).to(scores.device, torch.float32).contiguous()
        s = torch.as_tensor(s).to(scores.device, torch.float32).contiguous()
        if m.shape != (n,) or s.shape != (n,):
            raise _lib.PPVError(f'as_norm: {name} statistics must be [{n}], got {tuple(m.shape)} and {tuple(s.shape)}')
        stats += [m, s]
    with torch.cuda.device(scores.device):
        _lib.check(_lib.load().ppv_as_norm_apply(_lib.ptr(scores), M, N, *[_lib.ptr(t) for t in stats], _lib.current_stream()),
                   'ppv_as_norm_apply')
    return scores
