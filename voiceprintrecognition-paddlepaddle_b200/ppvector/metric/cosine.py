"""Batched cosine scoring on the GPU (libppv_b200: ppv_cosine_matrix / ppv_cosine_pairlist).

Replaces the CPU scoring of the reference: ``np.dot(a,b)/(|a||b|)`` (ppvector/predict.py:282),
``sklearn.metrics.pairwise.cosine_similarity`` (predict.py:178, trainer.py:419) and the per-trial Python loop of
``PPVectorTrainer.evaluate`` (trainer.py:416-423).
"""
import ctypes as C

import torch

from ppvector import _lib


def _prep(x, device='cuda'):
    """numpy / CPU inputs are uploaded (the reference hands numpy arrays to sklearn); compute is always on the GPU."""
    if not torch.is_tensor(x):
        x = torch.as_tensor(x)
    if not x.is_cuda:
        x = x.to(device)
    return x.to(torch.float32).contiguous()


def cosine_matrix(A, B):
    """A [M,D], B [N,D] -> [M,N] float32 CUDA tensor of cosine similarities."""
    A = _prep(A)
    B = _prep(B, A.device)
    M, D = A.shape
    N, D2 = B.shape
    assert D == D2
    lib = _lib.load()
    out = torch.empty((M, N), dtype=torch.float32, device=A.device)
    nbytes = lib.ppv_cosine_workspace_bytes(M, N, D)
    ws = torch.empty(nbytes, dtype=torch.uint8, device=A.device)
    with torch.cuda.device(A.device):
        _lib.check(lib.ppv_cosine_matrix(_lib.ptr(A), _lib.ptr(B), M, N, D, _lib.ptr(out), C.c_void_p(ws.data_ptr()), nbytes,
                                         _lib.current_stream()), 'ppv_cosine_matrix')
    return out


def cosine_pairlist(E, idx):
    """E [n,D] embeddings, idx [P,2] int32 pairs -> [P] float32 scores."""
    E = _prep(E)
    idx = torch.as_tensor(idx).to(device=E.device, dtype=torch.int32).contiguous()
    P = idx.shape[0]
    n, D = E.shape
    out = torch.empty((P,), dtype=torch.float32, device=E.device)
    if P == 0:
        return out
    with torch.cuda.device(E.device):
        _lib.check(_lib.load().ppv_cosine_pairlist(_lib.ptr(E), _lib.ptr(idx), P, n, D, _lib.ptr(out), _lib.current_stream()),
                   'ppv_cosine_pairlist')
    return out


def retrieval(features, db_features, threshold, names=None):
    """Enrol-DB lookup of ppvector/predict.py:173-187 (``__retrieval``): cosine of each query against the per-user mean embeddings,
    arg-max per query, accepted when the similarity reaches ``threshold``.  features [Q,D], db_features [U,D] ->
    list of [name_or_index, similarity rounded to 5 places] or [None, None] -- a transient speaker index of ``db_features`` searched
    for the top-1 on the GPU (ppvector.infer_utils.speaker_index; equal similarities: the lowest index, as numpy.argmax)."""
    from ppvector.infer_utils.speaker_index import SpeakerIndex
    db = _prep(db_features)
    index = SpeakerIndex(db, torch.arange(db.shape[0], device=db.device), db.shape[0], device=db.device)
    idx, best = index.search(_prep(features, db.device), k=1)
    return threshold_top1(idx[:, 0].cpu().tolist(), best[:, 0].cpu().tolist(), threshold, names)


def threshold_top1(idx, best, threshold, names=None):
    """[name_or_index, round(similarity, 5)] per query whose best similarity reaches ``threshold``, else [None, None]
    (predict.py:179-186)."""
    out = []
    for i, s in zip(idx, best):
        if s >= threshold:
            out.append([names[i] if names is not None else i, round(float(s), 5)])
        else:
            out.append([None, None])
    return out
