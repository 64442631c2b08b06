"""Device-resident speaker index of an enrolment database (libppv_b200: ppv_speaker_index_build / ppv_speaker_index_search).

Holds on the GPU the enrolment embeddings, the user id of each of them, the per-user mean embeddings and the library's search index
(an opaque buffer: its layout belongs to the library).  ``rebuild`` recomputes the means and the index in one launch -- enrolment changes
rebuild, there is no incremental path -- and ``search`` returns the k most similar users of each query without ever forming the
[queries x users] score matrix.  Replaces the per-user mean loop of ppvector/predict.py:154-163 and the sklearn cosine + argmax of
predict.py:173-187.
"""
import ctypes as C

import numpy as np
import torch

from ppvector import _lib


class SpeakerIndex:
    def __init__(self, embeddings, user_ids, num_users, device='cuda'):
        """embeddings [n, D] (enrolment order), user_ids [n] in [0, num_users), every user with at least one row."""
        self.device = torch.device(device)
        self.embeddings = torch.as_tensor(np.asarray(embeddings, dtype=np.float32) if not torch.is_tensor(embeddings) else embeddings)
        self.embeddings = self.embeddings.to(self.device, torch.float32).contiguous()
        self.user_ids = torch.as_tensor(np.asarray(user_ids) if not torch.is_tensor(user_ids) else user_ids).to(self.device, torch.int64)
        self.num_users = int(num_users)
        self.means = None
        self._index = None
        self.rebuild()

    @property
    def dim(self):
        return int(self.embeddings.shape[1])

    def rebuild(self):
        """Per-user means (fp32, each user's rows summed in enrolment order: bitwise numpy's E[rows].mean(axis=0)) and the search index."""
        n, D, U = int(self.embeddings.shape[0]), self.dim, self.num_users
        if n != int(self.user_ids.shape[0]):
            raise _lib.PPVError(f'SpeakerIndex: {n} embeddings but {int(self.user_ids.shape[0])} user ids')
        counts = torch.bincount(self.user_ids, minlength=U)
        if U < 1 or counts.shape[0] != U or bool((counts == 0).any()):
            raise _lib.PPVError(f'SpeakerIndex: every one of the {U} users needs at least one embedding')
        order = torch.argsort(self.user_ids, stable=True).to(torch.int32)
        offsets = torch.zeros(U + 1, dtype=torch.int32, device=self.device)
        offsets[1:] = torch.cumsum(counts, 0)
        lib = _lib.load()
        nbytes = lib.ppv_speaker_index_bytes(U, D)
        if nbytes == 0:
            raise _lib.PPVError(f'SpeakerIndex: unsupported shape (users {U}, dim {D}; 1 <= dim <= 256)')
        self.means = torch.empty((U, D), dtype=torch.float32, device=self.device)
        self._index = torch.empty(nbytes, dtype=torch.uint8, device=self.device)
        with torch.cuda.device(self.device):
            _lib.check(lib.ppv_speaker_index_build(_lib.ptr(self.embeddings), n, D, _lib.ptr(order), _lib.ptr(offsets), U, _lib.ptr(self.means),
                                                   C.c_void_p(self._index.data_ptr()), nbytes, _lib.current_stream()),
                       'ppv_speaker_index_build')

    def search(self, queries, k=1):
        """queries [Q, D] -> (idx [Q, k] int32, sim [Q, k] float32) CUDA tensors: the k most cosine-similar users per query, descending,
        equal similarities lowest user id first."""
        q = queries if torch.is_tensor(queries) else torch.as_tensor(np.asarray(queries, dtype=np.float32))
        q = q.to(self.device, torch.float32).contiguous()
        if q.dim() != 2 or q.shape[1] != self.dim:
            raise _lib.PPVError(f'SpeakerIndex.search: queries must be [Q, {self.dim}], got {tuple(q.shape)}')
        Q, k = int(q.shape[0]), int(k)
        lib = _lib.load()
        nbytes = lib.ppv_speaker_index_search_workspace_bytes(Q, self.num_users, self.dim, k)
        ws = torch.empty(max(nbytes, 1), dtype=torch.uint8, device=self.device)
        idx = torch.empty((Q, k), dtype=torch.int32, device=self.device)
        sim = torch.empty((Q, k), dtype=torch.float32, device=self.device)
        with torch.cuda.device(self.device):
            _lib.check(lib.ppv_speaker_index_search(_lib.ptr(q), Q, self.dim, C.c_void_p(self._index.data_ptr()), self._index.numel(),
                                                    self.num_users, k, _lib.ptr(idx), _lib.ptr(sim), C.c_void_p(ws.data_ptr()), nbytes,
                                                    _lib.current_stream()), 'ppv_speaker_index_search')
        return idx, sim
