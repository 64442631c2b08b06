"""Speaker diarization after the embeddings: spectral clustering on the GPU, post-processing on the host.
Drop-in for the reference's ppvector/infer_utils/speaker_diarization.py (same class names, defaults and results).

``SpectralCluster`` runs the clustering chain of the reference (:219-310) on the device (csrc/cluster.cu):
  cosine affinity (``ppv_cosine_matrix``, fp32) -> per-row pruning (``ppv_cluster_prune``) -> Laplacian (``ppv_cluster_laplacian``, fp64)
  -> the m = min(max(16, k), N) smallest eigenpairs (``ppv_sym_eig_smallest``: Householder tridiagonalisation, bisection, inverse
  iteration, back-transformation, fp64) -> k by the eigengap (host, from the m eigenvalues) -> k-means (``ppv_kmeans``).
The reference runs a full scipy ``eigh`` (O(N^3) on the CPU) and sklearn's k-means.  The k-means++ draws come from numpy's global
generator exactly as sklearn's ``k_means(..., random_state=None)`` takes them, so seeding ``np.random`` seeds both the same way.
At most 8192 windows (about 1.7 h of speech) per call; more raise ``PPVError``.

``SpeakerDiarization``: the label and segment post-processing (:89-216) is list logic over a few thousand segments and stays on
the host, quirks of the reference included (see ``_merge_by_cos``).  Windowing is infer_utils/chunking.py.  Voice-activity detection
(``segments_audio``) runs Kaldi's energy VAD on the GPU (infer_utils/vad.py) where the reference runs yeaudio's silero VAD; callers
may also pass voiced segments of their own.
"""
import ctypes as C

import numpy as np
import torch

from ppvector import _lib
from ppvector.infer_utils.chunking import chunk_segments
from ppvector.metric.cosine import cosine_matrix

__all__ = ['SpeakerDiarization', 'SpectralCluster']


class SpeakerDiarization(object):

    def __init__(self, seg_duration=1.5, seg_shift=0.75, sample_rate=16000, merge_threshold=0.78):
        """reference :11-24"""
        self.seg_duration = seg_duration
        self.seg_shift = seg_shift
        self.sample_rate = sample_rate
        self.merge_threshold = merge_threshold
        self.spectral_cluster = SpectralCluster()

    def segments_audio(self, audio_segment) -> list:
        """reference :26-45: the voiced spans of the recording (AudioSegment.vad, here the energy VAD), rounded to milliseconds, checked
        and cut into seg_duration windows -> [[start_s, end_s, window samples], ...]."""
        vad_segments = []
        samples = audio_segment.samples
        self.sample_rate = audio_segment.sample_rate
        for t in audio_segment.vad(return_seconds=True):
            st, ed = round(t['start'], 3), round(t['end'], 3)
            vad_segments.append([st, ed, samples[int(st * self.sample_rate):int(ed * self.sample_rate)]])
        self._check_audio_list(vad_segments)
        return self._chunk(vad_segments)

    def _check_audio_list(self, audio: list):
        """reference :47-57: ordered, consistent [start_s, end_s, samples] segments with more than 5 s of speech in all."""
        audio_duration = 0
        for i in range(len(audio)):
            seg = audio[i]
            assert seg[1] >= seg[0], '分割的时间戳错误'
            assert isinstance(seg[2], np.ndarray), '数据的类型不正确'
            assert int(seg[1] * self.sample_rate) - int(seg[0] * self.sample_rate) == seg[2].shape[0], '时间长度和数据长度不匹配'
            if i > 0:
                assert seg[0] >= audio[i - 1][1], 'modelscope error: Wrong time stamps.'
            audio_duration += seg[1] - seg[0]
        assert audio_duration > 5, f'音频时间过段，应当大于5秒，当前长度是{audio_duration}秒'

    def _chunk(self, vad_segments: list) -> list:
        """reference :60-87 -> [[start_s, end_s, window samples], ...] (chunking.chunk_segments)."""
        times, chunks = chunk_segments(vad_segments, self.seg_duration, self.seg_shift, self.sample_rate)
        return [[float(t[0]), float(t[1]), c] for t, c in zip(times, chunks)]

    def clustering(self, embeddings: np.ndarray, speaker_num=None):
        """reference :89-109 -> (labels after the cosine merge, per-label mean embeddings before it)."""
        labels = self.spectral_cluster(embeddings, oracle_num=speaker_num)
        labels = self._correct_labels(labels)
        spk_num = labels.max() + 1
        spk_center = [embeddings[labels == i].mean(0) for i in range(spk_num)]
        assert len(spk_center) > 0
        spk_center_embeddings = np.stack(spk_center, axis=0)
        labels = self._merge_by_cos(labels, spk_center, self.merge_threshold)
        return labels, spk_center_embeddings

    @staticmethod
    def _merge_by_cos(labels, spk_center_emb, cos_thr):
        """reference :113-136, quirk included: after a merge the label count drops but the centre list is not rebuilt, so the
        next round compares the first (count) centres of the original list -- the last centre drops out, not the merged one."""
        assert 0 < cos_thr <= 1
        while True:
            spk_num = labels.max() + 1
            if spk_num == 1:
                break
            spk_center = np.stack([spk_center_emb[i] for i in range(spk_num)], axis=0)
            norm_spk_center = spk_center / np.linalg.norm(spk_center, axis=1, keepdims=True)
            affinity = np.triu(np.matmul(norm_spk_center, norm_spk_center.T), 1)
            spks = np.unravel_index(np.argmax(affinity), affinity.shape)
            if affinity[spks] < cos_thr:
                break
            for i in range(len(labels)):
                if labels[i] == spks[1]:
                    labels[i] = spks[0]
                elif labels[i] > spks[1]:
                    labels[i] -= 1
        return labels

    def postprocess(self, segments: list, labels: np.ndarray) -> list:
        """reference :138-174: merge runs of one speaker, split overlaps at their midpoint, smooth segments under 1 s."""
        assert len(segments) == len(labels)
        distribute_res = [[segments[i][0], segments[i][1], labels[i]] for i in range(len(segments))]
        distribute_res = self._merge_seque(distribute_res)
        for i in range(1, len(distribute_res)):
            if distribute_res[i - 1][1] > distribute_res[i][0] + 1e-4:
                p = (distribute_res[i][0] + distribute_res[i - 1][1]) / 2
                distribute_res[i][0] = p
                distribute_res[i - 1][1] = p
        distribute_res = self._smooth(distribute_res)
        return [dict(speaker=r[2], start=round(r[0], 3), end=round(r[1], 3)) for r in distribute_res]

    @staticmethod
    def _correct_labels(labels):
        """reference :177-187: renumber labels in order of first appearance."""
        id2id, new_labels = {}, []
        for i in labels:
            if i not in id2id:
                id2id[i] = len(id2id)
            new_labels.append(id2id[i])
        return np.array(new_labels)

    @staticmethod
    def _merge_seque(distribute_res):
        """reference :190-198"""
        res = [distribute_res[0]]
        for i in range(1, len(distribute_res)):
            if distribute_res[i][2] != res[-1][2] or distribute_res[i][0] > res[-1][1]:
                res.append(distribute_res[i])
            else:
                res[-1][1] = distribute_res[i][1]
        return res

    def _smooth(self, res, min_duration=1):
        """reference :201-216; like the reference it raises IndexError when the only segment is shorter than min_duration."""
        for i in range(len(res)):
            res[i][0] = round(res[i][0], 2)
            res[i][1] = round(res[i][1], 2)
            if res[i][1] - res[i][0] < min_duration:
                if i == 0:
                    res[i][2] = res[i + 1][2]
                elif i == len(res) - 1:
                    res[i][2] = res[i - 1][2]
                elif res[i][0] - res[i - 1][1] <= res[i + 1][0] - res[i][1]:
                    res[i][2] = res[i - 1][2]
                else:
                    res[i][2] = res[i + 1][2]
        return self._merge_seque(res)


def _ws(nbytes, device):
    return torch.empty(max(int(nbytes), 1), dtype=torch.uint8, device=device)


class SpectralCluster:
    def __init__(self, min_num_spks=1, max_num_spks=15, pval=0.022):
        """reference :220-232"""
        self.min_num_spks = min_num_spks
        self.max_num_spks = max_num_spks
        self.pval = pval

    def __call__(self, X, oracle_num=None):
        """X [N, D] embeddings (numpy or tensor) -> labels [N] int numpy (reference :235-250)."""
        X = torch.as_tensor(np.asarray(X) if not torch.is_tensor(X) else X)
        X = (X if X.is_cuda else X.to('cuda')).to(torch.float32).contiguous()
        N = X.shape[0]
        P = cosine_matrix(X, X)
        L = self.laplacian(P, self.pval)
        m = min(max(self.max_num_spks + 1, oracle_num or 0), N)
        lambdas, vecs = self.smallest_eigs(L, m)
        if oracle_num is not None:
            k = int(oracle_num)
        else:
            k = int(np.argmax(self.get_eigen_gaps(lambdas[self.min_num_spks - 1:self.max_num_spks + 1]))) + self.min_num_spks
        labels, _ = self.kmeans(vecs, k, np.random.random_sample(1 + (k - 1) * (2 + int(np.log(k)))))
        return labels

    @staticmethod
    def laplacian(affinity, pval=0.022):
        """affinity [N, N] fp32 CUDA tensor, pruned in place (p_pruning, :260-275) -> Laplacian [N, N] fp64 CUDA tensor (:246, :277-283)."""
        lib = _lib.load()
        N = affinity.shape[0]
        L = torch.empty((N, N), dtype=torch.float64, device=affinity.device)
        with torch.cuda.device(affinity.device):
            _lib.check(lib.ppv_cluster_prune(_lib.ptr(affinity), N, float(pval), _lib.current_stream()), 'ppv_cluster_prune')
            _lib.check(lib.ppv_cluster_laplacian(_lib.ptr(affinity), N, _lib.ptr(L), _lib.current_stream()), 'ppv_cluster_laplacian')
        return L

    @staticmethod
    def smallest_eigs(L, m):
        """L [N, N] fp64 CUDA tensor (overwritten) -> (m smallest eigenvalues, numpy ascending; eigenvectors [N, m] fp64 CUDA tensor)."""
        lib = _lib.load()
        N = L.shape[0]
        evals = torch.empty((m,), dtype=torch.float64, device=L.device)
        evecs = torch.empty((N, m), dtype=torch.float64, device=L.device)
        nbytes = lib.ppv_sym_eig_workspace_bytes(N, m)
        ws = _ws(nbytes, L.device)
        with torch.cuda.device(L.device):
            _lib.check(lib.ppv_sym_eig_smallest(_lib.ptr(L), N, m, _lib.ptr(evals), _lib.ptr(evecs), C.c_void_p(ws.data_ptr()), nbytes,
                                                _lib.current_stream()), 'ppv_sym_eig_smallest')
        return evals.cpu().numpy(), evecs

    @staticmethod
    def kmeans(X, k, uniforms, max_iter=300):
        """k-means of the first k columns of X [N, >= k] fp64 CUDA tensor -> (labels int numpy, inertia) (cluster_embs, :299-301)."""
        lib = _lib.load()
        N, ld = X.shape
        u = torch.as_tensor(np.asarray(uniforms, dtype=np.float64)).to(X.device)
        labels = torch.empty((N,), dtype=torch.int32, device=X.device)
        inertia = torch.empty((1,), dtype=torch.float64, device=X.device)
        nbytes = lib.ppv_kmeans_workspace_bytes(N, k)
        ws = _ws(nbytes, X.device)
        with torch.cuda.device(X.device):
            _lib.check(lib.ppv_kmeans(_lib.ptr(X), ld, N, k, _lib.ptr(u), u.numel(), max_iter, _lib.ptr(labels), _lib.ptr(inertia),
                                      C.c_void_p(ws.data_ptr()), nbytes, _lib.current_stream()), 'ppv_kmeans')
        return labels.cpu().numpy().astype(np.int64), float(inertia.item())

    @staticmethod
    def get_eigen_gaps(eig_vals):
        """reference :304-310"""
        return [float(eig_vals[i + 1]) - float(eig_vals[i]) for i in range(len(eig_vals) - 1)]
