"""PPVectorPredictor -- drop-in for the embedding / contrast surface of ppvector/predict.py:24-283.

Same constructor arguments and the same ``predict`` / ``predict_batch`` / ``contrast`` contracts
(numpy in, numpy out).  Differences that are the point of this build:
  * the waveform batch goes host -> device once (pinned staging buffer) and waveform -> Fbank -> ECAPA-TDNN ->
    embedding is ONE library call (``ppv_model_forward_wav``); the reference featurises per utterance in a Python
    loop and runs the model in chunks of 32 (predict.py:262-267);
  * cosine scoring runs on the GPU (``ppvector.metric.cosine``);
  * ``use_gpu=False`` raises: this build has no CPU path;
  * ``speaker_diarization`` clusters on the GPU (infer_utils/speaker_diarization.py); the voice-activity segments come from the caller
    or, with ``vad=True``, from Kaldi's energy VAD on the GPU (infer_utils/vad.py) where the reference runs silero-vad;
  * the enrolment database (``audio_db_path``: ``register``, ``remove_user``, ``recognition``, ``get_users``, ``search_audio_db``) keeps
    its per-user mean embeddings in a device-resident speaker index (infer_utils/speaker_index.py), rebuilt in one launch whenever a
    user is registered or removed and searched by a fused top-k kernel; ``recognition_batch`` (extension) identifies a whole batch of
    utterances with one search.
"""
import os
import pickle
import shutil
from io import BufferedReader

import numpy as np
import torch
import yaml
from loguru import logger

from ppvector import _lib
from ppvector.data_utils.audio import AudioSegment
from ppvector.data_utils.featurizer import AudioFeaturizer
from ppvector.infer_utils.speaker_index import SpeakerIndex
from ppvector.metric.cosine import cosine_matrix, threshold_top1
from ppvector.models import build_model
from ppvector.utils.checkpoint import load_state_dict_file
from ppvector.utils.utils import dict_to_object, print_arguments


class PPVectorPredictor:
    def __init__(self, configs, threshold=0.6, audio_db_path=None, model_path='models/EcapaTdnn_Fbank/best_model/',
                 use_gpu=True, state_dict=None):
        """reference: predict.py:25-67.  ``state_dict`` (extension): weights given in memory instead of a file."""
        if not use_gpu:
            raise _lib.PPVError('use_gpu=False: this build of ppvector has no CPU path')
        assert torch.cuda.is_available(), 'GPU不可用'
        self.device = torch.device('cuda', torch.cuda.current_device())
        self.threshold = threshold
        if isinstance(configs, str):
            with open(configs, 'r', encoding='utf-8') as f:
                configs = yaml.load(f.read(), Loader=yaml.FullLoader)
            print_arguments(configs=configs)
        self.configs = dict_to_object(configs)
        self._audio_featurizer = AudioFeaturizer(feature_method=self.configs.preprocess_conf.feature_method,
                                                 method_args=self.configs.preprocess_conf.get('method_args', {}))
        backbone = build_model(input_size=self._audio_featurizer.feature_dim, configs=self.configs)
        if state_dict is None:
            if not os.path.exists(model_path):
                raise Exception("模型文件不存在，请检查{}是否存在！".format(model_path))
            state_dict = load_state_dict_file(model_path)
        # the reference wraps the backbone in nn.Sequential, hence the "0." key prefix (predict.py:59, checkpoint.py)
        state_dict = {(k[2:] if k.startswith('0.') else k): v for k, v in state_dict.items() if not k.startswith('1.')}
        backbone.load_state_dict({k: torch.as_tensor(np.asarray(v)) for k, v in state_dict.items()})
        self.predictor = backbone.eval().to(self.device)
        self._pinned = None
        self._pinned_out = None
        self.audio_db_path = audio_db_path
        self.users_name, self.users_audio_path, self.users_name_mean = [], [], []
        self.audio_feature, self.audio_feature_mean = None, None
        self._index = None
        if audio_db_path is not None:
            self.audio_indexes_path = os.path.join(audio_db_path, 'audio_indexes.bin')
            self._load_audio_db(audio_db_path)

    # ---- enrolment database: predict.py:89-187, 285-364 ------------------------------------------------------
    def _load_audio_indexes(self):
        """predict.py:89-102: the pickled index of embedded enrolment files; entries whose file is gone are dropped."""
        if not os.path.exists(self.audio_indexes_path):
            return
        with open(self.audio_indexes_path, 'rb') as f:
            indexes = pickle.load(f)
        for name, feature, path in zip(indexes['users_name'], indexes['faces_feature'], indexes['users_image_path']):
            if not os.path.exists(path):
                continue
            self.users_name.append(name)
            self.users_audio_path.append(path)
            self.audio_feature = feature[None] if self.audio_feature is None else np.vstack((self.audio_feature, feature))

    def _write_index(self):
        """predict.py:105-109 (same keys, same pickle layout)."""
        with open(self.audio_indexes_path, 'wb') as f:
            pickle.dump({'users_name': self.users_name, 'faces_feature': self.audio_feature, 'users_image_path': self.users_audio_path}, f)

    def _load_audio_db(self, audio_db_path):
        """predict.py:112-165: embed <db>/<user>/* files not yet in the index (predict_batch, eval batch size), rewrite the index,
        keep one mean embedding per user (users_name_mean in the reference's set() order; the means from the speaker index)."""
        self._load_audio_indexes()
        os.makedirs(audio_db_path, exist_ok=True)
        audios_path = []
        for name in os.listdir(audio_db_path):
            audio_dir = os.path.join(audio_db_path, name)
            if os.path.isdir(audio_dir):
                audios_path.extend(os.path.join(audio_dir, f).replace('\\', '/') for f in os.listdir(audio_dir))
        if len(audios_path) == 0:
            return
        known = set(self.users_audio_path)
        new = [p for p in audios_path if p not in known]
        bs = self.configs.dataset_conf.eval_conf.batch_size
        for i in range(0, len(new), bs):
            features = self.predict_batch(new[i:i + bs])
            self.audio_feature = features if self.audio_feature is None else np.vstack((self.audio_feature, features))
        for p in new:
            self.users_name.append(os.path.basename(os.path.dirname(p)))
            self.users_audio_path.append(p)
        assert len(self.audio_feature) == len(self.users_name) == len(self.users_audio_path), '加载的数量对不上！'
        self._write_index()
        self.users_name_mean = list(set(self.users_name))
        self._rebuild_index()
        logger.info(f'声纹库数据加载完成，一共有{len(self.audio_feature_mean)}个用户，分别是：{self.users_name_mean}')

    def _rebuild_index(self):
        """The speaker index of the enrolment rows: user i of users_name_mean owns the rows named users_name_mean[i]; audio_feature_mean
        is its [users, D] means (each user's rows summed in enrolment order, then divided: bitwise the reference's
        audio_feature[rows].mean(axis=0))."""
        if not self.users_name_mean:
            self._index = None
            self.audio_feature_mean = None if self.audio_feature is None else self.audio_feature[:0].copy()
            return
        user_id = {name: i for i, name in enumerate(self.users_name_mean)}
        self._index = SpeakerIndex(np.ascontiguousarray(self.audio_feature, dtype=np.float32), [user_id[n] for n in self.users_name],
                                   len(self.users_name_mean), self.device)
        self.audio_feature_mean = self._index.means.cpu().numpy()

    def _search(self, np_feature, k):
        assert self._index is not None, "数据库中没有音频数据，请先指定说话人特征数据库或者注册说话人"
        idx, sim = self._index.search(np.asarray(np_feature, dtype=np.float32), k=min(int(k), self._index.num_users))
        return idx.cpu().tolist(), sim.cpu().tolist()

    def _retrieval(self, np_feature):
        """predict.py:173-187: [name, similarity] of the best-matching user per query, [None, None] under the threshold (top-1 search
        of the speaker index)."""
        idx, sim = self._search(np_feature, 1)
        return threshold_top1([i[0] for i in idx], [s[0] for s in sim], self.threshold, names=self.users_name_mean)

    def recognition(self, audio_data, threshold=None, sample_rate=16000):
        """predict.py:324-335 -> [name, similarity], or [None, None] under the threshold."""
        if threshold:
            self.threshold = threshold
        feature = self.predict(audio_data, sample_rate=sample_rate)
        return self._retrieval(feature[None])[0]

    def recognition_batch(self, audios_data, threshold=None, sample_rate=16000, top_k=1):
        """Identification of a batch of utterances (extension): embedded together (predict_batch), then ONE top-k search of the speaker
        index.  Per utterance a list of up to ``top_k`` (<= 8) [name, similarity rounded to 5 places], most similar first, holding the
        users at or above ``threshold`` (None: the predictor's threshold, which this call does not change)."""
        threshold = self.threshold if threshold is None else threshold
        features = self.predict_batch(audios_data, sample_rate=sample_rate)
        idx, sim = self._search(features, top_k)
        return [[[self.users_name_mean[i], round(float(s), 5)] for i, s in zip(ri, rs) if s >= threshold] for ri, rs in zip(idx, sim)]

    def register(self, audio_data, user_name: str, sample_rate=16000):
        """predict.py:285-322 -> (True, "注册成功").  The audio goes through _load_audio (resample, dB normalisation) and the embedding
        path; the processed samples are stored as <db>/<user_name>/<n>.wav (32-bit float WAV), the index file is rewritten and the
        user's mean (or a new user) goes into the speaker index.  Deviations from the reference:
          * registering into an empty database works (the reference's np.vstack((None, feature)) raises there);
          * an existing file is never overwritten: n is the smallest unused number >= the number of files in the user's directory (the
            reference takes that number as is, which overwrites a file after a manual delete);
          * a predictor without a database (audio_db_path=None) raises ValueError (the reference fails with a TypeError)."""
        if self.audio_db_path is None:
            raise ValueError('register: this predictor has no enrolment database (audio_db_path=None)')
        audio_segment = self._load_audio(audio_data=audio_data, sample_rate=sample_rate)
        feature = self.predict(audio_data=audio_segment)
        self.audio_feature = feature[None] if self.audio_feature is None else np.vstack((self.audio_feature, feature))
        user_dir = os.path.join(self.audio_db_path, user_name)
        n = len(os.listdir(user_dir)) if os.path.exists(user_dir) else 0
        while os.path.exists(os.path.join(user_dir, f'{n}.wav')):
            n += 1
        audio_path = os.path.join(user_dir, f'{n}.wav')
        os.makedirs(user_dir, exist_ok=True)
        audio_segment.to_wav_file(audio_path)
        self.users_audio_path.append(audio_path.replace('\\', '/'))
        self.users_name.append(user_name)
        self._write_index()
        if user_name not in self.users_name_mean:
            self.users_name_mean.append(user_name)
        self._rebuild_index()
        return True, "注册成功"

    def remove_user(self, user_name):
        """predict.py:344-364 -> True, or False for an unknown user: drops every row of the user, rewrites the index file, deletes
        <db>/<user_name>/ and takes the user out of the speaker index."""
        if user_name not in self.users_name:
            return False
        keep = [i for i, v in enumerate(self.users_name) if v != user_name]
        self.users_name[:] = [self.users_name[i] for i in keep]
        self.users_audio_path[:] = [self.users_audio_path[i] for i in keep]
        self.audio_feature = self.audio_feature[keep]
        self._write_index()
        shutil.rmtree(os.path.join(self.audio_db_path, user_name))
        del self.users_name_mean[self.users_name_mean.index(user_name)]
        self._rebuild_index()
        return True

    def get_users(self):
        """predict.py:337-342"""
        return self.users_name

    # ---- audio loading: predict.py:189-216 ----------------------------------------------------------------
    def _load_audio(self, audio_data, sample_rate=16000):
        if isinstance(audio_data, str):
            audio_segment = AudioSegment.from_file(audio_data)
        elif isinstance(audio_data, BufferedReader):
            audio_segment = AudioSegment.from_file(audio_data)
        elif isinstance(audio_data, np.ndarray):
            audio_segment = AudioSegment.from_ndarray(audio_data, sample_rate)
        elif isinstance(audio_data, bytes):
            audio_segment = AudioSegment.from_bytes(audio_data)
        elif isinstance(audio_data, AudioSegment):
            audio_segment = audio_data
        else:
            raise Exception(f'不支持该数据类型，当前数据类型为：{type(audio_data)}')
        ds = self.configs.dataset_conf.dataset
        assert audio_segment.duration >= ds.min_duration, \
            f'音频太短，最小应该为{ds.min_duration}s，当前音频为{audio_segment.duration}s'
        if audio_segment.sample_rate != ds.sample_rate:
            audio_segment.resample(ds.sample_rate)
        if ds.use_dB_normalization:
            audio_segment.normalize(target_db=ds.target_dB)
        return audio_segment

    # ---- host buffers -> embeddings -----------------------------------------------------------------------
    def extract_embeddings(self, waveforms: np.ndarray, input_lens_ratio=None) -> np.ndarray:
        """[B,L] float32 host waveforms (already normalised / padded) -> [B,embd] float32 host embeddings.
        One pinned H2D copy, one fused library call, one D2H copy."""
        waveforms = np.ascontiguousarray(waveforms, dtype=np.float32)
        B, L = waveforms.shape
        if self._pinned is None or self._pinned.shape[0] < B or self._pinned.shape[1] != L:
            self._pinned = torch.empty((B, L), dtype=torch.float32).pin_memory()
        stage = self._pinned[:B]
        stage.copy_(torch.from_numpy(waveforms))
        return self.extract_embeddings_pinned(stage, input_lens_ratio).numpy().copy()

    def extract_embeddings_pinned(self, stage: torch.Tensor, input_lens_ratio=None) -> torch.Tensor:
        """As extract_embeddings, for a caller that already owns a pinned [B,L] float32 host tensor; returns a
        pinned host tensor (valid until the next call)."""
        B = stage.shape[0]
        wav = stage.to(self.device, non_blocking=True)
        emb = self.predictor.forward_wav(self._audio_featurizer, wav, input_lens_ratio)
        if self._pinned_out is None or self._pinned_out.shape[0] < B:
            self._pinned_out = torch.empty((B, emb.shape[1]), dtype=torch.float32).pin_memory()
        out = self._pinned_out[:B]
        out.copy_(emb, non_blocking=True)
        torch.cuda.current_stream().synchronize()
        return out

    def _lanes(self, n):
        """Compute lanes for the streaming calls.  Lane 0 is this predictor's model and featurizer; further lanes are replicas (same weights,
        own workspace, own featurizer scratch) that run on their own CUDA streams, so that two batches can be in the kernels at once: the
        persistent kernels of one batch leave SMs idle in their last tile round, between dependent launches and in the one-row-per-utterance
        layers (2-6 CTAs), and the other batch's kernels take them."""
        lanes = getattr(self, '_lane_objs', None)
        if lanes is None:
            lanes = self._lane_objs = [(self.predictor, self._audio_featurizer, None)]
        while len(lanes) < n:
            fz = AudioFeaturizer(feature_method=self.configs.preprocess_conf.feature_method,
                                 method_args=self.configs.preprocess_conf.get('method_args', {}))
            bb = build_model(input_size=fz.feature_dim, configs=self.configs)
            bb.load_state_dict(self.predictor.state_dict())
            bb = bb.eval().to(self.device)
            lanes.append((bb, fz, torch.cuda.Stream(self.device)))
        for bb, _, _ in lanes[1:n]:
            if getattr(bb, 'precision', None) != getattr(self.predictor, 'precision', None):
                bb.set_precision(self.predictor.precision)
        return lanes[:n]

    def _lanes_pdl(self, nl, restore=None):
        """PPV_LANES_PDL=0 launches the lanes' kernels WITHOUT programmatic dependent launch (ppv_set_pdl): an early-launched dependent CTA holds
        a whole SM while its primary drains.  Measured either way without a consistent winner (DESIGN.md 5a); the default keeps it on."""
        lib = _lib.load()
        if restore is not None:
            lib.ppv_set_pdl(restore)
            return None
        if nl > 1 and os.environ.get('PPV_LANES_PDL', '1') != '1':
            return lib.ppv_set_pdl(0)
        return None

    def embed_resident_stream(self, device_batches, input_lens_ratio=None, lanes=3):
        """Generator: device-resident [B,L] float32 waveform batches -> one device [B,embd] embedding tensor per batch, in order, batches dealt
        round robin to ``lanes`` compute lanes and paced like extract_embeddings_stream (a lane's next batch is enqueued behind its running
        one, then the host waits for the oldest batch and yields it; lanes + 1 batches queued at most).  A yielded tensor is complete (the
        host has synchronised on its lane) and stays valid for as long as the caller keeps it -- but a caller that keeps ALL of them makes
        every step allocate fresh device memory, and cudaMalloc synchronises the whole device, which stalls every lane: consume and drop."""
        from collections import deque
        main = torch.cuda.current_stream(self.device)
        L = self._lanes(max(1, int(lanes)))
        nl = len(L)
        streams = [main if st is None else st for _, _, st in L]
        start = torch.cuda.Event()
        start.record(main)
        inflight = deque()  # (embedding, completion event), oldest first
        for i, wav in enumerate(device_batches):
            model, fz, _ = L[i % nl]
            st = streams[i % nl]
            pdl_prev = self._lanes_pdl(nl)
            try:
                with torch.cuda.stream(st):
                    if i < nl and st is not main:
                        st.wait_event(start)  # inputs produced on the caller's stream
                    emb = model.forward_wav(fz, wav, input_lens_ratio)
                    ev = torch.cuda.Event()
                    ev.record(st)
            finally:
                if pdl_prev is not None:
                    self._lanes_pdl(nl, restore=pdl_prev)
            inflight.append((emb, ev))
            del emb
            if len(inflight) > nl:
                out, ev = inflight.popleft()
                ev.synchronize()
                yield out
                del out
        while inflight:
            out, ev = inflight.popleft()
            ev.synchronize()
            yield out
            del out

    def extract_embeddings_stream(self, pinned_batches, input_lens_ratio=None, lanes=3):
        """Pipelined form of extract_embeddings_pinned for a sequence of pinned [B,L] float32 host batches.  The H2D copy of a batch runs on
        a copy stream while earlier batches are in the kernels; batches are dealt round robin to ``lanes`` compute lanes (see _lanes), and the
        kernels of the next batch are enqueued BEFORE the host waits for the oldest batch's embeddings.  Yields one pinned host [B,embd]
        tensor per batch, in order (valid until the next item is requested); every batch still pays its own H2D and D2H -- they are
        overlapped, not skipped."""
        from collections import deque
        L = self._lanes(max(1, int(lanes)))
        nl = len(L)
        main = torch.cuda.current_stream(self.device)
        streams = [main if st is None else st for _, _, st in L]
        copy = getattr(self, '_copy_stream', None)
        if copy is None:
            copy = self._copy_stream = torch.cuda.Stream(self.device)
        nb = nl + 1      # device staging buffers: the batches in the kernels plus the one being copied
        ns = 2 * nl      # pinned outputs / completion events: a lane's next batch is enqueued while its previous result is still unread
        dev = [None] * nb
        ready = [torch.cuda.Event() for _ in range(nb)]
        free = [torch.cuda.Event() for _ in range(nb)]
        done = [torch.cuda.Event() for _ in range(ns)]
        outs = [None] * ns
        it = iter(pinned_batches)

        def stage(i, host):
            k = i % nb
            with torch.cuda.stream(copy):
                if i >= nb:
                    copy.wait_event(free[k])  # the kernels of batch i - nb have consumed this buffer
                if dev[k] is None or dev[k].shape != host.shape:
                    dev[k] = torch.empty(host.shape, dtype=torch.float32, device=self.device)
                dev[k].copy_(host, non_blocking=True)
                ready[k].record(copy)

        def launch(i):
            k, ln, sl = i % nb, i % nl, i % ns
            model, fz, _ = L[ln]
            st = streams[ln]
            with torch.cuda.stream(st):
                st.wait_event(ready[k])
                emb = model.forward_wav(fz, dev[k], input_lens_ratio)
                free[k].record(st)
                if outs[sl] is None or outs[sl].shape != emb.shape:
                    outs[sl] = torch.empty(emb.shape, dtype=torch.float32).pin_memory()
                outs[sl].copy_(emb, non_blocking=True)
                done[sl].record(st)

        def launch_no_pdl(i):  # see _lanes_pdl; the switch is process-wide, so it is flipped only around this generator's own launches
            prev = self._lanes_pdl(nl)
            try:
                launch(i)
            finally:
                if prev is not None:
                    self._lanes_pdl(nl, restore=prev)

        inflight = deque()
        i = 0
        nxt = next(it, None)
        while nxt is not None and len(inflight) < nl:
            stage(i, nxt)
            launch_no_pdl(i)
            inflight.append(i)
            i += 1
            nxt = next(it, None)
        while inflight:
            j = inflight.popleft()
            if nxt is not None:  # keep the lanes fed before blocking on the oldest batch
                stage(i, nxt)
                launch_no_pdl(i)
                inflight.append(i)
                i += 1
                nxt = next(it, None)
            done[j % ns].synchronize()
            yield outs[j % ns]

    def predict(self, audio_data, sample_rate=16000):
        """reference: predict.py:218-233 -> [embd] numpy"""
        seg = self._load_audio(audio_data=audio_data, sample_rate=sample_rate)
        return self.extract_embeddings(seg.samples[None, :])[0]

    def predict_batch(self, audios_data, sample_rate=16000, batch_size=32):
        """reference: predict.py:235-269.  Zero-pad to the longest of the WHOLE list, lens-ratio mask after CMN (featurizer.py:48-59),
        then the model in chunks of ``batch_size`` (predict.py:264-267).  Featurisation is per utterance, so chunking the padded
        waveforms gives the same embeddings as featurising the whole list at once, and bounds the workspace."""
        segs = [self._load_audio(audio_data=a, sample_rate=sample_rate).samples for a in audios_data]
        max_len = max(s.shape[0] for s in segs)
        inputs = np.zeros((len(segs), max_len), dtype=np.float32)
        ratio = np.zeros((len(segs),), dtype=np.float32)
        for i, s in enumerate(segs):
            inputs[i, :s.shape[0]] = s
            ratio[i] = s.shape[0] / max_len
        batch_size = max(1, int(batch_size))
        return np.concatenate([self.extract_embeddings(inputs[i:i + batch_size], ratio[i:i + batch_size])
                               for i in range(0, len(segs), batch_size)], axis=0)

    def diarization_embeddings(self, audio_data, sample_rate=16000, vad_segments=None, seg_duration=1.5, seg_shift=0.75, batch_size=256,
                               vad=False):
        """The embedding fan-out of the reference's ``speaker_diarization`` (predict.py:378-381): the recording (or the given voice-activity
        segments [(start_s, end_s), ...]) is cut into ``seg_duration`` windows every ``seg_shift`` seconds (infer_utils/chunking.py) and every
        window goes through the embedding path as ONE equal-length batch.  Returns (times [n, 2] seconds, embeddings [n, embd]).  Pass
        ``vad_segments`` from your VAD, or ``vad=True`` to find them with the energy VAD (infer_utils/vad.py) on the loaded audio; with
        neither, the whole recording is one segment."""
        from ppvector.infer_utils.chunking import fan_out_embeddings
        sr, segs = self._voiced_segments(audio_data, sample_rate, vad_segments, vad)
        return fan_out_embeddings(segs, self.extract_embeddings, seg_duration, seg_shift, sr, batch_size)

    def _voiced_segments(self, audio_data, sample_rate, vad_segments, vad=False):
        """-> (sample rate, [(start_s, end_s, samples), ...]) of the given voice-activity segments, of the segments the energy VAD finds
        on the loaded (resampled, dB-normalised) audio (vad=True), or of the whole recording."""
        if vad and vad_segments is not None:
            raise ValueError('pass either vad=True or vad_segments, not both')
        seg = self._load_audio(audio_data=audio_data, sample_rate=sample_rate)
        sr, x = seg.sample_rate, seg.samples
        if vad:
            vad_segments = [(t['start'], t['end']) for t in seg.vad(return_seconds=True)]
        spans = [(0.0, len(x) / sr)] if vad_segments is None else [(round(float(a), 3), round(float(b), 3)) for a, b in vad_segments]
        return sr, [(a, b, x[int(a * sr):int(b * sr)]) for a, b in spans]

    def speaker_diarization(self, audio_data, sample_rate=16000, speaker_num=None, search_audio_db=False, vad_segments=None, vad=False):
        """reference: predict.py:366-396 -> [{'speaker', 'start', 'end'}, ...].  The recording (or the given voice-activity segments
        [(start_s, end_s), ...]; None = the whole recording; vad=True: the segments the energy VAD finds, as the reference's
        segments_audio does with silero-vad) is cut into 1.5 s windows every 0.75 s and embedded as one batch
        (diarization_embeddings); the windows are clustered on the GPU (infer_utils/speaker_diarization.py: spectral clustering,
        ``speaker_num`` fixes the speaker count) and the segments post-processed as in the reference.  The voiced speech must total
        more than 5 s.  search_audio_db=True names each speaker from the enrolment database (``audio_db_path``)."""
        from ppvector.infer_utils.chunking import fan_out_embeddings
        from ppvector.infer_utils.speaker_diarization import SpeakerDiarization
        sr, segs = self._voiced_segments(audio_data, sample_rate, vad_segments, vad)
        sd = SpeakerDiarization(sample_rate=sr)
        sd._check_audio_list([list(s) for s in segs])
        times, features = fan_out_embeddings(segs, self.extract_embeddings, sd.seg_duration, sd.seg_shift, sr, 256)
        labels, spk_center_embeddings = sd.clustering(features, speaker_num=speaker_num)
        outputs = sd.postprocess([list(t) for t in times.tolist()], labels)
        if search_audio_db:
            assert getattr(self, 'audio_feature', None) is not None, "数据库中没有音频数据，请先指定说话人特征数据库或者注册说话人"
            names = self._retrieval(spk_center_embeddings)  # indexed with the post-merge labels, as the reference does
            outputs = [{'speaker': names[o['speaker']][0] if names[o['speaker']][0] else f"陌生人{o['speaker']}",
                        'start': o['start'], 'end': o['end']} for o in outputs]
        return outputs

    def contrast(self, audio_data1, audio_data2):
        """reference: predict.py:271-283 -> cosine similarity of the two embeddings"""
        feature1 = self.predict(audio_data1)
        feature2 = self.predict(audio_data2)
        e = torch.from_numpy(np.stack([feature1, feature2])).to(self.device)
        return float(cosine_matrix(e[:1], e[1:])[0, 0].item())
