"""PPVectorDataset -- the eval / extract_feature / plain-train subset of ppvector/data_utils/reader.py:16-163.

List file lines are ``path\\tlabel``; items are ``(feature [T,F] float32 CUDA tensor, speaker id)``.  Audio goes
wav -> float32 -> (resample) -> dB normalise -> crop (eval: from 0; train: random start; extract_feature: no crop) ->
``AudioFeaturizer`` on the GPU -> SpecAugment (train mode, reader.py:105-107, ``ppv_spec_augment``).  ``.npy`` entries are
pre-extracted features (reader.py:78-83).  Waveform augmentation (reader.py:143-163: speed / volume / noise / reverb), dB normalisation
and the crop run on the GPU (``ppvector.data_utils.audio_batch``, ``ppv_audio_prep`` / ``ppv_audio_prep_reverb``); ``load_batch`` prepares
a whole batch with one launch sequence (decode on the host, then audio prep -> ragged front end -> SpecAugment), which is what
``PPVectorTrainer.train`` uses.  With reverb the utterance grows by the response's length - 1 before the crop, as in the reference, so
the crop decision and its random start are taken on the reverberant length."""
import random

import numpy as np
import torch
from tqdm import tqdm

from ppvector.data_utils.audio import AudioSegment
from ppvector.data_utils.audio_batch import WaveAugmentor, augmented_len, prepare_batch
from ppvector.data_utils.featurizer import AudioFeaturizer
from ppvector.data_utils.spec_aug import SpecAugmentor


class PPVectorDataset(torch.utils.data.Dataset):
    def __init__(self, data_list_path, audio_featurizer: AudioFeaturizer, max_duration=3, min_duration=0.5, mode='train',
                 sample_rate=16000, aug_conf=None, num_speakers=None, use_dB_normalization=True, target_dB=-20,
                 device='cuda'):
        super().__init__()
        assert mode in ['train', 'eval', 'extract_feature']
        self.spec_augment = None
        self.wave_augment = None
        if mode == 'train' and aug_conf is not None:  # reader.py:143-151
            conf = dict(aug_conf) if isinstance(aug_conf, dict) else dict(vars(aug_conf))
            self.wave_augment = WaveAugmentor(conf, num_speakers=num_speakers, sample_rate=sample_rate, device=device)
            sa = conf.get('spec_aug')
            if sa is not None:
                self.spec_augment = SpecAugmentor(**(dict(sa) if isinstance(sa, dict) else dict(vars(sa))))
        self.data_list_path = data_list_path
        self.max_duration, self.min_duration, self.mode = max_duration, min_duration, mode
        self._target_sample_rate = sample_rate
        self._use_dB_normalization, self._target_dB = use_dB_normalization, target_dB
        self.num_speakers = num_speakers
        self.audio_featurizer = audio_featurizer
        self.device = torch.device(device)
        # frame count of a max_duration crop (reader.py:115-119 featurises random noise just to learn T)
        self.max_feature_len = audio_featurizer.num_frames(int(self.max_duration * self._target_sample_rate))
        with open(self.data_list_path, 'r', encoding='utf-8') as f:
            self.lines = [ln for ln in f.readlines() if ln.strip()]
        self.labels = [np.int64(line.strip().split('\t')[1]) for line in self.lines]
        if self.mode == 'eval':
            self.sort_list()

    def decode(self, idx):
        """(float32 samples at the target rate, label), or (None, label) for a .npy feature entry.  reader.py:85-93"""
        data_path, spk_id = self.lines[idx].strip().split('\t')
        if data_path.endswith('.npy'):
            return None, int(spk_id)
        seg = AudioSegment.from_file(data_path)
        if self.mode in ('train', 'extract_feature') and seg.duration < self.min_duration:
            return self.decode(idx + 1 if idx < len(self.lines) - 1 else 0)  # reader.py:88-89
        if seg.sample_rate != self._target_sample_rate:
            seg.resample(self._target_sample_rate)
        return seg.samples, int(spk_id)

    def _plan(self, x, spk_id):
        """The random decisions of one utterance, in the reference's order: augmentation draws (reader.py:153-163), then the crop start
        (reader.py:100-101) on the augmented length (speed-changed, plus a drawn room response's length - 1).
        -> (draw dict or None, (crop_start, crop_len or None), label)"""
        draw = self.wave_augment.draw(x.shape[0], spk_id) if self.wave_augment is not None else None
        new_len = augmented_len(x.shape[0], draw)
        crop = (0, None)
        n = int(self.max_duration * self._target_sample_rate)
        if self.mode != 'extract_feature' and new_len / float(self._target_sample_rate) > self.max_duration:
            crop = (random.randint(0, new_len - n) if self.mode == 'train' else 0, n)
        return draw, crop, (draw['spk_id'] if draw else spk_id)

    def _banks(self):
        """(noise bank, room response bank) of the wave augmentor, None where absent"""
        if self.wave_augment is None:
            return None, None
        return self.wave_augment.noise_bank, self.wave_augment.rir_bank

    def _npy_feature(self, idx):
        feature = np.load(self.lines[idx].strip().split('\t')[0])
        if feature.shape[0] > self.max_feature_len:
            s = random.randint(0, feature.shape[0] - self.max_feature_len) if self.mode == 'train' else 0
            feature = feature[s:s + self.max_feature_len, :]
        return torch.from_numpy(feature.astype(np.float32)).to(self.device)

    def load_batch(self, indices):
        """A whole batch with one launch sequence: -> (features [B,Tmax,F] CUDA, labels [B] int64, input_lens [B] int64), the output of
        collate_fn([self[i] for i in indices]) (collate_fn.py:5-23).  Lists that mix .npy features in fall back to the per-item path."""
        from ppvector.data_utils.collate_fn import collate_fn
        decoded = [self.decode(int(i)) for i in indices]
        if any(x is None for x, _ in decoded):
            return collate_fn([self[int(i)] for i in indices])
        plans = [self._plan(x, spk) for x, spk in decoded]
        noise_bank, rir_bank = self._banks()
        wav, lens = prepare_batch([x for x, _ in decoded], [p[0] for p in plans], [p[1] for p in plans], target_db=self._target_dB,
                                  normalize=self._use_dB_normalization, noise_bank=noise_bank, device=self.device, rir_bank=rir_bank)
        feats, frames = self.audio_featurizer.forward_ragged(wav, lens)
        if self.mode == 'train' and self.spec_augment is not None:  # reader.py:105-107
            feats = self.spec_augment(feats, num_frames=frames)
        return feats, torch.tensor([p[2] for p in plans], dtype=torch.int64), torch.tensor(frames, dtype=torch.int64)

    def __getitem__(self, idx):
        x, spk_id = self.decode(idx)
        if x is None:
            feature = self._npy_feature(idx)
        else:
            draw, crop, spk_id = self._plan(x, spk_id)
            noise_bank, rir_bank = self._banks()
            wav, lens = prepare_batch([x], [draw], [crop], target_db=self._target_dB, normalize=self._use_dB_normalization,
                                      noise_bank=noise_bank, device=self.device, rir_bank=rir_bank)
            feature = self.audio_featurizer(wav[0, :lens[0]]).squeeze(0)
        if self.mode == 'train' and self.spec_augment is not None:  # reader.py:105-107
            feature = self.spec_augment(feature)
        return feature, spk_id

    def __len__(self):
        return len(self.lines)

    def sort_list(self):
        """reader.py:122-138: eval lists are processed in order of increasing duration"""
        lengths = []
        for line in tqdm(self.lines, desc=f"对列表[{self.data_list_path}]进行长度排序"):
            data_path = line.split('\t')[0]
            if data_path.endswith('.npy'):
                lengths.append(np.load(data_path, mmap_mode='r').shape[0])
            else:
                lengths.append(AudioSegment.from_file(data_path).duration)
        order = np.argsort(lengths, kind='stable')
        self.lines = [self.lines[i] for i in order]
        self.labels = [self.labels[i] for i in order]
