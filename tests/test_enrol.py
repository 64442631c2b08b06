"""CPU: the enrolment database's host side -- the float WAV writer, the infer_recognition.py option table, and the numpy enrolment
oracle (tests/enrol_oracle.py) against a line-by-line transcription of the reference's register / remove_user / means."""
import os

import numpy as np

from enrol_oracle import EnrolDB, topk


def test_wav_writer_round_trips_bitwise(tmp_path):
    from ppvector.data_utils.audio import AudioSegment, read_wav
    rng = np.random.default_rng(0)
    x = rng.uniform(-1, 1, 16000 * 3 + 7).astype(np.float32)
    x[:4] = [0.0, -0.0, 1.0, np.float32(1e-38)]
    path = str(tmp_path / 'a.wav')
    AudioSegment(x, 22050).to_wav_file(path)
    y, sr = read_wav(path)
    assert sr == 22050 and y.dtype == np.float32 and y.tobytes() == x.tobytes()
    with open(path, 'rb') as f:
        head = f.read(44)
    assert head[:4] == b'RIFF' and head[8:16] == b'WAVEfmt ' and int.from_bytes(head[20:22], 'little') == 3  # IEEE float
    assert int.from_bytes(head[4:8], 'little') == os.path.getsize(path) - 8


def test_cli_options_match_reference():
    """infer_recognition.py: the reference's options with its defaults (record_seconds aside: no microphone capture), then the
    file-input ones."""
    import infer_recognition as cli
    table = [(n, t, d) for n, t, d, _ in cli.OPTIONS]
    assert table[:5] == [('configs', str, 'configs/cam++.yml'), ('use_gpu', bool, True), ('audio_db_path', str, 'audio_db/'),
                         ('threshold', float, 0.6), ('model_path', str, 'models/CAMPPlus_Fbank/best_model/')]
    assert [n for n, _, _ in table[5:]] == ['action', 'audio_path', 'user_name', 'top_k']


class ReferenceDB:
    """predict.py:154-163, :294-321 and :350-364 transcribed line by line (file I/O and embedding left out)."""

    def __init__(self, users_name, audio_feature):
        self.users_name, self.audio_feature = list(users_name), audio_feature
        self.users_audio_path = [f'p{i}' for i in range(len(users_name))]
        self.users_name_mean, self.audio_feature_mean = [], None
        for name in set(self.users_name):
            indexes = [idx for idx, val in enumerate(self.users_name) if val == name]
            feature = self.audio_feature[indexes].mean(axis=0)
            if self.audio_feature_mean is None:
                self.audio_feature_mean = feature
            else:
                self.audio_feature_mean = np.vstack((self.audio_feature_mean, feature))
            self.users_name_mean.append(name)
        if len(self.audio_feature_mean.shape) == 1:
            self.audio_feature_mean = self.audio_feature_mean[np.newaxis, :]

    def register(self, feature, user_name, audio_path):
        if self.audio_feature is None:
            self.audio_feature = feature
        else:
            self.audio_feature = np.vstack((self.audio_feature, feature))
        self.users_audio_path.append(audio_path)
        self.users_name.append(user_name)
        if user_name in self.users_name_mean:
            index = self.users_name_mean.index(user_name)
            indexes = [idx for idx, val in enumerate(self.users_name) if val == user_name]
            feature = self.audio_feature[indexes].mean(axis=0)
            self.audio_feature_mean[index] = feature
        else:
            self.users_name_mean.append(user_name)
            self.audio_feature_mean = np.vstack((self.audio_feature_mean, feature))

    def remove_user(self, user_name):
        if user_name in self.users_name:
            indexes = [i for i in range(len(self.users_name)) if self.users_name[i] == user_name]
            for index in sorted(indexes, reverse=True):
                del self.users_name[index]
                del self.users_audio_path[index]
                self.audio_feature = np.delete(self.audio_feature, index, axis=0)
            index = self.users_name_mean.index(user_name)
            del self.users_name_mean[index]
            self.audio_feature_mean = np.delete(self.audio_feature_mean, index, axis=0)
            return True
        else:
            return False


def assert_same(ref, ora):
    assert ora.users_name == ref.users_name and ora.users_audio_path == ref.users_audio_path
    assert ora.users_name_mean == ref.users_name_mean
    assert ora.audio_feature.tobytes() == ref.audio_feature.tobytes() and ora.audio_feature.shape == ref.audio_feature.shape
    assert ora.audio_feature_mean.tobytes() == ref.audio_feature_mean.tobytes()


def test_oracle_equals_reference_transcription():
    rng = np.random.default_rng(5)
    names = ['ann', 'bo', 'ann', 'cy', 'bo', 'ann']
    feats = rng.normal(size=(len(names), 192)).astype(np.float32)
    ref = ReferenceDB(names, feats.copy())
    ora = EnrolDB(names, feats.copy(), [f'p{i}' for i in range(len(names))])
    assert_same(ref, ora)
    steps = [('reg', 'bo'), ('reg', 'dee'), ('rm', 'ann'), ('rm', 'zed'), ('reg', 'ann'), ('reg', 'dee'), ('rm', 'cy'), ('reg', 'bo')]
    for j, (op, name) in enumerate(steps):
        if op == 'reg':
            f = rng.normal(size=192).astype(np.float32)
            ref.register(f, name, f'r{j}')
            ora.register(name, f, f'r{j}')
        else:
            assert ora.remove_user(name) == ref.remove_user(name)
        assert_same(ref, ora)
    q = rng.normal(size=(5, 192)).astype(np.float32)
    sims = ora.similarities(q)
    res = ora.retrieval(q, -1.0)
    assert [r[0] for r in res] == [ora.users_name_mean[int(np.argmax(s))] for s in sims]


def test_oracle_register_into_empty_and_next_path(tmp_path):
    ora = EnrolDB()
    ora.register('ann', np.ones(4, np.float32), 'x')
    assert ora.users_name_mean == ['ann'] and ora.audio_feature_mean.shape == (1, 4)
    assert EnrolDB.next_path(str(tmp_path), 'ann').endswith('ann/0.wav')
    os.makedirs(tmp_path / 'ann')
    for n in ('0.wav', '2.wav'):
        (tmp_path / 'ann' / n).write_bytes(b'')
    assert EnrolDB.next_path(str(tmp_path), 'ann').endswith('ann/3.wav')  # the reference's len(listdir) = 2 would overwrite 2.wav


def test_topk_ties_lowest_index_first():
    s = np.array([[0.5, 0.9, 0.9, 0.1, 0.9]])
    idx, val = topk(s, 4)
    assert idx.tolist() == [[1, 2, 4, 0]] and val.tolist() == [[0.9, 0.9, 0.9, 0.5]]
