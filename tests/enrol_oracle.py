"""numpy restatement of the reference's enrolment database (ppvector/predict.py): the per-user means of __load_audio_db (:154-163),
register (:285-322), remove_user (:344-364) and __retrieval (:173-187), on in-memory embeddings.  Similarities are fp64; ranking ties
go to the lowest user index (numpy.argmax's first maximum).  The three deviations of PPVectorPredictor.register are restated here:
registering into an empty database works, an existing file is never overwritten, and there is no database-less register."""
import os

import numpy as np


class EnrolDB:
    def __init__(self, users_name=(), audio_feature=None, users_audio_path=()):
        """predict.py:154-163: the rows already embedded (in index order), then one mean per user in set() order."""
        self.users_name = list(users_name)
        self.users_audio_path = list(users_audio_path)
        self.audio_feature = None if audio_feature is None else np.asarray(audio_feature, dtype=np.float32)
        self.users_name_mean, self.audio_feature_mean = [], None
        for name in set(self.users_name):
            self.users_name_mean.append(name)
            feature = self._mean(name)[None]
            self.audio_feature_mean = feature if self.audio_feature_mean is None else np.vstack((self.audio_feature_mean, feature))

    def _mean(self, name):
        return self.audio_feature[[i for i, v in enumerate(self.users_name) if v == name]].mean(axis=0)

    def index(self):
        """the pickled index (predict.py:105-109)"""
        return {'users_name': self.users_name, 'faces_feature': self.audio_feature, 'users_image_path': self.users_audio_path}

    @staticmethod
    def next_path(db_path, user_name):
        """predict.py:298-302, except that an existing file is skipped: the smallest unused <n>.wav with n >= the file count."""
        user_dir = os.path.join(db_path, user_name)
        n = len(os.listdir(user_dir)) if os.path.exists(user_dir) else 0
        while os.path.exists(os.path.join(user_dir, f'{n}.wav')):
            n += 1
        return os.path.join(user_dir, f'{n}.wav').replace('\\', '/')

    def register(self, user_name, feature, audio_path):
        """predict.py:294-321 with the embedding and the file path given."""
        feature = np.asarray(feature, dtype=np.float32)
        self.audio_feature = feature[None] if self.audio_feature is None else np.vstack((self.audio_feature, feature))
        self.users_audio_path.append(audio_path)
        self.users_name.append(user_name)
        if user_name in self.users_name_mean:
            self.audio_feature_mean[self.users_name_mean.index(user_name)] = self._mean(user_name)
        else:
            self.users_name_mean.append(user_name)
            self.audio_feature_mean = feature[None] if self.audio_feature_mean is None else np.vstack((self.audio_feature_mean, feature))

    def remove_user(self, user_name):
        """predict.py:350-364 (without the directory removal)"""
        if user_name not in self.users_name:
            return False
        for index in sorted([i for i, v in enumerate(self.users_name) if v == user_name], reverse=True):
            del self.users_name[index]
            del self.users_audio_path[index]
            self.audio_feature = np.delete(self.audio_feature, index, axis=0)
        index = self.users_name_mean.index(user_name)
        del self.users_name_mean[index]
        self.audio_feature_mean = np.delete(self.audio_feature_mean, index, axis=0)
        return True

    def similarities(self, queries):
        """fp64 cosine [Q, users] of the queries against the means (a zero-norm row scores 0)."""
        q = np.asarray(queries, dtype=np.float64)
        m = np.asarray(self.audio_feature_mean, dtype=np.float64)
        qn = np.linalg.norm(q, axis=1, keepdims=True)
        mn = np.linalg.norm(m, axis=1, keepdims=True)
        return (q / np.where(qn > 0, qn, 1.0)) @ (m / np.where(mn > 0, mn, 1.0)).T

    def retrieval(self, queries, threshold):
        """predict.py:173-187: [name, round(sim, 5)] of the arg-max per query, [None, None] under the threshold."""
        out = []
        for s in self.similarities(queries):
            i = int(np.argmax(s))
            out.append([self.users_name_mean[i], round(float(s[i]), 5)] if s[i] >= threshold else [None, None])
        return out


def topk(sim, k):
    """-> (idx [Q, k], sim [Q, k]): descending, equal similarities lowest index first."""
    sim = np.asarray(sim)
    order = np.lexsort((np.broadcast_to(np.arange(sim.shape[1]), sim.shape), -sim), axis=1)[:, :k]
    return order, np.take_along_axis(sim, order, axis=1)
