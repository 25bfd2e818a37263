"""What the sequential embedding models share (model/sequential_recommender/FPMC.py, TransRec.py, HRM.py, NPE.py).

``SeqTableRecommender``: the by-time train sequences, the variables' initialisation in the reference's order, the
optimizer bookkeeping of one fused epoch call, evaluate and predict.  Each model reads its own configuration keys.
``SeqEmbeddingRecommender`` adds what FPMC and TransRec share: the reference's constructor keys, the time-ordered
sampler of the chosen mode at high_order = 1 and the per-user last item that predict scores from.
``SeqWindowRecommender`` adds what HRM and NPE share: the pointwise sampler over windows of high_order items, the
reference's log lines and the per-user predict windows."""
from time import time

import numpy as np
import torch

from ...data.sampler import TimeOrderPairwiseSampler, TimeOrderPointwiseSampler
from ...util import timer
from ...util.tool import csr_to_user_dict_bytime
from ..AbstractRecommender import SeqAbstractRecommender
from .._engine import OptimizerState, get_initializer

PAIRWISE_LOSSES = ("bpr", "hinge", "square")          # util/learner.py:17-29
POINTWISE_LOSSES = ("cross_entropy", "square")        # util/learner.py:31-41


class SeqTableRecommender(SeqAbstractRecommender):
    """The dataset side of every sequential embedding model.  A subclass reads learning_rate, learner, init_method,
    stddev and batch_size (with its other keys) from the configuration and defines tables(), _run_epoch(),
    _device_rows() and _scores()."""

    def __init__(self, sess, dataset, conf):
        super(SeqTableRecommender, self).__init__(dataset, conf)
        self.num_users = dataset.num_users
        self.num_items = dataset.num_items
        self.dataset = dataset
        self.train_matrix = dataset.train_matrix
        self.train_dict = csr_to_user_dict_bytime(dataset.time_matrix, dataset.train_matrix)
        self.sess = sess
        self._data_iter = None
        self._step_loss = None

    def _init_tables(self, shapes, methods=None):
        """get_initializer on generator 2017, in the reference's variable order (tf.set_random_seed(2017)).  methods
        names each shape's initialiser (default: init_method for every shape); all draw from the one generator."""
        generator = torch.Generator().manual_seed(2017)
        methods = [self.init_method] * len(shapes) if methods is None else methods
        inits = {m: get_initializer(m, self.stddev, generator) for m in set(methods)}
        return [inits[m](s).cuda() for m, s in zip(methods, shapes)]

    def _init_training(self, tables):
        self.opt = OptimizerState(self.learner, self.learning_rate)
        self._grads = [torch.zeros_like(t) for t in tables]
        slots = [self.opt.slots_like(t) for t in tables]
        self._slots0, self._slots1 = [s[0] for s in slots], [s[1] for s in slots]

    def _epoch_buffers(self, n):
        steps = (n + self.batch_size - 1) // self.batch_size
        if self._step_loss is None or self._step_loss.numel() < steps:
            self._step_loss = torch.empty(max(steps, 1), dtype=torch.float32, device="cuda")
        return steps, self.opt.lr_t(steps), self.opt.take_stamps(steps)

    def _train_epoch(self):
        """One epoch of the sampler (a new order and new negatives) through the model's fused epoch call; returns the
        summed batch losses."""
        users, recent, items, third = self.data_iter().device_epoch()
        steps = self._run_epoch(users, recent, items, third)
        return float(self._step_loss[:steps].sum().item())

    @timer
    def evaluate(self):
        return self.evaluator.evaluate(self)

    def predict(self, user_ids, candidate_items_userids=None):
        """[len(user_ids), num_items] CUDA scores; with candidate lists, one score array per user."""
        ratings = self._scores(*self._device_rows(user_ids))
        if candidate_items_userids is not None:
            host = ratings.cpu().numpy()
            ratings = [host[r][np.asarray(items, dtype=np.int64)] for r, items in enumerate(candidate_items_userids)]
        return ratings


class SeqEmbeddingRecommender(SeqTableRecommender):
    def __init__(self, sess, dataset, conf):
        super(SeqEmbeddingRecommender, self).__init__(sess, dataset, conf)
        self.learning_rate = conf["learning_rate"]
        self.embedding_size = conf["embedding_size"]
        self.learner = conf["learner"]
        self.loss_function = conf["loss_function"]
        self.is_pairwise = conf["is_pairwise"]
        self.num_epochs = conf["epochs"]
        self.reg_mf = conf["reg_mf"]
        self.batch_size = conf["batch_size"]
        self.init_method = conf["init_method"]
        self.stddev = conf["stddev"]
        self.verbose = conf["verbose"]
        self.num_negatives = conf["num_neg"]
        # the last train item of every user (train_dict[u][-1]), -1 for a user without train items
        last = np.full(self.num_users, -1, dtype=np.int32)
        for u, seq in self.train_dict.items():
            last[u] = seq[-1]
        self._last = last

    def _check_loss(self):
        loss = self.loss_function.lower()
        if loss not in (PAIRWISE_LOSSES if self.is_pairwise is True else POINTWISE_LOSSES):
            raise Exception("please choose a suitable loss function")      # learner.py:27-28, 39-40
        self._loss = loss

    def data_iter(self):
        """The reference's sampler of the chosen mode (FPMC.py:99-105, TransRec.py:112-118), built once."""
        if self._data_iter is None:
            if self.is_pairwise is True:
                self._data_iter = TimeOrderPairwiseSampler(self.dataset, high_order=1, neg_num=1,
                                                           batch_size=self.batch_size, shuffle=True)
            else:
                self._data_iter = TimeOrderPointwiseSampler(self.dataset, high_order=1, neg_num=self.num_negatives,
                                                            batch_size=self.batch_size, shuffle=True)
        return self._data_iter

    def _device_rows(self, user_ids):
        users = np.asarray(user_ids, dtype=np.int64).reshape(-1)
        known = (users >= 0) & (users < self.num_users)
        last = np.where(known, self._last[np.where(known, users, 0)], -1)
        if (last < 0).any():
            raise KeyError(int(users[np.argmax(last < 0)]))             # train_dict[user_id] (FPMC.py:145)
        users = users.astype(np.int32)
        return torch.from_numpy(users).cuda(), torch.from_numpy(last).cuda()


def predict_windows(train_dict, num_users, high_order):
    """Every user's predict window train_dict[u][len(seq) - high_order:] as Python slices it (HRM.py:140-144,
    NPE.py:119-123): the last high_order items, or for a user with fewer than high_order train items the shorter
    seq[max(0, 2 * len - high_order):].  -> (recent int32 [num_users, high_order] padded with 0, length int32
    [num_users], 0 for a user without train items)."""
    recent = np.zeros((num_users, high_order), dtype=np.int32)
    length = np.zeros(num_users, dtype=np.int32)
    for u, seq in train_dict.items():
        w = seq[len(seq) - high_order:]
        recent[u, :len(w)] = w
        length[u] = len(w)
    return recent, length


class SeqWindowRecommender(SeqTableRecommender):
    """HRM and NPE: pointwise only, one TimeOrderPointwiseSampler(high_order, num_neg) epoch per fused call.  A
    subclass also reads high_order and num_neg."""

    def _check_loss(self):
        loss = self.loss_function.lower()
        if loss not in POINTWISE_LOSSES:
            raise Exception("please choose a suitable loss function")      # learner.py:39-40
        self._loss = loss

    def _init_windows(self):
        recent, length = predict_windows(self.train_dict, self.num_users, self.high_order)
        self._recent_len_host = length
        self._recent = torch.from_numpy(recent).cuda()
        self._recent_len = torch.from_numpy(length).cuda()

    def data_iter(self):
        """The reference's sampler (HRM.py:106-108, NPE.py:86-88), built once."""
        if self._data_iter is None:
            self._data_iter = TimeOrderPointwiseSampler(self.dataset, high_order=self.high_order,
                                                        neg_num=self.num_negatives, batch_size=self.batch_size,
                                                        shuffle=True)
        return self._data_iter

    def train_model(self):
        self.logger.info(self.evaluator.metrics_info())
        data_iter = self.data_iter()
        for epoch in range(1, self.num_epochs + 1):
            num_training_instances = len(data_iter)       # the number of batches (HRM.py:111, NPE.py:90)
            training_start_time = time()
            total_loss = self._train_epoch()
            self.logger.info("[iter %d : loss : %f, time: %f]" %
                             (epoch, total_loss / num_training_instances, time() - training_start_time))
            if epoch % self.verbose == 0:
                self.logger.info("epoch %d:\t%s" % (epoch, self.evaluate()))

    def _device_rows(self, user_ids):
        users = np.asarray(user_ids, dtype=np.int64).reshape(-1)
        known = (users >= 0) & (users < self.num_users)
        length = np.where(known, self._recent_len_host[np.where(known, users, 0)], 0)
        if (length == 0).any():
            raise KeyError(int(users[np.argmax(length == 0)]))          # train_dict[user_id] (HRM.py:140)
        return (torch.from_numpy(users.astype(np.int32)).cuda(),)
