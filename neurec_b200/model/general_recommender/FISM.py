"""FISM: factored item similarity models (Kabbur et al., KDD 2013).

Plug-in mirror of the reference's model/general_recommender/FISM.py:17-180 on the sm_90a kernels:
  * variables in the reference's order (:55-64): c1 [I, d] and embedding_Q [I, d] drawn with init_method from one
    generator seeded 2017, bias [I] zeros.  The reference's pad row c2 is never materialised: histories are rows of a
    CSR and the kernels skip nothing but the excluded item;
  * the epoch is the reference's instance generator (util/data_generator.py) restated as a fixed layout uploaded
    once, with new numbers every epoch from the process-wide sampler stream: the negatives are
    nrc_sample_negatives(seed, epoch) outside each user's train items, the order is nrc_shuffle_perm(seed, epoch)
    (DataIterator(shuffle=True)).  The batch loop (:119-138) is ``nrc_fism_train_epoch``;
      pointwise (data_generator.py:29-54): per user ascending, per train item i in row order, num_neg negatives
        (history = the whole row, n = |R_u| + 1 [sic], label 0), then the positive (history = the row without i,
        n = |R_u|, label 1);
      pairwise (data_generator.py:5-27): that generator removes items from the list it enumerates and appends the
        list itself, so a user with |R_u| > 1 gets the items at the even positions 0, 2, 4, ... of its row as
        positives, the k-th negative draw as the k-th negative, and one history for both sides of every sample: the
        items at the odd positions.  n = |R_u|, n_j = |R_u| + 1.  This is what the reference trains on;
  * predict (:154-180) is ``nrc_fism_query`` over the user's whole train row and ``nrc_fism_scores`` (n = |R_u|);
    with candidate lists, the candidates' scores are read from that row.  A user without train items raises KeyError
    (self.train_dict[u]).
Deviation: the reference's pointwise generator raises KeyError for a user without train items; here such a user
contributes no instance.
"""
from time import time

import numpy as np
import scipy.sparse as sp
import torch

from ... import ops
from ...data import sampler as _sampler
from ...util import timer
from ..AbstractRecommender import AbstractRecommender
from .._engine import OptimizerState, get_initializer

SEED = 2018
PAIRWISE_LOSSES = ("bpr", "hinge", "square")          # util/learner.py:17-29
POINTWISE_LOSSES = ("cross_entropy", "square")        # util/learner.py:31-41


def pointwise_layout(ptr, idx, num_neg):
    """The pointwise instances in the generator's order before the negatives are drawn: (rows, excl, num, labels)
    int32 / f32 [P (num_neg + 1)], with excl = the positive item in its slot and -1 in the negative slots."""
    deg = np.diff(ptr)
    k = num_neg + 1
    users = np.repeat(np.arange(len(deg), dtype=np.int32), deg)
    pos_slot = np.tile(np.arange(k) == num_neg, len(users))
    n = np.repeat(deg[users], k).astype(np.int32)
    excl = np.where(pos_slot, np.repeat(np.asarray(idx, np.int32), k), -1).astype(np.int32)
    return np.repeat(users, k), excl, np.where(pos_slot, n, n + 1).astype(np.int32), pos_slot.astype(np.float32)


def pairwise_layout(ptr, idx):
    """The pairwise instances as the generator produces them (see the module docstring): the odd-position CSR
    (hist_ptr int64, hist_idx int32) and per sample (rows, items, num, num_neg) int32."""
    deg = np.diff(ptr)
    pos = np.arange(len(idx)) - np.repeat(ptr[:-1], deg)
    row = np.repeat(np.arange(len(deg)), deg)
    many = np.repeat(deg > 1, deg)
    odd, even = many & (pos % 2 == 1), many & (pos % 2 == 0)
    hist_ptr = np.zeros(len(deg) + 1, np.int64)
    hist_ptr[1:] = np.cumsum(np.bincount(row[odd], minlength=len(deg)))
    num = deg[row[even]].astype(np.int32)
    return (hist_ptr, np.asarray(idx, np.int32)[odd]), (row[even].astype(np.int32), np.asarray(idx, np.int32)[even],
                                                        num, (num + 1).astype(np.int32))


class FISM(AbstractRecommender):
    def __init__(self, sess, dataset, conf):
        super(FISM, self).__init__(dataset, conf)
        self.batch_size = conf["batch_size"]
        self.num_epochs = conf["epochs"]
        self.embedding_size = conf["embedding_size"]
        self.regs = conf["regs"]
        self.lambda_bilinear = self.regs[0]
        self.gamma_bilinear = self.regs[1]
        self.alpha = conf["alpha"]
        self.num_negatives = conf["num_neg"]
        self.learning_rate = conf["learning_rate"]
        self.learner = conf["learner"]
        self.topK = conf["topk"]
        self.loss_function = conf["loss_function"]
        self.is_pairwise = conf["is_pairwise"]
        self.init_method = conf["init_method"]
        self.stddev = conf["stddev"]
        self.verbose = conf["verbose"]
        self.num_users = dataset.num_users
        self.num_items = dataset.num_items
        self.dataset = dataset
        self.sess = sess
        train = sp.csr_matrix(dataset.train_matrix)
        # csr_to_user_dict keeps each row in the matrix's own order; the sampler's exclusion list is the sorted row
        self._ptr = train.indptr.astype(np.int64)
        self._idx = train.indices.astype(np.int32)
        self._n = 0
        self._step_loss = None

    def build_graph(self):
        loss = self.loss_function.lower()
        if loss not in (PAIRWISE_LOSSES if self.is_pairwise is True else POINTWISE_LOSSES):
            raise Exception("please choose a suitable loss function")      # learner.py:27-28, 39-40
        self._loss = loss
        d, ni = self.embedding_size, self.num_items
        gen = torch.Generator().manual_seed(2017)
        init = get_initializer(self.init_method, self.stddev, gen)
        self.c1 = init([ni, d]).cuda()                                       # FISM.py:58-59
        self.embedding_Q = init([ni, d]).cuda()                              # FISM.py:62-63
        self.bias = torch.zeros(ni, dtype=torch.float32, device="cuda")      # FISM.py:64
        self.opt = OptimizerState(self.learner, self.learning_rate)
        self._grads = [torch.zeros_like(t) for t in self.tables()]
        slots = [self.opt.slots_like(t) for t in self.tables()]
        self._slots0, self._slots1 = [s[0] for s in slots], [s[1] for s in slots]
        z = lambda n: torch.zeros(n, dtype=torch.int32, device="cuda")
        self._touched = (z(ni), z(ni))
        self._init_instances()

    def tables(self):
        return [self.c1, self.embedding_Q, self.bias]

    def _init_instances(self):
        t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()
        ptr, idx = self._ptr, self._idx
        sorted_idx = np.concatenate([np.sort(idx[ptr[u]:ptr[u + 1]]) for u in range(self.num_users)] or
                                    [np.zeros(0, np.int32)]).astype(np.int32)
        self._train_ptr, self._train_idx, self._train_sorted = t(ptr), t(idx), t(sorted_idx)
        if self.is_pairwise is True:
            (hp, hi), (rows, items, num, num_neg) = pairwise_layout(ptr, idx)
            self._hist_ptr, self._hist_idx = t(hp), t(hi)
            self._rows, self._items, self._num, self._num_neg = t(rows), t(items), t(num), t(num_neg)
            self._excl = None
        else:
            rows, excl, num, labels = pointwise_layout(ptr, idx, self.num_negatives)
            self._hist_ptr, self._hist_idx = self._train_ptr, self._train_idx
            self._rows, self._excl, self._num, self._labels = t(rows), t(excl), t(num), t(labels)
            self._pos_users = t(np.repeat(np.arange(self.num_users, dtype=np.int32), np.diff(ptr)))
            self._pos_items = t(idx)
        self._n = int(self._rows.numel())

    def device_epoch(self, epoch):
        """Epoch `epoch` of the generator (FISM.py:112-118) as CUDA tensors in DataIterator's shuffled order:
        (rows, excl or None, num, items, third, num_neg or None); third is the negatives (pairwise) or the labels."""
        g = lambda a, perm: ops.gather_rows_i32(a, perm)
        perm = ops.shuffle_perm(self._n, SEED, epoch)
        if self.is_pairwise is True:
            neg = ops.sample_negatives(self._train_ptr, self._train_sorted, self._rows, 1, self.num_items, SEED,
                                       epoch).view(-1)
            return (g(self._rows, perm), None, g(self._num, perm), g(self._items, perm), g(neg, perm),
                    g(self._num_neg, perm))
        neg = ops.sample_negatives(self._train_ptr, self._train_sorted, self._pos_users, self.num_negatives,
                                   self.num_items, SEED, epoch)
        items = torch.cat([neg, self._pos_items.view(-1, 1)], 1).view(-1)
        labels = g(self._labels.view(torch.int32), perm).view(torch.float32)
        return g(self._rows, perm), g(self._excl, perm), g(self._num, perm), g(items, perm), labels, None

    def _train_epoch(self):
        """One epoch (new negatives and a new order) through nrc_fism_train_epoch; returns the summed batch losses."""
        epoch = _sampler._EPOCH_COUNTER_NEXT()
        rows, excl, num, items, third, num_neg = self.device_epoch(epoch)
        steps = (self._n + self.batch_size - 1) // self.batch_size
        if self._step_loss is None or self._step_loss.numel() < steps:
            self._step_loss = torch.empty(max(steps, 1), dtype=torch.float32, device="cuda")
        ops.fism_train_epoch(*self.tables(), self._hist_ptr, self._hist_idx, rows, excl, num, items, third, num_neg,
                             self.batch_size, self.is_pairwise is True, self._loss, self.alpha, self.lambda_bilinear,
                             self.gamma_bilinear, self.opt.kind, self.opt.lr_t(steps), self.opt.hyper, self._grads,
                             self._touched, self._slots0, self._slots1, self.opt.take_stamps(steps), self._step_loss)
        return float(self._step_loss[:steps].sum().item())

    def train_model(self):
        self.logger.info(self.evaluator.metrics_info())
        for epoch in range(1, self.num_epochs + 1):
            training_start_time = time()
            total_loss = self._train_epoch()
            self.logger.info("[iter %d : loss : %f, time: %f]" % (epoch, total_loss / max(self._n, 1),
                                                                 time() - training_start_time))
            if epoch % self.verbose == 0:
                self.logger.info("epoch %d:\t%s" % (epoch, self.evaluate()))

    @timer
    def evaluate(self):
        return self.evaluator.evaluate(self)

    def predict(self, user_ids, candidate_items_userids=None):
        """[len(user_ids), num_items] CUDA scores; with candidate lists, one score array per user."""
        users = np.asarray(user_ids, dtype=np.int64).reshape(-1)
        known = (users >= 0) & (users < self.num_users)
        deg = np.diff(self._ptr)
        known[known] = deg[users[known]] > 0
        if not known.all():
            raise KeyError(int(users[np.argmin(known)]))                    # self.train_dict[u] (FISM.py:159, 172)
        dev_users = torch.from_numpy(users.astype(np.int32)).cuda()
        ratings = ops.fism_scores(self.c1, self.embedding_Q, self.bias, self._train_ptr, self._train_idx, dev_users,
                                  self.alpha)
        if candidate_items_userids is not None:
            host = ratings.cpu().numpy()
            ratings = [host[r][np.asarray(items, dtype=np.int64)] for r, items in enumerate(candidate_items_userids)]
        return ratings
