"""Caser: convolutional sequence embedding over the last seq_L items.

Plug-in mirror of the reference's model/sequential_recommender/Caser.py:17-209 on the sm_90a kernels:
  * variables in the reference's creation order (:37-68, then the layers as build_graph first calls them): P [U, d],
    E [I, d] (+ the zero pad row at id I), W2 [I, 2d], b2 [I] (zeros), then the dense block (Kv, bv, Kh_h, bh_h for
    h = 1..L, W1, b1; layout in ops.caser_dense_floats).  Weights draw glorot-uniform with TF's fans from one
    generator seeded 2017; biases are zeros;
  * _generate_sequences (:144-172) is restated in numpy and its instances are uploaded once.  Every epoch draws its
    number from the process-wide sampler stream: the negatives are nrc_sample_negatives(seed, epoch) outside each
    user's train items, the order is nrc_shuffle_perm(seed, epoch) (DataIterator(shuffle=True), :130-131), and the
    batch loop (:132-139) is ``nrc_caser_train_epoch`` with its dropout masks keyed by (seed, epoch, step);
  * predict (:194-209) is ``nrc_caser_query`` over every user's last seq_L train items (pre-padded with the pad id)
    and nrc_mf_scores against W2, without the biases, as the reference's all_logits.
A user with fewer than seq_T train items has the pad id among its positives; that target reads a zero row and a zero
bias (what TF's GPU gather returns for the out-of-range id): its loss term counts and it gets no gradient.
"""
import numpy as np
import torch

from ... import ops
from ...data import sampler as _sampler
from ._base import SeqTableRecommender

SEED = 2018


def generate_sequences(train_dict, seq_L, seq_T, num_items):
    """Caser._generate_sequences (Caser.py:144-172) on the by-time train dict: for users in ascending id order, a user
    with at least seq_L + seq_T items gets one instance per window, latest window first; a shorter user gets one
    instance pre-padded with num_items.  -> (users int32 [n], seqs int32 [n, seq_L], pos int32 [n, seq_T],
    test_seq {user: int32 [seq_L]})."""
    n = seq_L + seq_T
    users, seqs, test = [], [], {}
    for u in np.unique(list(train_dict.keys())):
        s = np.asarray(train_dict[u], dtype=np.int32)
        if len(s) >= n:
            w = np.lib.stride_tricks.sliding_window_view(s, n)[::-1]
        else:
            w = np.concatenate([np.full(n - len(s), num_items, np.int32), s])[None, :]
        test[int(u)] = w[0, -seq_L:].copy()
        users.append(np.full(len(w), u, dtype=np.int32))
        seqs.append(w)
    if not users:
        return np.zeros(0, np.int32), np.zeros((0, seq_L), np.int32), np.zeros((0, seq_T), np.int32), test
    w = np.concatenate(seqs)
    return (np.concatenate(users), np.ascontiguousarray(w[:, :seq_L]), np.ascontiguousarray(w[:, -seq_T:]), test)


def glorot_uniform(shape, generator):
    """TF's glorot_uniform with its fans: a 2-D [in, out] shape, or a conv kernel [kh, kw, in, out] with receptive
    field kh * kw."""
    receptive = int(np.prod(shape[:-2])) if len(shape) > 2 else 1
    fan_in, fan_out = shape[-2] * receptive, shape[-1] * receptive
    lim = (6.0 / (fan_in + fan_out)) ** 0.5
    return ((torch.rand(tuple(shape), generator=generator) * 2 - 1) * lim).to(torch.float32)


class Caser(SeqTableRecommender):
    def __init__(self, sess, dataset, conf):
        super(Caser, self).__init__(sess, dataset, conf)
        self.lr = conf["lr"]
        self.l2_reg = conf["l2_reg"]
        self.factors_num = conf["factors_num"]
        self.batch_size = conf["batch_size"]
        self.epochs = conf["epochs"]
        self.seq_L = conf["seq_L"]
        self.seq_T = conf["seq_T"]
        self.nv = conf["nv"]
        self.nh = conf["nh"]
        self.dropout = conf["dropout"]
        self.neg_samples = conf["neg_samples"]
        self.learner, self.learning_rate = "adam", self.lr

    def build_graph(self):
        d, L, ni = self.factors_num, self.seq_L, self.num_items
        gen = torch.Generator().manual_seed(2017)
        self.user_embeddings = glorot_uniform([self.num_users, d], gen).cuda()
        self.seq_item_embeddings = glorot_uniform([ni, d], gen).cuda()
        self.item_embeddings = glorot_uniform([ni, 2 * d], gen).cuda()
        self.item_biases = torch.zeros(ni, dtype=torch.float32, device="cuda")
        parts = [glorot_uniform([L, 1, 1, self.nv], gen).reshape(-1), torch.zeros(self.nv)]
        for h in range(1, L + 1):
            parts += [glorot_uniform([h, d, 1, self.nh], gen).reshape(-1), torch.zeros(self.nh)]
        F = self.nv * d + self.nh * L
        parts += [glorot_uniform([F, d], gen).reshape(-1), torch.zeros(d)]
        self.dense = torch.cat(parts).cuda()
        assert self.dense.numel() == ops.caser_dense_floats(d, L, self.nv, self.nh)
        self._init_training(self.tables())
        self._work = ops.caser_work(d, L, self.nv, self.nh, self.batch_size)
        self._init_sequences()

    def tables(self):
        return [self.user_embeddings, self.seq_item_embeddings, self.item_embeddings, self.item_biases, self.dense]

    def _init_sequences(self):
        users, seqs, pos, test = generate_sequences(self.train_dict, self.seq_L, self.seq_T, self.num_items)
        windows = np.full((self.num_users, self.seq_L), self.num_items, dtype=np.int32)
        known = np.zeros(self.num_users, dtype=bool)
        for u, w in test.items():
            windows[u] = w
            known[u] = True
        self._known = known
        t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()
        self._users, self._seqs, self._pos, self._windows = t(users), t(seqs), t(pos), t(windows)
        # the train CSR the negatives exclude (rows = sorted train items)
        ptr = np.zeros(self.num_users + 1, dtype=np.int64)
        for u, items in self.train_dict.items():
            ptr[u + 1] = len(items)
        ptr = np.cumsum(ptr)
        idx = np.zeros(max(int(ptr[-1]), 1), dtype=np.int32)
        for u, items in self.train_dict.items():
            idx[ptr[u]:ptr[u + 1]] = np.sort(np.asarray(items, dtype=np.int32))
        self._train_ptr, self._train_idx = t(ptr), t(idx)

    def device_epoch(self, epoch):
        """Epoch `epoch` of the reference's loop (Caser.py:129-131) as CUDA tensors: users, seqs, pos, neg in shuffled
        order, the negatives drawn per instance before the shuffle."""
        n = self._users.numel()
        neg = ops.sample_negatives(self._train_ptr, self._train_idx, self._users, self.neg_samples, self.num_items,
                                   SEED, epoch)
        perm = ops.shuffle_perm(n, SEED, epoch)
        return tuple(ops.gather_rows_i32(a, perm) for a in (self._users, self._seqs, self._pos, neg))

    def _train_epoch(self):
        """One epoch (a new order, new negatives and new masks) through nrc_caser_train_epoch; returns the summed
        batch data losses."""
        epoch = _sampler._EPOCH_COUNTER_NEXT()
        users, seqs, pos, neg = self.device_epoch(epoch)
        steps, lr_t, _ = self._epoch_buffers(users.numel())
        ops.caser_train_epoch(*self.tables(), users, seqs, pos, neg, self.nv, self.nh, self.batch_size,
                              1.0 - self.dropout, self.l2_reg, SEED, epoch, lr_t, self.opt.hyper, self._grads,
                              self._slots0, self._slots1, self._work, self._step_loss)
        return float(self._step_loss[:steps].sum().item())

    def train_model(self):
        self.logger.info(self.evaluator.metrics_info())
        for epoch in range(self.epochs):
            self._train_epoch()
            self.logger.info("epoch %d:\t%s" % (epoch, self.evaluate()))

    def _device_rows(self, user_ids):
        users = np.asarray(user_ids, dtype=np.int64).reshape(-1)
        ok = (users >= 0) & (users < self.num_users)
        ok[ok] = self._known[users[ok]]
        if not ok.all():
            raise KeyError(int(users[np.argmin(ok)]))                     # self.user_test_seq[u] (Caser.py:198)
        return (torch.from_numpy(users.astype(np.int32)).cuda(),)

    def _scores(self, users):
        P, E, W2, _, dense = self.tables()
        return ops.caser_scores(P, E, W2, dense, users, self._windows, self.nv, self.nh)
