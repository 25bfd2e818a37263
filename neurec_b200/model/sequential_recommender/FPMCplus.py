"""FPMCplus: FPMC with attention over the window of recent items, conditioned on the candidate item.

Plug-in mirror of the reference's model/sequential_recommender/FPMCplus.py:16-205 on the sm_90a kernels:
  * tables UI [users, d], IU, IL, LI [items, d] and the attention MLP W [3d, w], b [1, w], h [w, 1] (:53-71);
    e_k = <h, tanh([UI_u, IL_i, LI_{l_k}] W + b)>, a = exp(e) / sum exp(e) over the window, and
    x(u, w, i) = <UI_u, IU_i> + <IL_i, sum_k a_k LI_{l_k}> (:73-106);
  * the epoch is TimeOrderPairwiseSampler(high_order) or TimeOrderPointwiseSampler(high_order, num_neg)'s device
    epoch (:134-140) and the batch loop (:141-171) is ``nrc_fpmcplus_train_epoch``: per batch the fused gradient
    kernel, the fixed-order sum of W's, b's and h's dense gradients, and one TF-1.12 optimizer launch over all seven
    variables;
  * predict (:177-205) is ``nrc_fpmcplus_scores`` over every item, from every user's last high_order train items by
    time.  A user with fewer train items gets the shorter window Python's slice gives, and the softmax runs over it
    (the reference's predict fails with a shape error there); at high_order = 1 the window is one item (the
    reference's graph is ill-formed at 1, where the sampler's window is [batch]).
"""
import torch

from ... import ops
from ._base import PAIRWISE_LOSSES, POINTWISE_LOSSES, SeqWindowRecommender
from ...data.sampler import TimeOrderPairwiseSampler, TimeOrderPointwiseSampler


class FPMCplus(SeqWindowRecommender):
    def __init__(self, sess, dataset, conf):
        super(FPMCplus, self).__init__(sess, dataset, conf)
        self.learning_rate = conf["learning_rate"]
        self.embedding_size = conf["embedding_size"]
        self.weight_size = conf["weight_size"]
        self.learner = conf["learner"]
        self.loss_function = conf["loss_function"]
        self.is_pairwise = conf["is_pairwise"]
        self.num_epochs = conf["epochs"]
        self.reg_mf = conf["reg_mf"]
        self.reg_w = conf["reg_w"]
        self.batch_size = conf["batch_size"]
        self.high_order = conf["high_order"]
        self.verbose = conf["verbose"]
        self.embed_init_method = conf["embed_init_method"]
        self.weight_init_method = conf["weight_init_method"]
        self.stddev = float(conf["stddev"])
        self.num_negatives = conf["num_neg"]

    def _check_loss(self):
        loss = self.loss_function.lower()
        if loss not in (PAIRWISE_LOSSES if self.is_pairwise is True else POINTWISE_LOSSES):
            raise Exception("please choose a suitable loss function")      # learner.py:27-28, 39-40
        self._loss = loss

    def data_iter(self):
        """The reference's sampler of the chosen mode (FPMCplus.py:134-140), built once."""
        if self._data_iter is None:
            if self.is_pairwise is True:
                self._data_iter = TimeOrderPairwiseSampler(self.dataset, high_order=self.high_order, neg_num=1,
                                                           batch_size=self.batch_size, shuffle=True)
            else:
                self._data_iter = TimeOrderPointwiseSampler(self.dataset, high_order=self.high_order,
                                                            neg_num=self.num_negatives, batch_size=self.batch_size,
                                                            shuffle=True)
        return self._data_iter

    def build_graph(self):
        self._check_loss()
        d, w, ni = self.embedding_size, self.weight_size, self.num_items
        emb, wgt = self.embed_init_method, self.weight_init_method
        (self.embeddings_UI, self.embeddings_IU, self.embeddings_IL, self.embeddings_LI, self.W,
         self.b) = self._init_tables([[self.num_users, d], [ni, d], [ni, d], [ni, d], [3 * d, w], [1, w]],
                                     [emb, emb, emb, emb, wgt, wgt])
        self.h = torch.ones((w, 1), dtype=torch.float32, device="cuda")
        self._init_training(self.tables())
        z = lambda n: torch.zeros(n, dtype=torch.int32, device="cuda")
        self._touched = (z(self.num_users), z(ni), z(ni))
        self._work = ops.fpmcplus_work(d, w, self.high_order, self.batch_size)
        self._init_windows()

    def tables(self):
        return [self.embeddings_UI, self.embeddings_IU, self.embeddings_IL, self.embeddings_LI, self.W, self.b,
                self.h]

    def _run_epoch(self, users, recent, items, third):
        steps, lr_t, first_stamp = self._epoch_buffers(users.numel())
        ops.fpmcplus_train_epoch(*self.tables(), users, recent, items, third, self.batch_size,
                                 self.is_pairwise is True, self._loss, self.reg_mf, self.reg_w, self.opt.kind, lr_t,
                                 self.opt.hyper, self._grads, self._touched, self._slots0, self._slots1, first_stamp,
                                 self._work, self._step_loss)
        return steps

    def _scores(self, users):
        return ops.fpmcplus_scores(*self.tables(), users, self._recent, self._recent_len)
