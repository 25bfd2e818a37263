"""NPE: neural personalized embedding (Nguyen et al., IJCAI 2018).

Plug-in mirror of the reference's model/sequential_recommender/NPE.py:16-142 on the sm_90a kernels:
  * three tables UI [users, d], IU and IL [items, d] (:44-52); with c the sum of IL over the window of the user's
    high_order previous items, x(u, w, i) = <relu(UI_u), relu(IU_i)> + <relu(IU_i), relu(c)> (:54-65);
  * pointwise only: the epoch is TimeOrderPointwiseSampler(high_order, num_neg)'s device epoch (:86-88) and the batch
    loop (:89-105) is ``nrc_npe_train_epoch``: per batch the fused gradient kernel and one TF-1.12 optimizer launch
    over UI, IU and IL;
  * predict (:114-142) is ``nrc_npe_query`` + ``nrc_mf_scores``: rows relu(UI_u) + relu(c) against relu(IU), from
    every user's last high_order train items by time (fewer when the user has fewer).
high_order must be at least 2: at 1 the sampler's window is [batch], and the reference's reduce_sum(axis=1) then sums
the embedding axis instead of the window, which makes its graph ill-formed.
"""
import torch

from ... import ops
from ._base import SeqWindowRecommender


class NPE(SeqWindowRecommender):
    def __init__(self, sess, dataset, conf):
        super(NPE, self).__init__(sess, dataset, conf)
        self.learning_rate = conf["learning_rate"]
        self.embedding_size = conf["embedding_size"]
        self.learner = conf["learner"]
        self.loss_function = conf["loss_function"]
        self.num_epochs = conf["epochs"]
        self.reg = conf["reg"]
        self.batch_size = conf["batch_size"]
        self.high_order = conf["high_order"]
        self.verbose = conf["verbose"]
        self.num_negatives = conf["num_neg"]
        self.init_method = conf["init_method"]
        self.stddev = conf["stddev"]
        if self.high_order < 2:
            raise ValueError("NPE needs high_order >= 2: with one recent item the window is [batch] and "
                             "reduce_sum(axis=1) would sum the embedding axis instead of the window (NPE.py:61)")

    def build_graph(self):
        self._check_loss()
        d = self.embedding_size
        self.embeddings_UI, self.embeddings_IU, self.embeddings_IL = self._init_tables(
            [[self.num_users, d], [self.num_items, d], [self.num_items, d]])
        self._init_training(self.tables())
        z = lambda n: torch.zeros(n, dtype=torch.int32, device="cuda")
        self._touched = (z(self.num_users), z(self.num_items), z(self.num_items))
        self._init_windows()

    def tables(self):
        return [self.embeddings_UI, self.embeddings_IU, self.embeddings_IL]

    def _run_epoch(self, users, recent, items, labels):
        steps, lr_t, first_stamp = self._epoch_buffers(users.numel())
        ops.npe_train_epoch(*self.tables(), users, recent, items, labels, self.batch_size, self._loss, self.reg,
                            self.opt.kind, lr_t, self.opt.hyper, self._grads, self._touched, self._slots0,
                            self._slots1, first_stamp, self._step_loss)
        return steps

    def _scores(self, users):
        return ops.npe_scores(*self.tables(), users, self._recent, self._recent_len)
