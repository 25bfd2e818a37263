"""TransRec: translation-based recommendation (He et al., RecSys 2017).

Plug-in mirror of the reference's model/sequential_recommender/TransRec.py:22-166 on the sm_90a kernels:
  * variables P [users, d], Q [items, d], b [items] and the global translation g [1, d] (:54-64); training scores
    x(u, l, i) = b_i - |(P_u + g) + Q_l - Q_i|^2, squared (:66-78);
  * the epoch is the time-ordered sampler's device epoch (:112-118) and the batch loop (:119-141) is
    ``nrc_transrec_train_epoch``: per batch the fused gradient kernel (g's dense gradient summed in one fixed order)
    and one TF-1.12 optimizer launch over P, Q, b (IndexedSlices rules) and g (dense rules);
  * predict (:102-107, 153-166) is ``nrc_transrec_scores``: b_j - |(P_u + g) + Q_l - Q_j|, NOT squared.
"""
import torch

from ... import ops
from ._base import SeqEmbeddingRecommender


class TransRec(SeqEmbeddingRecommender):
    def build_graph(self):
        self._check_loss()
        d = self.embedding_size
        self.user_embeddings, self.item_embeddings, self.item_biases, self.global_embedding = self._init_tables(
            [[self.num_users, d], [self.num_items, d], [self.num_items], [1, d]])
        self._init_training(self.tables())
        z = lambda n: torch.zeros(n, dtype=torch.int32, device="cuda")
        self._touched = (z(self.num_users), z(self.num_items), z(self.num_items))
        self._work = ops.transrec_work(d)

    def tables(self):
        return [self.user_embeddings, self.item_embeddings, self.item_biases, self.global_embedding]

    def _run_epoch(self, users, recent, items, third):
        steps, lr_t, first_stamp = self._epoch_buffers(users.numel())
        ops.transrec_train_epoch(*self.tables(), users, recent, items, third, self.batch_size, self.is_pairwise is True,
                                 self._loss, self.reg_mf, self.opt.kind, lr_t, self.opt.hyper, self._grads,
                                 self._touched, self._slots0, self._slots1, first_stamp, self._work, self._step_loss)
        return steps

    def train_model(self):
        self.logger.info(self.evaluator.metrics_info())
        self.data_iter()
        for epoch in range(self.num_epochs):
            # the reference computes the epoch's loss but does not log it (TransRec.py:143-144 are commented out)
            self._train_epoch()
            if epoch % self.verbose == 0:
                self.logger.info("epoch %d:\t%s" % (epoch, self.evaluate()))

    def _scores(self, users, recent):
        return ops.transrec_scores(*self.tables(), users, recent)
