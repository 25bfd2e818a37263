"""FPMC: factorizing personalized Markov chains (Rendle et al., WWW 2010).

Plug-in mirror of the reference's model/sequential_recommender/FPMC.py:16-165 on the sm_90a kernels:
  * four tables UI [users, d], IU, IL, LI [items, d] (:49-59); x(u, l, i) = <UI_u, IU_i> + <IL_i, LI_l> with l the
    user's item before i (:61-70);
  * the epoch is the time-ordered sampler's device epoch (:99-105; a new order and new negatives every epoch) and the
    batch loop (:106-128) is ``nrc_fpmc_train_epoch``: per batch the fused gather -> score -> loss -> gradient kernel
    and one TF-1.12 optimizer launch over the four tables;
  * predict (:140-165) is ``nrc_fpmc_scores`` over all items from every user's last train item.
"""
from time import time

import torch

from ... import ops
from ._base import SeqEmbeddingRecommender


class FPMC(SeqEmbeddingRecommender):
    def __init__(self, sess, dataset, conf):
        super(FPMC, self).__init__(sess, dataset, conf)
        self.topK = conf["topk"]

    def build_graph(self):
        self._check_loss()
        d = self.embedding_size
        self.embeddings_UI, self.embeddings_IU, self.embeddings_IL, self.embeddings_LI = self._init_tables(
            [[self.num_users, d], [self.num_items, d], [self.num_items, d], [self.num_items, d]])
        self._init_training(self.tables())
        z = lambda n: torch.zeros(n, dtype=torch.int32, device="cuda")
        self._touched = (z(self.num_users), z(self.num_items), z(self.num_items))

    def tables(self):
        return [self.embeddings_UI, self.embeddings_IU, self.embeddings_IL, self.embeddings_LI]

    def _run_epoch(self, users, recent, items, third):
        steps, lr_t, first_stamp = self._epoch_buffers(users.numel())
        ops.fpmc_train_epoch(*self.tables(), users, recent, items, third, self.batch_size, self.is_pairwise is True,
                             self._loss, self.reg_mf, self.opt.kind, lr_t, self.opt.hyper, self._grads, self._touched,
                             self._slots0, self._slots1, first_stamp, self._step_loss)
        return steps

    def train_model(self):
        self.logger.info(self.evaluator.metrics_info())
        data_iter = self.data_iter()
        for epoch in range(1, self.num_epochs + 1):
            num_training_instances = len(data_iter)       # the number of batches (FPMC.py:107)
            training_start_time = time()
            total_loss = self._train_epoch()
            self.logger.info("[iter %d : loss : %f, time: %f]" %
                             (epoch, total_loss / num_training_instances, time() - training_start_time))
            if epoch % self.verbose == 0:
                self.logger.info("epoch %d:\t%s" % (epoch, self.evaluate()))

    def _scores(self, users, recent):
        return ops.fpmc_scores(*self.tables(), users, recent)
