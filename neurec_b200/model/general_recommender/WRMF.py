"""WRMF: weighted regularised matrix factorisation for implicit feedback (Hu, Koren and Volinsky, ICDM 2008).

Plug-in mirror of the reference's model/general_recommender/WRMF.py:12-106 (same constructor, configuration keys,
log lines and predict contract).  The reference keeps two dense [num_users, num_items] host matrices (Cui, Pui,
:27-33) and runs one sess.run per user and one per item every epoch (:69-85).  Here an epoch is two calls of
``nrc_wrmf_half_step``: every user solved against the item table over the user-major CSR, then every item against
the new user table over the item-major CSR.  The rows of a half depend only on the other table, so one batched call
computes exactly what the reference's sequential loop does.
"""
from time import time

import numpy as np
import torch

from ... import ops
from ...util import timer
from ..AbstractRecommender import AbstractRecommender
from .._engine import get_initializer


class WRMF(AbstractRecommender):
    def __init__(self, sess, dataset, conf):
        super(WRMF, self).__init__(dataset, conf)
        self.embedding_size = conf["embedding_size"]
        self.alpha = conf["alpha"]
        self.topK = conf["topk"]
        self.num_epochs = conf["epochs"]
        self.reg_mf = conf["reg_mf"]
        self.init_method = conf["init_method"]
        self.stddev = conf["stddev"]
        self.verbose = conf["verbose"]
        self.dataset = dataset
        self.num_users = dataset.num_users
        self.num_items = dataset.num_items
        self.sess = sess                      # unused: there is no TF session

    def build_graph(self):
        gen = torch.Generator().manual_seed(2017)
        init = get_initializer(self.init_method, self.stddev, gen)
        self.user_embeddings = init([self.num_users, self.embedding_size]).cuda()     # WRMF.py:45-48
        self.item_embeddings = init([self.num_items, self.embedding_size]).cuda()
        users, items = self.dataset.get_train_interactions()
        u = torch.as_tensor(np.asarray(users, dtype=np.int32)).cuda()
        i = torch.as_tensor(np.asarray(items, dtype=np.int32)).cuda()
        self._user_csr = ops.csr_from_coo(u, i, self.num_users, self.num_items)
        self._item_csr = ops.csr_from_coo(i, u, self.num_items, self.num_users)
        # heaviest rows first, so that long rows do not finish last in the launch
        order = lambda ptr: torch.argsort(-torch.diff(ptr), stable=True).to(torch.int32)
        self._user_order = order(self._user_csr[0])
        self._item_order = order(self._item_csr[0])
        self._work = ops.wrmf_work(max(self.num_users, self.num_items), self.embedding_size)
        self._not_spd = torch.zeros((1,), dtype=torch.int32, device="cuda")

    def _train_epoch(self):
        # WRMF.py:74-85: every user against the item table, then every item against the new user table
        for fixed, (ptr, idx), order, out in ((self.item_embeddings, self._user_csr, self._user_order, self.user_embeddings),
                                              (self.user_embeddings, self._item_csr, self._item_order, self.item_embeddings)):
            ops.wrmf_half_step(fixed, ptr, idx, out, self.alpha, self.reg_mf, row_order=order, work=self._work,
                               not_spd=self._not_spd)

    def train_model(self):
        self.logger.info(self.evaluator.metrics_info())
        for epoch in range(1, self.num_epochs + 1):
            training_start_time = time()
            self._train_epoch()
            torch.cuda.synchronize()
            self.logger.info('iteration %i finished in %f seconds' % (epoch, time() - training_start_time))
            if epoch % self.verbose == 0:
                self.logger.info("epoch %d:\t%s" % (epoch, self.evaluate()))

    @timer
    def evaluate(self):
        return self.evaluator.evaluate(self)

    def get_eval_tables(self):
        """Fast path of UniEvaluator: predict is user_embeddings[users] . item_embeddings^T (WRMF.py:96-99)."""
        return self.user_embeddings, self.item_embeddings

    def predict(self, user_ids, candidate_items_userids=None):
        users = torch.as_tensor(np.asarray(user_ids, dtype=np.int32)).cuda()
        ratings = ops.mf_scores(self.user_embeddings, self.item_embeddings, users).cpu().numpy()
        if candidate_items_userids is not None:
            ratings = [r[np.asarray(items)] for r, items in zip(ratings, candidate_items_userids)]   # :100-105
        return ratings
