"""HRM: hierarchical representation model (Wang et al., SIGIR 2015).

Plug-in mirror of the reference's model/sequential_recommender/HRM.py:16-163 on the sm_90a kernels:
  * two tables P [users, d] and E [items, d] (:46-52); the window of the user's high_order previous items and the
    next item share E.  x(u, w, i) = <pool_P(P_u, pool_S(E[w])), E_i>, both pools elementwise, max when the conf
    value is "max" and mean otherwise (:62-84).  At high_order = 1 the reference's concat branch is the same formula;
  * pointwise only: the epoch is TimeOrderPointwiseSampler(high_order, num_neg)'s device epoch (:106-108) and the
    batch loop (:110-126) is ``nrc_hrm_train_epoch``: per batch the fused gather -> pool -> score -> loss -> gradient
    kernel and one TF-1.12 optimizer launch over P and E;
  * predict (:135-163) is ``nrc_hrm_query`` + ``nrc_mf_scores`` from every user's last high_order train items by time
    (fewer when the user has fewer; the reference's own predict fails with a shape error at high_order = 1, this one
    scores with the training formula).
"""
import torch

from ... import ops
from ._base import SeqWindowRecommender


class HRM(SeqWindowRecommender):
    def __init__(self, sess, dataset, conf):
        super(HRM, self).__init__(sess, dataset, conf)
        self.learning_rate = conf["learning_rate"]
        self.embedding_size = conf["embedding_size"]
        self.learner = conf["learner"]
        self.num_epochs = conf["epochs"]
        self.reg_mf = conf["reg_mf"]
        self.pre_agg = conf["pre_agg"]
        self.loss_function = conf["loss_function"]
        self.session_agg = conf["session_agg"]
        self.batch_size = conf["batch_size"]
        self.high_order = conf["high_order"]
        self.verbose = conf["verbose"]
        self.num_negatives = conf["num_neg"]
        self.init_method = conf["init_method"]
        self.stddev = conf["stddev"]

    def build_graph(self):
        self._check_loss()
        d = self.embedding_size
        self.user_embeddings, self.item_embeddings = self._init_tables([[self.num_users, d], [self.num_items, d]])
        self._init_training(self.tables())
        z = lambda n: torch.zeros(n, dtype=torch.int32, device="cuda")
        self._touched = (z(self.num_users), z(self.num_items))
        self._init_windows()

    def tables(self):
        return [self.user_embeddings, self.item_embeddings]

    def _pools(self):
        """(pre_agg, session_agg) as max flags: the reference's `== "max"` tests (HRM.py:69, 78)."""
        return self.pre_agg == "max", self.session_agg == "max"

    def _run_epoch(self, users, recent, items, labels):
        steps, lr_t, first_stamp = self._epoch_buffers(users.numel())
        ops.hrm_train_epoch(*self.tables(), users, recent, items, labels, self.batch_size, *self._pools(), self._loss,
                            self.reg_mf, self.opt.kind, lr_t, self.opt.hyper, self._grads, self._touched,
                            self._slots0, self._slots1, first_stamp, self._step_loss)
        return steps

    def _scores(self, users):
        return ops.hrm_scores(*self.tables(), users, self._recent, self._recent_len, *self._pools())
