"""ItemKNN: item-based neighbourhood recommender (item-item similarity, the best `neighbor` items per column,
ratings = R . W).

Plug-in mirror of the reference's model/general_recommender/ItemKNN.py:549-589 on the sm_90a kernels:
  * build_graph (:568-573) prepares the data as Compute_Similarity does (:319-435, :89-90), on the host with numpy:
    adjusted subtracts each user's average and pearson each item's, both averages stored into an array of the data's
    own dtype (so int64 ratings subtract truncated integer averages); tanimoto / jaccard, dice and tversky make the
    data binary; the per-item vectors (sums of squares, their roots or powers) come from the same numpy calls.  The
    similarity, the dot products and the neighbour selection are ``nrc_itemknn_similarity``; W_sparse (a host scipy
    CSR, float32) is kept for users who read it;
  * predict(users, None) (:583-585) is ``nrc_itemknn_scores``, computed per call: the same float64 sums as
    train.tocsc().dot(W_sparse) rounded to float32, without storing the dense [U, I] ratings matrix;
  * train_model (:575-577) logs metrics_info() and one evaluation.
Deviations: ties at the neighbour boundary are broken by the lower item id (numpy's introselect orders them its own
way); with candidate lists, predict reads the candidates' scores from the user's row (the reference returns None,
which its evaluator cannot use).
"""
import numpy as np
import scipy.sparse as sp
import torch

from ... import ops
from ...util import timer
from ..AbstractRecommender import AbstractRecommender

# similarity name -> transform of nrc_itemknn_similarity (ItemKNN.py:227-315)
KINDS = {"cosine": "norm", "adjusted": "norm", "asymmetric": "norm", "pearson": "norm", "jaccard": "tanimoto",
         "tanimoto": "tanimoto", "dice": "dice", "tversky": "tversky", "euclidean": "euclidean"}


def _subtract_average(X, axis):
    """X.data minus the average of each row (axis 1, on a CSR) or column (axis 0, on a CSC) that has entries; the
    averages live in an array of the sums' dtype, so integer data subtract truncated averages."""
    n = np.diff(X.indptr)
    sums = np.asarray(X.sum(axis=axis)).ravel()
    avg = np.zeros_like(sums)
    nz = n > 0
    avg[nz] = sums[nz] / n[nz]
    X.data -= np.repeat(avg, n)
    return X


def prepare(train, similarity, asymmetric_alpha=0.5):
    """The data and per-item vectors Compute_Similarity works from: (X as a CSC, kind, va f64 [I], vb f64 [I]).
    Raises the reference's ValueError for an unknown similarity name."""
    if similarity not in KINDS:
        raise ValueError("Cosine_Similarity: value for parameter 'mode' not recognized."
                         " Allowed values are: 'cosine', 'pearson', 'adjusted', 'asymmetric', 'jaccard', 'tanimoto',"
                         "dice, tversky."
                         " Passed value was '{}'".format(similarity))
    kind = KINDS[similarity]
    X = sp.csc_matrix(train, copy=True)
    if similarity == "adjusted":
        X = _subtract_average(X.tocsr(), 1).tocsc()
    elif similarity == "pearson":
        X = _subtract_average(X, 0)
    elif kind in ("tanimoto", "dice", "tversky"):
        X.data[:] = 1
    sq = np.asarray(X.power(2).sum(axis=0)).ravel()
    if kind in ("tanimoto", "dice", "tversky"):
        va = vb = sq
    elif kind == "euclidean":
        va, vb = sq, np.sqrt(sq)
    else:
        s = np.sqrt(sq)
        if similarity == "asymmetric":
            va, vb = np.power(s, 2 * asymmetric_alpha), np.power(s, 2 * (1 - asymmetric_alpha))
        else:
            va = vb = s
    return X, kind, np.asarray(va, np.float64), np.asarray(vb, np.float64)


def _dev_csr(M):
    """(ptr i64, idx i32, val f64) CUDA tensors of a canonical scipy CSR / CSC."""
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()
    return t(M.indptr.astype(np.int64)), t(M.indices.astype(np.int32)), t(M.data.astype(np.float64))


def similarity_device(train, similarity, neighbor, shrink=0, asymmetric_alpha=0.5, tversky_alpha=1.0,
                      tversky_beta=1.0):
    """W of Compute_Similarity(train, similarity, topK=neighbor, shrink, normalize=True, ...) on the device, in
    ops.itemknn_similarity's padded CSC form."""
    X, kind, va, vb = prepare(train, similarity, asymmetric_alpha)
    X.sort_indices()
    R = X.tocsr()
    R.sort_indices()
    rp, ri, rv = _dev_csr(R)
    cp, ci, cv = _dev_csr(X)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()
    return ops.itemknn_similarity(rp, ri, rv, cp, ci, cv, X.shape[1], kind, t(va), t(vb), shrink, tversky_alpha,
                                  tversky_beta, neighbor)


def w_to_scipy(W, num_items):
    """The padded CSC W of ops.itemknn_similarity as a host scipy CSR float32 [I, I] (W[k, c] = similarity)."""
    counts, rows, vals = (a.cpu().numpy() for a in W)
    kc = rows.shape[0]
    mask = np.arange(kc)[:, None] < counts[None, :]
    cols = np.broadcast_to(np.arange(num_items)[None, :], rows.shape)
    return sp.csr_matrix((vals.T[mask.T], (rows.T[mask.T], cols.T[mask.T])), shape=(num_items, num_items),
                         dtype=np.float32)


class ItemKNN(AbstractRecommender):
    def __init__(self, sess, dataset, conf):
        super(ItemKNN, self).__init__(dataset, conf)
        self.verbose = conf["verbose"]
        self.topK = conf["neighbor"]
        self.shrink = conf["shrink"]
        self.dataset = dataset
        self.train_matrix = self.dataset.train_matrix.tocsc()
        self.similarity = conf["similarity"]
        self.asymmetric_alpha = conf["asymmetric_alpha"]
        self.tversky_alpha = conf["tversky_alpha"]
        self.tversky_beta = conf["tversky_beta"]
        self.num_users = dataset.num_users
        self.num_items = dataset.num_items

    def build_graph(self):
        self.W = similarity_device(self.train_matrix, self.similarity, self.topK, self.shrink, self.asymmetric_alpha,
                                   self.tversky_alpha, self.tversky_beta)
        self.W_sparse = w_to_scipy(self.W, self.num_items)
        R = sp.csr_matrix(self.train_matrix)
        R.sort_indices()
        self._train = _dev_csr(R)

    def train_model(self):
        self.logger.info(self.evaluator.metrics_info())
        self.logger.info(self.evaluate())

    @timer
    def evaluate(self):
        return self.evaluator.evaluate(self)

    def predict(self, user_ids, candidate_items=None):
        """[len(user_ids), num_items] CUDA float32 scores; with candidate lists, one score array per user."""
        users = np.asarray(user_ids, dtype=np.int64).reshape(-1)
        if len(users) and (users.min() < 0 or users.max() >= self.num_users):
            raise IndexError("user id outside [0, %d)" % self.num_users)
        dev_users = torch.from_numpy(users.astype(np.int32)).cuda()
        ratings = ops.itemknn_scores(*self._train, self.W, dev_users)
        if candidate_items is not None:
            host = ratings.cpu().numpy()
            ratings = [host[r][np.asarray(items, dtype=np.int64)] for r, items in enumerate(candidate_items)]
        return ratings
