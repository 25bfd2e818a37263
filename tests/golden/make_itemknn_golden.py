"""Generates tests/golden/kat_itemknn.npz by running the UNMODIFIED reference's Compute_Similarity (ItemKNN.py).

Run from the repo root after build() (the reference's util.cython modules come from oracle/_ref):
``python tests/golden/make_itemknn_golden.py``.  The fixture is committed, so the tests never need the reference.

Inputs: the train matrix of the ratio-0.8 ml-100k split the reference's Dataset makes under np.random.seed(2018)
(the same split as ml100k_split.npz; its int64 ratings are stored here as `ratings`, aligned with that file's
train_indices), as ItemKNN passes it (train.tocsc()), once with its int64 ratings ("int") and once as float64 ones
("bin").  For every similarity name, shrink in {0, 10} and neighbor K in {5, 100}, with ItemKNN's arguments
(normalize=True, asymmetric_alpha=1, tversky 0.5 / 0.5), per configuration `<data>_<name>_s<shrink>`:
  *_k<K>_counts u8 [I]     entries per column of the reference's W
  *_tie<K> packed bits [I] the column's K-th largest value equals the best value not selected (read from the
                           reference's own run at neighbor = I; compared in W's float32, so a float64 near-tie
                           counts too)
  *_k<K>_crc u32 [I / 64]  itemknn_math.block_crcs of W: per block of 64 columns, the rows and value bits of every
                           untied column and the sorted values of every tied one
  *_k<K>_nan               the number of NaN values in W
plus `unknown_error`, the ValueError message for an unknown similarity name.
"""
import importlib
import os
import sys

import numpy as np
import scipy.sparse as sp

from make_golden import OUT

sys.path[:0] = [os.path.dirname(os.path.dirname(OUT)), os.path.dirname(OUT)]  # the repository, tests/

NAMES = ("cosine", "adjusted", "asymmetric", "pearson", "jaccard", "tanimoto", "dice", "tversky", "euclidean")


def column_ties(full, k):
    """Per column of the reference's neighbor = I run: the k-th largest value equals the (k+1)-th (zeros, which W
    does not store, included)."""
    ni = full.shape[1]
    out = np.zeros(ni, bool)
    for c in range(ni):
        v = full.data[full.indptr[c]:full.indptr[c + 1]].astype(np.float64)
        v = np.concatenate([v, np.zeros(ni - len(v))])
        v = -np.sort(-v)                      # NaN last
        if k < ni:
            a, b = v[k - 1], v[k]
            out[c] = (a == b) or (np.isnan(a) and np.isnan(b))
    return out


def itemknn():
    import oracle
    cwd = oracle.import_reference()
    os.chdir(cwd)
    sys.argv = ["main.py"]
    np.random.seed(2018)
    import random
    random.seed(2018)
    from util import Configurator
    from data.dataset import Dataset
    knn = importlib.import_module("model.general_recommender.ItemKNN")
    import itemknn_math as km
    conf = Configurator("NeuRec.properties", default_section="hyperparameters")
    ds = Dataset(conf)
    tr = ds.train_matrix.tocsr()
    tr.sort_indices()
    z = np.load(os.path.join(OUT, "ml100k_split.npz"))
    assert np.array_equal(tr.indptr, z["train_indptr"]) and np.array_equal(tr.indices, z["train_indices"])
    assert tr.dtype == np.int64, tr.dtype
    res = {"ratings": tr.data.astype(np.int8)}
    assert np.array_equal(res["ratings"], tr.data)
    try:
        knn.Compute_Similarity(tr.tocsc(), similarity="nope", topK=5, shrink=0, normalize=True)
        raise AssertionError("no ValueError for an unknown similarity")
    except ValueError as e:
        res["unknown_error"] = np.array(str(e))
    ni = tr.shape[1]
    data = {"int": tr.tocsc(), "bin": sp.csr_matrix((np.ones(tr.nnz), tr.indices, tr.indptr), shape=tr.shape).tocsc()}
    for dname, X in data.items():
        for name in NAMES:
            for shrink in (0, 10):
                key = "%s_%s_s%d" % (dname, name, shrink)
                ws = {}
                for k in (5, 100, ni):
                    sim = knn.Compute_Similarity(X, shrink=shrink, topK=k, normalize=True, similarity=name,
                                                 asymmetric_alpha=1, tversky_alpha=0.5, tversky_beta=0.5)
                    W = sim.compute_similarity().tocsc()
                    W.sort_indices()
                    ws[k] = W
                for k in (5, 100):
                    W = ws[k]
                    cols = {c: (W.indices[W.indptr[c]:W.indptr[c + 1]], W.data[W.indptr[c]:W.indptr[c + 1]])
                            for c in range(ni)}
                    ties = column_ties(ws[ni], k)
                    res["%s_k%d_counts" % (key, k)] = np.diff(W.indptr).astype(np.uint8)
                    res["%s_tie%d" % (key, k)] = np.packbits(ties)
                    res["%s_k%d_crc" % (key, k)] = km.block_crcs(cols, ties, ni)
                    res["%s_k%d_nan" % (key, k)] = np.int32(np.isnan(W.data).sum())
                print(key, W.nnz, int(column_ties(ws[ni], 5).sum()), flush=True)
    np.savez_compressed(os.path.join(OUT, "kat_itemknn.npz"), **res)
    print("itemknn fixture written")


if __name__ == "__main__":
    itemknn()
