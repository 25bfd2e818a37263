"""numpy float64 restatement of ItemKNN (the reference's ItemKNN.py:11-589) for the tests.

The data and the per-item vectors come from the plug-in's `prepare` (which the fixture pins against the reference's
own Compute_Similarity); from there every column is restated here in the reference's operation order: the dots as
X.T.dot(dense block) (scipy's csr_matvecs: users ascending), the diagonal zeroed, then the transform with numpy's
elementwise float64 operations (each correctly rounded, nothing fused).  Selection keeps the top min(K, I) by
(value descending, row ascending, NaN last), then the values != 0.0, cast to float32.  Scores are scipy's
train.tocsc().dot(W) rounded to float32, as the reference's evaluator sees them.
"""
import zlib

import numpy as np
import scipy.sparse as sp

from neurec_b200.model.general_recommender.ItemKNN import prepare  # noqa: F401  (re-exported for the tests)


def dots(X, c0, c1):
    """w[k, c - c0] for the columns [c0, c1) of the CSC X, as float64 (an integer Gram is exact)."""
    return np.asarray(X.T.dot(X[:, c0:c1].toarray()), dtype=np.float64).reshape(X.shape[1], c1 - c0)


def transform(kind, w, c, va, vb, shrink, ta, tb):
    """Column c's similarities from its dots w f64 [I] (w[c] is zeroed here first), in the reference's order."""
    w = np.array(w, dtype=np.float64)
    w[c] = 0.0
    with np.errstate(divide="ignore", invalid="ignore"):
        if kind == "norm":
            return w * (1 / (va[c] * vb + shrink + 1e-6))
        if kind == "tanimoto":
            return w * (1 / (va[c] + va - w + shrink + 1e-6))
        if kind == "dice":
            return w * (1 / (va[c] + va + shrink + 1e-6))
        if kind == "tversky":
            return w * (1 / (w + (va[c] - w) * ta + (va - w) * tb + shrink + 1e-6))
        assert kind == "euclidean"
        d = va + va[c]
        d = d - 2 * w
        d = d / (vb[c] * vb)
        d = np.sqrt(d)
        s = 1 / (d + shrink + 1e-9)
        s[c] = 0.0
        return s


def select(v, K):
    """(rows ascending, f32 values) kept from column values v: the top min(K, I) by (value descending, row
    ascending, NaN last), then those != 0.0."""
    K = min(int(K), len(v))
    order = np.lexsort((np.arange(len(v)), -v))
    top = np.sort(order[:K])
    top = top[v[top] != 0.0]
    return top.astype(np.int32), v[top].astype(np.float32)


def column(X, kind, va, vb, c, K, shrink=0, ta=1.0, tb=1.0):
    """One column of W: (rows, f32 values)."""
    return select(transform(kind, dots(X, c, c + 1)[:, 0], c, va, vb, shrink, ta, tb), K)


def similarity(X, kind, va, vb, K, shrink=0, ta=1.0, tb=1.0, columns=None, block=100):
    """{c: (rows, f32 values)} for the given columns (all by default), the dots computed in blocks of `block`."""
    ni = X.shape[1]
    columns = range(ni) if columns is None else columns
    want = sorted(set(int(c) for c in columns))
    out = {}
    i = 0
    while i < len(want):
        c0 = want[i]
        c1 = min(c0 + block, ni)
        blk = [c for c in want[i:] if c < c1]
        G = dots(X, c0, c1)
        for c in blk:
            out[c] = select(transform(kind, G[:, c - c0], c, va, vb, shrink, ta, tb), K)
        i += len(blk)
    return out


CRC_BLOCK = 64


def block_crcs(cols, ties, ni, block=CRC_BLOCK):
    """crc32 per block of `block` consecutive columns of a W given as {c: (rows, f32 values)}: a column without a
    boundary tie adds its rows (int32) and then its value bits in row order; a tied column adds only its values
    sorted ascending, since which of the tied rows are kept is implementation-defined.  NaN is hashed as one
    canonical NaN."""
    out = []
    for b0 in range(0, ni, block):
        h = 0
        for c in range(b0, min(b0 + block, ni)):
            r, v = cols[c]
            v = np.asarray(v, np.float32)
            v = np.where(np.isnan(v), np.float32(np.nan), v)
            if ties[c]:
                h = zlib.crc32(np.sort(v).tobytes(), h)
            else:
                h = zlib.crc32(np.ascontiguousarray(r, dtype=np.int32).tobytes(), h)
                h = zlib.crc32(v.tobytes(), h)
        out.append(h)
    return np.array(out, np.uint32)


def to_scipy(cols, ni):
    """{c: (rows, vals)} over every column -> scipy CSR float32 [I, I]."""
    r = np.concatenate([cols[c][0] for c in range(ni)]) if ni else np.zeros(0, np.int32)
    v = np.concatenate([cols[c][1] for c in range(ni)]) if ni else np.zeros(0, np.float32)
    cc = np.concatenate([np.full(len(cols[c][0]), c) for c in range(ni)]) if ni else np.zeros(0, np.int64)
    return sp.csr_matrix((v, (r, cc)), shape=(ni, ni), dtype=np.float32)


def scores(train, W, users):
    """The reference's ratings rows (train.tocsc().dot(W_sparse)) for `users`, as its evaluator casts them."""
    return np.asarray(sp.csc_matrix(train).dot(sp.csr_matrix(W)).toarray()[np.asarray(users)], dtype=np.float32)
