"""TEST INFRASTRUCTURE ONLY -- numpy restatement (fp32 or fp64) of the reference's FISM graph, its hand-derived
gradients, both instance generators and the batch loop, in the style of oracle/tf_math.py (whose losses, optimizer
rules and Adam lr_t it reuses).

Restated call sites (paths relative to the reference):
  model/general_recommender/FISM.py:55-94     variables, inference, pointwise and pairwise losses
  model/general_recommender/FISM.py:100-144   the batch loop (loss of every batch, regularisers included)
  model/general_recommender/FISM.py:154-180   predict
  util/data_generator.py:5-27                 _get_pairwise_all_likefism_data
  util/data_generator.py:29-54                _get_pointwise_all_likefism_data
A sample is (history row r of a CSR, excluded item e or -1, count n, target i, label z or negative j); pads of the
reference's padded histories read the zero row and are left out here.  Every gradient is an IndexedSlices whose rows
are the touched set of its variable; Q and b share the targets' touched set.  The gradients are checked against
torch.autograd in tests/test_fism.py.
"""
import numpy as np
import scipy.sparse as sp

from oracle.tf_math import DEFAULT_HYPER, SLOT_INIT, adam_lr_t, opt_apply

f32 = np.float32


def pairwise_loss_and_grad(kind, x, dtype=f32):
    """learner.py:18-29 in dtype -> (per-sample loss, dloss/dx); as oracle/tf_math.py's fp32 form."""
    x = np.asarray(x, dtype)
    one = dtype(1)
    if kind == "bpr":
        sp = np.where(x >= 0, np.log1p(np.exp(-np.abs(x))), -x + np.log1p(np.exp(-np.abs(x))))
        return sp.astype(dtype), (-one / (one + np.exp(x))).astype(dtype)
    if kind == "hinge":
        t = x + one
        return np.maximum(t, dtype(0)), (t > 0).astype(dtype)
    if kind == "square":
        t = one - x
        return t * t, dtype(-2) * t
    raise Exception("please choose a suitable loss function")


def pointwise_loss_and_grad(kind, z, x, dtype=f32):
    """learner.py:31-41 in dtype -> (per-sample loss contribution, dloss/dx); cross entropy is a batch mean."""
    x, z = np.asarray(x, dtype), np.asarray(z, dtype)
    one = dtype(1)
    if kind == "cross_entropy":
        inv_b = one / dtype(max(len(x), 1))
        e = np.exp(-np.abs(x))
        l = (np.maximum(x, dtype(0)) - x * z + np.log1p(e)) * inv_b
        s = np.where(x >= 0, one / (one + e), e / (one + e))
        return l.astype(dtype), ((s - z) * inv_b).astype(dtype)
    if kind == "square":
        t = z - x
        return t * t, dtype(-2) * t
    raise Exception("please choose a suitable loss function")


def pointwise_layout(ptr, idx, num_neg):
    """_get_pointwise_all_likefism_data's instances before the negatives are drawn: users ascending, each user's items
    in CSR order, num_neg negatives (history = the whole row, n = |R_u| + 1, label 0) then the positive (history = the
    row without i, n = |R_u|, label 1).  Users without train items give no instance.  -> dict of int32 rows, excl,
    num, items (-1 in the negative slots), labels f32, and pos_slot (bool, the positives)."""
    ptr = np.asarray(ptr, np.int64)
    deg = np.diff(ptr)
    k = num_neg + 1
    P = int(ptr[-1])
    users = np.repeat(np.arange(len(deg), dtype=np.int32), deg)
    pos_items = np.asarray(idx[:P], np.int32)
    rows = np.repeat(users, k)
    slot = np.tile(np.arange(k), P)
    pos_slot = slot == num_neg
    n = np.repeat(deg[users], k).astype(np.int32)
    num = np.where(pos_slot, n, n + 1).astype(np.int32)
    items = np.where(pos_slot, np.repeat(pos_items, k), -1).astype(np.int32)
    excl = items.copy()
    labels = pos_slot.astype(f32)
    return dict(rows=rows, excl=excl, num=num, items=items, labels=labels, pos_slot=pos_slot,
                pos_users=users, pos_items=pos_items)


def fill_negatives(layout, neg):
    """The epoch's targets: neg [P, num_neg] (drawn per positive, in positive order) fill the negative slots."""
    items = layout["items"].copy()
    items[~layout["pos_slot"]] = np.asarray(neg, np.int32).reshape(-1)
    return items


def pairwise_layout(ptr, idx):
    """_get_pairwise_all_likefism_data as it runs: it removes items from the list it enumerates, so a user with
    |R_u| > 1 gets the items at the even positions 0, 2, 4, ... of its row as positives (ceil(|R_u| / 2) samples),
    and the positive and negative histories of every sample are one list, the items at the odd positions.
    n = |R_u|, n_j = |R_u| + 1; sample k of a user takes the user's k-th negative draw.  -> (odd CSR ptr int64, idx
    int32) and dict of int32 rows, num, num_neg, items."""
    ptr = np.asarray(ptr, np.int64)
    deg = np.diff(ptr)
    hist_ptr = np.zeros(len(deg) + 1, np.int64)
    hist, rows, num, items = [], [], [], []
    for u in range(len(deg)):
        r = np.asarray(idx[ptr[u]:ptr[u + 1]], np.int32)
        odd = r[1::2] if deg[u] > 1 else r[:0]
        hist.append(odd)
        hist_ptr[u + 1] = hist_ptr[u] + len(odd)
        if deg[u] > 1:
            even = r[0::2]
            rows.append(np.full(len(even), u, np.int32))
            items.append(even)
            num.append(np.full(len(even), deg[u], np.int32))
    cat = lambda a: np.concatenate(a).astype(np.int32) if a else np.zeros(0, np.int32)
    num = cat(num)
    return (hist_ptr, cat(hist)), dict(rows=cat(rows), num=num, num_neg=(num + 1).astype(np.int32), items=cat(items))


def histories(hist_ptr, hist_idx, rows, excl=None):
    """The reference's per-sample history lists (before pad_sequences)."""
    out = []
    for s, r in enumerate(rows):
        h = np.asarray(hist_idx[hist_ptr[r]:hist_ptr[r + 1]], np.int32)
        if excl is not None and excl[s] >= 0:
            h = h[h != excl[s]]
        out.append(h)
    return out


def history_matrix(hist_ptr, hist_idx, rows, excl, num_items, dtype):
    """[len(rows), num_items] 0/1 CSR of the samples' histories (the exclusion applied): p = S @ c1."""
    hist_ptr = np.asarray(hist_ptr, np.int64)
    rows = np.asarray(rows, np.int64)
    beg = hist_ptr[rows]
    ln = hist_ptr[rows + 1] - beg
    sid = np.repeat(np.arange(len(rows)), ln)
    pos = np.arange(int(ln.sum())) - np.repeat(np.cumsum(ln) - ln, ln) + np.repeat(beg, ln)
    h = np.asarray(hist_idx, np.int64)[pos]
    if excl is not None:
        keep = h != np.repeat(np.asarray(excl, np.int64), ln)
        sid, h = sid[keep], h[keep]
    return sp.csr_matrix((np.ones(len(h), dtype), (sid, h)), shape=(len(rows), num_items))


def loss_and_grad(c1, Q, b, hist_ptr, hist_idx, rows, excl, num, items, third, num_neg, pairwise, loss, alpha, lam,
                  gamma, dtype=f32):
    """FISM._create_loss (FISM.py:77-88) for one batch -> (loss, (gC1, gQ, gb), (tC1, tItem)).  third: labels or
    negatives; excl None or -1 entries: no exclusion."""
    c1, Q, b = (np.asarray(a, dtype) for a in (c1, Q, b))
    lam, gamma = dtype(lam), dtype(gamma)
    S = history_matrix(hist_ptr, hist_idx, rows, excl, c1.shape[0], dtype)
    p = np.asarray(S @ c1, dtype)
    coeff = lambda n: np.power(np.asarray(n, dtype), -dtype(alpha)).astype(dtype)
    qi, bi, ci = Q[items], b[items], coeff(num)
    xi = (ci * (p * qi).sum(1, dtype=dtype) + bi).astype(dtype)
    gQ, gb = np.zeros_like(Q), np.zeros_like(b)
    sq = (qi * qi).sum(dtype=dtype)
    if pairwise:
        j = np.asarray(third, np.int64)
        qj, bj, cj = Q[j], b[j], coeff(num_neg)
        xj = (cj * (p * qj).sum(1, dtype=dtype) + bj).astype(dtype)
        lo, g = pairwise_loss_and_grad(loss, (xi - xj).astype(dtype), dtype)
        sq = sq + (qj * qj).sum(dtype=dtype)
        gi, gj = (g * ci)[:, None], (-g * cj)[:, None]
        gp = (gi * qi + gj * qj + lam * p).astype(dtype)
        np.add.at(gQ, items, (gi * p + gamma * qi).astype(dtype))
        np.add.at(gQ, j, (gj * p + gamma * qj).astype(dtype))
        np.add.at(gb, items, g)
        np.add.at(gb, j, -g)
        t_items = np.concatenate([items, j])
    else:
        lo, g = pointwise_loss_and_grad(loss, third, xi, dtype)
        gi = (g * ci)[:, None]
        gp = (gi * qi + lam * p).astype(dtype)
        np.add.at(gQ, items, (gi * p + gamma * qi).astype(dtype))
        np.add.at(gb, items, g)
        t_items = items
    gC1 = np.asarray(S.T @ gp, dtype)
    tC = np.asarray(S.sum(0)).reshape(-1) > 0
    tI = np.zeros(Q.shape[0], bool)
    tI[t_items] = True
    total = lo.sum(dtype=dtype) + lam * dtype(0.5) * (p * p).sum(dtype=dtype) + gamma * dtype(0.5) * sq
    return dtype(total), (gC1, gQ, gb), (tC, tI)


def query(c1, ptr, idx, users, dtype=np.float64):
    c1 = np.asarray(c1, dtype)
    return np.asarray(history_matrix(ptr, idx, users, None, c1.shape[0], dtype) @ c1, dtype)


def scores(c1, Q, b, ptr, idx, users, alpha):
    """FISM.predict (FISM.py:154-180) in fp64: [rows, num_items], the history the whole row, n = |R_u|."""
    p = query(c1, ptr, idx, users)
    n = np.diff(np.asarray(ptr, np.int64))[np.asarray(users)].astype(np.float64)
    return (n ** -float(alpha))[:, None] * (p @ np.asarray(Q, np.float64).T) + np.asarray(b, np.float64)[None, :]


class FISMTrainer:
    """CPU stand-in for build_graph + the sess.run((loss, optimizer)) batch loop; variables c1, Q, b."""

    def __init__(self, c1, Q, b, learner="adam", lr=1e-3, loss="square", alpha=0.5, lam=1e-4, gamma=1e-4,
                 pairwise=False):
        self.vars = [np.array(t, dtype=f32) for t in (c1, Q, b)]
        self.learner, self.lr, self.loss, self.alpha = learner, lr, loss, alpha
        self.lam, self.gamma, self.pairwise = lam, gamma, pairwise
        i0, i1 = SLOT_INIT[learner]
        mk = lambda a, v: None if v is None else np.full_like(a, v)
        self.slots = [(mk(a, i0), mk(a, i1)) for a in self.vars]
        self.t = 0

    def step(self, hist_ptr, hist_idx, rows, excl, num, items, third, num_neg):
        l, grads, (tC, tI) = loss_and_grad(*self.vars, hist_ptr, hist_idx, rows, excl, num, items, third, num_neg,
                                           self.pairwise, self.loss, self.alpha, self.lam, self.gamma)
        hyper = DEFAULT_HYPER[self.learner](self.lr)
        if self.learner == "adam":
            hyper[0] = adam_lr_t(self.lr, 1, start_step=self.t)[0]
        for var, g, (s0, s1), tch in zip(self.vars, grads, self.slots, (tC, tI, tI)):
            opt_apply(self.learner, var, g.reshape(var.shape), s0, s1, tch, hyper, dense_var=False)
        self.t += 1
        return l

    def epoch(self, hist_ptr, hist_idx, rows, excl, num, items, third, num_neg, batch_size):
        n = len(rows)
        losses = []
        for off in range(0, n, batch_size):
            sl = slice(off, min(n, off + batch_size))
            losses.append(self.step(hist_ptr, hist_idx, rows[sl], None if excl is None else excl[sl], num[sl],
                                    items[sl], third[sl], None if num_neg is None else num_neg[sl]))
        return np.asarray(losses, dtype=f32)
