"""TEST INFRASTRUCTURE ONLY -- numpy fp32 restatement of the reference's HRM and NPE graphs and batch loops, in the
style of tests/seq_math.py (whose trainer base it extends; losses and optimizer rules come from oracle/tf_math.py).

Restated call sites (paths relative to the reference):
  model/sequential_recommender/HRM.py:54-91,110-126   pooled window, pooled user, pointwise loss, batch loop
  model/sequential_recommender/NPE.py:54-71,89-105    summed window, relu products, pointwise loss, batch loop
  model/sequential_recommender/HRM.py:135-163, NPE.py:114-142   predict from each user's last high_order items
TensorFlow pieces: reduce_mean's gradient is grad / count (_MeanGrad); reduce_max's is (indicator / #equal) * grad
(_MinOrMaxGrad: ties split evenly); relu's is zero where its input is <= 0 (ReluGrad); every embedding_lookup
gradient is an IndexedSlices whose rows are the touched set of its variable, and l2_loss counts each gathered row,
window rows included.  The manual gradients are checked against torch.autograd in tests/test_seq_window.py.
"""
import numpy as np
import torch

from oracle.tf_math import pointwise_loss_and_grad
from seq_math import _mask, _SeqTrainer

f32 = np.float32


def _add_rows(dst, ids, rows):
    """dst[ids[k]] += rows[k] for every k, duplicates summed (np.add.at, through torch's index_add_ for speed)."""
    torch.from_numpy(dst).index_add_(0, torch.from_numpy(np.asarray(ids, np.int64).reshape(-1)),
                                     torch.from_numpy(np.ascontiguousarray(rows, dtype=f32)))


def _windows(recent, n):
    return np.asarray(recent, np.int64).reshape(n, -1)


def hrm_grad(P, E, users, recent, items, labels, pre_max, session_max, loss, reg=0.0):
    """HRM._create_loss (HRM.py:86-91) -> (loss, (gP, gE), (tP, tE)).  recent [batch, L] (or [batch] at L = 1);
    s = pool_S(E[w]), h = pool_P(P_u, s), x = <h, E_i>; tP <- users, tE <- window items + items."""
    P, E = np.asarray(P, f32), np.asarray(E, f32)
    u, i = np.asarray(users), np.asarray(items)
    w = _windows(recent, len(u))
    L = w.shape[1]
    R, p, e = E[w], P[u], E[i]                                        # [B, L, d], [B, d], [B, d]
    if session_max:
        s = R.max(1)
        ind = R == s[:, None, :]
        num = ind.sum(1).astype(f32)
    else:
        s = (R.sum(1, dtype=f32) / f32(L)).astype(f32)
    if pre_max:
        h = np.maximum(p, s)
        share = (f32(1.0) / np.where(p == s, f32(2.0), f32(1.0))).astype(f32)
    else:
        h = ((p + s) / f32(2.0)).astype(f32)
    x = (h * e).sum(1, dtype=f32)
    lo, g = pointwise_loss_and_grad(loss, labels, x)
    reg = f32(reg)
    dh = (g[:, None] * e).astype(f32)
    if pre_max:
        dp = np.where(p == h, share * dh, f32(0)).astype(f32)
        ds = np.where(s == h, share * dh, f32(0)).astype(f32)
    else:
        dp = ds = (dh / f32(2.0)).astype(f32)
    if session_max:
        dR = np.where(ind, (f32(1.0) / num)[:, None, :] * ds[:, None, :], f32(0)).astype(f32)
    else:
        dR = np.broadcast_to((ds / f32(L))[:, None, :], R.shape).astype(f32)
    gP, gE = np.zeros_like(P), np.zeros_like(E)
    _add_rows(gP, u, (dp + reg * p).astype(f32))
    _add_rows(gE, i, (g[:, None] * h + reg * e).astype(f32))
    _add_rows(gE, w.reshape(-1), (dR + reg * R).reshape(-1, E.shape[1]).astype(f32))
    sq = sum((t * t).sum(dtype=f32) for t in (p, R, e))
    total = lo.sum(dtype=f32) + reg * f32(0.5) * f32(sq)
    return f32(total), (gP, gE), (_mask(P.shape[0], u), _mask(E.shape[0], w.reshape(-1), i))


def npe_grad(UI, IU, IL, users, recent, items, labels, loss, reg=0.0):
    """NPE._create_loss (NPE.py:67-71) -> (loss, (gUI, gIU, gIL), (tU, tI, tL)).  c = sum_l IL[w_l],
    x = <relu(UI_u), relu(IU_i)> + <relu(IU_i), relu(c)>; tU <- users, tI <- items, tL <- window items."""
    UI, IU, IL = (np.asarray(a, f32) for a in (UI, IU, IL))
    u, i = np.asarray(users), np.asarray(items)
    w = _windows(recent, len(u))
    a, q, R = UI[u], IU[i], IL[w]
    c = R.sum(1, dtype=f32)
    ra, rq, rc = np.maximum(a, f32(0)), np.maximum(q, f32(0)), np.maximum(c, f32(0))
    x = (ra * rq + rq * rc).sum(1, dtype=f32)
    lo, g = pointwise_loss_and_grad(loss, labels, x)
    reg = f32(reg)
    g = g[:, None]
    gUI, gIU, gIL = np.zeros_like(UI), np.zeros_like(IU), np.zeros_like(IL)
    _add_rows(gUI, u, (np.where(a > 0, g * rq, f32(0)) + reg * a).astype(f32))
    _add_rows(gIU, i, (np.where(q > 0, g * ra + g * rc, f32(0)) + reg * q).astype(f32))
    dc = np.where(c > 0, g * rq, f32(0)).astype(f32)
    _add_rows(gIL, w.reshape(-1), (dc[:, None, :] + reg * R).reshape(-1, IL.shape[1]).astype(f32))
    sq = sum((t * t).sum(dtype=f32) for t in (a, q, R))
    total = lo.sum(dtype=f32) + reg * f32(0.5) * f32(sq)
    return f32(total), (gUI, gIU, gIL), (_mask(UI.shape[0], u), _mask(IU.shape[0], i), _mask(IL.shape[0], w.reshape(-1)))


def predict_window(seq, high_order):
    """The reference's cand_items[len(cand_items) - high_order:] (HRM.py:144, NPE.py:123), as Python evaluates it."""
    return list(seq)[len(seq) - high_order:]


def hrm_scores(P, E, users, windows, pre_max, session_max):
    """HRM.predict in fp64: [rows, num_items]; windows[r] is row r's window (any length >= 1)."""
    P, E = np.asarray(P, np.float64), np.asarray(E, np.float64)
    out = []
    for u, w in zip(users, windows):
        R = E[np.asarray(w, np.int64)]
        s = R.max(0) if session_max else R.mean(0)
        h = np.maximum(P[u], s) if pre_max else (P[u] + s) / 2
        out.append(E @ h)
    return np.asarray(out)


def npe_scores(UI, IU, IL, users, windows):
    """NPE.predict in fp64: [rows, num_items]."""
    UI, IU, IL = (np.asarray(a, np.float64) for a in (UI, IU, IL))
    rq = np.maximum(IU, 0)
    out = []
    for u, w in zip(users, windows):
        c = IL[np.asarray(w, np.int64)].sum(0)
        out.append(rq @ np.maximum(UI[u], 0) + rq @ np.maximum(c, 0))
    return np.asarray(out)


class HRMTrainer(_SeqTrainer):
    """HRM.build_graph + train_model's batch loop (HRM.py:97-126); variables P, E."""

    def __init__(self, P, E, learner="adam", lr=1e-3, loss="cross_entropy", reg=0.0, pre_max=True, session_max=True):
        super().__init__((P, E), learner, lr, loss, reg, False)
        self.pre_max, self.session_max = pre_max, session_max

    def step(self, users, recent, items, labels):
        l, grads, touched = hrm_grad(*self.vars, users, recent, items, labels, self.pre_max, self.session_max,
                                     self.loss, self.reg)
        self._apply(grads, touched, (False, False))
        return l


class NPETrainer(_SeqTrainer):
    """NPE.build_graph + train_model's batch loop (NPE.py:77-105); variables UI, IU, IL."""

    def __init__(self, UI, IU, IL, learner="adam", lr=1e-3, loss="cross_entropy", reg=0.1):
        super().__init__((UI, IU, IL), learner, lr, loss, reg, False)

    def step(self, users, recent, items, labels):
        l, grads, touched = npe_grad(*self.vars, users, recent, items, labels, self.loss, self.reg)
        self._apply(grads, touched, (False,) * 3)
        return l
