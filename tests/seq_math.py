"""TEST INFRASTRUCTURE ONLY -- numpy fp32 restatement of the reference's FPMC and TransRec graphs and batch loops,
in the style of oracle/tf_math.py (whose losses, optimizer rules and Adam lr_t it reuses).

Restated call sites (paths relative to the reference):
  model/sequential_recommender/FPMC.py:61-84,106-131       four-table score, pairwise / pointwise loss, batch loop
  model/sequential_recommender/TransRec.py:66-91,119-141   squared translation distance, loss, batch loop
  model/sequential_recommender/TransRec.py:102-107         prediction graph (Euclidean distance, not squared)
TensorFlow pieces as in oracle/tf_math.py: every embedding_lookup gradient is an IndexedSlices whose rows are the
touched set of its variable (several lookups of one variable concatenate and sum); TransRec's global vector g enters
through tf.tile and directly through l2_loss, so its gradient is a dense tensor (the Apply* optimizer formulas) and
its reg term is counted once per batch.  The manual gradients are checked against torch.autograd in
tests/test_sequential.py.
"""
import numpy as np

from oracle.tf_math import (DEFAULT_HYPER, SLOT_INIT, adam_lr_t, opt_apply, pairwise_loss_and_grad,
                            pointwise_loss_and_grad)

f32 = np.float32


def _loss(pairwise, kind, third, x_pos, x_neg=None):
    if pairwise:
        return pairwise_loss_and_grad(kind, x_pos - x_neg)
    return pointwise_loss_and_grad(kind, third, x_pos)


def _mask(rows, *ids):
    m = np.zeros(rows, bool)
    for a in ids:
        m[a] = True
    return m


def fpmc_grad(UI, IU, IL, LI, users, recent, items, third, pairwise, loss, reg=0.0):
    """FPMC._create_loss (FPMC.py:72-84) -> (loss, (gUI, gIU, gIL, gLI), (tU, tI, tL)).
    x(u, l, i) = <UI_u, IU_i> + <IL_i, LI_l>; tU <- users, tI <- items + negatives (IU and IL), tL <- recent."""
    UI, IU, IL, LI = (np.asarray(a, f32) for a in (UI, IU, IL, LI))
    u, l, i = users, recent, items
    a, ui, li, r = UI[u], IU[i], IL[i], LI[l]
    xi = (a * ui + li * r).sum(1, dtype=f32)
    reg = f32(reg)
    gUI, gIU, gIL, gLI = (np.zeros_like(t) for t in (UI, IU, IL, LI))
    sq = sum((t * t).sum(dtype=f32) for t in (a, ui, li, r))
    if pairwise:
        j = third
        uj, lj = IU[j], IL[j]
        xj = (a * uj + lj * r).sum(1, dtype=f32)
        lo, c = _loss(True, loss, None, xi, xj)
        sq = sq + (uj * uj).sum(dtype=f32) + (lj * lj).sum(dtype=f32)
        c = c[:, None]
        np.add.at(gUI, u, (c * (ui - uj) + reg * a).astype(f32))
        np.add.at(gIU, i, (c * a + reg * ui).astype(f32))
        np.add.at(gIU, j, (-c * a + reg * uj).astype(f32))
        np.add.at(gIL, i, (c * r + reg * li).astype(f32))
        np.add.at(gIL, j, (-c * r + reg * lj).astype(f32))
        np.add.at(gLI, l, (c * (li - lj) + reg * r).astype(f32))
        tI = _mask(IU.shape[0], i, j)
    else:
        lo, c = _loss(False, loss, third, xi)
        c = c[:, None]
        np.add.at(gUI, u, (c * ui + reg * a).astype(f32))
        np.add.at(gIU, i, (c * a + reg * ui).astype(f32))
        np.add.at(gIL, i, (c * r + reg * li).astype(f32))
        np.add.at(gLI, l, (c * li + reg * r).astype(f32))
        tI = _mask(IU.shape[0], i)
    total = lo.sum(dtype=f32) + reg * f32(0.5) * f32(sq)
    return f32(total), (gUI, gIU, gIL, gLI), (_mask(UI.shape[0], u), tI, _mask(LI.shape[0], l))


def transrec_grad(P, Q, B, G, users, recent, items, third, pairwise, loss, reg=0.0):
    """TransRec._create_loss (TransRec.py:80-91) -> (loss, (gP, gQ, gB, gG), (tP, tQ, tB)).
    v = ((P_u + g) + Q_l) - Q_i, x = b_i - |v|^2; tP <- users, tQ <- recent + items + negatives, tB <- items +
    negatives; gG is g's dense gradient [d] with reg * g counted once."""
    P, Q, B = (np.asarray(a, f32) for a in (P, Q, B))
    G = np.asarray(G, f32).reshape(-1)
    u, l, i = users, recent, items
    p, r, qi, bi = P[u], Q[l], Q[i], B[i]
    x = (p + G) + r
    vi = x - qi
    xi = bi - (vi * vi).sum(1, dtype=f32)
    reg = f32(reg)
    gP, gQ, gB = np.zeros_like(P), np.zeros_like(Q), np.zeros_like(B)
    sq = sum((t * t).sum(dtype=f32) for t in (p, r, qi, bi))
    two = f32(2.0)
    if pairwise:
        j = third
        qj, bj = Q[j], B[j]
        vj = x - qj
        xj = bj - (vj * vj).sum(1, dtype=f32)
        lo, c = _loss(True, loss, None, xi, xj)
        sq = sq + (qj * qj).sum(dtype=f32) + (bj * bj).sum(dtype=f32)
        e = -two * c[:, None] * (vi - vj)
        np.add.at(gQ, j, (-two * c[:, None] * vj + reg * qj).astype(f32))
        np.add.at(gB, j, (-c + reg * bj).astype(f32))
        tQ, tB = _mask(Q.shape[0], l, i, j), _mask(B.shape[0], i, j)
    else:
        lo, c = _loss(False, loss, third, xi)
        e = -two * c[:, None] * vi
        tQ, tB = _mask(Q.shape[0], l, i), _mask(B.shape[0], i)
    e = e.astype(f32)
    np.add.at(gP, u, (e + reg * p).astype(f32))
    np.add.at(gQ, l, (e + reg * r).astype(f32))
    np.add.at(gQ, i, (two * c[:, None] * vi + reg * qi).astype(f32))
    np.add.at(gB, i, (c + reg * bi).astype(f32))
    gG = (e.sum(0, dtype=f32) + reg * G).astype(f32)
    total = lo.sum(dtype=f32) + reg * f32(0.5) * (f32(sq) + (G * G).sum(dtype=f32))
    return f32(total), (gP, gQ, gB, gG), (_mask(P.shape[0], u), tQ, tB)


def fpmc_scores(UI, IU, IL, LI, users, recent):
    """FPMC.predict (FPMC.py:140-165) in fp64: [rows, num_items]."""
    UI, IU, IL, LI = (np.asarray(a, np.float64) for a in (UI, IU, IL, LI))
    return UI[users] @ IU.T + LI[recent] @ IL.T


def transrec_scores(P, Q, B, G, users, recent):
    """TransRec's prediction graph (TransRec.py:102-107) in fp64: b_j - |(P_u + g) + Q_l - Q_j|, from the differences."""
    P, Q, B = (np.asarray(a, np.float64) for a in (P, Q, B))
    x = (P[users] + np.asarray(G, np.float64).reshape(1, -1)) + Q[recent]
    d = x[:, None, :] - Q[None, :, :]
    return B[None, :] - np.sqrt((d * d).sum(-1))


class _SeqTrainer:
    """CPU stand-in for build_graph + the sess.run((loss, optimizer)) batch loop over the model's variables."""

    def __init__(self, tables, learner, lr, loss, reg, pairwise):
        self.vars = [np.array(t, dtype=f32) for t in tables]
        self.learner, self.lr, self.loss, self.reg, self.pairwise = learner, lr, loss, reg, pairwise
        i0, i1 = SLOT_INIT[learner]
        mk = lambda a, v: None if v is None else np.full_like(a, v)
        self.slots = [(mk(a, i0), mk(a, i1)) for a in self.vars]
        self.t = 0

    def _apply(self, grads, touched, dense):
        hyper = DEFAULT_HYPER[self.learner](self.lr)
        if self.learner == "adam":
            hyper[0] = adam_lr_t(self.lr, 1, start_step=self.t)[0]
        for var, g, (s0, s1), tch, dv in zip(self.vars, grads, self.slots, touched, dense):
            opt_apply(self.learner, var, g.reshape(var.shape), s0, s1, tch, hyper, dense_var=dv)
        self.t += 1

    def epoch(self, users, recent, items, third, batch_size):
        n = len(users)
        losses = []
        for off in range(0, n, batch_size):
            sl = slice(off, min(n, off + batch_size))
            losses.append(self.step(users[sl], recent[sl], items[sl], third[sl]))
        return np.asarray(losses, dtype=f32)


class FPMCTrainer(_SeqTrainer):
    """FPMC.build_graph + train_model's batch loop (FPMC.py:86-131); variables UI, IU, IL, LI."""

    def __init__(self, UI, IU, IL, LI, learner="adam", lr=1e-3, loss="cross_entropy", reg=0.01, pairwise=False):
        super().__init__((UI, IU, IL, LI), learner, lr, loss, reg, pairwise)

    def step(self, users, recent, items, third):
        l, grads, (tU, tI, tL) = fpmc_grad(*self.vars, users, recent, items, third, self.pairwise, self.loss, self.reg)
        self._apply(grads, (tU, tI, tI, tL), (False,) * 4)
        return l


class TransRecTrainer(_SeqTrainer):
    """TransRec.build_graph + train_model's batch loop (TransRec.py:93-141); variables P, Q, b, g (g dense)."""

    def __init__(self, P, Q, B, G, learner="adam", lr=1e-3, loss="bpr", reg=0.0, pairwise=True):
        super().__init__((P, Q, B, G), learner, lr, loss, reg, pairwise)

    def step(self, users, recent, items, third):
        l, grads, (tP, tQ, tB) = transrec_grad(*self.vars, users, recent, items, third, self.pairwise, self.loss,
                                               self.reg)
        self._apply(grads, (tP, tQ, tB, None), (False, False, False, True))
        return l
