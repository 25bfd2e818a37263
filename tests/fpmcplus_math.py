"""TEST INFRASTRUCTURE ONLY -- numpy restatement (fp32 or fp64) of the reference's FPMCplus graph, hand-derived
gradients, batch loop and predict, in the style of tests/seq_math.py (whose trainer base it extends; the fp32 losses
and optimizer rules come from oracle/tf_math.py).

Restated call sites (paths relative to the reference):
  model/sequential_recommender/FPMCplus.py:53-71     variables UI, IU, IL, LI, W [3d, w], b [1, w], h [w, 1]
  model/sequential_recommender/FPMCplus.py:73-106    attention MLP over the window, conditioned on the item
  model/sequential_recommender/FPMCplus.py:108-119   pairwise / pointwise loss and regularisers
  model/sequential_recommender/FPMCplus.py:141-171   batch loop
  model/sequential_recommender/FPMCplus.py:177-205   predict from each user's last high_order train items
TensorFlow pieces: tanh's gradient is grad * (1 - y * y) (TanhGrad); matmul gradients of W, b and h are dense
tensors (the Apply* optimizer formulas); every embedding_lookup gradient is an IndexedSlices whose rows are the
touched set of its variable, and l2_loss counts every gathered row, window rows included.  The manual gradients are
checked against torch.autograd in tests/test_fpmcplus.py.
"""
import numpy as np
import torch

from oracle.tf_math import pairwise_loss_and_grad, pointwise_loss_and_grad
from seq_math import _mask, _SeqTrainer

f32 = np.float32


def _losses(pairwise, kind, third, x, dt):
    """(per-sample loss, dl/dx) in dtype dt: oracle/tf_math's fp32 functions, or the same formulas in fp64."""
    if dt == f32:
        return pairwise_loss_and_grad(kind, x) if pairwise else pointwise_loss_and_grad(kind, third, x)
    if pairwise:
        if kind == "bpr":
            return np.logaddexp(0.0, -x), -1.0 / (1.0 + np.exp(x))
        if kind == "hinge":
            return np.maximum(x + 1.0, 0.0), (x + 1.0 > 0).astype(dt)
        return (1.0 - x) ** 2, -2.0 * (1.0 - x)
    z = np.asarray(third, dt)
    if kind == "cross_entropy":
        n = len(x)
        return (np.maximum(x, 0) - x * z + np.log1p(np.exp(-np.abs(x)))) / n, (1.0 / (1.0 + np.exp(-x)) - z) / n
    return (z - x) ** 2, -2.0 * (z - x)


def _add_rows(dst, ids, rows):
    """dst[ids[k]] += rows[k] for every k, duplicates summed."""
    torch.from_numpy(dst).index_add_(0, torch.from_numpy(np.asarray(ids, np.int64).reshape(-1)),
                                     torch.from_numpy(np.ascontiguousarray(rows, dtype=dst.dtype)))


def attention(a, il, R, W, b, h):
    """FPMCplus._attention_mlp (:73-93) for a batch: a = UI_u [B, d], il = IL_i [B, d], R = LI[window] [B, L, d]
    -> (tanh outputs t [B, L, w], attention weights [B, L]).  exp without a max shift, as the reference: exp(e) of
    an e beyond the dtype's range is inf, and inf / inf makes that row's weights NaN."""
    d = a.shape[1]
    A = a @ W[:d] + b.reshape(1, -1)
    B = il @ W[d:2 * d]
    C = R @ W[2 * d:]
    t = np.tanh((A + B)[:, None, :] + C)
    e = t @ h.reshape(-1)
    with np.errstate(over="ignore", invalid="ignore"):
        ex = np.exp(e)
        att = ex / ex.sum(1, keepdims=True)
    return t, att


def fpmcplus_grad(UI, IU, IL, LI, W, b, h, users, recent, items, third, pairwise, loss, reg_mf=0.0, reg_w=0.0,
                  dtype=f32):
    """FPMCplus._create_loss (:108-119) -> (loss, (gUI, gIU, gIL, gLI, gW, gb, gh), (tU, tI, tL)).  recent [B, L]
    (or [B] at L = 1); tU <- users, tI <- items + negatives (IU and IL), tL <- window items (LI)."""
    dt = dtype
    UI, IU, IL, LI, W = (np.asarray(v, dt) for v in (UI, IU, IL, LI, W))
    b, h = np.asarray(b, dt).reshape(-1), np.asarray(h, dt).reshape(-1)
    u, i = np.asarray(users), np.asarray(items)
    w = np.asarray(recent, np.int64).reshape(len(u), -1)
    d = UI.shape[1]
    a, R = UI[u], LI[w]

    def side(item):
        il = IL[item]
        t, att = attention(a, il, R, W, b, h)
        q = np.einsum("bd,bld->bl", il, R)
        s = np.einsum("bl,bld->bd", att, R)
        x = (a * IU[item]).sum(1) + (il * s).sum(1)
        return dict(il=il, iu=IU[item], t=t, att=att, q=q, s=s, x=x)

    P = side(i)
    sides = [(P, i, dt(1.0))]
    if pairwise:
        N = side(np.asarray(third))
        sides.append((N, np.asarray(third), dt(-1.0)))
        lo, c = _losses(True, loss, None, P["x"] - N["x"], dt)
    else:
        lo, c = _losses(False, loss, third, P["x"], dt)
    c = np.asarray(c, dt)
    gUI, gIU, gIL, gLI = (np.zeros_like(v) for v in (UI, IU, IL, LI))
    gW, gb, gh = np.zeros_like(W), np.zeros_like(b), np.zeros_like(h)
    reg_mf, reg_w = dt(reg_mf), dt(reg_w)
    for S, item, sign in sides:
        cs = (sign * c)[:, None]
        y = (S["att"] * S["q"]).sum(1, keepdims=True)
        de = cs * S["att"] * (S["q"] - y)                                      # dl/de [B, L]
        dz = (de[:, :, None] * h) * (dt(1.0) - S["t"] * S["t"])               # [B, L, w]
        dzs = dz.sum(1)
        gW[:d] += a.T @ dzs
        gW[d:2 * d] += S["il"].T @ dzs
        gW[2 * d:] += np.einsum("bld,blw->dw", R, dz)
        gb += dzs.sum(0)
        gh += np.einsum("bl,blw->w", de, S["t"])
        _add_rows(gUI, u, cs * S["iu"] + dzs @ W[:d].T)
        _add_rows(gIU, item, cs * a + reg_mf * S["iu"])
        _add_rows(gIL, item, cs * S["s"] + dzs @ W[d:2 * d].T + reg_mf * S["il"])
        _add_rows(gLI, w.reshape(-1), (S["att"][:, :, None] * (cs * S["il"])[:, None, :] + dz @ W[2 * d:].T)
                  .reshape(-1, d))
    _add_rows(gUI, u, reg_mf * a)
    _add_rows(gLI, w.reshape(-1), (reg_mf * R).reshape(-1, d))
    sq = sum((v * v).sum(dtype=dt) for v in [a, R] + [S["iu"] for S, _, _ in sides] + [S["il"] for S, _, _ in sides])
    total = lo.sum(dtype=dt) + reg_mf * dt(0.5) * dt(sq)
    if pairwise:
        gW += reg_w * W
        gh += reg_w * h
        total = total + reg_w * (dt(0.5) * (W * W).sum(dtype=dt) + dt(0.5) * (h * h).sum(dtype=dt))
    ids = [i] + ([np.asarray(third)] if pairwise else [])
    touched = (_mask(UI.shape[0], u), _mask(IU.shape[0], *ids), _mask(LI.shape[0], w.reshape(-1)))
    return dt(total), (gUI, gIU, gIL, gLI, gW, gb.reshape(1, -1), gh.reshape(-1, 1)), touched


def fpmcplus_scores(UI, IU, IL, LI, W, b, h, users, windows, dtype=np.float64):
    """FPMCplus.predict in `dtype`: [rows, num_items]; windows[r] is row r's window (any length >= 1), and the softmax
    runs over its length."""
    UI, IU, IL, LI, W = (np.asarray(v, dtype) for v in (UI, IU, IL, LI, W))
    b, h = np.asarray(b, dtype), np.asarray(h, dtype)
    ni = IU.shape[0]
    out = []
    for u, win in zip(users, windows):
        R = np.broadcast_to(LI[np.asarray(win, np.int64)], (ni, len(win), UI.shape[1]))
        a = np.broadcast_to(UI[u], (ni, UI.shape[1]))
        _, att = attention(a, IL, R, W, b, h)
        with np.errstate(invalid="ignore"):
            s = np.einsum("bl,bld->bd", att, R)
            out.append(IU @ UI[u] + (IL * s).sum(1))
    return np.asarray(out)


class FPMCplusTrainer(_SeqTrainer):
    """FPMCplus.build_graph + train_model's batch loop (:125-171); variables UI, IU, IL, LI (IndexedSlices) and
    W, b, h (dense)."""

    def __init__(self, UI, IU, IL, LI, W, b, h, learner="adam", lr=1e-3, loss="bpr", reg_mf=1e-5, reg_w=1e-3,
                 pairwise=True):
        super().__init__((UI, IU, IL, LI, W, b, h), learner, lr, loss, reg_mf, pairwise)
        self.reg_w = reg_w

    def step(self, users, recent, items, third):
        l, grads, (tU, tI, tL) = fpmcplus_grad(*self.vars, users, recent, items, third, self.pairwise, self.loss,
                                               self.reg, self.reg_w)
        self._apply(grads, (tU, tI, tI, tL, None, None, None), (False,) * 4 + (True,) * 3)
        return l
