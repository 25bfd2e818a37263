"""TEST INFRASTRUCTURE ONLY -- numpy restatement (fp32 or fp64) of the reference's Caser graph, hand-derived gradients
and batch loop, checked against torch.autograd in tests/test_caser.py and against the kernels in
tests/test_gpu_caser.py.

Restated call sites (paths relative to the reference):
  model/sequential_recommender/Caser.py:37-68     variables P, E (+ zero pad row), W2, b2; conv_v, conv_h, fc1
  model/sequential_recommender/Caser.py:70-118    the convolutional graph, the sigmoid losses and the l2 terms
  model/sequential_recommender/Caser.py:124-142   batch loop: Adam per batch
  model/sequential_recommender/Caser.py:194-209   predict: [z, P_u] W2^T without the biases
TensorFlow pieces, read from TF 1.12's source (TF itself is not installable here):
  * reduce_max's gradient (_MinOrMaxGrad) is (indicators / num_selected) * grad: tied maxima share it equally;
  * relu's gradient passes where its output is > 0; nn.dropout is (x / keep) * mask, its gradient (g * mask) / keep;
  * l2_regularizer(s)(w) = s * sum(w^2) / 2, so each table's gradient gets l2_reg * w on every row.  The lookups'
    IndexedSlices and that dense term are aggregated into IndexedSlices covering every row, so the four tables take
    Adam's sparse form on every row; the conv and FC weights (dense gradients) take ApplyAdam's form;
  * a pad target (id I, outside item_embeddings) reads a zero row and a zero bias, what the GPU gather returns.
"""
import numpy as np

from oracle import tf_math

f32 = np.float32


def dense_layout(d, L, nv, nh):
    """[(name, offset, shape)] of the dense block in TF's creation order, and its total size."""
    out, off = [], 0
    shapes = [("Kv", (L, 1, 1, nv)), ("bv", (nv,))]
    for h in range(1, L + 1):
        shapes += [("Kh%d" % h, (h, d, 1, nh)), ("bh%d" % h, (nh,))]
    shapes += [("W1", (nv * d + nh * L, d)), ("b1", (d,))]
    for name, shape in shapes:
        out.append((name, off, shape))
        off += int(np.prod(shape))
    return out, off


def unpack(dense, d, L, nv, nh):
    return {name: dense[off:off + int(np.prod(shape))].reshape(shape) for name, off, shape in dense_layout(d, L, nv, nh)[0]}


def pack(parts, d, L, nv, nh):
    layout, n = dense_layout(d, L, nv, nh)
    out = np.zeros(n, dtype=parts["W1"].dtype)
    for name, off, shape in layout:
        out[off:off + int(np.prod(shape))] = np.asarray(parts[name]).reshape(-1)
    return out


def forward(P, E, dense, d, L, nv, nh, users, seqs, mask=None, keep=1.0, dt=np.float64):
    """-> dict of the forward's intermediates; u = [z, P_u] [B, 2d]."""
    V = {k: v.astype(dt) for k, v in unpack(dense, d, L, nv, nh).items()}
    Ez = np.concatenate([E, np.zeros((1, d))]).astype(dt)
    X = Ez[np.asarray(seqs)]                                            # [B, L, d]
    B = X.shape[0]
    Kv = V["Kv"].reshape(L, nv)
    out_v = (np.einsum("blk,lf->bkf", X, Kv) + V["bv"]).reshape(B, d * nv)
    acts, out_h = [], []
    for h in range(1, L + 1):
        Kh = V["Kh%d" % h].reshape(h, d, nh)
        pre = np.stack([np.einsum("blk,lkf->bf", X[:, t:t + h], Kh) for t in range(L - h + 1)], 1) + V["bh%d" % h]
        a = np.maximum(pre, 0)
        acts.append(a)
        out_h.append(a.max(1))
    feat = np.concatenate([out_v] + out_h, 1)
    o = feat if mask is None else (feat / dt(keep)) * np.asarray(mask, dt)
    zp = o @ V["W1"] + V["b1"]
    z = np.maximum(zp, 0)
    u = np.concatenate([z, P[np.asarray(users)].astype(dt)], 1)
    return dict(V=V, X=X, acts=acts, o=o, z=z, u=u)


def query(P, E, dense, d, L, nv, nh, users, windows, dt=np.float64):
    """predict's user vectors [z, P_u] without dropout (windows: one row per user in `users`)."""
    return forward(P, E, dense, d, L, nv, nh, users, windows, dt=dt)["u"]


def loss_and_grad(P, E, W2, b2, dense, d, L, nv, nh, users, seqs, pos, neg, mask=None, keep=1.0, dt=np.float64):
    """Data loss and the gradients (gP, gE, gW2, gb2, gdense) of one batch, without the l2 terms."""
    I = E.shape[0]
    users, seqs, pos, neg = (np.asarray(a) for a in (users, seqs, pos, neg))
    f = forward(P, E, dense, d, L, nv, nh, users, seqs, mask, keep, dt)
    V, X, u, z, o = f["V"], f["X"], f["u"], f["z"], f["o"]
    B, T, N = len(users), pos.shape[1], neg.shape[1]
    tgt = np.concatenate([pos, neg], 1)
    W2z = np.concatenate([W2, np.zeros((1, 2 * d))]).astype(dt)
    b2z = np.concatenate([b2, [0.0]]).astype(dt)
    x = np.einsum("bk,bjk->bj", u, W2z[tgt]) + b2z[tgt]
    s = 1.0 / (1.0 + np.exp(-x))
    eps = dt(1e-24)
    loss = np.mean(-np.log(s[:, :T] + eps)) + np.mean(-np.log((1.0 - s[:, T:]) + eps))
    c = np.empty_like(x)
    c[:, :T] = (dt(-1.0 / (B * T)) * (1.0 / (s[:, :T] + eps))) * s[:, :T] * (1.0 - s[:, :T])
    c[:, T:] = (dt(1.0 / (B * N)) * (1.0 / ((1.0 - s[:, T:]) + eps))) * s[:, T:] * (1.0 - s[:, T:])
    real = tgt != I
    gW2 = np.zeros((I + 1, 2 * d), dt)
    np.add.at(gW2, tgt[real], (c[..., None] * u[:, None, :])[real])
    gb2 = np.zeros(I + 1, dt)
    np.add.at(gb2, tgt[real], c[real])
    du = np.einsum("bj,bjk->bk", c, W2z[tgt])
    gP = np.zeros(P.shape, dt)
    np.add.at(gP, users, du[:, d:])
    dzp = du[:, :d] * (z > 0)
    g = {"W1": o.T @ dzp, "b1": dzp.sum(0)}
    do = dzp @ V["W1"].T
    dfeat = do if mask is None else (do * np.asarray(mask, dt)) / dt(keep)
    dv = dfeat[:, :nv * d].reshape(B, d, nv)
    Kv = V["Kv"].reshape(L, nv)
    g["Kv"], g["bv"] = np.einsum("blk,bkf->lf", X, dv), dv.sum((0, 1))
    dX = np.einsum("bkf,lf->blk", dv, Kv)
    for h in range(1, L + 1):
        a = f["acts"][h - 1]
        gh = dfeat[:, nv * d + (h - 1) * nh:nv * d + h * nh]
        ind = (a == a.max(1, keepdims=True)).astype(dt)
        dpre = (ind / ind.sum(1, keepdims=True)) * gh[:, None, :] * (a > 0)
        Kh = V["Kh%d" % h].reshape(h, d, nh)
        gK = np.zeros_like(Kh)
        for t in range(L - h + 1):
            gK += np.einsum("blk,bf->lkf", X[:, t:t + h], dpre[:, t])
            dX[:, t:t + h] += np.einsum("bf,lkf->blk", dpre[:, t], Kh)
        g["Kh%d" % h], g["bh%d" % h] = gK, dpre.sum((0, 1))
    gE = np.zeros((I + 1, d), dt)
    np.add.at(gE, seqs, dX)
    return loss, (gP, gE[:I], gW2[:I], gb2[:I], pack(g, d, L, nv, nh))


class CaserTrainer(object):
    """The reference's batch loop in fp32: per batch, the data gradients plus l2_reg * var on every table, then Adam
    (the sparse form on the four tables, ApplyAdam's on the dense block)."""

    def __init__(self, P, E, W2, b2, dense, d, L, nv, nh, lr=1e-3, l2_reg=1e-3, keep=0.5):
        self.vars = [np.array(v, dtype=f32) for v in (P, E, W2, b2, dense)]
        self.s0 = [np.zeros_like(v) for v in self.vars]
        self.s1 = [np.zeros_like(v) for v in self.vars]
        self.shape, self.lr, self.reg, self.keep, self.t = (d, L, nv, nh), lr, f32(l2_reg), keep, 0

    def step(self, users, seqs, pos, neg, mask, lr_t):
        loss, grads = loss_and_grad(*self.vars, *self.shape, users, seqs, pos, neg, mask, self.keep, dt=f32)
        for k, (v, g) in enumerate(zip(self.vars, grads)):
            g = g.astype(f32) + (self.reg * v if k < 4 else 0)
            tf_math.opt_apply("adam", v, g, self.s0[k], self.s1[k], None, [lr_t, 0.9, 0.999, 1e-8], dense_var=k == 4)
        return loss

    def epoch(self, users, seqs, pos, neg, masks, batch_size):
        n = len(users)
        steps = (n + batch_size - 1) // batch_size
        lr_t = tf_math.adam_lr_t(self.lr, steps, start_step=self.t)
        out = np.zeros(steps, dtype=np.float64)
        for s in range(steps):
            sl = slice(s * batch_size, (s + 1) * batch_size)
            out[s] = self.step(users[sl], seqs[sl], pos[sl], neg[sl], masks[s], lr_t[s])
        self.t += steps
        return out
