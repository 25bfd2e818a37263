"""Every route the MF training kernels (csrc/train_mf.cu, csrc/epoch.cu, csrc/optim.cu) take from a shape, against
float64.

The routes depend on the SM count: the gradient kernel and the id-fed in-place step cap their grid at 8 CTAs of 8
warps per SM and loop beyond 64 * SMs triplets; the lazy-Adam kernel caps at 8 CTAs of 256 threads per SM and loops
beyond 2048 * SMs; the persistent epoch kernel has 16 warps per SM and loops when a batch has more samples; the
CSR-fed step runs one persistent grid of 768-thread CTAs and holds T = 8192 / dim head rows in shared memory.  Every
shape below is derived from the device's SM count, one case on each side of each boundary; each test asserts the route
it ran through nrc_mf_last_routes, and the last test of the file checks that the whole file saw every route.

Exact tests: tables of small integers times 2^-k, hinge or square loss (or BPR at x = 0, where g = -1/2 exactly), lr and
reg powers of two.  Every partial sum is then a multiple of its granule below 2^24 granules (asserted from the float64
magnitudes by `assert_exact`), so fp32 is exact in any summation order and every route must equal float64 bit for bit.
The optimizers' arithmetic is correctly rounded (`__f*_rn`), so with an exact gradient the tables and slots must equal
the numpy restatement (oracle/tf_math.py) bit for bit.

In-place steps read rows while other triplets of the same launch update them.  They are exact when every row a triplet
reads still holds its pre-launch value: users live on the first half of the dimensions, where every item agrees, so every
score difference is 0; a user row touched once, an item row touched once, or a head row (read from the shared-memory
tier or the replica) is read before it changes.  Rows that some other triplet could have moved first are left out of the
comparison, and the tests assert that they are few.

Rounded tests: realistic values.  Each entry must lie within C * 2^-24 * M of float64, where M is a first-order bound
on the rounding error of the chain, carried in float64 alongside the values; C = 2.  The hogwild tests add the
interleaving term: what reading rows other triplets already moved can change, propagated through the loss's Lipschitz
constant, with a factor 2.  Each of them also checks that it would notice a lost delta or an lr off by 2^-8."""
import ctypes
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import oracle
from oracle import tf_math

gpu = pytest.mark.gpu
U24 = 2.0 ** -24
C_BOUND = 2.0
SEEN = set()
HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
OPTS = ("gd", "adam", "adagrad", "rmsprop", "momentum")
HYPER = {"gd": [2.0 ** -4], "adam": [2.0 ** -4, 0.9, 0.999, 1e-8], "adagrad": [2.0 ** -4],
         "rmsprop": [2.0 ** -4, 0.9, 0.5, 1e-10], "momentum": [2.0 ** -4, 0.5]}


def dev(a):
    return None if a is None else torch.from_numpy(np.ascontiguousarray(a)).cuda()


def sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def routes():
    from neurec_b200 import ops
    return ops.mf_last_routes()


def tier_rows(dim):
    return 8192 // dim


# ---------------------------------------------------------------------------------------------------------------
# the route predicates of the host code and the shapes on each side of them (pure functions of the SM count)
# ---------------------------------------------------------------------------------------------------------------
def grad_capped(batch, n_sms):
    """Grad kernel and id-fed step: ceil(batch / 8) CTAs of 8 warps over the 8 * SMs cap."""
    return (batch + 7) // 8 > 8 * n_sms


def lazy_capped(count, n_sms):
    return (count + 255) // 256 > 8 * n_sms


def epoch_capped(batch, n_sms):
    return batch > 16 * n_sms


def grad_batches(n_sms):
    return [1, 64 * n_sms, 64 * n_sms + 1, 3 * 64 * n_sms + 7]


def epoch_batches(n_sms):
    return [16 * n_sms, 16 * n_sms + 1]


def lazy_counts(n_sms):
    return [3000, 2048 * n_sms + 5]


@pytest.mark.parametrize("n_sms", [114, 132])
def test_route_shapes_straddle_every_boundary(n_sms):
    """CPU: the shapes derived from the SM count land on both sides of every route predicate (114: H100 PCIe,
    132: H100 SXM)."""
    b = grad_batches(n_sms)
    assert [grad_capped(x, n_sms) for x in b] == [False, False, True, True]
    e = epoch_batches(n_sms)
    assert not epoch_capped(e[0], n_sms) and epoch_capped(e[1], n_sms)
    c = lazy_counts(n_sms)
    assert not lazy_capped(c[0], n_sms) and lazy_capped(c[1], n_sms)
    for dim in (32, 64, 128):
        T = tier_rows(dim)
        assert [min(n, T) for n in (T - 1, T, T + 1, 4 * T)] == [T - 1, T, T, T]


# ---------------------------------------------------------------------------------------------------------------
# exactness precondition and bounds
# ---------------------------------------------------------------------------------------------------------------
def granule_bits(values, limit=60):
    """The smallest k with every value a multiple of 2^-k."""
    v = np.abs(np.asarray(values, np.float64)).ravel()
    for k in range(limit):
        s = v * 2.0 ** k
        if np.array_equal(s, np.round(s)):
            return k
    raise AssertionError("values are not dyadic")


def assert_exact(values, magnitude, what=""):
    """Every value is a multiple of 2^-bits and every partial sum (bounded by `magnitude`) stays below 2^24 such
    granules: fp32 represents each exactly, in any summation order."""
    bits = granule_bits(values)
    assert (np.asarray(magnitude, np.float64) * 2.0 ** bits < 2.0 ** 24).all(), (what, float(np.max(magnitude)))


def assert_within(got, want, M, what, C=C_BOUND):
    err = np.abs(np.asarray(got, np.float64) - want)
    bound = C * U24 * M
    assert (err <= bound).all(), (what, float((err - bound).max()), float(np.max(M)))


def dyadic(rs, shape, lo=-4, hi=4, k=4):
    return (rs.randint(lo, hi + 1, shape) / 2.0 ** k).astype(np.float32)


# ---------------------------------------------------------------------------------------------------------------
# the float64 gradient of a batch with its exactness precondition
# ---------------------------------------------------------------------------------------------------------------
def loss_grad64(kind, x, z=None):
    if kind == "hinge":
        assert not (x == -1.0).any(), "a hinge case sits on the tie x = -1"
        return np.maximum(x + 1, 0), (x + 1 > 0).astype(np.float64)
    if kind == "square":
        t = (1.0 - x) if z is None else (z - x)
        return t * t, -2.0 * t
    if kind == "bpr":
        assert (x == 0).all()
        return np.full_like(x, np.log(2.0)), np.full_like(x, -0.5)
    raise ValueError(kind)


def grad64(U, V, users, items, third, loss, reg, pairwise=True):
    """-> (per-sample loss, gU, gV) in float64, asserting that fp32 computes each exactly in any order."""
    U = U.astype(np.float64); V = V.astype(np.float64)
    pu, qi = U[users], V[items]
    if pairwise:
        qj = V[third]
        x = (pu * qi).sum(1) - (pu * qj).sum(1)
        mag_x = (np.abs(pu) * (np.abs(qi) + np.abs(qj))).sum(1)
        l, g = loss_grad64(loss, x)
        du = g[:, None] * (qi - qj) + reg * pu
        dvi = g[:, None] * pu + reg * qi
        dvj = -g[:, None] * pu + reg * qj
        parts = [pu * qi, pu * qj, x, g, du, dvi, dvj]
    else:
        x = (pu * qi).sum(1)
        mag_x = (np.abs(pu) * np.abs(qi)).sum(1)
        l, g = loss_grad64(loss, x, np.asarray(third, np.float64))
        du = g[:, None] * qi + reg * pu
        dvi = g[:, None] * pu + reg * qi
        parts = [pu * qi, x, g, du, dvi]
    gU = np.zeros_like(U); gV = np.zeros_like(V)
    mU = np.zeros_like(U); mV = np.zeros_like(V)
    np.add.at(gU, users, du); np.add.at(mU, users, np.abs(du))
    np.add.at(gV, items, dvi); np.add.at(mV, items, np.abs(dvi))
    if pairwise:
        np.add.at(gV, third, dvj); np.add.at(mV, third, np.abs(dvj))
    for p in parts:
        assert_exact(p, 0)
    assert_exact(x, mag_x, "scores")
    assert_exact(gU, mU, "user gradient"); assert_exact(gV, mV, "item gradient")
    return l, gU, gV


def no_hinge_tie(rs, U, V, users, pos, neg, ni):
    """Redraw negatives until no hinge case has x = -1 exactly (the tie of max(x + 1, 0) is out of scope here)."""
    for _ in range(100):
        x = (U[users].astype(np.float64) * (V[pos].astype(np.float64) - V[neg])).sum(1)
        tie = x == -1.0
        if not tie.any():
            return neg
        neg[tie] = rs.randint(0, ni, int(tie.sum()))
    raise AssertionError("could not leave the hinge tie")


# ---------------------------------------------------------------------------------------------------------------
# nrc_mf_pairwise_grad / nrc_mf_pointwise_grad: always the generic loop
# ---------------------------------------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("dim", [1, 31, 32, 33, 127, 129, 256])
@pytest.mark.parametrize("loss,reg", [("hinge", 0.0), ("square", 2.0 ** -3), ("bpr", 2.0 ** -3), ("pw_square", 0.0)])
def test_grad_exact(dim, loss, reg):
    """Batches 0, 1, 64 * SMs, 64 * SMs + 1 and a multiple of it with heavy duplicate rows; gradients and stamps bit for
    bit, the loss within its summation bound."""
    from neurec_b200 import ops
    n_sms = sms()
    rs = np.random.RandomState(dim * 7 + len(loss))
    pairwise = loss != "pw_square"
    kind = "square" if loss == "pw_square" else loss
    for bi, B in enumerate([0] + grad_batches(n_sms)):
        nu, ni = (37, 53) if bi == 4 else (B + 5, 2 * B + 5)       # the last batch repeats rows hundreds of times
        U = dyadic(rs, (nu, dim), -1, 1, 2)
        V = dyadic(rs, (ni, dim), -1, 1, 2)
        users = rs.randint(0, nu, B).astype(np.int32)
        pos = rs.randint(0, ni, B).astype(np.int32)
        if kind == "bpr":           # users on the first half, items agreeing there: x = 0, g = -1/2 exactly
            h = max(1, dim // 2)
            U[:, h:] = 0
            V[:, :h] = V[0, :h]
        if pairwise:
            third = rs.randint(0, ni, B).astype(np.int32)
            if kind == "hinge":
                third = no_hinge_tie(rs, U, V, users, pos, third, ni)
        else:
            third = rs.randint(0, 2, B).astype(np.float32)
        l, gU, gV = grad64(U, V, users, pos, third, kind, reg, pairwise)
        dU, dV = dev(np.zeros_like(U)), dev(np.zeros_like(V))
        tU = dev(np.full(nu, 5, np.int32)); tV = dev(np.full(ni, 5, np.int32))
        lo = torch.zeros(1, device="cuda")
        before = routes()["grad"]
        fn = ops.mf_pairwise_grad if pairwise else ops.mf_pointwise_grad
        fn(dev(U), dev(V), dev(users), dev(pos), dev(third), kind, reg, dU, dV, tU, tV, 9, lo)
        r = routes()["grad"]
        if B == 0:
            assert r == before and not dU.any() and not dV.any() and float(lo) == 0
            continue
        assert r["vec"] == 0 and r["capped"] == int(grad_capped(B, n_sms)) and r["grid"] == min((B + 7) // 8, 8 * n_sms)
        SEEN.add(("grad", "capped" if r["capped"] else "single"))
        assert np.array_equal(dU.cpu().numpy(), gU) and np.array_equal(dV.cpu().numpy(), gV)
        want_tU = np.full(nu, 5); want_tU[users] = 9
        want_tV = np.full(ni, 5); want_tV[pos] = 9
        if pairwise:
            want_tV[third] = 9
        assert np.array_equal(tU.cpu().numpy(), want_tU) and np.array_equal(tV.cpu().numpy(), want_tV)
        reg_l = 0.5 * reg * ((U[users].astype(np.float64) ** 2).sum() + (V[pos].astype(np.float64) ** 2).sum()
                             + ((V[third].astype(np.float64) ** 2).sum() if pairwise else 0))
        want_l = l.sum() + reg_l
        # summation in any order, one rounding per sample's loss, and log1pf(1) for BPR
        M = (B + dim + 4) * (np.abs(l).sum() + reg_l)
        assert_within(float(lo), want_l, M, "loss")
        SEEN.add(("grad_loss", loss))


@gpu
@pytest.mark.parametrize("pairwise", [True, False])
def test_grad_rounded_bpr_and_cross_entropy(pairwise):
    """BPR and cross-entropy on realistic values with |x| up to ~100 (past expf's overflow for BPR's exp(x)): every
    gradient element within the first-order bound of the float64 chain."""
    from neurec_b200 import ops
    n_sms = sms()
    rs = np.random.RandomState(3 + pairwise)
    nu, ni, dim = 3000, 4000, 64
    B = 64 * n_sms + 1
    U = (rs.randn(nu, dim) * rs.choice([0.05, 2.0], (nu, 1))).astype(np.float32)
    V = (rs.randn(ni, dim) * rs.choice([0.05, 2.0], (ni, 1))).astype(np.float32)
    users = rs.randint(0, nu, B).astype(np.int32)
    pos = rs.randint(0, ni, B).astype(np.int32)
    third = rs.randint(0, ni, B).astype(np.int32) if pairwise else rs.randint(0, 2, B).astype(np.float32)
    reg = float(np.float32(1e-3))
    U64, V64 = U.astype(np.float64), V.astype(np.float64)
    pu, qi = U64[users], V64[pos]
    if pairwise:
        qj = V64[third]
        x = (pu * qi).sum(1) - (pu * qj).sum(1)
        Mx = dim * (np.abs(pu) * (np.abs(qi) + np.abs(qj))).sum(1) + np.abs(x)
        g = -1.0 / (1.0 + np.exp(x))
        # expf 2 ulp, add, divide: 4 units of g; d g / dx = g (1 + g) <= 1/4
        Mg = 4 * np.abs(g) + np.abs(g * (1 + g)) * Mx
        diff = qi - qj
        du = g[:, None] * diff + reg * pu
        dvi = g[:, None] * pu + reg * qi
        dvj = -g[:, None] * pu + reg * qj
        Mdu = Mg[:, None] * np.abs(diff) + 3 * (np.abs(g[:, None] * diff) + np.abs(reg * pu))
        Mdvi = Mg[:, None] * np.abs(pu) + 2 * (np.abs(g[:, None] * pu) + np.abs(reg * qi))
        Mdvj = Mg[:, None] * np.abs(pu) + 2 * (np.abs(g[:, None] * pu) + np.abs(reg * qj))
    else:
        z = third.astype(np.float64)
        x = (pu * qi).sum(1)
        Mx = dim * (np.abs(pu) * np.abs(qi)).sum(1)
        s = 1.0 / (1.0 + np.exp(-x))
        g = (s - z) / B
        Mg = (5 * (np.abs(s) + np.abs(s - z)) + 0.25 * Mx + np.abs(g) * B) / B
        du = g[:, None] * qi + reg * pu
        dvi = g[:, None] * pu + reg * qi
        Mdu = Mg[:, None] * np.abs(qi) + 2 * (np.abs(g[:, None] * qi) + np.abs(reg * pu))
        Mdvi = Mg[:, None] * np.abs(pu) + 2 * (np.abs(g[:, None] * pu) + np.abs(reg * qi))
    assert np.abs(x).max() > 80
    gU = np.zeros_like(U64); gV = np.zeros_like(V64); MU = np.zeros_like(U64); MV = np.zeros_like(V64)
    cU = np.bincount(users, minlength=nu)[:, None].astype(np.float64)
    np.add.at(gU, users, du); np.add.at(MU, users, Mdu + np.abs(du) * cU[users])
    np.add.at(gV, pos, dvi); np.add.at(MV, pos, Mdvi)
    if pairwise:
        np.add.at(gV, third, dvj); np.add.at(MV, third, Mdvj)
        cV = np.bincount(np.concatenate([pos, third]), minlength=ni)[:, None]
        aV = np.zeros_like(V64); np.add.at(aV, pos, np.abs(dvi)); np.add.at(aV, third, np.abs(dvj))
    else:
        cV = np.bincount(pos, minlength=ni)[:, None]
        aV = np.zeros_like(V64); np.add.at(aV, pos, np.abs(dvi))
    MV += aV * cV
    dU, dV = dev(np.zeros_like(U)), dev(np.zeros_like(V))
    tU = dev(np.zeros(nu, np.int32)); tV = dev(np.zeros(ni, np.int32))
    lo = torch.zeros(1, device="cuda")
    if pairwise:
        ops.mf_pairwise_grad(dev(U), dev(V), dev(users), dev(pos), dev(third), "bpr", reg, dU, dV, tU, tV, 1, lo)
    else:
        ops.mf_pointwise_grad(dev(U), dev(V), dev(users), dev(pos), dev(third), "cross_entropy", reg, dU, dV, tU, tV, 1,
                              lo)
    assert routes()["grad"]["capped"] == 1
    assert_within(dU.cpu().numpy(), gU, MU, "user gradient")
    assert_within(dV.cpu().numpy(), gV, MV, "item gradient")
    SEEN.add(("grad_rounded", "bpr" if pairwise else "cross_entropy"))


# ---------------------------------------------------------------------------------------------------------------
# nrc_mf_epoch_fused: the persistent epoch kernel
# ---------------------------------------------------------------------------------------------------------------
def epoch_csr(rs, nu, ni, deg):
    rows = [rs.choice(ni, deg, replace=False) for _ in range(nu)]
    tp, ti = oracle.lists_to_csr(rows)
    return tp, ti, np.repeat(np.arange(nu, dtype=np.int32), np.diff(tp))


class EpochRun:
    """Device state of nrc_mf_epoch_fused and the numpy restatement stepped alongside it."""

    def __init__(self, U, V, opt, tp, ti, pu, ni, shuffle, drop_last, bs, loss, reg, seed=5, epoch=2):
        from neurec_b200 import ops
        self.ops = ops
        self.opt, self.loss, self.reg, self.bs = opt, loss, reg, bs
        self.args = (dev(tp), dev(ti), dev(pu), dev(ti))
        self.ni, self.shuffle, self.drop_last, self.seed, self.epoch = ni, shuffle, drop_last, seed, epoch
        i0, i1 = tf_math.SLOT_INIT[opt]
        mk = lambda a, v: np.full_like(a, 0.0 if v is None else v)
        self.host = {"U": U.copy(), "V": V.copy(), "s0U": mk(U, i0), "s1U": mk(U, i1), "s0V": mk(V, i0),
                     "s1V": mk(V, i1)}
        self.d = {k: dev(v) for k, v in self.host.items()}
        self.gU, self.gV = torch.zeros_like(self.d["U"]), torch.zeros_like(self.d["V"])
        self.tU = torch.zeros(U.shape[0], dtype=torch.int32, device="cuda")
        self.tV = torch.zeros(V.shape[0], dtype=torch.int32, device="cuda")
        wu, wi, wj = oracle.epoch_build(tp, ti, pu, ti, 1, ni, True, shuffle, seed, epoch)
        n = len(wu)
        self.n_used = (n // bs) * bs if drop_last else n
        self.steps = -(-self.n_used // bs)
        self.w = (wu, wi, wj[:, 0])
        self.ws = [torch.empty(n, dtype=torch.int32, device="cuda") for _ in range(3)]
        self.step_loss = torch.zeros(max(self.steps, 1), device="cuda")
        self.pows = torch.tensor([0.9, 0.999], device="cuda")
        self.stamp = 1
        self.t = 0

    def batch(self, s):
        sl = slice(s * self.bs, min(self.n_used, (s + 1) * self.bs))
        return tuple(a[sl] for a in self.w)

    def exact_next(self, s):
        """The gradient of step s is exact in fp32 (raises otherwise)."""
        u, i, j = self.batch(s)
        return grad64(self.host["U"], self.host["V"], u, i, j, self.loss, self.reg)

    def run(self, first, num):
        d = self.d
        self.ops.mf_epoch_fused(d["U"], d["V"], *self.args, 1, True, self.shuffle, self.drop_last, self.seed,
                                self.epoch, self.bs, first, num, self.loss, self.reg, self.opt, HYPER[self.opt],
                                self.pows, self.gU, self.gV, self.tU, self.tV, d["s0U"], d["s1U"], d["s0V"], d["s1V"],
                                self.stamp, self.ws[0], self.ws[1], self.ws[2], self.step_loss)
        self.stamp += num
        for s in range(first, first + num):     # the numpy restatement, op for op (tf_math.opt_apply)
            u, i, j = self.batch(s)
            h = self.host
            _, gU, gV, tU, tV = tf_math.mf_pairwise_grad(h["U"], h["V"], u, i, j, self.loss, self.reg)
            hyper = list(HYPER[self.opt])
            if self.opt == "adam":
                hyper[0] = tf_math.adam_lr_t(hyper[0], 1, start_step=self.t)[0]
            tf_math.opt_apply(self.opt, h["U"], gU, h["s0U"], h["s1U"], tU, hyper)
            tf_math.opt_apply(self.opt, h["V"], gV, h["s0V"], h["s1V"], tV, hyper)
            self.t += 1

    def assert_equal(self):
        for k in ("U", "V", "s0U", "s1U", "s0V", "s1V"):
            if k[:2] == "s1" and self.opt not in ("adam", "rmsprop") or k[:2] == "s0" and self.opt == "gd":
                continue
            assert np.array_equal(self.d[k].cpu().numpy(), self.host[k]), k
        assert not self.gU.any() and not self.gV.any()       # the accumulators are zeroed for the next step


EPOCH_DIMS = [(128, 4), (64, 2), (32, 1), (20, 0), (256, 0), (1, 0), (3, 0), (33, 0), (130, 0)]


@gpu
@pytest.mark.parametrize("dim,vec", EPOCH_DIMS)
@pytest.mark.parametrize("opt", OPTS)
def test_epoch_fused_exact(dim, vec, opt):
    """One step on each side of 16 * SMs samples per batch (the hinge loss, then square with reg), tables and slots
    bit for bit against tf_math's optimizer; GD and momentum keep stepping, with steps [1, k) in a second launch
    (first_step > 0), while the float64 chain stays exact.  The float4 optimizer pass for dim % 4 == 0, the per-element
    pass (which reads `touched` per element) otherwise."""
    n_sms = sms()
    rs = np.random.RandomState(dim + len(opt))
    nu, ni = 300, 2000            # about a third of the item rows are untouched by a step
    tp, ti, pu = epoch_csr(rs, nu, ni, 15)
    for bs, loss, reg, drop_last in ((epoch_batches(n_sms)[0], "hinge", 0.0, False),
                                     (epoch_batches(n_sms)[1], "square", 2.0 ** -3, True)):
        U = dyadic(rs, (nu, dim), -1, 1, 2)
        V = dyadic(rs, (ni, dim), -1, 1, 2)
        U[:, 4:] = 0              # |x| <= 1/2 at the first step: no hinge case on the tie x = -1
        R = EpochRun(U, V, opt, tp, ti, pu, ni, True, drop_last, bs, loss, reg)
        assert R.steps >= 2
        R.exact_next(0)
        R.run(0, 1)
        r = routes()["epoch"]
        assert r["vec"] == vec and r["opt_vec4"] == int(dim % 4 == 0) and r["grid"] == n_sms
        assert r["capped"] == int(epoch_capped(bs, n_sms))
        R.assert_equal()
        SEEN.add(("epoch_vec", vec)); SEEN.add(("epoch_opt_vec4", r["opt_vec4"])); SEEN.add(("epoch_opt", opt))
        SEEN.add(("epoch_capped", r["capped"]))
        if opt in ("gd", "momentum"):      # later steps, one launch each (first_step > 0), while still exact
            for s in range(1, R.steps):
                try:
                    R.exact_next(s)
                except AssertionError:
                    break
                R.run(s, 1)
                R.assert_equal()
                SEEN.add(("epoch_first_step", "> 0"))
        if drop_last:
            assert R.n_used % bs == 0 and R.n_used < len(R.w[0])
            SEEN.add(("epoch_drop_last", 1))


@gpu
def test_epoch_fused_pointwise_short_last_batch():
    """Pointwise cross-entropy: the last batch of the epoch is short and its gradients are scaled by 1 / cnt, not
    1 / batch_size.  One step at the last batch (first_step > 0) within the float64 chain's bound."""
    from neurec_b200 import ops
    rs = np.random.RandomState(17)
    nu, ni, dim, bs = 60, 200, 64, 350
    tp, ti, pu = epoch_csr(rs, nu, ni, 20)
    U = (rs.randn(nu, dim) * 0.3).astype(np.float32)
    V = (rs.randn(ni, dim) * 0.3).astype(np.float32)
    wu, wi, wl = oracle.epoch_build(tp, ti, pu, ti, 1, ni, False, True, 3, 0)
    n = len(wu)
    steps = -(-n // bs)
    last = steps - 1
    cnt = n - last * bs
    assert 0 < cnt < bs
    dU, dV = dev(U), dev(V)
    z = lambda t: torch.zeros_like(t)
    ws = [torch.empty(n, dtype=torch.int32, device="cuda") for _ in range(3)]
    sl = torch.zeros(steps, device="cuda")
    tU = torch.zeros(nu, dtype=torch.int32, device="cuda"); tV = torch.zeros(ni, dtype=torch.int32, device="cuda")
    gU, gV = z(dU), z(dV)
    # steps [0, last) with lr 0 build the workspace and leave the tables; then the short step alone
    ops.mf_epoch_fused(dU, dV, dev(tp), dev(ti), dev(pu), dev(ti), 1, False, True, False, 3, 0, bs, 0, last,
                       "cross_entropy", 0.0, "gd", [0.0], None, gU, gV, tU, tV, None, None, None, None, 1, *ws, sl)
    assert np.array_equal(dU.cpu().numpy(), U)
    lr = 0.5
    ops.mf_epoch_fused(dU, dV, dev(tp), dev(ti), dev(pu), dev(ti), 1, False, True, False, 3, 0, bs, last, 1,
                       "cross_entropy", 0.0, "gd", [lr], None, gU, gV, tU, tV, None, None, None, None, 100, *ws, sl)
    u, i, zl = wu[last * bs:], wi[last * bs:], wl[last * bs:].astype(np.float64)
    U64, V64 = U.astype(np.float64), V.astype(np.float64)
    x = (U64[u] * V64[i]).sum(1)
    e = np.exp(-np.abs(x))
    s = np.where(x >= 0, 1 / (1 + e), e / (1 + e))
    g = (s - zl) / cnt
    Mg = (6 * np.abs(s) + np.abs(s - zl) + 0.25 * dim * (np.abs(U64[u]) * np.abs(V64[i])).sum(1)) / cnt + 2 * np.abs(g)
    wantU, wantV = U64.copy(), V64.copy()
    MU, MV = np.abs(U64).copy(), np.abs(V64).copy()
    cu = np.bincount(u, minlength=nu)[:, None]; ci = np.bincount(i, minlength=ni)[:, None]
    np.add.at(wantU, u, -lr * g[:, None] * V64[i]); np.add.at(MU, u, lr * (Mg[:, None] + 3 * np.abs(g)[:, None] * cu[u]) * np.abs(V64[i]))
    np.add.at(wantV, i, -lr * g[:, None] * U64[u]); np.add.at(MV, i, lr * (Mg[:, None] + 3 * np.abs(g)[:, None] * ci[i]) * np.abs(U64[u]))
    assert_within(dU.cpu().numpy(), wantU, MU, "users")
    assert_within(dV.cpu().numpy(), wantV, MV, "items")
    # 1 / batch_size instead of 1 / cnt would be far outside the bound
    assert (np.abs(wantU - U64) * (bs / cnt - 1) > C_BOUND * U24 * MU).any()
    SEEN.add(("epoch_short_last_batch", 1))


# ---------------------------------------------------------------------------------------------------------------
# in-place SGD: shard sets on one device, the exact construction and the expected tables
# ---------------------------------------------------------------------------------------------------------------
def shard_set(full, world, rank, per_shard):
    """`world` separate allocations of `per_shard` rows on this device; rows past the table stay zero."""
    from neurec_b200.util import peer
    dim = full.shape[1]
    blocks = []
    for r in range(world):
        b = np.zeros((per_shard, dim), np.float32)
        part = full[r * per_shard:(r + 1) * per_shard]
        b[:len(part)] = part
        blocks.append(dev(b))
    S = peer.ShardSet(blocks[rank], [b.data_ptr() for b in blocks], rank, "local", None)
    S.blocks = blocks
    return S


def gather_shards(S, n):
    return torch.cat(S.blocks).cpu().numpy()[:n]


def set_hot(S, full, n_hot):
    """The replicated head by hand (ShardSet.enable_hot all-reduces over a process group)."""
    if n_hot:
        S.n_hot = n_hot
        S.hot = dev(full[:n_hot])
        S.hot_delta = torch.zeros_like(S.hot)


def apply_hot(S, per_shard):
    """sync_hot + writeback_hot of every shard, on one device."""
    from neurec_b200 import _lib
    from neurec_b200.ops import _p, _stream
    if not S.n_hot:
        return
    _lib.check(_lib.load().nrc_mf_hot_apply(_p(S.hot), _p(S.hot_delta), S.hot.numel(), _stream()))
    assert not S.hot_delta.any()
    for r, b in enumerate(S.blocks):
        lo, hi = r * per_shard, min(S.n_hot, (r + 1) * per_shard)
        if hi > lo:
            b[:hi - lo] = S.hot[lo:hi]


def x_zero_tables(rs, nu, ni, dim):
    """Users on the first half of the dimensions, every item equal there: every score difference is 0."""
    h = dim // 2
    U = np.zeros((nu, dim), np.float32)
    U[:, :h] = dyadic(rs, (nu, h), -8, 8, 4)
    V = dyadic(rs, (ni, dim), -8, 8, 4)
    V[:, :h] = V[0, :h]
    return U, V


def sgd_expected(U, V, wu, wi, wj, lr, reg):
    """float64 in-place step with g = -1/2 and every read at the pre-launch value, asserted exact in fp32."""
    U64, V64 = U.astype(np.float64), V.astype(np.float64)
    pu, qi, qj = U64[wu], V64[wi], V64[wj]
    assert ((pu * (qi - qj)).sum(1) == 0).all()
    g = -0.5
    du = -lr * (g * (qi - qj) + reg * pu)
    dvi = -lr * (g * pu + reg * qi)
    dvj = -lr * (-g * pu + reg * qj)
    wU, wV = U64.copy(), V64.copy()
    mU, mV = np.abs(U64), np.abs(V64)
    np.add.at(wU, wu, du); np.add.at(mU, wu, np.abs(du))
    np.add.at(wV, wi, dvi); np.add.at(mV, wi, np.abs(dvi))
    np.add.at(wV, wj, dvj); np.add.at(mV, wj, np.abs(dvj))
    for p in (du, dvi, dvj, g * (qi - qj), reg * pu, g * pu, reg * qi, reg * qj):
        assert_exact(p, 0)
    assert_exact(np.concatenate([wU.ravel(), wV.ravel()]), np.concatenate([mU.ravel(), mV.ravel()]), "tables")
    return wU, wV


def clean_rows(wu, wi, wj, n_hot, nu, ni):
    """Rows whose every touch is by a triplet that read pre-launch values only: triplets whose user or non-head item
    another triplet also touches are dirty, and so are the rows they touch."""
    cu = np.bincount(wu, minlength=nu)
    ci = np.bincount(np.concatenate([wi, wj]), minlength=ni)
    dirty = (cu[wu] > 1) | ((wi >= n_hot) & (ci[wi] > 1)) | ((wj >= n_hot) & (ci[wj] > 1))
    okU = np.ones(nu, bool); okV = np.ones(ni, bool)
    okU[wu[dirty]] = False; okV[wi[dirty]] = False; okV[wj[dirty]] = False
    return okU, okV, dirty


def csr_layout(rs, n_pos, first, count, ni, n_hot, world, per_shard):
    """Users of one positive, except user A (33 positives, the last at position `first`) and user B (32 positives,
    the first at position first + count - 1): with the shuffle off each is touched once by the window and A takes the
    RED, B the store.  Non-head positives are distinct, a third of the positives are Zipf draws from the head, and the
    positives next to `first` are the ids on both sides of every shard boundary and the last item."""
    degs = []
    p = 0
    while p < n_pos:
        if p == first - 32:
            degs.append(33)
        elif p == first + count - 1:
            degs.append(32)
        else:
            degs.append(1)
        p += degs[-1]
    nu = len(degs)
    n_pos = p
    special = sorted({ni - 1} | {b for r in range(1, world) for b in (r * per_shard - 1, r * per_shard)
                                 if n_hot <= b < ni})
    pool = rs.permutation(np.arange(n_hot, ni))
    pool = pool[~np.isin(pool, special)]
    items = np.empty(n_pos, np.int64)
    items[:] = pool[:n_pos]
    if n_hot:
        head = rs.random_sample(n_pos) < 1 / 3
        items[head] = np.minimum((n_hot * rs.random_sample(int(head.sum())) ** 3).astype(np.int64), n_hot - 1)
    items[first + 1:first + 1 + len(special)] = special
    rows, p = [], 0
    for d in degs:
        r = items[p:p + d]
        if d > 1:               # long rows: distinct non-head items
            r = pool[n_pos + p:n_pos + p + d]
        rows.append(np.sort(r))
        p += d
    tp, ti = oracle.lists_to_csr(rows)
    assert len(ti) == n_pos
    return tp, ti, np.repeat(np.arange(nu, dtype=np.int32), np.diff(tp)), nu


def sgd_csr_case(dim, world, self_rank, n_hot, shuffle, same_csr, count, seed=0):
    """One exact CSR-fed window [first, first + count) on `world` item shards of this device; returns the route."""
    from neurec_b200 import ops
    n_sms = sms()
    rs = np.random.RandomState(seed + dim + 10 * world + n_hot)
    ni = 100_003
    per_shard = -(-ni // world) + (5 if world > 1 else 0)        # the last shard only partly filled
    if world > 1:
        assert (world - 1) * per_shard < ni < world * per_shard
    first = 1000 if count else 50
    n_pos = max(6000, first + count + 100)
    tp, ti, pu, nu = csr_layout(rs, n_pos, first, max(count, 2), ni, n_hot, world, per_shard)
    U, V = x_zero_tables(rs, nu, ni, dim)
    lr, reg = 2.0 ** -4, 2.0 ** -3
    for seed in range(seed, seed + 20):      # shuffle off: a draw whose negatives leave A's and B's triplets clean
        wu, wi, wj = oracle.epoch_build(tp, ti, pu, ti, 1, ni, True, shuffle, seed, 4)
        wu, wi, wj = wu[first:first + count], wi[first:first + count], wj[first:first + count, 0]
        okU, okV, dirty = clean_rows(wu, wi, wj, n_hot, nu, ni)
        if shuffle or count == 0 or (okU[pu[first]] and okU[pu[first + count - 1]]):
            break
    assert count == 0 or dirty.mean() < 0.06
    wantU, wantV = sgd_expected(U, V, wu, wi, wj, lr, reg)
    S = shard_set(V, world, self_rank, per_shard)
    set_hot(S, V, n_hot)
    dU = dev(U)
    t_idx = dev(ti)
    loss = torch.zeros(1, device="cuda")
    before = routes()["sgd_csr"]
    ops.mf_bpr_sgd_epoch(dU, S, dev(tp), t_idx, dev(pu), t_idx if same_csr else t_idx.clone(), ni, shuffle, seed, 4,
                         first, count, lr, reg, loss)
    r = routes()["sgd_csr"]
    apply_hot(S, per_shard)
    gU, gV = dU.cpu().numpy(), gather_shards(S, ni)
    assert np.array_equal(gU[okU], wantU[okU]) and np.array_equal(gV[okV], wantV[okV])
    if count == 0:
        assert r == before and np.array_equal(gU, U) and np.array_equal(gV, V)
        return r
    if not shuffle:       # A (33 positives) and B (32) each touched once by the window and checked
        assert okU[pu[first]] and okU[pu[first + count - 1]]
        assert np.diff(tp)[pu[first]] == 33 and np.diff(tp)[pu[first + count - 1]] == 32
    assert r["vec"] == dim // 32 and r["sharded"] == int(world > 1) and r["user_once"] == int(same_csr)
    assert r["tier_rows"] == min(n_hot, tier_rows(dim))
    return r


T_CASES = ["0", "T-1", "T", "T+1", "4T"]


@gpu
@pytest.mark.parametrize("dim", [32, 64, 128])
@pytest.mark.parametrize("n_hot_of", T_CASES)
def test_sgd_csr_exact_tier_boundary(dim, n_hot_of):
    """Head rows on both sides of the shared-memory tier's T rows: tier, replica beyond it, per-CTA flush and
    nrc_mf_hot_apply bit for bit; shuffle on, a window of 769 (two CTAs) starting inside the epoch."""
    T = tier_rows(dim)
    n_hot = {"0": 0, "T-1": T - 1, "T": T, "T+1": T + 1, "4T": 4 * T}[n_hot_of]
    r = sgd_csr_case(dim, 1, 0, n_hot, True, True, 769)
    SEEN.add(("sgd_csr_tier", dim // 32, n_hot_of))


@gpu
@pytest.mark.parametrize("dim", [32, 64, 128])
@pytest.mark.parametrize("world,self_rank", [(2, 0), (2, 1), (3, 2), (8, 0), (8, 7)])
def test_sgd_csr_exact_sharded(dim, world, self_rank):
    """The SHARDED kernel on `world` separate allocations of one device ("remote" rows are ordinary device memory):
    item ids on both sides of every shard boundary, a last shard only partly filled, a head of T + 1 rows, the shuffle
    off with users of 33 and 32 positives at the window's ends, and pos_items a copy of the CSR at world 3."""
    T = tier_rows(dim)
    same = world != 3
    r = sgd_csr_case(dim, world, self_rank, T + 1 if world != 8 else 0, False, same, 768)
    assert r["sharded"] == 1
    SEEN.add(("sgd_csr_sharded", dim // 32))
    SEEN.add(("sgd_csr_user_once", r["user_once"]))


@gpu
@pytest.mark.parametrize("shuffle,same_csr", [(False, True), (False, False), (True, False)])
def test_sgd_csr_exact_store_rule(shuffle, same_csr):
    """Users of 33 and 32 positives each touched once by the window (the shuffle off): 33 takes the RED, 32 the store,
    both exact; with pos_items a copy of the CSR every user row takes the RED."""
    r = sgd_csr_case(64, 1, 0, 0, shuffle, same_csr, 768)
    SEEN.add(("sgd_csr_user_once", r["user_once"]))


@gpu
def test_sgd_csr_empty_window():
    """count 0 launches nothing and leaves the hook as it was."""
    sgd_csr_case(32, 2, 1, 0, True, True, 0)


@gpu
@pytest.mark.parametrize("dim", [32, 64, 128])
@pytest.mark.parametrize("world", [1, 2])
@pytest.mark.parametrize("which", ["below", "capped"])
def test_sgd_csr_exact_persistent_windows(dim, world, which):
    """Windows of about SMs * 768 positions and three times that (the persistent grid loops), reg 0 and every item row
    equal: every score difference is 0, user rows stay as they are (a zero delta) and every item is a head row (n_hot =
    num_items), read from the tier or the replica.  Item rows repeat thousands of times (Zipf positives) and their summed
    deltas must be exact: the tier's shared-memory atomics, the per-CTA flush and nrc_mf_hot_apply."""
    from neurec_b200 import ops
    n_sms = sms()
    rs = np.random.RandomState(dim + world)
    nu, ni, deg = 8000, 3000, 80
    rows = [np.unique(np.minimum((ni * rs.random_sample(deg) ** 2).astype(np.int64), ni - 1)) for _ in range(nu)]
    tp, ti = oracle.lists_to_csr(rows)
    pu = np.repeat(np.arange(nu, dtype=np.int32), np.diff(tp))
    count = 768 * n_sms - 5 if which == "below" else 3 * 768 * n_sms + 7
    first = 333
    assert first + count <= len(ti)
    U = dyadic(rs, (nu, dim), -8, 8, 4)
    V = np.repeat(dyadic(rs, (1, dim), -8, 8, 4), ni, 0)
    lr = 2.0 ** -4
    wu, wi, wj = oracle.epoch_build(tp, ti, pu, ti, 1, ni, True, True, 8, 1)
    wu, wi, wj = wu[first:first + count], wi[first:first + count], wj[first:first + count, 0]
    U64 = U.astype(np.float64)
    wantV = V.astype(np.float64)
    mV = np.abs(wantV)
    np.add.at(wantV, wi, lr * 0.5 * U64[wu]); np.add.at(mV, wi, np.abs(lr * 0.5 * U64[wu]))
    np.add.at(wantV, wj, -lr * 0.5 * U64[wu]); np.add.at(mV, wj, np.abs(lr * 0.5 * U64[wu]))
    assert_exact(wantV, mV, "items")
    assert np.bincount(wi, minlength=ni).max() > 500
    per_shard = -(-ni // world)
    S = shard_set(V, world, world - 1, per_shard)
    set_hot(S, V, ni)
    dU = dev(U)
    loss = torch.zeros(1, device="cuda")
    ops.mf_bpr_sgd_epoch(dU, S, dev(tp), dev(ti), dev(pu), dev(ti), ni, True, 8, 1, first, count, lr, 0.0, loss)
    r = routes()["sgd_csr"]
    apply_hot(S, per_shard)
    assert np.array_equal(dU.cpu().numpy(), U)
    assert np.array_equal(gather_shards(S, ni), wantV)
    assert_within(float(loss), count * np.log(2.0), count * (count + 4) * np.log(2.0), "loss")
    grid_cap = r["grid"] if r["capped"] else None
    assert r["tier_rows"] == tier_rows(dim) and r["sharded"] == int(world > 1)
    if which == "capped":
        assert r["capped"] == 1 and count > 768 * grid_cap
    else:
        assert r["capped"] == 0 and r["grid"] == -(-count // 768)
    SEEN.add(("sgd_csr_capped", r["capped"]))
    SEEN.add(("sgd_csr_tier", dim // 32, "num_items"))


def sgd_ids_case(dim, world, self_rank, B, seed=0):
    """The id-fed step on a batch whose users and items are all distinct: every read is pre-launch, so exact."""
    from neurec_b200 import ops
    rs = np.random.RandomState(seed + dim + world)
    nu, ni = B + 17, 2 * B + 29
    U, V = x_zero_tables(rs, nu, ni, dim)
    users = rs.permutation(nu)[:B].astype(np.int32)
    it = rs.permutation(ni)[:2 * B].astype(np.int32)
    pos, neg = it[:B], it[B:]
    lr, reg = 2.0 ** -4, 2.0 ** -3
    wantU, wantV = sgd_expected(U, V, users, pos, neg, lr, reg)
    loss = torch.zeros(1, device="cuda")
    if world == 0:
        dU, dV = dev(U), dev(V)
        ops.mf_bpr_sgd_fused(dU, dV, dev(users), dev(pos), dev(neg), lr, reg, loss)
        gU, gV = dU.cpu().numpy(), dV.cpu().numpy()
    else:
        pu_, pi_ = -(-nu // world) + 3, -(-ni // world) + 1
        SU, SV = shard_set(U, world, self_rank, pu_), shard_set(V, world, self_rank, pi_)
        ops.mf_bpr_sgd_sharded(SU, SV, self_rank, dev(users), dev(pos), dev(neg), lr, reg, loss)
        gU, gV = gather_shards(SU, nu), gather_shards(SV, ni)
    assert np.array_equal(gU, wantU) and np.array_equal(gV, wantV)
    reg_l = 0.5 * reg * float((U[users].astype(np.float64) ** 2).sum() + (V[pos].astype(np.float64) ** 2).sum()
                              + (V[neg].astype(np.float64) ** 2).sum())
    assert_within(float(loss), B * np.log(2.0) + reg_l, (B + dim + 4) * (B * np.log(2.0) + reg_l), "loss")
    return routes()["sgd_ids"]


@gpu
@pytest.mark.parametrize("dim", [32, 64, 128])
@pytest.mark.parametrize("world,self_rank", [(0, 0), (1, 0), (2, 1), (3, 0), (8, 7)])
def test_sgd_ids_exact(dim, world, self_rank):
    """nrc_mf_bpr_sgd_fused (world 0 here) and nrc_mf_bpr_sgd_sharded, user and item shards, at 64 * SMs and
    64 * SMs + 1 triplets (the grid loops)."""
    n_sms = sms()
    for B in grad_batches(n_sms)[1:3]:
        r = sgd_ids_case(dim, world, self_rank, B)
        assert r["vec"] == dim // 32 and r["sharded"] == int(world > 0) and r["capped"] == int(grad_capped(B, n_sms))
        SEEN.add(("sgd_ids", dim // 32, r["sharded"], r["capped"]))


_ENV_CASE = """
import sys
sys.path.insert(0, %r); sys.path.insert(0, %r)
import test_gpu_mf_routes as t
r = t.sgd_csr_case(64, 3, 1, 0, True, True, 769)
assert r["sharded"] == 1
r = t.sgd_ids_case(128, 2, 0, 700)
assert r["sharded"] == 1
print("ok")
"""


@gpu
@pytest.mark.parametrize("env", ["NRC_PEER_VEC_RED=0", "NRC_FORCE_REMOTE_PATH=1"])
def test_sgd_sharded_switches_in_a_fresh_process(env):
    """Scalar REDs for rows of other shards, and the remote path for local rows too: both switches are read once per
    process, so the sharded cases run in a fresh interpreter."""
    k, v = env.split("=")
    e = dict(os.environ, **{k: v})
    r = subprocess.run([sys.executable, "-c", _ENV_CASE % (ROOT, HERE)], env=e, capture_output=True, text=True,
                       timeout=600)
    assert r.returncode == 0 and r.stdout.strip().endswith("ok"), r.stdout[-3000:] + r.stderr[-3000:]
    SEEN.add(("sgd_env", k))


# ---------------------------------------------------------------------------------------------------------------
# repeated rows read in place: rounding plus interleaving
# ---------------------------------------------------------------------------------------------------------------
def hogwild_bound(U, V, wu, wi, wj, lr):
    """Expected tables (every delta taken at the pre-launch tables, reg 0) and the per-element bound: the rounding of
    each delta and of the sum into the row, plus twice what reading rows other triplets already moved can change."""
    U64, V64 = U.astype(np.float64), V.astype(np.float64)
    nu, ni = U.shape[0], V.shape[0]
    pu, qi, qj = U64[wu], V64[wi], V64[wj]
    diff = qi - qj
    x = (pu * diff).sum(1)
    g = -1.0 / (1.0 + np.exp(x))
    du, dvi, dvj = -lr * g[:, None] * diff, -lr * g[:, None] * pu, lr * g[:, None] * pu
    AU, AV = np.zeros_like(U64), np.zeros_like(V64)
    np.add.at(AU, wu, np.abs(du)); np.add.at(AV, wi, np.abs(dvi)); np.add.at(AV, wj, np.abs(dvj))
    au = AU[wu] - np.abs(du)                     # the other triplets' deltas on the rows this triplet reads
    ai = AV[wi] - np.abs(dvi); aj = AV[wj] - np.abs(dvj)
    aij = ai + aj
    dx = (au * np.abs(diff) + np.abs(pu) * aij + au * aij).sum(1)
    dg = 0.25 * dx
    Iu = lr * (dg[:, None] * (np.abs(diff) + aij) + np.abs(g)[:, None] * aij)
    Ii = lr * (dg[:, None] * (np.abs(pu) + au) + np.abs(g)[:, None] * au)
    D = U.shape[1]
    Mg = 4 * np.abs(g) + 0.25 * D * (np.abs(pu) * (np.abs(qi) + np.abs(qj))).sum(1)
    Ru = lr * (Mg[:, None] * np.abs(diff) + 4 * np.abs(g)[:, None] * np.abs(diff))
    Ri = lr * (Mg[:, None] * np.abs(pu) + 3 * np.abs(g)[:, None] * np.abs(pu))
    cU = np.bincount(wu, minlength=nu)[:, None]
    cV = np.bincount(np.concatenate([wi, wj]), minlength=ni)[:, None]
    wU, wV = U64.copy(), V64.copy()
    np.add.at(wU, wu, du); np.add.at(wV, wi, dvi); np.add.at(wV, wj, dvj)
    IU, IV, RU, RV = (np.zeros_like(a) for a in (U64, V64, U64, V64))
    np.add.at(IU, wu, Iu); np.add.at(IV, wi, Ii); np.add.at(IV, wj, Ii)
    np.add.at(RU, wu, Ru); np.add.at(RV, wi, Ri); np.add.at(RV, wj, Ri)
    BU = C_BOUND * (U24 * (RU + (cU + 1) * (np.abs(U64) + AU)) + 2 * IU)
    BV = C_BOUND * (U24 * (RV + (cV + 1) * (np.abs(V64) + AV)) + 2 * IV)
    return wU, wV, BU, BV, (du, dvi, dvj)


@gpu
@pytest.mark.parametrize("dim,shuffle,same_csr,n_hot", [(128, True, True, 0), (64, False, True, 0),
                                                        (32, True, False, 0), (64, True, True, 128)])
def test_sgd_csr_hogwild_bound(dim, shuffle, same_csr, n_hot):
    """Users of 2, 32 and 33 positives read and update their rows in place while other triplets of the launch do:
    every element within rounding plus interleaving of the first-order step, and the bound is tight enough that
    dropping any one triplet's delta, or lr off by 2^-8, leaves it."""
    from neurec_b200 import ops
    from neurec_b200.util import peer
    rs = np.random.RandomState(dim + shuffle)
    nu, ni = 4000, 60_000
    deg = np.full(nu, 2)
    deg[:40] = 32; deg[40:80] = 33
    rows = [rs.choice(ni, d, replace=False) for d in deg]
    tp, ti = oracle.lists_to_csr(rows)
    pu = np.repeat(np.arange(nu, dtype=np.int32), np.diff(tp))
    first, count = 37, len(ti) - 37 - 11
    U = (rs.randn(nu, dim) * 0.1).astype(np.float32)
    V = (rs.randn(ni, dim) * 0.1).astype(np.float32)
    lr = float(np.float32(5e-4))
    wu, wi, wj = oracle.epoch_build(tp, ti, pu, ti, 1, ni, True, shuffle, 9, 2)
    wu, wi, wj = wu[first:first + count], wi[first:first + count], wj[first:first + count, 0]
    wU, wV, BU, BV, (du, dvi, dvj) = hogwild_bound(U, V, wu, wi, wj, lr)
    dU, dV = dev(U), dev(V)
    S = peer.single(dV)
    set_hot(S, V, n_hot)
    t_idx = dev(ti)
    loss = torch.zeros(1, device="cuda")
    ops.mf_bpr_sgd_epoch(dU, S, dev(tp), t_idx, dev(pu), t_idx if same_csr else t_idx.clone(), ni, shuffle, 9, 2,
                         first, count, lr, 0.0, loss)
    r = routes()["sgd_csr"]
    assert r["user_once"] == int(same_csr)
    if n_hot:
        S.blocks = [dV]
        apply_hot(S, ni)
    gU, gV = dU.cpu().numpy(), dV.cpu().numpy()
    assert (np.abs(gU - wU) <= BU).all(), float((np.abs(gU - wU) - BU).max())
    assert (np.abs(gV - wV) <= BV).all(), float((np.abs(gV - wV) - BV).max())
    # sensitivity: every triplet's delta leaves the bound somewhere on its rows; so does lr * (1 + 2^-8)
    cu = np.bincount(wu, minlength=nu)
    multi = cu[wu] > 1
    assert multi.mean() > 0.5 and (cu[wu][np.isin(wu, np.arange(40, 80))] > 1).any()
    lost = (np.abs(du) > BU[wu]).any(1) | (np.abs(dvi) > BV[wi]).any(1) | (np.abs(dvj) > BV[wj]).any(1)
    assert lost.all(), int((~lost).sum())
    assert ((np.abs(wU - U) * 2.0 ** -8) > BU).any() and ((np.abs(wV - V) * 2.0 ** -8) > BV).any()
    SEEN.add(("sgd_csr_hogwild", dim // 32))


@gpu
def test_sgd_ids_hogwild_bound():
    """The id-fed step with repeated users and items, above 64 * SMs triplets: within the same bound, and as tight."""
    from neurec_b200 import ops
    n_sms = sms()
    rs = np.random.RandomState(5)
    B, nu, ni, dim = 64 * n_sms + 1, 3000, 40_000, 64
    U = (rs.randn(nu, dim) * 0.1).astype(np.float32)
    V = (rs.randn(ni, dim) * 0.1).astype(np.float32)
    users = rs.randint(0, nu, B).astype(np.int32)
    pos = rs.randint(0, ni, B).astype(np.int32)
    neg = rs.randint(0, ni, B).astype(np.int32)
    lr = float(np.float32(5e-4))
    wU, wV, BU, BV, (du, dvi, dvj) = hogwild_bound(U, V, users, pos, neg, lr)
    dU, dV = dev(U), dev(V)
    ops.mf_bpr_sgd_fused(dU, dV, dev(users), dev(pos), dev(neg), lr, 0.0, torch.zeros(1, device="cuda"))
    assert routes()["sgd_ids"]["capped"] == 1
    gU, gV = dU.cpu().numpy(), dV.cpu().numpy()
    assert (np.abs(gU - wU) <= BU).all() and (np.abs(gV - wV) <= BV).all()
    lost = (np.abs(du) > BU[users]).any(1) | (np.abs(dvi) > BV[pos]).any(1) | (np.abs(dvj) > BV[neg]).any(1)
    assert lost.all()
    assert ((np.abs(wU - U) * 2.0 ** -8) > BU).any()


# ---------------------------------------------------------------------------------------------------------------
# lazy Adam
# ---------------------------------------------------------------------------------------------------------------
def lazy_adam64(x, m, v, g, Mg, lr_t, b1, b2, eps):
    """One LazyAdam element update in float64 with its first-order rounding bound (in units of 2^-24)."""
    m1 = b1 * m + (1 - b1) * g
    v1 = b2 * v + (1 - b2) * g * g
    Mm = (1 - b1) * Mg + 3 * (np.abs(b1 * m) + np.abs((1 - b1) * g))
    Mv = (1 - b2) * 2 * np.abs(g) * Mg + 4 * (np.abs(b2 * v) + (1 - b2) * g * g)
    sq = np.sqrt(v1)
    den = sq + eps
    Mden = 0.5 * Mv / np.maximum(sq, 1e-30) + sq + den          # sqrtf's input error, its rounding, the add
    s = lr_t * m1 / den
    Ms = lr_t * Mm / den + np.abs(s) * Mden / den + 2 * np.abs(s)
    return x - s, m1, v1, Ms + np.abs(x) + np.abs(s), Mm, Mv


@gpu
@pytest.mark.parametrize("dim", [32, 64, 128])
@pytest.mark.parametrize("shuffle", [True, False])
def test_lazy_adam_rounded(dim, shuffle):
    """Rows touched once by the window (the others are left out, and few): var, m and v within the float64 chain's
    bound; untouched rows and slots bit-identical.  first > 0, and at dim 32 a count beyond 2048 * SMs (the grid
    loops)."""
    from neurec_b200 import ops
    n_sms = sms()
    rs = np.random.RandomState(dim + shuffle)
    count = lazy_counts(n_sms)[1] if dim == 32 else lazy_counts(n_sms)[0]
    first = 101
    n_pos = first + count + 50
    ni = 2_000_003 if dim == 32 else 400_000
    nu = n_pos
    items = rs.choice(ni, n_pos, replace=False).astype(np.int32)
    tp = np.arange(nu + 1, dtype=np.int64)
    ti = items.copy()
    pu = np.arange(nu, dtype=np.int32)
    U = (rs.randn(nu, dim) * 0.1).astype(np.float32)
    V = (rs.randn(ni, dim) * 0.1).astype(np.float32)
    mU = (rs.randn(nu, dim) * 1e-3).astype(np.float32); vU = (rs.rand(nu, dim) * 1e-5).astype(np.float32)
    mV = (rs.randn(ni, dim) * 1e-3).astype(np.float32); vV = (rs.rand(ni, dim) * 1e-5).astype(np.float32)
    lr_t, b1, b2, eps, reg = (float(np.float32(a)) for a in (1e-3, 0.9, 0.999, 1e-8, 1e-3))
    wu, wi, wj = oracle.epoch_build(tp, ti, pu, ti, 1, ni, True, shuffle, 6, 3)
    wu, wi, wj = wu[first:first + count], wi[first:first + count], wj[first:first + count, 0]
    ci = np.bincount(np.concatenate([wi, wj]), minlength=ni)
    clean = (ci[wi] == 1) & (ci[wj] == 1)
    assert clean.mean() > 0.4
    d = {k: dev(a) for k, a in dict(U=U, mU=mU, vU=vU, V=V, mV=mV, vV=vV).items()}
    loss = torch.zeros(1, device="cuda")
    ops.mf_bpr_lazy_adam_epoch(d["U"], d["mU"], d["vU"], d["V"], d["mV"], d["vV"], dev(tp), dev(ti), dev(pu), dev(ti),
                               ni, shuffle, 6, 3, first, count, lr_t, reg, loss, b1, b2, eps)
    r = routes()["lazy_adam"]
    assert r["vec"] == dim // 32 and r["capped"] == int(lazy_capped(count, n_sms))
    SEEN.add(("lazy_adam", dim // 32, r["capped"]))
    g = {k: t.cpu().numpy() for k, t in d.items()}
    # untouched rows: bit-identical
    tu = np.zeros(nu, bool); tu[wu] = True
    tv = np.zeros(ni, bool); tv[wi] = True; tv[wj] = True
    for k, a, t in (("U", U, tu), ("mU", mU, tu), ("vU", vU, tu), ("V", V, tv), ("mV", mV, tv), ("vV", vV, tv)):
        assert np.array_equal(g[k][~t], a[~t]), k
    u, i, j = wu[clean], wi[clean], wj[clean]
    f = lambda a: a.astype(np.float64)
    pu_, qi, qj = f(U[u]), f(V[i]), f(V[j])
    x = (pu_ * qi).sum(1) - (pu_ * qj).sum(1)
    Mx = dim * (np.abs(pu_) * (np.abs(qi) + np.abs(qj))).sum(1)
    gs = -1.0 / (1.0 + np.exp(x))
    Mgs = 4 * np.abs(gs) + 0.25 * Mx
    for key, rows, grad, Mgrad, var in (
            ("U", u, gs[:, None] * (qi - qj) + reg * pu_, Mgs[:, None] * np.abs(qi - qj) + 3 * (np.abs(gs[:, None] * (qi - qj)) + reg * np.abs(pu_)), pu_),
            ("V", i, gs[:, None] * pu_ + reg * qi, Mgs[:, None] * np.abs(pu_) + 2 * (np.abs(gs[:, None] * pu_) + reg * np.abs(qi)), qi),
            ("V", j, -gs[:, None] * pu_ + reg * qj, Mgs[:, None] * np.abs(pu_) + 2 * (np.abs(gs[:, None] * pu_) + reg * np.abs(qj)), qj)):
        m0 = f((mU if key == "U" else mV)[rows]); v0 = f((vU if key == "U" else vV)[rows])
        wx, wm, wv, Mx_, Mm, Mv = lazy_adam64(var, m0, v0, grad, Mgrad, lr_t, b1, b2, eps)
        assert_within(g[key][rows], wx, Mx_, key)
        assert_within(g["m" + key][rows], wm, Mm, "m" + key)
        assert_within(g["v" + key][rows], wv, Mv, "v" + key)


# ---------------------------------------------------------------------------------------------------------------
# nrc_mf_train_step_host and nrc_mf_train_epoch
# ---------------------------------------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("opt", OPTS)
def test_train_step_host_matches_train_epoch(opt):
    """The host-fed step (H2D copies, both phases, loss copied back) gives the bits of one nrc_mf_train_epoch step,
    and those are tf_math's step bit for bit on an exact batch (hinge, dyadic tables)."""
    from neurec_b200 import _lib, ops
    from neurec_b200.ops import _p, _stream
    rs = np.random.RandomState(len(opt))
    nu, ni, dim, B = 300, 400, 48, 2000
    U = dyadic(rs, (nu, dim), -1, 1, 2)
    V = dyadic(rs, (ni, dim), -1, 1, 2)
    users = rs.randint(0, nu, B).astype(np.int32)
    pos = rs.randint(0, ni, B).astype(np.int32)
    neg = no_hinge_tie(rs, U, V, users, pos, rs.randint(0, ni, B).astype(np.int32), ni)
    grad64(U, V, users, pos, neg, "hinge", 2.0 ** -3)
    hyper = list(HYPER[opt])
    i0, i1 = tf_math.SLOT_INIT[opt]
    mk = lambda a, v: np.full_like(a, 0.0 if v is None else v)
    # the oracle
    hU, hV = U.copy(), V.copy()
    s = [mk(U, i0), mk(U, i1), mk(V, i0), mk(V, i1)]
    want_l, gU, gV, tU, tV = tf_math.mf_pairwise_grad(hU, hV, users, pos, neg, "hinge", 2.0 ** -3)
    tf_math.opt_apply(opt, hU, gU, s[0], s[1], tU, hyper)
    tf_math.opt_apply(opt, hV, gV, s[2], s[3], tV, hyper)
    out = []
    for path in ("host", "epoch"):
        dU, dV = dev(U), dev(V)
        sl = [dev(a) for a in (mk(U, i0), mk(U, i1), mk(V, i0), mk(V, i1))]
        gd = [torch.zeros_like(dU), torch.zeros_like(dV)]
        t = [torch.zeros(nu, dtype=torch.int32, device="cuda"), torch.zeros(ni, dtype=torch.int32, device="cuda")]
        h = np.zeros(4, np.float32); h[:len(hyper)] = hyper
        if path == "host":
            staging = torch.empty(12 * B + 16, dtype=torch.uint8, device="cuda")
            lh = np.zeros(1, np.float32)
            _lib.check(_lib.load().nrc_mf_train_step_host(
                _p(dU), _p(dV), nu, ni, dim, users.ctypes.data, pos.ctypes.data, neg.ctypes.data, B, 1,
                _lib.LOSS_IDS["hinge"], 2.0 ** -3, _lib.OPT_IDS[opt], h.ctypes.data, _p(gd[0]), _p(gd[1]), _p(t[0]),
                _p(t[1]), _p(sl[0]), _p(sl[1]), _p(sl[2]), _p(sl[3]), 7, _p(staging), lh.ctypes.data, _stream()))
            l = float(lh[0])
        else:
            st = torch.zeros(1, device="cuda")
            ops.mf_train_epoch(dU, dV, dev(users), dev(pos), dev(neg), B, True, "hinge", 2.0 ** -3, opt, [hyper[0]],
                               hyper, gd[0], gd[1], t[0], t[1], sl[0], sl[1], sl[2], sl[3], 7, st)
            l = float(st)
        r = routes()
        assert r["grad"]["capped"] == 0 and r["opt_apply"]["grid"] >= 1
        out.append((dU.cpu().numpy(), dV.cpu().numpy(), [a.cpu().numpy() for a in sl], l))
        assert np.array_equal(out[-1][0], hU) and np.array_equal(out[-1][1], hV), path
        assert not gd[0].any() and not gd[1].any()
    assert out[0][3] == out[1][3] == float(want_l)       # dyadic per-sample losses: the sum is exact too
    for a, b in zip(out[0][2], out[1][2]):
        assert np.array_equal(a, b)
    SEEN.add(("train_step_host", opt))


@gpu
def test_opt_apply_grid_loops():
    """The multi-tensor optimizer apply beyond 2048 * SMs elements (the grid loops): momentum on touched rows only,
    bit for bit against tf_math."""
    from neurec_b200 import ops
    n_sms = sms()
    rs = np.random.RandomState(2)
    rows, dim = 2048 * n_sms // 16 + 3, 16
    var = (rs.randn(rows, dim)).astype(np.float32)
    grad = (rs.randn(rows, dim)).astype(np.float32)
    s0 = (rs.randn(rows, dim)).astype(np.float32)
    touched = rs.randint(0, 2, rows).astype(np.int32) * 4
    want_var, want_s0 = var.copy(), s0.copy()
    tf_math.opt_apply("momentum", want_var, grad, want_s0, None, touched == 4, [0.01, 0.9])
    d = [dev(a) for a in (var, grad, s0)]
    ops.opt_apply_rows("momentum", d[0], d[1], d[2], None, dev(touched), 4, [0.01, 0.9])
    r = routes()["opt_apply"]
    assert r["capped"] == 1 and r["grid"] == 8 * n_sms
    assert np.array_equal(d[0].cpu().numpy(), want_var) and np.array_equal(d[2].cpu().numpy(), want_s0)
    assert not d[1].any()
    SEEN.add(("opt_apply_capped", 1))


# ---------------------------------------------------------------------------------------------------------------
# limits and errors: the library's error, nothing written, the hook unchanged
# ---------------------------------------------------------------------------------------------------------------
@gpu
def test_limits_and_errors_write_nothing():
    from neurec_b200 import _lib, ops
    from neurec_b200.ops import _p, _stream
    lib = _lib.load()
    rs = np.random.RandomState(1)
    nu, ni = 50, 80
    tp, ti, pu = epoch_csr(rs, nu, ni, 5)
    n_pos = len(ti)

    def tables(dim):
        return dev((rs.randn(nu, dim)).astype(np.float32)), dev((rs.randn(ni, dim)).astype(np.float32))

    def unchanged(tensors, fn, code):
        snap = [t.clone() for t in tensors]
        before = routes()
        rc = fn()
        torch.cuda.synchronize()
        assert rc == code, (rc, lib.nrc_last_error())
        assert routes() == before
        for a, b in zip(tensors, snap):
            assert torch.equal(a, b)

    U, V = tables(48)
    ids = dev(np.zeros(4, np.int32))
    loss = torch.zeros(1, device="cuda")
    E = _lib.NRC_E_LIMIT
    dtp, dti, dpu = dev(tp), dev(ti), dev(pu)
    PA = lambda ts: (ctypes.c_void_p * len(ts))(*[t.data_ptr() if t is not None else None for t in ts])
    # dim 48 on every fixed-VEC entry point
    unchanged([U, V], lambda: lib.nrc_mf_bpr_sgd_fused(_p(U), _p(V), 48, _p(ids), _p(ids), _p(ids), 4, 0.1, 0.0,
                                                       _p(loss), _stream()), E)
    unchanged([U, V], lambda: lib.nrc_mf_bpr_sgd_sharded(PA([U]), PA([V]), 1, 0, nu, ni, 48, _p(ids), _p(ids),
                                                         _p(ids), 4, 0.1, 0.0, _p(loss), _stream()), E)
    epoch_args = lambda u, shards, world, rank, ips, dim, first, count, hot, hd, n_hot, nitems=ni: (
        _p(u), shards, world, rank, ips, dim, _p(dtp), _p(dti), _p(dpu), _p(dti), n_pos, nitems, 1, 3, 0, first, count,
        0.1, 0.0, _p(loss), _p(hot), _p(hd), n_hot, _stream())
    unchanged([U, V], lambda: lib.nrc_mf_bpr_sgd_epoch_hot(*epoch_args(U, PA([V]), 1, 0, ni, 48, 0, 10, None, None, 0)),
              E)
    unchanged([U, V], lambda: lib.nrc_mf_bpr_lazy_adam_epoch(_p(U), _p(U), _p(U), _p(V), _p(V), _p(V), 48, _p(dtp),
                                                             _p(dti), _p(dpu), _p(dti), n_pos, ni, 1, 3, 0, 0, 10,
                                                             1e-3, 0.9, 0.999, 1e-8, 0.0, _p(loss), _stream()), E)
    U, V = tables(32)
    halves = [V[:40].clone(), V[40:].clone()]
    # world 0 and 9, a NULL shard, shards that do not cover num_items
    for w in (0, 9):
        unchanged([U] + halves, lambda: lib.nrc_mf_bpr_sgd_epoch_hot(
            *epoch_args(U, PA(halves + halves[:1] * 7), w, 0, 40, 32, 0, 10, None, None, 0)), E)
        unchanged([U, V] + halves, lambda: lib.nrc_mf_bpr_sgd_sharded(
            PA([U] * 9), PA(halves * 5), w, 0, nu, 40, 32, _p(ids), _p(ids), _p(ids), 4, 0.1, 0.0, _p(loss),
            _stream()), E)
    unchanged([U] + halves, lambda: lib.nrc_mf_bpr_sgd_epoch_hot(
        *epoch_args(U, PA([halves[0], None]), 2, 0, 40, 32, 0, 10, None, None, 0)), _lib.NRC_E_VALUE)
    unchanged([U, V] + halves, lambda: lib.nrc_mf_bpr_sgd_sharded(
        PA([U, None]), PA(halves), 2, 0, nu, 40, 32, _p(ids), _p(ids), _p(ids), 4, 0.1, 0.0, _p(loss), _stream()),
        _lib.NRC_E_VALUE)
    unchanged([U] + halves, lambda: lib.nrc_mf_bpr_sgd_epoch_hot(
        *epoch_args(U, PA(halves), 2, 0, 39, 32, 0, 10, None, None, 0)), _lib.NRC_E_VALUE)
    # n_hot beyond the table, n_hot without its buffers
    hot, hd = V.clone(), torch.zeros_like(V)
    unchanged([U, V, hot, hd], lambda: lib.nrc_mf_bpr_sgd_epoch_hot(
        *epoch_args(U, PA([V]), 1, 0, ni, 32, 0, 10, hot, hd, ni + 1)), _lib.NRC_E_VALUE)
    unchanged([U, V, hot, hd], lambda: lib.nrc_mf_bpr_sgd_epoch_hot(
        *epoch_args(U, PA([V]), 1, 0, ni, 32, 0, 10, None, hd, 4)), _lib.NRC_E_VALUE)
    unchanged([U, V, hot, hd], lambda: lib.nrc_mf_bpr_sgd_epoch_hot(
        *epoch_args(U, PA([V]), 1, 0, ni, 32, 0, 10, hot, None, 4)), _lib.NRC_E_VALUE)
    # hot_apply with n_floats not a multiple of 4
    hd.fill_(1.0)
    unchanged([hot, hd], lambda: lib.nrc_mf_hot_apply(_p(hot), _p(hd), 6, _stream()), _lib.NRC_E_VALUE)
    unchanged([hot, hd], lambda: lib.nrc_mf_hot_apply(_p(hot), _p(hd), -4, _stream()), _lib.NRC_E_VALUE)
    # windows past the epoch
    for first, count in ((n_pos - 3, 4), (-1, 2), (0, n_pos + 1)):
        unchanged([U, V], lambda: lib.nrc_mf_bpr_sgd_epoch_hot(
            *epoch_args(U, PA([V]), 1, 0, ni, 32, first, count, None, None, 0)), _lib.NRC_E_VALUE)
        unchanged([U, V], lambda: lib.nrc_mf_bpr_lazy_adam_epoch(
            _p(U), _p(U), _p(U), _p(V), _p(V), _p(V), 32, _p(dtp), _p(dti), _p(dpu), _p(dti), n_pos, ni, 1, 3, 0,
            first, count, 1e-3, 0.9, 0.999, 1e-8, 0.0, _p(loss), _stream()), _lib.NRC_E_VALUE)
    # epoch steps past the epoch
    z = torch.zeros_like
    ws = torch.empty(n_pos, dtype=torch.int32, device="cuda")
    tU, tV = torch.zeros(nu, dtype=torch.int32, device="cuda"), torch.zeros(ni, dtype=torch.int32, device="cuda")
    steps = -(-n_pos // 64)
    with pytest.raises(ValueError):
        ops.mf_epoch_fused(U, V, dtp, dti, dpu, dti, 1, True, True, False, 3, 0, 64, steps - 1, 2, "bpr", 0.0, "gd",
                           [0.1], None, z(U), z(V), tU, tV, None, None, None, None, 1, ws, ws, ws,
                           torch.zeros(steps, device="cuda"))
    SEEN.add(("limits", 1))


REQUIRED = ({("grad", "single"), ("grad", "capped")}
            | {("grad_loss", l) for l in ("hinge", "square", "bpr", "pw_square")}
            | {("grad_rounded", l) for l in ("bpr", "cross_entropy")}
            | {("epoch_vec", v) for v in (4, 2, 1, 0)} | {("epoch_opt_vec4", v) for v in (0, 1)}
            | {("epoch_opt", o) for o in OPTS} | {("epoch_capped", c) for c in (0, 1)}
            | {("epoch_first_step", "> 0"), ("epoch_drop_last", 1), ("epoch_short_last_batch", 1)}
            | {("sgd_csr_tier", v, t) for v in (1, 2, 4) for t in T_CASES + ["num_items"]}
            | {("sgd_csr_sharded", v) for v in (1, 2, 4)} | {("sgd_csr_user_once", u) for u in (0, 1)}
            | {("sgd_csr_capped", c) for c in (0, 1)} | {("sgd_csr_hogwild", v) for v in (1, 2, 4)}
            | {("sgd_ids", v, s, c) for v in (1, 2, 4) for s in (0, 1) for c in (0, 1)}
            | {("sgd_env", k) for k in ("NRC_PEER_VEC_RED", "NRC_FORCE_REMOTE_PATH")}
            | {("lazy_adam", 2, 0), ("lazy_adam", 4, 0), ("lazy_adam", 1, 1)}
            | {("train_step_host", o) for o in OPTS} | {("opt_apply_capped", 1), ("limits", 1)})


@gpu
def test_every_route_was_seen(request):
    """Across this file the hook reported every route of the MF training kernels, the SHARDED forms of both in-place
    kernels and the per-element optimizer pass among them.  Only meaningful when the whole file ran: a run of
    selected tests skips it."""
    here = {it.nodeid for it in request.session.items if it.fspath == request.node.fspath}
    if len(here) < 100:
        pytest.skip("only part of the file ran")
    assert REQUIRED <= SEEN, sorted(REQUIRED - SEEN)
