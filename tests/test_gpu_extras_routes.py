"""Every route the data-side kernels (csrc/extras.cu), the negative samplers (csrc/sampler.cu) and LightGCN's BPR
gradient (csrc/lightgcn.cu) take from a shape, against float64 or a bit-exact restatement.

The routes depend on the SM count: the warp-per-row kernels (APR's normaliser, SBPR's gradient, the CSR sort and
compaction, the split ranks, the row ids, LightGCN's gradient) cap their grid at 8 CTAs of 8 warps per SM and loop
beyond 64 * SMs rows; the thread-per-element kernels of extras.cu (the row gather, SBPR's epoch builder, the COO count
and scatter passes) cap at 8 CTAs of 256 threads per SM and loop beyond 2048 * SMs elements; the samplers cap at 16
CTAs of 256 threads per SM and loop beyond 4096 * SMs elements; the row-pointer scan is one CTA that carries its sums
across 1024-row chunks.  Every shape below is derived from the device's SM count, one case on each side of each
boundary; each test asserts the route it ran through nrc_extras_last_routes, and the last test of the file checks that
the whole file saw every route.

The reference is written here in float64 (`R`), independently of oracle/tf_math.py's fp32 restatements; a CPU test
checks it against torch.autograd.  Each value carries M, a first-order bound on the rounding error of the fp32 chain
that computes it.  Exact cases use tables of small integers times 2^-k, power-of-two reg, scale and s_uk, hinge or
square loss (BPR only at x = 0, by cloning the negative's rows from the positive's); with `R.exact` set every operation
of the reference asserts that fp32 computes it exactly in any order, so the kernel must equal float64 bit for bit.
Rounded cases: each entry within 2 * 2^-24 * M of float64.  The data kernels and samplers are integer or counter-based
and are compared bit for bit with oracle/ (its C restatement of the Philox draws) and numpy."""
import ctypes
import os

import numpy as np
import pytest
import scipy.sparse as sp
import torch

import oracle
from oracle import tf_math

gpu = pytest.mark.gpu
U24 = 2.0 ** -24
C_BOUND = 2.0
SEEN = set()
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")
OPTS = ("gd", "adam", "adagrad", "rmsprop", "momentum")
HYPER = {"gd": [2.0 ** -4], "adam": [2.0 ** -4, 0.9, 0.999, 1e-8], "adagrad": [2.0 ** -4],
         "rmsprop": [2.0 ** -4, 0.9, 0.5, 1e-10], "momentum": [2.0 ** -4, 0.5]}
SBPR_DIMS = [1, 31, 32, 33, 64, 65, 256]
NORM_DIMS = [1, 2, 31, 32, 33, 64, 65, 255, 256]


def dev(a):
    return None if a is None else torch.from_numpy(np.ascontiguousarray(a)).cuda()


def host(t):
    return t.cpu().numpy()


def sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def routes():
    from neurec_b200 import ops
    return ops.extras_last_routes()


# ---------------------------------------------------------------------------------------------------------------
# the route predicates of the host code and the shapes on each side of them (pure functions of the SM count)
# ---------------------------------------------------------------------------------------------------------------
def warp_grid(rows, n_sms):
    """Warp-per-row kernels: ceil(rows / 8) CTAs of 8 warps, at most 8 per SM."""
    return min(max((rows + 7) // 8, 1), 8 * n_sms), (rows + 7) // 8 > 8 * n_sms


def elem_grid(n, n_sms):
    """Thread-per-element kernels of extras.cu: ceil(n / 256) CTAs, at most 8 per SM."""
    return min(max((n + 255) // 256, 1), 8 * n_sms), (n + 255) // 256 > 8 * n_sms


def sampler_grid(n, n_sms):
    """The samplers' thread-per-element kernels: ceil(n / 256) CTAs, at most 16 per SM."""
    return min((n + 255) // 256, 16 * n_sms), (n + 255) // 256 > 16 * n_sms


def warp_rows(n_sms):
    return [64 * n_sms, 64 * n_sms + 1]


def sbpr_batches(n_sms):
    """1, both sides of 64 * SMs, and a multiple that repeats rows hundreds of times."""
    return [1, 64 * n_sms, 64 * n_sms + 1, 2 * 64 * n_sms + 7]


def csr_shapes(n_sms):
    """(rows, entries): both sides of one and two scan chunks, of 64 * SMs rows and of 2048 * SMs entries."""
    return ([(r, 5000) for r in (1023, 1024, 1025, 2049)] + [(r, 20000) for r in (64 * n_sms - 1, 64 * n_sms + 1)]
            + [(1500, e) for e in (2048 * n_sms - 1, 2048 * n_sms + 1)])


def sampler_rows(n_sms, neg_num):
    """Users whose n * neg_num lands on both sides of 4096 * SMs."""
    c = 4096 * n_sms
    return [c // neg_num, c // neg_num + 1]


@pytest.mark.parametrize("n_sms", [114, 132])
def test_route_shapes_straddle_every_boundary(n_sms):
    """CPU: the shapes derived from the SM count land on both sides of every route predicate (114: H100 PCIe,
    132: H100 SXM)."""
    assert [warp_grid(b, n_sms)[1] for b in sbpr_batches(n_sms)] == [False, False, True, True]
    assert warp_grid(64 * n_sms, n_sms)[0] == 8 * n_sms
    assert [warp_grid(r, n_sms)[1] for r in warp_rows(n_sms)] == [False, True]
    shapes = csr_shapes(n_sms)
    assert {(r + 1023) // 1024 for r, _ in shapes} >= {1, 2, 3}
    assert {warp_grid(r, n_sms)[1] for r, _ in shapes} == {False, True}
    assert [elem_grid(e, n_sms)[1] for _, e in shapes[-2:]] == [False, True]
    assert elem_grid(2048 * n_sms, n_sms) == (8 * n_sms, False)
    for k in (1, 3):
        assert [sampler_grid(n * k, n_sms)[1] for n in sampler_rows(n_sms, k)] == [False, True]
    # Ciao's 221 734 positives tiled twice loop in the epoch builder on both SM counts
    assert elem_grid(2 * 221734, n_sms)[1] and not elem_grid(221734 // 2, n_sms)[1]
    # Gowalla's 810 128 interactions and 29 858 users cross every data-kernel boundary
    assert elem_grid(810128, n_sms)[1] and warp_grid(29858, n_sms)[1] and (29858 + 1023) // 1024 > 1


# ---------------------------------------------------------------------------------------------------------------
# exactness precondition, bounds and the float64 value class
# ---------------------------------------------------------------------------------------------------------------
def granule_bits(*arrays):
    """The smallest k with every value of every array a multiple of 2^-k."""
    bits = 0
    for a in arrays:
        v = np.abs(np.asarray(a, np.float64)).ravel()
        v = v[(v != 0) & np.isfinite(v)]
        if v.size == 0:
            continue
        m, e = np.frexp(v)
        mant = (m * 2.0 ** 53).astype(np.int64)
        low = np.frexp((mant & -mant).astype(np.float64))[1] - 1
        bits = max(bits, int((53 - e - low).max()))
    return bits


def is_exact(operands, magnitude):
    bits = granule_bits(*operands)
    return bits < 150 and bool((np.asarray(magnitude, np.float64) * 2.0 ** bits < 2.0 ** 24).all())


def assert_exact(operands, magnitude, what=""):
    """Every operand is a multiple of 2^-bits and every partial result (bounded by `magnitude`) stays below 2^24 such
    granules: fp32 represents each exactly, in any summation order."""
    assert is_exact(operands, magnitude), (what, granule_bits(*operands), float(np.max(magnitude)))


def assert_within(got, want, M, what, C=C_BOUND, floor=0.0):
    """|got - want| <= C * 2^-24 * M (+ floor, an absolute allowance where fp32 atomics flush subnormals)."""
    err = np.abs(np.asarray(got, np.float64) - want)
    bound = C * U24 * np.asarray(M, np.float64) + floor
    assert (err <= bound).all(), (what, float((err - bound).max()), float(np.max(M)))


class R:
    """A float64 value v of an fp32 chain with m, a first-order bound on that chain's rounding error in units of
    2^-24.  While R.exact is set, every operation also asserts that fp32 computes it exactly (assert_exact)."""
    exact = False

    def __init__(self, v, m=None):
        self.v = np.asarray(v, np.float64)
        self.m = np.zeros_like(self.v) if m is None else np.asarray(m, np.float64)

    @staticmethod
    def of(o):
        return o if isinstance(o, R) else R(o)

    def __getitem__(self, k):
        return R(self.v[k], np.broadcast_to(self.m, self.v.shape)[k])

    def __neg__(self):
        return R(-self.v, self.m)

    def __add__(self, o):
        o = R.of(o)
        v = self.v + o.v
        if R.exact:
            assert_exact([self.v, o.v], np.abs(self.v) + np.abs(o.v), "add")
        return R(v, self.m + o.m + np.abs(v))

    __radd__ = __add__

    def __sub__(self, o):
        return self + (-R.of(o))

    def __rsub__(self, o):
        return R.of(o) - self

    def __mul__(self, o):
        o = R.of(o)
        v = self.v * o.v
        if R.exact:
            assert_exact([v], np.abs(v), "mul")
        return R(v, np.abs(self.v) * o.m + np.abs(o.v) * self.m + np.abs(v))

    __rmul__ = __mul__

    def __truediv__(self, o):
        """Correctly rounded division by an exact (per-row) divisor."""
        k = np.asarray(o.v if isinstance(o, R) else o, np.float64)
        v = self.v / k
        if R.exact:
            assert_exact([v], np.abs(v), "div")
        return R(v, self.m / np.abs(k) + np.abs(v))

    def sum(self, axis):
        """A sum in any order (warp shuffles, atomics)."""
        n = self.v.shape[axis]
        mag = np.abs(self.v).sum(axis)
        if R.exact:
            assert_exact([self.v], mag, "sum")
        return R(self.v.sum(axis), self.m.sum(axis) + max(n - 1, 0) * mag)


def cat(parts, axis):
    return R(np.concatenate([p.v for p in parts], axis),
             np.concatenate([np.broadcast_to(p.m, p.v.shape) for p in parts], axis))


def where(mask, a, b=0.0):
    a, b = R.of(a), R.of(b)
    return R(np.where(mask, a.v, b.v), np.where(mask, a.m, b.m))


def scatter(n_rows, pairs):
    """Rows added by atomics into a zeroed accumulator: sum of (ids, contributions [k, ...]) over `pairs`; each of a
    row's adds rounds at most its partial sum."""
    ids = np.concatenate([np.asarray(i).ravel() for i, _ in pairs])
    d = cat([c for _, c in pairs], 0)
    S = sp.csr_matrix((np.ones(len(ids)), (ids, np.arange(len(ids)))), shape=(n_rows, len(ids)))
    mag = S @ np.abs(d.v)
    if R.exact:
        assert_exact([d.v], mag, "scatter")
    cnt = np.bincount(ids, minlength=n_rows).astype(np.float64).reshape((-1,) + (1,) * (d.v.ndim - 1))
    return R(S @ d.v, S @ np.broadcast_to(d.m, d.v.shape) + cnt * mag)


def pair_loss(kind, x):
    """learner.cuh pairwise_loss_grad -> (per-sample loss, dl/dx)."""
    if kind == "hinge":
        if R.exact:
            assert not (x.v == -1.0).any(), "a hinge case sits on the tie x = -1"
        t = x + 1.0
        return where(t.v > 0, t), R((t.v > 0).astype(np.float64))
    if kind == "square":
        t = 1.0 - x
        return t * t, -2.0 * t
    if kind == "bpr":
        if R.exact:
            assert (x.v == 0).all(), "exact BPR cases sit at x = 0"
        with np.errstate(over="ignore"):
            g = -1.0 / (1.0 + np.exp(x.v))
        l = np.logaddexp(0.0, -x.v)
        return R(l, 4 * np.abs(l) + np.abs(g) * x.m), R(g, 4 * np.abs(g) + np.abs(g * (1 + g)) * x.m)
    raise ValueError(kind)


def loss_sum(lo):
    """The batch loss (atomics in any order) and whether fp32 sums it exactly."""
    saved, R.exact = R.exact, False
    try:
        s = lo.sum(0)
    finally:
        R.exact = saved
    return s, saved and is_exact([lo.v], np.abs(lo.v).sum())


def dyadic(rs, shape, lo=-1, hi=1, k=2):
    return (rs.randint(lo, hi + 1, shape) / 2.0 ** k).astype(np.float32)


def sparse_dyadic(rs, shape, density=0.3, k=2):
    """Small integers times 2^-k, most of them 0: scores and gradient sums stay far below 2^24 granules."""
    return dyadic(rs, shape, -1, 1, k) * (rs.rand(*shape) < density)


# ---------------------------------------------------------------------------------------------------------------
# SBPR (SBPR.py:66-92): x_* = <p, q_*> + b_*;  loss = l((x_i - x_k) / s) + l(x_k - x_j) + reg * l2_loss(...)
# ---------------------------------------------------------------------------------------------------------------
def sbpr_ref(U, V, Bv, users, pos, soc, neg, suk, kind, reg):
    """-> (per-sample loss, gU, gV, gB, touched users, touched items)."""
    pu, qi, qk, qj = R(U[users]), R(V[pos]), R(V[soc]), R(V[neg])
    bi, bk, bj = R(Bv[pos]), R(Bv[soc]), R(Bv[neg])
    s = np.asarray(suk, np.float64)
    xi, xk, xj = (pu * qi).sum(1) + bi, (pu * qk).sum(1) + bk, (pu * qj).sum(1) + bj
    l1, g1 = pair_loss(kind, (xi - xk) / s)
    l2, g2 = pair_loss(kind, xk - xj)
    saved = R.exact
    R.exact = saved and kind != "bpr"         # BPR's loss is never dyadic: only bounded
    try:
        lo = l1 + l2
        if reg:
            sq = cat([pu * pu, qi * qi, qk * qk, qj * qj], 1).sum(1)
            lo = lo + (reg * 0.5) * (((sq + bi * bi) + bk * bk) + bj * bj)
    finally:
        R.exact = saved
    ci = g1 / s
    ck, cj = g2 - ci, -g2
    c = lambda a: a[:, None]
    gU = scatter(U.shape[0], [(users, ((c(ci) * qi + c(ck) * qk) + c(cj) * qj) + reg * pu)])
    gV = scatter(V.shape[0], [(pos, c(ci) * pu + reg * qi), (soc, c(ck) * pu + reg * qk),
                              (neg, c(cj) * pu + reg * qj)])
    gB = scatter(V.shape[0], [(pos, ci + reg * bi), (soc, ck + reg * bk), (neg, cj + reg * bj)])
    tU = np.zeros(U.shape[0], bool); tU[users] = True
    tV = np.zeros(V.shape[0], bool); tV[pos] = True; tV[soc] = True; tV[neg] = True
    return lo, gU, gV, gB, tU, tV


def sbpr_torch_loss(t, users, pos, soc, neg, suk, kind, reg):
    U, V, Bv = t
    x = lambda i: (U[users] * V[i]).sum(1) + Bv[i]
    s = torch.tensor(suk, dtype=torch.float64)

    def l(y):
        if kind == "bpr":
            return torch.nn.functional.softplus(-y)
        if kind == "hinge":
            return torch.clamp(y + 1.0, min=0.0)
        return (1.0 - y) ** 2
    sq = sum((a * a).sum(1) for a in (U[users], V[pos], V[soc], V[neg])) + Bv[pos] ** 2 + Bv[soc] ** 2 + Bv[neg] ** 2
    return (l((x(pos) - x(soc)) / s) + l(x(soc) - x(neg)) + reg * 0.5 * sq).sum()


@pytest.mark.parametrize("kind", ["bpr", "hinge", "square"])
def test_sbpr_reference_matches_autograd(kind):
    """CPU: the float64 SBPR reference's loss and gradients equal torch.autograd's, with every s_uk in 1..5, repeated
    users and items, and social items equal to the positive or the negative."""
    rs = np.random.RandomState(len(kind))
    nu, ni, D, B = 5, 9, 6, 40
    T = [rs.randn(nu, D) * 0.7, rs.randn(ni, D) * 0.7, rs.randn(ni) * 0.7]
    users, pos, soc, neg = (rs.randint(0, n, B) for n in (nu, ni, ni, ni))
    soc[::5], soc[1::5] = pos[::5], neg[1::5]
    suk = np.arange(B) % 5 + 1.0
    lo, gU, gV, gB, _, _ = sbpr_ref(*T, users, pos, soc, neg, suk, kind, 0.25)
    t = [torch.tensor(a, dtype=torch.float64, requires_grad=True) for a in T]
    loss = sbpr_torch_loss(t, users, pos, soc, neg, suk, kind, 0.25)
    loss.backward()
    assert abs(loss.item() - lo.v.sum()) <= 1e-12 * max(1.0, abs(loss.item()))
    for a, w in zip(t, (gU, gV, gB)):
        np.testing.assert_allclose(w.v, a.grad.numpy(), rtol=1e-12, atol=1e-12)


def sbpr_scores64(U, V, Bv, users, items):
    return (U[users].astype(np.float64) * V[items]).sum(1) + Bv[items]


def sbpr_case(rs, B, D, kind, heavy=False, suks=(1, 2, 4)):
    """Tables and ids of one exact batch: repeated users and items, social items equal to the positive (every fifth
    sample) or the negative (the next ones); BPR at x = 0 on both pairs (pos, social and negative rows cloned)."""
    nu, ni = (37, 216) if heavy else (B + 5, 3 * B + 6)
    U, V, Bv = sparse_dyadic(rs, (nu, D)), sparse_dyadic(rs, (ni, D)), dyadic(rs, (ni,))
    users = rs.randint(0, nu, B).astype(np.int32)
    pos, soc, neg = (rs.randint(0, ni, B).astype(np.int32) for _ in range(3))
    suk = rs.choice(np.asarray(suks, np.float32), B)
    if B > 1:
        users[1] = users[0]
    at_pos, at_neg = np.arange(B) % 5 == 0, np.arange(B) % 5 == 1
    if kind == "bpr":                         # items 3t, 3t+1, 3t+2 share one row: x_i = x_k = x_j
        pos -= pos % 3
        soc, neg = pos + 1, pos + 2
        for t in (V, Bv):
            t[1::3] = t[0::3][:len(t[1::3])]
            t[2::3] = t[0::3][:len(t[2::3])]
        return U, V, Bv, users, pos, soc, neg, suk
    for _ in range(200):
        soc[at_pos], soc[at_neg] = pos[at_pos], neg[at_neg]
        xi, xk, xj = (sbpr_scores64(U, V, Bv, users, a) for a in (pos, soc, neg))
        tie = ((xi - xk) / suk == -1.0) | (xk - xj == -1.0)
        if kind != "hinge" or not tie.any():
            break
        neg[tie] = rs.randint(0, ni, int(tie.sum()))
        free = tie & ~at_pos & ~at_neg
        soc[free] = rs.randint(0, ni, int(free.sum()))
    return U, V, Bv, users, pos, soc, neg, suk


def sbpr_device_grad(U, V, Bv, users, pos, soc, neg, suk, kind, reg, stamp=9, loss0=0.5):
    """One gradient call into zeroed accumulators, stamps filled with 5 and the loss cell at loss0 -> host arrays
    and the route record of the call."""
    from neurec_b200 import ops
    dU, dV, dB = dev(U), dev(V), dev(Bv)
    g = [torch.zeros_like(t) for t in (dU, dV, dB)]
    tU = torch.full((U.shape[0],), 5, dtype=torch.int32, device="cuda")
    tV = torch.full((V.shape[0],), 5, dtype=torch.int32, device="cuda")
    lo = torch.full((1,), loss0, device="cuda")
    ops.sbpr_grad(dU, dV, dB, dev(users), dev(pos), dev(soc), dev(neg), dev(suk), kind, reg, *g, tU, tV, stamp, lo)
    return float(lo), [host(a) for a in g], host(tU), host(tV), routes()["sbpr_grad"]


def check_sbpr(case, kind, reg, exact):
    U, V, Bv, users, pos, soc, neg, suk = case
    R.exact = exact
    try:
        lo, gU, gV, gB, tU, tV = sbpr_ref(U, V, Bv, users, pos, soc, neg, suk, kind, reg)
        want_l, loss_exact = loss_sum(lo)
    finally:
        R.exact = False
    got_l, g, sU, sV, r = sbpr_device_grad(U, V, Bv, users, pos, soc, neg, suk, kind, reg)
    # fp32 atomicAdd on global memory flushes subnormal operands and results to zero (the |x| = 85 pairs give
    # gradients near 2^-126): up to 2^-126 per add into a row, on top of the rounding bound
    adds = (np.bincount(users, minlength=U.shape[0])[:, None],
            np.bincount(np.concatenate([pos, soc, neg]), minlength=V.shape[0])[:, None],
            np.bincount(np.concatenate([pos, soc, neg]), minlength=V.shape[0]))
    for a, w, name, cnt in zip(g, (gU, gV, gB), ("gU", "gV", "gB"), adds):
        if exact:
            assert np.array_equal(a.astype(np.float64), w.v), (name, float(np.abs(a - w.v).max()))
        else:
            assert_within(a, w.v, w.m, name, floor=2.0 ** -126 * cnt)
    assert np.array_equal(sU, np.where(tU, 9, 5)) and np.array_equal(sV, np.where(tV, 9, 5))
    # the batch loss is added into *loss (0.5 there before the call)
    if loss_exact:
        assert got_l == 0.5 + float(want_l.v), (got_l, float(want_l.v))
    else:
        assert_within(got_l, 0.5 + want_l.v, want_l.m + np.abs(0.5 + want_l.v), "loss")
    return r


@gpu
@pytest.mark.parametrize("dim", SBPR_DIMS)
@pytest.mark.parametrize("kind,suks", [("hinge", (1, 2, 4)), ("square", (1, 2, 4)), ("bpr", (1, 2, 4))])
def test_sbpr_grad_exact(kind, suks, dim):
    """Batches 1, 64 * SMs, 64 * SMs + 1 and a heavy-duplicate multiple: gradients, stamps and the loss bit for bit
    (BPR at x = 0, its loss within the bound)."""
    n_sms = sms()
    rs = np.random.RandomState(dim * 7 + len(kind))
    reg = 0.0 if kind == "hinge" and dim % 2 else 2.0 ** -3
    batches = sbpr_batches(n_sms)
    for bi, B in enumerate(batches):
        case = sbpr_case(rs, B, dim, kind, heavy=bi == len(batches) - 1, suks=suks)
        r = check_sbpr(case, kind, reg, exact=True)
        grid, capped = warp_grid(B, n_sms)
        assert (r["grid"], r["capped"]) == (grid, capped)
        SEEN.add(("sbpr_grad", kind, int(capped)))
    SEEN.add(("sbpr_dim", dim))


def sbpr_rounded_case(rs, B, D, heavy):
    nu, ni = (37, 216) if heavy else (B + 5, 3 * B + 6)
    U = (rs.randn(nu, D) * 0.3).astype(np.float32)
    V = (rs.randn(ni, D) * 0.3).astype(np.float32)
    Bv = (rs.randn(ni) * 0.3).astype(np.float32)
    users = rs.randint(0, nu, B).astype(np.int32)
    pos, soc, neg = (rs.randint(4, ni, B).astype(np.int32) for _ in range(3))
    soc[::5], soc[1::5] = pos[::5], neg[1::5]
    suk = rs.choice(np.asarray([1, 2, 3, 4, 5], np.float32), B)
    # items 0..3 carry biases that put both pairs of user 0 (a zero row) at |x| = 85 (beyond 80, below 88.7 where
    # expf stays finite)
    Bv[:4] = [170.0, 85.0, 0.0, -85.0]
    U[0] = 0.0
    for b, (i, k, j) in zip(range(0, min(B, 8)), [(0, 1, 2), (2, 1, 0), (1, 2, 3), (3, 2, 1)] * 2):
        users[b], pos[b], soc[b], neg[b], suk[b] = 0, i, k, j, 1.0
    return U, V, Bv, users, pos, soc, neg, suk


@gpu
@pytest.mark.parametrize("dim", [1, 33, 64, 256])
def test_sbpr_grad_rounded(dim):
    """BPR with realistic tables, s_uk in 1..5 (3 and 5 round the division) and pairs with |x| > 80: gradients within
    2 * 2^-24 * M of float64, stamps exact."""
    n_sms = sms()
    rs = np.random.RandomState(dim + 101)
    batches = sbpr_batches(n_sms)
    for bi, B in enumerate(batches):
        case = sbpr_rounded_case(rs, B, dim, heavy=bi == len(batches) - 1)
        r = check_sbpr(case, "bpr", 2.0 ** -6, exact=False)
        assert (r["grid"], r["capped"]) == warp_grid(B, n_sms)
        SEEN.add(("sbpr_rounded", int(r["capped"])))


def sbpr_epoch_case(rs, n, bs, D, kind):
    """n samples in which step s reads only users s * 8 + [0, 8) and items s * 16 + [0, 16): no step reads a row an
    earlier step moved, so every step's gradient is exact from the tables before the epoch."""
    steps = -(-n // bs)
    nu, ni = 8 * (steps + 1), 16 * (steps + 1)
    s = np.arange(n) // bs
    U, V, Bv = sparse_dyadic(rs, (nu, D)), sparse_dyadic(rs, (ni, D)), dyadic(rs, (ni,))
    users = (s * 8 + rs.randint(0, 8, n)).astype(np.int32)
    pos, soc, neg = ((s * 16 + rs.randint(0, 16, n)).astype(np.int32) for _ in range(3))
    suk = rs.choice(np.asarray([1, 2, 4], np.float32), n)
    for _ in range(200):
        xi, xk, xj = (sbpr_scores64(U, V, Bv, users, a) for a in (pos, soc, neg))
        tie = ((xi - xk) / suk == -1.0) | (xk - xj == -1.0)
        if kind != "hinge" or not tie.any():
            break
        neg[tie] = s[tie] * 16 + rs.randint(0, 16, int(tie.sum()))
    return U, V, Bv, users, pos, soc, neg, suk


@gpu
@pytest.mark.parametrize("opt", OPTS)
def test_sbpr_epoch_exact(opt):
    """A short last batch, batch_size > n and n = 0, first_stamp > 1: tables, slots, stamps and every step's loss equal
    tf_math.opt_apply on the float64 gradients bit for bit."""
    from neurec_b200 import ops
    rs = np.random.RandomState(OPTS.index(opt) + 31)
    D, reg = 33, 2.0 ** -3
    kind = "hinge" if OPTS.index(opt) % 2 else "square"
    for n, bs, first in ((3 * 64 + 5, 64, 7), (5, 64, 1), (0, 64, 3)):
        steps = -(-n // bs)
        U, V, Bv, users, pos, soc, neg, suk = sbpr_epoch_case(rs, n, bs, D, kind)
        T = [U, V, Bv]
        i0, i1 = tf_math.SLOT_INIT[opt]
        H = [a.copy() for a in T]
        S0 = [None if i0 is None else np.full_like(a, i0) for a in T]
        S1 = [None if i1 is None else np.full_like(a, i1) for a in T]
        dT, dS0, dS1 = [dev(a) for a in T], [dev(a) for a in S0], [dev(a) for a in S1]
        grads = [torch.zeros_like(t) for t in dT]
        tU = torch.zeros(U.shape[0], dtype=torch.int32, device="cuda")
        tV = torch.zeros(V.shape[0], dtype=torch.int32, device="cuda")
        lr_t = tf_math.adam_lr_t(HYPER["adam"][0], max(steps, 1)) if opt == "adam" else \
            np.full(max(steps, 1), HYPER[opt][0], np.float32)
        step_loss = torch.full((max(steps, 1),), 7.0, device="cuda")
        before = routes()["sbpr_grad"]
        got_steps = ops.sbpr_train_epoch(*dT, dev(users), dev(pos), dev(soc), dev(neg), dev(suk), bs, kind, reg, opt,
                                         lr_t, HYPER[opt], *grads, tU, tV, dS0[0], dS1[0], dS0[1], dS1[1], dS0[2],
                                         dS1[2], first, step_loss)
        assert got_steps == steps
        want_tU, want_tV = np.zeros(U.shape[0], np.int32), np.zeros(V.shape[0], np.int32)
        want_loss = np.full(max(steps, 1), 7.0, np.float32)
        for s in range(steps):
            sl = slice(s * bs, min(n, (s + 1) * bs))
            R.exact = True
            try:
                lo, gU, gV, gB, mU, mV = sbpr_ref(*H, users[sl], pos[sl], soc[sl], neg[sl], suk[sl], kind, reg)
                l, loss_exact = loss_sum(lo)
            finally:
                R.exact = False
            assert loss_exact
            want_loss[s] = l.v
            hyper = list(HYPER[opt])
            if opt == "adam":
                hyper[0] = lr_t[s]
            for k, (var, gk, m) in enumerate(zip(H, (gU, gV, gB), (mU, mV, mV))):
                g32 = gk.v.astype(np.float32)
                assert np.array_equal(g32, gk.v)
                tf_math.opt_apply(opt, var, g32, S0[k], S1[k], m, hyper)
            want_tU[mU], want_tV[mV] = first + s, first + s
        for k in range(3):
            assert np.array_equal(host(dT[k]), H[k]), (n, k)
            for dsl, hsl in ((dS0[k], S0[k]), (dS1[k], S1[k])):
                if hsl is not None:
                    assert np.array_equal(host(dsl), hsl), (n, k)
            assert not grads[k].any()
        assert np.array_equal(host(tU), want_tU) and np.array_equal(host(tV), want_tV)
        assert np.array_equal(host(step_loss), want_loss)
        if n == 0:
            assert routes()["sbpr_grad"] == before
        else:
            assert routes()["sbpr_grad"]["grid"] == warp_grid(n - (steps - 1) * bs, sms())[0]
        SEEN.add(("sbpr_epoch", opt, n == 0))


@pytest.fixture(scope="module")
def ciao():
    z = np.load(os.path.join(GOLDEN, "ciao_split.npz"))
    d = {k: z[k] for k in z.files}
    d["num_users"], d["num_items"] = int(z["num_users"]), int(z["num_items"])
    for k in ("train_indptr", "trust_indptr"):
        d[k] = d[k].astype(np.int64)
    for k in ("train_indices", "trust_indices"):
        d[k] = d[k].astype(np.int32)
    sptr, sidx = oracle.social_items_csr(d["train_indptr"], d["train_indices"], d["trust_indptr"], d["trust_indices"])
    d["social_indptr"], d["social_indices"] = sptr, sidx
    eligible = np.diff(sptr) > 0
    deg = np.diff(d["train_indptr"])
    d["pos_users"] = np.repeat(np.arange(d["num_users"], dtype=np.int32), np.where(eligible, deg, 0))
    d["pos_items"] = d["train_indices"][np.repeat(eligible, deg)]
    d["max_excluded"] = int((deg + np.diff(sptr))[eligible].max())
    return d


@gpu
@pytest.mark.parametrize("shuffle,epoch", [(True, 3), (False, 0)])
def test_sbpr_epoch_build_beyond_the_cap(ciao, shuffle, epoch):
    """Ciao's positives tiled twice (above 2048 * SMs samples): the whole epoch and windows on both sides of the cap
    and straddling it, bit for bit against oracle.sbpr_epoch_build."""
    from neurec_b200 import ops
    n_sms, c = sms(), ciao
    pu, pi = np.tile(c["pos_users"], 2), np.tile(c["pos_items"], 2)
    n = len(pu)
    cap = 2048 * n_sms
    assert n > cap + 1000
    csr = [c[k] for k in ("train_indptr", "train_indices", "social_indptr", "social_indices", "trust_indptr",
                          "trust_indices")]
    want = oracle.sbpr_epoch_build(*csr, pu, pi, c["num_items"], shuffle, 2018, epoch)
    dcsr = [dev(a) for a in csr]
    for first, count in ((0, n), (0, cap), (0, cap + 1), (n - cap - 1, cap + 1), (cap - 3, 7), (1000, cap - 1)):
        got = ops.sbpr_epoch_build(*dcsr, dev(pu), dev(pi), c["num_items"], c["max_excluded"], shuffle, 2018, epoch,
                                   first, count)
        for g, w, name in zip(got, want, ("users", "pos", "social", "neg", "suk")):
            assert np.array_equal(host(g), w[first:first + count]), (first, count, name)
        r = routes()["sbpr_epoch_build"]
        assert (r["grid"], r["capped"]) == elem_grid(count, n_sms)
        SEEN.add(("sbpr_build", int(r["capped"])))


# ---------------------------------------------------------------------------------------------------------------
# APR's normaliser: x * rsqrt(max(sum x^2, 1e-12)) * scale
# ---------------------------------------------------------------------------------------------------------------
RSQRT_ULP = 2          # CUDA C Programming Guide, mathematical functions: rsqrtf's maximum error is 2 ulp
EPS32 = float(np.float32(1e-12))


def l2_normalize_ref(x, scale):
    """-> (float64 value, bound M in units of 2^-24): sum of squares with fmaf (dim roundings, relative), max with
    the epsilon, rsqrtf (RSQRT_ULP ulp = 2 * RSQRT_ULP units of 2^-24 relative, plus half the sum's relative error),
    then two rounded products."""
    x = np.asarray(x, np.float64)
    ss = (x * x).sum(1, keepdims=True)
    big = ss >= EPS32
    inv = 1.0 / np.sqrt(np.where(big, ss, EPS32))
    v = x * inv * scale
    # the sum of squares: ceil(dim / 32) fmaf per lane and 5 shuffle adds, each within 2^-24 of the whole sum
    rel = 2 * RSQRT_ULP + 2 + 1 + np.where(big, 0.5 * (x.shape[1] + 5), 0.0)
    return v, np.abs(v) * rel


@gpu
@pytest.mark.parametrize("dim", NORM_DIMS)
def test_l2_normalize_rows(dim):
    """Rows on both sides of 64 * SMs, zero rows, rows whose sum of squares is below 1e-12 (the epsilon branch), and
    in-place use: within the bound set by rsqrtf's documented error; zero rows exactly zero."""
    from neurec_b200 import ops
    n_sms = sms()
    rs = np.random.RandomState(dim)
    for rows in warp_rows(n_sms):
        x = rs.randn(rows, dim).astype(np.float32) * np.float32(3.0)
        x[::97] = 0.0
        x[5::89] *= np.float32(1e-9)          # sum of squares ~ dim * 1e-17: the epsilon branch
        v, M = l2_normalize_ref(x, 0.375)
        assert ((x[5::89].astype(np.float64) ** 2).sum(1) < EPS32 / 10).all()
        got = host(ops.l2_normalize_rows(dev(x), 0.375))
        assert_within(got, v, M, ("l2", dim, rows), C=1.0)
        assert (got[::97] == 0).all()
        r = routes()["l2_normalize_rows"]
        assert (r["grid"], r["capped"]) == warp_grid(rows, n_sms)
        t = dev(x)
        ops.l2_normalize_rows(t, 0.375, out=t)
        assert np.array_equal(host(t), got)
        SEEN.add(("l2", int(r["capped"])))
    SEEN.add(("l2_dim", dim))


@gpu
def test_gather_rows_i32():
    """out[p] = src[index[p] % rows] on both sides of 2048 * SMs elements, widths 1, 3 and 32."""
    from neurec_b200 import ops
    n_sms = sms()
    rs = np.random.RandomState(5)
    for width in (1, 3, 32):
        src = rs.randint(-2 ** 31, 2 ** 31 - 1, (1000, width)).astype(np.int32)
        for total in (2048 * n_sms, 2048 * n_sms + width):
            n = total // width
            index = rs.randint(0, 10 ** 6, n).astype(np.int64)
            got = host(ops.gather_rows_i32(dev(src), dev(index)))
            assert np.array_equal(got, src[index % 1000])
            r = routes()["gather_rows_i32"]
            assert (r["grid"], r["capped"]) == elem_grid(n * width, n_sms)
            SEEN.add(("gather", int(r["capped"])))


# ---------------------------------------------------------------------------------------------------------------
# LightGCN's BPR gradient (LightGCN.py:99-104, 156-166)
# ---------------------------------------------------------------------------------------------------------------
def lightgcn_grad_ref(E, E0, nu, users, pos, neg, reg, scale):
    """-> (mf loss per sample, emb loss per sample, G, Rg): x = <E_u, E_i> - <E_u, E_j>; G += scale * dl/dE,
    Rg += reg * E0 of every row a sample reads."""
    n, D = E.shape
    ru, ri, rj = users, nu + pos, nu + neg
    a, bi, bj = R(E[ru]), R(E[ri]), R(E[rj])
    x = (a * bi).sum(1) - (a * bj).sum(1)
    l, g = pair_loss("bpr", x)
    sq = cat([R(E0[ru]) * R(E0[ru]), R(E0[ri]) * R(E0[ri]), R(E0[rj]) * R(E0[rj])], 1).sum(1)
    emb = (reg * 0.5) * sq
    gs = (g * scale)[:, None]
    G = scatter(n, [(ru, gs * (bi - bj)), (ri, gs * a), (rj, -gs * a)])
    Rg = scatter(n, [(r, reg * R(E0[r])) for r in (ru, ri, rj)])
    return l, emb, G, Rg


def test_lightgcn_grad_reference_matches_autograd():
    """CPU: the float64 LightGCN gradient reference equals torch.autograd's d(mf loss)/dE times scale and
    d(emb loss)/dE0, with repeated users and items and a negative equal to the positive."""
    rs = np.random.RandomState(3)
    nu, ni, D, B = 4, 6, 5, 30
    E, E0 = rs.randn(nu + ni, D), rs.randn(nu + ni, D)
    users, pos, neg = rs.randint(0, nu, B), rs.randint(0, ni, B), rs.randint(0, ni, B)
    neg[::7] = pos[::7]
    l, emb, G, Rg = lightgcn_grad_ref(E, E0, nu, users, pos, neg, 0.25, 0.25)
    tE = torch.tensor(E, requires_grad=True)
    tE0 = torch.tensor(E0, requires_grad=True)
    x = (tE[users] * tE[nu + pos]).sum(1) - (tE[users] * tE[nu + neg]).sum(1)
    mf = torch.nn.functional.softplus(-x).sum()
    em = 0.25 * 0.5 * sum((tE0[r] ** 2).sum() for r in (users, nu + pos, nu + neg))
    (mf + em).backward()
    assert abs(mf.item() - l.v.sum()) <= 1e-12 * mf.item() and abs(em.item() - emb.v.sum()) <= 1e-12 * em.item()
    np.testing.assert_allclose(G.v, 0.25 * tE.grad.numpy(), rtol=1e-12, atol=1e-12)
    np.testing.assert_allclose(Rg.v, tE0.grad.numpy(), rtol=1e-12, atol=1e-12)


def lightgcn_case(rs, B, D, nu, ni, exact):
    """Exact: dyadic tables, the negative's rows cloned from the positive's (x = 0, g = -1/2).  Rounded: realistic."""
    n = nu + ni
    if exact:
        E, E0 = sparse_dyadic(rs, (n, D)), dyadic(rs, (n, D))
        pos = 2 * rs.randint(0, ni // 2, B)
        neg = pos + 1
        E[nu + 1::2] = E[nu::2][:len(E[nu + 1::2])]
    else:
        E, E0 = (rs.randn(n, D) * 0.3).astype(np.float32), (rs.randn(n, D) * 0.3).astype(np.float32)
        pos, neg = rs.randint(0, ni, B), rs.randint(0, ni, B)
    users = rs.randint(0, nu, B)
    return E, E0, users.astype(np.int32), pos.astype(np.int32), neg.astype(np.int32)


@gpu
@pytest.mark.parametrize("dim", [1, 33, 64, 128])
@pytest.mark.parametrize("exact", [True, False])
def test_lightgcn_bpr_grad(dim, exact):
    """Batches on both sides of 64 * SMs and a heavy-duplicate multiple; reg = 0 leaves R untouched.  Exact at x = 0
    with scale 1/4: G, R and the emb loss bit for bit, the mf loss within its bound; rounded otherwise."""
    from neurec_b200 import ops
    n_sms = sms()
    rs = np.random.RandomState(dim * 3 + exact)
    for bi, B in enumerate(sbpr_batches(n_sms)):
        heavy = bi == 3
        nu, ni = (29, 64) if heavy else (B + 3, 2 * B + 4)
        E, E0, users, pos, neg = lightgcn_case(rs, B, dim, nu, ni, exact)
        for reg in ((2.0 ** -3, 0.0) if bi in (1, 2) else (2.0 ** -3,)):
            R.exact = exact
            try:
                l, emb, G, Rg = lightgcn_grad_ref(E, E0, nu, users, pos, neg, reg, 0.25)
                want_emb, emb_exact = loss_sum(emb)
            finally:
                R.exact = False
            want_mf, _ = loss_sum(l)
            gG = torch.zeros(E.shape, device="cuda")
            gR = torch.full(E.shape, 0.0 if reg else 3.0, device="cuda")
            loss2 = torch.tensor([0.5, 0.25], device="cuda")
            ops.lightgcn_bpr_grad(dev(E), dev(E0), nu, dev(users), dev(pos), dev(neg), reg, 0.25, gG, gR, loss2)
            got_G, got_R, got_l = host(gG), host(gR), host(loss2).astype(np.float64)
            if exact:
                assert np.array_equal(got_G, G.v), float(np.abs(got_G - G.v).max())
                assert np.array_equal(got_R, Rg.v) if reg else (got_R == 3.0).all()
                assert emb_exact and got_l[1] == 0.25 + want_emb.v
            else:
                assert_within(got_G, G.v, G.m, "G")
                if reg:
                    assert_within(got_R, Rg.v, Rg.m, "R")
                else:
                    assert (got_R == 3.0).all()
                assert_within(got_l[1], 0.25 + want_emb.v, want_emb.m + 0.25 + want_emb.v, "emb")
            assert_within(got_l[0], 0.5 + want_mf.v, want_mf.m + 0.5 + want_mf.v, "mf")
            r = routes()["lightgcn_bpr_grad"]
            assert (r["grid"], r["capped"]) == warp_grid(B, n_sms)
            SEEN.add(("lightgcn_grad", exact, int(r["capped"]), reg == 0))


def csr_dev(A):
    return dev(A.indptr.astype(np.int64)), dev(A.indices.astype(np.int32)), dev(A.data.astype(np.float32))


def degree_order(A):
    return dev(np.argsort(-np.diff(A.indptr), kind="stable").astype(np.int32))


@gpu
@pytest.mark.parametrize("adj_type", ["norm", "gcmc"])
@pytest.mark.parametrize("n_layers,dim", [(2, 32), (6, 50), (6, 32), (2, 50)])
def test_lightgcn_epoch_asymmetric(ml100k, adj_type, n_layers, dim):
    """The asymmetric adjacencies with their explicit transpose (LightGCN.py:89-93), 2 and 6 layers (the conf
    default), widths 32 (the fast SpMM) and 50 (the generic one), 3 steps against tf_math.LightGCNTrainer.  The
    backward must read A^T: through A the result moves by far more than the tolerance."""
    from neurec_b200 import ops
    d = ml100k
    nu, ni, bs, steps = d["num_users"], d["num_items"], 1024, 3
    A = tf_math.lightgcn_adj(d["train_indptr"], d["train_indices"], nu, ni, adj_type)
    AT = A.T.tocsr(); AT.sort_indices()
    assert abs(A - AT).max() > 1e-3
    rs = np.random.RandomState(n_layers * 100 + dim)
    lim = np.sqrt(6.0 / (nu + dim))
    e0 = rs.uniform(-lim, lim, (nu + ni, dim)).astype(np.float32)
    all_users = np.repeat(np.arange(nu, dtype=np.int32), np.diff(d["train_indptr"]))
    perm = rs.permutation(len(all_users))[:bs * steps - 300]
    users, pos = all_users[perm], d["train_indices"][perm]
    neg = rs.randint(0, ni, len(users)).astype(np.int32)
    tr = tf_math.LightGCNTrainer(A, e0, nu, n_layers, 0.01, 1e-3)
    want = tr.epoch(users, pos, neg, bs)
    de0 = dev(e0)
    z = lambda: torch.zeros_like(de0)
    m, v, ef, gf, ge, wa, wb = z(), z(), z(), z(), z(), z(), z()
    sl = torch.zeros(steps, 2, device="cuda")
    n = ops.lightgcn_train_epoch(csr_dev(A), csr_dev(AT), degree_order(A), nu, ni, n_layers, de0, m, v, dev(users),
                                 dev(pos), dev(neg), bs, 1e-3, tf_math.adam_lr_t(0.01, steps),
                                 [0.01, 0.9, 0.999, 1e-8], ef, gf, ge, (wa, wb), sl)
    assert n == steps
    assert np.allclose(host(sl), want, rtol=1e-4)
    assert np.abs(host(de0) - tr.e0).max() < 5e-5
    assert not gf.any() and not ge.any()
    r = routes()["lightgcn_bpr_grad"]
    assert (r["grid"], r["capped"]) == warp_grid(len(users) - (steps - 1) * bs, sms())
    SEEN.add(("lightgcn_epoch", adj_type, n_layers, dim))


@gpu
@pytest.mark.parametrize("dim", [32, 33])
def test_lightgcn_step_exact_adam(dim):
    """One step on a small asymmetric graph with power-of-two values and the negative's rows cloned from the
    positive's (x = 0): the propagation, the BPR gradient and the backward through A^T are exact, so the Adam result
    equals tf_math.opt_apply on the float64 gradient bit for bit."""
    from neurec_b200 import ops
    rs = np.random.RandomState(dim)
    nu, ni, L, B, reg = 24, 40, 3, 64, 2.0 ** -3
    n = nu + ni
    dense = (rs.rand(n, n) < 0.08) * rs.choice([0.5, 0.25, -0.25], (n, n))
    pos = 2 * rs.randint(0, ni // 2, B)
    neg = pos + 1
    dense[nu + 1::2] = dense[nu::2]           # row U + j = row U + i: (A^k E0)[U + j] = (A^k E0)[U + i]
    A = sp.csr_matrix(dense.astype(np.float32)); A.sort_indices()
    AT = A.T.tocsr(); AT.sort_indices()
    e0 = dyadic(rs, (n, dim))
    e0[nu + 1::2] = e0[nu::2]
    users = rs.randint(0, nu, B).astype(np.int32)
    # float64 forward, gradient and backward; every intermediate is dyadic and small (asserted)
    Ad, ATd = A.astype(np.float64), AT.astype(np.float64)
    x, layers = e0.astype(np.float64), [e0.astype(np.float64)]
    for _ in range(L):
        assert (abs(Ad) @ np.abs(x) * 2.0 ** (granule_bits(Ad.data) + granule_bits(x)) < 2.0 ** 24).all()
        x = Ad @ x
        layers.append(x)
    E = sum(layers) / (L + 1)
    assert_exact([E], sum(np.abs(y) for y in layers), "mean")
    R.exact = True
    try:
        l, emb, G, Rg = lightgcn_grad_ref(E, e0, nu, users, pos.astype(np.int32), neg.astype(np.int32), reg,
                                          1.0 / (L + 1))
        want_emb, _ = loss_sum(emb)
    finally:
        R.exact = False
    t = G.v
    for _ in range(L):
        mag = abs(ATd) @ np.abs(t) + np.abs(G.v)
        bits = max(granule_bits(ATd.data) + granule_bits(t), granule_bits(G.v))
        assert (mag * 2.0 ** bits < 2.0 ** 24).all(), bits
        t = G.v + ATd @ t
    g = Rg.v + t
    assert_exact([g], np.abs(Rg.v) + np.abs(t), "grad")
    g32 = g.astype(np.float32)
    assert np.array_equal(g32, g)
    lr_t = tf_math.adam_lr_t(0.01, 1)
    want, m_w, v_w = e0.copy(), np.zeros_like(e0), np.zeros_like(e0)
    tf_math.opt_apply("adam", want, g32, m_w, v_w, None, [lr_t[0], 0.9, 0.999, 1e-8], dense_var=True)
    de0 = dev(e0)
    z = lambda: torch.zeros_like(de0)
    m, v, ef, gf, ge, wa, wb = z(), z(), z(), z(), z(), z(), z()
    sl = torch.zeros(1, 2, device="cuda")
    ops.lightgcn_train_epoch(csr_dev(A), csr_dev(AT), None, nu, ni, L, de0, m, v, dev(users), dev(pos.astype(np.int32)),
                             dev(neg.astype(np.int32)), B, reg, lr_t, [0.01, 0.9, 0.999, 1e-8], ef, gf, ge, (wa, wb), sl)
    assert np.array_equal(host(ef), E.astype(np.float32))
    assert np.array_equal(host(m), m_w) and np.array_equal(host(v), v_w)
    assert np.array_equal(host(de0), want)
    assert float(host(sl)[0, 1]) == float(want_emb.v)
    SEEN.add(("lightgcn_exact", dim))


# ---------------------------------------------------------------------------------------------------------------
# interactions -> CSR, the train / test split and the row ids
# ---------------------------------------------------------------------------------------------------------------
def coo_case(rs, num_rows, nnz, num_cols=3000):
    """nnz interactions over num_rows rows with duplicates: empty rows (every third), one row of more than 4096
    entries, one row that repeats a single id, the rest random."""
    live = np.arange(num_rows)[np.arange(num_rows) % 3 != 1]
    long_n = min(4200, nnz // 3)
    rep_n = min(50, nnz // 10)
    rest = nnz - long_n - rep_n
    rows = np.concatenate([np.full(long_n, live[0]), np.full(rep_n, live[-1]), rs.choice(live[1:-1], rest)])
    cols = np.concatenate([rs.randint(0, num_cols, long_n), np.full(rep_n, 7), rs.randint(0, num_cols, rest)])
    p = rs.permutation(nnz)
    return rows[p].astype(np.int32), cols[p].astype(np.int32)


def check_csr(rows, cols, num_rows, num_cols):
    from neurec_b200 import ops
    n_sms = sms()
    ip, ix = ops.csr_from_coo(dev(rows), dev(cols), num_rows, num_cols)
    wp, wx = oracle.csr_from_coo(rows, cols, num_rows)
    assert np.array_equal(host(ip), wp) and np.array_equal(host(ix), wx)
    r = routes()["csr_from_coo"]
    assert (r["grid"], r["capped"]) == (elem_grid(len(rows), n_sms) if len(rows) else (0, 0))
    assert (r["row_grid"], r["row_capped"]) == warp_grid(num_rows, n_sms)
    assert r["scan_chunks"] == (num_rows + 1023) // 1024
    SEEN.add(("csr", r["capped"], r["row_capped"], min(r["scan_chunks"], 3)))
    # the row ids of the same CSR
    ids = host(ops.csr_row_ids(ip))
    assert np.array_equal(ids, np.repeat(np.arange(num_rows, dtype=np.int32), np.diff(wp)))
    r = routes()["csr_row_ids"]
    assert (r["grid"], r["capped"]) == warp_grid(num_rows, n_sms)
    SEEN.add(("row_ids", r["capped"]))


@gpu
def test_csr_from_coo_and_row_ids():
    """1023, 1024, 1025 and 2049 rows (one to three scan chunks), 64 * SMs +- 1 rows and 2048 * SMs +- 1 entries,
    with empty rows, a row of one repeated id and a row of more than 4096 entries: bit for bit against
    oracle.csr_from_coo, and the row ids against numpy."""
    rs = np.random.RandomState(0)
    for num_rows, nnz in csr_shapes(sms()):
        check_csr(*coo_case(rs, num_rows, nnz), num_rows, 3000)
    check_csr(np.zeros(0, np.int32), np.zeros(0, np.int32), 1500, 10)


@gpu
def test_csr_from_coo_gowalla(gowalla):
    """Gowalla's 810 128 train interactions and 29 858 users, shuffled and with 1000 duplicates."""
    g = gowalla
    nu = g["num_users"]
    rows = np.repeat(np.arange(nu, dtype=np.int32), np.diff(g["train_indptr"]))
    cols = g["train_indices"]
    rs = np.random.RandomState(1)
    extra = rs.randint(0, len(rows), 1000)
    rows, cols = np.concatenate([rows, rows[extra]]), np.concatenate([cols, cols[extra]])
    p = rs.permutation(len(rows))
    check_csr(rows[p], cols[p], nu, g["num_items"])


def split_case(rs, num_users, n):
    """Every third user empty, users with 1, 2, 3 and 4 interactions, tied times."""
    live = np.arange(num_users)[np.arange(num_users) % 3 != 1]
    small = np.concatenate([np.full(k, live[k]) for k in (1, 2, 3, 4)] + [np.full(3, live[5])])
    users = np.concatenate([small, rs.choice(live[6:], n - len(small))])
    users = users[rs.permutation(n)].astype(np.int32)
    keys = rs.randint(0, 50, n).astype(np.int64) * 10 ** 9 - 25 * 10 ** 9      # ties, negative times
    return users, keys


@gpu
@pytest.mark.parametrize("mode,by_time", [("ratio", True), ("ratio", False), ("loo", True), ("loo", False)])
def test_split_interactions(mode, by_time):
    """The split at the CSR shapes (scan chunks, 64 * SMs +- 1 users, 2048 * SMs +- 1 interactions), with empty users,
    leave-one-out users of at most 3 interactions and tied times: bit for bit against oracle.split_interactions."""
    from neurec_b200 import ops
    n_sms = sms()
    rs = np.random.RandomState(len(mode) + by_time)
    for num_users, n in csr_shapes(n_sms):
        users, keys = split_case(rs, num_users, n)
        keys = keys if by_time else None
        got = host(ops.split_interactions(dev(users), dev(keys), num_users, mode, 0.7, seed=11))
        want = oracle.split_interactions(users, keys, num_users, mode, 0.7, seed=11)
        assert np.array_equal(got, want), (num_users, n)
        r = routes()["split_interactions"]
        assert (r["grid"], r["capped"]) == elem_grid(n, n_sms)
        assert (r["row_grid"], r["row_capped"]) == warp_grid(num_users, n_sms)
        assert r["scan_chunks"] == (num_users + 1023) // 1024
        SEEN.add(("split", mode, r["capped"], r["row_capped"], min(r["scan_chunks"], 3)))


# ---------------------------------------------------------------------------------------------------------------
# the samplers
# ---------------------------------------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("neg_num", [1, 3])
def test_sample_negatives(neg_num):
    """n * neg_num on both sides of 4096 * SMs, first_index > 0, a user whose train row leaves exactly one item:
    bit for bit against oracle.philox_sample_negatives."""
    from neurec_b200 import ops
    n_sms = sms()
    rs = np.random.RandomState(neg_num)
    nu, ni = 500, 300
    rows = [np.sort(rs.choice(ni, rs.randint(0, 60), replace=False)) for _ in range(nu)]
    rows[7] = np.delete(np.arange(ni), 123)                     # every item but 123
    tp, ti = oracle.lists_to_csr(rows)
    for n in sampler_rows(n_sms, neg_num):
        users = rs.randint(0, nu, n).astype(np.int32)
        users[::101] = 7
        got = host(ops.sample_negatives(dev(tp), dev(ti), dev(users), neg_num, ni, 2018, 5, first_index=12345))
        want = oracle.philox_sample_negatives(tp, ti, users, neg_num, ni, 2018, 5, first_index=12345)
        assert np.array_equal(got, want)
        assert (got[::101] == 123).all()
        r = routes()["sample_negatives"]
        assert (r["grid"], r["capped"]) == sampler_grid(n * neg_num, n_sms)
        SEEN.add(("negatives", neg_num, r["capped"]))


def cut_rows(rs, total, edges):
    """Row offsets over [0, total): a one-element row at every edge in `edges`, random rows of 1..20 elsewhere."""
    cuts = set(int(c) for c in np.cumsum(rs.randint(1, 21, total // 5)) if c < total)
    for e in edges:
        if 0 < e < total:
            cuts |= {e, e + 1} if e + 1 < total else {e}
    return np.asarray([0] + sorted(cuts) + [total], np.int64)


@gpu
def test_batch_randint_choice_replace():
    """The replace form on both sides of 4096 * SMs elements, with one-element rows at the block and grid-stride
    edges: bit for bit against oracle.philox_batch_choice, never an excluded value."""
    from neurec_b200 import ops
    n_sms = sms()
    rs = np.random.RandomState(9)
    high = 40
    c = 4096 * n_sms
    for total in (c, c + 1, 2 * c + 77):
        edges = [255, 256, 257, c - 1, c, total - 1]
        op = cut_rows(rs, total, edges)
        n_rows = len(op) - 1
        excl = [np.sort(rs.choice(high, rs.randint(0, 30), replace=False)) for _ in range(n_rows)]
        ep, ei = oracle.lists_to_csr(excl)
        got = host(ops.batch_randint_choice(high, dev(op), total, True, dev(ep), dev(ei), seed=3, stream_id=4))
        want = oracle.philox_batch_choice(high, op, True, (ep, ei), seed=3, stream_id=4)
        assert np.array_equal(got, want)
        rid = np.repeat(np.arange(n_rows), np.diff(op))
        for e in edges:
            if e < total:
                assert got[e] not in set(excl[rid[e]].tolist())
        r = routes()["batch_randint_choice"]
        assert (r["grid"], r["capped"], r["replace"]) == sampler_grid(total, n_sms) + (1,)
        SEEN.add(("choice_replace", r["capped"]))


@gpu
def test_batch_randint_choice_no_replace_not_enough_integers():
    """The no-replace form with rows where high - |exclusion| equals, exceeds by one and falls one short of the row's
    size: the first and last give -1 (random_choice.pyx:36-37), the others are distinct, outside the exclusion and
    bit for bit the oracle's, as if the short rows were absent."""
    from neurec_b200 import ops
    rs = np.random.RandomState(2)
    high = 30
    sizes, excl = [], []
    for k in range(300):
        e = np.sort(rs.choice(high, rs.randint(0, 20), replace=False))
        room = high - len(e)
        size = [room, room - 1, room + 1][k % 3] if k % 7 == 0 else int(rs.randint(1, max(2, room // 2)))
        sizes.append(max(size, 1)); excl.append(e)
    op = np.concatenate([[0], np.cumsum(sizes)]).astype(np.int64)
    ep, ei = oracle.lists_to_csr(excl)
    got = host(ops.batch_randint_choice(high, dev(op), int(op[-1]), False, dev(ep), dev(ei), seed=8, stream_id=1))
    want = oracle.philox_batch_choice(high, op, False, (ep, ei), seed=8, stream_id=1)
    short = np.asarray([high - len(e) <= s for s, e in zip(sizes, excl)])
    assert short.sum() >= 20 and (~short).sum() > 200
    for k in range(300):
        g, w = got[op[k]:op[k + 1]], want[op[k]:op[k + 1]]
        if short[k]:
            assert (g == -1).all(), k
        else:
            assert np.array_equal(g, w), k
            assert len(set(g.tolist())) == len(g) and not set(g.tolist()) & set(excl[k].tolist())
    r = routes()["batch_randint_choice"]
    assert (r["grid"], r["capped"], r["replace"]) == (2, 0, 0)
    SEEN.add(("choice_noreplace", 1))


# ---------------------------------------------------------------------------------------------------------------
# limits and errors: the library's error, nothing written, the hook unchanged
# ---------------------------------------------------------------------------------------------------------------
@gpu
def test_limits_and_errors_write_nothing():
    from neurec_b200 import _lib
    lib = _lib.load()
    buf = torch.full((4096,), 7, dtype=torch.int32, device="cuda")
    fb = torch.full((4096,), 7.0, device="cuda")
    ip = torch.zeros(64, dtype=torch.int64, device="cuda")
    P, F, I = buf.data_ptr(), fb.data_ptr(), ip.data_ptr()
    lr = np.ones(4, np.float32)
    h = lr.ctypes.data
    calls = {
        "l2_normalize_rows": [lambda: lib.nrc_l2_normalize_rows(F, -1, 4, 1.0, F, None),
                              lambda: lib.nrc_l2_normalize_rows(F, 4, 0, 1.0, F, None),
                              lambda: lib.nrc_l2_normalize_rows(None, 4, 4, 1.0, F, None)],
        "gather_rows_i32": [lambda: lib.nrc_gather_rows_i32(P, 0, 1, I, 4, P, None),
                            lambda: lib.nrc_gather_rows_i32(P, 4, 0, I, 4, P, None),
                            lambda: lib.nrc_gather_rows_i32(P, 4, 1, I, -1, P, None)],
        "sbpr_epoch_build": [lambda: lib.nrc_sbpr_epoch_build(I, P, I, P, I, P, P, P, 4, 0, 0, 1, 1, 0, 0, 4, P, P, P,
                                                              P, F, None),
                             lambda: lib.nrc_sbpr_epoch_build(I, P, I, P, I, P, P, P, -1, 10, 0, 1, 1, 0, 0, 0, P, P,
                                                              P, P, F, None),
                             lambda: lib.nrc_sbpr_epoch_build(I, P, I, P, I, P, P, P, 4, 10, 10, 1, 1, 0, 0, 4, P, P,
                                                              P, P, F, None),
                             lambda: lib.nrc_sbpr_epoch_build(I, P, I, P, I, P, P, P, 4, 10, 0, 1, 1, 0, 2, 3, P, P,
                                                              P, P, F, None),
                             lambda: lib.nrc_sbpr_epoch_build(I, P, I, P, I, P, P, P, 4, 10, 0, 1, 1, 0, -1, 2, P, P,
                                                              P, P, F, None)],
        "sbpr_grad": [lambda: lib.nrc_sbpr_grad(F, F, F, 0, P, P, P, P, F, 4, 0, 0.0, F, F, F, P, P, 1, F, None),
                      lambda: lib.nrc_sbpr_grad(F, F, F, 4, P, P, P, P, F, -1, 0, 0.0, F, F, F, P, P, 1, F, None),
                      lambda: lib.nrc_sbpr_grad(F, F, F, 4, P, P, P, P, F, 4, 3, 0.0, F, F, F, P, P, 1, F, None),
                      lambda: lib.nrc_sbpr_train_epoch(F, F, F, 4, 4, 4, P, P, P, P, F, 4, 0, 0, 0.0, 0, h, h, F,
                                                       F, F, P, P, F, F, F, F, F, F, 1, F, None),
                      lambda: lib.nrc_sbpr_train_epoch(F, F, F, 4, 4, 0, P, P, P, P, F, 4, 4, 0, 0.0, 0, h, h, F,
                                                       F, F, P, P, F, F, F, F, F, F, 1, F, None),
                      lambda: lib.nrc_sbpr_train_epoch(F, F, F, 4, 4, 4, P, P, P, P, F, -1, 4, 0, 0.0, 0, h, h, F,
                                                       F, F, P, P, F, F, F, F, F, F, 1, F, None)],
        "csr_from_coo": [lambda: lib.nrc_csr_from_coo(P, P, 4, 0, 4, I, P, I, P, P, None),
                         lambda: lib.nrc_csr_from_coo(P, P, 4, 4, 0, I, P, I, P, P, None),
                         lambda: lib.nrc_csr_from_coo(P, P, -1, 4, 4, I, P, I, P, P, None)],
        "split_interactions": [lambda: lib.nrc_split_interactions(P, None, 4, 0, 0, 0.5, 1, P, I, P, P, None),
                               lambda: lib.nrc_split_interactions(P, None, -1, 4, 0, 0.5, 1, P, I, P, P, None),
                               lambda: lib.nrc_split_interactions(P, None, 4, 4, 2, 0.5, 1, P, I, P, P, None),
                               lambda: lib.nrc_split_interactions(P, None, 4, 4, 0, 1.5, 1, P, I, P, P, None),
                               lambda: lib.nrc_split_interactions(P, None, 4, 4, 0, -0.5, 1, P, I, P, P, None)],
        "csr_row_ids": [lambda: lib.nrc_csr_row_ids(I, -1, P, None)],
        "sample_negatives": [lambda: lib.nrc_sample_negatives(I, P, P, 4, 0, 10, 1, 0, 0, P, None),
                             lambda: lib.nrc_sample_negatives(I, P, P, 4, 1, 0, 1, 0, 0, P, None),
                             lambda: lib.nrc_sample_negatives(I, P, P, -1, 1, 10, 1, 0, 0, P, None)],
        "batch_randint_choice": [lambda: lib.nrc_batch_randint_choice(0, I, 2, 4, 1, None, None, 1, 0, P, None),
                                 lambda: lib.nrc_batch_randint_choice(10, I, -1, 4, 1, None, None, 1, 0, P, None),
                                 lambda: lib.nrc_batch_randint_choice(10, I, 2, -1, 0, None, None, 1, 0, P, None)],
        "lightgcn_bpr_grad": [lambda: lib.nrc_lightgcn_bpr_grad(F, F, 2, 0, P, P, P, 4, 0.0, 1.0, F, F, F, None),
                              lambda: lib.nrc_lightgcn_bpr_grad(F, F, 2, 4, P, P, P, -1, 0.0, 1.0, F, F, F, None),
                              lambda: lib.nrc_lightgcn_train_epoch(I, P, F, None, None, None, None, 2, 2, 4, 1, F, F,
                                                                   F, P, P, P, 4, 0, 0.0, h, h, F, F, F, F, F, F,
                                                                   None),
                              lambda: lib.nrc_lightgcn_train_epoch(I, P, F, None, None, None, None, 2, 2, 4, 0, F, F,
                                                                   F, P, P, P, 4, 4, 0.0, h, h, F, F, F, F, F, F,
                                                                   None)],
    }
    # empty inputs succeed and launch nothing
    empty = {
        "l2_normalize_rows": lambda: lib.nrc_l2_normalize_rows(F, 0, 4, 1.0, F, None),
        "gather_rows_i32": lambda: lib.nrc_gather_rows_i32(P, 4, 1, I, 0, P, None),
        "sbpr_epoch_build": lambda: lib.nrc_sbpr_epoch_build(I, P, I, P, I, P, P, P, 4, 10, 0, 1, 1, 0, 2, 0, P, P, P,
                                                             P, F, None),
        "sbpr_grad": lambda: lib.nrc_sbpr_grad(F, F, F, 4, P, P, P, P, F, 0, 0, 0.0, F, F, F, P, P, 1, F, None),
        "csr_row_ids": lambda: lib.nrc_csr_row_ids(I, 0, P, None),
        "sample_negatives": lambda: lib.nrc_sample_negatives(I, P, P, 0, 1, 10, 1, 0, 0, P, None),
        "batch_randint_choice": lambda: lib.nrc_batch_randint_choice(10, I, 2, 0, 1, None, None, 1, 0, P, None),
        "lightgcn_bpr_grad": lambda: lib.nrc_lightgcn_bpr_grad(F, F, 2, 4, P, P, P, 0, 0.0, 1.0, F, F, F, None),
    }
    torch.cuda.synchronize()
    before = routes()
    for name, fns in calls.items():
        for k, fn in enumerate(fns):
            rc = fn()
            assert rc in (-1, -5), (name, k, rc)
            assert lib.nrc_last_error(), (name, k)
    for name, fn in empty.items():
        assert fn() == 0, name
    torch.cuda.synchronize()
    assert (buf == 7).all() and (fb == 7.0).all()
    assert routes() == before
    SEEN.add(("limits", 1))


REQUIRED = ({("sbpr_grad", k, c) for k in ("hinge", "square", "bpr") for c in (0, 1)}
            | {("sbpr_dim", d) for d in SBPR_DIMS} | {("sbpr_rounded", c) for c in (0, 1)}
            | {("sbpr_epoch", o, z) for o in OPTS for z in (False, True)} | {("sbpr_build", c) for c in (0, 1)}
            | {("l2", c) for c in (0, 1)} | {("l2_dim", d) for d in NORM_DIMS} | {("gather", c) for c in (0, 1)}
            | {("lightgcn_grad", e, c, z) for e in (True, False) for c in (0, 1) for z in (False, True)}
            | {("lightgcn_epoch", a, L, d) for a in ("norm", "gcmc") for L in (2, 6) for d in (32, 50)}
            | {("lightgcn_exact", d) for d in (32, 33)}
            | {("csr", c, rc, k) for c, rc, k in ((0, 0, 1), (0, 0, 2), (0, 0, 3), (0, 1, 3), (1, 0, 2), (0, 1, 3))}
            | {("csr", 1, 1, 3)} | {("row_ids", c) for c in (0, 1)}
            | {("split", m, c, rc, k) for m in ("ratio", "loo") for c, rc, k in ((0, 0, 1), (0, 0, 3), (0, 1, 3),
                                                                                  (1, 0, 2))}
            | {("negatives", k, c) for k in (1, 3) for c in (0, 1)} | {("choice_replace", c) for c in (0, 1)}
            | {("choice_noreplace", 1)} | {("limits", 1)})


@gpu
def test_every_route_was_seen(request):
    """Across this file the hook reported every route of these kernels.  Only meaningful when the whole file ran: a
    run of selected tests skips it."""
    here = {it.nodeid for it in request.session.items if it.fspath == request.node.fspath}
    if len(here) < 60:
        pytest.skip("only part of the file ran")
    assert REQUIRED <= SEEN, sorted(REQUIRED - SEEN, key=str)
