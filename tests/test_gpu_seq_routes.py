"""Every route the sequential kernels (csrc/sequential.cu: FPMC, TransRec, HRM, NPE) take from a shape, against float64.

The routes depend on the SM count: the FPMC, HRM and NPE gradient kernels cap their grid at 8 CTAs of 8 warps per SM
and loop beyond 64 * SMs samples; TransRec's caps at 128 CTAs and loops beyond 1024 samples, and sums g's gradient per
lane, per CTA and across CTAs; the query and relu passes cap at 16 CTAs of 256 threads per SM and loop beyond
4096 * SMs elements; the score kernels tile 8 rows by 256 items per CTA.  Every shape below is derived from the device's
SM count, one case on each side of each boundary; each test asserts the route it ran through nrc_seq_last_routes, and
the last test of the file checks that the whole file saw every route.

The reference is written here in float64 (`R`), independently of the fp32 restatements in seq_math.py and
seq_window_math.py; a CPU test checks it against torch.autograd.  Each value carries M, a first-order bound on the
rounding error of the fp32 chain that computes it.

Exact tests: tables of small integers times 2^-k, hinge or square loss (BPR at x = 0 by cloning the negative's rows
from the positive's, so g = -1/2; pointwise cross entropy at x = 0 only at power-of-two batches, since inv_b = fl(1/B)),
HRM mean pools only over power-of-two windows and max ties of 1, 2 or 4 rows, reg and lr powers of two.  With
`R.exact` set, every operation of the reference asserts that fp32 computes it exactly in any order (its operands are
multiples of 2^-k and every partial result stays below 2^24 such granules), so every route must equal float64 bit for
bit.  Hinge cases stay off the tie x = -1, where the kernel's gradient is 0.

Rounded tests: realistic values; each entry within C * 2^-24 * M of float64, C = 2."""
import ctypes

import numpy as np
import pytest
import scipy.sparse as sp
import torch

from oracle import tf_math

gpu = pytest.mark.gpu
U24 = 2.0 ** -24
C_BOUND = 2.0
SEEN = set()
OPTS = ("gd", "adam", "adagrad", "rmsprop", "momentum")
HYPER = {"gd": [2.0 ** -4], "adam": [2.0 ** -4, 0.9, 0.999, 1e-8], "adagrad": [2.0 ** -4],
         "rmsprop": [2.0 ** -4, 0.9, 0.5, 1e-10], "momentum": [2.0 ** -4, 0.5]}
DIMS = [1, 31, 32, 33, 63, 64, 65, 255, 256]
WINDOWS = [1, 2, 4, 63, 64]
POOLS = [(1, 1), (1, 0), (0, 1), (0, 0)]            # (session_max, pre_max)


def dev(a):
    return None if a is None else torch.from_numpy(np.ascontiguousarray(a)).cuda()


def host(t):
    return t.cpu().numpy()


def sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def routes():
    from neurec_b200 import ops
    return ops.seq_last_routes()


# ---------------------------------------------------------------------------------------------------------------
# the route predicates of the host code and the shapes on each side of them (pure functions of the SM count)
# ---------------------------------------------------------------------------------------------------------------
def grad_grid(batch, n_sms):
    """FPMC / HRM / NPE gradients: ceil(batch / 8) CTAs of 8 warps, at most 8 per SM."""
    return min((batch + 7) // 8, 8 * n_sms), (batch + 7) // 8 > 8 * n_sms


def transrec_grid(batch):
    return min((batch + 7) // 8, 128), (batch + 7) // 8 > 128


def elementwise_grid(total, n_sms):
    """Query and relu passes: one thread per element, at most 16 CTAs of 256 threads per SM."""
    return min((total + 255) // 256, 16 * n_sms), (total + 255) // 256 > 16 * n_sms


def grad_batches(n_sms):
    """1, both sides of 64 * SMs, and a multiple that repeats rows hundreds of times."""
    return [1, 64 * n_sms, 64 * n_sms + 1, 2 * 64 * n_sms + 7]


TRANSREC_BATCHES = [8, 9, 1024, 1025, 3 * 1024 + 7]
CE_BATCHES = [1, 256, 16384]                        # powers of two: inv_b = 1 / B exactly


def query_rows(dim, n_sms):
    """rows * dim on both sides of 4096 * SMs."""
    return [4096 * n_sms // dim, 4096 * n_sms // dim + 1]


@pytest.mark.parametrize("n_sms", [114, 132])
def test_route_shapes_straddle_every_boundary(n_sms):
    """CPU: the shapes derived from the SM count land on both sides of every route predicate (114: H100 PCIe,
    132: H100 SXM)."""
    assert [grad_grid(b, n_sms)[1] for b in grad_batches(n_sms)] == [False, False, True, True]
    assert grad_grid(64 * n_sms, n_sms)[0] == 8 * n_sms
    assert [transrec_grid(b) for b in TRANSREC_BATCHES] == [(1, False), (2, False), (128, False), (128, True),
                                                             (128, True)]
    assert [grad_grid(b, n_sms)[1] for b in CE_BATCHES] == [False, False, True]
    for dim in (64, 16, 256):
        r = query_rows(dim, n_sms)
        assert [elementwise_grid(x * dim, n_sms)[1] for x in r] == [False, True]
        assert elementwise_grid(r[0] * dim, n_sms)[0] == 16 * n_sms
    # the unrolled t < D loops hold one to eight elements per lane, with masked lanes on both sides of each step
    assert sorted({-(-d // 32) for d in DIMS}) == [1, 2, 3, 8]
    assert {d % 32 for d in DIMS} == {0, 1, 31}


# ---------------------------------------------------------------------------------------------------------------
# exactness precondition and bounds
# ---------------------------------------------------------------------------------------------------------------
def granule_bits(*arrays):
    """The smallest k with every value of every array a multiple of 2^-k (None when one is not dyadic)."""
    bits = 0
    for a in arrays:
        v = np.abs(np.asarray(a, np.float64)).ravel()
        v = v[(v != 0) & np.isfinite(v)]
        if v.size == 0:
            continue
        m, e = np.frexp(v)
        mant = (m * 2.0 ** 53).astype(np.int64)
        low = np.frexp((mant & -mant).astype(np.float64))[1] - 1      # index of the lowest set bit
        bits = max(bits, int((53 - e - low).max()))
    return bits


def assert_exact(operands, magnitude, what=""):
    """Every operand is a multiple of 2^-bits and every partial result (bounded by `magnitude`) stays below 2^24 such
    granules: fp32 represents each exactly, in any summation order."""
    bits = granule_bits(*operands)
    assert bits < 150 and (np.asarray(magnitude, np.float64) * 2.0 ** bits < 2.0 ** 24).all(), \
        (what, bits, float(np.max(magnitude)))


def assert_within(got, want, M, what, C=C_BOUND):
    err = np.abs(np.asarray(got, np.float64) - want)
    bound = C * U24 * np.asarray(M, np.float64)
    assert (err <= bound).all(), (what, float((err - bound).max()), float(np.max(M)))


def dyadic(rs, shape, lo=-1, hi=1, k=2):
    return (rs.randint(lo, hi + 1, shape) / 2.0 ** k).astype(np.float32)


def distinct_columns(rs, n, dim, k=5):
    """Every column a permutation of n distinct multiples of 2^-k: two rows tie in an element only when they are the
    same row, so the tie count of a max pool is the multiplicity of the maximal row in the window."""
    return np.stack([(rs.permutation(n) - n // 2) / 2.0 ** k for _ in range(dim)], 1).astype(np.float32)


class R:
    """A float64 value v of an fp32 chain with m, a first-order bound on that chain's rounding error in units of
    2^-24 (|fp32 - v| <= 2^-24 * m to first order).  While R.exact is set, every operation also asserts that fp32
    computes it exactly (assert_exact)."""
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

    def __radd__(self, o):
        return self + o

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

    def __rmul__(self, o):
        return self * o

    def __truediv__(self, k):
        """Division by a (per-row) count, correctly rounded."""
        k = np.asarray(k, np.float64)
        v = self.v / k
        if R.exact:
            assert_exact([v], np.abs(v), "div")
        return R(v, self.m / k + np.abs(v))

    def sum(self, axis):
        """A sum in any order (warp shuffles, atomics)."""
        n = self.v.shape[axis]
        mag = np.abs(self.v).sum(axis)
        if R.exact:
            assert_exact([self.v], mag, "sum")
        return R(self.v.sum(axis), self.m.sum(axis) + max(n - 1, 0) * mag)

    def sqrt(self):
        v = np.sqrt(self.v)
        return R(v, np.where(v > 0, self.m / (2 * np.where(v > 0, v, 1)), np.sqrt(self.m)) + v)


def cat(parts, axis):
    return R(np.concatenate([p.v for p in parts], axis), np.concatenate([np.broadcast_to(p.m, p.v.shape)
                                                                         for p in parts], axis))


def rmax(a, b):
    b = R.of(b)
    return R(np.maximum(a.v, b.v), np.maximum(np.broadcast_to(a.m, a.v.shape), b.m))


def where(mask, a, b=0.0):
    a, b = R.of(a), R.of(b)
    return R(np.where(mask, a.v, b.v), np.where(mask, a.m, b.m))


def scatter(n_rows, pairs):
    """Rows gathered by ids and added into a zeroed accumulator by atomics: sum of (ids, contributions [k, D]) over
    `pairs`; each of a row's count adds rounds at most its partial sum."""
    ids = np.concatenate([np.asarray(i).ravel() for i, _ in pairs])
    d = cat([c for _, c in pairs], 0)
    S = sp.csr_matrix((np.ones(len(ids)), (ids, np.arange(len(ids)))), shape=(n_rows, len(ids)))
    mag = S @ np.abs(d.v)
    if R.exact:
        assert_exact([d.v], mag, "scatter")
    cnt = np.bincount(ids, minlength=n_rows).astype(np.float64).reshape((-1,) + (1,) * (d.v.ndim - 1))
    return R(S @ d.v, S @ np.broadcast_to(d.m, d.v.shape) + cnt * mag)


def touched(n, *ids):
    t = np.zeros(n, bool)
    for i in ids:
        t[np.asarray(i).ravel()] = True
    return t


# ---------------------------------------------------------------------------------------------------------------
# the float64 reference: losses and the four models
# ---------------------------------------------------------------------------------------------------------------
def pair_loss(kind, x):
    """learner.pairwise_loss -> (per-sample loss, dl/dx)."""
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


def point_loss(kind, x, z):
    """learner.pointwise_loss -> (per-sample loss, dl/dx); cross entropy is the batch mean."""
    z = np.asarray(z, np.float64)
    if kind == "square":
        t = R(z) - x
        return t * t, -2.0 * t
    if kind == "cross_entropy":
        B = len(z)
        if R.exact:
            assert (x.v == 0).all() and B & (B - 1) == 0, "exact cross entropy sits at x = 0 with B a power of two"
        e = np.exp(-np.abs(x.v))
        s = np.where(x.v >= 0, 1.0 / (1.0 + e), e / (1.0 + e))
        l = (np.maximum(x.v, 0) - x.v * z + np.log1p(e)) / B
        g = (s - z) / B
        Ml = (5 * (np.maximum(x.v, 0) + np.abs(x.v * z) + np.log1p(e)) + np.abs(s - z) * x.m) / B + np.abs(l)
        Mg = (5 * (np.abs(s) + np.abs(s - z)) + 0.25 * x.m) / B + 2 * np.abs(g)
        return R(l, Ml), R(g, Mg)
    raise ValueError(kind)


def with_reg(l, reg, sq, kind):
    """Per-sample loss l + reg / 2 * sq; BPR and cross entropy are never exact, so their loss is only bounded."""
    saved = R.exact
    R.exact = saved and kind not in ("bpr", "cross_entropy")
    try:
        return (l + (reg * 0.5) * sq) if reg else l
    finally:
        R.exact = saved


def batch_loss(lo, kind, extra=None):
    saved = R.exact
    R.exact = saved and kind not in ("bpr", "cross_entropy")
    try:
        return lo.sum(0) if extra is None else lo.sum(0) + extra
    finally:
        R.exact = saved


def fpmc_ref(T, users, recent, items, third, pairwise, kind, reg):
    UI, IU, IL, LI = T
    a, ui, li, r = R(UI[users]), R(IU[items]), R(IL[items]), R(LI[recent])
    x = cat([a * ui, li * r], 1).sum(1)
    sq = [a * a, ui * ui, li * li, r * r]
    if pairwise:
        uj, lj = R(IU[third]), R(IL[third])
        x = x - cat([a * uj, lj * r], 1).sum(1)
        sq += [uj * uj, lj * lj]
        l, c = pair_loss(kind, x)
    else:
        l, c = point_loss(kind, x, third)
    lo = with_reg(l, reg, cat(sq, 1).sum(1), kind)
    c = c[:, None]
    nu, ni = UI.shape[0], IU.shape[0]
    if pairwise:
        g = [scatter(nu, [(users, c * (ui - uj) + reg * a)]),
             scatter(ni, [(items, c * a + reg * ui), (third, -c * a + reg * uj)]),
             scatter(ni, [(items, c * r + reg * li), (third, -c * r + reg * lj)]),
             scatter(ni, [(recent, c * (li - lj) + reg * r)])]
        t = [touched(nu, users), touched(ni, items, third), touched(ni, recent)]
    else:
        g = [scatter(nu, [(users, c * ui + reg * a)]), scatter(ni, [(items, c * a + reg * ui)]),
             scatter(ni, [(items, c * r + reg * li)]), scatter(ni, [(recent, c * li + reg * r)])]
        t = [touched(nu, users), touched(ni, items), touched(ni, recent)]
    return batch_loss(lo, kind), g, t


def transrec_ref(T, users, recent, items, third, pairwise, kind, reg):
    P, Q, Bv, G = T
    p, r, qi, G_ = R(P[users]), R(Q[recent]), R(Q[items]), R(G.reshape(1, -1))
    xv = (p + G_) + r
    vi = xv - qi
    bi = R(Bv[items])
    x = bi - (vi * vi).sum(1)
    sq = [p * p, r * r, qi * qi]
    bsq = bi * bi
    if pairwise:
        qj, bj = R(Q[third]), R(Bv[third])
        vj = xv - qj
        x = x - (bj - (vj * vj).sum(1))
        sq += [qj * qj]
        bsq = bsq + bj * bj
        l, c = pair_loss(kind, x)
    else:
        l, c = point_loss(kind, x, third)
    lo = with_reg(l, reg, cat(sq, 1).sum(1) + bsq, kind)
    c1 = c[:, None]
    c2 = 2.0 * c1
    nu, ni = P.shape[0], Q.shape[0]
    e = -c2 * (vi - vj) if pairwise else -c2 * vi
    gQ = [(recent, e + reg * r), (items, c2 * vi + reg * qi)]
    gB = [(items, c + reg * bi)]
    if pairwise:
        gQ.append((third, -c2 * vj + reg * qj))
        gB.append((third, -c + reg * bj))
    gG = e.sum(0) + reg * R(G)
    total = batch_loss(lo, kind, (reg * 0.5) * (R(G) * R(G)).sum(0) if reg else None)
    g = [scatter(nu, [(users, e + reg * p)]), scatter(ni, gQ), scatter(ni, gB), gG]
    t = [touched(nu, users), touched(ni, recent, items, *([third] if pairwise else [])),
         touched(ni, items, *([third] if pairwise else []))]
    return total, g, t


def hrm_ref(T, users, recent, items, labels, smax, pmax, kind, reg):
    P, E = T
    B, L = recent.shape
    p, e, W = R(P[users]), R(E[items]), R(E[recent])
    if smax:
        s = R(W.v.max(1))
        cnt = (W.v == s.v[:, None, :]).sum(1)
    else:
        s = W.sum(1) / L
    if pmax:
        if not R.exact:            # no max decision may sit within rounding of a tie it does not make exactly
            assert ((p.v == s.v) | (np.abs(p.v - s.v) > 4 * U24 * s.m)).all()
        h = rmax(p, s)
    else:
        h = (p + s) / 2
    x = (h * e).sum(1)
    l, c = point_loss(kind, x, labels)
    WW = W * W
    lo = with_reg(l, reg, cat([R(WW.v.reshape(B, -1), WW.m.reshape(B, -1)), p * p + e * e], 1).sum(1), kind)
    c1 = c[:, None]
    dh = c1 * e
    if pmax:
        share = np.where(p.v == s.v, 0.5, 1.0)
        dp = where(p.v == h.v, R(share) * dh)
        ds = where(s.v == h.v, R(share) * dh)
    else:
        dp = dh / 2
        ds = dh / 2
    if smax:
        inv = R(1.0 / cnt, np.where(cnt & (cnt - 1) == 0, 0.0, 1.0 / cnt))      # fl(1 / cnt)
        dv = where(W.v == s.v[:, None, :], inv[:, None, :] * ds[:, None, :])
    else:
        dv = ds[:, None, :] / L
    dW = dv + reg * W
    D = P.shape[1]
    g = [scatter(P.shape[0], [(users, dp + reg * p)]),
         scatter(E.shape[0], [(items, c1 * h + reg * e), (recent.ravel(), R(dW.v.reshape(-1, D),
                                                                            dW.m.reshape(-1, D)))])]
    t = [touched(P.shape[0], users), touched(E.shape[0], items, recent)]
    return batch_loss(lo, kind), g, t


def npe_ref(T, users, recent, items, labels, kind, reg):
    UI, IU, IL = T
    B, L = recent.shape
    a, q, W = R(UI[users]), R(IU[items]), R(IL[recent])
    ctx = W.sum(1)
    if not R.exact:                # no relu gate may sit within rounding of 0 unless it is exactly 0
        assert ((ctx.v == 0) | (np.abs(ctx.v) > 4 * U24 * ctx.m)).all()
    ra, rq, rc = rmax(a, 0.0), rmax(q, 0.0), rmax(ctx, 0.0)
    x = (ra * rq + rq * rc).sum(1)
    l, c = point_loss(kind, x, labels)
    WW = W * W
    lo = with_reg(l, reg, cat([R(WW.v.reshape(B, -1), WW.m.reshape(B, -1)), a * a + q * q], 1).sum(1), kind)
    c1 = c[:, None]
    dctx = where(ctx.v > 0, c1 * rq)
    dW = dctx[:, None, :] + reg * W
    D = UI.shape[1]
    g = [scatter(UI.shape[0], [(users, where(a.v > 0, c1 * rq) + reg * a)]),
         scatter(IU.shape[0], [(items, where(q.v > 0, c1 * ra + c1 * rc) + reg * q)]),
         scatter(IL.shape[0], [(recent.ravel(), R(dW.v.reshape(-1, D), dW.m.reshape(-1, D)))])]
    t = [touched(UI.shape[0], users), touched(IU.shape[0], items), touched(IL.shape[0], recent)]
    return batch_loss(lo, kind), g, t


# ---------------------------------------------------------------------------------------------------------------
# the reference against torch.autograd (CPU)
# ---------------------------------------------------------------------------------------------------------------
def torch_loss(model, t, users, recent, items, third, pairwise, kind, reg, smax=None, pmax=None):
    F = torch.nn.functional
    T = lambda a: torch.as_tensor(np.asarray(a))
    u, l, i = T(users).long(), T(recent).long(), T(items).long()
    pair = {"bpr": lambda x: -F.logsigmoid(x), "hinge": lambda x: F.relu(x + 1), "square": lambda x: (1 - x) ** 2}

    def point(x):
        z = T(third).double()
        if kind == "cross_entropy":
            return F.binary_cross_entropy_with_logits(x, z, reduction="mean")
        return ((z - x) ** 2).sum()

    rows = []
    if model == "fpmc":
        UI, IU, IL, LI = t
        x = (UI[u] * IU[i]).sum(1) + (IL[i] * LI[l]).sum(1)
        rows = [UI[u], IU[i], IL[i], LI[l]]
        if pairwise:
            j = T(third).long()
            x = x - (UI[u] * IU[j]).sum(1) - (IL[j] * LI[l]).sum(1)
            rows += [IU[j], IL[j]]
    elif model == "transrec":
        P, Q, Bv, G = t
        d = lambda q, b: b - (((P[u] + G) + Q[l] - q) ** 2).sum(1)
        x = d(Q[i], Bv[i])
        rows = [P[u], Q[l], Q[i], Bv[i], G]
        if pairwise:
            j = T(third).long()
            x = x - d(Q[j], Bv[j])
            rows += [Q[j], Bv[j]]
    elif model == "hrm":
        P, E = t
        W = E[l]
        s = W.amax(1) if smax else W.mean(1)                 # amax splits the gradient evenly over ties, as TF
        h = torch.stack([P[u], s]).amax(0) if pmax else (P[u] + s) / 2
        x = (h * E[i]).sum(1)
        rows = [P[u], E[i], W]
    else:
        UI, IU, IL = t
        c = IL[l].sum(1)
        x = (F.relu(UI[u]) * F.relu(IU[i]) + F.relu(IU[i]) * F.relu(c)).sum(1)
        rows = [UI[u], IU[i], IL[l]]
    loss = pair[kind](x).sum() if pairwise else point(x)
    return loss + reg * 0.5 * sum((r ** 2).sum() for r in rows)


def ref_call(model, T, users, recent, items, third, pairwise, kind, reg, smax=None, pmax=None):
    if model == "fpmc":
        return fpmc_ref(T, users, recent, items, third, pairwise, kind, reg)
    if model == "transrec":
        return transrec_ref(T, users, recent, items, third, pairwise, kind, reg)
    if model == "hrm":
        return hrm_ref(T, users, recent, items, third, smax, pmax, kind, reg)
    return npe_ref(T, users, recent, items, third, kind, reg)


AUTOGRAD_CASES = ([("fpmc", p, k, None, None) for p, k in ((1, "bpr"), (1, "hinge"), (1, "square"),
                                                           (0, "cross_entropy"), (0, "square"))]
                  + [("transrec", p, k, None, None) for p, k in ((1, "bpr"), (1, "hinge"), (1, "square"),
                                                               (0, "cross_entropy"), (0, "square"))]
                  + [("hrm", 0, k, sm, pm) for k in ("cross_entropy", "square") for sm, pm in POOLS]
                  + [("npe", 0, k, None, None) for k in ("cross_entropy", "square")])


@pytest.mark.parametrize("model,pairwise,kind,smax,pmax", AUTOGRAD_CASES)
@pytest.mark.parametrize("ties", [False, True])
def test_reference_matches_autograd(model, pairwise, kind, smax, pmax, ties):
    """CPU: the float64 reference's loss and gradients equal torch.autograd's in float64, on small cases with repeated
    users, items and window ids.  With `ties`, integer tables force max ties of every count, P_u == s, and exact
    zeros at relu's inputs."""
    rs = np.random.RandomState(len(model) * 7 + pairwise + len(kind))
    nu, ni, D, B = 7, 11, 5, 13
    L = 4 if model in ("hrm", "npe") else None
    shapes = {"fpmc": [(nu, D), (ni, D), (ni, D), (ni, D)], "transrec": [(nu, D), (ni, D), (ni,), (D,)],
              "hrm": [(nu, D), (ni, D)], "npe": [(nu, D), (ni, D), (ni, D)]}[model]
    T = [(rs.randint(-2, 3, s) if ties else rs.randn(*s)).astype(np.float32) for s in shapes]
    users, items = rs.randint(0, nu, B), rs.randint(0, ni, B)
    recent = rs.randint(0, ni, (B, L) if L else B)
    third = rs.randint(0, ni, B) if pairwise else rs.randint(0, 2, B).astype(np.float32)
    if not ties:
        T = [a * 0.3 for a in T]
    if ties and model == "hrm":
        T[0][:3] = T[1][recent[:3]].max(1) if smax else T[0][:3]        # P_u == s in every element
        users[:3] = [0, 1, 2]
    if ties and model == "npe":
        recent[0] = [1, 2, 1, 2]
        T[2][2] = -T[2][1]                                              # a window summing to exactly 0
    reg = 0.25
    want_l, want_g, _ = ref_call(model, T, users, recent, items, third, pairwise, kind, reg, smax, pmax)
    t = [torch.tensor(a, dtype=torch.float64, requires_grad=True) for a in T]
    loss = torch_loss(model, t, users, recent, items, third, pairwise, kind, reg, smax, pmax)
    loss.backward()
    assert abs(loss.item() - float(want_l.v)) <= 1e-12 * max(1.0, abs(loss.item()))
    for k, (a, w) in enumerate(zip(t, want_g)):
        np.testing.assert_allclose(w.v, a.grad.numpy(), rtol=1e-12, atol=1e-12, err_msg=str(k))


# ---------------------------------------------------------------------------------------------------------------
# the gradient kernels, exact
# ---------------------------------------------------------------------------------------------------------------
MODES = {"fpmc": [(1, "hinge"), (1, "square"), (1, "bpr"), (0, "square"), (0, "cross_entropy")],
         "transrec": [(1, "hinge"), (1, "square"), (1, "bpr"), (0, "square")],
         "hrm": [(0, "square")], "npe": [(0, "square")]}


def sparse_dyadic(rs, shape, density=0.3, k=2):
    """Small integers times 2^-k, most of them 0: scores and gradient sums stay far below 2^24 granules."""
    return dyadic(rs, shape, -1, 1, k) * (rs.rand(*shape) < density)


def grad_case(model, rs, B, D, pairwise, kind, L=2, heavy=False, smax=None, pmax=None):
    """Tables, ids and labels of one exact batch; repeated users and items, window rows (or the recent item) that are
    also the sample's next item."""
    nu, ni = (37, 216) if heavy else (B + 5, 2 * B + 6)
    if model == "fpmc":
        T = [sparse_dyadic(rs, (nu, D))] + [sparse_dyadic(rs, (ni, D)) for _ in range(3)]
        if kind == "cross_entropy":            # <UI_u, IU_i> = <IL_i, LI_l> = 0: x = 0
            h = max(1, D // 2)
            T[0][:, h:] = 0; T[1][:, :h] = 0; T[2][:, h:] = 0; T[3][:, :h] = 0
    elif model == "transrec":
        T = [sparse_dyadic(rs, (nu, D), 0.1), sparse_dyadic(rs, (ni, D), 0.1), dyadic(rs, (ni,)),
             sparse_dyadic(rs, (D,), 0.1)]
    elif model == "hrm":
        T = [sparse_dyadic(rs, (nu, D), 0.1), sparse_dyadic(rs, (ni, D), 0.1)]
    else:
        T = [sparse_dyadic(rs, (nu, D)), sparse_dyadic(rs, (ni, D)), sparse_dyadic(rs, (ni, D))]
    users = rs.randint(0, nu, B).astype(np.int32)
    items = rs.randint(0, ni, B).astype(np.int32)
    windowed = model in ("hrm", "npe")
    recent = rs.randint(0, ni, (B, L) if windowed else B).astype(np.int32)
    if B > 1:
        users[1] = users[0]
        sel = slice(0, B, 8)
        if windowed:
            recent[sel, 0] = items[sel]
        else:
            recent[sel] = items[sel]
    if pairwise:
        third = rs.randint(0, ni, B).astype(np.int32)
        if kind == "bpr":                      # the negative's rows are the positive's: x = 0, g = -1/2
            items &= ~1
            third = items + 1
            for t in T[1:3]:                   # IU, IL (FPMC) or Q, b (TransRec)
                t[1::2] = t[0::2]
        if kind == "hinge":
            for _ in range(100):
                x = score64(model, T, users, recent, items, third)
                if not (x == -1.0).any():
                    break
                third[x == -1.0] = rs.randint(0, ni, int((x == -1.0).sum()))
    else:
        third = rs.randint(0, 2, B).astype(np.float32)
        if windowed:                           # labels at the score except every seventh: the loss sum stays exact
            third = score_window64(model, T, users, recent, items, smax, pmax).astype(np.float32)
            third[::7] += rs.randint(0, 2, len(third[::7])) * 2 - 1
    return T, users, recent, items, third


def score64(model, T, users, recent, items, third=None):
    """FPMC / TransRec scores x_i, or the differences x_i - x_j, in float64."""
    T = [a.astype(np.float64) for a in T]
    if model == "fpmc":
        UI, IU, IL, LI = T
        f = lambda i: (UI[users] * IU[i]).sum(1) + (IL[i] * LI[recent]).sum(1)
    else:
        P, Q, Bv, G = T
        f = lambda i: Bv[i] - (((P[users] + G) + Q[recent] - Q[i]) ** 2).sum(1)
    return f(items) if third is None else f(items) - f(third)


TOUCH_SIZES = {"fpmc": (0, 1, 1), "transrec": (0, 1, 1), "hrm": (0, 1), "npe": (0, 1, 1)}


def device_grad(model, T, users, recent, items, third, pairwise, kind, reg, smax=None, pmax=None, stamp=9):
    """One gradient call into zeroed accumulators and touched arrays filled with 5 -> (loss, grads, touched) on the
    host, and the route record of the call."""
    from neurec_b200 import ops
    dT = [dev(a) for a in T]
    g = [torch.zeros_like(t) for t in dT]
    n = (T[0].shape[0], T[1].shape[0])
    tch = [torch.full((n[k],), 5, dtype=torch.int32, device="cuda") for k in TOUCH_SIZES[model]]
    lo = torch.zeros(1, device="cuda")
    ids = (dev(users), dev(recent), dev(items), dev(third))
    if model == "fpmc":
        ops.fpmc_grad(*dT, *ids, pairwise, kind, reg, *g, *tch, stamp, lo)
    elif model == "transrec":
        ops.transrec_grad(*dT, *ids, pairwise, kind, reg, *g, *tch, stamp, ops.transrec_work(T[0].shape[1]), lo)
    elif model == "hrm":
        ops.hrm_grad(*dT, *ids, pmax, smax, kind, reg, *g, *tch, stamp, lo)
    else:
        ops.npe_grad(*dT, *ids, kind, reg, *g, *tch, stamp, lo)
    return float(lo), [host(a) for a in g], [host(t) for t in tch], routes()[model + "_grad"]


def check_grad(model, T, users, recent, items, third, pairwise, kind, reg, smax=None, pmax=None, exact=True):
    """Kernel against the float64 reference: gradients and stamps bit for bit (exact) or within the bound, the batch
    loss bit for bit where it is dyadic, else within its bound.  Returns the route record."""
    R.exact = exact
    try:
        want_l, want_g, want_t = ref_call(model, T, users, recent, items, third, pairwise, kind, reg, smax, pmax)
    finally:
        R.exact = False
    lo, g, t, r = device_grad(model, T, users, recent, items, third, pairwise, kind, reg, smax, pmax)
    for k, (a, w) in enumerate(zip(g, want_g)):
        if exact:
            a = a.reshape(w.v.shape)
            assert np.array_equal(a, w.v), (model, k, float(np.abs(a - w.v).max()))
        else:
            assert_within(a.reshape(w.v.shape), w.v, w.m, (model, k))
    for a, w in zip(t, want_t):
        assert np.array_equal(a, np.where(w, 9, 5))
    if exact and kind not in ("bpr", "cross_entropy"):
        assert lo == float(want_l.v), (lo, float(want_l.v))
    else:
        assert_within(lo, want_l.v, want_l.m, "loss")
    return r


@gpu
@pytest.mark.parametrize("dim", DIMS)
@pytest.mark.parametrize("model,pairwise,kind,smax,pmax",
                         [(m, p, k, None, None) for m in ("fpmc", "transrec", "npe") for p, k in MODES[m]]
                         + [("hrm", 0, "square", sm, pm) for sm, pm in POOLS])
def test_grad_exact(model, pairwise, kind, smax, pmax, dim):
    """Batches on both sides of each grid cap and a heavy-duplicate multiple (TransRec: 8, 9, 1024, 1025, 3079; cross
    entropy at 1, 256 and 16384), windows of 2: gradients, g's gradient, stamps and the loss bit for bit."""
    n_sms = sms()
    rs = np.random.RandomState(dim * 13 + len(model) + 3 * pairwise + len(kind))
    if model == "transrec":
        batches = TRANSREC_BATCHES
    elif kind == "cross_entropy":
        batches = CE_BATCHES
    else:
        batches = grad_batches(n_sms)
    reg = 0.0 if kind == "hinge" else 2.0 ** -3
    for bi, B in enumerate(batches):
        heavy = bi == len(batches) - 1 and kind != "cross_entropy"
        case = grad_case(model, rs, B, dim, pairwise, kind, heavy=heavy, smax=smax, pmax=pmax)
        r = check_grad(model, *case, pairwise, kind, reg, smax, pmax)
        grid, capped = transrec_grid(B) if model == "transrec" else grad_grid(B, n_sms)
        assert r["grid_x"] == grid and r["capped"] == capped and r["pairwise"] == pairwise
        assert r["window"] == (2 if model in ("hrm", "npe") else -1)
        assert (r["session_max"], r["pre_max"]) == ((smax, pmax) if model == "hrm" else (-1, -1))
        SEEN.add(("grad", model, pairwise, int(capped)))
        if model == "transrec":
            SEEN.add(("transrec_ctas", B))
    SEEN.add(("grad_loss", model, kind) if model != "hrm" else ("hrm_pools", smax, pmax))


def window_of(rs, L, ids):
    """A window of L ids in which every id appears 1, 2 or 4 times."""
    out, fresh = [], iter(rs.permutation(ids))
    while len(out) < L:
        fits = [k for k in (1, 2, 4) if len(out) + k <= L]
        out += [next(fresh)] * fits[rs.randint(len(fits))]
    return rs.permutation(out)


def score_window64(model, T, users, recent, items, smax=None, pmax=None):
    """HRM / NPE scores in float64."""
    T = [a.astype(np.float64) for a in T]
    if model == "hrm":
        W = T[1][recent]
        s = W.max(1) if smax else W.mean(1)
        h = np.maximum(T[0][users], s) if pmax else (T[0][users] + s) / 2
        return (h * T[1][items]).sum(1)
    r = lambda a: np.maximum(a, 0)
    return (r(T[0][users]) * r(T[1][items]) + r(T[1][items]) * r(T[2][recent].sum(1))).sum(1)


@gpu
# a mean over a window that is not a power of two is not exact: the rounded tests take HRM's mean at L = 63
@pytest.mark.parametrize("model,smax,pmax,L", [("hrm", sm, pm, L) for sm, pm in POOLS for L in WINDOWS
                                               if sm or L & (L - 1) == 0] + [("npe", None, None, L) for L in WINDOWS])
def test_grad_windows_exact(model, smax, pmax, L):
    """Windows of 1, 2, 4, 63 and 64 at batches 1, 64 * SMs and 64 * SMs + 1.  HRM: tables whose columns hold distinct
    values, so max ties come only from rows repeated 1, 2 or 4 times in a window; users whose row equals the window's
    maximum (P_u == s, the 1/2 share).  NPE: windows that sum to exactly 0 at relu.  Labels equal the score except on
    every seventh sample, so most samples pass only their reg terms and the long accumulations stay exact."""
    n_sms = sms()
    rs = np.random.RandomState(L * 31 + (smax or 0) * 2 + (pmax or 0))
    for B in (1, 64 * n_sms, 64 * n_sms + 1):
        D = 9
        nu, ni = 40, 80
        users = rs.randint(4, nu, B).astype(np.int32)
        recent = np.stack([window_of(rs, L, np.arange(ni)) for _ in range(min(B, 64))])[rs.randint(0, min(B, 64), B)]
        recent = recent.astype(np.int32)
        items = rs.randint(0, ni, B).astype(np.int32)
        items[::5] = recent[::5, 0]
        labels = rs.randint(0, 2, B).astype(np.float32)
        if model == "hrm":
            T = [dyadic(rs, (nu, D), -8, 8, 4), distinct_columns(rs, ni, D, 4) if smax else dyadic(rs, (ni, D))]
            k = max(1, B // 3)                                # users 0-3 over one window, their rows its pool
            recent[:k] = window_of(rs, L, np.arange(ni))
            users[:k] = rs.randint(0, 4, k)
            W0 = T[1][recent[0]]
            T[0][:4] = W0.max(0) if smax else W0.mean(0)
        else:
            T = [dyadic(rs, (nu, D)), dyadic(rs, (ni, D)), dyadic(rs, (ni, D))]
            T[2][1::2] = -T[2][0::2]                          # row 2k + 1 cancels row 2k
            if L % 2 == 0:
                k = max(1, B // 2)
                pairs = rs.randint(0, ni // 2, (k, L // 2)) * 2
                recent[:k] = np.stack([pairs, pairs + 1], 2).reshape(k, L)
        x = score_window64(model, T, users, recent, items, smax, pmax)
        labels = x.astype(np.float32)
        assert (labels == x).all()
        labels[::7] += 1
        # HRM without reg: its loss sums reg * |E[w]|^2 over 64 distinct-valued rows per sample, past 2^24 granules
        r = check_grad(model, T, users, recent, items, labels, 0, "square", 0.0 if model == "hrm" else 2.0 ** -3,
                       smax, pmax)
        grid, capped = grad_grid(B, n_sms)
        assert r["window"] == L and r["grid_x"] == grid and r["capped"] == capped
        if model == "hrm" and smax:
            W = T[1][recent]
            s = W.max(1)
            cnt = (W == s[:, None, :]).sum(1)
            assert set(np.unique(cnt)) <= {1, 2, 4}
        if model == "hrm":
            W0 = T[1][recent[0]]
            assert (T[0][users[0]] == (W0.max(0) if smax else W0.mean(0))).all()
        if model == "npe" and L % 2 == 0:
            assert (T[2][recent].sum(1) == 0).all(1).any()
        SEEN.add(("window", model, L, int(capped)))


# ---------------------------------------------------------------------------------------------------------------
# the gradient kernels, rounded
# ---------------------------------------------------------------------------------------------------------------
ROUNDED = [("fpmc", 1, "bpr", None, None, 1), ("fpmc", 0, "cross_entropy", None, None, 1),
           ("transrec", 1, "bpr", None, None, 1), ("transrec", 0, "cross_entropy", None, None, 1),
           ("hrm", 0, "cross_entropy", 0, 0, 3), ("hrm", 0, "cross_entropy", 0, 0, 63),
           ("hrm", 0, "cross_entropy", 1, 1, 4), ("hrm", 0, "square", 1, 0, 4),
           ("npe", 0, "cross_entropy", None, None, 3)]


@gpu
@pytest.mark.parametrize("model,pairwise,kind,smax,pmax,L", ROUNDED)
def test_grad_rounded(model, pairwise, kind, smax, pmax, L):
    """Realistic values past 64 * SMs samples (TransRec: past 1024): BPR and cross entropy with |x| past 80, HRM's mean
    over 3 and 63 items, max ties of three rows (fl(1/3) * grad): every gradient entry and the loss within the
    first-order bound of the float64 chain."""
    n_sms = sms()
    rs = np.random.RandomState(len(model) + 10 * L + pairwise)
    B = 1025 if model == "transrec" else 64 * n_sms + 1
    D = 16 if L > 4 else 64
    nu, ni = 3000, 4000
    scale = lambda n: rs.choice([0.05, 4.0], (n, 1))
    if model == "fpmc":
        T = [(rs.randn(nu, D) * scale(nu))] + [rs.randn(ni, D) * scale(ni) for _ in range(3)]
    elif model == "transrec":
        T = [rs.randn(nu, D) * scale(nu), rs.randn(ni, D) * scale(ni), rs.randn(ni) * 20, rs.randn(D) * 0.3]
    elif model == "hrm":
        T = [rs.randn(nu, D) * scale(nu), rs.randn(ni, D) * scale(ni)]
    else:
        T = [rs.randn(nu, D) * scale(nu), rs.randn(ni, D) * scale(ni), rs.randn(ni, D) * scale(ni)]
    T = [a.astype(np.float32) for a in T]
    users, items = rs.randint(0, nu, B).astype(np.int32), rs.randint(0, ni, B).astype(np.int32)
    if model in ("hrm", "npe"):
        recent = rs.randint(0, ni, (B, L)).astype(np.int32)
        if smax and L == 4:
            recent[:, 1:3] = recent[:, :1]                 # one row three times: max ties of count 3
        x = score_window64(model, T, users, recent, items, smax, pmax)
    else:
        recent = rs.randint(0, ni, B).astype(np.int32)
    third = rs.randint(0, ni, B).astype(np.int32) if pairwise else rs.randint(0, 2, B).astype(np.float32)
    if model in ("fpmc", "transrec"):
        x = score64(model, T, users, recent, items, third if pairwise else None)
    if kind != "square":
        assert np.abs(x).max() > 80
    r = check_grad(model, T, users, recent, items, third, pairwise, kind, float(np.float32(1e-3)), smax, pmax,
                   exact=False)
    grid, capped = transrec_grid(B) if model == "transrec" else grad_grid(B, n_sms)
    assert r["capped"] == capped == 1 and r["grid_x"] == grid
    if model == "hrm" and smax:
        W = T[1][recent]
        assert 3 in (W == W.max(1, keepdims=True)).sum(1)
    SEEN.add(("rounded", model, kind, L))


# ---------------------------------------------------------------------------------------------------------------
# the score kernels
# ---------------------------------------------------------------------------------------------------------------
def scores_ref(model, T, users, recent):
    if model == "fpmc":
        UI, IU, IL, LI = [R(a) for a in T]
        a, l = UI[users][:, None, :], LI[recent][:, None, :]
        return cat([a * IU.v[None], R(IL.v[None]) * l], 2).sum(2), None
    P, Q, Bv, G = T
    xq = (R(P[users]) + R(G[None])) + R(Q[recent])
    d = R(xq.v[:, None, :], xq.m[:, None, :]) - R(Q[None])
    acc = (d * d).sum(2)
    saved, R.exact = R.exact, False            # the distance is only bounded; the exact test rounds it as fp32 does
    try:
        return R(Bv[None]) - acc.sqrt(), acc
    finally:
        R.exact = saved


@gpu
@pytest.mark.parametrize("dim", [1, 32, 256])
@pytest.mark.parametrize("model", ["fpmc", "transrec"])
def test_scores(model, dim):
    """Rows 1, 7, 8, 9, 41 (groups of 8 with a partial last one) by items 1, 255, 256, 257 (tiles of 256 with a partial
    last one), widths up to 256 (shared memory full): bit for bit on dyadic tables (TransRec: the distance sum is exact,
    then fp32's correctly rounded sqrt and subtraction), within the bound on realistic values."""
    from neurec_b200 import ops
    rs = np.random.RandomState(dim + len(model))
    nu = 50
    for rows in (1, 7, 8, 9, 41):
        for ni in (1, 255, 256, 257):
            for exact in (True, False):
                if exact:
                    T = ([dyadic(rs, (nu, dim))] + [dyadic(rs, (ni, dim)) for _ in range(3)] if model == "fpmc" else
                         [dyadic(rs, (nu, dim)), dyadic(rs, (ni, dim)), dyadic(rs, (ni,), -8, 8), dyadic(rs, (dim,))])
                else:
                    T = ([rs.randn(nu, dim)] + [rs.randn(ni, dim) for _ in range(3)] if model == "fpmc" else
                         [rs.randn(nu, dim), rs.randn(ni, dim), rs.randn(ni), rs.randn(dim)])
                    T = [a.astype(np.float32) for a in T]
                users = rs.randint(0, nu, rows).astype(np.int32)
                recent = rs.randint(0, ni, rows).astype(np.int32)
                R.exact = exact
                try:
                    want, acc = scores_ref(model, T, users, recent)
                finally:
                    R.exact = False
                fn = ops.fpmc_scores if model == "fpmc" else ops.transrec_scores
                got = host(fn(*[dev(a) for a in T], dev(users), dev(recent)))
                r = routes()[model + "_scores"]
                assert r["grid_x"] == (rows + 7) // 8 and r["grid_y"] == (ni + 255) // 256 and r["capped"] == -1
                if exact and model == "fpmc":
                    assert np.array_equal(got, want.v)
                elif exact:
                    s = np.sqrt(acc.v).astype(np.float32)      # acc is exact in fp32: sqrtf is correctly rounded
                    assert np.array_equal(got, T[2][None] - s)
                else:
                    assert_within(got, want.v, want.m, (model, rows, ni))
        SEEN.add(("scores", model, dim))


# ---------------------------------------------------------------------------------------------------------------
# the query kernels and the relu pass
# ---------------------------------------------------------------------------------------------------------------
def query_ref(model, T, recent, recent_len, smax=None, pmax=None):
    """Every user's query row over its window's actual length, with its bound."""
    nu, L = recent.shape
    live = np.arange(L)[None, :] < recent_len[:, None]
    if model == "hrm":
        P, E = T
        W = E[recent].astype(np.float64)
        if smax:
            s = R(np.where(live[..., None], W, -np.inf).max(1))
        else:
            s = R(np.where(live[..., None], W, 0.0)).sum(1) / recent_len[:, None]
        p = R(P)
        return rmax(p, s) if pmax else (p + s) / 2
    UI, IU, IL = T
    ctx = R(np.where(live[..., None], IL[recent].astype(np.float64), 0.0)).sum(1)
    return rmax(R(UI), 0.0) + rmax(ctx, 0.0)


@gpu
@pytest.mark.parametrize("L", [3, 64])
@pytest.mark.parametrize("model,smax,pmax", [("hrm", sm, pm) for sm, pm in POOLS] + [("npe", None, None)])
def test_query(model, smax, pmax, L):
    """rows * dim on both sides of 4096 * SMs; windows shorter than L and windows of 64: every query element within the
    bound of float64 (max pools exactly)."""
    from neurec_b200 import _lib
    from neurec_b200.ops import _p, _stream
    lib = _lib.load()
    n_sms = sms()
    rs = np.random.RandomState(L + (smax or 0) * 2 + (pmax or 0))
    D, nu, ni = 64, 300, 500
    T = [rs.randn(n, D).astype(np.float32) for n in ((nu, ni) if model == "hrm" else (nu, ni, ni))]
    recent = rs.randint(0, ni, (nu, L)).astype(np.int32)
    recent_len = rs.randint(1, L + 1, nu).astype(np.int32)
    recent_len[:5] = L
    want = query_ref(model, T, recent, recent_len, smax, pmax)
    dT = [dev(a) for a in T]
    d_recent, d_len = dev(recent), dev(recent_len)
    for rows in query_rows(D, n_sms):
        users = rs.randint(0, nu, rows).astype(np.int32)
        d_users = dev(users)
        out = torch.zeros((rows, D), device="cuda")
        if model == "hrm":
            rc = lib.nrc_hrm_query(_p(dT[0]), _p(dT[1]), D, L, _p(d_users), rows, _p(d_recent), _p(d_len), int(pmax),
                                   int(smax), _p(out), _stream())
        else:
            rc = lib.nrc_npe_query(_p(dT[0]), _p(dT[1]), _p(dT[2]), ni, D, L, _p(d_users), rows, _p(d_recent),
                                   _p(d_len), _p(out), None, _stream())
        _lib.check(rc)
        got = host(out)
        if model == "hrm" and smax and pmax:
            assert np.array_equal(got, want.v[users])
        else:
            assert_within(got, want.v[users], want.m[users], (model, rows))
        r = routes()[model + "_query"]
        grid, capped = elementwise_grid(rows * D, n_sms)
        assert r["grid_x"] == grid and r["capped"] == capped and r["window"] == L
        assert (r["session_max"], r["pre_max"]) == ((smax, pmax) if model == "hrm" else (-1, -1))
        SEEN.add(("query", model, smax, pmax, int(capped)))


@gpu
def test_relu_pass():
    """NPE's relu over the item rows, num_items * dim on both sides of 4096 * SMs, bit for bit; with no query rows the
    query kernel does not launch and its record stays."""
    from neurec_b200 import _lib
    from neurec_b200.ops import _p, _stream
    lib = _lib.load()
    n_sms = sms()
    rs = np.random.RandomState(4)
    D = 16
    for ni in query_rows(D, n_sms):
        IU = rs.randn(ni, D).astype(np.float32)
        IU[::3, ::2] = 0
        out = torch.full((ni, D), 7.0, device="cuda")
        d_iu = dev(IU)
        before = routes()["npe_query"]
        _lib.check(lib.nrc_npe_query(None, _p(d_iu), None, ni, D, 2, None, 0, None, None, None, _p(out), _stream()))
        assert np.array_equal(host(out), np.maximum(IU, 0))
        r = routes()
        grid, capped = elementwise_grid(ni * D, n_sms)
        assert r["npe_query"] == before and r["npe_relu"]["grid_x"] == grid and r["npe_relu"]["capped"] == capped
        SEEN.add(("relu", int(capped)))


@gpu
def test_query_passes_visit_each_element_once():
    """The query kernels are maps: a grid-stride loop that revisits elements (stepping by one CTA instead of the whole
    grid) writes the same values, and only its time shows it.  Over 4 * 4096 * SMs elements at L = 1 (a capped grid,
    four elements per thread) each query pass must take less than 50 times NPE's relu pass over as many elements;
    a grid that revisits takes about 16 * SMs / 2 times as long as one that does not."""
    from neurec_b200 import _lib
    from neurec_b200.ops import _p, _stream
    lib = _lib.load()
    n_sms = sms()
    D = 64
    rows = 4 * 4096 * n_sms // D
    rs = np.random.RandomState(8)
    tabs = [dev(rs.randn(rows, D).astype(np.float32)) for _ in range(3)]
    users = dev(np.arange(rows, dtype=np.int32))
    recent = dev(rs.randint(0, rows, (rows, 1)).astype(np.int32))
    rlen = dev(np.ones(rows, np.int32))
    out = torch.empty((rows, D), device="cuda")
    calls = {"hrm": lambda: lib.nrc_hrm_query(_p(tabs[0]), _p(tabs[1]), D, 1, _p(users), rows, _p(recent), _p(rlen),
                                              0, 0, _p(out), _stream()),
             "npe": lambda: lib.nrc_npe_query(_p(tabs[0]), _p(tabs[1]), _p(tabs[2]), rows, D, 1, _p(users), rows,
                                              _p(recent), _p(rlen), _p(out), None, _stream()),
             "relu": lambda: lib.nrc_npe_query(None, _p(tabs[1]), None, rows, D, 1, None, 0, None, None, None,
                                               _p(out), _stream())}

    def median_ms(fn):
        _lib.check(fn())
        times = []
        for _ in range(5):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            _lib.check(fn())
            b.record()
            b.synchronize()
            times.append(a.elapsed_time(b))
        return float(np.median(times))

    t = {k: median_ms(fn) for k, fn in calls.items()}
    r = routes()
    assert r["npe_relu"]["capped"] == 1 and r["hrm_query"]["capped"] == 1 and r["npe_query"]["capped"] == 1
    assert t["hrm"] < 50 * t["relu"] and t["npe"] < 50 * t["relu"], t
    SEEN.add(("query_once", 1))


# ---------------------------------------------------------------------------------------------------------------
# the *_train_epoch batch loops
# ---------------------------------------------------------------------------------------------------------------
EPOCH_CASES = [(m, o) for m in ("fpmc", "hrm", "npe") for o in OPTS] + [("transrec", o) for o in ("gd", "momentum")]
# TransRec's g moves every step and is read by the next: without reg and with lr 1/4 its granule stays coarse
TRANSREC_HYPER = {"gd": [2.0 ** -2], "momentum": [2.0 ** -2, 0.5]}
# variable k of each model: the touched array that selects its rows (None: g's dense gradient)
EPOCH_TOUCH = {"fpmc": (0, 1, 1, 2), "transrec": (0, 1, 2, None), "hrm": (0, 1), "npe": (0, 1, 2)}


def epoch_batch(model, rs, n, bs, D, L):
    """n samples in which step s reads only users s * 8 + [0, 8) and items s * 16 + [0, 16): no step reads a row an
    earlier step moved (g aside), so every step's gradient is exact from the tables before the epoch."""
    steps = -(-n // bs)
    nu, ni = 8 * (steps + 1), 16 * (steps + 1)
    s = np.arange(n) // bs
    users = (s * 8 + rs.randint(0, 8, n)).astype(np.int32)
    items = (s * 16 + rs.randint(0, 16, n)).astype(np.int32)
    windowed = model in ("hrm", "npe")
    recent = ((s * 16)[:, None] + rs.randint(0, 16, (n, L))).astype(np.int32) if windowed else \
        (s * 16 + rs.randint(0, 16, n)).astype(np.int32)
    if model == "fpmc":
        T = [sparse_dyadic(rs, (nu, D))] + [sparse_dyadic(rs, (ni, D)) for _ in range(3)]
    elif model == "transrec":
        T = [sparse_dyadic(rs, (nu, D), 0.1), sparse_dyadic(rs, (ni, D), 0.1), dyadic(rs, (ni,)),
             sparse_dyadic(rs, (D,), 0.1)]
    elif model == "hrm":
        T = [sparse_dyadic(rs, (nu, D)), sparse_dyadic(rs, (ni, D))]
    else:
        T = [sparse_dyadic(rs, (nu, D)), sparse_dyadic(rs, (ni, D)), sparse_dyadic(rs, (ni, D))]
    if windowed:
        third = rs.randint(0, 2, n).astype(np.float32)
    else:
        third = (s * 16 + rs.randint(0, 16, n)).astype(np.int32)
        for _ in range(100):
            x = score64(model, T, users, recent, items, third)
            if not (x == -1.0).any():
                break
            tie = x == -1.0
            third[tie] = s[tie] * 16 + rs.randint(0, 16, int(tie.sum()))
    return T, users, recent, items, third


@gpu
@pytest.mark.parametrize("model,opt", EPOCH_CASES)
def test_epoch_exact(model, opt):
    """A short last batch, batch_size > n and n = 0, first_stamp > 1, windows of 2 (HRM, with the pools of the case)
    and 3 (NPE): tables, slots, stamps and every step's loss equal tf_math.opt_apply on the float64 gradients bit for
    bit.  TransRec's g moves every step, under gd and momentum with power-of-two hyperparameters."""
    from neurec_b200 import ops
    # (TransRec: a seed whose later steps, where g has moved, also stay off the hinge tie)
    rs = np.random.RandomState(OPTS.index(opt) * 5 + len(model) + 7 * (model == "transrec"))
    D, L = 33, {"hrm": 2, "npe": 3}.get(model)
    smax, pmax = POOLS[OPTS.index(opt) % 4] if model == "hrm" else (None, None)
    pairwise = 1 if model in ("fpmc", "transrec") else 0
    kind = "hinge" if pairwise else "square"
    reg = 0.0 if model == "transrec" else 2.0 ** -3
    hyper0 = TRANSREC_HYPER[opt] if model == "transrec" else HYPER[opt]
    for n, bs, first in ((3 * 64 + 5, 64, 7), (5, 64, 1), (0, 64, 3)):
        steps = -(-n // bs)
        T, users, recent, items, third = epoch_batch(model, rs, n, bs, D, L)
        i0, i1 = tf_math.SLOT_INIT[opt]
        H = [a.copy() for a in T]
        S0 = [None if i0 is None else np.full_like(a, i0) for a in T]
        S1 = [None if i1 is None else np.full_like(a, i1) for a in T]
        dT, dS0, dS1 = [dev(a) for a in T], [dev(a) for a in S0], [dev(a) for a in S1]
        grads = [torch.zeros_like(t) for t in dT]
        sizes = (T[0].shape[0], T[1].shape[0])
        tch = [torch.zeros(sizes[k], dtype=torch.int32, device="cuda") for k in TOUCH_SIZES[model]]
        lr_t = tf_math.adam_lr_t(HYPER["adam"][0], max(steps, 1)) if opt == "adam" else \
            np.full(max(steps, 1), hyper0[0], np.float32)
        step_loss = torch.full((max(steps, 1),), 7.0, device="cuda")
        before = routes()[model + "_grad"]
        ids = (dev(users), dev(recent), dev(items), dev(third), bs)
        tail = (reg, opt, lr_t, hyper0, grads, tch, dS0, dS1, first)
        if model == "fpmc":
            got_steps = ops.fpmc_train_epoch(*dT, *ids, pairwise, kind, *tail, step_loss)
        elif model == "transrec":
            got_steps = ops.transrec_train_epoch(*dT, *ids, pairwise, kind, *tail, ops.transrec_work(D), step_loss)
        elif model == "hrm":
            got_steps = ops.hrm_train_epoch(*dT, *ids, pmax, smax, kind, *tail, step_loss)
        else:
            got_steps = ops.npe_train_epoch(*dT, *ids, kind, *tail, step_loss)
        assert got_steps == steps
        want_t = [np.zeros(sizes[k], np.int32) for k in TOUCH_SIZES[model]]
        want_loss = np.full(max(steps, 1), 7.0, np.float32)
        for s in range(steps):                # the float64 gradient of each step, then the optimizer op for op
            sl = slice(s * bs, min(n, (s + 1) * bs))
            R.exact = True
            try:
                l, g, t = ref_call(model, H, users[sl], recent[sl], items[sl], third[sl], pairwise, kind, reg, smax,
                                   pmax)
            finally:
                R.exact = False
            want_loss[s] = l.v
            assert want_loss[s] == l.v
            hyper = list(hyper0)
            if opt == "adam":
                hyper[0] = lr_t[s]
            for k, (var, gk) in enumerate(zip(H, g)):
                tk = EPOCH_TOUCH[model][k]
                gk32 = gk.v.astype(np.float32)
                assert np.array_equal(gk32, gk.v)
                tf_math.opt_apply(opt, var, gk32.reshape(var.shape), S0[k], S1[k], None if tk is None else t[tk],
                                  hyper, dense_var=tk is None)
            for k, m in enumerate(t):
                want_t[k][m] = first + s
        for k in range(len(T)):
            assert np.array_equal(host(dT[k]), H[k]), (n, k)
            for dsl, hsl in ((dS0[k], S0[k]), (dS1[k], S1[k])):
                if hsl is not None and not (opt == "momentum" and hsl is S1[k]):
                    assert np.array_equal(host(dsl), hsl), (n, k)
            assert not grads[k].any()
        for a, w in zip(tch, want_t):
            assert np.array_equal(host(a), w)
        assert np.array_equal(host(step_loss), want_loss)
        if n == 0:
            assert routes()[model + "_grad"] == before
            SEEN.add(("epoch_n0", model))
        else:
            last = n - (steps - 1) * bs                       # the record is the last batch's
            r = routes()[model + "_grad"]
            assert r["window"] == (L or -1)
            assert r["grid_x"] == (transrec_grid(last) if model == "transrec" else grad_grid(last, sms()))[0]
        SEEN.add(("epoch", model, opt))


# ---------------------------------------------------------------------------------------------------------------
# limits and errors: the library's error, nothing written, the hook unchanged
# ---------------------------------------------------------------------------------------------------------------
@gpu
def test_limits_and_errors_write_nothing():
    from neurec_b200 import _lib
    from neurec_b200.ops import _p, _stream
    lib = _lib.load()
    E_LIMIT, E_VALUE = _lib.NRC_E_LIMIT, _lib.NRC_E_VALUE
    D = 8
    tabs = [dev(np.ones((6, D), np.float32)) for _ in range(4)]
    bias, G = dev(np.ones(6, np.float32)), dev(np.ones(D, np.float32))
    gr = [torch.zeros_like(t) for t in tabs]
    tch = [torch.zeros(6, dtype=torch.int32, device="cuda") for _ in range(3)]
    ids, win = dev(np.zeros(4, np.int32)), dev(np.zeros((4, 65), np.int32))
    lab = dev(np.zeros(4, np.float32))
    loss = torch.zeros(1, device="cuda")
    work = torch.zeros(129 * 256 + 1, device="cuda")
    out = torch.zeros((4, D), device="cuda")
    watched = tabs + gr + tch + [loss, out, work]
    h = np.array([0.1, 0.9, 0.999, 1e-8], np.float32)
    slots = (ctypes.c_void_p * 4)(*[t.data_ptr() for t in tabs])
    step_loss = torch.zeros(4, device="cuda")
    watched.append(step_loss)
    P = lambda k: _p(tabs[k])

    def unchanged(code, fn):
        snap = [t.clone() for t in watched]
        before = routes()
        rc = fn()
        torch.cuda.synchronize()
        assert rc == code, (rc, lib.nrc_last_error())
        assert routes() == before
        for a, b in zip(watched, snap):
            assert torch.equal(a, b)

    fpmc = lambda dim, pw, loss_kind: lib.nrc_fpmc_grad(
        P(0), P(1), P(2), P(3), dim, _p(ids), _p(ids), _p(ids), _p(ids), 4, pw, loss_kind, 0.1, _p(gr[0]), _p(gr[1]),
        _p(gr[2]), _p(gr[3]), _p(tch[0]), _p(tch[1]), _p(tch[2]), 3, _p(loss), _stream())
    transrec = lambda dim, loss_kind, w: lib.nrc_transrec_grad(
        P(0), P(1), _p(bias), _p(G), dim, _p(ids), _p(ids), _p(ids), _p(ids), 4, 1, loss_kind, 0.1, _p(gr[0]),
        _p(gr[1]), _p(gr[2]), _p(gr[3]), _p(tch[0]), _p(tch[1]), _p(tch[2]), 3, w, _p(loss), _stream())
    hrm = lambda dim, L, loss_kind: lib.nrc_hrm_grad(
        P(0), P(1), dim, L, _p(ids), _p(win), _p(ids), _p(lab), 4, 1, 1, loss_kind, 0.1, _p(gr[0]), _p(gr[1]),
        _p(tch[0]), _p(tch[1]), 3, _p(loss), _stream())
    npe = lambda dim, L, loss_kind: lib.nrc_npe_grad(
        P(0), P(1), P(2), dim, L, _p(ids), _p(win), _p(ids), _p(lab), 4, loss_kind, 0.1, _p(gr[0]), _p(gr[1]),
        _p(gr[2]), _p(tch[0]), _p(tch[1]), _p(tch[2]), 3, _p(loss), _stream())
    BPR, HINGE, CE = (_lib.LOSS_IDS[k] for k in ("bpr", "hinge", "cross_entropy"))
    for dim in (0, 257):
        unchanged(E_LIMIT, lambda: fpmc(dim, 1, BPR))
        unchanged(E_LIMIT, lambda: transrec(dim, BPR, _p(work)))
        unchanged(E_LIMIT, lambda: hrm(dim, 2, CE))
        unchanged(E_LIMIT, lambda: npe(dim, 2, CE))
    for L in (0, 65):
        unchanged(E_LIMIT, lambda: hrm(D, L, CE))
        unchanged(E_LIMIT, lambda: npe(D, L, CE))
    unchanged(E_VALUE, lambda: fpmc(D, 1, CE))             # a loss the mode does not define
    unchanged(E_VALUE, lambda: fpmc(D, 0, HINGE))
    unchanged(E_VALUE, lambda: transrec(D, CE, _p(work)))
    unchanged(E_VALUE, lambda: hrm(D, 2, BPR))
    unchanged(E_VALUE, lambda: npe(D, 2, HINGE))
    unchanged(E_VALUE, lambda: transrec(D, BPR, None))     # NULL work
    # the epochs: an unknown optimizer, NULL slots, NULL lr_t, NULL work
    fe = lambda opt, s0, lr, ld=BPR: lib.nrc_fpmc_train_epoch(
        P(0), P(1), P(2), P(3), 6, 6, D, _p(ids), _p(ids), _p(ids), _p(ids), 4, 2, 1, ld, 0.1, opt, lr, h.ctypes.data,
        _p(gr[0]), _p(gr[1]), _p(gr[2]), _p(gr[3]), _p(tch[0]), _p(tch[1]), _p(tch[2]), s0, slots, 1, _p(step_loss),
        _stream())
    unchanged(E_VALUE, lambda: fe(99, slots, h.ctypes.data))
    unchanged(E_VALUE, lambda: fe(0, None, h.ctypes.data))
    unchanged(E_VALUE, lambda: fe(1, slots, None))
    unchanged(E_VALUE, lambda: fe(0, slots, h.ctypes.data, CE))
    unchanged(E_VALUE, lambda: lib.nrc_transrec_train_epoch(
        P(0), P(1), _p(bias), _p(G), 6, 6, D, _p(ids), _p(ids), _p(ids), _p(ids), 4, 2, 1, BPR, 0.1, 0, h.ctypes.data,
        h.ctypes.data, _p(gr[0]), _p(gr[1]), _p(gr[2]), _p(gr[3]), _p(tch[0]), _p(tch[1]), _p(tch[2]), slots, slots, 1,
        None, _p(step_loss), _stream()))
    unchanged(E_VALUE, lambda: lib.nrc_hrm_train_epoch(
        P(0), P(1), 6, 6, D, 2, _p(ids), _p(win), _p(ids), _p(lab), 4, 2, 1, 1, CE, 0.1, 5, h.ctypes.data,
        h.ctypes.data, _p(gr[0]), _p(gr[1]), _p(tch[0]), _p(tch[1]), slots, slots, 1, _p(step_loss), _stream()))
    unchanged(E_LIMIT, lambda: lib.nrc_npe_train_epoch(
        P(0), P(1), P(2), 6, 6, D, 65, _p(ids), _p(win), _p(ids), _p(lab), 4, 2, CE, 0.1, 0, h.ctypes.data,
        h.ctypes.data, _p(gr[0]), _p(gr[1]), _p(gr[2]), _p(tch[0]), _p(tch[1]), _p(tch[2]), slots, slots, 1,
        _p(step_loss), _stream()))
    # the queries: rows < 0, window 65, dim 0
    unchanged(E_VALUE, lambda: lib.nrc_hrm_query(P(0), P(1), D, 2, _p(ids), -1, _p(win), _p(ids), 1, 1, _p(out),
                                                 _stream()))
    unchanged(E_LIMIT, lambda: lib.nrc_hrm_query(P(0), P(1), D, 65, _p(ids), 4, _p(win), _p(ids), 1, 1, _p(out),
                                                 _stream()))
    unchanged(E_VALUE, lambda: lib.nrc_npe_query(P(0), P(1), P(2), 6, D, 2, _p(ids), -1, _p(win), _p(ids), _p(out),
                                                 None, _stream()))
    unchanged(E_LIMIT, lambda: lib.nrc_npe_query(P(0), P(1), P(2), 6, 0, 2, _p(ids), 4, _p(win), _p(ids), _p(out),
                                                 None, _stream()))
    # the score kernels: item tiles past 65535 (NULL pointers: nothing is allocated), dim 257, rows < 0
    for n_items, dim, rows, code in ((65535 * 256 + 1, D, 4, E_LIMIT), (6, 257, 4, E_LIMIT), (6, D, -1, E_VALUE)):
        unchanged(code, lambda: lib.nrc_fpmc_scores(None, None, None, None, n_items, dim, None, None, rows, None,
                                                    _stream()))
        unchanged(code, lambda: lib.nrc_transrec_scores(None, None, None, None, n_items, dim, None, None, rows, None,
                                                        _stream()))
    # the largest item count passes its checks; with no rows nothing launches
    unchanged(_lib.NRC_OK, lambda: lib.nrc_fpmc_scores(None, None, None, None, 65535 * 256, D, None, None, 0, None,
                                                       _stream()))
    SEEN.add(("limits", 1))


REQUIRED = ({("grad", m, p, c) for m in ("fpmc", "transrec") for p in (0, 1) for c in (0, 1)}
            | {("grad", m, 0, c) for m in ("hrm", "npe") for c in (0, 1)}
            | {("transrec_ctas", b) for b in TRANSREC_BATCHES}
            | {("grad_loss", m, k) for m in ("fpmc", "transrec", "npe") for _, k in MODES[m]}
            | {("hrm_pools", sm, pm) for sm, pm in POOLS}
            | {("window", "npe", L, c) for L in WINDOWS for c in (0, 1)}
            | {("window", "hrm", L, c) for L in WINDOWS for c in (0, 1)}
            | {("rounded", m, k, L) for m, _, k, _, _, L in ROUNDED}
            | {("scores", m, d) for m in ("fpmc", "transrec") for d in (1, 32, 256)}
            | {("query", "hrm", sm, pm, c) for sm, pm in POOLS for c in (0, 1)} | {("query", "npe", None, None, c)
                                                                                  for c in (0, 1)}
            | {("relu", c) for c in (0, 1)} | {("query_once", 1)}
            | {("epoch", m, o) for m, o in EPOCH_CASES} | {("epoch_n0", m) for m in ("fpmc", "transrec", "hrm", "npe")}
            | {("limits", 1)})


@gpu
def test_every_route_was_seen(request):
    """Across this file the hook reported every route of the sequential kernels.  Only meaningful when the whole file
    ran: a run of selected tests skips it."""
    here = {it.nodeid for it in request.session.items if it.fspath == request.node.fspath}
    if len(here) < 150:
        pytest.skip("only part of the file ran")
    assert REQUIRED <= SEEN, sorted(REQUIRED - SEEN, key=str)
