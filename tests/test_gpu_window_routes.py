"""Every route Caser (csrc/caser.cu), FPMCplus (the fpmcplus_* kernels of csrc/sequential.cu) and FISM's epoch
(csrc/fism.cu) take from a shape, against float64: bit for bit on exact constructions, and entry by entry within a
first-order rounding bound on Gaussian inputs (the "rounded cases" section).

The routes depend on the SM count: Caser's gradient and query kernels run one CTA per sample and cap their grid at
2 * SMs; its reg pass and FPMCplus's projection pass cap at 16 CTAs of 256 threads per SM (4096 * SMs elements); the
FPMCplus gradient caps at 8 CTAs of 8 warps per SM (64 * SMs samples).  Both dense gradients are summed in chunks of
32 samples by a last-CTA-finishes pass that resets its counters for the next launch.  Caser stages its dense block in
shared memory while it and the per-sample work fit kCaserSmemFloats; FPMCplus's pair kernel holds as many rows per
CTA (R, at most 8) as its shared-memory budget allows.  Every shape below is derived from the device's SM count or
from those formulas, one case on each side of each boundary; each test asserts the route it ran through the models'
route hooks, and the last test of the file checks that the whole file saw every route.

Exact constructions (every route must equal the float64 restatements of caser_math, fpmcplus_math and fism_math bit
for bit):
  * Caser: dyadic tables and weights; every sample has its own targets, and each target's bias is minus its dot
    product with the sample's [z, P_u], so every logit is exactly 0, sigmoid = 1/2 and dl/dx = -+1 / (2 B T) (B * T and
    B * N powers of two).  Dropout keep in {1, 1/2, 1/4}; leading pads, a fully padded window, pad targets; windows
    redrawn until every max-pool over a positive maximum ties 1, 2 or 4 positions.  Only the loss (logf) is bounded.
  * FPMCplus: b = +-64 per attention column and small dyadic W, so every tanh saturates to exactly +-1 (|z| >= 20 is
    asserted, where float64's tanh saturates as well) and every window position has the same energy: attention weights
    are exactly 1 (L = 1) or 1/2 (L = 2), tanh' = 0, and the attention parameters' gradients are exactly their reg
    term.  Hinge (off the tie x = -1) and square losses.
  * FISM: alpha = 0 and dyadic tables.
Epochs: every step reads rows no other step reads, so each step's gradient is exact from the tables before the epoch,
and the optimizer step is tf_math.opt_apply's op for op."""
import ctypes

import numpy as np
import pytest
import torch

import caser_math as cm
import fism_math as fm
import fpmcplus_math as fpm
from oracle import tf_math
from test_gpu_graph_routes import dropout_mask_ref
from test_gpu_seq_routes import R, cat, pair_loss, point_loss, scatter, where

gpu = pytest.mark.gpu
U24 = 2.0 ** -24
SEEN = set()
OPTS = ("gd", "adam", "adagrad", "rmsprop", "momentum")
HYPER = {"gd": [2.0 ** -4], "adam": [2.0 ** -4, 0.9, 0.999, 1e-8], "adagrad": [2.0 ** -4],
         "rmsprop": [2.0 ** -4, 0.9, 0.5, 1e-10], "momentum": [2.0 ** -4, 0.5]}
CASER_SMEM_FLOATS = 56 * 1024                     # kCaserSmemFloats
FPMCPLUS_PAIR_FLOATS = 25600                      # kFpmcPlusPairSmemFloats


def dev(a):
    return None if a is None else torch.from_numpy(np.ascontiguousarray(a)).cuda()


def host(t):
    return t.cpu().numpy()


def sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def dyadic(rs, shape, lo=-1, hi=1, k=2, density=1.0):
    v = rs.randint(lo, hi + 1, shape) / 2.0 ** k
    if density < 1.0:
        v = v * (rs.rand(*shape) < density)
    return v.astype(np.float32)


def exact32(a):
    """The float64 array holds fp32 values only (a necessary condition of a bit-for-bit comparison)."""
    a = np.asarray(a, np.float64)
    return np.array_equal(a.astype(np.float32).astype(np.float64), a)


# ---------------------------------------------------------------------------------------------------------------
# the route predicates of the host code and the shapes on each side of them (pure functions of the SM count)
# ---------------------------------------------------------------------------------------------------------------
def pow2_batches(n_sms):
    """Powers of two on each side of Caser's 2 * SMs CTAs (B * T stays a power of two): the largest one the cap
    admits and the next one."""
    lo = 1 << (2 * n_sms).bit_length() - 1
    return lo, 2 * lo


def elementwise_capped(total, n_sms):
    return (total + 255) // 256 > 16 * n_sms


def fpmcplus_grad_grid(batch, n_sms):
    return min((batch + 7) // 8, 8 * n_sms), (batch + 7) // 8 > 8 * n_sms


def caser_dense(d, L, nv, nh):
    return cm.dense_layout(d, L, nv, nh)[1]


def caser_staged(d, L, nv, nh):
    """caser_staged: the dense block plus the CTA's per-sample floats fit kCaserSmemFloats."""
    F, NH = nv * d + nh * L, nh * L * (L + 1) // 2
    return caser_dense(d, L, nv, nh) + L * d + NH + F + 3 * d + 64 <= CASER_SMEM_FLOATS


def caser_smem_boundary(d=40, L=8, nv=2):
    """(largest staged nh, smallest unstaged nh) at (d, L, nv)."""
    nh = 1
    while caser_staged(d, L, nv, nh + 1):
        nh += 1
    return (d, L, nv, nh), (d, L, nv, nh + 1)


def fpmcplus_pair_rows(d, w, L):
    return min(8, (FPMCPLUS_PAIR_FLOATS - w) // (w * (1 + L) + d * (1 + L) + 1))


PAIR_SHAPES = [(16, 16, 2), (64, 64, 56), (256, 128, 64)]          # R = 8, 3, 1 (d, w, L)


def projection_shape(n_sms, above):
    """(num_items, rows) of an FPMCplus score call at d = 2, w = 1, L = 2 whose projection pass has exactly
    4096 * SMs elements (+1 above): num_items * (w + 2 d) + rows * (1 + L) * w."""
    target = 4096 * n_sms + int(above)
    for rows in range(1, 10):
        if (target - 3 * rows) % 5 == 0:
            return (target - 3 * rows) // 5, rows
    raise AssertionError(target)


def caser_reg_shape(n_sms, d, above):
    """(num_users, num_items) with nu d + ni (3 d + 1) = 4096 * SMs (+1 above)."""
    target = 4096 * n_sms + int(above)
    for nu in range(64, 64 + 3 * d + 1):
        if (target - nu * d) % (3 * d + 1) == 0:
            return nu, (target - nu * d) // (3 * d + 1)
    raise AssertionError(target)


@pytest.mark.parametrize("n_sms", [114, 132])
def test_route_shapes_straddle_every_boundary(n_sms):
    """CPU: the shapes derived from the SM count land on both sides of every route predicate (114: H100 PCIe,
    132: H100 SXM), and the formula-derived shapes on both sides of the shared-memory ones."""
    lo, hi = pow2_batches(n_sms)
    assert lo <= 2 * n_sms < hi and lo & (lo - 1) == 0
    assert [fpmcplus_grad_grid(b, n_sms)[1] for b in (64 * n_sms, 64 * n_sms + 1)] == [False, True]
    for above in (False, True):
        ni, rows = projection_shape(n_sms, above)
        assert ni * 5 + rows * 3 == 4096 * n_sms + above
        assert elementwise_capped(ni * 5 + rows * 3, n_sms) == above
        nu, ni = caser_reg_shape(n_sms, 8, above)
        assert nu * 8 + ni * 25 == 4096 * n_sms + above
    a, b = caser_smem_boundary()
    assert caser_staged(*a) and not caser_staged(*b) and b[3] <= 64
    assert [fpmcplus_pair_rows(*s) for s in PAIR_SHAPES] == [8, 3, 1]
    assert sorted({(B + 31) // 32 for B in (1, 32, 33, 70)}) == [1, 2, 3]


# ---------------------------------------------------------------------------------------------------------------
# Caser: exact cases
# ---------------------------------------------------------------------------------------------------------------
def caser_ties(acts):
    """[B, L * nh] tie counts of every max-pool whose maximum is positive (1 elsewhere)."""
    out = []
    for a in acts:
        mx = a.max(1)
        cnt = (a == mx[:, None, :]).sum(1)
        out.append(np.where(mx > 0, cnt, 1))
    return np.concatenate(out, 1)


def caser_weights(rs, d, L, nv, nh):
    """Dyadic conv and FC weights.  conv_h biases <= 0, so positions over pads only are relu zeros (they would tie
    any number of positions), and b1 > 0, so most of z passes its relu."""
    parts = {}
    for name, _, shape in cm.dense_layout(d, L, nv, nh)[0]:
        if name.startswith("Kv") or name.startswith("Kh"):
            parts[name] = dyadic(rs, shape, -1, 1, 2, 0.6)
        elif name == "W1":
            parts[name] = dyadic(rs, shape, -1, 1, 3, 0.4)
        elif name.startswith("bh"):
            parts[name] = dyadic(rs, shape, -2, 0, 2)
        elif name == "b1":
            parts[name] = dyadic(rs, shape, 1, 4, 3)
        else:
            parts[name] = dyadic(rs, shape, -2, 2, 3)
    return cm.pack(parts, d, L, nv, nh).astype(np.float32)


def window_of(rs, L, ids):
    """A window of L ids in which every id appears 1, 2 or 4 times."""
    out, fresh = [], iter(rs.permutation(ids))
    while len(out) < L:
        fits = [k for k in (1, 2, 4) if len(out) + k <= L]
        out += [next(fresh)] * fits[rs.randint(len(fits))]
    return rs.permutation(out)


def caser_case(rs, d, L, nv, nh, T, N, B, mask=None, keep=1.0, nu=None, ni=None, disjoint=False, pads=True):
    """Tables, dense block and batch of one exact Caser batch (see the module docstring).  disjoint: no row of any
    table is read by two samples.  -> (P, E, W2, b2, dense), (users, seqs, pos, neg), tie counts."""
    K = T + N
    nu = nu or (B + 1 if disjoint else max(2, B // 3))
    ni = ni or (B * max(K, L) + 4)
    P = dyadic(rs, (nu, d), -1, 1, 2, 0.5)
    E = dyadic(rs, (ni, d), -2, 2, 2)
    W2 = dyadic(rs, (ni, 2 * d), -1, 1, 2, 0.5)
    b2 = dyadic(rs, (ni,), -2, 2, 3)
    dense = caser_weights(rs, d, L, nv, nh)
    if disjoint:
        users = rs.permutation(nu)[:B].astype(np.int32)
        seqs = rs.permutation(ni)[:B * L].reshape(B, L).astype(np.int32)
    else:
        users = rs.randint(0, nu, B).astype(np.int32)
        if B > 1:
            users[1] = users[0]
        seqs = np.stack([window_of(rs, L, np.arange(ni)) for _ in range(B)]).astype(np.int32)
    tg = rs.permutation(ni)[:B * K].reshape(B, K).astype(np.int32)
    pos, neg = tg[:, :T].copy(), tg[:, T:].copy()
    if pads and not disjoint:
        if L > 1:
            seqs[0, :L - 1] = ni                                   # a short history's leading pads
        if B > 2:
            seqs[2] = ni                                           # a fully padded window
        if B > 1:
            pos[0, 0] = ni                                         # pad targets: a zero row and bias
            neg[-1, -1] = ni
    redraw = [b for b in range(B) if not (pads and b == 2 and B > 2 and not disjoint)]
    for _ in range(200):
        f = cm.forward(P, E, dense, d, L, nv, nh, users, seqs, mask, keep)
        ties = caser_ties(f["acts"])
        bad = [b for b in redraw if not np.isin(ties[b], (1, 2, 4)).all()]
        if not bad:
            break
        for b in bad:
            if disjoint:
                seqs[b] = rs.randint(0, ni, L)
            elif b == 0 and pads and L > 1:
                seqs[b, -1] = rs.randint(0, ni)
            else:
                seqs[b] = window_of(rs, L, np.arange(ni))
    else:
        raise AssertionError("no tie-safe windows")
    assert np.isin(ties, (1, 2, 4)).all()
    u = f["u"]
    tgt = np.concatenate([pos, neg], 1)
    real = tgt != ni
    for b in range(B):                                             # every logit exactly 0
        for j, t in enumerate(tgt[b]):
            if t != ni:
                b2[t] = -np.dot(u[b], W2[t].astype(np.float64))
    assert exact32(b2) and real.any()
    return (P, E, W2, b2, dense), (users, seqs, pos, neg), ties


def caser_loss_bound(B, T, N, want):
    return (B * (T + N) + 16) * U24 * 4 * abs(want) + 1e-7


def caser_routes():
    from neurec_b200 import ops
    return ops.caser_last_routes()


def caser_device_grad(tabs, batch, nv, nh, mask, keep, work=None, fill=7.0):
    from neurec_b200 import ops
    d, L = tabs[0].shape[1], batch[1].shape[1]
    B = len(batch[0])
    g = [torch.zeros(t.shape, dtype=torch.float32, device="cuda") for t in tabs]
    g[4].fill_(fill)                                             # overwritten, not accumulated
    work = ops.caser_work(d, L, nv, nh, B) if work is None else work
    lo = torch.zeros(1, device="cuda")
    ops.caser_grad(*[dev(t) for t in tabs], *[dev(a) for a in batch], nv, nh, dev(mask), keep, g, work, lo)
    torch.cuda.synchronize()
    return float(lo), [host(x) for x in g]


# d, L, nv, nh, T, N, B ("lo" / "hi": the powers of two around 2 * SMs), keep, masked
CASER_EXACT = [
    (3, 1, 1, 1, 1, 1, 1, 1.0, False),
    (4, 2, 2, 2, 2, 2, 32, 0.5, True),
    (50, 5, 4, 16, 2, 4, 64, 0.25, True),                        # the conf's d, L, nv, nh; two chunks
    (8, 16, 2, 3, 1, 1, "lo", 0.5, True),                        # the largest window
    (6, 4, 2, 2, 1, 2, "hi", 1.0, False),
    ("staged", 1, 1, 16, 0.5, True),
    ("unstaged", 1, 1, 16, 1.0, False),
]


def caser_exact_shape(case, n_sms):
    if case[0] in ("staged", "unstaged"):
        shape = caser_smem_boundary()[case[0] == "unstaged"]
        return shape + case[1:]
    d, L, nv, nh, T, N, B, keep, masked = case
    lo, hi = pow2_batches(n_sms)
    return d, L, nv, nh, T, N, {"lo": lo, "hi": hi}.get(B, B), keep, masked


@gpu
@pytest.mark.parametrize("ci", range(len(CASER_EXACT)))
def test_caser_grad_exact(ci):
    """Windows 1, 2, 5 and 16; batches 1, 32, 64 and the powers of two on each side of 2 * SMs; the largest staged
    and the smallest unstaged dense block; keep 1, 1/2 and 1/4: every table gradient and the dense block bit for bit,
    the loss within the bound of its logf terms."""
    n_sms = sms()
    d, L, nv, nh, T, N, B, keep, masked = caser_exact_shape(CASER_EXACT[ci], n_sms)
    rs = np.random.RandomState(100 + ci)
    F = nv * d + nh * L
    mask = (rs.rand(B, F) < 0.5).astype(np.float32) if masked else None
    tabs, batch, ties = caser_case(rs, d, L, nv, nh, T, N, B, mask, keep)
    want_l, want = cm.loss_and_grad(*[t.astype(np.float64) for t in tabs], d, L, nv, nh, *batch, mask, keep)
    lo, got = caser_device_grad(tabs, batch, nv, nh, mask, keep)
    for name, g, w in zip(("P", "E", "W2", "b2", "dense"), got, want):
        assert exact32(w), name
        assert np.array_equal(g.astype(np.float64), w), (name, float(np.abs(g - w).max()))
    assert abs(lo - want_l) <= caser_loss_bound(B, T, N, want_l), (lo, want_l)
    r = caser_routes()
    cap = 2 * n_sms
    staged = caser_staged(d, L, nv, nh)
    assert r["grad"] == dict(staged=int(staged), grid_x=min(B, cap), grid_y=-1, capped=int(B > cap), window=L,
                             masked=int(masked))
    assert r["wgrad"]["grid_x"] == (caser_dense(d, L, nv, nh) + 255) // 256 and r["wgrad"]["grid_y"] == (B + 31) // 32
    if L >= 4:
        assert {2, 4} <= set(np.unique(ties))
    SEEN.add(("caser_grad", int(staged), int(B > cap)))
    SEEN.add(("caser_window", L))
    SEEN.add(("caser_chunks", (B + 31) // 32))
    SEEN.update(("caser_ties", int(t)) for t in np.unique(ties))


@gpu
def test_caser_wgrad_counters_reset_between_launches():
    """Launches with 2, 1, 3 and 2 chunks (64, 1, 70 and 33 samples, the last two with a short last chunk) one after
    another on one work buffer: each writes its whole dense gradient (the output starts at 7), the exact ones bit for
    bit against float64 and the others bit for bit against the same launch on a fresh work buffer."""
    from neurec_b200 import ops
    d, L, nv, nh = 5, 3, 2, 2
    rs = np.random.RandomState(17)
    work = ops.caser_work(d, L, nv, nh, 70)
    for B, exact in ((64, True), (1, True), (70, False), (33, False), (64, True)):
        T, N = (1, 1)
        tabs, batch, _ = caser_case(rs, d, L, nv, nh, T, N, B, None, 1.0)
        lo, got = caser_device_grad(tabs, batch, nv, nh, None, 1.0, work=work)
        if exact:
            _, want = cm.loss_and_grad(*[t.astype(np.float64) for t in tabs], d, L, nv, nh, *batch)
            assert np.array_equal(got[4].astype(np.float64), want[4]), B
        else:
            _, fresh = caser_device_grad(tabs, batch, nv, nh, None, 1.0)
            assert np.array_equal(got[4], fresh[4]), B
            _, want = cm.loss_and_grad(*[t.astype(np.float64) for t in tabs], d, L, nv, nh, *batch)
            assert not (got[4] == 7.0).any()
            assert np.abs(got[4] - want[4]).max() <= 1e-5 * max(np.abs(want[4]).max(), 1e-6)
        assert caser_routes()["wgrad"]["grid_y"] == (B + 31) // 32
        SEEN.add(("caser_chunks", (B + 31) // 32))
    SEEN.add(("caser_counters", 1))


@gpu
@pytest.mark.parametrize("staged", [True, False])
def test_caser_query_exact(staged):
    """Rows on both sides of 2 * SMs, windows with pads and a fully padded one: [z, P_u] bit for bit."""
    from neurec_b200 import ops
    n_sms = sms()
    d, L, nv, nh = caser_smem_boundary()[0 if staged else 1]
    rs = np.random.RandomState(5 + staged)
    nu, ni = 40, 90
    P = dyadic(rs, (nu, d), -1, 1, 2, 0.5)
    E = dyadic(rs, (ni, d), -2, 2, 2)
    W2 = dyadic(rs, (ni, 2 * d), -1, 1, 2)
    dense = caser_weights(rs, d, L, nv, nh)
    windows = rs.randint(0, ni, (nu, L)).astype(np.int32)
    windows[3, :L - 1] = ni
    windows[4] = ni
    for rows in (2 * n_sms, 2 * n_sms + 1):
        users = rs.randint(0, nu, rows).astype(np.int32)
        users[:2] = [3, 4]
        want = cm.query(P, E, dense, d, L, nv, nh, users, windows[users])
        got = host(ops.caser_query(dev(P), dev(E), dev(W2), dev(dense), dev(users), dev(windows), nv, nh))
        assert exact32(want) and np.array_equal(got.astype(np.float64), want)
        r = caser_routes()["query"]
        capped = rows > 2 * n_sms
        assert r == dict(staged=int(staged), grid_x=min(rows, 2 * n_sms), grid_y=-1, capped=int(capped), window=L,
                         masked=0)
        SEEN.add(("caser_query", int(staged), int(capped)))


def caser_epoch_call(tabs, batch, nv, nh, bs, keep, reg, seed, epoch, lr_t, slots=None, work=None):
    """One nrc_caser_train_epoch on device copies -> (tables, slots, step losses, grads, steps)."""
    from neurec_b200 import ops
    d, L = tabs[0].shape[1], batch[1].shape[1]
    dv = [dev(t) for t in tabs]
    s0 = [torch.zeros_like(v) for v in dv] if slots is None else [dev(s) for s in slots[0]]
    s1 = [torch.zeros_like(v) for v in dv] if slots is None else [dev(s) for s in slots[1]]
    grads = [torch.zeros_like(v) for v in dv]
    steps = max(1, -(-len(batch[0]) // bs))
    step_loss = torch.full((steps,), 7.0, device="cuda")
    work = ops.caser_work(d, L, nv, nh, bs) if work is None else work
    got = ops.caser_train_epoch(*dv, *[dev(a) for a in batch], nv, nh, bs, keep, reg, seed, epoch, lr_t,
                                HYPER["adam"], grads, s0, s1, work, step_loss)
    return [host(v) for v in dv], ([host(s) for s in s0], [host(s) for s in s1]), host(step_loss), \
        [host(g) for g in grads], got


@gpu
@pytest.mark.parametrize("above", [False, True])
def test_caser_epoch_first_step_exact(above):
    """One step whose reg pass covers 4096 * SMs elements (+1: the capped grid): dropout masks of the documented key,
    l2_reg 1/8; tables, Adam slots and the dense block bit for bit against tf_math.opt_apply on the float64
    gradient, the step loss within its logf bound."""
    from neurec_b200 import ops
    n_sms = sms()
    d, L, nv, nh, T, N, B, keep, reg = 8, 3, 2, 2, 2, 2, 32, 0.5, 2.0 ** -3
    nu, ni = caser_reg_shape(n_sms, d, above)
    rs = np.random.RandomState(31 + above)
    seed, epoch = 2018, 3
    F = nv * d + nh * L
    mask = dropout_mask_ref(B * F, keep, seed, epoch << 32).reshape(B, F)        # the documented key, on the host
    tabs, batch, _ = caser_case(rs, d, L, nv, nh, T, N, B, mask, keep, nu=nu, ni=ni)
    lr_t = tf_math.adam_lr_t(HYPER["adam"][0], 1)
    got_t, (g0, g1), got_loss, grads, steps = caser_epoch_call(tabs, batch, nv, nh, 64, keep, reg, seed, epoch, lr_t)
    assert steps == 1
    want_l, want = cm.loss_and_grad(*[t.astype(np.float64) for t in tabs], d, L, nv, nh, *batch, mask, keep)
    H = [t.copy() for t in tabs]
    S0, S1 = [np.zeros_like(t) for t in tabs], [np.zeros_like(t) for t in tabs]
    for k in range(5):
        g = want[k] + (reg * H[k].astype(np.float64) if k < 4 else 0.0)
        assert exact32(g), k
        tf_math.opt_apply("adam", H[k], g.astype(np.float32), S0[k], S1[k], None,
                          [lr_t[0]] + HYPER["adam"][1:], dense_var=k == 4)
    for k in range(5):
        assert np.array_equal(got_t[k], H[k]), k
        assert np.array_equal(g0[k], S0[k]) and np.array_equal(g1[k], S1[k]), k
        assert not grads[k].any() or k == 4
    assert abs(float(got_loss[0]) - want_l) <= caser_loss_bound(B, T, N, want_l)
    r = caser_routes()["reg"]
    total = nu * d + ni * (3 * d + 1)
    assert r["capped"] == int(elementwise_capped(total, n_sms)) == int(above)
    assert r["grid_x"] == min((total + 255) // 256, 16 * n_sms)
    SEEN.add(("caser_reg", int(above)))


@gpu
def test_caser_epoch_steps_equal_single_steps():
    """No row shared between samples: a k-step epoch (a short last batch) equals k one-step calls bit for bit
    (tables, slots, the dense block; every step's loss, summed by atomics, within its bound); batch_size > n runs one
    step; n = 0 runs none and writes nothing."""
    d, L, nv, nh, T, N = 6, 4, 2, 3, 1, 2
    bs, n = 16, 3 * 16 + 5
    rs = np.random.RandomState(41)
    tabs, batch, _ = caser_case(rs, d, L, nv, nh, T, N, n, None, 1.0, disjoint=True)
    steps = -(-n // bs)
    lr_t = tf_math.adam_lr_t(HYPER["adam"][0], steps)
    all_t, all_s, all_l, all_g, got = caser_epoch_call(tabs, batch, nv, nh, bs, 1.0, 2.0 ** -3, 5, 9, lr_t)
    assert got == steps
    cur_t, cur_s = [t.copy() for t in tabs], None
    for s in range(steps):
        sl = slice(s * bs, min(n, (s + 1) * bs))
        cur_t, cur_s, lo, _, one = caser_epoch_call(cur_t, [a[sl] for a in batch], nv, nh, bs, 1.0, 2.0 ** -3, 5, 9,
                                                    lr_t[s:s + 1], slots=cur_s)
        assert one == 1                       # the step loss's atomics add in any order
        assert abs(float(lo[0]) - float(all_l[s])) <= caser_loss_bound(len(batch[0][sl]), T, N, float(all_l[s])), s
    for k in range(5):
        assert np.array_equal(all_t[k], cur_t[k]), k
        assert np.array_equal(all_s[0][k], cur_s[0][k]) and np.array_equal(all_s[1][k], cur_s[1][k]), k
    assert caser_routes()["grad"]["grid_x"] == n - (steps - 1) * bs
    # batch_size > n: one step; n = 0: no step, nothing written, the records kept
    _, _, _, _, one = caser_epoch_call(tabs, [a[:5] for a in batch], nv, nh, 64, 1.0, 0.0, 5, 9, lr_t[:1])
    assert one == 1 and caser_routes()["grad"]["grid_x"] == 5
    before = caser_routes()
    t0, _, l0, _, zero = caser_epoch_call(tabs, [a[:0] for a in batch], nv, nh, 64, 1.0, 0.0, 5, 9, lr_t[:1])
    assert zero == 0 and caser_routes() == before and l0[0] == 7.0
    assert all(np.array_equal(a, b) for a, b in zip(t0, tabs))
    SEEN.add(("caser_epoch", 1))


# ---------------------------------------------------------------------------------------------------------------
# FPMCplus: exact cases
# ---------------------------------------------------------------------------------------------------------------
def fpmcplus_tables(rs, nu, ni, d, w, density=0.3, split=False):
    """Dyadic tables and a saturating attention MLP: b = +-64, |UI W_U + IL W_I + LI W_L| <= 24 for d <= 256.
    split: columns 0 and 1 instead saturate to +-s and -+s with s = LI_l[0] = +-1 of the window item, at equal h, so
    every window position keeps the same energy while h's data gradient sum_k de_k t_k is not 0 (it carries the
    softmax backward's sign)."""
    tabs = [dyadic(rs, (n, d), -1, 1, 2, density) for n in (nu, ni, ni, ni)]
    W = dyadic(rs, (3 * d, w), -1, 1, 3, 0.3)
    b = (rs.choice([-64.0, 64.0], (1, w))).astype(np.float32)
    h = dyadic(rs, (w, 1), -1, 1, 2)
    h[h == 0] = 0.25
    if split:
        tabs[3][:, 0] = rs.choice([-1.0, 1.0], ni)
        W[2 * d, :2] = 64.0, -64.0
        b[0, :2] = 0.0
        h[1] = h[0]
    return tabs + [W, b, h]


def fpmcplus_pre_activations(tabs, users, recent, items):
    UI, IU, IL, LI, W, b, h = [t.astype(np.float64) for t in tabs]
    d = UI.shape[1]
    z = (UI[users] @ W[:d] + b)[:, None, :] + (IL[items] @ W[d:2 * d])[:, None, :] + LI[recent] @ W[2 * d:]
    return z


def fpmcplus_score64(tabs, users, recent, items, third):
    UI, IU, IL, LI = [t.astype(np.float64) for t in tabs[:4]]
    x = lambda i: (UI[users] * IU[i]).sum(1) + (IL[i] * LI[recent].mean(1)).sum(1)
    return x(items) - x(third)


def fpmcplus_case(rs, B, d, w, L, pairwise, kind, nu=None, ni=None, steps_of=None, split=False):
    """One exact FPMCplus batch; steps_of (bs): sample s reads users s // bs * 8 + [0, 8) and items, negatives and
    window ids s // bs * 16 + [0, 16) only."""
    if steps_of:
        s = np.arange(B) // steps_of
        steps = int(s.max()) + 1 if B else 1
        nu, ni = 8 * (steps + 1), 16 * (steps + 1)
        users = (s * 8 + rs.randint(0, 8, B)).astype(np.int32)
        pick = lambda shape: ((s * 16).reshape((-1,) + (1,) * (len(shape) - 1)) + rs.randint(0, 16, shape))
        items, recent = pick((B,)).astype(np.int32), pick((B, L)).astype(np.int32)
        third_ids = lambda m: pick((B,))[m]
    else:
        nu, ni = nu or B + 5, ni or 2 * B + 6
        users, items = rs.randint(0, nu, B).astype(np.int32), rs.randint(0, ni, B).astype(np.int32)
        recent = rs.randint(0, ni, (B, L)).astype(np.int32)
        if B > 8:
            users[1] = users[0]
            recent[::8, 0] = items[::8]
        third_ids = lambda m: rs.randint(0, ni, int(m.sum()))
    tabs = fpmcplus_tables(rs, nu, ni, d, w, split=split)
    if pairwise:
        third = np.zeros(B, np.int32)
        redo = np.ones(B, bool)
        for _ in range(100):
            third[redo] = third_ids(redo)
            redo = fpmcplus_score64(tabs, users, recent, items, third) == -1.0 if kind == "hinge" else redo & False
            if not redo.any():
                break
    else:
        third = rs.randint(0, 2, B).astype(np.float32)
    z = fpmcplus_pre_activations(tabs, users, recent, items)
    assert B == 0 or np.abs(z).min() >= 20
    if pairwise and B:
        assert np.abs(fpmcplus_pre_activations(tabs, users, recent, third)).min() >= 20
    return tabs, users, recent, items, third


def fpmcplus_ref(tabs, users, recent, items, third, pairwise, kind, reg_mf, reg_w):
    return fpm.fpmcplus_grad(*tabs, users, recent, items, third, pairwise, kind, reg_mf, reg_w, dtype=np.float64)


# d, w, L, B ("cap": 64 * SMs, "cap+1": one more), pairwise, loss
FPMCPLUS_EXACT = [
    (5, 4, 1, 1, 1, "hinge"), (16, 16, 2, "cap", 1, "square"), (33, 40, 2, "cap+1", 1, "hinge"),
    (8, 8, 1, "cap+1", 0, "square"), (16, 16, 2, "cap", 0, "square"), (256, 128, 2, 37, 0, "square"),
    (32, 128, 1, 33, 1, "square"),
]


def fpmcplus_routes():
    from neurec_b200 import ops
    return ops.fpmcplus_last_routes()


@gpu
@pytest.mark.parametrize("d,w,L,B,pairwise,kind", FPMCPLUS_EXACT)
def test_fpmcplus_grad_exact(d, w, L, B, pairwise, kind):
    """Batches 1, 33, 37 and on both sides of 64 * SMs, windows 1 and 2, widths up to 256 and 128: every table
    gradient, h's, the stamps and the loss bit for bit; W takes exactly reg_w * W (pairwise; 0 pointwise), b exactly
    0, and h its reg term except on the two split columns of a window of 2."""
    from neurec_b200 import ops
    n_sms = sms()
    B = {"cap": 64 * n_sms, "cap+1": 64 * n_sms + 1}.get(B, B)
    rs = np.random.RandomState(d * 3 + w + L + pairwise)
    split = L == 2 and w >= 2
    tabs, users, recent, items, third = fpmcplus_case(rs, B, d, w, L, pairwise, kind, split=split)
    reg_mf, reg_w = 2.0 ** -3, 2.0 ** -2
    want_l, want_g, want_t = fpmcplus_ref(tabs, users, recent, items, third, pairwise, kind, reg_mf, reg_w)
    dt = [dev(t) for t in tabs]
    g = [torch.zeros_like(t) for t in dt]
    nu, ni = tabs[0].shape[0], tabs[1].shape[0]
    tch = [torch.full((n,), 5, dtype=torch.int32, device="cuda") for n in (nu, ni, ni)]
    lo = torch.zeros(1, device="cuda")
    work = ops.fpmcplus_work(d, w, L, B)
    ops.fpmcplus_grad(*dt, dev(users), dev(recent), dev(items), dev(third), pairwise, kind, reg_mf, reg_w, g, tch, 9,
                      work, lo)
    got = [host(x) for x in g]
    for k, (a, ref) in enumerate(zip(got, want_g)):
        assert exact32(ref), k
        assert np.array_equal(a.astype(np.float64), ref), (k, float(np.abs(a - ref).max()))
    rw = reg_w if pairwise else 0.0
    assert np.array_equal(got[4], tabs[4] * np.float32(rw)) and not got[5].any()
    assert np.array_equal(got[6][2:], tabs[6][2:] * np.float32(rw))
    if split:
        assert (got[6][:2] != tabs[6][:2] * np.float32(rw)).all()
    for a, ref in zip(tch, want_t):
        assert np.array_equal(host(a), np.where(ref, 9, 5))
    assert float(lo) == float(want_l), (float(lo), float(want_l))
    grid, capped = fpmcplus_grad_grid(B, n_sms)
    r = fpmcplus_routes()
    assert r["grad"] == dict(pairwise=pairwise, grid_x=grid, grid_y=-1, capped=int(capped), window=L, rows=-1)
    assert r["wgrad"]["grid_y"] == (B + 31) // 32 and r["wgrad"]["grid_x"] == (3 * d * w + 2 * w + 255) // 256
    SEEN.add(("fpmcplus_grad", pairwise, int(capped), L))


@gpu
@pytest.mark.parametrize("opt", OPTS)
@pytest.mark.parametrize("pairwise,kind", [(1, "hinge"), (0, "square")])
def test_fpmcplus_epoch_exact(pairwise, kind, opt):
    """A short last batch, batch_size > n, n = 0, first_stamp > 1, windows of 2: tables, slots, stamps and every
    step's loss bit for bit against tf_math.opt_apply on the float64 gradients.  reg_w = 0, so W, b and h take zero
    gradients and stay saturating through the epoch under every optimizer; their slots are checked as well."""
    from neurec_b200 import ops
    rs = np.random.RandomState(OPTS.index(opt) * 3 + pairwise)
    d, w, L, reg = 9, 8, 2, 2.0 ** -3
    for n, bs, first in ((3 * 64 + 5, 64, 7), (5, 64, 1), (0, 64, 3)):
        steps = -(-n // bs)
        T = fpmcplus_case(rs, n, d, w, L, pairwise, kind, steps_of=bs)
        tabs, users, recent, items, third = T
        i0, i1 = tf_math.SLOT_INIT[opt]
        H = [a.copy() for a in tabs]
        S0 = [None if i0 is None else np.full_like(a, i0) for a in tabs]
        S1 = [None if i1 is None else np.full_like(a, i1) for a in tabs]
        dT, dS0, dS1 = [dev(a) for a in tabs], [dev(a) for a in S0], [dev(a) for a in S1]
        grads = [torch.zeros_like(t) for t in dT]
        nu, ni = tabs[0].shape[0], tabs[1].shape[0]
        tch = [torch.zeros(k, dtype=torch.int32, device="cuda") for k in (nu, ni, ni)]
        lr_t = tf_math.adam_lr_t(HYPER["adam"][0], max(steps, 1)) if opt == "adam" else \
            np.full(max(steps, 1), HYPER[opt][0], np.float32)
        step_loss = torch.full((max(steps, 1),), 7.0, device="cuda")
        before = fpmcplus_routes()
        got = ops.fpmcplus_train_epoch(*dT, dev(users), dev(recent), dev(items), dev(third), bs, pairwise, kind, reg,
                                       0.0, opt, lr_t, HYPER[opt], grads, tch, dS0, dS1, first,
                                       ops.fpmcplus_work(d, w, L, bs), step_loss)
        assert got == steps
        want_t = [np.zeros(k, np.int32) for k in (nu, ni, ni)]
        want_loss = np.full(max(steps, 1), 7.0, np.float32)
        for s in range(steps):
            sl = slice(s * bs, min(n, (s + 1) * bs))
            l, g, t = fpmcplus_ref(H, users[sl], recent[sl], items[sl], third[sl], pairwise, kind, reg, 0.0)
            want_loss[s] = l
            assert want_loss[s] == l
            hyper = list(HYPER[opt])
            if opt == "adam":
                hyper[0] = lr_t[s]
            for k, (var, gk) in enumerate(zip(H, g)):
                assert exact32(gk), k
                tk = (t[0], t[1], t[1], t[2], None, None, None)[k]
                tf_math.opt_apply(opt, var, gk.astype(np.float32).reshape(var.shape), S0[k], S1[k], tk, hyper,
                                  dense_var=tk is None)
            for k, m in enumerate(t):
                want_t[k][m] = first + s
        for k in range(7):
            assert np.array_equal(host(dT[k]), H[k]), (n, k)
            for dsl, hsl in ((dS0[k], S0[k]), (dS1[k], S1[k])):
                if hsl is not None and not (opt == "momentum" and hsl is S1[k]):
                    assert np.array_equal(host(dsl), hsl), (n, k)
            assert not grads[k].any()
        for a, wt in zip(tch, want_t):
            assert np.array_equal(host(a), wt)
        assert np.array_equal(host(step_loss), want_loss)
        if n == 0:
            assert fpmcplus_routes() == before
        else:
            last = n - (steps - 1) * bs
            assert fpmcplus_routes()["grad"]["grid_x"] == fpmcplus_grad_grid(last, sms())[0]
    SEEN.add(("fpmcplus_epoch", pairwise, opt))


@gpu
@pytest.mark.parametrize("shape", PAIR_SHAPES + ["proj_below", "proj_above"])
def test_fpmcplus_scores_exact(shape):
    """The pair kernel at R = 8, 3 and 1 rows per CTA with a row count R does not divide and window lengths 1, 2, 4,
    ..., L; the projection pass on both sides of 4096 * SMs elements.  h sums to 0 against the saturated signs, so
    every exp(e) is exactly 1 and the scores are exact: bit for bit against float64."""
    from neurec_b200 import ops
    n_sms = sms()
    rs = np.random.RandomState(len(str(shape)) * 7 + (shape[0] if isinstance(shape, tuple) else 1))
    if isinstance(shape, tuple):
        d, w, L = shape
        ni, rows = 300, 3 * fpmcplus_pair_rows(d, w, L) + 2 if fpmcplus_pair_rows(d, w, L) > 1 else 5
    else:
        d, w, L = 2, 2, 2
        ni, rows = projection_shape(n_sms, shape == "proj_above")
        w = 1
    nu = max(rows, 4)
    tabs = fpmcplus_tables(rs, nu, ni, d, w)
    if w > 1:
        tabs[5][0, 0::2], tabs[5][0, 1::2] = 64.0, -64.0            # tanh +1 and -1 in pairs
        tabs[6][:] = 0.5                                            # equal h against +1 and -1: e = 0
        if w % 2:
            tabs[6][-1] = 0.0
    else:
        tabs[6][:] = 0.0                                            # e = 0
    users = np.arange(rows, dtype=np.int32) % nu
    lens = [1 << k for k in range(8) if (1 << k) <= L]
    recent = rs.randint(0, ni, (nu, L)).astype(np.int32)
    length = np.asarray([lens[u % len(lens)] for u in range(nu)], np.int32)
    length[0] = L if L & (L - 1) == 0 else length[0]
    windows = [recent[u, :length[u]] for u in users]
    want = fpm.fpmcplus_scores(*tabs, users, windows)
    got = host(ops.fpmcplus_scores(*[dev(t) for t in tabs], dev(users), dev(recent), dev(length)))
    assert exact32(want) and np.array_equal(got.astype(np.float64), want)
    r = fpmcplus_routes()
    R = fpmcplus_pair_rows(d, w, L)
    assert r["pair"] == dict(pairwise=-1, grid_x=-(-rows // R), grid_y=(ni + 255) // 256, capped=-1, window=L, rows=R)
    total = ni * (w + 2 * d) + rows * (1 + L) * w
    assert r["project"]["capped"] == int(elementwise_capped(total, n_sms))
    if isinstance(shape, tuple):
        assert rows % R != 0 or R == 1
        SEEN.add(("fpmcplus_pair", R))
    else:
        SEEN.add(("fpmcplus_project", r["project"]["capped"]))


# ---------------------------------------------------------------------------------------------------------------
# FISM: exact epochs
# ---------------------------------------------------------------------------------------------------------------
def fism_epoch_case(rs, n, bs, d, pairwise):
    """n samples, one history row each; step s reads c1 rows and targets of item block s only (block 128: histories
    from its first 64 items, and every positive's excluded item is a history item no other sample of the step has).
    -> tables, (hist_ptr, hist_idx), samples."""
    steps = max(1, -(-n // bs))
    ni = 128 * (steps + 1)
    s = np.arange(n) // bs
    hists, excl, items = [], np.full(n, -1, np.int32), np.zeros(n, np.int32)
    fresh = {}
    for k in range(n):
        base = 128 * s[k]
        h = list(base + rs.choice(64, rs.randint(0, 9), replace=False))
        items[k] = base + rs.randint(0, 128)
        if not pairwise and k % 2 == 0:
            j = fresh.setdefault(s[k], iter(base + 64 + rs.permutation(64)))
            e = int(next(j))
            h.insert(rs.randint(0, len(h) + 1), e)
            excl[k] = items[k] = e
        hists.append(np.asarray(h, np.int32))
    ptr = np.zeros(n + 1, np.int64)
    ptr[1:] = np.cumsum([len(h) for h in hists])
    idx = np.concatenate(hists + [np.zeros(0, np.int32)]).astype(np.int32)
    rows = np.arange(n, dtype=np.int32)
    num = np.asarray([len(h) for h in hists], np.int32) + 1
    c1, Q = dyadic(rs, (ni, d), -2, 2, 2, 0.5), dyadic(rs, (ni, d), -2, 2, 2, 0.5)
    b = dyadic(rs, (ni,), -2, 2, 2)
    if pairwise:
        third = np.zeros(n, np.int32)
        redo = np.ones(n, bool)
        for _ in range(100):
            third[redo] = (128 * s + rs.randint(0, 128, n))[redo]
            p = fm.history_matrix(ptr, idx, rows, None, ni, np.float64) @ c1.astype(np.float64)
            xd = (p * Q[items]).sum(1) + b[items] - (p * Q[third]).sum(1) - b[third]
            redo = xd == -1.0
            if not redo.any():
                break
        return (c1, Q, b), (ptr, idx), [rows, None, num, items, third, (num + 1).astype(np.int32)]
    third = rs.randint(0, 2, n).astype(np.float32)
    return (c1, Q, b), (ptr, idx), [rows, None if n == 0 else excl, num, items, third, None]


@gpu
@pytest.mark.parametrize("opt", OPTS)
@pytest.mark.parametrize("pairwise,kind", [(0, "square"), (1, "hinge")])
def test_fism_epoch_exact(pairwise, kind, opt):
    """alpha = 0, lambda and gamma 1/4 and 1/8, a short last batch, batch_size > n, n = 0, first_stamp > 1: c1, Q, b,
    their slots, both touched stamps and every step's loss bit for bit against fism_math in float64 and
    tf_math.opt_apply; the accumulators end zeroed.  An excluded item's c1 row takes neither a gradient nor a stamp."""
    from neurec_b200 import ops
    rs = np.random.RandomState(OPTS.index(opt) * 2 + pairwise + 50)
    d, lam, gamma = 12, 0.25, 0.125
    for n, bs, first in ((3 * 64 + 5, 64, 7), (5, 64, 1), (0, 64, 3)):
        steps = -(-n // bs)
        tabs, (ptr, idx), arrs = fism_epoch_case(rs, n, bs, d, pairwise)
        ni = tabs[0].shape[0]
        i0, i1 = tf_math.SLOT_INIT[opt]
        H = [a.copy() for a in tabs]
        S0 = [None if i0 is None else np.full_like(a, i0) for a in tabs]
        S1 = [None if i1 is None else np.full_like(a, i1) for a in tabs]
        dT, dS0, dS1 = [dev(a) for a in tabs], [dev(a) for a in S0], [dev(a) for a in S1]
        grads = [torch.zeros_like(t) for t in dT]
        tch = [torch.zeros(ni, dtype=torch.int32, device="cuda") for _ in range(2)]
        lr_t = tf_math.adam_lr_t(HYPER["adam"][0], max(steps, 1)) if opt == "adam" else \
            np.full(max(steps, 1), HYPER[opt][0], np.float32)
        step_loss = torch.full((max(steps, 1),), 7.0, device="cuda")
        before = ops.fism_last_routes()
        got = ops.fism_train_epoch(*dT, dev(ptr), dev(idx), *[dev(a) for a in arrs], bs, pairwise, kind, 0.0, lam,
                                   gamma, opt, lr_t, HYPER[opt], grads, tch, dS0, dS1, first, step_loss)
        assert got == steps
        want_t = [np.zeros(ni, np.int32) for _ in range(2)]
        want_loss = np.full(max(steps, 1), 7.0, np.float32)
        rows, excl, num, items, third, num_neg = arrs
        for s in range(steps):
            sl = slice(s * bs, min(n, (s + 1) * bs))
            l, g, (tC, tI) = fm.loss_and_grad(*H, ptr, idx, rows[sl], None if excl is None else excl[sl], num[sl],
                                              items[sl], third[sl], None if num_neg is None else num_neg[sl],
                                              pairwise, kind, 0.0, lam, gamma, dtype=np.float64)
            want_loss[s] = l
            assert want_loss[s] == l
            hyper = list(HYPER[opt])
            if opt == "adam":
                hyper[0] = lr_t[s]
            for k, (var, gk, tk) in enumerate(zip(H, g, (tC, tI, tI))):
                assert exact32(gk), k
                tf_math.opt_apply(opt, var, gk.astype(np.float32).reshape(var.shape), S0[k], S1[k], tk, hyper)
            want_t[0][tC] = first + s
            want_t[1][tI] = first + s
            if excl is not None:                      # the excluded rows the step does not otherwise read
                ex = excl[sl][excl[sl] >= 0]
                assert ex.size and not tC[ex].any()
        for k in range(3):
            assert np.array_equal(host(dT[k]), H[k]), (n, k)
            for dsl, hsl in ((dS0[k], S0[k]), (dS1[k], S1[k])):
                if hsl is not None and not (opt == "momentum" and hsl is S1[k]):
                    assert np.array_equal(host(dsl), hsl), (n, k)
            assert not grads[k].any()
        for a, wt in zip(tch, want_t):
            assert np.array_equal(host(a), wt)
        assert np.array_equal(host(step_loss), want_loss)
        if n == 0:
            assert ops.fism_last_routes() == before
        else:
            assert ops.fism_last_routes()["grad"]["pairwise"] == pairwise
    SEEN.add(("fism_epoch", pairwise, opt))


# ---------------------------------------------------------------------------------------------------------------
# rounded cases: every entry within a first-order bound of float64
# ---------------------------------------------------------------------------------------------------------------
# The float64 references below follow the kernels' chains with R (test_gpu_seq_routes): each value carries m, a
# first-order bound on its fp32 rounding error in units of 2^-24, built from the absolute values of the same graph.
# Every chain a kernel sums in one loop is summed here in one R.sum over all its terms, and the transcendental ops carry
# their documented CUDA error (expf, tanhf: 2 ulp; logf: 1 ulp).  Each compared entry must lie within C_BOUND * 2^-24
# * m of float64; no relu, max or hinge decision may sit within rounding of its threshold (checked on the reference).
C_BOUND = 2.0


def rdiv(a, b):
    a, b = R.of(a), R.of(b)
    v = a.v / b.v
    return R(v, a.m / np.abs(b.v) + np.abs(a.v) * b.m / b.v ** 2 + np.abs(v))


def rexp(x):
    v = np.exp(x.v)
    return R(v, v * x.m + 4 * v)


def rtanh(x):
    v = np.tanh(x.v)
    return R(v, (1 - v * v) * x.m + 4 * np.abs(v))


def rlog(x):
    v = np.log(x.v)
    return R(v, x.m / x.v + 2 * np.abs(v))


def rsum(parts, axis):
    """One fp32 chain over every term of `parts` (concatenated along `axis`)."""
    return cat(parts, axis).sum(axis)


class Undecided(AssertionError):
    """A decision within rounding of its threshold; .rows: the samples (first axis) that hold one."""

    def __init__(self, what, rows):
        super().__init__(what, rows)
        self.rows = rows


def assert_decided(v, m, what):
    """A relu / hinge / max decision at 0 is exact (v == 0) or clear of the rounding of v."""
    v, m = np.asarray(v), np.broadcast_to(m, np.shape(v))
    bad = ~((v == 0) | (np.abs(v) > 4 * C_BOUND * U24 * m))
    if bad.any():
        raise Undecided(what, np.unique(np.nonzero(bad)[0]))


def assert_bounded(got, want, what):
    err = np.abs(np.asarray(got, np.float64) - want.v)
    bound = C_BOUND * U24 * np.broadcast_to(want.m, want.v.shape)
    assert (err <= bound).all(), (what, float((err - bound).max()), float(np.max(want.m)))


def rrelu(x, what):
    assert_decided(x.v, x.m, what)
    return where(x.v > 0, x)


def caser_ref(P, E, W2, b2, dense, d, L, nv, nh, users, seqs, pos, neg, mask, keep):
    """nrc_caser_grad's chain in R -> (loss, [gP, gE, gW2, gb2, gdense])."""
    V = {k: v.astype(np.float64) for k, v in cm.unpack(dense.astype(np.float64), d, L, nv, nh).items()}
    I = E.shape[0]
    Ez = np.concatenate([E.astype(np.float64), np.zeros((1, d))])
    X = R(Ez[seqs])                                                   # [B, L, d]
    B, T, N = len(users), pos.shape[1], neg.shape[1]
    Kv = V["Kv"].reshape(L, nv)
    out_v = rsum([R(X.v[:, :, :, None]) * R(Kv[None, :, None, :]), R(np.broadcast_to(V["bv"], (B, 1, d, nv)))], 1)
    out_v = R(out_v.v.reshape(B, d * nv), out_v.m.reshape(B, d * nv))
    pooled, pools = [], []
    for h in range(1, L + 1):
        Kh = V["Kh%d" % h].reshape(h * d, nh)
        pre = []
        for t in range(L - h + 1):
            xs = X.v[:, t:t + h].reshape(B, h * d)
            pre.append(rsum([R(xs[:, :, None]) * R(Kh[None]), R(np.broadcast_to(V["bh%d" % h], (B, 1, nh)))], 1))
        a = rrelu(cat([R(p.v[:, None], p.m[:, None]) for p in pre], 1), ("conv_h", h))     # [B, np, nh]
        mx = a.v.max(1, keepdims=True)
        tied = a.v == mx
        assert_decided(np.where(tied, 1.0, mx - a.v), a.m + np.max(np.where(tied, a.m, 0), 1, keepdims=True),
                       ("max", h))
        pooled.append(R(mx[:, 0], np.max(np.where(tied, a.m, 0), 1)))
        pools.append((a, tied))
    feat = cat([out_v] + pooled, 1)
    mk = np.ones_like(feat.v) if mask is None else np.asarray(mask, np.float64)
    o = (feat / keep) * R(mk) if mask is not None else feat
    W1, b1 = V["W1"], V["b1"]
    zp = rsum([R(o.v[:, :, None], o.m[:, :, None]) * R(W1[None]), R(np.broadcast_to(b1, (B, 1, d)))], 1)
    z = rrelu(zp, "z")
    Pu = R(P.astype(np.float64)[users])
    u = cat([z, Pu], 1)
    tgt = np.concatenate([pos, neg], 1)
    real = tgt != I
    W2z = np.concatenate([W2.astype(np.float64), np.zeros((1, 2 * d))])
    b2z = np.concatenate([b2.astype(np.float64), [0.0]])
    x = rsum([R(u.v[:, None, :], u.m[:, None, :]) * R(W2z[tgt]), R(b2z[tgt][:, :, None])], 2)
    x = where(real, x, 0.0)
    s = rdiv(1.0, 1.0 + rexp(-x))
    inv_bt, inv_bn = R(1.0 / (B * T), 1.0 / (B * T)), R(1.0 / (B * N), 1.0 / (B * N))
    sp, sn = s[:, :T], s[:, T:]
    lp = -rlog(sp + 1e-24) * inv_bt
    ln = -rlog((1.0 - sn) + 1e-24) * inv_bn
    loss = cat([lp, ln], 1).sum(1).sum(0)
    cp = ((-inv_bt) * rdiv(1.0, sp + 1e-24)) * sp * (1.0 - sp)
    cn = (inv_bn * rdiv(1.0, (1.0 - sn) + 1e-24)) * sn * (1.0 - sn)
    c = cat([cp, cn], 1)                                              # [B, T + N]
    cu = R(c.v[:, :, None], c.m[:, :, None]) * R(u.v[:, None, :], u.m[:, None, :])
    gW2 = scatter(I, [(tgt[real], R(cu.v[real], cu.m[real]))])
    gb2 = scatter(I, [(tgt[real], R(c.v[real], c.m[real]))])
    du = (R(c.v[:, :, None], c.m[:, :, None]) * R(W2z[tgt])).sum(1)   # pad terms are 0
    gP = scatter(P.shape[0], [(users, du[:, d:])])
    dz = where(z.v > 0, du[:, :d])
    g = {"W1": (R(o.v[:, :, None], o.m[:, :, None]) * R(dz.v[:, None, :], dz.m[:, None, :])).sum(0),
         "b1": dz.sum(0)}
    do = (R(W1[None]) * R(dz.v[:, None, :], dz.m[:, None, :])).sum(2)
    dfeat = (do * R(mk)) / keep if mask is not None else do
    dv = R(dfeat.v[:, :nv * d].reshape(B, d, nv), dfeat.m[:, :nv * d].reshape(B, d, nv))
    g["Kv"] = (R(X.v[:, :, :, None]) * R(dv.v[:, None], dv.m[:, None])).sum(2).sum(0)   # per sample over k, then b
    g["bv"] = dv.sum(1).sum(0)
    terms = [R(dv.v[:, None, :, :], dv.m[:, None, :, :]) * R(Kv[None, :, None, :])]   # [B, L, d, nv]
    for h in range(1, L + 1):
        a, tied = pools[h - 1]
        gh = dfeat[:, nv * d + (h - 1) * nh:nv * d + h * nh]
        cnt = tied.sum(1, keepdims=True)
        inv = R(1.0 / cnt, np.where(cnt & (cnt - 1) == 0, 0.0, 1.0 / cnt))
        dpre = where(tied & (a.v > 0), inv * R(gh.v[:, None, :], gh.m[:, None, :]))      # [B, np, nh]
        Kh = V["Kh%d" % h].reshape(h, d, nh)
        prods = R(np.stack([X.v[:, l:l + L - h + 1] for l in range(h)], 1)[..., None]) * \
            R(dpre.v[:, None, :, None, :], dpre.m[:, None, :, None, :])                  # [B, h, np, d, nh]
        flat = R(prods.v.transpose(1, 3, 4, 0, 2).reshape(h, d, nh, -1), prods.m.transpose(1, 3, 4, 0, 2)
                 .reshape(h, d, nh, -1))
        g["Kh%d" % h] = flat.sum(3)
        g["bh%d" % h] = R(dpre.v.reshape(B * (L - h + 1), nh), dpre.m.reshape(B * (L - h + 1), nh)).sum(0)
        for t in range(L - h + 1):                                     # window row t + l takes dpre[t] Kh[l]
            q = R(dpre.v[:, t][:, None, None, :], dpre.m[:, t][:, None, None, :]) * R(Kh[None])  # [B, h, d, nh]
            pad = np.zeros((B, L, d, nh))
            pv, pm = pad.copy(), pad.copy()
            pv[:, t:t + h], pm[:, t:t + h] = q.v, q.m
            terms.append(R(pv, pm))
    dX = rsum(terms, 3)                                                # [B, L, d]
    live = seqs != I
    gE = scatter(I, [(seqs[live], R(dX.v[live], dX.m[live]))])
    gd = cm.pack({k: v.v for k, v in g.items()}, d, L, nv, nh)
    gdm = cm.pack({k: np.broadcast_to(v.m, v.v.shape) for k, v in g.items()}, d, L, nv, nh)
    return loss, [gP, gE, gW2, gb2, R(gd, gdm)]


def fpmcplus_rref(tabs, users, recent, items, third, pairwise, kind, reg, reg_w):
    """nrc_fpmcplus_grad's chain in R -> (loss, [gUI, gIU, gIL, gLI, gW, gb, gh])."""
    UI, IU, IL, LI, W, b, h = [t.astype(np.float64) for t in tabs]
    b, h = b.reshape(-1), h.reshape(-1)
    B, L = recent.shape
    D, w = UI.shape[1], W.shape[1]
    WU, WI, WL = W[:D], W[D:2 * D], W[2 * D:]
    a = UI[users]
    Rl = LI[recent]                                                   # [B, L, D]

    def proj(x, Wb, bias=None):                                       # x [..., D] @ Wb [D, w] (+ bias)
        xv = x.v if isinstance(x, R) else x
        xm = x.m if isinstance(x, R) else np.zeros_like(xv)
        p = R(xv[..., :, None], xm[..., :, None]) * R(Wb)
        if bias is not None:
            return rsum([p, R(np.broadcast_to(bias, p.v.shape[:-2] + (1, w)))], -2)
        return p.sum(-2)

    A = proj(a, WU, b)                                                # [B, w]
    C = proj(Rl, WL)                                                  # [B, L, w]

    def side(item):
        il = IL[item]
        Bi = proj(il, WI)
        z = (R(A.v[:, None], A.m[:, None]) + R(Bi.v[:, None], Bi.m[:, None])) + C
        t = rtanh(z)                                                  # [B, L, w]
        e = (R(h[None, None]) * t).sum(2)                             # [B, L]
        ex = rexp(e)
        att = rdiv(ex, ex.sum(1)[:, None])
        q = (R(il[:, None, :]) * R(Rl)).sum(2)                        # [B, L]
        y = (att * q).sum(1)
        x = rsum([R(a) * R(IU[item]), R(y.v[:, None], y.m[:, None])], 1)
        return dict(il=il, iu=IU[item], t=t, att=att, q=q, y=y, x=x, item=item)

    S = [side(items)]
    if pairwise:
        S.append(side(third))
        x = S[0]["x"] - S[1]["x"]
        if kind == "hinge":
            assert_decided(x.v + 1.0, x.m, "hinge")
        lo, c = pair_loss(kind, x)
    else:
        lo, c = point_loss(kind, S[0]["x"], third)
    sq = cat([R(a) * R(a), (R(Rl) * R(Rl)).sum(1)] + [R(sd[k]) * R(sd[k]) for sd in S for k in ("iu", "il")], 1)
    loss = lo + (reg * 0.5) * sq.sum(1) if reg else lo
    sign = [1.0, -1.0]
    zs, gls, gh_terms, si = [], [], [], []
    for k, sd in enumerate(S):
        cs = c * sign[k]
        de = R(cs.v[:, None], cs.m[:, None]) * sd["att"] * (sd["q"] - R(sd["y"].v[:, None], sd["y"].m[:, None]))
        one_t2 = 1.0 - sd["t"] * sd["t"]
        dz = (R(de.v[:, :, None], de.m[:, :, None]) * R(h[None, None])) * one_t2      # [B, L, w]
        zs.append(dz.sum(1))
        gls.append(dz)
        gh_terms.append(R(de.v[:, :, None], de.m[:, :, None]) * sd["t"])
        si.append((R(sd["att"].v[:, :, None], sd["att"].m[:, :, None]) * R(Rl)).sum(1))   # [B, D]
    gA = zs[0] + zs[1] if pairwise else zs[0]
    gL = gls[0] + gls[1] if pairwise else gls[0]
    flat = lambda r: R(r.v.reshape(-1, *r.v.shape[2:]), r.m.reshape(-1, *r.m.shape[2:]))
    gWU = (R(a[:, :, None]) * R(gA.v[:, None], gA.m[:, None])).sum(0)
    gWI = rsum([R(S[k]["il"][:, :, None]) * R(zs[k].v[:, None], zs[k].m[:, None]) for k in range(len(S))], 0)
    gWL = (R(Rl[..., None]) * R(gL.v[:, :, None], gL.m[:, :, None]))
    gWL = flat(gWL).sum(0)
    gW = cat([gWU, gWI, gWL], 0)
    gb = gA.sum(0)
    gh = rsum([flat(x_) for x_ in gh_terms], 0)
    if pairwise and reg_w:
        gW = gW + reg_w * R(W)
        gh = gh + reg_w * R(h)
    back = lambda g, Wb: (R(Wb[None]) * R(g.v[..., None, :], g.m[..., None, :])).sum(-1)   # Wb [D, w] g [.., w]
    vU = back(gA, WU)
    c1 = R(c.v[:, None], c.m[:, None])
    ui = S[0]["iu"]
    if pairwise:
        uj = S[1]["iu"]
        gUI = (c1 * (R(ui) - R(uj)) + vU) + reg * R(a)
        gIU = [(S[0]["item"], c1 * R(a) + reg * R(ui)), (S[1]["item"], -c1 * R(a) + reg * R(uj))]
    else:
        gUI = (c1 * R(ui) + vU) + reg * R(a)
        gIU = [(S[0]["item"], c1 * R(a) + reg * R(ui))]
    gIL = [(S[k]["item"], ((c1 * sign[k]) * si[k] + back(zs[k], WI)) + reg * R(S[k]["il"])) for k in range(len(S))]
    gli = c1[:, None] * (R(S[0]["att"].v[..., None], S[0]["att"].m[..., None]) * R(S[0]["il"][:, None]))
    if pairwise:
        gli = gli - c1[:, None] * (R(S[1]["att"].v[..., None], S[1]["att"].m[..., None]) * R(S[1]["il"][:, None]))
    gLIrows = (gli + back(gL, WL)) + reg * R(Rl)
    nu, ni = UI.shape[0], IU.shape[0]
    g = [scatter(nu, [(users, gUI)]), scatter(ni, gIU), scatter(ni, gIL), scatter(ni, [(recent.ravel(), flat(gLIrows))]),
         gW, gb, gh]
    total = loss.sum(0)
    if pairwise and reg_w:
        total = total + reg_w * (0.5 * (R(W) * R(W)).sum(1).sum(0) + 0.5 * (R(h) * R(h)).sum(0))
    return total, g


def gaussian_caser(rs, nu, ni, d, L, nv, nh):
    P, E = (rs.randn(nu, d) * 0.3).astype(np.float32), (rs.randn(ni, d) * 0.3).astype(np.float32)
    W2, b2 = (rs.randn(ni, 2 * d) * 0.3).astype(np.float32), (rs.randn(ni) * 0.1).astype(np.float32)
    parts = {}
    for name, _, shape in cm.dense_layout(d, L, nv, nh)[0]:
        fan = int(np.prod(shape[:-1])) if len(shape) > 1 else 1
        parts[name] = rs.randn(*shape) * (1.0 / np.sqrt(fan)) + (0.05 if len(shape) == 1 else 0.0)
    return P, E, W2, b2, cm.pack(parts, d, L, nv, nh).astype(np.float32)


# d, L, nv, nh, T, N, B ("cap+1": 2 * SMs + 1)
CASER_ROUNDED = [(7, 1, 2, 3, 3, 3, 33), (8, 2, 2, 2, 3, 3, 70), (50, 5, 4, 16, 3, 3, "cap+1"),
                 (8, 16, 2, 3, 1, 2, 20), ("staged", 2, 2, 9), ("unstaged", 2, 2, 9)]


@gpu
@pytest.mark.parametrize("ci", range(len(CASER_ROUNDED)))
def test_caser_grad_rounded(ci):
    """Gaussian tables and weights, keep 1/2, windows 1, 2, 5 and 16 with pads, 33, 70 and 2 * SMs + 1 samples, the
    largest staged and the smallest unstaged dense block: every entry of every gradient and the loss within the
    first-order bound of the float64 chain (sigmoid away from 1/2, so each side's derivative shows)."""
    n_sms = sms()
    case = CASER_ROUNDED[ci]
    if case[0] in ("staged", "unstaged"):
        d, L, nv, nh = caser_smem_boundary()[case[0] == "unstaged"]
        T, N, B = case[1:]
    else:
        d, L, nv, nh, T, N, B = case
        B = 2 * n_sms + 1 if B == "cap+1" else B
    rs = np.random.RandomState(300 + ci)
    nu, ni = 40, 97
    tabs = gaussian_caser(rs, nu, ni, d, L, nv, nh)
    users = rs.randint(0, nu, B).astype(np.int32)
    seqs = rs.randint(0, ni, (B, L)).astype(np.int32)
    pos, neg = rs.randint(0, ni, (B, T)).astype(np.int32), rs.randint(0, ni, (B, N)).astype(np.int32)
    seqs[0, :L - 1] = ni
    pos[0, 0] = ni
    if B > 2:
        seqs[2] = ni
    keep = 0.5
    mask = (rs.rand(B, nv * d + nh * L) < keep).astype(np.float32)
    for _ in range(20):                       # redraw the windows of samples with a decision within rounding
        try:
            want_l, want = caser_ref(*tabs, d, L, nv, nh, users, seqs, pos, neg, mask, keep)
            break
        except Undecided as e:
            assert not (B > 2 and 2 in e.rows), e.args
            for b in e.rows:
                seqs[b, 0 if b else L - 1:] = rs.randint(0, ni, L if b else 1)
    else:
        raise AssertionError("no decided windows")
    lo, got = caser_device_grad(tabs, (users, seqs, pos, neg), nv, nh, mask, keep)
    for name, g, w in zip(("P", "E", "W2", "b2", "dense"), got, want):
        assert_bounded(g.reshape(w.v.shape), w, name)
    assert_bounded(lo, want_l, "loss")
    r = caser_routes()
    cap = 2 * n_sms
    staged = caser_staged(d, L, nv, nh)
    assert r["grad"] == dict(staged=int(staged), grid_x=min(B, cap), grid_y=-1, capped=int(B > cap), window=L,
                             masked=1)
    assert r["wgrad"]["grid_y"] == (B + 31) // 32
    SEEN.add(("caser_rounded", int(staged), int(B > cap), L))


# pairwise, loss, d, w, L, B ("cap+1": 64 * SMs + 1)
FPMCPLUS_ROUNDED = [(1, "bpr", 16, 16, 3, "cap+1"), (1, "hinge", 33, 40, 2, 300), (1, "square", 16, 16, 64, 50),
                    (0, "cross_entropy", 16, 16, 3, "cap+1"), (0, "square", 8, 8, 1, 100),
                    (1, "bpr", 32, 128, 64, 20), (0, "cross_entropy", 5, 4, 1, 1), (1, "hinge", 7, 5, 1, "cap+1")]


@gpu
@pytest.mark.parametrize("pairwise,kind,d,w,L,B", FPMCPLUS_ROUNDED)
def test_fpmcplus_grad_rounded(pairwise, kind, d, w, L, B):
    """Gaussian tables and attention MLP (tanh' and the softmax weights away from their exact values) under every
    loss, windows 1, 2, the conf's 3 and 64, on both sides of 64 * SMs: every entry of the seven gradients and the
    loss within the first-order bound of the float64 chain."""
    from neurec_b200 import ops
    n_sms = sms()
    B = 64 * n_sms + 1 if B == "cap+1" else B
    rs = np.random.RandomState(d + w + L + len(kind) + pairwise)
    nu, ni = 200, 300
    tabs = [(rs.randn(n, d) * 0.3).astype(np.float32) for n in (nu, ni, ni, ni)]
    tabs += [(rs.randn(3 * d, w) / np.sqrt(d)).astype(np.float32), (rs.randn(1, w) * 0.3).astype(np.float32),
             (rs.randn(w, 1) * 0.5 + 1.0).astype(np.float32)]
    users, items = rs.randint(0, nu, B).astype(np.int32), rs.randint(0, ni, B).astype(np.int32)
    recent = rs.randint(0, ni, (B, L)).astype(np.int32)
    third = rs.randint(0, ni, B).astype(np.int32) if pairwise else (rs.rand(B) < 0.3).astype(np.float32)
    reg, reg_w = float(np.float32(0.01)), float(np.float32(0.05))
    for _ in range(20):                       # redraw the negatives of samples on the hinge's tie
        try:
            want_l, want = fpmcplus_rref(tabs, users, recent, items, third, pairwise, kind, reg, reg_w)
            break
        except Undecided as e:
            third[e.rows] = rs.randint(0, ni, len(e.rows))
    else:
        raise AssertionError("no decided negatives")
    dt = [dev(t) for t in tabs]
    g = [torch.zeros_like(t) for t in dt]
    tch = [torch.zeros(n, dtype=torch.int32, device="cuda") for n in (nu, ni, ni)]
    lo = torch.zeros(1, device="cuda")
    ops.fpmcplus_grad(*dt, dev(users), dev(recent), dev(items), dev(third), pairwise, kind, reg, reg_w, g, tch, 9,
                      ops.fpmcplus_work(d, w, L, B), lo)
    for k, (a, ref) in enumerate(zip(g, want)):
        assert_bounded(host(a).reshape(ref.v.shape), ref, k)
    assert_bounded(float(lo), want_l, "loss")
    grid, capped = fpmcplus_grad_grid(B, n_sms)
    r = fpmcplus_routes()
    assert r["grad"] == dict(pairwise=pairwise, grid_x=grid, grid_y=-1, capped=int(capped), window=L, rows=-1)
    SEEN.add(("fpmcplus_rounded", pairwise, kind, L, int(capped)))


# ---------------------------------------------------------------------------------------------------------------
# limits and errors: the library's error, nothing written, the hooks unchanged
# ---------------------------------------------------------------------------------------------------------------
@gpu
def test_limits_and_errors_write_nothing():
    from neurec_b200 import _lib, ops
    from neurec_b200.ops import _p, _stream
    lib = _lib.load()
    E_LIMIT, E_VALUE = _lib.NRC_E_LIMIT, _lib.NRC_E_VALUE
    D = 8
    tabs = [dev(np.ones((6, 3 * D), np.float32)) for _ in range(7)]
    gr = [torch.zeros_like(t) for t in tabs]
    tch = [torch.zeros(6, dtype=torch.int32, device="cuda") for _ in range(3)]
    ids, win = dev(np.zeros(4, np.int32)), dev(np.zeros((4, 65), np.int32))
    lab = dev(np.zeros(4, np.float32))
    ptr = dev(np.array([0, 1, 2, 3, 4, 4, 4], np.int64))
    loss = torch.zeros(1, device="cuda")
    work = torch.zeros(1 << 16, device="cuda")
    out = torch.zeros((4, 2 * D), device="cuda")
    step_loss = torch.zeros(4, device="cuda")
    watched = tabs + gr + tch + [loss, out, work, step_loss]
    h = np.array([0.1, 0.9, 0.999, 1e-8], np.float32)
    slots = (ctypes.c_void_p * 7)(*[t.data_ptr() for t in tabs])
    P = lambda k: _p(tabs[k])
    G = lambda k: _p(gr[k])
    routes = lambda: (ops.caser_last_routes(), ops.fpmcplus_last_routes(), ops.fism_last_routes())

    def unchanged(code, fn):
        snap = [t.clone() for t in watched]
        before = routes()
        rc = fn()
        torch.cuda.synchronize()
        assert rc == code, (rc, lib.nrc_last_error())
        assert routes() == before
        for a, b in zip(watched, snap):
            assert torch.equal(a, b)

    # Caser: dim, L, filters, targets, batch chunks, keep; the epoch's keep and batch size; the query's L and rows
    caser = lambda dim=D, L=2, T=1, nv=1, nh=1, N=1, batch=4, mask=None, keep=1.0: lib.nrc_caser_grad(
        P(0), P(1), P(2), P(3), P(4), 6, dim, L, T, nv, nh, N, _p(ids), _p(win), _p(ids), _p(ids), batch, mask, keep,
        G(0), G(1), G(2), G(3), G(4), _p(work), _p(loss), _stream())
    for kw, code in ((dict(dim=0), E_LIMIT), (dict(dim=257), E_LIMIT), (dict(L=0), E_LIMIT), (dict(L=17), E_LIMIT),
                     (dict(nv=0), E_LIMIT), (dict(nv=65), E_LIMIT), (dict(nh=0), E_LIMIT), (dict(nh=65), E_LIMIT),
                     (dict(T=0), E_VALUE), (dict(N=0), E_VALUE), (dict(T=33, N=32), E_LIMIT),
                     (dict(batch=65535 * 32 + 1), E_LIMIT), (dict(batch=-1), E_VALUE),
                     (dict(mask=_p(lab), keep=0.0), E_VALUE), (dict(mask=_p(lab), keep=1.5), E_VALUE)):
        unchanged(code, lambda: caser(**kw))
    unchanged(_lib.NRC_OK, lambda: caser(batch=0))
    ce = lambda keep=0.5, bs=2, L=2: lib.nrc_caser_train_epoch(
        P(0), P(1), P(2), P(3), P(4), 6, 6, D, L, 1, 1, 1, 1, _p(ids), _p(win), _p(ids), _p(ids), 4, bs, keep, 0.1,
        1, 1, h.ctypes.data, h.ctypes.data, G(0), G(1), G(2), G(3), G(4), slots, slots, _p(work), _p(step_loss),
        _stream())
    unchanged(E_VALUE, lambda: ce(keep=0.0))
    unchanged(E_VALUE, lambda: ce(bs=0))
    unchanged(E_LIMIT, lambda: ce(bs=65535 * 32 + 1))
    unchanged(E_LIMIT, lambda: ce(L=17))
    unchanged(E_LIMIT, lambda: lib.nrc_caser_query(P(0), P(1), P(4), 6, D, 17, 1, 1, _p(ids), 4, _p(win), _p(out),
                                                   _stream()))
    unchanged(E_VALUE, lambda: lib.nrc_caser_query(P(0), P(1), P(4), 6, D, 2, 1, 1, _p(ids), -1, _p(win), _p(out),
                                                   _stream()))
    # FPMCplus: dim, weight_size, window, loss of the mode, batch chunks, NULL work; the epoch; the scores
    fp = lambda dim=D, w=4, L=2, pw=1, kind="hinge", batch=4, wk=True: lib.nrc_fpmcplus_grad(
        P(0), P(1), P(2), P(3), P(4), P(5), P(6), dim, w, L, _p(ids), _p(win), _p(ids), _p(ids), batch, pw,
        _lib.LOSS_IDS[kind], 0.1, 0.1, G(0), G(1), G(2), G(3), G(4), G(5), G(6), _p(tch[0]), _p(tch[1]), _p(tch[2]), 3,
        _p(work) if wk else None, _p(loss), _stream())
    for kw, code in ((dict(dim=0), E_LIMIT), (dict(dim=257), E_LIMIT), (dict(w=0), E_LIMIT), (dict(w=129), E_LIMIT),
                     (dict(L=0), E_LIMIT), (dict(L=65), E_LIMIT), (dict(pw=0, kind="hinge"), E_VALUE),
                     (dict(pw=1, kind="cross_entropy"), E_VALUE), (dict(batch=65535 * 32 + 1), E_LIMIT),
                     (dict(wk=False), E_VALUE)):
        unchanged(code, lambda: fp(**kw))
    fe = lambda bs=2, opt=0: lib.nrc_fpmcplus_train_epoch(
        P(0), P(1), P(2), P(3), P(4), P(5), P(6), 6, 6, D, 4, 2, _p(ids), _p(win), _p(ids), _p(ids), 4, bs, 1,
        _lib.LOSS_IDS["hinge"], 0.1, 0.1, opt, h.ctypes.data, h.ctypes.data, G(0), G(1), G(2), G(3), G(4), G(5), G(6),
        _p(tch[0]), _p(tch[1]), _p(tch[2]), slots, slots, 1, _p(work), _p(step_loss), _stream())
    unchanged(E_LIMIT, lambda: fe(bs=65535 * 32 + 1))
    unchanged(E_VALUE, lambda: fe(opt=99))
    for n_items, dim, rows, code in ((65535 * 256 + 1, D, 4, E_LIMIT), (6, 0, 4, E_LIMIT), (6, D, -1, E_VALUE)):
        unchanged(code, lambda: lib.nrc_fpmcplus_scores(P(0), P(1), P(2), P(3), P(4), P(5), P(6), n_items, dim, 4, 2,
                                                        _p(ids), rows, _p(win), _p(ids), _p(work), _p(out), _stream()))
    # FISM: dim, the loss of each mode, alpha, num_items, NULL num_neg; the epoch's optimizer and batch size; query
    fg = lambda dim=D, pw=0, kind="square", alpha=0.5, ni=6, nn=True: lib.nrc_fism_grad(
        P(0), P(1), P(2), ni, dim, _p(ptr), _p(ids), _p(ids), None, _p(ids), _p(ids), _p(ids) if pw else _p(lab),
        _p(ids) if nn else None, 4, pw, _lib.LOSS_IDS[kind], alpha, 0.1, 0.1, G(0), G(1), G(2), _p(tch[0]),
        _p(tch[1]), 3, _p(loss), _stream())
    for kw, code in ((dict(dim=0), E_LIMIT), (dict(dim=257), E_LIMIT), (dict(pw=0, kind="hinge"), E_VALUE),
                     (dict(pw=0, kind="bpr"), E_VALUE), (dict(pw=1, kind="cross_entropy"), E_VALUE),
                     (dict(alpha=float("inf")), E_VALUE), (dict(alpha=float("nan")), E_VALUE), (dict(ni=0), E_VALUE),
                     (dict(pw=1, kind="bpr", nn=False), E_VALUE)):
        unchanged(code, lambda: fg(**kw))
    fie = lambda bs=2, opt=0, dim=D: lib.nrc_fism_train_epoch(
        P(0), P(1), P(2), 6, dim, _p(ptr), _p(ids), _p(ids), None, _p(ids), _p(ids), _p(lab), None, 4, bs, 0,
        _lib.LOSS_IDS["square"], 0.5, 0.1, 0.1, opt, h.ctypes.data, h.ctypes.data, G(0), G(1), G(2), _p(tch[0]),
        _p(tch[1]), slots, slots, 1, _p(step_loss), _stream())
    unchanged(E_VALUE, lambda: fie(opt=99))
    unchanged(E_VALUE, lambda: fie(bs=0))
    unchanged(E_LIMIT, lambda: fie(dim=257))
    unchanged(E_LIMIT, lambda: lib.nrc_fism_query(P(0), 6, 257, _p(ptr), _p(ids), _p(ids), 4, _p(out), _stream()))
    unchanged(E_VALUE, lambda: lib.nrc_fism_query(P(0), 6, D, _p(ptr), _p(ids), _p(ids), -1, _p(out), _stream()))
    unchanged(E_VALUE, lambda: lib.nrc_fism_scores(P(0), P(1), P(2), 6, D, float("nan"), _p(ptr), _p(ids), 4,
                                                   _p(out), _stream()))
    SEEN.add(("limits", 1))


# ---------------------------------------------------------------------------------------------------------------
# the exact constructions against torch.autograd (CPU)
# ---------------------------------------------------------------------------------------------------------------
def test_exact_constructions_match_autograd():
    """CPU: the zero-logit Caser batch and the saturated FPMCplus batch are what the exact GPU tests say they are --
    every Caser sigmoid is 1/2 and every FPMCplus attention weight is 1/L with tanh' = 0 -- and on them the float64
    restatements equal torch.autograd exactly (Caser) and to rounding (FPMCplus, whose W and h gradients are exactly
    the reg term)."""
    from test_caser import _autograd as caser_autograd
    from test_fpmcplus import _autograd as fpmcplus_autograd
    rs = np.random.RandomState(3)
    d, L, nv, nh, T, N, B, keep = 4, 4, 2, 2, 2, 2, 8, 0.5
    mask = (rs.rand(B, nv * d + nh * L) < 0.5).astype(np.float32)
    tabs, batch, ties = caser_case(rs, d, L, nv, nh, T, N, B, mask, keep)
    t64 = [t.astype(np.float64) for t in tabs]
    f = cm.forward(*t64[:2], t64[4], d, L, nv, nh, *batch[:2], mask, keep)
    tgt = np.concatenate(batch[2:], 1)
    real = tgt != tabs[1].shape[0]
    x = np.einsum("bk,bjk->bj", f["u"], np.concatenate([t64[2], np.zeros((1, 2 * d))])[tgt]) + \
        np.concatenate([t64[3], [0.0]])[tgt]
    assert (x == 0).all() and real.any() and 2 in ties
    want_l, want = caser_autograd(*t64, d, L, nv, nh, *batch, mask, keep)
    lo, got = cm.loss_and_grad(*t64, d, L, nv, nh, *batch, mask, keep)
    assert abs(lo - want_l) <= 1e-15 * want_l and abs(lo - 2 * np.log(2)) <= 1e-15
    for g, w in zip(got, want):
        assert np.array_equal(g, w)
    for pairwise, kind, L in ((1, "hinge", 2), (1, "square", 1), (0, "square", 2)):
        tabs, users, recent, items, third = fpmcplus_case(rs, 12, 5, 6, L, pairwise, kind)
        t, att = fpm.attention(tabs[0][users].astype(np.float64), tabs[2][items].astype(np.float64),
                               tabs[3][recent].astype(np.float64), *[a.astype(np.float64) for a in tabs[4:]])
        assert (np.abs(t) == 1).all() and (att == 1.0 / L).all()
        want_l, want = fpmcplus_autograd(tabs, users, recent, items, third, pairwise, kind, 0.125, 0.25)
        lo, got, _ = fpmcplus_ref(tabs, users, recent, items, third, pairwise, kind, 0.125, 0.25)
        assert abs(lo - want_l) <= 1e-12 * abs(want_l)
        for k, (g, w) in enumerate(zip(got, want)):
            np.testing.assert_allclose(g, w.reshape(g.shape), rtol=1e-12, atol=1e-12, err_msg=str(k))
        rw = 0.25 if pairwise else 0.0
        assert np.array_equal(got[4], rw * tabs[4].astype(np.float64)) and not got[5].any()
        assert np.array_equal(got[6], rw * tabs[6].astype(np.float64))


@pytest.mark.parametrize("L", [1, 3])
def test_rounded_references_match_autograd(L):
    """CPU: the R references' values (the bounded GPU tests' float64 side) equal torch.autograd on Gaussian cases with
    pads, dropout and repeated ids, for Caser and for FPMCplus under every loss."""
    from test_caser import _autograd as caser_autograd
    from test_fpmcplus import _autograd as fpmcplus_autograd
    rs = np.random.RandomState(7 + L)
    d, nv, nh, B, T, N = 4, 2, 3, 6, 2, 3
    P, E, W2, b2, dense = gaussian_caser(rs, 7, 11, d, L, nv, nh)
    users, seqs = rs.randint(0, 7, B), rs.randint(0, 11, (B, L))
    pos, neg = rs.randint(0, 11, (B, T)), rs.randint(0, 11, (B, N))
    seqs[0, :L - 1], pos[0, 0], users[1] = 11, 11, users[0]
    mask = (rs.rand(B, nv * d + nh * L) < 0.5).astype(np.float32)
    want_l, want = caser_autograd(*[a.astype(np.float64) for a in (P, E, W2, b2, dense)], d, L, nv, nh, users, seqs,
                                  pos, neg, mask, 0.5)
    lo, got = caser_ref(P, E, W2, b2, dense, d, L, nv, nh, users, seqs, pos, neg, mask, 0.5)
    assert abs(float(lo.v) - want_l) <= 1e-12 * abs(want_l)
    for g, w in zip(got, want):
        np.testing.assert_allclose(g.v, w, rtol=1e-10, atol=1e-12)
    for pairwise, kind in ((1, "bpr"), (1, "hinge"), (1, "square"), (0, "cross_entropy"), (0, "square")):
        nu, ni, d, w, B = 6, 9, 5, 4, 20
        tabs = [(rs.randn(n, d) * 0.5).astype(np.float32) for n in (nu, ni, ni, ni)]
        tabs += [(rs.randn(3 * d, w) * 0.4).astype(np.float32), (rs.randn(1, w) * 0.3).astype(np.float32),
                 (rs.randn(w, 1) * 0.7 + 1).astype(np.float32)]
        u, i, win = rs.randint(0, nu, B), rs.randint(0, ni, B), rs.randint(0, ni, (B, L))
        u[1], win[0, -1] = u[0], win[0, 0]
        third = rs.randint(0, ni, B) if pairwise else (rs.rand(B) < 0.3).astype(np.float32)
        want_l, want = fpmcplus_autograd(tabs, u, win, i, third, pairwise, kind, 0.05, 0.2)
        lo, got = fpmcplus_rref(tabs, u, win, i, third, pairwise, kind, 0.05, 0.2)
        assert abs(float(lo.v) - want_l) <= 1e-12 * abs(want_l), kind
        for k, (g, ww) in enumerate(zip(got, want)):
            np.testing.assert_allclose(g.v, ww.reshape(g.v.shape), rtol=1e-10, atol=1e-12, err_msg=(kind, k))


REQUIRED = ({("caser_grad", s, c) for s, c in ((1, 0), (1, 1), (0, 0))}
            | {("caser_window", L) for L in (1, 2, 5, 16)}
            | {("caser_chunks", c) for c in (1, 2, 3)} | {("caser_ties", t) for t in (1, 2, 4)}
            | {("caser_counters", 1)} | {("caser_query", s, c) for s in (0, 1) for c in (0, 1)}
            | {("caser_reg", c) for c in (0, 1)} | {("caser_epoch", 1)}
            | {("fpmcplus_grad", p, c, L) for p, c, L in ((1, 0, 1), (1, 0, 2), (1, 1, 2), (0, 1, 1), (0, 0, 2))}
            | {("fpmcplus_epoch", p, o) for p in (0, 1) for o in OPTS}
            | {("fpmcplus_pair", R) for R in (8, 3, 1)} | {("fpmcplus_project", c) for c in (0, 1)}
            | {("fism_epoch", p, o) for p in (0, 1) for o in OPTS}
            | {("caser_rounded", s, c, L) for s, c, L in ((0, 0, 8), (1, 0, 8), (1, 0, 1), (1, 0, 2), (1, 1, 5),
                                                          (1, 0, 16))}
            | {("fpmcplus_rounded", p, k, L, c) for p, k, _, _, L, c in
               [(p, k, d, w, L, int(B == "cap+1")) for p, k, d, w, L, B in FPMCPLUS_ROUNDED]}
            | {("limits", 1)})


@gpu
def test_every_route_was_seen(request):
    """Across this file the hooks reported every route listed in REQUIRED.  Only meaningful when the whole file ran:
    a run of selected tests skips it."""
    here = {it.nodeid for it in request.session.items if it.fspath == request.node.fspath}
    if len(here) < 60:
        pytest.skip("only part of the file ran")
    assert REQUIRED <= SEEN, sorted(REQUIRED - SEEN, key=str)
