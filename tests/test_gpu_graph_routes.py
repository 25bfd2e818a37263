"""Every route the graph kernels (csrc/lightgcn.cu SpMM, csrc/ngcf.cu, csrc/spectral.cu) take from a shape, against
float64.

The routes depend on the SM count: the SpMM, the NGCF layer kernels and the BPR gradient cap their grid at 8 CTAs
(64 warps) per SM and loop beyond 64 * SMs rows, units or triplets; the NGCF backward runs 2 CTAs per SM over
32-row tiles; SpectralCF splits an A_hat product into two K halves when it has >= 1024 rows and fewer than one
32-row tile per SM.  Every shape below is derived from the device's SM count (`*_cases(sms)`), one case on each
side of each boundary; each test asserts the route it ran through nrc_graph_last_routes, and the last test of the
file checks that the whole file saw every route.

Exact tests: small-integer tables, CSR values and dense operators from {0, +-2^-k}, identity or relu, hinge or
square loss, reg 0 or a power of two.  Every partial sum is then a multiple of its granularity below 2^24 granules
(asserted from the float64 magnitudes by `assert_exact`), so fp32 is exact in any summation order and every route
must equal the float64 reference bit for bit.

Rounded tests: realistic values.  Each entry must lie within C * 2^-24 * M of float64, where M is a first-order
bound on the rounding error the chain can carry, evaluated in float64 alongside the values (`*_chain`): for a sum
of n products it is n times the same sum on absolute values (any order, fma or not); element-wise operations add
one unit of their result per rounding (two for rsqrtf, expf, tanhf: their documented ulp bounds); errors of the
inputs propagate through the absolute values of the local derivatives.  C = 2 for every quantity: the chain is
first order and C covers the second-order terms (each below 2^-24 relative to the first-order ones)."""
import functools
import os

import numpy as np
import pytest
import scipy.sparse as sp
import torch

from oracle import tf_math

gpu = pytest.mark.gpu
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
U24 = 2.0 ** -24
C_BOUND = 2.0
SEEN = set()


def dev(a):
    return None if a is None else torch.from_numpy(np.ascontiguousarray(a)).cuda()


def sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def routes():
    from neurec_b200 import ops
    return ops.graph_last_routes()


# ---------------------------------------------------------------------------------------------------------------
# the route predicates of the host code and the shapes on each side of them (pure functions of the SM count)
# ---------------------------------------------------------------------------------------------------------------
def spmm_capped(n, n_sms):
    """More than one 8-row unit per CTA (fast) or one row per warp (exact): ceil(n / 8) CTAs over the 8 * SMs cap."""
    return (n + 7) // 8 > 8 * n_sms


def spectral_split(N, n_sms):
    """The A_hat products (K = N) run in two K halves: >= 1024 rows and fewer 32-row tiles than SMs."""
    return 2 if N >= 1024 and (N + 31) // 32 < n_sms else 1


def spectral_dw_slices(N):
    per = ((N + 63) // 64 + 31) // 32 * 32
    return (N + per - 1) // per


def ngcf_bwd_tiles(N, n_sms):
    tiles = (N + 31) // 32
    return -(-tiles // min(2 * n_sms, tiles))


def per_warp(n, n_sms):
    """Most items per warp of a kernel with ceil(n / 8) CTAs of 8 warps, capped at 8 CTAs per SM."""
    return -(-n // (min((n + 7) // 8, 8 * n_sms) * 8))


def spmm_synth_sizes(n_sms):
    return {"synth_small": 1203, "synth_capped": 64 * n_sms + 5}


def spectral_cases(n_sms):
    """(N, d, layers): below 1024 rows; 1024 and 1031; the conf shape on ml-100k; the last split size and the first
    unsplit one; one size past 32 * SMs rows."""
    last = 32 * (n_sms - 1)
    return [(290, 3, 8), (290, 1, 0), (1024, 8, 1), (1031, 3, 2), (2625, 100, 2), (1031, 128, 1),
            (last, 4, 1), (last + 1, 4, 1), (32 * n_sms + 7, 3, 1)]


def dropout_sizes(n_sms):
    """Element counts: tiny, ragged, and one whose grid (capped at 8 CTAs of 256 threads per SM, 4 elements per
    thread) loops."""
    return [1, 3, 4, 5, 1000, 4 * 2048 * n_sms + 13]


@pytest.mark.parametrize("n_sms", [114, 132])
def test_route_shapes_straddle_every_boundary(n_sms):
    """CPU: the shapes derived from the SM count land on both sides of every route predicate (114: H100 PCIe,
    132: H100 SXM)."""
    syn = spmm_synth_sizes(n_sms)
    assert not spmm_capped(syn["synth_small"], n_sms) and spmm_capped(syn["synth_capped"], n_sms)
    assert syn["synth_capped"] % 8 and syn["synth_small"] % 8
    assert not spmm_capped(2625, n_sms) and spmm_capped(70839, n_sms)          # ml-100k, gowalla
    assert ngcf_bwd_tiles(2625, n_sms) == 1 and ngcf_bwd_tiles(70839, n_sms) > 1
    assert per_warp(2625, n_sms) == 1 and per_warp(70839, n_sms) > 1
    assert per_warp(64 * n_sms + 1, n_sms) == 2 and per_warp(64 * n_sms, n_sms) == 1
    splits = {N: spectral_split(N, n_sms) for N, _, _ in spectral_cases(n_sms)}
    last = 32 * (n_sms - 1)
    assert splits[290] == 1 and splits[1024] == 2 and splits[1031] == 2 and splits[2625] == 2
    assert splits[last] == 2 and splits[last + 1] == 1 and splits[32 * n_sms + 7] == 1
    assert spectral_split(1023, n_sms) == 1
    n_big = dropout_sizes(n_sms)[-1]
    assert (n_big + 3) // 4 > 256 * 8 * n_sms


# ---------------------------------------------------------------------------------------------------------------
# exactness precondition and bounds
# ---------------------------------------------------------------------------------------------------------------
def assert_exact(values, magnitude, bits, what=""):
    """Every value is a multiple of 2^-bits and every partial sum (bounded by `magnitude`) stays below 2^24 such
    granules: fp32 represents each exactly, in any summation order."""
    v = np.asarray(values, np.float64) * 2.0 ** bits
    assert np.array_equal(v, np.round(v)), what
    assert (np.asarray(magnitude, np.float64) * 2.0 ** bits < 2.0 ** 24).all(), (what, float(np.max(magnitude)))


def as_f32_exact(a):
    out = np.asarray(a, np.float64).astype(np.float32)
    assert np.array_equal(out.astype(np.float64), a)
    return out


def assert_within(got, want, M, what, C=C_BOUND):
    err = np.abs(np.asarray(got, np.float64) - want)
    bound = C * U24 * M
    assert (err <= bound).all(), (what, float((err - bound).max()), float(np.max(M)))


def abs_csr(A):
    B = A.copy()
    B.data = np.abs(B.data)
    return B


def row_nnz(A):
    return np.diff(A.indptr).astype(np.float64)[:, None]


# ---------------------------------------------------------------------------------------------------------------
# graphs
# ---------------------------------------------------------------------------------------------------------------
@functools.lru_cache(maxsize=None)
def split(name):
    """The train CSR of the ml-100k / gowalla fixtures (tests/golden)."""
    z = np.load(os.path.join(GOLDEN, "%s_split.npz" % name))
    return {"num_users": int(z["num_users"]), "num_items": int(z["num_items"]),
            "train_indptr": z["train_indptr"].astype(np.int64), "train_indices": z["train_indices"].astype(np.int32)}


@functools.lru_cache(maxsize=None)
def _graph(name, adj_type):
    d = split(name)
    A = tf_math.lightgcn_adj(d["train_indptr"], d["train_indices"], d["num_users"], d["num_items"], adj_type)
    return d["num_users"], d["num_items"], A.astype(np.float64)


def synthetic_graph(n, seed):
    """n x n CSR: empty rows, rows of 191, 192 and 193 non-zeros (one short of, at and one past the long-row
    threshold), one row of 1100 (> 8 warps x 32 x 4 loads), the rest up to 40 non-zeros."""
    rs = np.random.RandomState(seed)
    rows = [np.unique(rs.randint(0, n, k)) for k in rs.randint(0, 41, n)]
    for r in rs.choice(n, 40, replace=False):
        rows[r] = np.zeros(0, np.int64)
    for r, k in zip(rs.choice(n, 7, replace=False), [191, 192, 193, 1100, 191, 193, 0]):
        rows[r] = np.sort(rs.permutation(n)[:k])
    deg = np.array([len(r) for r in rows])
    indptr = np.zeros(n + 1, np.int64)
    indptr[1:] = np.cumsum(deg)
    A = sp.csr_matrix((np.ones(indptr[-1]), np.concatenate(rows), indptr), shape=(n, n))
    return A


def dyadic_values(A, rs, sparse=False):
    """Values of A replaced by +-2^-k, k in {0, 1, 2}; sparse: only about 2 non-zero values per row, the rest 0 (the
    structure stays), so repeated products keep their magnitudes."""
    B = A.copy().astype(np.float64)
    nnz = B.nnz
    B.data = rs.choice([-1.0, 1.0], nnz) * 2.0 ** -rs.randint(0, 3, nnz)
    if sparse:
        deg = np.repeat(np.maximum(np.diff(B.indptr), 1), np.diff(B.indptr))
        B.data *= rs.rand(nnz) < np.minimum(1.0, 2.0 / deg)
    return B


def order_of(A, kind, seed=0):
    if kind == "natural":
        return None
    if kind == "degree":
        return np.argsort(-np.diff(A.indptr), kind="stable").astype(np.int32)
    return np.random.RandomState(seed).permutation(A.shape[0]).astype(np.int32)


def csr_dev(A):
    return dev(A.indptr.astype(np.int64)), dev(A.indices.astype(np.int32)), dev(A.data.astype(np.float32))


def spmm_graph(name):
    if name in ("gowalla", "ml100k"):
        return _graph(name, "pre")[2]
    n = spmm_synth_sizes(sms())[name]
    return synthetic_graph(n, n)


@pytest.fixture
def exact_mode(request):
    from neurec_b200 import ops
    ops.spmm_set_exact(request.param)
    yield request.param
    ops.spmm_set_exact(False)


def check_spmm_route(n, dim, exact):
    r = routes()
    fast = (not exact) and dim in (32, 64, 128)
    width = dim // 4 if fast else (dim // 32 if dim in (32, 64, 128) else 0)
    assert (r["spmm_fast"], r["spmm_width"], r["spmm_capped"]) == (int(fast), width, int(spmm_capped(n, sms()))), r
    SEEN.add(("spmm", "fast" if fast else "exact", width))
    SEEN.add(("spmm_capped", "fast" if fast else "exact", r["spmm_capped"]))


# ---------------------------------------------------------------------------------------------------------------
# a. SpMM: exact on dyadic inputs, every route, with the fused epilogue
# ---------------------------------------------------------------------------------------------------------------
SPMM_DIMS = [32, 64, 128, 1, 50, 129, 256]


def spmm_exact_reference(graph, dim):
    """Dyadic values on the graph, integer x, bias and running sum; the float64 product after its precondition."""
    rs = np.random.RandomState(dim)
    A = dyadic_values(graph, rs)
    n = A.shape[0]
    X = rs.randint(-4, 5, (n, dim)).astype(np.float64)
    B = rs.randint(-8, 9, (n, dim)).astype(np.float64)
    S = rs.randint(-8, 9, (n, dim)).astype(np.float64)
    want = A @ X
    M = abs_csr(A) @ np.abs(X)
    assert_exact(want, M, 2, "A.x")
    assert_exact((S + B + want) / 4, np.abs(S) + np.abs(B) + M, 4, "epilogue")
    return A, X, B, S, want


@pytest.mark.parametrize("n_sms", [114, 132])
def test_spmm_exact_preconditions(n_sms):
    """CPU: the synthetic graphs of both SM counts hold the long, short and empty rows they are built for, and the
    float64 references of the exact SpMM tests meet the exactness precondition."""
    for name, n in spmm_synth_sizes(n_sms).items():
        G = synthetic_graph(n, n)
        deg = np.diff(G.indptr)
        assert {191, 192, 193} <= set(deg.tolist()) and deg.max() > 8 * 32 * 4 and (deg == 0).any()
        for dim in SPMM_DIMS:
            spmm_exact_reference(G, dim)


@gpu
@pytest.mark.parametrize("exact_mode", [False, True], ids=["fast", "exact"], indirect=True)
@pytest.mark.parametrize("dim", SPMM_DIMS)
@pytest.mark.parametrize("graph", ["gowalla", "synth_small", "synth_capped"])
def test_spmm_exact_on_dyadic_inputs(graph, dim, exact_mode):
    """y = A.x, then y = bias + A.x with sum = (sum + y) / 4: bit for bit the float64 product, in the degree order,
    the natural order and (synthetic graphs) a random row order, where a long row can sit anywhere in its unit."""
    from neurec_b200 import ops
    A, X, B, S, want = spmm_exact_reference(spmm_graph(graph), dim)
    n = A.shape[0]
    ip, ix, va = csr_dev(A)
    dX = dev(X.astype(np.float32))
    orders =["degree", "natural"] + (["random"] if graph != "gowalla" else [])
    for kind in orders:
        order = dev(order_of(A, kind, dim))
        got = ops.spmm_csr(ip, ix, va, dX, row_order=order).cpu().numpy()
        check_spmm_route(n, dim, exact_mode)
        assert np.array_equal(got, as_f32_exact(want)), kind
    dS = dev(S.astype(np.float32))
    y = ops.spmm_csr(ip, ix, va, dX, row_order=dev(order_of(A, "degree")), bias=dev(B.astype(np.float32)), sum_=dS,
                     div=4.0).cpu().numpy()
    assert np.array_equal(y, as_f32_exact(B + want))
    assert np.array_equal(dS.cpu().numpy(), as_f32_exact((S + B + want) / 4))
    if graph != "gowalla":
        assert np.diff(A.indptr).max() > 8 * 32 * 4 and (np.diff(A.indptr) == 0).any()


@gpu
@pytest.mark.parametrize("dim", [32, 64, 128])
@pytest.mark.parametrize("graph", ["gowalla", "synth_small", "synth_capped"])
def test_fast_spmm_rounded_and_deterministic(graph, dim):
    """The fast kernel on the real 'pre' values (synthetic graphs: random values) and Gaussian x: within
    C * 2^-24 * nnz(row) * (|A| |x|) of float64 on every route, and bit-identical across two runs."""
    from neurec_b200 import ops
    rs = np.random.RandomState(7 + dim)
    A = spmm_graph(graph).copy()
    if graph != "gowalla":
        A.data = rs.randn(A.nnz)
    A32 = A.astype(np.float32)
    A = A32.astype(np.float64)
    n = A.shape[0]
    X = rs.randn(n, dim).astype(np.float32)
    want = A @ X.astype(np.float64)
    M = row_nnz(A) * (abs_csr(A) @ np.abs(X).astype(np.float64))
    ip, ix, va = csr_dev(A)
    dX = dev(X)
    for kind in ["degree", "natural", "random"]:
        order = dev(order_of(A, kind, dim))
        got = ops.spmm_csr(ip, ix, va, dX, row_order=order).cpu().numpy()
        check_spmm_route(n, dim, False)
        assert_within(got, want, M, (graph, kind))
        again = ops.spmm_csr(ip, ix, va, dX, row_order=order).cpu().numpy()
        assert np.array_equal(got, again), kind
    assert np.abs(want).max() > 0.1


@gpu
@pytest.mark.parametrize("n_layers", [0, 1, 2, 6])
@pytest.mark.parametrize("graph,dim", [("gowalla", 64), ("gowalla", 32), ("synth_capped", 128), ("synth_small", 50)])
def test_lightgcn_propagate_exact(graph, dim, n_layers):
    """mean(E_0, A E_0, ..., A^L E_0) bit for bit (0 layers: a copy; layer 0 reads the running sum from E_0; the
    last layer divides by L + 1 -- an exact sum divided once, which float64 rounds to the same fp32), fast and
    exact SpMM."""
    from neurec_b200 import ops
    rs = np.random.RandomState(dim + n_layers)
    A = dyadic_values(spmm_graph(graph), rs, sparse=True)
    absA = abs_csr(A)
    n = A.shape[0]
    e0 = rs.randint(-4, 5, (n, dim)).astype(np.float64)
    x, m, s, ms = e0, np.abs(e0), e0.copy(), np.abs(e0)
    for k in range(n_layers):
        x, m = A @ x, absA @ m
        s, ms = s + x, ms + m
        assert_exact(s, ms, 2 * (k + 1), "layer %d" % k)
    want = as_f32_exact(s).astype(np.float32) if n_layers == 0 else (s / (n_layers + 1)).astype(np.float32)
    ref, _ = tf_math.lightgcn_propagate(A.astype(np.float32), e0.astype(np.float32), n_layers)
    assert np.array_equal(ref, want)                 # tf_math's fp32 chain agrees (its sums are exact too)
    ip, ix, va = csr_dev(A)
    for exact in (False, True):
        ops.spmm_set_exact(exact)
        try:
            before = routes()
            out = torch.full((n, dim), 7.0, device="cuda")
            work = (torch.full_like(out, 3.0), torch.full_like(out, 5.0))
            got = ops.lightgcn_propagate(ip, ix, va, dev(order_of(A, "degree")), dev(e0.astype(np.float32)), n_layers,
                                         e_final=out, work=work).cpu().numpy()
        finally:
            ops.spmm_set_exact(False)
        assert np.array_equal(got, want), exact
        if n_layers:
            check_spmm_route(n, dim, exact)
        else:
            assert routes() == before                # a copy: no SpMM launched
    SEEN.add(("propagate_layers", n_layers))


@gpu
def test_lightgcn_train_epoch_one_layer(ml100k):
    """nrc_lightgcn_train_epoch with one layer (the first layer is the last: the forward reads sum_in = E_0, writes
    no Y and divides by 2; the backward writes only grad_e0) against LightGCNTrainer, with the tolerances of the
    three-layer test in test_gpu_lightgcn.py."""
    from neurec_b200 import ops
    d = ml100k
    nu, ni, dim, L, bs, steps = d["num_users"], d["num_items"], 64, 1, 1024, 4
    A = tf_math.lightgcn_adj(d["train_indptr"], d["train_indices"], nu, ni, "pre")
    rs = np.random.RandomState(14)
    lim = np.sqrt(6.0 / (nu + dim))
    e0 = rs.uniform(-lim, lim, (nu + ni, dim)).astype(np.float32)
    all_users = np.repeat(np.arange(nu, dtype=np.int32), np.diff(d["train_indptr"]))
    perm = rs.permutation(len(all_users))[:bs * steps - 100]
    users, pos = all_users[perm], d["train_indices"][perm]
    neg = rs.randint(0, ni, len(users)).astype(np.int32)
    tr = tf_math.LightGCNTrainer(A, e0, nu, L, 0.01, 1e-3)
    want = tr.epoch(users, pos, neg, bs)
    de0 = dev(e0)
    z = lambda: torch.zeros_like(de0)
    m, v, ef, gf, ge = z(), z(), z(), z(), z()
    wa, wb = torch.full_like(de0, 9.0), torch.full_like(de0, 9.0)
    sl = torch.zeros(steps, 2, device="cuda")
    order = dev(order_of(A, "degree"))
    n = ops.lightgcn_train_epoch(csr_dev(A), None, order, nu, ni, L, de0, m, v, dev(users), dev(pos), dev(neg), bs,
                                 1e-3, tf_math.adam_lr_t(0.01, steps), [0.01, 0.9, 0.999, 1e-8], ef, gf, ge, (wa, wb),
                                 sl)
    assert n == steps
    check_spmm_route(nu + ni, dim, False)
    assert np.allclose(sl.cpu().numpy(), want, rtol=1e-4)
    assert np.abs(de0.cpu().numpy() - tr.e0).max() < 5e-5
    assert np.abs(tr.e0 - e0).max() > 5e-3
    assert float(gf.abs().max()) == 0.0 and float(ge.abs().max()) == 0.0
    assert bool((wa == 9.0).all()) and bool((wb == 9.0).all())        # one layer: no intermediate Y written


# ---------------------------------------------------------------------------------------------------------------
# b. NGCF: forward and gradients within C * 2^-24 * M of float64
# ---------------------------------------------------------------------------------------------------------------
NGCF_ALPHA = tf_math.LEAKY_ALPHA
NGCF_EPS = tf_math.L2NORM_EPS


def _mm_err(X, eX, W, n_terms):
    """value and error bound (units of 2^-24) of X @ W with exact W and X carrying eX: n_terms roundings per term."""
    return X @ W, eX @ np.abs(W) + n_terms * (np.abs(X) @ np.abs(W))


def _leaky_err(z, ez):
    """leaky-relu with its error: slope times the input error away from the kink, the input error itself (slope <=
    1, continuous) within its band; one rounding of x * 0.2f plus the 0.2f constant on the negative side."""
    band = (np.abs(z) <= C_BOUND * U24 * ez) & (ez > 0)
    slope = np.where(z > 0, 1.0, NGCF_ALPHA)
    return np.where(z > 0, z, NGCF_ALPHA * z), np.where(band, 1.0, slope) * ez + 2.0 * (z < 0) * np.abs(NGCF_ALPHA * z)


def ngcf_chain(A, AT, e0, W, masks, keep, nu, users, pos, neg, reg, n_sms, forward_only=False):
    """Values of nrc_ngcf_grad's quantities in float64 and their first-order error bounds (units of 2^-24)."""
    absA, absAT, degA, degAT = abs_csr(A), abs_csr(AT), row_nnz(A), row_nnz(AT)
    N = e0.shape[0]
    ego, e_ego = e0, np.zeros_like(e0)
    outs, eouts, cache = [e0], [np.zeros_like(e0)], []
    for k, (Wgc, bgc, Wbi, bbi) in enumerate(W):
        din, dout = Wgc.shape
        side = A @ ego
        e_side = absA @ e_ego + degA * (absA @ np.abs(ego))
        z1, e_z1 = _mm_err(side, e_side, Wgc, din + 1)
        z1, e_z1 = z1 + bgc, e_z1 + (din + 1) * np.abs(bgc)
        bi = ego * side
        e_bi = np.abs(ego) * e_side + np.abs(side) * e_ego + np.abs(bi)
        z2, e_z2 = _mm_err(bi, e_bi, Wbi, din + 1)
        z2, e_z2 = z2 + bbi, e_z2 + (din + 1) * np.abs(bbi)
        l1, el1 = _leaky_err(z1, e_z1)
        l2, el2 = _leaky_err(z2, e_z2)
        h, e_h = l1 + l2, el1 + el2 + np.abs(l1 + l2)
        m = np.ones_like(h) if masks is None else masks[k].astype(np.float64)
        hd, e_hd = h * m / keep, e_h * m / keep                 # keep 1 or 1/2: exact scaling
        sq = (hd * hd).sum(1, keepdims=True)
        e_sq = (2 * np.abs(hd) * e_hd).sum(1, keepdims=True) + (dout + 1) * sq
        live = sq > NGCF_EPS
        inv = 1.0 / np.sqrt(np.maximum(sq, NGCF_EPS))
        e_inv = np.where(live, 0.5 * inv / np.maximum(sq, NGCF_EPS) * e_sq, 0.0) + 2 * inv
        y = hd * inv
        outs.append(y)
        eouts.append(inv * e_hd + np.abs(hd) * e_inv + np.abs(y))
        cache.append(dict(ego=ego, e_ego=e_ego, side=side, e_side=e_side, z1=z1, e_z1=e_z1, z2=z2, e_z2=e_z2, bi=bi,
                          e_bi=e_bi, m=m, hd=hd, e_hd=e_hd, sq=sq, e_sq=e_sq, live=live, inv=inv, e_inv=e_inv))
        ego, e_ego = hd, e_hd
    allE, eA = np.concatenate(outs, 1), np.concatenate(eouts, 1)
    R = dict(all=allE, e_all=eA, cache=cache)
    if forward_only:
        return R
    ru, ri, rj = np.asarray(users), nu + np.asarray(pos), nu + np.asarray(neg)
    D = allE.shape[1]
    eu, ei, ej, xu, xi, xj = allE[ru], allE[ri], allE[rj], eA[ru], eA[ri], eA[rj]
    di, dj = (eu * ei).sum(1), (eu * ej).sum(1)
    e_x = ((np.abs(eu) * xi + np.abs(ei) * xu).sum(1) + D * np.abs(eu * ei).sum(1)
           + (np.abs(eu) * xj + np.abs(ej) * xu).sum(1) + D * np.abs(eu * ej).sum(1) + np.abs(di - dj))
    x = di - dj
    g = -1.0 / (1.0 + np.exp(x))
    e_g = 0.25 * e_x + 4 * np.abs(g)
    l = np.where(x >= 0, np.log1p(np.exp(-x)), -x + np.log1p(np.exp(x)))
    B = len(ru)
    R["mf"], R["e_mf"] = l.sum(), (np.abs(g) * e_x + 4 * l).sum() + B * l.sum()
    sqb = (eu * eu + ei * ei + ej * ej).sum(1)
    e_sqb = (2 * (np.abs(eu) * xu + np.abs(ei) * xi + np.abs(ej) * xj)).sum(1) + 3 * D * sqb
    R["emb"], R["e_emb"] = reg * 0.5 * sqb.sum(), reg * 0.5 * (e_sqb + 3 * sqb).sum() + B * reg * 0.5 * sqb.sum()
    G, eG, aG, cnt = (np.zeros_like(allE) for _ in range(4))
    gg, eg = g[:, None], e_g[:, None]
    for rows, c, ec in ((ru, gg * (ei - ej) + reg * eu,
                         np.abs(ei - ej) * eg + np.abs(gg) * (xi + xj) + reg * xu
                         + 3 * (np.abs(gg * (ei - ej)) + np.abs(reg * eu))),
                        (ri, gg * eu + reg * ei, np.abs(eu) * eg + np.abs(gg) * xu + reg * xi
                         + 3 * (np.abs(gg * eu) + np.abs(reg * ei))),
                        (rj, -gg * eu + reg * ej, np.abs(eu) * eg + np.abs(gg) * xu + reg * xj
                         + 3 * (np.abs(gg * eu) + np.abs(reg * ej)))):
        np.add.at(G, rows, c)
        np.add.at(eG, rows, ec)
        np.add.at(aG, rows, np.abs(c))
        np.add.at(cnt, rows, 1.0)
    eG = eG + cnt * aG                                       # RED chain: one rounding per contribution
    tiles = (N + 31) // 32
    grid = min(2 * n_sms, tiles)
    chain = 32 * -(-tiles // grid) + grid                     # dW: fma chain over the CTA's tiles, then one RED per CTA
    dims = [e0.shape[1]] + [w[0].shape[1] for w in W]
    offs = np.cumsum([0] + dims)
    dn, e_dn = None, None
    grads = [None] * len(W)
    for k in range(len(W) - 1, -1, -1):
        Wgc, _, Wbi, _ = W[k]
        c = cache[k]
        din, dout = Wgc.shape
        gn, e_gn = G[:, offs[k + 1]:offs[k + 2]], eG[:, offs[k + 1]:offs[k + 2]]
        hd, e_hd, inv, e_inv, live = c["hd"], c["e_hd"], c["inv"], c["e_inv"], c["live"]
        dot = (gn * hd).sum(1, keepdims=True)
        e_dot = (np.abs(gn) * e_hd + np.abs(hd) * e_gn).sum(1, keepdims=True) + dout * np.abs(gn * hd).sum(1, keepdims=True)
        t1 = gn * inv
        e_t1 = e_gn * inv + np.abs(gn) * e_inv + np.abs(t1)
        T = live * hd * dot * inv ** 3
        e_T = live * (e_hd * np.abs(dot) * inv ** 3 + np.abs(hd) * e_dot * inv ** 3
                      + 3 * np.abs(hd * dot) * inv ** 2 * e_inv + 4 * np.abs(T))
        dhd, e_dhd = t1 - T, e_t1 + e_T + np.abs(t1 - T)
        if dn is not None:
            dhd, e_dhd = dhd + dn, e_dhd + e_dn + np.abs(dhd + dn)
        dh, e_dh = dhd * c["m"] / keep, e_dhd * c["m"] / keep
        s1, s2 = np.where(c["z1"] > 0, 1.0, NGCF_ALPHA), np.where(c["z2"] > 0, 1.0, NGCF_ALPHA)
        dz1, dz2 = dh * s1, dh * s2
        e_dz1 = s1 * e_dh + 2 * (c["z1"] <= 0) * np.abs(dz1)
        e_dz2 = s2 * e_dh + 2 * (c["z2"] <= 0) * np.abs(dz2)
        side, e_side, bi, e_bi, ego, e_ego = c["side"], c["e_side"], c["bi"], c["e_bi"], c["ego"], c["e_ego"]
        dWgc = side.T @ dz1
        e_dWgc = np.abs(side).T @ e_dz1 + e_side.T @ np.abs(dz1) + chain * (np.abs(side).T @ np.abs(dz1))
        dWbi = bi.T @ dz2
        e_dWbi = np.abs(bi).T @ e_dz2 + e_bi.T @ np.abs(dz2) + chain * (np.abs(bi).T @ np.abs(dz2))
        db1, e_db1 = dz1.sum(0), e_dz1.sum(0) + chain * np.abs(dz1).sum(0)
        db2, e_db2 = dz2.sum(0), e_dz2.sum(0) + chain * np.abs(dz2).sum(0)
        grads[k] = [(dWgc, e_dWgc), (db1, e_db1), (dWbi, e_dWbi), (db2, e_db2)]
        a, e_a = dz1 @ Wgc.T, e_dz1 @ np.abs(Wgc).T + dout * (np.abs(dz1) @ np.abs(Wgc).T)
        b, e_b = dz2 @ Wbi.T, e_dz2 @ np.abs(Wbi).T + dout * (np.abs(dz2) @ np.abs(Wbi).T)
        dside = a + b * ego
        e_dside = e_a + e_b * np.abs(ego) + np.abs(b) * e_ego + 2 * np.abs(b * ego) + np.abs(dside)
        dego = b * side
        e_dego = e_b * np.abs(side) + np.abs(b) * e_side + np.abs(dego)
        dn = dego + AT @ dside
        e_dn = e_dego + absAT @ e_dside + degAT * (absAT @ np.abs(dside)) + np.abs(dn)
        c.update(dz1=dz1, dz2=dz2)
    R["dE0"] = G[:, :dims[0]] + dn
    R["e_dE0"] = eG[:, :dims[0]] + e_dn + np.abs(R["dE0"])
    R["grads"] = grads
    return R


def pack(weights):
    return np.concatenate([np.concatenate([np.asarray(w, np.float32).reshape(-1) for w in ws]) for ws in weights])


@functools.lru_cache(maxsize=None)
def ngcf_graph(name, isolate=0):
    """The 'norm' adjacency D^-1 (A + I) of ml-100k or gowalla as float64 CSR and its transpose; isolate > 0 drops
    every train interaction of that many users, which then only have their self-loop."""
    d = split(name)
    ip, ix = d["train_indptr"], d["train_indices"]
    if isolate:
        deg = np.diff(ip).copy()
        deg[:isolate] = 0
        keep = np.ones(len(ix), bool)
        keep[:ip[isolate]] = False
        ix = ix[keep]
        ip = np.concatenate([[0], np.cumsum(deg)]).astype(np.int64)
    A = tf_math.ngcf_adj(ip, ix, d["num_users"], d["num_items"], "norm").astype(np.float32)
    AT = A.T.tocsr()
    AT.sort_indices()
    return d["num_users"], d["num_items"], A.astype(np.float64), AT.astype(np.float64)


def ngcf_inputs(A, AT, nu, ni, emb, layers, keep, batch, seed, zero_rows=0, tiny=0, no_bias=False):
    """Tables of scale 0.1 and xavier weights in fp32; masks (keep < 1: Bernoulli, else ones) with every
    pre-activation that lies within its rounding bound of the kink masked out, layer by layer (the kink of a kept
    entry cannot flip between fp32 and float64); zero_rows users get an all-zero mask row in the first layer
    (sq = 0 exactly); tiny: the first `tiny` users (isolated by the caller) get rows of scale 1e-8 so that
    0 < sq < 1e-12."""
    rs = np.random.RandomState(seed)
    N = nu + ni
    e0 = (rs.randn(N, emb) * 0.1).astype(np.float32)
    if tiny:
        e0[:tiny] *= np.float32(1e-7)
    W = tf_math.ngcf_init_weights(rs, emb, layers)
    if no_bias:
        W = [(w[0], np.zeros_like(w[1]), w[2], np.zeros_like(w[3])) for w in W]
    W64 = [tuple(np.asarray(w, np.float64) for w in ws) for ws in W]
    masks = [(rs.rand(N, w) < keep).astype(np.float32) if keep < 1 else np.ones((N, w), np.float32) for w in layers]
    if zero_rows:
        masks[0][tiny:tiny + zero_rows] = 0.0
    users = rs.randint(0, nu, batch).astype(np.int32)
    users[:tiny + zero_rows] = np.arange(tiny + zero_rows)                    # those rows carry a gradient
    pos = rs.randint(0, ni, batch).astype(np.int32)
    neg = rs.randint(0, ni, batch).astype(np.int32)
    e64 = e0.astype(np.float64)
    for k in range(len(layers)):
        R = ngcf_chain(A, AT, e64, W64[:k + 1], [m.astype(np.float64) for m in masks[:k + 1]], keep, nu, users,
                       pos, neg, 0.0, 132, forward_only=True)
        c = R["cache"][k]
        near = ((np.abs(c["z1"]) <= C_BOUND * U24 * c["e_z1"] * 1.01) & (c["e_z1"] > 0)) | \
               ((np.abs(c["z2"]) <= C_BOUND * U24 * c["e_z2"] * 1.01) & (c["e_z2"] > 0))
        masks[k][near] = 0.0
    return e0, W, W64, masks, users, pos, neg


def ngcf_reference(graph, emb, layers, keep, batch, n_sms):
    """Inputs of one NGCF case and its float64 chain, checked against tf_math.ngcf_loss_and_grad and the guards."""
    nu, ni, A, AT = ngcf_graph(graph)
    inputs = ngcf_inputs(A, AT, nu, ni, emb, layers, keep, batch, len(layers) + emb)
    e0, W, W64, masks, users, pos, neg = inputs
    reg = 2.0 ** -10
    M64 = [m.astype(np.float64) for m in masks]
    R = ngcf_chain(A, AT, e0.astype(np.float64), W64, M64, keep, nu, users, pos, neg, reg, n_sms)
    check_ngcf_guards(R, masks)
    mf, emb_l, dE0, grads, allE = tf_math.ngcf_loss_and_grad(A, AT, e0.astype(np.float64), W64, nu, users, pos, neg,
                                                             reg, M64, keep)
    assert np.allclose(R["all"], allE, rtol=0, atol=1e-12) and np.allclose(R["dE0"], dE0, rtol=1e-10, atol=1e-12)
    assert np.isclose(R["mf"], mf, rtol=1e-12) and np.isclose(R["emb"], emb_l, rtol=1e-12)
    for k in range(len(layers)):
        for j in range(4):
            assert np.allclose(R["grads"][k][j][0].reshape(-1), grads[k][j].reshape(-1), rtol=1e-9, atol=1e-12)
    return reg, R, inputs


@pytest.mark.parametrize("emb,layers,keep", [(16, [16, 16], 0.5), (33, [1, 33], 1.0)])
def test_ngcf_reference_cpu(emb, layers, keep):
    """CPU: the float64 chain of the NGCF tests equals tf_math, the masks keep every kink and sq out of its band,
    and the forward bounds stay below 2^-10 of the value scale."""
    reg, R, _ = ngcf_reference("ml100k", emb, layers, keep, 300, 132)
    assert (C_BOUND * U24 * R["e_all"] <= 2.0 ** -10 * np.abs(R["all"]).max()).all()
    assert np.abs(R["dE0"]).max() > 0


NGCF_CASES = [  # (graph, emb, layers, keep, batch)
    ("ml100k", 16, [16, 16], 1.0, 512),
    ("ml100k", 16, [16, 16], 0.5, 512),
    ("ml100k", 64, [64, 64, 64, 64], 1.0, 256),
    ("ml100k", 64, [64, 64, 64, 64], 0.5, 256),
    ("ml100k", 1, [1, 33], 1.0, 300),
    ("ml100k", 33, [1, 33], 0.5, 300),
    ("ml100k", 32, [63, 31], 1.0, 300),
    ("ml100k", 63, [63, 31], 0.5, 300),
    ("gowalla", 16, [16, 16], 0.5, 2048),
    ("gowalla", 64, [64, 64, 64, 64], 1.0, 1024),
    ("gowalla", 32, [63, 31], 0.5, "big"),                  # a batch of 64 * SMs + 77 triplets
]


def run_ngcf(shape, A, AT, e0, W, masks, keep, users, pos, neg, reg):
    from neurec_b200 import ops
    N, dt = shape.n_nodes, shape.d_total
    csr, tcsr = csr_dev(A), csr_dev(AT)
    order, torder = dev(order_of(A, "degree")), dev(order_of(AT, "degree"))
    dm = None if masks is None else dev(np.concatenate([m.reshape(-1) for m in masks]))
    fwd = ops.ngcf_forward(shape, csr, order, dev(e0), dev(pack(W)), dm, keep).cpu().numpy()
    rf = routes()
    all_emb = torch.empty((N, dt), device="cuda")
    G = torch.zeros((N, dt), device="cuda")
    gE = torch.full((N, shape.emb_dim), 3.0, device="cuda")
    gW = torch.full((shape.weights_size(),), 3.0, device="cuda")
    work = torch.full((shape.work_floats(),), 5.0, device="cuda")
    loss2 = torch.zeros(2, device="cuda")
    ops.ngcf_grad(shape, csr, order, tcsr, torder, dev(e0), dev(pack(W)), dm, keep, dev(users), dev(pos), dev(neg),
                  reg, all_emb, G, gE, gW, work, loss2)
    rg = routes()
    assert float(G.abs().max()) == 0.0
    return fwd, rf, all_emb.cpu().numpy(), gE.cpu().numpy(), gW.cpu().numpy(), loss2.cpu().numpy(), rg


def check_ngcf_routes(rf, rg, N, batch):
    n = sms()
    assert rf["ngcf_fwd_rows"] == per_warp(N, n) and rf["ngcf_bwd_tiles"] == -1 and rf["ngcf_bpr_triplets"] == -1, rf
    assert rg["ngcf_fwd_rows"] == per_warp(N, n), rg
    assert rg["ngcf_bwd_tiles"] == ngcf_bwd_tiles(N, n) and rg["ngcf_bpr_triplets"] == per_warp(batch, n), rg
    SEEN.add(("ngcf_fwd_rows", "many" if rg["ngcf_fwd_rows"] > 1 else 1))
    SEEN.add(("ngcf_bwd_tiles", "many" if rg["ngcf_bwd_tiles"] > 1 else 1))
    SEEN.add(("ngcf_bpr_triplets", "many" if rg["ngcf_bpr_triplets"] > 1 else 1))


def assert_ngcf(R, fwd, all_emb, gE, gW, loss2, W, layers):
    assert_within(fwd, R["all"], R["e_all"], "forward")
    assert_within(all_emb, R["all"], R["e_all"], "all_emb")
    assert_within(gE, R["dE0"], R["e_dE0"], "dE0")
    got = np.split(gW, np.cumsum([w.size for ws in W for w in ws])[:-1])
    for k in range(len(layers)):
        for j, name in enumerate(("dW_gc", "db_gc", "dW_bi", "db_bi")):
            v, e = R["grads"][k][j]
            assert_within(got[4 * k + j].reshape(np.shape(v)), v, e, (name, k))
    assert_within(loss2[0], R["mf"], R["e_mf"], "mf_loss")
    assert_within(loss2[1], R["emb"], R["e_emb"], "emb_loss")


def check_ngcf_guards(R, masks):
    """No kept pre-activation within its bound of the kink; every sq clear of 1e-12 or exactly 0."""
    for k, c in enumerate(R["cache"]):
        kept = c["m"] != 0
        for z, ez in ((c["z1"], c["e_z1"]), (c["z2"], c["e_z2"])):
            assert not (kept & (np.abs(z) <= C_BOUND * U24 * ez) & (ez > 0)).any(), k
        sq, e_sq = c["sq"], c["e_sq"]
        assert ((sq == 0) | (np.abs(sq - NGCF_EPS) > C_BOUND * U24 * e_sq + 1e-6 * NGCF_EPS)).all(), k


@gpu
@pytest.mark.parametrize("graph,emb,layers,keep,batch", NGCF_CASES)
def test_ngcf_within_bound(graph, emb, layers, keep, batch):
    """nrc_ngcf_forward and nrc_ngcf_grad (all_emb, dE0, every packed weight and bias, both losses) against the
    float64 chain, which equals tf_math.ngcf_loss_and_grad."""
    from neurec_b200 import ops
    nu, ni, A, AT = ngcf_graph(graph)
    N = nu + ni
    if batch == "big":
        batch = 64 * sms() + 77
    reg, R, (e0, W, W64, masks, users, pos, neg) = ngcf_reference(graph, emb, layers, keep, batch, sms())
    shape = ops.NgcfShape.make(nu, ni, emb, layers)
    fwd, rf, all_emb, gE, gW, loss2, rg = run_ngcf(shape, A, AT, e0, W, masks, keep, users, pos, neg, reg)
    check_ngcf_routes(rf, rg, N, batch)
    assert_ngcf(R, fwd, all_emb, gE, gW, loss2, W, layers)
    assert np.abs(gW).max() > 0 and np.abs(gE).max() > 0
    SEEN.add(("ngcf_layers", len(layers)))
    SEEN.add(("ngcf_widths", max(layers) > 32))


@gpu
def test_ngcf_zero_and_tiny_rows():
    """Rows whose dropped-out first layer is all zero (sq = 0: l2_normalize's epsilon branch, lv = 0 in the
    backward) and isolated users with rows of scale 1e-8 and no biases (0 < sq < 1e-12 in every layer: the clamp
    and lv = 0 with hd != 0), every one of them in the batch."""
    from neurec_b200 import ops
    nu, ni, A, AT = ngcf_graph("ml100k", isolate=6)
    emb, layers, keep = 16, [16, 16], 0.5
    e0, W, W64, masks, users, pos, neg = ngcf_inputs(A, AT, nu, ni, emb, layers, keep, 400, 3, zero_rows=5, tiny=6,
                                                     no_bias=True)
    M64 = [m.astype(np.float64) for m in masks]
    reg = 0.0
    R = ngcf_chain(A, AT, e0.astype(np.float64), W64, M64, keep, nu, users, pos, neg, reg, sms())
    check_ngcf_guards(R, masks)
    sq0, sq1 = R["cache"][0]["sq"][:, 0], R["cache"][1]["sq"][:, 0]
    assert (sq0[6:11] == 0).all() and ((sq0[:6] > 0) & (sq0[:6] < NGCF_EPS)).all(), sq0[:11]
    assert ((sq1[:6] > 0) & (sq1[:6] < NGCF_EPS)).all(), sq1[:6]
    shape = ops.NgcfShape.make(nu, ni, emb, layers)
    fwd, rf, all_emb, gE, gW, loss2, rg = run_ngcf(shape, A, AT, e0, W, masks, keep, users, pos, neg, reg)
    check_ngcf_routes(rf, rg, nu + ni, len(users))
    assert_ngcf(R, fwd, all_emb, gE, gW, loss2, W, layers)
    assert np.abs(R["dE0"][:6]).max() > 1.0                  # the clamped rows carry a large, checked gradient
    SEEN.add(("ngcf_sq", "zero"))
    SEEN.add(("ngcf_sq", "below_eps"))


# ---------------------------------------------------------------------------------------------------------------
# c. SpectralCF: exact on dyadic inputs on every split route; rounded with the smooth activations
# ---------------------------------------------------------------------------------------------------------------
def spectral_exact_inputs(N, d, K, seed):
    """A_hat with one or two entries of +-1 per row, filters with one +-1 per column (signed near-permutations:
    magnitudes do not grow with the layers), integer tables in [-2, 2]."""
    rs = np.random.RandomState(seed)
    A = np.zeros((N, N))
    for r in range(N):
        k = 1 + (rs.rand() < 0.3)
        A[r, rs.choice(N, k, replace=False)] = rs.choice([-1.0, 1.0], k)
    F = np.zeros((K, d, d))
    for k in range(K):
        for c in range(d):
            F[k, rs.randint(d), c] = rs.choice([-1.0, 1.0])
    e0 = rs.randint(-2, 3, (N, d)).astype(np.float64)
    return A, F, e0


def spectral_magnitudes(A, F, e0, act, users, pos, neg, nu, reg, loss):
    """The float64 forward / backward of tf_math on absolute values (relu masks and hinge steps of the real chain):
    a bound of every partial sum."""
    absA, d = np.abs(A), e0.shape[1]
    allE, sides = tf_math.spectralcf_forward(A, e0, list(F), act)
    mags, m = [np.abs(e0)], np.abs(e0)
    for k in range(len(F)):
        s = absA @ m
        m = s @ np.abs(F[k])
        mags.append(m)
    mall = np.concatenate(mags, 1)
    ue, ie = allE[:nu], allE[nu:]
    x = (ue[users] * ie[pos]).sum(1) - (ue[users] * ie[neg]).sum(1)
    mx = (mall[:nu][users] * (mall[nu:][pos] + mall[nu:][neg])).sum(1)
    g = np.abs({"hinge": (x + 1 > 0) * 1.0, "square": -2 * (1 - x)}[loss]) + (2 * mx if loss == "square" else 0)
    MG = np.zeros_like(allE)
    np.add.at(MG, users, g[:, None] * (mall[nu:][pos] + mall[nu:][neg]) + reg * mall[:nu][users])
    np.add.at(MG, nu + pos, g[:, None] * mall[:nu][users] + reg * mall[nu:][pos])
    np.add.at(MG, nu + neg, g[:, None] * mall[:nu][users] + reg * mall[nu:][neg])
    carry = np.zeros((A.shape[0], d))
    out = [mall, mx, MG]
    for k in range(len(F), 0, -1):
        dZ = MG[:, k * d:(k + 1) * d] + carry
        out.append(np.abs(sides[k - 1]).T @ dZ)
        carry = absA.T @ (dZ @ np.abs(F[k - 1]).T)
        out.append(carry)
    return out


def run_spectral(A, F, e0, act, nu, users, pos, neg, loss, reg, explicit_t):
    from neurec_b200 import ops
    N, d = e0.shape
    K = F.shape[0]
    dA, dF, de0 = dev(A.astype(np.float32)), dev(F.astype(np.float32)), dev(e0.astype(np.float32))
    dAT = dev(np.ascontiguousarray(A.T).astype(np.float32)) if explicit_t else None
    work = torch.full((max(1, N * d * (K + 3)),), 7.0, device="cuda")
    fwd = ops.spectralcf_forward(dA, de0, dF, act, work=work).cpu().numpy()
    rf = routes()
    fwd2 = ops.spectralcf_forward(dA, de0, dF, act, work=torch.full_like(work, -3.0)).cpu().numpy()
    all_emb = torch.empty((N, d * (K + 1)), device="cuda")
    G = torch.zeros_like(all_emb)
    touched = torch.zeros(N, dtype=torch.int32, device="cuda")
    gE = torch.full((N, d), 3.0, device="cuda")
    gF = torch.full((max(K, 1), d, d), 3.0, device="cuda")[:K]
    loss_out = torch.zeros(1, device="cuda")
    ops.spectralcf_grad(nu, dA, dAT, de0, dF, act, dev(users), dev(pos), dev(neg), loss, reg, all_emb, G, touched, gE,
                        gF, torch.full_like(work, 11.0), loss_out)
    rg = routes()
    assert float(G.abs().max()) == 0.0
    return fwd, fwd2, rf, all_emb.cpu().numpy(), gE.cpu().numpy(), gF.cpu().numpy(), float(loss_out.item()), rg


def check_spectral_routes(rf, rg, N, K):
    n = sms()
    s = spectral_split(N, n) if K else 0
    assert (rf["spectral_fwd_split"], rf["spectral_bwd_split"], rf["spectral_dw_split"]) == (s, -1, -1), rf
    dw = spectral_dw_slices(N) if K else 0
    assert (rg["spectral_fwd_split"], rg["spectral_bwd_split"], rg["spectral_dw_split"]) == (s, s, dw), rg
    SEEN.add(("spectral_split", s))
    if K:
        SEEN.add(("spectral_dw", "split" if dw > 1 else 1))


def spectral_batch(nu, ni, B, seed):
    rs = np.random.RandomState(seed)
    return (rs.randint(0, nu, B).astype(np.int32), rs.randint(0, ni, B).astype(np.int32),
            rs.randint(0, ni, B).astype(np.int32))


SPECTRAL_EXACT = [  # (act, loss, reg, explicit A_hat^T); square loss only up to d = 8 and 2 layers (else
    ("identity", "hinge", 0.0, False),                  # hinge): its gradient grows with x, which grows with d and K
    ("relu", "square", 0.5, True), ("relu", "hinge", 0.25, False),
]


def spectral_exact_reference(case, act, loss, reg, n_sms):
    N, d, K = spectral_cases(n_sms)[case]
    loss = loss if d <= 8 and K <= 2 else "hinge"
    nu = N // 3
    A, F, e0 = spectral_exact_inputs(N, d, K, case)
    users, pos, neg = spectral_batch(nu, N - nu, 97, case)
    total, dE0, dW, allE = tf_math.spectralcf_loss_and_grad(A, e0, list(F), nu, users, pos, neg, reg, loss, act)
    mall, mx, MG, *back = spectral_magnitudes(A, F, e0, act, users, pos, neg, nu, reg, loss)
    rb = {0.0: 0, 0.5: 1, 0.25: 2}[reg]
    assert_exact(allE, mall, 0, "forward")
    m_emb = sum((mall[rows] ** 2).sum() for rows in (users, nu + pos, nu + neg))
    m_loss = ((1 + mx) ** (2 if loss == "square" else 1)).sum()
    assert_exact(total, m_loss + reg * m_emb, rb + 1, "loss")
    assert_exact(dE0, MG[:, :d] + (back[-1] if K else 0), rb, "dE0")
    for k in range(K):
        assert_exact(dW[k], back[2 * (K - 1 - k)], rb, ("dW", k))
    return N, d, K, nu, loss, A, F, e0, (users, pos, neg), (total, dE0, dW, allE)


@pytest.mark.parametrize("n_sms", [114, 132])
def test_spectralcf_exact_preconditions(n_sms):
    """CPU: the float64 references of every exact SpectralCF case meet the exactness precondition."""
    for case in range(len(spectral_cases(n_sms))):
        for act, loss, reg, _ in SPECTRAL_EXACT:
            spectral_exact_reference(case, act, loss, reg, n_sms)


@gpu
@pytest.mark.parametrize("act,loss,reg,explicit_t", SPECTRAL_EXACT)
@pytest.mark.parametrize("case", range(9))
def test_spectralcf_exact(case, act, loss, reg, explicit_t):
    """nrc_spectralcf_forward and nrc_spectralcf_grad (all-embedding table, dE0, every dW_k, loss) bit for bit the
    float64 tf_math chain, on both sides of the split predicate; the forward is bit-identical across two runs
    (the split-2 products add two partials onto zero)."""
    N, d, K, nu, loss, A, F, e0, (users, pos, neg), (total, dE0, dW, allE) = \
        spectral_exact_reference(case, act, loss, reg, sms())
    fwd, fwd2, rf, all_emb, gE, gF, l, rg = run_spectral(A, F, e0, act, nu, users, pos, neg, loss, reg, explicit_t)
    check_spectral_routes(rf, rg, N, K)
    assert np.array_equal(fwd, as_f32_exact(allE)) and np.array_equal(fwd, fwd2)
    assert np.array_equal(all_emb, fwd)
    assert np.array_equal(gE, as_f32_exact(dE0))
    for k in range(K):
        assert np.array_equal(gF[k], as_f32_exact(dW[k])), k
    assert l == as_f32_exact(np.float64(total))
    SEEN.add(("spectral_layers", K))
    SEEN.add(("spectral_dim", d))


_SELU_L, _SELU_A = 1.0507009873554805, 1.6732632423543772


def _act_err(act, z, y):
    """Rounding error bound (units of 2^-24) of the kernel's activation: sigmoid / tanh 4 units of the output
    (expf or tanhf 2 ulp, the add and divide); elu / selu 2 ulp of expf(z) itself (the subtraction of 1 cancels)
    plus 3 units of the output."""
    if act in ("sigmoid", "tanh"):
        return 4 * np.abs(y)
    scale = 1.0 if act == "elu" else _SELU_L * _SELU_A
    return (z <= 0) * 2 * scale * np.exp(np.minimum(z, 0)) + 3 * np.abs(y)


def spectral_chain(A, F, e0, act, nu, users, pos, neg, reg, chain_dw):
    """float64 values (tf_math) and first-order error bounds (units of 2^-24) of nrc_spectralcf_grad's quantities:
    products of n terms carry n times their absolute sums; an activation carries its derivative times the input error
    plus `_act_err`, its backward factor act'(y) the
    derivative of act' in y times y's error plus 3 units."""
    N, d = e0.shape
    absA = np.abs(A)
    total, dE0, dW, allE = tf_math.spectralcf_loss_and_grad(A, e0, list(F), nu, users, pos, neg, reg, "bpr", act)
    _, sides = tf_math.spectralcf_forward(A, e0, list(F), act)
    E, eE, errs, e_sides, zs = e0, np.zeros_like(e0), [np.zeros_like(e0)], [], []
    for k in range(len(F)):
        s = sides[k]
        es = absA @ eE + N * (absA @ np.abs(E))
        z = s @ F[k]
        ez = es @ np.abs(F[k]) + d * (np.abs(s) @ np.abs(F[k]))
        y = allE[:, (k + 1) * d:(k + 2) * d]
        dy = tf_math.activation_grad_from_output(act, y)
        eE = np.abs(dy) * ez + _act_err(act, z, y)
        E = y
        errs.append(eE)
        e_sides.append(es)
        zs.append((z, ez))
    eA = np.concatenate(errs, 1)
    D = allE.shape[1]
    ue, ie, xe_u, xe_i = allE[:nu], allE[nu:], eA[:nu], eA[nu:]
    pu, qi, qj, epu, eqi, eqj = ue[users], ie[pos], ie[neg], xe_u[users], xe_i[pos], xe_i[neg]
    x = (pu * qi).sum(1) - (pu * qj).sum(1)
    e_x = ((np.abs(pu) * (eqi + eqj) + epu * (np.abs(qi) + np.abs(qj))).sum(1)
           + D * (np.abs(pu) * (np.abs(qi) + np.abs(qj))).sum(1) + np.abs(x))
    g = -1.0 / (1.0 + np.exp(x))
    e_g = 0.25 * e_x + 4 * np.abs(g)
    G, eG, aG, cnt = (np.zeros_like(allE) for _ in range(4))
    gg, eg = g[:, None], e_g[:, None]
    for rows, c, ec in ((users, gg * (qi - qj) + reg * pu,
                         np.abs(qi - qj) * eg + np.abs(gg) * (eqi + eqj) + reg * epu + 3 * (np.abs(gg * (qi - qj)) + reg * np.abs(pu))),
                        (nu + pos, gg * pu + reg * qi, np.abs(pu) * eg + np.abs(gg) * epu + reg * eqi + 3 * (np.abs(gg * pu) + reg * np.abs(qi))),
                        (nu + neg, -gg * pu + reg * qj, np.abs(pu) * eg + np.abs(gg) * epu + reg * eqj + 3 * (np.abs(gg * pu) + reg * np.abs(qj)))):
        np.add.at(G, rows, c)
        np.add.at(eG, rows, ec)
        np.add.at(aG, rows, np.abs(c))
        np.add.at(cnt, rows, 1.0)
    eG = eG + cnt * aG
    carry, e_carry = np.zeros((N, d)), np.zeros((N, d))
    e_dW = [None] * len(F)
    for k in range(len(F), 0, -1):
        y = allE[:, k * d:(k + 1) * d]
        ey = eA[:, k * d:(k + 1) * d]
        a = tf_math.activation_grad_from_output(act, y)
        da = {"sigmoid": np.abs(1 - 2 * y), "tanh": 2 * np.abs(y), "elu": (y <= 0) * 1.0, "selu": (y <= 0) * 1.0}[act]
        ea = da * ey + 3 * np.abs(a)
        if act == "selu":       # act' jumps from scale * alpha to scale at 0: within z's band either may be taken
            z, ez = zs[k - 1]
            ea = ea + ((np.abs(z) <= C_BOUND * U24 * ez) & (ez > 0)) * (_SELU_L * _SELU_A - _SELU_L) / U24
        t = G[:, k * d:(k + 1) * d] + carry
        et = eG[:, k * d:(k + 1) * d] + e_carry + np.abs(t)
        dZ = t * a
        edZ = et * np.abs(a) + np.abs(t) * ea + np.abs(dZ)
        s, es = sides[k - 1], e_sides[k - 1]
        e_dW[k - 1] = np.abs(s).T @ edZ + es.T @ np.abs(dZ) + chain_dw * (np.abs(s).T @ np.abs(dZ))
        dS = dZ @ F[k - 1].T
        edS = edZ @ np.abs(F[k - 1]).T + d * (np.abs(dZ) @ np.abs(F[k - 1]).T)
        carry = A.T @ dS
        e_carry = absA.T @ edS + N * (absA.T @ np.abs(dS))
    e_dE0 = eG[:, :d] + e_carry + np.abs(dE0)
    return dict(all=allE, e_all=eA, dE0=dE0, e_dE0=e_dE0, dW=dW, e_dW=e_dW, loss=total)


@gpu
@pytest.mark.parametrize("act", ["sigmoid", "tanh", "elu", "selu"])
def test_spectralcf_rounded_conf_shape(ml100k, act):
    """The conf shape (ml-100k, d = 100, 2 layers, BPR, reg 1e-3 rounded to fp32) on a random dense operator of
    row sums about 1 and the init scale of the tables: within C * 2^-24 * M of float64 on the split-2 route, which
    is bit-identical across two runs."""
    nu, ni = ml100k["num_users"], ml100k["num_items"]
    N, d, K = nu + ni, 100, 2
    rs = np.random.RandomState(ord(act[0]))
    A = (rs.rand(N, N) * (rs.rand(N, N) < 0.01) * 0.2).astype(np.float32).astype(np.float64)
    F = (rs.randn(K, d, d) * np.sqrt(2.0 / (2 * d))).astype(np.float32).astype(np.float64)
    e0 = (rs.randn(N, d) * 0.3).astype(np.float32).astype(np.float64)
    users, pos, neg = spectral_batch(nu, ni, 256, 5)
    reg = float(np.float32(1e-3))
    per = ((N + 63) // 64 + 31) // 32 * 32
    chain_dw = per + (N + per - 1) // per               # the fma chain of one K slice, then one RED per slice
    R = spectral_chain(A, F, e0, act, nu, users, pos, neg, reg, chain_dw)
    assert np.abs(R["all"][:, d:]).max() > 0.1
    fwd, fwd2, rf, all_emb, gE, gF, l, rg = run_spectral(A, F, e0, act, nu, users, pos, neg, "bpr", reg, False)
    check_spectral_routes(rf, rg, N, K)
    assert rf["spectral_fwd_split"] == 2
    assert np.array_equal(fwd, fwd2)
    assert_within(fwd, R["all"], R["e_all"], "forward")
    assert_within(all_emb, R["all"], R["e_all"], "all_emb")
    assert_within(gE, R["dE0"], R["e_dE0"], "dE0")
    for k in range(K):
        assert_within(gF[k], R["dW"][k], R["e_dW"][k], ("dW", k))
    assert np.isclose(l, R["loss"], rtol=1e-5)
    SEEN.add(("spectral_act", act))


# ---------------------------------------------------------------------------------------------------------------
# d. the dropout mask, bit for bit
# ---------------------------------------------------------------------------------------------------------------
def philox4x32_10(c, k0, k1):
    """Philox4x32-10 (Salmon et al., SC'11) on uint64 arrays holding 32-bit words."""
    M0, M1, W0, W1, mask = 0xD2511F53, 0xCD9E8D57, 0x9E3779B9, 0xBB67AE85, 0xFFFFFFFF
    c0, c1, c2, c3 = (np.asarray(x, np.uint64) for x in c)
    k0, k1 = np.uint64(k0), np.uint64(k1)
    for _ in range(10):
        p0, p1 = np.uint64(M0) * c0, np.uint64(M1) * c2
        c0, c1, c2, c3 = (p1 >> np.uint64(32)) ^ c1 ^ k0, p1 & np.uint64(mask), (p0 >> np.uint64(32)) ^ c3 ^ k1, \
            p0 & np.uint64(mask)
        k0, k1 = (k0 + np.uint64(W0)) & np.uint64(mask), (k1 + np.uint64(W1)) & np.uint64(mask)
    return c0, c1, c2, c3


def dropout_mask_ref(n, keep, seed, stream_id):
    """The kernel's keep mask: word t of counter (q, q >> 32, 'DROP', stream_id) under key (seed, seed >> 32 ^
    stream_id >> 32) gives element 4 q + t the value 1 when (word >> 8) * 2^-24 < keep."""
    q = np.arange((n + 3) // 4, dtype=np.uint64)
    words = philox4x32_10((q & np.uint64(0xFFFFFFFF), q >> np.uint64(32), np.full_like(q, 0x44524F50),
                           np.full_like(q, stream_id & 0xFFFFFFFF)),
                          seed & 0xFFFFFFFF, ((seed >> 32) ^ (stream_id >> 32)) & 0xFFFFFFFF)
    w = np.stack(words, 1).reshape(-1)[:n]
    u = (w >> np.uint64(8)).astype(np.float64) * 2.0 ** -24
    return (u < np.float64(np.float32(keep))).astype(np.float32)


def test_philox_reference_known_answer():
    """CPU: the restatement reproduces the published Philox4x32-10 known-answer vectors (Random123 kat_vectors)."""
    out = philox4x32_10([0, 0, 0, 0], 0, 0)
    assert [int(x) for x in out] == [0x6627E8D5, 0xE169C58D, 0xBC57AC4C, 0x9B00DBD8]
    out = philox4x32_10([0xFFFFFFFF] * 4, 0xFFFFFFFF, 0xFFFFFFFF)
    assert [int(x) for x in out] == [0x408F276D, 0x41C83B0E, 0xA20BC7C6, 0x6D5451FD]


@gpu
@pytest.mark.parametrize("keep", [1.0, 0.5, 2.0 ** -10])
@pytest.mark.parametrize("stream_id", [3, (5 << 32) | 3])
def test_dropout_mask_bit_exact(keep, stream_id):
    """nrc_dropout_mask equals the numpy restatement for every element count, on two streams whose high words
    differ (they enter the key), and the two streams give different masks."""
    from neurec_b200 import ops
    for n in dropout_sizes(sms()):
        got = ops.dropout_mask(n, keep, 2017 | (7 << 32), stream_id).cpu().numpy()
        want = dropout_mask_ref(n, keep, 2017 | (7 << 32), stream_id)
        assert np.array_equal(got, want), n
        if keep == 1.0:
            assert (got == 1.0).all()
    if keep < 1:
        big = dropout_sizes(sms())[-1]
        other = dropout_mask_ref(big, keep, 2017 | (7 << 32), stream_id ^ (5 << 32))
        assert not np.array_equal(other, dropout_mask_ref(big, keep, 2017 | (7 << 32), stream_id))
        assert abs(dropout_mask_ref(big, keep, 1, stream_id).mean() - keep) < 5 * np.sqrt(keep / big) + 1e-6


# ---------------------------------------------------------------------------------------------------------------
# e. limits: the library's error, nothing written
# ---------------------------------------------------------------------------------------------------------------
def _raises_limit(fn, code_name="NRC_E_LIMIT"):
    from neurec_b200 import _lib
    with pytest.raises(_lib.NrcError) as e:
        fn()
    assert e.value.rc == getattr(_lib, code_name), str(e.value)


@gpu
def test_limits_write_nothing():
    """SpMM dim 257; NGCF embedding 65, width 65 and 5 layers; SpectralCF d = 129 and 9 layers: each call returns
    the library's error before any launch: outputs and the route record stay as they were."""
    from neurec_b200 import _lib, ops
    rs = np.random.RandomState(0)
    A = sp.random(50, 50, density=0.1, random_state=rs, format="csr", dtype=np.float32)
    A.sort_indices()
    ip, ix, va = csr_dev(A)
    before = routes()
    y = torch.full((50, 257), 7.0, device="cuda")
    s = torch.full((50, 257), 5.0, device="cuda")
    _raises_limit(lambda: ops.spmm_csr(ip, ix, va, torch.ones(50, 257, device="cuda"), y=y, sum_=s))
    torch.cuda.synchronize()
    assert bool((y == 7.0).all()) and bool((s == 5.0).all()) and routes() == before

    def ngcf_shape(emb, layers):
        sh = ops.NgcfShape()
        sh.num_users, sh.num_items, sh.emb_dim, sh.n_layers = 20, 30, emb, len(layers)
        for i, v in enumerate(layers[:4]):
            sh.layers[i] = v
        return sh

    for emb, layers in ((65, [16]), (16, [16, 65]), (16, [16, 16, 16, 16, 16])):
        sh = ngcf_shape(emb, layers)
        all_emb = torch.full((50, 400), 7.0, device="cuda")
        work = torch.full((1 << 16,), 5.0, device="cuda")
        _raises_limit(lambda: ops.ngcf_forward(sh, (ip, ix, va), None, torch.ones(50, emb, device="cuda"),
                                               torch.ones(20000, device="cuda"), None, 1.0, all_emb=all_emb,
                                               work=work))
        G = torch.zeros((50, 400), device="cuda")
        gE = torch.full((50, emb), 3.0, device="cuda")
        gW = torch.full((20000,), 3.0, device="cuda")
        loss2 = torch.zeros(2, device="cuda")
        t = torch.zeros(4, dtype=torch.int32, device="cuda")
        _raises_limit(lambda: ops.ngcf_grad(sh, (ip, ix, va), None, None, None, torch.ones(50, emb, device="cuda"),
                                            torch.ones(20000, device="cuda"), None, 1.0, t, t, t, 0.0, all_emb, G, gE,
                                            gW, work, loss2))
        torch.cuda.synchronize()
        assert bool((all_emb == 7.0).all()) and bool((work == 5.0).all()) and float(G.abs().max()) == 0.0
        assert bool((gE == 3.0).all()) and bool((gW == 3.0).all()) and float(loss2.abs().max()) == 0.0
        assert routes() == before

    for d, K, code in ((129, 1, "NRC_E_LIMIT"), (129, 0, "NRC_E_LIMIT"), (8, 9, None)):
        N, nu = 64, 20
        a_hat = torch.ones((N, N), device="cuda")
        e0 = torch.ones((N, d), device="cuda")
        filters = torch.ones((K, d, d), device="cuda")
        all_emb = torch.full((N, d * (K + 1)), 7.0, device="cuda")
        work = torch.full((N * d * (K + 3),), 5.0, device="cuda")
        grad_all = torch.zeros_like(all_emb)
        gE = torch.full((N, d), 3.0, device="cuda")
        gF = torch.full((K, d, d), 3.0, device="cuda")
        loss = torch.zeros(1, device="cuda")
        t = torch.zeros(4, dtype=torch.int32, device="cuda")
        calls = (lambda: ops.spectralcf_forward(a_hat, e0, filters, "identity", all_emb=all_emb, work=work),
                 lambda: ops.spectralcf_grad(nu, a_hat, None, e0, filters, "identity", t, t, t, "bpr", 0.0, all_emb,
                                             grad_all, torch.zeros(N, dtype=torch.int32, device="cuda"), gE, gF, work,
                                             loss))
        for call in calls:
            if code:
                _raises_limit(call, code)
            else:
                with pytest.raises(ValueError):                  # the reference's shape error (NRC_E_VALUE)
                    call()
            torch.cuda.synchronize()
            assert bool((all_emb == 7.0).all()) and bool((work == 5.0).all()) and float(grad_all.abs().max()) == 0
            assert bool((gE == 3.0).all()) and bool((gF == 3.0).all()) and float(loss.abs().max()) == 0
            assert routes() == before
    assert _lib.NRC_E_LIMIT != _lib.NRC_E_VALUE


# ---------------------------------------------------------------------------------------------------------------
# f. route completeness (runs last)
# ---------------------------------------------------------------------------------------------------------------
REQUIRED = {
    ("spmm", "fast", 8), ("spmm", "fast", 16), ("spmm", "fast", 32),
    ("spmm", "exact", 0), ("spmm", "exact", 1), ("spmm", "exact", 2), ("spmm", "exact", 4),
    ("spmm_capped", "fast", 0), ("spmm_capped", "fast", 1), ("spmm_capped", "exact", 0), ("spmm_capped", "exact", 1),
    ("ngcf_fwd_rows", 1), ("ngcf_fwd_rows", "many"), ("ngcf_bwd_tiles", 1), ("ngcf_bwd_tiles", "many"),
    ("ngcf_bpr_triplets", 1), ("ngcf_bpr_triplets", "many"),
    ("spectral_split", 0), ("spectral_split", 1), ("spectral_split", 2), ("spectral_dw", "split"),
    # not reported by the hook; recorded from the shapes the tests ran
    ("propagate_layers", 0), ("propagate_layers", 1), ("propagate_layers", 2), ("propagate_layers", 6),
    ("ngcf_layers", 2), ("ngcf_layers", 4), ("ngcf_widths", True), ("ngcf_widths", False),
    ("ngcf_sq", "zero"), ("ngcf_sq", "below_eps"),
    ("spectral_layers", 0), ("spectral_layers", 1), ("spectral_layers", 8),
    ("spectral_dim", 1), ("spectral_dim", 3), ("spectral_dim", 128),
    ("spectral_act", "sigmoid"), ("spectral_act", "tanh"), ("spectral_act", "elu"), ("spectral_act", "selu"),
}


@gpu
def test_every_route_was_seen(request):
    """Across this file the hook reported every route of the graph kernels.  Only meaningful when the whole file
    ran: a run of selected tests skips it."""
    here = {it.nodeid for it in request.session.items if it.fspath == request.node.fspath}
    every = {it.nodeid for it in request.node.parent.collect()}
    if here != every:
        pytest.skip("only part of this file was selected")
    assert REQUIRED <= SEEN, sorted(REQUIRED - SEEN)
