"""The SIMT evaluator on every route its shapes select, against the C oracle, bit for bit.

nrc_eval_mf picks its selection form by shape alone (ops.eval_last_routes reports which one ran):
  0  heap replay for every user (top_k >= 32)
  1  fast pass, 2 users per warp (at most 16 users per SM)
  2  fast pass on 128-item tiles (more users, fast-pass shared memory <= 200 KB)
  3  fast pass on 64-item tiles (dims too large for the 128-item tile)
and every fast form is followed by the heap replay of the users it could not decide.  The score-matrix
kernel (nrc_eval_score_matrix, nrc_arg_topk) has a fast pass for top_k <= 31 and shrinks from 8 to 4 warps
per CTA when a warp's heap and metric scratch exceed 12 KB.  Every case compares ranks and metric rows with
the oracle (equal_nan: Recall / NDCG of an empty test row are 0/0) and asserts the route it meant to reach.
"""
import numpy as np
import pytest
import torch

import oracle
from conftest import random_csr

pytestmark = pytest.mark.gpu
ALL = [1, 2, 3, 4, 5]
THREADS = 8


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def envelope_ok(dim, top_k, num_items):
    """nrc_eval_mf's shared-memory envelope as include/neurec_b200.h states it."""
    L = min(2 * top_k, num_items)
    d4 = (dim + 3) & ~3
    return 256 * (2 * d4 + 4 + 2 * L + 3 * top_k) <= 227 * 1024


def batch_csr(users, ptr, idx):
    """Rows of a CSR indexed by user id, re-indexed by batch row (as the oracle takes the test sets)."""
    rows = [idx[ptr[u]:ptr[u + 1]] for u in users]
    p = np.zeros(len(users) + 1, np.int64)
    p[1:] = np.cumsum([len(r) for r in rows])
    return p, (np.concatenate(rows) if rows else np.zeros(0, np.int32)).astype(np.int32)


def oracle_mf(U, V, users, tp, ti, sp, si, K, scores=False):
    """(results, ranks[, masked scores]) of the oracle's predict -> mask -> evaluate."""
    S = oracle.mask_train(oracle.mf_scores(U, V, users, THREADS), users, tp, ti)
    out = oracle.evaluate_matrix(S, *batch_csr(users, sp, si), ALL, K, thread_num=THREADS, return_ranks=True)
    return out + (S,) if scores else out


def undecided(S, K):
    """Rows the tie-free fast pass must leave to the heap replay: the K+1 best non-NaN scores are not finite and
    strictly decreasing, or a NaN sits in the heap seed [0, L)."""
    L = min(2 * K, S.shape[1])
    top = -np.sort(-np.where(np.isnan(S), -np.inf, S), axis=1)[:, :K + 1]
    top = np.pad(top, ((0, 0), (0, K + 1 - top.shape[1])), constant_values=-np.inf)
    ok = (top[:, :-1] > top[:, 1:]).all(1) & (top[:, K] > -np.inf) & ~np.isnan(S[:, :L]).any(1)
    return int((~ok).sum())


def run_mf(U, V, users, tp, ti, sp, si, K):
    from neurec_b200 import ops
    res, ranks = ops.eval_mf(dev(U), dev(V), dev(users), dev(tp), dev(ti), dev(sp), dev(si), ALL, K,
                             return_ranks=True)
    return res.cpu().numpy(), ranks.cpu().numpy()


def assert_same(got, want):
    assert np.array_equal(got[1], want[1])
    assert np.array_equal(got[0], want[0], equal_nan=True)


@pytest.fixture(autouse=True)
def _no_forced_exact():
    from neurec_b200 import _lib
    _lib.load().nrc_eval_force_exact(0)
    yield


def n_users(kind):
    return {"sm16": 16 * sms(), "sm16+1": 16 * sms() + 1}.get(kind, kind)


def tables(rs, nu, ni, dim, ints):
    if ints:   # few distinct scores: ties inside the top K+1 of most users
        return (rs.randint(-1, 2, (nu, dim)).astype(np.float32), rs.randint(-1, 2, (ni, dim)).astype(np.float32))
    return (rs.randn(nu, dim) * 0.1).astype(np.float32), (rs.randn(ni, dim) * 0.1).astype(np.float32)


# (users, dim, top_k, num_items, integer tables, form)
FORM_CASES = [
    ("sm16", 64, 20, 1001, False, 1),
    ("sm16", 7, 31, 999, True, 1),
    ("sm16+1", 64, 20, 1001, False, 2),
    ("sm16+1", 64, 20, 1001, True, 2),
    (3000, 7, 31, 999, False, 2),          # dim % 4 != 0: scalar V-tile load
    (3003, 10, 1, 517, True, 2),
    (2222, 128, 31, 1283, False, 2),
    (2222, 200, 20, 900, False, 2),
    (2222, 256, 6, 900, False, 2),         # the largest top_k the 128-item tile takes at dim 256
    (2222, 256, 7, 900, False, 3),
    (2500, 301, 20, 700, False, 3),        # scalar V-tile load on 64-item tiles
    (2222, 300, 20, 650, True, 3),
    (2222, 448, 1, 650, False, 3),         # the largest dim the envelope takes
    (3000, 64, 32, 1001, False, 0),
    (3000, 33, 100, 1001, True, 0),
    ("sm16+1", 64, 20, 20, False, 2),      # num_items == top_k: nobody is decided by the fast pass
    ("sm16+1", 64, 20, 21, False, 2),      # num_items == top_k + 1
    (300, 7, 31, 31, False, 1),
    (500, 33, 32, 33, False, 0),
]


@pytest.mark.parametrize("case", FORM_CASES, ids=lambda c: "u%s-d%d-k%d-n%d-%s" % (c[0], c[1], c[2], c[3], "int" if c[4] else "f"))
def test_eval_mf_every_form_vs_oracle(case):
    from neurec_b200 import ops
    kind, dim, K, N, ints, form = case
    B = n_users(kind)
    rs = np.random.RandomState(dim * 1000 + K + N)
    nu = max(B, 3500)
    U, V = tables(rs, nu, N, dim, ints)
    users = rs.randint(0, nu, B).astype(np.int32)                 # arbitrary order, repeats
    tp, ti = random_csr(rs, nu, N, rs.randint(0, max(2, min(N - K - 1, 40)), nu))
    sp, si = random_csr(rs, nu, N, rs.randint(0, 8, nu))            # some empty test rows
    got = run_mf(U, V, users, tp, ti, sp, si, K)
    assert ops.eval_last_routes()["mf_form"] == form
    und = ops.eval_last_undecided()
    *want, S = oracle_mf(U, V, users, tp, ti, sp, si, K, scores=True)
    assert_same(got, tuple(want))
    if form:   # the replay after the fast pass ran for exactly the users with ties or too few items
        assert und == undecided(S, K)
        if ints or N <= K + 1:
            assert und > 0


def special_train_rows(nu, N, K, rs):
    """Train rows that stress the per-tile mask walk and the heap seed."""
    L = min(2 * K, N)
    kinds = [
        [],                                                         # empty
        np.setdiff1d(np.arange(N), rs.choice(N, K // 2 + 1, replace=False)),   # fewer than K+1 unmasked
        np.arange(130, 170),                                        # run of 40 inside one 64- / 128-item tile
        np.arange(100, 150),                                        # run across the tile boundary at 128
        np.arange(0, L, 2),                                         # inside the heap seed [0, L)
        np.array([0, L - 1, L, 63, 64, 127, 128, 191, 192, 255, 256, N - 1]),  # tile and seed edges
        np.concatenate([np.arange(L), np.arange(250, 330)]),        # the whole seed + a run of 80
    ]
    return oracle.lists_to_csr([np.asarray(kinds[u % len(kinds)])[np.asarray(kinds[u % len(kinds)]) < N]
                                for u in range(nu)])


@pytest.mark.parametrize("kind,dim,K,form", [("sm16", 64, 20, 1), ("sm16+1", 64, 20, 2), ("sm16+1", 300, 20, 3),
                                            ("sm16+1", 256, 31, 3), ("sm16+1", 64, 32, 0)])
def test_eval_mf_masks_and_truth_rows(kind, dim, K, form):
    from neurec_b200 import ops
    B = n_users(kind)
    N = 1001
    rs = np.random.RandomState(dim + K)
    U, V = tables(rs, B, N, dim, False)
    users = rs.permutation(B).astype(np.int32)
    tp, ti = special_train_rows(B, N, K, rs)
    sp, si = random_csr(rs, B, N, np.where(np.arange(B) % 3 == 0, 0, rs.randint(1, 10, B)))   # empty test rows
    got = run_mf(U, V, users, tp, ti, sp, si, K)
    assert ops.eval_last_routes()["mf_form"] == form
    want = oracle_mf(U, V, users, tp, ti, sp, si, K)
    assert_same(got, want)
    assert np.isnan(want[0]).any()          # 0/0 metrics of the empty test rows were compared


@pytest.mark.parametrize("dim,kmax", [(64, 110), (448, 1)])
def test_eval_mf_envelope(dim, kmax):
    """The largest accepted top_k (from the header's formula) gives the oracle's results; one more is refused with
    NRC_E_LIMIT before anything is written; eval_mf_auto then takes the materialised route to the same results."""
    from neurec_b200 import _lib, ops
    N, B = 1000, 64
    assert max(k for k in range(1, 513) if envelope_ok(dim, k, N)) == kmax
    rs = np.random.RandomState(dim)
    U, V = tables(rs, B, N, dim, False)
    users = np.arange(B, dtype=np.int32)
    tp, ti = random_csr(rs, B, N, rs.randint(0, 30, B))
    sp, si = random_csr(rs, B, N, rs.randint(0, 6, B))
    assert_same(run_mf(U, V, users, tp, ti, sp, si, kmax), oracle_mf(U, V, users, tp, ti, sp, si, kmax))
    K = kmax + 1
    t = [dev(x) for x in (U, V, users, tp, ti, sp, si)]
    res = torch.full((B, 5 * K), -7.0, device="cuda")
    ranks = torch.full((B, K), -7, dtype=torch.int32, device="cuda")
    m = np.asarray(ALL, np.int32)
    rc = _lib.load().nrc_eval_mf(*[ops._p(x) for x in t[:2]], dim, N, ops._p(t[2]), B, *[ops._p(x) for x in t[3:]],
                                 m.ctypes.data, 5, K, ops._p(res), ops._p(ranks), ops._stream())
    assert rc == _lib.NRC_E_LIMIT
    torch.cuda.synchronize()
    assert (res == -7).all() and (ranks == -7).all()
    got = ops.eval_mf_auto(*t, ALL, K, return_ranks=True)
    assert_same((got[0].cpu().numpy(), got[1].cpu().numpy()), oracle_mf(U, V, users, tp, ti, sp, si, K))


def score_rows(rs, B, N, kind):
    S = rs.randn(B, N).astype(np.float32)
    if kind == "ints":
        S = rs.randint(0, 4, (B, N)).astype(np.float32)
    S[0] = -np.inf                                                  # all -inf
    S[1, rs.rand(N) < 0.5] = np.inf                                 # mixed +-inf
    S[1, rs.rand(N) < 0.3] = -np.inf
    return S


# (rows, rating_len, top_k, fast pass, warps of the score matrix); arg_topk checked at the same top_k
ROWS_CASES = [
    (70, 1000, 20, 1, 8),
    (70, 20, 5, 1, 8),                     # rating_len < 32
    (70, 31, 31, 0, 8),                    # rating_len == top_k
    (70, 32, 31, 1, 8),                    # rating_len == top_k + 1
    (40, 3000, 400, 0, 8),
    (40, 3000, 438, 0, 8),                 # the largest top_k with 8 warps
    (40, 3000, 439, 0, 4),
    (40, 3000, 512, 0, 4),
]


@pytest.mark.parametrize("case", ROWS_CASES, ids=lambda c: "n%d-k%d" % (c[1], c[2]))
@pytest.mark.parametrize("kind", ["randn", "ints"])
def test_score_matrix_and_arg_topk_routes(case, kind):
    from neurec_b200 import ops
    B, N, K, fast, warps = case
    rs = np.random.RandomState(N + K)
    S = score_rows(rs, B, N, kind)
    ip, ix = random_csr(rs, B, N, rs.randint(0, 12, B))
    want = oracle.evaluate_matrix(S, ip, ix, ALL, K, thread_num=THREADS, return_ranks=True)
    got = ops.eval_score_matrix(dev(S), dev(ip), dev(ix), ALL, K, return_ranks=True)
    assert ops.eval_last_routes()["rows_fast"] == fast and ops.eval_last_routes()["rows_warps"] == warps
    assert_same((got[0].cpu().numpy(), got[1].cpu().numpy()), want)
    assert np.array_equal(ops.arg_topk(dev(S), K).cpu().numpy(), oracle.arg_topk(S, K, THREADS))


@pytest.mark.parametrize("K,warps", [(600, 8), (614, 8), (615, 4), (1024, 4)])
def test_arg_topk_large_top_k(K, warps):
    from neurec_b200 import ops
    rs = np.random.RandomState(K)
    S = score_rows(rs, 40, 2000, "ints")
    got = ops.arg_topk(dev(S), K).cpu().numpy()
    r = ops.eval_last_routes()
    assert (r["rows_fast"], r["rows_warps"]) == (0, warps)
    assert np.array_equal(got, oracle.arg_topk(S, K, THREADS))


def test_host_variants_stream_several_chunks():
    """rating_len 100 003: 167 rows per 64 MB chunk, so 400 rows take three chunks (the last partial) through both
    staging buffers and streams; the host, device and oracle results agree."""
    from neurec_b200 import ops
    B, N, K = 400, 100003, 20
    rs = np.random.RandomState(5)
    S = rs.randn(B, N).astype(np.float32)
    S[::7, :2000] = np.round(S[::7, :2000])                         # ties in some rows
    ip, ix = random_csr(rs, B, N, rs.randint(0, 10, B))
    want, wranks = oracle.evaluate_matrix(S, ip, ix, ALL, K, thread_num=THREADS, return_ranks=True)
    res_h, ranks_h = ops.eval_score_matrix_host(S, ip, ix, ALL, K, return_ranks=True)
    assert np.array_equal(ranks_h, wranks) and np.array_equal(res_h, want, equal_nan=True)
    res_d, ranks_d = ops.eval_score_matrix(dev(S), dev(ip), dev(ix), ALL, K, return_ranks=True)
    assert np.array_equal(ranks_d.cpu().numpy(), wranks) and np.array_equal(res_d.cpu().numpy(), want, equal_nan=True)
    assert np.array_equal(ops.arg_topk_host(S, 40), oracle.arg_topk(S, 40, THREADS))


# ------------------------------------------------------------------------------------- non-finite scores
def nonfinite_tables(rs, nu, ni, dim, K, kind):
    """NaN scores inside / outside the heap seed [0, L): NaN item rows, NaN user rows, inf * 0 products."""
    L = min(2 * K, ni)
    U = (rs.randn(nu, dim) * 0.1).astype(np.float32)
    V = (rs.randn(ni, dim) * 0.1).astype(np.float32)
    if kind == "item_in":
        V[[1, L - 1]] = np.nan
    elif kind == "item_out":
        V[[L, ni - 3]] = np.nan
    elif kind == "user":
        U[::7] = np.nan
    else:   # inf * 0: NaN at items 2 and ni - 5 for every third user, +-inf there for the others
        V[[2, ni - 5], 1] = np.inf
        U[::3, 1] = 0.0
    return U, V


NONFINITE = ["item_in", "item_out", "user", "inf0"]


@pytest.mark.parametrize("kind", NONFINITE)
@pytest.mark.parametrize("users,dim,K,form", [("sm16", 64, 20, 1), ("sm16+1", 64, 20, 2), ("sm16+1", 300, 20, 3),
                                              ("sm16+1", 64, 32, 0)])
def test_non_finite_scores_eval_mf(kind, users, dim, K, form):
    from neurec_b200 import ops
    B, N = n_users(users), 1001
    rs = np.random.RandomState(dim + K)
    U, V = nonfinite_tables(rs, B, N, dim, K, kind)
    us = np.arange(B, dtype=np.int32)
    tp, ti = random_csr(rs, B, N, rs.randint(0, 30, B))
    sp, si = random_csr(rs, B, N, rs.randint(0, 6, B))
    got = run_mf(U, V, us, tp, ti, sp, si, K)
    assert ops.eval_last_routes()["mf_form"] == form
    und = ops.eval_last_undecided()
    *want, S = oracle_mf(U, V, us, tp, ti, sp, si, K, scores=True)
    assert_same(got, tuple(want))
    if form:
        assert und == undecided(S, K)


@pytest.mark.parametrize("kind", NONFINITE)
@pytest.mark.parametrize("K", [5, 20, 40])
def test_non_finite_scores_score_matrix_and_arg_topk(kind, K):
    from neurec_b200 import ops
    B, N = 300, 700
    rs = np.random.RandomState(K)
    U, V = nonfinite_tables(rs, B, N, 16, K, kind)
    S = oracle.mf_scores(U, V, np.arange(B, dtype=np.int32))
    ip, ix = random_csr(rs, B, N, rs.randint(0, 6, B))
    want = oracle.evaluate_matrix(S, ip, ix, ALL, K, thread_num=THREADS, return_ranks=True)
    got = ops.eval_score_matrix(dev(S), dev(ip), dev(ix), ALL, K, return_ranks=True)
    assert ops.eval_last_routes()["rows_fast"] == (1 if K < 32 else 0)
    assert_same((got[0].cpu().numpy(), got[1].cpu().numpy()), want)
    assert np.array_equal(ops.arg_topk(dev(S), K).cpu().numpy(), oracle.arg_topk(S, K, THREADS))
    assert np.array_equal(ops.arg_topk_host(S, K), oracle.arg_topk(S, K, THREADS))


@pytest.mark.parametrize("kind", NONFINITE)
@pytest.mark.parametrize("dim", [64, 128])
def test_non_finite_scores_tensor_core_path(kind, dim):
    from neurec_b200 import ops
    B, N, K = 256, 16411, 20
    rs = np.random.RandomState(dim)
    U, V = nonfinite_tables(rs, B, N, dim, K, kind)
    us = rs.permutation(B).astype(np.int32)
    tp, ti = random_csr(rs, B, N, rs.randint(0, 40, B))
    sp, si = random_csr(rs, B, N, rs.randint(0, 6, B))
    res, ranks = ops.eval_mf_tc(dev(U), dev(V), dev(us), dev(tp), dev(ti), dev(sp), dev(si), ALL, K, return_ranks=True)
    assert_same((res.cpu().numpy(), ranks.cpu().numpy()), oracle_mf(U, V, us, tp, ti, sp, si, K))


# ------------------------------------------------------------------------------------- item-sharded pieces
@pytest.mark.parametrize("dim", [4, 68, 128])
def test_mf_score_pairs_vs_oracle(dim):
    from neurec_b200 import ops
    B, C, N = 200, 45, 3001
    rs = np.random.RandomState(dim)
    Ur = (rs.randn(B, dim) * 0.1).astype(np.float32)
    V = (rs.randn(N, dim) * 0.1).astype(np.float32)
    items = rs.randint(0, N, (B, C)).astype(np.int32)
    items[rs.rand(B, C) < 0.1] = -1
    tp, ti = oracle.lists_to_csr([rs.choice(items[b][items[b] >= 0], 5) for b in range(B)])   # masked candidates
    got = ops.mf_score_pairs(dev(Ur), dev(V), dev(items), dev(tp), dev(ti)).cpu().numpy()
    full = oracle.mf_scores(Ur, V, np.arange(B, dtype=np.int32), THREADS)
    oracle.mask_train(full, np.arange(B, dtype=np.int32), tp, ti)
    want = np.where(items >= 0, np.take_along_axis(full, np.maximum(items, 0), 1), -np.inf).astype(np.float32)
    assert np.array_equal(got, want)


def merge_reference(ids, sc, K):
    """(score desc, id asc) over the candidates that are neither NaN nor -inf; tie when equal scores sit inside the
    top K+1, fewer than K+1 candidates exist, or any candidate is NaN."""
    B = ids.shape[0]
    ranks = np.full((B, K), -1, np.int32)
    ties = 0
    for b in range(B):
        ok = ~np.isnan(sc[b]) & (sc[b] > -np.inf)
        order = np.lexsort((ids[b][ok], -sc[b][ok]))
        top = order[:K + 1]
        ranks[b, :min(K, len(top))] = ids[b][ok][top[:K]]
        v = sc[b][ok][top]
        ties += int(len(v) < K + 1 or (v[:-1] == v[1:]).any() or np.isnan(sc[b]).any())
    return ranks, ties


@pytest.mark.parametrize("K,C", [(1, 2), (1, 33), (1, 512), (31, 32), (31, 33), (31, 512), (384, 385), (384, 512),
                                 (400, 401), (400, 512), (511, 512)])
def test_merge_candidates_vs_numpy(K, C):
    from neurec_b200 import ops
    B, N = 48, 20000
    rs = np.random.RandomState(K * 1000 + C)
    ids = np.stack([rs.choice(N, C, replace=False) for _ in range(B)]).astype(np.int32)
    sc = (rs.randn(B, C)).astype(np.float32)
    sc[::4] = np.round(sc[::4] * 4)                                # exact ties
    sc[9] = np.arange(C, dtype=np.float32)                         # distinct scores
    pad = rs.rand(B, C) < 0.05                                     # -1 / -inf padding
    pad[5, :] = True
    ids[pad] = -1
    sc[pad] = -np.inf
    sc[7, rs.randint(0, C)] = np.nan                               # a NaN candidate
    sc[11] = np.arange(C, dtype=np.float32)
    sc[11, C // 2] = np.inf                                         # one +inf: ranked first, no tie
    sc[13, [0, C - 1]] = np.inf                                     # two +inf: a tie
    ids[[11, 13]] = np.stack([rs.choice(N, C, replace=False) for _ in range(2)])
    fin = ~np.isnan(sc) & (sc > -np.inf)
    truth = [rs.choice(ids[b][fin[b]], min(5, int(fin[b].sum())), replace=False) for b in range(B)]
    tp, ti = oracle.lists_to_csr(truth)
    res, ranks, ties = ops.eval_merge_candidates(dev(ids), dev(sc), dev(tp), dev(ti), ALL, K, return_ranks=True)
    want_ranks, want_ties = merge_reference(ids, sc, K)
    assert np.array_equal(ranks.cpu().numpy(), want_ranks)
    assert int(ties.item()) == want_ties
    # metrics: the oracle on a matrix whose top K is exactly that ranking
    S = np.full((B, N), -np.inf, np.float32)
    for b in range(B):
        r = want_ranks[b][want_ranks[b] >= 0]
        S[b, r] = np.arange(K, K - len(r), -1, dtype=np.float32)
    assert int(want_ranks[11, 0]) == int(ids[11, C // 2]) and want_ranks[13, 0] >= 0
    want = oracle.evaluate_matrix(S, tp, ti, ALL, K, thread_num=THREADS)
    assert np.array_equal(res.cpu().numpy(), want, equal_nan=True)


# ------------------------------------------------------------------------------------- glue
@pytest.mark.parametrize("dim", [1, 7, 33, 300])
def test_mf_scores_is_the_oracle_fma_chain(dim):
    from neurec_b200 import ops
    rs = np.random.RandomState(dim)
    U = rs.randn(300, dim).astype(np.float32)
    V = rs.randn(1001, dim).astype(np.float32)
    users = rs.randint(0, 300, 257).astype(np.int32)
    got = ops.mf_scores(dev(U), dev(V), dev(users)).cpu().numpy()
    assert np.array_equal(got, oracle.mf_scores(U, V, users, THREADS))


def test_mask_rows_equals_oracle_with_repeated_users():
    from neurec_b200 import ops
    rs = np.random.RandomState(2)
    nu, N = 500, 777
    tp, ti = random_csr(rs, nu, N, rs.randint(0, 200, nu))
    users = np.concatenate([rs.randint(0, nu, 300), [3, 3, 3]]).astype(np.int32)
    S = rs.randn(len(users), N).astype(np.float32)
    got = ops.mask_rows(dev(S), dev(users), dev(tp), dev(ti)).cpu().numpy()
    assert np.array_equal(got, oracle.mask_train(S.copy(), users, tp, ti))


def test_mean_rows_is_numpy_mean():
    from neurec_b200 import ops
    rs = np.random.RandomState(3)
    for rows in (1, 127, 128, 129, 257, 100001):
        for cols in (1, 31, 33, 250):
            a = rs.rand(rows, cols).astype(np.float32)
            assert np.array_equal(ops.mean_rows(dev(a)).cpu().numpy(), np.mean(a, axis=0)), (rows, cols)
    for rows in (262145, 1000003, 4194319):   # one column: numpy's pairwise split tree 12 to 16 levels deep
        a = rs.rand(rows, 1).astype(np.float32)
        assert np.array_equal(ops.mean_rows(dev(a)).cpu().numpy(), np.mean(a, axis=0)), rows


# ------------------------------------------------------------------------------------- surface
def test_uni_evaluator_beyond_the_fused_envelope():
    """dim 64 takes top_k <= 110 in the fused kernel; UniEvaluator at top_k 200 gives the oracle's metrics."""
    from neurec_b200.evaluator.uni_evaluator import UniEvaluator
    nu, ni, dim, K = 300, 1000, 64, 200
    assert not envelope_ok(dim, K, ni)
    rs = np.random.RandomState(8)
    U = (rs.randn(nu, dim) * 0.1).astype(np.float32)
    V = (rs.randn(ni, dim) * 0.1).astype(np.float32)
    tp, ti = random_csr(rs, nu, ni, rs.randint(1, 60, nu))
    sp, si = random_csr(rs, nu, ni, rs.randint(1, 8, nu))
    train = {u: ti[tp[u]:tp[u + 1]].tolist() for u in range(nu)}
    test = {u: si[sp[u]:sp[u + 1]].tolist() for u in range(nu)}

    class Model:
        def get_eval_tables(self):
            return dev(U), dev(V)
    ev = UniEvaluator(train, test, metric=["Precision", "Recall", "NDCG"], top_k=[10, 100, 200])
    got = ev.evaluate(Model())
    users = np.arange(nu, dtype=np.int32)
    bp, bi = batch_csr(users, sp, si)
    rows = oracle.eval_mf(U, V, users, tp, ti, bp, bi, [1, 2, 4], K, thread_num=THREADS)
    final = np.mean(rows, axis=0).reshape(3, K)[:, [9, 99, 199]].reshape(-1)
    assert got == "\t".join([("%.8f" % x).ljust(12) for x in final])
