"""White-box tests of the tensor-core evaluator's candidate passes: the lists tc_candidate_kernel writes
(read back through nrc_eval_tc_debug_candidates, which runs a pass exactly as nrc_eval_mf_tc does) are
checked against the invariants the exact re-scoring relies on.  tests/test_tc_algorithm_model.py states
them on a numpy model of the algorithm; here they are checked on the real kernel's output:

  I1  every id is an unmasked item in [0, N) inside its list's item segment (and, with two filter
      threads per user, inside its half of the tile); no item twice for a user; every list ascending;
  I2  |approximate score - exact score| <= margin / 2 for every candidate, and the margin is
      2 (2^-7 + 2^-11) |u| max_i |v_i| 1.001;
  I3  main pass (threshold rank K + 1): every unmasked item whose exact score is >= the exact (K+1)-th
      best is a candidate, ties at the cut included;
  I4  replay pass (threshold rank L = min(2K, N)): every item >= L that enters the reference's heap
      (evaluate.h:38-41, strict >) when the exact scores are offered in item order is a candidate.

Exact scores are the oracle's fp32 FMA chain (oracle.mf_scores)."""
import heapq

import numpy as np
import pytest
import torch

import oracle
from conftest import random_csr
from test_tc_algorithm_model import CASES, adversarial_top1_tables

pytestmark = pytest.mark.gpu

EPS_REL = 2.0 ** -7 + 2.0 ** -11
KS = (1, 5, 16, 31)
# tables whose scores mostly lie within the margin of each other (or tie in masses; with heavy-tailed item
# norms the margin, which scales with the LARGEST item norm, dwarfs the typical score): with few segments
# most lists overflow, by design; only many short segments give overflow-free lists there
OVERFLOWING = {"cancelling", "heavy_tail_norms", "worst_rounding", "worst_rounding_up"}


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def tile_items(dim):
    return 128 if dim <= 128 else 64


def expected_segments(N, dim, g):
    """Forced segment count -> (segments, items per segment), the rule of run_pass."""
    T = -(-N // tile_items(dim))
    G = T if g == 0 else min(g, T)
    seg_tiles = -(-T // G)
    return -(-T // seg_tiles), seg_tiles * tile_items(dim)


def subnormal_tables(rs, nu, n, d):
    """User entries ~1e-20, item entries spread over 1e-19 .. 1e-17: products and partial sums fall in
    the fp32 subnormal range (< 2^-126 ~ 1.2e-38)."""
    U = (rs.choice([-1.0, 1.0], (nu, d)) * rs.uniform(0.5, 2.0, (nu, d)) * 1e-20).astype(np.float32)
    V = (rs.choice([-1.0, 1.0], (n, d)) * 10.0 ** rs.uniform(-19, -17, (n, d))).astype(np.float32)
    return U, V


def make_tables(kind, nu, n, d, seed):
    """User table [nu, d] and item table [n, d] of one kind."""
    rs = np.random.RandomState(seed)
    if kind == "subnormal":
        return subnormal_tables(rs, nu, n, d)
    if kind == "integers":                      # mass ties: integer scores, exact in bf16 and fp32
        return (rs.randint(-2, 3, (nu, d)).astype(np.float32), rs.randint(-2, 3, (n, d)).astype(np.float32))
    if kind == "gauss_dups":
        U = (rs.randn(nu, d) * 0.1).astype(np.float32)
        U[rs.rand(nu) < 0.08] = 0.0                                   # all-zero user rows (margin 0)
        V = (rs.randn(n, d) * 0.1).astype(np.float32)
        hubs = (rs.randn(4, d) * 0.3).astype(np.float32)              # larger rows: they reach the top lists
        for j, pos in enumerate(np.linspace(0, n - 1, 24).astype(int)):
            V[pos] = hubs[j % 4]                                      # identical rows in different segments
        V[n - 1] = hubs[0]
        return U, V
    if kind == "top1_decoys":                   # two bf16-rounding decoys in front of the exact top-1
        u, V = adversarial_top1_tables(n_items=n, d=d)
        V[3:] *= rs.uniform(0.2, 1.0, size=(n - 3, 1)).astype(np.float32)
        return np.stack([u * np.float32(2.0 ** (j % 7 - 3)) for j in range(nu)]), V
    _, V = CASES[kind](rs, n, d)
    U = np.stack([CASES[kind](np.random.RandomState(seed * 1000 + j), 1, d)[0] * np.float32(2.0 ** (j % 5 - 2))
                  for j in range(nu)]).astype(np.float32)
    return U, V


class Problem:
    def __init__(self, kind, n_users, N, dim, seed):
        self.N, self.dim = N, dim
        nu = n_users + 17                                             # evaluate a permuted subset of the rows
        self.U, self.V = make_tables(kind, nu, N, dim, seed)
        rs = np.random.RandomState(seed + 1)
        self.users = rs.permutation(nu)[:n_users].astype(np.int32)
        self.tp, self.ti = random_csr(rs, nu, N, rs.randint(0, min(80, N // 2), nu))
        S = oracle.mf_scores(self.U, self.V, self.users, thread_num=8)
        self.exact = S.copy()
        oracle.mask_train(S, self.users, self.tp, self.ti)
        self.exm = S                                                  # masked exact scores (train items -inf)
        self.masked = np.isneginf(S) & ~np.isneginf(self.exact)
        un = np.sqrt((self.U[self.users].astype(np.float64) ** 2).sum(1))
        vmax = np.sqrt((self.V.astype(np.float64) ** 2).sum(1)).max()
        self.margin = 2.0 * EPS_REL * un * vmax * 1.001
        self.d = dict(U=dev(self.U), V=dev(self.V), users=dev(self.users), tp=dev(self.tp), ti=dev(self.ti))

    def lists(self, pass_, lq, G, CH, cap):
        from neurec_b200 import ops
        ops.eval_tc_force_segments(G if G > 0 else 1 << 30)
        ops.eval_tc_epilogue_warps(8 * CH)
        try:
            segs, seg_items = expected_segments(self.N, self.dim, G)
            ch = CH if pass_ == 0 else 1                              # the replay pass keeps one thread per user
            cap = min(cap, -(-seg_items // ch))                       # no list can hold more than its columns
            cand, val, cnt, margin, got_seg = ops.eval_tc_debug_candidates(
                pass_, self.d["U"], self.d["V"], self.d["users"], self.d["tp"], self.d["ti"], lq, cap, segs * ch)
            torch.cuda.synchronize()
        finally:
            ops.eval_tc_force_segments(0)
            ops.eval_tc_epilogue_warps(8)
        assert cnt.shape[1] == segs * ch and got_seg == seg_items, (cnt.shape, segs, ch, got_seg, seg_items)
        return cand.cpu().numpy(), val.cpu().numpy(), cnt.cpu().numpy(), margin.cpu().numpy(), ch, seg_items, cap


def reference_heap_entries(s, L):
    """Items >= L that enter the reference's heap (evaluate.h:38-41): seeded with the first L scores,
    an item replaces the root when its score is strictly greater.  The root never decreases, so blocks
    of items below the current root are skipped with one vector comparison."""
    h = [float(x) for x in s[:L]]
    heapq.heapify(h)
    out = []
    for b0 in range(L, len(s), 4096):
        blk = s[b0:b0 + 4096]
        for t in np.nonzero(blk > h[0])[0]:
            v = float(blk[t])
            if v > h[0]:
                heapq.heapreplace(h, v)
                out.append(b0 + int(t))
    return out


def check_pass(P, pass_, K, G, CH):
    """Runs one pass and checks I1-I4 on its lists (every violated invariant is reported, not only the
    first); returns the number of users with an overflowed list."""
    N, n = P.N, len(P.users)
    L = min(2 * K, N)
    lq, cap = (K + 1, 1024) if pass_ == 0 else (L, 2048)
    cand, val, cnt, margin, ch, seg_items, cap = P.lists(pass_, lq, G, CH, cap)
    ctx = (pass_, K, G, CH, N, P.dim)
    NT = tile_items(P.dim)
    failed = []

    def expect(ok, name, *detail):
        if not ok:
            failed.append((name,) + detail)

    # I2 (margin): the device's fp32 margin is the formula to fp32 rounding
    expect(np.allclose(margin.astype(np.float64), P.margin, rtol=1e-5, atol=0.0), "I2 margin formula")
    assert cnt.min() >= 0
    valid = np.arange(cap)[None, None, :] < np.minimum(cnt, cap)[:, :, None]
    rows, slots, _ = np.nonzero(valid)
    ids, vals = cand[valid], val[valid]
    # I1
    assert ((ids >= 0) & (ids < N)).all(), ctx
    expect(not P.masked[rows, ids].any(), "I1 train item")
    expect((ids // seg_items == slots // ch).all(), "I1 segment")
    if ch == 2:
        expect(((ids % NT) // (NT // 2) == slots % 2).all(), "I1 half tile")
    inner = valid[:, :, 1:]
    expect((cand[:, :, 1:][inner] > cand[:, :, :-1][inner]).all(), "I1 ascending")
    key = rows.astype(np.int64) * N + ids
    expect(len(np.unique(key)) == len(key), "I1 duplicate")
    # I2 (error bound) for every candidate
    err = np.abs(vals.astype(np.float64) - P.exact[rows, ids].astype(np.float64))
    bad = err > 0.5 * margin[rows].astype(np.float64)
    expect(not bad.any(), "I2 error bound", int(bad.sum()), float(err[bad].max()) if bad.any() else 0.0)
    # I3 / I4 on the users whose lists all fit
    over = (cnt > cap).any(1)
    member = np.zeros((n, N), bool)
    member[rows, ids] = True
    if pass_ == 0:
        kth = -np.partition(-P.exm, K, axis=1)[:, K]                # exact (K+1)-th best, -inf if fewer unmasked
        for r in np.nonzero(~over)[0]:
            e = P.exm[r]
            must = np.isfinite(e) & (e >= kth[r])
            if margin[r] > 0:
                missing = np.nonzero(must & ~member[r])[0]
                expect(len(missing) == 0, "I3 top K+1", int(r), missing[:8].tolist())
            else:
                # zero user row: every score is 0, the kernel keeps the first K+1 unmasked items of each
                # list (the strict > of the filter); the top K+1 VALUES must still be among the candidates
                top = np.sort(np.where(member[r], e, -np.inf))[::-1][:K + 1]
                expect(np.array_equal(top, np.sort(e)[::-1][:K + 1]), "I3 zero row", int(r))
    else:
        for r in np.nonzero(~over)[0]:
            entering = reference_heap_entries(P.exm[r].astype(np.float64), L)
            missing = [i for i in entering if not member[r, i]]
            expect(not missing, "I4 heap entries", int(r), missing[:8])
    assert not failed, (ctx, sorted({f[0] for f in failed}), failed[:4])
    return int(over.sum())


SHAPES = [(dim, N) for dim in (64, 128, 192) for N in (45, 5000, 20049, 70001)]


@pytest.mark.parametrize("dim,N", SHAPES)
def test_candidate_lists_invariants_across_shapes_and_segments(dim, N):
    """Gaussian tables with all-zero user rows and identical item rows in different segments; forced
    segment counts 1, 2, 5 and one segment per tile, one and two filter threads per user, K = 1 .. 31
    (<= 16 at dim 192), both passes; user counts that are not multiples of 64."""
    n = 70 if N > 50_000 else 130
    P = Problem("gauss_dups", n, N, dim, seed=dim + N)
    ks = [k for k in KS if dim < 192 or k <= 16]
    i = 0
    for G in (1, 2, 5, 0):
        for CH in (1, 2):
            for pass_ in (0, 1):
                K = ks[i % len(ks)]
                i += 1
                over = check_pass(P, pass_, K, G, CH)
                assert over <= n // 10, (dim, N, G, CH, pass_, K, over)


@pytest.mark.parametrize("dim", [64, 192])
@pytest.mark.parametrize("kind", sorted(CASES) + ["integers", "subnormal"])
def test_candidate_lists_invariants_on_adversarial_tables(kind, dim):
    """Every adversarial table of the algorithm model (cancelling sums, worst-case bf16 rounding, heavy-tailed
    norms, tiny times huge), integer tables (mass ties) and products in the fp32 subnormal range."""
    N, n = 20049, 70
    P = Problem(kind, n, N, dim, seed=len(kind) * 7 + dim)
    ks = [k for k in KS if dim < 192 or k <= 16]
    i = 0
    for G in (1, 5, 0):
        for CH in (1, 2):
            for pass_ in (0, 1):
                K = ks[i % len(ks)]
                i += 1
                over = check_pass(P, pass_, K, G, CH)
                if kind not in OVERFLOWING:
                    assert over <= n // 10, (kind, dim, G, CH, pass_, K, over)
                elif G == 0:
                    assert over == 0                                  # one tile per segment: lists cannot overflow


@pytest.mark.parametrize("dim", [128, 192])
def test_candidate_lists_keep_the_exact_top1_behind_bf16_decoys(dim):
    """The algorithm model's counter-example to the round-1 margin (tests/test_tc_algorithm_model.py::
    adversarial_top1_tables): two decoys whose bf16 scores round up come first, the exact top-1 rounds down.
    The main pass must keep it (I3), with one and with two filter threads per user."""
    N, n = 20049, 70
    P = Problem("top1_decoys", n, N, dim, seed=dim)
    for G in (1, 0):
        for CH in (1, 2):
            for K in (1, 5):
                over = check_pass(P, 0, K, G, CH)
                if K == 1:   # at K = 5 the fillers' scores crowd the cut: long segments overflow, by design
                    assert over <= n // 10
