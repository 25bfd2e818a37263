"""GPU parity tests of the tensor-core (wgmma) evaluator path: bit-identical ranks and
metric rows to the oracle (and therefore to nrc_eval_mf), including masks, ties and candidate
overflow (which must fall back to the exact heap replay)."""
import ctypes

import numpy as np
import pytest
import torch

import oracle
from conftest import random_csr

pytestmark = pytest.mark.gpu
ALL = [1, 2, 3, 4, 5]


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


@pytest.mark.parametrize("K,sw", [(64, 0), (128, 0), (64, 1), (128, 1), (256, 1)])
def test_tcgen05_gemm_building_block(K, sw):
    """nrc_tc_gemm_debug: the wgmma building block of the candidate kernel (name kept from the first MMA path)."""
    from neurec_b200 import _lib
    lib = _lib.load()
    g = torch.Generator(device="cuda").manual_seed(K + sw)
    A = torch.randn(128, K, device="cuda", generator=g).bfloat16()
    B = torch.randn(256, K, device="cuda", generator=g).bfloat16()
    out = torch.zeros(128, 256, device="cuda")
    _lib.check(lib.nrc_tc_gemm_debug(ctypes.c_void_p(A.data_ptr()), ctypes.c_void_p(B.data_ptr()), K, sw,
                                     ctypes.c_void_p(out.data_ptr()), None))
    torch.cuda.synchronize()
    ref = A.double() @ B.double().T          # bf16 products are exact; only the fp32 accumulation differs
    assert (out.double() - ref).abs().max().item() < 2e-4


@pytest.mark.parametrize("n_tile", [128, 64])
@pytest.mark.parametrize("K,sw", [(64, 0), (128, 0), (64, 1), (128, 1), (256, 1)])
def test_wgmma_gemm_building_block_both_n_tiles(K, sw, n_tile):
    """nrc_tc_gemm_debug_ntile: the wgmma building block with either instruction the candidate kernel issues,
    m64n128k16 (dim <= 128) and m64n64k16 (dim 192), both operand layouts."""
    from neurec_b200 import ops
    g = torch.Generator(device="cuda").manual_seed(K + sw)
    A = torch.randn(128, K, device="cuda", generator=g).bfloat16()
    B = torch.randn(256, K, device="cuda", generator=g).bfloat16()
    out = ops.tc_gemm_debug(A, B, swizzle=sw, n_tile=n_tile)
    torch.cuda.synchronize()
    ref = A.double() @ B.double().T          # bf16 products are exact; only the fp32 accumulation differs
    assert (out.double() - ref).abs().max().item() < 2e-4


def _accumulation_operands(pattern, k, rs):
    """bf16-exact operands A [128, k], B [256, k] whose fp32 accumulation is hard to get right."""
    if pattern == "unit_plus_tiny":
        # per k16 block: one product of size ~1 and fifteen just under 2^-24 of it, all of one sign per
        # dot product; the unit product sits at a row- / column-dependent position of the block
        A = np.full((128, k), 2.0 ** -12 * (1 - 2.0 ** -8))
        B = np.full((256, k), 2.0 ** -12)
        pa, pb = rs.randint(0, 16, 128), rs.randint(0, 16, 256)
        pb[:128] = pa                                          # half of the pairs: the designed pattern exactly
        for b in range(k // 16):
            A[np.arange(128), 16 * b + pa] = 1.0
            B[np.arange(256), 16 * b + pb] = 1.0
        A *= rs.choice([-1.0, 1.0], (128, 1)) * 2.0 ** rs.randint(-20, 20, (128, 1))
        B *= 2.0 ** rs.randint(-20, 20, (256, 1))
    elif pattern == "cancelling":
        # +-x pairs: the products cancel up to small residues
        x = 2.0 ** rs.randint(-6, 6, (128, k // 2)) * (1 + rs.randint(0, 128, (128, k // 2)) / 128.0)
        A = np.repeat(x, 2, axis=1)
        y = 2.0 ** rs.randint(-6, 6, (256, k // 2)) * (1 + rs.randint(0, 128, (256, k // 2)) / 128.0)
        B = np.repeat(y, 2, axis=1)
        B[:, 1::2] *= -(1 - rs.randint(0, 3, (256, k // 2)) * 2.0 ** -7)
    else:
        A, B = rs.randn(128, k), rs.randn(256, k)
    return torch.tensor(A, dtype=torch.float32).bfloat16(), torch.tensor(B, dtype=torch.float32).bfloat16()


@pytest.mark.parametrize("sw", [0, 1])
@pytest.mark.parametrize("n_tile", [128, 64])
def test_wgmma_accumulation_error_within_half_the_margin_budget(n_tile, sw):
    """The margin (tc_prepare_users_kernel) leaves 2^-11 |u||v| for the tensor core's fp32 accumulation and
    the exact FMA chain together.  Measured on adversarial operands at k = 256: |out - sum bf16(a) bf16(b)
    (fp64)| must stay below 2^-12 sum |a_k b_k|, half of that budget."""
    from neurec_b200 import ops
    rs = np.random.RandomState(n_tile + sw)
    worst = 0.0
    for pattern in ("unit_plus_tiny", "cancelling", "gauss"):
        A, B = _accumulation_operands(pattern, 256, rs)
        out = ops.tc_gemm_debug(A.cuda(), B.cuda(), swizzle=sw, n_tile=n_tile).cpu().double()
        a, b = A.double(), B.double()
        ref, mag = a @ b.T, a.abs() @ b.abs().T
        err = (out - ref).abs()
        assert (err <= 2.0 ** -12 * mag).all(), (pattern, float((err / mag.clamp_min(1e-300)).max()))
        worst = max(worst, float((err / mag.clamp_min(1e-300)).max()) / 2.0 ** -12)
    print("n_tile %d swizzle %d: largest |error| / (2^-12 sum|ab|) = %.3g" % (n_tile, sw, worst))


def _problem(nu, ni, dim, seed, scale=0.1, int_tables=False):
    rs = np.random.RandomState(seed)
    if int_tables:
        U = rs.randint(-2, 3, size=(nu, dim)).astype(np.float32)
        V = rs.randint(-2, 3, size=(ni, dim)).astype(np.float32)
    else:
        U = (rs.randn(nu, dim) * scale).astype(np.float32)
        V = (rs.randn(ni, dim) * scale).astype(np.float32)
    tp, ti = random_csr(rs, nu, ni, rs.randint(1, 80, nu))
    sp, si = random_csr(rs, nu, ni, rs.randint(1, 12, nu))
    return U, V, tp, ti, sp, si


@pytest.mark.parametrize("nu,ni,dim,K", [(300, 5000, 64, 20), (129, 2049, 128, 10), (500, 12345, 128, 31),
                                         (77, 300, 64, 5), (260, 7001, 192, 16)])
def test_tc_eval_bit_exact_vs_oracle(nu, ni, dim, K):
    from neurec_b200 import ops
    U, V, tp, ti, sp, si = _problem(nu, ni, dim, nu + ni)
    users = np.random.RandomState(1).permutation(nu).astype(np.int32)
    tip = np.zeros(nu + 1, np.int64); tip[1:] = np.cumsum(sp[users + 1] - sp[users])
    tix = np.concatenate([si[sp[u]:sp[u + 1]] for u in users])
    want, wranks = oracle.eval_mf(U, V, users, tp, ti, tip, tix, ALL, K, thread_num=4, return_ranks=True)
    args = (dev(U), dev(V), dev(users), dev(tp), dev(ti), dev(sp), dev(si), ALL, K)
    got, ranks = ops.eval_mf_tc(*args, return_ranks=True)
    assert np.array_equal(ranks.cpu().numpy(), wranks)
    assert np.array_equal(got.cpu().numpy(), want)
    got2, ranks2 = ops.eval_mf(*args, return_ranks=True)               # and identical to the SIMT path
    assert torch.equal(ranks, ranks2) and torch.equal(got, got2)


def test_tc_eval_ties_and_overflow_fall_back_to_heap_replay():
    from neurec_b200 import ops
    # integer tables: massive exact ties -> undecidable users -> heap replay must reproduce libstdc++ order
    U, V, tp, ti, sp, si = _problem(140, 900, 64, 5, int_tables=True)
    users = np.arange(140, dtype=np.int32)
    want, wranks = oracle.eval_mf(U, V, users, tp, ti, sp, si, ALL, 20, return_ranks=True)
    args = (dev(U), dev(V), dev(users), dev(tp), dev(ti), dev(sp), dev(si), ALL, 20)
    got, ranks = ops.eval_mf_tc(*args, return_ranks=True)
    assert np.array_equal(ranks.cpu().numpy(), wranks) and np.array_equal(got.cpu().numpy(), want)
    # tiny candidate buffer: (almost) every user overflows and is re-done exactly
    U, V, tp, ti, sp, si = _problem(150, 4000, 128, 6)
    users = np.arange(150, dtype=np.int32)
    want, wranks = oracle.eval_mf(U, V, users, tp, ti, sp, si, ALL, 20, return_ranks=True)
    got, ranks = ops.eval_mf_tc(dev(U), dev(V), dev(users), dev(tp), dev(ti), dev(sp), dev(si), ALL, 20,
                                return_ranks=True, cand_cap=24)
    assert np.array_equal(ranks.cpu().numpy(), wranks) and np.array_equal(got.cpu().numpy(), want)


def test_tc_eval_candidate_list_heap_replay_matches_reference_heap():
    """Force every user through the candidate-list heap replay (the tie path): the first 2K items seed
    the heap, the candidates are a superset of everything that later enters it, so ranks and metrics
    must still be bit-identical -- also with integer tables where most of the catalogue ties."""
    from neurec_b200 import ops, _lib
    lib = _lib.load()
    try:
        lib.nrc_eval_force_exact(1)
        for (nu, ni, dim, K, ints) in ((200, 6000, 64, 20, False), (130, 3000, 128, 7, False),
                                       (140, 5000, 64, 20, True), (64, 45, 64, 31, False), (150, 4001, 192, 16, False),
                                       (140, 3000, 192, 12, True)):
            U, V, tp, ti, sp, si = _problem(nu, ni, dim, 17 + ni, int_tables=ints)
            if ni < 100:
                rs = np.random.RandomState(4)
                tp, ti = random_csr(rs, nu, ni, rs.randint(0, 20, nu))
                sp, si = random_csr(rs, nu, ni, rs.randint(1, 6, nu))
            users = np.arange(nu, dtype=np.int32)
            want, wranks = oracle.eval_mf(U, V, users, tp, ti, sp, si, ALL, K, return_ranks=True)
            got, ranks = ops.eval_mf_tc(dev(U), dev(V), dev(users), dev(tp), dev(ti), dev(sp), dev(si), ALL, K,
                                        return_ranks=True)
            assert np.array_equal(ranks.cpu().numpy(), wranks), (nu, ni, dim, K, ints)
            assert np.array_equal(got.cpu().numpy(), want)
            n = ctypes.c_int32(0)
            lib.nrc_eval_last_undecided(ctypes.byref(n))
            assert n.value == nu          # every user went through a heap replay
    finally:
        lib.nrc_eval_force_exact(0)


def test_tc_eval_large_scale_matches_simt_path():
    """200 k items x 2 000 users, d=128: the tensor-core path must agree bit for bit with the SIMT
    fused evaluator (itself pinned on the oracle) -- checks the error-margin argument at scale,
    with score magnitudes that make bf16 rounding errors comparable to the top-K gaps."""
    from neurec_b200 import ops
    g = torch.Generator(device="cuda").manual_seed(11)
    nu, ni, dim, K = 2000, 200_000, 128, 20
    U = torch.randn(nu, dim, device="cuda", generator=g) * 0.1
    V = torch.randn(ni, dim, device="cuda", generator=g) * 0.1
    rs = np.random.RandomState(3)
    tp, ti = random_csr(rs, nu, ni, np.full(nu, 50))
    sp, si = random_csr(rs, nu, ni, np.full(nu, 10))
    users = torch.arange(nu, dtype=torch.int32, device="cuda")
    a = ops.eval_mf_tc(U, V, users, dev(tp), dev(ti), dev(sp), dev(si), ALL, K, return_ranks=True)
    b = ops.eval_mf(U, V, users, dev(tp), dev(ti), dev(sp), dev(si), ALL, K, return_ranks=True)
    assert torch.equal(a[1], b[1]) and torch.equal(a[0], b[0])


def test_uni_evaluator_routes_large_catalogues_to_the_tensor_core_path(monkeypatch):
    """UniEvaluator picks nrc_eval_mf_tc above TC_MIN_ITEMS; the printed metric string (the thing
    main.py logs, uni_evaluator.py:150-156) must not change by a character."""
    from neurec_b200.evaluator.uni_evaluator import UniEvaluator
    from neurec_b200 import ops
    nu, ni, dim = 1100, 3000, 64
    U, V, tp, ti, sp, si = _problem(nu, ni, dim, 77)
    train = {u: ti[tp[u]:tp[u + 1]].tolist() for u in range(nu)}
    test = {u: si[sp[u]:sp[u + 1]].tolist() for u in range(nu)}

    class Model:
        def get_eval_tables(self):
            return dev(U), dev(V)
    ev = UniEvaluator(train, test, metric=["Precision", "Recall", "MAP", "NDCG", "MRR"], top_k=[5, 10, 20])
    plain = ev.evaluate(Model())
    calls = []
    real = ops.eval_mf_tc
    monkeypatch.setattr(ops, "eval_mf_tc", lambda *a, **k: (calls.append(1), real(*a, **k))[1])
    monkeypatch.setattr(ops, "TC_MIN_ITEMS", 1000)
    assert ev.evaluate(Model()) == plain
    assert calls == [1]


@pytest.mark.parametrize("K", [1, 5])
def test_tc_eval_adversarial_bf16_rounding_keeps_the_exact_top1(K):
    """Round-1 verdict's counter-example (tests/test_tc_algorithm_model.py::adversarial_top1_tables):
    bf16 rounding pushes two decoys UP and the exact top-1 DOWN by almost 2^-7 relative each.  With the
    round-1 margin (2^-8) the true top-1 was never a candidate; with eps = 2^-7 + 2^-11 it must be.
    Padded past TC_MIN_ITEMS (16 384) so this is the shape UniEvaluator routes to the tensor cores."""
    from neurec_b200 import ops
    from test_tc_algorithm_model import adversarial_top1_tables
    ni, dim = 16_500, 128
    u, V = adversarial_top1_tables(n_items=ni, d=dim)
    rs = np.random.RandomState(5)
    V[3:] *= rs.uniform(0.2, 1.0, size=(ni - 3, 1)).astype(np.float32)      # distinct fillers, all far below
    place = rs.permutation(ni)                                               # decoys / target anywhere in the stream
    V = np.ascontiguousarray(V[np.argsort(place)])
    target = int(place[2])
    nu = 140
    U = np.stack([u * np.float32(2.0 ** (j % 7 - 3)) for j in range(nu)])   # power-of-two scales keep the roundings
    users = np.arange(nu, dtype=np.int32)
    tp, ti = random_csr(rs, nu, ni, np.full(nu, 3))
    for r in range(nu):                                                      # never mask the three special items
        row = ti[tp[r]:tp[r + 1]]
        assert not (set(row.tolist()) & {int(place[0]), int(place[1]), target})
    sp, si = random_csr(rs, nu, ni, np.full(nu, 4))
    want, wranks = oracle.eval_mf(U, V, users, tp, ti, sp, si, ALL, K, return_ranks=True)
    assert (wranks[:, 0] == target).all()
    got, ranks = ops.eval_mf_tc(dev(U), dev(V), dev(users), dev(tp), dev(ti), dev(sp), dev(si), ALL, K,
                                return_ranks=True)
    assert np.array_equal(ranks.cpu().numpy(), wranks)
    assert np.array_equal(got.cpu().numpy(), want)


def test_tc_eval_sixteen_epilogue_warps_give_the_same_bits():
    """The 16-warp epilogue (two threads per user, one per half item tile, own threshold + candidate list
    each) must select exactly what the 8-warp layout selects: ranks and metric rows bit-identical to the
    oracle, also with masks, ties (integer tables) and a catalogue that is not a multiple of the tile."""
    from neurec_b200 import ops
    try:
        ops.eval_tc_epilogue_warps(16)
        for (nu, ni, dim, K, ints) in ((300, 5000, 64, 20, False), (129, 20049, 128, 10, False), (140, 900, 64, 20, True),
                                       (500, 12345, 128, 31, False)):
            U, V, tp, ti, sp, si = _problem(nu, ni, dim, nu + ni + 1, int_tables=ints)
            users = np.arange(nu, dtype=np.int32)
            want, wranks = oracle.eval_mf(U, V, users, tp, ti, sp, si, ALL, K, thread_num=4, return_ranks=True)
            got, ranks = ops.eval_mf_tc(dev(U), dev(V), dev(users), dev(tp), dev(ti), dev(sp), dev(si), ALL, K,
                                        return_ranks=True)
            assert np.array_equal(ranks.cpu().numpy(), wranks), (nu, ni, dim, K)
            assert np.array_equal(got.cpu().numpy(), want)
    finally:
        ops.eval_tc_epilogue_warps(8)


def _force_exact(on):
    from neurec_b200 import _lib
    _lib.check(_lib.load().nrc_eval_force_exact(int(on)))


@pytest.mark.parametrize("dim,ni,K", [(64, 20049, 20), (192, 20001, 12)])
def test_tc_eval_forced_segments_bit_exact(dim, ni, K):
    """The replay pass over G > 1 item segments (lists replayed in slot order) on integer tables (mass ties),
    with and without the tie-free main pass: ranks and metric rows equal the oracle's for every G and both
    epilogue layouts."""
    from neurec_b200 import ops
    nu = 130
    U, V, tp, ti, sp, si = _problem(nu, ni, dim, 41 + dim, int_tables=True)
    users = np.arange(nu, dtype=np.int32)
    want, wranks = oracle.eval_mf(U, V, users, tp, ti, sp, si, ALL, K, thread_num=8, return_ranks=True)
    d = (dev(U), dev(V), dev(users), dev(tp), dev(ti), dev(sp), dev(si))
    try:
        for G in (1, 2, 3, 7, 16):
            ops.eval_tc_force_segments(G)
            # the route: the replay pass really runs over G lists per user
            lists = ops.eval_tc_debug_candidates(1, d[0], d[1], d[2][:3], d[3], d[4], min(2 * K, ni), 2048, 64)
            assert lists[2].shape[1] == G
            for CH in (1, 2):
                ops.eval_tc_epilogue_warps(8 * CH)
                for exact in (1, 0):
                    _force_exact(exact)
                    got, ranks = ops.eval_mf_tc(*d, ALL, K, return_ranks=True)
                    replayed, full = ops.eval_tc_last_fallbacks()
                    assert np.array_equal(ranks.cpu().numpy(), wranks), (G, CH, exact)
                    assert np.array_equal(got.cpu().numpy(), want), (G, CH, exact)
                    assert replayed > 0, (G, CH, exact, replayed, full)
                    if exact:
                        assert replayed + full == nu
    finally:
        _force_exact(0)
        ops.eval_tc_force_segments(0)
        ops.eval_tc_epilogue_warps(8)


@pytest.mark.parametrize("G", [2, 3, 7])
def test_tc_eval_ties_straddling_segment_boundaries(G):
    """Identical item rows on both sides of every segment boundary: their scores tie at the top, so which of
    them the reference's heap keeps, and in which order, depends on the order the replay visits its lists."""
    from neurec_b200 import ops
    nu, ni, dim, K = 130, 24000, 64, 10
    rs = np.random.RandomState(G)
    V = (rs.randn(ni, dim) * 0.1).astype(np.float32)
    hubs = (rs.randn(3, dim) * 0.4).astype(np.float32)
    T = -(-ni // 128)
    seg_items = -(-T // G) * 128
    for b in range(seg_items, ni, seg_items):
        for off in (-3, -2, -1, 0, 1, 2):                                  # every hub on both sides
            V[b + off] = hubs[off % 3]
    U = (hubs[rs.randint(0, 3, nu)] + rs.randn(nu, dim).astype(np.float32) * 0.02).astype(np.float32)
    U[::5] = (rs.randn(nu // 5, dim) * 0.1).astype(np.float32)            # and some users without a hub
    users = np.arange(nu, dtype=np.int32)
    tp, ti = random_csr(rs, nu, ni, rs.randint(0, 30, nu))
    sp, si = random_csr(rs, nu, ni, rs.randint(1, 12, nu))
    want, wranks = oracle.eval_mf(U, V, users, tp, ti, sp, si, ALL, K, thread_num=8, return_ranks=True)
    d = (dev(U), dev(V), dev(users), dev(tp), dev(ti), dev(sp), dev(si))
    try:
        ops.eval_tc_force_segments(G)
        assert ops.eval_tc_debug_candidates(1, d[0], d[1], d[2], d[3], d[4], 2 * K, 2048, G)[4] == seg_items
        for exact in (0, 1):
            _force_exact(exact)
            got, ranks = ops.eval_mf_tc(*d, ALL, K, return_ranks=True)
            replayed, full = ops.eval_tc_last_fallbacks()
            assert replayed > nu // 2 and full == 0, (exact, replayed, full)
            assert np.array_equal(ranks.cpu().numpy(), wranks), exact
            assert np.array_equal(got.cpu().numpy(), want), exact
    finally:
        _force_exact(0)
        ops.eval_tc_force_segments(0)


def test_tc_eval_replay_pass_overflow_falls_back_to_full_replay():
    """{0, 1} tables, dim 64, ~50 k items: for half of the users 40 items tie at the top (the main pass keeps
    few candidates, but the top K+1 tie) and 3 000 more tie just below, so that the replay pass's threshold
    (the 2K-th best) lets more than 2 048 of them through -- the list overflows and the user is re-ranked
    by the full-catalogue heap replay (eval_mf_kernel)."""
    from neurec_b200 import ops
    nu, ni, dim, K = 70, 50_000, 64, 31
    rs = np.random.RandomState(9)
    V = (rs.rand(ni, dim) < 0.5).astype(np.float32)
    V[:, :3] = 0.0
    V[:40, :3] = 1.0                                                   # score 3 for the special users
    two = 40 + rs.permutation(ni - 40)[:3000]
    for j, i in enumerate(two):                                        # score 2
        V[i, [c for c in range(3) if c != j % 3]] = 1.0
    one = np.setdiff1d(np.arange(40, ni), two)
    V[one, rs.randint(0, 3, len(one))] = 1.0                           # score 1
    U = (rs.rand(nu, dim) < 0.3).astype(np.float32)
    special = np.arange(0, nu, 2)
    U[special] = 0.0
    U[special, :3] = 1.0
    users = np.arange(nu, dtype=np.int32)
    tp, ti = random_csr(rs, nu, ni, rs.randint(0, 6, nu))
    sp, si = random_csr(rs, nu, ni, rs.randint(1, 12, nu))
    want, wranks = oracle.eval_mf(U, V, users, tp, ti, sp, si, ALL, K, thread_num=8, return_ranks=True)
    d = (dev(U), dev(V), dev(users), dev(tp), dev(ti), dev(sp), dev(si))
    try:
        ops.eval_tc_force_segments(1)
        sp_users = dev(special.astype(np.int32))
        c0 = ops.eval_tc_debug_candidates(0, d[0], d[1], sp_users, d[3], d[4], K + 1, 1024, 1)[2].cpu().numpy()
        c1 = ops.eval_tc_debug_candidates(1, d[0], d[1], sp_users, d[3], d[4], 2 * K, 2048, 1)[2].cpu().numpy()
        assert (c0 <= 1024).all() and (c1 > 2048).all(), (c0.max(), c1.min())
        got, ranks = ops.eval_mf_tc(*d, ALL, K, return_ranks=True)
        replayed, full = ops.eval_tc_last_fallbacks()
        assert replayed >= len(special) and full >= len(special), (replayed, full)
        assert np.array_equal(ranks.cpu().numpy(), wranks)
        assert np.array_equal(got.cpu().numpy(), want)
    finally:
        ops.eval_tc_force_segments(0)


def test_tc_eval_bf16_item_cache_versions():
    """nrc_eval_tc_items_version: user batches of one table version equal one call; an in-place change of the
    table under a new version, and a different table of the same shape under the same version, are
    converted again."""
    from neurec_b200 import ops
    nu, ni, dim, K = 300, 17_000, 64, 10
    U, V, tp, ti, sp, si = _problem(nu, ni, dim, 23)
    users = np.arange(nu, dtype=np.int32)
    d = [dev(U), dev(V), dev(users), dev(tp), dev(ti), dev(sp), dev(si)]

    def oracle_on(Vh):
        return oracle.eval_mf(U, Vh, users, tp, ti, sp, si, ALL, K, thread_num=8, return_ranks=True)

    def run(Vd, rows=None):
        u = d[2] if rows is None else d[2][rows]
        got, ranks = ops.eval_mf_tc(d[0], Vd, u, d[3], d[4], d[5], d[6], ALL, K, return_ranks=True)
        return got.cpu().numpy(), ranks.cpu().numpy()

    try:
        ops.eval_tc_items_version(1)
        want, wranks = oracle_on(V)
        got, ranks = run(d[1])
        assert np.array_equal(ranks, wranks) and np.array_equal(got, want)
        a, b = run(d[1], slice(0, 150)), run(d[1], slice(150, nu))
        assert np.array_equal(np.concatenate([a[1], b[1]]), ranks)
        assert np.array_equal(np.concatenate([a[0], b[0]]), got)
        # in place, new version: must be converted again
        V2 = (V[::-1] * np.float32(1.5)).copy()
        d[1].copy_(dev(V2))
        ops.eval_tc_items_version(2)
        want2, wranks2 = oracle_on(V2)
        got, ranks = run(d[1])
        assert np.array_equal(ranks, wranks2) and np.array_equal(got, want2)
        # another table of the same shape under the same version
        V3 = (np.random.RandomState(5).randn(ni, dim) * 0.1).astype(np.float32)
        d3 = dev(V3)
        want3, wranks3 = oracle_on(V3)
        got, ranks = run(d3)
        assert np.array_equal(ranks, wranks3) and np.array_equal(got, want3)
        got, ranks = run(d[1])                                         # and back
        assert np.array_equal(ranks, wranks2) and np.array_equal(got, want2)
    finally:
        ops.eval_tc_items_version(0)


@pytest.mark.parametrize("dim", [64, 128, 192])
def test_tc_eval_adversarial_tables_at_routing_shape(dim):
    """Every adversarial table of the algorithm model, and products in the fp32 subnormal range, at the shape
    eval_mf_auto routes to the tensor cores (16 500 items)."""
    from neurec_b200 import ops
    from test_tc_algorithm_model import CASES
    from test_gpu_tc_candidates import make_tables
    nu, ni, K = 130, 16_500, 10
    for case in sorted(CASES) + ["subnormal"]:
        U, V = make_tables(case, nu, ni, dim, seed=dim + len(case))
        rs = np.random.RandomState(dim)
        tp, ti = random_csr(rs, nu, ni, rs.randint(0, 40, nu))
        sp, si = random_csr(rs, nu, ni, rs.randint(1, 12, nu))
        users = np.arange(nu, dtype=np.int32)
        want, wranks = oracle.eval_mf(U, V, users, tp, ti, sp, si, ALL, K, thread_num=8, return_ranks=True)
        got, ranks = ops.eval_mf_tc(dev(U), dev(V), dev(users), dev(tp), dev(ti), dev(sp), dev(si), ALL, K,
                                    return_ranks=True)
        assert np.array_equal(ranks.cpu().numpy(), wranks), case
        assert np.array_equal(got.cpu().numpy(), want), case
