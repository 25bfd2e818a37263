"""CPU tests: the oracle against the golden vectors captured from the REAL reference
(tests/golden/make_golden.py), among them the outputs of the reference's own compiled headers.
No GPU needed."""
import os
import subprocess
import sys

import numpy as np
import pytest

import oracle
from oracle import tf_math
from conftest import ROOT, parse_result_string

ALL = [1, 2, 3, 4, 5]


def test_kat2_evaluator_golden(golden_eval):
    g = golden_eval
    out, ranks = oracle.evaluate_matrix(g["kat2_scores"], g["kat2_truth_indptr"],
                                        g["kat2_truth_indices"], ALL, 5, return_ranks=True)
    assert np.array_equal(out, g["kat2_out"])
    assert np.array_equal(ranks, g["kat2_top5"])
    out2 = oracle.evaluate_matrix(g["kat2_scores"], g["kat2_truth_indptr"],
                                  g["kat2_truth_indices"], [4, 1, 3, 2, 5], 5, thread_num=2)
    assert np.array_equal(out2, g["kat2_out_41325"])


def test_kat3_tie_order_golden(golden_eval):
    g = golden_eval
    assert np.array_equal(oracle.arg_topk(np.zeros((1, 40), np.float32), 5), g["tie_zeros_top5"])
    assert g["tie_zeros_top5"].tolist() == [[3, 4, 1, 0, 2]]  # SURVEY.md KAT-3
    m3 = np.zeros((1, 40), np.float32); m3[0, ::3] = 1
    assert np.array_equal(oracle.arg_topk(m3, 8), g["tie_mult3_top8"])
    inf = np.full((1, 40), -np.inf, np.float32); inf[0, 7] = 1; inf[0, 3] = 2
    assert np.array_equal(oracle.arg_topk(inf, 5), g["tie_inf_top5"])
    assert np.array_equal(oracle.arg_topk(g["tie_scores"], 20), g["tie_top20"])
    assert np.array_equal(oracle.arg_topk(g["tie_scores"], 40, thread_num=3), g["tie_top40"])
    out = oracle.evaluate_matrix(g["tie_scores"], g["tie_truth_indptr"], g["tie_truth_indices"],
                                 ALL, 20)
    assert np.array_equal(out, g["tie_out_k20"])


def test_restatement_vs_reference_headers_golden():
    """The C restatement against what the reference's compiled arg_topk.h / evaluate.h returned on the same
    seeded matrices (tests/golden/make_golden.py headers): random and integer-tied scores, -inf masks."""
    sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))
    from make_golden import header_trials
    g = np.load(os.path.join(ROOT, "tests", "golden", "kat_headers.npz"))
    pt = pm = 0
    for S, k, ip, ix in header_trials():
        top = oracle.arg_topk(S, k).ravel()
        assert np.array_equal(top, g["topk"][pt:pt + top.size])
        met = oracle.evaluate_matrix(S, ip, ix, ALL, k).ravel()
        assert np.array_equal(met, g["metrics"][pm:pm + met.size], equal_nan=True)
        pt += top.size; pm += met.size
    assert pt == g["topk"].size and pm == g["metrics"].size


def _fresh(code):
    r = subprocess.run([sys.executable, "-c", "import sys; sys.path.insert(0, %r)\n" % ROOT + code],
                       capture_output=True, text=True, check=True)
    return r.stdout.strip().splitlines()[-1]


def test_kat1_libc_sampler_golden(golden_sampler):
    """glibc rand() stream (seed 1) in a fresh process reproduces the reference's draws."""
    g = golden_sampler
    got = _fresh(
        "import oracle, json, numpy as np\n"
        "a = oracle.batch_randint_choice(100, [5], True, oracle.lists_to_csr([[1,2,3]]))\n"
        "b = oracle.batch_randint_choice(40981, [4], True, None)\n"
        "print(json.dumps({'a': a.tolist(), 'b': b.tolist()}))")
    import json
    got = json.loads(got)
    assert got["a"] == g["a"]["a"] == [93, 69, 35, 0, 34]
    assert got["b"] == g["a"]["b"]
    got = json.loads(_fresh(
        "import oracle, json, numpy as np\n"
        "a = oracle.batch_randint_choice(100, [5], True, oracle.lists_to_csr([[1,2,3]]))\n"
        "c = oracle.batch_randint_choice(1682, [3,2], True, oracle.lists_to_csr([[0,1],[5]]))\n"
        "d = oracle.batch_randint_choice(50, [1], True, oracle.lists_to_csr([list(range(40))]))\n"
        "e = oracle.batch_randint_choice(30, [10], False, oracle.lists_to_csr([[0,1,2]]))\n"
        "print(json.dumps({'c': c.tolist(), 'd': d.tolist(), 'e': e.tolist()}))"))
    assert got["c"] == g["b"]["c"][0] + g["b"]["c"][1]
    assert got["d"] == [g["b"]["d"]]
    assert got["e"] == g["b"]["e"]


def test_pairwise_sampler_epoch_golden(golden_sampler, ml100k):
    """First negatives of the reference's PairwiseSampler epoch on ml-100k == the C
    restatement fed the same (user, n_pos, exclusion) rows in a fresh process."""
    g = golden_sampler["pairwise"]
    import json
    got = json.loads(_fresh(
        "import oracle, json, numpy as np\n"
        "z = np.load(%r)\n"
        "ip = z['train_indptr'].astype(np.int64); ix = z['train_indices'].astype(np.int32)\n"
        "sizes = np.diff(ip)[:3].astype(np.int32)\n"
        "neg = oracle.batch_randint_choice(int(z['num_items']), sizes, True, (ip[:4], ix[:ip[3]]))\n"
        "print(json.dumps(neg[:64].tolist()))" % (ROOT + "/tests/golden/ml100k_split.npz")))
    assert got == g["neg"]
    # positives are flattened in ascending-user order (sampler.py:24-39)
    users = np.repeat(np.arange(ml100k["num_users"]), np.diff(ml100k["train_indptr"]))
    assert users[:64].tolist() == g["users"]
    assert ml100k["train_indices"][:64].tolist() == g["pos"]
    assert g["len"] == (len(ml100k["train_indices"]) + 511) // 512 == 157


def test_kat5_ml100k_full_evaluator(ml100k, golden_ml100k_eval):
    """Whole UniEvaluator pass on the ml-100k split: oracle (fp32 FMA-chain predict) vs the
    reference run (np.matmul predict).  Scores differ in the last ulp, so a near-tie may flip:
    the north-star tolerance is 1e-5 on the averaged metrics."""
    d = ml100k
    rng = np.random.RandomState(1)
    U = (rng.randn(d["num_users"], 64) * .01).astype(np.float32)
    V = (rng.randn(d["num_items"], 64) * .01).astype(np.float32)
    users = np.arange(d["num_users"], dtype=np.int32)
    res = oracle.eval_mf(U, V, users, d["train_indptr"], d["train_indices"], d["test_indptr"],
                         d["test_indices"], [1, 2, 4, 3, 5], 20, thread_num=4)
    mean = res.mean(axis=0).reshape(5, 20)[:, [9, 19]].reshape(-1)
    want = parse_result_string(golden_ml100k_eval["eval_topk_10_20"])
    assert np.abs(mean - want).max() < 1e-5
    # exact-predict variant: same scores as the reference (np.matmul) => identical string
    S = np.matmul(U, V.T)
    oracle.mask_train(S, users, d["train_indptr"], d["train_indices"])
    res2 = oracle.evaluate_matrix(S, d["test_indptr"], d["test_indices"], [1, 2, 4, 3, 5], 20)
    # the reference evaluates in batches of 128 and np.mean's the concatenation (fp32)
    final = np.mean(res2, axis=0).reshape(5, 20)[:, [9, 19]].reshape(-1)
    buf = '\t'.join([("%.8f" % x).ljust(12) for x in final])
    assert buf == golden_ml100k_eval["eval_topk_10_20"]


def test_mf_scores_are_fma_chain():
    rs = np.random.RandomState(3)
    U = rs.randn(5, 24).astype(np.float32); V = rs.randn(11, 24).astype(np.float32)
    S = oracle.mf_scores(U, V, np.arange(5, dtype=np.int32))
    import math
    for b in range(5):
        for i in range(11):
            acc = np.float32(0)
            for k in range(24):  # fma = exact product + add, one rounding
                acc = np.float32(math.fma(float(U[b, k]), float(V[i, k]), float(acc))) \
                    if hasattr(math, "fma") else acc
            if hasattr(math, "fma"):
                # double fma then a float rounding can double-round; allow 1 ulp
                assert abs(float(S[b, i]) - float(acc)) <= abs(float(acc)) * 2e-7 + 1e-12
    assert np.allclose(S, U @ V.T, rtol=1e-5, atol=1e-6)


# ------------------------------------------------------------------------- tf_math pins
def _num_grad(f, x, eps=1e-3):
    g = np.zeros_like(x, dtype=np.float64)
    it = np.nditer(x, flags=["multi_index"])
    for _ in it:
        i = it.multi_index
        old = x[i]
        x[i] = old + eps; fp = f()
        x[i] = old - eps; fm = f()
        x[i] = old
        g[i] = (fp - fm) / (2 * eps)
    return g


@pytest.mark.parametrize("loss", ["bpr", "hinge", "square"])
def test_pairwise_grad_matches_finite_differences(loss):
    rs = np.random.RandomState(0)
    U = rs.randn(6, 5); V = rs.randn(7, 5)
    users = np.array([0, 1, 1, 5, 0]); pos = np.array([2, 2, 3, 6, 2]); neg = np.array([4, 0, 2, 1, 5])
    _, gU, gV, _, _ = tf_math.mf_pairwise_grad(U, V, users, pos, neg, loss, reg=0.05)

    def f64loss(Ux, Vx):
        x = (Ux[users] * Vx[pos]).sum(1) - (Ux[users] * Vx[neg]).sum(1)
        l = {"bpr": np.log1p(np.exp(-x)), "hinge": np.maximum(x + 1, 0), "square": (1 - x) ** 2}[loss]
        return l.sum() + 0.05 * 0.5 * ((Ux[users] ** 2).sum() + (Vx[pos] ** 2).sum() + (Vx[neg] ** 2).sum())

    U64, V64 = U.copy(), V.copy()
    nU = _num_grad(lambda: f64loss(U64, V64), U64, 1e-5)
    nV = _num_grad(lambda: f64loss(U64, V64), V64, 1e-5)
    assert np.allclose(gU, nU, rtol=2e-3, atol=2e-4)
    assert np.allclose(gV, nV, rtol=2e-3, atol=2e-4)


@pytest.mark.parametrize("loss", ["cross_entropy", "square"])
def test_pointwise_grad_matches_finite_differences(loss):
    rs = np.random.RandomState(1)
    U = rs.randn(6, 4); V = rs.randn(7, 4)
    users = np.array([0, 1, 1, 5]); items = np.array([2, 2, 3, 6]); z = np.array([1., 0., 1., 0.])
    _, gU, gV, _, _ = tf_math.mf_pointwise_grad(U, V, users, items, z, loss, reg=0.1)

    def f64loss(Ux, Vx):
        x = (Ux[users] * Vx[items]).sum(1)
        if loss == "cross_entropy":
            l = (np.maximum(x, 0) - x * z + np.log1p(np.exp(-np.abs(x)))).mean()
        else:
            l = ((z - x) ** 2).sum()
        return l + 0.1 * 0.5 * ((Ux[users] ** 2).sum() + (Vx[items] ** 2).sum())

    U64, V64 = U.copy(), V.copy()
    assert np.allclose(gU, _num_grad(lambda: f64loss(U64, V64), U64, 1e-5), rtol=2e-3, atol=2e-4)
    assert np.allclose(gV, _num_grad(lambda: f64loss(U64, V64), V64, 1e-5), rtol=2e-3, atol=2e-4)


def test_adam_sparse_is_dense_over_whole_table():
    """TF-1.12 Adam on IndexedSlices moves rows whose gradient is zero (m, v decay)."""
    var = np.ones((4, 3), np.float32); m = np.full((4, 3), 0.5, np.float32); v = np.full((4, 3), 0.25, np.float32)
    g = np.zeros((4, 3), np.float32); g[1] = 1.0
    tf_math.opt_apply("adam", var, g, m, v, None, [0.1, 0.9, 0.999, 1e-8])
    assert np.all(var[0] < 1.0) and np.allclose(m[0], 0.45) and np.allclose(v[0], 0.25 * 0.999)
    lr_t = tf_math.adam_lr_t(1e-3, 3)
    assert np.allclose(lr_t, [1e-3 * np.sqrt(1 - .999 ** t) / (1 - .9 ** t) for t in (1, 2, 3)], rtol=1e-5)


def test_numpy_axis0_mean_is_sequential_fp32():
    """nrc_mean_rows restates np.mean(axis=0): sequential fp32 row adds, then / n."""
    rs = np.random.RandomState(0)
    a = rs.rand(5000, 7).astype(np.float32)
    acc = a[0].copy()
    for r in range(1, len(a)):
        acc = (acc + a[r]).astype(np.float32)
    assert np.array_equal(np.mean(a, axis=0), acc / np.float32(len(a)))


# ----------------------------------------------------------------------------- NGCF restatement
def _ngcf_problem(dtype, seed=3, nu=23, ni=31, d=8, layers=(6, 5)):
    from oracle import tf_math
    rs = np.random.RandomState(seed)
    rows = [np.unique(rs.randint(0, ni, rs.randint(1, 7))) for _ in range(nu)]
    indptr = np.zeros(nu + 1, np.int64); indptr[1:] = np.cumsum([len(r) for r in rows])
    A = tf_math.ngcf_adj(indptr, np.concatenate(rows).astype(np.int32), nu, ni, "norm").astype(dtype)
    e0 = (rs.randn(nu + ni, d) * 0.3).astype(dtype)
    W = [tuple(w.astype(dtype) for w in ws) for ws in tf_math.ngcf_init_weights(rs, d, list(layers))]
    masks = [(rs.rand(nu + ni, k) < 0.9).astype(dtype) for k in layers]
    users = rs.randint(0, nu, 40); pos = rs.randint(0, ni, 40); neg = rs.randint(0, ni, 40)
    return A, e0, W, masks, nu, users, pos, neg


def test_ngcf_adjacency_is_row_normalised_with_self_loops():
    """NGCF.py:308-310: 'norm' = D^-1 (A + I): every row sums to 1, the diagonal is 1/(deg+1)."""
    A, e0, *_ = _ngcf_problem(np.float64)
    assert np.allclose(np.asarray(A.sum(1)).ravel(), 1.0)
    deg = np.diff(A.indptr) - 1
    assert np.allclose(A.diagonal(), 1.0 / (deg + 1))


def test_ngcf_forward_shapes_and_normalisation():
    from oracle import tf_math
    A, e0, W, masks, nu, *_ = _ngcf_problem(np.float32)
    allE, cache = tf_math.ngcf_forward(A, e0, W, masks, keep=0.9)
    assert allE.dtype == np.float32 and allE.shape == (e0.shape[0], 8 + 6 + 5)
    assert np.array_equal(allE[:, :8], e0)                                   # layer 0 is the raw table
    n1 = np.linalg.norm(allE[:, 8:14], axis=1)
    assert np.allclose(n1[n1 > 0], 1.0, atol=1e-5)                           # l2_normalize(axis=1)
    # n_fold slabs are a no-op: concatenated slab products == one product
    fold = (A.shape[0]) // 7
    slabs = [A[i * fold:(A.shape[0] if i == 6 else (i + 1) * fold)] @ e0 for i in range(7)]
    assert np.array_equal(np.concatenate(slabs, 0), A @ e0)


def test_ngcf_gradients_match_finite_differences():
    """Manual backprop of NGCF.py:160-202 + 94-110 (normalise, always-on dropout, leaky-relu, W_gc /
    W_bi GEMMs, SpMM, concat) against central differences in fp64."""
    from oracle import tf_math
    A, e0, W, masks, nu, users, pos, neg = _ngcf_problem(np.float64)
    AT = A.T.tocsr()
    reg = 0.05

    def total(e0_, W_):
        mf, emb, *_ = tf_math.ngcf_loss_and_grad(A, AT, e0_, W_, nu, users, pos, neg, reg, masks, keep=0.9)
        return mf + emb
    mf, emb, dE0, grads, _ = tf_math.ngcf_loss_and_grad(A, AT, e0, W, nu, users, pos, neg, reg, masks, keep=0.9)
    rs = np.random.RandomState(0)
    h = 1e-6
    for _ in range(12):                                                       # embedding table entries
        r, c = rs.randint(e0.shape[0]), rs.randint(e0.shape[1])
        p, m = e0.copy(), e0.copy(); p[r, c] += h; m[r, c] -= h
        fd = (total(p, W) - total(m, W)) / (2 * h)
        assert abs(fd - dE0[r, c]) < 1e-5 * max(1.0, abs(fd)), (r, c, fd, dE0[r, c])
    for k in range(len(W)):                                                   # every weight tensor of every layer
        for t in range(4):
            r, c = rs.randint(W[k][t].shape[0]), rs.randint(W[k][t].shape[1])
            Wp = [list(w) for w in W]; Wm = [list(w) for w in W]
            Wp[k][t] = W[k][t].copy(); Wp[k][t][r, c] += h
            Wm[k][t] = W[k][t].copy(); Wm[k][t][r, c] -= h
            fd = (total(e0, [tuple(w) for w in Wp]) - total(e0, [tuple(w) for w in Wm])) / (2 * h)
            assert abs(fd - grads[k][t][r, c]) < 1e-5 * max(1.0, abs(fd)), (k, t, fd, grads[k][t][r, c])


def test_ngcf_trainer_learns_the_training_pairs():
    """NGCFTrainer (BPR softplus + TF Adam over E_0 and all layer weights, always-on dropout): the loss
    of a fixed batch goes down and positives end up ranked above negatives."""
    from oracle import tf_math
    A, e0, W, masks, nu, users, pos, neg = _ngcf_problem(np.float32, seed=9, nu=40, ni=60, d=8, layers=(8, 8))
    rs = np.random.RandomState(1)
    pos = np.array([A[u].indices[A[u].indices >= nu][0] - nu for u in users])   # a train item of each user
    neg = rs.randint(0, 60, len(users))
    tr = tf_math.NGCFTrainer(A, e0 * 0.1, W, nu, lr=0.01, reg=1e-4, keep=0.9, rs=np.random.RandomState(2))
    first = [float(tr.step(users, pos, neg)[0]) for _ in range(5)]
    for _ in range(150):
        tr.step(users, pos, neg)
    last = [float(tr.step(users, pos, neg)[0]) for _ in range(5)]
    assert np.mean(last) < 0.6 * np.mean(first)
    Ue, Ie = tr.embeddings(masks=None)
    assert Ue.shape == (nu, 8 + 8 + 8) and Ie.shape == (60, 24) and Ue.dtype == np.float32
    x = (Ue[users] * Ie[pos]).sum(1) - (Ue[users] * Ie[neg]).sum(1)
    assert (x > 0).mean() > 0.8


def test_torch_timing_port_follows_the_parity_oracle(ml100k):
    """oracle/torch_port.py (the multi-threaded CPU arm bench.py times) against oracle/tf_math.py (the
    parity oracle): same losses and tables after a few steps, for every step kind it times."""
    from oracle import torch_port
    d = ml100k
    nu, ni = d["num_users"], d["num_items"]
    rs = np.random.RandomState(0)
    U0 = (rs.randn(nu, 16) * 0.1).astype(np.float32); V0 = (rs.randn(ni, 16) * 0.1).astype(np.float32)
    for pairwise, loss, learner in ((True, "bpr", "adam"), (True, "bpr", "gd"), (False, "cross_entropy", "adam"),
                                    (False, "square", "gd")):
        a = tf_math.MFTrainer(U0, V0, learner, 1e-2, loss, 1e-3, pairwise)
        b = torch_port.MFStep(U0, V0, learner, 1e-2, loss, 1e-3, pairwise)
        for s in range(4):
            u = rs.randint(0, nu, 300).astype(np.int32); i = rs.randint(0, ni, 300).astype(np.int32)
            t = rs.randint(0, ni, 300).astype(np.int32) if pairwise else rs.randint(0, 2, 300).astype(np.float32)
            la, lb = a.step(u, i, t), b.step(u.tolist(), i.tolist(), t.tolist())
            assert abs(float(la) - lb) < 1e-3 * max(1.0, abs(lb))
        assert np.abs(a.U - b.U.numpy()).max() < 2e-5 and np.abs(a.V - b.V.numpy()).max() < 2e-5
    A = tf_math.lightgcn_adj(d["train_indptr"], d["train_indices"], nu, ni, "pre")
    e0 = (rs.randn(nu + ni, 16) * 0.1).astype(np.float32)
    a = tf_math.LightGCNTrainer(A, e0, nu, 2, 0.01, 1e-3)
    b = torch_port.LightGCNStep(A, e0, nu, 2, 0.01, 1e-3)
    for s in range(3):
        u = rs.randint(0, nu, 200).astype(np.int32); i = rs.randint(0, ni, 200).astype(np.int32); j = rs.randint(0, ni, 200).astype(np.int32)
        la = a.step(u, i, j)
        lb = b.step(u.tolist(), i.tolist(), j.tolist())
        assert abs(float(la[0]) - lb) < 1e-3 * max(1.0, abs(lb))
    assert np.abs(a.e0 - b.e0.numpy()).max() < 5e-5


def test_candidate_ranking_model_equals_the_reference(ml100k):
    """rec.evaluate.neg > 0 (evaluator/backend/cpp/uni_evaluator.py:123-131): the padded-matrix model of that branch the
    GPU test compares the product with (tests/test_surface.py::test_candidate_ranking_branch) reproduces the string the
    REAL reference's ProxyEvaluator printed for the same inputs (tests/golden/kat_neg_eval.json)."""
    import json
    import os
    d = ml100k
    with open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "kat_neg_eval.json")) as f:
        kat = json.load(f)
    nu, ni = d["num_users"], d["num_items"]
    rows_of = lambda p, i: {u: d[i][d[p][u]:d[p][u + 1]].astype(int).tolist() for u in range(nu) if d[p][u + 1] > d[p][u]}
    train_d, test_d = rows_of("train_indptr", "train_indices"), rows_of("test_indptr", "test_indices")
    rs = np.random.RandomState(2)
    neg_d = {}
    for u in test_d:
        seen = set(train_d[u]) | set(test_d[u])
        neg_d[u] = [int(i) for i in rs.choice(ni, 60) if i not in seen][:40]
    U = (rs.randn(nu, 16)).astype(np.float32); V = (rs.randn(ni, 16)).astype(np.float32)
    rows = []
    for u in test_d:
        c = list(test_d[u]) + neg_d[u]
        s = np.matmul(U[u], V[c].T)[None, :].astype(np.float32)
        pad = np.full((1, max(10, len(c))), -np.inf, np.float32); pad[0, :len(c)] = s
        ip, ix = oracle.lists_to_csr([range(len(test_d[u]))])
        rows.append(oracle.evaluate_matrix(pad, ip, ix, [2, 4], 10)[0])
    got = np.mean(np.stack(rows), axis=0, dtype=np.float32)
    want = np.array([float(x) for x in kat["eval"].split()], np.float32)
    assert got.shape == want.shape == (20,)
    assert np.abs(got - want).max() < 5e-8 + 1e-8          # the string carries 8 decimals
    assert "\t".join(("%.8f" % x).ljust(12) for x in got) == kat["eval"]


def test_adjacency_restatements_equal_the_reference_classes(ml100k):
    """LightGCN.create_adj_mat for 'plain', 'norm', 'gcmc', 'pre', 'mean' (LightGCN.py:35-78) and NGCF.get_adj_mat('norm')
    (NGCF.py:288-319) run by the REAL reference classes on the ml-100k split (tests/golden/kat_adjacency.json): the
    oracle's restatements give the same sparsity pattern and the same fp32 values, crc for crc."""
    import json
    import os
    import zlib
    with open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "kat_adjacency.json")) as f:
        kat = json.load(f)
    d = ml100k
    nu, ni = d["num_users"], d["num_items"]

    def digest(A):
        A = A.tocoo().astype(np.float32).tocsr()
        A.sort_indices()
        return (int(A.nnz), zlib.crc32(A.indptr.astype(np.int64).tobytes()), zlib.crc32(A.indices.astype(np.int32).tobytes()),
                zlib.crc32(A.data.astype(np.float32).tobytes()))
    for t in ("plain", "norm", "gcmc", "pre", "mean"):
        w = kat["lightgcn_" + t]
        got = digest(tf_math.lightgcn_adj(d["train_indptr"], d["train_indices"], nu, ni, t))
        assert got == (w["nnz"], w["indptr_crc32"], w["indices_crc32"], w["data_crc32"]), t
    w = kat["ngcf_norm"]
    got = digest(tf_math.ngcf_adj(d["train_indptr"], d["train_indices"], nu, ni, "norm"))
    assert got == (w["nnz"], w["indptr_crc32"], w["indices_crc32"], w["data_crc32"])


@pytest.mark.skipif(oracle.ref_lib() is None, reason="oracle/_ref (the compiled reference headers) is not built")
@pytest.mark.parametrize("trial", range(12))
def test_oracle_equals_reference_headers_on_non_finite_scores(trial):
    """The oracle is the truth the GPU evaluator is held to for non-finite scores as well: on matrices with NaN
    inside and outside the heap seed [0, L), +-inf, all -inf rows and empty truth rows, arg_topk and evaluate_matrix
    equal the reference's compiled arg_topk.h / evaluate.h (libstdc++'s partial_sort_copy keeps a NaN that seeds
    its heap, which reorders the ranking; a NaN offered later is never admitted)."""
    rs = np.random.RandomState(700 + trial)
    for _ in range(40):
        B, N, K = 8, int(rs.randint(2, 400)), int(rs.randint(1, 40))
        K = min(K, N)
        L = min(2 * K, N)
        S = rs.randn(B, N).astype(np.float32)
        if trial % 2:
            S = np.round(S * 2).astype(np.float32)          # ties
        S[rs.rand(B, N) < 0.05] = np.inf
        S[rs.rand(B, N) < 0.05] = -np.inf
        lo, hi = [(0, N), (0, L), (L, N)][trial % 3]
        for b in range(B):
            if hi > lo:
                S[b, rs.randint(lo, hi, size=rs.randint(1, 4))] = np.nan
        S[0] = -np.inf                                      # a row with nothing finite
        S[1, :L] = np.nan                                   # a NaN heap root
        for k in (K, L):
            assert np.array_equal(oracle.arg_topk(S, k), oracle.arg_topk(S, k, impl="reference"))
        truth = [rs.choice(N, rs.randint(0, min(N, 5) + 1), replace=False) for _ in range(B)]
        truth[2] = []
        ip, ix = oracle.lists_to_csr(truth)
        want = oracle.evaluate_matrix(S, ip, ix, ALL, K, impl="reference")
        assert np.array_equal(oracle.evaluate_matrix(S, ip, ix, ALL, K), want, equal_nan=True)
