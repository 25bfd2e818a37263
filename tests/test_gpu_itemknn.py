"""GPU parity of ItemKNN (csrc/itemknn.cu) through the C ABI against the restatement in tests/itemknn_math.py: the
similarity kernel on every route its shapes select (nrc_itemknn_last_routes), W's rows and float32 values bit for
bit on integer and non-integer data, K from 1 to I, cold items; ml-100k against the reference's own W
(tests/golden/kat_itemknn.npz); the scores bit for bit against scipy's train.tocsc().dot(W); the plug-in and
main.py."""
import os
import re
import subprocess
import sys
import zlib

import numpy as np
import pytest
import scipy.sparse as sp
import torch

import itemknn_math as km
from test_gpu_sequential import BASE_CONF, _Conf, write_timed_dataset
from test_itemknn import NAMES, check_against_fixture, ml100k_train, same_bits

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")
REACHED = set()
ROW_SMEM = 220 * 1024          # itemknn.cu's kKnnRowSmem: tier 0 up to ROW_SMEM / 8 items, tier 1 up to / 4
CONF = dict(recommender="ItemKNN", neighbor=5, shrink=0, similarity="euclidean", asymmetric_alpha=1,
            tversky_alpha=0.5, tversky_beta=0.5, verbose=1)


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _csr_dev(M):
    return dev(M.indptr.astype(np.int64)), dev(M.indices.astype(np.int32)), dev(M.data.astype(np.float64))


def synth(rs, nu, ni, per_user, values, cold=()):
    """A U x I train matrix with about per_user items per user and no entry in the `cold` columns: int64 ratings
    1..5 ("int"), float64 ones ("bin") or non-integer float64 ratings ("float")."""
    allowed = np.setdiff1d(np.arange(ni), np.asarray(cold, np.int64))
    rows = [np.unique(rs.choice(allowed, rs.randint(1, 2 * per_user), replace=True)) for _ in range(nu)]
    ptr = np.concatenate([[0], np.cumsum([len(r) for r in rows])]).astype(np.int64)
    idx = np.concatenate(rows).astype(np.int32)
    if values == "int":
        data = rs.randint(1, 6, len(idx)).astype(np.int64)
    elif values == "bin":
        data = np.ones(len(idx))
    else:
        data = rs.randint(1, 6, len(idx)) * rs.uniform(0.3, 1.7, len(idx))
    return sp.csr_matrix((data, idx, ptr), shape=(nu, ni))


def device_w(X, kind, va, vb, K, shrink=0, ta=0.5, tb=0.5, integral=None):
    Xc = sp.csc_matrix(X)
    Xc.sort_indices()
    R = Xc.tocsr()
    R.sort_indices()
    W = torch_ops().itemknn_similarity(*_csr_dev(R), *_csr_dev(Xc), X.shape[1], kind, dev(va), dev(vb), shrink, ta,
                                       tb, K, integral=integral)
    r = torch_ops().itemknn_last_routes()["similarity"]
    REACHED.add(("similarity", r["acc"], r["tier"], r["capped"]))
    return W, r


def torch_ops():
    from neurec_b200 import ops
    return ops


def check_columns(W, X, kind, va, vb, K, shrink=0, ta=0.5, tb=0.5, columns=None):
    """W's columns equal the restatement's: rows, and the float32 values bit for bit (NaN where it has NaN)."""
    counts, rows, vals = (t.cpu().numpy() for t in W)
    want = km.similarity(X, kind, va, vb, K, shrink, ta, tb, columns)
    for c, (r, v) in want.items():
        n = counts[c]
        assert n == len(r), (c, n, len(r))
        assert np.array_equal(rows[:n, c], r), c
        assert same_bits(vals[:n, c], v), c
    return want


def dev_cols(W):
    counts, rows, vals = (t.cpu().numpy() for t in W)
    return {c: (rows[:counts[c], c], vals[:counts[c], c]) for c in range(len(counts))}


@pytest.mark.parametrize("values", ["int", "bin", "float"])
@pytest.mark.parametrize("name", NAMES)
def test_small_catalogue_every_kind_bit_for_bit(name, values):
    """Tier 0, uncapped: every similarity on integer, binary and non-integer data, K in {1, 5, more than any column's
    candidates, I}, with cold items (euclidean's NaN between two cold items, kept once the selection reaches it);
    integer data on both accumulators."""
    rs = np.random.RandomState(zlib.crc32((name + values).encode()))
    nu, ni = 150, 257
    X0 = synth(rs, nu, ni, 6, values, cold=[3, 100, 256])
    X, kind, va, vb = km.prepare(X0.tocsc(), name, 0.75)
    for K in (1, 5, 150, ni):
        for integral in ((None, False) if values != "float" else (None,)):
            for shrink in (0, 3):
                W, r = device_w(X, kind, va, vb, K, shrink, 0.5, 0.25, integral=integral)
                assert r["tier"] == 0 and r["capped"] == 0 and r["k"] == K
                # tanimoto, dice and tversky make even non-integer data binary, so integral
                assert r["acc"] == (0 if integral is None and np.array_equal(X.data, np.round(X.data)) else 1)
                check_columns(W, X, kind, va, vb, K, shrink, 0.5, 0.25)


def test_capped_grid_and_cold_columns():
    """More columns than the 4 * SMs CTAs: each CTA takes several columns in turn, on both accumulators."""
    rs = np.random.RandomState(5)
    ni = 4 * _sms() + 37
    X0 = synth(rs, 300, ni, 12, "int", cold=[0, 7, ni - 1])
    for name in ("euclidean", "cosine", "pearson"):
        X, kind, va, vb = km.prepare(X0.tocsc(), name)
        for integral in (None, False):
            W, r = device_w(X, kind, va, vb, 5, integral=integral)
            assert r["capped"] == 1 and r["grid"] == 4 * _sms() and r["tier"] == 0
            check_columns(W, X, kind, va, vb, 5)


@pytest.mark.parametrize("ni,integral,tier", [
    (ROW_SMEM // 8 + 123, None, 1), (ROW_SMEM // 8 + 123, False, 2), (ROW_SMEM // 4 + 77, None, 2)])
def test_large_catalogue_global_rows(ni, integral, tier):
    """Catalogues whose row does not fit in shared memory: an int32 accumulator in shared memory with the keys in
    global work (tier 1), or both in global work (tier 2); every cold column and 200 others checked."""
    rs = np.random.RandomState(ni)
    cold = rs.choice(ni, 40, replace=False)
    X0 = synth(rs, 500, ni, 40, "bin", cold=cold)
    cols = np.concatenate([cold, rs.choice(ni, 200, replace=False), [0, ni - 1]])
    for name, K in (("cosine", 5), ("euclidean", 3)):
        X, kind, va, vb = km.prepare(X0.tocsc(), name)
        W, r = device_w(X, kind, va, vb, K, integral=integral)
        assert r["tier"] == tier and r["acc"] == (0 if integral is None else 1) and r["smem"] == (ni * 4 if tier == 1 else 0)
        check_columns(W, X, kind, va, vb, K, columns=cols)


@pytest.fixture(scope="module")
def kat():
    return dict(np.load(os.path.join(GOLDEN, "kat_itemknn.npz")))


@pytest.mark.parametrize("binary", [False, True], ids=["int64", "float64_binary"])
def test_ml100k_against_the_reference(kat, binary):
    """Every similarity at shrink 0 and 10: W at neighbor 5 equals the reference's on every column without a
    boundary tie, and at neighbor 100 has the reference's count and sorted values on every column."""
    train = ml100k_train(binary)
    ni = train.shape[1]
    for name in NAMES:
        for shrink in (0, 10):
            X, kind, va, vb = km.prepare(train, name, 1)
            w5 = dev_cols(device_w(X, kind, va, vb, 5, shrink)[0])
            w100 = dev_cols(device_w(X, kind, va, vb, 100, shrink)[0])
            check_against_fixture(kat, "%s_%s_s%d" % ("bin" if binary else "int", name, shrink), ni, w5, w100)


def _scores_all(R, W, users, batch=512):
    from neurec_b200 import ops
    out = []
    for b in range(0, len(users), batch):
        out.append(ops.itemknn_scores(*_csr_dev(R), W, dev(users[b:b + batch].astype(np.int32))).cpu().numpy())
        r = ops.itemknn_last_routes()["scores"]
        REACHED.add(("scores", r["capped"]))
    return np.concatenate(out)


@pytest.mark.parametrize("case", ["ml100k_euclidean_k5", "ml100k_cosine_k100", "float_pearson_k40"])
def test_scores_bit_for_bit_against_scipy(case):
    """Every user's row equals np.float32(train.tocsc().dot(W)) with W the device's, bit for bit."""
    from neurec_b200.model.general_recommender.ItemKNN import w_to_scipy
    if case.startswith("ml100k"):
        train = ml100k_train()
        name, K = ("euclidean", 5) if "euclidean" in case else ("cosine", 100)
        batch = 512
    else:
        train = synth(np.random.RandomState(9), 9 * _sms(), 700, 15, "float").tocsc()
        name, K = "pearson", 40
        batch = 9 * _sms()
    X, kind, va, vb = km.prepare(train, name, 1)
    W, _ = device_w(X, kind, va, vb, K)
    R = sp.csr_matrix(train)
    R.sort_indices()
    users = np.arange(train.shape[0])
    got = _scores_all(R, W, users, batch)
    want = km.scores(train, w_to_scipy(W, train.shape[1]), users)
    assert np.array_equal(got.view(np.uint32), want.view(np.uint32))


def test_plug_in_build_predict_and_evaluate(kat):
    """The plug-in on ml-100k at the conf defaults: W_sparse equals the reference's on untied columns, predict rows
    are the scores of scipy's product, candidate lists read from the row, and one evaluation runs."""
    from neurec_b200.data import Dataset
    from neurec_b200.model.general_recommender.ItemKNN import ItemKNN
    z = np.load(os.path.join(GOLDEN, "ml100k_split.npz"))
    train = ml100k_train().tocsr()
    shape = train.shape
    test = sp.csr_matrix((np.ones(len(z["test_indices"])), z["test_indices"].astype(np.int32),
                          z["test_indptr"].astype(np.int64)), shape=shape)
    ds = Dataset.from_csr("ml-100k", train, test)
    m = ItemKNN(None, ds, _Conf(BASE_CONF, **CONF))
    m.build_graph()
    Ws = m.W_sparse.tocsc()
    Ws.sort_indices()
    cols = {c: (Ws.indices[Ws.indptr[c]:Ws.indptr[c + 1]], Ws.data[Ws.indptr[c]:Ws.indptr[c + 1]])
            for c in range(shape[1])}
    assert Ws.nnz == 8240 and Ws.dtype == np.float32
    X, kind, va, vb = km.prepare(train.tocsc(), "euclidean", 1)
    check_against_fixture(kat, "int_euclidean_s0", shape[1], cols,
                          dev_cols(device_w(X, kind, va, vb, 100)[0]))
    users = [0, 5, 17, 942]
    got = m.predict(users)
    assert isinstance(got, torch.Tensor) and got.is_cuda and got.dtype == torch.float32 and got.shape == (4, shape[1])
    want = km.scores(train, m.W_sparse, users)
    assert np.array_equal(got.cpu().numpy().view(np.uint32), want.view(np.uint32))
    cand = [[1, 2, 3], [10], [0, 1681], [5, 5, 7]]
    for r, w, c in zip(m.predict(users, cand), got.cpu().numpy(), cand):
        assert isinstance(r, np.ndarray) and np.array_equal(r, w[c])
    vals = [float(x) for x in m.evaluate().split()]
    assert len(vals) == 10 and all(0.0 <= v <= 1.0 for v in vals)


def test_main_runs_itemknn(tmp_path):
    data = tmp_path / "dataset"
    write_timed_dataset(str(data))
    cmd = [sys.executable, os.path.join(ROOT, "main.py"), "--recommender=ItemKNN", "--data.input.path=%s" % data,
           "--data.input.dataset=toy", "--topk=[5,10]", "--test_batch_size=64", "--similarity=cosine",
           "--neighbor=20"]
    for f in ("NeuRec.properties", "conf"):
        os.symlink(os.path.join(ROOT, f), tmp_path / f)
    r = subprocess.run(cmd, cwd=tmp_path, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    out = r.stdout + r.stderr
    assert "metrics:\tPrecision@5 " in out and "NDCG@10" in out
    rows = re.findall(r"((?:[0-9]+\.[0-9]+[ \t]+){9}[0-9]+\.[0-9]+)", out)
    assert rows, out[-3000:]
    vals = np.array([float(x) for x in rows[-1].split()])
    assert np.isfinite(vals).all() and (vals >= 0).all() and (vals <= 1).all() and vals.max() > 0


def test_every_route_was_reached():
    """Runs last in this file: the int32 and float64 accumulators in shared memory, tier 1, tier 2 on both
    accumulators, the grid capped and not; the score kernel capped and not."""
    if len(REACHED) == 0:
        pytest.skip("the route tests did not run in this session")
    sims = {(a, t) for k, a, t, _ in (r for r in REACHED if r[0] == "similarity")}
    assert sims >= {(0, 0), (1, 0), (0, 1), (0, 2), (1, 2)}
    assert {r[3] for r in REACHED if r[0] == "similarity"} == {0, 1}
    assert ("scores", 0) in REACHED and ("scores", 1) in REACHED
