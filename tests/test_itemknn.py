"""CPU tests of ItemKNN: the numpy restatement (tests/itemknn_math.py) against the reference's own Compute_Similarity
on ml-100k (tests/golden/kat_itemknn.npz, written by tests/golden/make_itemknn_golden.py), the scoring order against
scipy, the conf values, model resolution, the reference's ValueError and the ABI's argument checks."""
import os
import sys

import numpy as np
import pytest
import scipy.sparse as sp

import itemknn_math as km

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")
NAMES = ("cosine", "adjusted", "asymmetric", "pearson", "jaccard", "tanimoto", "dice", "tversky", "euclidean")
REFERENCE_CONF = dict(neighbor=5, shrink=0, similarity="euclidean", asymmetric_alpha=1, tversky_alpha=0.5,
                      tversky_beta=0.5, verbose=1)


def ml100k_train(binary=False):
    """The ml-100k train matrix as ItemKNN gets it (train.tocsc()): int64 ratings, or float64 ones."""
    z = np.load(os.path.join(GOLDEN, "ml100k_split.npz"))
    r = np.load(os.path.join(GOLDEN, "kat_itemknn.npz"))["ratings"]
    data = np.ones(len(r)) if binary else r.astype(np.int64)
    shape = (int(z["num_users"]), int(z["num_items"]))
    return sp.csr_matrix((data, z["train_indices"].astype(np.int32), z["train_indptr"].astype(np.int64)),
                         shape=shape).tocsc()


@pytest.fixture(scope="module")
def kat():
    return dict(np.load(os.path.join(GOLDEN, "kat_itemknn.npz")))


def same_bits(a, b):
    return np.array_equal(np.asarray(a, np.float32).view(np.uint32), np.asarray(b, np.float32).view(np.uint32)) or (
        np.array_equal(np.isnan(a), np.isnan(b)) and np.array_equal(np.nan_to_num(a), np.nan_to_num(b)))


def check_against_fixture(kat, key, ni, w5, w100):
    """W ({c: (rows, f32 values)}) at neighbor 5 and 100 against the reference's: the same count in every column, the
    same rows and value bits in every column without a boundary tie, the same multiset of values in every tied column
    (compared through itemknn_math.block_crcs, 64 columns per crc), the same number of NaN.  Returns the number of
    tied columns at neighbor 5."""
    for K, w in ((5, w5), (100, w100)):
        want = kat["%s_k%d_counts" % (key, K)].astype(np.int64)
        got = np.array([len(w[c][0]) for c in range(ni)])
        bad = np.flatnonzero(got != want)
        assert len(bad) == 0, (key, K, "counts differ in columns", bad[:10])
        ties = np.unpackbits(kat["%s_tie%d" % (key, K)])[:ni].astype(bool)
        bad = np.flatnonzero(km.block_crcs(w, ties, ni) != kat["%s_k%d_crc" % (key, K)])
        assert len(bad) == 0, (key, K, "W differs in the column blocks starting at", bad[:10] * km.CRC_BLOCK)
        nan = sum(int(np.isnan(w[c][1]).sum()) for c in range(ni))
        assert nan == int(kat["%s_k%d_nan" % (key, K)]), (key, K, nan)
    return int(np.unpackbits(kat[key + "_tie5"])[:ni].sum())


@pytest.mark.parametrize("binary", [False, True], ids=["int64", "float64_binary"])
@pytest.mark.parametrize("name", NAMES)
def test_restatement_equals_the_reference_on_ml100k(kat, name, binary):
    train = ml100k_train(binary)
    ni = train.shape[1]
    for shrink in (0, 10):
        key = "%s_%s_s%d" % ("bin" if binary else "int", name, shrink)
        X, kind, va, vb = km.prepare(train, name, 1)
        w5 = km.similarity(X, kind, va, vb, 5, shrink, 0.5, 0.5)
        w100 = km.similarity(X, kind, va, vb, 100, shrink, 0.5, 0.5)
        check_against_fixture(kat, key, ni, w5, w100)


def test_fixture_pins_the_facts_the_device_must_reproduce(kat):
    """Euclidean at K = 5 on the int64 ratings: 8 240 entries, no NaN, nothing in the 34 cold columns; adjusted and
    pearson on float64 binary data centre every entry to 0 (empty W); pearson on int64 ratings subtracts truncated
    averages (its W differs from the one with exact averages)."""
    train = ml100k_train()
    assert train.dtype == np.int64
    cold = np.flatnonzero(np.diff(train.indptr) == 0)
    assert len(cold) == 34
    counts = kat["int_euclidean_s0_k5_counts"]
    assert counts.sum() == 8240 and int(kat["int_euclidean_s0_k5_nan"]) == 0
    assert not counts[cold].any() and (counts[np.diff(train.indptr) > 0] == 5).all()
    for name in ("adjusted", "pearson"):
        for s in (0, 10):
            assert kat["bin_%s_s%d_k5_counts" % (name, s)].sum() == 0
            assert kat["bin_%s_s%d_k100_counts" % (name, s)].sum() == 0
    X, kind, va, vb = km.prepare(train, "pearson", 1)
    assert X.dtype == np.int64
    Xf = sp.csc_matrix(train, dtype=np.float64)
    n = np.diff(Xf.indptr)
    avg = np.zeros(Xf.shape[1])
    avg[n > 0] = np.asarray(Xf.sum(0)).ravel()[n > 0] / n[n > 0]
    assert not np.array_equal(X.data, Xf.data - np.repeat(avg, n))


def test_unknown_similarity_raises_the_reference_error(kat):
    with pytest.raises(ValueError) as e:
        km.prepare(ml100k_train(), "nope")
    assert str(e.value) == str(kat["unknown_error"])


def test_selection_rule_on_ties_negatives_and_nan():
    v = np.array([0.5, np.nan, 0.5, -1.0, 0.0, 0.5, -0.0, np.nan, 2.0])
    assert km.select(v, 2)[0].tolist() == [0, 8]
    assert km.select(v, 3)[0].tolist() == [0, 2, 8]
    assert km.select(v, 6)[0].tolist() == [0, 2, 5, 8]             # the zeros selected, then dropped
    assert km.select(v, 7)[0].tolist() == [0, 2, 3, 5, 8]          # a negative value is kept
    r, w = km.select(v, 9)
    assert r.tolist() == [0, 1, 2, 3, 5, 7, 8] and np.isnan(w[[1, 5]]).all()  # NaN last, and kept once reached


def test_scores_are_scipys_sum_order():
    """ratings[u, j] as scipy forms train.tocsc().dot(W): per (u, j) the float64 sum over column j's entries in
    ascending k of X[u, k] * W[k, j], from 0 -- the order the score kernel walks; checked on non-integer data where
    another order would round differently."""
    rs = np.random.RandomState(3)
    nu, ni = 60, 90
    X = sp.random(nu, ni, density=0.3, random_state=rs, format="csr") * 3.7
    W = sp.random(ni, ni, density=0.2, random_state=rs, format="csc", dtype=np.float32)
    want = km.scores(X, W, np.arange(nu))
    X.sort_indices()
    W.sort_indices()
    got = np.zeros((nu, ni), np.float32)
    for u in range(nu):
        row = dict(zip(X.indices[X.indptr[u]:X.indptr[u + 1]], X.data[X.indptr[u]:X.indptr[u + 1]]))
        for j in range(ni):
            acc = 0.0
            for k, w in zip(W.indices[W.indptr[j]:W.indptr[j + 1]], W.data[W.indptr[j]:W.indptr[j + 1]]):
                if k in row:
                    acc = acc + row[k] * float(w)
            got[u, j] = np.float32(acc)
    assert np.array_equal(got.view(np.uint32), want.view(np.uint32))


def test_conf_parses_to_the_reference_values(tmp_path, monkeypatch):
    from neurec_b200.util import Configurator
    (tmp_path / "conf").mkdir()
    (tmp_path / "conf" / "ItemKNN.properties").write_text(open(os.path.join(ROOT, "conf", "ItemKNN.properties")).read())
    (tmp_path / "NeuRec.properties").write_text(open(os.path.join(ROOT, "NeuRec.properties")).read())
    monkeypatch.chdir(tmp_path)
    monkeypatch.setattr(sys, "argv", ["main.py", "--recommender=ItemKNN"])
    conf = Configurator("NeuRec.properties", default_section="hyperparameters")
    for key, value in REFERENCE_CONF.items():
        assert conf[key] == value and type(conf[key]) is type(value), key


def test_main_resolves_itemknn():
    import main
    from neurec_b200.model.general_recommender.ItemKNN import ItemKNN
    assert main.resolve_model("ItemKNN") is ItemKNN
    with pytest.raises(ImportError, match="HRM, NPE, FPMCplus, Caser, FISM, ItemKNN"):
        main.resolve_model("NAIS")


def _lib():
    from neurec_b200 import _build, _lib as lib
    if not os.path.isfile(lib.LIB_PATH):
        _build.build()
    return lib


def test_abi_rejects_bad_arguments_before_any_cuda_call():
    """Every check runs before any CUDA call, so a rejected call writes nothing; host pointers stand in for the
    device arrays (they are never touched)."""
    lib = _lib()
    L = lib.load()
    n = None
    buf = np.zeros(8, np.float32)
    x = buf.ctypes.data

    def sim(nu=4, ni=10, kind=0, k=5, shrink=0.0, ta=0.5, tb=0.5, arr=x, work=n, work_bytes=0):
        return L.nrc_itemknn_similarity(nu, ni, x, x, x, arr, x, x, kind, x, x, shrink, ta, tb, k, 1, 10.0, work,
                                        work_bytes, x, x, x, n)

    assert L.nrc_itemknn_work_bytes(1000) == 0 and L.nrc_itemknn_work_bytes(0) == 0
    with pytest.raises(ValueError, match="num_items"):
        lib.check(sim(ni=0))
    with pytest.raises(ValueError, match="num_users"):
        lib.check(sim(nu=-1))
    for kind in (-1, 5):
        with pytest.raises(ValueError, match="kind"):
            lib.check(sim(kind=kind))
    with pytest.raises(ValueError, match="neighbor"):
        lib.check(sim(k=0))
    for kw in (dict(shrink=float("nan")), dict(ta=float("nan")), dict(tb=float("nan"))):
        with pytest.raises(ValueError, match="NaN"):
            lib.check(sim(**kw))
    with pytest.raises(ValueError, match="required"):
        lib.check(sim(arr=n))
    with pytest.raises(ValueError, match="nrc_itemknn_work_bytes"):
        lib.check(sim(ni=60000, work=x, work_bytes=8))
    with pytest.raises(ValueError, match="neighbor"):
        lib.check(L.nrc_itemknn_scores(10, x, x, x, 0, x, x, x, x, 2, x, n))
    with pytest.raises(ValueError, match="batch"):
        lib.check(L.nrc_itemknn_scores(10, x, x, x, 5, x, x, x, x, -1, x, n))
    with pytest.raises(ValueError, match="required"):
        lib.check(L.nrc_itemknn_scores(10, n, x, x, 5, x, x, x, x, 2, x, n))
    with pytest.raises(lib.NrcError) as e:
        lib.check(L.nrc_itemknn_scores(220 * 1024 // 8 * 32 + 1, x, x, x, 5, x, x, x, x, 2, x, n))
    assert e.value.rc == lib.NRC_E_LIMIT
    lib.check(L.nrc_itemknn_scores(10, n, n, n, 5, n, n, n, n, 0, n, n))    # an empty batch needs no arrays
    assert buf.tolist() == [0.0] * 8
    out = np.zeros(12, np.int32)
    with pytest.raises(ValueError):
        lib.check(L.nrc_itemknn_last_routes(None))
    lib.check(L.nrc_itemknn_last_routes(out.ctypes.data))
