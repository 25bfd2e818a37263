"""CPU tests of FISM: the numpy restatement (tests/fism_math.py) against torch float64 autograd of the reference's
padded graph, both instance layouts against the reference's own generators (tests/golden/kat_fism_layout.json), the
conf values, model resolution and the ABI's argument checks."""
import json
import os
import sys
import zlib

import numpy as np
import pytest
import torch

import fism_math as fm

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")
MODES = [(True, "bpr"), (True, "hinge"), (True, "square"), (False, "cross_entropy"), (False, "square")]
REFERENCE_CONF = dict(epochs=100, batch_size=256, embedding_size=16, regs=[0.0001, 0.0001], alpha=0.5,
                      learning_rate=0.001, learner="adam", is_pairwise=False, num_neg=4, loss_function="square",
                      init_method="normal", stddev=0.01, verbose=1)


def _ml100k_csr():
    z = np.load(os.path.join(GOLDEN, "ml100k_split.npz"))
    return z["train_indptr"].astype(np.int64), z["train_indices"].astype(np.int32), int(z["num_items"])


def _crc(a):
    return int(zlib.crc32(np.ascontiguousarray(np.asarray(a), dtype=np.int32).tobytes()))


def _hist_crc(hist_ptr, hist_idx, rows, excl=None):
    lists = fm.histories(hist_ptr, hist_idx, rows, excl)
    lens = [len(h) for h in lists]
    return {"n_rows": int(sum(lens)), "lens_crc32": _crc(lens), "items_crc32": _crc(np.concatenate(lists))}


def test_layouts_equal_the_reference_generators_on_ml100k():
    """The pointwise and pairwise instances of the reference's generators, run by the reference on the ml-100k train
    CSR: the restatement and the plug-in's layout reproduce their histories, counts, positives and labels exactly
    (the pairwise generator's even-position positives and shared odd-position history included)."""
    from neurec_b200.model.general_recommender import FISM as plug
    with open(os.path.join(GOLDEN, "kat_fism_layout.json")) as f:
        kat = json.load(f)
    ptr, idx, ni = _ml100k_csr()
    assert ni == kat["num_items"]
    want = kat["pointwise"]
    L = fm.pointwise_layout(ptr, idx, want["num_neg"])
    assert len(L["rows"]) == want["n"] == 401835
    assert _hist_crc(ptr, idx, L["rows"], L["excl"]) == want["histories"]
    assert want["histories"]["n_rows"] == 64883548
    assert _crc(L["num"]) == want["num_idx_crc32"]
    assert _crc(L["labels"].astype(np.int32)) == want["labels_crc32"]
    assert _crc(L["items"][L["pos_slot"]]) == want["positives_crc32"]
    rows, excl, num, labels = plug.pointwise_layout(ptr, idx, want["num_neg"])
    for a, b in ((rows, L["rows"]), (excl, L["excl"]), (num, L["num"]), (labels, L["labels"])):
        assert np.array_equal(a, b)
    want = kat["pairwise"]
    (hp, hi), P = fm.pairwise_layout(ptr, idx)
    assert len(P["rows"]) == want["n"] == 40381
    h = _hist_crc(hp, hi, P["rows"])
    assert h == want["histories_pos"] == want["histories_neg"] and h["n_rows"] == 3248097
    assert _crc(P["num"]) == want["num_idx_pos_crc32"] and _crc(P["num_neg"]) == want["num_idx_neg_crc32"]
    assert _crc(P["items"]) == want["positives_crc32"]
    (php, phi), (rows, items, num, num_neg) = plug.pairwise_layout(ptr, idx)
    assert np.array_equal(php, hp) and np.array_equal(phi, hi)
    for a, b in ((rows, P["rows"]), (items, P["items"]), (num, P["num"]), (num_neg, P["num_neg"])):
        assert np.array_equal(a, b)


def test_pairwise_layout_on_toy_rows():
    """A row of 5 gives positives at positions 0, 2, 4 and the history [1, 3]; rows of one item give nothing."""
    ptr = np.array([0, 5, 6, 8], np.int64)
    idx = np.array([10, 11, 12, 13, 14, 7, 3, 4], np.int32)
    (hp, hi), P = fm.pairwise_layout(ptr, idx)
    assert hp.tolist() == [0, 2, 2, 3] and hi.tolist() == [11, 13, 4]
    assert P["rows"].tolist() == [0, 0, 0, 2] and P["items"].tolist() == [10, 12, 14, 3]
    assert P["num"].tolist() == [5, 5, 5, 2] and P["num_neg"].tolist() == [6, 6, 6, 3]


def _autograd(c1, Q, b, hists, num, items, third, num_neg, pairwise, loss, alpha, lam, gamma):
    """The reference's graph in torch float64: histories padded with id I, which reads the constant zero row c2."""
    I, d = c1.shape
    t = lambda a: torch.tensor(a, dtype=torch.float64, requires_grad=True)
    C1, QQ, B = t(c1), t(Q), t(b)
    width = max(1, max(len(h) for h in hists))
    pad = np.full((len(hists), width), I, np.int64)
    for s, h in enumerate(hists):
        pad[s, :len(h)] = h
    emb = torch.cat([C1, torch.zeros(1, d, dtype=torch.float64)], 0)
    p = emb[torch.from_numpy(pad)].sum(1)
    it = torch.from_numpy(np.asarray(items, np.int64))

    def out(ids, n):
        coeff = torch.pow(torch.tensor(np.asarray(n, np.float64)), -float(alpha))
        return coeff * (p * QQ[ids]).sum(1) + B[ids]

    x = out(it, num)
    if pairwise:
        jt = torch.from_numpy(np.asarray(third, np.int64))
        y = x - out(jt, num_neg)
        if loss == "bpr":
            lo = torch.nn.functional.softplus(-y).sum()
        elif loss == "hinge":
            lo = torch.clamp(y + 1.0, min=0.0).sum()
        else:
            lo = ((1.0 - y) ** 2).sum()
        reg = gamma * ((QQ[jt] ** 2).sum() / 2 + (QQ[it] ** 2).sum() / 2)
    else:
        z = torch.tensor(np.asarray(third, np.float64))
        if loss == "cross_entropy":
            lo = torch.nn.functional.binary_cross_entropy_with_logits(x, z, reduction="mean")
        else:
            lo = ((z - x) ** 2).sum()
        reg = gamma * (QQ[it] ** 2).sum() / 2
    total = lo + lam * (p ** 2).sum() / 2 + reg
    total.backward()
    return float(total.detach()), [C1.grad.numpy(), QQ.grad.numpy(), B.grad.numpy()]


@pytest.mark.parametrize("alpha", [0.0, 0.5])
@pytest.mark.parametrize("pairwise,loss", MODES)
def test_restatement_vs_autograd(pairwise, loss, alpha):
    """Loss and all three gradients of a batch with repeated users, targets and history rows across samples, an
    excluded item, an empty history and counts that differ from the history lengths."""
    rs = np.random.RandomState(7 + int(alpha * 10) + 3 * len(loss))
    ni, d, B = 40, 6, 24
    c1, Q = rs.randn(ni, d) * 0.3, rs.randn(ni, d) * 0.3
    b = rs.randn(ni) * 0.2
    rows_h = [rs.choice(ni, rs.randint(1, 12), replace=False) for _ in range(6)] + [np.zeros(0, np.int64)]
    hp = np.zeros(len(rows_h) + 1, np.int64)
    hp[1:] = np.cumsum([len(h) for h in rows_h])
    hi = np.concatenate(rows_h).astype(np.int32)
    rows = rs.randint(0, len(rows_h), B).astype(np.int32)
    rows[:3] = [2, 2, 6]
    excl = np.full(B, -1, np.int32)
    if not pairwise:
        excl[1] = hi[hp[2]]
        excl[4] = hi[hp[rows[4] + 1] - 1] if hp[rows[4] + 1] > hp[rows[4]] else -1
    num = (np.diff(hp)[rows] + rs.randint(0, 3, B)).astype(np.int32)
    num[num == 0] = 1
    items = rs.randint(0, ni, B).astype(np.int32)
    items[5:8] = items[0]
    third = rs.randint(0, ni, B).astype(np.int32) if pairwise else rs.randint(0, 2, B).astype(np.float64)
    if pairwise:
        third[8:10] = items[0]                                   # a negative that is another sample's target
    num_neg = (num + 1).astype(np.int32) if pairwise else None
    lam, gamma = 0.03, 0.05
    want_l, want = _autograd(c1, Q, b, fm.histories(hp, hi, rows, excl), num, items, third, num_neg, pairwise, loss,
                             alpha, lam, gamma)
    got_l, got, (tC, tI) = fm.loss_and_grad(c1, Q, b, hp, hi, rows, excl, num, items, third, num_neg, pairwise, loss,
                                            alpha, lam, gamma, dtype=np.float64)
    assert abs(got_l - want_l) <= 1e-12 * max(1.0, abs(want_l))
    for g, w in zip(got, want):
        np.testing.assert_allclose(g, w, rtol=1e-10, atol=1e-12)
    used = np.concatenate(fm.histories(hp, hi, rows, excl))
    assert np.array_equal(np.flatnonzero(tC), np.unique(used))
    assert np.array_equal(np.flatnonzero(tI), np.unique(np.concatenate([items, third]) if pairwise else items))


def test_conf_parses_to_the_reference_values(tmp_path, monkeypatch):
    from neurec_b200.util import Configurator
    (tmp_path / "conf").mkdir()
    (tmp_path / "conf" / "FISM.properties").write_text(open(os.path.join(ROOT, "conf", "FISM.properties")).read())
    (tmp_path / "NeuRec.properties").write_text(open(os.path.join(ROOT, "NeuRec.properties")).read())
    monkeypatch.chdir(tmp_path)
    monkeypatch.setattr(sys, "argv", ["main.py", "--recommender=FISM"])
    conf = Configurator("NeuRec.properties", default_section="hyperparameters")
    for key, value in REFERENCE_CONF.items():
        assert conf[key] == value and type(conf[key]) is type(value), key


def test_main_resolves_fism():
    import main
    from neurec_b200.model.general_recommender.FISM import FISM
    assert main.resolve_model("FISM") is FISM
    with pytest.raises(ImportError, match="HRM, NPE, FPMCplus, Caser, FISM"):
        main.resolve_model("NAIS")


def _lib():
    from neurec_b200 import _build, _lib as lib
    if not os.path.isfile(lib.LIB_PATH):
        _build.build()
    return lib


def test_abi_rejects_bad_arguments_before_any_cuda_call():
    """Every check runs before any CUDA call, so a rejected call writes nothing; NULL device pointers stand in for
    the tables (they are never touched)."""
    lib = _lib()
    L = lib.load()
    n = None
    buf = np.zeros(8, np.float32)
    x = buf.ctypes.data                                    # a non-NULL host pointer; never dereferenced here

    def grad(dim=16, ni=10, pairwise=0, loss=2, batch=4, alpha=0.5, num_neg=x, tables=x, grads=x):
        return L.nrc_fism_grad(tables, tables, tables, ni, dim, x, x, x, n, x, x, x, num_neg, batch, pairwise, loss,
                               alpha, 0.0, 0.0, grads, grads, grads, grads, grads, 1, n, n)

    def epoch(dim=16, pairwise=0, loss=2, batch_size=4, opt=1, alpha=0.5, slots=x):
        return L.nrc_fism_train_epoch(x, x, x, 10, dim, x, x, x, n, x, x, x, x, 8, batch_size, pairwise, loss, alpha,
                                      0.0, 0.0, opt, x, x, x, x, x, x, x, slots, slots, 1, x, n)

    for call in (grad, epoch):
        for dim in (0, 257):
            with pytest.raises(lib.NrcError) as e:
                lib.check(call(dim=dim))
            assert e.value.rc == lib.NRC_E_LIMIT
        for pairwise, loss in ((0, 0), (0, 1), (1, 3)):
            with pytest.raises(ValueError, match="suitable loss"):
                lib.check(call(pairwise=pairwise, loss=loss))
        for alpha in (float("nan"), float("inf")):
            with pytest.raises(ValueError, match="alpha"):
                lib.check(call(alpha=alpha))
    with pytest.raises(ValueError, match="num_items"):
        lib.check(grad(ni=0))
    with pytest.raises(ValueError, match="batch"):
        lib.check(grad(batch=-1))
    with pytest.raises(ValueError, match="num_neg"):
        lib.check(grad(pairwise=1, loss=0, num_neg=n))
    with pytest.raises(ValueError, match="required"):
        lib.check(grad(tables=n))
    with pytest.raises(ValueError, match="required"):
        lib.check(grad(grads=n))
    with pytest.raises(ValueError, match="batch_size"):
        lib.check(epoch(batch_size=0))
    with pytest.raises(ValueError, match="optimizer"):
        lib.check(epoch(opt=9))
    with pytest.raises(ValueError, match="required"):
        lib.check(epoch(slots=n))
    with pytest.raises(lib.NrcError) as e:
        lib.check(L.nrc_fism_query(n, 10, 300, n, n, n, 2, n, n))
    assert e.value.rc == lib.NRC_E_LIMIT
    with pytest.raises(ValueError, match="required"):
        lib.check(L.nrc_fism_query(n, 10, 16, n, n, n, 2, n, n))
    with pytest.raises(ValueError, match="alpha"):
        lib.check(L.nrc_fism_scores(x, x, x, 10, 16, float("nan"), x, x, 2, x, n))
    with pytest.raises(ValueError, match="required"):
        lib.check(L.nrc_fism_scores(n, x, x, 10, 16, 0.5, x, x, 2, x, n))
    with pytest.raises(lib.NrcError) as e:
        lib.check(L.nrc_fism_scores(x, x, x, 65535 * 256 + 1, 16, 0.5, x, x, 2, x, n))
    assert e.value.rc == lib.NRC_E_LIMIT
    assert buf.tolist() == [0.0] * 8
    out = np.zeros(18, np.int32)
    with pytest.raises(ValueError):
        lib.check(L.nrc_fism_last_routes(None))
    lib.check(L.nrc_fism_last_routes(out.ctypes.data))
