"""FPMCplus on the CPU: the restatement in tests/fpmcplus_math.py against a torch float64 autograd graph of the
reference's FPMCplus.py:53-119, the conf file against the reference's values, model resolution, the predict windows
and the ABI's argument checks."""
import os
import sys

import numpy as np
import pytest
import torch

import fpmcplus_math as fpm
from conftest import ROOT

T = lambda a: torch.tensor(np.asarray(a, dtype=np.float64), dtype=torch.float64, requires_grad=True)
I = lambda a: torch.as_tensor(np.asarray(a, dtype=np.int64))

# the reference's conf/FPMCplus.properties, key by key, with the types its parser gives
REFERENCE_CONF = {"epochs": 500, "batch_size": 128, "embedding_size": 16, "weight_size": 16, "high_order": 3,
                  "reg_mf": 0.00001, "reg_w": 0.001, "learning_rate": 0.001, "learner": "adam", "is_pairwise": True,
                  "num_neg": 4, "loss_function": "BPR", "embed_init_method": "tnormal",
                  "weight_init_method": "he_normal", "stddev": 0.01, "verbose": 1}
MODES = [(True, "bpr"), (True, "hinge"), (True, "square"), (False, "cross_entropy"), (False, "square")]


def test_conf_parses_to_the_reference_values(tmp_path, monkeypatch):
    from neurec_b200.util import Configurator
    (tmp_path / "conf").mkdir()
    (tmp_path / "conf" / "FPMCplus.properties").write_text(open(os.path.join(ROOT, "conf", "FPMCplus.properties")).read())
    (tmp_path / "NeuRec.properties").write_text(open(os.path.join(ROOT, "NeuRec.properties")).read())
    monkeypatch.chdir(tmp_path)
    monkeypatch.setattr(sys, "argv", ["main.py", "--recommender=FPMCplus"])
    conf = Configurator("NeuRec.properties", default_section="hyperparameters")
    for key, value in REFERENCE_CONF.items():
        assert conf[key] == value and type(conf[key]) is type(value), key


def test_main_resolves_fpmcplus():
    import main
    from neurec_b200.model.sequential_recommender.FPMCplus import FPMCplus
    assert main.resolve_model("FPMCplus") is FPMCplus
    with pytest.raises(ImportError, match="HRM, NPE, FPMCplus"):
        main.resolve_model("Fossil")


def test_fpmcplus_checks_the_loss_of_its_mode():
    from neurec_b200.model.sequential_recommender.FPMCplus import FPMCplus
    m = FPMCplus.__new__(FPMCplus)
    for pairwise, ok, bad in ((True, ("BPR", "hinge", "square"), ("cross_entropy",)),
                              (False, ("cross_entropy", "square"), ("bpr", "hinge"))):
        m.is_pairwise = pairwise
        for loss in ok:
            m.loss_function = loss
            m._check_loss()
            assert m._loss == loss.lower()
        for loss in bad:
            m.loss_function = loss
            with pytest.raises(Exception, match="please choose a suitable loss function"):
                m._check_loss()


# ------------------------------------------------------------------------------- restatement vs torch.autograd
def _loss(pairwise, kind, z, x):                   # util/learner.py:17-41
    if pairwise:
        if kind == "bpr":
            return torch.nn.functional.softplus(-x).sum()
        if kind == "hinge":
            return torch.clamp(x + 1.0, min=0).sum()
        return ((1.0 - x) ** 2).sum()
    if kind == "cross_entropy":
        return torch.nn.functional.binary_cross_entropy_with_logits(x, z, reduction="mean")
    return ((z - x) ** 2).sum()


def _l2(*ts):                                      # util/tool.py:216-217
    return sum((t ** 2).sum() for t in ts) / 2


def _autograd(tabs, u, w, i, third, pairwise, loss, reg_mf, reg_w):
    """FPMCplus.py:53-119 as a torch float64 graph (the concat, one matmul, tanh, h, exp / sum, as written)."""
    UI, IU, IL, LI, W, b, h = (T(t) for t in tabs)
    d = UI.shape[1]
    L = w.shape[1]

    def inference(item):
        a, iu, il, r = UI[I(u)], IU[I(item)], IL[I(item)], LI[I(w)]
        cat = torch.cat([a[:, None, :].expand(-1, L, -1), il[:, None, :].expand(-1, L, -1), r], 2)
        mlp = torch.tanh(cat.reshape(-1, 3 * d) @ W + b)
        e = (mlp @ h).reshape(-1, L)
        ex = torch.exp(e)
        att = (ex / ex.sum(1, keepdim=True))[:, :, None]
        s = (att * r).sum(1)
        return a, iu, il, r, (a * iu + il * s).sum(1)

    a, iu, il, r, x = inference(i)
    if pairwise:
        _, iuj, ilj, _, xj = inference(third)
        total = _loss(True, loss, None, x - xj) + reg_mf * _l2(a, iu, il, r, iuj, ilj) + reg_w * _l2(W, h)
    else:
        total = _loss(False, loss, torch.as_tensor(third, dtype=torch.float64), x) + reg_mf * _l2(a, iu, il, r)
    total.backward()
    return float(total.detach()), [t.grad.numpy() for t in (UI, IU, IL, LI, W, b, h)]


def _case(rs, n, L, nu, ni, d, w, pairwise):
    tabs = [(rs.randn(k, d) * 0.5).astype(np.float32) for k in (nu, ni, ni, ni)]
    tabs += [(rs.randn(3 * d, w) * 0.4).astype(np.float32), (rs.randn(1, w) * 0.3).astype(np.float32),
             (rs.randn(w, 1) * 0.7 + 1.0).astype(np.float32)]
    u, i = rs.randint(0, nu, n), rs.randint(0, ni, n)
    win = rs.randint(0, ni, (n, L))
    u[1] = u[0]                                         # a repeated user
    win[0, -1] = win[0, 0]                              # an id twice in one window
    win[2, 0], i[3] = i[2], win[3, 0]                   # items that are both in a window and a target
    if pairwise:
        third = rs.randint(0, ni, n)
        third[4] = i[5]                                 # a negative that is another sample's positive
        third[6] = win[6, 1 % L]                        # a negative inside its own window
    else:
        third = (rs.rand(n) < 0.3).astype(np.float32)
    return tabs, u, win, i, third


@pytest.mark.parametrize("L", [1, 3, 5])
@pytest.mark.parametrize("pairwise,loss", MODES)
def test_restatement_equals_autograd(pairwise, loss, L):
    rs = np.random.RandomState(11 + 7 * L + len(loss) + pairwise)
    nu, ni, d, w = 6, 9, 5, 4
    tabs, u, win, i, third = _case(rs, 24, L, nu, ni, d, w, pairwise)
    reg_mf, reg_w = 0.05, 0.2
    want_l, want_g = _autograd(tabs, u, win, i, third, pairwise, loss, reg_mf, reg_w)
    for dt, rtol in ((np.float64, 1e-10), (np.float32, 2e-5)):
        lo, grads, (tU, tI, tL) = fpm.fpmcplus_grad(*tabs, u, win, i, third, pairwise, loss, reg_mf, reg_w, dtype=dt)
        assert abs(float(lo) - want_l) <= rtol * abs(want_l), (dt, lo, want_l)
        for k, (g, ref) in enumerate(zip(grads, want_g)):
            assert g.shape == ref.shape
            assert np.allclose(g, ref, rtol=rtol, atol=rtol * max(1.0, np.abs(ref).max())), (dt, k)
    # the pointwise loss has no reg_w term: W and h get only their data gradients there
    if not pairwise:
        _, g0 = _autograd(tabs, u, win, i, third, pairwise, loss, reg_mf, 0.0)
        assert np.array_equal(g0[4], want_g[4]) and np.array_equal(g0[6], want_g[6])
    assert np.array_equal(np.flatnonzero(tU), np.unique(u)) and np.array_equal(np.flatnonzero(tL), np.unique(win))
    ids = np.concatenate([i, third]) if pairwise else i
    assert np.array_equal(np.flatnonzero(tI), np.unique(ids))


def test_scores_restatement_equals_the_training_score():
    """predict's x(u, window, j) is the training graph's x for that user, window and item."""
    rs = np.random.RandomState(5)
    tabs, u, win, i, third = _case(rs, 8, 3, 6, 9, 5, 4, False)
    want = fpm.fpmcplus_scores(*tabs, [u[0]], [win[0]])[0]
    for j in range(9):
        _, att = fpm.attention(tabs[0][[u[0]]].astype(np.float64), tabs[2][[j]].astype(np.float64),
                               tabs[3][win[[0]]].astype(np.float64), *[t.astype(np.float64) for t in tabs[4:]])
        s = (att[0][:, None] * tabs[3][win[0]]).sum(0)
        x = tabs[0][u[0]].astype(np.float64) @ tabs[1][j] + tabs[2][j].astype(np.float64) @ s
        assert abs(want[j] - x) <= 1e-12 * max(1.0, abs(x))


def test_scores_overflow_where_the_reference_overflows():
    """exp(e) without a max shift: an e beyond fp32's exp range overflows to inf, and inf / inf is NaN for that
    (user, item) in fp32; fp64 still holds it."""
    d, w = 2, 4
    UI, IU, IL = np.ones((1, d)), np.ones((2, d)), np.array([[1.0, 0.0], [0.0, 0.0]])
    LI = np.ones((3, d))
    W = np.zeros((3 * d, w))
    W[d] = 50.0                                          # tanh saturates at sign(IL_j[0])
    b, h = np.zeros((1, w)), np.full((w, 1), 30.0)       # |h|_1 = 120 > 88
    got32 = fpm.fpmcplus_scores(UI, IU, IL, LI, W, b, h, [0], [[0, 1, 2]], dtype=np.float32)
    got64 = fpm.fpmcplus_scores(UI, IU, IL, LI, W, b, h, [0], [[0, 1, 2]])
    assert np.isnan(got32[0, 0]) and np.isfinite(got32[0, 1]) and np.isfinite(got64).all()


# ------------------------------------------------------------------------------------ predict windows
def test_predict_uses_the_short_windows_of_short_histories():
    """The plug-in reads its predict windows from predict_windows: a user with fewer train items than high_order gets
    the shorter window of the reference's slice."""
    from neurec_b200.model.sequential_recommender import FPMCplus as mod
    from neurec_b200.model.sequential_recommender._base import SeqWindowRecommender, predict_windows
    assert issubclass(mod.FPMCplus, SeqWindowRecommender)
    assert mod.FPMCplus._init_windows is SeqWindowRecommender._init_windows
    train_dict = {0: np.array([4, 5, 6, 7]), 1: np.array([8]), 2: np.array([1, 2])}
    recent, length = predict_windows(train_dict, 4, 3)
    assert length.tolist() == [3, 1, 1, 0]
    assert recent[0].tolist() == [5, 6, 7] and recent[1, 0] == 8 and recent[2, 0] == 2


def test_init_draws_stay_those_of_one_initialiser():
    """_init_tables with one method per shape: the same generator stream as one initialiser for every shape."""
    from neurec_b200.model.sequential_recommender._base import SeqTableRecommender
    m = SeqTableRecommender.__new__(SeqTableRecommender)
    m.init_method, m.stddev = "tnormal", 0.01
    shapes = [[5, 4], [7, 4]]
    orig = torch.Tensor.cuda
    try:
        torch.Tensor.cuda = lambda self, *a, **k: self
        a = m._init_tables(shapes)
        b = m._init_tables(shapes, ["tnormal", "tnormal"])
        c = m._init_tables(shapes + [[6, 3]], ["tnormal", "tnormal", "he_normal"])
    finally:
        torch.Tensor.cuda = orig
    assert all(torch.equal(x, y) for x, y in zip(a, b)) and all(torch.equal(x, y) for x, y in zip(a, c))
    assert c[2].shape == (6, 3)


# ------------------------------------------------------------------------------------ ABI argument checks
def _lib():
    from neurec_b200 import _build, _lib as lib
    if not os.path.isfile(lib.LIB_PATH):
        _build.build()
    return lib


def test_abi_rejects_bad_arguments_before_any_cuda_call():
    lib = _lib()
    L = lib.load()
    ce, bpr = lib.LOSS_IDS["cross_entropy"], lib.LOSS_IDS["bpr"]
    n = None

    def grad(dim, wsz, window, pairwise, loss, batch=4):
        return L.nrc_fpmcplus_grad(n, n, n, n, n, n, n, dim, wsz, window, n, n, n, n, batch, pairwise, loss, 0.0, 0.0,
                                   n, n, n, n, n, n, n, n, n, n, 1, n, n, n)

    def epoch(dim, wsz, window, pairwise, loss, opt=1):
        return L.nrc_fpmcplus_train_epoch(n, n, n, n, n, n, n, 3, 5, dim, wsz, window, n, n, n, n, 8, 4, pairwise,
                                          loss, 0.0, 0.0, opt, n, n, n, n, n, n, n, n, n, n, n, n, n, n, 1, n, n, n)

    for call in (grad, epoch):
        for pairwise, loss in ((1, ce), (0, bpr), (0, lib.LOSS_IDS["hinge"]), (1, 99)):
            with pytest.raises(ValueError, match="please choose a suitable loss function"):
                lib.check(call(16, 16, 3, pairwise, loss))
        for dim, wsz, window in ((0, 16, 3), (257, 16, 3), (16, 0, 3), (16, 129, 3), (16, 16, 0), (16, 16, 65)):
            with pytest.raises(lib.NrcError) as e:
                lib.check(call(dim, wsz, window, 1, bpr))
            assert e.value.rc == lib.NRC_E_LIMIT
    with pytest.raises(ValueError, match="required"):                    # NULL tables, gradients and work
        lib.check(grad(16, 16, 3, 1, bpr))
    with pytest.raises(ValueError, match="please select a suitable optimizer"):
        lib.check(epoch(16, 16, 3, 1, bpr, opt=9))
    with pytest.raises(lib.NrcError) as e:
        lib.check(grad(16, 16, 3, 1, bpr, batch=65535 * 32 + 1))
    assert e.value.rc == lib.NRC_E_LIMIT
    for dim, wsz, window in ((0, 16, 3), (16, 129, 3), (16, 16, 65)):
        assert L.nrc_fpmcplus_work_floats(dim, wsz, window, 128) == lib.NRC_E_LIMIT
        with pytest.raises(lib.NrcError) as e:
            lib.check(L.nrc_fpmcplus_scores(n, n, n, n, n, n, n, 10, dim, wsz, window, n, 2, n, n, n, n, n))
        assert e.value.rc == lib.NRC_E_LIMIT
    assert L.nrc_fpmcplus_work_floats(16, 16, 3, 0) == lib.NRC_E_VALUE
    with pytest.raises(ValueError, match="required"):
        lib.check(L.nrc_fpmcplus_scores(n, n, n, n, n, n, n, 10, 16, 16, 3, n, 2, n, n, n, n, n))
    out = np.zeros(24, np.int32)
    with pytest.raises(ValueError):
        lib.check(L.nrc_fpmcplus_last_routes(None))
    lib.check(L.nrc_fpmcplus_last_routes(out.ctypes.data))
