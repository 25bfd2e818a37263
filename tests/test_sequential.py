"""FPMC and TransRec without a GPU: the conf files, the models' registration, the sequential base class, the fp32
restatement's hand-derived gradients (tests/seq_math.py) against torch.autograd in float64, and the C ABI's argument
checks (which run before any CUDA call)."""
import os
import sys

import numpy as np
import pytest
import scipy.sparse as sp
import torch

import seq_math
from conftest import ROOT

T = lambda a: torch.tensor(np.asarray(a, dtype=np.float64), dtype=torch.float64, requires_grad=True)
I = lambda a: torch.as_tensor(np.asarray(a, dtype=np.int64))

# the reference's conf/FPMC.properties and conf/TransRec.properties, key by key, with the types its parser gives
REFERENCE_CONF = {
    "FPMC": {"epochs": 500, "batch_size": 512, "embedding_size": 16, "reg_mf": 0.01, "learning_rate": 0.001,
             "learner": "adam", "is_pairwise": False, "num_neg": 4, "loss_function": "cross_entropy",
             "init_method": "uniform", "stddev": 0.01, "verbose": 1},
    "TransRec": {"epochs": 500, "batch_size": 1024, "embedding_size": 50, "reg_mf": 0.0, "learning_rate": 0.001,
                 "learner": "adam", "is_pairwise": True, "num_neg": 4, "loss_function": "bpr",
                 "init_method": "tnormal", "stddev": 0.01, "verbose": 1},
}
MODES = [(True, "bpr"), (True, "hinge"), (True, "square"), (False, "cross_entropy"), (False, "square")]


@pytest.mark.parametrize("model", ["FPMC", "TransRec"])
def test_conf_parses_to_the_reference_values(tmp_path, monkeypatch, model):
    from neurec_b200.util import Configurator
    (tmp_path / "conf").mkdir()
    name = "%s.properties" % model
    (tmp_path / "conf" / name).write_text(open(os.path.join(ROOT, "conf", name)).read())
    (tmp_path / "NeuRec.properties").write_text(open(os.path.join(ROOT, "NeuRec.properties")).read())
    monkeypatch.chdir(tmp_path)
    monkeypatch.setattr(sys, "argv", ["main.py", "--recommender=%s" % model])
    conf = Configurator("NeuRec.properties", default_section="hyperparameters")
    for key, value in REFERENCE_CONF[model].items():
        assert conf[key] == value and type(conf[key]) is type(value), key


def test_main_resolves_the_sequential_models():
    import main
    from neurec_b200.model.sequential_recommender.FPMC import FPMC
    from neurec_b200.model.sequential_recommender.TransRec import TransRec
    assert main.resolve_model("FPMC") is FPMC and main.resolve_model("TransRec") is TransRec
    with pytest.raises(ImportError, match="FPMC, TransRec"):
        main.resolve_model("GRU4Rec")


def test_sequential_base_needs_times():
    """AbstractRecommender.py:48-52: the ValueError (message as the reference spells it) comes before the base
    constructor reads the configuration."""
    from neurec_b200.data import Dataset
    from neurec_b200.model.AbstractRecommender import SeqAbstractRecommender
    from neurec_b200.model.sequential_recommender.FPMC import FPMC
    train = sp.csr_matrix(np.eye(4, 6, dtype=np.float32))
    ds = Dataset.from_csr("toy", train, train)
    for make in (lambda: SeqAbstractRecommender(ds, {}), lambda: FPMC(None, ds, {})):
        with pytest.raises(ValueError, match="^Dataset does not contant time infomation!$"):
            make()


# ------------------------------------------------------------------------------- restatement vs torch.autograd
def _pair_loss(kind, x):          # util/learner.py:19-29
    if kind == "bpr":
        return -torch.nn.functional.logsigmoid(x).sum()
    if kind == "hinge":
        return torch.clamp(x + 1.0, min=0).sum()
    return ((1.0 - x) ** 2).sum()


def _point_loss(kind, z, x):      # util/learner.py:31-41
    if kind == "cross_entropy":
        return torch.nn.functional.binary_cross_entropy_with_logits(x, z, reduction="mean")
    return ((z - x) ** 2).sum()


def _l2(*ts):                     # util/tool.py:216-217
    return sum((t ** 2).sum() for t in ts) / 2


def _batch(rs, n, nu, ni, pairwise):
    u, l, i = rs.randint(0, nu, n), rs.randint(0, ni, n), rs.randint(0, ni, n)
    u[1], l[2], i[3] = u[0], i[0], l[1]            # repeated users, an item that is both recent and next
    third = rs.randint(0, ni, n) if pairwise else (rs.rand(n) < 0.3).astype(np.float32)
    return u, l, i, third


def _close(got, want):
    assert np.allclose(got, want, rtol=2e-5, atol=2e-6), np.abs(got - want).max()


@pytest.mark.parametrize("pairwise,loss", MODES)
def test_fpmc_grad_restatement_equals_autograd(pairwise, loss):
    """FPMC.py:61-84 written as a torch float64 graph; the restatement is fp32 (tolerance: fp32 rounding)."""
    rs = np.random.RandomState(0)
    nu, ni, d, reg = 7, 11, 5, 0.03
    tabs = [rs.randn(nu, d) * 0.5] + [rs.randn(ni, d) * 0.5 for _ in range(3)]
    tabs = [t.astype(np.float32) for t in tabs]
    u, l, i, third = _batch(rs, 24, nu, ni, pairwise)
    lo, grads, (tU, tI, tL) = seq_math.fpmc_grad(*tabs, u, l, i, third, pairwise, loss, reg)
    UI, IU, IL, LI = (T(t) for t in tabs)

    def infer(items):
        ui, iu, il, li = UI[I(u)], IU[I(items)], IL[I(items)], LI[I(l)]
        return ui, iu, il, li, (ui * iu + il * li).sum(1)
    a, iu_i, il_i, li_l, xi = infer(i)
    if pairwise:
        _, iu_j, il_j, _, xj = infer(third)
        total = _pair_loss(loss, xi - xj) + reg * _l2(a, iu_i, il_i, li_l, iu_j, il_j)
    else:
        total = _point_loss(loss, torch.as_tensor(third, dtype=torch.float64), xi) + reg * _l2(a, iu_i, il_i, li_l)
    total.backward()
    assert abs(float(total.detach()) - float(lo)) < 1e-5 * abs(float(total.detach()))
    for g, t in zip(grads, (UI, IU, IL, LI)):
        _close(g, t.grad.numpy())
    assert np.array_equal(np.flatnonzero(tU), np.unique(u)) and np.array_equal(np.flatnonzero(tL), np.unique(l))
    assert np.array_equal(np.flatnonzero(tI), np.unique(np.concatenate([i, third]) if pairwise else i))


@pytest.mark.parametrize("pairwise,loss", MODES)
def test_transrec_grad_restatement_equals_autograd(pairwise, loss):
    """TransRec.py:66-91 written as a torch float64 graph: g tiled over the batch and once in l2_loss."""
    rs = np.random.RandomState(1)
    nu, ni, d, reg = 6, 13, 4, 0.05
    P, Q = (rs.randn(nu, d) * 0.3).astype(np.float32), (rs.randn(ni, d) * 0.3).astype(np.float32)
    B, G = (rs.randn(ni) * 0.3).astype(np.float32), (rs.randn(1, d) * 0.3).astype(np.float32)
    u, l, i, third = _batch(rs, 20, nu, ni, pairwise)
    lo, (gP, gQ, gB, gG), (tP, tQ, tB) = seq_math.transrec_grad(P, Q, B, G, u, l, i, third, pairwise, loss, reg)
    tp, tq, tb, tg = T(P), T(Q), T(B), T(G)

    def infer(items):
        p, r, q, b = tp[I(u)], tq[I(l)], tq[I(items)], tb[I(items)]
        v = p + tg.tile(len(u), 1) + r - q
        return p, r, q, b, b - (v ** 2).sum(1)
    p1, r1, q1, b1, xi = infer(i)
    if pairwise:
        _, _, q2, b2, xj = infer(third)
        total = _pair_loss(loss, xi - xj) + reg * _l2(p1, r1, q2, q1, b1, b2, tg)
    else:
        total = _point_loss(loss, torch.as_tensor(third, dtype=torch.float64), xi) + reg * _l2(p1, r1, q1, b1, tg)
    total.backward()
    assert abs(float(total.detach()) - float(lo)) < 1e-5 * abs(float(total.detach()))
    for g, t in ((gP, tp), (gQ, tq), (gB, tb), (gG, tg)):
        _close(g, t.grad.numpy().reshape(g.shape))
    assert np.array_equal(np.flatnonzero(tP), np.unique(u))
    nxt = np.concatenate([i, third]) if pairwise else i
    assert np.array_equal(np.flatnonzero(tQ), np.unique(np.concatenate([l, nxt])))
    assert np.array_equal(np.flatnonzero(tB), np.unique(nxt))


def test_transrec_global_reg_counts_once_per_batch():
    """g's reg term is reg * g for the batch, not per sample: zero samples' worth of score gradient leaves reg * g."""
    rs = np.random.RandomState(2)
    P, Q = np.zeros((3, 4), np.float32), np.zeros((5, 4), np.float32)
    B, G = np.zeros(5, np.float32), (rs.randn(1, 4)).astype(np.float32)
    u, l, i, j = (np.arange(3) % 3, np.arange(3), np.arange(3), np.arange(3))
    # x_i == x_j for every sample and the square loss at 0 has slope -2: the samples' g-terms cancel (i == j)
    _, (_, _, _, gG), _ = seq_math.transrec_grad(P, Q, B, G, u, l, i, j, True, "square", 0.1)
    _close(gG, np.float32(0.1) * G.reshape(-1))


# ------------------------------------------------------------------------------------ ABI argument checks
def _lib():
    from neurec_b200 import _build, _lib as lib
    if not os.path.isfile(lib.LIB_PATH):
        _build.build()
    return lib


def test_abi_rejects_bad_loss_and_width_before_any_cuda_call():
    lib = _lib()
    L = lib.load()
    bpr, ce = lib.LOSS_IDS["bpr"], lib.LOSS_IDS["cross_entropy"]
    n = None

    def fpmc(dim, pairwise, loss):
        return L.nrc_fpmc_grad(n, n, n, n, dim, n, n, n, n, 4, pairwise, loss, 0.0, n, n, n, n, n, n, n, 1, n, n)

    def transrec(dim, pairwise, loss):
        return L.nrc_transrec_grad(n, n, n, n, dim, n, n, n, n, 4, pairwise, loss, 0.0, n, n, n, n, n, n, n, 1, n, n, n)

    def fpmc_epoch(dim, pairwise, loss):
        return L.nrc_fpmc_train_epoch(n, n, n, n, 3, 5, dim, n, n, n, n, 8, 4, pairwise, loss, 0.0, 1, n, n, n, n, n,
                                      n, n, n, n, n, n, 1, n, n)

    def transrec_epoch(dim, pairwise, loss):
        return L.nrc_transrec_train_epoch(n, n, n, n, 3, 5, dim, n, n, n, n, 8, 4, pairwise, loss, 0.0, 1, n, n, n, n,
                                          n, n, n, n, n, n, n, 1, n, n, n)

    for call in (fpmc, transrec, fpmc_epoch, transrec_epoch):
        for pairwise, loss in ((1, ce), (0, bpr), (1, 99)):
            with pytest.raises(ValueError, match="please choose a suitable loss function"):
                lib.check(call(16, pairwise, loss))
        for dim in (0, 257):
            with pytest.raises(lib.NrcError) as e:
                lib.check(call(dim, 1, bpr))
            assert e.value.rc == lib.NRC_E_LIMIT
    for dim in (0, 257):
        for rc in (L.nrc_fpmc_scores(n, n, n, n, 10, dim, n, n, 2, n, n),
                   L.nrc_transrec_scores(n, n, n, n, 10, dim, n, n, 2, n, n), L.nrc_transrec_work_floats(dim)):
            with pytest.raises(lib.NrcError) as e:
                lib.check(int(rc))
            assert e.value.rc == lib.NRC_E_LIMIT
    assert L.nrc_transrec_work_floats(50) == 128 * 50 + 1
