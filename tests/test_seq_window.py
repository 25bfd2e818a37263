"""HRM and NPE without a GPU: the conf files, the models' registration, the fp32 restatement's hand-derived gradients
(tests/seq_window_math.py) against torch.autograd in float64, the predict windows, and the C ABI's argument checks
(which run before any CUDA call)."""
import os
import sys

import numpy as np
import pytest
import scipy.sparse as sp
import torch

import seq_window_math as swm
from conftest import ROOT

T = lambda a: torch.tensor(np.asarray(a, dtype=np.float64), dtype=torch.float64, requires_grad=True)
I = lambda a: torch.as_tensor(np.asarray(a, dtype=np.int64))

# the reference's conf/HRM.properties and conf/NPE.properties, key by key, with the types its parser gives
REFERENCE_CONF = {
    "HRM": {"epochs": 3, "batch_size": 256, "embedding_size": 16, "reg_mf": 0, "topK": 10, "learning_rate": 0.001,
            "learner": "adam", "pre_agg": "max", "session_agg": "max", "high_order": 2, "num_neg": 4,
            "loss_function": "cross_entropy", "init_method": "normal", "stddev": 0.01, "verbose": 1},
    "NPE": {"epochs": 100, "batch_size": 256, "embedding_size": 64, "reg": 0.1, "learning_rate": 0.001,
            "learner": "adam", "high_order": 3, "num_neg": 4, "loss_function": "cross_entropy",
            "init_method": "tnormal", "stddev": 0.01, "verbose": 1},
}
LOSSES = ["cross_entropy", "square"]
AGGS = [(True, True), (True, False), (False, True), (False, False)]


@pytest.mark.parametrize("model", ["HRM", "NPE"])
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


def test_main_resolves_the_window_models():
    import main
    from neurec_b200.model.sequential_recommender.HRM import HRM
    from neurec_b200.model.sequential_recommender.NPE import NPE
    assert main.resolve_model("HRM") is HRM and main.resolve_model("NPE") is NPE
    with pytest.raises(ImportError, match="HRM, NPE"):
        main.resolve_model("Fossil")


def _timed_dataset():
    from neurec_b200.data import Dataset
    train = sp.csr_matrix(np.eye(4, 6, dtype=np.float32))
    return Dataset.from_csr("toy", train, train, time_matrix=train)


def test_models_need_times_and_npe_a_window_of_two(tmp_path, monkeypatch):
    from neurec_b200.data import Dataset
    from neurec_b200.model.sequential_recommender.HRM import HRM
    from neurec_b200.model.sequential_recommender.NPE import NPE
    train = sp.csr_matrix(np.eye(4, 6, dtype=np.float32))
    ds = Dataset.from_csr("toy", train, train)
    for cls in (HRM, NPE):
        with pytest.raises(ValueError, match="^Dataset does not contant time infomation!$"):
            cls(None, ds, {})
    monkeypatch.chdir(tmp_path)                                 # the model's log file
    conf = dict(REFERENCE_CONF["NPE"], recommender="NPE", high_order=1, metric=["Precision"], topk=[5],
                group_view=None, test_batch_size=128, num_thread=1)

    class _Conf(dict):
        def params_str(self):
            return "test"
    with pytest.raises(ValueError, match="high_order >= 2"):
        NPE(None, _timed_dataset(), _Conf(conf))


def test_window_models_take_pointwise_losses_only():
    from neurec_b200.model.sequential_recommender._base import SeqWindowRecommender
    m = SeqWindowRecommender.__new__(SeqWindowRecommender)
    for loss in ("bpr", "hinge", "nope"):
        m.loss_function = loss
        with pytest.raises(Exception, match="please choose a suitable loss function"):
            m._check_loss()
    for loss in ("cross_entropy", "Square"):
        m.loss_function = loss
        m._check_loss()
        assert m._loss == loss.lower()


# ------------------------------------------------------------------------------- restatement vs torch.autograd
def _point_loss(kind, z, x):      # util/learner.py:31-41
    if kind == "cross_entropy":
        return torch.nn.functional.binary_cross_entropy_with_logits(x, z, reduction="mean")
    return ((z - x) ** 2).sum()


def _l2(*ts):                     # util/tool.py:216-217
    return sum((t ** 2).sum() for t in ts) / 2


def _batch(rs, n, L, nu, ni):
    u, i = rs.randint(0, nu, n), rs.randint(0, ni, n)
    w = rs.randint(0, ni, (n, L))
    u[1] = u[0]                                        # a repeated user
    w[0, -1] = w[0, 0]                                 # an id twice in one window
    w[2, 0], i[3] = i[2], w[3, 0]                      # items that are both in a window and a target
    z = (rs.rand(n) < 0.3).astype(np.float32)
    return u, w, i, z


def _close(got, want):
    assert np.allclose(got, want, rtol=2e-5, atol=2e-6), np.abs(got - want).max()


def _hrm_autograd(P, E, u, w, i, z, pre_max, session_max, loss, reg):
    tp, te = T(P), T(E)
    R, p, e = te[I(w)], tp[I(u)], te[I(i)]
    s = torch.amax(R, 1) if session_max else R.mean(1)        # amax splits the gradient among ties, as TF does
    cat = torch.stack([p, s], 1)
    h = torch.amax(cat, 1) if pre_max else cat.mean(1)
    total = _point_loss(loss, torch.as_tensor(z, dtype=torch.float64), (h * e).sum(1)) + reg * _l2(p, R, e)
    total.backward()
    return float(total.detach()), (tp.grad.numpy(), te.grad.numpy())


@pytest.mark.parametrize("ties", [False, True])
@pytest.mark.parametrize("loss", LOSSES)
@pytest.mark.parametrize("pre_max,session_max", AGGS)
@pytest.mark.parametrize("L", [1, 3])
def test_hrm_grad_restatement_equals_autograd(L, pre_max, session_max, loss, ties):
    """HRM.py:62-91 as a torch float64 graph.  ties: integer-valued tables, so window maxima and P_u == s tie often
    (and exactly); the split must equal amax's."""
    rs = np.random.RandomState(L * 10 + ties)
    nu, ni, d, reg = 6, 9, 5, 0.03
    if ties:
        P, E = rs.randint(-2, 3, (nu, d)).astype(np.float32), rs.randint(-2, 3, (ni, d)).astype(np.float32)
    else:
        P, E = (rs.randn(nu, d) * 0.5).astype(np.float32), (rs.randn(ni, d) * 0.5).astype(np.float32)
    u, w, i, z = _batch(rs, 24, L, nu, ni)
    lo, grads, (tP, tE) = swm.hrm_grad(P, E, u, w, i, z, pre_max, session_max, loss, reg)
    want_l, want_g = _hrm_autograd(P, E, u, w, i, z, pre_max, session_max, loss, reg)
    assert abs(want_l - float(lo)) < 1e-5 * abs(want_l)
    for g, wg in zip(grads, want_g):
        _close(g, wg)
    if ties and session_max and L > 1:
        R = E[w]
        assert ((R == R.max(1, keepdims=True)).sum(1) > 1).any()          # the batch has split window maxima
    assert np.array_equal(np.flatnonzero(tP), np.unique(u))
    assert np.array_equal(np.flatnonzero(tE), np.unique(np.concatenate([w.reshape(-1), i])))


@pytest.mark.parametrize("ties", [False, True])
@pytest.mark.parametrize("loss", LOSSES)
@pytest.mark.parametrize("L", [2, 4])
def test_npe_grad_restatement_equals_autograd(L, loss, ties):
    """NPE.py:54-71 as a torch float64 graph.  ties: integer-valued tables put exact zeros at relu's input."""
    rs = np.random.RandomState(100 + L * 10 + ties)
    nu, ni, d, reg = 6, 9, 5, 0.05
    if ties:
        tabs = [rs.randint(-2, 3, (n, d)).astype(np.float32) for n in (nu, ni, ni)]
    else:
        tabs = [(rs.randn(n, d) * 0.5).astype(np.float32) for n in (nu, ni, ni)]
    u, w, i, z = _batch(rs, 24, L, nu, ni)
    lo, grads, (tU, tI, tL) = swm.npe_grad(*tabs, u, w, i, z, loss, reg)
    UI, IU, IL = (T(t) for t in tabs)
    a, q, R = UI[I(u)], IU[I(i)], IL[I(w)]
    c = R.sum(1)
    x = (torch.relu(a) * torch.relu(q) + torch.relu(q) * torch.relu(c)).sum(1)
    total = _point_loss(loss, torch.as_tensor(z, dtype=torch.float64), x) + reg * _l2(a, q, R)
    total.backward()
    assert abs(float(total.detach()) - float(lo)) < 1e-5 * abs(float(total.detach()))
    for g, t in zip(grads, (UI, IU, IL)):
        _close(g, t.grad.numpy())
    if ties:
        assert (tabs[0][u] == 0).any() and (c.detach().numpy() == 0).any()    # relu sees exact zeros
    assert np.array_equal(np.flatnonzero(tU), np.unique(u)) and np.array_equal(np.flatnonzero(tI), np.unique(i))
    assert np.array_equal(np.flatnonzero(tL), np.unique(w))


def test_hrm_at_one_recent_item_is_the_concat_branch():
    """HRM.py:75-77: at high_order = 1 the reference concatenates P_u with the recent row itself; pooling a window of
    one row is that row, so the two graphs agree (the window arrives as [batch])."""
    rs = np.random.RandomState(7)
    P, E = (rs.randn(5, 4) * 0.5).astype(np.float32), (rs.randn(8, 4) * 0.5).astype(np.float32)
    u, w, i, z = _batch(rs, 10, 1, 5, 8)
    for pre_max, session_max in AGGS:
        a = swm.hrm_grad(P, E, u, w, i, z, pre_max, session_max, "cross_entropy", 0.01)
        b = swm.hrm_grad(P, E, u, w[:, 0], i, z, pre_max, True, "cross_entropy", 0.01)
        assert a[0] == b[0] and all(np.array_equal(x, y) for x, y in zip(a[1], b[1]))


# ------------------------------------------------------------------------------------ predict windows
@pytest.mark.parametrize("L", [1, 2, 3, 4])
def test_predict_window_is_pythons_slice(L):
    """train_dict[u][len - L:] for every length 1..2L: the last L items, or seq[max(0, 2 len - L):] when len < L."""
    from neurec_b200.model.sequential_recommender._base import predict_windows
    seqs = {n - 1: list(range(100 + 10 * n, 100 + 10 * n + n)) for n in range(1, 2 * L + 1)}
    seqs[2 * L + 1] = []                                        # a user id the train dict does not hold
    recent, length = predict_windows({u: np.asarray(s) for u, s in seqs.items() if s}, 2 * L + 2, L)
    for u, seq in seqs.items():
        want = seq[len(seq) - L:] if seq else []
        assert want == swm.predict_window(seq, L)
        n = len(seq)
        assert len(want) == (L if n >= L else min(n, L - n))
        assert length[u] == len(want) and recent[u, :len(want)].tolist() == want
        assert not recent[u, len(want):].any()
    assert length[2 * L] == 0 and length[2 * L + 1] == 0


# ------------------------------------------------------------------------------------ ABI argument checks
def _lib():
    from neurec_b200 import _build, _lib as lib
    if not os.path.isfile(lib.LIB_PATH):
        _build.build()
    return lib


def test_abi_rejects_bad_loss_width_and_window_before_any_cuda_call():
    lib = _lib()
    L = lib.load()
    ce, bpr = lib.LOSS_IDS["cross_entropy"], lib.LOSS_IDS["bpr"]
    n = None

    def hrm(dim, window, loss):
        return L.nrc_hrm_grad(n, n, dim, window, n, n, n, n, 4, 1, 1, loss, 0.0, n, n, n, n, 1, n, n)

    def npe(dim, window, loss):
        return L.nrc_npe_grad(n, n, n, dim, window, n, n, n, n, 4, loss, 0.0, n, n, n, n, n, n, 1, n, n)

    def hrm_epoch(dim, window, loss):
        return L.nrc_hrm_train_epoch(n, n, 3, 5, dim, window, n, n, n, n, 8, 4, 1, 1, loss, 0.0, 1, n, n, n, n, n, n,
                                     n, n, 1, n, n)

    def npe_epoch(dim, window, loss):
        return L.nrc_npe_train_epoch(n, n, n, 3, 5, dim, window, n, n, n, n, 8, 4, loss, 0.0, 1, n, n, n, n, n, n, n,
                                     n, n, n, 1, n, n)

    for call in (hrm, npe, hrm_epoch, npe_epoch):
        for loss in (bpr, lib.LOSS_IDS["hinge"], 99):
            with pytest.raises(ValueError, match="please choose a suitable loss function"):
                lib.check(call(16, 2, loss))
        for dim, window in ((0, 2), (257, 2), (16, 0), (16, 65), (16, -1)):
            with pytest.raises(lib.NrcError) as e:
                lib.check(call(dim, window, ce))
            assert e.value.rc == lib.NRC_E_LIMIT
    for dim, window in ((0, 2), (257, 2), (16, 0), (16, 65)):
        for rc in (L.nrc_hrm_query(n, n, dim, window, n, 2, n, n, 1, 1, n, n),
                   L.nrc_npe_query(n, n, n, 10, dim, window, n, 2, n, n, n, n, n)):
            with pytest.raises(lib.NrcError) as e:
                lib.check(int(rc))
            assert e.value.rc == lib.NRC_E_LIMIT
