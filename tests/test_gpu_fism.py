"""GPU parity of FISM (csrc/fism.cu) through the C ABI against the restatement in tests/fism_math.py: the gradient
kernel on every route its shapes select (nrc_fism_last_routes), bit for bit on dyadic inputs at alpha = 0 and within a
first-order bound otherwise; one ml-100k epoch per mode under all five optimizers; the query and scores; argument
errors; the plug-in with a checkpoint restore; main.py in both modes."""
import os
import re
import subprocess
import sys

import numpy as np
import pytest
import scipy.sparse as sp
import torch

import fism_math as fm
from oracle import tf_math
from test_gpu_sequential import BASE_CONF, _Conf, dev, host, write_timed_dataset

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")
REACHED = set()
U = 2.0 ** -24
CONF = dict(recommender="FISM", epochs=1, batch_size=256, embedding_size=16, regs=[0.0001, 0.0001], alpha=0.5,
            learning_rate=0.001, learner="adam", is_pairwise=False, num_neg=4, loss_function="square",
            init_method="normal", stddev=0.01, verbose=1)
LR = {"adam": 1e-3, "gd": 1e-3, "adagrad": 1e-2, "rmsprop": 1e-3, "momentum": 1e-3}


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _lanes(d):
    vec = 4 if d % 4 == 0 else 1
    lpr = 1
    while lpr < d // vec and lpr < 32:
        lpr <<= 1
    return vec, lpr


def _ml100k():
    z = np.load(os.path.join(GOLDEN, "ml100k_split.npz"))
    return (z["train_indptr"].astype(np.int64), z["train_indices"].astype(np.int32), int(z["num_users"]),
            int(z["num_items"]))


def _dyadic(rs, shape, scale=0.5, density=0.2):
    return (rs.randint(-2, 3, shape) * (rs.rand(*shape) < density) * scale).astype(np.float32)


def _history_csr(rs, ni, lengths):
    rows = [np.sort(rs.choice(ni, n, replace=False)) for n in lengths]
    ptr = np.zeros(len(rows) + 1, np.int64)
    ptr[1:] = np.cumsum(lengths)
    return ptr, (np.concatenate(rows) if rows else np.zeros(0)).astype(np.int32)


def _batch(rs, ptr, idx, ni, B, pairwise):
    nrows = len(ptr) - 1
    deg = np.diff(ptr)
    rows = rs.randint(0, nrows, B).astype(np.int32)
    rows[:min(B, 2)] = np.argmax(deg)                                   # the longest history, twice
    items = rs.randint(0, ni, B).astype(np.int32)
    if pairwise:
        excl = None
        third = rs.randint(0, ni, B).astype(np.int32)
        num = (deg[rows] + 1).astype(np.int32)
        num_neg = (num + 1).astype(np.int32)
    else:
        excl = np.full(B, -1, np.int32)
        has = deg[rows] > 0
        pick = ptr[rows] + rs.randint(0, 1 << 30, B) % np.maximum(deg[rows], 1)
        sel = np.flatnonzero(has)[::2]                                  # positives: the target left out of its row
        excl[sel] = idx[pick[sel]]
        items[sel] = excl[sel]
        third = (rs.rand(B) < 0.3).astype(np.float32)
        num = np.maximum(deg[rows], 1).astype(np.int32)
        num_neg = None
    return rows, excl, num, items, third, num_neg


def _run_grad(c1, Q, b, ptr, idx, batch, pairwise, loss, alpha, lam, gamma):
    from neurec_b200 import ops
    rows, excl, num, items, third, num_neg = batch
    z = lambda a: torch.zeros(a.shape, dtype=torch.float32, device="cuda")
    grads = [z(c1), z(Q), z(b)]
    touched = (torch.zeros(len(Q), dtype=torch.int32, device="cuda"),
               torch.zeros(len(Q), dtype=torch.int32, device="cuda"))
    lo = torch.zeros(1, device="cuda")
    d = lambda a: None if a is None else dev(a)
    ops.fism_grad(dev(c1), dev(Q), dev(b), dev(ptr), dev(idx), dev(rows), d(excl), dev(num), dev(items), dev(third),
                  d(num_neg), pairwise, loss, alpha, lam, gamma, grads, touched, 7, lo)
    torch.cuda.synchronize()
    return float(lo), [host(g) for g in grads], [host(t) == 7 for t in touched]


# d, pairwise, loss, B (None: both sides of 64 * SMs), lengths: 1 .. 590 (the longest ml-100k row)
ROUTE_CASES = [
    (1, False, "square"), (3, True, "square"), (16, False, "square"), (16, True, "hinge"), (50, True, "square"),
    (64, False, "square"), (128, True, "square"), (256, False, "square"), (256, True, "hinge"),
]


@pytest.mark.parametrize("capped", [False, True])
@pytest.mark.parametrize("d,pairwise,loss", ROUTE_CASES)
def test_grad_exact_on_dyadic_inputs(d, pairwise, loss, capped):
    """alpha = 0 (powf(n, -0) = 1 exactly) and dyadic tables: every product and partial sum is exact in fp32, so the
    kernel's gradients equal the float64 restatement bit for bit in any summation order."""
    rs = np.random.RandomState(d * 7 + capped)
    ni = 4096
    lengths = np.concatenate([[590, 1, 0, 2, 31, 32, 33, 97], rs.randint(1, 60, 56)])
    ptr, idx = _history_csr(rs, ni, lengths)
    cap = 64 * _sms()
    B = cap + 37 if capped else 200
    c1, Q, b = _dyadic(rs, (ni, d)), _dyadic(rs, (ni, d)), _dyadic(rs, (ni,), 0.5, 0.5)
    batch = _batch(rs, ptr, idx, ni, B, pairwise)
    lam, gamma = 0.5, 0.25
    got_l, got, (tC, tI) = _run_grad(c1, Q, b, ptr, idx, batch, pairwise, loss, 0.0, lam, gamma)
    want_l, want, (wC, wI) = fm.loss_and_grad(c1, Q, b, ptr, idx, *batch[:5], batch[5], pairwise, loss, 0.0, lam,
                                              gamma, dtype=np.float64)
    for name, g, w in zip(("c1", "Q", "b"), got, want):
        assert np.array_equal(g.astype(np.float64), w), name
    assert np.array_equal(tC, wC) and np.array_equal(tI, wI)
    assert abs(got_l - want_l) <= (B + 64) * U * max(1.0, abs(want_l))       # every loss term is >= 0
    from neurec_b200 import ops
    r = ops.fism_last_routes()["grad"]
    vec, lpr = _lanes(d)
    blocks = (B + 1) // 2
    assert r == dict(pairwise=int(pairwise), vec=vec, lanes=lpr, grid_x=min(blocks, cap // 2), grid_y=-1,
                     capped=int(blocks > cap // 2))
    REACHED.add(("grad", vec, lpr, pairwise, bool(r["capped"])))


@pytest.mark.parametrize("pairwise,loss", [(True, "bpr"), (True, "square"), (False, "cross_entropy"),
                                           (False, "square")])
@pytest.mark.parametrize("d", [5, 16, 256])
def test_grad_rounded_within_bound(d, pairwise, loss):
    """alpha = 0.5 on Gaussian tables against float64: within 2 * 2^-24 * M, M = (the longest add chain + 8) times
    the largest magnitude of the compared array, plus powf's documented 4-ulp error carried through the score into
    the loss derivative."""
    rs = np.random.RandomState(d + 3 * len(loss))
    ni = 1024
    lengths = np.concatenate([[590, 1, 2, 33], rs.randint(1, 200, 60)])
    ptr, idx = _history_csr(rs, ni, lengths)
    c1, Q = (rs.randn(ni, d) * 0.05).astype(np.float32), (rs.randn(ni, d) * 0.05).astype(np.float32)
    b = (rs.randn(ni) * 0.05).astype(np.float32)
    B = 300
    batch = _batch(rs, ptr, idx, ni, B, pairwise)
    got_l, got, _ = _run_grad(c1, Q, b, ptr, idx, batch, pairwise, loss, 0.5, 1e-3, 2e-3)
    want_l, want, _ = fm.loss_and_grad(c1, Q, b, ptr, idx, *batch[:5], batch[5], pairwise, loss, 0.5, 1e-3, 2e-3,
                                       dtype=np.float64)
    K = 590 + d + B
    slope = {"bpr": 0.25, "square": 2.0, "cross_entropy": 0.25 / B}[loss]
    p = np.abs(fm.query(np.abs(c1), ptr, idx, batch[0]))
    x_abs = float((p * np.abs(Q[batch[3]])).sum(1).max() + np.abs(b).max())
    for name, g, w in zip(("c1", "Q", "b"), got, want):
        scale = float(np.abs(w).max())
        tol = 2 * U * (K + 8) * scale * (1 + slope * x_abs)
        err = float(np.abs(g.astype(np.float64) - w).max())
        assert err <= tol, (name, err, tol)
    assert abs(got_l - want_l) <= 2 * U * (K + 8) * max(1.0, abs(want_l)) * (1 + slope * x_abs)
    from neurec_b200 import ops
    r = ops.fism_last_routes()["grad"]
    REACHED.add(("grad", r["vec"], r["lanes"], pairwise, bool(r["capped"])))


def _epoch_inputs(ptr, idx, ni, pairwise, epoch, seed=2018):
    """One epoch of the plug-in's layout with the device's negatives and order (nrc_sample_negatives,
    nrc_shuffle_perm), as host arrays for the restatement and device arrays for the kernel."""
    from neurec_b200 import ops
    from neurec_b200.model.general_recommender.FISM import pairwise_layout, pointwise_layout
    sorted_idx = np.concatenate([np.sort(idx[ptr[u]:ptr[u + 1]]) for u in range(len(ptr) - 1)]).astype(np.int32)
    if pairwise:
        (hp, hi), (rows, items, num, num_neg) = pairwise_layout(ptr, idx)
        neg = host(ops.sample_negatives(dev(ptr), dev(sorted_idx), dev(rows), 1, ni, seed, epoch)).reshape(-1)
        arrs = [rows, None, num, items, neg, num_neg]
    else:
        hp, hi = ptr, idx
        rows, excl, num, labels = pointwise_layout(ptr, idx, 4)
        pos_users = np.repeat(np.arange(len(ptr) - 1, dtype=np.int32), np.diff(ptr))
        neg = host(ops.sample_negatives(dev(ptr), dev(sorted_idx), dev(pos_users), 4, ni, seed, epoch))
        items = np.concatenate([neg, idx[:, None]], 1).reshape(-1)
        arrs = [rows, excl, num, items, labels, None]
    perm = host(ops.shuffle_perm(len(rows), seed, epoch))
    return (hp, hi), [None if a is None else np.ascontiguousarray(a[perm]) for a in arrs]


@pytest.mark.parametrize("opt", ["adam", "gd", "adagrad", "rmsprop", "momentum"])
@pytest.mark.parametrize("pairwise,loss", [(False, "square"), (True, "bpr")])
def test_epoch_vs_restatement_on_ml100k(pairwise, loss, opt):
    """One nrc_fism_train_epoch on the ml-100k train CSR (pointwise: 401 835 samples, 1 570 steps; pairwise: 40 381
    samples, 158 steps) against FISMTrainer fed the same negatives and order."""
    from neurec_b200 import ops
    ptr, idx, nu, ni = _ml100k()
    (hp, hi), arrs = _epoch_inputs(ptr, idx, ni, pairwise, epoch=9)
    rs = np.random.RandomState(3)
    c1, Q = (rs.randn(ni, 16) * 0.01).astype(np.float32), (rs.randn(ni, 16) * 0.01).astype(np.float32)
    b = np.zeros(ni, np.float32)
    lr, bs = LR[opt], 256
    tr = fm.FISMTrainer(c1, Q, b, opt, lr, loss, 0.5, 1e-4, 1e-4, pairwise)
    want = tr.epoch(hp, hi, *arrs[:5], arrs[5], bs)
    n = len(arrs[0])
    steps = (n + bs - 1) // bs
    assert steps == (158 if pairwise else 1570)
    dv = [dev(c1), dev(Q), dev(b)]
    grads = [torch.zeros_like(v) for v in dv]
    i0, i1 = tf_math.SLOT_INIT[opt]
    mk = lambda v, val: None if val is None else torch.full_like(v, val)
    s0, s1 = [mk(v, i0) for v in dv], [mk(v, i1) for v in dv]
    touched = (torch.zeros(ni, dtype=torch.int32, device="cuda"), torch.zeros(ni, dtype=torch.int32, device="cuda"))
    step_loss = torch.zeros(steps, device="cuda")
    d = lambda a: None if a is None else dev(a)
    got_steps = ops.fism_train_epoch(*dv, dev(hp), dev(hi), *[d(a) for a in arrs], bs, pairwise, loss, 0.5, 1e-4,
                                     1e-4, opt, tf_math.adam_lr_t(lr, steps), tf_math.DEFAULT_HYPER[opt](lr), grads,
                                     touched, s0, s1, 1, step_loss)
    assert got_steps == steps
    got_loss = host(step_loss).astype(np.float64)
    assert np.abs(got_loss - want).max() <= 2e-3 * np.abs(want).max(), np.abs(got_loss - want).max()
    for name, v, ref in zip(("c1", "Q", "b"), dv, tr.vars):
        err = np.abs(host(v) - ref).max()
        assert err <= 2e-3 * max(np.abs(ref).max(), 1e-3), (name, err)
    for g in grads:
        assert not g.any()                                              # the optimizer launch zeroes them


@pytest.mark.parametrize("d", [1, 7, 16, 64, 256])
def test_query_and_scores_vs_fp64(d):
    """p_u over each whole row and n^(-alpha) <p_u, Q_j> + b_j over the catalogue, both sides of the query's grid
    cap, against float64."""
    from neurec_b200 import ops
    ptr, idx, nu, ni = _ml100k()
    rs = np.random.RandomState(d)
    c1, Q = (rs.randn(ni, d) * 0.1).astype(np.float32), (rs.randn(ni, d) * 0.1).astype(np.float32)
    b = (rs.randn(ni) * 0.1).astype(np.float32)
    for users in (np.array([0, 5, 17, 942, 5], np.int32),
                  rs.randint(0, nu, 64 * _sms() + 9).astype(np.int32)):
        q = ops.fism_query(dev(c1), dev(ptr), dev(idx), dev(users))
        want_q = fm.query(c1, ptr, idx, users)
        K = int(np.diff(ptr).max())
        env = fm.query(np.abs(c1), ptr, idx, users)
        assert (np.abs(host(q) - want_q) <= 2 * U * K * env + 1e-30).all()
        r = ops.fism_last_routes()["query"]
        vec, lpr = _lanes(d)
        assert r["vec"] == vec and r["lanes"] == lpr
        REACHED.add(("query", bool(r["capped"])))
        s = host(ops.fism_scores(dev(c1), dev(Q), dev(b), dev(ptr), dev(idx), dev(users), 0.5))
        want = fm.scores(c1, Q, b, ptr, idx, users, 0.5)
        n = np.diff(ptr)[users].astype(np.float64)[:, None]
        bound = 2 * U * (K + d + 8) * (n ** -0.5 * (env @ np.abs(Q.astype(np.float64)).T) + np.abs(b)[None, :])
        assert (np.abs(s - want) <= bound).all(), np.abs(s - want).max()
        r = ops.fism_last_routes()["scores"]
        assert r["grid_x"] == (len(users) + 7) // 8 and r["grid_y"] == (ni + 255) // 256 and r["vec"] == vec
        REACHED.add(("scores", vec))


def test_argument_errors_on_device_tensors():
    from neurec_b200 import _lib, ops
    ptr, idx, nu, ni = _ml100k()
    c1 = torch.zeros(ni, 300, device="cuda")
    with pytest.raises(_lib.NrcError) as e:
        ops.fism_query(c1, dev(ptr), dev(idx), dev(np.arange(3, dtype=np.int32)))
    assert e.value.rc == _lib.NRC_E_LIMIT
    with pytest.raises(TypeError):
        ops.fism_query(torch.zeros(ni, 16, device="cuda"), dev(ptr.astype(np.int32)), dev(idx),
                       dev(np.arange(3, dtype=np.int32)))
    Q = torch.ones(ni, 16, device="cuda")
    grads = [torch.zeros(ni, 16, device="cuda"), torch.zeros(ni, 16, device="cuda"), torch.zeros(ni, device="cuda")]
    touched = (torch.zeros(ni, dtype=torch.int32, device="cuda"), torch.zeros(ni, dtype=torch.int32, device="cuda"))
    r = dev(np.zeros(4, np.int32))
    with pytest.raises(ValueError, match="suitable loss"):
        ops.fism_grad(Q, Q, grads[2], dev(ptr), dev(idx), r, None, r, r, r, r, True, "cross_entropy", 0.5, 0.0, 0.0,
                      grads, touched, 1)
    with pytest.raises(ValueError, match="alpha"):
        ops.fism_grad(Q, Q, grads[2], dev(ptr), dev(idx), r, None, r, r, torch.zeros(4, device="cuda"), None, False,
                      "square", float("inf"), 0.0, 0.0, grads, touched, 1)
    torch.cuda.synchronize()
    assert not any(g.any() for g in grads) and not any(t.any() for t in touched)


def _dataset():
    from neurec_b200.data import Dataset
    ptr, idx, nu, ni = _ml100k()
    z = np.load(os.path.join(GOLDEN, "ml100k_split.npz"))
    mk = lambda p, i: sp.csr_matrix((np.ones(len(i), np.float32), i.astype(np.int32), p.astype(np.int64)),
                                    shape=(nu, ni))
    return Dataset.from_csr("ml-100k", mk(ptr, idx), mk(z["test_indptr"], z["test_indices"]))


def _plug_in(ds, **over):
    from neurec_b200.model.general_recommender.FISM import FISM
    m = FISM(None, ds, _Conf(BASE_CONF, **dict(CONF, **over)))
    m.build_graph()
    return m


@pytest.mark.parametrize("pairwise", [False, True])
def test_plug_in_epoch_predict_evaluate_and_checkpoint(tmp_path, monkeypatch, pairwise):
    from neurec_b200.data import sampler as smp
    from neurec_b200.model._engine import get_initializer
    from neurec_b200.util import checkpoint
    monkeypatch.chdir(tmp_path)
    ds = _dataset()
    ptr, idx, nu, ni = _ml100k()
    over = dict(is_pairwise=True, loss_function="bpr") if pairwise else {}
    m = _plug_in(ds, **over)
    g = torch.Generator().manual_seed(2017)
    init = get_initializer("normal", 0.01, g)
    assert torch.equal(m.c1.cpu(), init([ni, 16])) and torch.equal(m.embedding_Q.cpu(), init([ni, 16]))
    assert not m.bias.any()
    start = [host(t).copy() for t in m.tables()]
    smp.reseed(21)
    total = m._train_epoch()
    (hp, hi), arrs = _epoch_inputs(ptr, idx, ni, pairwise, 21)
    tr = fm.FISMTrainer(*start, "adam", 1e-3, "bpr" if pairwise else "square", 0.5, 1e-4, 1e-4, pairwise)
    want = tr.epoch(hp, hi, *arrs[:5], arrs[5], 256)
    assert abs(total - float(want.sum())) <= 2e-3 * abs(float(want.sum()))
    for t, ref in zip(m.tables(), tr.vars):
        assert np.abs(host(t) - ref).max() <= 2e-3 * max(np.abs(ref).max(), 1e-3)
    users = [0, 5, 17, 942]
    tabs = [host(t) for t in m.tables()]
    got = m.predict(users)
    assert isinstance(got, torch.Tensor) and got.is_cuda and got.shape == (4, ni)
    want_s = fm.scores(*tabs, ptr, idx, np.array(users), 0.5)
    assert np.abs(host(got) - want_s).max() <= 1e-5 * max(1.0, np.abs(want_s).max())
    cand = [[1, 2, 3], [10], [0, 1681], [5, 5, 7]]
    for r, w, c in zip(m.predict(users, cand), host(got), cand):
        assert isinstance(r, np.ndarray) and np.array_equal(r, w[c])
    with pytest.raises(KeyError):
        m.predict([0, nu + 5])
    vals = [float(x) for x in m.evaluate().split()]
    assert len(vals) == 10 and all(0.0 <= v <= 1.0 for v in vals)
    # checkpoint: the resumed model draws the same epoch (negatives and order) bit for bit, and its epoch loss is
    # the continuing run's within the bound of reordered fp32 sums
    path = str(tmp_path / "fism.ckpt")
    checkpoint.save(m, path)
    next_epoch = smp._EPOCH_COUNTER.value
    ea = [None if a is None else host(a) for a in m.device_epoch(next_epoch)]
    la = m._train_epoch()
    smp.reseed(0)
    b = _plug_in(ds, **over)
    checkpoint.load(b, path)
    assert smp._EPOCH_COUNTER.value == next_epoch
    eb = [None if a is None else host(a) for a in b.device_epoch(next_epoch)]
    for x, y in zip(ea, eb):
        assert (x is None and y is None) or np.array_equal(x, y)
    lb = b._train_epoch()
    assert abs(la - lb) <= 1e-4 * abs(la)


@pytest.mark.parametrize("pairwise", [False, True])
def test_main_runs_fism(tmp_path, pairwise):
    data = tmp_path / "dataset"
    write_timed_dataset(str(data))
    cmd = [sys.executable, os.path.join(ROOT, "main.py"), "--recommender=FISM", "--data.input.path=%s" % data,
           "--data.input.dataset=toy", "--topk=[5,10]", "--test_batch_size=64", "--epochs=2"]
    if pairwise:
        cmd += ["--is_pairwise=True", "--loss_function=bpr"]
    for f in ("NeuRec.properties", "conf"):
        os.symlink(os.path.join(ROOT, f), tmp_path / f)
    r = subprocess.run(cmd, cwd=tmp_path, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    out = r.stdout
    assert "metrics:\tPrecision@5 " in out and "NDCG@10" in out
    epochs = re.findall(r"epoch (\d+):\t([0-9.\t ]+)", out)
    assert [int(e[0]) for e in epochs] == [1, 2]
    vals = np.array([[float(x) for x in e[1].split()] for e in epochs])
    assert vals.shape[1] == 10 and np.isfinite(vals).all() and (vals >= 0).all() and (vals <= 1).all()
    losses = re.findall(r"\[iter (\d+) : loss : ([0-9.eE+-]+), time: [0-9.]+\]", out)
    assert [int(e[0]) for e in losses] == [1, 2] and all(np.isfinite(float(e[1])) for e in losses)


def test_every_route_was_reached():
    """Runs last in this file: the gradient kernel with float4 and scalar loads, one and several rows per warp load,
    both modes, capped and not; the query kernel capped and not; the score kernel with both load widths."""
    if len(REACHED) == 0:
        pytest.skip("the route tests did not run in this session")
    grads = {r for r in REACHED if r[0] == "grad"}
    assert {r[1] for r in grads} == {1, 4}
    assert {r[2] for r in grads} >= {1, 4, 16, 32}
    assert {r[3] for r in grads} == {True, False} and {r[4] for r in grads} == {True, False}
    assert ("query", True) in REACHED and ("query", False) in REACHED
    assert ("scores", 1) in REACHED and ("scores", 4) in REACHED
