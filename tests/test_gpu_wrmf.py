"""WRMF on the device (csrc/wrmf.cu, nrc_wrmf_half_step) against the fp64 CSR restatement of the reference's
model/general_recommender/WRMF.py:51-61 (tests/test_wrmf.py pins that restatement on the reference's dense form).

A half-step's fp32 result is judged by its normwise backward error against A and b formed in fp64 from the fp32
tables, under a bound derived from how the kernel sums (the Gram slices, each row's outer products and b) and from
Cholesky's backward error, and by its forward error against the fp64 solve within kappa_inf(A) times that bound."""
import os
import re
import subprocess
import sys

import numpy as np
import pytest
import scipy.sparse as sp
import torch

from conftest import ROOT, random_csr
from test_wrmf import objective, row_system, transpose_csr

pytestmark = pytest.mark.gpu
U32 = 2.0 ** -24
ALPHA, REG = 10.0, 0.1


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def gamma(n):
    return n * U32 / (1.0 - n * U32)


def gram_depth(num_fixed):
    """Additions each entry of Y^T Y goes through: one slice of rows (csrc/wrmf.cu gram_slices), then every slice."""
    if num_fixed == 0:
        return 0
    slices = min(256, (num_fixed + 127) // 128)
    return -(-num_fixed // slices) + slices


def half_step(fixed, ptr, idx, alpha=ALPHA, reg=REG, row_order=None, out=None):
    from neurec_b200 import ops
    fixed_d = fixed if isinstance(fixed, torch.Tensor) else dev(fixed)
    if out is None:
        out = torch.full((len(ptr) - 1, fixed_d.shape[1]), np.nan, dtype=torch.float32, device="cuda")
    ops.wrmf_half_step(fixed_d, dev(ptr), dev(idx), out, alpha, reg,
                       row_order=None if row_order is None else dev(row_order))
    return out.cpu().numpy()


def check_rows(fixed32, ptr, idx, got, alpha=ALPHA, reg=REG, rows=None):
    """Backward and forward error of every row of `got` (fp32) against the fp64 system; returns the largest
    backward error as a fraction of its bound.  Empty rows must be exactly 0."""
    Y = np.asarray(fixed32, np.float64)
    G, absG = Y.T @ Y, np.abs(Y).T @ np.abs(Y)
    depth_g = gram_depth(Y.shape[0])
    d = Y.shape[1]
    worst = 0.0
    for r in (range(len(ptr) - 1) if rows is None else rows):
        J = idx[ptr[r]:ptr[r + 1]]
        x = got[r].astype(np.float64)
        if len(J) == 0:
            assert np.all(got[r] == 0.0), r
            continue
        A, b = row_system(Y, G, J, alpha, reg)
        Yr = np.abs(Y[J])
        # |dA| from forming A in fp32: G's sums, the row's outer products, scaling by alpha, the two additions
        dA_form = gamma(depth_g + 3) * absG + alpha * gamma(len(J) + 3) * (Yr.T @ Yr) + U32 * reg * np.eye(d)
        db = gamma(len(J) + 2) * (1.0 + alpha) * Yr.sum(axis=0)
        # Cholesky factor and both triangular solves: (A + dA) x = b with |dA| <= gamma(3d + 1) |R^T| |R|
        R = np.linalg.cholesky(A)
        dA_chol = gamma(3 * d + 1) * (np.abs(R) @ np.abs(R).T)
        nx, nb, nA = np.abs(x).max(), np.abs(b).max(), np.abs(A).sum(axis=1).max()
        bound = (np.abs(dA_form + dA_chol).sum(axis=1).max() * nx + np.abs(db).max()) / (nA * nx + nb)
        eta = np.abs(A @ x - b).max() / (nA * nx + nb)
        assert eta <= bound, (r, eta, bound)
        worst = max(worst, eta / bound)
        x64 = np.linalg.solve(A, b)
        kappa = nA * np.abs(np.linalg.inv(A)).sum(axis=1).max()
        fwd = np.abs(x - x64).max() / np.abs(x64).max()
        # Higham, Thm 7.2: |dx| / |x| <= 2 kappa eps / (1 - kappa eps) for a backward error eps with kappa eps < 1
        limit = 2 * kappa * bound / (1 - kappa * bound) if kappa * bound < 0.5 else 4 * kappa * bound
        assert fwd <= limit, (r, fwd, kappa, bound)
    return worst


def _case(d, num_fixed, degrees, seed):
    rs = np.random.RandomState(seed)
    fixed = (rs.randn(num_fixed, d) * 0.1).astype(np.float32)
    if num_fixed == 0:
        degrees = np.zeros_like(degrees)
    ptr, idx = random_csr(rs, len(degrees), max(num_fixed, 1), degrees)
    return fixed, ptr, idx


DIMS = [1, 3, 16, 32, 33, 64, 100, 128]


@pytest.mark.parametrize("d", DIMS)
def test_half_step_against_fp64(d):
    """Rows of 0, 1 and >= 2000 entries over a fixed table of 40 000 rows, and rows over a table with fewer rows
    than d (Y^T Y singular, reg > 0 makes A definite)."""
    degrees = np.array([0, 1, 2400, 3000, 1, 0, 7, 64, 250, 2100] + [5, 40, 600] * 4)
    fixed, ptr, idx = _case(d, 40000, degrees, seed=d)
    got = half_step(fixed, ptr, idx)
    assert np.diff(ptr).max() >= 2000 and np.diff(ptr).min() == 0
    check_rows(fixed, ptr, idx, got)
    small = d // 2
    fixed, ptr, idx = _case(d, small, np.array([0, 1, small, 2, 0, 1]), seed=100 + d)
    got = half_step(fixed, ptr, idx, reg=0.5)
    check_rows(fixed, ptr, idx, got, reg=0.5)


@pytest.mark.parametrize("d", [3, 16, 64, 128])
def test_half_step_is_deterministic_and_row_independent(d):
    rs = np.random.RandomState(7)
    degrees = rs.randint(0, 400, 300)
    degrees[::37] = 2500
    fixed, ptr, idx = _case(d, 41000, degrees, seed=d + 1)
    a = half_step(fixed, ptr, idx)
    b = half_step(fixed, ptr, idx)
    assert np.array_equal(a.view(np.uint32), b.view(np.uint32))
    order = np.argsort(-np.diff(ptr), kind="stable").astype(np.int32)
    c = half_step(fixed, ptr, idx, row_order=order)
    assert np.array_equal(a.view(np.uint32), c.view(np.uint32))
    keep = rs.rand(300) < 0.3
    sub = [idx[ptr[r]:ptr[r + 1]] if keep[r] else idx[:0] for r in range(300)]
    sptr = np.cumsum([0] + [len(s) for s in sub]).astype(np.int64)
    s = half_step(fixed, sptr, np.concatenate(sub).astype(np.int32))
    assert np.array_equal(s[keep].view(np.uint32), a[keep].view(np.uint32))
    assert np.all(s[~keep] == 0.0)


@pytest.mark.parametrize("d", [16, 64])
def test_not_positive_definite_rows_raise_and_stay_unchanged(d):
    from neurec_b200 import ops
    from neurec_b200._lib import NrcError
    fixed = torch.zeros((50, d), dtype=torch.float32, device="cuda")
    rs = np.random.RandomState(0)
    ptr, idx = random_csr(rs, 9, 50, [0, 3, 10, 1, 0, 50, 2, 2, 8])
    out = torch.full((9, d), 7.0, device="cuda")
    with pytest.raises(NrcError, match=r"\b9 of 9 rows\b"):
        ops.wrmf_half_step(fixed, dev(ptr), dev(idx), out, ALPHA, 0.0)
    assert torch.all(out == 7.0)


def test_rejected_calls_write_nothing():
    from neurec_b200 import _lib, ops
    lib = _lib.load()
    fixed = torch.randn((64, 129), device="cuda")
    ptr = dev(np.array([0, 2, 3], np.int64)); idx = dev(np.array([1, 5, 9], np.int32))
    out = torch.full((2, 129), 3.0, device="cuda")
    not_spd = torch.full((1,), 12345, dtype=torch.int32, device="cuda")
    work = ops.wrmf_work(64, 128)
    p = lambda t: t.data_ptr()
    call = lambda dim, alpha, reg: lib.nrc_wrmf_half_step(p(fixed), 64, p(ptr), p(idx), None, 2, dim, alpha, reg,
                                                          p(out), p(work), p(not_spd), None)
    cases = [(0, ALPHA, REG, _lib.NRC_E_LIMIT), (129, ALPHA, REG, _lib.NRC_E_LIMIT), (-4, ALPHA, REG, _lib.NRC_E_LIMIT)]
    cases += [(16, a, REG, _lib.NRC_E_VALUE) for a in (-1.0, float("nan"), float("inf"))]
    cases += [(16, ALPHA, r, _lib.NRC_E_VALUE) for r in (-1e-3, float("nan"), float("inf"))]
    for dim, alpha, reg, code in cases:
        assert call(dim, alpha, reg) == code, (dim, alpha, reg)
        torch.cuda.synchronize()
        assert torch.all(out == 3.0) and int(not_spd.item()) == 12345, (dim, alpha, reg)
    with pytest.raises(ValueError):
        ops.wrmf_half_step(fixed[:, :16].contiguous(), ptr, idx, out[:, :16].contiguous(), -1.0, REG)


def _initial_tables(num_users, num_items, d):
    from neurec_b200.model._engine import get_initializer
    init = get_initializer("uniform", 0.01, torch.Generator().manual_seed(2017))
    return init([num_users, d]).numpy(), init([num_items, d]).numpy()


@pytest.mark.parametrize("d", [16, 64])
def test_objective_never_increases_over_five_epochs(ml100k, d):
    """Each half-step is the exact minimiser over its table, so the fp64 objective of the fp32 tables cannot rise.
    Slack: 1e-7 of the objective, far above what rounding a minimiser to fp32 can add (second order in its error)
    and far below one half-step's decrease here."""
    g = ml100k
    ptr, idx = g["train_indptr"], g["train_indices"]
    tptr, tidx = transpose_csr(ptr, idx, g["num_items"])
    X, Y = _initial_tables(g["num_users"], g["num_items"], d)
    f = [objective(X, Y, ptr, idx, ALPHA, REG)]
    Xd, Yd = dev(X), dev(Y)
    for _ in range(5):
        half_step(Yd, ptr, idx, out=Xd)
        f.append(objective(Xd.cpu().numpy(), Y, ptr, idx, ALPHA, REG))
        half_step(Xd, tptr, tidx, out=Yd)
        Y = Yd.cpu().numpy()
        f.append(objective(Xd.cpu().numpy(), Y, ptr, idx, ALPHA, REG))
    f = np.array(f)
    assert np.all(f[1:] <= f[:-1] + 1e-7 * f[:-1]), f
    assert f[-1] < 0.5 * f[0]


@pytest.mark.parametrize("d", [16, 64])
def test_one_epoch_against_fp64_als(ml100k, d):
    """Both halves of the first epoch from the plug-in's initial item table, each against the fp64 solve of the
    same system (the item half's fixed table is the user table the device wrote)."""
    g = ml100k
    ptr, idx = g["train_indptr"], g["train_indices"]
    tptr, tidx = transpose_csr(ptr, idx, g["num_items"])
    _, Y0 = _initial_tables(g["num_users"], g["num_items"], d)
    X = half_step(Y0, ptr, idx)
    check_rows(Y0, ptr, idx, X)
    Y = half_step(X, tptr, tidx)
    check_rows(X, tptr, tidx, Y)


def test_gowalla_epoch_decreases_the_objective(gowalla):
    g = gowalla
    ptr, idx = g["train_indptr"], g["train_indices"]
    tptr, tidx = transpose_csr(ptr, idx, g["num_items"])
    X, Y = _initial_tables(g["num_users"], g["num_items"], 64)
    f0 = objective(X, Y, ptr, idx, ALPHA, REG)
    X1 = half_step(Y, ptr, idx)
    Y1 = half_step(X1, tptr, tidx)
    assert np.isfinite(X1).all() and np.isfinite(Y1).all()
    f1 = objective(X1, Y, ptr, idx, ALPHA, REG)
    f2 = objective(X1, Y1, ptr, idx, ALPHA, REG)
    assert f2 <= f1 < f0
    rows = np.argsort(-np.diff(ptr))[:3].tolist() + [0, 1, 2]                 # the heaviest users and a few others
    check_rows(Y, ptr, idx, X1, rows=rows)


# ------------------------------------------------------------------------------------------------ plug-in
class _Conf(dict):
    def params_str(self):
        return "test"


CONF = {"metric": ["Precision", "Recall", "NDCG", "MAP", "MRR"], "group_view": None, "topk": [10, 20],
        "test_batch_size": 128, "num_thread": 8, "recommender": "WRMF", "embedding_size": 16, "alpha": 10,
        "epochs": 3, "reg_mf": 0.1, "init_method": "uniform", "stddev": 0.01, "verbose": 1}


def _model(ml100k):
    from neurec_b200.data import Dataset
    from neurec_b200.model.general_recommender.WRMF import WRMF
    d = ml100k
    shape = (d["num_users"], d["num_items"])
    mk = lambda p, i: sp.csr_matrix((np.ones(len(d[i]), np.float32), d[i], d[p]), shape=shape)
    ds = Dataset.from_csr("ml-100k", mk("train_indptr", "train_indices"), mk("test_indptr", "test_indices"))
    m = WRMF(None, ds, _Conf(CONF))
    m.build_graph()
    return m


def test_plug_in_predict_and_checkpoint_resume(ml100k, tmp_path, monkeypatch):
    from neurec_b200.util import checkpoint
    monkeypatch.chdir(tmp_path)
    a = _model(ml100k)
    a._train_epoch()
    U, V = a.user_embeddings.cpu().numpy(), a.item_embeddings.cpu().numpy()
    users = [0, 5, 17, 942]
    want = U[users] @ V.T
    got = a.predict(users)
    assert np.abs(got - want).max() <= 1e-5 * np.abs(want).max()
    cand = [[1, 2, 3], [10], [0, 1681], [5, 5, 7]]
    for r, w, c in zip(a.predict(users, cand), want, cand):
        assert np.abs(np.asarray(r) - w[c]).max() <= 1e-5 * np.abs(want).max()
    a._train_epoch()
    path = str(tmp_path / "wrmf.ckpt")
    checkpoint.save(a, path)
    a._train_epoch()
    b = _model(ml100k)
    assert not torch.equal(a.item_embeddings, b.item_embeddings)
    checkpoint.load(b, path)
    b._train_epoch()
    assert torch.equal(a.user_embeddings, b.user_embeddings) and torch.equal(a.item_embeddings, b.item_embeddings)


def test_main_runs_wrmf(tmp_path):
    from test_surface import _write_synthetic_dataset
    data = tmp_path / "dataset"
    _write_synthetic_dataset(str(data))
    cmd = [sys.executable, os.path.join(ROOT, "main.py"), "--data.input.path=%s" % data, "--data.input.dataset=toy",
           "--topk=[5,10]", "--test_batch_size=64", "--recommender=WRMF", "--epochs=3"]
    for name in ("NeuRec.properties", "conf"):
        os.symlink(os.path.join(ROOT, name), tmp_path / name)
    r = subprocess.run(cmd, cwd=tmp_path, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    out = r.stdout
    assert "metrics:\tPrecision@5 " in out and "NDCG@10" in out
    assert [int(e) for e in re.findall(r"iteration (\d+) finished in [0-9.]+ seconds", out)] == [1, 2, 3]
    epochs = re.findall(r"epoch (\d+):\t([0-9.\t ]+)", out)
    assert [int(e[0]) for e in epochs] == [1, 2, 3]
    vals = np.array([[float(x) for x in e[1].split()] for e in epochs])
    assert vals.shape[1] == 10 and np.isfinite(vals).all() and (vals >= 0).all() and (vals <= 1).all()
    assert vals[-1, 4] > vals[0, 4]                                            # NDCG@5 improves
