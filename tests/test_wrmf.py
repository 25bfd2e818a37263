"""WRMF (implicit-feedback ALS) without a GPU: the conf file, the model's registration, and the fp64 restatement of
the reference's dense formulation (model/general_recommender/WRMF.py:27-33,51-61) against the CSR form the kernel
computes.  The GPU tests (test_gpu_wrmf.py) use the CSR form below as their fp64 reference."""
import os
import sys

import numpy as np
import pytest

from conftest import ROOT, random_csr


def dense_als_epoch(X, Y, train_dense, alpha, reg):
    """WRMF.py:27-33 (Cui, Pui), 51-61 (one solve per row) and 74-85 (users, then items), literally, in fp64."""
    X, Y = X.astype(np.float64).copy(), Y.astype(np.float64).copy()
    num_users, num_items = train_dense.shape
    d = X.shape[1]
    Cui = np.zeros((num_users, num_items))
    Pui = np.zeros((num_users, num_items))
    Cui[train_dense] = alpha
    Pui[train_dense] = 1.0
    lambda_eye = reg * np.eye(d)
    for u in range(num_users):
        Cu, Pu = Cui[u].reshape([-1, 1]), Pui[u].reshape([-1, 1])
        YTY = Y.T @ Y
        YTCuIY = Y.T @ (Cu * Y)
        YTCupu = Y.T @ ((Cu + 1) * Pu)
        X[u] = np.linalg.solve(YTY + YTCuIY + lambda_eye, YTCupu)[:, 0]
    for i in range(num_items):
        Ci, Pi = Cui[:, i].reshape([-1, 1]), Pui[:, i].reshape([-1, 1])
        XTX = X.T @ X
        XTCIIX = X.T @ (Ci * X)
        XTCIpi = X.T @ ((Ci + 1) * Pi)
        Y[i] = np.linalg.solve(XTX + XTCIIX + lambda_eye, XTCIpi)[:, 0]
    return X, Y


def row_system(fixed64, G, indices, alpha, reg):
    """A = G + alpha sum y y^T + reg I and b = (1 + alpha) sum y over one CSR row, fp64."""
    Yr = fixed64[indices]
    A = G + alpha * (Yr.T @ Yr) + reg * np.eye(G.shape[0])
    b = (1.0 + alpha) * Yr.sum(axis=0)
    return A, b


def csr_half_step(fixed, indptr, indices, alpha, reg):
    """One half-step in the CSR form of nrc_wrmf_half_step, fp64 (fixed is widened from whatever it holds)."""
    Y = np.asarray(fixed, dtype=np.float64)
    G = Y.T @ Y
    out = np.zeros((len(indptr) - 1, Y.shape[1]))
    for r in range(len(indptr) - 1):
        A, b = row_system(Y, G, indices[indptr[r]:indptr[r + 1]], alpha, reg)
        out[r] = np.linalg.solve(A, b)
    return out


def transpose_csr(indptr, indices, num_cols):
    rows = np.repeat(np.arange(len(indptr) - 1, dtype=np.int32), np.diff(indptr))
    order = np.lexsort((rows, indices))
    tptr = np.zeros(num_cols + 1, np.int64)
    tptr[1:] = np.cumsum(np.bincount(indices, minlength=num_cols))
    return tptr, rows[order].astype(np.int32)


def objective(X, Y, indptr, indices, alpha, reg):
    """sum_ui c_ui (p_ui - x_u.y_i)^2 + reg (|X|^2 + |Y|^2), c = 1 + alpha on train entries and 1 elsewhere, in fp64
    without a dense matrix: sum over all (u, i) of s^2 is tr(X^T X Y^T Y), the train entries add c (1 - s)^2 - s^2."""
    X, Y = np.asarray(X, np.float64), np.asarray(Y, np.float64)
    rows = np.repeat(np.arange(len(indptr) - 1), np.diff(indptr))
    total = np.sum((X.T @ X) * (Y.T @ Y))
    for c in range(0, len(rows), 1 << 17):
        s = np.einsum("ij,ij->i", X[rows[c:c + (1 << 17)]], Y[indices[c:c + (1 << 17)]])
        total += np.sum((1.0 + alpha) * (1.0 - s) ** 2 - s ** 2)
    return total + reg * (np.sum(X * X) + np.sum(Y * Y))


def test_conf_parses_to_the_reference_values(tmp_path, monkeypatch):
    from neurec_b200.util import Configurator
    (tmp_path / "conf").mkdir()
    (tmp_path / "conf" / "WRMF.properties").write_text(open(os.path.join(ROOT, "conf", "WRMF.properties")).read())
    (tmp_path / "NeuRec.properties").write_text(open(os.path.join(ROOT, "NeuRec.properties")).read())
    monkeypatch.chdir(tmp_path)
    monkeypatch.setattr(sys, "argv", ["main.py", "--recommender=WRMF"])
    conf = Configurator("NeuRec.properties", default_section="hyperparameters")
    want = {"epochs": 300, "embedding_size": 16, "reg_mf": 0.1, "alpha": 10, "init_method": "uniform",
            "stddev": 0.01, "verbose": 1}
    for key, value in want.items():
        assert conf[key] == value and type(conf[key]) is type(value), key


def test_main_resolves_wrmf():
    import main
    from neurec_b200.model.general_recommender.WRMF import WRMF
    assert main.resolve_model("WRMF") is WRMF


@pytest.mark.parametrize("seed,num_users,num_items,d,alpha,reg", [
    (0, 13, 17, 4, 10.0, 0.1), (1, 9, 30, 7, 2.5, 0.01), (2, 20, 6, 8, 40.0, 1.0), (3, 5, 5, 3, 0.0, 0.5)])
def test_dense_reference_equals_csr_form(seed, num_users, num_items, d, alpha, reg):
    """The reference's dense Cui / Pui formulation and the CSR form agree to 1e-12 over a whole epoch, with empty
    users and items among the rows."""
    rs = np.random.RandomState(seed)
    ptr, idx = random_csr(rs, num_users, num_items, rs.randint(0, num_items // 2 + 1, num_users))
    train = np.zeros((num_users, num_items), bool)
    for u in range(num_users):
        train[u, idx[ptr[u]:ptr[u + 1]]] = True
    X0 = rs.uniform(-0.01, 0.01, (num_users, d))
    Y0 = rs.uniform(-0.5, 0.5, (num_items, d))
    Xd, Yd = dense_als_epoch(X0, Y0, train, alpha, reg)
    X = csr_half_step(Y0, ptr, idx, alpha, reg)
    tptr, tidx = transpose_csr(ptr, idx, num_items)
    Y = csr_half_step(X, tptr, tidx, alpha, reg)
    assert np.abs(Xd - X).max() <= 1e-12 * max(1.0, np.abs(Xd).max())
    assert np.abs(Yd - Y).max() <= 1e-12 * max(1.0, np.abs(Yd).max())
    assert np.all(X[np.diff(ptr) == 0] == 0) and np.all(Y[np.diff(tptr) == 0] == 0)
    # the objective the GPU tests track is the one both halves minimise
    f0 = objective(X0, Y0, ptr, idx, alpha, reg)
    f1 = objective(X, Y0, ptr, idx, alpha, reg)
    f2 = objective(X, Y, ptr, idx, alpha, reg)
    C = np.where(train, 1.0 + alpha, 1.0)
    dense = lambda X_, Y_: np.sum(C * (train - X_ @ Y_.T) ** 2) + reg * (np.sum(X_ ** 2) + np.sum(Y_ ** 2))
    assert abs(f2 - dense(X, Y)) <= 1e-10 * abs(dense(X, Y))
    assert f0 >= f1 >= f2
