"""GPU parity of FPMCplus (csrc/sequential.cu) through the C ABI against the restatement in tests/fpmcplus_math.py:
the gradient kernels on every route their shapes select (nrc_fpmcplus_last_routes), bit-identical dense gradients,
one fused epoch per optimizer on the time-ordered ml-100k train set, the scores against fp64 (full and short windows,
and exp's overflow), argument errors, the plug-in (epoch, predict, evaluate, checkpoint) and main.py."""
import os
import re
import subprocess
import sys

import numpy as np
import pytest
import torch

import fpmcplus_math as fpm
from oracle import tf_math
from test_gpu_seq_window import _short_history_dataset
from test_gpu_sequential import BASE_CONF, _Conf, dev, host, ml100k_time_ordered, write_timed_dataset

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

MODES = [(True, "bpr"), (True, "hinge"), (True, "square"), (False, "cross_entropy"), (False, "square")]
LR = {"adam": 1e-3, "gd": 0.02, "adagrad": 0.01, "rmsprop": 1e-3, "momentum": 0.01}
EPS = 2.0 ** -24
REACHED = set()


@pytest.fixture(scope="module")
def ml100k_seq():
    return ml100k_time_ordered()


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _vars(rs, nu, ni, d, w, scale=0.3):
    tabs = [(rs.randn(n, d) * scale).astype(np.float32) for n in (nu, ni, ni, ni)]
    return tabs + [(rs.randn(3 * d, w) * (1.0 / np.sqrt(d))).astype(np.float32),
                   (rs.randn(1, w) * 0.3).astype(np.float32), (rs.randn(w, 1) * 0.5 + 1.0).astype(np.float32)]


def _batch(rs, n, L, nu, ni, pairwise):
    u, i = rs.randint(0, nu, n).astype(np.int32), rs.randint(0, ni, n).astype(np.int32)
    win = rs.randint(0, ni, (n, L)).astype(np.int32)
    if n > 6:
        u[1] = u[0]
        win[0, -1] = win[0, 0]
        win[2, 0], i[3] = i[2], win[3, 0]
    third = rs.randint(0, ni, n).astype(np.int32) if pairwise else (rs.rand(n) < 0.3).astype(np.float32)
    return u, win, i, third


def _touched(nu, ni):
    z = lambda n: torch.zeros(n, dtype=torch.int32, device="cuda")
    return (z(nu), z(ni), z(ni))


def _grad_bound(tabs, u, win, i, third, pairwise, loss, d, w, L):
    """A first-order bound on the fp32 rounding of one batch, from the same graph on absolute values in fp64: each
    score is a (d + L + 4)-term chain over terms of size M_x, and each energy a (d + w + 4)-term chain through tanh
    (|tanh'| <= 1) over terms of size M_e; an energy error moves the score by at most 2 max|q| per unit.  Gradients
    carry the same relative rounding of their own terms, so they are compared relative to the largest entry."""
    t = [np.abs(v.astype(np.float64)) for v in tabs]
    UI, IU, IL, LI, W, b, h = t
    R = LI[win]
    ids = [i] + ([third] if pairwise else [])
    tot = 0.0
    for item in ids:
        m_x = (UI[u] * IU[item]).sum(1) + (IL[item][:, None, :] * R).sum(2).max(1)
        pre = (UI[u] @ W[:d] + b)[:, None, :] + (IL[item] @ W[d:2 * d])[:, None, :] + R @ W[2 * d:]
        m_e = (pre * h.reshape(-1)).sum(2).max(1) + h.sum()
        q = (IL[item][:, None, :] * R).sum(2).max(1)
        tot += float(((d + L + 4) * m_x + (d + w + 4) * m_e * 2 * q).sum())
    scale = 1.0 if not (not pairwise and loss == "cross_entropy") else 1.0 / len(u)
    return 4 * EPS * tot * (2.0 if loss == "square" else 1.0) * scale


# --------------------------------------------------------------------------------------------- gradient kernels
def _grad_cases():
    sms = 132
    cases = [(1, 1, 1, 7), (16, 16, 3, 128), (33, 40, 2, 300), (256, 128, 3, 40), (16, 16, 64, 50),
             (5, 3, 3, 64 * sms + 37)]
    return cases


@pytest.mark.parametrize("d,w,L,batch", _grad_cases())
@pytest.mark.parametrize("pairwise,loss", MODES)
def test_grad_kernel_vs_restatement(pairwise, loss, d, w, L, batch):
    """Loss within the rounding bound of _grad_bound plus the atomic adds' half ulps; every gradient within 3e-5 of
    its largest entry plus that bound's share (fp32 atomics sum duplicate ids in another order than index_add_);
    accumulators are added into; the touched sets are exactly the documented ones; and the routes are the ones the
    shape selects."""
    from neurec_b200 import ops
    rs = np.random.RandomState(d * 7 + w * 3 + L + batch % 97)
    nu, ni = 200, 300
    tabs = _vars(rs, nu, ni, d, w)
    u, win, i, third = _batch(rs, batch, L, nu, ni, pairwise)
    reg_mf, reg_w = 0.01, 0.05
    want_l, want_g, want_t = fpm.fpmcplus_grad(*tabs, u, win, i, third, pairwise, loss, reg_mf, reg_w)
    dt = [dev(t) for t in tabs]
    base = [(rs.randn(*t.shape) * 0.01).astype(np.float32) for t in tabs]
    g = [dev(b) for b in base]
    tch = _touched(nu, ni)
    for t in tch:
        t.fill_(3)
    out = torch.full((1,), 0.5, device="cuda")
    work = ops.fpmcplus_work(d, w, L, batch)
    ops.fpmcplus_grad(*dt, dev(u), dev(win), dev(i), dev(third), pairwise, loss, reg_mf, reg_w, g, tch, 9, work, out)
    got_l = out.item() - 0.5
    bound = _grad_bound(tabs, u, win, i, third, pairwise, loss, d, w, L)
    tol = 1e-5 * abs(float(want_l)) + bound + batch * EPS * (0.5 + abs(float(want_l))) + 1e-6
    assert abs(got_l - float(want_l)) <= tol, (got_l, want_l, tol)
    for k, (gg, b0, ref) in enumerate(zip(g, base, want_g)):
        scale = max(1.0, float(np.abs(ref).max()))
        err = np.abs((host(gg) - b0) - ref).max()
        assert err <= 3e-5 * scale, (k, err, scale)
    for t, ref in zip(tch, want_t):
        hh = host(t)
        assert np.array_equal(hh == 9, ref) and np.all(hh[~ref] == 3)
    assert float(work[:(3 * d * w + 2 * w + 255) // 256].abs().sum()) == 0       # counters left at 0
    r = ops.fpmcplus_last_routes()
    sms = _sms()
    capped = int(batch > 64 * sms)
    assert r["grad"] == dict(pairwise=int(pairwise), grid_x=min((batch + 7) // 8, 8 * sms), grid_y=-1,
                             capped=capped, window=L, rows=-1)
    assert r["wgrad"] == dict(pairwise=int(pairwise), grid_x=(3 * d * w + 2 * w + 255) // 256,
                              grid_y=(batch + 31) // 32, capped=-1, window=L, rows=-1)
    REACHED.add(("grad", pairwise, capped, L == 64, d == 256 and w == 128))


@pytest.mark.parametrize("pairwise", [True, False])
def test_dense_gradients_are_bit_identical_across_launches(pairwise):
    from neurec_b200 import ops
    rs = np.random.RandomState(4)
    nu, ni, d, w, L, batch = 300, 500, 16, 16, 3, 3000
    tabs = _vars(rs, nu, ni, d, w)
    u, win, i, third = _batch(rs, batch, L, nu, ni, pairwise)
    dt = [dev(t) for t in tabs]
    work = ops.fpmcplus_work(d, w, L, batch)
    got = []
    for _ in range(2):
        g = [torch.zeros_like(t) for t in dt]
        ops.fpmcplus_grad(*dt, dev(u), dev(win), dev(i), dev(third), pairwise, "square", 0.01, 0.05, g,
                          _touched(nu, ni), 1, work, torch.zeros(1, device="cuda"))
        got.append([x.clone() for x in g[4:]])
    assert all(torch.equal(a, b) for a, b in zip(*got))
    assert all(float(x.abs().max()) > 0 for x in got[0])


def test_grad_kernel_rejects_without_writing():
    from neurec_b200 import ops
    rs = np.random.RandomState(0)
    dt = [dev(t) for t in _vars(rs, 5, 6, 8, 4)]
    g = [torch.zeros_like(t) for t in dt]
    tch = _touched(5, 6)
    ids, lab = dev(np.zeros(4, np.int32)), dev(np.zeros(4, np.float32))
    work = ops.fpmcplus_work(8, 4, 3, 4)
    out = torch.zeros(1, device="cuda")
    before = ops.fpmcplus_last_routes()
    for pairwise, loss, recent, third in ((True, "cross_entropy", dev(np.zeros((4, 3), np.int32)), ids),
                                          (False, "bpr", dev(np.zeros((4, 3), np.int32)), lab),
                                          (False, "cross_entropy", dev(np.zeros((4, 65), np.int32)), lab)):
        with pytest.raises((ValueError, RuntimeError)):
            ops.fpmcplus_grad(*dt, ids, recent, ids, third, pairwise, loss, 0.1, 0.1, g, tch, 1, work, out)
    with pytest.raises(ValueError):
        ops.fpmcplus_grad(*dt, ids, dev(np.zeros((4, 3), np.int32)), ids, lab, False, "square", 0.1, 0.1, g, tch, 1,
                          None, out)
    torch.cuda.synchronize()
    assert all(float(t.abs().sum()) == 0 for t in g) and out.item() == 0
    assert all(int(t.abs().sum()) == 0 for t in tch)
    assert ops.fpmcplus_last_routes() == before


# --------------------------------------------------------------------------------------------- fused epochs
def _epoch(ds, pairwise, L, bs, num_neg=4, first_epoch=11):
    from neurec_b200.data import sampler as smp
    smp.reseed(first_epoch)
    if pairwise:
        s = smp.TimeOrderPairwiseSampler(ds, high_order=L, neg_num=1, batch_size=bs, shuffle=True)
    else:
        s = smp.TimeOrderPointwiseSampler(ds, high_order=L, neg_num=num_neg, batch_size=bs, shuffle=True)
    return s.device_epoch()


@pytest.mark.parametrize("opt", ["adam", "gd", "adagrad", "rmsprop", "momentum"])
@pytest.mark.parametrize("pairwise", [True, False])
def test_train_epoch_vs_trainer_on_ml100k(ml100k_seq, pairwise, opt):
    """One epoch of the time-ordered ml-100k train set at the conf file's shape (d = w = 16, L = 3, batch 128), fed
    identically to the kernels and to the fp32 trainer: step losses, all seven variables and their slots."""
    from neurec_b200 import ops
    ds = ml100k_seq
    nu, ni, d, w, L, bs = ds.num_users, ds.num_items, 16, 16, 3, 128
    tabs = _vars(np.random.RandomState(3), nu, ni, d, w, scale=0.1)
    epoch = _epoch(ds, pairwise, L, bs)
    ep_h = [host(t) for t in epoch]
    loss = "bpr" if pairwise else "cross_entropy"
    lr = LR[opt]
    tr = fpm.FPMCplusTrainer(*tabs, learner=opt, lr=lr, loss=loss, reg_mf=1e-3, reg_w=1e-3, pairwise=pairwise)
    want = tr.epoch(*ep_h, bs)
    steps = len(want)
    dt = [dev(t) for t in tabs]
    i0, i1 = tf_math.SLOT_INIT[opt]
    mk = lambda a, v: None if v is None else torch.full_like(a, v)
    slots = [(mk(t, i0), mk(t, i1)) for t in dt]
    grads = [torch.zeros_like(t) for t in dt]
    lr_t = tf_math.adam_lr_t(lr, steps) if opt == "adam" else np.full(steps, lr, np.float32)
    step_loss = torch.zeros(steps, device="cuda")
    n = ops.fpmcplus_train_epoch(*dt, *epoch, bs, pairwise, loss, 1e-3, 1e-3, opt, lr_t, tf_math.DEFAULT_HYPER[opt](lr),
                                 grads, _touched(nu, ni), [s[0] for s in slots], [s[1] for s in slots], 1,
                                 ops.fpmcplus_work(d, w, L, bs), step_loss)
    assert n == steps
    assert np.allclose(host(step_loss), want, rtol=1e-4, atol=1e-6)
    for k, (t, ref, t0) in enumerate(zip(dt, tr.vars, tabs)):
        assert np.abs(host(t) - ref).max() < 5e-5 * max(1.0, np.abs(ref).max()), k
        assert np.abs(ref - t0).max() > 1e-6, k                         # every variable moved
    for (s0, s1), (r0, r1) in zip(slots, tr.slots):
        for s, r in ((s0, r0), (s1, r1)):
            if s is not None:
                assert np.abs(host(s) - r).max() <= 1e-4 * max(1e-3, np.abs(r).max())
    assert all(float(g.abs().max()) == 0 for g in grads)


# --------------------------------------------------------------------------------------------- scores
def _score_bound(tabs, users, windows):
    t = [np.abs(v.astype(np.float64)) for v in tabs]
    UI, IU, IL, LI, W, b, h = t
    d = UI.shape[1]
    out = []
    for u, win in zip(users, windows):
        R = LI[np.asarray(win)]
        m_x = IU @ UI[u] + (IL @ R.T).max(1)
        pre = (UI[u] @ W[:d] + b.reshape(-1))[None, None, :] + (IL @ W[d:2 * d])[:, None, :] + (R @ W[2 * d:])[None]
        m_e = (pre * h.reshape(-1)).sum(2).max(1) + h.sum()
        q = (IL @ R.T).max(1)
        out.append((d + len(win) + 4) * m_x + (d + W.shape[1] + 4) * m_e * 2 * q)
    return 4 * EPS * np.asarray(out)


@pytest.mark.parametrize("d,w,L", [(1, 1, 1), (16, 16, 3), (33, 40, 2), (256, 128, 3), (16, 16, 64), (64, 128, 64),
                                   (256, 128, 64)])
def test_scores_vs_fp64(d, w, L):
    """Every user of a dataset with histories shorter and longer than the window, the window as Python slices it and
    the softmax over its length.  The pair kernel's rows per CTA shrink where a row's window does not fit the
    shared-memory budget (one at the widest shapes)."""
    from neurec_b200 import ops
    from neurec_b200.model.sequential_recommender._base import predict_windows
    ds, nu = _short_history_dataset(min(L, 5), ni=300)
    ni = ds.num_items
    train_dict = ds.get_user_train_dict(by_time=True)
    recent, length = predict_windows(train_dict, nu, L)
    users = np.asarray(sorted(train_dict), np.int32)
    windows = [list(train_dict[u])[len(train_dict[u]) - L:] for u in users]
    assert min(len(x) for x in windows) < L or L == 1
    tabs = _vars(np.random.RandomState(d + w + L), nu, ni, d, w)
    got = host(ops.fpmcplus_scores(*[dev(t) for t in tabs], dev(users), dev(recent), dev(length)))
    want = fpm.fpmcplus_scores(*tabs, users, windows)
    assert got.shape == (len(users), ni)
    assert np.all(np.abs(got - want) <= _score_bound(tabs, users, windows) + 1e-12), np.abs(got - want).max()
    r = ops.fpmcplus_last_routes()
    per_row = (w + d) * (1 + L) + 1
    rows = min(8, (25600 - w) // per_row)
    assert r["pair"] == dict(pairwise=-1, grid_x=(len(users) + rows - 1) // rows, grid_y=(ni + 255) // 256,
                             capped=-1, window=L, rows=rows)
    assert r["project"]["capped"] == 0 and r["project"]["window"] == L
    REACHED.add(("pair", rows))


def test_scores_projection_capped_grid():
    """A catalogue large enough that the projection pass's grid is capped (threads take several elements)."""
    from neurec_b200 import ops
    rs = np.random.RandomState(8)
    nu, ni, d, w, L = 4, 30000, 16, 16, 3
    tabs = _vars(rs, nu, ni, d, w)
    users = np.arange(nu, dtype=np.int32)
    recent = rs.randint(0, ni, (nu, L)).astype(np.int32)
    length = np.asarray([3, 1, 2, 3], np.int32)
    got = host(ops.fpmcplus_scores(*[dev(t) for t in tabs], dev(users), dev(recent), dev(length)))
    assert ops.fpmcplus_last_routes()["project"]["capped"] == 1
    windows = [recent[u, :length[u]] for u in users]
    want = fpm.fpmcplus_scores(*tabs, users, windows)
    assert np.all(np.abs(got - want) <= _score_bound(tabs, users, windows) + 1e-12)


def test_scores_overflow_as_the_reference():
    """|h|_1 > 88: where some exp(e_k) overflows in fp32 the reference's inf / inf makes the score NaN, and where
    every exp(e_k) underflows 0 / 0 does; the NaNs land where the fp32 restatement puts them and every other score is
    within the fp64 bound."""
    from neurec_b200 import ops
    rs = np.random.RandomState(9)
    nu, ni, d, w, L = 6, 400, 4, 8, 3
    tabs = _vars(rs, nu, ni, d, w)
    tabs[4][:] = 0
    tabs[4][d] = 40.0                                    # z follows the sign of IL_j[0], saturating tanh
    tabs[4][2 * d + 1] = 40.0                            # ... plus that of LI_l[1]
    tabs[6][:] = 15.0                                    # |h|_1 = 120
    tabs[2][:, 0] = rs.choice([-1.0, 0.0, 1.0], ni)
    tabs[3][:, 1] = rs.choice([-1.0, 1.0], ni)
    users = np.arange(nu, dtype=np.int32)
    recent = rs.randint(0, ni, (nu, L)).astype(np.int32)
    length = np.full(nu, L, np.int32)
    got = host(ops.fpmcplus_scores(*[dev(t) for t in tabs], dev(users), dev(recent), dev(length)))
    want32 = fpm.fpmcplus_scores(*tabs, users, list(recent), dtype=np.float32)
    nan = np.isnan(want32)
    assert nan.any() and (~nan).any()
    assert np.array_equal(np.isnan(got), nan)
    want = fpm.fpmcplus_scores(*tabs, users, list(recent))
    fin = ~nan & np.isfinite(want)
    assert np.allclose(got[fin], want[fin], rtol=1e-4, atol=1e-4)


# --------------------------------------------------------------------------------------------- plug-in
MODEL_CONF = dict(recommender="FPMCplus", epochs=1, batch_size=128, embedding_size=16, weight_size=16, high_order=3,
                  reg_mf=1e-5, reg_w=1e-3, learning_rate=0.001, learner="adam", is_pairwise=True, num_neg=4,
                  loss_function="BPR", embed_init_method="tnormal", weight_init_method="he_normal", stddev=0.01,
                  verbose=1)


def _plug_in(ds, **over):
    from neurec_b200.model.sequential_recommender.FPMCplus import FPMCplus
    m = FPMCplus(None, ds, _Conf(BASE_CONF, **dict(MODEL_CONF, **over)))
    m.build_graph()
    return m


def test_plug_in_initialises_in_the_reference_order(ml100k_seq, tmp_path, monkeypatch):
    """Generator 2017 in variable order: tables by embed_init_method, W and b by weight_init_method, h ones."""
    from neurec_b200.model._engine import get_initializer
    monkeypatch.chdir(tmp_path)
    m = _plug_in(ml100k_seq)
    gen = torch.Generator().manual_seed(2017)
    emb, wgt = get_initializer("tnormal", 0.01, gen), get_initializer("he_normal", 0.01, gen)
    nu, ni = ml100k_seq.num_users, ml100k_seq.num_items
    want = [emb([nu, 16]), emb([ni, 16]), emb([ni, 16]), emb([ni, 16]), wgt([48, 16]), wgt([1, 16])]
    for t, ref in zip(m.tables(), want):
        assert torch.equal(t.cpu(), ref)
    assert torch.equal(m.h.cpu(), torch.ones(16, 1))


@pytest.mark.parametrize("pairwise", [True, False])
def test_plug_in_epoch_predict_evaluate_and_checkpoint(ml100k_seq, tmp_path, monkeypatch, pairwise):
    from neurec_b200 import ops
    from neurec_b200.data import sampler as smp
    from neurec_b200.util import checkpoint
    monkeypatch.chdir(tmp_path)
    ds = ml100k_seq
    over = {} if pairwise else dict(is_pairwise=False, loss_function="cross_entropy")
    m = _plug_in(ds, **over)
    rs = np.random.RandomState(6)
    for t in m.tables()[:4]:
        t.copy_(dev((rs.randn(*t.shape) * 0.1).astype(np.float32)))
    init = [host(t).copy() for t in m.tables()]
    smp.reseed(21)
    total = m._train_epoch()
    epoch = _epoch(ds, pairwise, 3, 128, first_epoch=21)
    tr = fpm.FPMCplusTrainer(*init, learner="adam", lr=1e-3, loss=m._loss, reg_mf=1e-5, reg_w=1e-3,
                             pairwise=pairwise)
    want = tr.epoch(*[host(t) for t in epoch], 128)
    assert abs(total - float(want.sum(dtype=np.float64))) <= 1e-4 * abs(float(want.sum()))
    # Adam's step is scale-free: where a dense W or b entry's gradient cancels to rounding level over a step, the
    # step's sign follows the rounding, so the plug-in's variables are compared at lr-scale drift (the table-level
    # comparison of every optimizer is test_train_epoch_vs_trainer_on_ml100k)
    for t, ref in zip(m.tables(), tr.vars):
        assert np.abs(host(t) - ref).max() < 5e-4 * max(1.0, np.abs(ref).max())
    # predict: every item from the user's last 3 train items by time, and the candidate path
    users = [0, 5, 17, 942]
    train_dict = ds.get_user_train_dict(by_time=True)
    windows = [list(train_dict[u])[len(train_dict[u]) - 3:] for u in users]
    tabs = [host(t) for t in m.tables()]
    want_s = fpm.fpmcplus_scores(*tabs, users, windows)
    got = m.predict(users)
    assert isinstance(got, torch.Tensor) and got.is_cuda and got.shape == (4, ds.num_items)
    assert np.all(np.abs(host(got) - want_s) <= _score_bound(tabs, users, windows) + 1e-12)
    cand = [[1, 2, 3], [10], [0, 1681], [5, 5, 7]]
    for r, w, c in zip(m.predict(users, cand), host(got), cand):
        assert isinstance(r, np.ndarray) and np.array_equal(r, w[c])
    with pytest.raises(KeyError):
        m.predict([0, ds.num_users + 5])
    # evaluate(): the evaluator's generic route -- mask the train items, score matrix, mean of the rows
    got_s = m.evaluate()
    test_dict, train_all = ds.get_user_test_dict(), ds.get_user_train_dict()
    test_users = list(test_dict.keys())
    ptr = np.zeros(ds.num_users + 1, np.int64)
    for u, it in train_all.items():
        ptr[u + 1] = len(it)
    ptr = np.cumsum(ptr)
    idx = np.concatenate([np.unique(np.asarray(train_all[u], np.int32)) for u in sorted(train_all)])
    rows = []
    for off in range(0, len(test_users), BASE_CONF["test_batch_size"]):
        bu = test_users[off:off + BASE_CONF["test_batch_size"]]
        scores = m.predict(bu).contiguous()
        ops.mask_rows(scores, dev(np.asarray(bu, np.int32)), dev(ptr), dev(idx))
        tptr = np.zeros(len(bu) + 1, np.int64)
        tptr[1:] = np.cumsum([len(np.unique(test_dict[u])) for u in bu])
        tidx = np.concatenate([np.unique(np.asarray(test_dict[u], np.int32)) for u in bu])
        rows.append(ops.eval_score_matrix(scores, dev(tptr), dev(tidx), [1, 2, 4, 3, 5], 20))
    final = host(ops.mean_rows(torch.cat(rows, 0))).reshape(5, 20)[:, [9, 19]].reshape(-1)
    assert got_s == "\t".join([("%.8f" % x).ljust(12) for x in final])
    # checkpoint: W, b, h and their slots come back bit for bit, and the resumed epoch continues the run
    path = str(tmp_path / "fpmcplus.ckpt")
    checkpoint.save(m, path)
    saved = torch.load(path, map_location="cpu")["tensors"]
    assert {"W", "b", "h", "_slots0.4", "_slots1.6"} <= set(saved)
    la = m._train_epoch()
    smp.reseed(0)
    b = _plug_in(ds, **over)
    checkpoint.load(b, path)
    live = checkpoint.state_dict(b)["tensors"]
    assert set(saved) - {"_step_loss"} <= set(live)
    for k, v in saved.items():
        if k in live:
            assert torch.equal(live[k], v), k
    lb = b._train_epoch()
    assert abs(la - lb) <= 1e-5 * abs(la)


def test_plug_in_short_histories(tmp_path, monkeypatch):
    """Users with fewer train items than high_order are scored over the shorter window; KeyError for a user without
    train items."""
    from neurec_b200 import ops
    monkeypatch.chdir(tmp_path)
    ds, nu = _short_history_dataset(3)
    train_dict = ds.get_user_train_dict(by_time=True)
    users = sorted(train_dict)
    m = _plug_in(ds)
    windows = [list(train_dict[u])[len(train_dict[u]) - 3:] for u in users]
    assert [int(x) for x in host(m._recent_len)[users]] == [len(w) for w in windows]
    got = m.predict(users)
    tabs = [host(t) for t in m.tables()]
    want = fpm.fpmcplus_scores(*tabs, users, windows)
    assert np.all(np.abs(host(got) - want) <= _score_bound(tabs, users, windows) + 1e-12)
    kern = ops.fpmcplus_scores(*m.tables(), dev(np.asarray(users, np.int32)), m._recent, m._recent_len)
    assert torch.equal(got, kern)
    with pytest.raises(KeyError):
        m.predict([users[0], nu - 1])


# --------------------------------------------------------------------------------------------- main.py
def test_main_runs_fpmcplus(tmp_path):
    data = tmp_path / "dataset"
    write_timed_dataset(str(data))
    cmd = [sys.executable, os.path.join(ROOT, "main.py"), "--recommender=FPMCplus", "--data.input.path=%s" % data,
           "--data.input.dataset=toy", "--topk=[5,10]", "--test_batch_size=64", "--epochs=4", "--learning_rate=0.01"]
    for f in ("NeuRec.properties", "conf"):
        os.symlink(os.path.join(ROOT, f), tmp_path / f)
    r = subprocess.run(cmd, cwd=tmp_path, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    out = r.stdout
    assert "metrics:\tPrecision@5 " in out and "NDCG@10" in out
    epochs = re.findall(r"epoch (\d+):\t([0-9.\t ]+)", out)
    vals = np.array([[float(x) for x in e[1].split()] for e in epochs])
    assert vals.shape[1] == 10 and np.isfinite(vals).all() and (vals >= 0).all() and (vals <= 1).all()
    losses = re.findall(r"\[iter (\d+) : loss : ([0-9.eE+-]+), time: [0-9.]+\]", out)
    assert [int(e[0]) for e in epochs] == [1, 2, 3, 4] and [int(e[0]) for e in losses] == [1, 2, 3, 4]
    lv = [float(e[1]) for e in losses]
    assert np.isfinite(lv).all() and lv[-1] < lv[0]


def test_every_route_was_reached():
    """Runs last in this file: the gradient kernel in both forms, capped and not, at the window and width caps, and
    the pair kernel with 8 rows per CTA and with 1."""
    if len(REACHED) == 0:
        pytest.skip("the route tests did not run in this session")
    for pairwise in (True, False):
        assert ("grad", pairwise, 1, False, False) in REACHED and ("grad", pairwise, 0, True, False) in REACHED
        assert ("grad", pairwise, 0, False, True) in REACHED
    assert ("pair", 8) in REACHED and ("pair", 1) in REACHED
