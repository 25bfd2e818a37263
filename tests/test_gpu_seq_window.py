"""GPU parity of HRM and NPE (csrc/sequential.cu) through the C ABI against the fp32 restatement in
tests/seq_window_math.py: the gradient kernels on every width class, window length and pooling, one fused epoch per
optimizer on the time-ordered ml-100k train set, the query kernels + nrc_mf_scores against fp64, the plug-ins
(epoch, predict, evaluate, checkpoint) and main.py."""
import os
import re
import subprocess
import sys

import numpy as np
import pytest
import scipy.sparse as sp
import torch

import seq_window_math as swm
from oracle import tf_math
from test_gpu_sequential import BASE_CONF, _Conf, dev, host, ml100k_time_ordered, write_timed_dataset

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

LR = {"adam": 1e-3, "gd": 0.05, "adagrad": 0.01, "rmsprop": 1e-3, "momentum": 0.02}
# (model, pre_max, session_max, integer-valued tables that force max ties)
VARIANTS = [("hrm", pm, sm, ties) for pm in (True, False) for sm in (True, False) for ties in (False, True)] + \
           [("npe", None, None, False), ("npe", None, None, True)]


@pytest.fixture(scope="module")
def ml100k_seq():
    return ml100k_time_ordered()


def _tables(model, rs, nu, ni, d, scale=0.1, ties=False):
    shapes = [(nu, d), (ni, d)] if model == "hrm" else [(nu, d), (ni, d), (ni, d)]
    if ties:
        return [rs.randint(-2, 3, s).astype(np.float32) for s in shapes]
    return [(rs.randn(*s) * scale).astype(np.float32) for s in shapes]


def _touched(model, nu, ni):
    z = lambda n: torch.zeros(n, dtype=torch.int32, device="cuda")
    return (z(nu), z(ni)) if model == "hrm" else (z(nu), z(ni), z(ni))


def _loss_rounding(model, tabs, users, recent, items, labels, pm, sm, loss, d, L):
    """A bound on |fp32 batch loss - exact| beyond the loss formula's own rounding: each sample's score is a d-term
    sum after an L-term pool, so it carries up to (d + L + 4) eps of its terms' magnitudes M_b, which moves the loss
    by |dl/dx_b| times that (it matters where x cancels); each warp's loss then enters the accumulator by one fp32
    atomic add (at most half an ulp of the running sum; integer tables make many samples' losses equal, so these
    roundings need not cancel)."""
    t = [np.abs(a.astype(np.float64)) for a in tabs]
    w = recent.reshape(len(users), -1)
    if model == "hrm":
        s = t[1][w].max(1) if sm else t[1][w].mean(1)
        h = np.maximum(t[0][users], s) if pm else (t[0][users] + s) / 2
        m = (h * t[1][items]).sum(1)
        x = swm.hrm_scores(*[a.astype(np.float64) for a in tabs], users, w, pm, sm)[np.arange(len(users)), items]
    else:
        m = (t[1][items] * (t[0][users] + t[2][w].sum(1))).sum(1)
        x = swm.npe_scores(*[a.astype(np.float64) for a in tabs], users, w)[np.arange(len(users)), items]
    dl = 2 * np.abs(labels - x) if loss == "square" else np.full(len(x), 1.0 / len(x))
    return float((dl * m).sum()) * 2.0 ** -23 * (d + L + 4)


def _grad_call(model, dt, batch, pm, sm, loss, reg, g, tch, stamp, out):
    from neurec_b200 import ops
    if model == "hrm":
        ops.hrm_grad(*dt, *batch, pm, sm, loss, reg, *g, *tch, stamp, out)
    else:
        ops.npe_grad(*dt, *batch, loss, reg, *g, *tch, stamp, out)


# --------------------------------------------------------------------------------------------- gradient kernels
@pytest.mark.parametrize("batch", [1, 1000])
@pytest.mark.parametrize("L", [1, 2, 3, 5, 64])
@pytest.mark.parametrize("d", [1, 7, 16, 50, 64, 128, 256])
@pytest.mark.parametrize("model,pre_max,session_max,ties", VARIANTS)
def test_grad_kernel_vs_restatement(model, pre_max, session_max, ties, d, L, batch):
    """Both losses, reg 0 and 0.01, repeated users, items and window ids: loss within rel 1e-5 plus the rounding
    bound of _loss_rounding, gradients within 2e-5
    of the largest gradient entry (fp32 atomics sum duplicate ids in another order than np.add.at), accumulators
    added into, the touched sets exactly the documented ones.  Integer tables make window maxima and P_u == s tie
    exactly, and put exact zeros at relu's inputs."""
    rs = np.random.RandomState(d * 131 + L * 7 + batch)
    nu, ni = 300, 500
    tabs = _tables(model, rs, nu, ni, d, ties=ties)
    users, items = rs.randint(0, nu, batch).astype(np.int32), rs.randint(0, ni, batch).astype(np.int32)
    recent = rs.randint(0, ni, (batch, L)).astype(np.int32)
    if batch > 1:
        users[1] = users[0]
        recent[0, -1] = recent[0, 0]
        recent[2, 0], items[3] = items[2], recent[3, 0]
    labels = (rs.rand(batch) < 0.3).astype(np.float32)
    dt = [dev(t) for t in tabs]
    x_err = {loss: _loss_rounding(model, tabs, users, recent, items, labels, pre_max, session_max, loss, d, L)
             for loss in ("cross_entropy", "square")}
    for loss in ("cross_entropy", "square"):
        for reg in (0.0, 0.01):
            if model == "hrm":
                want_l, want_g, want_t = swm.hrm_grad(*tabs, users, recent, items, labels, pre_max, session_max, loss,
                                                      reg)
            else:
                want_l, want_g, want_t = swm.npe_grad(*tabs, users, recent, items, labels, loss, reg)
            base = [(rs.randn(*t.shape) * 0.01).astype(np.float32) for t in tabs]
            g = [dev(b) for b in base]
            tch = _touched(model, nu, ni)
            for t in tch:
                t.fill_(3)
            out = torch.full((1,), 0.5, device="cuda")
            _grad_call(model, dt, [dev(users), dev(recent), dev(items), dev(labels)], pre_max, session_max, loss, reg,
                       g, tch, 9, out)
            got_l = out.item() - 0.5
            atomics = batch * 2.0 ** -24 * (0.5 + abs(float(want_l)))
            tol = 1e-5 * abs(float(want_l)) + 1e-6 + x_err[loss] + atomics
            assert abs(got_l - float(want_l)) <= tol, (loss, reg, got_l, want_l, tol)
            scale = max(float(np.abs(w).max()) for w in want_g)
            for k, (gg, b, w) in enumerate(zip(g, base, want_g)):
                err = np.abs((host(gg) - b) - w).max()
                assert err <= 2e-5 * max(1.0, scale), (loss, reg, k, err, scale)
            for t, w in zip(tch, want_t):
                h = host(t)
                assert np.array_equal(h == 9, w) and np.all(h[~w] == 3)


@pytest.mark.parametrize("model", ["hrm", "npe"])
def test_grad_kernel_rejects_without_writing(model):
    from neurec_b200 import ops
    rs = np.random.RandomState(0)
    dt = [dev(t) for t in _tables(model, rs, 5, 6, 8)]
    g = [torch.zeros_like(t) for t in dt]
    tch = _touched(model, 5, 6)
    ids, lab = dev(np.zeros(4, np.int32)), dev(np.zeros(4, np.float32))
    out = torch.zeros(1, device="cuda")
    for loss, recent in (("bpr", dev(np.zeros((4, 2), np.int32))), ("cross_entropy", dev(np.zeros((4, 65), np.int32)))):
        with pytest.raises((ValueError, RuntimeError)):
            _grad_call(model, dt, [ids, recent, ids, lab], True, True, loss, 0.1, g, tch, 1, out)
    torch.cuda.synchronize()
    assert all(float(t.abs().sum()) == 0 for t in g) and out.item() == 0
    assert all(int(t.abs().sum()) == 0 for t in tch)


# --------------------------------------------------------------------------------------------- fused epochs
CONF_SHAPE = {"hrm": dict(L=2, d=16, bs=256, reg=0.01, instances=78481),
              "npe": dict(L=3, d=64, bs=256, reg=0.1, instances=77538)}


def _epoch(ds, L, bs, num_neg=4, first_epoch=11):
    from neurec_b200.data import sampler as smp
    smp.reseed(first_epoch)
    s = smp.TimeOrderPointwiseSampler(ds, high_order=L, neg_num=num_neg, batch_size=bs, shuffle=True)
    return s, s.device_epoch()


@pytest.mark.parametrize("opt", ["adam", "gd", "adagrad", "rmsprop", "momentum"])
@pytest.mark.parametrize("model", ["hrm", "npe"])
def test_train_epoch_vs_trainer_on_ml100k(ml100k_seq, model, opt):
    """One epoch of the time-ordered ml-100k train set at the conf file's window, width and batch size (HRM with max
    pools), fed identically to the kernels and to the fp32 trainer.  reg is the conf's for NPE except under adagrad and
    rmsprop (see below) and 0.01 for HRM (the conf's is 0)."""
    from neurec_b200 import ops
    ds = ml100k_seq
    nu, ni = ds.num_users, ds.num_items
    c = dict(CONF_SHAPE[model])
    lr = LR[opt]
    if model == "npe" and opt in ("adagrad", "rmsprop"):
        # these steps do not shrink with the gradient: an entry that relu gates off gets only reg * w, which walks it
        # around 0 in lr-sized steps, and on which side of 0 it lands (whether relu passes the data gradient) then
        # turns on rounding-level differences.  Without reg such an entry stays where it is.
        c["reg"] = 0.0
    tabs = _tables(model, np.random.RandomState(3), nu, ni, c["d"])
    sampler, epoch = _epoch(ds, c["L"], c["bs"])
    assert len(sampler._users_np) == c["instances"] and epoch[0].numel() == c["instances"] * 5
    assert tuple(epoch[1].shape) == (c["instances"] * 5, c["L"])
    ep_h = [host(t) for t in epoch]
    if model == "hrm":
        tr = swm.HRMTrainer(*tabs, learner=opt, lr=lr, reg=c["reg"], pre_max=True, session_max=True)
    else:
        tr = swm.NPETrainer(*tabs, learner=opt, lr=lr, reg=c["reg"])
    want = tr.epoch(*ep_h, c["bs"])
    steps = len(want)
    dt = [dev(t) for t in tabs]
    i0, i1 = tf_math.SLOT_INIT[opt]
    mk = lambda a, v: None if v is None else torch.full_like(a, v)
    slots = [(mk(t, i0), mk(t, i1)) for t in dt]
    grads = [torch.zeros_like(t) for t in dt]
    lr_t = tf_math.adam_lr_t(lr, steps) if opt == "adam" else np.full(steps, lr, np.float32)
    step_loss = torch.zeros(steps, device="cuda")
    args = (*epoch, c["bs"])
    tail = ("cross_entropy", c["reg"], opt, lr_t, tf_math.DEFAULT_HYPER[opt](lr), grads, _touched(model, nu, ni),
            [s[0] for s in slots], [s[1] for s in slots], 1, step_loss)
    if model == "hrm":
        n = ops.hrm_train_epoch(*dt, *args, True, True, *tail)
    else:
        n = ops.npe_train_epoch(*dt, *args, *tail)
    assert n == steps
    assert np.allclose(host(step_loss), want, rtol=1e-4)
    for i, (t, ref, t0) in enumerate(zip(dt, tr.vars, tabs)):
        assert np.abs(host(t) - ref).max() < 3e-5, i
        assert np.abs(ref - t0).max() > 1e-5, i                         # every variable moved
    assert all(float(g.abs().max()) == 0 for g in grads)                 # the optimizer launch consumes the gradients


# --------------------------------------------------------------------------------------------- query + scores
def _short_history_dataset(L, ni=300):
    """Users whose train sequences have every length 1 .. 2L + 1, one user without train items, in a dataset with
    times (each user's items in time order are a random permutation slice)."""
    from neurec_b200.data import Dataset
    rs = np.random.RandomState(L)
    rows, cols, times = [], [], []
    lengths = list(range(1, 2 * L + 2)) * 3
    for u, n in enumerate(lengths):
        it = rs.choice(ni, n, replace=False)
        rows += [u] * n
        cols += list(it)
        times += list(rs.permutation(n) + 1.0)
    nu = len(lengths) + 1                                               # the last user has no train items
    mk = lambda data: sp.csr_matrix((np.asarray(data, np.float64), (rows, cols)), shape=(nu, ni))
    train = mk(np.ones(len(rows)))
    return Dataset.from_csr("short", train, train, time_matrix=mk(times)), nu


@pytest.mark.parametrize("d", [1, 16, 64, 256])
@pytest.mark.parametrize("L", [1, 2, 3, 5])
@pytest.mark.parametrize("model,pre_max,session_max", [("hrm", True, True), ("hrm", True, False),
                                                       ("hrm", False, True), ("hrm", False, False),
                                                       ("npe", None, None)])
def test_query_scores_vs_fp64(model, pre_max, session_max, L, d):
    """Query rows + nrc_mf_scores for every user of a dataset with histories shorter and longer than the window, the
    window as Python slices it.  Tolerance: the fp32 pools' and the d-term FMA chain's rounding, relative to the same
    computation on absolute values."""
    from neurec_b200 import ops
    from neurec_b200.model.sequential_recommender._base import predict_windows
    ds, nu = _short_history_dataset(L)
    ni = ds.num_items
    train_dict = ds.get_user_train_dict(by_time=True)
    recent, length = predict_windows(train_dict, nu, L)
    users = np.asarray(sorted(train_dict), np.int32)
    windows = [swm.predict_window(list(train_dict[u]), L) for u in users]
    assert min(len(w) for w in windows) == 1 and sorted({len(w) for w in windows}) == sorted(
        {(L if n >= L else min(n, L - n)) for n in range(1, 2 * L + 2)})
    rs = np.random.RandomState(L * 31 + d)
    tabs = _tables(model, rs, nu, ni, d, scale=0.3)
    dt = [dev(t) for t in tabs]
    args = (dev(users), dev(recent), dev(length))
    eps = 6e-8
    t64 = [t.astype(np.float64) for t in tabs]
    if model == "hrm":
        got = host(ops.hrm_scores(*dt, *args, pre_max, session_max))
        want = swm.hrm_scores(*t64, users, windows, pre_max, session_max)
        mag = swm.hrm_scores(*[np.abs(t) for t in t64], users, windows, pre_max, session_max)
    else:
        got = host(ops.npe_scores(*dt, *args))
        want = swm.npe_scores(*t64, users, windows)
        UI, IU, IL = (np.abs(t) for t in t64)
        mag = np.asarray([IU @ (UI[u] + IL[np.asarray(w)].sum(0)) for u, w in zip(users, windows)])
    assert got.shape == (len(users), ni)
    tol = 2 * eps * (d + L + 4) * mag
    assert np.all(np.abs(got - want) <= tol + 1e-12), np.abs(got - want).max()


# --------------------------------------------------------------------------------------------- plug-ins
MODEL_CONF = {
    "HRM": dict(recommender="HRM", epochs=1, batch_size=256, embedding_size=16, reg_mf=0.01, topK=10,
                learning_rate=0.001, learner="adam", pre_agg="max", session_agg="max", high_order=2, num_neg=4,
                loss_function="cross_entropy", init_method="normal", stddev=0.01, verbose=1),
    "NPE": dict(recommender="NPE", epochs=1, batch_size=256, embedding_size=64, reg=0.1, learning_rate=0.001,
                learner="adam", high_order=3, num_neg=4, loss_function="cross_entropy", init_method="tnormal",
                stddev=0.01, verbose=1),
}


def _plug_in(name, ds, **over):
    from neurec_b200.model.sequential_recommender.HRM import HRM
    from neurec_b200.model.sequential_recommender.NPE import NPE
    m = {"HRM": HRM, "NPE": NPE}[name](None, ds, _Conf(BASE_CONF, **dict(MODEL_CONF[name], **over)))
    m.build_graph()
    return m


@pytest.mark.parametrize("name", ["HRM", "NPE"])
def test_plug_in_epoch_predict_evaluate_and_checkpoint(ml100k_seq, tmp_path, monkeypatch, name):
    from neurec_b200 import ops
    from neurec_b200.data import sampler as smp
    from neurec_b200.util import checkpoint
    monkeypatch.chdir(tmp_path)
    ds = ml100k_seq
    m = _plug_in(name, ds)
    conf = MODEL_CONF[name]
    L = conf["high_order"]
    # Adam on 0.01-scale tables takes steps of either sign where a gradient cancels to rounding level, so the plumbing
    # is compared on 0.1-scale tables (as for FPMC)
    rs = np.random.RandomState(6)
    for t in m.tables():
        t.copy_(dev((rs.randn(*t.shape) * 0.1).astype(np.float32)))
    init = [host(t).copy() for t in m.tables()]
    smp.reseed(21)
    total = m._train_epoch()
    _, epoch = _epoch(ds, L, conf["batch_size"], conf["num_neg"], first_epoch=21)
    if name == "HRM":
        tr = swm.HRMTrainer(*init, learner="adam", lr=conf["learning_rate"], reg=conf["reg_mf"])
    else:
        tr = swm.NPETrainer(*init, learner="adam", lr=conf["learning_rate"], reg=conf["reg"])
    want = tr.epoch(*[host(t) for t in epoch], conf["batch_size"])
    assert abs(total - float(want.sum(dtype=np.float64))) <= 1e-4 * abs(float(want.sum()))
    for t, ref in zip(m.tables(), tr.vars):
        assert np.abs(host(t) - ref).max() < 3e-5
    # predict: query + nrc_mf_scores from every user's last high_order train items (by time), and the candidate path
    users = [0, 5, 17, 942]
    train_dict = ds.get_user_train_dict(by_time=True)
    windows = [list(train_dict[u])[len(train_dict[u]) - L:] for u in users]
    t64 = [host(t).astype(np.float64) for t in m.tables()]
    want_s = (swm.hrm_scores(*t64, users, windows, True, True) if name == "HRM"
              else swm.npe_scores(*t64, users, windows))
    got = m.predict(users)
    assert isinstance(got, torch.Tensor) and got.is_cuda and got.shape == (4, ds.num_items)
    assert np.abs(host(got) - want_s).max() <= 1e-5 * max(1.0, np.abs(want_s).max())
    cand = [[1, 2, 3], [10], [0, 1681], [5, 5, 7]]
    for r, w, c in zip(m.predict(users, cand), host(got), cand):
        assert isinstance(r, np.ndarray) and np.array_equal(r, w[c])
    with pytest.raises(KeyError):                                        # a user without train items
        m.predict([0, ds.num_users + 5])
    # evaluate(): the evaluator's generic route -- mask the train items, score matrix, mean of the rows
    got_s = m.evaluate()
    test_dict, train_dict = ds.get_user_test_dict(), ds.get_user_train_dict()
    test_users = list(test_dict.keys())
    ptr = np.zeros(ds.num_users + 1, np.int64)
    for u, it in train_dict.items():
        ptr[u + 1] = len(it)
    ptr = np.cumsum(ptr)
    idx = np.concatenate([np.unique(np.asarray(train_dict[u], np.int32)) for u in sorted(train_dict)])
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
    # checkpoint: the restored state is bit-identical, and the resumed epoch continues the run
    path = str(tmp_path / "seq.ckpt")
    checkpoint.save(m, path)
    saved = torch.load(path, map_location="cpu")["tensors"]
    la = m._train_epoch()
    smp.reseed(0)
    b = _plug_in(name, ds)
    checkpoint.load(b, path)
    live = checkpoint.state_dict(b)["tensors"]
    assert set(saved) - {"_step_loss"} <= set(live)                   # scratch a fresh model allocates on use
    for k, v in saved.items():
        if k in live:
            assert torch.equal(live[k], v), k
    # the resumed epoch differs from the uninterrupted one only by the gradient atomics' summation order; Adam's
    # scale-free step on relu-gated NPE entries amplifies that in the tables, so the two runs are compared by loss
    lb = b._train_epoch()
    assert abs(la - lb) <= 1e-5 * abs(la)


def test_plug_in_windows_and_short_histories(tmp_path, monkeypatch):
    """The plug-ins' predict windows on users with fewer train items than high_order (scored over the shorter window,
    as the reference's slice gives it), and KeyError for a user without train items."""
    from neurec_b200 import ops
    monkeypatch.chdir(tmp_path)
    ds, nu = _short_history_dataset(3)
    train_dict = ds.get_user_train_dict(by_time=True)
    users = sorted(train_dict)
    for name in ("HRM", "NPE"):
        m = _plug_in(name, ds, high_order=3)
        windows = [list(train_dict[u])[len(train_dict[u]) - 3:] for u in users]
        assert [int(x) for x in host(m._recent_len)[users]] == [len(w) for w in windows]
        got = m.predict(users)
        t64 = [host(t).astype(np.float64) for t in m.tables()]
        want = (swm.hrm_scores(*t64, users, windows, True, True) if name == "HRM"
                else swm.npe_scores(*t64, users, windows))
        assert np.abs(host(got) - want).max() <= 1e-5 * max(1e-3, np.abs(want).max())
        kern = (ops.hrm_scores(*m.tables(), dev(np.asarray(users, np.int32)), m._recent, m._recent_len, True, True)
                if name == "HRM" else
                ops.npe_scores(*m.tables(), dev(np.asarray(users, np.int32)), m._recent, m._recent_len))
        assert torch.equal(got, kern)
        with pytest.raises(KeyError):
            m.predict([users[0], nu - 1])


# --------------------------------------------------------------------------------------------- main.py
@pytest.mark.parametrize("name", ["HRM", "NPE"])
def test_main_runs_the_window_models(tmp_path, name):
    data = tmp_path / "dataset"
    write_timed_dataset(str(data))
    cmd = [sys.executable, os.path.join(ROOT, "main.py"), "--recommender=%s" % name, "--data.input.path=%s" % data,
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
    assert [int(e[0]) for e in epochs] == [1, 2, 3, 4]                  # epochs 1..N (HRM.py:110, NPE.py:89)
    assert [int(e[0]) for e in losses] == [1, 2, 3, 4]
    lv = [float(e[1]) for e in losses]
    assert np.isfinite(lv).all() and lv[-1] < lv[0]
