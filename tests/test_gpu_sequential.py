"""GPU parity of FPMC and TransRec (csrc/sequential.cu) through the C ABI against the fp32 restatement in
tests/seq_math.py: the gradient kernels on every width class and mode, one fused epoch per optimizer on the
time-ordered ml-100k train set, the score kernels against fp64, the plug-ins and main.py."""
import os
import re
import subprocess
import sys

import numpy as np
import pytest
import scipy.sparse as sp
import torch

import seq_math
from oracle import tf_math

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")

MODES = [(True, "bpr"), (True, "hinge"), (True, "square"), (False, "cross_entropy"), (False, "square")]
LR = {"adam": 1e-3, "gd": 0.05, "adagrad": 0.01, "rmsprop": 1e-3, "momentum": 0.02}


def _lr(model, pairwise, opt):
    """Learning rates that keep one epoch stable: pairwise losses are sums over the batch (pointwise cross entropy is
    a mean), and TransRec's g takes the gradient of every sample."""
    if not pairwise:
        return LR[opt]
    small = {"fpmc": {"gd": 1e-3, "momentum": 5e-4}, "transrec": {"gd": 1e-4, "momentum": 1e-4}}[model]
    return small.get(opt, LR[opt])


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def host(t):
    return t.cpu().numpy()


def ml100k_time_ordered():
    """The ratio-0.8 by-time split of ml-100k the reference made (kat_split_ml100k.npz), users and items remapped to
    dense ids, as a Dataset with its time matrix: 79 424 (user, recent, next) instances at high_order = 1."""
    from neurec_b200.data import Dataset
    z = np.load(os.path.join(GOLDEN, "kat_split_ml100k.npz"))
    n = int(z["n"])
    users = np.unique(z["user"], return_inverse=True)[1]
    items = np.unique(z["item"], return_inverse=True)[1]
    times = z["time"].astype(np.float64)
    train = np.unpackbits(z["ratio"])[:n].astype(bool)
    shape = (int(users.max()) + 1, int(items.max()) + 1)
    mk = lambda m, data: sp.csr_matrix((data[m], (users[m], items[m])), shape=shape)
    ones = np.ones(n, np.float32)
    return Dataset.from_csr("ml-100k", mk(train, ones), mk(~train, ones), time_matrix=mk(train, times))


@pytest.fixture(scope="module")
def ml100k_seq():
    return ml100k_time_ordered()


def _tables(model, rs, nu, ni, d, scale=0.1):
    if model == "fpmc":
        return [(rs.randn(nu, d) * scale).astype(np.float32)] + [(rs.randn(ni, d) * scale).astype(np.float32)
                                                                 for _ in range(3)]
    return [(rs.randn(nu, d) * scale).astype(np.float32), (rs.randn(ni, d) * scale).astype(np.float32),
            (rs.randn(ni) * scale).astype(np.float32), (rs.randn(1, d) * scale).astype(np.float32)]


def _touched(model, nu, ni):
    z = lambda n: torch.zeros(n, dtype=torch.int32, device="cuda")
    return (z(nu), z(ni), z(ni))


# --------------------------------------------------------------------------------------------- gradient kernels
@pytest.mark.parametrize("batch", [1, 1000])
@pytest.mark.parametrize("d", [1, 7, 16, 50, 64, 128, 256])
@pytest.mark.parametrize("pairwise,loss", MODES)
@pytest.mark.parametrize("model", ["fpmc", "transrec"])
def test_grad_kernel_vs_restatement(model, pairwise, loss, d, batch):
    """Loss within rel 1e-5; gradients within 2e-5 of the largest gradient entry (fp32 atomics sum duplicate ids in
    another order than np.add.at); accumulators are added into; the touched sets are exactly the documented ones."""
    from neurec_b200 import ops
    rs = np.random.RandomState(d * 7 + batch)
    nu, ni = 300, 500
    tabs = _tables(model, rs, nu, ni, d)
    users, recent, items = rs.randint(0, nu, batch), rs.randint(0, ni, batch), rs.randint(0, ni, batch)
    third = rs.randint(0, ni, batch).astype(np.int32) if pairwise else (rs.rand(batch) < 0.3).astype(np.float32)
    users, recent, items = (a.astype(np.int32) for a in (users, recent, items))
    for reg in (0.0, 0.01):
        fn = seq_math.fpmc_grad if model == "fpmc" else seq_math.transrec_grad
        want_l, want_g, want_t = fn(*tabs, users, recent, items, third, pairwise, loss, reg)
        base = [(rs.randn(*t.shape) * 0.01).astype(np.float32) for t in tabs]     # accumulators are added into
        dt = [dev(t) for t in tabs]
        g = [dev(b) for b in base]
        tch = _touched(model, nu, ni)
        for t in tch:
            t.fill_(3)
        out = torch.full((1,), 0.5, device="cuda")
        args = [dev(users), dev(recent), dev(items), dev(third), pairwise, loss, reg]
        if model == "fpmc":
            ops.fpmc_grad(*dt, *args, *g, *tch, 9, out)
        else:
            ops.transrec_grad(*dt, *args, *g, *tch, 9, ops.transrec_work(d), out)
        got_l = out.item() - 0.5
        assert abs(got_l - float(want_l)) <= 1e-5 * abs(float(want_l)) + 1e-6, (got_l, want_l)
        scale = max(float(np.abs(w).max()) for w in want_g)
        for name, gg, b, w in zip("0123", g, base, want_g):
            err = np.abs((host(gg) - b).reshape(w.shape) - w).max()
            assert err <= 2e-5 * max(1.0, scale), (name, err, scale)
        for t, w in zip(tch, want_t):
            h = host(t)
            assert np.array_equal(h == 9, w) and np.all(h[~w] == 3)


def test_grad_kernel_rejects_without_writing():
    from neurec_b200 import ops
    rs = np.random.RandomState(0)
    tabs = [dev(t) for t in _tables("transrec", rs, 5, 6, 8)]
    g = [torch.zeros_like(t) for t in tabs]
    ids = dev(np.zeros(4, np.int32))
    out = torch.zeros(1, device="cuda")
    for bad in ("cross_entropy", "hinge"):
        with pytest.raises(ValueError, match="suitable loss"):
            ops.transrec_grad(*tabs, ids, ids, ids, ids if bad == "cross_entropy" else dev(np.zeros(4, np.float32)),
                              bad == "cross_entropy", bad, 0.1, *g, *_touched("transrec", 5, 6), 1,
                              ops.transrec_work(8), out)
    torch.cuda.synchronize()
    assert all(float(t.abs().sum()) == 0 for t in g) and out.item() == 0


# --------------------------------------------------------------------------------------------- fused epochs
def _epoch(ds, pairwise, bs, num_neg=4, first_epoch=11):
    from neurec_b200.data import sampler as smp
    smp.reseed(first_epoch)
    if pairwise:
        s = smp.TimeOrderPairwiseSampler(ds, high_order=1, neg_num=1, batch_size=bs, shuffle=True)
    else:
        s = smp.TimeOrderPointwiseSampler(ds, high_order=1, neg_num=num_neg, batch_size=bs, shuffle=True)
    return s, s.device_epoch()


def _run_epoch(model, dt, grads, touched, slots, epoch, bs, pairwise, loss, reg, opt, lr, lr_t, stamp, work):
    from neurec_b200 import ops
    users, recent, items, third = epoch
    steps = (users.numel() + bs - 1) // bs
    step_loss = torch.zeros(steps, device="cuda")
    s0, s1 = [s[0] for s in slots], [s[1] for s in slots]
    args = (users, recent, items, third, bs, pairwise, loss, reg, opt, lr_t, tf_math.DEFAULT_HYPER[opt](lr), grads,
            touched, s0, s1, stamp)
    if model == "fpmc":
        n = ops.fpmc_train_epoch(*dt, *args, step_loss)
    else:
        n = ops.transrec_train_epoch(*dt, *args, work, step_loss)
    assert n == steps
    return host(step_loss)


@pytest.mark.parametrize("opt", ["adam", "gd", "adagrad", "rmsprop", "momentum"])
@pytest.mark.parametrize("pairwise", [True, False])
@pytest.mark.parametrize("model", ["fpmc", "transrec"])
def test_train_epoch_vs_trainer_on_ml100k(ml100k_seq, model, pairwise, opt):
    """One epoch of the time-ordered ml-100k train set (79 424 instances; pointwise x5 with 4 negatives) at the
    model's default width and batch size, fed identically to the kernels and to the fp32 trainer."""
    from neurec_b200 import ops
    ds = ml100k_seq
    nu, ni = ds.num_users, ds.num_items
    d, bs = (16, 512) if model == "fpmc" else (50, 1024)
    loss = "bpr" if pairwise else "cross_entropy"
    lr, reg = _lr(model, pairwise, opt), 0.01
    rs = np.random.RandomState(3)
    tabs = _tables(model, rs, nu, ni, d)
    sampler, epoch = _epoch(ds, pairwise, bs)
    assert len(sampler._users_np) == 79424 and epoch[0].numel() == 79424 * (1 if pairwise else 5)
    ep_h = [host(t) for t in epoch]
    Trainer = seq_math.FPMCTrainer if model == "fpmc" else seq_math.TransRecTrainer
    tr = Trainer(*tabs, learner=opt, lr=lr, loss=loss, reg=reg, pairwise=pairwise)
    want = tr.epoch(*ep_h, bs)
    steps = len(want)
    dt = [dev(t) for t in tabs]
    i0, i1 = tf_math.SLOT_INIT[opt]
    mk = lambda a, v: None if v is None else torch.full_like(a, v)
    slots = [(mk(t, i0), mk(t, i1)) for t in dt]
    grads = [torch.zeros_like(t) for t in dt]
    touched = _touched(model, nu, ni)
    work = ops.transrec_work(d)
    lr_t = tf_math.adam_lr_t(lr, steps) if opt == "adam" else np.full(steps, lr, np.float32)
    got = _run_epoch(model, dt, grads, touched, slots, epoch, bs, pairwise, loss, reg, opt, lr, lr_t, 1, work)
    assert np.allclose(got, want, rtol=1e-4)
    for i, (t, ref, t0) in enumerate(zip(dt, tr.vars, tabs)):
        assert np.abs(host(t).reshape(ref.shape) - ref).max() < 3e-5, i
        assert np.abs(ref - t0).max() > 1e-5, i                         # every variable moved
    assert all(float(g.abs().max()) == 0 for g in grads)                 # the optimizer launch consumes the gradients
    if model == "transrec" and opt == "momentum":
        # an item that occurs only as the recent item of a whole epoch: its Q row moves, its bias stays bit-unchanged
        # although it has momentum from the first epoch (b's touched set is the next items and negatives only)
        _, ep2 = _epoch(ds, pairwise, bs, first_epoch=12)
        users2, recent2, items2, third2 = (host(t) for t in ep2)
        x = int(recent2[0])
        items2 = np.where(items2 == x, (x + 1) % ni, items2).astype(np.int32)
        if pairwise:
            third2 = np.where(third2 == x, (x + 2) % ni, third2).astype(np.int32)
        ep2 = [dev(a) for a in (users2, recent2, items2, third2)]
        assert float(slots[2][0][x]) != 0.0
        B1, Q1, trB1 = host(dt[2]).copy(), host(dt[1]).copy(), tr.vars[2].copy()
        want2 = tr.epoch(users2, recent2, items2, third2, bs)
        got2 = _run_epoch(model, dt, grads, touched, slots, ep2, bs, pairwise, loss, reg, opt, lr,
                          np.full(len(want2), lr, np.float32), 1 + steps, work)
        assert np.allclose(got2, want2, rtol=1e-4)
        assert host(dt[2])[x] == B1[x] and tr.vars[2][x] == trB1[x]
        assert np.abs(host(dt[1])[x] - Q1[x]).max() > 0
        assert np.abs(host(dt[2]) - tr.vars[2]).max() < 3e-5


@pytest.mark.parametrize("opt", ["adam", "rmsprop"])
def test_transrec_global_takes_the_dense_update(opt):
    """g's gradient is a dense tensor: after each step g equals, bit for bit, the Apply* formula applied to the
    gradient the kernel computed (its cross-CTA sum has one fixed order, so a second call gives the same bits), and
    the IndexedSlices formula gives other bits."""
    from neurec_b200 import ops
    rs = np.random.RandomState(4)
    nu, ni, d, bs, lr, reg = 200, 300, 50, 1024, LR[opt], 0.01
    tabs = _tables("transrec", rs, nu, ni, d)
    dt = [dev(t) for t in tabs]
    i0, i1 = tf_math.SLOT_INIT[opt]
    mk = lambda a, v: None if v is None else torch.full_like(a, v)
    slots = [(mk(t, i0), mk(t, i1)) for t in dt]
    grads = [torch.zeros_like(t) for t in dt]
    touched = _touched("transrec", nu, ni)
    work = ops.transrec_work(d)
    G = tabs[3].reshape(-1).copy()
    dense_s = [np.full(d, i0, np.float32), np.full(d, i1, np.float32)]
    Gs, sparse_s = G.copy(), [a.copy() for a in dense_s]
    lr_t = tf_math.adam_lr_t(lr, 4)
    for step in range(4):
        ids = [rs.randint(0, n, bs).astype(np.int32) for n in (nu, ni, ni, ni)]
        batch = [dev(a) for a in ids]
        gG = [torch.zeros_like(t) for t in dt]
        ops.transrec_grad(*dt, *batch, True, "bpr", reg, *gG, *_touched("transrec", nu, ni), 1, work,
                          torch.zeros(1, device="cuda"))
        g = host(gG[3]).reshape(-1)
        hyper = tf_math.DEFAULT_HYPER[opt](lr)
        if opt == "adam":
            hyper[0] = lr_t[step]
        tf_math.opt_apply(opt, G, g, dense_s[0], dense_s[1], None, hyper, dense_var=True)
        tf_math.opt_apply(opt, Gs, g, sparse_s[0], sparse_s[1], None, hyper, dense_var=False)
        _run_epoch("transrec", dt, grads, touched, slots, batch, bs, True, "bpr", reg, opt, lr, lr_t[step:step + 1],
                   1 + step, work)
        assert np.array_equal(host(dt[3]).reshape(-1), G), step
    assert not np.array_equal(G, Gs)


# --------------------------------------------------------------------------------------------- score kernels
@pytest.mark.parametrize("rows", [1, 13, 100])
@pytest.mark.parametrize("d", [1, 7, 16, 50, 256])
@pytest.mark.parametrize("model", ["fpmc", "transrec"])
def test_score_kernel_vs_fp64(model, d, rows):
    """All 1 682 items (not a multiple of the 256-item tile) for row counts around the 8-row group.  Tolerance: fp32
    summation over d terms, relative to the sum of the terms' magnitudes."""
    from neurec_b200 import ops
    rs = np.random.RandomState(d + rows)
    nu, ni = 120, 1682
    tabs = _tables(model, rs, nu, ni, d, scale=0.3)
    users, recent = rs.randint(0, nu, rows).astype(np.int32), rs.randint(0, ni, rows).astype(np.int32)
    fn = ops.fpmc_scores if model == "fpmc" else ops.transrec_scores
    got = host(fn(*[dev(t) for t in tabs], dev(users), dev(recent)))
    assert got.shape == (rows, ni)
    t64 = [t.astype(np.float64) for t in tabs]
    eps = 6e-8
    if model == "fpmc":
        want = seq_math.fpmc_scores(*t64, users, recent)
        # 2d fused multiply-adds, each rounding relative to the running sum of magnitudes
        tol = 2 * eps * (2 * d + 2) * seq_math.fpmc_scores(*[np.abs(t) for t in t64], users, recent)
    else:
        want = seq_math.transrec_scores(*t64, users, recent)
        P, Q, B, G = t64
        # x = (P_u + g) + Q_l carries 2 roundings of |P_u| + |g| + |Q_l| per element; the distance then moves by at
        # most the 2-norm of those errors, and the d-term sum of squares adds (d + 2) eps of the distance itself
        m = np.sqrt(((np.abs(P[users]) + np.abs(G) + np.abs(Q[recent])) ** 2).sum(1))[:, None]
        tol = 2 * eps * (2 * m + (d + 2) * (B[None, :] - want) + np.abs(B)[None, :])
    assert np.all(np.abs(got - want) <= tol + 1e-9), np.abs(got - want).max()


def test_transrec_score_is_exactly_the_bias_at_zero_distance():
    """x = (P_u + g) + Q_l equal to Q_j scores exactly b_j (the distance is summed from differences, not expanded)."""
    from neurec_b200 import ops
    rs = np.random.RandomState(5)
    P, Q, B, G = _tables("transrec", rs, 10, 300, 50, scale=0.3)
    users, recent = np.array([3, 7], np.int32), np.array([11, 12], np.int32)
    Q[200] = (P[3] + G[0]) + Q[11]
    Q[201] = (P[7] + G[0]) + Q[12]
    got = host(ops.transrec_scores(dev(P), dev(Q), dev(B), dev(G), dev(users), dev(recent)))
    assert got[0, 200] == B[200] and got[1, 201] == B[201]
    assert np.all(got[0, np.arange(300) != 200] < B[np.arange(300) != 200])


# --------------------------------------------------------------------------------------------- plug-ins
class _Conf(dict):
    def params_str(self):
        return "test"


BASE_CONF = {"metric": ["Precision", "Recall", "NDCG", "MAP", "MRR"], "group_view": None, "topk": [10, 20],
             "test_batch_size": 128, "num_thread": 8}
MODEL_CONF = {
    "FPMC": dict(recommender="FPMC", epochs=1, batch_size=512, embedding_size=16, reg_mf=0.01, learning_rate=0.001,
                 learner="adam", is_pairwise=False, num_neg=4, loss_function="cross_entropy", init_method="uniform",
                 stddev=0.01, verbose=1),
    "TransRec": dict(recommender="TransRec", epochs=1, batch_size=1024, embedding_size=50, reg_mf=0.0,
                     learning_rate=0.001, learner="adam", is_pairwise=True, num_neg=4, loss_function="bpr",
                     init_method="tnormal", stddev=0.01, verbose=1),
}


def _plug_in(name, ds):
    from neurec_b200.model.sequential_recommender.FPMC import FPMC
    from neurec_b200.model.sequential_recommender.TransRec import TransRec
    cls = {"FPMC": FPMC, "TransRec": TransRec}[name]
    m = cls(None, ds, _Conf(BASE_CONF, **MODEL_CONF[name]))
    m.build_graph()
    return m


@pytest.mark.parametrize("name", ["FPMC", "TransRec"])
def test_plug_in_epoch_predict_and_evaluate(ml100k_seq, tmp_path, monkeypatch, name):
    from neurec_b200 import ops
    from neurec_b200.data import sampler as smp
    monkeypatch.chdir(tmp_path)
    ds = ml100k_seq
    m = _plug_in(name, ds)
    # Adam's step is m / sqrt(v): on the default 0.01-scale tables, a row gradient whose terms cancel to rounding level
    # takes a step of either sign, so the plumbing is compared on 0.1-scale tables, where both sides stay within
    # rounding of each other
    rs = np.random.RandomState(6)
    for t in m.tables():
        t.copy_(dev((rs.randn(*t.shape) * 0.1).astype(np.float32)))
    init = [host(t).copy() for t in m.tables()]
    conf = MODEL_CONF[name]
    smp.reseed(21)
    total = m._train_epoch()
    # the same epoch through the trainer, from the same initial tables
    _, epoch = _epoch(ds, conf["is_pairwise"], conf["batch_size"], conf["num_neg"], first_epoch=21)
    Trainer = seq_math.FPMCTrainer if name == "FPMC" else seq_math.TransRecTrainer
    tr = Trainer(*init, learner="adam", lr=conf["learning_rate"], loss=conf["loss_function"], reg=conf["reg_mf"],
                 pairwise=conf["is_pairwise"])
    want = tr.epoch(*[host(t) for t in epoch], conf["batch_size"])
    assert abs(total - float(want.sum(dtype=np.float64))) <= 1e-4 * abs(float(want.sum()))
    for t, ref in zip(m.tables(), tr.vars):
        assert np.abs(host(t).reshape(ref.shape) - ref).max() < 3e-5
    # predict: the score kernel from every user's last train item (by time), and the candidate path
    users = [0, 5, 17, 942]
    last = np.array([ds.get_user_train_dict(by_time=True)[u][-1] for u in users], np.int32)
    t64 = [host(t).astype(np.float64) for t in m.tables()]
    fn = seq_math.fpmc_scores if name == "FPMC" else seq_math.transrec_scores
    want_s = fn(*t64, np.asarray(users), last)
    got = m.predict(users)
    assert isinstance(got, torch.Tensor) and got.is_cuda and got.shape == (4, ds.num_items)
    kern = (ops.fpmc_scores if name == "FPMC" else ops.transrec_scores)(*m.tables(), dev(np.asarray(users, np.int32)),
                                                                          dev(last))
    assert torch.equal(got, kern)
    assert np.abs(host(got) - want_s).max() <= 1e-5 * max(1.0, np.abs(want_s).max())
    cand = [[1, 2, 3], [10], [0, 1681], [5, 5, 7]]
    for r, w, c in zip(m.predict(users, cand), host(got), cand):
        assert isinstance(r, np.ndarray) and np.array_equal(r, w[c])
    # evaluate(): the evaluator's generic route -- mask the train items, score matrix, mean of the rows
    got_s = m.evaluate()
    test_dict, train_dict = ds.get_user_test_dict(), ds.get_user_train_dict()
    test_users = list(test_dict.keys())                                  # the evaluator's row order
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
    with pytest.raises(KeyError):                                        # a user without train items
        m.predict([0, ds.num_users + 5])


# --------------------------------------------------------------------------------------------- main.py
def write_timed_dataset(path, nu=120, ni=200, seed=0):
    """A small UIRT dataset with times: every user walks a chain of items (i -> i + 1 mostly), so the next item
    depends on the previous one."""
    rs = np.random.RandomState(seed)
    rows = []
    for u in range(nu):
        start = rs.randint(ni)
        item, seen = start, set()
        for t in range(25):
            while item in seen:
                item = (item + 1) % ni
            seen.add(item)
            rows.append("%d\t%d\t%d\t%d" % (u + 1, item + 1, rs.randint(1, 6), 880000000 + 1000 * t + rs.randint(10)))
            item = (item + (1 if rs.rand() < 0.8 else rs.randint(2, 20))) % ni
    os.makedirs(path, exist_ok=True)
    with open(os.path.join(path, "toy.rating"), "w") as f:
        f.write("\n".join(rows) + "\n")


@pytest.mark.parametrize("name", ["FPMC", "TransRec"])
def test_main_runs_the_sequential_models(tmp_path, name):
    data = tmp_path / "dataset"
    write_timed_dataset(str(data))
    cmd = [sys.executable, os.path.join(ROOT, "main.py"), "--recommender=%s" % name, "--data.input.path=%s" % data,
           "--data.input.dataset=toy", "--topk=[5,10]", "--test_batch_size=64", "--epochs=6", "--learning_rate=0.01"]
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
    if name == "FPMC":        # epochs 1..N, loss per batch of the sampler (FPMC.py:106-131)
        assert [int(e[0]) for e in epochs] == [1, 2, 3, 4, 5, 6]
        assert [int(e[0]) for e in losses] == [1, 2, 3, 4, 5, 6]
        lv = [float(e[1]) for e in losses]
        assert lv[-1] < lv[0]
    else:                     # epochs 0..N-1, no loss line (TransRec.py:119-147)
        assert [int(e[0]) for e in epochs] == [0, 1, 2, 3, 4, 5]
        assert losses == []
