"""GPU parity of Caser (csrc/caser.cu) through the C ABI against the restatement in tests/caser_math.py: the gradient
kernel on every route its shapes select (nrc_caser_last_routes) against float64, bit-identical dense gradients, one
fused ml-100k epoch at the conf defaults against the fp32 restatement fed the same epoch, the query and scores
against float64, argument errors, the plug-in (epoch, predict, evaluate, checkpoint, short histories) and main.py."""
import os
import re
import subprocess
import sys

import numpy as np
import pytest
import torch

import caser_math as cm
from test_gpu_seq_window import _short_history_dataset
from test_gpu_sequential import BASE_CONF, _Conf, dev, host, ml100k_time_ordered, write_timed_dataset

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REACHED = set()
SMEM_FLOATS = 56 * 1024                     # kCaserSmemFloats
CONF = dict(recommender="Caser", lr=0.001, l2_reg=0.001, factors_num=50, seq_L=5, seq_T=3, nv=4, nh=16, dropout=0.5,
            neg_samples=3, batch_size=256, epochs=1)


@pytest.fixture(scope="module")
def ml100k_seq():
    return ml100k_time_ordered()


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _staged(d, L, nv, nh):
    F, NH = nv * d + nh * L, nh * L * (L + 1) // 2
    return cm.dense_layout(d, L, nv, nh)[1] + L * d + NH + F + 3 * d + 64 <= SMEM_FLOATS


def _vars(rs, nu, ni, d, L, nv, nh):
    P = (rs.randn(nu, d) * 0.3).astype(np.float32)
    E = (rs.randn(ni, d) * 0.3).astype(np.float32)
    W2 = (rs.randn(ni, 2 * d) * 0.3).astype(np.float32)
    b2 = (rs.randn(ni) * 0.1).astype(np.float32)
    parts = {}
    for name, _, shape in cm.dense_layout(d, L, nv, nh)[0]:
        fan = int(np.prod(shape[:-1])) if len(shape) > 1 else 1
        parts[name] = rs.randn(*shape) * (1.0 / np.sqrt(fan)) + (0.05 if len(shape) == 1 else 0.0)
    return P, E, W2, b2, cm.pack(parts, d, L, nv, nh).astype(np.float32)


def _batch(rs, B, L, T, N, nu, ni, pads):
    users = rs.randint(0, nu, B).astype(np.int32)
    seqs = rs.randint(0, ni, (B, L)).astype(np.int32)
    pos, neg = rs.randint(0, ni, (B, T)).astype(np.int32), rs.randint(0, ni, (B, N)).astype(np.int32)
    if pads:
        seqs[0, :L - 1] = ni
        pos[0, 0] = ni
        if B > 2:
            seqs[2, :] = ni
            users[1] = users[0]
            seqs[1, 0] = seqs[0, -1]
    return users, seqs, pos, neg


def _grads(P, E, W2, b2, dense):
    z = lambda a: torch.zeros(a.shape, dtype=torch.float32, device="cuda")
    return [z(P), z(E), z(W2), z(b2), z(dense)]


def _close(got, want, what, rel=2e-4):
    scale = max(float(np.abs(want).max()), 1e-6)
    err = float(np.abs(got.astype(np.float64) - want).max()) if want.size else 0.0
    assert err <= rel * scale, "%s: max error %.3g against max |want| %.3g" % (what, err, scale)


GRAD_CASES = [  # d, L, nv, nh, T, N, B (None: 2 * SMs + 5), pads, masked
    (1, 1, 1, 1, 1, 1, 1, False, False),
    (7, 2, 2, 3, 3, 3, 37, True, True),
    (50, 5, 4, 16, 3, 3, 256, True, True),
    (50, 5, 4, 16, 3, 3, None, False, True),
    (33, 16, 2, 1, 1, 63, 9, True, True),
    (256, 2, 64, 2, 3, 3, 5, False, False),
    (256, 16, 64, 64, 32, 32, 3, True, True),
]


@pytest.mark.parametrize("case", GRAD_CASES)
def test_grad_vs_fp64(case):
    """nrc_caser_grad against the float64 restatement on the fp32 inputs: every table gradient, the dense block's
    and the loss, with the staged / global weight route and the grid cap the shape selects."""
    from neurec_b200 import ops
    d, L, nv, nh, T, N, B, pads, masked = case
    B = 2 * _sms() + 5 if B is None else B
    rs = np.random.RandomState(d * 131 + L * 7 + B)
    nu, ni = 40, 97
    vars_ = _vars(rs, nu, ni, d, L, nv, nh)
    users, seqs, pos, neg = _batch(rs, B, L, T, N, nu, ni, pads)
    F = nv * d + nh * L
    keep = 0.5
    mask = (rs.rand(B, F) < keep).astype(np.float32) if masked else None
    want_loss, want = cm.loss_and_grad(*[v.astype(np.float64) for v in vars_], d, L, nv, nh, users, seqs, pos, neg,
                                       mask, keep)
    dv = [dev(v) for v in vars_]
    grads = _grads(*vars_)
    grads[4].fill_(7.0)                                                  # overwritten, not accumulated
    work = ops.caser_work(d, L, nv, nh, B)
    loss = torch.zeros(1, device="cuda")
    ops.caser_grad(*dv, dev(users), dev(seqs), dev(pos), dev(neg), nv, nh, None if mask is None else dev(mask), keep,
                   grads, work, loss)
    torch.cuda.synchronize()
    for name, g, w in zip(("P", "E", "W2", "b2", "dense"), grads, want):
        _close(host(g), w, name)
    assert abs(float(loss) - want_loss) <= 1e-5 * max(1.0, abs(want_loss))
    r = ops.caser_last_routes()
    cap = 2 * _sms()
    staged = _staged(d, L, nv, nh)
    assert r["grad"] == dict(staged=int(staged), grid_x=min(B, cap), grid_y=-1, capped=int(B > cap), window=L,
                             masked=int(masked))
    assert r["wgrad"]["grid_x"] == (cm.dense_layout(d, L, nv, nh)[1] + 255) // 256
    assert r["wgrad"]["grid_y"] == (B + 31) // 32
    REACHED.add(("grad", staged, B > cap, masked))


def test_dense_gradient_is_the_same_bits_on_every_call():
    from neurec_b200 import ops
    d, L, nv, nh, T, N, B = 50, 5, 4, 16, 3, 3, 256
    rs = np.random.RandomState(11)
    vars_ = _vars(rs, 60, 200, d, L, nv, nh)
    batch = [dev(a) for a in _batch(rs, B, L, T, N, 60, 200, True)]
    mask = dev((rs.rand(B, nv * d + nh * L) < 0.5).astype(np.float32))
    dv = [dev(v) for v in vars_]
    work = ops.caser_work(d, L, nv, nh, B)
    outs = []
    for _ in range(3):
        grads = _grads(*vars_)
        ops.caser_grad(*dv, *batch, nv, nh, mask, 0.5, grads, work)
        outs.append(host(grads[4]).copy())
    assert np.array_equal(outs[0], outs[1]) and np.array_equal(outs[0], outs[2])


def _restated_epoch(m_users, m_seqs, m_pos, train_ptr, train_idx, N, ni, seed, epoch):
    """The device epoch reproduced through the existing primitives with the documented keys."""
    from neurec_b200 import ops
    neg = ops.sample_negatives(train_ptr, train_idx, m_users, N, ni, seed, epoch)
    perm = ops.shuffle_perm(m_users.numel(), seed, epoch)
    return [ops.gather_rows_i32(a, perm) for a in (m_users, m_seqs, m_pos, neg)]


def _masks(n, batch_size, F, keep, seed, epoch):
    from neurec_b200 import ops
    out = []
    for s in range((n + batch_size - 1) // batch_size):
        bs = min(batch_size, n - s * batch_size)
        out.append(host(ops.dropout_mask(bs * F, keep, seed, (epoch << 32) | s)).reshape(bs, F))
    return out


def test_epoch_vs_fp32_restatement_on_ml100k(ml100k_seq):
    """One nrc_caser_train_epoch at the conf defaults (73 766 instances, 289 steps with a short last one) against
    CaserTrainer fed the same permutation, negatives and masks."""
    from neurec_b200 import ops
    from neurec_b200.model.sequential_recommender.Caser import generate_sequences
    ds = ml100k_seq
    d, L, T, nv, nh, N, bsz, keep, reg = 50, 5, 3, 4, 16, 3, 256, 0.5, 1e-3
    nu, ni = ds.num_users, ds.num_items
    td = ds.get_user_train_dict(by_time=True)
    users, seqs, pos, _ = generate_sequences(td, L, T, ni)
    ptr = np.zeros(nu + 1, np.int64)
    for u, it in td.items():
        ptr[u + 1] = len(it)
    ptr = np.cumsum(ptr)
    idx = np.concatenate([np.sort(np.asarray(td[u], np.int32)) for u in sorted(td)])
    seed, epoch = 2018, 5
    eu, es, ep, en = _restated_epoch(dev(users), dev(seqs), dev(pos), dev(ptr), dev(idx), N, ni, seed, epoch)
    n = len(users)
    masks = _masks(n, bsz, nv * d + nh * L, keep, seed, epoch)
    rs = np.random.RandomState(2)
    init = _vars(rs, nu, ni, d, L, nv, nh)
    tr = cm.CaserTrainer(*init, d, L, nv, nh, lr=1e-3, l2_reg=reg, keep=keep)
    want = tr.epoch(host(eu), host(es), host(ep), host(en), masks, bsz)
    dv = [dev(v) for v in init]
    grads = _grads(*init)
    s0, s1 = [torch.zeros_like(v) for v in dv], [torch.zeros_like(v) for v in dv]
    from oracle import tf_math
    steps = (n + bsz - 1) // bsz
    step_loss = torch.zeros(steps, device="cuda")
    got_steps = ops.caser_train_epoch(*dv, eu, es, ep, en, nv, nh, bsz, keep, reg, seed, epoch,
                                      tf_math.adam_lr_t(1e-3, steps), [1e-3, 0.9, 0.999, 1e-8], grads, s0, s1,
                                      ops.caser_work(d, L, nv, nh, bsz), step_loss)
    assert got_steps == steps == 289
    got_loss = host(step_loss).astype(np.float64)
    assert np.abs(got_loss - want).max() <= 1e-4 * np.abs(want).max(), np.abs(got_loss - want).max()
    for name, v, ref in zip(("P", "E", "W2", "b2", "dense"), dv, tr.vars):
        _close(host(v), ref.astype(np.float64), name, rel=5e-4)
    r = ops.caser_last_routes()
    assert r["reg"]["grid_x"] > 0 and r["grad"]["masked"] == 1 and r["grad"]["staged"] == 1
    REACHED.add(("reg", r["reg"]["capped"]))


@pytest.mark.parametrize("d,L,nv,nh", [(1, 1, 1, 1), (50, 5, 4, 16), (256, 16, 64, 64)])
def test_query_and_scores_vs_fp64(d, L, nv, nh):
    """[z, P_u] over each user's window (pad ids included) and the scores against W2 without the biases."""
    from neurec_b200 import ops
    rs = np.random.RandomState(d + L)
    nu, ni = 30, 301
    P, E, W2, b2, dense = _vars(rs, nu, ni, d, L, nv, nh)
    windows = rs.randint(0, ni, (nu, L)).astype(np.int32)
    windows[3, :L - 1] = ni
    windows[4, :] = ni
    users = np.array([0, 3, 4, 29, 3], np.int32)
    want_q = cm.query(P.astype(np.float64), E.astype(np.float64), dense.astype(np.float64), d, L, nv, nh, users,
                      windows[users])
    q = ops.caser_query(dev(P), dev(E), dev(W2), dev(dense), dev(users), dev(windows), nv, nh)
    _close(host(q), want_q, "query")
    s = ops.caser_scores(dev(P), dev(E), dev(W2), dev(dense), dev(users), dev(windows), nv, nh)
    _close(host(s), want_q @ W2.astype(np.float64).T, "scores")
    r = ops.caser_last_routes()["query"]
    assert r["staged"] == int(_staged(d, L, nv, nh)) and r["grid_x"] == len(users) and r["masked"] == 0
    REACHED.add(("query", bool(r["staged"])))


def test_argument_errors_on_device_tensors():
    from neurec_b200 import _lib, ops
    rs = np.random.RandomState(1)
    P, E, W2, b2, dense = _vars(rs, 5, 9, 4, 2, 1, 1)
    users, seqs, pos, neg = (dev(a) for a in _batch(rs, 3, 2, 1, 1, 5, 9, False))
    with pytest.raises(_lib.NrcError) as e:
        ops.caser_query(dev(P), dev(E), dev(W2), dev(dense), users, dev(np.zeros((5, 17), np.int32)), 1, 1)
    assert e.value.rc == _lib.NRC_E_LIMIT
    with pytest.raises(ValueError, match="keep"):
        ops.caser_grad(dev(P), dev(E), dev(W2), dev(b2), dev(dense), users, seqs, pos, neg, 1, 1,
                       torch.ones(3, 6, device="cuda"), 0.0, _grads(P, E, W2, b2, dense), ops.caser_work(4, 2, 1, 1, 3))
    with pytest.raises(TypeError):
        ops.caser_query(dev(P), dev(E), dev(W2), dev(dense), users.long(), dev(np.zeros((5, 2), np.int32)), 1, 1)


def _plug_in(ds, **over):
    from neurec_b200.model.sequential_recommender.Caser import Caser
    m = Caser(None, ds, _Conf(BASE_CONF, **dict(CONF, **over)))
    m.build_graph()
    return m


def test_plug_in_initialises_in_the_reference_order(ml100k_seq, tmp_path, monkeypatch):
    from neurec_b200.model.sequential_recommender.Caser import glorot_uniform
    monkeypatch.chdir(tmp_path)
    m = _plug_in(ml100k_seq)
    g = torch.Generator().manual_seed(2017)
    nu, ni = ml100k_seq.num_users, ml100k_seq.num_items
    for t, shape in zip(m.tables()[:3], ([nu, 50], [ni, 50], [ni, 100])):
        assert torch.equal(t.cpu(), glorot_uniform(shape, g))
    assert not m.item_biases.any()
    parts = cm.unpack(host(m.dense), 50, 5, 4, 16)
    assert np.array_equal(parts["Kv"], glorot_uniform([5, 1, 1, 4], g).numpy()) and not parts["bv"].any()
    for h in range(1, 6):
        assert np.array_equal(parts["Kh%d" % h], glorot_uniform([h, 50, 1, 16], g).numpy())
        assert not parts["bh%d" % h].any()
    assert np.array_equal(parts["W1"], glorot_uniform([280, 50], g).numpy()) and not parts["b1"].any()


def _first_step_grads(m, epoch):
    """The gradients of the first step of epoch `epoch` of plug-in m, from its current state (m is not changed)."""
    from neurec_b200 import ops
    users, seqs, pos, neg = m.device_epoch(epoch)
    bs = min(m.batch_size, users.numel())
    F = m.nv * m.factors_num + m.nh * m.seq_L
    mask = ops.dropout_mask(bs * F, 1.0 - m.dropout, 2018, epoch << 32).view(bs, F)
    grads = [torch.zeros_like(t) for t in m.tables()]
    ops.caser_grad(*m.tables(), users[:bs], seqs[:bs], pos[:bs], neg[:bs], m.nv, m.nh, mask, 1.0 - m.dropout, grads,
                   ops.caser_work(m.factors_num, m.seq_L, m.nv, m.nh, bs))
    return grads


def test_plug_in_epoch_predict_evaluate_and_checkpoint(ml100k_seq, tmp_path, monkeypatch):
    from neurec_b200 import ops
    from neurec_b200.data import sampler as smp
    from neurec_b200.util import checkpoint
    monkeypatch.chdir(tmp_path)
    ds = ml100k_seq
    m = _plug_in(ds)
    init = [host(t).copy() for t in m.tables()]
    smp.reseed(21)
    total = m._train_epoch()
    eu, es, ep, en = _restated_epoch(m._users, m._seqs, m._pos, m._train_ptr, m._train_idx, 3, ds.num_items, 2018,
                                     21)
    masks = _masks(eu.numel(), 256, 280, 0.5, 2018, 21)
    tr = cm.CaserTrainer(*init, 50, 5, 4, 16, lr=1e-3, l2_reg=1e-3, keep=0.5)
    want = tr.epoch(host(eu), host(es), host(ep), host(en), masks, 256)
    assert abs(total - float(want.sum())) <= 1e-4 * abs(float(want.sum()))
    for t, ref in zip(m.tables(), tr.vars):
        assert np.abs(host(t) - ref).max() < 5e-4 * max(1.0, np.abs(ref).max())
    # predict: every item from the user's last 5 train items by time, no biases; the candidate path
    users = [0, 5, 17, 942]
    td = ds.get_user_train_dict(by_time=True)
    windows = np.array([list(td[u])[-5:] for u in users], np.int32)
    tabs = [host(t).astype(np.float64) for t in m.tables()]
    want_s = cm.query(tabs[0], tabs[1], tabs[4], 50, 5, 4, 16, users, windows) @ tabs[2].T
    got = m.predict(users)
    assert isinstance(got, torch.Tensor) and got.is_cuda and got.shape == (4, ds.num_items)
    _close(host(got), want_s, "predict")
    cand = [[1, 2, 3], [10], [0, 1681], [5, 5, 7]]
    for r, w, c in zip(m.predict(users, cand), host(got), cand):
        assert isinstance(r, np.ndarray) and np.array_equal(r, w[c])
    with pytest.raises(KeyError):
        m.predict([0, ds.num_users + 5])
    result = m.evaluate()
    vals = [float(x) for x in result.split()]
    assert len(vals) == 10 and all(0.0 <= v <= 1.0 for v in vals)
    # checkpoint: tables, the dense block, Adam slots and beta powers and the epoch counter come back, so the resumed
    # epoch draws the same instances, negatives and masks from the same state: its first step's dense gradient (summed
    # in a fixed order) is the same bits, and its loss is the continuing run's.  The tables' row gradients are summed
    # by atomics in a varying order, and max-pool and relu switches let two runs drift apart over an epoch, so the
    # tables after the epoch are not compared bit for bit.
    path = str(tmp_path / "caser.ckpt")
    checkpoint.save(m, path)
    saved = torch.load(path, map_location="cpu")["tensors"]
    assert {"dense", "item_embeddings", "_slots0.4", "_slots1.4"} <= set(saved)
    next_epoch = smp._EPOCH_COUNTER.value
    ga = _first_step_grads(m, next_epoch)
    la = m._train_epoch()
    smp.reseed(0)
    b = _plug_in(ds)
    checkpoint.load(b, path)
    live = checkpoint.state_dict(b)["tensors"]
    for k, v in saved.items():
        if k in live and k != "_step_loss":
            assert torch.equal(live[k], v), k
    assert smp._EPOCH_COUNTER.value == next_epoch
    assert torch.equal(_first_step_grads(b, next_epoch)[4], ga[4])
    lb = b._train_epoch()
    assert abs(la - lb) <= 1e-5 * abs(la)


def test_plug_in_short_histories(tmp_path, monkeypatch):
    """Users with fewer than seq_L + seq_T train items get one pre-padded instance, users with fewer than seq_T have
    the pad id among their positives; the epoch stays finite and predict reads the pre-padded windows."""
    monkeypatch.chdir(tmp_path)
    ds, nu = _short_history_dataset(3)
    m = _plug_in(ds, seq_L=3, seq_T=3, batch_size=16)
    ni = ds.num_items
    assert int((host(m._pos) == ni).sum()) > 0 and int((host(m._seqs) == ni).sum()) > 0
    total = m._train_epoch()
    assert np.isfinite(total)
    for t in m.tables():
        assert torch.isfinite(t).all()
    td = ds.get_user_train_dict(by_time=True)
    users = sorted(td)
    got = host(m.predict(users))
    tabs = [host(t).astype(np.float64) for t in m.tables()]
    windows = np.array([([ni] * 3 + list(td[u]))[-3:] for u in users], np.int32)
    _close(got, cm.query(tabs[0], tabs[1], tabs[4], 50, 3, 4, 16, users, windows) @ tabs[2].T, "short predict")
    with pytest.raises(KeyError):
        m.predict([users[0], nu - 1])


def test_main_runs_caser(tmp_path):
    data = tmp_path / "dataset"
    write_timed_dataset(str(data))
    cmd = [sys.executable, os.path.join(ROOT, "main.py"), "--recommender=Caser", "--data.input.path=%s" % data,
           "--data.input.dataset=toy", "--topk=[5,10]", "--test_batch_size=64", "--epochs=3", "--lr=0.01"]
    for f in ("NeuRec.properties", "conf"):
        os.symlink(os.path.join(ROOT, f), tmp_path / f)
    r = subprocess.run(cmd, cwd=tmp_path, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    out = r.stdout
    assert "metrics:\tPrecision@5 " in out and "NDCG@10" in out
    epochs = re.findall(r"epoch (\d+):\t([0-9.\t ]+)", out)
    assert [int(e[0]) for e in epochs] == [0, 1, 2]
    vals = np.array([[float(x) for x in e[1].split()] for e in epochs])
    assert vals.shape[1] == 10 and np.isfinite(vals).all() and (vals >= 0).all() and (vals <= 1).all()
    assert "[iter" not in out                                           # train_model logs no loss


def test_every_route_was_reached():
    """Runs last in this file: the gradient kernel staged and not, capped and not, with and without a mask, and the
    query kernel on both weight routes."""
    if len(REACHED) == 0:
        pytest.skip("the route tests did not run in this session")
    grads = {r for r in REACHED if r[0] == "grad"}
    assert {r[1] for r in grads} == {True, False} and {r[2] for r in grads} == {True, False}
    assert {r[3] for r in grads} == {True, False}
    assert ("query", True) in REACHED and ("query", False) in REACHED
