"""GPU parity of the device-resident epoch (csrc/epoch.cu): the shuffle bijection, the epoch
builder and the persistent one-launch-per-epoch MF trainer against their CPU restatements
(oracle.shuffle_perm / oracle.epoch_build / tf_math.MFTrainer).  Replaces data/sampler.py:71-90,
121-147, 189-206, util/data_iterator.py:45-63,133-155 and the batch loop of MF.py:92-108."""
import numpy as np
import pytest
import torch

import oracle
from oracle import tf_math

pytestmark = pytest.mark.gpu


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


@pytest.mark.parametrize("n", [1, 2, 3, 5, 64, 257, 4097, 80367, 401835, 1 << 20])
def test_shuffle_perm_bit_exact(n):
    from neurec_b200 import ops
    for seed, epoch in ((2018, 0), (7, 123456789012)):
        got = ops.shuffle_perm(n, seed, epoch).cpu().numpy()
        assert np.array_equal(got, oracle.shuffle_perm(n, seed, epoch))
    assert np.array_equal(ops.shuffle_perm(n, 1, 1, shuffle=False).cpu().numpy(), np.arange(n))


def _flat(d):
    users = np.repeat(np.arange(d["num_users"], dtype=np.int32), np.diff(d["train_indptr"]))
    return users, d["train_indices"]


@pytest.mark.parametrize("pairwise,neg_num,shuffle", [(True, 1, True), (True, 3, True), (True, 1, False),
                                                      (False, 4, True), (False, 2, False), (False, 1, True)])
def test_epoch_build_bit_exact(ml100k, pairwise, neg_num, shuffle):
    from neurec_b200 import ops
    d = ml100k
    pu, pi = _flat(d)
    ni = d["num_items"]
    args = (dev(d["train_indptr"]), dev(d["train_indices"]), dev(pu), dev(pi), neg_num, ni, pairwise, shuffle, 2018, 5)
    u, i, t = (x.cpu().numpy() for x in ops.epoch_build(*args))
    wu, wi, wt = oracle.epoch_build(d["train_indptr"], d["train_indices"], pu, pi, neg_num, ni, pairwise, shuffle, 2018, 5)
    assert np.array_equal(u, wu) and np.array_equal(i, wi) and np.array_equal(t, wt)
    assert t.dtype == (np.int32 if pairwise else np.float32)
    # any window of the epoch is the same slice (how drop_last and multi-call epochs are cut)
    n = len(wu)
    u2, i2, t2 = (x.cpu().numpy() for x in ops.epoch_build(*args, first=1000, n_out=n - 3000))
    assert np.array_equal(u2, wu[1000:n - 2000]) and np.array_equal(i2, wi[1000:n - 2000]) and np.array_equal(t2, wt[1000:n - 2000])
    with pytest.raises(ValueError):
        ops.epoch_build(*args, first=10, n_out=n)


def _mf_state(nu, ni, dim, learner, seed=3):
    rs = np.random.RandomState(seed)
    U0 = (rs.randn(nu, dim) * 0.05).astype(np.float32)
    V0 = (rs.randn(ni, dim) * 0.05).astype(np.float32)
    i0, i1 = tf_math.SLOT_INIT[learner]
    dU, dV = dev(U0), dev(V0)
    mk = lambda a, v: None if v is None else torch.full_like(a, v)
    st = dict(U=dU, V=dV, gU=torch.zeros_like(dU), gV=torch.zeros_like(dV),
              tU=torch.zeros(nu, dtype=torch.int32, device="cuda"), tV=torch.zeros(ni, dtype=torch.int32, device="cuda"),
              s0U=mk(dU, i0), s1U=mk(dU, i1), s0V=mk(dV, i0), s1V=mk(dV, i1),
              pows=torch.tensor([0.9, 0.999], device="cuda") if learner == "adam" else None)
    return U0, V0, st


def _run_fused(ops, d, st, pairwise, neg_num, bs, loss, reg, learner, lr, seed, epoch, first_step, num_steps,
               first_stamp, ws, step_loss, drop_last=False, shuffle=True):
    pu, pi = _flat(d)
    ops.mf_epoch_fused(st["U"], st["V"], dev(d["train_indptr"]), dev(d["train_indices"]), dev(pu), dev(pi), neg_num,
                       pairwise, shuffle, drop_last, seed, epoch, bs, first_step, num_steps, loss, reg, learner,
                       tf_math.DEFAULT_HYPER[learner](lr), st["pows"], st["gU"], st["gV"], st["tU"], st["tV"],
                       st["s0U"], st["s1U"], st["s0V"], st["s1V"], first_stamp, ws[0], ws[1], ws[2], step_loss)


@pytest.mark.parametrize("pairwise,loss,learner,dim,bs,reg,steps", [
    (True, "bpr", "adam", 64, 512, 0.0, 157),          # BASELINE config 1: a FULL ml-100k epoch
    (True, "bpr", "adam", 128, 512, 1e-3, 12),
    (True, "hinge", "gd", 32, 300, 1e-3, 9),
    (True, "square", "momentum", 20, 512, 0.0, 7),     # generic-dim path, touched-row optimizer
    (False, "cross_entropy", "adam", 32, 256, 0.0, 40),
    (False, "square", "adagrad", 64, 1000, 1e-4, 6),
    (False, "cross_entropy", "rmsprop", 24, 256, 1e-4, 6),
])
def test_fused_epoch_matches_the_oracle_trainer(ml100k, pairwise, loss, learner, dim, bs, reg, steps):
    from neurec_b200 import ops
    d = ml100k
    nu, ni = d["num_users"], d["num_items"]
    neg_num = 1 if pairwise else 4
    lr = 1e-3 if learner == "adam" else 1e-2
    U0, V0, st = _mf_state(nu, ni, dim, learner)
    pu, pi = _flat(d)
    wu, wi, wt = oracle.epoch_build(d["train_indptr"], d["train_indices"], pu, pi, neg_num, ni, pairwise, True, 2018, 3)
    n = len(wu)
    total_steps = (n + bs - 1) // bs
    assert steps <= total_steps
    if pairwise:
        wt = wt[:, 0]
    tr = tf_math.MFTrainer(U0, V0, learner, lr, loss, reg, pairwise)
    want = tr.epoch(wu[:steps * bs], wi[:steps * bs], wt[:steps * bs], bs)
    ws = tuple(torch.empty(n, dtype=torch.int32, device="cuda") for _ in range(3))
    step_loss = torch.full((total_steps,), 7.0, device="cuda")
    _run_fused(ops, d, st, pairwise, neg_num, bs, loss, reg, learner, lr, 2018, 3, 0, steps, 1, ws, step_loss)
    got = step_loss.cpu().numpy()
    # the epoch arrays the kernel built for itself are the oracle's
    assert np.array_equal(ws[0].cpu().numpy(), wu) and np.array_equal(ws[1].cpu().numpy(), wi)
    third = ws[2].cpu().numpy()
    assert np.array_equal(third if pairwise else third.view(np.float32), wt)
    assert np.allclose(got[:steps], want, rtol=2e-4, atol=1e-5), np.abs(got[:steps] - want).max()
    assert (got[steps:] == 0).all()                                     # zeroed for the whole epoch
    tol = 2e-5 if steps > 100 else 5e-6
    assert np.abs(st["U"].cpu().numpy() - tr.U).max() < tol and np.abs(st["V"].cpu().numpy() - tr.V).max() < tol
    assert float(st["gU"].abs().max()) == 0.0 and float(st["gV"].abs().max()) == 0.0   # accumulators left clean
    if learner == "adam":                                              # beta powers advanced like TF's variables
        p1, p2 = np.float32(0.9), np.float32(0.999)
        for _ in range(steps):
            p1, p2 = np.float32(p1 * np.float32(0.9)), np.float32(p2 * np.float32(0.999))
        assert np.array_equal(st["pows"].cpu().numpy(), np.array([p1, p2], np.float32))


def test_fused_epoch_can_be_cut_into_calls_and_honours_drop_last(ml100k):
    from neurec_b200 import ops
    d = ml100k
    nu, ni, dim, bs = d["num_users"], d["num_items"], 64, 4096
    pu, pi = _flat(d)
    n = len(pu)
    total = n // bs                                                      # drop_last: 19 full batches
    U0, V0, a = _mf_state(nu, ni, dim, "adam")
    _, _, b = _mf_state(nu, ni, dim, "adam")
    mk = lambda: tuple(torch.empty(n, dtype=torch.int32, device="cuda") for _ in range(3))
    la, lb = torch.zeros(total, device="cuda"), torch.zeros(total, device="cuda")
    _run_fused(ops, d, a, True, 1, bs, "bpr", 0.0, "adam", 1e-3, 11, 0, 0, total, 1, mk(), la, drop_last=True)
    wsb = mk()
    _run_fused(ops, d, b, True, 1, bs, "bpr", 0.0, "adam", 1e-3, 11, 0, 0, 5, 1, wsb, lb, drop_last=True)
    _run_fused(ops, d, b, True, 1, bs, "bpr", 0.0, "adam", 1e-3, 11, 0, 5, total - 5, 6, wsb, lb, drop_last=True)
    assert np.allclose(la.cpu().numpy(), lb.cpu().numpy(), rtol=1e-5)
    assert np.abs(a["U"].cpu().numpy() - b["U"].cpu().numpy()).max() < 1e-6
    wu, wi, wt = oracle.epoch_build(d["train_indptr"], d["train_indices"], pu, pi, 1, ni, True, True, 11, 0)
    tr = tf_math.MFTrainer(U0, V0, "adam", 1e-3, "bpr", 0.0, True)
    want = tr.epoch(wu[:total * bs], wi[:total * bs], wt[:total * bs, 0], bs)
    assert np.allclose(la.cpu().numpy(), want, rtol=2e-4)
    with pytest.raises(ValueError):                                      # one step past the trimmed epoch
        _run_fused(ops, d, b, True, 1, bs, "bpr", 0.0, "adam", 1e-3, 11, 0, total, 1, 1, wsb, lb, drop_last=True)
    with pytest.raises(ValueError):                                      # MF.py:88: one negative per positive
        _run_fused(ops, d, b, True, 2, bs, "bpr", 0.0, "adam", 1e-3, 11, 0, 0, 1, 1, wsb, lb)
    with pytest.raises(ValueError):                                      # learner.py:27-28
        _run_fused(ops, d, b, True, 1, bs, "cross_entropy", 0.0, "adam", 1e-3, 11, 0, 0, 1, 1, wsb, lb)


def test_fused_epoch_equals_the_two_kernel_epoch(ml100k):
    """Same epoch through nrc_epoch_build + nrc_mf_train_epoch (a launch pair per step) and through the
    persistent kernel: same losses and tables up to the order of the atomics."""
    from neurec_b200 import ops
    d = ml100k
    nu, ni, dim, bs = d["num_users"], d["num_items"], 64, 512
    pu, pi = _flat(d)
    _, _, a = _mf_state(nu, ni, dim, "adam")
    _, _, b = _mf_state(nu, ni, dim, "adam")
    u, i, t = ops.epoch_build(dev(d["train_indptr"]), dev(d["train_indices"]), dev(pu), dev(pi), 1, ni, True, True, 4, 9)
    steps = (len(pu) + bs - 1) // bs
    la, lb = torch.zeros(steps, device="cuda"), torch.zeros(steps, device="cuda")
    ops.mf_train_epoch(a["U"], a["V"], u, i, t.view(-1), bs, True, "bpr", 0.0, "adam", tf_math.adam_lr_t(1e-3, steps),
                       [1e-3, 0.9, 0.999, 1e-8], a["gU"], a["gV"], a["tU"], a["tV"], a["s0U"], a["s1U"], a["s0V"],
                       a["s1V"], 1, la)
    ws = tuple(torch.empty(len(pu), dtype=torch.int32, device="cuda") for _ in range(3))
    _run_fused(ops, d, b, True, 1, bs, "bpr", 0.0, "adam", 1e-3, 4, 9, 0, steps, 1, ws, lb)
    assert np.allclose(la.cpu().numpy(), lb.cpu().numpy(), rtol=1e-4)
    assert np.abs(a["U"].cpu().numpy() - b["U"].cpu().numpy()).max() < 2e-6
    assert np.abs(a["V"].cpu().numpy() - b["V"].cpu().numpy()).max() < 2e-6


@pytest.mark.parametrize("dim", [128, 64, 32])
def test_csr_fed_sgd_kernel_equals_build_then_step(dim):
    """nrc_mf_bpr_sgd_epoch (sampler + shuffle + in-place BPR/SGD in one kernel, BASELINE config 5)
    against (a) nrc_epoch_build + nrc_mf_bpr_sgd_fused on the same positions and (b) the numpy
    restatement, on an epoch without repeated rows (where the in-place step is order-free)."""
    from neurec_b200 import ops
    from neurec_b200.util import peer
    nu, ni, n = 300, 400_000, 300
    rs = np.random.RandomState(dim)
    tp = np.arange(nu + 1, dtype=np.int64)                      # one positive per user
    pos_items = rs.permutation(ni)[:nu].astype(np.int32)
    pos_users = np.arange(nu, dtype=np.int32)
    for seed in range(50):                                       # a duplicate-free epoch (checked on the host)
        wu, wi, wj = oracle.epoch_build(tp, pos_items, pos_users, pos_items, 1, ni, True, True, seed, 2)
        if len(np.unique(np.concatenate([wi, wj[:, 0]]))) == 2 * n:
            break
    else:
        pytest.skip("no duplicate-free epoch found")
    U0 = (rs.randn(nu, dim) * 0.1).astype(np.float32)
    V0 = (rs.randn(ni, dim) * 0.1).astype(np.float32)
    lr, reg = 0.05, 0.01
    # (b) numpy
    pu, qi, qj = U0[wu], V0[wi], V0[wj[:, 0]]
    x = (pu * qi).sum(1) - (pu * qj).sum(1)
    wl, g = tf_math.pairwise_loss_and_grad("bpr", x)
    g = g[:, None].astype(np.float32)
    Uw, Vw = U0.copy(), V0.copy()
    Uw[wu] -= np.float32(lr) * (g * (qi - qj) + np.float32(reg) * pu)
    Vw[wi] -= np.float32(lr) * (g * pu + np.float32(reg) * qi)
    Vw[wj[:, 0]] -= np.float32(lr) * (-g * pu + np.float32(reg) * qj)
    want_loss = float(np.sum(wl, dtype=np.float64) + 0.5 * reg * np.sum(pu * pu + qi * qi + qj * qj, dtype=np.float64))
    # CSR-fed kernel, cut into two calls
    dU, dV = dev(U0), dev(V0)
    loss = torch.zeros(1, device="cuda")
    a = (dev(tp), dev(pos_items), dev(pos_users), dev(pos_items), ni, True, seed, 2)
    ops.mf_bpr_sgd_epoch(dU, peer.single(dV), *a, 0, 111, lr, reg, loss)
    ops.mf_bpr_sgd_epoch(dU, peer.single(dV), *a, 111, n - 111, lr, reg, loss)
    assert np.abs(dU.cpu().numpy() - Uw).max() < 2e-6 and np.abs(dV.cpu().numpy() - Vw).max() < 2e-6
    assert abs(float(loss) - want_loss) < 1e-3 * want_loss
    # (a) build + step
    eU, eV = dev(U0), dev(V0)
    u, i, j = ops.epoch_build(dev(tp), dev(pos_items), dev(pos_users), dev(pos_items), 1, ni, True, True, seed, 2)
    l2 = torch.zeros(1, device="cuda")
    ops.mf_bpr_sgd_fused(eU, eV, u, i, j.view(-1), lr, reg, l2)
    assert np.abs(eU.cpu().numpy() - dU.cpu().numpy()).max() < 1e-6
    assert np.abs(eV.cpu().numpy() - dV.cpu().numpy()).max() < 1e-6
    with pytest.raises(ValueError):
        ops.mf_bpr_sgd_epoch(dU, peer.single(dV), *a, 10, n, lr, reg, loss)


def test_csr_fed_sgd_kernel_with_repeated_rows_sums_every_contribution():
    """Hot rows (Zipf items, few users): in-place REDs must not lose updates -- with lr so small that
    reads of already-updated rows change the gradient only in second order, the result must match
    the sum of all per-triplet updates computed on the pre-step tables."""
    from neurec_b200 import ops
    from neurec_b200.util import peer
    nu, ni, dim = 64, 500, 128
    rs = np.random.RandomState(1)
    rows = [np.unique(rs.zipf(1.3, 40) % ni).astype(np.int32) for _ in range(nu)]
    tp, ti = oracle.lists_to_csr(rows)
    pos_users = np.repeat(np.arange(nu, dtype=np.int32), np.diff(tp))
    n = len(ti)
    U0 = (rs.randn(nu, dim) * 0.1).astype(np.float32); V0 = (rs.randn(ni, dim) * 0.1).astype(np.float32)
    lr = 1e-4
    wu, wi, wj = oracle.epoch_build(tp, ti, pos_users, ti, 1, ni, True, True, 9, 0)
    g_all = tf_math.mf_pairwise_grad(U0, V0, wu, wi, wj[:, 0], "bpr", 0.0)
    dU, dV = dev(U0), dev(V0)
    loss = torch.zeros(1, device="cuda")
    ops.mf_bpr_sgd_epoch(dU, peer.single(dV), dev(tp), dev(ti), dev(pos_users), dev(ti), ni, True, 9, 0, 0, n, lr, 0.0, loss)
    assert abs(float(loss) - float(g_all[0])) < 1e-3 * float(g_all[0])
    assert np.abs(dU.cpu().numpy() - (U0 - np.float32(lr) * g_all[1])).max() < 5e-6
    assert np.abs(dV.cpu().numpy() - (V0 - np.float32(lr) * g_all[2])).max() < 5e-6


@pytest.mark.parametrize("dim", [128, 32])
def test_replicated_head_gives_the_same_tables(dim):
    """ShardSet.enable_hot: rows [0, n_hot) are read from the replica and their deltas accumulated next to it;
    after sync_hot + writeback_hot a duplicate-free epoch leaves bit-identical tables (row + (0 + delta) = row +
    delta), and with repeated rows every contribution is summed (first-order check)."""
    from neurec_b200 import ops
    from neurec_b200.util import peer
    nu, ni, n = 300, 400_000, 300
    rs = np.random.RandomState(dim + 7)
    tp = np.arange(nu + 1, dtype=np.int64)
    pos_items = rs.permutation(ni)[:nu].astype(np.int32)
    pos_users = np.arange(nu, dtype=np.int32)
    for seed in range(50):
        wu, wi, wj = oracle.epoch_build(tp, pos_items, pos_users, pos_items, 1, ni, True, True, seed, 2)
        if len(np.unique(np.concatenate([wi, wj[:, 0]]))) == 2 * n:
            break
    else:
        pytest.skip("no duplicate-free epoch found")
    n_hot = ni // 2
    assert (wi < n_hot).any() and (wi >= n_hot).any() and (wj < n_hot).any() and (wj >= n_hot).any()
    U0 = (rs.randn(nu, dim) * 0.1).astype(np.float32); V0 = (rs.randn(ni, dim) * 0.1).astype(np.float32)
    a = (dev(tp), dev(pos_items), dev(pos_users), dev(pos_items), ni, True, seed, 2)
    dU, dV, l0 = dev(U0), dev(V0), torch.zeros(1, device="cuda")
    ops.mf_bpr_sgd_epoch(dU, peer.single(dV), *a, 0, n, 0.05, 0.01, l0)
    eU, eV, l1 = dev(U0), dev(V0), torch.zeros(1, device="cuda")
    sh = peer.single(eV).enable_hot(n_hot)
    ops.mf_bpr_sgd_epoch(eU, sh, *a, 0, n, 0.05, 0.01, l1)
    assert torch.equal(eV[:n_hot], dev(V0[:n_hot]))             # the owners' copies of replicated rows are untouched ...
    assert float(sh.hot_delta.abs().max()) > 0                  # ... their deltas wait in the accumulator
    sh.sync_hot(); sh.writeback_hot()
    assert float(sh.hot_delta.abs().max()) == 0
    assert torch.equal(eU, dU) and torch.equal(eV, dV)
    assert abs(float(l0) - float(l1)) < 1e-4 * abs(float(l0))
    # repeated rows, everything replicated
    nu, ni = 64, 512
    rows = [np.unique(rs.zipf(1.3, 40) % ni).astype(np.int32) for _ in range(nu)]
    tp, ti = oracle.lists_to_csr(rows)
    pos_users = np.repeat(np.arange(nu, dtype=np.int32), np.diff(tp))
    U0 = (rs.randn(nu, dim) * 0.1).astype(np.float32); V0 = (rs.randn(ni, dim) * 0.1).astype(np.float32)
    wu, wi, wj = oracle.epoch_build(tp, ti, pos_users, ti, 1, ni, True, True, 9, 0)
    g_all = tf_math.mf_pairwise_grad(U0, V0, wu, wi, wj[:, 0], "bpr", 0.0)
    dU, dV = dev(U0), dev(V0)
    sh = peer.single(dV).enable_hot(ni)
    ops.mf_bpr_sgd_epoch(dU, sh, dev(tp), dev(ti), dev(pos_users), dev(ti), ni, True, 9, 0, 0, len(ti), 1e-4, 0.0,
                         torch.zeros(1, device="cuda"))
    sh.sync_hot(); sh.writeback_hot()
    assert np.abs(dV.cpu().numpy() - (V0 - np.float32(1e-4) * g_all[2])).max() < 5e-6


@pytest.mark.parametrize("dim", [128, 64])
def test_csr_fed_sgd_kernel_large_launch_with_uneven_cta_shares(dim):
    """~60 k triplets in one launch, not a multiple of the grid size, so the persistent grid's CTAs take shares of
    unequal length: loss and both tables against the sum of the per-triplet gradients."""
    from neurec_b200 import ops
    from neurec_b200.util import peer
    nu, ni = 3000, 20000
    rs = np.random.RandomState(dim)
    rows = [np.unique(rs.randint(0, ni, 21)).astype(np.int32) for _ in range(nu)]
    tp, ti = oracle.lists_to_csr(rows)
    pos_users = np.repeat(np.arange(nu, dtype=np.int32), np.diff(tp))
    n = len(ti)
    assert n > 3 * 148 * 128
    U0 = (rs.randn(nu, dim) * 0.1).astype(np.float32); V0 = (rs.randn(ni, dim) * 0.1).astype(np.float32)
    lr, reg = 1e-4, 0.01
    wu, wi, wj = oracle.epoch_build(tp, ti, pos_users, ti, 1, ni, True, True, 5, 1)
    g_all = tf_math.mf_pairwise_grad(U0, V0, wu, wi, wj[:, 0], "bpr", reg)
    dU, dV = dev(U0), dev(V0)
    loss = torch.zeros(1, device="cuda")
    ops.mf_bpr_sgd_epoch(dU, peer.single(dV), dev(tp), dev(ti), dev(pos_users), dev(ti), ni, True, 5, 1, 0, n, lr, reg, loss)
    assert abs(float(loss) - float(g_all[0])) < 1e-3 * float(g_all[0])
    assert np.abs(dU.cpu().numpy() - (U0 - np.float32(lr) * g_all[1])).max() < 5e-6
    assert np.abs(dV.cpu().numpy() - (V0 - np.float32(lr) * g_all[2])).max() < 5e-6


@pytest.mark.parametrize("pairwise,loss,opt,mf_dim,layers,steps", [
    (False, "cross_entropy", "adam", 32, [64, 32, 16], 40),     # BASELINE configs[1] (conf/NeuMF.properties + embedding 32)
    (True, "bpr", "adam", 16, [64, 32, 16], 12),                # pairwise NeuMF: two differently-initialised towers
    (True, "bpr", "adam", 0, [64, 32, 16], 10),                 # MLP pairwise: shared tower, both passes feed dW
    (False, "square", "rmsprop", 8, [32, 16], 8),               # another tower shape, touched-row optimizer
    (False, "cross_entropy", "gd", 4, [48, 24], 6),             # widths that take the generic layer paths
])
def test_fused_ncf_epoch_matches_the_oracle_trainer(ml100k, pairwise, loss, opt, mf_dim, layers, steps):
    """nrc_ncf_epoch_fused (sampler + shuffle + every NeuMF / MLP step in one persistent launch) vs
    tf_math.NCFTrainer on the epoch arrays of oracle.epoch_build."""
    from neurec_b200 import ops
    from test_gpu_ncf import make_params, KEYS
    d = ml100k
    nu, ni, bs = d["num_users"], d["num_items"], 256
    nt = 2 if (pairwise and mf_dim == 16) else 1
    neg_num = 1 if pairwise else 4
    P, mlp_dim = make_params(nu, ni, mf_dim, layers, nt, 7, scale=0.01)
    pu, pi = _flat(d)
    wu, wi, wt = oracle.epoch_build(d["train_indptr"], d["train_indices"], pu, pi, neg_num, ni, pairwise, True, 77, 5)
    if pairwise:
        wt = wt[:, 0]
    n = len(wu)
    lr = 1e-3 if opt == "adam" else 1e-2
    tr = tf_math.NCFTrainer(P, mlp_dim, layers, nt, opt, lr, loss, 1e-4, 1e-4, pairwise)
    want = tr.epoch(wu[:steps * bs], wi[:steps * bs], wt[:steps * bs], bs)
    shape = ops.NcfShape.make(nu, ni, mf_dim, layers, nt)
    dP = {k: (dev(v) if v is not None else None) for k, v in P.items()}
    i0, i1 = tf_math.SLOT_INIT[opt]
    mk = lambda val: {k: (None if v is None or val is None else torch.full_like(v, val)) for k, v in dP.items()}
    G, S0, S1 = mk(0.0), mk(i0), mk(i1)
    tU = torch.zeros(nu, dtype=torch.int32, device="cuda"); tI = torch.zeros(ni, dtype=torch.int32, device="cuda")
    total_steps = (n + bs - 1) // bs
    step_loss = torch.full((total_steps,), 3.0, device="cuda")
    ws = tuple(torch.empty(n, dtype=torch.int32, device="cuda") for _ in range(3))
    pows = torch.tensor([0.9, 0.999], device="cuda") if opt == "adam" else None
    args = (shape, dP, dev(d["train_indptr"]), dev(d["train_indices"]), dev(pu), dev(pi), neg_num, pairwise, True, False,
            77, 5, bs)
    tail = (loss, 1e-4, 1e-4, opt, tf_math.DEFAULT_HYPER[opt](lr), pows, G, S0, S1, tU, tI)
    cut = steps // 2                                                 # the epoch cut into two calls
    ops.ncf_epoch_fused(*args, 0, cut, *tail, 1, ws[0], ws[1], ws[2], step_loss)
    ops.ncf_epoch_fused(*args, cut, steps - cut, *tail, 1 + cut, ws[0], ws[1], ws[2], step_loss)
    got = step_loss.cpu().numpy()
    assert np.array_equal(ws[0].cpu().numpy(), wu) and np.array_equal(ws[1].cpu().numpy(), wi)
    assert np.allclose(got[:steps], want, rtol=2e-4, atol=1e-6), np.abs(got[:steps] - want).max()
    assert (got[steps:] == 0).all()
    for k in KEYS:
        if P[k] is not None:
            assert np.abs(dP[k].cpu().numpy() - tr.P[k]).max() < 3e-5, k
    assert np.abs(tr.P["dense"] - P["dense"]).max() > 1e-5          # the towers really moved
    for k in KEYS[:4]:
        if G[k] is not None:
            assert float(G[k].abs().max()) == 0.0                    # accumulators left clean


@pytest.mark.parametrize("dim", [128, 64])
def test_lazy_adam_variant_on_a_duplicate_free_epoch(dim):
    """nrc_mf_bpr_lazy_adam_epoch (the explicitly-named lazy variant for huge tables, SURVEY 8d): on an
    epoch without repeated rows it is exactly LazyAdam -- only the batch's rows move, by the Adam
    formulas with this step's lr_t; untouched rows and their slots stay bit-identical."""
    from neurec_b200 import ops
    nu, ni, n = 300, 300_000, 300
    rs = np.random.RandomState(dim + 1)
    tp = np.arange(nu + 1, dtype=np.int64)
    pos_items = rs.permutation(ni)[:nu].astype(np.int32)
    pos_users = np.arange(nu, dtype=np.int32)
    for seed in range(50):
        wu, wi, wj = oracle.epoch_build(tp, pos_items, pos_users, pos_items, 1, ni, True, True, seed, 0)
        if len(np.unique(np.concatenate([wi, wj[:, 0]]))) == 2 * n:
            break
    else:
        pytest.skip("no duplicate-free epoch found")
    wj = wj[:, 0]
    U0 = (rs.randn(nu, dim) * 0.1).astype(np.float32); V0 = (rs.randn(ni, dim) * 0.1).astype(np.float32)
    mU0 = (rs.randn(nu, dim) * 0.01).astype(np.float32); vU0 = (rs.rand(nu, dim) * 0.01).astype(np.float32)
    mV0 = (rs.randn(ni, dim) * 0.01).astype(np.float32); vV0 = (rs.rand(ni, dim) * 0.01).astype(np.float32)
    lr_t, b1, b2, eps, reg = np.float32(3e-3), np.float32(0.9), np.float32(0.999), np.float32(1e-8), np.float32(1e-3)
    pu, qi, qj = U0[wu], V0[wi], V0[wj]
    x = (pu * qi).sum(1) - (pu * qj).sum(1)
    wl, g = tf_math.pairwise_loss_and_grad("bpr", x)
    g = g[:, None].astype(np.float32)

    def lazy(var, m, v, rows, grad):
        m[rows] = b1 * m[rows] + (np.float32(1) - b1) * grad
        v[rows] = b2 * v[rows] + (np.float32(1) - b2) * grad * grad
        var[rows] = var[rows] - lr_t * m[rows] / (np.sqrt(v[rows]) + eps)
    Uw, mUw, vUw, Vw, mVw, vVw = (a.copy() for a in (U0, mU0, vU0, V0, mV0, vV0))
    lazy(Uw, mUw, vUw, wu, g * (qi - qj) + reg * pu)
    lazy(Vw, mVw, vVw, wi, g * pu + reg * qi)
    lazy(Vw, mVw, vVw, wj, -g * pu + reg * qj)
    d = [dev(a) for a in (U0, mU0, vU0, V0, mV0, vV0)]
    loss = torch.zeros(1, device="cuda")
    ops.mf_bpr_lazy_adam_epoch(*d, dev(tp), dev(pos_items), dev(pos_users), dev(pos_items), ni, True, seed, 0, 0, n,
                               float(lr_t), float(reg), loss)
    for got, want, name in zip(d, (Uw, mUw, vUw, Vw, mVw, vVw), "U mU vU V mV vV".split()):
        assert np.abs(got.cpu().numpy() - want).max() < 2e-6, name
    untouched = np.setdiff1d(np.arange(ni), np.concatenate([wi, wj]))
    assert np.array_equal(d[3].cpu().numpy()[untouched], V0[untouched])
    assert np.array_equal(d[4].cpu().numpy()[untouched], mV0[untouched])
