"""The CSR-fed BPR/SGD step's store path for user rows (nrc_mf_bpr_sgd_epoch with pos_items == train_indices): a user
row that no other triplet of the launch touches is written with a plain store of value + delta, every other update is
a RED.  A store taken where it must not be loses a whole delta; these tests are built so that such a loss is many
times their tolerance."""
import numpy as np
import pytest
import torch

import oracle
from oracle import tf_math

pytestmark = pytest.mark.gpu


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def run(U0, V0, tp, ti, pos_users, ni, shuffle, seed, epoch, windows, lr, reg, same_csr=True, n_hot=0):
    """One call per (first, count) window; same_csr passes train_indices itself as pos_items (the store path),
    otherwise a copy of it (REDs only).  Returns the tables (head written back) and the summed loss."""
    from neurec_b200 import ops
    from neurec_b200.util import peer
    dU, dV = dev(U0), dev(V0)
    sh = peer.single(dV)
    if n_hot:
        sh.enable_hot(n_hot)
    t_idx = dev(ti)
    pos = t_idx if same_csr else t_idx.clone()
    loss = torch.zeros(1, device="cuda")
    for first, count in windows:
        ops.mf_bpr_sgd_epoch(dU, sh, dev(tp), t_idx, dev(pos_users), pos, ni, shuffle, seed, epoch, first, count, lr,
                             reg, loss)
        sh.sync_hot()
    sh.writeback_hot()
    return dU.cpu().numpy(), dV.cpu().numpy(), float(loss)


def window_triplets(tp, ti, pos_users, ni, shuffle, seed, epoch, first, count):
    wu, wi, wj = oracle.epoch_build(tp, ti, pos_users, ti, 1, ni, True, shuffle, seed, epoch)
    return wu[first:first + count], wi[first:first + count], wj[first:first + count, 0]


def first_order(U0, V0, wu, wi, wj, lr, reg):
    """The sum of every triplet's update taken at the pre-step tables."""
    _, gU, gV, _, _ = tf_math.mf_pairwise_grad(U0, V0, wu, wi, wj, "bpr", reg)
    return U0 - np.float32(lr) * gU, V0 - np.float32(lr) * gV


@pytest.mark.parametrize("dim", [32, 64, 128])
def test_rows_touched_once_equal_a_numpy_step_bit_for_bit(dim):
    """One positive per user, every item of the launch distinct: no row is touched twice.  The tables are built so
    that every score difference is 0 (g = -1/2 exactly) and every product and sum is exact in fp32: users live on the
    first half of the dimensions, where all items agree, and items differ on the second half.  The store path must
    give the numpy step's bits, and the bits of the same launch with REDs only."""
    nu, ni, n = 700, 2_000_000, 700
    rs = np.random.RandomState(dim)
    tp = np.arange(nu + 1, dtype=np.int64)
    pos_users = np.arange(nu, dtype=np.int32)
    for seed in range(50):
        ti = rs.permutation(ni)[:nu].astype(np.int32)
        ti.sort()
        pos_users = np.arange(nu, dtype=np.int32)
        wu, wi, wj = window_triplets(tp, ti, pos_users, ni, True, seed, 3, 0, n)
        if len(np.unique(np.concatenate([wi, wj]))) == 2 * n:
            break
    else:
        pytest.skip("no launch with distinct items found")
    h = dim // 2
    U0 = np.zeros((nu, dim), np.float32)
    U0[:, :h] = rs.randint(-8, 9, (nu, h)) / np.float32(16)
    V0 = np.zeros((ni, dim), np.float32)
    V0[:, :h] = rs.randint(-8, 9, h) / np.float32(16)            # the same first half for every item
    V0[:, h:] = rs.randint(-8, 9, (ni, dim - h)) / np.float32(16)
    lr, reg = 2.0 ** -4, 2.0 ** -3
    g = np.float32(-0.5)
    pu, qi, qj = U0[wu], V0[wi], V0[wj]
    want_U, want_V = U0.copy(), V0.copy()
    f = np.float32
    want_U[wu] = pu + (-f(lr) * (g * (qi - qj) + f(reg) * pu))
    want_V[wi] = qi + (-f(lr) * (g * pu + f(reg) * qi))
    want_V[wj] = qj + (-f(lr) * (-g * pu + f(reg) * qj))
    gU, gV, _ = run(U0, V0, tp, ti, pos_users, ni, True, seed, 3, [(0, n)], lr, reg)
    assert np.array_equal(gU, want_U) and np.array_equal(gV, want_V)
    rU, rV, _ = run(U0, V0, tp, ti, pos_users, ni, True, seed, 3, [(0, n)], lr, reg, same_csr=False)
    assert np.array_equal(rU, gU) and np.array_equal(rV, gV)


@pytest.mark.parametrize("shuffle", [True, False])
def test_users_touched_twice_keep_both_deltas(shuffle):
    """Every user has exactly two positives and the launch covers the whole epoch, so every user row is updated by
    two triplets and none may take the store.  Each delta is more than ten times the tolerance."""
    nu, ni, dim = 5000, 100_000, 128
    rs = np.random.RandomState(11)
    rows = [np.sort(rs.choice(ni, 2, replace=False)).astype(np.int32) for _ in range(nu)]
    tp, ti = oracle.lists_to_csr(rows)
    pos_users = np.repeat(np.arange(nu, dtype=np.int32), np.diff(tp))
    n = len(ti)
    U0 = (rs.randn(nu, dim) * 0.1).astype(np.float32)
    V0 = (rs.randn(ni, dim) * 0.1).astype(np.float32)
    lr = 1e-3
    wu, wi, wj = window_triplets(tp, ti, pos_users, ni, shuffle, 4, 0, 0, n)
    assert (np.bincount(wu, minlength=nu) == 2).all()
    want_U, want_V = first_order(U0, V0, wu, wi, wj, lr, 0.0)
    one = np.abs(want_U - U0).max(1)
    assert np.median(one) > 10 * 5e-6                 # losing either delta of a row is far outside the tolerance
    gU, gV, _ = run(U0, V0, tp, ti, pos_users, ni, shuffle, 4, 0, [(0, n)], lr, 0.0)
    assert np.abs(gU - want_U).max() < 5e-6 and np.abs(gV - want_V).max() < 5e-6


def mixed_csr(rs, nu, ni):
    """Rows of 1 to 7 positives and a few of 40 (longer than the rows checked for a single visit).  Item ids have
    density ~ 1/sqrt(id): the lowest ids are the most popular (the replicated head), none so popular that reading it
    mid-launch moves a gradient by more than second order."""
    deg = rs.randint(1, 8, nu)
    deg[rs.choice(nu, 8, replace=False)] = 40
    items = (ni * rs.random_sample(int(deg.sum())) ** 2).astype(np.int32)
    ends = np.cumsum(deg)
    rows = [np.unique(items[e - d:e]) for d, e in zip(deg, ends)]
    tp, ti = oracle.lists_to_csr(rows)
    return tp, ti, np.repeat(np.arange(nu, dtype=np.int32), np.diff(tp))


@pytest.mark.parametrize("dim,shuffle,same_csr,n_hot", [
    (128, True, True, 0), (128, True, True, 64), (128, True, True, 16384), (64, True, True, 16384),
    (32, True, True, 0), (128, False, True, 0), (64, False, True, 64), (128, True, False, 0), (32, True, False, 16384)])
def test_mixed_windows_match_the_first_order_step(dim, shuffle, same_csr, n_hot):
    """Users of 1 to 40 positives, windows that start inside the epoch (first > 0) and whose length leaves the
    persistent grid's CTAs unequal shares, split over two calls; with and without a replicated head (in the shared-
    memory tier only, or beyond it), with and without the shuffle, and with pos_items a copy of the CSR (REDs only).
    lr is small enough that reading a row another triplet already moved is second order, and large enough that a
    lost delta is not."""
    nu, ni = 200_000, 30_000
    rs = np.random.RandomState(dim + 2 * shuffle + n_hot)
    tp, ti, pos_users = mixed_csr(rs, nu, ni)
    n = len(ti)
    first = 1234
    count = min(n - first, 132 * 768 + 517)
    mid = first + count // 3
    U0 = (rs.randn(nu, dim) * 0.1).astype(np.float32)
    V0 = (rs.randn(ni, dim) * 0.1).astype(np.float32)
    lr = 1e-3
    wu1, wi1, wj1 = window_triplets(tp, ti, pos_users, ni, shuffle, 7, 1, first, mid - first)
    wu2, wi2, wj2 = window_triplets(tp, ti, pos_users, ni, shuffle, 7, 1, mid, first + count - mid)
    # the first call's result is the second call's pre-step table
    U1, V1 = first_order(U0, V0, wu1, wi1, wj1, lr, 0.0)
    want_U, want_V = first_order(U1, V1, wu2, wi2, wj2, lr, 0.0)
    cu = np.bincount(wu2, minlength=nu)
    assert (cu[wu2] == 1).any() and (cu[wu2] > 1).any()     # both kinds of user row in the launch
    if shuffle:
        assert (cu[wu2] == 1).mean() > 0.5
    gU, gV, loss = run(U0, V0, tp, ti, pos_users, ni, shuffle, 7, 1, [(first, mid - first), (mid, first + count - mid)],
                       lr, 0.0, same_csr=same_csr, n_hot=n_hot)
    assert np.abs(gU - want_U).max() < 5e-6 and np.abs(gV - want_V).max() < 5e-6
    want_loss = float(tf_math.mf_pairwise_grad(U0, V0, wu1, wi1, wj1, "bpr", 0.0)[0]) + \
        float(tf_math.mf_pairwise_grad(U1, V1, wu2, wi2, wj2, "bpr", 0.0)[0])
    assert abs(loss - want_loss) < 1e-3 * want_loss
