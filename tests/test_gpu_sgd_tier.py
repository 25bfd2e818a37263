"""The CSR-fed BPR/SGD kernel's shared-memory tier (csrc/train_mf.cu, mf_bpr_sgd_stream_kernel): head rows
[0, T) are read from each CTA's copy and their deltas summed per CTA before one flush into the replica's delta
buffer.  T = 64 rows at dim 128; the head is set just below, at and well above it."""
import numpy as np
import pytest
import torch

import oracle
from oracle import tf_math

pytestmark = pytest.mark.gpu

TIER_ROWS_D128 = 64


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def zipf_csr(nu, ni, max_pos, seed):
    """1..max_pos positives per user, items by bench.synth_shard_csr's law: continuous Zipf(1.05), most popular first."""
    rs = np.random.RandomState(seed)
    deg = rs.randint(1, max_pos + 1, nu)
    users = np.repeat(np.arange(nu, dtype=np.int64), deg)
    a = 1.05
    r = (((ni ** (1 - a) - 1) * rs.rand(len(users)) + 1) ** (1 / (1 - a))).astype(np.int64)
    items = np.clip(r, 1, ni) - 1
    key = np.unique(users * ni + items)                 # sorted, duplicate-free rows
    u, i = key // ni, (key % ni).astype(np.int32)
    tp = np.zeros(nu + 1, np.int64)
    tp[1:] = np.cumsum(np.bincount(u, minlength=nu))
    return tp, i, u.astype(np.int32)


@pytest.mark.parametrize("n_hot", [TIER_ROWS_D128 - 1, TIER_ROWS_D128, 4 * TIER_ROWS_D128])
def test_zipf_epoch_over_the_whole_grid_sums_every_contribution(n_hot):
    """More triplets than 256 per CTA of any grid the kernel can launch (8 CTAs of 256 threads per SM at most), so
    every CTA samples several chunks and flushes its own tier.  With lr small enough that in-place reads of rows
    outside the head are second order, the tables after sync_hot + writeback_hot are the pre-step tables plus the
    sum of every per-triplet update, and the loss is the sum of the per-triplet losses."""
    from neurec_b200 import ops
    from neurec_b200.util import peer
    dim, nu, ni = 128, 100_000, 50_000
    tp, ti, pu = zipf_csr(nu, ni, 5, seed=n_hot)
    n = len(ti)
    assert n > torch.cuda.get_device_properties(0).multi_processor_count * 8 * 256
    rs = np.random.RandomState(1)
    U0 = (rs.randn(nu, dim) * 0.1).astype(np.float32)
    V0 = (rs.randn(ni, dim) * 0.1).astype(np.float32)
    lr = 1e-4
    wu, wi, wj = oracle.epoch_build(tp, ti, pu, ti, 1, ni, True, True, 13, 1)
    assert np.bincount(wi, minlength=ni)[0] > 1000            # row 0 is updated thousands of times in one launch
    assert (wi >= n_hot).mean() > 0.2                          # rows past the head are updated in place
    g_all = tf_math.mf_pairwise_grad(U0, V0, wu, wi, wj[:, 0], "bpr", 0.0)
    dU, dV = dev(U0), dev(V0)
    sh = peer.single(dV).enable_hot(n_hot)
    loss = torch.zeros(1, device="cuda")
    ops.mf_bpr_sgd_epoch(dU, sh, dev(tp), dev(ti), dev(pu), dev(ti), ni, True, 13, 1, 0, n, lr, 0.0, loss)
    assert torch.equal(dV[:n_hot], dev(V0[:n_hot]))            # the head's deltas wait next to the replica
    sh.sync_hot(); sh.writeback_hot()
    assert abs(float(loss) - float(g_all[0])) < 1e-3 * float(g_all[0])
    assert np.abs(dU.cpu().numpy() - (U0 - np.float32(lr) * g_all[1])).max() < 5e-6
    assert np.abs(dV.cpu().numpy() - (V0 - np.float32(lr) * g_all[2])).max() < 5e-6
