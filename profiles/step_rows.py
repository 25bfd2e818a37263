"""How many of one benchmark step's in-place row updates land on a row that no other triplet of the step touches.

    python profiles/step_rows.py [--step S]

CPU only (about ten seconds): the bench shape's train CSR for rank 0 at N = 1 (bench.synth_shard_csr on the host),
the positions of the epoch from oracle.epoch_build (the kernel's sampler and shuffle, restated bit for bit), and the
2^20 triplets of step S (default 0, the first step of epoch 0).  Rows of the replicated head (item ids below n_hot)
are not updated in place and are counted apart.  For such a row -- one reader and one writer, the warp of its
triplet -- a plain store of value + delta gives the bits an atomic add gives.  Also prints the user share by the
kernel's own rule (no other CSR position of the user's row has its inverse-shuffled position inside the step), which
must equal the counted one, and the step's accesses of the replicated head by rank band.  Prints one JSON object.
"""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    import bench
    import oracle
    ap = argparse.ArgumentParser()
    ap.add_argument("--step", type=int, default=0)
    args = ap.parse_args()
    cfg = bench.ShardedCfg
    ptr, idx = bench.synth_shard_csr(cfg, 0, 1, device="cpu")
    users = np.repeat(np.arange(len(ptr) - 1, dtype=np.int32), np.diff(ptr))
    wu, wi, wj = oracle.epoch_build(ptr, idx, users, idx, 1, cfg.items_per_gpu, True, True, bench.SEED, 0)
    lo = args.step * cfg.batch
    u, i, j = wu[lo:lo + cfg.batch], wi[lo:lo + cfg.batch], wj[lo:lo + cfg.batch, 0]
    n_hot = bench.n_hot_of(cfg, 1)
    cu = np.bincount(u, minlength=cfg.users_per_gpu)
    items = np.concatenate([i, j])
    ci = np.bincount(items[items >= n_hot], minlength=cfg.items_per_gpu)
    once_u = int((cu[u] == 1).sum())
    # the kernel's rule for user rows: no other CSR position of the row is visited inside the step's window (perm^-1
    # of each position, rows of at most 32 positives); it must agree with the count above
    n = len(idx)
    inv = np.empty(n, np.int64)
    inv[oracle.shuffle_perm(n, bench.SEED, 0, True)] = np.arange(n)
    visited = ((inv - lo) >= 0) & ((inv - lo) < cfg.batch)
    per_row = np.add.reduceat(visited.astype(np.int64), ptr[:-1])
    rule_u = int(((per_row[u] == 1) & (np.diff(ptr)[u] <= 32)).sum())
    cold_i, cold_j = i[i >= n_hot], j[j >= n_hot]
    once_i, once_j = int((ci[cold_i] == 1).sum()), int((ci[cold_j] == 1).sum())
    total = len(u) + len(cold_i) + len(cold_j)
    # accesses of the replicated head per step by rank band: [0, 64) the shared-memory tier at d = 128, the rest are
    # read from `hot` and RED-added into `hot_delta` in global memory
    bands = [0, 64, 256, 1024, 4096, n_hot]
    head = {"%d-%d" % (a, b): int(((items >= a) & (items < b)).sum()) for a, b in zip(bands[:-1], bands[1:]) if b > a}
    print(json.dumps({
        "step": args.step, "triplets": len(u), "n_hot": n_hot,
        "user_updates": len(u), "user_touched_once": once_u / len(u),
        "user_touched_once_kernel_rule": rule_u / len(u), "head_accesses_by_rank": head,
        "negative_updates_outside_head": len(cold_j), "negatives_in_head": float((j < n_hot).mean()),
        "negative_touched_once": once_j / len(cold_j),
        "positive_updates_outside_head": len(cold_i), "positive_touched_once": once_i / len(cold_i),
        "positives_in_head": int((i < n_hot).sum()), "positives_in_shared_memory_tier": int((i < 64).sum()),
        "in_place_updates": total, "touched_once": once_u + once_i + once_j,
        "touched_once_share": (once_u + once_i + once_j) / total}))


if __name__ == "__main__":
    main()
