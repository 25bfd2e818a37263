"""Time of FISM training epochs and full-catalogue scoring on the device.

    python profiles/fism_epoch.py OUT_DIR [--repeats 5] [--warmup 1]

Workloads (conf/FISM.properties' defaults: d 16, alpha 0.5, regs 1e-4, Adam, batch 256, num_neg 4):
  * ml-100k pointwise: the reference's ratio-0.8 split (tests/golden/ml100k_split.npz), 401 835 samples, 1 570 steps;
  * ml-100k pairwise (bpr): 40 381 samples over the odd-position histories, 158 steps;
  * gowalla pointwise: tests/golden/gowalla_split.npz, 4 050 640 samples, 15 823 steps;
  * scoring every item for every user: ml-100k (943 x 1 682) and gowalla (29 858 x 40 981, in batches of 1 024 users).
Reported per epoch: the median time of one nrc_fism_train_epoch over an epoch already on the device (CUDA events,
--repeats after --warmup untimed ones), the step time, and, from the shapes, the history rows gathered (as many row
gradients added) with their bytes (d floats each way) and float adds, as rates over the epoch time.  Scoring: CUDA
events around query + scores.  The card's name and power limit are read in the same run; the JSON goes to
OUT_DIR/fism_epoch.json.
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
GOLDEN = os.path.join(ROOT, "tests", "golden")


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    name, power, clock = [s.strip() for s in q.stdout.splitlines()[0].split(",")]
    return {"name": name, "power_limit": power, "max_sm_clock": clock}


def events_ms(fn, repeats, warmup):
    import torch
    for _ in range(warmup):
        fn()
    out = []
    for _ in range(repeats):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        out.append(a.elapsed_time(b))
    return float(np.median(out))


def load(name):
    z = np.load(os.path.join(GOLDEN, name))
    return z["train_indptr"].astype(np.int64), z["train_indices"].astype(np.int32), int(z["num_users"]), \
        int(z["num_items"])


def epoch(ptr, idx, ni, pairwise, repeats, warmup, d=16, bs=256):
    import torch
    from neurec_b200 import ops
    from neurec_b200.model.general_recommender.FISM import pairwise_layout, pointwise_layout
    dev = lambda a: None if a is None else torch.from_numpy(np.ascontiguousarray(a)).cuda()
    rs = np.random.RandomState(0)
    if pairwise:
        (hp, hi), (rows, items, num, num_neg) = pairwise_layout(ptr, idx)
        third, excl = rs.randint(0, ni, len(rows)).astype(np.int32), None
    else:
        hp, hi = ptr, idx
        rows, excl, num, third = pointwise_layout(ptr, idx, 4)
        items = np.where(excl >= 0, excl, rs.randint(0, ni, len(rows))).astype(np.int32)
        num_neg = None
    perm = rs.permutation(len(rows))
    arrs = [None if a is None else dev(a[perm]) for a in (rows, excl, num, items, third, num_neg)]
    deg = np.diff(hp)[rows] - (0 if excl is None else (excl >= 0))
    n = len(rows)
    steps = (n + bs - 1) // bs
    tabs = [torch.randn(ni, d, device="cuda") * 0.01, torch.randn(ni, d, device="cuda") * 0.01,
            torch.zeros(ni, device="cuda")]
    grads = [torch.zeros_like(t) for t in tabs]
    s0, s1 = [torch.zeros_like(t) for t in tabs], [torch.zeros_like(t) for t in tabs]
    touched = (torch.zeros(ni, dtype=torch.int32, device="cuda"), torch.zeros(ni, dtype=torch.int32, device="cuda"))
    step_loss = torch.zeros(steps, device="cuda")
    lr_t = np.full(steps, 1e-3, np.float32)
    hp_d, hi_d = dev(hp), dev(hi)
    run = lambda: ops.fism_train_epoch(*tabs, hp_d, hi_d, *arrs, bs, pairwise, "bpr" if pairwise else "square", 0.5,
                                       1e-4, 1e-4, "adam", lr_t, [1e-3, 0.9, 0.999, 1e-8], grads, touched, s0, s1, 1,
                                       step_loss)
    ms = events_ms(run, repeats, warmup)
    rows_total = int(deg.sum())
    dp = deg[perm]
    per_batch_max = [int(dp[s * bs:(s + 1) * bs].max()) for s in range(steps)]
    return {"samples": n, "steps": steps, "epoch_ms": ms, "step_us": 1e3 * ms / steps,
            "history_rows": rows_total, "history_rows_per_s": rows_total / (ms * 1e-3),
            "row_gradient_adds_per_s": rows_total * d / (ms * 1e-3),
            "history_bytes_read": rows_total * d * 4, "row_gradient_bytes_added": rows_total * d * 4,
            "float_adds_gather": rows_total * d, "mean_longest_history_per_step": float(np.mean(per_batch_max)),
            "mean_history": float(deg.mean())}


def scoring(ptr, idx, nu, ni, repeats, warmup, d=16, chunk=1024):
    import torch
    from neurec_b200 import ops
    c1, Q, b = torch.randn(ni, d, device="cuda"), torch.randn(ni, d, device="cuda"), torch.randn(ni, device="cuda")
    hp, hi = torch.from_numpy(ptr).cuda(), torch.from_numpy(idx).cuda()
    users = torch.arange(nu, dtype=torch.int32, device="cuda")

    def run():
        for s in range(0, nu, chunk):
            ops.fism_scores(c1, Q, b, hp, hi, users[s:s + chunk], 0.5)
    ms = events_ms(run, repeats, warmup)
    return {"users": nu, "items": ni, "ms": ms, "scores_per_s": nu * ni / (ms * 1e-3),
            "score_bytes_written": nu * ni * 4, "write_bytes_per_s": nu * ni * 4 / (ms * 1e-3)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("out_dir")
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    a = ap.parse_args()
    import torch
    assert torch.cuda.is_available(), "fism_epoch.py measures on a CUDA device"
    res = {"card": card(), "command": "python profiles/fism_epoch.py OUT_DIR --repeats %d --warmup %d" %
           (a.repeats, a.warmup)}
    ml, gw = load("ml100k_split.npz"), load("gowalla_split.npz")
    work = [("ml100k_pointwise", lambda: epoch(ml[0], ml[1], ml[3], False, a.repeats, a.warmup)),
            ("ml100k_pairwise", lambda: epoch(ml[0], ml[1], ml[3], True, a.repeats, a.warmup)),
            ("gowalla_pointwise", lambda: epoch(gw[0], gw[1], gw[3], False, max(1, a.repeats // 2), a.warmup)),
            ("ml100k_scores", lambda: scoring(*ml, a.repeats, a.warmup)),
            ("gowalla_scores", lambda: scoring(*gw, a.repeats, a.warmup))]
    for name, fn in work:
        res[name] = fn()
        print(name, json.dumps(res[name]), flush=True)
    os.makedirs(a.out_dir, exist_ok=True)
    with open(os.path.join(a.out_dir, "fism_epoch.json"), "w") as f:
        json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
