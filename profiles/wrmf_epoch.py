"""Time of one WRMF epoch (two nrc_wrmf_half_step calls) on the device, and of the reference's formulation on the CPU.

    python profiles/wrmf_epoch.py OUT.json [--epochs 20] [--warmup 3] [--cpu-rows 40]

Shapes: ml-100k at d = 16 and d = 64, gowalla at d = 64 (the golden splits under tests/golden), alpha = 10,
reg_mf = 0.1, item table initialised as the plug-in does.  Device times are CUDA events around each half-step over
--epochs epochs after --warmup untimed ones.  The rate is the algorithm's flop per half-step, counted here from the
shapes, over the event time, next to NVIDIA's 67 TFLOP/s FP32 data-sheet figure for the H100 SXM (a figure for a
700 W card; the card's name and power limit are read in the same run).

The CPU arm restates the reference's one-row-per-call formulation (WRMF.py:51-61,74-85: a dense confidence column,
Y^T Y + Y^T diag(Cu) Y + lambda I formed per row, then a dense solve) in numpy fp32 with np.linalg.solve, times it
on --cpu-rows users and as many items, and extrapolates to all rows.  It is a restatement, not the reference
(which runs the same algebra through one TensorFlow session call per row).
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
PEAK_FP32_TFLOPS = 67.0
ALPHA, REG = 10.0, 0.1


def load_split(name):
    z = np.load(os.path.join(ROOT, "tests", "golden", "%s_split.npz" % name))
    return (int(z["num_users"]), int(z["num_items"]), z["train_indptr"].astype(np.int64),
            z["train_indices"].astype(np.int32))


def transpose_csr(indptr, indices, num_cols):
    rows = np.repeat(np.arange(len(indptr) - 1, dtype=np.int32), np.diff(indptr))
    order = np.lexsort((rows, indices))
    tptr = np.zeros(num_cols + 1, np.int64)
    tptr[1:] = np.cumsum(np.bincount(indices, minlength=num_cols))
    return tptr, rows[order].astype(np.int32)


def half_flop(n_fixed, n_rows, nnz, d):
    """Gram 2 n_fixed d^2, outer products 2 nnz d^2, per row Cholesky d^3 / 3 and two triangular solves 2 d^2."""
    return 2.0 * n_fixed * d * d + 2.0 * nnz * d * d + n_rows * (d ** 3 / 3.0 + 2.0 * d * d)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    name, power, clock = [s.strip() for s in q.stdout.splitlines()[0].split(",")]
    return {"name": name, "power_limit": power, "max_sm_clock": clock}


def device_epochs(num_users, num_items, ptr, idx, d, epochs, warmup):
    import torch
    from neurec_b200 import _lib, ops
    from neurec_b200.model._engine import get_initializer
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()
    tptr, tidx = transpose_csr(ptr, idx, num_items)
    init = get_initializer("uniform", 0.01, torch.Generator().manual_seed(2017))
    X, Y = init([num_users, d]).cuda(), init([num_items, d]).cuda()
    user_csr, item_csr = (t(ptr), t(idx)), (t(tptr), t(tidx))
    order = lambda p: t(np.argsort(-np.diff(p), kind="stable").astype(np.int32))
    user_order, item_order = order(ptr), order(tptr)
    work = ops.wrmf_work(max(num_users, num_items), d)
    not_spd = torch.zeros(1, dtype=torch.int32, device="cuda")
    halves = ((Y, user_csr, user_order, X), (X, item_csr, item_order, Y))
    for _ in range(warmup):
        for fixed, (p, i), o, out in halves:
            ops.wrmf_half_step(fixed, p, i, out, ALPHA, REG, row_order=o, work=work, not_spd=not_spd)
    ev = [[torch.cuda.Event(enable_timing=True) for _ in range(3)] for _ in range(epochs)]
    torch.cuda.synchronize()
    for e in range(epochs):
        ev[e][0].record()
        for h, (fixed, (p, i), o, out) in enumerate(halves):
            # the raw call: ops.wrmf_half_step reads not_spd back, which would put a host sync inside the window
            rc =_lib.load().nrc_wrmf_half_step(ops._p(fixed), fixed.shape[0], ops._p(p), ops._p(i), ops._p(o),
                                                p.numel() - 1, d, ALPHA, REG, ops._p(out), ops._p(work),
                                                ops._p(not_spd), ops._stream())
            _lib.check(rc)
            ev[e][h + 1].record()
    torch.cuda.synchronize()
    assert int(not_spd.item()) == 0 and bool(torch.isfinite(X).all()) and bool(torch.isfinite(Y).all())
    user_ms = np.array([ev[e][0].elapsed_time(ev[e][1]) for e in range(epochs)])
    item_ms = np.array([ev[e][1].elapsed_time(ev[e][2]) for e in range(epochs)])
    return user_ms, item_ms


def cpu_rows(fixed, ptr, idx, rows, d):
    """Seconds per row of the reference's per-row formulation (numpy fp32), over the given rows."""
    n = fixed.shape[0]
    lambda_eye = np.float32(REG) * np.eye(d, dtype=np.float32)
    start = time.perf_counter()
    for r in rows:
        C = np.zeros((n, 1), np.float32)
        P = np.zeros((n, 1), np.float32)
        C[idx[ptr[r]:ptr[r + 1]]] = ALPHA
        P[idx[ptr[r]:ptr[r + 1]]] = 1.0
        YTY = fixed.T @ fixed
        YTCY = fixed.T @ (C * fixed)
        YTCp = fixed.T @ ((C + 1) * P)
        np.linalg.solve(YTY + YTCY + lambda_eye, YTCp)
    return (time.perf_counter() - start) / len(rows)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("out")
    ap.add_argument("--epochs", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--cpu-rows", type=int, default=40)
    a = ap.parse_args()
    result = {"card": card(), "peak_fp32_tflops_datasheet": PEAK_FP32_TFLOPS, "alpha": ALPHA, "reg_mf": REG,
              "epochs_timed": a.epochs, "warmup_epochs": a.warmup, "shapes": []}
    rs = np.random.RandomState(0)
    for name, d in (("ml100k", 16), ("ml100k", 64), ("gowalla", 64)):
        nu, ni, ptr, idx = load_split(name)
        nnz = int(ptr[-1])
        user_ms, item_ms = device_epochs(nu, ni, ptr, idx, d, a.epochs, a.warmup)
        f_user, f_item = half_flop(ni, nu, nnz, d), half_flop(nu, ni, nnz, d)
        epoch_ms = user_ms + item_ms
        tptr, tidx = transpose_csr(ptr, idx, ni)
        Y = (rs.rand(ni, d).astype(np.float32) - 0.5) * 0.02
        X = (rs.rand(nu, d).astype(np.float32) - 0.5) * 0.02
        k = min(a.cpu_rows, nu, ni)
        cpu_user = cpu_rows(Y, ptr, idx, rs.choice(nu, k, replace=False), d)
        cpu_item = cpu_rows(X, tptr, tidx, rs.choice(ni, k, replace=False), d)
        cpu_epoch_s = cpu_user * nu + cpu_item * ni
        tf = lambda flop, ms: flop / (ms * 1e-3) / 1e12
        result["shapes"].append({
            "dataset": name, "dim": d, "num_users": nu, "num_items": ni, "nnz": nnz,
            "user_half_ms_median": float(np.median(user_ms)), "item_half_ms_median": float(np.median(item_ms)),
            "epoch_ms_median": float(np.median(epoch_ms)), "epoch_ms_min": float(epoch_ms.min()),
            "epoch_ms_max": float(epoch_ms.max()),
            "flop_user_half": f_user, "flop_item_half": f_item,
            "tflops_user_half": tf(f_user, np.median(user_ms)), "tflops_item_half": tf(f_item, np.median(item_ms)),
            "tflops_epoch": tf(f_user + f_item, np.median(epoch_ms)),
            "share_of_fp32_datasheet_epoch": tf(f_user + f_item, np.median(epoch_ms)) / PEAK_FP32_TFLOPS,
            "cpu_restatement": {"what": "numpy fp32 restatement of the reference's one-row-per-call formulation "
                                        "(dense confidence column, np.linalg.solve per row), timed on %d users and %d "
                                        "items, extrapolated to all rows" % (k, k),
                                "s_per_user_row": cpu_user, "s_per_item_row": cpu_item,
                                "epoch_s_extrapolated": cpu_epoch_s},
            "speedup_vs_cpu_restatement": cpu_epoch_s / (np.median(epoch_ms) * 1e-3),
        })
        print(json.dumps(result["shapes"][-1]), flush=True)
    os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
    with open(a.out, "w") as f:
        json.dump(result, f, indent=1)
        f.write("\n")


if __name__ == "__main__":
    main()
