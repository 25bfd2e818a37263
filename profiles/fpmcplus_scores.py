"""Time of FPMCplus's full-catalogue scoring (nrc_fpmcplus_scores) at a gowalla-sized shape, on the device.

    python profiles/fpmcplus_scores.py OUT_DIR [--repeats 5] [--warmup 1]

Workload: 29 858 users x 40 981 items (the gowalla split's counts), synthetic tables drawn from numpy seed 0 (tables
N(0, 0.1), W N(0, 1 / sqrt(d)), b N(0, 0.3), h N(1, 0.5)), the conf file's d = weight_size = 16 and high_order L = 3,
every user's window three random items.  Each repeat scores every user against every item in one call (the
projection pass, then the pair kernel); CUDA events around it, medians over --repeats after --warmup calls.

Counted per (user, item) pair: L w = 48 tanh, L w = 48 FMAs of h . tanh plus 2 L w = 96 adds of (A + B) + C, and
(L + 1) d = 64 FMAs of the two dot products: 208 FP32 operations that are not tanh (160 of them FMAs, 2 flops each).
Reported: pairs/s, tanh/s, and the counted FP32 flops/s of the non-tanh work against the data sheet's 67 TFLOP/s
FP32 for the H100 SXM, and tanh/s against an SFU bound: the accurate tanhf as compiled for sm_90a takes one
MUFU.EX2 and one MUFU.RCP for |x| >= 0.6 (a polynomial on the FP32 pipe below), and an SM issues 16 MUFU operations
per clock, so SMs x 16 x the maximum SM clock / 2 bounds tanh/s where every argument takes that path.
The card's name and power limit are read in the same run; the JSON goes to OUT_DIR/fpmcplus_scores.json.
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
USERS, ITEMS, D, W, L = 29858, 40981, 16, 16, 3
FP32_TFLOPS = 67.0


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    name, power, clock = [s.strip() for s in q.stdout.splitlines()[0].split(",")]
    return {"name": name, "power_limit": power, "max_sm_clock": clock}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("out_dir")
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    a = ap.parse_args()
    import torch
    from neurec_b200 import ops
    assert torch.cuda.is_available(), "this measurement needs a CUDA device"
    out_dir = os.path.abspath(a.out_dir)
    os.makedirs(out_dir, exist_ok=True)
    rs = np.random.RandomState(0)
    dev = lambda x: torch.from_numpy(np.ascontiguousarray(x)).cuda()
    tabs = [dev((rs.randn(n, D) * 0.1).astype(np.float32)) for n in (USERS, ITEMS, ITEMS, ITEMS)]
    tabs += [dev((rs.randn(3 * D, W) / np.sqrt(D)).astype(np.float32)), dev((rs.randn(1, W) * 0.3).astype(np.float32)),
             dev((rs.randn(W, 1) * 0.5 + 1.0).astype(np.float32))]
    users = dev(np.arange(USERS, dtype=np.int32))
    recent = dev(rs.randint(0, ITEMS, (USERS, L)).astype(np.int32))
    length = dev(np.full(USERS, L, np.int32))
    call = lambda: ops.fpmcplus_scores(*tabs, users, recent, length)
    for _ in range(a.warmup):
        out = call()
    del out
    times = []
    for _ in range(a.repeats):
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        s.record()
        out = call()
        e.record()
        torch.cuda.synchronize()
        times.append(s.elapsed_time(e))
        nonfinite = int((~torch.isfinite(out)).sum())
        del out
    ms = float(np.median(times))
    c = card()
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    sfu_bound = sms * 16 * float(c["max_sm_clock"].split()[0]) * 1e6 / 2
    pairs = USERS * ITEMS
    flops = pairs * (2 * (L * W + (L + 1) * D) + 2 * L * W)
    result = {"card": c, "sms": sms, "users": USERS, "items": ITEMS, "dim": D, "weight_size": W, "window": L,
              "repeats": a.repeats, "warmup": a.warmup, "call_ms": {"median": ms, "min": float(min(times)),
                                                                   "max": float(max(times))},
              "pairs_per_s": pairs / (ms * 1e-3), "tanh_per_s": pairs * L * W / (ms * 1e-3),
              "counted_fp32_flops_per_s": flops / (ms * 1e-3),
              "counted_fp32_share_of_67_tflops": flops / (ms * 1e-3) / (FP32_TFLOPS * 1e12),
              "tanh_sfu_bound_per_s": sfu_bound, "tanh_share_of_sfu_bound": pairs * L * W / (ms * 1e-3) / sfu_bound,
              "nonfinite_scores": nonfinite,
              "routes": ops.fpmcplus_last_routes()}
    with open(os.path.join(out_dir, "fpmcplus_scores.json"), "w") as f:
        json.dump(result, f, indent=1)
        f.write("\n")
    print(json.dumps(result))


if __name__ == "__main__":
    main()
