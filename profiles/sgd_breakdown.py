"""Where the time of the CSR-fed BPR/SGD step (the default bprmf-sharded workload at N = 1) goes, on one GPU.

    python profiles/sgd_breakdown.py OUT.json [--root TREE] [--label NAME] [--items a,b,...]

Each item runs the workload's step kernel in a fresh process (the library reads its knobs once) against the
library built in TREE (default: this repository), at the bench shape unless the item says otherwise, and records
the mean kernel time of 20 timed launches (CUDA events, bench.measure_sharded's `launch_us`).  Results are merged
into OUT.json under NAME, next to the card's name and power limit read in the same run.

  bench          the bench shape as it is
  local_red      NRC_SGD_LOCAL_BULK=0: local rows updated by vector REDs instead of one bulk reduce-add per row
                 (a knob of trees whose kernel has both forms)
  no_head        NRC_BENCH_N_HOT=0: no replicated head, the popular rows are updated in place
  uniform_pos    positives uniform over the catalogue (zipf_a = 0), head kept: the step without the skew
  prebuilt_ids   ids of the same positions built by ops.epoch_build beforehand (untimed), then ops.mf_bpr_sgd_fused
                 timed, against the CSR-fed kernel on the same tables in the same process (both without a head)
  probe          profiles/row_update_probe.cu: read / read + store / read + RED.v4 / read + bulk reduce-add of 3 x 2^20
                 rows of a 12.5 M x 128 table; row ids uniform, Zipf, and the step's mix of the two
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ITEMS = ("bench", "local_red", "no_head", "uniform_pos", "prebuilt_ids", "probe")

SHARDED = """
import json, os, sys
sys.path.insert(0, %(root)r)
import bench
cfg = bench.ShardedCfg
for k, v in %(cfg)r.items():
    setattr(cfg, k, v)
line = bench.measure_sharded(20, 5, 1, 0, [], with_cpu=False, cfg=cfg)
print(json.dumps({"ms_per_step": line["ms_per_step"], "launch_us": line["roofline"]["launch_us"],
                  "launch_us_min": line["roofline"]["launch_us_min"], "launch_us_max": line["roofline"]["launch_us_max"],
                  "GBps_algorithmic": line["roofline"]["achieved"], "lazy_adam_launch_us": line["lazy_adam"]["roofline"]["launch_us"]}))
"""

PREBUILT = """
import json, sys
sys.path.insert(0, %(root)r)
import numpy as np, torch
import bench
from neurec_b200 import ops
from neurec_b200.util import peer
cfg, K, W = bench.ShardedCfg, 20, 5
ptr, idx = bench.synth_shard_csr(cfg, 0, 1)
T = bench.TrainData(ptr, idx)
g = torch.Generator(device="cuda").manual_seed(30)
U = torch.empty((cfg.users_per_gpu, cfg.dim), device="cuda").normal_(0, 0.01, generator=g)
V = torch.empty((cfg.items_per_gpu, cfg.dim), device="cuda").normal_(0, 0.01, generator=g)
ni, bs = cfg.items_per_gpu, cfg.batch
spe = T.n_pos // bs
pos = [(s // spe, (s %% spe) * bs) for s in range(W + K)]        # (epoch, first) of every step, as bench.py steps
ids = [ops.epoch_build(T.ptr, T.idx, T.users, T.idx, 1, ni, True, True, bench.SEED, e, first=f, n_out=bs) for e, f in pos]
loss = torch.zeros(1, device="cuda")
VS = peer.single(V)
def fused(s):
    u, i, j = ids[s]
    ops.mf_bpr_sgd_fused(U, V, u, i, j.view(-1), cfg.lr, 0.0, loss)
def stream(s):
    ops.mf_bpr_sgd_epoch(U, VS, T.ptr, T.idx, T.users, T.idx, ni, True, bench.SEED, pos[s][0], pos[s][1], bs, cfg.lr, 0.0, loss)
def time_of(fn):
    for s in range(W):
        fn(s)
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2 * K)]
    torch.cuda.synchronize()
    for k in range(K):
        ev[2 * k].record(); fn(W + k); ev[2 * k + 1].record()
    torch.cuda.synchronize()
    return float(np.mean([ev[2 * k].elapsed_time(ev[2 * k + 1]) for k in range(K)])) * 1e3
out = {}
for rnd in range(2):
    out.setdefault("csr_fed_launch_us", []).append(time_of(stream))
    out.setdefault("prebuilt_fused_launch_us", []).append(time_of(fused))
print(json.dumps(out))
"""


def last_json(stdout):
    return json.loads(stdout.strip().splitlines()[-1])


def run_py(code, env=None):
    e = dict(os.environ)
    e.update(env or {})
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, env=e)
    if r.returncode:
        raise RuntimeError(r.stderr[-4000:])
    return last_json(r.stdout)


def sharded(root, env=None, cfg=None):
    return run_py(SHARDED % {"root": root, "cfg": cfg or {}}, env)


def probe():
    work = tempfile.mkdtemp()
    exe = os.path.join(work, "row_update_probe")
    subprocess.run([os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc"), "-gencode", "arch=compute_90a,code=sm_90a", "-O3",
                    "-o", exe, os.path.join(ROOT, "profiles", "row_update_probe.cu")], check=True)
    r = subprocess.run([exe], capture_output=True, text=True, check=True)
    return [json.loads(x) for x in r.stdout.splitlines() if x.startswith("{")]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("out")
    ap.add_argument("--root", default=ROOT)
    ap.add_argument("--label", default="this tree")
    ap.add_argument("--items", default=",".join(ITEMS))
    args = ap.parse_args()
    root = os.path.abspath(args.root)
    res = {}
    for item in args.items.split(","):
        if item == "bench":
            res[item] = sharded(root)
        elif item == "local_red":
            res[item] = sharded(root, env={"NRC_SGD_LOCAL_BULK": "0"})
        elif item == "no_head":
            res[item] = sharded(root, env={"NRC_BENCH_N_HOT": "0"})
        elif item == "uniform_pos":
            res[item] = sharded(root, cfg={"zipf_a": 0.0})
        elif item == "prebuilt_ids":
            res[item] = run_py(PREBUILT % {"root": root}, env={"NRC_BENCH_N_HOT": "0"})
        elif item == "probe":
            res[item] = probe()
        else:
            raise SystemExit("unknown item %r" % item)
        print(item, json.dumps(res[item]), flush=True)
    out = {}
    if os.path.exists(args.out):
        with open(args.out) as f:
            out = json.load(f)
    out["gpu"] = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                                capture_output=True, text=True).stdout.strip()
    out[args.label] = res
    with open(args.out, "w") as f:
        json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
