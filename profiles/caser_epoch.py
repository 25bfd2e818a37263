"""Time of one Caser training epoch, the split of one of its steps between launches, the per-step table passes at a
gowalla-sized shape, and full evaluation, on the device.

    python profiles/caser_epoch.py OUT_DIR [--repeats 10] [--warmup 2]

Workloads:
  * ml-100k at conf/Caser.properties' defaults: the time-ordered train set of the reference's ratio-0.8 split
    (tests/golden/kat_split_ml100k.npz; 943 users, 1 682 items), 73 766 instances at (seq_L, seq_T) = (5, 3), batch
    256 (289 steps), d 50, nv 4, nh 16, 3 negatives, dropout 0.5, l2_reg 1e-3, Adam;
  * gowalla-sized: 29 858 users and 40 981 items (the tables P, E, W2 and b2 hold 7.68 M floats) with 30 random train
    items per user, the same hyper-parameters, 64 steps of 256 instances.
Reported:
  * fused_epoch_ms: CUDA events around one nrc_caser_train_epoch on an epoch already on the device (median over
    --repeats after --warmup untimed repeats);
  * step_split_us: per kernel, the device time per step from torch.profiler over one fused epoch run in a separate,
    profiled pass: the dropout mask, the reg pass, the gradient kernel, the dense-gradient reduction and the Adam
    launch;
  * at the gowalla-sized shape, the reg pass and the Adam launch per step against the HBM bytes they must move (reg:
    read var, write grad, 8 B per table float; Adam: read var, grad, m, v and write var, m, v, 28 B per float), as
    bytes over time against 3.35 TB/s;
  * evaluate_ms: the plug-in's evaluation on ml-100k (NeuRec.properties' options), host clock after a synchronise;
    gowalla_scores_ms: CUDA events around the query and scores of all 29 858 users x 40 981 items in batches of 1 024.
The card's name and power limit are read in the same run; the JSON goes to OUT_DIR/caser_epoch.json.
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "profiles"))
HBM_BYTES_PER_S = 3.35e12
KERNELS = {"mask": "dropout_mask_kernel", "reg": "caser_reg_kernel", "grad": "caser_grad_kernel",
           "wgrad": "caser_wgrad_kernel", "adam": "opt_apply_kernel"}


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


def kernel_split(fn, steps):
    """Device time per step of each launch kind, from torch.profiler over one call of fn."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    tot = {k: 0.0 for k in KERNELS}
    for e in prof.key_averages():
        for k, pat in KERNELS.items():
            if pat in e.key:
                tot[k] += e.device_time_total
    return {k: v / steps for k, v in tot.items()}


class Epoch(object):
    """Device arrays and state for one Caser epoch call at the conf defaults."""

    def __init__(self, train_dict, nu, ni, d=50, L=5, T=3, nv=4, nh=16, N=3, bsz=256, limit=None):
        import torch
        from neurec_b200 import ops
        from neurec_b200.model.sequential_recommender.Caser import generate_sequences
        from oracle import tf_math
        users, seqs, pos, _ = generate_sequences(train_dict, L, T, ni)
        ptr = np.zeros(nu + 1, np.int64)
        for u, it in train_dict.items():
            ptr[u + 1] = len(it)
        ptr = np.cumsum(ptr)
        idx = np.concatenate([np.sort(np.asarray(train_dict[u], np.int32)) for u in sorted(train_dict)])
        t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()
        du = t(users)
        neg = ops.sample_negatives(t(ptr), t(idx), du, N, ni, 2018, 0)
        perm = ops.shuffle_perm(len(users), 2018, 0)
        self.batch = [ops.gather_rows_i32(a, perm) for a in (du, t(seqs), t(pos), neg)]
        if limit is not None:
            self.batch = [a[:limit].contiguous() for a in self.batch]
        self.n = self.batch[0].numel()
        self.steps = (self.n + bsz - 1) // bsz
        rs = np.random.RandomState(0)
        self.vars = [t((rs.randn(*s) * 0.05).astype(np.float32)) for s in
                     ((nu, d), (ni, d), (ni, 2 * d), (ni,), (ops.caser_dense_floats(d, L, nv, nh),))]
        self.grads = [torch.zeros_like(v) for v in self.vars]
        self.s0 = [torch.zeros_like(v) for v in self.vars]
        self.s1 = [torch.zeros_like(v) for v in self.vars]
        self.work = ops.caser_work(d, L, nv, nh, bsz)
        self.loss = torch.zeros(self.steps, device="cuda")
        self.lr_t = tf_math.adam_lr_t(1e-3, self.steps)
        self.shape = (nv, nh, bsz)
        self.table_floats = sum(v.numel() for v in self.vars[:4])
        self.dense_floats = self.vars[4].numel()

    def run(self):
        from neurec_b200 import ops
        nv, nh, bsz = self.shape
        ops.caser_train_epoch(*self.vars, *self.batch, nv, nh, bsz, 0.5, 1e-3, 2018, 1, self.lr_t,
                              [1e-3, 0.9, 0.999, 1e-8], self.grads, self.s0, self.s1, self.work, self.loss)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("out_dir")
    ap.add_argument("--repeats", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    args = ap.parse_args()
    import torch
    from neurec_b200 import ops
    from seq_epoch import ml100k_time_ordered
    assert torch.cuda.is_available(), "caser_epoch.py measures on the GPU"
    res = {"card": card()}
    # ml-100k at the defaults
    ds = ml100k_time_ordered()
    td = ds.get_user_train_dict(by_time=True)
    e = Epoch(td, ds.num_users, ds.num_items)
    ms = events_ms(e.run, args.repeats, args.warmup)
    split = kernel_split(e.run, e.steps)
    res["ml100k"] = {"instances": e.n, "steps": e.steps, "fused_epoch_ms": ms, "step_us": 1e3 * ms / e.steps,
                     "step_split_us": split, "routes": ops.caser_last_routes()}
    # gowalla-sized tables
    nu, ni = 29858, 40981
    rs = np.random.RandomState(1)
    gd = {u: list(rs.choice(ni, 30, replace=False)) for u in range(nu)}
    g = Epoch(gd, nu, ni, limit=64 * 256)
    gms = events_ms(g.run, args.repeats, args.warmup)
    gsplit = kernel_split(g.run, g.steps)
    tf, df = g.table_floats, g.dense_floats
    reg_bytes, adam_bytes = 8.0 * tf, 28.0 * (tf + df)
    res["gowalla_sized"] = {
        "users": nu, "items": ni, "table_floats": tf, "dense_floats": df, "steps": g.steps, "fused_ms": gms,
        "step_us": 1e3 * gms / g.steps, "step_split_us": gsplit,
        "reg_bytes": reg_bytes, "reg_tb_s": reg_bytes / (gsplit["reg"] * 1e-6) / 1e12,
        "reg_share_of_hbm": reg_bytes / (gsplit["reg"] * 1e-6) / HBM_BYTES_PER_S,
        "adam_bytes": adam_bytes, "adam_tb_s": adam_bytes / (gsplit["adam"] * 1e-6) / 1e12,
        "adam_share_of_hbm": adam_bytes / (gsplit["adam"] * 1e-6) / HBM_BYTES_PER_S}
    # full evaluation on ml-100k through the plug-in; scoring every gowalla-sized user
    from neurec_b200.model.sequential_recommender.Caser import Caser
    conf = {"metric": ["Precision", "Recall", "NDCG", "MAP", "MRR"], "group_view": None, "topk": [10, 20],
            "test_batch_size": 128, "num_thread": 8, "recommender": "Caser", "lr": 0.001, "l2_reg": 0.001,
            "factors_num": 50, "seq_L": 5, "seq_T": 3, "nv": 4, "nh": 16, "dropout": 0.5, "neg_samples": 3,
            "batch_size": 256, "epochs": 1}

    class Conf(dict):
        def params_str(self):
            return "profile"

    cwd = os.getcwd()
    os.chdir(tempfile.mkdtemp())
    m = Caser(None, ds, Conf(conf))
    m.build_graph()
    m._train_epoch()
    ev = []
    for r in range(args.warmup + args.repeats):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        m.evaluate()
        torch.cuda.synchronize()
        if r >= args.warmup:
            ev.append(1e3 * (time.perf_counter() - t0))
    os.chdir(cwd)
    windows = torch.randint(0, ni, (nu, 5), dtype=torch.int32, device="cuda")
    P, E, W2, _, dense = g.vars

    def score_all():
        for off in range(0, nu, 1024):
            users = torch.arange(off, min(nu, off + 1024), dtype=torch.int32, device="cuda")
            ops.caser_scores(P, E, W2, dense, users, windows, 4, 16)

    res["evaluate_ms"] = float(np.median(ev))
    res["gowalla_scores_ms"] = events_ms(score_all, args.repeats, args.warmup)
    os.makedirs(args.out_dir, exist_ok=True)
    with open(os.path.join(args.out_dir, "caser_epoch.json"), "w") as f:
        json.dump(res, f, indent=1)
    print(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
