"""Time of one FPMC, TransRec, HRM, NPE and FPMCplus training epoch, and of one full evaluation of each, on the device.

    python profiles/seq_epoch.py OUT_DIR [--repeats 20] [--warmup 3]

Workload: the time-ordered ml-100k train set (the reference's ratio-0.8 split in tests/golden/kat_split_ml100k.npz,
users and items remapped to dense ids: 943 users, 1 682 items, 79 424 (user, recent, next) instances at
high_order = 1, 78 481 at 2 and 77 538 at 3), each model at its conf file's defaults:
  * FPMC      pointwise cross_entropy, num_neg 4 (397 120 samples), batch 512 (776 steps), d 16, adam, reg 0.01;
  * TransRec  pairwise bpr (79 424 samples), batch 1024 (78 steps), d 50, adam, reg 0;
  * HRM       high_order 2, max / max pools, cross_entropy, num_neg 4 (392 405 samples), batch 256 (1 533 steps),
              d 16, adam, reg 0;
  * NPE       high_order 3, cross_entropy, num_neg 4 (387 690 samples), batch 256 (1 515 steps), d 64, adam, reg 0.1;
  * FPMCplus  high_order 3, pairwise bpr (77 538 samples), batch 128 (606 steps), d 16, weight_size 16, adam,
              reg_mf 1e-5, reg_w 1e-3.
Per model, medians over --repeats after --warmup untimed repeats:
  * fused_epoch_ms: CUDA events around the one fused epoch call (nrc_<model>_train_epoch: per batch the gradient
    kernel(s) and one optimizer launch) on an epoch already on the device;
  * plug_in_epoch_ms: the plug-in's whole epoch (the sampler's device epoch, Adam's per-step lr_t on the host, the
    fused call, the loss read back), host clock around it;
  * score_kernel_ms: CUDA events around scoring all 943 users x 1 682 items (the score kernel; for HRM and NPE the
    query kernel and nrc_mf_scores; for FPMCplus the projection pass and the pair kernel);
  * evaluate_ms: the plug-in's evaluation with NeuRec.properties' options (predict in batches of 128 users, train
    items masked, five metrics at top 10 and 20), host clock after a device synchronise.
The card's name and power limit are read in the same run; the JSON goes to OUT_DIR/seq_epoch.json.
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
MODELS = ("FPMC", "TransRec", "HRM", "NPE", "FPMCplus")


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    name, power, clock = [s.strip() for s in q.stdout.splitlines()[0].split(",")]
    return {"name": name, "power_limit": power, "max_sm_clock": clock}


def ml100k_time_ordered():
    from scipy import sparse as sp
    from neurec_b200.data import Dataset
    z = np.load(os.path.join(ROOT, "tests", "golden", "kat_split_ml100k.npz"))
    n = int(z["n"])
    users = np.unique(z["user"], return_inverse=True)[1]
    items = np.unique(z["item"], return_inverse=True)[1]
    train = np.unpackbits(z["ratio"])[:n].astype(bool)
    shape = (int(users.max()) + 1, int(items.max()) + 1)
    mk = lambda m, data: sp.csr_matrix((data[m], (users[m], items[m])), shape=shape)
    ones = np.ones(n, np.float32)
    return Dataset.from_csr("ml-100k", mk(train, ones), mk(~train, ones),
                            time_matrix=mk(train, z["time"].astype(np.float64)))


def load_conf(name):
    """NeuRec.properties + conf/<name>.properties as main.py reads them (defaults only)."""
    from neurec_b200.util import Configurator
    cwd, argv = os.getcwd(), sys.argv
    try:
        os.chdir(ROOT)
        sys.argv = [argv[0], "--recommender=%s" % name]
        return Configurator("NeuRec.properties", default_section="hyperparameters")
    finally:
        os.chdir(cwd)
        sys.argv = argv


def measure(name, conf, ds, repeats, warmup):
    import torch
    from neurec_b200 import ops
    from neurec_b200.model.sequential_recommender.FPMC import FPMC
    from neurec_b200.model.sequential_recommender.FPMCplus import FPMCplus
    from neurec_b200.model.sequential_recommender.HRM import HRM
    from neurec_b200.model.sequential_recommender.NPE import NPE
    from neurec_b200.model.sequential_recommender.TransRec import TransRec
    m = {"FPMC": FPMC, "TransRec": TransRec, "HRM": HRM, "NPE": NPE, "FPMCplus": FPMCplus}[name](None, ds, conf)
    m.build_graph()
    sampler = m.data_iter()
    epoch = sampler.device_epoch()
    n, bs = epoch[0].numel(), m.batch_size
    steps = (n + bs - 1) // bs
    lr_t = m.opt.lr_t(steps)
    step_loss = torch.empty(steps, device="cuda")
    reg = m.reg if name == "NPE" else m.reg_mf
    users = torch.arange(ds.num_users, dtype=torch.int32, device="cuda")

    def fused_call():
        opt = (m.opt.kind, lr_t, m.opt.hyper, m._grads, m._touched, m._slots0, m._slots1, m.opt.take_stamps(steps))
        if name == "FPMC":
            ops.fpmc_train_epoch(*m.tables(), *epoch, bs, m.is_pairwise is True, m._loss, reg, *opt, step_loss)
        elif name == "TransRec":
            ops.transrec_train_epoch(*m.tables(), *epoch, bs, m.is_pairwise is True, m._loss, reg, *opt, m._work,
                                     step_loss)
        elif name == "FPMCplus":
            ops.fpmcplus_train_epoch(*m.tables(), *epoch, bs, m.is_pairwise is True, m._loss, reg, m.reg_w, *opt,
                                     m._work, step_loss)
        elif name == "HRM":
            ops.hrm_train_epoch(*m.tables(), *epoch, bs, *m._pools(), m._loss, reg, *opt, step_loss)
        else:
            ops.npe_train_epoch(*m.tables(), *epoch, bs, m._loss, reg, *opt, step_loss)

    if name in ("FPMC", "TransRec"):
        last = torch.from_numpy(m._last).cuda()
        scores = ops.fpmc_scores if name == "FPMC" else ops.transrec_scores
        score_call = lambda: scores(*m.tables(), users, last)
    else:
        score_call = lambda: m._scores(users)

    def events(fn):
        for _ in range(warmup):
            fn()
        ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(repeats)]
        torch.cuda.synchronize()
        for a, b in ev:
            a.record()
            fn()
            b.record()
        torch.cuda.synchronize()
        return np.array([a.elapsed_time(b) for a, b in ev])

    def wall(fn):
        for _ in range(warmup):
            fn()
        out = []
        for _ in range(repeats):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            fn()
            torch.cuda.synchronize()
            out.append((time.perf_counter() - t0) * 1e3)
        return np.array(out)

    fused_ms = events(fused_call)
    plug_ms = wall(m._train_epoch)
    score_ms = events(score_call)
    eval_ms = wall(lambda: m.evaluator.evaluate(m))
    assert all(bool(torch.isfinite(t).all()) for t in m.tables())
    stat = lambda a: {"median": float(np.median(a)), "min": float(a.min()), "max": float(a.max())}
    return {"model": name, "dim": m.embedding_size, "pairwise": getattr(m, "is_pairwise", False) is True,
            "high_order": sampler.high_order, "loss": m._loss, "learner": m.learner, "reg": reg, "batch_size": bs,
            "samples": n, "steps": steps,
            "instances": int(len(sampler._users_np)), "num_users": ds.num_users, "num_items": ds.num_items,
            "fused_epoch_ms": stat(fused_ms), "fused_step_us_median": float(np.median(fused_ms)) * 1e3 / steps,
            "plug_in_epoch_ms": stat(plug_ms), "score_kernel_ms": stat(score_ms), "evaluate_ms": stat(eval_ms)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("out_dir")
    ap.add_argument("--repeats", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    a = ap.parse_args()
    import torch
    assert torch.cuda.is_available(), "this measurement needs a CUDA device"
    out_dir = os.path.abspath(a.out_dir)
    os.makedirs(out_dir, exist_ok=True)
    confs = {name: load_conf(name) for name in MODELS}
    os.chdir(tempfile.mkdtemp())                        # the models' log files stay out of the tree
    ds = ml100k_time_ordered()
    result = {"card": card(), "repeats": a.repeats, "warmup": a.warmup, "models": []}
    for name in MODELS:
        result["models"].append(measure(name, confs[name], ds, a.repeats, a.warmup))
        print(json.dumps(result["models"][-1]), flush=True)
    with open(os.path.join(out_dir, "seq_epoch.json"), "w") as f:
        json.dump(result, f, indent=1)
        f.write("\n")
    print(json.dumps(result["card"]))


if __name__ == "__main__":
    main()
