"""Time of every SIMT evaluator form and of the tensor-core evaluator, on a gowalla-sized catalogue.

    python profiles/eval_forms.py OUT.json [--lib PATH] [--repeats 10] [--warmup 3] [--dump OUT.npz]
                                           [--against OTHER.npz]

Cases (40 981 items and the train/test sets of tests/golden/gowalla_split.npz; seeded N(0, 0.1) tables):
  * nrc_eval_mf, mf_form 2 (tie-free pass, 128-item tiles): 29 858 users, top_k 20, d = 64 and d = 128;
  * nrc_eval_mf, mf_form 1 (2 users per warp): 16 users per SM, top_k 20, d = 64;
  * nrc_eval_mf, mf_form 0 (heap replay only): 29 858 users, top_k 50, d = 64;
  * nrc_eval_mf, mf_form 3 (tie-free pass, 64-item tiles): 29 858 users, top_k 20, d = 256;
  * nrc_eval_score_matrix over 8 192 materialised, masked score rows, top_k 20, with its tie-free pass and without
    it (nrc_eval_force_exact), and nrc_arg_topk over the same rows;
  * nrc_eval_mf_tc: 29 858 users, top_k 20, d = 64 and d = 128.
Each case asserts the route the library reports (nrc_eval_last_routes) and is timed by CUDA events around one call:
--repeats timed calls after --warmup untimed ones; the median, minimum and maximum go to the JSON with the card's
name and power limit, read in the same run.  --lib loads another build of libneurec_b200.so through the same C ABI
(include/neurec_b200.h), so one script times two builds; --dump saves every case's ranks and metric rows, and
--against compares them with another run's dump (identical bits expected).
"""
import argparse
import ctypes
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

METRICS = np.array([1, 2, 3, 4, 5], np.int32)   # Precision, Recall, MAP, NDCG, MRR


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    name, power, clock = [s.strip() for s in q.stdout.splitlines()[0].split(",")]
    return {"name": name, "power_limit": power, "max_sm_clock": clock}


def load_lib(path):
    from neurec_b200 import _lib
    lib = ctypes.CDLL(path)
    for name, (ret, argtypes) in _lib.declared_functions().items():
        fn = getattr(lib, name)
        fn.restype, fn.argtypes = ret, argtypes
    return lib


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("out")
    ap.add_argument("--lib", default=os.path.join(ROOT, "neurec_b200", "libneurec_b200.so"))
    ap.add_argument("--repeats", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--dump", default=None)
    ap.add_argument("--against", default=None)
    a = ap.parse_args()

    import torch
    assert torch.cuda.is_available(), "eval_forms.py needs a CUDA device"
    lib = load_lib(os.path.abspath(a.lib))

    def ok(rc):
        if rc != 0:
            raise RuntimeError("rc %d: %s" % (rc, lib.nrc_last_error().decode()))

    p = lambda t: None if t is None else ctypes.c_void_p(t.data_ptr())
    stream = lambda: ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    m_ptr = METRICS.ctypes.data_as(ctypes.c_void_p)
    M = len(METRICS)

    z = np.load(os.path.join(ROOT, "tests", "golden", "gowalla_split.npz"))
    nu, ni = int(z["num_users"]), int(z["num_items"])
    dev = lambda x: torch.from_numpy(np.ascontiguousarray(x)).cuda()
    tp, ti = dev(z["train_indptr"].astype(np.int64)), dev(z["train_indices"].astype(np.int32))
    sp, si = dev(z["test_indptr"].astype(np.int64)), dev(z["test_indices"].astype(np.int32))
    rs = np.random.RandomState(0)
    tables = {}

    def table(d):
        if d not in tables:
            tables[d] = (dev((rs.randn(nu, d) * 0.1).astype(np.float32)), dev((rs.randn(ni, d) * 0.1).astype(np.float32)))
        return tables[d]

    def routes():
        r = (ctypes.c_int32 * 3)()
        ok(lib.nrc_eval_last_routes(r))
        return list(r)

    def timed(call):
        for _ in range(a.warmup):
            call()
        ts = []
        for _ in range(a.repeats):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            call()
            e1.record()
            e1.synchronize()
            ts.append(e0.elapsed_time(e1))
        return {"median_ms": float(np.median(ts)), "min_ms": float(min(ts)), "max_ms": float(max(ts))}

    sms = torch.cuda.get_device_properties(0).multi_processor_count
    cases, outputs = {}, {}

    def mf_case(name, form, n, d, K, tc=False):
        U, V = table(d)
        users = dev(np.arange(n, dtype=np.int32) % nu)
        res = torch.empty((n, M * K), dtype=torch.float32, device="cuda")
        ranks = torch.empty((n, K), dtype=torch.int32, device="cuda")
        if tc:
            call = lambda: ok(lib.nrc_eval_mf_tc(p(U), p(V), d, ni, p(users), n, p(tp), p(ti), p(sp), p(si), m_ptr, M,
                                                 K, 0, p(res), p(ranks), stream()))
        else:
            call = lambda: ok(lib.nrc_eval_mf(p(U), p(V), d, ni, p(users), n, p(tp), p(ti), p(sp), p(si), m_ptr, M, K,
                                              p(res), p(ranks), stream()))
        call()
        torch.cuda.synchronize()
        if not tc:
            assert routes()[0] == form, (name, routes())
        else:
            r, f = ctypes.c_int32(), ctypes.c_int32()
            ok(lib.nrc_eval_tc_last_fallbacks(ctypes.byref(r), ctypes.byref(f)))
        cases[name] = dict(timed(call), users=n, items=ni, dim=d, top_k=K, mf_form=None if tc else form)
        outputs[name + "/ranks"], outputs[name + "/results"] = ranks.cpu().numpy(), res.cpu().numpy()

    mf_case("eval_mf_form2_d64", 2, nu, 64, 20)
    mf_case("eval_mf_form2_d128", 2, nu, 128, 20)
    mf_case("eval_mf_form1_d64", 1, 16 * sms, 64, 20)
    mf_case("eval_mf_form0_d64_k50", 0, nu, 64, 50)
    mf_case("eval_mf_form3_d256", 3, nu, 256, 20)
    mf_case("eval_mf_tc_d64", None, nu, 64, 20, tc=True)
    mf_case("eval_mf_tc_d128", None, nu, 128, 20, tc=True)

    # materialised rows: the fused path's scores, train items masked to -inf
    R, K = 8192, 20
    U, V = table(64)
    users = dev(np.arange(R, dtype=np.int32))
    S = torch.empty((R, ni), dtype=torch.float32, device="cuda")
    ok(lib.nrc_mf_scores(p(U), p(V), 64, ni, p(users), R, p(S), stream()))
    ok(lib.nrc_mask_rows(p(S), ni, R, p(users), p(tp), p(ti), stream()))
    sub = z["test_indptr"][:R + 1].astype(np.int64)
    rp, ri = dev(sub), dev(z["test_indices"][:sub[-1]].astype(np.int32))
    for name, exact in (("score_matrix_fast", 0), ("score_matrix_exact", 1)):
        res = torch.empty((R, M * K), dtype=torch.float32, device="cuda")
        ranks = torch.empty((R, K), dtype=torch.int32, device="cuda")
        ok(lib.nrc_eval_force_exact(exact))
        call = lambda: ok(lib.nrc_eval_score_matrix(p(S), ni, R, p(rp), p(ri), m_ptr, M, K, p(res), p(ranks), stream()))
        call()
        torch.cuda.synchronize()
        assert routes()[1] == 1 - exact, (name, routes())
        cases[name] = dict(timed(call), rows=R, items=ni, top_k=K, rows_fast=1 - exact, rows_warps=routes()[2])
        outputs[name + "/ranks"], outputs[name + "/results"] = ranks.cpu().numpy(), res.cpu().numpy()
    ok(lib.nrc_eval_force_exact(0))
    top = torch.empty((R, K), dtype=torch.int32, device="cuda")
    call = lambda: ok(lib.nrc_arg_topk(p(S), ni, R, K, p(top), stream()))
    call()
    torch.cuda.synchronize()
    assert routes()[1] == 1, routes()
    cases["arg_topk"] = dict(timed(call), rows=R, items=ni, top_k=K, rows_fast=1, rows_warps=routes()[2])
    outputs["arg_topk/ranks"] = top.cpu().numpy()

    out = {"card": card(), "lib": os.path.relpath(os.path.abspath(a.lib), ROOT), "repeats": a.repeats,
           "warmup": a.warmup, "cases": cases}
    if a.dump:
        np.savez_compressed(a.dump, **outputs)
    if a.against:
        other = np.load(a.against)
        out["identical_to"] = os.path.basename(a.against)
        out["identical"] = {k: bool(np.array_equal(outputs[k], other[k])) for k in sorted(outputs)}
    with open(a.out, "w") as f:
        json.dump(out, f, indent=1)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
