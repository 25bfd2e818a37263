"""Time of ItemKNN's similarity build and full-catalogue scoring on the device.

    python profiles/itemknn_build.py OUT_DIR [--repeats 3] [--warmup 1]

Workloads: the ml-100k ratio-0.8 split with its int64 ratings (tests/golden/ml100k_split.npz + the ratings in
tests/golden/kat_itemknn.npz) and the gowalla split as float64 ones (tests/golden/gowalla_split.npz), each under cosine
and euclidean at neighbor 5 and 800.  Reported per case: the route nrc_itemknn_last_routes took, the median time of
one nrc_itemknn_similarity (CUDA events, --repeats after --warmup untimed ones; the host preparation and the uploads
are outside the timed region), and, from the shapes, the products of the dot phase (the sum over users of n_u^2) and
the I^2 candidates the selection scans, as rates over that time; the time of nrc_itemknn_scores over the first
--score-users users (every user of ml-100k) in batches of 1 024, with the (user, W entry) lookups it makes.  The card's name and power limit are read in the same run; the JSON goes to
OUT_DIR/itemknn_build.json.
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


def train(name):
    import scipy.sparse as sp
    z = np.load(os.path.join(GOLDEN, name + "_split.npz"))
    ptr, idx = z["train_indptr"].astype(np.int64), z["train_indices"].astype(np.int32)
    if name == "ml100k":
        data = np.load(os.path.join(GOLDEN, "kat_itemknn.npz"))["ratings"].astype(np.int64)
    else:
        data = np.ones(len(idx))
    return sp.csr_matrix((data, idx, ptr), shape=(int(z["num_users"]), int(z["num_items"]))).tocsc()


def case(X0, similarity, K, repeats, warmup, max_users, batch=1024):
    import torch
    from neurec_b200 import ops
    from neurec_b200.model.general_recommender.ItemKNN import _dev_csr, prepare
    X, kind, va, vb = prepare(X0, similarity, 1)
    X.sort_indices()
    R = X.tocsr()
    R.sort_indices()
    nu, ni = X.shape
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()
    args = (*_dev_csr(R), *_dev_csr(X), ni, kind, t(va), t(vb), 0, 0.5, 0.5, K)
    holder = {}

    def build():
        holder["W"] = ops.itemknn_similarity(*args)

    ms = events_ms(build, repeats, warmup)
    route = ops.itemknn_last_routes()["similarity"]
    products = int((np.diff(R.indptr).astype(np.int64) ** 2).sum())
    S = X0.tocsr()
    S.sort_indices()
    tr = _dev_csr(S)
    scored = min(nu, max_users)
    users = torch.arange(scored, dtype=torch.int32, device="cuda")

    def score():
        for b in range(0, scored, batch):
            ops.itemknn_scores(*tr, holder["W"], users[b:b + batch])

    sms = events_ms(score, repeats, warmup)
    nnz = int(holder["W"][0].sum())
    return {"similarity": similarity, "neighbor": K, "users": nu, "items": ni, "route": route,
            "similarity_ms": ms, "dot_products": products, "dot_products_per_s": products / (ms * 1e-3),
            "candidates": ni * ni, "candidates_per_s": ni * ni / (ms * 1e-3), "w_entries": nnz,
            "scored_users": scored, "scores_ms": sms, "score_lookups": scored * nnz,
            "score_lookups_per_s": scored * nnz / (sms * 1e-3)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("out_dir")
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--score-users", type=int, default=2048)
    a = ap.parse_args()
    import torch
    torch.cuda.init()
    res = {"card": card(), "repeats": a.repeats, "warmup": a.warmup, "cases": []}
    for data in ("ml100k", "gowalla"):
        X0 = train(data)
        for similarity in ("cosine", "euclidean"):
            for K in (5, 800):
                r = dict(case(X0, similarity, K, a.repeats, a.warmup, a.score_users), dataset=data)
                res["cases"].append(r)
                print(json.dumps(r), flush=True)
    os.makedirs(a.out_dir, exist_ok=True)
    with open(os.path.join(a.out_dir, "itemknn_build.json"), "w") as f:
        json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
