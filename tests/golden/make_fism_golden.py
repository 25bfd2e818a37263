"""Generates tests/golden/kat_fism_layout.json by running the UNMODIFIED reference's FISM instance generators.

Run from the repo root:  ``python tests/golden/make_fism_golden.py``  (needs the reference, like make_golden.py).
The fixture is committed, so the tests never need the reference.

What is captured: util/data_generator.py's _get_pointwise_all_likefism_data (num_negatives = 4, train_dict from the
reference's csr_to_user_dict) and _get_pairwise_all_likefism_data, run by the reference on the train CSR of the
ratio-0.8 ml-100k split (ml100k_split.npz): counts and crc32 of the histories (lengths, then the items of every
history in order), num_idx, the positives and the labels.  The random negatives are not pinned.
"""
import importlib
import json
import os
import zlib

import numpy as np
import scipy.sparse as sp

from make_golden import OUT


def crc(a):
    return int(zlib.crc32(np.ascontiguousarray(np.asarray(a), dtype=np.int32).tobytes()))


def hist_crc(lists):
    lens = [len(h) for h in lists]
    flat = np.concatenate([np.asarray(h, np.int32) for h in lists]) if lists else np.zeros(0, np.int32)
    return {"n_rows": int(sum(lens)), "lens_crc32": crc(lens), "items_crc32": crc(flat)}


def fism():
    import oracle
    cwd = oracle.import_reference()
    os.chdir(cwd)
    gen = importlib.import_module("util.data_generator")
    tool = importlib.import_module("util.tool")
    z = np.load(os.path.join(OUT, "ml100k_split.npz"))
    nu, ni = int(z["num_users"]), int(z["num_items"])
    train = sp.csr_matrix((np.ones(len(z["train_indices"]), np.float32), z["train_indices"].astype(np.int32),
                           z["train_indptr"].astype(np.int64)), shape=(nu, ni))

    class _Data:
        num_users, num_items, train_matrix = nu, ni, train

    np.random.seed(2018)
    users, num_idx, items, labels = gen._get_pointwise_all_likefism_data(_Data, 4, tool.csr_to_user_dict(train))
    labels = np.asarray(labels, np.int32)
    res = {"num_users": nu, "num_items": ni, "pointwise": {
        "num_neg": 4, "n": len(users), "histories": hist_crc(users), "num_idx_crc32": crc(num_idx),
        "labels_crc32": crc(labels), "positives_crc32": crc(np.asarray(items, np.int32)[labels == 1])}}
    up, un, nip, nin, ip, _ = gen._get_pairwise_all_likefism_data(_Data)
    res["pairwise"] = {"n": len(up), "histories_pos": hist_crc(up), "histories_neg": hist_crc(un),
                       "num_idx_pos_crc32": crc(nip), "num_idx_neg_crc32": crc(nin), "positives_crc32": crc(ip)}
    with open(os.path.join(OUT, "kat_fism_layout.json"), "w") as fo:
        json.dump(res, fo, indent=1)
    print("fism fixture written", res)


if __name__ == "__main__":
    fism()
