"""Generates tests/golden/kat_caser_sequences.json by running the UNMODIFIED reference's Caser._generate_sequences.

Run from the repo root:  ``python tests/golden/make_caser_golden.py``  (needs /root/reference, like make_golden.py).
The fixture is committed; the GPU box never runs this script and never reads /root/reference.

What is captured: Caser._generate_sequences (model/sequential_recommender/Caser.py:144-172) run by the reference on the
by-time train sequences of the ratio-0.8 ml-100k split (kat_split_ml100k.npz, make_golden.py's by_time_dict), items
remapped to dense ids, at (seq_L, seq_T) = (5, 3) and at (12, 8), which pre-pads the users with fewer than 20 train
items: counts and crc32 of its users, windows, positives and predict windows, and the number of pad ids among the
windows and the positives.
"""
import importlib
import json
import os
import zlib

import numpy as np

from make_golden import OUT, by_time_dict


def caser():
    import oracle
    cwd = oracle.import_reference()
    os.chdir(cwd)
    Caser = importlib.import_module("model.sequential_recommender.Caser").Caser
    z = np.load(os.path.join(OUT, "kat_split_ml100k.npz"))
    n = int(z["n"])
    items = np.unique(z["item"], return_inverse=True)[1]
    d = by_time_dict(z["user"].astype(np.int64), items, z["time"].astype(np.int64), np.unpackbits(z["ratio"])[:n])
    num_items = int(items.max()) + 1
    crc = lambda a: int(zlib.crc32(np.ascontiguousarray(a, dtype=np.int32).tobytes()))
    res = {"num_items": num_items, "settings": {}}
    for L, T in ((5, 3), (12, 8)):
        m = Caser.__new__(Caser)                       # only the generator's inputs: no session, dataset or graph
        m.user_pos_train, m.seq_L, m.seq_T, m.items_num = d, L, T, num_items
        users, seqs, pos = m._generate_sequences()
        tu = sorted(m.user_test_seq)
        res["settings"]["%d,%d" % (L, T)] = {
            "n": len(users), "users_crc32": crc(users), "seqs_crc32": crc(np.stack(seqs)), "pos_crc32": crc(np.stack(pos)),
            "n_test": len(tu), "test_users_crc32": crc(tu),
            "test_seq_crc32": crc(np.stack([m.user_test_seq[u] for u in tu])),
            "pad_pos": int((np.stack(pos) == num_items).sum()), "pad_seq": int((np.stack(seqs) == num_items).sum())}
    with open(os.path.join(OUT, "kat_caser_sequences.json"), "w") as fo:
        json.dump(res, fo, indent=1)
    print("caser fixture written", res)


if __name__ == "__main__":
    caser()
