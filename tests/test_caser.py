"""Caser on the CPU: the restatement in tests/caser_math.py against a torch float64 autograd graph of the reference's
Caser.py:70-118 (conv2d on kernels permuted from TF's layout, so the flatten order is checked too), the sequence
generator against the reference's own output on ml-100k (tests/golden/kat_caser_sequences.json), the conf file
against the reference's values, model resolution and the ABI's argument checks."""
import json
import os
import sys
import zlib

import numpy as np
import pytest
import torch
import torch.nn.functional as Fn

import caser_math as cm
from conftest import ROOT

GOLDEN = os.path.join(ROOT, "tests", "golden")

# the reference's conf/Caser.properties, key by key, with the types its parser gives
REFERENCE_CONF = {"lr": 0.001, "l2_reg": 0.001, "factors_num": 50, "seq_L": 5, "seq_T": 3, "nv": 4, "nh": 16,
                  "dropout": 0.5, "neg_samples": 3, "batch_size": 256, "epochs": 1000}


def _autograd(P, E, W2, b2, dense, d, L, nv, nh, users, seqs, pos, neg, mask, keep):
    """The reference's graph in torch float64: conv2d over the [L, d] image (TF's NHWC kernels [kh, kw, in, out]
    permuted to [out, in, kh, kw]), amax (ties share the gradient, as TF's reduce_max), dropout as (x / keep) * mask."""
    t = lambda a: torch.tensor(np.asarray(a, np.float64), requires_grad=True)
    vP, vE, vW2, vb2, vD = t(P), t(E), t(W2), t(b2), t(dense)
    lay = {name: (off, shape) for name, off, shape in cm.dense_layout(d, L, nv, nh)[0]}
    part = lambda name: vD[lay[name][0]:lay[name][0] + int(np.prod(lay[name][1]))].reshape(lay[name][1])
    Ez = torch.cat([vE, torch.zeros(1, d, dtype=torch.float64)])
    img = Ez[torch.as_tensor(seqs)].unsqueeze(1)                           # [B, 1, L, d]
    B = img.shape[0]
    out_v = Fn.conv2d(img, part("Kv").permute(3, 2, 0, 1), part("bv"))    # [B, nv, 1, d]
    out_v = out_v.permute(0, 2, 3, 1).reshape(B, d * nv)                  # TF's (b, 1, d, nv) flattened
    pools = []
    for h in range(1, L + 1):
        c = torch.relu(Fn.conv2d(img, part("Kh%d" % h).permute(3, 2, 0, 1), part("bh%d" % h)))   # [B, nh, L-h+1, 1]
        pools.append(torch.amax(c.squeeze(3), dim=2))
    feat = torch.cat([out_v] + pools, 1)
    o = feat if mask is None else (feat / keep) * torch.as_tensor(np.asarray(mask, np.float64))
    z = torch.relu(o @ part("W1") + part("b1"))
    u = torch.cat([z, vP[torch.as_tensor(users)]], 1)
    tgt = torch.as_tensor(np.concatenate([pos, neg], 1))
    W2z = torch.cat([vW2, torch.zeros(1, 2 * d, dtype=torch.float64)])
    b2z = torch.cat([vb2, torch.zeros(1, dtype=torch.float64)])
    x = (u.unsqueeze(1) * W2z[tgt]).sum(-1) + b2z[tgt]
    T = pos.shape[1]
    s = torch.sigmoid(x)
    loss = torch.mean(-torch.log(s[:, :T] + 1e-24)) + torch.mean(-torch.log(1 - s[:, T:] + 1e-24))
    loss.backward()
    return loss.item(), [v.grad.numpy() for v in (vP, vE, vW2, vb2, vD)]


def _case(rs, d, L, nv, nh, B, T, N, nu=7, ni=11, pads=False, ties=False):
    P = rs.randn(nu, d) * 0.5
    E = rs.randn(ni, d) * 0.5
    W2 = rs.randn(ni, 2 * d) * 0.5
    b2 = rs.randn(ni) * 0.1
    dense = rs.randn(cm.dense_layout(d, L, nv, nh)[1]) * 0.4
    users = rs.randint(0, nu, B)
    seqs = rs.randint(0, ni, (B, L))
    pos, neg = rs.randint(0, ni, (B, T)), rs.randint(0, ni, (B, N))
    if pads:
        seqs[0, :L - 1] = ni                                             # a short user's pre-padded window
        pos[0, 0] = ni                                                   # and a pad id among its positives
        seqs[-1, 0] = ni
    if ties:
        # identical window rows give identical conv_h outputs at every position (forced max ties); a negative
        # bias on some filters gives exact relu zeros
        seqs[0, :] = seqs[0, 0]
        lay = {name: off for name, off, _ in cm.dense_layout(d, L, nv, nh)[0]}
        for h in range(1, L + 1):
            dense[lay["bh%d" % h]:lay["bh%d" % h] + nh:2] = -50.0
    return P, E, W2, b2, dense, users, seqs, pos, neg


CASES = [  # d, L, nv, nh, B, T, N, pads, ties, masked
    (4, 3, 2, 3, 5, 2, 3, False, False, False),
    (5, 4, 3, 2, 6, 3, 2, True, False, True),
    (3, 5, 2, 4, 4, 3, 3, False, True, False),
    (6, 2, 1, 2, 3, 1, 1, True, True, True),
    (2, 1, 1, 1, 2, 1, 2, False, False, True),
]


@pytest.mark.parametrize("case", CASES)
def test_restatement_equals_autograd(case):
    d, L, nv, nh, B, T, N, pads, ties, masked = case
    rs = np.random.RandomState(sum(case[:7]))
    P, E, W2, b2, dense, users, seqs, pos, neg = _case(rs, d, L, nv, nh, B, T, N, pads=pads, ties=ties)
    F = nv * d + nh * L
    mask = (rs.rand(B, F) < 0.6).astype(np.float64) if masked else None
    keep = 0.6 if masked else 1.0
    want_loss, want = _autograd(P, E, W2, b2, dense, d, L, nv, nh, users, seqs, pos, neg, mask, keep)
    loss, got = cm.loss_and_grad(P, E, W2, b2, dense, d, L, nv, nh, users, seqs, pos, neg, mask, keep)
    assert abs(loss - want_loss) <= 1e-12 * max(1.0, abs(want_loss))
    for g, w in zip(got, want):
        assert g.shape == w.shape
        np.testing.assert_allclose(g, w, rtol=1e-10, atol=1e-12)
    if pads:
        # the pad target's loss term counts (x = 0) but it sends no gradient; pad window rows send none
        assert np.all(np.isfinite(got[1])) and got[2].shape[0] == E.shape[0]
    if ties:
        f = cm.forward(P, E, dense, d, L, nv, nh, users, seqs)
        assert any((a[0] == a[0].max(0)).sum(0).max() > 1 for a in f["acts"][:-1])
        assert any((a == 0).any() for a in f["acts"])


def test_means_run_over_the_batch_that_is_present():
    """A partial last batch: the loss and its gradients are the means over its own rows (DataIterator keeps it)."""
    rs = np.random.RandomState(3)
    d, L, nv, nh, T, N = 4, 3, 2, 2, 2, 3
    P, E, W2, b2, dense, users, seqs, pos, neg = _case(rs, d, L, nv, nh, 5, T, N)
    part = slice(3, 5)
    loss, g = cm.loss_and_grad(P, E, W2, b2, dense, d, L, nv, nh, users[part], seqs[part], pos[part], neg[part])
    want_loss, want = _autograd(P, E, W2, b2, dense, d, L, nv, nh, users[part], seqs[part], pos[part], neg[part],
                                None, 1.0)
    assert abs(loss - want_loss) <= 1e-12
    np.testing.assert_allclose(g[4], want[4], rtol=1e-10, atol=1e-12)
    # the same two samples inside a batch of 5 weigh 2/5 as much
    _, g_all = cm.loss_and_grad(P, E, W2, b2, dense, d, L, nv, nh, users, seqs, pos, neg)
    assert not np.allclose(g_all[4], g[4])


def test_query_is_the_forward_without_dropout():
    rs = np.random.RandomState(4)
    d, L, nv, nh = 5, 4, 2, 3
    P, E, W2, b2, dense, users, seqs, pos, neg = _case(rs, d, L, nv, nh, 3, 1, 1)
    u = cm.query(P, E, dense, d, L, nv, nh, users, seqs)
    f = cm.forward(P, E, dense, d, L, nv, nh, users, seqs, mask=np.ones((3, nv * d + nh * L)), keep=1.0)
    np.testing.assert_array_equal(u, f["u"])
    np.testing.assert_array_equal(u[:, d:], P[users])


def _by_time_ml100k():
    z = np.load(os.path.join(GOLDEN, "kat_split_ml100k.npz"))
    n = int(z["n"])
    users, times = z["user"].astype(np.int64), z["time"].astype(np.int64)
    items = np.unique(z["item"], return_inverse=True)[1]                 # dense item ids, as make_caser_golden.py
    flags = np.unpackbits(z["ratio"])[:n]
    uid = np.unique(users, return_inverse=True)[1]                      # same construction as make_golden.by_time_dict
    keep = np.nonzero(flags)[0]
    order = keep[np.lexsort((keep, times[keep], uid[keep]))]
    d = {}
    for e in order:
        d.setdefault(int(uid[e]), []).append(int(items[e]))
    return d


def test_sequences_equal_the_reference_on_ml100k():
    """Caser._generate_sequences run by the REAL reference (tests/golden/make_caser_golden.py) on the by-time train
    sequences of the ratio-0.8 ml-100k split: the plug-in's numpy restatement gives the same instances and predict
    windows, bit for bit, at (L, T) = (5, 3) and at (12, 8), where short users are pre-padded."""
    from neurec_b200.model.sequential_recommender.Caser import generate_sequences
    with open(os.path.join(GOLDEN, "kat_caser_sequences.json")) as f:
        kat = json.load(f)
    d = _by_time_ml100k()
    crc = lambda a, dt: int(zlib.crc32(np.ascontiguousarray(a, dtype=dt).tobytes()))
    for key, want in kat["settings"].items():
        L, T = (int(x) for x in key.split(","))
        users, seqs, pos, test = generate_sequences(d, L, T, kat["num_items"])
        assert len(users) == want["n"]
        assert crc(users, np.int32) == want["users_crc32"]
        assert crc(seqs, np.int32) == want["seqs_crc32"]
        assert crc(pos, np.int32) == want["pos_crc32"]
        tu = sorted(test)
        assert len(tu) == want["n_test"]
        assert crc(tu, np.int32) == want["test_users_crc32"]
        assert crc(np.stack([test[u] for u in tu]), np.int32) == want["test_seq_crc32"]
        assert int((pos == kat["num_items"]).sum()) == want["pad_pos"]
        assert int((seqs == kat["num_items"]).sum()) == want["pad_seq"]


def test_conf_parses_to_the_reference_values(tmp_path, monkeypatch):
    from neurec_b200.util import Configurator
    (tmp_path / "conf").mkdir()
    (tmp_path / "conf" / "Caser.properties").write_text(open(os.path.join(ROOT, "conf", "Caser.properties")).read())
    (tmp_path / "NeuRec.properties").write_text(open(os.path.join(ROOT, "NeuRec.properties")).read())
    monkeypatch.chdir(tmp_path)
    monkeypatch.setattr(sys, "argv", ["main.py", "--recommender=Caser"])
    conf = Configurator("NeuRec.properties", default_section="hyperparameters")
    for key, value in REFERENCE_CONF.items():
        assert conf[key] == value and type(conf[key]) is type(value), key


def test_main_resolves_caser():
    import main
    from neurec_b200.model.sequential_recommender.Caser import Caser
    assert main.resolve_model("Caser") is Caser
    with pytest.raises(ImportError, match="HRM, NPE, FPMCplus, Caser"):
        main.resolve_model("SASRec")


def test_glorot_uniform_uses_tf_fans():
    from neurec_b200.model.sequential_recommender.Caser import glorot_uniform
    g = torch.Generator().manual_seed(0)
    x = glorot_uniform([3, 50, 1, 16], g)                               # fan_in 150, fan_out 2400
    assert x.shape == (3, 50, 1, 16) and float(x.abs().max()) <= (6.0 / 2550) ** 0.5
    g2 = torch.Generator().manual_seed(0)
    np.testing.assert_array_equal(x.numpy(), ((torch.rand(3, 50, 1, 16, generator=g2) * 2 - 1) *
                                              (6.0 / 2550) ** 0.5).numpy())


def _lib():
    from neurec_b200 import _build, _lib as lib
    if not os.path.isfile(lib.LIB_PATH):
        _build.build()
    return lib


def test_abi_rejects_bad_arguments_before_any_cuda_call():
    lib = _lib()
    L = lib.load()
    n = None

    def grad(dim, sl, st, nv, nh, neg, batch=4, mask=None, keep=1.0):
        return L.nrc_caser_grad(n, n, n, n, n, 10, dim, sl, st, nv, nh, neg, n, n, n, n, batch, mask, keep, n, n, n, n,
                                n, n, n, n)

    def epoch(dim, sl, st, nv, nh, neg, keep=0.5, batch_size=4):
        return L.nrc_caser_train_epoch(n, n, n, n, n, 3, 10, dim, sl, st, nv, nh, neg, n, n, n, n, 8, batch_size, keep,
                                       0.0, 1, 0, n, n, n, n, n, n, n, n, n, n, n, n)

    for call in (grad, epoch):
        for shape in ((0, 5, 3, 4, 16, 3), (257, 5, 3, 4, 16, 3), (50, 0, 3, 4, 16, 3), (50, 17, 3, 4, 16, 3),
                      (50, 5, 3, 0, 16, 3), (50, 5, 3, 65, 16, 3), (50, 5, 3, 4, 0, 3), (50, 5, 3, 4, 65, 3),
                      (50, 5, 32, 4, 16, 33)):
            with pytest.raises(lib.NrcError) as e:
                lib.check(call(*shape))
            assert e.value.rc == lib.NRC_E_LIMIT, shape
        for shape in ((50, 5, 0, 4, 16, 3), (50, 5, 3, 4, 16, 0)):
            with pytest.raises(ValueError, match="positive"):
                lib.check(call(*shape))
    with pytest.raises(ValueError, match="required"):                    # NULL tables, gradients and work
        lib.check(grad(50, 5, 3, 4, 16, 3))
    mask = np.ones(4, np.float32)
    for keep in (0.0, 1.5):
        with pytest.raises(ValueError, match="keep"):
            lib.check(grad(50, 5, 3, 4, 16, 3, mask=mask.ctypes.data, keep=keep))
        with pytest.raises(ValueError, match="keep"):
            lib.check(epoch(50, 5, 3, 4, 16, 3, keep=keep))
    with pytest.raises(ValueError, match="batch_size"):
        lib.check(epoch(50, 5, 3, 4, 16, 3, batch_size=0))
    with pytest.raises(lib.NrcError) as e:
        lib.check(grad(50, 5, 3, 4, 16, 3, batch=65535 * 32 + 1))
    assert e.value.rc == lib.NRC_E_LIMIT
    with pytest.raises(ValueError, match="required"):
        lib.check(epoch(50, 5, 3, 4, 16, 3))
    for shape in ((0, 5, 4, 16), (50, 17, 4, 16), (50, 5, 65, 16)):
        assert L.nrc_caser_dense_floats(*shape) == lib.NRC_E_LIMIT
        assert L.nrc_caser_work_floats(*shape, 256) == lib.NRC_E_LIMIT
        with pytest.raises(lib.NrcError) as e:
            lib.check(L.nrc_caser_query(n, n, n, 10, *shape, n, 2, n, n, n))
        assert e.value.rc == lib.NRC_E_LIMIT
    assert L.nrc_caser_work_floats(50, 5, 4, 16, 0) == lib.NRC_E_VALUE
    assert L.nrc_caser_dense_floats(50, 5, 4, 16) == cm.dense_layout(50, 5, 4, 16)[1] == 26154
    with pytest.raises(ValueError, match="required"):
        lib.check(L.nrc_caser_query(n, n, n, 10, 50, 5, 4, 16, n, 2, n, n, n))
    out = np.zeros(24, np.int32)
    with pytest.raises(ValueError):
        lib.check(L.nrc_caser_last_routes(None))
    lib.check(L.nrc_caser_last_routes(out.ctypes.data))
