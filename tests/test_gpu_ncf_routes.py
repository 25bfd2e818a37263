"""Every route the NCF kernels take from a shape, against oracle/tf_math evaluated in float64.

nrc_ncf_grad / nrc_ncf_train_epoch / nrc_ncf_scores (csrc/ncf.cu) and nrc_ncf_epoch_fused (csrc/ncf_epoch.cu) pick
their code from the shape.  Each test asserts the route it ran through nrc_ncf_last_routes, and the last test of
the file checks that the whole file saw every route.

Exact tests: small-integer tables, sparse integer weights and biases, square or hinge loss, GD with a power-of-two
learning rate, reg 0 or a power of two.  Every intermediate is then a dyadic rational, and its partial sums in any
order stay below 2^24 times its granularity (asserted from the float64 magnitudes), so fp32 is exact whatever the
summation order and every route must equal the float64 reference bit for bit.  Integer inputs also put many
pre-activations at exactly 0, which pins ReluGrad's convention: the gradient passes only where the output is > 0.

Rounded tests: the conf's init scales, BPR and cross-entropy.  Each entry must lie within C * 2^-24 * M of the
float64 value, where M is the same chain evaluated in float64 on absolute values under the reference's relu masks
(`chain64`) and C is stated in `c_forward` / `c_grad`."""
import numpy as np
import pytest
import torch

import oracle
from oracle import tf_math

pytestmark = pytest.mark.gpu
KEYS = ("mf_user", "mf_item", "mlp_user", "mlp_item", "dense")
U24 = 2.0 ** -24
LR_EXACT = 2.0 ** -6

# name: (mf_dim, layers, n_towers, pairwise).  Routes each one takes (asserted below through the hook):
SHAPES = {
    "default": (16, [64, 32, 16], 1, False),    # conf/NeuMF.properties: every fast route
    "two_tower": (16, [64, 32, 16], 2, True),   # pairwise NeuMF: 2 x 6768 tower floats copied per step (> 8192)
    "odd": (10, [20, 10], 1, False),            # scalar tables, quartet dW, generic forms, a 630-float tower
    "odd_pair": (10, [20, 10], 2, True),
    "mlp_pair": (0, [48, 24], 1, True),         # pairwise MLP: one tower shared by both passes
    "deep": (5, [128, 64, 32, 16], 1, False),   # four layers, a 128-wide one; scalar tables
    "wide": (0, [16, 160, 8], 1, False),        # a 160-wide layer: split and generic forms in one tower
    "gmf": (8, [], 1, False),                   # GMF only: no dense layers
    "one_layer": (4, [12], 2, True),            # one layer; mlp width 6 -> scalar tables
}
# epoch-kernel routes: (dW blocked, tables float4, split-forward mask, split-backward mask)
EPOCH_ROUTES = {
    "default": (1, 1, 0b111, 0b111), "two_tower": (1, 1, 0b111, 0b111), "odd": (0, 0, 0, 0),
    "odd_pair": (0, 0, 0, 0), "mlp_pair": (1, 1, 0, 0), "deep": (1, 0, 0b1111, 0b1111),
    "wide": (1, 1, 0b101, 0b011), "gmf": (0, 1, 0, 0), "one_layer": (1, 0, 0, 0),
}
SEEN = set()


def dev(a):
    return None if a is None else torch.from_numpy(np.ascontiguousarray(a)).cuda()


def host(d):
    return {k: (None if v is None else v.cpu().numpy()) for k, v in d.items()}


def record(n_layers):
    """The hook's report of the last NCF launch, added to SEEN."""
    from neurec_b200 import ops
    r = ops.ncf_last_routes()
    if r["sample_fast"] >= 0:
        SEEN.add(("sample", "fast" if r["sample_fast"] else "generic"))
        SEEN.add(("wgrad_slices", r["wgrad_slices"]))
    if r["epoch_tables_vec4"] >= 0:
        SEEN.add(("epoch_tables", "float4" if r["epoch_tables_vec4"] else "scalar"))
        SEEN.add(("epoch_layers", n_layers))
        if n_layers:
            SEEN.add(("epoch_dw", "blocked" if r["epoch_dw_blocked"] else "quartet"))
        for l in range(n_layers):
            SEEN.add(("fwd_layer", "split" if (r["fwd_split"] >> l) & 1 else "generic"))
            SEEN.add(("bwd_layer", "split" if (r["bwd_split"] >> l) & 1 else "generic"))
    if r["scores_tile"] >= 0:
        SEEN.add(("scores", "tile" if r["scores_tile"] else "generic"))
    return r


def check_epoch_routes(name, r):
    blocked, vec4, fwd, bwd = EPOCH_ROUTES[name]
    assert (r["epoch_dw_blocked"], r["epoch_tables_vec4"], r["fwd_split"], r["bwd_split"]) == (blocked, vec4, fwd, bwd), r
    assert r["sample_fast"] == -1 and r["scores_tile"] == -1, r
    mf_dim, layers, nt, _ = SHAPES[name]
    total = tf_math.ncf_dense_layout(layers[0] // 2 if layers else 0, layers, nt)[2]
    if total > 8192:                    # the weight copy's loop beyond its 8 unrolled float4 per thread
        SEEN.add(("epoch_copy", "beyond_8192"))
    if total % 4:                       # the copy's ragged last float4
        SEEN.add(("epoch_copy", "tail"))


def check_batch_routes(name, r, batch):
    _, layers, _, _ = SHAPES[name]
    assert r["sample_fast"] == (1 if layers == [64, 32, 16] else 0), r
    assert r["wgrad_slices"] == ((16 if batch >= 64 else 1) if layers else 0), r
    assert r["epoch_tables_vec4"] == -1 and r["scores_tile"] == -1, r


# ---------------------------------------------------------------------------------------------------------------
# float64 reference chain and its magnitudes
# ---------------------------------------------------------------------------------------------------------------
def loss_grad64(loss, x, labels):
    """dl/dx of learner.py's losses in float64 and the largest |d^2 l / dx^2| (Lip)."""
    if loss == "bpr":
        return -1.0 / (1.0 + np.exp(x)), 0.25
    if loss == "hinge":
        return (x + 1.0 > 0) * 1.0, 0.0
    if loss == "cross_entropy":
        return (1.0 / (1.0 + np.exp(-x)) - labels) / len(x), 0.25 / len(x)
    return (-2.0 * (1.0 - x), 2.0) if labels is None else (-2.0 * (labels - x), 2.0)


def chain64(P, c, users, items, third, ref=None, grads=True):
    """float64 forward and backward of one batch, as tf_math.ncf_grad computes it.  With `ref` (an earlier
    result of this function): the same chain on absolute values of every input, under ref's relu masks, with
    the loss gradient replaced by |g| + Lip * M_x.  That gives, for every quantity, a magnitude M that bounds
    its partial sums in any order and its first-order rounding error (in units of 2^-24 per operation)."""
    mf_dim, layers, nt, pairwise = c["mf_dim"], c["layers"], c["n_towers"], c["pairwise"]
    mlp_dim = layers[0] // 2 if layers else 0
    lay, tsz, _ = tf_math.ncf_dense_layout(mlp_dim, layers, nt)
    f = np.abs if ref is not None else (lambda a: a)
    Q = {k: (None if v is None else f(np.asarray(v, np.float64))) for k, v in P.items()}
    passes = [(items, 0)] + ([(third, 1 if nt == 2 else 0)] if pairwise else [])
    R = {"y": [], "z": [], "h": [], "m": []}
    for p, (it, tw) in enumerate(passes):
        y = np.zeros(len(users))
        if mf_dim:
            y = y + (Q["mf_user"][users] * Q["mf_item"][it]).sum(1)
        zs, hs, ms = [], [], []
        if layers:
            h = np.concatenate([Q["mlp_user"][users], Q["mlp_item"][it]], 1)
            for li, (wo, inn, out, bo) in enumerate(lay):
                W = Q["dense"][tw * tsz + wo:tw * tsz + wo + inn * out].reshape(inn, out)
                z = h @ W + Q["dense"][tw * tsz + bo:tw * tsz + bo + out]
                m = (ref["z"][p][li] if ref is not None else z) > 0
                hs.append(h); zs.append(z); ms.append(m)
                h = np.where(m, z, 0.0)
            hs.append(h)
            y = y + h.sum(1)
        R["y"].append(y); R["z"].append(zs); R["h"].append(hs); R["m"].append(ms)
    if not grads:
        return R
    labels = None if pairwise else np.asarray(third, np.float64)
    if ref is None:
        R["x"] = R["y"][0] - R["y"][1] if pairwise else R["y"][0]
        g, _ = loss_grad64(c["loss"], R["x"], labels)
    else:
        R["x"] = R["y"][0] + R["y"][1] if pairwise else R["y"][0]
        g = np.abs(ref["g"]) + loss_grad64(c["loss"], ref["x"], labels)[1] * R["x"]
    R["g"] = g
    G = {k: (None if v is None else np.zeros_like(v)) for k, v in Q.items()}
    for p, (it, tw) in enumerate(passes):
        gp = (g if (p == 0 or ref is not None) else -g)[:, None]
        if mf_dim:
            pu, qi = Q["mf_user"][users], Q["mf_item"][it]
            np.add.at(G["mf_user"], users, gp * qi + (c["reg_mf"] * pu if p == 0 else 0))
            np.add.at(G["mf_item"], it, gp * pu + c["reg_mf"] * qi)
        if layers:
            delta = gp * R["m"][p][-1]
            for li in range(len(lay) - 1, -1, -1):
                wo, inn, out, bo = lay[li]
                W = Q["dense"][tw * tsz + wo:tw * tsz + wo + inn * out].reshape(inn, out)
                G["dense"][tw * tsz + wo:tw * tsz + wo + inn * out] += (R["h"][p][li].T @ delta).reshape(-1)
                G["dense"][tw * tsz + bo:tw * tsz + bo + out] += delta.sum(0)
                delta = delta @ W.T
                if li > 0:
                    delta = delta * R["m"][p][li - 1]
            mu, mi = Q["mlp_user"][users], Q["mlp_item"][it]
            np.add.at(G["mlp_user"], users, delta[:, :mlp_dim] + (c["reg_mlp"] * mu if p == 0 else 0))
            np.add.at(G["mlp_item"], it, delta[:, mlp_dim:] + c["reg_mlp"] * mi)
    R["G"] = G
    return R


def c_forward(c, upto=None):
    """C of a forward value: every layer's dot product (in terms + bias) and, for the prediction, the GMF dot
    and the sum over the last layer's outputs.  gamma_n <= 1.01 n 2^-24 bounds n chained roundings of sums of
    products in any order (fma or not; the split forms only reorder), relu under a fixed mask is exact, and a
    relu that flips moves its output by at most its own error (relu is continuous).  Factor 2: second-order
    terms and headroom."""
    layers = c["layers"]
    ins = [2 * (layers[0] // 2)] + layers[:-1] if layers else []
    n = sum(i + 1 for i in ins[:upto])
    if upto is None:
        n += c["mf_dim"] + (layers[-1] if layers else 0) + 1
    return 2 * (n + 2)


def c_grad(c, batch):
    """C of a gradient entry: the forward chain to the prediction, the loss gradient (its error is at most
    Lip * err(x) + 4 ulp of g, which M covers through |g| + Lip * M_x), the backward dot products (out terms
    per layer), the sum over the batch's samples and passes (dW, or the rows a batch repeats) and the
    regulariser term.  Needs masks that do not flip: asserted by `assert_out_of_band`."""
    passes = 2 if c["pairwise"] else 1
    return c_forward(c) + 2 * (sum(c["layers"]) + passes * batch + 8)


def band_ok(R, A, c):
    """Per sample: no pre-activation of any pass within its forward error bound of 0 (a relu mask that could
    flip between fp32 and float64)."""
    ok = np.ones(len(R["y"][0]), bool)
    for p in range(len(R["z"])):
        for li, (z, mz) in enumerate(zip(R["z"][p], A["z"][p])):
            ok &= ((np.abs(z) > c_forward(c, li + 1) * U24 * mz) | (mz == 0)).all(1)
    return ok


def assert_within(got, want, M, C, what):
    err = np.abs(got.astype(np.float64) - want)
    bound = C * U24 * M
    assert (err <= bound).all(), (what, float((err - bound).max()), float(M.max()), C)


def assert_exact_regime(A, c, lr_bits=0, var=None):
    """Every partial sum of the exact tests' chain is a multiple of its granularity below 2^24 granules."""
    reg_bits = max([0] + [-int(np.log2(r)) for r in (c["reg_mf"], c["reg_mlp"]) if r])
    for y in A["y"]:
        assert (y < 2.0 ** 24).all()
    for p in range(len(A["z"])):
        for z in A["z"][p]:
            assert (z < 2.0 ** 24).all()
    assert (A["g"] < 2.0 ** 24).all()
    for k, g in A["G"].items():
        if g is None:
            continue
        assert (g * 2.0 ** reg_bits < 2.0 ** 24).all(), k
        if var is not None:
            assert ((np.abs(var[k]) + g * 2.0 ** -lr_bits) * 2.0 ** (reg_bits + lr_bits) < 2.0 ** 24).all(), k


def as_f32_exact(a):
    out = a.astype(np.float32)
    assert np.array_equal(out.astype(np.float64), a)
    return out


# ---------------------------------------------------------------------------------------------------------------
# inputs
# ---------------------------------------------------------------------------------------------------------------
def cfg(name, loss, reg_mf=0.0, reg_mlp=0.0):
    mf_dim, layers, nt, pairwise = SHAPES[name]
    return dict(mf_dim=mf_dim, layers=layers, n_towers=nt, pairwise=pairwise, loss=loss, reg_mf=reg_mf,
                reg_mlp=reg_mlp)


def int_params(c, nu, ni, rs):
    """Tables in [-2, 2]; weights in {-1, 0, 1} with about 3 non-zeros per output column, biases in {-1, 0, 1}."""
    mf_dim, layers, nt = c["mf_dim"], c["layers"], c["n_towers"]
    mlp_dim = layers[0] // 2 if layers else 0
    ri = lambda *s: rs.randint(-2, 3, s).astype(np.float32)
    P = {"mf_user": ri(nu, mf_dim) if mf_dim else None, "mf_item": ri(ni, mf_dim) if mf_dim else None,
         "mlp_user": ri(nu, mlp_dim) if layers else None, "mlp_item": ri(ni, mlp_dim) if layers else None,
         "dense": None}
    if layers:
        lay, tsz, total = tf_math.ncf_dense_layout(mlp_dim, layers, nt)
        d = np.zeros(total, np.float32)
        for t in range(nt):
            for (wo, inn, out, bo) in lay:
                d[t * tsz + wo:t * tsz + wo + inn * out] = rs.randint(-1, 2, inn * out) * (rs.rand(inn * out) < 3.0 / inn)
                d[t * tsz + bo:t * tsz + bo + out] = rs.randint(-1, 2, out)
        P["dense"] = d
    return P


def real_params(c, nu, ni, seed, scale):
    from test_gpu_ncf import make_params
    return make_params(nu, ni, c["mf_dim"], c["layers"], c["n_towers"], seed, scale)[0]


def decided_biases(P, c, nu, ni, rs):
    """Biases of +-3 sigma of each unit's pre-activation over all (user, item) pairs, layer by layer: deep
    towers at the init scale put many last-layer pre-activations within rounding of 0, which a batch of the
    epoch kernel cannot be chosen around.  The arithmetic the kernel does is the same."""
    mf_dim, layers, nt = c["mf_dim"], c["layers"], c["n_towers"]
    if not layers:
        return P
    P = dict(P, dense=P["dense"].copy())
    lay, tsz, _ = tf_math.ncf_dense_layout(layers[0] // 2, layers, nt)
    users, items = np.repeat(np.arange(nu), ni), np.tile(np.arange(ni), nu)
    for t in range(nt):
        h = np.concatenate([P["mlp_user"][users], P["mlp_item"][items]], 1).astype(np.float64)
        for (wo, inn, out, bo) in lay:
            s = h @ P["dense"][t * tsz + wo:t * tsz + wo + inn * out].reshape(inn, out)
            b = ((3.0 * s.std(0) + 0.2 * np.abs(s).max(0)) * rs.choice([-1.0, 1.0], out)).astype(np.float32)
            P["dense"][t * tsz + bo:t * tsz + bo + out] = b
            h = np.maximum(s + b, 0.0)
    return P


def synthetic_csr(nu, ni, seed, max_deg=16):
    rs = np.random.RandomState(seed)
    tp, ti = oracle.lists_to_csr([rs.choice(ni, rs.randint(1, max_deg), replace=False) for _ in range(nu)])
    return tp, ti, np.repeat(np.arange(nu, dtype=np.int32), np.diff(tp))


def epoch_arrays(tp, ti, pu, ni, pairwise, neg_num, shuffle, seed, epoch):
    wu, wi, wt = oracle.epoch_build(tp, ti, pu, ti, neg_num, ni, pairwise, shuffle, seed, epoch)
    return wu, wi, (wt[:, 0] if pairwise else wt)


def run_epoch(c, P, tp, ti, pu, nu, ni, opt, lr, bs, num_steps, shuffle=True, drop_last=False, seed=7, epoch=0,
              neg_num=1):
    """nrc_ncf_epoch_fused over steps [0, num_steps) -> (parameters, workspace arrays, step losses, routes)."""
    from neurec_b200 import ops
    pairwise = c["pairwise"]
    shape = ops.NcfShape.make(nu, ni, c["mf_dim"], c["layers"], c["n_towers"])
    dP = {k: dev(v) for k, v in P.items()}
    i0, i1 = tf_math.SLOT_INIT[opt]
    mk = lambda val: {k: (None if v is None or val is None else torch.full_like(v, val)) for k, v in dP.items()}
    G, S0, S1 = mk(0.0), mk(i0), mk(i1)
    tU = torch.zeros(nu, dtype=torch.int32, device="cuda"); tI = torch.zeros(ni, dtype=torch.int32, device="cuda")
    n = len(pu) * (1 if pairwise else neg_num + 1)
    n_used = (n // bs) * bs if drop_last else n
    step_loss = torch.full((max(1, (n_used + bs - 1) // bs),), 3.0, device="cuda")
    ws = tuple(torch.empty(n, dtype=torch.int32, device="cuda") for _ in range(3))
    pows = torch.tensor([0.9, 0.999], device="cuda") if opt == "adam" else None
    hyper = tf_math.DEFAULT_HYPER[opt](lr)
    ops.ncf_epoch_fused(shape, dP, dev(tp), dev(ti), dev(pu), dev(ti), neg_num, pairwise, shuffle, drop_last, seed,
                        epoch, bs, 0, num_steps, c["loss"], c["reg_mf"], c["reg_mlp"], opt, hyper, pows, G, S0, S1, tU,
                        tI, 1, ws[0], ws[1], ws[2], step_loss)
    r = record(len(c["layers"]))
    third = ws[2].cpu().numpy() if pairwise else ws[2].view(torch.float32).cpu().numpy()
    for k in KEYS[:4]:
        if G[k] is not None:
            assert float(G[k].abs().max()) == 0.0, k          # accumulators left clean
    return host(dP), (ws[0].cpu().numpy(), ws[1].cpu().numpy(), third), step_loss.cpu().numpy(), r


def run_grad(c, P, users, items, third, nu, ni):
    from neurec_b200 import ops
    shape = ops.NcfShape.make(nu, ni, c["mf_dim"], c["layers"], c["n_towers"])
    dP = {k: dev(v) for k, v in P.items()}
    dG = {k: (None if v is None else torch.zeros_like(v)) for k, v in dP.items()}
    tU = torch.zeros(nu, dtype=torch.int32, device="cuda"); tI = torch.zeros(ni, dtype=torch.int32, device="cuda")
    loss = torch.zeros(1, device="cuda")
    ops.ncf_grad(shape, dP, dev(users), dev(items), dev(third), c["pairwise"], c["loss"], c["reg_mf"], c["reg_mlp"],
                 dG, tU, tI, 3, loss)
    r = record(len(c["layers"]))
    return host(dG), float(loss.item()), r


def run_train_epoch_gd(c, P, users, items, third, nu, ni, lr, bs):
    from neurec_b200 import ops
    shape = ops.NcfShape.make(nu, ni, c["mf_dim"], c["layers"], c["n_towers"])
    dP = {k: dev(v) for k, v in P.items()}
    G = {k: (None if v is None else torch.zeros_like(v)) for k, v in dP.items()}
    none = {k: None for k in KEYS}
    tU = torch.zeros(nu, dtype=torch.int32, device="cuda"); tI = torch.zeros(ni, dtype=torch.int32, device="cuda")
    steps = (len(users) + bs - 1) // bs
    ops.ncf_train_epoch(shape, dP, dev(users), dev(items), dev(third), bs, c["pairwise"], c["loss"], c["reg_mf"],
                        c["reg_mlp"], "gd", np.full(steps, lr, np.float32), [lr], G, none, none, tU, tI, 1,
                        torch.zeros(steps, device="cuda"))
    r = record(len(c["layers"]))
    return host(dP), r


# ---------------------------------------------------------------------------------------------------------------
# a. exact: every route equals the float64 reference bit for bit
# ---------------------------------------------------------------------------------------------------------------
EXACT = [  # (shape, loss, batch, reg_mf, reg_mlp)
    ("default", "square", 64, 0.5, 0.25),
    ("two_tower", "square", 63, 0.0, 0.5),
    ("odd", "square", 1, 0.5, 0.0),             # a batch of one
    ("odd_pair", "hinge", 63, 0.0, 0.0),
    ("mlp_pair", "hinge", 64, 0.0, 0.25),
    ("deep", "square", 63, 0.0, 0.0),
    ("wide", "square", 64, 0.5, 0.5),
    ("gmf", "square", 63, 0.5, 0.0),
    ("one_layer", "square", 64, 0.25, 0.25),
]


@pytest.mark.parametrize("name,loss,bs,reg_mf,reg_mlp", EXACT)
def test_exact_one_step_on_every_path(name, loss, bs, reg_mf, reg_mlp):
    """One GD step (lr 2^-6) through nrc_ncf_epoch_fused; the gradients of nrc_ncf_grad and the one-step tables
    of nrc_ncf_train_epoch on the batch the epoch kernel drew: all equal to float64 tf_math.ncf_grad exactly,
    so the epoch kernel and the per-batch path are bit-identical after one step."""
    c = cfg(name, loss, reg_mf, reg_mlp)
    nu, ni = 40, 70
    rs = np.random.RandomState(100 + bs)
    P = int_params(c, nu, ni, rs)
    tp, ti, pu = synthetic_csr(nu, ni, 5)
    newP, (wu, wi, wt), _, r = run_epoch(c, P, tp, ti, pu, nu, ni, "gd", LR_EXACT, bs, 1)
    check_epoch_routes(name, r)
    ref_u, ref_i, ref_t = epoch_arrays(tp, ti, pu, ni, c["pairwise"], 1, True, 7, 0)
    assert np.array_equal(wu, ref_u) and np.array_equal(wi, ref_i) and np.array_equal(wt, ref_t)
    users, items, third = wu[:bs], wi[:bs], wt[:bs]

    P64 = {k: (None if v is None else v.astype(np.float64)) for k, v in P.items()}
    R = chain64(P64, c, users, items, third)
    A = chain64(P64, c, users, items, third, ref=R)
    assert_exact_regime(A, c, lr_bits=6, var=P64)
    _, Gt, _, _ = tf_math.ncf_grad(P64, users, items, third, c["pairwise"], loss, reg_mf, reg_mlp,
                                   c["layers"][0] // 2 if c["layers"] else 0, c["layers"], c["n_towers"])
    zero_pre = 0
    for k in KEYS:
        if P[k] is not None:
            assert np.array_equal(R["G"][k], Gt[k]), k                # this file's chain is tf_math's
    for p in range(len(R["z"])):
        zero_pre += sum(int((z == 0).sum()) for z in R["z"][p])
    if c["layers"]:
        assert zero_pre > 0                                            # ReluGrad at an output of exactly 0 is tested
    want = {k: (None if P[k] is None else as_f32_exact(P64[k] - LR_EXACT * Gt[k])) for k in KEYS}

    for k in KEYS:                                                     # the epoch kernel, one step
        if P[k] is not None:
            assert np.array_equal(newP[k], want[k]), k
    G, _, rb = run_grad(c, P, users, items, third, nu, ni)             # the per-batch gradients
    check_batch_routes(name, rb, bs)
    for k in KEYS:
        if P[k] is not None:
            assert np.array_equal(G[k], as_f32_exact(Gt[k])), k
    stepP, rt = run_train_epoch_gd(c, P, users, items, third, nu, ni, LR_EXACT, bs)
    check_batch_routes(name, rt, bs)
    for k in KEYS:                                                     # the per-batch path, one step
        if P[k] is not None:
            assert np.array_equal(stepP[k], want[k]), k
            assert np.array_equal(stepP[k], newP[k]), k


SCORES = [  # (shape name or explicit (mf_dim, layers), n_users, n_items, tile kernel?)
    ((0, [64, 32, 16]), 1, 1, True),
    ((1, [64, 32, 16]), 2, 127, True),
    ((5, [64, 32, 16]), 3, 128, True),
    ((64, [64, 32, 16]), 5, 129, True),
    ((16, [64, 32, 16]), 943, 1682, True),
    ((65, [64, 32, 16]), 5, 129, False),        # GMF wider than the tile kernel keeps per user
    ((10, [20, 10]), 3, 128, False),
    ((5, [128, 64, 32, 16]), 2, 127, False),
    ((0, [48, 24]), 5, 1682, False),
    ((0, [16, 160, 8]), 1, 129, False),
    ((8, []), 3, 1, False),
    ((4, [12]), 2, 129, False),
]


def scores_users(n_users, nu, rs):
    if n_users <= 5:        # unsorted, with a repeat from 2 users on
        return np.array([7, 7, 3, 41, 0][:n_users] if n_users != 2 else [9, 9], np.int32) % nu
    return rs.randint(0, nu, n_users).astype(np.int32)


@pytest.mark.parametrize("exact", [True, False], ids=["exact", "rounded"])
@pytest.mark.parametrize("shape,n_users,n_items,tile", SCORES)
def test_scores_match_float64(shape, n_users, n_items, tile, exact):
    """nrc_ncf_scores on the tile kernel and the warp-per-pair kernel: bit-exact on integer parameters, within
    c_forward * 2^-24 * M on the conf's init scale (0.3 here)."""
    from neurec_b200 import ops
    mf_dim, layers = shape
    c = dict(mf_dim=mf_dim, layers=layers, n_towers=1, pairwise=False)
    nu = 943 if n_users == 943 else 50
    rs = np.random.RandomState(n_items + mf_dim)
    P = int_params(c, nu, n_items, rs) if exact else real_params(c, nu, n_items, n_items + mf_dim, 0.3)
    users = scores_users(n_users, nu, rs)
    got = ops.ncf_scores(ops.NcfShape.make(nu, n_items, mf_dim, layers, 1), {k: dev(v) for k, v in P.items()},
                         dev(users)).cpu().numpy()
    r = record(len(layers))
    assert r["scores_tile"] == (1 if tile else 0) and r["sample_fast"] == -1 and r["epoch_tables_vec4"] == -1, r
    P64 = {k: (None if v is None else v.astype(np.float64)) for k, v in P.items()}
    C = c_forward(c)
    mlp_dim = layers[0] // 2 if layers else 0
    for u in np.unique(users):
        uu, it = np.full(n_items, u), np.arange(n_items)
        R = chain64(P64, c, uu, it, None, grads=False)
        M = chain64(P64, c, uu, it, None, ref=R, grads=False)["y"][0]
        want = tf_math.ncf_predict(P64, uu, it, mlp_dim, layers)
        assert np.allclose(R["y"][0], want, rtol=1e-12, atol=1e-12 * M.max())
        for row in np.nonzero(users == u)[0]:
            if exact:
                assert (M < 2.0 ** 24).all()
                assert np.array_equal(got[row], as_f32_exact(want)), (u, row)
            else:
                assert_within(got[row], want, M, C, ("scores", u))
    if not exact:
        assert np.abs(got).max() > 1e-2


# ---------------------------------------------------------------------------------------------------------------
# b. rounded: realistic scales against float64 with a per-entry bound
# ---------------------------------------------------------------------------------------------------------------
ROUNDED = [  # (shape, scale, reg_mf, reg_mlp)
    ("default", 0.01, 1e-3, 1e-3),
    ("two_tower", 0.1, 0.0, 0.01),
    ("odd", 0.3, 0.01, 0.0),
    ("odd_pair", 0.1, 0.0, 0.0),
    ("mlp_pair", 0.3, 0.0, 1e-3),
    ("deep", 0.1, 0.0, 0.0),
    ("wide", 0.3, 0.0, 0.0),
    ("gmf", 0.1, 0.01, 0.0),
    ("one_layer", 0.3, 1e-3, 1e-3),
]


def loss_of(name):
    return "bpr" if SHAPES[name][3] else "cross_entropy"


@pytest.mark.parametrize("name,scale,reg_mf,reg_mlp", ROUNDED)
def test_rounded_gradients_within_bound(name, scale, reg_mf, reg_mlp):
    """nrc_ncf_grad on a batch of 203 at the conf's init scales, BPR or cross-entropy, against float64."""
    c = cfg(name, loss_of(name), reg_mf, reg_mlp)
    nu, ni, bs = 60, 90, 203
    P = real_params(c, nu, ni, 3, scale)
    P64 = {k: (None if v is None else v.astype(np.float64)) for k, v in P.items()}
    rs = np.random.RandomState(4)
    pool = 8 * bs                                   # keep the first 203 samples whose relu masks cannot flip
    users, items = rs.randint(0, nu, pool).astype(np.int32), rs.randint(0, ni, pool).astype(np.int32)
    third = rs.randint(0, ni, pool).astype(np.int32) if c["pairwise"] else (rs.rand(pool) < 0.3).astype(np.float32)
    R = chain64(P64, c, users, items, third, grads=False)
    keep = np.nonzero(band_ok(R, chain64(P64, c, users, items, third, ref=R, grads=False), c))[0][:bs]
    assert len(keep) == bs
    users, items, third = users[keep], items[keep], third[keep]
    R = chain64(P64, c, users, items, third)
    A = chain64(P64, c, users, items, third, ref=R)
    assert band_ok(R, A, c).all()
    G, loss, r = run_grad(c, P, users, items, third, nu, ni)
    check_batch_routes(name, r, bs)
    l64, Gt, _, _ = tf_math.ncf_grad(P64, users, items, third, c["pairwise"], c["loss"], reg_mf, reg_mlp,
                                     c["layers"][0] // 2 if c["layers"] else 0, c["layers"], c["n_towers"])
    C = c_grad(c, bs)
    for k in KEYS:
        if P[k] is not None:
            assert np.allclose(R["G"][k], Gt[k], rtol=1e-12, atol=1e-12 * A["G"][k].max())
            assert_within(G[k], Gt[k], A["G"][k], C, k)
            assert np.abs(Gt[k]).max() > 0, k
    assert np.isclose(loss, l64, rtol=1e-5)


# "deep" is left out: at the init scale its four-layer tower leaves some last-layer pre-activation within
# rounding of 0 in every batch of every epoch tried; its epoch route is covered bit for bit by the exact test.
@pytest.mark.parametrize("name,scale,reg_mf,reg_mlp", [r for r in ROUNDED if r[0] != "deep"])
def test_rounded_gd_step_of_the_epoch_kernel_within_bound(name, scale, reg_mf, reg_mlp):
    """One GD step with lr = 1 through nrc_ncf_epoch_fused (the update carries the gradient at full weight),
    against the float64 step on the batch the kernel drew.  The epoch index is the first whose first batch
    keeps every relu mask out of its flip band (found with the sampler's CPU restatement, then asserted)."""
    c = cfg(name, loss_of(name), reg_mf, reg_mlp)
    nu, ni, bs = 50, 80, 64
    P = decided_biases(real_params(c, nu, ni, 6, scale), c, nu, ni, np.random.RandomState(8))
    P64 = {k: (None if v is None else v.astype(np.float64)) for k, v in P.items()}
    tp, ti, pu = synthetic_csr(nu, ni, 9)
    for epoch in range(64):
        wu, wi, wt = epoch_arrays(tp, ti, pu, ni, c["pairwise"], 1, True, 7, epoch)
        R = chain64(P64, c, wu[:bs], wi[:bs], wt[:bs])
        A = chain64(P64, c, wu[:bs], wi[:bs], wt[:bs], ref=R)
        if band_ok(R, A, c).all():
            break
    else:
        pytest.fail("no epoch of 64 keeps its first batch out of the relu flip band")
    newP, (gu, gi, gt), step_loss, r = run_epoch(c, P, tp, ti, pu, nu, ni, "gd", 1.0, bs, 1, epoch=epoch)
    check_epoch_routes(name, r)
    assert np.array_equal(gu[:bs], wu[:bs]) and np.array_equal(gi[:bs], wi[:bs]) and np.array_equal(gt[:bs], wt[:bs])
    C = c_grad(c, bs)
    for k in KEYS:
        if P[k] is not None:
            assert_within(newP[k], P64[k] - R["G"][k], A["G"][k] + np.abs(P64[k]), C, k)
    assert (step_loss[1:] == 0).all()


# ---------------------------------------------------------------------------------------------------------------
# whole epochs on the oracle trainer: partial last batch, drop_last, shuffle off, every loss and optimizer
# ---------------------------------------------------------------------------------------------------------------
EPOCHS = [  # (shape, loss, opt, lr, shuffle, drop_last, neg_num)
    ("default", "cross_entropy", "adam", 1e-3, True, False, 4),
    ("odd_pair", "hinge", "adagrad", 1e-2, True, True, 1),
    ("deep", "square", "momentum", 1e-3, False, False, 1),
    ("mlp_pair", "square", "rmsprop", 1e-3, True, False, 1),
    ("wide", "cross_entropy", "gd", 5e-2, True, False, 2),
    ("gmf", "square", "momentum", 1e-3, False, True, 1),
    ("one_layer", "bpr", "adagrad", 1e-2, True, False, 1),
    ("odd", "square", "rmsprop", 1e-3, True, False, 1),
]


@pytest.mark.parametrize("name,loss,opt,lr,shuffle,drop_last,neg_num", EPOCHS)
def test_whole_epoch_matches_the_oracle_trainer(name, loss, opt, lr, shuffle, drop_last, neg_num):
    """Every step of one epoch of a 300-user synthetic CSR in one nrc_ncf_epoch_fused call against
    tf_math.NCFTrainer on the epoch arrays of oracle.epoch_build (fp32 against fp32 in another order: 3e-5 absolute
    on every parameter, 2e-4 relative on each step's loss)."""
    c = cfg(name, loss, 1e-4, 1e-4)
    nu, ni, bs = 300, 500, 128
    P = real_params(c, nu, ni, 12, 0.05)
    tp, ti, pu = synthetic_csr(nu, ni, 13)
    wu, wi, wt = epoch_arrays(tp, ti, pu, ni, c["pairwise"], neg_num, shuffle, 21, 3)
    n = len(wu)
    assert n % bs != 0                                  # a partial last batch, kept or dropped
    n_used = (n // bs) * bs if drop_last else n
    steps = (n_used + bs - 1) // bs
    if not drop_last:
        SEEN.add(("epoch_batch", "partial"))
    mlp_dim = c["layers"][0] // 2 if c["layers"] else 0
    tr = tf_math.NCFTrainer(P, mlp_dim, c["layers"], c["n_towers"], opt, lr, loss, 1e-4, 1e-4, c["pairwise"])
    want = tr.epoch(wu[:n_used], wi[:n_used], wt[:n_used], bs)
    newP, (gu, gi, gt), got, r = run_epoch(c, P, tp, ti, pu, nu, ni, opt, lr, bs, steps, shuffle=shuffle,
                                           drop_last=drop_last, seed=21, epoch=3, neg_num=neg_num)
    check_epoch_routes(name, r)
    # the kernel builds the samples the epoch uses (drop_last: not the dropped tail)
    assert np.array_equal(gu[:n_used], wu[:n_used]) and np.array_equal(gi[:n_used], wi[:n_used])
    assert np.array_equal(gt[:n_used], wt[:n_used])
    assert len(got) == steps and len(want) == steps
    assert np.allclose(got, want, rtol=2e-4, atol=1e-6), np.abs(got - want).max()
    for k in KEYS:
        if P[k] is not None:
            assert np.abs(newP[k] - tr.P[k]).max() < 3e-5, k
            assert np.abs(tr.P[k] - P[k]).max() > 3e-4, k           # every table moved well past the tolerance


# ---------------------------------------------------------------------------------------------------------------
# d. a shape over the epoch kernel's shared-memory limit
# ---------------------------------------------------------------------------------------------------------------
def test_over_the_shared_memory_limit_returns_limit_and_launches_nothing():
    """Pairwise NeuMF with layers [128, 64, 32, 16]: two towers of 27 376 floats plus two sample groups of
    2 * 2 * 368 + 136 floats and 64 reduction slots are 232 128 B, over the epoch kernel's 200 KB.  The call
    returns NRC_E_LIMIT before any launch: parameters, accumulators, workspace, step losses and the route
    report stay as they were.  (The NeuMF plug-in passes the NrcError on from its first epoch.)"""
    from neurec_b200 import _lib, ops
    c = dict(mf_dim=8, layers=[128, 64, 32, 16], n_towers=2, pairwise=True, loss="bpr", reg_mf=0.0, reg_mlp=0.0)
    nu, ni = 30, 40
    P = real_params(c, nu, ni, 1, 0.1)
    tp, ti, pu = synthetic_csr(nu, ni, 2)
    n = len(pu)
    ops.ncf_scores(ops.NcfShape.make(nu, ni, 10, [20, 10], 1), {k: dev(v) for k, v in real_params(
        cfg("odd", "bpr"), nu, ni, 1, 0.1).items()}, dev(np.arange(3, dtype=np.int32)))
    before = ops.ncf_last_routes()
    shape = ops.NcfShape.make(nu, ni, 8, c["layers"], 2)
    dP = {k: dev(v) for k, v in P.items()}
    G = {k: torch.zeros_like(v) for k, v in dP.items()}
    none = {k: None for k in KEYS}
    tU = torch.zeros(nu, dtype=torch.int32, device="cuda"); tI = torch.zeros(ni, dtype=torch.int32, device="cuda")
    ws = tuple(torch.full((n,), -7, dtype=torch.int32, device="cuda") for _ in range(3))
    step_loss = torch.full((4,), 3.0, device="cuda")
    with pytest.raises(_lib.NrcError, match="shared memory") as e:
        ops.ncf_epoch_fused(shape, dP, dev(tp), dev(ti), dev(pu), dev(ti), 1, True, True, False, 7, 0, 64, 0, 1, "bpr",
                            0.0, 0.0, "gd", [0.1], None, G, none, none, tU, tI, 1, ws[0], ws[1], ws[2], step_loss)
    assert "error %d" % _lib.NRC_E_LIMIT in str(e.value)
    torch.cuda.synchronize()
    assert ops.ncf_last_routes() == before
    for k in KEYS:
        assert np.array_equal(dP[k].cpu().numpy(), P[k]), k
        assert float(G[k].abs().max()) == 0.0, k
    assert all(bool((w == -7).all()) for w in ws)
    assert bool((step_loss == 3.0).all()) and int(tU.abs().max()) == 0 and int(tI.abs().max()) == 0


# ---------------------------------------------------------------------------------------------------------------
# c. route completeness (runs last)
# ---------------------------------------------------------------------------------------------------------------
REQUIRED = {
    ("sample", "fast"), ("sample", "generic"), ("wgrad_slices", 16), ("wgrad_slices", 1), ("wgrad_slices", 0),
    ("epoch_dw", "blocked"), ("epoch_dw", "quartet"), ("epoch_tables", "float4"), ("epoch_tables", "scalar"),
    ("fwd_layer", "split"), ("fwd_layer", "generic"), ("bwd_layer", "split"), ("bwd_layer", "generic"),
    ("epoch_layers", 0), ("epoch_layers", 1), ("epoch_layers", 2), ("epoch_layers", 3), ("epoch_layers", 4),
    ("scores", "tile"), ("scores", "generic"),
    # not reported by the hook; recorded from the shapes and epochs the tests ran
    ("epoch_copy", "beyond_8192"), ("epoch_copy", "tail"), ("epoch_batch", "partial"),
}


def test_every_route_was_seen(request):
    """Across this file the hook reported every route of the NCF kernels.  Only meaningful when the whole file
    ran: a run of selected tests skips it."""
    here = {it.nodeid for it in request.session.items if it.fspath == request.node.fspath}
    every = {it.nodeid for it in request.node.parent.collect()}
    if here != every:
        pytest.skip("only part of this file was selected")
    assert REQUIRED <= SEEN, sorted(REQUIRED - SEEN)
