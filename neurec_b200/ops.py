"""Tensor-facing wrappers of the C ABI (torch.Tensor is only the device buffer).

Every function launches hand-written sm_90a kernels from ``libneurec_b200.so`` on the
current torch CUDA stream.  Nothing here computes on the CPU.
"""
from __future__ import annotations

import ctypes

import numpy as np
import torch

from . import _lib
from ._lib import LOSS_IDS, METRIC_IDS, OPT_IDS, check

launch_count = 0  # kernels launched through this module (bench.py reports it)


def _p(t):
    if t is None:
        return None
    return ctypes.c_void_p(t.data_ptr())


def _stream():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def _req(t, dtype, name):
    if not (isinstance(t, torch.Tensor) and t.is_cuda and t.dtype == dtype and t.is_contiguous()):
        raise TypeError("'%s' must be a contiguous CUDA tensor of dtype %s" % (name, dtype))
    return t


def _metric_arr(metric):
    ids = [METRIC_IDS[m] if isinstance(m, str) else int(m) for m in metric]
    return np.asarray(ids, dtype=np.int32)


def _count(n=1):
    global launch_count
    launch_count += n


# ------------------------------------------------------------------------------- evaluator
def eval_score_matrix(scores, test_indptr, test_indices, metric, top_k, return_ranks=False):
    """Device drop-in of CPPEvaluator.eval_score_matrix (cpp_evaluator.pyx:28-42)."""
    _req(scores, torch.float32, "scores")
    _req(test_indptr, torch.int64, "test_indptr")
    _req(test_indices, torch.int32, "test_indices")
    B, N = scores.shape
    m = _metric_arr(metric)
    res = torch.empty((B, len(m) * top_k), dtype=torch.float32, device=scores.device)
    ranks = torch.empty((B, top_k), dtype=torch.int32, device=scores.device) if return_ranks else None
    check(_lib.load().nrc_eval_score_matrix(_p(scores), N, B, _p(test_indptr), _p(test_indices),
                                            m.ctypes.data, len(m), top_k, _p(res), _p(ranks),
                                            _stream()))
    _count()
    return (res, ranks) if return_ranks else res


def eval_score_matrix_host(scores, test_indptr, test_indices, metric, top_k, return_ranks=False):
    """Host-buffer drop-in (numpy in, numpy out); H2D/D2H happen inside the call."""
    scores = np.ascontiguousarray(scores, dtype=np.float32)
    test_indptr = np.ascontiguousarray(test_indptr, dtype=np.int64)
    test_indices = np.ascontiguousarray(test_indices, dtype=np.int32)
    B, N = scores.shape
    m = _metric_arr(metric)
    res = np.empty((B, len(m) * top_k), dtype=np.float32)
    ranks = np.empty((B, top_k), dtype=np.int32) if return_ranks else None
    check(_lib.load().nrc_eval_score_matrix_host(
        scores.ctypes.data, N, B, test_indptr.ctypes.data, test_indices.ctypes.data,
        m.ctypes.data, len(m), top_k, res.ctypes.data,
        ranks.ctypes.data if ranks is not None else None))
    _count()
    return (res, ranks) if return_ranks else res


def arg_topk(scores, top_k):
    """Device drop-in of util.cython.arg_topk.arg_topk (arg_topk.pyx:16-35)."""
    _req(scores, torch.float32, "scores")
    U, N = scores.shape
    out = torch.empty((U, top_k), dtype=torch.int32, device=scores.device)
    check(_lib.load().nrc_arg_topk(_p(scores), N, U, top_k, _p(out), _stream()))
    _count()
    return out


def arg_topk_host(scores, top_k):
    scores = np.ascontiguousarray(scores, dtype=np.float32)
    U, N = scores.shape
    out = np.empty((U, top_k), dtype=np.int32)
    check(_lib.load().nrc_arg_topk_host(scores.ctypes.data, N, U, top_k, out.ctypes.data))
    _count()
    return out


def eval_mf(user_table, item_table, users, train_indptr, train_indices, test_indptr,
            test_indices, metric, top_k, return_ranks=False, want_results=True):
    """Fused predict -> mask -> top-K -> metrics (uni_evaluator.py:132-146, MF.py:120-122)."""
    _req(user_table, torch.float32, "user_table")
    _req(item_table, torch.float32, "item_table")
    _req(users, torch.int32, "users")
    _req(train_indptr, torch.int64, "train_indptr")
    _req(train_indices, torch.int32, "train_indices")
    _req(test_indptr, torch.int64, "test_indptr")
    _req(test_indices, torch.int32, "test_indices")
    N, D = item_table.shape
    B = users.numel()
    m = _metric_arr(metric)
    dev = users.device
    res = torch.empty((B, len(m) * top_k), dtype=torch.float32, device=dev) if want_results else None
    ranks = torch.empty((B, top_k), dtype=torch.int32, device=dev) if return_ranks else None
    check(_lib.load().nrc_eval_mf(_p(user_table), _p(item_table), D, N, _p(users), B,
                                  _p(train_indptr), _p(train_indices), _p(test_indptr),
                                  _p(test_indices), m.ctypes.data, len(m), top_k, _p(res),
                                  _p(ranks), _stream()))
    _count()
    return (res, ranks) if return_ranks else res


def eval_mf_tc(user_table, item_table, users, train_indptr, train_indices, test_indptr, test_indices,
               metric, top_k, return_ranks=False, cand_cap=0):
    """eval_mf with the score step on the tensor cores (wgmma candidate pass + exact re-score);
    bit-identical results, meant for catalogues of millions of items."""
    N, D = item_table.shape
    B = users.numel()
    m = _metric_arr(metric)
    res = torch.empty((B, len(m) * top_k), dtype=torch.float32, device=users.device)
    ranks = torch.empty((B, top_k), dtype=torch.int32, device=users.device) if return_ranks else None
    check(_lib.load().nrc_eval_mf_tc(_p(user_table), _p(item_table), D, N, _p(users), B, _p(train_indptr),
                                     _p(train_indices), _p(test_indptr), _p(test_indices), m.ctypes.data,
                                     len(m), top_k, int(cand_cap), _p(res), _p(ranks), _stream()))
    _count(5)
    return (res, ranks) if return_ranks else res


def mf_score_pairs(user_rows, item_table, items, train_indptr, train_indices):
    """Exact fp32 scores of `items` [B, C] (ids into item_table, -1 = none) for the gathered user rows
    [B, dim]; masked (train CSR indexed by ROW) or missing candidates score -inf (nrc_mf_score_pairs)."""
    _req(user_rows, torch.float32, "user_rows"); _req(item_table, torch.float32, "item_table")
    _req(items, torch.int32, "items")
    B, C = items.shape
    out = torch.empty((B, C), dtype=torch.float32, device=items.device)
    check(_lib.load().nrc_mf_score_pairs(_p(user_rows), _p(item_table), item_table.shape[1], _p(items), B, C,
                                         _p(train_indptr), _p(train_indices), _p(out), _stream()))
    _count()
    return out


def eval_merge_candidates(cand_ids, cand_scores, test_indptr, test_indices, metric, top_k, return_ranks=False):
    """Per row the top_k of C (score, global id) candidates + metrics (nrc_eval_merge_candidates).
    Returns (results, [ranks,] tie_count tensor)."""
    _req(cand_ids, torch.int32, "cand_ids"); _req(cand_scores, torch.float32, "cand_scores")
    B, C = cand_ids.shape
    m = _metric_arr(metric)
    res = torch.empty((B, len(m) * top_k), dtype=torch.float32, device=cand_ids.device)
    ranks = torch.empty((B, top_k), dtype=torch.int32, device=cand_ids.device) if return_ranks else None
    ties = torch.zeros(1, dtype=torch.int32, device=cand_ids.device)
    check(_lib.load().nrc_eval_merge_candidates(_p(cand_ids), _p(cand_scores), C, B, _p(test_indptr), _p(test_indices),
                                                m.ctypes.data, len(m), int(top_k), _p(res), _p(ranks), _p(ties),
                                                _stream()))
    _count()
    return (res, ranks, ties) if return_ranks else (res, ties)


TC_MIN_ITEMS = 16384     # catalogue size from which eval_mf_auto takes the tensor-core pass (crossover not re-measured on H100)


def use_tensor_core_eval(n_items, dim, top_k, n_users):
    """Routing rule of eval_mf_auto: the tensor-core candidate pass needs dim 64 or 128 with top_k <= 31 (one
    lane per kept score) or dim 192 with top_k <= 16 (shared-memory budget of the tie-replay pass)
    and pays off from TC_MIN_ITEMS items / ~1 k users up."""
    fits = (dim in (64, 128) and 1 <= top_k <= 31) or (dim == 192 and 1 <= top_k <= 16)
    return n_items >= TC_MIN_ITEMS and fits and n_users >= 1024


def eval_mf_auto(user_table, item_table, users, train_indptr, train_indices, test_indptr, test_indices,
                 metric, top_k, return_ranks=False):
    """eval_mf, with the score step on the tensor cores when the catalogue is large enough for the
    candidate pass to pay off, and materialised score rows when (dim, top_k) lie outside the fused
    kernel's shared-memory envelope (results are bit-identical on every route)."""
    n_items, dim = item_table.shape
    if use_tensor_core_eval(n_items, dim, top_k, users.numel()):
        return eval_mf_tc(user_table, item_table, users, train_indptr, train_indices, test_indptr, test_indices,
                          metric, top_k, return_ranks)
    try:
        return eval_mf(user_table, item_table, users, train_indptr, train_indices, test_indptr, test_indices,
                       metric, top_k, return_ranks)
    except _lib.NrcError as e:
        if e.rc != _lib.NRC_E_LIMIT:
            raise
    return eval_mf_materialised(user_table, item_table, users, train_indptr, train_indices, test_indptr,
                                test_indices, metric, top_k, return_ranks)


EVAL_CHUNK_BYTES = 256 << 20   # score rows eval_mf_materialised holds at a time


def eval_mf_materialised(user_table, item_table, users, train_indptr, train_indices, test_indptr, test_indices,
                         metric, top_k, return_ranks=False):
    """eval_mf in user chunks through materialised scores: nrc_mf_scores (the fused kernel's FMA chain)
    -> nrc_mask_rows -> nrc_eval_score_matrix, so the results are the fused kernel's bit for bit.  It
    takes every dim and top_k <= 512, at the cost of writing [chunk, num_items] scores to memory."""
    n_items = item_table.shape[0]
    B = users.numel()
    chunk = max(1, EVAL_CHUNK_BYTES // (4 * n_items))
    res, ranks = [], []
    for a in range(0, B, chunk):
        u = users[a:a + chunk]
        s = mask_rows(mf_scores(user_table, item_table, u), u, train_indptr, train_indices)
        # the batch rows' test sets as a CSR indexed by row, as nrc_eval_score_matrix reads it
        beg = test_indptr[u.long()]
        cnt = test_indptr[u.long() + 1] - beg
        tp = torch.zeros(u.numel() + 1, dtype=torch.int64, device=u.device)
        torch.cumsum(cnt, 0, out=tp[1:])
        src = torch.repeat_interleave(beg - tp[:-1], cnt) + torch.arange(int(tp[-1]), device=u.device)
        ti = test_indices[src].contiguous()
        out = eval_score_matrix(s, tp, ti, metric, top_k, return_ranks)
        res.append(out[0] if return_ranks else out)
        if return_ranks:
            ranks.append(out[1])
    if B == 0:
        m = _metric_arr(metric)
        res = [torch.empty((0, len(m) * top_k), dtype=torch.float32, device=users.device)]
        ranks = [torch.empty((0, top_k), dtype=torch.int32, device=users.device)]
    res = torch.cat(res)
    return (res, torch.cat(ranks)) if return_ranks else res


def eval_tc_items_version(version):
    """Non-zero: eval_mf_tc reuses its bf16 item-table copy while (table pointer, shape, version) are
    unchanged (one fixed model evaluated in several user batches); 0: convert on every call."""
    check(_lib.load().nrc_eval_tc_items_version(int(version)))


def eval_tc_epilogue_warps(warps):
    """8 or 16 epilogue warps in the tensor-core candidate kernel (same results; tuning knob)."""
    check(_lib.load().nrc_eval_tc_epilogue_warps(int(warps)))


def eval_tc_last_launch():
    """(kernel_ms, flops) of the last candidate-kernel launch made by eval_mf_tc."""
    import ctypes
    ms, fl = ctypes.c_float(0.0), ctypes.c_double(0.0)
    check(_lib.load().nrc_eval_tc_last_launch(ctypes.byref(ms), ctypes.byref(fl)))
    return ms.value, fl.value


def eval_tc_force_segments(g):
    """Test hook: 0 = heuristic number of item segments in the tensor-core passes, g >= 1 = min(g, tiles)."""
    check(_lib.load().nrc_eval_tc_force_segments(int(g)))


def eval_tc_debug_candidates(pass_, user_table, item_table, users, train_indptr, train_indices, lq, cap, max_slots):
    """Test hook: one tensor-core candidate pass as eval_mf_tc runs it.  Returns (cand [n, nslots, cap] int32,
    cand_val [n, nslots, cap] float32 approximate scores, cnt [n, nslots] int32 (> cap: overflow), margin [n]
    float32, seg_items); entries of a list past min(cnt, cap) are undefined."""
    _req(user_table, torch.float32, "user_table")
    _req(item_table, torch.float32, "item_table")
    _req(users, torch.int32, "users")
    N, D = item_table.shape
    n = users.numel()
    dev = users.device
    cand = torch.empty((n * max_slots * cap,), dtype=torch.int32, device=dev)
    val = torch.empty((n * max_slots * cap,), dtype=torch.float32, device=dev)
    cnt = torch.empty((n * max_slots,), dtype=torch.int32, device=dev)
    margin = torch.empty((n,), dtype=torch.float32, device=dev)
    ns, seg = ctypes.c_int32(0), ctypes.c_int32(0)
    check(_lib.load().nrc_eval_tc_debug_candidates(
        int(pass_), _p(user_table), _p(item_table), D, N, _p(users), n, _p(train_indptr), _p(train_indices),
        int(lq), int(cap), int(max_slots), _p(cand), _p(val), _p(cnt), _p(margin), ctypes.byref(ns),
        ctypes.byref(seg), _stream()))
    _count(3)
    s = ns.value
    return (cand[:n * s * cap].view(n, s, cap), val[:n * s * cap].view(n, s, cap), cnt[:n * s].view(n, s),
            margin, seg.value)


def eval_tc_last_fallbacks():
    """(users of the last eval_mf_tc call re-ranked by the candidate-list heap replay, users re-ranked by the
    full-catalogue heap replay after a candidate list overflowed)."""
    r, f = ctypes.c_int32(0), ctypes.c_int32(0)
    check(_lib.load().nrc_eval_tc_last_fallbacks(ctypes.byref(r), ctypes.byref(f)))
    return r.value, f.value


def tc_gemm_debug(a, b, swizzle=1, n_tile=128):
    """Test hook: out f32 [128, 256] = a bf16 [128, k] . b bf16 [256, k]^T through wgmma m64n{n_tile}k16."""
    _req(a, torch.bfloat16, "a")
    _req(b, torch.bfloat16, "b")
    assert a.shape[0] == 128 and b.shape[0] == 256 and a.shape[1] == b.shape[1]
    out = torch.empty((128, 256), dtype=torch.float32, device=a.device)
    check(_lib.load().nrc_tc_gemm_debug_ntile(_p(a), _p(b), a.shape[1], int(swizzle), int(n_tile), _p(out),
                                              _stream()))
    _count()
    return out


def eval_last_undecided():
    """Users of the last eval_mf / eval_mf_tc call that needed a heap replay (ties, overflow)."""
    import ctypes
    n = ctypes.c_int32(0)
    check(_lib.load().nrc_eval_last_undecided(ctypes.byref(n)))
    return n.value


EVAL_ROUTES = ("mf_form", "rows_fast", "rows_warps")


def eval_last_routes():
    """Kernel forms of the most recent evaluator launches (nrc_eval_last_routes) as {name: value}; -1 = none yet.
    mf_form: 0 heap replay for every user, 1 fast pass with 2 users per warp, 2 fast pass on 128-item tiles,
    3 fast pass on 64-item tiles (last eval_mf); rows_fast, rows_warps: the last score-matrix / arg-top-k launch."""
    out = (ctypes.c_int32 * len(EVAL_ROUTES))()
    check(_lib.load().nrc_eval_last_routes(out))
    return dict(zip(EVAL_ROUTES, out))


def mf_scores(user_table, item_table, users):
    """MF.predict(users, None) on device: [len(users), num_items] fp32 (MF.py:120-122)."""
    _req(user_table, torch.float32, "user_table"); _req(item_table, torch.float32, "item_table")
    _req(users, torch.int32, "users")
    N, D = item_table.shape
    out = torch.empty((users.numel(), N), dtype=torch.float32, device=users.device)
    check(_lib.load().nrc_mf_scores(_p(user_table), _p(item_table), D, N, _p(users), users.numel(),
                                    _p(out), _stream()))
    _count()
    return out


def mask_rows(scores, users, train_indptr, train_indices):
    """In place scores[b, train(users[b])] = -inf (uni_evaluator.py:140-143)."""
    _req(scores, torch.float32, "scores")
    _req(users, torch.int32, "users")
    B, N = scores.shape
    check(_lib.load().nrc_mask_rows(_p(scores), N, B, _p(users), _p(train_indptr), _p(train_indices),
                                    _stream()))
    _count()
    return scores


def mean_rows(results):
    """np.mean(results, axis=0) with numpy's fp32 summation order (uni_evaluator.py:150)."""
    _req(results, torch.float32, "results")
    rows, cols = results.shape
    out = torch.empty((cols,), dtype=torch.float32, device=results.device)
    check(_lib.load().nrc_mean_rows(_p(results), rows, cols, _p(out), _stream()))
    _count()
    return out


# --------------------------------------------------------------------------------- sampler
def sample_negatives(train_indptr, train_indices, users, neg_num, num_items, seed, stream_id,
                     first_index=0):
    """_sampling_negative_items (sampler.py:71-90): [n, neg_num] negatives, on device."""
    _req(train_indptr, torch.int64, "train_indptr")
    _req(train_indices, torch.int32, "train_indices")
    _req(users, torch.int32, "users")
    n = users.numel()
    out = torch.empty((n, max(int(neg_num), 0)), dtype=torch.int32, device=users.device)
    check(_lib.load().nrc_sample_negatives(_p(train_indptr), _p(train_indices), _p(users), n,
                                           int(neg_num), int(num_items), int(seed),
                                           int(stream_id), int(first_index), _p(out), _stream()))
    _count()
    return out


def batch_randint_choice(high, out_indptr, total_out, replace=True, excl_indptr=None,
                         excl_indices=None, seed=0, stream_id=0):
    """batch_randint_choice (random_choice.pyx:64-89) on device CSR inputs; flat output."""
    _req(out_indptr, torch.int64, "out_indptr")
    n_rows = out_indptr.numel() - 1
    out = torch.empty((int(total_out),), dtype=torch.int32, device=out_indptr.device)
    check(_lib.load().nrc_batch_randint_choice(int(high), _p(out_indptr), n_rows, int(total_out),
                                               1 if replace else 0, _p(excl_indptr),
                                               _p(excl_indices), int(seed), int(stream_id),
                                               _p(out), _stream()))
    _count()
    return out


# ----------------------------------------------------------------------------- device epoch
def shuffle_perm(n, seed, epoch, shuffle=True, device="cuda"):
    """RandomSampler's per-epoch order (data_iterator.py:45-63) as a keyed bijection: int64 [n]."""
    out = torch.empty((int(n),), dtype=torch.int64, device=device)
    check(_lib.load().nrc_shuffle_perm(int(n), 1 if shuffle else 0, int(seed), int(epoch), _p(out), _stream()))
    _count()
    return out


def epoch_build(train_indptr, train_indices, pos_users, pos_items, neg_num, num_items, pairwise, shuffle,
                seed, epoch, first=0, n_out=None):
    """One epoch of Pairwise/PointwiseSampler as device arrays (nrc_epoch_build): users i32 [n],
    items i32 [n], third = i32 [n, neg_num] negatives (pairwise) or f32 [n] labels (pointwise)."""
    _req(train_indptr, torch.int64, "train_indptr"); _req(train_indices, torch.int32, "train_indices")
    _req(pos_users, torch.int32, "pos_users"); _req(pos_items, torch.int32, "pos_items")
    if int(neg_num) <= 0:
        raise ValueError("'neg_num' must be a positive integer.")
    n_pos = pos_users.numel()
    n_samples = n_pos if pairwise else n_pos * (int(neg_num) + 1)
    n_out = n_samples - first if n_out is None else int(n_out)
    dev = pos_users.device
    users = torch.empty((n_out,), dtype=torch.int32, device=dev)
    items = torch.empty((n_out,), dtype=torch.int32, device=dev)
    third = torch.empty((n_out, int(neg_num)), dtype=torch.int32, device=dev) if pairwise else \
        torch.empty((n_out,), dtype=torch.float32, device=dev)
    check(_lib.load().nrc_epoch_build(_p(train_indptr), _p(train_indices), _p(pos_users), _p(pos_items), n_pos,
                                      int(neg_num), int(num_items), 1 if pairwise else 0, 1 if shuffle else 0,
                                      int(seed), int(epoch), int(first), n_out, _p(users), _p(items), _p(third),
                                      _stream()))
    _count()
    return users, items, third


def mf_epoch_fused(U, V, train_indptr, train_indices, pos_users, pos_items, neg_num, pairwise, shuffle, drop_last,
                   seed, epoch, batch_size, first_step, num_steps, loss, reg, opt, hyper, adam_pows, gU, gV, tU, tV,
                   s0U, s1U, s0V, s1V, first_stamp, ws_users, ws_items, ws_third, step_loss):
    """Steps [first_step, first_step + num_steps) of one MF epoch -- shuffle, negative sampling and
    every step -- in one persistent cooperative launch (nrc_mf_epoch_fused)."""
    h = np.zeros(4, dtype=np.float32)
    h[:len(hyper)] = hyper
    check(_lib.load().nrc_mf_epoch_fused(
        _p(U), _p(V), U.shape[0], V.shape[0], U.shape[1], _p(train_indptr), _p(train_indices), _p(pos_users),
        _p(pos_items), pos_users.numel(), int(neg_num), 1 if pairwise else 0, 1 if shuffle else 0,
        1 if drop_last else 0, int(seed), int(epoch), int(batch_size), int(first_step), int(num_steps),
        LOSS_IDS[loss], float(reg), OPT_IDS[opt], h.ctypes.data, _p(adam_pows), _p(gU), _p(gV), _p(tU), _p(tV),
        _p(s0U), _p(s1U), _p(s0V), _p(s1V), int(first_stamp), _p(ws_users), _p(ws_items), _p(ws_third),
        _p(step_loss), _stream()))
    _count()


# -------------------------------------------------------------------------------- training
def mf_pairwise_grad(U, V, users, pos, neg, loss, reg, gU, gV, tU, tV, stamp, loss_out):
    check(_lib.load().nrc_mf_pairwise_grad(_p(U), _p(V), U.shape[1], _p(users), _p(pos), _p(neg),
                                           users.numel(), LOSS_IDS[loss], float(reg), _p(gU),
                                           _p(gV), _p(tU), _p(tV), int(stamp), _p(loss_out),
                                           _stream()))
    _count()


def mf_pointwise_grad(U, V, users, items, labels, loss, reg, gU, gV, tU, tV, stamp, loss_out):
    check(_lib.load().nrc_mf_pointwise_grad(_p(U), _p(V), U.shape[1], _p(users), _p(items),
                                            _p(labels), users.numel(), LOSS_IDS[loss], float(reg),
                                            _p(gU), _p(gV), _p(tU), _p(tV), int(stamp),
                                            _p(loss_out), _stream()))
    _count()


def mf_bpr_sgd_fused(U, V, users, pos, neg, lr, reg, loss_out):
    """Single-pass BPR + SGD for huge tables (see nrc_mf_bpr_sgd_fused)."""
    check(_lib.load().nrc_mf_bpr_sgd_fused(_p(U), _p(V), U.shape[1], _p(users), _p(pos), _p(neg),
                                           users.numel(), float(lr), float(reg), _p(loss_out), _stream()))
    _count()


def mf_bpr_sgd_sharded(user_shards, item_shards, self_rank, users, pos, neg, lr, reg, loss_out):
    """The single-pass BPR + SGD step on row-sharded tables (nrc_mf_bpr_sgd_sharded): `user_shards`
    / `item_shards` are neurec_b200.util.peer.ShardSet objects (this rank's own block and peer
    mappings of the others); ids are global."""
    w = user_shards.world
    assert w == item_shards.world and w >= 1
    check(_lib.load().nrc_mf_bpr_sgd_sharded(user_shards.ptr_array(), item_shards.ptr_array(), w, int(self_rank),
                                             user_shards.shape[0], item_shards.shape[0], user_shards.shape[1],
                                             _p(users), _p(pos), _p(neg), users.numel(), float(lr), float(reg),
                                             _p(loss_out), _stream()))
    _count()


def mf_bpr_sgd_epoch(user_table, item_shards, train_indptr, train_indices, pos_users, pos_items, num_items, shuffle,
                     seed, epoch, first, count, lr, reg, loss_out):
    """Triplets [first, first + count) of a shuffled BPR + SGD epoch straight from the train CSR
    (nrc_mf_bpr_sgd_epoch): sampling, shuffling, scoring and the in-place update in ONE kernel.
    `user_table` is this rank's row block (pos_users are local ids), `item_shards` a ShardSet; with a
    replicated head (ShardSet.enable_hot) call item_shards.sync_hot() after every step."""
    _req(user_table, torch.float32, "user_table")
    _req(train_indptr, torch.int64, "train_indptr"); _req(train_indices, torch.int32, "train_indices")
    _req(pos_users, torch.int32, "pos_users"); _req(pos_items, torch.int32, "pos_items")
    n_hot = getattr(item_shards, "n_hot", 0)
    check(_lib.load().nrc_mf_bpr_sgd_epoch_hot(_p(user_table), item_shards.ptr_array(), item_shards.world,
                                               item_shards.rank, item_shards.shape[0], user_table.shape[1],
                                               _p(train_indptr), _p(train_indices), _p(pos_users), _p(pos_items),
                                               pos_users.numel(), int(num_items), 1 if shuffle else 0, int(seed),
                                               int(epoch), int(first), int(count), float(lr), float(reg), _p(loss_out),
                                               _p(item_shards.hot) if n_hot else None,
                                               _p(item_shards.hot_delta) if n_hot else None, int(n_hot), _stream()))
    _count()


def mf_bpr_lazy_adam_epoch(U, mU, vU, V, mV, vV, train_indptr, train_indices, pos_users, pos_items, num_items, shuffle,
                           seed, epoch, first, count, lr_t, reg, loss_out, beta1=0.9, beta2=0.999, eps=1e-8):
    """The explicitly-named lazy-Adam variant of mf_bpr_sgd_epoch (nrc_mf_bpr_lazy_adam_epoch)."""
    check(_lib.load().nrc_mf_bpr_lazy_adam_epoch(_p(U), _p(mU), _p(vU), _p(V), _p(mV), _p(vV), U.shape[1],
                                                 _p(train_indptr), _p(train_indices), _p(pos_users), _p(pos_items),
                                                 pos_users.numel(), int(num_items), 1 if shuffle else 0, int(seed),
                                                 int(epoch), int(first), int(count), float(lr_t), float(beta1),
                                                 float(beta2), float(eps), float(reg), _p(loss_out), _stream()))
    _count()


MF_KERNELS = ("grad", "sgd_ids", "sgd_csr", "lazy_adam", "epoch", "opt_apply")
MF_ROUTE_FIELDS = ("vec", "sharded", "user_once", "tier_rows", "grid", "capped", "opt_vec4")


def mf_last_routes():
    """Routes of the most recent launch of each MF training kernel group (nrc_mf_last_routes) as
    {kernel: {field: value}}; -1 = no such launch yet or a field the group does not decide."""
    nf = len(MF_ROUTE_FIELDS)
    out = (ctypes.c_int32 * (len(MF_KERNELS) * nf))()
    check(_lib.load().nrc_mf_last_routes(out))
    return {k: dict(zip(MF_ROUTE_FIELDS, out[i * nf:(i + 1) * nf])) for i, k in enumerate(MF_KERNELS)}


def opt_apply_rows(opt, var, grad, slot0, slot1, touched, stamp, hyper):
    h = np.zeros(4, dtype=np.float32)
    h[:len(hyper)] = hyper
    rows, dim = var.shape
    check(_lib.load().nrc_opt_apply_rows(OPT_IDS[opt], _p(var), _p(grad), _p(slot0), _p(slot1),
                                         _p(touched), int(stamp), rows, dim, h.ctypes.data,
                                         _stream()))
    _count()


def opt_apply_multi(opt, variables, stamp, hyper):
    """variables: list of (var, grad, slot0|None, slot1|None, touched|None, dense_var:bool);
    every variable of the model is updated by ONE kernel launch."""
    n = len(variables)
    PA = ctypes.c_void_p * n
    ptr = lambda t: t.data_ptr() if t is not None else None
    var = PA(*[ptr(v[0]) for v in variables])
    grad = PA(*[ptr(v[1]) for v in variables])
    s0 = PA(*[ptr(v[2]) for v in variables])
    s1 = PA(*[ptr(v[3]) for v in variables])
    tch = PA(*[ptr(v[4]) for v in variables])
    shp = [(v[0].shape[0], v[0].numel() // v[0].shape[0]) if v[0].dim() > 1 else (1, v[0].numel())
           for v in variables]
    rows = (ctypes.c_int64 * n)(*[s[0] for s in shp])
    dims = (ctypes.c_int32 * n)(*[s[1] for s in shp])
    dense = (ctypes.c_int32 * n)(*[1 if v[5] else 0 for v in variables])
    h = np.zeros(4, dtype=np.float32)
    h[:len(hyper)] = hyper
    cast = lambda a: ctypes.cast(a, ctypes.c_void_p)
    check(_lib.load().nrc_opt_apply_multi(OPT_IDS[opt], n, cast(var), cast(grad), cast(s0), cast(s1),
                                          cast(tch), cast(rows), cast(dims), cast(dense), int(stamp),
                                          h.ctypes.data, _stream()))
    _count()


def spmm_set_exact(on):
    """True: sequential, separately rounded accumulation (bit-identical to scipy / TF's CPU kernel);
    False (default): the fast order (nrc_spmm_set_exact)."""
    check(_lib.load().nrc_spmm_set_exact(1 if on else 0))


def spmm_csr(indptr, indices, values, x, row_order=None, bias=None, y=None, sum_=None, div=0.0,
             want_y=True):
    """y = A.x in CSR order (LightGCN.py:140); optional fused epilogue, see nrc_spmm_csr."""
    _req(indptr, torch.int64, "indptr"); _req(indices, torch.int32, "indices")
    _req(values, torch.float32, "values"); _req(x, torch.float32, "x")
    n_rows = indptr.numel() - 1
    dim = x.shape[1]
    if y is None and want_y:
        y = torch.empty((n_rows, dim), dtype=torch.float32, device=x.device)
    check(_lib.load().nrc_spmm_csr(_p(indptr), _p(indices), _p(values), _p(row_order), n_rows, _p(x),
                                   dim, _p(bias), _p(y), _p(sum_), float(div), _stream()))
    _count()
    return y


GRAPH_ROUTES = ("spmm_fast", "spmm_width", "spmm_capped", "ngcf_fwd_rows", "ngcf_bwd_tiles", "ngcf_bpr_triplets",
                "spectral_fwd_split", "spectral_bwd_split", "spectral_dw_split")


def graph_last_routes():
    """Routes of the most recent SpMM / NGCF / SpectralCF launches (nrc_graph_last_routes) as {name: value}; -1 = no
    such launch yet or not decided by the last call of that group."""
    out = (ctypes.c_int32 * len(GRAPH_ROUTES))()
    check(_lib.load().nrc_graph_last_routes(out))
    return dict(zip(GRAPH_ROUTES, out))


def lightgcn_propagate(indptr, indices, values, row_order, e0, n_layers, e_final=None, work=None):
    """mean(E_0, A E_0, ..., A^L E_0) (LightGCN.py:132-149)."""
    n, dim = e0.shape
    if e_final is None:
        e_final = torch.empty_like(e0)
    if work is None:
        work = (torch.empty_like(e0), torch.empty_like(e0))
    check(_lib.load().nrc_lightgcn_propagate(_p(indptr), _p(indices), _p(values), _p(row_order), n, dim,
                                             int(n_layers), _p(e0), _p(e_final), _p(work[0]),
                                             _p(work[1]), _stream()))
    _count(n_layers)
    return e_final


def lightgcn_bpr_grad(e_final, e0, num_users, users, pos, neg, reg, scale, grad_final, grad_reg, loss2):
    check(_lib.load().nrc_lightgcn_bpr_grad(_p(e_final), _p(e0), int(num_users), e0.shape[1], _p(users),
                                            _p(pos), _p(neg), users.numel(), float(reg), float(scale),
                                            _p(grad_final), _p(grad_reg), _p(loss2), _stream()))
    _count()


def lightgcn_train_epoch(csr, t_csr, row_order, num_users, num_items, n_layers, e0, m, v, users, pos,
                         neg, batch_size, reg, lr_t, hyper, e_final, grad_final, grad_e0, work,
                         step_loss2):
    n = users.numel()
    steps = (n + batch_size - 1) // batch_size
    lr_t = np.ascontiguousarray(lr_t, dtype=np.float32)
    h = np.zeros(4, dtype=np.float32)
    h[:len(hyper)] = hyper
    t = t_csr if t_csr is not None else (None, None, None)
    check(_lib.load().nrc_lightgcn_train_epoch(
        _p(csr[0]), _p(csr[1]), _p(csr[2]), _p(t[0]), _p(t[1]), _p(t[2]), _p(row_order), int(num_users),
        int(num_items), e0.shape[1], int(n_layers), _p(e0), _p(m), _p(v), _p(users), _p(pos), _p(neg), n,
        int(batch_size), float(reg), lr_t.ctypes.data, h.ctypes.data, _p(e_final), _p(grad_final),
        _p(grad_e0), _p(work[0]), _p(work[1]), _p(step_loss2), _stream()))
    _count(steps * (2 * n_layers + 3))
    return steps


class NcfShape(ctypes.Structure):
    """ctypes mirror of nrc_ncf_shape (include/neurec_b200.h)."""
    _fields_ = [("num_users", ctypes.c_int32), ("num_items", ctypes.c_int32),
                ("mf_dim", ctypes.c_int32), ("mlp_dim", ctypes.c_int32),
                ("n_layers", ctypes.c_int32), ("layers", ctypes.c_int32 * 4),
                ("n_towers", ctypes.c_int32)]

    @classmethod
    def make(cls, num_users, num_items, mf_dim, layers, n_towers=1):
        layers = list(layers or [])
        if len(layers) > 4:
            raise ValueError("at most 4 dense layers are supported")
        s = cls()
        s.num_users, s.num_items, s.mf_dim = int(num_users), int(num_items), int(mf_dim)
        s.mlp_dim = int(layers[0] / 2) if layers else 0   # NeuMF.py:58 int(self.layers[0]/2)
        s.n_layers = len(layers)
        for i, v in enumerate(layers):
            s.layers[i] = int(v)
        s.n_towers = int(n_towers)
        return s

    def dense_size(self):
        n = _lib.load().nrc_ncf_dense_size(ctypes.byref(self))
        check(n if n < 0 else 0)
        return n


NCF_ROUTES = ("sample_fast", "wgrad_slices", "epoch_dw_blocked", "epoch_tables_vec4", "fwd_split", "bwd_split",
              "scores_tile")


def ncf_last_routes():
    """Code paths of the most recent NCF launch (nrc_ncf_last_routes) as {name: value}; -1 = not decided by it.
    fwd_split / bwd_split are bitmasks over the epoch kernel's layers."""
    out = (ctypes.c_int32 * len(NCF_ROUTES))()
    check(_lib.load().nrc_ncf_last_routes(out))
    return dict(zip(NCF_ROUTES, out))


def ncf_grad(shape, P, users, items, third, pairwise, loss, reg_mf, reg_mlp, G, tU, tI, stamp,
             loss_out):
    """P / G: dicts with keys mf_user, mf_item, mlp_user, mlp_item, dense (tensors or None)."""
    k = ("mf_user", "mf_item", "mlp_user", "mlp_item", "dense")
    check(_lib.load().nrc_ncf_grad(ctypes.byref(shape), *[_p(P[n]) for n in k], _p(users), _p(items),
                                   _p(third), users.numel(), 1 if pairwise else 0, LOSS_IDS[loss],
                                   float(reg_mf), float(reg_mlp), *[_p(G[n]) for n in k], _p(tU),
                                   _p(tI), int(stamp), _p(loss_out), _stream()))
    _count()


def ncf_scores(shape, P, users):
    """NeuMF.predict(users, None): [len(users), num_items] scores on device (NeuMF.py:163-168)."""
    k = ("mf_user", "mf_item", "mlp_user", "mlp_item", "dense")
    out = torch.empty((users.numel(), shape.num_items), dtype=torch.float32, device=users.device)
    check(_lib.load().nrc_ncf_scores(ctypes.byref(shape), *[_p(P[n]) for n in k], _p(users),
                                     users.numel(), shape.num_items, _p(out), _stream()))
    _count()
    return out


def ncf_train_epoch(shape, P, users, items, third, batch_size, pairwise, loss, reg_mf, reg_mlp, opt,
                    lr_t, hyper, G, S0, S1, tU, tI, first_stamp, step_loss):
    k = ("mf_user", "mf_item", "mlp_user", "mlp_item", "dense")
    n = users.numel()
    steps = (n + batch_size - 1) // batch_size
    lr_t = np.ascontiguousarray(lr_t, dtype=np.float32)
    h = np.zeros(4, dtype=np.float32)
    h[:len(hyper)] = hyper
    PA = ctypes.c_void_p * 5
    arr = lambda D: ctypes.cast(PA(*[(D[x].data_ptr() if D.get(x) is not None else None) for x in k]),
                                ctypes.c_void_p)
    check(_lib.load().nrc_ncf_train_epoch(
        ctypes.byref(shape), *[_p(P[x]) for x in k], _p(users), _p(items), _p(third), n, int(batch_size),
        1 if pairwise else 0, LOSS_IDS[loss], float(reg_mf), float(reg_mlp), OPT_IDS[opt],
        lr_t.ctypes.data, h.ctypes.data, arr(G), arr(S0), arr(S1), _p(tU), _p(tI), int(first_stamp),
        _p(step_loss), _stream()))
    _count(3 * steps)
    return steps


def ncf_epoch_fused(shape, P, train_indptr, train_indices, pos_users, pos_items, neg_num, pairwise, shuffle,
                    drop_last, seed, epoch, batch_size, first_step, num_steps, loss, reg_mf, reg_mlp, opt, hyper,
                    adam_pows, G, S0, S1, tU, tI, first_stamp, ws_users, ws_items, ws_third, step_loss):
    """Steps [first_step, first_step + num_steps) of one NeuMF / MLP epoch -- shuffle, negative
    sampling and every step -- in one persistent cooperative launch (nrc_ncf_epoch_fused)."""
    k = ("mf_user", "mf_item", "mlp_user", "mlp_item", "dense")
    h = np.zeros(4, dtype=np.float32)
    h[:len(hyper)] = hyper
    PA = ctypes.c_void_p * 5
    arr = lambda D: ctypes.cast(PA(*[(D[x].data_ptr() if D.get(x) is not None else None) for x in k]),
                                ctypes.c_void_p)
    check(_lib.load().nrc_ncf_epoch_fused(
        ctypes.byref(shape), *[_p(P[x]) for x in k], _p(train_indptr), _p(train_indices), _p(pos_users),
        _p(pos_items), pos_users.numel(), int(neg_num), 1 if pairwise else 0, 1 if shuffle else 0,
        1 if drop_last else 0, int(seed), int(epoch), int(batch_size), int(first_step), int(num_steps),
        LOSS_IDS[loss], float(reg_mf), float(reg_mlp), OPT_IDS[opt], h.ctypes.data, _p(adam_pows), arr(G), arr(S0),
        arr(S1), _p(tU), _p(tI), int(first_stamp), _p(ws_users), _p(ws_items), _p(ws_third), _p(step_loss), _stream()))
    _count()


def mf_train_epoch(U, V, users, items, third, batch_size, pairwise, loss, reg, opt, lr_t, hyper,
                   gU, gV, tU, tV, s0U, s1U, s0V, s1V, first_stamp, step_loss):
    n = users.numel()
    steps = (n + batch_size - 1) // batch_size
    lr_t = np.ascontiguousarray(lr_t, dtype=np.float32)
    assert lr_t.size >= max(steps, 1)
    h = np.zeros(4, dtype=np.float32)
    h[:len(hyper)] = hyper
    check(_lib.load().nrc_mf_train_epoch(
        _p(U), _p(V), U.shape[0], V.shape[0], U.shape[1], _p(users), _p(items), _p(third), n,
        int(batch_size), 1 if pairwise else 0, LOSS_IDS[loss], float(reg), OPT_IDS[opt],
        lr_t.ctypes.data, h.ctypes.data, _p(gU), _p(gV), _p(tU), _p(tV), _p(s0U), _p(s1U),
        _p(s0V), _p(s1V), int(first_stamp), _p(step_loss), _stream()))
    _count(2 * steps)
    return steps


# ------------------------------------------------------------------------------------ NGCF
class NgcfShape(ctypes.Structure):
    """ctypes mirror of nrc_ngcf_shape (include/neurec_b200.h)."""
    _fields_ = [("num_users", ctypes.c_int32), ("num_items", ctypes.c_int32), ("emb_dim", ctypes.c_int32),
                ("n_layers", ctypes.c_int32), ("layers", ctypes.c_int32 * 4)]

    @classmethod
    def make(cls, num_users, num_items, emb_dim, layers):
        layers = list(layers)
        if not 1 <= len(layers) <= 4:
            raise ValueError("NGCF supports 1 to 4 propagation layers")
        s = cls()
        s.num_users, s.num_items, s.emb_dim, s.n_layers = int(num_users), int(num_items), int(emb_dim), len(layers)
        for i, v in enumerate(layers):
            s.layers[i] = int(v)
        return s

    @property
    def n_nodes(self):
        return self.num_users + self.num_items

    @property
    def d_total(self):
        return self.emb_dim + sum(self.layers[i] for i in range(self.n_layers))

    def weights_size(self):
        n = _lib.load().nrc_ngcf_weights_size(ctypes.byref(self))
        check(n if n < 0 else 0)
        return n

    def work_floats(self):
        n = _lib.load().nrc_ngcf_work_floats(ctypes.byref(self))
        check(int(n) if n < 0 else 0)
        return int(n)

    def mask_floats(self):
        return self.n_nodes * sum(self.layers[i] for i in range(self.n_layers))


def dropout_mask(n, keep, seed, stream_id, out=None, device="cuda"):
    """tf.nn.dropout's keep mask (1.0 with probability keep) from the counter-based generator."""
    if out is None:
        out = torch.empty((int(n),), dtype=torch.float32, device=device)
    check(_lib.load().nrc_dropout_mask(int(n), float(keep), int(seed), int(stream_id), _p(out), _stream()))
    _count()
    return out


def ngcf_forward(shape, csr, row_order, e0, weights, masks, keep, all_emb=None, work=None):
    """_create_ngcf_embed (NGCF.py:160-202): the concatenated embeddings [N, d_total]."""
    if all_emb is None:
        all_emb = torch.empty((shape.n_nodes, shape.d_total), dtype=torch.float32, device=e0.device)
    if work is None:
        work = torch.empty(shape.work_floats(), dtype=torch.float32, device=e0.device)
    check(_lib.load().nrc_ngcf_forward(ctypes.byref(shape), _p(csr[0]), _p(csr[1]), _p(csr[2]), _p(row_order), _p(e0),
                                       _p(weights), _p(masks), float(keep), _p(all_emb), _p(work), _stream()))
    _count(2 * shape.n_layers + 1)
    return all_emb


def ngcf_grad(shape, csr, row_order, t_csr, t_row_order, e0, weights, masks, keep, users, pos, neg, reg, all_emb,
              grad_all, grad_e0, grad_weights, work, loss2):
    """Loss + gradients of one NGCF batch (nrc_ngcf_grad)."""
    t = t_csr if t_csr is not None else (None, None, None)
    check(_lib.load().nrc_ngcf_grad(ctypes.byref(shape), _p(csr[0]), _p(csr[1]), _p(csr[2]), _p(row_order), _p(t[0]),
                                    _p(t[1]), _p(t[2]), _p(t_row_order), _p(e0), _p(weights), _p(masks), float(keep),
                                    _p(users), _p(pos), _p(neg), users.numel(), float(reg), _p(all_emb), _p(grad_all),
                                    _p(grad_e0), _p(grad_weights), _p(work), _p(loss2), _stream()))
    _count(4 * shape.n_layers + 4)


# ------------------------------------------------- SURVEY 8(f) ranks 3-4: APR, SBPR, time order, CSR build
def l2_normalize_rows(x, scale, out=None):
    """tf.nn.l2_normalize(x, 1) * scale (APR.py:103-104,117-118) on a f32 [rows, dim] table."""
    _req(x, torch.float32, "x")
    out = torch.empty_like(x) if out is None else _req(out, torch.float32, "out")
    check(_lib.load().nrc_l2_normalize_rows(_p(x), x.shape[0], x.shape[1], float(scale), _p(out), _stream()))
    _count()
    return out


def gather_rows_i32(src, index, out=None):
    """out[p] = src[index[p] % len(src)] for an int32 [rows, width] (or [rows]) table and an int64 index."""
    _req(src, torch.int32, "src"); _req(index, torch.int64, "index")
    width = 1 if src.dim() == 1 else int(src.shape[1])
    shape = (index.numel(),) if src.dim() == 1 else (index.numel(), width)
    out = torch.empty(shape, dtype=torch.int32, device=src.device) if out is None else out
    check(_lib.load().nrc_gather_rows_i32(_p(src), src.shape[0], width, _p(index), index.numel(), _p(out), _stream()))
    _count()
    return out


def sbpr_epoch_build(train_indptr, train_indices, social_indptr, social_indices, trust_indptr, trust_indices,
                     pos_users, pos_items, num_items, max_excluded, shuffle, seed, epoch, first=0, count=None):
    """One epoch of SBPR._get_pairwise_all_data + DataIterator (SBPR.py:103-149) as device arrays:
    users, pos, social, neg i32 [count] and s_uk f32 [count]."""
    for t, n in ((train_indptr, "train_indptr"), (social_indptr, "social_indptr"), (trust_indptr, "trust_indptr")):
        _req(t, torch.int64, n)
    for t, n in ((train_indices, "train_indices"), (social_indices, "social_indices"), (trust_indices, "trust_indices"),
                 (pos_users, "pos_users"), (pos_items, "pos_items")):
        _req(t, torch.int32, n)
    n_pos = pos_users.numel()
    count = n_pos - first if count is None else int(count)
    dev = pos_users.device
    mk = lambda dt: torch.empty((count,), dtype=dt, device=dev)
    ou, oi, ok, oj, os_ = mk(torch.int32), mk(torch.int32), mk(torch.int32), mk(torch.int32), mk(torch.float32)
    check(_lib.load().nrc_sbpr_epoch_build(_p(train_indptr), _p(train_indices), _p(social_indptr), _p(social_indices),
                                           _p(trust_indptr), _p(trust_indices), _p(pos_users), _p(pos_items), n_pos,
                                           int(num_items), int(max_excluded), 1 if shuffle else 0, int(seed), int(epoch),
                                           int(first), count, _p(ou), _p(oi), _p(ok), _p(oj), _p(os_), _stream()))
    _count()
    return ou, oi, ok, oj, os_


def sbpr_grad(U, V, B, users, pos, social, neg, suk, loss, reg, gU, gV, gB, tU, tV, stamp, loss_out):
    check(_lib.load().nrc_sbpr_grad(_p(U), _p(V), _p(B), U.shape[1], _p(users), _p(pos), _p(social), _p(neg), _p(suk),
                                    users.numel(), LOSS_IDS[loss], float(reg), _p(gU), _p(gV), _p(gB), _p(tU), _p(tV),
                                    int(stamp), _p(loss_out), _stream()))
    _count()


def sbpr_train_epoch(U, V, B, users, pos, social, neg, suk, batch_size, loss, reg, opt, lr_t, hyper, gU, gV, gB, tU, tV,
                     s0U, s1U, s0V, s1V, s0B, s1B, first_stamp, step_loss):
    n = users.numel()
    steps = (n + batch_size - 1) // batch_size
    lr_t = np.ascontiguousarray(lr_t, dtype=np.float32)
    assert lr_t.size >= max(steps, 1)
    h = np.zeros(4, dtype=np.float32)
    h[:len(hyper)] = hyper
    check(_lib.load().nrc_sbpr_train_epoch(
        _p(U), _p(V), _p(B), U.shape[0], V.shape[0], U.shape[1], _p(users), _p(pos), _p(social), _p(neg), _p(suk), n,
        int(batch_size), LOSS_IDS[loss], float(reg), OPT_IDS[opt], lr_t.ctypes.data, h.ctypes.data, _p(gU), _p(gV),
        _p(gB), _p(tU), _p(tV), _p(s0U), _p(s1U), _p(s0V), _p(s1V), _p(s0B), _p(s1B), int(first_stamp), _p(step_loss),
        _stream()))
    _count(2 * steps)
    return steps


# ------------------------------------------------------------------------- sequential: FPMC, TransRec
def _slot_array(slots):
    """HOST array of the variables' slot pointers (None -> NULL) for the *_train_epoch entry points."""
    return (ctypes.c_void_p * len(slots))(*[None if s is None else s.data_ptr() for s in slots])


def _epoch_prologue(users, batch_size, lr_t, hyper):
    n = users.numel()
    steps = (n + batch_size - 1) // batch_size
    lr_t = np.ascontiguousarray(lr_t, dtype=np.float32)
    assert lr_t.size >= max(steps, 1)
    h = np.zeros(4, dtype=np.float32)
    h[:len(hyper)] = hyper
    return n, steps, lr_t, h


def fpmc_grad(UI, IU, IL, LI, users, recent, items, third, pairwise, loss, reg, gUI, gIU, gIL, gLI, tU, tI, tL, stamp,
              loss_out):
    """Loss + row gradients of one FPMC batch (FPMC.py:61-84); `third` = negatives (i32) or labels (f32)."""
    check(_lib.load().nrc_fpmc_grad(_p(UI), _p(IU), _p(IL), _p(LI), UI.shape[1], _p(users), _p(recent), _p(items),
                                    _p(third), users.numel(), 1 if pairwise else 0, LOSS_IDS[loss], float(reg), _p(gUI),
                                    _p(gIU), _p(gIL), _p(gLI), _p(tU), _p(tI), _p(tL), int(stamp), _p(loss_out),
                                    _stream()))
    _count()


def fpmc_train_epoch(UI, IU, IL, LI, users, recent, items, third, batch_size, pairwise, loss, reg, opt, lr_t, hyper,
                     grads, touched, slots0, slots1, first_stamp, step_loss):
    """One FPMC epoch (FPMC.py:106-131): grads = (gUI, gIU, gIL, gLI), touched = (tU, tI, tL), slots0 / slots1 the
    four variables' optimizer slots (None where the optimizer keeps none).  Returns the number of steps."""
    n, steps, lr_t, h = _epoch_prologue(users, batch_size, lr_t, hyper)
    s0, s1 = _slot_array(slots0), _slot_array(slots1)
    check(_lib.load().nrc_fpmc_train_epoch(
        _p(UI), _p(IU), _p(IL), _p(LI), UI.shape[0], IU.shape[0], UI.shape[1], _p(users), _p(recent), _p(items),
        _p(third), n, int(batch_size), 1 if pairwise else 0, LOSS_IDS[loss], float(reg), OPT_IDS[opt],
        lr_t.ctypes.data, h.ctypes.data, *[_p(g) for g in grads], *[_p(t) for t in touched],
        ctypes.cast(s0, ctypes.c_void_p), ctypes.cast(s1, ctypes.c_void_p),
        int(first_stamp), _p(step_loss), _stream()))
    _count(2 * steps)
    return steps


def fpmc_scores(UI, IU, IL, LI, users, recent):
    """FPMC.predict(users, None) on the device: f32 [len(users), num_items] for rows (users[r], recent[r])."""
    for t, name in ((UI, "UI"), (IU, "IU"), (IL, "IL"), (LI, "LI")):
        _req(t, torch.float32, name)
    _req(users, torch.int32, "users"); _req(recent, torch.int32, "recent")
    out = torch.empty((users.numel(), IU.shape[0]), dtype=torch.float32, device=users.device)
    check(_lib.load().nrc_fpmc_scores(_p(UI), _p(IU), _p(IL), _p(LI), IU.shape[0], UI.shape[1], _p(users), _p(recent),
                                      users.numel(), _p(out), _stream()))
    _count()
    return out


def transrec_work(dim, device="cuda"):
    """Zero-filled scratch of the TransRec gradient (g's per-CTA partial sums and a completion counter)."""
    n = _lib.load().nrc_transrec_work_floats(int(dim))
    check(int(n) if n < 0 else 0)
    return torch.zeros(int(n), dtype=torch.float32, device=device)


def transrec_grad(P, Q, B, G, users, recent, items, third, pairwise, loss, reg, gP, gQ, gB, gG, tP, tQ, tB, stamp, work,
                  loss_out):
    """Loss + gradients of one TransRec batch (TransRec.py:66-91); gG is g's dense gradient f32 [d]."""
    check(_lib.load().nrc_transrec_grad(_p(P), _p(Q), _p(B), _p(G), P.shape[1], _p(users), _p(recent), _p(items),
                                        _p(third), users.numel(), 1 if pairwise else 0, LOSS_IDS[loss], float(reg),
                                        _p(gP), _p(gQ), _p(gB), _p(gG), _p(tP), _p(tQ), _p(tB), int(stamp), _p(work),
                                        _p(loss_out), _stream()))
    _count()


def transrec_train_epoch(P, Q, B, G, users, recent, items, third, batch_size, pairwise, loss, reg, opt, lr_t, hyper,
                         grads, touched, slots0, slots1, first_stamp, work, step_loss):
    """One TransRec epoch (TransRec.py:119-141): grads = (gP, gQ, gB, gG), touched = (tP, tQ, tB), slots in the order
    P, Q, b, g.  Returns the number of steps."""
    n, steps, lr_t, h = _epoch_prologue(users, batch_size, lr_t, hyper)
    s0, s1 = _slot_array(slots0), _slot_array(slots1)
    check(_lib.load().nrc_transrec_train_epoch(
        _p(P), _p(Q), _p(B), _p(G), P.shape[0], Q.shape[0], P.shape[1], _p(users), _p(recent), _p(items), _p(third), n,
        int(batch_size), 1 if pairwise else 0, LOSS_IDS[loss], float(reg), OPT_IDS[opt], lr_t.ctypes.data,
        h.ctypes.data, *[_p(g) for g in grads], *[_p(t) for t in touched],
        ctypes.cast(s0, ctypes.c_void_p), ctypes.cast(s1, ctypes.c_void_p),
        int(first_stamp), _p(work), _p(step_loss), _stream()))
    _count(2 * steps)
    return steps


def transrec_scores(P, Q, B, G, users, recent):
    """TransRec's prediction graph on the device: f32 [len(users), num_items], b_j - |(P_u + g) + Q_l - Q_j|."""
    for t, name in ((P, "P"), (Q, "Q"), (B, "B"), (G, "G")):
        _req(t, torch.float32, name)
    _req(users, torch.int32, "users"); _req(recent, torch.int32, "recent")
    out = torch.empty((users.numel(), Q.shape[0]), dtype=torch.float32, device=users.device)
    check(_lib.load().nrc_transrec_scores(_p(P), _p(Q), _p(B), _p(G), Q.shape[0], P.shape[1], _p(users), _p(recent),
                                          users.numel(), _p(out), _stream()))
    _count()
    return out


# ------------------------------------------------------------------------- sequential over a window: HRM, NPE
def _window(recent):
    """recent i32 [n, L] (or [n] at L = 1) -> L."""
    return 1 if recent.dim() == 1 else recent.shape[1]


def hrm_grad(P, E, users, recent, items, labels, pre_agg, session_agg, loss, reg, gP, gE, tP, tE, stamp, loss_out):
    """Loss + row gradients of one HRM batch (HRM.py:62-91); recent i32 [batch, L]; pre_agg / session_agg True = max."""
    check(_lib.load().nrc_hrm_grad(_p(P), _p(E), P.shape[1], _window(recent), _p(users), _p(recent), _p(items),
                                   _p(labels), users.numel(), int(bool(pre_agg)), int(bool(session_agg)),
                                   LOSS_IDS[loss], float(reg), _p(gP), _p(gE), _p(tP), _p(tE), int(stamp),
                                   _p(loss_out), _stream()))
    _count()


def hrm_train_epoch(P, E, users, recent, items, labels, batch_size, pre_agg, session_agg, loss, reg, opt, lr_t, hyper,
                    grads, touched, slots0, slots1, first_stamp, step_loss):
    """One HRM epoch (HRM.py:104-129): grads = (gP, gE), touched = (tP, tE), slots in the order P, E.  Returns the
    number of steps."""
    n, steps, lr_t, h = _epoch_prologue(users, batch_size, lr_t, hyper)
    s0, s1 = _slot_array(slots0), _slot_array(slots1)
    check(_lib.load().nrc_hrm_train_epoch(
        _p(P), _p(E), P.shape[0], E.shape[0], P.shape[1], _window(recent), _p(users), _p(recent), _p(items),
        _p(labels), n, int(batch_size), int(bool(pre_agg)), int(bool(session_agg)), LOSS_IDS[loss], float(reg),
        OPT_IDS[opt], lr_t.ctypes.data, h.ctypes.data, *[_p(g) for g in grads], *[_p(t) for t in touched],
        ctypes.cast(s0, ctypes.c_void_p), ctypes.cast(s1, ctypes.c_void_p), int(first_stamp), _p(step_loss),
        _stream()))
    _count(2 * steps)
    return steps


def _query_args(users, recent, recent_len):
    _req(users, torch.int32, "users"); _req(recent, torch.int32, "recent"); _req(recent_len, torch.int32, "recent_len")
    return _window(recent), _p(users), users.numel(), _p(recent), _p(recent_len)


def hrm_scores(P, E, users, recent, recent_len, pre_agg, session_agg):
    """HRM.predict(users, None) on the device: f32 [len(users), num_items].  recent i32 [num_users, L] / recent_len
    i32 [num_users] hold every user's predict window; the query rows h go through nrc_mf_scores."""
    _req(P, torch.float32, "P"); _req(E, torch.float32, "E")
    q = torch.empty((users.numel(), P.shape[1]), dtype=torch.float32, device=users.device)
    check(_lib.load().nrc_hrm_query(_p(P), _p(E), P.shape[1], *_query_args(users, recent, recent_len),
                                    int(bool(pre_agg)), int(bool(session_agg)), _p(q), _stream()))
    _count()
    return mf_scores(q, E, torch.arange(users.numel(), dtype=torch.int32, device=users.device))


def npe_scores(UI, IU, IL, users, recent, recent_len):
    """NPE.predict(users, None) on the device: f32 [len(users), num_items], the query rows relu(UI_u) + relu(c)
    against relu(IU) through nrc_mf_scores."""
    for t, name in ((UI, "UI"), (IU, "IU"), (IL, "IL")):
        _req(t, torch.float32, name)
    q = torch.empty((users.numel(), UI.shape[1]), dtype=torch.float32, device=users.device)
    items = torch.empty_like(IU)
    check(_lib.load().nrc_npe_query(_p(UI), _p(IU), _p(IL), IU.shape[0], UI.shape[1],
                                    *_query_args(users, recent, recent_len), _p(q), _p(items), _stream()))
    _count(2)
    return mf_scores(q, items, torch.arange(users.numel(), dtype=torch.int32, device=users.device))


def npe_grad(UI, IU, IL, users, recent, items, labels, loss, reg, gUI, gIU, gIL, tU, tI, tL, stamp, loss_out):
    """Loss + row gradients of one NPE batch (NPE.py:54-71); recent i32 [batch, L]."""
    check(_lib.load().nrc_npe_grad(_p(UI), _p(IU), _p(IL), UI.shape[1], _window(recent), _p(users), _p(recent),
                                   _p(items), _p(labels), users.numel(), LOSS_IDS[loss], float(reg), _p(gUI), _p(gIU),
                                   _p(gIL), _p(tU), _p(tI), _p(tL), int(stamp), _p(loss_out), _stream()))
    _count()


def npe_train_epoch(UI, IU, IL, users, recent, items, labels, batch_size, loss, reg, opt, lr_t, hyper, grads, touched,
                    slots0, slots1, first_stamp, step_loss):
    """One NPE epoch (NPE.py:84-108): grads = (gUI, gIU, gIL), touched = (tU, tI, tL), slots in the order UI, IU, IL.
    Returns the number of steps."""
    n, steps, lr_t, h = _epoch_prologue(users, batch_size, lr_t, hyper)
    s0, s1 = _slot_array(slots0), _slot_array(slots1)
    check(_lib.load().nrc_npe_train_epoch(
        _p(UI), _p(IU), _p(IL), UI.shape[0], IU.shape[0], UI.shape[1], _window(recent), _p(users), _p(recent),
        _p(items), _p(labels), n, int(batch_size), LOSS_IDS[loss], float(reg), OPT_IDS[opt], lr_t.ctypes.data,
        h.ctypes.data, *[_p(g) for g in grads], *[_p(t) for t in touched], ctypes.cast(s0, ctypes.c_void_p),
        ctypes.cast(s1, ctypes.c_void_p), int(first_stamp), _p(step_loss), _stream()))
    _count(2 * steps)
    return steps


# ------------------------------------------------------------------------- FPMCplus: attention over the window
def fpmcplus_work(dim, weight_size, window, batch_size, device="cuda"):
    """Zero-filled scratch of the FPMCplus gradient for batches of up to batch_size samples (the dense gradients'
    per-sample factors, per-chunk partial sums and completion counters)."""
    n = _lib.load().nrc_fpmcplus_work_floats(int(dim), int(weight_size), int(window), int(batch_size))
    check(int(n) if n < 0 else 0)
    return torch.zeros(int(n), dtype=torch.float32, device=device)


def fpmcplus_grad(UI, IU, IL, LI, W, b, h, users, recent, items, third, pairwise, loss, reg_mf, reg_w, grads, touched,
                  stamp, work, loss_out):
    """Loss + gradients of one FPMCplus batch (FPMCplus.py:53-119); recent i32 [batch, L], grads = (gUI, gIU, gIL, gLI,
    gW, gb, gh) (the last three dense), touched = (tU, tI, tL)."""
    check(_lib.load().nrc_fpmcplus_grad(
        _p(UI), _p(IU), _p(IL), _p(LI), _p(W), _p(b), _p(h), UI.shape[1], W.shape[1], _window(recent), _p(users),
        _p(recent), _p(items), _p(third), users.numel(), 1 if pairwise else 0, LOSS_IDS[loss], float(reg_mf),
        float(reg_w), *[_p(g) for g in grads], *[_p(t) for t in touched], int(stamp), _p(work), _p(loss_out),
        _stream()))
    _count(2)


def fpmcplus_train_epoch(UI, IU, IL, LI, W, b, h, users, recent, items, third, batch_size, pairwise, loss, reg_mf,
                         reg_w, opt, lr_t, hyper, grads, touched, slots0, slots1, first_stamp, work, step_loss):
    """One FPMCplus epoch (FPMCplus.py:141-171): grads and slots in the order UI, IU, IL, LI, W, b, h; touched =
    (tU, tI, tL).  Returns the number of steps."""
    n, steps, lr_t, hy = _epoch_prologue(users, batch_size, lr_t, hyper)
    s0, s1 = _slot_array(slots0), _slot_array(slots1)
    check(_lib.load().nrc_fpmcplus_train_epoch(
        _p(UI), _p(IU), _p(IL), _p(LI), _p(W), _p(b), _p(h), UI.shape[0], IU.shape[0], UI.shape[1], W.shape[1],
        _window(recent), _p(users), _p(recent), _p(items), _p(third), n, int(batch_size), 1 if pairwise else 0,
        LOSS_IDS[loss], float(reg_mf), float(reg_w), OPT_IDS[opt], lr_t.ctypes.data, hy.ctypes.data,
        *[_p(g) for g in grads], *[_p(t) for t in touched], ctypes.cast(s0, ctypes.c_void_p),
        ctypes.cast(s1, ctypes.c_void_p), int(first_stamp), _p(work), _p(step_loss), _stream()))
    _count(3 * steps)
    return steps


def fpmcplus_scores(UI, IU, IL, LI, W, b, h, users, recent, recent_len):
    """FPMCplus.predict(users, None) on the device: f32 [len(users), num_items].  recent i32 [num_users, L] /
    recent_len i32 [num_users] hold every user's predict window (see nrc_hrm_query)."""
    for t, name in ((UI, "UI"), (IU, "IU"), (IL, "IL"), (LI, "LI"), (W, "W"), (b, "b"), (h, "h")):
        _req(t, torch.float32, name)
    L, pu, rows, pr, pl = _query_args(users, recent, recent_len)
    lib = _lib.load()
    n = lib.nrc_fpmcplus_score_work_floats(IU.shape[0], UI.shape[1], W.shape[1], L, rows)
    check(int(n) if n < 0 else 0)
    work = torch.empty(max(int(n), 1), dtype=torch.float32, device=users.device)
    out = torch.empty((rows, IU.shape[0]), dtype=torch.float32, device=users.device)
    check(lib.nrc_fpmcplus_scores(_p(UI), _p(IU), _p(IL), _p(LI), _p(W), _p(b), _p(h), IU.shape[0], UI.shape[1],
                                  W.shape[1], L, pu, rows, pr, pl, _p(work), _p(out), _stream()))
    _count(2)
    return out


FPMCPLUS_KERNELS = ("grad", "wgrad", "project", "pair")
FPMCPLUS_ROUTE_FIELDS = ("pairwise", "grid_x", "grid_y", "capped", "window", "rows")


def fpmcplus_last_routes():
    """Routes of the most recent launch of each FPMCplus kernel (nrc_fpmcplus_last_routes) as {kernel: {field:
    value}}; -1 = no such launch yet or a field the kernel does not decide."""
    nf = len(FPMCPLUS_ROUTE_FIELDS)
    out = (ctypes.c_int32 * (len(FPMCPLUS_KERNELS) * nf))()
    check(_lib.load().nrc_fpmcplus_last_routes(out))
    return {k: dict(zip(FPMCPLUS_ROUTE_FIELDS, out[i * nf:(i + 1) * nf])) for i, k in enumerate(FPMCPLUS_KERNELS)}


# ------------------------------------------------------------------------- Caser: convolutions over the window
def caser_dense_floats(dim, seq_L, nv, nh):
    """Floats of Caser's dense block (every conv and FC weight and bias, layout in nrc_caser_dense_floats)."""
    n = _lib.load().nrc_caser_dense_floats(int(dim), int(seq_L), int(nv), int(nh))
    check(int(n) if n < 0 else 0)
    return int(n)


def caser_work(dim, seq_L, nv, nh, batch_size, device="cuda"):
    """Zero-filled scratch of the Caser gradient and epoch for batches of up to batch_size samples."""
    n = _lib.load().nrc_caser_work_floats(int(dim), int(seq_L), int(nv), int(nh), int(batch_size))
    check(int(n) if n < 0 else 0)
    return torch.zeros(int(n), dtype=torch.float32, device=device)


def _caser_sizes(P, W2, seqs, nv, nh):
    return P.shape[1], _window(seqs), int(nv), int(nh), W2.shape[0]


def caser_grad(P, E, W2, b2, dense, users, seqs, pos, neg, nv, nh, mask, keep, grads, work, loss_out=None):
    """Loss and gradients of one Caser batch (Caser.py:70-118): seqs i32 [batch, L], pos i32 [batch, T], neg i32
    [batch, N], mask f32 [batch, F] or None; grads = (gP, gE, gW2, gb2) accumulated, gDense overwritten."""
    d, L, nv, nh, ni = _caser_sizes(P, W2, seqs, nv, nh)
    check(_lib.load().nrc_caser_grad(
        _p(P), _p(E), _p(W2), _p(b2), _p(dense), ni, d, L, pos.shape[1], nv, nh, neg.shape[1], _p(users), _p(seqs),
        _p(pos), _p(neg), users.numel(), _p(mask), float(keep), *[_p(g) for g in grads], _p(work), _p(loss_out),
        _stream()))
    _count(2)


def caser_train_epoch(P, E, W2, b2, dense, users, seqs, pos, neg, nv, nh, batch_size, keep, l2_reg, seed, epoch, lr_t,
                      hyper, grads, slots0, slots1, work, step_loss):
    """One Caser epoch (Caser.py:128-139) over an already shuffled and sampled epoch: grads and slots in the order
    P, E, W2, b2, dense.  Returns the number of steps."""
    d, L, nv, nh, ni = _caser_sizes(P, W2, seqs, nv, nh)
    n, steps, lr_t, hy = _epoch_prologue(users, batch_size, lr_t, hyper)
    s0, s1 = _slot_array(slots0), _slot_array(slots1)
    check(_lib.load().nrc_caser_train_epoch(
        _p(P), _p(E), _p(W2), _p(b2), _p(dense), P.shape[0], ni, d, L, pos.shape[1], nv, nh, neg.shape[1], _p(users),
        _p(seqs), _p(pos), _p(neg), n, int(batch_size), float(keep), float(l2_reg), int(seed), int(epoch),
        lr_t.ctypes.data, hy.ctypes.data, *[_p(g) for g in grads], ctypes.cast(s0, ctypes.c_void_p),
        ctypes.cast(s1, ctypes.c_void_p), _p(work), _p(step_loss), _stream()))
    _count(5 * steps)
    return steps


def caser_query(P, E, W2, dense, users, windows, nv, nh):
    """Caser.predict's user vectors [z, P_u] (Caser.py:194-209): f32 [len(users), 2d] over windows i32 [num_users, L]."""
    for t, name in ((P, "P"), (E, "E"), (W2, "W2"), (dense, "dense")):
        _req(t, torch.float32, name)
    _req(users, torch.int32, "users"); _req(windows, torch.int32, "windows")
    d, L, nv, nh, ni = _caser_sizes(P, W2, windows, nv, nh)
    out = torch.empty((users.numel(), 2 * d), dtype=torch.float32, device=users.device)
    check(_lib.load().nrc_caser_query(_p(P), _p(E), _p(dense), ni, d, L, nv, nh, _p(users), users.numel(),
                                      _p(windows), _p(out), _stream()))
    _count()
    return out


def caser_scores(P, E, W2, dense, users, windows, nv, nh):
    """Caser.predict(users, None) on the device: f32 [len(users), num_items], [z, P_u] W2^T without the biases."""
    q = caser_query(P, E, W2, dense, users, windows, nv, nh)
    return mf_scores(q, W2, torch.arange(users.numel(), dtype=torch.int32, device=users.device))


CASER_KERNELS = ("grad", "wgrad", "query", "reg")
CASER_ROUTE_FIELDS = ("staged", "grid_x", "grid_y", "capped", "window", "masked")


def caser_last_routes():
    """Routes of the most recent launch of each Caser kernel (nrc_caser_last_routes) as {kernel: {field: value}};
    -1 = no such launch yet or a field the kernel does not decide."""
    nf = len(CASER_ROUTE_FIELDS)
    out = (ctypes.c_int32 * (len(CASER_KERNELS) * nf))()
    check(_lib.load().nrc_caser_last_routes(out))
    return {k: dict(zip(CASER_ROUTE_FIELDS, out[i * nf:(i + 1) * nf])) for i, k in enumerate(CASER_KERNELS)}


# ------------------------------------------------------------------------- FISM: item similarity over the history
def _fism_samples(hist_ptr, hist_idx, rows, excl, num, items, third, num_neg, pairwise):
    _req(hist_ptr, torch.int64, "hist_ptr"); _req(hist_idx, torch.int32, "hist_idx")
    for t, name in ((rows, "rows"), (num, "num"), (items, "items")):
        _req(t, torch.int32, name)
    if excl is not None:
        _req(excl, torch.int32, "excl")
    _req(third, torch.int32 if pairwise else torch.float32, "third")
    if pairwise:
        _req(num_neg, torch.int32, "num_neg")
    return rows.numel()


def fism_grad(c1, Q, b, hist_ptr, hist_idx, rows, excl, num, items, third, num_neg, pairwise, loss, alpha, lam, gamma,
              grads, touched, stamp, loss_out=None):
    """Loss and row gradients of one FISM batch (FISM.py:69-94): sample s sums c1 over history row rows[s] of the CSR
    (hist_ptr, hist_idx) without item excl[s] (excl None or -1: none); `third` = negatives (i32, pairwise, with
    num_neg their counts) or labels (f32).  grads = (gC1, gQ, gb) and touched = (tC1, tItem) are accumulated."""
    n = _fism_samples(hist_ptr, hist_idx, rows, excl, num, items, third, num_neg, pairwise)
    check(_lib.load().nrc_fism_grad(
        _p(c1), _p(Q), _p(b), Q.shape[0], Q.shape[1], _p(hist_ptr), _p(hist_idx), _p(rows), _p(excl), _p(num),
        _p(items), _p(third), _p(num_neg) if pairwise else None, n, 1 if pairwise else 0, LOSS_IDS[loss],
        float(alpha), float(lam), float(gamma), *[_p(g) for g in grads], *[_p(t) for t in touched], int(stamp),
        _p(loss_out), _stream()))
    _count()


def fism_train_epoch(c1, Q, b, hist_ptr, hist_idx, rows, excl, num, items, third, num_neg, batch_size, pairwise, loss,
                     alpha, lam, gamma, opt, lr_t, hyper, grads, touched, slots0, slots1, first_stamp, step_loss):
    """One FISM epoch (FISM.py:112-138) over an already built and shuffled epoch: grads, slots in the order c1, Q, b;
    touched = (tC1, tItem).  Returns the number of steps."""
    _fism_samples(hist_ptr, hist_idx, rows, excl, num, items, third, num_neg, pairwise)
    n, steps, lr_t, h = _epoch_prologue(rows, batch_size, lr_t, hyper)
    s0, s1 = _slot_array(slots0), _slot_array(slots1)
    check(_lib.load().nrc_fism_train_epoch(
        _p(c1), _p(Q), _p(b), Q.shape[0], Q.shape[1], _p(hist_ptr), _p(hist_idx), _p(rows), _p(excl), _p(num),
        _p(items), _p(third), _p(num_neg) if pairwise else None, n, int(batch_size), 1 if pairwise else 0,
        LOSS_IDS[loss], float(alpha), float(lam), float(gamma), OPT_IDS[opt], lr_t.ctypes.data, h.ctypes.data,
        *[_p(g) for g in grads], *[_p(t) for t in touched], ctypes.cast(s0, ctypes.c_void_p),
        ctypes.cast(s1, ctypes.c_void_p), int(first_stamp), _p(step_loss), _stream()))
    _count(2 * steps)
    return steps


def fism_query(c1, hist_ptr, hist_idx, users):
    """FISM.predict's user rows (FISM.py:154-180): f32 [len(users), d], the sum of c1 over each user's history row."""
    _req(c1, torch.float32, "c1"); _req(hist_ptr, torch.int64, "hist_ptr"); _req(hist_idx, torch.int32, "hist_idx")
    _req(users, torch.int32, "users")
    out = torch.empty((users.numel(), c1.shape[1]), dtype=torch.float32, device=users.device)
    check(_lib.load().nrc_fism_query(_p(c1), c1.shape[0], c1.shape[1], _p(hist_ptr), _p(hist_idx), _p(users),
                                     users.numel(), _p(out), _stream()))
    _count()
    return out


def fism_scores(c1, Q, b, hist_ptr, hist_idx, users, alpha):
    """FISM.predict(users, None) on the device: f32 [len(users), num_items], n^(-alpha) <p_u, Q_j> + b_j with n the
    length of the user's history row."""
    for t, name in ((Q, "Q"), (b, "b")):
        _req(t, torch.float32, name)
    p = fism_query(c1, hist_ptr, hist_idx, users)
    out = torch.empty((users.numel(), Q.shape[0]), dtype=torch.float32, device=users.device)
    check(_lib.load().nrc_fism_scores(_p(p), _p(Q), _p(b), Q.shape[0], Q.shape[1], float(alpha), _p(hist_ptr),
                                      _p(users), users.numel(), _p(out), _stream()))
    _count()
    return out


FISM_KERNELS = ("grad", "query", "scores")
FISM_ROUTE_FIELDS = ("pairwise", "vec", "lanes", "grid_x", "grid_y", "capped")


def fism_last_routes():
    """Routes of the most recent launch of each FISM kernel (nrc_fism_last_routes) as {kernel: {field: value}};
    -1 = no such launch yet or a field the kernel does not decide."""
    nf = len(FISM_ROUTE_FIELDS)
    out = (ctypes.c_int32 * (len(FISM_KERNELS) * nf))()
    check(_lib.load().nrc_fism_last_routes(out))
    return {k: dict(zip(FISM_ROUTE_FIELDS, out[i * nf:(i + 1) * nf])) for i, k in enumerate(FISM_KERNELS)}


# ------------------------------------------------------------------------- ItemKNN: neighbourhood similarity
ITEMKNN_KINDS = {"norm": 0, "tanimoto": 1, "dice": 2, "tversky": 3, "euclidean": 4}


def itemknn_similarity(csr_ptr, csr_idx, csr_val, csc_ptr, csc_idx, csc_val, num_items, kind, va, vb, shrink,
                       tversky_alpha, tversky_beta, neighbor, integral=None, gram_bound=None):
    """Compute_Similarity(...).compute_similarity() (ItemKNN.py:11-547) on the device: W in padded CSC form,
    (counts i32 [I], rows i32 [Kc, I], vals f32 [Kc, I]) with Kc = min(neighbor, I) and column c's entries at
    [:counts[c], c], rows ascending.  X comes as its CSR and its CSC (f64 values, already centred or made binary);
    va, vb f64 [I] are the per-item vectors (see nrc_itemknn_similarity); kind is a key of ITEMKNN_KINDS.
    integral / gram_bound default to what the values show: integral when every value is an integer, the bound
    max|x|^2 * (the longest column)."""
    for t, name in ((csr_ptr, "csr_ptr"), (csc_ptr, "csc_ptr")):
        _req(t, torch.int64, name)
    for t, name in ((csr_idx, "csr_idx"), (csc_idx, "csc_idx")):
        _req(t, torch.int32, name)
    for t, name in ((csr_val, "csr_val"), (csc_val, "csc_val"), (va, "va"), (vb, "vb")):
        _req(t, torch.float64, name)
    ni = int(num_items)
    if kind not in ITEMKNN_KINDS:
        raise ValueError("similarity kind '%s' is not one of %s" % (kind, sorted(ITEMKNN_KINDS)))
    if ni < 1 or int(neighbor) < 1:
        raise ValueError("num_items >= 1 and neighbor >= 1 required")
    if csc_ptr.numel() != ni + 1 or va.numel() != ni or vb.numel() != ni:
        raise ValueError("csc_ptr must hold num_items + 1 entries and va, vb num_items")
    if csr_idx.numel() != csc_idx.numel() or csr_val.numel() != csr_idx.numel() or csc_val.numel() != csc_idx.numel():
        raise ValueError("the CSR and the CSC must hold the same entries")
    if integral is None:
        integral = bool(csr_val.numel() == 0 or torch.equal(csr_val, torch.round(csr_val)))
    if gram_bound is None:
        top = float(csr_val.abs().max()) if csr_val.numel() else 0.0
        longest = int((csc_ptr[1:] - csc_ptr[:-1]).max()) if ni else 0
        gram_bound = top * top * longest
    kc = min(int(neighbor), ni)
    dev = csr_val.device
    counts = torch.empty(ni, dtype=torch.int32, device=dev)
    rows = torch.empty((kc, ni), dtype=torch.int32, device=dev)
    vals = torch.empty((kc, ni), dtype=torch.float32, device=dev)
    L = _lib.load()
    nbytes = int(L.nrc_itemknn_work_bytes(ni))
    work = torch.empty(max(nbytes, 1), dtype=torch.uint8, device=dev) if nbytes else None
    check(L.nrc_itemknn_similarity(
        csr_ptr.numel() - 1, ni, _p(csr_ptr), _p(csr_idx), _p(csr_val), _p(csc_ptr), _p(csc_idx), _p(csc_val),
        ITEMKNN_KINDS[kind], _p(va), _p(vb), float(shrink), float(tversky_alpha), float(tversky_beta), int(neighbor),
        1 if integral else 0, float(gram_bound), _p(work), nbytes, _p(counts), _p(rows), _p(vals), _stream()))
    _count()
    return counts, rows, vals


def itemknn_scores(csr_ptr, csr_idx, csr_val, W, users):
    """ItemKNN.predict(users, None) (ItemKNN.py:573, 583-585) on the device: f32 [len(users), I], the f64 sum of
    X[u, k] * W[k, j] over column j's entries in ascending k (scipy's order for train.tocsc().dot(W)) rounded once.
    W = (counts, rows, vals) from itemknn_similarity; X is the un-centred train CSR (f64 values)."""
    _req(csr_ptr, torch.int64, "csr_ptr"); _req(csr_idx, torch.int32, "csr_idx"); _req(csr_val, torch.float64, "csr_val")
    counts, rows, vals = W
    _req(counts, torch.int32, "counts"); _req(rows, torch.int32, "rows"); _req(vals, torch.float32, "vals")
    _req(users, torch.int32, "users")
    ni = counts.numel()
    if rows.dim() != 2 or rows.shape != vals.shape or rows.shape[1] != ni:
        raise ValueError("W's rows and vals must be [min(neighbor, I), I]")
    out = torch.empty((users.numel(), ni), dtype=torch.float32, device=users.device)
    check(_lib.load().nrc_itemknn_scores(ni, _p(csr_ptr), _p(csr_idx), _p(csr_val), max(rows.shape[0], 1),
                                         _p(counts), _p(rows), _p(vals), _p(users), users.numel(), _p(out),
                                         _stream()))
    _count()
    return out


ITEMKNN_KERNELS = ("similarity", "scores")
ITEMKNN_ROUTE_FIELDS = ("acc", "tier", "grid", "capped", "k", "smem")


def itemknn_last_routes():
    """Routes of the most recent launch of each ItemKNN kernel (nrc_itemknn_last_routes) as {kernel: {field: value}};
    -1 = no such launch yet or a field the kernel does not decide."""
    nf = len(ITEMKNN_ROUTE_FIELDS)
    out = (ctypes.c_int32 * (len(ITEMKNN_KERNELS) * nf))()
    check(_lib.load().nrc_itemknn_last_routes(out))
    return {k: dict(zip(ITEMKNN_ROUTE_FIELDS, out[i * nf:(i + 1) * nf])) for i, k in enumerate(ITEMKNN_KERNELS)}


SEQ_KERNELS = ("fpmc_grad", "transrec_grad", "hrm_grad", "npe_grad", "fpmc_scores", "transrec_scores", "hrm_query",
               "npe_query", "npe_relu")
SEQ_ROUTE_FIELDS = ("pairwise", "session_max", "pre_max", "grid_x", "grid_y", "capped", "window")


def seq_last_routes():
    """Routes of the most recent launch of each sequential kernel group (nrc_seq_last_routes) as
    {kernel: {field: value}}; -1 = no such launch yet or a field the group does not decide."""
    nf = len(SEQ_ROUTE_FIELDS)
    out = (ctypes.c_int32 * (len(SEQ_KERNELS) * nf))()
    check(_lib.load().nrc_seq_last_routes(out))
    return {k: dict(zip(SEQ_ROUTE_FIELDS, out[i * nf:(i + 1) * nf])) for i, k in enumerate(SEQ_KERNELS)}


EXTRAS_KERNELS = ("l2_normalize_rows", "gather_rows_i32", "sbpr_epoch_build", "sbpr_grad", "csr_from_coo",
                  "split_interactions", "csr_row_ids", "sample_negatives", "batch_randint_choice", "lightgcn_bpr_grad")
EXTRAS_ROUTE_FIELDS = ("grid", "capped", "row_grid", "row_capped", "scan_chunks", "replace")


def extras_last_routes():
    """Routes of the most recent launch of each data-side, sampler and LightGCN-gradient kernel group
    (nrc_extras_last_routes) as {kernel: {field: value}}; -1 = no such launch yet or a field the group does not decide."""
    nf = len(EXTRAS_ROUTE_FIELDS)
    out = (ctypes.c_int32 * (len(EXTRAS_KERNELS) * nf))()
    check(_lib.load().nrc_extras_last_routes(out))
    return {k: dict(zip(EXTRAS_ROUTE_FIELDS, out[i * nf:(i + 1) * nf])) for i, k in enumerate(EXTRAS_KERNELS)}


def csr_from_coo(rows, cols, num_rows, num_cols):
    """Interactions -> (indptr i64 [num_rows + 1], indices i32 [distinct]) with ascending duplicate-free rows
    (Dataset.to_csr_matrix + csr_to_user_dict, dataset.py:288-296, tool.py:56-65).  ValueError on ids out of range."""
    _req(rows, torch.int32, "rows"); _req(cols, torch.int32, "cols")
    if rows.numel() != cols.numel():
        raise ValueError("rows and cols must have the same length")
    nnz, dev = rows.numel(), rows.device
    indptr = torch.empty((num_rows + 1,), dtype=torch.int64, device=dev)
    indices = torch.empty((max(nnz, 1),), dtype=torch.int32, device=dev)
    w64 = torch.empty((2 * (num_rows + 1),), dtype=torch.int64, device=dev)
    w32 = torch.empty((max(2 * nnz, 1),), dtype=torch.int32, device=dev)
    bad = torch.empty((1,), dtype=torch.int32, device=dev)
    check(_lib.load().nrc_csr_from_coo(_p(rows), _p(cols), nnz, int(num_rows), int(num_cols), _p(indptr), _p(indices),
                                       _p(w64), _p(w32), _p(bad), _stream()))
    _count(6)
    if int(bad.item()):
        raise ValueError("interaction ids outside [0, %d) x [0, %d)" % (num_rows, num_cols))
    return indptr, indices[:int(indptr[-1].item())]


ACT_IDS = {"identity": 0, "sigmoid": 1, "tanh": 2, "relu": 3, "elu": 4, "selu": 5}


def _act_id(name):
    if name not in ACT_IDS:
        raise NotImplementedError("ERROR")                      # util/tool.py:32-33
    return ACT_IDS[name]


def spectralcf_work(num_nodes, dim, num_layers, device="cuda"):
    n = int(_lib.load().nrc_spectralcf_work_floats(int(num_nodes), int(dim), int(num_layers)))
    return torch.empty((max(n, 1),), dtype=torch.float32, device=device)


def spectralcf_forward(a_hat, e0, filters, activation, all_emb=None, work=None):
    """SpectralCF._create_inference (SpectralCF.py:63-83): [E_0 | act((A_hat E_0) W_1) | ...] f32 [N, d (K + 1)]."""
    _req(a_hat, torch.float32, "a_hat"); _req(e0, torch.float32, "e0"); _req(filters, torch.float32, "filters")
    N, d = e0.shape
    K = filters.shape[0]
    if all_emb is None:
        all_emb = torch.empty((N, d * (K + 1)), dtype=torch.float32, device=e0.device)
    work = spectralcf_work(N, d, K, e0.device) if work is None else work
    check(_lib.load().nrc_spectralcf_forward(N, d, K, _p(a_hat), _p(e0), _p(filters), _act_id(activation), _p(all_emb),
                                             _p(work), _stream()))
    _count(1 + 2 * K)
    return all_emb


def spectralcf_grad(num_users, a_hat, a_hat_t, e0, filters, activation, users, pos, neg, loss, reg, all_emb, grad_all,
                    touched, grad_e0, grad_filters, work, loss_out):
    """One batch of SpectralCF's loss + backward (nrc_spectralcf_grad)."""
    N, d = e0.shape
    K = filters.shape[0]
    check(_lib.load().nrc_spectralcf_grad(int(num_users), N - int(num_users), d, K, _p(a_hat), _p(a_hat_t), _p(e0),
                                          _p(filters), _act_id(activation), _p(users), _p(pos), _p(neg), users.numel(),
                                          LOSS_IDS[loss.lower()], float(reg), _p(all_emb), _p(grad_all), _p(touched),
                                          _p(grad_e0), _p(grad_filters), _p(work), _p(loss_out), _stream()))
    _count(3 + 6 * K)


def wrmf_work(num_rows_max, dim, device="cuda"):
    n = int(_lib.load().nrc_wrmf_work_floats(int(num_rows_max), int(dim)))
    return torch.empty((max(n, 1),), dtype=torch.float32, device=device)


def wrmf_half_step(fixed, indptr, indices, out, alpha, reg, row_order=None, work=None, not_spd=None):
    """One WRMF half-step (WRMF.py:51-61): every row of the CSR (indptr, indices) over the fixed table is solved
    in one call and written to out f32 [len(indptr) - 1, dim].  NrcError naming the count when some rows' matrices
    are not positive definite (those rows are left unchanged)."""
    _req(fixed, torch.float32, "fixed"); _req(out, torch.float32, "out")
    _req(indptr, torch.int64, "indptr"); _req(indices, torch.int32, "indices")
    if row_order is not None:
        _req(row_order, torch.int32, "row_order")
    num_fixed, dim = fixed.shape
    num_rows = indptr.numel() - 1
    if out.shape != (num_rows, dim):
        raise ValueError("out must be [%d, %d], got %s" % (num_rows, dim, tuple(out.shape)))
    work = wrmf_work(num_fixed, dim, fixed.device) if work is None else _req(work, torch.float32, "work")
    if work.numel() < _lib.load().nrc_wrmf_work_floats(num_fixed, dim):
        raise ValueError("work holds %d floats, the call needs nrc_wrmf_work_floats(%d, %d)" % (work.numel(), num_fixed, dim))
    if not_spd is None:
        not_spd = torch.empty((1,), dtype=torch.int32, device=fixed.device)
    check(_lib.load().nrc_wrmf_half_step(_p(fixed), num_fixed, _p(indptr), _p(indices), _p(row_order), num_rows, dim,
                                         float(alpha), float(reg), _p(out), _p(work), _p(not_spd), _stream()))
    _count(3)
    bad = int(not_spd.item())
    if bad:
        raise _lib.NrcError("WRMF: %d of %d rows have a matrix that is not positive definite (reg_mf = %g); "
                            "they were left unchanged" % (bad, num_rows, reg))
    return out


def split_interactions(users, keys, num_users, mode="ratio", ratio=0.8, seed=0):
    """Per-user train / test split of an interaction list on the device (data/utils.py:59-106): int32 [n] of 1 (train)
    / 0 (test).  keys: int64 CUDA tensor of interaction times (by_time=True) or None (by_time=False)."""
    _req(users, torch.int32, "users")
    if keys is not None:
        _req(keys, torch.int64, "keys")
    if mode not in ("ratio", "loo"):
        raise ValueError("There is not splitter '%s'" % mode)             # dataset.py:160-161
    n, dev = users.numel(), users.device
    out = torch.zeros((n,), dtype=torch.int32, device=dev)
    w64 = torch.empty((2 * (int(num_users) + 1),), dtype=torch.int64, device=dev)
    w32 = torch.empty((max(n, 1),), dtype=torch.int32, device=dev)
    bad = torch.empty((1,), dtype=torch.int32, device=dev)
    check(_lib.load().nrc_split_interactions(_p(users), _p(keys), n, int(num_users), 0 if mode == "ratio" else 1,
                                             float(ratio), int(seed), _p(out), _p(w64), _p(w32), _p(bad), _stream()))
    _count(4)
    if int(bad.item()):
        raise ValueError("user ids outside [0, %d)" % num_users)
    return out


def csr_row_ids(indptr, nnz=None, out=None):
    """Row id of every CSR entry (the sampler's flattened `users_list`, data/sampler.py:24-39), int32 [nnz]."""
    _req(indptr, torch.int64, "indptr")
    if out is None:
        out = torch.empty((int(indptr[-1].item()) if nnz is None else int(nnz),), dtype=torch.int32, device=indptr.device)
    check(_lib.load().nrc_csr_row_ids(_p(indptr), indptr.numel() - 1, _p(out), _stream()))
    _count()
    return out
