"""The inverse of the epoch bijection (csrc/epoch.cuh: feistel_perm_inv), which the CSR-fed BPR/SGD step uses to find
the user rows one triplet of a launch touches alone.  The header's host side is compiled here and checked against the
oracle's restatement of the forward bijection (oracle.shuffle_perm); the rule the kernel applies is checked on the
benchmark's first step."""
import ctypes
import os
import subprocess

import numpy as np
import pytest

import oracle

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

HARNESS = r"""
#include "neurec_b200/csrc/epoch.cuh"
extern "C" int perm_pair(int64_t n, int shuffle, uint64_t seed, uint64_t epoch, int64_t* fwd, int64_t* inv) {
    nrc::Feistel F;
    const int rc = nrc::feistel_init(F, n, shuffle, seed, epoch);
    if (rc) return rc;
    for (int64_t p = 0; p < n; ++p) { fwd[p] = nrc::feistel_perm(F, p); inv[p] = nrc::feistel_perm_inv(F, p); }
    return 0;
}
"""


@pytest.fixture(scope="module")
def perm_pair(tmp_path_factory):
    from neurec_b200 import _build
    if _build.needs_build():
        _build.build()
    d = tmp_path_factory.mktemp("perm_inv")
    src, so = d / "harness.cu", d / "harness.so"
    src.write_text(HARNESS)
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    libdir = os.path.dirname(_build.LIB)
    subprocess.run([nvcc, "-std=c++17", "-shared", "-Xcompiler", "-fPIC", "-I", ROOT, "-o", str(so), str(src),
                    "-L", libdir, "-lneurec_b200", "-Xlinker", "-rpath=" + libdir], check=True)
    lib = ctypes.CDLL(str(so))
    lib.perm_pair.argtypes = [ctypes.c_int64, ctypes.c_int, ctypes.c_uint64, ctypes.c_uint64, ctypes.c_void_p,
                              ctypes.c_void_p]

    def call(n, shuffle, seed, epoch):
        fwd, inv = np.empty(n, np.int64), np.empty(n, np.int64)
        assert lib.perm_pair(n, 1 if shuffle else 0, seed, epoch, fwd.ctypes.data, inv.ctypes.data) == 0
        return fwd, inv
    return call


@pytest.mark.parametrize("n", [0, 1, 2, 3, 5, 17, 64, 1000, 4097, 65536, 300_001])
@pytest.mark.parametrize("shuffle,seed,epoch", [(True, 2018, 0), (True, 7, 3), (True, 1 << 40, 12345), (False, 5, 1)])
def test_inverse_bijection(perm_pair, n, shuffle, seed, epoch):
    fwd, inv = perm_pair(n, shuffle, seed, epoch)
    assert np.array_equal(fwd, oracle.shuffle_perm(n, seed, epoch, shuffle))
    p = np.arange(n, dtype=np.int64)
    assert np.array_equal(inv[fwd], p) and np.array_equal(fwd[inv], p)
    if not shuffle:
        assert np.array_equal(inv, p)


def test_single_visit_rule_on_the_benchmark_step():
    """The kernel's rule -- user u of the triplet at position p is touched by no other triplet of [first, first +
    count) when no other CSR position q of u's row has perm^-1(q) in that window (rows up to 32 positives) -- gives
    the share profiles/step_rows.py counts for the benchmark's first step (0.845)."""
    import bench
    cfg = bench.ShardedCfg
    ptr, idx = bench.synth_shard_csr(cfg, 0, 1, device="cpu")
    n = len(idx)
    perm = oracle.shuffle_perm(n, bench.SEED, 0, True)
    inv = np.empty(n, np.int64)
    inv[perm] = np.arange(n)
    first, count = 0, cfg.batch
    users = np.repeat(np.arange(len(ptr) - 1, dtype=np.int64), np.diff(ptr))
    idx_w = perm[first:first + count]
    u = users[idx_w]
    # per CSR position: is it visited in the window?  A row is touched once iff exactly one of its positions is.
    visited = ((inv - first) >= 0) & ((inv - first) < count)
    per_row = np.add.reduceat(visited.astype(np.int64), ptr[:-1]) if n else np.zeros(0, np.int64)
    deg = np.diff(ptr)
    once = (per_row[u] == 1) & (deg[u] <= 32)
    share = float(once.mean())
    assert abs(share - float((np.bincount(u, minlength=len(ptr) - 1)[u] == 1).mean())) == 0
    assert abs(share - 0.845) < 0.005
