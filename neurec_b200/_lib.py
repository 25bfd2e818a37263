"""ctypes binding of the C ABI declared in include/neurec_b200.h.

There is no CPU fallback: when ``libneurec_b200.so`` is missing, loading raises and every
product entry point fails loudly (``python -c "import __graft_entry__ as g; g.build()"``
builds it in-tree with nvcc for sm_90a).
"""
from __future__ import annotations

import ctypes
import os
import re

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(HERE, "libneurec_b200.so")
HEADER = os.path.join(os.path.dirname(HERE), "include", "neurec_b200.h")

NRC_OK, NRC_E_VALUE, NRC_E_TYPE, NRC_E_NOTIMPL, NRC_E_CUDA, NRC_E_LIMIT = 0, -1, -2, -3, -4, -5

METRIC_IDS = {"Precision": 1, "Recall": 2, "MAP": 3, "NDCG": 4, "MRR": 5}
LOSS_IDS = {"bpr": 0, "hinge": 1, "square": 2, "cross_entropy": 3}
OPT_IDS = {"gd": 0, "adam": 1, "adagrad": 2, "rmsprop": 3, "momentum": 4}

_CT = {
    "int": ctypes.c_int, "int32_t": ctypes.c_int32, "int64_t": ctypes.c_int64,
    "uint64_t": ctypes.c_uint64, "float": ctypes.c_float, "double": ctypes.c_double,
}


class NrcError(RuntimeError):
    """`rc` is the NRC_E_* code of a failed call (None when the library could not be loaded)."""

    def __init__(self, msg, rc=None):
        super().__init__(msg)
        self.rc = rc


def declared_functions(header: str = HEADER):
    """Parse ``include/neurec_b200.h`` -> {name: (restype, [argtypes])}."""
    text = open(header).read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    out = {}
    for m in re.finditer(r"(const char\*|int64_t|int)\s+(nrc_\w+)\s*\(([^)]*)\)\s*;", text):
        ret, name, args = m.group(1), m.group(2), m.group(3)
        argtypes = []
        args = args.strip()
        if args and args != "void":
            for a in args.split(","):
                a = a.strip()
                if "*" in a:
                    argtypes.append(ctypes.c_void_p)
                else:
                    ty = a.replace("const", "").split()[0]
                    argtypes.append(_CT[ty])
        out[name] = ({"const char*": ctypes.c_char_p, "int64_t": ctypes.c_int64}.get(ret, ctypes.c_int), argtypes)
    return out


_LIB = None


def load() -> ctypes.CDLL:
    """Load the CUDA library; raises NrcError when it has not been built."""
    global _LIB
    if _LIB is None:
        if not os.path.isfile(LIB_PATH):
            raise NrcError(
                "neurec_b200: %s is missing -- the CUDA library is the only implementation of "
                "the hot path (no CPU fallback). Build it with "
                "`python -c 'import __graft_entry__ as g; g.build()'`." % LIB_PATH)
        lib = ctypes.CDLL(LIB_PATH)
        for name, (ret, argtypes) in declared_functions().items():
            fn = getattr(lib, name)  # AttributeError if the library lacks a declared symbol
            fn.restype = ret
            fn.argtypes = argtypes
        _LIB = lib
    return _LIB


def check(rc: int) -> None:
    """Translate an NRC_E_* return code into the exception the reference raises."""
    if rc == NRC_OK:
        return
    msg = load().nrc_last_error().decode("utf-8", "replace")
    if rc == NRC_E_VALUE:
        raise ValueError(msg)
    if rc == NRC_E_TYPE:
        raise TypeError(msg)
    if rc == NRC_E_NOTIMPL:
        raise NotImplementedError(msg)
    raise NrcError("neurec_b200 error %d: %s" % (rc, msg), rc)
