"""The CPU oracle in table mode: _mm256_rsqrt_ps from the committed RSQRTPS table (tests/rsqrt_oracle.cpp), so that it
reproduces the reference's Adagrad as run on an Intel CPU on any host.

    with table_mode(oracle):
        w = oracle.Worker(...)   # every oracle object made and dropped inside the block
        ...

Inside the block the `oracle` module calls the table-mode library (the same C++ as oracle/persia_oracle.cpp, built
beside it with the instruction replaced), with set_rsqrt_exact(False) = the table.  The library is compiled once per
source version into the temporary directory, so the tree is never written.
"""
import contextlib
import ctypes as C
import hashlib
import json
import os
import subprocess
import tempfile
import threading

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
SRC = os.path.join(HERE, "rsqrt_oracle.cpp")
ORACLE_SRC = os.path.join(ROOT, "oracle", "persia_oracle.cpp")
TABLE_JSON = os.path.join(HERE, "golden", "intel_rsqrtps_table.json")
_FLAGS = ["-O2", "-std=c++17", "-mavx2", "-mfma", "-mf16c", "-ffp-contract=off", "-fPIC", "-Wall",
          "-Wno-unused-function", "-pthread", "-shared"]

_lib = None
_lock = threading.Lock()


def table_entries():
    """The 2048 committed entries (f32 bit patterns, uint32)."""
    with open(TABLE_JSON) as f:
        return np.array([int(e, 16) for e in json.load(f)["entries"]], np.uint32)


def build():
    h = hashlib.sha256()
    for p in (SRC, ORACLE_SRC):
        with open(p, "rb") as f:
            h.update(f.read())
    h.update(" ".join(_FLAGS).encode())
    d = os.path.join(tempfile.gettempdir(), f"persia_b200_rsqrt_oracle_{os.getuid()}")
    os.makedirs(d, exist_ok=True)
    so = os.path.join(d, f"librsqrt_oracle_{h.hexdigest()[:16]}.so")
    if not os.path.exists(so):
        tmp = f"{so}.{os.getpid()}.tmp"
        subprocess.check_call([os.environ.get("CXX", "g++")] + _FLAGS + ["-o", tmp, SRC])
        os.replace(tmp, so)
    os.utime(so)  # newer than the oracle's source: oracle.lib() rebuilds its own library otherwise
    return so


def lib(oracle):
    """The table-mode library, its signatures bound as the oracle module binds its own, the table loaded."""
    global _lib
    with _lock:
        if _lib is None:
            saved_lib, saved_so = oracle._lib, oracle._SO
            try:
                oracle._lib, oracle._SO = None, build()
                L = oracle.lib()
            finally:
                oracle._lib, oracle._SO = saved_lib, saved_so
            u64, vp = C.c_uint64, C.c_void_p
            for name, res, args in (("po_set_rsqrt_table", None, [vp]), ("po_rsqrt_table_many", None, [vp, u64, vp]),
                                    ("po_rsqrt_intrinsic_many", None, [vp, u64, vp]),
                                    ("po_rsqrt_table_mismatches", u64, [u64, u64])):
                getattr(L, name).restype, getattr(L, name).argtypes = res, args
            t = table_entries()
            L.po_set_rsqrt_table(t.ctypes.data_as(vp))
            _lib = L
        return _lib


@contextlib.contextmanager
def table_mode(oracle):
    """The oracle module in table mode for the block; exact-rsqrt mode (set_rsqrt_exact(True)) stays available in it."""
    L = lib(oracle)
    saved = oracle._lib
    oracle._lib = L
    try:
        oracle.set_rsqrt_exact(False)
        yield oracle
    finally:
        L.po_set_rsqrt_exact(0)
        oracle._lib = saved


def _bits_call(oracle, name, x):
    x = np.ascontiguousarray(x).view(np.uint32)
    out = np.empty_like(x)
    getattr(lib(oracle), name)(x.ctypes.data_as(C.c_void_p), x.size, out.ctypes.data_as(C.c_void_p))
    return out


def rsqrt_table(oracle, x):
    """The table model of every element of x (float32 or its bit patterns), as uint32 bit patterns."""
    return _bits_call(oracle, "po_rsqrt_table_many", x)


def rsqrt_intrinsic(oracle, x):
    """This host's RSQRTPS of every element of x, as uint32 bit patterns."""
    return _bits_call(oracle, "po_rsqrt_intrinsic_many", x)


def mismatches(oracle, lo, hi):
    """Inputs in the bit-pattern range [lo, hi) where the table model and this host's RSQRTPS differ."""
    return int(lib(oracle).po_rsqrt_table_mismatches(lo, hi))
