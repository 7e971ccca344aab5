"""CPU-only: the C-ABI library loads and exports every symbol include/persia_b200.h declares."""
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _declared():
    src = open(os.path.join(ROOT, "include", "persia_b200.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(pb_[a-z0-9_]+)\s*\(", src)))


def test_library_exports_every_declared_symbol():
    from persia_b200 import build, native

    build.build()
    lib = native.load()
    names = _declared()
    assert len(names) >= 20
    for n in names:
        assert hasattr(lib, n), f"{n} declared in include/persia_b200.h but not exported"
    assert set(names) == set(native.SYMBOLS), "ctypes binding and header disagree"
    assert lib.pb_version() >= 100


def test_no_cpu_fallback_in_product_path():
    """persia_b200/ must not import or call the oracle."""
    for dp, _, fs in os.walk(os.path.join(ROOT, "persia_b200")):
        for f in fs:
            if f.endswith((".py", ".cu", ".cuh", ".cpp", ".h")):
                txt = open(os.path.join(dp, f)).read()
                assert "import oracle" not in txt and "from oracle" not in txt and "persia_oracle" not in txt, f


def test_missing_library_fails_loudly(monkeypatch):
    from persia_b200 import native

    monkeypatch.setattr(native, "_lib", None)
    monkeypatch.setattr(native, "SO_PATH", "/nonexistent/libpersia_b200.so")
    with pytest.raises(native.PersiaB200Error):
        native.load()


def test_refusals_from_every_abi_file_reach_pb_last_error():
    """The checkpoint, sharded, view and batch calls each refuse a bad argument before touching a device, and the
    message of each refusal is what pb_last_error reads next: one error state for every file of the C ABI."""
    import ctypes as C

    from persia_b200 import build, native as N

    build.build()
    lib = N.load()
    out = C.c_void_p()
    assert lib.pb_image_create(0, 0, C.byref(out)) == N.PB_ERR_INVALID
    assert b"zero max_chunk" in lib.pb_last_error()
    bases = (C.c_uint64 * 1)(256)
    assert lib.pb_xchg_create(0, 0, 0, 1, 16, 0, bases, C.byref(out)) == N.PB_ERR_INVALID
    assert lib.pb_last_error() == b"bad argument"
    blob = C.create_string_buffer(int(lib.pb_table_view_bytes()))
    assert lib.pb_view_open(0, blob, C.byref(out)) == N.PB_ERR_INVALID
    assert b"not a table view" in lib.pb_last_error()
    ids = (C.c_uint64 * 1)(1)
    occ = (C.c_uint32 * 2)(0, 1)
    assert lib.pb_forward(None, None, ids, 1, None, occ, 1, 0, None, None) == N.PB_ERR_INVALID
    assert lib.pb_last_error() == b"null argument"
