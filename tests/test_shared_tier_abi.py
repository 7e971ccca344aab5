"""CPU-only: the tier blob of pb_table_export_tier_view has the layout include/persia_b200.h describes, the tiered view
calls refuse bad arguments before touching a device, and persia_core splits a table with a shared tier at any
replica_size (PERSIA_B200_SHARED_TIER) while the refusal without it stays."""
import ctypes as C
import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from test_remote_view_abi import _Blob  # noqa: E402


class _TierBlob(C.Structure):
    """magic, version, the exporting pid and random number, its device, whether the handle is valid, the device pointers
    of the tier's index cells and mapped rows, the cells' CUDA IPC handle (64 bytes), the rows' memfd number and byte
    size, and the tier's geometry."""
    _fields_ = [("magic", C.c_uint32), ("version", C.c_uint32), ("pid", C.c_uint64), ("nonce", C.c_uint64),
                ("device", C.c_int32), ("ipc", C.c_uint32), ("cells", C.c_uint64), ("rows", C.c_uint64),
                ("handle", C.c_char * 64), ("fd", C.c_int32), ("pad0", C.c_uint32), ("bytes", C.c_uint64),
                ("n_cells", C.c_uint32), ("capacity", C.c_uint32), ("stride", C.c_uint32), ("dim", C.c_uint32)]


def _lib():
    from persia_b200 import build, native as N

    build.build()
    return N, N.load()


def _view(version=1, pid=7, nonce=9):
    b = _Blob()
    b.magic, b.version, b.pid, b.nonce, b.n_cells, b.dim, b.stride, b.capacity = 0x57564250, version, pid, nonce, 1024, 16, 16, 100
    return bytes(b)


def _tier(pid=7, nonce=9, **kw):
    t = _TierBlob()
    t.magic, t.version, t.pid, t.nonce, t.n_cells, t.capacity, t.stride, t.dim = 0x54564250, 1, pid, nonce, 2048, 1000, 16, 16
    t.bytes = 4 * t.capacity * t.stride
    for k, v in kw.items():
        setattr(t, k, v)
    return bytes(t)


def test_tier_blob_layout():
    N, lib = _lib()
    assert int(lib.pb_tier_view_bytes()) == C.sizeof(_TierBlob) == 144
    assert int(lib.pb_table_view_bytes()) == C.sizeof(_Blob)  # the table's blob is unchanged


def test_tiered_view_refusals_before_any_device_work():
    N, lib = _lib()
    h = C.c_void_p()
    buf = C.create_string_buffer(C.sizeof(_TierBlob))
    assert lib.pb_table_export_tier_view(None, buf) == N.PB_ERR_INVALID
    assert lib.pb_view_open_tiered(0, _view(2), None, C.byref(h)) == N.PB_ERR_INVALID
    assert lib.pb_view_open_tiered(0, None, _tier(), C.byref(h)) == N.PB_ERR_INVALID
    # a tiered table's blob alone: refused, so that no reader ignores the tier
    assert lib.pb_view_open(0, _view(2), C.byref(h)) == N.PB_ERR_STATE
    assert b"pb_view_open_tiered" in lib.pb_last_error()
    # not a tier blob, or one of another geometry or export
    assert lib.pb_view_open_tiered(0, _view(2), bytes(C.sizeof(_TierBlob)), C.byref(h)) == N.PB_ERR_INVALID
    assert b"not a tier view" in lib.pb_last_error()
    assert lib.pb_view_open_tiered(0, _view(2), _tier(n_cells=1000), C.byref(h)) == N.PB_ERR_INVALID
    assert lib.pb_view_open_tiered(0, _view(2), _tier(dim=8), C.byref(h)) == N.PB_ERR_INVALID
    assert lib.pb_view_open_tiered(0, _view(2), _tier(bytes=12), C.byref(h)) == N.PB_ERR_INVALID
    assert lib.pb_view_open_tiered(0, _view(2), _tier(pid=8), C.byref(h)) == N.PB_ERR_INVALID
    assert b"another table's export" in lib.pb_last_error()
    assert lib.pb_view_open_tiered(0, _view(2), _tier(nonce=10), C.byref(h)) == N.PB_ERR_INVALID
    # a table without a shared tier is opened with pb_view_open
    assert lib.pb_view_open_tiered(0, _view(1), _tier(), C.byref(h)) == N.PB_ERR_INVALID
    assert b"no shared host tier" in lib.pb_last_error()


def test_hbm_split_shared():
    from persia_b200.persia_core import hbm_split

    assert hbm_split(1 << 20, "1000", 4, shared=True) == (1000, (1 << 20) - 1000)
    assert hbm_split(1 << 20, "1000", 1, shared=True) == (1000, (1 << 20) - 1000)
    assert hbm_split(1 << 20, None, 4, shared=True) == (1 << 20, 0)
    assert hbm_split(1 << 20, str(1 << 21), 4, shared=True) == (1 << 20, 0)
    with pytest.raises(RuntimeError) as e:
        hbm_split(1 << 20, "1000", 2)
    assert "one GPU only" in str(e.value) and "PERSIA_B200_HBM_ROWS" in str(e.value)
    with pytest.raises(RuntimeError):
        hbm_split(1 << 20, "0", 2, shared=True)


def test_shared_tier_switch(monkeypatch):
    from persia_b200 import persia_core as pc

    monkeypatch.delenv("PERSIA_B200_SHARED_TIER", raising=False)
    assert not pc.shared_tier_on()
    monkeypatch.setenv("PERSIA_B200_SHARED_TIER", "0")
    assert not pc.shared_tier_on()
    monkeypatch.setenv("PERSIA_B200_SHARED_TIER", "1")
    assert pc.shared_tier_on()
