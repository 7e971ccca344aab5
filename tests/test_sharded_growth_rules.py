"""CPU: PERSIA_B200_GROW=shared (exportable growable tables, at any replica_size) and its refusals, the entry points
of exportable growth in the symbol list, and the version-3 view blob's checks, all before any device is touched."""
import ctypes as C
import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from test_remote_view_abi import _Blob  # noqa: E402  (the blob layout, unchanged by version 3)


@pytest.mark.parametrize("replica_size", [1, 2, 4, 8])
def test_shared_at_every_replica_size(replica_size):
    from persia_b200.persia_core import growth_on

    assert growth_on("shared", replica_size=replica_size) == "shared"
    assert growth_on(" shared ", replica_size=replica_size, hbm_rows="") == "shared"
    with pytest.raises(RuntimeError, match="PERSIA_B200_HBM_ROWS"):
        growth_on("shared", replica_size=replica_size, hbm_rows="4096")


def test_one_still_refused_on_r_gpus_and_points_to_shared():
    from persia_b200.persia_core import growth_on

    with pytest.raises(RuntimeError, match="one GPU only.*shared"):
        growth_on("1", replica_size=2)
    with pytest.raises(RuntimeError, match="PERSIA_B200_GROW must be"):
        growth_on("Shared")


def test_grow_mode_of_a_shard():
    from persia_b200 import native as N
    from persia_b200.shard import grow_mode

    assert [grow_mode(g) for g in (False, None, 0, "0", "")] == [N.GROW_OFF] * 5
    assert [grow_mode(g) for g in (True, 1, "1")] == [N.GROW_ON] * 3
    assert [grow_mode(g) for g in ("shared", 2)] == [N.GROW_SHARED] * 2
    with pytest.raises(ValueError):
        grow_mode("yes")


def test_symbols():
    from persia_b200 import native as N

    assert N.SYMBOLS["pb_table_set_growth"][1] == [N._vp, N._i32]
    assert N.SYMBOLS["pb_view_address"][1] == [N._vp, C.c_char_p, N._u64]
    assert N.SYMBOLS["pb_table_add_reader"][1] == [N._vp, C.c_char_p]
    assert (N.GROW_OFF, N.GROW_ON, N.GROW_SHARED) == (0, 1, 2)


def _grow_blob(rows_span, cells_span, gran, max_cells, n_cells=1024, capacity=1000, dim=16, stride=16):
    b = _Blob()
    b.magic, b.version, b.pid, b.nonce = 0x57564250, 3, 7, 9
    b.n_cells, b.capacity, b.dim, b.stride, b.pad = n_cells, capacity, dim, stride, max_cells
    spans = {0: cells_span, 1: rows_span}  # handle[cells], handle[rows]: (span, granularity)
    for i, span in spans.items():
        C.memmove(C.addressof(b) + _Blob.handle.offset + 64 * i, (C.c_uint64 * 2)(span, gran), 16)
    return bytes(b)


def test_version_3_blob_checks():
    from persia_b200 import build, native as N

    build.build()
    lib = N.load()
    assert int(lib.pb_table_view_bytes()) == C.sizeof(_Blob)  # the same size as every other version
    h = C.c_void_p()
    g = 2 << 20
    rows, cells = g * 1, g * 1  # 1000 rows x 64 bytes, 2051 cells x 16 bytes: each within one granule
    # malformed: no granularity, a span off the granularity, rows or cells larger than their spans, max_cells not a
    # power of two or below n_cells
    for blob in (_grow_blob(rows, cells, 0, 2048), _grow_blob(rows + 1, cells, g, 2048),
                 _grow_blob(1024, cells, 1024, 2048), _grow_blob(rows, 1024, 1024, 2048),
                 _grow_blob(rows, cells, g, 3000), _grow_blob(rows, cells, g, 512)):
        assert lib.pb_view_open(0, blob, C.byref(h)) == N.PB_ERR_INVALID
        assert b"growable table geometry is malformed" in lib.pb_last_error()
    # a growable table has no tier: the tiered open refuses its blob
    assert lib.pb_view_open_tiered(0, _grow_blob(rows, cells, g, 2048), bytes(144), C.byref(h)) == N.PB_ERR_INVALID
    assert lib.pb_table_add_reader(None, b"x") == N.PB_ERR_INVALID
    assert lib.pb_view_address(None, C.create_string_buffer(8), 8) == N.PB_ERR_INVALID
