"""CPU-only: the view blob of pb_table_export_view has the layout include/persia_b200.h describes, and the view calls
refuse bad arguments before touching a device."""
import ctypes as C
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


class _Blob(C.Structure):
    """The blob's fields: magic, version, the exporting pid, a random number of the exporting process, its device, whether the IPC handles are valid, the device
    pointers and CUDA IPC handles (64 bytes each) of the index cells, rows, counters and write-sequence word, and the
    table's geometry."""
    _fields_ = [("magic", C.c_uint32), ("version", C.c_uint32), ("pid", C.c_uint64), ("nonce", C.c_uint64),
                ("device", C.c_int32),
                ("ipc", C.c_uint32), ("ptr", C.c_uint64 * 4), ("handle", (C.c_char * 64) * 4), ("dim", C.c_uint32),
                ("stride", C.c_uint32), ("state_floats", C.c_uint32), ("n_cells", C.c_uint32), ("capacity", C.c_uint32),
                ("pad", C.c_uint32)]


def test_view_blob_layout_and_refusals():
    from persia_b200 import build, native as N

    build.build()
    lib = N.load()
    assert int(lib.pb_table_view_bytes()) == C.sizeof(_Blob)
    blob = C.create_string_buffer(C.sizeof(_Blob))
    assert lib.pb_table_export_view(None, blob) == N.PB_ERR_INVALID
    h = C.c_void_p()
    assert lib.pb_view_open(0, blob, C.byref(h)) == N.PB_ERR_INVALID  # not a view: zero magic
    assert b"not a table view" in lib.pb_last_error()
    b = _Blob.from_buffer_copy(blob.raw)
    b.magic, b.version, b.n_cells, b.dim, b.stride = 0x57564250, 1, 1000, 16, 16  # n_cells not a power of two
    assert lib.pb_view_open(0, bytes(b), C.byref(h)) == N.PB_ERR_INVALID
    assert lib.pb_view_close(None) == N.PB_OK
    assert lib.pb_forward_remote(None, None, 1, 0, None, None, 0, None, None, 0, None, None) == N.PB_ERR_INVALID
