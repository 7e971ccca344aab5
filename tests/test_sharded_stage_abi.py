"""CPU-only: the stage exchange of pb_tier_stage_sharded has the area layout include/persia_b200.h describes, and its
calls refuse bad arguments before touching a device."""
import ctypes as C
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def _round256(v):
    return (v + 255) // 256 * 256


def test_stage_bytes_layout_and_zeros():
    from persia_b200 import build, native as N

    build.build()
    lib = N.load()
    ctrl = _round256(5 * 16 * 4)  # XC_WORDS x 16 u32 flag and count words
    assert ctrl == 512
    for R, cap in ((1, 1), (2, 100), (4, 4096), (16, 12345)):
        assert int(lib.pb_xchg_stage_bytes(R, cap)) == ctrl + _round256(R * cap * 8), (R, cap)
    for R, cap in ((0, 8), (17, 8), (2, 0), (16, 1 << 28)):
        assert int(lib.pb_xchg_stage_bytes(R, cap)) == 0, (R, cap)
    # much smaller than a batch exchange of the same pair count: no rows, gradients or chain words
    assert int(lib.pb_xchg_stage_bytes(2, 1000)) < int(lib.pb_xchg_bytes(2, 1000, 1, 0))


def test_stage_calls_refuse_bad_arguments_before_the_device():
    from persia_b200 import build, native as N

    build.build()
    lib = N.load()
    h = C.c_void_p()
    bases = (C.c_uint64 * 2)(256, 512)
    assert lib.pb_xchg_create_stage(0, 2, 0, 8, None, C.byref(h)) == N.PB_ERR_INVALID
    assert lib.pb_xchg_create_stage(0, 2, 0, 8, bases, None) == N.PB_ERR_INVALID
    assert lib.pb_xchg_create_stage(0, 2, 2, 8, bases, C.byref(h)) == N.PB_ERR_INVALID  # rank >= R
    assert lib.pb_xchg_create_stage(0, 0, 0, 8, bases, C.byref(h)) == N.PB_ERR_INVALID
    assert lib.pb_xchg_create_stage(0, 2, 0, 0, bases, C.byref(h)) == N.PB_ERR_INVALID
    assert lib.pb_xchg_create_stage(0, 2, 0, 8, (C.c_uint64 * 2)(256, 300), C.byref(h)) == N.PB_ERR_INVALID
    assert b"256-byte aligned" in lib.pb_last_error()
    assert h.value is None
    off = (C.c_uint32 * 2)(0, 0)
    pf = (C.c_uint64 * 1)(0)
    assert lib.pb_tier_stage_sharded(None, None, None, 0, off, pf, 1, 8, None, 0) == N.PB_ERR_INVALID
    assert lib.pb_tier_stage_sharded(None, None, None, 0, None, None, 1, 8, None, 0) == N.PB_ERR_INVALID
    assert b"null argument" in lib.pb_last_error()
    assert lib.pb_xchg_destroy(None) == N.PB_OK
