"""ctypes binding of libpersia_b200.so (include/persia_b200.h).

There is no CPU fallback: if the library is missing or a call fails, this raises.  PyTorch is used by
the callers only to own device memory and streams; the signatures here are plain pointers and sizes.
"""
import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
SO_PATH = os.environ.get("PERSIA_B200_LIB") or os.path.join(_HERE, "libpersia_b200.so")  # override: kernel experiments

PB_MAX_SLOTS = 128
OPT_SGD, OPT_ADAGRAD, OPT_ADAGRAD_VW, OPT_ADAM = 0, 1, 2, 3

PHASE_SEND, PHASE_SERVE, PHASE_FINISH, PHASE_ALL = 1, 2, 4, 7
PB_OK, PB_ERR_INVALID, PB_ERR_CUDA, PB_ERR_STATE, PB_ERR_CAPACITY, PB_ERR_BATCH = 0, -1, -2, -3, -4, -5


class PersiaB200Error(RuntimeError):
    """Every fallible call of the reference maps PersiaError -> RuntimeError (persia-core/src/lib.rs:94-98)."""

    def __init__(self, code, msg):
        super().__init__(f"[pb {code}] {msg}")
        self.code = code


class TableCfg(C.Structure):
    _fields_ = [("dim", C.c_uint32), ("capacity", C.c_uint64)]


class OptimCfg(C.Structure):
    _fields_ = [("kind", C.c_int), ("lr", C.c_float), ("wd", C.c_float), ("g_square_momentum", C.c_float),
                ("initialization", C.c_float), ("eps", C.c_float), ("beta1", C.c_float), ("beta2", C.c_float)]


class HyperCfg(C.Structure):
    _fields_ = [("init_lower", C.c_float), ("init_upper", C.c_float), ("admit_probability", C.c_float),
                ("enable_weight_bound", C.c_int), ("weight_bound", C.c_float)]


class SlotsCfg(C.Structure):
    _fields_ = [("n_slots", C.c_uint32), ("prefix_bit", C.c_uint32), ("prefix", C.c_uint64 * PB_MAX_SLOTS),
                ("sqrt_scaling", C.c_uint8 * PB_MAX_SLOTS)]


# every symbol include/persia_b200.h declares: name -> (restype, argtypes)
_vp, _u32, _u64, _i32 = C.c_void_p, C.c_uint32, C.c_uint64, C.c_int
SYMBOLS = {
    "pb_last_error": (C.c_char_p, []),
    "pb_version": (_i32, []),
    "pb_table_create": (_i32, [_i32, C.POINTER(TableCfg), C.POINTER(_vp)]),
    "pb_table_destroy": (_i32, [_vp]),
    "pb_table_set_optimizer": (_i32, [_vp, C.POINTER(OptimCfg)]),
    "pb_table_configure": (_i32, [_vp, C.POINTER(HyperCfg)]),
    "pb_table_size": (_i32, [_vp, C.POINTER(_u64), _vp]),
    "pb_table_clear": (_i32, [_vp, _vp]),
    "pb_table_entry_len": (_i32, [_vp, C.POINTER(_u32)]),
    "pb_table_set_eviction": (_i32, [_vp, _u32, _u64, _u64, _u32]),
    "pb_table_spill": (_i32, [_vp, _u64, _u32, _vp, _vp, _u32, _vp, _vp]),
    "pb_table_counters": (_i32, [_vp, C.POINTER(_u64 * 5), _vp]),
    "pb_lookup": (_i32, [_vp, _vp, _u32, _i32, _vp, _vp]),
    "pb_update": (_i32, [_vp, _vp, _vp, _u32, _vp]),
    "pb_set_rows": (_i32, [_vp, _vp, _vp, _u32, _vp]),
    "pb_get_rows": (_i32, [_vp, _vp, _u32, _vp, _vp, _vp]),
    "pb_table_export_signs": (_i32, [_vp, _vp, _vp, _u32, _vp, _vp]),
    "pb_add_prefix": (_i32, [_vp, _u32, C.POINTER(_u32), C.POINTER(_u64), _u32, _u32, _vp, _vp]),
    "pb_shard_of": (_i32, [_vp, _u32, _u32, _vp, _vp]),
    "pb_hash_stack": (_i32, [_vp, _u32, _u32, _u64, _vp, _vp]),
    "pb_farmhash64": (_i32, [_vp, _u32, _vp, _vp]),
    "pb_partition_by_shard": (_i32, [_vp, _u32, _u32, _vp, _vp, _vp, _u64, _vp]),
    "pb_partition_workspace": (_u64, [_u32]),
    "pb_ctx_create": (_i32, [_i32, _u32, _u32, C.POINTER(_vp)]),
    "pb_ctx_destroy": (_i32, [_vp]),
    "pb_ctx_set_slots": (_i32, [_vp, C.POINTER(SlotsCfg)]),
    "pb_ctx_batch_stats": (_i32, [_vp, C.POINTER(_u32 * 6), _vp]),
    "pb_forward": (_i32, [_vp, _vp, _vp, _u32, _vp, C.POINTER(_u32), _u32, _i32, _vp, _vp]),
    "pb_backward": (_i32, [_vp, _vp, C.POINTER(_vp), _i32, C.POINTER(C.c_float), _vp, _vp]),
    "pb_forward_raw": (_i32, [_vp, _vp, _vp, _u32, _vp, _u32, _u32, _i32, _vp, _vp, _vp, _vp, _vp, _vp]),
    "pb_backward_raw": (_i32, [_vp, _vp, _vp, _i32, C.c_float, _vp, _vp]),
    "pb_xchg_bytes": (_u64, [_u32, _u32, _u32, _i32]),
    "pb_xchg_create": (_i32, [_i32, _u32, _u32, _u32, _u32, _i32, C.POINTER(_u64), C.POINTER(_vp)]),
    "pb_xchg_destroy": (_i32, [_vp]),
    "pb_xchg_status": (_i32, [_vp, C.POINTER(_u32 * 2), _vp]),
    "pb_forward_sharded": (_i32, [_vp, _vp, _vp, _vp, _u32, _vp, C.POINTER(_u32), _u32, _i32, _vp, _vp, _i32]),
    "pb_backward_sharded": (_i32, [_vp, _vp, _vp, C.POINTER(_vp), _i32, C.POINTER(C.c_float), _vp, _vp, _i32]),
    "pb_forward_raw_sharded": (_i32, [_vp, _vp, _vp, _vp, _u32, _vp, _u32, _u32, _i32, _vp, _vp, _vp, _vp, _vp, _vp, _i32]),
    "pb_backward_raw_sharded": (_i32, [_vp, _vp, _vp, _vp, _i32, C.c_float, _vp, _vp, _i32]),
    "pb_launch_count": (_u64, []),
    "pb_profile_enable": (_i32, [_i32]),
    "pb_profile_read": (_i32, [C.POINTER(C.c_double), C.POINTER(_u64), _i32]),
}

_lib = None


def load():
    """Loads the library (once).  Loading needs libcudart but no GPU; compute calls need a device."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(SO_PATH):
        raise PersiaB200Error(PB_ERR_STATE, f"{SO_PATH} is missing: run `python -c 'import __graft_entry__ as g; "
                                            f"g.build()'` (persia_b200/build.py); there is no CPU fallback")
    lib = C.CDLL(SO_PATH, mode=C.RTLD_GLOBAL)
    for name, (res, args) in SYMBOLS.items():
        fn = getattr(lib, name)
        fn.restype = res
        fn.argtypes = args
    _lib = lib
    return lib


def check(rc):
    if rc != 0:
        raise PersiaB200Error(rc, load().pb_last_error().decode("utf-8", "replace"))
