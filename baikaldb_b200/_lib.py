"""ctypes binding of libbkgpu.so (the C ABI in include/bkgpu.h).

The library is the product; this module only loads it.  There is no Python or CPU fallback: if
the shared object is missing, import of the operators fails loudly."""
from __future__ import annotations

import ctypes
import os
from ctypes import POINTER, Structure, byref, c_char, c_char_p, c_double, c_int, c_int32, c_int64, c_size_t, c_uint8, \
    c_uint32, c_uint64, c_void_p

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("BKGPU_LIB") or os.path.join(_HERE, "libbkgpu.so")  # BKGPU_LIB: A/B builds while tuning

OK, EINVAL, EUNSUPPORTED, ENODEV, ENOMEM, ESTATE, ECANCELLED, ETOOBIG, ENCCL = 0, -1, -2, -3, -4, -5, -6, -7, -8
ERROR_NAMES = {EINVAL: "EINVAL", EUNSUPPORTED: "EUNSUPPORTED", ENODEV: "ENODEV", ENOMEM: "ENOMEM", ESTATE: "ESTATE",
               ECANCELLED: "ECANCELLED", ETOOBIG: "ETOOBIG", ENCCL: "ENCCL"}


class BkgpuColumn(Structure):
    _fields_ = [("tuple_id", c_int32), ("slot_id", c_int32), ("prim_type", c_int32), ("elem_size", c_int32),
                ("values", c_void_p), ("validity", c_void_p), ("length", c_int64)]


class BkgpuBinaryColumn(Structure):
    _fields_ = [("offsets", c_void_p), ("data", c_void_p), ("validity", c_void_p), ("validity_offset", c_int64), ("length", c_int64)]


class BkgpuStats(Structure):
    _fields_ = [("rows_scanned", c_int64), ("rows_filtered", c_int64), ("rows_returned", c_int64),
                ("kernel_launches", c_int64), ("h2d_bytes", c_int64), ("d2h_bytes", c_int64),
                ("main_kernel_ms", c_double), ("main_kernel_launches", c_int64), ("main_kernel_bytes", c_int64),
                ("collective_ms", c_double), ("main_kernel_name", c_char * 64)]


# every symbol include/bkgpu.h declares: (name, restype, argtypes)
SYMBOLS = [
    ("bkgpu_version", c_char_p, []),
    ("bkgpu_device_count", c_int, []),
    ("bkgpu_last_error", c_char_p, [c_void_p]),
    ("bkgpu_plan_explain", c_int, [c_char_p, c_size_t, c_char_p, c_size_t]),
    ("bkgpu_init", c_int, [POINTER(c_void_p), c_char_p, c_size_t, c_int, c_void_p]),
    ("bkgpu_set_option", c_int, [c_void_p, c_char_p, c_int64]),
    ("bkgpu_open", c_int, [c_void_p]),
    ("bkgpu_push", c_int, [c_void_p, POINTER(BkgpuColumn), c_int, c_int64, c_int]),
    ("bkgpu_finish", c_int, [c_void_p]),
    ("bkgpu_get_next", c_int, [c_void_p, POINTER(BkgpuColumn), POINTER(c_int), POINTER(c_int64), POINTER(c_int)]),
    ("bkgpu_reset", c_int, [c_void_p]),
    ("bkgpu_cancel", None, [c_void_p]),
    ("bkgpu_close", None, [c_void_p]),
    ("bkgpu_get_stats", c_int, [c_void_p, POINTER(BkgpuStats)]),
    ("bkgpu_region_register", c_int, [c_int, c_int64, POINTER(BkgpuColumn), c_int, c_int64, c_int]),
    ("bkgpu_region_evict", c_int, [c_int, c_int64]),
    ("bkgpu_region_info", c_int, [c_int, c_int64, POINTER(c_int64), POINTER(c_size_t)]),
    ("bkgpu_release_cache", None, []),
    ("bkgpu_parse_datetime", c_int, [c_char_p, c_size_t, c_int, POINTER(c_uint64)]),
    ("bkgpu_cast_image", c_int, [c_uint64, c_int, c_int, POINTER(c_uint64)]),
    ("bkgpu_hll_estimate", c_int, [c_char_p, c_size_t, POINTER(c_uint64)]),
    ("bkgpu_push_region", c_int, [c_void_p, c_int64]),
    ("bkgpu_partial_capacity", c_int, [c_void_p, POINTER(c_size_t)]),
    ("bkgpu_partial_export", c_int, [c_void_p, c_void_p, c_size_t]),
    ("bkgpu_partial_merge", c_int, [c_void_p, c_void_p, c_size_t, c_int]),
    ("bkgpu_nccl_unique_id", c_int, [POINTER(c_uint8)]),
    ("bkgpu_nccl_comm_create", c_int, [POINTER(c_void_p), POINTER(c_uint8), c_int, c_int, c_int]),
    ("bkgpu_nccl_comm_destroy", None, [c_void_p]),
    ("bkgpu_host_alloc", c_void_p, [c_size_t]),
    ("bkgpu_host_free", None, [c_void_p]),
    ("bkgpu_device_alloc", c_void_p, [c_int, c_size_t]),
    ("bkgpu_device_free", None, [c_int, c_void_p]),
    ("bkgpu_memcpy_h2d", c_int, [c_int, c_void_p, c_void_p, c_size_t]),
    ("bkgpu_memcpy_d2h", c_int, [c_int, c_void_p, c_void_p, c_size_t]),
    ("bkgpu_gen_column", c_int, [c_int, c_void_p, c_int32, c_int32, c_uint64, c_uint32, c_int64, c_int64, c_int64,
                                 c_int64, c_double]),
    ("bkgpu_dict_build", c_int, [POINTER(c_void_p), c_int, c_void_p, POINTER(BkgpuBinaryColumn), c_int, c_int]),
    ("bkgpu_dict_size", c_int, [c_void_p, POINTER(c_int64), POINTER(c_int64)]),
    ("bkgpu_dict_copy", c_int, [c_void_p, c_void_p, c_void_p, c_int]),
    ("bkgpu_dict_codes", c_int, [c_void_p, c_int, c_void_p, c_void_p, POINTER(c_int64)]),
    ("bkgpu_dict_free", None, [c_void_p]),
]

_lib = None


class BkgpuError(RuntimeError):
    def __init__(self, code: int, message: str):
        super().__init__(f"bkgpu {ERROR_NAMES.get(code, code)}: {message}")
        self.code = code
        self.message = message


def lib() -> ctypes.CDLL:
    """Load libbkgpu.so (built by ``__graft_entry__.build()`` / ``make -C csrc``)."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise ImportError(f"{LIB_PATH} is missing: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
                              "(there is no CPU fallback for this path)")
        L = ctypes.CDLL(LIB_PATH, mode=ctypes.RTLD_GLOBAL)
        for name, restype, argtypes in SYMBOLS:
            fn = getattr(L, name)
            fn.restype = restype
            fn.argtypes = argtypes
        _lib = L
    return _lib


def check(rc: int, plan=None) -> None:
    if rc != OK:
        msg = lib().bkgpu_last_error(plan)
        raise BkgpuError(rc, msg.decode(errors="replace") if msg else "")


def explain(plan_bytes: bytes) -> str:
    buf = ctypes.create_string_buffer(1 << 16)
    rc = lib().bkgpu_plan_explain(plan_bytes, len(plan_bytes), buf, len(buf))
    if rc != OK:
        raise BkgpuError(rc, buf.value.decode(errors="replace"))
    return buf.value.decode()


__all__ = ["lib", "check", "explain", "BkgpuColumn", "BkgpuBinaryColumn", "BkgpuStats", "BkgpuError", "SYMBOLS", "LIB_PATH", "byref"]
