"""ctypes binding of ``include/rpk.h`` -- the same C-ABI a cgo binding would call (INTEGRATION.md).

There is no CPU implementation behind this module: if ``librpk.so`` is missing, or no sm_90 GPU (H100) is
present, construction fails loudly.
"""
from __future__ import annotations

import ctypes as C
import os

_PKG = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_PKG, "lib", "librpk.so")

RPK_OK, RPK_EINVAL, RPK_ECUDA, RPK_ENOMEM, RPK_ESTATE, RPK_ENODEV = 0, -1, -2, -3, -4, -5
ERR_NAMES = {0: "RPK_OK", -1: "RPK_EINVAL", -2: "RPK_ECUDA", -3: "RPK_ENOMEM", -4: "RPK_ESTATE", -5: "RPK_ENODEV"}


class RpkStats(C.Structure):
    _fields_ = [
        ("select_calls", C.c_uint64), ("offer_scores", C.c_uint64), ("status_calls", C.c_uint64),
        ("status_records", C.c_uint64), ("last_select_kernel_ms", C.c_float), ("last_select_total_ms", C.c_float),
        ("last_status_kernel_ms", C.c_float), ("last_status_total_ms", C.c_float),
        ("select_kernel_kind", C.c_uint32), ("n_gpus", C.c_uint32), ("distinct_mem", C.c_uint32),
        ("distinct_vcpu", C.c_uint32), ("distinct_ram", C.c_uint32), ("packed_bits", C.c_uint32),
    ]


# Every function include/rpk.h declares, in its order: name -> (restype, argtypes).  Each parameter has the width and
# signedness of its C type; every pointer or array parameter is a pointer type (data pointers are plain c_void_p, so
# numpy and torch buffers pass as addresses).  tests/test_abi.py checks this table against the header.
_p, _pp, _int, _u32, _size = C.c_void_p, C.POINTER(C.c_void_p), C.c_int, C.c_uint32, C.c_size_t
ABI = {
    "rpk_create": (_int, [_int, C.POINTER(C.c_int), _pp]),
    "rpk_destroy": (None, [_p]),
    "rpk_last_error": (C.c_char_p, [_p]),
    "rpk_abi_version": (_int, []),
    "rpk_host_alloc": (_p, [_size]),
    "rpk_host_free": (None, [_p]),
    "rpk_offers_upload": (_int, [_p, _u32, _p, _p, _p, _p, _p, _p]),
    "rpk_offers_refresh": (_int, [_p, _u32, _p, _p, _p, _p, _p, _p, _p]),
    "rpk_select": (_int, [_p, _u32, _p, _p, _p, _p, _p, _p, _p]),
    "rpk_pods_reset": (_int, [_p, _u32]),
    "rpk_pods_grow": (_int, [_p, _u32]),
    "rpk_pods_seed_slots": (_int, [_p, _u32, _p, _p, _p, _p, _p, _p]),
    "rpk_select_slots": (_int, [_p, _u32, _p, _p, _p]),
    "rpk_explain": (_int, [_p, _u32, _p, _p, _p, _p, _p, _p]),
    "rpk_explain_slots": (_int, [_p, _u32, _p, _p]),
    "rpk_pods_mark_pending": (_int, [_p, _u32, _p, _p]),
    "rpk_select_pending": (_int, [_p, _u32, _p, _p, _p, _p]),
    "rpk_select_pending_changed": (_int, [_p, _u32, _p, _p, _p, _p, _p, _p]),
    "rpk_select_device": (_int, [_p, _int, _u32, _p, _p, _p, _p, _p, _p, _p, _p]),
    "rpk_select_device_gather": (_int, [_p, _int, _u32, _p, _p, _p, _p, _p, _int, _pp, _u32, _p, _p]),
    "rpk_select_device_gather_top5": (_int, [_p, _int, _u32, _p, _p, _p, _p, _p, _int, _pp, _pp, _u32, _p]),
    "rpk_select_slots_device": (_int, [_p, _int, _u32, _p, _p, _p, _p]),
    "rpk_select_slots_device_gather": (_int, [_p, _int, _u32, _p, _int, _pp, _u32, _p, _p]),
    "rpk_select_slots_device_gather_top5": (_int, [_p, _int, _u32, _p, _int, _pp, _pp, _u32, _p]),
    "rpk_pods_pending_list_device": (_int, [_p, _int, _p, _p, _p]),
    "rpk_results_xchg_bytes": (_size, [_int, _u32]),
    "rpk_select_pending_changed_gather": (_int, [_p, _int, _int, _int, _pp, _u32, _p, _p, _p]),
    "rpk_select_pending_changed_device_gather": (_int, [_p, _int, _int, _int, _pp, _u32, _p, _p]),
    "rpk_ipc_alloc": (_int, [_p, _int, _size, _pp, C.c_char_p]),
    "rpk_ipc_open": (_int, [_p, _int, C.c_char_p, _pp]),
    "rpk_ipc_close": (_int, [_p, _int, _p]),
    "rpk_ipc_free": (_int, [_p, _int, _p]),
    "rpk_peer_fence": (_int, [_p, _int, _int, _pp, _int, _u32, _p]),
    "rpk_peer_bind": (_int, [_p, _int, _int, _pp, _int]),
    "rpk_peer_wait": (_int, [_p, _int, C.c_uint, _p]),
    "rpk_peer_inline_wait": (_int, [_p, _int, _int]),
    "rpk_best_device_ptr": (_p, [_p, _int]),
    "rpk_test_capture_buffers": (_int, [_p, _int, _pp, _size, C.POINTER(C.c_size_t)]),
    "rpk_status_diff": (_int, [_p, _u32, _p, _u32, _p, _p, _p]),
    "rpk_status_diff_codes": (_int, [_p, _u32, _p, _u32, _p, _p, _p, _p]),
    "rpk_status_seed": (_int, [_p, _u32, _p, _u32]),
    "rpk_status_seed_slots": (_int, [_p, _u32, _p, _p, _u32]),
    "rpk_status_diff_slots": (_int, [_p, _u32, _p, _p, _u32, _p, _p, _p]),
    "rpk_status_diff_slots_device": (_int, [_p, _int, _u32, _u32, _u32, _p, _p, _u32, _p, _p, _p, _p, _p]),
    "rpk_status_reset": (_int, [_p, _u32]),
    "rpk_status_grow": (_int, [_p, _u32]),
    "rpk_tick": (_int, [_p, _u32, _p, _p, _p, _p, _p, _p, _p, _u32, _p, _u32, _p, _p, _p]),
    "rpk_status_diff_device": (_int, [_p, _int, _u32, _p, _u32, _p, _p, _p, _p]),
    "rpk_status_diff_device_codes": (_int, [_p, _int, _u32, _p, _u32, _p, _p, _p, _p, _p]),
    "rpk_xchg_bytes": (_size, [_int, _u32]),
    "rpk_status_diff_device_gather": (_int, [_p, _int, _u32, _p, _u32, _p, _u32, _int, _pp, _u32, _int, _p, _p]),
    "rpk_status_diff_slots_device_gather": (_int, [_p, _int, _u32, _u32, _u32, _p, _p, _u32, _p, _int, _pp, _u32, _int, _p, _p]),
    "rpk_stats_get": (_int, [_p, C.POINTER(RpkStats)]),
    "rpk_launch_count": (C.c_uint64, [_p]),
}
SYMBOLS = list(ABI)


class RpkError(RuntimeError):
    def __init__(self, code: int, msg: str):
        super().__init__(f"{ERR_NAMES.get(code, code)}: {msg}")
        self.code = code


_lib = None


def load():
    """Load ``librpk.so`` (built in-tree by ``__graft_entry__.build()`` / ``make -C csrc``)."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise ImportError(f"{LIB_PATH} is missing: build it with `make -C {os.path.join(_PKG, 'csrc')}` "
                          "(there is no CPU fallback)")
    L = C.CDLL(LIB_PATH)
    for name, (restype, argtypes) in ABI.items():
        fn = getattr(L, name)
        fn.restype, fn.argtypes = restype, argtypes
    _lib = L
    return L
