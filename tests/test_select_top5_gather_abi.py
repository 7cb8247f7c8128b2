"""CPU checks of rpk_select_device_gather_top5's boundary: the header declares it, the Python binding declares it with
the header's parameter types, and the library refuses a NULL ctx before it touches CUDA."""
import ctypes as C

import rpk
from test_abi import c_sig, ctypes_sig, header_prototypes

NAME = "rpk_select_device_gather_top5"


def test_declared_in_the_header_and_the_binding():
    ret, params = header_prototypes()[NAME]
    restype, argtypes = rpk._ffi.ABI[NAME]
    assert ret == "int" and restype is C.c_int
    assert [c_sig(p, True) for p in params] == [ctypes_sig(t) for t in argtypes]
    # the assignment vectors, then the top-5 vectors, then row0 and the stream
    assert [p.split()[-1].lstrip("*") for p in params[-5:]] == ["n_out", "d_best_full", "d_top5_full", "row0", "stream"]


def test_null_ctx_is_refused():
    lib = rpk._ffi.load()
    ptrs = (C.c_void_p * 1)(None)
    assert lib.rpk_select_device_gather_top5(None, 0, 1, None, None, None, None, None, 1, ptrs, ptrs, 0, None) == rpk._ffi.RPK_EINVAL
