"""Refusals of every device entry point, and of the host sweep rpk_status_seed: each fault a call refuses returns its
code, names the function called at the start of rpk_last_error, launches nothing and, with flags bound, signals nothing.

Every ctx here binds a two-rank peer group on shard 0, so a gather with n_out > 1 is a bound gather that would signal
if it ran.  The buffers are real and large enough for the call, so only the fault under test stands between a call and
its launches."""
import ctypes as C
import importlib

import numpy as np
import pytest

import rpk

pytestmark = pytest.mark.gpu

EINVAL, ESTATE = rpk._ffi.RPK_EINVAL, rpk._ffi.RPK_ESTATE
P = 64       # rows, slots, records and table sizes of every call
STRIDE = 32  # a valid status stride; 8 is the bad one


class Rig:
    """three one-GPU ctxs -- "full" (offer and pod tables), "pods" (pod table only), "bare" (neither) -- with flags
    bound, and the device buffers every call reads or writes"""

    def __init__(self):
        import torch

        peer = importlib.import_module("k8s-runpod-kubelet_b200.peer")
        dev = torch.device("cuda", 0)
        self.engines, self.flags = {}, {}
        offers = rpk.synth.make_offers(300)
        for kind in ("full", "pods", "bare"):
            eng = rpk.Engine(1)
            if kind == "full":
                eng.upload_offers(offers)
            if kind != "bare":
                eng.pods_reset(P)
            flags = eng.ipc_alloc(64 * 4)[0]
            eng.peer_bind([flags, flags], 0)
            self.engines[kind] = eng
            self.flags[kind] = peer.as_int32_tensor(flags, 64, dev)

        def buf(n, dtype=torch.int32):
            return torch.zeros(n, dtype=dtype, device=dev)

        self.keep = []

        def ptr(t):
            self.keep.append(t)
            return t.data_ptr()

        self.mem = ptr(torch.full((P,), 8, dtype=torch.int32, device=dev))
        self.slots = ptr(torch.arange(P, dtype=torch.int32, device=dev))
        self.best = [ptr(buf(P)) for _ in range(2)]
        self.top5 = [ptr(buf(5 * P)) for _ in range(2)]
        self.n = ptr(buf(1))
        self.records = ptr(buf(P * STRIDE, torch.uint8))
        self.hash_prev = ptr(buf(P, torch.int64))
        self.idx = ptr(buf(P))
        self.code = ptr(buf(P, torch.int16))
        lib = self.engines["full"]._lib
        self.xchg = [ptr(buf(lib.rpk_xchg_bytes(2, P), torch.uint8)) for _ in range(2)]
        self.res_xchg = ptr(buf(lib.rpk_results_xchg_bytes(1, P), torch.uint8))
        self.host_records = np.zeros(P * STRIDE, np.uint8)
        self.n_pending, self.n_reselected = C.c_uint32(), C.c_uint32()

    def close(self):
        for eng in self.engines.values():
            eng.close()


@pytest.fixture(scope="module")
def rig():
    r = Rig()
    yield r
    r.close()


def arr(ptrs):
    return (C.c_void_p * len(ptrs))(*ptrs)


def cols(r):
    return (r.mem, None, None, None, None)


def host(x):
    return C.cast(C.byref(x), C.c_void_p)


# (id, ctx, function, shard -> arguments after ctx, code).  The shard is 0 unless the case is the out-of-range one.
CASES = [
    ("shard", "full", "rpk_select_device", lambda r, s: (s, P, *cols(r), r.best[0], None, None), EINVAL),
    ("offers", "bare", "rpk_select_device", lambda r, s: (s, P, *cols(r), r.best[0], None, None), ESTATE),
    ("output", "full", "rpk_select_device", lambda r, s: (s, P, *cols(r), None, None, None), EINVAL),
    ("shard", "full", "rpk_select_device_gather", lambda r, s: (s, P, *cols(r), 2, arr(r.best), 0, None, None), EINVAL),
    ("offers", "bare", "rpk_select_device_gather", lambda r, s: (s, P, *cols(r), 2, arr(r.best), 0, None, None), ESTATE),
    ("output", "full", "rpk_select_device_gather", lambda r, s: (s, P, *cols(r), 2, arr([r.best[0], None]), 0, None, None),
     EINVAL),
    ("shard", "full", "rpk_select_device_gather_top5", lambda r, s: (s, P, *cols(r), 2, arr(r.best), arr(r.top5), 0, None),
     EINVAL),
    ("offers", "bare", "rpk_select_device_gather_top5", lambda r, s: (s, P, *cols(r), 2, arr(r.best), arr(r.top5), 0, None),
     ESTATE),
    ("output", "full", "rpk_select_device_gather_top5",
     lambda r, s: (s, P, *cols(r), 2, arr(r.best), arr([r.top5[0], None]), 0, None), EINVAL),
    ("shard", "full", "rpk_select_slots_device", lambda r, s: (s, P, r.slots, r.best[0], None, None), EINVAL),
    ("pods", "bare", "rpk_select_slots_device", lambda r, s: (s, P, r.slots, r.best[0], None, None), ESTATE),
    ("offers", "pods", "rpk_select_slots_device", lambda r, s: (s, P, r.slots, r.best[0], None, None), ESTATE),
    ("output", "full", "rpk_select_slots_device", lambda r, s: (s, P, r.slots, None, None, None), EINVAL),
    ("shard", "full", "rpk_select_slots_device_gather", lambda r, s: (s, P, r.slots, 2, arr(r.best), 0, None, None), EINVAL),
    ("pods", "bare", "rpk_select_slots_device_gather", lambda r, s: (s, P, r.slots, 2, arr(r.best), 0, None, None), ESTATE),
    ("offers", "pods", "rpk_select_slots_device_gather", lambda r, s: (s, P, r.slots, 2, arr(r.best), 0, None, None),
     ESTATE),
    ("output", "full", "rpk_select_slots_device_gather",
     lambda r, s: (s, P, r.slots, 2, arr([r.best[0], None]), 0, None, None), EINVAL),
    ("shard", "full", "rpk_select_slots_device_gather_top5",
     lambda r, s: (s, P, r.slots, 2, arr(r.best), arr(r.top5), 0, None), EINVAL),
    ("pods", "bare", "rpk_select_slots_device_gather_top5",
     lambda r, s: (s, P, r.slots, 2, arr(r.best), arr(r.top5), 0, None), ESTATE),
    ("offers", "pods", "rpk_select_slots_device_gather_top5",
     lambda r, s: (s, P, r.slots, 2, arr(r.best), arr(r.top5), 0, None), ESTATE),
    ("output", "full", "rpk_select_slots_device_gather_top5",
     lambda r, s: (s, P, r.slots, 2, arr(r.best), arr([r.top5[0], None]), 0, None), EINVAL),
    ("shard", "full", "rpk_pods_pending_list_device", lambda r, s: (s, r.idx, r.n, None), EINVAL),
    ("pods", "bare", "rpk_pods_pending_list_device", lambda r, s: (s, r.idx, r.n, None), ESTATE),
    ("output", "full", "rpk_pods_pending_list_device", lambda r, s: (s, r.idx, None, None), EINVAL),
    ("shard", "full", "rpk_select_pending_changed_gather",
     lambda r, s: (s, 1, 0, arr([r.res_xchg]), P, host(r.n_pending), host(r.n_reselected), None), EINVAL),
    ("pods", "bare", "rpk_select_pending_changed_gather",
     lambda r, s: (s, 1, 0, arr([r.res_xchg]), P, host(r.n_pending), host(r.n_reselected), None), ESTATE),
    ("offers", "pods", "rpk_select_pending_changed_gather",
     lambda r, s: (s, 1, 0, arr([r.res_xchg]), P, host(r.n_pending), host(r.n_reselected), None), ESTATE),
    ("output", "full", "rpk_select_pending_changed_gather",
     lambda r, s: (s, 1, 0, None, P, host(r.n_pending), host(r.n_reselected), None), EINVAL),
    ("shard", "full", "rpk_status_diff_device", lambda r, s: (s, P, r.records, STRIDE, r.hash_prev, r.idx, r.n, None), EINVAL),
    ("output", "full", "rpk_status_diff_device", lambda r, s: (s, P, r.records, STRIDE, r.hash_prev, r.idx, None, None),
     EINVAL),
    ("stride", "full", "rpk_status_diff_device", lambda r, s: (s, P, r.records, 8, r.hash_prev, r.idx, r.n, None), EINVAL),
    ("shard", "full", "rpk_status_diff_device_codes",
     lambda r, s: (s, P, r.records, STRIDE, r.hash_prev, r.idx, r.code, r.n, None), EINVAL),
    ("output", "full", "rpk_status_diff_device_codes",
     lambda r, s: (s, P, r.records, STRIDE, r.hash_prev, r.idx, r.code, None, None), EINVAL),
    ("stride", "full", "rpk_status_diff_device_codes",
     lambda r, s: (s, P, r.records, 8, r.hash_prev, r.idx, r.code, r.n, None), EINVAL),
    ("shard", "full", "rpk_status_diff_slots_device",
     lambda r, s: (s, P, 0, P, r.slots, r.records, STRIDE, r.hash_prev, r.idx, r.code, r.n, None), EINVAL),
    ("output", "full", "rpk_status_diff_slots_device",
     lambda r, s: (s, P, 0, P, r.slots, r.records, STRIDE, r.hash_prev, r.idx, r.code, None, None), EINVAL),
    ("stride", "full", "rpk_status_diff_slots_device",
     lambda r, s: (s, P, 0, P, r.slots, r.records, 8, r.hash_prev, r.idx, r.code, r.n, None), EINVAL),
    ("shard", "full", "rpk_status_diff_device_gather",
     lambda r, s: (s, P, r.records, STRIDE, r.hash_prev, 0, 2, arr(r.xchg), P, 0, r.n, None), EINVAL),
    ("output", "full", "rpk_status_diff_device_gather",
     lambda r, s: (s, P, r.records, STRIDE, r.hash_prev, 0, 2, arr([r.xchg[0], None]), P, 0, r.n, None), EINVAL),
    ("stride", "full", "rpk_status_diff_device_gather",
     lambda r, s: (s, P, r.records, 8, r.hash_prev, 0, 2, arr(r.xchg), P, 0, r.n, None), EINVAL),
    ("shard", "full", "rpk_status_diff_slots_device_gather",
     lambda r, s: (s, P, 0, P, r.slots, r.records, STRIDE, r.hash_prev, 2, arr(r.xchg), P, 0, r.n, None), EINVAL),
    ("output", "full", "rpk_status_diff_slots_device_gather",
     lambda r, s: (s, P, 0, P, r.slots, r.records, STRIDE, r.hash_prev, 2, arr([r.xchg[0], None]), P, 0, r.n, None), EINVAL),
    ("stride", "full", "rpk_status_diff_slots_device_gather",
     lambda r, s: (s, P, 0, P, r.slots, r.records, 8, r.hash_prev, 2, arr(r.xchg), P, 0, r.n, None), EINVAL),
    ("shard", "full", "rpk_peer_fence", lambda r, s: (s, 2, arr([r.idx, r.idx]), 0, 1, None), EINVAL),
    ("output", "full", "rpk_peer_fence", lambda r, s: (s, 2, arr([r.idx, None]), 0, 1, None), EINVAL),
    ("shard", "full", "rpk_peer_wait", lambda r, s: (s, 1, None), EINVAL),
    ("stride", "full", "rpk_status_seed", lambda r, s: (P, r.host_records.ctypes.data, 8), EINVAL),
]


@pytest.mark.parametrize("fault,kind,fn,args,code", CASES, ids=[f"{c[2]}-{c[0]}-{c[1]}" for c in CASES])
def test_refusal_names_the_call_and_enqueues_nothing(rig, fault, kind, fn, args, code):
    import torch

    eng = rig.engines[kind]
    shard = 1 if fault == "shard" else 0
    torch.cuda.synchronize()
    flags0 = rig.flags[kind].cpu().numpy().copy()
    c0 = eng.launch_count()
    rc = getattr(eng._lib, fn)(eng._ctx, *args(rig, shard))
    msg = (eng._lib.rpk_last_error(eng._ctx) or b"").decode()
    assert rc == code, (fn, fault, rc, msg)
    assert msg.startswith(fn + ":"), (fn, fault, msg)
    assert eng.launch_count() == c0, f"{fn} ({fault}): launched"
    torch.cuda.synchronize()
    assert np.array_equal(rig.flags[kind].cpu().numpy(), flags0), f"{fn} ({fault}): signalled"
