"""``Engine`` -- thin Python host wrapper over the C-ABI (``include/rpk.h``).

It adds nothing to the computation: numpy columns in (host entry points) or torch CUDA tensors in (device
entry points), the C library does the rest on the GPU.  Method names follow the reference's vocabulary:
``upload_offers`` replaces the per-pod GraphQL decode of ``gpuTypes`` (runpod_client.go:447-455), ``select``
replaces the body of ``GetGPUTypes`` (:465-509) for a whole batch of pods, ``status_diff`` replaces the diff
predicate of ``updateAllPodStatuses`` (kubelet.go:857-880).
"""
from __future__ import annotations

import ctypes as C
import functools

import numpy as np

from . import _ffi

# torch dtypes each device argument accepts; the kernels read and write exactly this element width
_DEV_DTYPES = {
    "req_mem_gb": ("int32",), "req_vcpu": ("int32",), "req_ram_gb": ("int32",), "max_price": ("float64",),
    "cloud": ("uint8",), "d_best": ("int32",), "d_top5": ("int32",), "d_records": ("uint8",),
    "d_hash_prev": ("int64", "uint64"), "d_changed_idx": ("int32", "uint32"), "d_changed_code": ("int16", "uint16"),
    "d_n_changed": ("int32", "uint32"), "d_slots": ("int32", "uint32"),
}


@functools.cache
def _dev_dtypes(name):
    import torch

    return tuple(getattr(torch, d) for d in _DEV_DTYPES[name])


def _np_ptr(a, dtype, n=None, name="array"):
    if a is None:
        return None
    if not isinstance(a, np.ndarray) or a.dtype != dtype or not a.flags.c_contiguous:
        raise TypeError(f"{name}: expected a C-contiguous numpy array of {np.dtype(dtype).name}")
    if n is not None and a.size != n:
        raise ValueError(f"{name}: expected {n} elements, got {a.size}")
    return C.c_void_p(a.ctypes.data)


def _ptr_array(ptrs):
    """raw device pointers (None: none) -> (count, void*[] holding them) for the C side's pointer-array parameters"""
    ptrs = [int(p) for p in ptrs or ()]
    return len(ptrs), (C.c_void_p * max(len(ptrs), 1))(*ptrs)


def _changed_list(cap: int, want_codes: bool):
    """Host outputs of a changed list of capacity ``cap`` -> (changed_idx, changed_code | None, n_changed) pointers for
    the C call, and a function returning (indices, codes | None) trimmed to the count the call wrote."""
    idx = np.empty(max(cap, 1), np.uint32)
    codes = np.empty(max(cap, 1), np.uint16) if want_codes else None
    n = C.c_uint32(0)
    ptrs = (C.c_void_p(idx.ctypes.data), C.c_void_p(codes.ctypes.data) if want_codes else None, C.cast(C.byref(n), C.c_void_p))
    return ptrs, lambda: (idx[: n.value].copy(), codes[: n.value].copy() if want_codes else None)


class Engine:
    """One ``rpk_ctx``.  ``n_gpus > 1`` = one process driving several GPUs (the Go kubelet's shape)."""

    def __init__(self, n_gpus: int = 1, device_ids=None):
        self._lib = _ffi.load()
        self._ctx = C.c_void_p()
        ids = None
        if device_ids is not None:
            ids = (C.c_int * len(device_ids))(*device_ids)
            n_gpus = len(device_ids)
        rc = self._lib.rpk_create(n_gpus, ids, C.byref(self._ctx))
        if rc != 0:
            msg = self._lib.rpk_last_error(None)
            self._ctx = C.c_void_p()
            raise _ffi.RpkError(rc, (msg or b"").decode())
        self.n_gpus = n_gpus
        self.device_ids = list(device_ids) if device_ids is not None else list(range(n_gpus))  # as rpk_create reads NULL
        self.G = 0

    # -- plumbing ------------------------------------------------------------------------------------
    def _check(self, rc: int):
        if rc != 0:
            raise _ffi.RpkError(rc, (self._lib.rpk_last_error(self._ctx) or b"").decode())

    def _device(self, shard: int):
        """CUDA device id of ``shard``; None for a shard out of range, which the C side refuses (RPK_EINVAL)"""
        return self.device_ids[shard] if 0 <= shard < self.n_gpus else None

    def _stream(self, stream, shard: int):
        """``stream`` as given, else torch's current stream on the shard's GPU (its default stream, 0, is passed as
        cudaStreamLegacy = 1: a NULL stream would select the ctx's own stream)"""
        if stream is not None:
            return C.c_void_p(stream)
        import torch

        return C.c_void_p(torch.cuda.current_stream(self._device(shard)).cuda_stream or 1)

    def _dev_ptr(self, t, name: str, shard: int, n=None, at_least=None):
        """torch tensor for device argument ``name`` (None passes as NULL) -> raw device pointer; torch is only the
        allocator here.  The C side sees nothing but the pointer, so everything that would make a kernel fault or write
        out of bounds is refused here: a tensor that is not CUDA, not on the shard's GPU, of a dtype ``name`` does not
        accept, or not contiguous (TypeError), or that does not hold exactly ``n`` / at least ``at_least`` elements
        (ValueError).  Alignment is left to the C side, which refuses a misaligned view with RPK_EINVAL."""
        if t is None:
            return None
        if not t.is_cuda:
            raise TypeError(f"{name}: expected a CUDA tensor, got one on {t.device}")
        dev = self._device(shard)
        if dev is not None and t.device.index != dev:
            raise TypeError(f"{name}: expected a tensor on cuda:{dev} (shard {shard}), got one on {t.device}")
        if t.dtype not in _dev_dtypes(name):
            raise TypeError(f"{name}: expected a tensor of {' or '.join(_DEV_DTYPES[name])}, got {t.dtype}")
        if not t.is_contiguous():
            raise TypeError(f"{name}: expected a contiguous tensor")
        k = t.numel()
        if n is not None and k != n:
            raise ValueError(f"{name}: expected {n} elements, got {k}")
        if at_least is not None and k < at_least:
            raise ValueError(f"{name}: expected at least {at_least} elements, got {k}")
        return C.c_void_p(t.data_ptr())

    def _dev_pods(self, pods: dict, shard: int):
        """device pod columns -> (P, pointers of req_mem_gb, req_vcpu, req_ram_gb, max_price, cloud)"""
        P = int(pods["req_mem_gb"].numel())
        return P, [self._dev_ptr(pods.get(k), k, shard, P) for k in ("req_mem_gb", "req_vcpu", "req_ram_gb", "max_price", "cloud")]

    def close(self):
        if getattr(self, "_ctx", None) is not None and self._ctx.value:
            self._lib.rpk_destroy(self._ctx)
            self._ctx = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()

    def stats(self) -> dict:
        s = _ffi.RpkStats()
        self._check(self._lib.rpk_stats_get(self._ctx, C.byref(s)))
        return {k: getattr(s, k) for k, _ in s._fields_}

    def launch_count(self) -> int:
        return int(self._lib.rpk_launch_count(self._ctx))

    # -- offers --------------------------------------------------------------------------------------
    def upload_offers(self, offers: dict):
        G = int(offers["mem_gb"].shape[0])
        self._check(self._lib.rpk_offers_upload(
            self._ctx, G, _np_ptr(offers["mem_gb"], np.int32, G, "mem_gb"), _np_ptr(offers.get("vcpu"), np.int32, G, "vcpu"),
            _np_ptr(offers.get("ram_gb"), np.int32, G, "ram_gb"), _np_ptr(offers["secure_price"], np.float64, G, "secure_price"),
            _np_ptr(offers["community_price"], np.float64, G, "community_price"), _np_ptr(offers["flags"], np.uint8, G, "flags")))
        self.G = G

    # -- selection -----------------------------------------------------------------------------------
    def select(self, pods: dict, want_top5: bool = False, out_best=None, out_top5=None):
        """Host columns in, ``(best[P], top5[P,5] | None)`` out (numpy)."""
        P = int(pods["req_mem_gb"].shape[0])
        best = out_best if out_best is not None else np.empty(P, np.int32)
        top5 = (out_top5 if out_top5 is not None else np.empty((P, 5), np.int32)) if want_top5 else None
        self._check(self._lib.rpk_select(
            self._ctx, P, _np_ptr(pods["req_mem_gb"], np.int32, P, "req_mem_gb"), _np_ptr(pods.get("req_vcpu"), np.int32, P, "req_vcpu"),
            _np_ptr(pods.get("req_ram_gb"), np.int32, P, "req_ram_gb"), _np_ptr(pods.get("max_price"), np.float64, P, "max_price"),
            _np_ptr(pods.get("cloud"), np.uint8, P, "cloud"), _np_ptr(best, np.int32, P, "best"),
            _np_ptr(top5, np.int32, P * 5, "top5") if top5 is not None else None))
        return best, top5

    # -- pod-requirement table: selection over slot lists -----------------------------------------------
    def pods_reset(self, N: int):
        """(Re)size the pod table to N slots, every row the columns of a pod with no annotations (rpk_pods_reset)."""
        self._check(self._lib.rpk_pods_reset(self._ctx, N))

    def pods_seed_slots(self, slots: np.ndarray, pods: dict):
        """Row slots[i] := row i of the host columns ``pods`` (as ``select`` takes them; slots strictly ascending)."""
        n = int(pods["req_mem_gb"].shape[0])
        slots = np.ascontiguousarray(slots, np.uint32)  # keep the converted array alive across the call
        self._check(self._lib.rpk_pods_seed_slots(
            self._ctx, n, _np_ptr(slots, np.uint32, n, "slots"), _np_ptr(pods["req_mem_gb"], np.int32, n, "req_mem_gb"),
            _np_ptr(pods.get("req_vcpu"), np.int32, n, "req_vcpu"), _np_ptr(pods.get("req_ram_gb"), np.int32, n, "req_ram_gb"),
            _np_ptr(pods.get("max_price"), np.float64, n, "max_price"), _np_ptr(pods.get("cloud"), np.uint8, n, "cloud")))

    def select_slots(self, slots: np.ndarray, want_top5: bool = False, out_best=None, out_top5=None):
        """``select`` over rows of the pod table: ``(best[n], top5[n,5] | None)`` for the rows held at ``slots`` (any
        order, repeats allowed)."""
        slots = np.ascontiguousarray(slots, np.uint32)  # keep the converted array alive across the call
        n = int(slots.size)
        best = out_best if out_best is not None else np.empty(n, np.int32)
        top5 = (out_top5 if out_top5 is not None else np.empty((n, 5), np.int32)) if want_top5 else None
        self._check(self._lib.rpk_select_slots(
            self._ctx, n, _np_ptr(slots, np.uint32, n, "slots"), _np_ptr(best, np.int32, n, "best"),
            _np_ptr(top5, np.int32, n * 5, "top5") if top5 is not None else None))
        return best, top5

    def select_device(self, pods: dict, d_best, d_top5=None, shard: int = 0, stream=None):
        """torch CUDA columns in, result enqueued on ``stream`` (default: torch's current stream on the shard's GPU)."""
        P, cols = self._dev_pods(pods, shard)
        self._check(self._lib.rpk_select_device(
            self._ctx, shard, P, *cols, self._dev_ptr(d_best, "d_best", shard, P), self._dev_ptr(d_top5, "d_top5", shard, P * 5),
            self._stream(stream, shard)))

    def select_device_gather(self, pods: dict, full_ptrs, row0: int, d_top5=None, shard: int = 0, stream=None, top5_ptrs=None):
        """Shard + fused all-gather: results land at [row0, row0+P) of every vector in ``full_ptrs`` (raw
        device pointers: own vector first or anywhere, peers' via IPC / peer access).  ``top5_ptrs`` (one per vector of
        ``full_ptrs``, one of them on the shard's GPU) gathers the gpuTypeIds lists too: elements [5*row0, 5*(row0+P)) of
        every one of them (rpk_select_device_gather_top5); ``d_top5`` keeps the lists local instead."""
        P, cols = self._dev_pods(pods, shard)
        n_out, outs = _ptr_array(full_ptrs)
        if top5_ptrs is not None:
            if d_top5 is not None:
                raise ValueError("d_top5 and top5_ptrs: pass one (top5_ptrs gathers the lists into every vector)")
            n_t5, t5 = _ptr_array(top5_ptrs)
            if n_t5 != n_out:
                raise ValueError(f"top5_ptrs: expected one vector per vector of full_ptrs ({n_out}), got {n_t5}")
            self._check(self._lib.rpk_select_device_gather_top5(
                self._ctx, shard, P, *cols, n_out, outs, t5, row0, self._stream(stream, shard)))
            return
        self._check(self._lib.rpk_select_device_gather(
            self._ctx, shard, P, *cols, n_out, outs, row0, self._dev_ptr(d_top5, "d_top5", shard, P * 5), self._stream(stream, shard)))

    def select_slots_device(self, d_slots, d_best, d_top5=None, shard: int = 0, stream=None):
        """``select_device`` over rows of the pod table: ``d_best[i]`` (and ``d_top5[5i, 5i+5)``) for the row held at slot
        ``d_slots[i]`` (a torch CUDA tensor on the shard's GPU; any order, repeats allowed; an entry outside the table
        gives -1 and five -1), enqueued on ``stream``."""
        n = int(d_slots.numel())
        self._check(self._lib.rpk_select_slots_device(
            self._ctx, shard, n, self._dev_ptr(d_slots, "d_slots", shard), self._dev_ptr(d_best, "d_best", shard, at_least=n),
            self._dev_ptr(d_top5, "d_top5", shard, at_least=5 * n), self._stream(stream, shard)))

    def select_slots_device_gather(self, d_slots, full_ptrs, row0: int, d_top5=None, shard: int = 0, stream=None, top5_ptrs=None):
        """``select_device_gather`` over rows of the pod table listed in ``d_slots``: the results land at [row0, row0+n)
        of every vector in ``full_ptrs`` and, with ``top5_ptrs``, the lists at [5*row0, 5*(row0+n)) of every one of
        those (rpk_select_slots_device_gather, rpk_select_slots_device_gather_top5)."""
        n = int(d_slots.numel())
        slots = self._dev_ptr(d_slots, "d_slots", shard)
        n_out, outs = _ptr_array(full_ptrs)
        if top5_ptrs is not None:
            if d_top5 is not None:
                raise ValueError("d_top5 and top5_ptrs: pass one (top5_ptrs gathers the lists into every vector)")
            n_t5, t5 = _ptr_array(top5_ptrs)
            if n_t5 != n_out:
                raise ValueError(f"top5_ptrs: expected one vector per vector of full_ptrs ({n_out}), got {n_t5}")
            self._check(self._lib.rpk_select_slots_device_gather_top5(
                self._ctx, shard, n, slots, n_out, outs, t5, row0, self._stream(stream, shard)))
            return
        self._check(self._lib.rpk_select_slots_device_gather(
            self._ctx, shard, n, slots, n_out, outs, row0, self._dev_ptr(d_top5, "d_top5", shard, at_least=5 * n),
            self._stream(stream, shard)))

    # -- cross-process peer vectors (CUDA IPC) ------------------------------------------------------------
    def ipc_alloc(self, nbytes: int, shard: int = 0):
        """-> (device pointer, 64-byte handle) of a fresh cudaMalloc buffer other processes can map."""
        ptr = C.c_void_p()
        handle = C.create_string_buffer(64)
        self._check(self._lib.rpk_ipc_alloc(self._ctx, shard, nbytes, C.byref(ptr), handle))
        return int(ptr.value), handle.raw

    def ipc_open(self, handle: bytes, shard: int = 0) -> int:
        if len(handle) != 64:  # rpk_ipc_open reads 64 bytes
            raise ValueError(f"handle: expected the 64-byte CUDA IPC handle ipc_alloc returns, got {len(handle)} bytes")
        ptr = C.c_void_p()
        self._check(self._lib.rpk_ipc_open(self._ctx, shard, handle, C.byref(ptr)))
        return int(ptr.value)

    def peer_fence(self, flag_ptrs, my_rank: int, epoch: int, shard: int = 0, stream=None):
        """Signal every peer and wait for every peer on ``stream`` (one tiny kernel; see rpk_peer_fence)."""
        n, flags = _ptr_array(flag_ptrs)
        self._check(self._lib.rpk_peer_fence(self._ctx, shard, n, flags, my_rank, epoch & 0xFFFFFFFF, self._stream(stream, shard)))

    def peer_bind(self, flag_ptrs, my_rank: int, shard: int = 0):
        """Bind the peer group's flag arrays: gathers on this shard signal by themselves from now on (rpk_peer_bind)."""
        n, flags = _ptr_array(flag_ptrs)
        self._check(self._lib.rpk_peer_bind(self._ctx, shard, n, flags, my_rank))

    def peer_inline_wait(self, on: bool = True, shard: int = 0):
        """Bound gathers also wait for every peer's signal before they complete (no rpk_peer_wait launch needed)."""
        self._check(self._lib.rpk_peer_inline_wait(self._ctx, shard, 1 if on else 0))

    def peer_wait(self, what: int = 1, shard: int = 0, stream=None):
        """The wait half of the fence (bit 0: select gather, bit 1: status gather)."""
        self._check(self._lib.rpk_peer_wait(self._ctx, shard, what, self._stream(stream, shard)))

    def best_device_ptr(self, shard: int = 0) -> int:
        return int(self._lib.rpk_best_device_ptr(self._ctx, shard) or 0)

    # -- status sweep --------------------------------------------------------------------------------
    def status_reset(self, N: int):
        self._check(self._lib.rpk_status_reset(self._ctx, N))

    def status_seed(self, records: np.ndarray):
        N, stride = records.shape
        self._check(self._lib.rpk_status_seed(self._ctx, N, _np_ptr(records, np.uint8, N * stride, "records"), stride))

    def status_diff(self, records: np.ndarray, want_hashes: bool = False, want_codes: bool = False):
        """-> (changed_idx ascending, hashes | None) or, with ``want_codes``, (changed_idx, codes, hashes | None)"""
        N, stride = records.shape
        out, changed = _changed_list(N, want_codes)
        hashes = np.empty(N, np.uint64) if want_hashes else None
        self._check(self._lib.rpk_status_diff_codes(
            self._ctx, N, _np_ptr(records, np.uint8, N * stride, "records"), stride, *out, _np_ptr(hashes, np.uint64, N, "hashes")))
        idx, codes = changed()
        return (idx, codes, hashes) if want_codes else (idx, hashes)

    def status_seed_slots(self, slots: np.ndarray, records: np.ndarray):
        """Previous state of individual slots (records[i] -> slot slots[i]); nothing is reported."""
        n, stride = records.shape
        slots = np.ascontiguousarray(slots, np.uint32)  # keep the converted array alive across the call
        self._check(self._lib.rpk_status_seed_slots(self._ctx, n, _np_ptr(slots, np.uint32, n, "slots"),
                                                    _np_ptr(records, np.uint8, n * stride, "records"), stride))

    def status_diff_slots(self, slots: np.ndarray, records: np.ndarray, want_codes: bool = False):
        """Diff of the listed slots only (records[i] is this sweep's state of slot slots[i]; slots strictly ascending):
        -> (changed slot ids ascending, codes | None).  Slots not listed are neither compared nor touched."""
        n, stride = records.shape
        slots = np.ascontiguousarray(slots, np.uint32)  # keep the converted array alive across the call
        out, changed = _changed_list(n, want_codes)
        self._check(self._lib.rpk_status_diff_slots(
            self._ctx, n, _np_ptr(slots, np.uint32, n, "slots"), _np_ptr(records, np.uint8, n * stride, "records"), stride, *out))
        return changed()

    def tick(self, pods: dict | None, records: np.ndarray, want_top5: bool = False, want_codes: bool = True, out_best=None):
        """One kubelet tick: selection over ``pods`` (None: none pending) and the status sweep over ``records`` enqueued
        together (rpk_tick).  -> (best | None, top5 | None, changed_idx, codes | None)"""
        N, stride = records.shape
        P = int(pods["req_mem_gb"].shape[0]) if pods else 0
        best = (out_best if out_best is not None else np.empty(P, np.int32)) if P else None
        top5 = np.empty((P, 5), np.int32) if (want_top5 and P) else None
        out, changed = _changed_list(N, want_codes)
        g = (lambda k, dt: _np_ptr(pods.get(k), dt, P, k)) if P else (lambda k, dt: None)
        self._check(self._lib.rpk_tick(
            self._ctx, P, g("req_mem_gb", np.int32), g("req_vcpu", np.int32), g("req_ram_gb", np.int32), g("max_price", np.float64),
            g("cloud", np.uint8), _np_ptr(best, np.int32, P, "best") if P else None, _np_ptr(top5, np.int32, P * 5, "top5") if top5 is not None else None,
            N, _np_ptr(records, np.uint8, N * stride, "records"), stride, *out))
        return (best, top5, *changed())

    def status_diff_device(self, d_records, stride: int, d_hash_prev, d_changed_idx, d_n_changed, shard: int = 0, stream=None,
                           d_changed_code=None):
        N = int(d_hash_prev.numel())
        self._check(self._lib.rpk_status_diff_device_codes(
            self._ctx, shard, N, self._dev_ptr(d_records, "d_records", shard, N * stride), stride,
            self._dev_ptr(d_hash_prev, "d_hash_prev", shard), self._dev_ptr(d_changed_idx, "d_changed_idx", shard, at_least=N),
            self._dev_ptr(d_changed_code, "d_changed_code", shard, at_least=N),
            self._dev_ptr(d_n_changed, "d_n_changed", shard, at_least=1), self._stream(stream, shard)))

    def status_diff_slots_device(self, d_slots, d_records, stride: int, d_hash_prev, d_changed_idx, d_n_changed, idx_base: int = 0,
                                 d_changed_code=None, shard: int = 0, stream=None):
        """Diff of the listed slots against a caller-owned hash column holding global slots [idx_base, idx_base + N)
        (N = d_hash_prev.numel()); entries outside that range are skipped.  Enqueued on ``stream``."""
        N, n = int(d_hash_prev.numel()), int(d_slots.numel())
        self._check(self._lib.rpk_status_diff_slots_device(
            self._ctx, shard, N, idx_base, n, self._dev_ptr(d_slots, "d_slots", shard),
            self._dev_ptr(d_records, "d_records", shard, n * stride), stride, self._dev_ptr(d_hash_prev, "d_hash_prev", shard),
            self._dev_ptr(d_changed_idx, "d_changed_idx", shard, at_least=n),
            self._dev_ptr(d_changed_code, "d_changed_code", shard, at_least=n),
            self._dev_ptr(d_n_changed, "d_n_changed", shard, at_least=1), self._stream(stream, shard)))

    def xchg_bytes(self, n_ranks: int, cap: int) -> int:
        return int(self._lib.rpk_xchg_bytes(n_ranks, cap))

    def status_diff_device_gather(self, d_records, stride: int, d_hash_prev, idx_base: int, xchg_ptrs, cap: int, my_rank: int,
                                  d_n_changed, shard: int = 0, stream=None):
        """Sharded sweep: this rank's changed list (count, global ids, codes) lands in region ``my_rank`` of every
        rank's exchange buffer (rpk_status_diff_device_gather)."""
        N = int(d_hash_prev.numel())
        n_ranks, xchg = _ptr_array(xchg_ptrs)
        self._check(self._lib.rpk_status_diff_device_gather(
            self._ctx, shard, N, self._dev_ptr(d_records, "d_records", shard, N * stride), stride,
            self._dev_ptr(d_hash_prev, "d_hash_prev", shard), idx_base, n_ranks, xchg, cap, my_rank,
            self._dev_ptr(d_n_changed, "d_n_changed", shard, at_least=1), self._stream(stream, shard)))

    def status_diff_slots_device_gather(self, d_slots, d_records, stride: int, d_hash_prev, idx_base: int, xchg_ptrs, cap: int,
                                        my_rank: int, d_n_changed, shard: int = 0, stream=None):
        """Sharded slot-list sweep: the listed slots that lie in this rank's column (global slots [idx_base, idx_base + N),
        N = d_hash_prev.numel()) are compared, and the changed ones (count, global ids in list order, codes) land in
        region ``my_rank`` of every rank's exchange buffer (rpk_status_diff_slots_device_gather)."""
        N, n = int(d_hash_prev.numel()), int(d_slots.numel())
        n_ranks, xchg = _ptr_array(xchg_ptrs)
        self._check(self._lib.rpk_status_diff_slots_device_gather(
            self._ctx, shard, N, idx_base, n, self._dev_ptr(d_slots, "d_slots", shard),
            self._dev_ptr(d_records, "d_records", shard, n * stride), stride, self._dev_ptr(d_hash_prev, "d_hash_prev", shard),
            n_ranks, xchg, cap, my_rank, self._dev_ptr(d_n_changed, "d_n_changed", shard, at_least=1), self._stream(stream, shard)))
