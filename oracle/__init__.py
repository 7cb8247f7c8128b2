"""ctypes loader for the CPU oracle (``rpk_oracle.c``).

TEST INFRASTRUCTURE ONLY -- see the header of ``rpk_oracle.c``.  Importable
from ``tests/``, ``__graft_entry__.smoke()`` and the CPU arms of ``bench.py``;
never from the product package.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_SO = os.path.join(_HERE, "librpk_oracle.so")
_lib = None

CLOUD_SECURE, CLOUD_COMMUNITY, CLOUD_OTHER = 0, 1, 2


def build(force: bool = False) -> str:
    src = os.path.join(_HERE, "rpk_oracle.c")
    if force or not os.path.exists(_SO) or os.path.getmtime(_SO) < os.path.getmtime(src):
        subprocess.check_call(["make", "-C", _HERE, "-s"] + (["-B"] if force else []))
    return _SO


def _p(a, ct):
    return None if a is None else a.ctypes.data_as(C.POINTER(ct))


def lib():
    global _lib
    if _lib is None:
        build()
        L = C.CDLL(_SO)
        L.rpk_oracle_extract_gpu_memory.restype = C.c_int64
        L.rpk_oracle_extract_gpu_memory.argtypes = [C.c_char_p]
        L.rpk_oracle_clamp_i32.restype = C.c_int32
        L.rpk_oracle_clamp_i32.argtypes = [C.c_int64]
        L.rpk_oracle_validate_cloud_type.restype = C.c_int
        L.rpk_oracle_validate_cloud_type.argtypes = [C.c_char_p]
        L.rpk_oracle_annotation_with_fallback.restype = C.c_char_p
        L.rpk_oracle_annotation_with_fallback.argtypes = [C.c_char_p, C.c_char_p, C.c_char_p]
        L.rpk_oracle_xxh64.restype = C.c_uint64
        L.rpk_oracle_xxh64.argtypes = [C.c_char_p, C.c_size_t, C.c_uint64]
        L.rpk_oracle_get_gpu_types.restype = C.c_int
        L.rpk_oracle_select.restype = C.c_int
        L.rpk_oracle_status_diff.restype = C.c_uint32
        L.rpk_oracle_record_hashes.restype = None
        L.rpk_oracle_record_codes.restype = None
        L.rpk_oracle_translate.restype = C.c_uint32
        L.rpk_oracle_translate.argtypes = [C.c_char_p, C.c_char_p, C.c_int]
        _lib = L
    return _lib


def extract_gpu_memory(s: str | None) -> int:
    return int(lib().rpk_oracle_extract_gpu_memory(None if s is None else s.encode()))


def clamp_i32(v: int) -> int:
    return int(lib().rpk_oracle_clamp_i32(v))


def validate_cloud_type(s: str | None) -> int:
    return int(lib().rpk_oracle_validate_cloud_type(None if s is None else s.encode()))


def annotation_with_fallback(pod_val, job_val, default):
    enc = lambda v: None if v is None else v.encode()  # noqa: E731
    out = lib().rpk_oracle_annotation_with_fallback(enc(pod_val), enc(job_val), enc(default))
    return None if out is None else out.decode()


def xxh64(data: bytes, seed: int = 0) -> int:
    return int(lib().rpk_oracle_xxh64(data, len(data), seed))


def _offer_args(offers):
    """offers: dict with mem_gb,i32 / vcpu,i32|None / ram_gb,i32|None / secure_price,f64 / community_price,f64 / flags,u8."""
    G = int(offers["mem_gb"].shape[0])
    return G, [
        C.c_uint32(G),
        _p(offers["mem_gb"], C.c_int32),
        _p(offers.get("vcpu"), C.c_int32),
        _p(offers.get("ram_gb"), C.c_int32),
        _p(offers["secure_price"], C.c_double),
        _p(offers["community_price"], C.c_double),
        _p(offers["flags"], C.c_uint8),
    ]


def get_gpu_types(offers, min_ram: int, max_price: float, cloud: int, req_vcpu: int = 0, req_ram: int = 0):
    """One reference-shaped GetGPUTypes call -> list of <=5 offer indices."""
    _, oa = _offer_args(offers)
    out5 = np.full(5, -1, np.int32)
    k = lib().rpk_oracle_get_gpu_types(*oa, C.c_int64(min_ram), C.c_int32(req_vcpu), C.c_int32(req_ram),
                                       C.c_double(max_price), C.c_int(cloud), _p(out5, C.c_int32))
    if k < 0:
        raise MemoryError("oracle allocation failed")
    return [int(x) for x in out5[:k]]


def select(offers, pods, want_top5: bool = True, n_threads: int = 1):
    """P x G grid, one GetGPUTypes per pod.  pods: dict req_mem_gb / req_vcpu|None / req_ram_gb|None /
    max_price,f64|None / cloud,u8|None.  Returns (best[P], top5[P,5] | None)."""
    _, oa = _offer_args(offers)
    P = int(pods["req_mem_gb"].shape[0])
    best = np.full(P, -2, np.int32)
    top5 = np.full((P, 5), -2, np.int32) if want_top5 else None
    rc = lib().rpk_oracle_select(*oa, C.c_uint32(P), _p(pods["req_mem_gb"], C.c_int32), _p(pods.get("req_vcpu"), C.c_int32),
                                 _p(pods.get("req_ram_gb"), C.c_int32), _p(pods.get("max_price"), C.c_double),
                                 _p(pods.get("cloud"), C.c_uint8), _p(best, C.c_int32), _p(top5, C.c_int32),
                                 C.c_int(n_threads))
    if rc != 0:
        raise MemoryError("oracle allocation failed")
    return best, top5


class StatusTable:
    """Previous-state table of the reference's sweep (Provider.podStatus, kubelet.go:42): per slot the decoded
    (status, ports) pair, compared as string + bool (``rpk_oracle_status_diff``), or "never seen".

    Records are canonical slots of any stride 16..256 (include/rpk.h).  Their prefix does not depend on the stride,
    so one table follows the engine across stride changes: the state is kept at the widest stride seen so far
    (``self.stride``), a wider table copies every slot's bytes into the new width, and narrower records are
    zero-padded to the table's width before they are compared."""

    def __init__(self, N: int, stride: int = 32):
        self.N, self.stride = N, stride
        self.prev = np.zeros((N, stride), np.uint8)
        self.has_prev = np.zeros(N, np.uint8)

    def _fit(self, records: np.ndarray) -> np.ndarray:
        """``records`` at the table's width (the table widens first when the records are wider)"""
        s = records.shape[1]
        assert records.dtype == np.uint8 and records.ndim == 2 and 16 <= s <= 256 and s % 16 == 0
        if s > self.stride:
            wide = np.zeros((self.prev.shape[0], s), np.uint8)
            wide[:, : self.stride] = self.prev
            self.prev, self.stride = wide, s
        if s < self.stride:
            wide = np.zeros((records.shape[0], self.stride), np.uint8)
            wide[:, :s] = records
            return wide
        return np.ascontiguousarray(records)

    def diff(self, records: np.ndarray) -> np.ndarray:
        """rpk_status_diff: ascending changed slots; their state is replaced (kubelet.go:875-880)"""
        assert records.shape[0] == self.N
        recs = self._fit(records)
        idx = np.empty(self.N, np.uint32)
        n = lib().rpk_oracle_status_diff(C.c_uint32(self.N), C.c_uint32(self.stride), _p(recs, C.c_uint8),
                                         _p(self.prev, C.c_uint8), _p(self.has_prev, C.c_uint8), _p(idx, C.c_uint32))
        return idx[:n].copy()

    def seed(self, records: np.ndarray) -> None:
        """rpk_status_seed: every slot's state := its record; nothing is reported"""
        assert records.shape[0] == self.N
        self.prev[:] = self._fit(records)
        self.has_prev[:] = 1

    def seed_slots(self, slots: np.ndarray, records: np.ndarray) -> None:
        """rpk_status_seed_slots: state of slot slots[i] := records[i] (distinct slots); no other slot is touched"""
        slots = np.asarray(slots, np.int64)
        assert records.shape[0] == len(slots) and len(np.unique(slots)) == len(slots)
        assert len(slots) == 0 or (slots.min() >= 0 and slots.max() < self.N)
        self.prev[slots] = self._fit(records)
        self.has_prev[slots] = 1

    def reset(self, N: int) -> None:
        """rpk_status_reset: N slots, none seen (every slot reports on the next diff)"""
        self.N = N
        self.prev = np.zeros((N, self.stride), np.uint8)
        self.has_prev = np.zeros(N, np.uint8)

    def grow(self, N: int) -> None:
        """rpk_status_grow: slots [self.N, N) are appended, never seen; every other slot keeps its state"""
        assert N >= self.N
        prev, has_prev = self.prev, self.has_prev
        self.reset(N)
        self.prev[: len(prev)] = prev
        self.has_prev[: len(has_prev)] = has_prev

    def prev_hashes(self) -> np.ndarray:
        """the device's previous-hash column for this state: the record hash of a seen slot, 0 for a slot never seen"""
        return np.where(self.has_prev != 0, record_hashes(self.prev), np.uint64(0))


def record_hashes(records: np.ndarray) -> np.ndarray:
    N, stride = records.shape
    out = np.empty(N, np.uint64)
    lib().rpk_oracle_record_hashes(C.c_uint32(N), C.c_uint32(stride), _p(records, C.c_uint8), _p(out, C.c_uint64))
    return out


def record_codes(records: np.ndarray) -> np.ndarray:
    """translateRunPodStatus (kubelet.go:1848-2024) of every record, as the code of include/rpk.h."""
    N, stride = records.shape
    out = np.empty(N, np.uint16)
    lib().rpk_oracle_record_codes(C.c_uint32(N), C.c_uint32(stride), _p(records, C.c_uint8), _p(out, C.c_uint16))
    return out


def translate(status: str, message: str, has_exposed_ports: bool) -> int:
    return int(lib().rpk_oracle_translate(status.encode(), message.encode(), int(has_exposed_ports)))
