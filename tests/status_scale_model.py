"""An exact restatement of the status sweep that stays cheap on tables of hundreds of millions of slots, for the scale
tests (test_status_scale_gpu.py).  oracle.StatusTable keeps N x stride bytes of previous records; this keeps one int32
per slot.

A slot holds a KEY, one int32 k = (pool id, ports, flag) = (pool_id * 2 + ports) * 2 + flag, whose canonical record at a
stride is ``lut(stride)[k]`` (the statuses of ``status_cases.status_pool()``: known and unknown ones, near misses, and
twins that differ only in their last byte at every capacity up to 125 characters).  The compared fields of a key are
its CLASS, k >> 1 = (pool id, ports); the message flag is not compared.  Per key the record's hash and code come from
the oracle's own functions (``hashes``, ``codes``).  test_status_scale_model.py asserts that two keys of one stride hash
alike exactly when their classes are equal, so "the hash changed" and "the compared fields changed" are the same thing,
and holds every operation below to oracle.StatusTable.

The state is one int32 per slot: the class of the record last seen, or -1 for a slot never seen."""
import functools

import numpy as np

import oracle
import rpk
from status_cases import capacity, status_pool

POOL = list(dict.fromkeys(status_pool()))
LENS = np.array([len(s) for s in POOL])
K = 4 * len(POOL)  # keys
NEVER = -1


def key(pool_id, ports, flag):
    return ((np.asarray(pool_id, np.int32) * 2 + np.asarray(ports, np.int32)) * 2 + np.asarray(flag, np.int32)).astype(np.int32)


@functools.lru_cache(maxsize=None)
def lut(stride: int) -> np.ndarray:
    """[K, stride] canonical records; the rows of statuses longer than the stride's capacity stay zero (never drawn)"""
    out = np.zeros((K, stride), np.uint8)
    for i, s in enumerate(POOL):
        if len(s) <= capacity(stride):
            for p in (0, 1):
                for f in (0, 1):
                    out[(i * 2 + p) * 2 + f] = rpk.synth.encode_record(s, bool(p), stride, bool(f))
    return out


@functools.lru_cache(maxsize=None)
def fitting_keys(stride: int) -> np.ndarray:
    """the keys whose status fits a slot of this stride, ascending"""
    return np.nonzero(LENS[np.arange(K) >> 2] <= capacity(stride))[0].astype(np.int32)


@functools.lru_cache(maxsize=None)
def hashes(stride: int) -> np.ndarray:
    return oracle.record_hashes(lut(stride))


@functools.lru_cache(maxsize=None)
def codes(stride: int) -> np.ndarray:
    return oracle.record_codes(lut(stride))


# ---- key columns ---------------------------------------------------------------------------------------------------
def draw(rng, n: int, stride: int) -> np.ndarray:
    """n keys that fit the stride: half a known status (the common case), half any fitting key"""
    fit = fitting_keys(stride)
    known = fit[(fit >> 2) < len(rpk.synth.STATUS_SET)]
    out = fit[rng.integers(0, len(fit), n, dtype=np.int32)]
    half = rng.random(n, dtype=np.float32) < 0.5
    out[half] = known[rng.integers(0, len(known), int(half.sum()), dtype=np.int32)]
    return out


def step(rng, keys: np.ndarray, stride: int, frac: float = 0.2, flip: float = 1 / 3) -> np.ndarray:
    """a fraction of slots take a fresh draw, and the flag (not compared) flips on a third of all slots"""
    out = keys.copy()
    m = rng.random(len(keys), dtype=np.float32) < frac
    out[m] = draw(rng, int(m.sum()), stride)
    out[rng.random(len(keys), dtype=np.float32) < flip] ^= 1
    return out


def other_class(keys: np.ndarray, stride: int) -> np.ndarray:
    """for each key, a key of the next fitting class (cyclically), with the same flag: the compared fields differ"""
    fc = np.unique(fitting_keys(stride) >> 1)
    j = np.searchsorted(fc, keys >> 1)
    return (fc[(j + 1) % len(fc)] * 2 + (keys & 1)).astype(np.int32)


def records(keys: np.ndarray, stride: int) -> np.ndarray:
    return lut(stride)[keys]


# ---- the sweep -----------------------------------------------------------------------------------------------------
class Model:
    """The previous-state table of the sweep over N slots (or of a caller-owned hash column of N rows)"""

    def __init__(self, N: int):
        self.state = np.full(N, NEVER, np.int32)

    @property
    def N(self) -> int:
        return len(self.state)

    def reset(self, N: int) -> None:
        self.state = np.full(N, NEVER, np.int32)

    def grow(self, N: int) -> None:
        assert N >= self.N
        self.state = np.concatenate([self.state, np.full(N - self.N, NEVER, np.int32)])

    def seed(self, keys: np.ndarray) -> None:
        assert len(keys) == self.N
        self.state = keys >> 1

    def seed_slots(self, slots, keys: np.ndarray) -> None:
        self.state[np.asarray(slots, np.int64)] = keys >> 1

    def diff(self, keys: np.ndarray, stride: int, idx_base: int = 0, want_hashes: bool = True):
        """-> (changed ids ascending (uint32, slot + idx_base), their codes, the hash column after the sweep | None)"""
        assert len(keys) == self.N
        cls = keys >> 1
        changed = np.flatnonzero(self.state != cls)
        self.state = cls
        ids = (changed + idx_base).astype(np.uint32)
        return ids, codes(stride)[keys[changed]], hashes(stride)[keys] if want_hashes else None

    def diff_slots(self, slots, keys: np.ndarray, stride: int, idx_base: int = 0, col_n: int | None = None):
        """keys[i] is this sweep's state of global slot slots[i] (distinct); the state holds global slots
        [idx_base, idx_base + col_n) (col_n: the whole state).  -> (changed ids in list order (uint32), their codes);
        entries outside the column are skipped."""
        slots = np.asarray(slots, np.uint32)
        assert len(slots) == len(keys)
        col_n = self.N if col_n is None else col_n
        assert col_n <= self.N
        row = slots - np.uint32(idx_base)  # below idx_base wraps around: outside
        inside = np.flatnonzero(row < col_n)
        r = row[inside].astype(np.int64)
        cls = keys[inside] >> 1
        ch = self.state[r] != cls
        self.state[r[ch]] = cls[ch]
        pos = inside[ch]
        return slots[pos], codes(stride)[keys[pos]]

    def column(self) -> np.ndarray:
        """the device's previous-hash column for this state: the hash of the class seen, 0 for a slot never seen (a
        key's hash does not depend on the stride it is encoded at, and every key fits stride 256)"""
        h = hashes(256)[np.maximum(self.state, 0) * 2]
        return np.where(self.state >= 0, h, np.uint64(0))
