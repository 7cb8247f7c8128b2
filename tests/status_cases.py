"""Status-sweep inputs shared by the CPU and GPU tests: the adversarial corpus for the per-slot code, and seeded
logical tables that can be encoded at any stride for multi-call sequences.

The kernels pick the one known status a record can be from its length (every known status has its own) and then
compare two masked 64-bit lanes, so the strings that can fool them are the near-misses: a known status with one
byte changed at any position, one byte short or long, lower-cased, and unknown strings of a known status's length.
"""
import numpy as np

import rpk

KNOWN = list(rpk.synth.STATUS_SET)
STRIDES = list(range(16, 257, 16))


def status_corpus() -> list:
    out = []
    for s in KNOWN:
        out.append(s)
        for i in range(len(s)):
            for x in (0x01, 0x20):  # neighbouring code point / case flip of that one byte
                out.append(s[:i] + bytes([s[i] ^ x]) + s[i + 1:])
        out += [s[:-1], s[1:], s + b"G", s + b"_", b"X" + s, s.lower(), s.capitalize()]
    # unknown strings with the length of a known one (records of len 8..13), some sharing a known one's first lane
    for n in range(6, 12):
        out += [b"Q" * n, b"PAUSED__"[:n].ljust(n, b"Z"), (b"RUNNING_" * 2)[:n], (b"TERMINA" + b"XXXXX")[:n]]
    out += [b"", b"R", b"X", b"\x7f", b"RUNNINGRUNN"]
    return list(dict.fromkeys(out))


def corpus_records(stride: int):
    """-> (records[n, stride], statuses[n], ports[n], flags[n]): the corpus x ports 0/1 x message flag 0/1"""
    rows, sts, ports, flags = [], [], [], []
    for s in status_corpus():
        for p in (False, True):
            for f in (False, True):
                rows.append(rpk.synth.encode_record(s, p, stride, f))
                sts.append(s)
                ports.append(p)
                flags.append(f)
    return np.ascontiguousarray(np.stack(rows)), sts, np.array(ports), np.array(flags)


def translated_codes(statuses, ports, flags) -> np.ndarray:
    """oracle.translate on the decoded strings; a set flag stands for a statusMessage containing "fail" (kubelet.go:1907)"""
    import oracle

    return np.array([oracle.translate(s.decode("ascii"), "pod failed" if f else "all good", bool(p))
                     for s, p, f in zip(statuses, ports, flags)], np.uint16)


def capacity(stride: int) -> int:
    """longest status a canonical slot of this stride holds (len = chars + 2 <= min(stride - 1, 127))"""
    return min(stride - 1, 127) - 2


def status_pool() -> list:
    """Statuses of every length class a slot can hold: the known and unknown ones, near-misses, and strings on both
    sides of every stride's capacity (13, 29, 45, ..., 125 characters) and of the 32-byte hash stripe, each with a
    twin that differs only in its last byte."""
    pool = KNOWN + list(rpk.synth.UNKNOWN_STATUS) + [b"", b"R", b"RUNNINg", b"TERMINATINH", b"EXITEDX"]
    alphabet = b"ABCDEFGHIJKLMNOPQRSTUVWXYZ_0123456789"
    for n in (12, 13, 14, 20, 23, 24, 29, 30, 31, 45, 46, 61, 62, 63, 77, 78, 93, 94, 109, 110, 124, 125):
        base = bytes(alphabet[(i * 7 + n) % len(alphabet)] for i in range(n))
        pool += [base, base[:-1] + bytes([base[-1] ^ 1])]
    return pool


class LogicalTable:
    """N slots of (status, ports, message flag), drawn from ``status_pool()`` by a seeded generator and encoded as
    canonical records at whatever stride a call uses -- the same logical table at two strides has two encodings."""

    def __init__(self, N: int, rng: np.random.Generator):
        self.pool = status_pool()
        self.lens = np.array([len(s) for s in self.pool])
        self.known = np.arange(len(KNOWN))
        self.rng = rng
        self.N = N
        self.ids = self._draw(N, 16)
        self.ports = rng.random(N) < 0.8
        self.flags = rng.random(N) < 0.3
        self._lut = {}

    def _draw(self, n: int, stride: int) -> np.ndarray:
        fits = np.nonzero(self.lens <= capacity(stride))[0]
        any_fit = fits[self.rng.integers(0, len(fits), n)]
        return np.where(self.rng.random(n) < 0.5, self.known[self.rng.integers(0, len(self.known), n)], any_fit)

    def step(self, stride: int, frac: float) -> None:
        """a fraction of slots take a fresh (status, ports) draw -- every slot whose status does not fit ``stride`` does
        -- and the message flag (not a compared field) moves on about a third of all slots"""
        m = (self.rng.random(self.N) < frac) | (self.lens[self.ids] > capacity(stride))
        k = int(m.sum())
        self.ids[m] = self._draw(k, stride)
        self.ports[m] = self.rng.random(k) < 0.8
        f = self.rng.random(self.N) < 0.3
        self.flags[f] = ~self.flags[f]

    def lut(self, stride: int) -> np.ndarray:
        if stride not in self._lut:
            lut = np.zeros((len(self.pool), 2, 2, stride), np.uint8)
            for i, s in enumerate(self.pool):
                if len(s) <= capacity(stride):
                    for p in (0, 1):
                        for f in (0, 1):
                            lut[i, p, f] = rpk.synth.encode_record(s, bool(p), stride, bool(f))
            self._lut[stride] = lut
        return self._lut[stride]

    def records(self, stride: int, rows=None) -> np.ndarray:
        ids, ports, flags = self.ids, self.ports, self.flags
        if rows is not None:
            ids, ports, flags = ids[rows], ports[rows], flags[rows]
        assert (self.lens[ids] <= capacity(stride)).all()
        return np.ascontiguousarray(self.lut(stride)[ids, ports.astype(np.int64), flags.astype(np.int64)])
