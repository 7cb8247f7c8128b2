"""References of rpk_explain (include/rpk.h, rpk_explanation) for the explain tests.

Two independent restatements of the same semantics:
  - ``explain(offers, pods, n_threads)``: the C loop of explain_ref.c (GetGPUTypes' filter loop with its predicate split
    apart, rows split over threads as oracle.select splits them), built with gcc into a temporary directory on first use;
  - ``explain_np(offers, pods)``: a numpy restatement over whole row x offer blocks, which shares no code with it.
Both return the dict ``Engine.explain`` returns.  ``KAT_ROWS`` are the hand-checked rows of the issue's known-answer
table on the offer table of tests/golden/select_kat.json (SURVEY.md 8(c))."""
import ctypes as C
import hashlib
import json
import os
import subprocess
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
WORDS = 14  # uint32 words of one rpk_explanation


def fields(raw):
    """P * 14 uint32 words -> the dict Engine.explain returns"""
    w = raw.reshape(-1, WORDS)
    return {"n_feasible": w[:, 0], "n_unoffered": w[:, 1], "n_fail": w[:, 2:6], "n_only": w[:, 6:10],
            "nearest": w[:, 10:14].view(np.int32)}


def as_words(ex):
    """the dict form -> P * 14 uint32 words (the C structs), for bit-for-bit comparisons"""
    P = len(ex["n_feasible"])
    w = np.empty((P, WORDS), np.uint32)
    w[:, 0], w[:, 1] = ex["n_feasible"], ex["n_unoffered"]
    w[:, 2:6], w[:, 6:10] = ex["n_fail"], ex["n_only"]
    w[:, 10:14] = np.asarray(ex["nearest"], np.int32).view(np.uint32)
    return w.reshape(-1)


_lib = None


def _ref_lib():
    global _lib
    if _lib is None:
        src = os.path.join(HERE, "explain_ref.c")
        tag = hashlib.sha256(open(src, "rb").read()).hexdigest()[:16]
        so = os.path.join(tempfile.gettempdir(), f"rpk_explain_ref_{os.getuid()}_{tag}.so")
        if not os.path.exists(so):
            tmp = f"{so}.{os.getpid()}"
            subprocess.check_call(["gcc", "-O2", "-fPIC", "-Wall", "-Wextra", "-std=c11", "-shared", "-o", tmp, src, "-lpthread"])
            os.replace(tmp, so)
        _lib = C.CDLL(so)
        _lib.explain_ref.restype = C.c_int
    return _lib


def _p(a, ct):
    return None if a is None else np.ascontiguousarray(a).ctypes.data_as(C.POINTER(ct))


def explain(offers, pods, n_threads: int = 1):
    """the C reference over every row of ``pods`` (columns as Engine.explain takes them)"""
    G, P = len(offers["mem_gb"]), len(pods["req_mem_gb"])
    keep = [np.ascontiguousarray(v) if v is not None else None for v in (
        offers["mem_gb"], offers.get("vcpu"), offers.get("ram_gb"), offers["secure_price"], offers["community_price"], offers["flags"],
        pods["req_mem_gb"], pods.get("req_vcpu"), pods.get("req_ram_gb"), pods.get("max_price"), pods.get("cloud"))]
    types = [C.c_int32, C.c_int32, C.c_int32, C.c_double, C.c_double, C.c_uint8, C.c_int32, C.c_int32, C.c_int32, C.c_double, C.c_uint8]
    ptrs = [_p(a, t) for a, t in zip(keep, types)]
    raw = np.full(max(P, 1) * WORDS, 0xA5A5A5A5, np.uint32)
    rc = _ref_lib().explain_ref(C.c_uint32(G), *ptrs[:6], C.c_uint32(P), *ptrs[6:], C.c_void_p(raw.ctypes.data), C.c_int(n_threads))
    if rc != 0:
        raise MemoryError("explain_ref allocation failed")
    return fields(raw[: P * WORDS])


def explain_np(offers, pods, block: int = 1 << 22):
    """numpy restatement: per cloud, the offered offers in (price, index) order; per block of rows, the four failure
    masks over them; nearest[r] = the first column of that order failing r alone"""
    G, P = len(offers["mem_gb"]), len(pods["req_mem_gb"])
    zero = np.zeros(P, np.int32)
    rm = np.asarray(pods["req_mem_gb"], np.int64)
    rv = np.asarray(pods.get("req_vcpu") if pods.get("req_vcpu") is not None else zero, np.int64)
    rr = np.asarray(pods.get("req_ram_gb") if pods.get("req_ram_gb") is not None else zero, np.int64)
    mx = np.asarray(pods.get("max_price") if pods.get("max_price") is not None else np.full(P, 0.5), np.float64)
    cl = np.asarray(pods.get("cloud") if pods.get("cloud") is not None else np.zeros(P, np.uint8), np.uint8)
    om = np.asarray(offers["mem_gb"], np.int64)
    ov = np.asarray(offers.get("vcpu") if offers.get("vcpu") is not None else np.zeros(G, np.int32), np.int64)
    orr = np.asarray(offers.get("ram_gb") if offers.get("ram_gb") is not None else np.zeros(G, np.int32), np.int64)
    out = {"n_feasible": np.zeros(P, np.uint32), "n_unoffered": np.full(P, G, np.uint32),
           "n_fail": np.zeros((P, 4), np.uint32), "n_only": np.zeros((P, 4), np.uint32), "nearest": np.full((P, 4), -1, np.int32)}
    for c, (bit, price_col) in enumerate(((1, "secure_price"), (2, "community_price"))):
        price = np.asarray(offers[price_col], np.float64)
        offered = ((np.asarray(offers["flags"]) & bit) != 0) & (price > 0)
        idx = np.nonzero(offered)[0]
        idx = idx[np.lexsort((idx, price[idx]))]  # price order, ties by offer index
        rows = np.nonzero(cl == c)[0]
        if not len(rows):
            continue
        out["n_unoffered"][rows] = G - len(idx)
        step = max(1, block // max(len(idx), 1))
        for b0 in range(0, len(rows), step):
            r = rows[b0:b0 + step]
            fail = np.stack([~(price[idx][None, :] < mx[r, None]), om[idx][None, :] < rm[r, None],
                             ov[idx][None, :] < rv[r, None], orr[idx][None, :] < rr[r, None]])  # [4, rows, offers]
            nf = fail.sum(axis=0)
            out["n_feasible"][r] = (nf == 0).sum(axis=1)
            out["n_fail"][r] = fail.sum(axis=2).T
            only = fail & (nf == 1)[None]
            out["n_only"][r] = only.sum(axis=2).T
            if len(idx):
                first = only.argmax(axis=2)
                out["nearest"][r] = np.where(only.any(axis=2), idx[first], -1).T
    return out


def kat_offers():
    """the ten offers of SURVEY.md 8(c) (tests/golden/select_kat.json), index = position"""
    rows = json.load(open(os.path.join(HERE, "golden", "select_kat.json")))["offers"]
    return {"mem_gb": np.array([o["memGb"] for o in rows], np.int32), "vcpu": None, "ram_gb": None,
            "secure_price": np.array([o["securePrice"] for o in rows], np.float64),
            "community_price": np.array([o["communityPrice"] for o in rows], np.float64),
            "flags": np.array([int(o["secureCloud"]) | int(o["communityCloud"]) << 1 for o in rows], np.uint8)}


KAT_IDS = [o["id"] for o in json.load(open(os.path.join(HERE, "golden", "select_kat.json")))["offers"]]

# ((req_mem_gb, max_price, cloud), n_feasible, n_unoffered, n_fail, n_only, nearest)
KAT_ROWS = [
    ((80, 0.5, 0), 0, 2, [3, 7, 0, 0], [1, 5, 0, 0], [6, 0, -1, -1]),
    ((24, 0.2, 1), 0, 3, [5, 2, 0, 0], [5, 2, 0, 0], [1, 0, -1, -1]),
    ((16, 0.5, 0), 5, 2, [3, 0, 0, 0], [3, 0, 0, 0], [9, -1, -1, -1]),
    ((16, 0.5, 2), 0, 10, [0, 0, 0, 0], [0, 0, 0, 0], [-1, -1, -1, -1]),
]


def kat_pods():
    return {"req_mem_gb": np.array([k[0][0] for k in KAT_ROWS], np.int32), "req_vcpu": None, "req_ram_gb": None,
            "max_price": np.array([k[0][1] for k in KAT_ROWS], np.float64), "cloud": np.array([k[0][2] for k in KAT_ROWS], np.uint8)}


def kat_expected():
    return {"n_feasible": np.array([k[1] for k in KAT_ROWS], np.uint32), "n_unoffered": np.array([k[2] for k in KAT_ROWS], np.uint32),
            "n_fail": np.array([k[3] for k in KAT_ROWS], np.uint32), "n_only": np.array([k[4] for k in KAT_ROWS], np.uint32),
            "nearest": np.array([k[5] for k in KAT_ROWS], np.int32)}


def assert_same(got, want, label=""):
    """bit-for-bit equality of two explanations, with the first differing row in the message"""
    a, b = as_words(got).reshape(-1, WORDS), as_words(want).reshape(-1, WORDS)
    assert a.shape == b.shape, f"{label}: {a.shape} rows != {b.shape}"
    bad = np.nonzero((a != b).any(axis=1))[0]
    assert not len(bad), f"{label}: {len(bad)} rows differ, first row {bad[0]}: got {a[bad[0]].view(np.int32)}, want {b[bad[0]].view(np.int32)}"
