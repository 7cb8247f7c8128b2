#!/usr/bin/env python
"""Select by slot list (rpk_select_slots) against the select from host columns (rpk_select), on the GPU.

    python tools/select_slots_probe.py [--out profiles/h100_select_slots.json] [--runs 25]

One H100, G = 100k offers (synth.make_offers(100_000)), a tracked pod table of N = 1M slots seeded with
synth.make_pods(1M).  For P pending pods in {4096, 125k, 1M} -- the first P slots, and a random ascending subset of P
slots (one list at 1M: every slot) -- and with and without the top-5 lists, three arms are alternated in one run:
  columns          rpk_select from pinned host columns (rpk_host_alloc) holding the P rows: 21 bytes up per row
  slots            rpk_select_slots from a pinned slot list: 4 bytes up per row
  slots_unchecked  the same call in a copy of the library built (in a temporary directory, from the objects build()
                   left and rpk_api.cu compiled with -DRPK_MEASURE_UNCHECKED_SLOTS) without the host range check of
                   each sub-batch's part of the list: slots - slots_unchecked is what the check costs the call
Wall clock around each call (every arm ends in a stream synchronise); 5 warm-up calls per arm, then the median [min, max]
of the runs.  The arms' outputs are compared in the same run.  At 125k and 1M rows (random subset, top-5) one more call
of each arm runs under torch.profiler, and its kernel and copy timeline is stored with the row.  The card's name and
power limit are read through NVML (nvidia-smi if pynvml is missing) in the same run, and the SM clock right after each
row's timed calls."""
import argparse
import ctypes as C
import json
import os
import re
import shutil
import statistics
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import rpk  # noqa: E402

N = 1 << 20
G = 100_000
COLS = (("req_mem_gb", np.int32), ("req_vcpu", np.int32), ("req_ram_gb", np.int32), ("max_price", np.float64), ("cloud", np.uint8))


def _nvml():
    import pynvml as nv

    nv.nvmlInit()
    return nv, nv.nvmlDeviceGetHandleByIndex(0)


def _smi(fields):
    out = subprocess.run(["nvidia-smi", f"--query-gpu={fields}", "--format=csv,noheader,nounits", "-i", "0"],
                         capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    return [x.strip() for x in out.split(",")]


def card():
    try:
        nv, h = _nvml()
        name = nv.nvmlDeviceGetName(h)
        return {"name": name.decode() if isinstance(name, bytes) else name,
                "power_limit_w": nv.nvmlDeviceGetPowerManagementLimit(h) / 1000.0, "source": "nvml"}
    except Exception:
        name, limit = _smi("name,power.limit")
        return {"name": name, "power_limit_w": float(limit), "source": "nvidia-smi"}


def sm_clock():
    try:
        nv, h = _nvml()
        return nv.nvmlDeviceGetClockInfo(h, nv.NVML_CLOCK_SM)
    except Exception:
        return float(_smi("clocks.sm")[0])


def build_unchecked(tmp):
    """librpk.so without the host range check of rpk_select_slots: rpk_api.cu compiled with the flags of csrc/Makefile
    plus -DRPK_MEASURE_UNCHECKED_SLOTS, linked with the other objects build() left in build/"""
    csrc = os.path.join(ROOT, "k8s-runpod-kubelet_b200", "csrc")
    mk = open(os.path.join(csrc, "Makefile")).read()

    def var(k):
        return re.search(rf"^{k} [:?]?= (.*)$", mk, re.M).group(1)

    arch = var("ARCH").split()
    flags = var("NVCCFLAGS").replace("$(ARCH)", var("ARCH")).split()
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    objs = []
    for src in var("SRCS").split():
        if src == "rpk_api.cu":
            obj = os.path.join(tmp, "rpk_api_unchecked.o")
            subprocess.check_call([nvcc, *flags, "-DRPK_MEASURE_UNCHECKED_SLOTS", "-c", src, "-o", obj], cwd=csrc)
        else:
            obj = os.path.join(csrc, "..", "build", src[:-3] + ".o")
        objs.append(obj)
    lib = os.path.join(tmp, "librpk_unchecked.so")
    subprocess.check_call([nvcc, *arch, "-shared", "-o", lib, *objs, "-lcudart_static", "-lpthread", "-ldl", "-lrt"])
    return lib


def engine_on(path):
    """an rpk.Engine on cuda:0 whose calls go to the library at `path` (same C-ABI)"""
    L = C.CDLL(path)
    for name, (restype, argtypes) in rpk._ffi.ABI.items():
        fn = getattr(L, name)
        fn.restype, fn.argtypes = restype, argtypes
    eng = rpk.Engine.__new__(rpk.Engine)
    eng._lib, eng._ctx, eng.n_gpus, eng.device_ids, eng.G = L, C.c_void_p(), 1, [0], 0
    eng._check(L.rpk_create(1, None, C.byref(eng._ctx)))
    return eng


class Pinned:
    """numpy arrays over pinned host memory from rpk_host_alloc"""

    def __init__(self):
        self.lib = rpk._ffi.load()
        self.ptrs = []

    def array(self, n, dtype):
        nbytes = max(int(n) * np.dtype(dtype).itemsize, 1)
        p = self.lib.rpk_host_alloc(nbytes)
        assert p, "rpk_host_alloc failed"
        self.ptrs.append(p)
        return np.frombuffer((C.c_uint8 * nbytes).from_address(p), dtype=dtype, count=int(n))

    def free(self):
        for p in self.ptrs:
            self.lib.rpk_host_free(p)
        self.ptrs = []


def stat(ts):
    return {"median": statistics.median(ts), "min": min(ts), "max": max(ts)}


def timeline(fn):
    """the kernels and copies of one call of fn (torch.profiler, a run of its own after the timed runs): name, stream,
    start and duration in microseconds from the first event"""
    import torch
    from torch.profiler import ProfilerActivity, profile

    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "trace.json")
        prof.export_chrome_trace(path)
        with open(path) as f:
            evs = json.load(f)["traceEvents"]
    evs = [e for e in evs if e.get("cat") in ("kernel", "gpu_memcpy") and "dur" in e]
    t0 = min((e["ts"] for e in evs), default=0)
    return [{"name": e["name"][:48], "stream": e.get("args", {}).get("stream"), "start_us": round(e["ts"] - t0, 1),
             "dur_us": round(e["dur"], 1)} for e in sorted(evs, key=lambda e: e["ts"])]


ARMS = ("columns", "slots", "slots_unchecked")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "h100_select_slots.json"))
    ap.add_argument("--runs", type=int, default=25)
    a = ap.parse_args()
    import torch

    if not torch.cuda.is_available():
        raise SystemExit("select_slots_probe: no GPU (numbers here are only measured on the device)")
    gpu = card()
    offers = rpk.synth.make_offers(G)
    pods = rpk.synth.make_pods(N)
    pin = Pinned()
    rows = []
    tmp = tempfile.TemporaryDirectory()
    eng = rpk.Engine(1)
    raw = engine_on(build_unchecked(tmp.name))
    try:
        for e in (eng, raw):
            e.upload_offers(offers)
            e.pods_reset(N)
            e.pods_seed_slots(np.arange(N, dtype=np.uint32), pods)
        rng = np.random.default_rng(17)
        for P in (4096, 125_000, N):
            for subset in (("every slot",) if P == N else ("first P", "random ascending")):
                sl = np.arange(P, dtype=np.uint32) if subset != "random ascending" else np.sort(rng.choice(N, P, replace=False)).astype(np.uint32)
                h_slots = pin.array(P, np.uint32)
                h_slots[:] = sl
                h_cols = {}
                for k, dt in COLS:
                    h_cols[k] = pin.array(P, dt)
                    h_cols[k][:] = pods[k][sl]
                for top5 in (True, False):
                    outs = {arm: (pin.array(P, np.int32), pin.array(P * 5, np.int32).reshape(P, 5) if top5 else None) for arm in ARMS}
                    calls = {"columns": lambda: eng.select(h_cols, want_top5=top5, out_best=outs["columns"][0], out_top5=outs["columns"][1]),
                             "slots": lambda: eng.select_slots(h_slots, want_top5=top5, out_best=outs["slots"][0], out_top5=outs["slots"][1]),
                             "slots_unchecked": lambda: raw.select_slots(h_slots, want_top5=top5, out_best=outs["slots_unchecked"][0],
                                                                         out_top5=outs["slots_unchecked"][1])}
                    ts = {arm: [] for arm in ARMS}
                    for i in range(a.runs + 5):
                        for arm in ARMS[i % 3:] + ARMS[:i % 3]:  # each arm first, second and third in turn
                            t0 = time.perf_counter()
                            calls[arm]()
                            t1 = time.perf_counter()
                            if i >= 5:
                                ts[arm].append((t1 - t0) * 1e3)
                        for arm in ARMS[1:]:
                            assert np.array_equal(outs["columns"][0], outs[arm][0]), (arm, P, subset, top5, i)
                            if top5:
                                assert np.array_equal(outs["columns"][1], outs[arm][1]), (arm, P, subset, top5, i)
                    clock = sm_clock()
                    st = {arm: stat(ts[arm]) for arm in ARMS}
                    c, s, u = st["columns"], st["slots"], st["slots_unchecked"]
                    row = {"P": P, "subset": subset, "top5": top5, "columns_ms": c, "slots_ms": s, "slots_unchecked_ms": u,
                           "range_check_ms_median": s["median"] - u["median"],
                           "upload_bytes": {"columns": 21 * P, "slots": 4 * P}, "speedup_median": c["median"] / s["median"],
                           "speedup_unchecked_median": c["median"] / u["median"],
                           "outside_spread": s["max"] < c["min"] or c["max"] < s["min"],
                           "unchecked_outside_spread": u["max"] < c["min"] or c["max"] < u["min"],
                           "outputs_identical": True, "sm_clock_mhz_after_timed_runs": clock}
                    if P >= 125_000 and top5 and subset != "first P":
                        row["timeline"] = {arm: timeline(calls[arm]) for arm in ARMS}
                    rows.append(row)
                    print(json.dumps({k: v for k, v in row.items() if k != "timeline"}), flush=True)
    finally:
        eng.close()
        raw.close()
        pin.free()
        tmp.cleanup()
    out = {"tool": "tools/select_slots_probe.py", "gpu": gpu, "G": G, "tracked_N": N, "runs": a.runs,
           "timing": "wall clock around each call (ends in a stream synchronise), arms rotated, 5 warm-up calls per arm, "
                     "median [min, max] of the runs", "rows": rows}
    os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
    with open(a.out, "w") as f:
        json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
