#!/usr/bin/env python
"""Select over the pending set kept on the device (rpk_select_pending) against the select by slot list
(rpk_select_slots) and the select from host columns (rpk_select), on the GPU.

    python tools/select_pending_probe.py [--out profiles/h100_select_pending.json] [--runs 25]

One H100, G = 100k offers, a pod table of N = 1M slots seeded with synth.make_pods(1M), as tools/select_slots_probe.py.
For P pending pods in {4096, 125k, 1M} -- the first P slots, and a random ascending subset (one set at 1M: every slot)
-- and with and without the top-5 lists, these arms are alternated in one run:
  columns            rpk_select from pinned host columns holding the P rows: 21 bytes up per row
  slots              rpk_select_slots from a pinned slot list: 4 bytes up per row, checked on the host
  pending            rpk_select_pending with slots_out: nothing up; the list is built on the device and copied back
  pending_nolist     rpk_select_pending without slots_out
  pending_one_select (1M only) pending in a copy of the library built, in a temporary directory, with
  pending_one_select_nolist  -DRPK_MEASURE_PENDING_ONE_SELECT: one select over the whole list instead of the row
                     sub-batches of the host pipeline
Wall clock around each call (every arm ends in a synchronise); 5 warm-up calls per arm, then the median [min, max] of the
runs.  The arms' outputs are compared in the same run.  k_pod_pending alone is timed with CUDA events around
rpk_pods_pending_list_device, the L2 flushed before each launch, at N = 1M and 16.8M and three densities.  The card's
name and power limit are read through NVML in the same run, and the SM clock right after each row's timed calls."""
import argparse
import json
import os
import re
import shutil
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import rpk  # noqa: E402
from select_slots_probe import COLS, G, N, Pinned, card, engine_on, sm_clock, stat  # noqa: E402


def build_one_select(tmp):
    """librpk.so whose rpk_select_pending runs one select over the whole list: rpk_api.cu compiled with the flags
    of csrc/Makefile plus -DRPK_MEASURE_PENDING_ONE_SELECT, linked with the other objects build() left in build/"""
    csrc = os.path.join(ROOT, "k8s-runpod-kubelet_b200", "csrc")
    mk = open(os.path.join(csrc, "Makefile")).read()

    def var(k):
        return re.search(rf"^{k} [:?]?= (.*)$", mk, re.M).group(1)

    flags = var("NVCCFLAGS").replace("$(ARCH)", var("ARCH")).split()
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    objs = []
    for src in var("SRCS").split():
        if src == "rpk_api.cu":
            obj = os.path.join(tmp, "rpk_api_one_select.o")
            subprocess.check_call([nvcc, *flags, "-DRPK_MEASURE_PENDING_ONE_SELECT", "-c", src, "-o", obj], cwd=csrc)
        else:
            obj = os.path.join(csrc, "..", "build", src[:-3] + ".o")
        objs.append(obj)
    lib = os.path.join(tmp, "librpk_one_select.so")
    subprocess.check_call([nvcc, *var("ARCH").split(), "-shared", "-o", lib, *objs, "-lcudart_static", "-lpthread", "-ldl", "-lrt"])
    return lib


def kernel_alone(runs):
    """k_pod_pending by itself: CUDA events around rpk_pods_pending_list_device, a 256 MB fill before each launch so
    that the flags come from HBM"""
    import torch

    rows = []
    rng = np.random.default_rng(19)
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
    with rpk.Engine(1) as eng:
        for n_slots in (1 << 20, 1 << 24):
            eng.pods_reset(n_slots)
            d_out = torch.empty(n_slots, dtype=torch.int32, device="cuda")
            d_n = torch.zeros(1, dtype=torch.int32, device="cuda")
            for density in (0.004, 0.125, 1.0):
                flags = (rng.random(n_slots) < density).astype(np.uint8)
                eng.pods_mark_pending(np.arange(n_slots, dtype=np.uint32), flags)
                ts = []
                for i in range(runs + 5):
                    flush.fill_(i & 0xFF)
                    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    t0.record()
                    eng.pods_pending_list_device(d_out, d_n)
                    t1.record()
                    torch.cuda.synchronize()
                    if i >= 5:
                        ts.append(t0.elapsed_time(t1) * 1e3)
                assert int(d_n.item()) == int(flags.sum())
                assert np.array_equal(d_out[: int(d_n.item())].cpu().numpy().view(np.uint32), np.flatnonzero(flags))
                row = {"N": n_slots, "density": density, "n_pending": int(flags.sum()), "kernel_us": stat(ts),
                       "sm_clock_mhz_after_timed_runs": sm_clock()}
                rows.append(row)
                print(json.dumps(row), flush=True)
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "h100_select_pending.json"))
    ap.add_argument("--runs", type=int, default=25)
    a = ap.parse_args()
    import torch

    if not torch.cuda.is_available():
        raise SystemExit("select_pending_probe: no GPU (numbers here are only measured on the device)")
    gpu = card()
    offers = rpk.synth.make_offers(G)
    pods = rpk.synth.make_pods(N)
    pin = Pinned()
    rows = []
    tmp = tempfile.TemporaryDirectory()
    eng = rpk.Engine(1)
    sub = engine_on(build_one_select(tmp.name))
    try:
        for e in (eng, sub):
            e.upload_offers(offers)
            e.pods_reset(N)
            e.pods_seed_slots(np.arange(N, dtype=np.uint32), pods)
        rng = np.random.default_rng(17)
        every = np.arange(N, dtype=np.uint32)
        for P in (4096, 125_000, N):
            for subset in (("every slot",) if P == N else ("first P", "random ascending")):
                sl = np.arange(P, dtype=np.uint32) if subset != "random ascending" else np.sort(rng.choice(N, P, replace=False)).astype(np.uint32)
                flags = np.zeros(N, np.uint8)
                flags[sl] = 1
                for e in (eng, sub):
                    e.pods_mark_pending(every, flags)
                h_slots = pin.array(P, np.uint32)
                h_slots[:] = sl
                h_cols = {}
                for k, dt in COLS:
                    h_cols[k] = pin.array(P, dt)
                    h_cols[k][:] = pods[k][sl]
                arms = ("columns", "slots", "pending", "pending_nolist") + (("pending_one_select", "pending_one_select_nolist") if P == N else ())
                for top5 in (True, False):
                    outs = {arm: (pin.array(P, np.int32), pin.array(P * 5, np.int32).reshape(P, 5) if top5 else None, pin.array(P, np.uint32))
                            for arm in arms}

                    def pending(e, arm, want_slots):
                        b, t, s = outs[arm]
                        return lambda: e.select_pending(P, want_top5=top5, want_slots=want_slots, out_best=b, out_top5=t, out_slots=s)

                    calls = {"columns": lambda: eng.select(h_cols, want_top5=top5, out_best=outs["columns"][0], out_top5=outs["columns"][1]),
                             "slots": lambda: eng.select_slots(h_slots, want_top5=top5, out_best=outs["slots"][0], out_top5=outs["slots"][1])}
                    for arm in arms[2:]:
                        calls[arm] = pending(sub if "one_select" in arm else eng, arm, not arm.endswith("nolist"))
                    ts = {arm: [] for arm in arms}
                    for i in range(a.runs + 5):
                        r = i % len(arms)
                        for arm in arms[r:] + arms[:r]:  # each arm in every position in turn
                            t0 = time.perf_counter()
                            calls[arm]()
                            t1 = time.perf_counter()
                            if i >= 5:
                                ts[arm].append((t1 - t0) * 1e3)
                        for arm in arms[1:]:
                            assert np.array_equal(outs["columns"][0], outs[arm][0]), (arm, P, subset, top5, i)
                            if top5:
                                assert np.array_equal(outs["columns"][1], outs[arm][1]), (arm, P, subset, top5, i)
                        for arm in ("pending", "pending_one_select"):
                            assert arm not in outs or np.array_equal(outs[arm][2], sl), (arm, P, subset, top5, i)
                    clock = sm_clock()
                    st = {arm: stat(ts[arm]) for arm in arms}
                    c = st["columns"]
                    row = {"P": P, "subset": subset, "top5": top5, **{arm + "_ms": st[arm] for arm in arms},
                           "speedup_vs_columns_median": {arm: c["median"] / st[arm]["median"] for arm in arms[1:]},
                           "outside_spread_of_columns": {arm: st[arm]["max"] < c["min"] or c["max"] < st[arm]["min"] for arm in arms[1:]},
                           "outputs_identical": True, "sm_clock_mhz_after_timed_runs": clock}
                    rows.append(row)
                    print(json.dumps(row), flush=True)
    finally:
        eng.close()
        sub.close()
        pin.free()
        tmp.cleanup()
    out = {"tool": "tools/select_pending_probe.py", "gpu": gpu, "G": G, "tracked_N": N, "runs": a.runs,
           "timing": "wall clock around each call (ends in a synchronise), arms rotated, 5 warm-up calls per arm, "
                     "median [min, max] of the runs; kernel_alone: CUDA events, L2 flushed before each launch",
           "rows": rows, "kernel_alone": kernel_alone(a.runs)}
    os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
    with open(a.out, "w") as f:
        json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
