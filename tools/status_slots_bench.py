#!/usr/bin/env python
"""Slot-list status diff against the whole-table sweep, on the GPU.

    python tools/status_slots_bench.py [--out profiles/h100_status_slots.json] [--runs 25]

* host call, the streaming config's shape (C5: 100 status mutations per 10 ms over 100k tracked slots, stride 16):
  rpk_status_diff_slots over the 100 fetched slots against rpk_status_diff_codes over the whole table, alternated in
  one run; wall clock around each call (both end in a stream synchronise).
* device kernel: rpk_status_diff_slots_device over n = 1 %, 10 % and 100 % of N listed slots next to
  rpk_status_diff_device_codes over the whole column, N = 1M and 16.8M at strides 16 and 32; CUDA events around each
  launch, L2 flushed (256 MiB write) before each, median of the runs.  Every sweep after the first reports nothing
  (the records do not change), so both sides time the compare, not the copy of a changed list.
The card's name and power limit are read in the same run and stored with the numbers."""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import rpk  # noqa: E402


def card():
    import torch

    name, limit = torch.cuda.get_device_name(0), None
    try:
        import pynvml as nv

        nv.nvmlInit()
        limit = nv.nvmlDeviceGetPowerManagementLimit(nv.nvmlDeviceGetHandleByIndex(0)) / 1000.0
    except Exception:
        try:
            out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                                 capture_output=True, text=True, timeout=30).stdout.strip()
            limit = float(out.splitlines()[0])
        except Exception:
            limit = None
    return {"name": name, "power_limit_w": limit}


def host_c5(runs: int):
    N, stride, n = 100_000, 16, 100
    rng = np.random.default_rng(5)
    recs = rpk.synth.make_status_records(N, 0, stride=stride)
    with rpk.Engine(1) as full, rpk.Engine(1) as part:
        full.status_diff(recs, want_codes=True)
        part.status_reset(N)
        part.status_seed(recs)
        t_full, t_part = [], []
        for i in range(runs + 5):
            slots = np.sort(rng.choice(N, n, replace=False)).astype(np.uint32)
            recs[slots, 1] ^= 1  # this tick's mutations
            sub = np.ascontiguousarray(recs[slots])
            t0 = time.perf_counter()
            got_p, _ = part.status_diff_slots(slots, sub, want_codes=True)
            t1 = time.perf_counter()
            got_f, _, _ = full.status_diff(recs, want_codes=True)
            t2 = time.perf_counter()
            assert np.array_equal(got_p, got_f), i
            if i >= 5:
                t_part.append((t1 - t0) * 1e3)
                t_full.append((t2 - t1) * 1e3)
    return {"N": N, "stride": stride, "listed": n, "runs": runs, "slots_ms_median": statistics.median(t_part),
            "full_ms_median": statistics.median(t_full), "speedup": statistics.median(t_full) / statistics.median(t_part)}


def device(runs: int):
    import torch

    dev = torch.device("cuda", 0)
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    rows = []
    with rpk.Engine(1) as eng:
        for N in (1 << 20, 1 << 24):
            for stride in (16, 32):
                recs = torch.from_numpy(rpk.synth.make_status_records(N, 0, stride=stride)).to(dev)
                col = torch.zeros(N, dtype=torch.int64, device=dev)
                idx = torch.empty(N, dtype=torch.int32, device=dev)
                code = torch.empty(N, dtype=torch.int16, device=dev)
                cnt = torch.zeros(1, dtype=torch.int32, device=dev)

                def timed(fn):
                    fn()  # sizes scratch; the state is seen from here on
                    ts = []
                    for i in range(runs):
                        flush.fill_(i & 0xFF)
                        ev[0].record()
                        fn()
                        ev[1].record()
                        torch.cuda.synchronize()
                        ts.append(ev[0].elapsed_time(ev[1]) * 1e3)
                    return statistics.median(ts)

                full_us = timed(lambda: eng.status_diff_device(recs, stride, col, idx, cnt, d_changed_code=code))
                rows.append({"N": N, "stride": stride, "listed": N, "kind": "full", "kernel_us_median": full_us})
                g = np.random.default_rng(N + stride)
                for pct in (1, 10, 100):
                    n = N * pct // 100
                    slots = np.arange(N, dtype=np.uint32) if pct == 100 else np.sort(g.choice(N, n, replace=False)).astype(np.uint32)
                    d_slots = torch.from_numpy(slots.view(np.int32)).to(dev)
                    d_sub = recs if pct == 100 else recs[torch.from_numpy(slots.astype(np.int64)).to(dev)].contiguous()
                    us = timed(lambda: eng.status_diff_slots_device(d_slots, d_sub, stride, col, idx, cnt, d_changed_code=code))
                    rows.append({"N": N, "stride": stride, "listed": n, "kind": f"slots {pct}%", "kernel_us_median": us,
                                 "ratio_to_full": us / full_us})
                    del d_slots, d_sub
                del recs, col, idx, code
                torch.cuda.empty_cache()
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "h100_status_slots.json"))
    ap.add_argument("--runs", type=int, default=25)
    a = ap.parse_args()
    import torch

    if not torch.cuda.is_available():
        raise SystemExit("status_slots_bench: no GPU (numbers here are only measured on the device)")
    out = {"tool": "tools/status_slots_bench.py", "gpu": card(), "host_c5": host_c5(200), "device": device(a.runs),
           "device_timing": "CUDA events around one launch, L2 flushed before each, median of the runs"}
    out["gpu_after"] = card()
    os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
    with open(a.out, "w") as f:
        json.dump(out, f, indent=1)
    print(json.dumps(out, indent=1))


if __name__ == "__main__":
    main()
