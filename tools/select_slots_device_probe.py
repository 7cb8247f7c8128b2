#!/usr/bin/env python
"""The device select over a slot list (rpk_select_slots_device_gather) against the same select on resident columns, on
one GPU.

    python tools/select_slots_device_probe.py [--calls 25] [--out profiles/h100_select_slots_device.json]

G = 100k offers (synth.make_offers(100_000)) and a pod table of N = 1M slots seeded with synth.make_pods(1M).  For n
pending rows in {125k, 1M}, listed in table order (slots 0..n-1) or as a random ascending subset, with and without the
top-5 lists, three arms alternate call by call:
  A  rpk_select_device_gather on the n rows' five columns, already on the GPU: the lower bound
  B  rpk_select_slots_device_gather on the device list: the gather of the rows from the pod table, then the same select
  C  what a caller does without B: torch.index_select of the five table columns (kept on the GPU), then arm A's call
B - A is what the gather costs; C - B what the slot list saves over the caller's own gather.

Each call is timed with CUDA events on the calling stream; the L2 is flushed (256 MiB write) between calls, outside the
event pair; 5 warm-up rounds, then the median [min, max] of the timed calls.  All arms' outputs must be identical (the
run fails otherwise).  Card name, power limit and SM clock are read through NVML in the same run."""
import argparse
import importlib
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

G = 100_000
N = 1 << 20
SIZES = (125_000, 1_000_000)
COLS = ("req_mem_gb", "req_vcpu", "req_ram_gb", "max_price", "cloud")


def nvml_info():
    import torch

    out = {"card": torch.cuda.get_device_name(0), "power_limit_w": None, "sm_mhz": None, "sm_max_mhz": None}
    try:
        import pynvml

        pynvml.nvmlInit()
        vis = os.environ.get("CUDA_VISIBLE_DEVICES")
        idx = int(vis.split(",")[0]) if vis and vis.split(",")[0].isdigit() else 0
        h = pynvml.nvmlDeviceGetHandleByIndex(idx)
        name = pynvml.nvmlDeviceGetName(h)
        out["card"] = name.decode() if isinstance(name, bytes) else name
        out["power_limit_w"] = pynvml.nvmlDeviceGetPowerManagementLimit(h) / 1000.0
        out["sm_mhz"] = pynvml.nvmlDeviceGetClockInfo(h, pynvml.NVML_CLOCK_SM)
        out["sm_max_mhz"] = pynvml.nvmlDeviceGetMaxClockInfo(h, pynvml.NVML_CLOCK_SM)
        out["source"] = "NVML"
    except Exception as e:  # noqa: BLE001 -- the timings are still useful without it; the JSON says so
        out["source"] = f"NVML unavailable ({e})"
    return out


def stats_us(ms):
    us = sorted(1e3 * m for m in ms)
    return {"median": statistics.median(us), "min": us[0], "max": us[-1], "n": len(us)}


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--calls", type=int, default=25, help="timed calls per arm and case (at least 25)")
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "h100_select_slots_device.json"))
    args = ap.parse_args()
    args.calls = max(args.calls, 25)

    import numpy as np
    import torch

    pkg = importlib.import_module("k8s-runpod-kubelet_b200")
    synth = pkg.synth
    dev = torch.device("cuda", 0)
    offers = synth.make_offers(G)
    pods = synth.make_pods(N)
    eng = pkg.Engine(1)
    eng.upload_offers(offers)
    eng.pods_reset(N)
    eng.pods_seed_slots(np.arange(N, dtype=np.uint32), pods)
    table = {k: torch.from_numpy(np.ascontiguousarray(pods[k])).to(dev) for k in COLS}  # arm C's copy of the table
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
    torch.cuda.set_stream(torch.cuda.Stream(device=dev, priority=-1))   # the select's stream priority, as in bench.py
    rng = np.random.default_rng(7)
    rows, all_identical = [], True
    for n in SIZES:
        for order in ("table order", "random ascending"):
            sl = np.arange(n, dtype=np.uint32) if order == "table order" else np.sort(rng.choice(N, n, replace=False)).astype(np.uint32)
            d_sl = torch.from_numpy(sl.view(np.int32)).to(dev)
            d_idx = d_sl.long()
            d_cols = {k: table[k].index_select(0, d_idx) for k in COLS}   # arm A's resident columns
            for top5 in (False, True):
                out = {a: (torch.empty(n, dtype=torch.int32, device=dev),
                           torch.empty(5 * n, dtype=torch.int32, device=dev) if top5 else None) for a in "ABC"}

                def arm_a():
                    eng.select_device_gather(d_cols, [out["A"][0].data_ptr()], 0, d_top5=out["A"][1])

                def arm_b():
                    eng.select_slots_device_gather(d_sl, [out["B"][0].data_ptr()], 0, d_top5=out["B"][1])

                def arm_c():
                    cols = {k: table[k].index_select(0, d_idx) for k in COLS}
                    eng.select_device_gather(cols, [out["C"][0].data_ptr()], 0, d_top5=out["C"][1])

                arms = {"A": arm_a, "B": arm_b, "C": arm_c}
                for _ in range(args.warmup):
                    for fn in arms.values():
                        fn()
                torch.cuda.synchronize()
                ms = {a: [] for a in arms}
                for i in range(args.calls * len(arms)):   # A, B, C, A, B, C, ...
                    a = "ABC"[i % 3]
                    flush.fill_(i & 0xFF)
                    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    e0.record(); arms[a](); e1.record()
                    e1.synchronize()
                    ms[a].append(e0.elapsed_time(e1))
                torch.cuda.synchronize()
                same = all(torch.equal(out["A"][0], out[a][0]) and (not top5 or torch.equal(out["A"][1], out[a][1]))
                           for a in "BC")
                all_identical = all_identical and same
                s = {a: stats_us(v) for a, v in ms.items()}
                row = {"n": n, "list": order, "top5": top5, "A_columns_us": s["A"], "B_slots_us": s["B"],
                       "C_index_select_then_columns_us": s["C"], "B_minus_A_us": s["B"]["median"] - s["A"]["median"],
                       "C_minus_B_us": s["C"]["median"] - s["B"]["median"], "outputs_identical": same}
                rows.append(row)
                print(f"n={n} {order} top5={top5}: A {s['A']['median']:.1f} us [{s['A']['min']:.1f}, {s['A']['max']:.1f}], "
                      f"B {s['B']['median']:.1f} [{s['B']['min']:.1f}, {s['B']['max']:.1f}], "
                      f"C {s['C']['median']:.1f} [{s['C']['min']:.1f}, {s['C']['max']:.1f}]; B - A {row['B_minus_A_us']:.1f}, "
                      f"C - B {row['C_minus_B_us']:.1f}; identical {same}", flush=True)
    gpu = nvml_info()
    doc = {
        "tool": "tools/select_slots_device_probe.py",
        "what": "device select over a slot list (B, rpk_select_slots_device_gather) vs resident columns (A, "
                "rpk_select_device_gather) vs torch.index_select of the table columns then A (C)",
        "gpu": gpu, "G": G, "tracked_N": N, "offers": "synth.make_offers(100000)", "pods": "synth.make_pods(1M) seeded into the table",
        "outputs": "one assignment vector (n_out = 1), top-5 lists in a local vector when asked for",
        "timing": f"CUDA events around each call, arms alternating A, B, C, {args.calls} calls per arm after {args.warmup} "
                  "warm-up rounds, L2 flushed (256 MiB write) between calls outside the event pair; microseconds",
        "outputs_identical": all_identical, "rows": rows,
    }
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, "w") as f:
        json.dump(doc, f, indent=1)
    print(f"wrote {args.out}; outputs {'identical' if all_identical else 'DIFFER'}", flush=True)
    eng.close()
    if not all_identical:
        sys.exit(1)


if __name__ == "__main__":
    main()
