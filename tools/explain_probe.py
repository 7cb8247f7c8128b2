#!/usr/bin/env python
"""rpk_explain_slots beside rpk_select_slots (with top-5, as the Provider's tick asks for it) on the same slot lists (1 GPU):
G synthetic offers (default 100k), a pod table of --table slots seeded with synthetic pods, and random lists of 1k, 10k,
100k and 1M slots.  Each call is timed on the host around the whole call (it ends in a stream synchronise) after
--warmup calls, --reps times, alternating explain and select; the JSON holds the median, min and max per call and the
row-offer evaluations per second of the explain (n_slots x G over the median).  A separate torch.profiler run records
k_explain's kernel time per size.  The card's name, power limit and SM clock are read in the same run.

    python tools/explain_probe.py [--offers 100000] [--table 1000000] [--reps 20] [--out profiles/h100_explain.json]
"""
import argparse
import importlib
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
        name, power, mhz = [s.strip() for s in q.split(",")]
        return {"gpu": name, "power_limit": power, "sm_max_clock": mhz}
    except Exception as e:  # the timings do not depend on it; say that it is missing
        return {"gpu": None, "card_query_error": str(e)}


def stats_ms(ts):
    return {"median_ms": statistics.median(ts) * 1e3, "min_ms": min(ts) * 1e3, "max_ms": max(ts) * 1e3, "reps": len(ts)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--offers", type=int, default=100_000)
    ap.add_argument("--table", type=int, default=1_000_000)
    ap.add_argument("--sizes", default="1000,10000,100000,1000000")
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "h100_explain.json"))
    a = ap.parse_args()
    import torch

    rpk = importlib.import_module("k8s-runpod-kubelet_b200")
    offers = rpk.synth.make_offers(a.offers, correlated=True)
    pods = rpk.synth.make_pods(a.table)
    res = {"card": card(), "offers": a.offers, "pod_table": a.table, "sizes": []}
    with rpk.Engine(1) as eng:
        eng.upload_offers(offers)
        eng.pods_reset(a.table)
        eng.pods_seed_slots(np.arange(a.table, dtype=np.uint32), pods)
        lists = {n: np.random.default_rng(n).integers(0, a.table, n).astype(np.uint32) for n in map(int, a.sizes.split(","))}
        for n, sl in lists.items():
            out = np.empty(n * 14, np.uint32)
            best, top5 = np.empty(n, np.int32), np.empty((n, 5), np.int32)
            calls = {"explain_slots": lambda: eng.explain_slots(sl, out=out),
                     "select_slots_top5": lambda: eng.select_slots(sl, want_top5=True, out_best=best, out_top5=top5)}
            for fn in calls.values():
                for _ in range(a.warmup):
                    fn()
            ts = {k: [] for k in calls}
            for _ in range(a.reps):
                for k, fn in calls.items():
                    t0 = time.perf_counter()
                    fn()
                    ts[k].append(time.perf_counter() - t0)
            row = {"n_slots": n, **{k: stats_ms(v) for k, v in ts.items()}}
            row["explain_row_offer_evals_per_s"] = n * a.offers / (row["explain_slots"]["median_ms"] * 1e-3)
            res["sizes"].append(row)
            print(json.dumps(row), flush=True)
        # kernel time in a run of its own
        from torch.profiler import ProfilerActivity, profile

        for row in res["sizes"]:
            sl = lists[row["n_slots"]]
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                for _ in range(5):
                    eng.explain_slots(sl)
                torch.cuda.synchronize()
            k = [e.device_time for e in prof.events() if e.name.endswith("k_explain(rpk::ExplainArgs)") or "k_explain" in e.name]
            if k:
                row["k_explain_kernel_ms_median"] = statistics.median(k) / 1e3
                row["kernel_row_offer_evals_per_s"] = row["n_slots"] * a.offers / (row["k_explain_kernel_ms_median"] * 1e-3)
    os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
    with open(a.out, "w") as f:
        json.dump(res, f, indent=1)
    print(json.dumps({"card": res["card"], "out": a.out}))


if __name__ == "__main__":
    main()
