#!/usr/bin/env python
"""Where K0 of a persistent select goes (1 GPU): the class sort's two kernels (k_pod_classify, k_pod_scatter) and the
start of the grid kernel (k_select_persist), per row count, alone and beside a status sweep of --slots slots on a
low-priority side stream.  Every step flushes L2 (256 MiB write), enqueues the select on a high-priority stream and
synchronises; torch.profiler with CUDA activities records the kernels.  Prints one JSON line per (rows, sweep) case
with the medians over --steps steps, all in microseconds from the start of k_pod_classify:

    classify_us      k_pod_classify's duration
    scatter_end_us   k_pod_scatter's end: K0 as a whole
    scatter_tail_us  k_pod_scatter's end minus k_pod_classify's end (the scatter starts early: programmatic launch)
    k1_start_us      k_select_persist's start, k1_end_us its end (the select)

    python tools/k0_phases.py [--pods 125000,1000000] [--slots 1000000] [--steps 20] [--out results/k0_phases.json]
"""
import argparse
import importlib
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

KERNELS = {"k_pod_classify": "classify", "k_pod_scatter": "scatter", "k_select_persist": "k1"}


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
        name, power, mhz = [s.strip() for s in q.split(",")]
        return {"gpu": name, "power_limit": power, "sm_max_clock": mhz}
    except Exception as e:  # the timings do not depend on it; say that it is missing
        return {"gpu": None, "card_query_error": str(e)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--pods", default="125000,1000000")
    ap.add_argument("--offers", type=int, default=100_000)
    ap.add_argument("--slots", type=int, default=1_000_000, help="status sweep beside the select in the second case of each row count")
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--out", default=os.path.join(ROOT, "results", "k0_phases.json"))
    args = ap.parse_args()

    import torch
    from torch.profiler import ProfilerActivity, profile

    pkg = importlib.import_module("k8s-runpod-kubelet_b200")
    synth = pkg.synth
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(0)
    eng = pkg.Engine(1, device_ids=[0])
    eng.upload_offers(synth.make_offers(args.offers))
    NS = args.slots
    recs = [torch.from_numpy(synth.make_status_records(NS, i, 0.01 * i).reshape(-1)).to(dev) for i in range(2)]
    hp = torch.zeros(NS, dtype=torch.int64, device=dev)
    chg = torch.empty(NS, dtype=torch.int32, device=dev)
    nch = torch.zeros(1, dtype=torch.int32, device=dev)
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
    main_st = torch.cuda.Stream(device=dev, priority=-1)
    side = torch.cuda.Stream(device=dev, priority=0)
    os.makedirs(os.path.dirname(args.out), exist_ok=True)
    out = {**card(), "offers": args.offers, "steps": args.steps, "cases": []}
    for P in [int(x) for x in args.pods.split(",")]:
        d_pods = {k: torch.from_numpy(v).to(dev) for k, v in synth.make_pods(P, row0=0).items()}
        best = torch.empty(P, dtype=torch.int32, device=dev)
        for sweep in (False, True):
            def step(i):
                flush.fill_(i & 0xFF)
                main_st.wait_stream(torch.cuda.current_stream())
                side.wait_stream(torch.cuda.current_stream())
                if sweep:
                    eng.status_diff_device(recs[i & 1], 32, hp, chg, nch, stream=side.cuda_stream)
                eng.select_device(d_pods, best, stream=main_st.cuda_stream)
                torch.cuda.synchronize()

            for i in range(args.warmup):
                step(i)
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                for i in range(args.steps):
                    step(args.warmup + i)
            path = os.path.join(os.path.dirname(args.out), "k0_phases.pt.trace.json")
            prof.export_chrome_trace(path)
            kern = [e for e in json.load(open(path))["traceEvents"] if e.get("cat") == "kernel"]
            os.remove(path)
            kern.sort(key=lambda e: e["ts"])
            steps, cur = [], None
            for e in kern:  # a select is k_pod_classify, k_pod_scatter, k_select_persist in that order
                tag = next((v for k, v in KERNELS.items() if k in e["name"]), None)
                if tag == "classify":
                    cur = {}
                    steps.append(cur)
                if tag and cur is not None:
                    cur[tag] = (e["ts"], e["ts"] + e["dur"])
            rows = []
            for s in steps:
                if set(s) != set(KERNELS.values()):
                    continue
                t0 = s["classify"][0]
                rows.append({"classify_us": s["classify"][1] - t0, "scatter_end_us": s["scatter"][1] - t0,
                             "scatter_tail_us": s["scatter"][1] - s["classify"][1], "k1_start_us": s["k1"][0] - t0,
                             "k1_end_us": s["k1"][1] - t0})
            if not rows:
                sys.exit(f"no complete select in the trace (P={P}, sweep={sweep})")
            case = {"P": P, "G": args.offers, "sweep_slots": NS if sweep else 0, "selects": len(rows),
                    **{k: round(statistics.median(r[k] for r in rows), 1) for k in rows[0]}}
            print(json.dumps(case), flush=True)
            out["cases"].append(case)
    json.dump(out, open(args.out, "w"), indent=1)


if __name__ == "__main__":
    main()
