#!/usr/bin/env python
"""Where a bench step goes (1 GPU): eager bench-shaped steps -- the status sweep enqueued on a low-priority side
stream, then the select (K0 classify + scatter, K1) on a high-priority stream, L2 flushed between steps -- under
torch.profiler with CUDA activities.  Prints one JSON line per step with every kernel's start and end relative to
the step's first kernel, and a summary line with the medians.  Run it on its own: tracing slows the host.

    python tools/step_trace.py [--pods 1000000] [--slots 1000000] [--steps 6] [--out-dir results]
"""
import argparse
import importlib
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

KERNELS = {"k_status_stream": "sweep", "k_pod_classify": "classify", "k_pod_scatter": "scatter", "k_select_persist": "k1"}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--pods", type=int, default=1_000_000)
    ap.add_argument("--offers", type=int, default=100_000)
    ap.add_argument("--slots", type=int, default=1_000_000)
    ap.add_argument("--steps", type=int, default=6)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--out-dir", default=os.path.join(ROOT, "results"))
    args = ap.parse_args()

    import torch
    from torch.profiler import ProfilerActivity, profile

    pkg = importlib.import_module("k8s-runpod-kubelet_b200")
    synth = pkg.synth
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(0)
    eng = pkg.Engine(1, device_ids=[0])
    eng.upload_offers(synth.make_offers(args.offers))
    d_pods = {k: torch.from_numpy(v).to(dev) for k, v in synth.make_pods(args.pods, row0=0).items()}
    NS = args.slots
    recs = [torch.from_numpy(synth.make_status_records(NS, i, 0.01 * i).reshape(-1)).to(dev) for i in range(2)]
    hp = torch.zeros(NS, dtype=torch.int64, device=dev)
    chg = torch.empty(NS, dtype=torch.int32, device=dev)
    code = torch.empty(NS, dtype=torch.int16, device=dev)
    nch = torch.zeros(1, dtype=torch.int32, device=dev)
    best = torch.empty(args.pods, dtype=torch.int32, device=dev)
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
    main_st = torch.cuda.Stream(device=dev, priority=-1)
    side = torch.cuda.Stream(device=dev, priority=0)

    def step(i):
        flush.fill_(i & 0xFF)
        main_st.wait_stream(torch.cuda.current_stream())
        side.wait_stream(torch.cuda.current_stream())
        eng.status_diff_device(recs[i & 1], 32, hp, chg, nch, stream=side.cuda_stream, d_changed_code=code)
        eng.select_device(d_pods, best, stream=main_st.cuda_stream)
        torch.cuda.synchronize()

    for i in range(args.warmup):
        step(i)
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for i in range(args.steps):
            step(args.warmup + i)
    os.makedirs(args.out_dir, exist_ok=True)
    path = os.path.join(args.out_dir, "step_trace.pt.trace.json")
    prof.export_chrome_trace(path)

    kern = [e for e in json.load(open(path))["traceEvents"] if e.get("cat") == "kernel"]
    kern.sort(key=lambda e: e["ts"])
    steps, cur = [], None
    for e in kern:  # a step is everything between two flush kernels
        tag = next((v for k, v in KERNELS.items() if k in e["name"]), None)
        if tag is None:
            cur = None
            continue
        if cur is None:
            cur = {}
            steps.append(cur)
        cur[tag] = (e["ts"], e["ts"] + e["dur"], e.get("args", {}).get("stream"))
    rows = []
    for s in steps:
        if set(s) != set(KERNELS.values()):
            continue
        t0 = min(v[0] for v in s.values())
        row = {k: {"start_us": round(v[0] - t0, 1), "end_us": round(v[1] - t0, 1), "stream": v[2]} for k, v in s.items()}
        row["step_us"] = round(max(v[1] for v in s.values()) - t0, 1)
        row["select_us"] = round(s["k1"][1] - s["classify"][0], 1)  # K0 start to K1 end
        rows.append(row)
        print(json.dumps(row), flush=True)
    if not rows:
        sys.exit("no complete step in the trace")
    med = lambda f: round(statistics.median(f(r) for r in rows), 1)
    summary = {"summary": True, "steps": len(rows), "gpu": torch.cuda.get_device_name(0), "pods": args.pods, "offers": args.offers, "slots": NS,
               "step_us": med(lambda r: r["step_us"]), "select_us": med(lambda r: r["select_us"]),
               **{f"{k}_{e}_us": med(lambda r, k=k, e=e: r[k][e + "_us"]) for k in KERNELS.values() for e in ("start", "end")},
               "trace": os.path.basename(path)}
    print(json.dumps(summary), flush=True)
    json.dump({"steps": rows, "summary": summary}, open(os.path.join(args.out_dir, "step_trace.json"), "w"), indent=1)


if __name__ == "__main__":
    main()
