#!/usr/bin/env python
"""K1 tuning sweep (1 GPU): time rpk_select_device (k_pod_classify + k_pod_scatter + the persistent k_select_persist)
for several row counts and RPK_TUNE settings -- the per-GPU work of the N-GPU strong-scaling bench is P/N rows, so
P = 125k here is what each GPU does at N = 8.  --variants is a '|'-separated list of RPK_TUNE values (spaces become
commas), e.g. "|stagekb=110|ipw=8 pdl=off"; the default times the defaults only.

    python tools/k1_tune.py [--iters 20] [--variants ""] [--out results/k1_tune.json]
"""
import argparse
import importlib
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    os.environ["RPK_TUNE_RELOAD"] = "1"  # this tool sweeps RPK_TUNE inside one process
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--offers", type=int, default=100_000)
    ap.add_argument("--pods", default="125000,250000,1000000")
    ap.add_argument("--variants", default="")
    ap.add_argument("--status-slots", type=int, default=0, help="run a status sweep of this many slots on a side stream alongside")
    ap.add_argument("--prio", action="store_true", help="select on a high-priority stream, the sweep on a low-priority one")
    ap.add_argument("--out", default=os.path.join(ROOT, "results", "k1_tune.json"))
    args = ap.parse_args()

    import torch

    pkg = importlib.import_module("k8s-runpod-kubelet_b200")
    synth = pkg.synth
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(0)
    G = args.offers
    offers = synth.make_offers(G)
    eng = pkg.Engine(1, device_ids=[0])
    eng.upload_offers(offers)
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
    side = torch.cuda.Stream(device=dev, priority=0)
    main = torch.cuda.Stream(device=dev, priority=-1) if args.prio else torch.cuda.current_stream()
    out = []
    ref = {}
    for P in [int(x) for x in args.pods.split(",")]:
        pods_np = synth.make_pods(P, row0=0)
        d_pods = {k: torch.from_numpy(v).to(dev) for k, v in pods_np.items()}
        best = torch.empty(P, dtype=torch.int32, device=dev)
        NS = args.status_slots
        if NS:
            recs = [torch.from_numpy(synth.make_status_records(NS, i, 0.01 * i).reshape(-1)).to(dev) for i in range(2)]
            hp = torch.zeros(NS, dtype=torch.int64, device=dev)
            chg = torch.empty(NS, dtype=torch.int32, device=dev)
            nch = torch.zeros(1, dtype=torch.int32, device=dev)
        for var in args.variants.split("|"):
            os.environ["RPK_TUNE"] = var.replace(" ", ",")
            for _ in range(3):
                eng.select_device(d_pods, best)
            torch.cuda.synchronize()
            ms = []
            for i in range(args.iters):
                flush.fill_(i & 0xFF)
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                main.wait_stream(torch.cuda.current_stream())
                e0.record(main)
                if NS:
                    side.wait_event(e0)
                    eng.status_diff_device(recs[i & 1], 32, hp, chg, nch, stream=side.cuda_stream)
                eng.select_device(d_pods, best, stream=main.cuda_stream or None)
                if NS:
                    main.wait_stream(side)  # the step ends when both are done
                e1.record(main)
                torch.cuda.synchronize()
                ms.append(e0.elapsed_time(e1))
            key = P
            if key not in ref:
                ref[key] = best.clone()
            same = bool((best == ref[key]).all())
            ms.sort()
            row = {"P": P, "G": G, "tune": os.environ["RPK_TUNE"], "status_slots": NS, "us_mean": 1e3 * sum(ms) / len(ms),
                   "us_median": 1e3 * ms[len(ms) // 2], "us_min": 1e3 * ms[0], "scores_per_s": P * G / (sum(ms) / len(ms) * 1e-3),
                   "same_result_as_first_variant": same}
            print(json.dumps(row), flush=True)
            out.append(row)
    os.makedirs(os.path.dirname(args.out), exist_ok=True)
    json.dump(out, open(args.out, "w"), indent=1)


if __name__ == "__main__":
    main()
