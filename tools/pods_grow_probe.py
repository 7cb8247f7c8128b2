#!/usr/bin/env python
"""Growing the pod and status tables in place (rpk_pods_grow + rpk_status_grow) against what a caller had to do before:
reset both tables at the new size and upload everything again.

    python tools/pods_grow_probe.py [--out profiles/h100_pods_grow.json] [--rounds 10]

One H100, G = 100k offers, a pod table of N0 = 1M slots seeded with synth.make_pods, P pending slots in {125k, 1M} (a
random subset; every slot at 1M), every pending list reported once by rpk_select_pending_changed, and a tracked status
table of N0 slots seeded (stride 32).  Each round builds a fresh pair of ctxs with that history and grows them, in
alternating order, to N = 2 N0 (new buffers and copies) or N = 1.2 N0 (inside the 25 % slack: no allocation):
  A  rpk_pods_reset(N) + rpk_pods_seed_slots of every tracked row + rpk_pods_mark_pending of every flag +
     rpk_status_reset(N) + rpk_status_seed(N), then the next rpk_select_pending_changed
  B  rpk_pods_grow(N) + rpk_status_grow(N), then the same tick
Wall clock around the grow calls and around the tick, each ending in a synchronise (every call is a host call that
returns after its work); median [min, max] of the rounds.  After every round B's per-slot mirror of reported lists must
equal A's.  The card's name, power limit and SM clock are read through NVML in the same run."""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import rpk  # noqa: E402
from select_slots_probe import G, N as N0, card, sm_clock, stat  # noqa: E402

STRIDE = 32


def setup(offers, pods, flags, recs):
    """a ctx with the probe's history: the table seeded, the flags marked, every list reported, the status seeded;
    -> (engine, per-slot mirror of the reported lists)"""
    eng = rpk.Engine(1)
    every = np.arange(N0, dtype=np.uint32)
    eng.upload_offers(offers)
    eng.pods_reset(N0)
    eng.pods_seed_slots(every, pods)
    eng.pods_mark_pending(every, flags)
    mirror = np.full((N0, 5), -2, np.int32)
    _, _, sl, _, t5 = eng.select_pending_changed(N0)
    mirror[sl] = t5
    eng.status_reset(N0)
    eng.status_seed(recs)
    return eng, mirror


def arm_a(eng, N, pods, flags, recs):
    every = np.arange(N0, dtype=np.uint32)
    wide = np.zeros((N, STRIDE), np.uint8)
    wide[:N0] = recs
    t0 = time.perf_counter()
    eng.pods_reset(N)
    eng.pods_seed_slots(every, pods)
    eng.pods_mark_pending(every, flags)
    eng.status_reset(N)
    eng.status_seed(wide)
    return time.perf_counter() - t0


def arm_b(eng, N):
    t0 = time.perf_counter()
    eng.pods_grow(N)
    eng.status_grow(N)
    return time.perf_counter() - t0


def tick(eng, mirror, N):
    t0 = time.perf_counter()
    n_p, n_r, sl, _, t5 = eng.select_pending_changed(N)
    t = time.perf_counter() - t0
    grown = np.full((N, 5), -2, np.int32)
    grown[:N0] = mirror
    grown[sl] = t5
    return t, n_r, len(sl), grown


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "h100_pods_grow.json"))
    ap.add_argument("--rounds", type=int, default=10)
    args = ap.parse_args()
    import torch

    if not torch.cuda.is_available():
        raise SystemExit("no GPU: this probe measures on the GPU only")
    info = card()
    offers = rpk.synth.make_offers(G, correlated=True)
    pods = rpk.synth.make_pods(N0)
    recs = rpk.synth.make_status_records(N0, 0, stride=STRIDE)
    rows = []
    for P in (125_000, N0):
        flags = np.zeros(N0, np.uint8)
        flags[np.random.default_rng(P).choice(N0, P, replace=False) if P < N0 else slice(None)] = 1
        for factor in (2.0, 1.2):
            N = int(N0 * factor)
            t = {"A_grow": [], "A_tick": [], "B_grow": [], "B_tick": []}
            counts = {}
            for r in range(args.rounds + 1):  # round 0 warms up every shape and is not kept
                a, ma = setup(offers, pods, flags, recs)
                b, mb = setup(offers, pods, flags, recs)
                for arm in ("AB" if r % 2 == 0 else "BA"):
                    if arm == "A":
                        g = arm_a(a, N, pods, flags, recs)
                        tk, n_r, n_c, ma = tick(a, ma, N)
                    else:
                        g = arm_b(b, N)
                        tk, n_r, n_c, mb = tick(b, mb, N)
                    if r:
                        t[arm + "_grow"].append(g * 1e3)
                        t[arm + "_tick"].append(tk * 1e3)
                    counts[arm] = {"n_reselected": n_r, "n_changed": n_c}
                pend = np.flatnonzero(flags)
                assert np.array_equal(ma[pend], mb[pend]), f"P={P} x{factor}: B's mirror differs from A's"
                a.close()
                b.close()
            rows.append({"P": P, "N0": N0, "N": N, "factor": factor, "counts": counts,
                         **{k: stat(v) for k, v in t.items()}, "sm_clock_mhz": sm_clock()})
            print(json.dumps(rows[-1]), flush=True)
    out = {"card": info, "G": G, "N0": N0, "stride": STRIDE, "rounds": args.rounds, "unit": "ms (wall clock)", "rows": rows}
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, "w") as f:
        json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
