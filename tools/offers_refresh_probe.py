#!/usr/bin/env python
"""Offer-table refresh (rpk_offers_refresh) against upload (rpk_offers_upload) ahead of the pending tick, on the GPU.

    python tools/offers_refresh_probe.py [--out profiles/h100_offers_refresh.json] [--runs 25]

One H100, G = 100k offers (synth.make_offers), a pod table of N = 1M slots seeded with synth.make_pods(1M), P pending
slots in {125k, 1M} (a random ascending subset; every slot at 1M).  Two ctxs with the same history, one per arm:
  A  rpk_offers_upload(new table) + rpk_select_pending_changed
  B  rpk_offers_refresh(new table) + rpk_select_pending_changed
Before every round both ctxs upload the base table and run one tick (untimed), so every stored result is current and
B's change window is empty.  The new table of a round differs from the base by one case:
  identical       no offer changed
  unlisted_price  one offer that no pending list holds: both prices x1.5
  listed_up       the offer the most pending lists hold: both prices x1.5
  listed_down     the same offer: both prices x0.8
  16_offers       16 random offers with positive prices: both prices x1.1
  delta_max       RPK_OFFERS_DELTA_MAX random offers with positive prices: both prices x1.1 (the window at capacity)
  delta_max_plus1 one offer more: B invalidates wholesale, as A
Each round times, per arm, the table call alone, the table call + the tick after it, and then one steady tick (nothing
changed since; B's window still holds the round's offers, so B runs k_pod_stale_reach where A runs k_pod_stale).  Arms
alternate in rotated order; wall clock around calls that end in a synchronise; 3 warm-up rounds, then median [min, max]
of the runs.  After every call B's per-slot mirror must equal A's.  Kernels alone (torch.profiler device time, a 256 MB
fill before each call, P = 1M): k_pod_stale on A's tick after an upload and on its steady tick, k_pod_stale_reach on
B's tick after a refresh of 1, 8 and RPK_OFFERS_DELTA_MAX offers and on the steady tick after it.  The card's name,
power limit and SM clock are read in the same run."""
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
from select_slots_probe import G, N, Pinned, card, sm_clock, stat  # noqa: E402

DELTA_MAX = 16  # RPK_OFFERS_DELTA_MAX
CASES = ("identical", "unlisted_price", "listed_up", "listed_down", "16_offers", "delta_max", "delta_max_plus1")
WARMUP = 3


def scaled(base, gs, f):
    o = {k: (v.copy() if v is not None else None) for k, v in base.items()}
    o["secure_price"][gs] *= f
    o["community_price"][gs] *= f
    return o


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "h100_offers_refresh.json"))
    ap.add_argument("--runs", type=int, default=25)
    a = ap.parse_args()
    import torch

    if not torch.cuda.is_available():
        raise SystemExit("offers_refresh_probe: no GPU (numbers here are only measured on the device)")
    gpu = card()
    base = rpk.synth.make_offers(G)
    pods = rpk.synth.make_pods(N)
    every = np.arange(N, dtype=np.uint32)
    pin = Pinned()
    rng = np.random.default_rng(29)
    rows, alone = [], {}
    ea, eb = rpk.Engine(1), rpk.Engine(1)
    try:
        for P in (125_000, N):
            sl = every if P == N else np.sort(rng.choice(N, P, replace=False)).astype(np.uint32)
            flags = np.zeros(N, np.uint8)
            flags[sl] = 1
            outs, mirrors = {}, {}
            for arm, e in (("A", ea), ("B", eb)):
                e.upload_offers(base)
                e.pods_reset(N)
                e.pods_seed_slots(every, pods)
                e.pods_mark_pending(every, flags)
                outs[arm] = (pin.array(P, np.uint32), pin.array(P, np.int32), pin.array(P * 5, np.int32).reshape(P, 5))
                mirrors[arm] = np.full((N, 5), -9, np.int32)

            def tick(arm):
                e = ea if arm == "A" else eb
                o = outs[arm]
                return e.select_pending_changed(P, out_slots=o[0], out_best=o[1], out_top5=o[2])

            def apply(arm, got):  # the caller's mirror: outside the timed calls
                mirrors[arm][got[2]] = got[4]

            def same():
                assert np.array_equal(mirrors["A"][sl], mirrors["B"][sl]), "B's mirror differs from A's"

            for arm in ("A", "B"):
                apply(arm, tick(arm))
            t5 = mirrors["A"][sl]
            used = np.bincount(t5[t5 >= 0].ravel(), minlength=G)
            top, unlisted = int(used.argmax()), int(np.flatnonzero(used == 0)[0])
            movable = np.flatnonzero((base["secure_price"] > 0) & (base["community_price"] > 0))  # x1.1 changes them
            picks = rng.choice(movable, DELTA_MAX + 1, replace=False)
            tables = {"identical": scaled(base, [], 1.0), "unlisted_price": scaled(base, [unlisted], 1.5),
                      "listed_up": scaled(base, [top], 1.5), "listed_down": scaled(base, [top], 0.8),
                      "16_offers": scaled(base, picks[:16], 1.1), "delta_max": scaled(base, picks[:DELTA_MAX], 1.1),
                      "delta_max_plus1": scaled(base, picks, 1.1)}
            for case in CASES:
                new = tables[case]
                ts = {k: [] for k in ("A_table", "A_total", "A_steady", "B_table", "B_total", "B_steady")}
                nr = {"A": [], "B": []}
                n_changed = []
                for i in range(a.runs + WARMUP):
                    for arm, e in (("A", ea), ("B", eb)):  # back to the base table, every result current
                        e.upload_offers(base)
                        apply(arm, tick(arm))
                    same()
                    for arm in (("A", "B") if i % 2 == 0 else ("B", "A")):
                        e = ea if arm == "A" else eb
                        t0 = time.perf_counter()
                        if arm == "A":
                            e.upload_offers(new)
                        else:
                            n = e.refresh_offers(new)
                        t1 = time.perf_counter()
                        got = tick(arm)
                        t2 = time.perf_counter()
                        apply(arm, got)
                        t3 = time.perf_counter()
                        steady = tick(arm)
                        t4 = time.perf_counter()
                        assert steady[1] == 0, f"{case}: a steady tick reselected {steady[1]}"
                        if i >= WARMUP:
                            ts[arm + "_table"].append((t1 - t0) * 1e3)
                            ts[arm + "_total"].append((t2 - t0) * 1e3)
                            ts[arm + "_steady"].append((t4 - t3) * 1e3)
                            nr[arm].append(got[1])
                            if arm == "B":
                                n_changed.append(n)
                    same()
                clock = sm_clock()
                st = {k: stat(v) for k, v in ts.items()}
                row = {"P": P, "case": case, "n_offers_changed": stat(n_changed),
                       "A_upload_ms": st["A_table"], "B_refresh_ms": st["B_table"],
                       "A_upload_plus_tick_ms": st["A_total"], "B_refresh_plus_tick_ms": st["B_total"],
                       "A_steady_tick_after_ms": st["A_steady"], "B_steady_tick_after_ms": st["B_steady"],
                       "A_reselected": stat(nr["A"]), "B_reselected": stat(nr["B"]),
                       "B_total_faster_outside_spread": st["B_total"]["max"] < st["A_total"]["min"],
                       "B_total_slower_outside_spread": st["B_total"]["min"] > st["A_total"]["max"],
                       "mirror_B_equals_A": True, "sm_clock_mhz_after_timed_runs": clock}
                rows.append(row)
                print(json.dumps(row), flush=True)
            if P == N:
                alone = kernels_alone(ea, eb, base, tables, picks, tick, apply, a.runs)
                print(json.dumps({"P": P, "kernels_alone": alone}), flush=True)
    finally:
        ea.close()
        eb.close()
        pin.free()
    out = {"tool": "tools/offers_refresh_probe.py", "gpu": gpu, "G": G, "tracked_N": N, "runs": a.runs,
           "delta_max": DELTA_MAX,
           "timing": "wall clock around calls that end in a synchronise, arms alternated, 3 warm-up rounds, median [min, "
                     "max] of the runs; kernels_alone: torch.profiler device time, L2 flushed before each call",
           "rows": rows, "kernels_alone": alone}
    os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
    with open(a.out, "w") as f:
        json.dump(out, f, indent=1)


def kernels_alone(ea, eb, base, tables, picks, tick, apply, runs):
    import torch
    from torch.profiler import ProfilerActivity, profile

    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
    times = {}

    def timed(key, arm, reach):
        flush.fill_(len(times) & 0xFF)
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            got = tick(arm)
        apply(arm, got)
        for ev in prof.events():
            if ev.device_type.name == "CUDA" and "k_pod_stale" in ev.name and ("k_pod_stale_reach" in ev.name) == reach:
                times.setdefault(key, []).append(ev.device_time if hasattr(ev, "device_time") else ev.cuda_time)

    windows = {"1": scaled(base, picks[:1], 1.1), "8": scaled(base, picks[:8], 1.1), str(DELTA_MAX): tables["delta_max"]}
    for _ in range(runs):
        for e, arm in ((ea, "A"), (eb, "B")):
            e.upload_offers(base)
            apply(arm, tick(arm))
        ea.upload_offers(tables["listed_up"])
        timed("k_pod_stale_after_upload", "A", False)
        timed("k_pod_stale_steady", "A", False)
        for w, t in windows.items():
            eb.upload_offers(base)
            apply("B", tick("B"))
            eb.refresh_offers(t)
            timed(f"k_pod_stale_reach_window_{w}_after_refresh", "B", True)
            timed(f"k_pod_stale_reach_window_{w}_steady", "B", True)
    return {k + "_us": stat(v) for k, v in times.items()}


if __name__ == "__main__":
    main()
