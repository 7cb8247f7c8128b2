#!/usr/bin/env python
"""Pending results (rpk_select_pending_changed) against the full pending select (rpk_select_pending), on the GPU.

    python tools/select_pending_changed_probe.py [--out profiles/h100_select_pending_changed.json] [--runs 25]

One H100, G = 100k offers, a pod table of N = 1M slots seeded with synth.make_pods(1M), as tools/select_pending_probe.py.
For P pending slots in {4096, 125k, 1M} (a random ascending subset; every slot at 1M) two arms alternate, in rotated
order, in one run:
  A  rpk_select_pending with top-5 and slots_out: every pending row selected, 24 B per row back
  B  rpk_select_pending_changed: only stale rows reselected, only changed rows back; its per-slot mirror is compared
     with A's output after every call
in five states, each re-established before every round, outside the timed calls:
  steady          nothing changed since B's last call
  seed_1pct       1 % of the pending rows re-seeded with new columns
  same_offers     the identical offer table uploaded again
  one_price       one offer's price toggled between x1 and x1.5, the offer picked so that about 1 % of the lists hold it
  every_list      the offer table toggled between two orders of the same offers: every non-empty list changes
Wall clock around each call (both end in a synchronise; B's mirror update is outside), pinned outputs, 5 warm-up rounds, then the median [min, max]
of the runs.  k_pod_stale and k_pod_result_diff alone: their device time from torch.profiler over B calls in the
every_list state (every pending row stale, every row diffed), a 256 MB fill (L2 flush) before each call.  The card's
name and power limit are read through NVML in the same run, and the SM clock right after each row's timed calls."""
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
from select_slots_probe import COLS, G, N, Pinned, card, sm_clock, stat  # noqa: E402

STATES = ("steady", "seed_1pct", "same_offers", "one_price", "every_list")


def kernels_alone(eng, offers, flipped, P, runs):
    import torch
    from torch.profiler import ProfilerActivity, profile

    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
    times = {"k_pod_stale": [], "k_pod_result_diff": []}
    for i in range(runs):
        eng.upload_offers(flipped if i % 2 else offers)
        flush.fill_(i & 0xFF)
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            eng.select_pending_changed(P)
        for ev in prof.events():
            for k in times:
                if k in ev.name and ev.device_type.name == "CUDA":
                    times[k].append(ev.device_time if hasattr(ev, "device_time") else ev.cuda_time)
    eng.upload_offers(offers)
    return {k + "_us": stat(v) for k, v in times.items() if v}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "h100_select_pending_changed.json"))
    ap.add_argument("--runs", type=int, default=25)
    a = ap.parse_args()
    import torch

    if not torch.cuda.is_available():
        raise SystemExit("select_pending_changed_probe: no GPU (numbers here are only measured on the device)")
    gpu = card()
    offers = rpk.synth.make_offers(G)
    rev = np.arange(G)[::-1].copy()
    flipped = {k: np.ascontiguousarray(v[rev]) for k, v in offers.items()}
    pods = rpk.synth.make_pods(N)
    alt = rpk.synth.make_pods(N, seed=99)
    pin = Pinned()
    rows, alone = [], {}
    rng = np.random.default_rng(23)
    eng = rpk.Engine(1)
    try:
        eng.upload_offers(offers)
        every = np.arange(N, dtype=np.uint32)
        for P in (4096, 125_000, N):
            sl = every if P == N else np.sort(rng.choice(N, P, replace=False)).astype(np.uint32)
            eng.pods_reset(N)
            eng.pods_seed_slots(every, pods)
            flags = np.zeros(N, np.uint8)
            flags[sl] = 1
            eng.pods_mark_pending(every, flags)
            oa = (pin.array(P, np.int32), pin.array(P * 5, np.int32).reshape(P, 5), pin.array(P, np.uint32))
            ob = (pin.array(P, np.uint32), pin.array(P, np.int32), pin.array(P * 5, np.int32).reshape(P, 5))
            mirror_t = np.full((N, 5), -9, np.int32)
            mirror_b = np.full(N, -9, np.int32)
            eng.select_pending(P, want_top5=True, out_best=oa[0], out_top5=oa[1], out_slots=oa[2])
            # the offer whose share of the lists is closest to 1 %
            cnt = np.bincount(oa[1][oa[1] >= 0].ravel(), minlength=G)
            g1 = int(np.argmin(np.abs(cnt - 0.01 * P)))
            hit = np.sort(rng.choice(sl, max(1, P // 100), replace=False)).astype(np.uint32)
            def b_call():
                return eng.select_pending_changed(P, out_slots=ob[0], out_best=ob[1], out_top5=ob[2])

            def apply(got):  # the caller's mirror: outside the timed call
                mirror_b[got[2]], mirror_t[got[2]] = got[3], got[4]

            for state in STATES:
                eng.upload_offers(offers)
                eng.pods_seed_slots(hit, {k: np.ascontiguousarray(pods[k][hit]) for k, _ in COLS})
                apply(b_call())
                ts = {"A": [], "B": []}
                nr, nc = [], []
                for i in range(a.runs + 5):
                    if state == "seed_1pct":
                        src = alt if i % 2 == 0 else pods
                        eng.pods_seed_slots(hit, {k: np.ascontiguousarray(src[k][hit]) for k, _ in COLS})
                    elif state == "same_offers":
                        eng.upload_offers(offers)
                    elif state == "one_price":
                        o = {k: v.copy() for k, v in offers.items()}
                        if i % 2 == 0:
                            o["secure_price"][g1] *= 1.5  # dearer: only the lists that hold it can change
                            o["community_price"][g1] *= 1.5
                        eng.upload_offers(o)
                    elif state == "every_list":
                        eng.upload_offers(flipped if i % 2 == 0 else offers)
                    arms = ("A", "B") if i % 2 == 0 else ("B", "A")
                    for arm in arms:
                        t0 = time.perf_counter()
                        if arm == "A":
                            eng.select_pending(P, want_top5=True, out_best=oa[0], out_top5=oa[1], out_slots=oa[2])
                        else:
                            got = b_call()
                        t1 = time.perf_counter()
                        if i >= 5:
                            ts[arm].append((t1 - t0) * 1e3)
                    apply(got)
                    n_p, n_r, s = got[:3]
                    assert n_p == P and np.array_equal(oa[2], sl)
                    assert np.array_equal(mirror_b[sl], oa[0]) and np.array_equal(mirror_t[sl], oa[1]), (P, state, i)
                    if i >= 5:
                        nr.append(n_r)
                        nc.append(len(s))
                clock = sm_clock()
                sa, sb = stat(ts["A"]), stat(ts["B"])
                row = {"P": P, "state": state, "A_select_pending_ms": sa, "B_select_pending_changed_ms": sb,
                       "n_reselected": stat(nr), "n_changed": stat(nc), "speedup_median": sa["median"] / sb["median"],
                       "B_faster_outside_spread": sb["max"] < sa["min"], "B_slower_outside_spread": sb["min"] > sa["max"],
                       "mirror_equals_A": True, "sm_clock_mhz_after_timed_runs": clock}
                rows.append(row)
                print(json.dumps(row), flush=True)
            alone[str(P)] = kernels_alone(eng, offers, flipped, P, a.runs)
            print(json.dumps({"P": P, "kernels_alone": alone[str(P)]}), flush=True)
    finally:
        eng.close()
        pin.free()
    out = {"tool": "tools/select_pending_changed_probe.py", "gpu": gpu, "G": G, "tracked_N": N, "runs": a.runs,
           "timing": "wall clock around each call (ends in a synchronise), arms alternated, 5 warm-up rounds, median [min, "
                     "max] of the runs; kernels_alone: torch.profiler device time, every pending row stale, L2 flushed "
                     "before each call",
           "rows": rows, "kernels_alone": alone}
    os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
    with open(a.out, "w") as f:
        json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
