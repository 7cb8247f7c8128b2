#!/usr/bin/env python
"""Pending results for one process per GPU (rpk_select_pending_changed_gather) against what such a caller runs without
it, and against the host call, on the GPU.

    python tools/select_pending_changed_gather_probe.py [--out profiles/h100_select_pending_changed_gather.json] [--runs 25]

One H100, G = 100k offers, a pod table of N = 1M slots seeded with synth.make_pods(1M).  The group has one rank
(n_ranks = 1): it owns the whole table, writes into one local exchange buffer, is bound to a one-rank flag group and
has the inline wait on.  n_ranks also sets the owned range, so a second GPU-local buffer cannot stand in for a peer here:
the cost of the peer stores over NVLink is not measured.  For P pending slots in {125k, 1M} (a random ascending subset;
every slot at 1M) three arms alternate, in rotated order, in one run:
  A  rpk_pods_pending_list_device + a read of the count + rpk_select_slots_device_gather_top5 over the whole list: what
     a one-process-per-GPU caller runs today, every pending row selected and its 24 B written out
  B  rpk_select_pending_changed_gather: only stale rows reselected, only changed rows written (its inline wait ends it)
  C  rpk_select_pending_changed, the host call, on a second ctx with the same history
in four states, each re-established before every round, outside the timed calls:
  steady          nothing changed since the last call
  seed_1pct       1 % of the pending rows re-seeded, alternately with new and with the old columns
  one_price       one offer's price toggled between x1 and x1.5, the offer picked so that about 1 % of the lists hold it
  every_list      the offer table toggled between two orders of the same offers: every non-empty list changes
Wall clock around each call, which ends in a device synchronise, 5 warm-up rounds, then the median [min, max] of the
runs.  After every round B's region must equal C's output bit for bit.  The card's name and power limit are read in the
same run, and the SM clock right after each row's timed calls."""
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

STATES = ("steady", "seed_1pct", "one_price", "every_list")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "h100_select_pending_changed_gather.json"))
    ap.add_argument("--runs", type=int, default=25)
    a = ap.parse_args()
    import torch

    if not torch.cuda.is_available():
        raise SystemExit("select_pending_changed_gather_probe: no GPU (numbers here are only measured on the device)")
    gpu = card()
    offers = rpk.synth.make_offers(G)
    rev = np.arange(G)[::-1].copy()
    flipped = {k: np.ascontiguousarray(v[rev]) for k, v in offers.items()}
    pods = rpk.synth.make_pods(N)
    alt = rpk.synth.make_pods(N, seed=99)
    every = np.arange(N, dtype=np.uint32)
    pin = Pinned()
    rows = []
    rng = np.random.default_rng(29)
    eb, ec = rpk.Engine(1), rpk.Engine(1)  # B (and A, which keeps no results) / C
    dev = torch.device("cuda", 0)
    try:
        words = eb.results_xchg_bytes(1, N) // 4
        xbuf = torch.zeros(words, dtype=torch.int32, device=dev)
        flags = torch.zeros(64, dtype=torch.int32, device=dev)
        eb.peer_bind([flags.data_ptr()], 0)
        d_list, d_n = torch.empty(N, dtype=torch.int32, device=dev), torch.zeros(1, dtype=torch.int32, device=dev)
        best, t5 = torch.empty(N, dtype=torch.int32, device=dev), torch.empty(5 * N, dtype=torch.int32, device=dev)
        oc = (pin.array(N, np.uint32), pin.array(N, np.int32), pin.array(N * 5, np.int32).reshape(N, 5))

        def both(fn):
            fn(eb)
            fn(ec)

        def arm_a():
            eb.pods_pending_list_device(d_list, d_n)
            n = int(d_n.item())
            eb.select_slots_device_gather(d_list[:n], [best.data_ptr()], 0, top5_ptrs=[t5.data_ptr()])
            torch.cuda.synchronize()

        def arm_b():
            eb.select_pending_changed_gather([xbuf.data_ptr()], N, 0)
            torch.cuda.synchronize()

        def arm_c():
            return ec.select_pending_changed(N, out_slots=oc[0], out_best=oc[1], out_top5=oc[2])

        for P in (125_000, N):
            sl = every if P == N else np.sort(rng.choice(N, P, replace=False)).astype(np.uint32)
            eb.peer_inline_wait(False)
            both(lambda e: e.upload_offers(offers))
            both(lambda e: e.pods_reset(N))
            both(lambda e: e.pods_seed_slots(every, pods))
            fl = np.zeros(N, np.uint8)
            fl[sl] = 1
            both(lambda e: e.pods_mark_pending(every, fl))
            lists = ec.select_slots(sl, want_top5=True)[1]
            cnt = np.bincount(lists[lists >= 0].ravel(), minlength=G)
            g1 = int(np.argmin(np.abs(cnt - 0.01 * P)))  # the offer whose share of the lists is closest to 1 %
            hit = np.sort(rng.choice(sl, max(1, P // 100), replace=False)).astype(np.uint32)
            arm_b()  # sizes B's scratch before the inline wait is turned on
            eb.peer_inline_wait(True)
            arm_c()
            for state in STATES:
                both(lambda e: e.upload_offers(offers))
                both(lambda e: e.pods_seed_slots(hit, {k: np.ascontiguousarray(pods[k][hit]) for k, _ in COLS}))
                arm_b()
                arm_c()
                ts = {"A": [], "B": [], "C": []}
                nr, nc = [], []
                for i in range(a.runs + 5):
                    if state == "seed_1pct":
                        src = alt if i % 2 == 0 else pods
                        both(lambda e: e.pods_seed_slots(hit, {k: np.ascontiguousarray(src[k][hit]) for k, _ in COLS}))
                    elif state == "one_price":
                        o = {k: v.copy() for k, v in offers.items()}
                        if i % 2 == 0:
                            o["secure_price"][g1] *= 1.5
                            o["community_price"][g1] *= 1.5
                        both(lambda e: e.upload_offers(o))
                    elif state == "every_list":
                        both(lambda e: e.upload_offers(flipped if i % 2 == 0 else offers))
                    order = ("A", "B", "C")[i % 3:] + ("A", "B", "C")[:i % 3]
                    for arm in order:
                        t0 = time.perf_counter()
                        if arm == "A":
                            arm_a()
                        elif arm == "B":
                            arm_b()
                        else:
                            got = arm_c()
                        t1 = time.perf_counter()
                        if i >= 5:
                            ts[arm].append((t1 - t0) * 1e3)
                    n_p, n_r, s, b, t = got
                    rs, rb, rt = rpk.results_region(xbuf, 1, N, 0)
                    assert n_p == P and np.array_equal(rs, s) and np.array_equal(rb, b) and np.array_equal(rt, t), (P, state, i)
                    if i >= 5:
                        nr.append(n_r)
                        nc.append(len(s))
                clock = sm_clock()
                sa, sb, sc = stat(ts["A"]), stat(ts["B"]), stat(ts["C"])
                row = {"P": P, "state": state, "A_list_count_slots_gather_top5_ms": sa, "B_select_pending_changed_gather_ms": sb,
                       "C_select_pending_changed_host_ms": sc, "n_reselected": stat(nr), "n_changed": stat(nc),
                       "B_vs_A_speedup_median": sa["median"] / sb["median"], "B_faster_than_A_outside_spread": sb["max"] < sa["min"],
                       "B_slower_than_A_outside_spread": sb["min"] > sa["max"], "B_regions_equal_C": True,
                       "sm_clock_mhz_after_timed_runs": clock}
                rows.append(row)
                print(json.dumps(row), flush=True)
    finally:
        eb.close()
        ec.close()
        pin.free()
    out = {"tool": "tools/select_pending_changed_gather_probe.py", "gpu": gpu, "G": G, "tracked_N": N, "runs": a.runs,
           "n_ranks": 1, "unmeasured": "the peer stores over NVLink (one rank, one local buffer)",
           "timing": "wall clock around each call (ends in a device synchronise), arms rotated, 5 warm-up rounds, median "
                     "[min, max] of the runs",
           "rows": rows}
    os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
    with open(a.out, "w") as f:
        json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
