#!/usr/bin/env python
"""The device form of the pending results for one process per GPU (rpk_select_pending_changed_device_gather), eager and
replayed from a CUDA graph, against the host-sync form (rpk_select_pending_changed_gather), on the GPU.

    python tools/select_pending_changed_device_gather_probe.py [--out profiles/h100_select_pending_changed_device_gather.json] [--runs 20]

One H100, G = 100k offers, a pod table of N = 1M slots seeded with synth.make_pods(1M), one rank (n_ranks = 1, one local
exchange buffer, a bound one-rank flag group, the inline wait on), as tools/select_pending_changed_gather_probe.py.  For
P pending slots in {4096, 125k, 1M} (a random ascending subset; every slot at 1M) three arms, each on a ctx of its own
with the same history, alternate in rotated order in one run:
  B  rpk_select_pending_changed_gather (one host synchronise inside, its inline wait ends it)
  D  rpk_select_pending_changed_device_gather, eager, then a stream synchronise
  E  a CUDA-graph replay of D's call, then a stream synchronise
in four states, each re-established before every round, outside the timed calls:
  steady          nothing changed since the last call
  seed_1pct       1 % of the pending rows re-seeded, alternately with new and with the old columns
  one_price       one offer's price toggled between x1 and x1.5 by an upload, the offer picked so that about 1 % of the lists
                  hold it
  every_list      the offer table toggled between two orders of the same offers: every non-empty list changes
An upload invalidates a captured graph, so in one_price and every_list E re-captures its call after each round's upload,
outside the timed call.  Wall clock around each call, which ends in a synchronise, 5 warm-up rounds, then the median
[min, max] of the runs.  After every round D's and E's regions must equal B's bit for bit.  The card's name and power
limit are read in the same run, and the SM clock right after each row's timed calls."""
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
from select_slots_probe import COLS, G, N, card, sm_clock, stat  # noqa: E402

STATES = ("steady", "seed_1pct", "one_price", "every_list")
ARMS = ("B", "D", "E")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "h100_select_pending_changed_device_gather.json"))
    ap.add_argument("--runs", type=int, default=20)
    a = ap.parse_args()
    import torch

    if not torch.cuda.is_available():
        raise SystemExit("select_pending_changed_device_gather_probe: no GPU (numbers here are only measured on the device)")
    gpu = card()
    offers = rpk.synth.make_offers(G)
    rev = np.arange(G)[::-1].copy()
    flipped = {k: np.ascontiguousarray(v[rev]) for k, v in offers.items()}
    pods = rpk.synth.make_pods(N)
    alt = rpk.synth.make_pods(N, seed=99)
    every = np.arange(N, dtype=np.uint32)
    rows = []
    rng = np.random.default_rng(31)
    dev = torch.device("cuda", 0)
    eng = {arm: rpk.Engine(1) for arm in ARMS}
    stream = torch.cuda.Stream(device=dev)
    graph = [None]
    try:
        words = eng["B"].results_xchg_bytes(1, N) // 4
        xbuf = {arm: torch.zeros(words, dtype=torch.int32, device=dev) for arm in ARMS}
        flags = {arm: torch.zeros(64, dtype=torch.int32, device=dev) for arm in ARMS}
        counts = {arm: torch.zeros(2, dtype=torch.int32, device=dev) for arm in ("D", "E")}
        for arm in ARMS:
            eng[arm].peer_bind([flags[arm].data_ptr()], 0)

        def each(fn):
            for arm in ARMS:
                fn(eng[arm])

        def call(arm):
            eng[arm].select_pending_changed_device_gather([xbuf[arm].data_ptr()], N, 0, d_counts=counts[arm],
                                                          stream=stream.cuda_stream)

        def capture():
            graph[0] = None
            torch.cuda.synchronize()
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g, stream=stream, capture_error_mode="thread_local"):
                call("E")
            graph[0] = g

        def run(arm):
            if arm == "B":
                eng["B"].select_pending_changed_gather([xbuf["B"].data_ptr()], N, 0, stream=stream.cuda_stream)
            elif arm == "D":
                call("D")
            else:
                with torch.cuda.stream(stream):
                    graph[0].replay()
            stream.synchronize()

        for P in (4096, 125_000, N):
            sl = every if P == N else np.sort(rng.choice(N, P, replace=False)).astype(np.uint32)
            graph[0] = None
            for arm in ARMS:
                eng[arm].peer_inline_wait(False)
            each(lambda e: e.upload_offers(offers))
            each(lambda e: e.pods_reset(N))
            each(lambda e: e.pods_seed_slots(every, pods))
            fl = np.zeros(N, np.uint8)
            fl[sl] = 1
            each(lambda e: e.pods_mark_pending(every, fl))
            lists = eng["B"].select_slots(sl, want_top5=True)[1]
            cnt = np.bincount(lists[lists >= 0].ravel(), minlength=G)
            g1 = int(np.argmin(np.abs(cnt - 0.01 * P)))  # the offer whose share of the lists is closest to 1 %
            hit = np.sort(rng.choice(sl, max(1, P // 100), replace=False)).astype(np.uint32)
            for arm in ARMS:  # the first call sizes every buffer before the inline wait is turned on
                if arm == "B":
                    run("B")
                else:
                    call(arm)
                    stream.synchronize()
                eng[arm].peer_inline_wait(True)
            for state in STATES:
                each(lambda e: e.upload_offers(offers))
                each(lambda e: e.pods_seed_slots(hit, {k: np.ascontiguousarray(pods[k][hit]) for k, _ in COLS}))
                capture()
                for arm in ARMS:
                    run(arm)
                ts = {arm: [] for arm in ARMS}
                nr, nc = [], []
                for i in range(a.runs + 5):
                    if state == "seed_1pct":
                        src = alt if i % 2 == 0 else pods
                        each(lambda e: e.pods_seed_slots(hit, {k: np.ascontiguousarray(src[k][hit]) for k, _ in COLS}))
                    elif state == "one_price":
                        o = {k: v.copy() for k, v in offers.items()}
                        if i % 2 == 0:
                            o["secure_price"][g1] *= 1.5
                            o["community_price"][g1] *= 1.5
                        each(lambda e: e.upload_offers(o))
                        capture()
                    elif state == "every_list":
                        each(lambda e: e.upload_offers(flipped if i % 2 == 0 else offers))
                        capture()
                    for arm in ARMS[i % 3:] + ARMS[:i % 3]:
                        t0 = time.perf_counter()
                        run(arm)
                        t1 = time.perf_counter()
                        if i >= 5:
                            ts[arm].append((t1 - t0) * 1e3)
                    rb = rpk.results_region(xbuf["B"], 1, N, 0)
                    for arm in ("D", "E"):
                        rx = rpk.results_region(xbuf[arm], 1, N, 0)
                        assert all(np.array_equal(x, y) for x, y in zip(rb, rx)), (P, state, i, arm)
                    assert counts["D"].tolist() == counts["E"].tolist() and counts["D"][0].item() == P, (P, state, i)
                    if i >= 5:
                        nr.append(int(counts["D"][1].item()))
                        nc.append(len(rb[0]))
                clock = sm_clock()
                sb, sd, se = stat(ts["B"]), stat(ts["D"]), stat(ts["E"])
                row = {"P": P, "state": state, "B_select_pending_changed_gather_ms": sb,
                       "D_device_gather_eager_sync_ms": sd, "E_device_gather_graph_replay_sync_ms": se,
                       "n_reselected": stat(nr), "n_changed": stat(nc),
                       "B_vs_D_speedup_median": sb["median"] / sd["median"], "B_vs_E_speedup_median": sb["median"] / se["median"],
                       "E_faster_than_B_outside_spread": se["max"] < sb["min"], "E_slower_than_B_outside_spread": se["min"] > sb["max"],
                       "D_faster_than_B_outside_spread": sd["max"] < sb["min"], "D_slower_than_B_outside_spread": sd["min"] > sb["max"],
                       "D_E_regions_equal_B": True, "sm_clock_mhz_after_timed_runs": clock}
                rows.append(row)
                print(json.dumps(row), flush=True)
    finally:
        graph[0] = None
        for e in eng.values():
            e.close()
    out = {"tool": "tools/select_pending_changed_device_gather_probe.py", "gpu": gpu, "G": G, "tracked_N": N, "runs": a.runs,
           "n_ranks": 1, "unmeasured": "the peer stores over NVLink (one rank, one local buffer); E's re-capture after an upload",
           "timing": "wall clock around each call (ends in a synchronise of the call's stream), arms rotated, 5 warm-up rounds, "
                     "median [min, max] of the runs",
           "rows": rows}
    os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
    with open(a.out, "w") as f:
        json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
