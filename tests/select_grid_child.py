"""Child process of test_select_grid_gpu.py::test_capped_grid.  RPK_TUNE is read once per process, so the cap on row
tiles per launch of the packed / wide grid (gridtiles=N) runs in a process of its own.  With a small cap, a 100k-offer
table and batches of 1000 to 250 000 rows put tiles that hold rows into several launches, and the last of them (the one
that clears the group counts) into a later launch than the first: every launch after the first must start at its own
tile, and the tile tickets, done and the counts must carry across the launches and be zero again for the next call.

The synth 100k table is uploaded forced to each grid kind, and one context runs device selects of descending then
ascending batch sizes on it; every row of best (and top-5 on every other call) is checked against the oracle.  The
script asserts through persist_plan_model.py that each call spans the launches it is meant to, exits non-zero on the
first difference, and prints "ok <setting>" last."""
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
for p in (ROOT, HERE):
    if p not in sys.path:
        sys.path.insert(0, p)

import persist_plan_model as model  # noqa: E402
import rpk  # noqa: E402
import select_plan_cases as sc  # noqa: E402

KINDS = (("generic", 1), ("packed_pos", 3), ("packed", 2))
SIZES = (250_000, 50_000, 3_000, 50_000, 250_000, 1_000)  # R = 16, 2, 1, 2, 16, 1


def fail(what):
    print("FAIL", os.environ.get("RPK_TUNE"), what, flush=True)
    sys.exit(1)


def main():
    setting = os.environ.get("RPK_TUNE", "")
    cap = model.tune_value(setting, "gridtiles=")
    if cap <= 0:
        fail("no gridtiles= setting")
    sms = sc.sm_count()
    offers = sc.table("synth100k")
    G = len(offers["mem_gb"])
    dist = model.distinct(offers)
    pods, wb, wt = sc.batch("synth100k", max(SIZES), seed=5)
    with rpk.Engine(1) as eng:
        for force, kind in KINDS:
            with sc.forced(force):
                eng.upload_offers(offers)
            if eng.stats()["select_kernel_kind"] != kind:
                fail(f"{force}: kind {eng.stats()['select_kernel_kind']}, not {kind}")
            S = model.grid_segments(kind, G)[0]
            for i, P in enumerate(SIZES):
                p = sc.head(pods, P)
                R = model.rows_per_warp(P, sms)
                launches = model.grid_launches(P, R, S, grid_tiles=cap)
                last = model.valid_tiles(model.row_groups(kind, dist, p), R) - 1  # the tile that clears the counts
                if not (len(launches) >= 2 and last // cap >= 1):
                    fail(f"{force} P={P}: {len(launches)} launches, last tile with rows {last}")
                top5 = i % 2 == 0
                try:
                    sc.check(f"{force} P={P} R={R} gridtiles={cap}", *sc.run_device(eng, p, top5), wb[:P],
                             wt[:P] if top5 else None)
                except AssertionError as e:
                    fail(str(e))
                print(f"{force} P={P} R={R}: {len(launches)} launches, last tile with rows in launch "
                      f"{last // cap + 1}: ok", flush=True)
    print("ok", setting, flush=True)


if __name__ == "__main__":
    main()
