"""Child process of test_select_plans_gpu.py::test_tuned_plan.  RPK_TUNE (stagekb=, ipw=, k0ctas=, pdl=off) is read
once per process, so every setting runs in a process of its own: this script asserts through persist_plan_model.py
that each of its cases reaches the plan the setting is meant to produce, runs it through the named entry point and
exits non-zero on the first difference from the oracle; the last line is "ok <setting>"."""
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


def fail(what):
    print("FAIL", os.environ.get("RPK_TUNE"), what, flush=True)
    sys.exit(1)


def check(ok, what):
    if not ok:
        fail(what)


# (table, rows, entry point, top-5, what the plan must be); rows "ipw1-edge": the least batch with direct items at ipw=1
CASES = {
    # slice staging, one sub-range per stage: 49 stages x 12 row groups = 588 queues, several per CTA
    "stagekb=4": [("synth100k", 40_000, "host", True, lambda pl, q, sms: pl.slice and (pl.S, pl.per) == (49, 1) and q == 588 > sms),
                  ("synth100k", 40_000, "device", False, lambda pl, q, sms: pl.slice and pl.per == 1 and q > sms)],
    # price staging, one sub-range per stage: 74 stages x 2 clouds = 148 queues
    "stagekb=1": [("synth150k", 40_000, "device", True, lambda pl, q, sms: not pl.slice and (pl.S, pl.per) == (74, 1) and q == 148 > sms),
                  ("synth150k", 20_000, "host", False, lambda pl, q, sms: not pl.slice and pl.per == 1 and q == 148)],
    # qspan = 1: every sub-range is an item of its own, ten tickets per row block
    "ipw=64": [("synth20k", 40_000, "host", True, lambda pl, q, sms: pl.qspan == 1 and pl.tickets_per_block == pl.nsub == 10),
               ("synth20k", 40_000, "device", False, lambda pl, q, sms: pl.qspan == 1 and pl.tickets_per_block == 10)],
    # direct items over 49 sub-ranges from about 135k rows, merged items one row below that
    "ipw=1": [("synth100k", "ipw1-edge", "device", True, lambda pl, q, sms: pl.direct and pl.nsub == 49),
              ("synth100k", "ipw1-edge-1", "device", False, lambda pl, q, sms: not pl.direct and pl.tickets_per_block == 2),
              ("synth100k", "ipw1-edge", "host", False, lambda pl, q, sms: pl.direct)],
    # K0 with one CTA / three CTAs looping over every 512-row chunk
    "k0ctas=1": [("synth20k", 100_000, "host", True, lambda pl, q, sms: pl.k0_blocks == 1),
                 ("synth20k", 100_000, "device", False, lambda pl, q, sms: pl.k0_blocks == 1)],
    "k0ctas=3": [("synth20k", 100_000, "device", True, lambda pl, q, sms: pl.k0_blocks == 3),
                 ("synth20k", 100_000, "host", False, lambda pl, q, sms: pl.k0_blocks == 3)],
    # plain launches instead of programmatic dependent launches
    "pdl=off": [("synth20k", 40_000, "host", True, lambda pl, q, sms: pl.S == 1),
                ("synth100k", 200_000, "device", True, lambda pl, q, sms: pl.slice and not pl.direct)],
}


def main():
    setting = os.environ.get("RPK_TUNE", "")
    stage_kb, ipw, k0 = model.tune_from_env(setting)
    sms = sc.sm_count()
    edge = (ipw * sms * model.PWARPS - 1) * model.RPI + 1 if ipw else 0
    with rpk.Engine(1) as eng:
        loaded = None
        for name, rows, entry, top5, regime in CASES[setting]:
            P = {"ipw1-edge": edge, "ipw1-edge-1": edge - 1}.get(rows, rows)
            offers = sc.table(name)
            pods = sc.pods_for(name, P, seed=3)
            dist = model.distinct(offers)
            pl = model.plan(len(offers["mem_gb"]), P, [len(d) for d in dist], sms, stage_kb=stage_kb, items_per_warp=ipw,
                            k0ctas=k0)
            check(model.persistent(P), f"{name} {P}: the batch does not take the persistent kernel")
            if entry == "host":
                check(model.host_sub_batches(P) == [P], f"{name} {P}: several host sub-batches")
            check(regime(pl, model.queues(pl, dist, pods), sms), f"{name} {P} {entry}: plan {vars(pl)}")
            if loaded != name:
                eng.upload_offers(offers)
                loaded = name
            wb, wt = sc.expected(offers, pods)
            run = sc.run_host if entry == "host" else sc.run_device
            try:
                sc.check(f"{name} {P} rows {entry}", *run(eng, pods, top5), wb, wt)
            except AssertionError as e:
                fail(str(e))
            print(f"{name} {P} rows {entry} top5={top5}: ok", flush=True)
    print("ok", setting, flush=True)


if __name__ == "__main__":
    main()
