"""Child process of test_ctx_lifetime_gpu.py: six cycles of create, use and close of one context, in a process of its
own so that free device memory moves with this context only.  Every cycle allocates each kind of buffer a context
holds: a 1M-offer bit-sliced table (with its transposed and per-mem-threshold views), the host select's lanes (600k
rows in three sub-batches, persistent kernel, top-5), the single-copy small batch, the device entry point's scratch, the
sweep's look-back state and changed list, a slot-list sweep and a tick.  After each cycle it prints free device memory;
it exits non-zero if a cycle's results differ from the first cycle's, or the small select from the oracle.  The last
two lines are {"free_bytes": [...]} and "ok"."""
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
for p in (ROOT, HERE):
    if p not in sys.path:
        sys.path.insert(0, p)

import numpy as np  # noqa: E402
import torch  # noqa: E402

import oracle  # noqa: E402
import rpk  # noqa: E402

CYCLES = 6
SLOTS = 1_000_000
STRIDE = 16
DEV_ROWS = 20_000


def fail(what):
    print("FAIL", what, flush=True)
    sys.exit(1)


def inputs():
    synth = rpk.synth
    recs = [synth.make_status_records(SLOTS, sweep, 0.1 if sweep else 0.0, stride=STRIDE) for sweep in range(3)]
    slots = np.arange(5, SLOTS, 7, dtype=np.uint32)
    return {"offers": synth.make_offers(1_000_000, correlated=True), "big": synth.make_pods(600_000),
            "small": synth.make_pods(1_000, seed=synth.SEED + 1), "dev": synth.make_pods(DEV_ROWS, seed=synth.SEED + 2),
            "recs": recs, "slots": slots, "slot_recs": np.ascontiguousarray(recs[1][slots])}


def cycle(x):
    out = {}
    eng = rpk.Engine(1)
    eng.upload_offers(x["offers"])
    out["big_best"], out["big_top5"] = eng.select(x["big"], want_top5=True)
    out["small_best"], _ = eng.select(x["small"])
    d = {k: None if v is None else torch.from_numpy(np.ascontiguousarray(v)).cuda() for k, v in x["dev"].items()}
    d_best = torch.empty(DEV_ROWS, dtype=torch.int32, device="cuda")
    torch.cuda.synchronize()
    eng.select_device(d, d_best)
    torch.cuda.synchronize()
    out["dev_best"] = d_best.cpu().numpy()
    out["diff_idx"], out["diff_codes"], _ = eng.status_diff(x["recs"][0], want_codes=True)
    out["slots_idx"], out["slots_codes"] = eng.status_diff_slots(x["slots"], x["slot_recs"], want_codes=True)
    out["tick_best"], _, out["tick_idx"], out["tick_codes"] = eng.tick(x["small"], x["recs"][2])
    eng.close()
    return out


def main():
    x = inputs()
    first, free = None, []
    for c in range(CYCLES):
        got = cycle(x)
        if first is None:
            first = got
            want, _ = oracle.select(x["offers"], x["small"], want_top5=False, n_threads=os.cpu_count() or 1)
            if not np.array_equal(got["small_best"], want) or not np.array_equal(got["tick_best"], want):
                fail("cycle 1: the 1000-row select differs from the oracle")
        else:
            bad = [k for k in first if not np.array_equal(first[k], got[k])]
            if bad:
                fail(f"cycle {c + 1}: {bad} differ from cycle 1")
        torch.cuda.synchronize()
        torch.cuda.empty_cache()
        free.append(torch.cuda.mem_get_info()[0])
        print(f"cycle {c + 1}: {free[-1] / 2**20:.1f} MiB free", flush=True)
    print(json.dumps({"free_bytes": free}), flush=True)
    print("ok", flush=True)


if __name__ == "__main__":
    main()
