#!/usr/bin/env python
"""What the exchange costs on the slot-list sweep, on one GPU.

    python tools/status_slots_gather_probe.py [--out profiles/h100_status_slots_gather.json] [--runs 25]

Three arms over the same resident records, alternated call by call:
  A  rpk_status_diff_slots_device_gather: the listed slots, changed list pushed into the exchange buffers;
  B  rpk_status_diff_slots_device: the listed slots, changed list and codes left on the GPU;
  C  rpk_status_diff_device_gather: the whole column, with the exchange.
Lists of 1 %, 10 % and 100 % of N = 1M and 16.8M slots, strides 16, 32 and 64.  The records alternate between two
tables that differ in 1 % of the slots, so every call reports about 1 % of what it compares and the exchange moves a
real changed list.  Setup as tools/top5_gather_probe.py runs a single process: a bound one-rank peer group with the
inline wait on and two exchange buffers, the second one local to the GPU, so the push and the signal run but cross no
NVLink.  CUDA events around each launch, L2 flushed (256 MiB write) before each, outside the event pair; median of the
runs.  Parity in the same run: after the last call A's region equals B's changed list and codes, and at 100 % also C's.
The card's name and power limit are read in the same run and stored with the numbers."""
import argparse
import json
import os
import statistics
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
import rpk  # noqa: E402
from status_slots_bench import card  # noqa: E402


def stats_us(ts):
    ts = sorted(ts)
    return {"median": statistics.median(ts), "min": ts[0], "max": ts[-1], "n": len(ts)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "h100_status_slots_gather.json"))
    ap.add_argument("--runs", type=int, default=25)
    a = ap.parse_args()
    import torch

    if not torch.cuda.is_available():
        raise SystemExit("status_slots_gather_probe: no GPU (numbers here are only measured on the device)")
    dev = torch.device("cuda", 0)
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
    rows, parity_ok = [], True
    gpu = card()
    with rpk.Engine(1) as eng:
        flags = eng.ipc_alloc(64 * 4)[0]
        eng.peer_bind([flags], 0)
        for N in (1 << 20, 1 << 24):
            for stride in (16, 32, 64):
                g = np.random.default_rng(N + stride)
                r0 = rpk.synth.make_status_records(N, 0, stride=stride)
                r1 = rpk.synth.make_status_records(N, 1, 0.01, stride=stride)
                recs = [torch.from_numpy(r).to(dev) for r in (r0, r1)]
                del r0, r1
                xb = eng.xchg_bytes(2, N)
                xch = [torch.zeros(xb // 4, dtype=torch.int32, device=dev) for _ in range(2)]
                ptrs = [x.data_ptr() for x in xch]
                cnt = torch.zeros(1, dtype=torch.int32, device=dev)
                idx = torch.empty(N, dtype=torch.int32, device=dev)
                code = torch.empty(N, dtype=torch.int16, device=dev)
                for pct in (1, 10, 100):
                    n = N * pct // 100
                    slots = np.arange(N, dtype=np.uint32) if pct == 100 else np.sort(g.choice(N, n, replace=False)).astype(np.uint32)
                    d_slots = torch.from_numpy(slots.view(np.int32)).to(dev)
                    sel = torch.from_numpy(slots.astype(np.int64)).to(dev)
                    subs = recs if pct == 100 else [r[sel].contiguous() for r in recs]
                    cols = {k: torch.zeros(N, dtype=torch.int64, device=dev) for k in "ABC"}
                    turn = {"A": 0, "B": 0, "C": 0}

                    def arm(k):
                        p = turn[k] & 1
                        turn[k] += 1
                        if k == "A":
                            eng.status_diff_slots_device_gather(d_slots, subs[p], stride, cols["A"], 0, ptrs, N, 0, cnt)
                        elif k == "B":
                            eng.status_diff_slots_device(d_slots, subs[p], stride, cols["B"], idx, cnt, d_changed_code=code)
                        else:
                            eng.status_diff_device_gather(recs[p], stride, cols["C"], 0, ptrs, N, 0, cnt)

                    for k in "ABC":  # size the scratch before the inline wait is on; the state is seen from here on
                        arm(k)
                    torch.cuda.synchronize()
                    eng.peer_inline_wait(True)
                    ts = {k: [] for k in "ABC"}
                    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
                    for i in range(3 * a.runs):
                        k = "ABC"[i % 3]
                        flush.fill_(i & 0xFF)
                        ev[0].record()
                        arm(k)
                        ev[1].record()
                        ev[1].synchronize()
                        ts[k].append(ev[0].elapsed_time(ev[1]) * 1e3)
                    eng.peer_inline_wait(False)
                    # parity: every arm has made the same number of calls, so one more call of each sees the same
                    # records against the same state: A's region (in both buffers) equals B's list, and at 100 % C's
                    arm("B")
                    torch.cuda.synchronize()
                    kb = int(cnt.item())
                    want = (idx[:kb].cpu().numpy(), code[:kb].cpu().numpy())
                    arm("A")
                    torch.cuda.synchronize()
                    ok = True
                    for x in xch:
                        h = x.cpu().numpy()
                        ka = int(h[0])
                        ok &= ka == kb and np.array_equal(h[8:8 + ka], want[0]) and np.array_equal(h[8 + 2 * N:].view(np.int16)[:ka], want[1])
                    if pct == 100:
                        arm("C")
                        torch.cuda.synchronize()
                        h = xch[1].cpu().numpy()
                        ok &= int(h[0]) == kb and np.array_equal(h[8:8 + kb], want[0])
                    parity_ok &= bool(ok)
                    sa, sb, sc_ = stats_us(ts["A"]), stats_us(ts["B"]), stats_us(ts["C"])
                    rows.append({"N": N, "stride": stride, "listed": n, "listed_pct": pct, "changed_per_call": kb,
                                 "A_slots_gather_us": sa, "B_slots_device_us": sb, "C_whole_table_gather_us": sc_,
                                 "A_minus_B_us": sa["median"] - sb["median"], "A_over_C": sa["median"] / sc_["median"],
                                 "parity_ok": bool(ok)})
                    print(f"N={N} stride={stride} {pct:3d}%: A {sa['median']:.1f} us  B {sb['median']:.1f} us  "
                          f"C {sc_['median']:.1f} us  changed {kb}  parity {ok}", flush=True)
                    del d_slots, sel, subs, cols
                del recs, xch, idx, code
                torch.cuda.empty_cache()
        eng.peer_bind(None, 0)
    out = {"tool": "tools/status_slots_gather_probe.py", "gpu": gpu, "gpu_after": card(), "parity_ok": parity_ok,
           "setup": "one GPU, bound one-rank peer group, inline wait on, two exchange buffers (the second GPU-local: the "
                    "push and the signal run, no NVLink); records alternate between two tables differing in 1 % of slots",
           "timing": f"CUDA events around one launch, L2 flushed (256 MiB write) before each outside the events, arms A, B, C "
                     f"alternated call by call, {a.runs} calls per arm; microseconds",
           "rows": rows}
    os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
    with open(a.out, "w") as f:
        json.dump(out, f, indent=1)
    print(f"wrote {a.out}; parity {'ok' if parity_ok else 'FAILED'}")
    if not parity_ok:
        sys.exit(3)


if __name__ == "__main__":
    main()
