#!/usr/bin/env python
"""What the gpuTypeIds lists cost on the sharded select path: the all-gather of the assignments alone
(rpk_select_device_gather, arm A) against the all-gather of the assignments and every row's top-5 list
(rpk_select_device_gather_top5, arm B), on the same resident pod columns, arms alternating call by call.

Setup as bench.py runs the gather: a bound peer group (rpk_peer_bind) with the inline wait on, so a call completes only
once every rank's slices have landed.  Under `torchrun --nproc_per_node N` the vectors are IPC-mapped across the N GPUs
(peer.exchange_peer_buffer) and each rank gathers its shard into all of them.  Run as a single process (N = 1) the group
has one rank and the second vector of each kind is a local one: the push kernel and the signal still run, the push
copies GPU-local instead of over NVLink.

Each call is timed with CUDA events on the calling stream; the L2 is flushed (256 MiB write) between calls, outside the
event pair.  Parity is checked in the same run: both arms' assignments are identical, arm B's lists equal
rpk_select(..., top5) on the same inputs, and 2 000 sampled rows equal the oracle.  Card name, power limit and SM clock
are read through NVML in the same run.  Rank 0 writes the JSON (default profiles/h100_top5_gather.json).

    python tools/top5_gather_probe.py [--calls 25] [--out PATH]
    torchrun --nproc_per_node 8 tools/top5_gather_probe.py
"""
import argparse
import importlib
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

G = 100_000
PODS = (125_000, 1_000_000)   # rows of the whole batch, sharded over the ranks (125k: one rank's share of 1M at N = 8)


def nvml_info(local_rank):
    """card name, power limit, current / max SM clock of this rank's GPU (None where NVML is unavailable)"""
    import torch

    out = {"card": torch.cuda.get_device_name(local_rank), "power_limit_w": None, "sm_mhz": None, "sm_max_mhz": None}
    try:
        import pynvml

        pynvml.nvmlInit()
        vis = os.environ.get("CUDA_VISIBLE_DEVICES")
        idx = int(vis.split(",")[local_rank]) if vis and vis.split(",")[local_rank].isdigit() else local_rank
        h = pynvml.nvmlDeviceGetHandleByIndex(idx)
        name = pynvml.nvmlDeviceGetName(h)
        out["card"] = name.decode() if isinstance(name, bytes) else name
        out["power_limit_w"] = pynvml.nvmlDeviceGetPowerManagementLimit(h) / 1000.0
        out["sm_mhz"] = pynvml.nvmlDeviceGetClockInfo(h, pynvml.NVML_CLOCK_SM)
        out["sm_max_mhz"] = pynvml.nvmlDeviceGetMaxClockInfo(h, pynvml.NVML_CLOCK_SM)
        out["source"] = "NVML"
    except Exception as e:  # noqa: BLE001 -- the numbers are still useful without it; the JSON says so
        out["source"] = f"NVML unavailable ({e})"
    return out


def stats_us(ms):
    us = sorted(1e3 * m for m in ms)
    return {"median": statistics.median(us), "min": us[0], "max": us[-1], "n": len(us)}


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--calls", type=int, default=25, help="timed calls per arm and size (at least 25)")
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--sample", type=int, default=2000, help="rows compared with the oracle per size")
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "h100_top5_gather.json"))
    args = ap.parse_args()
    args.calls = max(args.calls, 25)

    import numpy as np
    import torch
    import torch.distributed as dist

    import oracle

    pkg = importlib.import_module("k8s-runpod-kubelet_b200")
    peer = importlib.import_module("k8s-runpod-kubelet_b200.peer")
    synth = pkg.synth
    world = int(os.environ.get("WORLD_SIZE", "1"))
    rank = int(os.environ.get("RANK", "0"))
    local_rank = int(os.environ.get("LOCAL_RANK", "0"))
    torch.cuda.set_device(local_rank)
    dev = torch.device("cuda", local_rank)
    if world > 1:
        dist.init_process_group("nccl", device_id=dev)

    offers = synth.make_offers(G)
    eng = pkg.Engine(1, device_ids=[local_rank])
    eng.upload_offers(offers)
    n_out = max(world, 2)

    def vectors(nbytes):
        """-> [device pointer of every vector of one kind]: one per rank, or two local ones on a single GPU"""
        if world > 1:
            return peer.exchange_peer_buffer(eng, nbytes, rank, world)[1]
        return [eng.ipc_alloc(nbytes)[0] for _ in range(n_out)]

    flags = peer.exchange_peer_buffer(eng, 64 * 4, rank, world)[1] if world > 1 else [eng.ipc_alloc(64 * 4)[0]]
    eng.peer_bind(flags, rank)
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
    torch.cuda.set_stream(torch.cuda.Stream(device=dev, priority=-1))   # the select's stream priority, as in bench.py
    rng = np.random.default_rng(7)
    results, parity = {}, {}
    for P in sorted(set(PODS)):
        lo, hi = P * rank // world, P * (rank + 1) // world
        pods = synth.make_pods(P)
        d_pods = {k: torch.from_numpy(np.ascontiguousarray(v[lo:hi])).to(dev) for k, v in pods.items()}
        best_a, best_b, lists = vectors(P * 4), vectors(P * 4), vectors(P * 20)
        arm_a = lambda: eng.select_device_gather(d_pods, best_a, lo)
        arm_b = lambda: eng.select_device_gather(d_pods, best_b, lo, top5_ptrs=lists)
        arm_a(); arm_b()   # size the scratch before the inline wait is on (an allocating call synchronises its device)
        torch.cuda.synchronize()
        eng.peer_inline_wait(True)
        for _ in range(args.warmup):
            arm_a(); arm_b()
        torch.cuda.synchronize()
        ms = {"A": [], "B": []}
        for i in range(2 * args.calls):   # A, B, A, B, ...
            arm, fn = ("A", arm_a) if i % 2 == 0 else ("B", arm_b)
            flush.fill_(i & 0xFF)
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(); fn(); e1.record()
            e1.synchronize()
            ms[arm].append(e0.elapsed_time(e1))
        eng.peer_inline_wait(False)
        torch.cuda.synchronize()

        # parity, on this rank's copies of the full vectors (every rank holds all P rows after the gather)
        own = lambda ptrs, n: peer.as_int32_tensor(ptrs[rank if world > 1 else 0], n, dev).cpu().numpy()
        ba, bb, tb = own(best_a, P), own(best_b, P), own(lists, 5 * P).reshape(P, 5)
        hb, ht = eng.select(pods, want_top5=True)
        idx = np.sort(rng.choice(P, size=min(args.sample, P), replace=False))
        ob, ot = oracle.select(offers, {k: v[idx] for k, v in pods.items()}, want_top5=True, n_threads=8)
        copies_equal = True
        if world == 1:   # the second local vector of each kind received the push
            copies_equal = bool(np.array_equal(peer.as_int32_tensor(best_b[1], P, dev).cpu().numpy(), bb)
                                and np.array_equal(peer.as_int32_tensor(lists[1], 5 * P, dev).cpu().numpy().reshape(P, 5), tb))
        parity[str(P)] = {
            "best_A_equals_best_B": bool(np.array_equal(ba, bb)),
            "lists_B_equal_rpk_select_top5": bool(np.array_equal(tb, ht) and np.array_equal(bb, hb)),
            "sampled_rows_equal_oracle": bool(np.array_equal(bb[idx], ob) and np.array_equal(tb[idx], ot)),
            "pushed_copies_equal": copies_equal,
            "sampled_rows": int(len(idx)),
        }
        a, b = stats_us(ms["A"]), stats_us(ms["B"])
        results[str(P)] = {"rows_per_rank": hi - lo, "A_best_only_us": a, "B_best_and_top5_us": b,
                           "top5_list_and_its_push_us": b["median"] - a["median"]}
        print(f"rank {rank} P={P} ({hi - lo} rows here): A {a['median']:.1f} us [{a['min']:.1f}, {a['max']:.1f}], "
              f"B {b['median']:.1f} us [{b['min']:.1f}, {b['max']:.1f}], B - A {b['median'] - a['median']:.1f} us; "
              f"parity {parity[str(P)]}", flush=True)

    gpu = nvml_info(local_rank)
    rec = {"rank": rank, "gpu": gpu, "results": results, "parity": parity}
    recs = [rec]
    if world > 1:
        recs = [None] * world
        dist.all_gather_object(recs, rec)
    if rank == 0:
        ok = all(all(v for k, v in p.items() if k != "sampled_rows") for r in recs for p in r["parity"].values())
        doc = {
            "what": "sharded select: all-gather of the assignments (A, rpk_select_device_gather) vs the assignments plus "
                    "every row's top-5 list (B, rpk_select_device_gather_top5); B - A = the top-5 list and its push",
            "gpus": world,
            "setup": "bound peer group, inline wait on; " + ("vectors IPC-mapped across the GPUs" if world > 1 else
                     "one rank: the second vector of each kind is GPU-local (push runs, no NVLink)"),
            "G": G, "offers": "synth.make_offers(100000)", "pods": "synth.make_pods(P), rows sharded evenly over the ranks",
            "timing": f"CUDA events around each call, arms alternating, {args.calls} calls per arm after {args.warmup} warm-up "
                      "pairs, L2 flushed (256 MiB write) between calls outside the event pair; microseconds",
            "gpu": gpu, "parity_ok": ok, "ranks": recs,
        }
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(doc, f, indent=1)
        print(f"wrote {args.out}; parity {'ok' if ok else 'FAILED'}", flush=True)
    if world > 1:
        dist.barrier()
        dist.destroy_process_group()
    eng.close()


if __name__ == "__main__":
    main()
