"""Small end-to-end run for compute-sanitizer (memcheck / racecheck / synccheck): every kernel kind, top-5,
the latency and the pipelined host paths, both status kernels.  Usage on the GPU box:
    compute-sanitizer --tool memcheck python tools/sanitize_smoke.py
"""
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import oracle  # noqa: E402
import rpk  # noqa: E402

ONLY_MULTI = os.environ.get("RPK_SANITIZE_ONLY_MULTI") == "1"  # the 2-GPU part alone (a 2-GPU box is charged twice)
eng = rpk.Engine(1)
offers = rpk.synth.make_offers(20_000, correlated=True)
for force in () if ONLY_MULTI else (None, "bitmap_grouped", "packed_pos", "packed", "generic"):
    os.environ.pop("RPK_FORCE_KERNEL", None)
    if force:
        os.environ["RPK_FORCE_KERNEL"] = force
    eng.upload_offers(offers)
    for P in (37, 5000, 140_000):  # latency path, one sub-batch, two pipelined sub-batches
        pods = rpk.synth.make_pods(P, seed=P)
        best, t5 = eng.select(pods, want_top5=True)
        ob, ot = oracle.select(offers, pods, n_threads=8)
        assert np.array_equal(best, ob) and np.array_equal(t5, ot), (force, P)
os.environ.pop("RPK_FORCE_KERNEL", None)
# the pod table: one seed, then a select by slot on the latency path and on the pipelined path (the gather indexes the
# table with caller input)
if not ONLY_MULTI:
    eng.upload_offers(offers)
    pods = pods_t = rpk.synth.make_pods(200_000, seed=11)
    eng.pods_reset(200_000)
    eng.pods_seed_slots(np.arange(200_000, dtype=np.uint32), pods)
    for n in (37, 140_000):
        sl = np.random.default_rng(n).integers(0, 200_000, n).astype(np.uint32)
        best, t5 = eng.select_slots(sl, want_top5=True)
        ob, ot = oracle.select(offers, {k: np.ascontiguousarray(v[sl]) for k, v in pods.items()}, n_threads=8)
        assert np.array_equal(best, ob) and np.array_equal(t5, ot), n
for stride in () if ONLY_MULTI else (16, 32, 64):
    tab = oracle.StatusTable(30_000, stride)
    e2 = rpk.Engine(1)
    for sweep, frac in enumerate([0.0, 0.2, 1.0]):
        recs = rpk.synth.make_status_records(30_000, sweep, frac, stride=stride)
        got, codes, hashes = e2.status_diff(recs, want_hashes=True, want_codes=True)
        want = tab.diff(recs)
        assert np.array_equal(got, want) and np.array_equal(hashes, oracle.record_hashes(recs))
        assert np.array_equal(codes, oracle.record_codes(recs)[want])
    e2.status_seed_slots(np.array([5, 77], np.uint32), np.ascontiguousarray(recs[[5, 77]]))
    sl = np.arange(3, 30_000, 7, dtype=np.uint32)  # the slot-list sweep: only the listed slots are compared
    nxt = rpk.synth.make_status_records(30_000, 3, 0.5, stride=stride)[sl]
    got, codes = e2.status_diff_slots(sl, nxt, want_codes=True)
    assert np.array_equal(got, sl[oracle.record_hashes(nxt) != oracle.record_hashes(np.ascontiguousarray(recs[sl]))])
    e2.close()
# the big-table build of the stream kernel (>= 4M slots), ragged last unit
for stride in () if ONLY_MULTI else (32, 16):
    N = (1 << 22) + 37
    e2 = rpk.Engine(1)
    base = rpk.synth.make_status_records(N, 0, stride=stride)
    e2.status_seed(base)
    nxt = rpk.synth.make_status_records(N, 2, 0.01, stride=stride)
    got, codes, _ = e2.status_diff(nxt, want_codes=True)
    tab = oracle.StatusTable(N, stride)
    tab.diff(base)
    want = tab.diff(nxt)
    assert np.array_equal(got, want) and np.array_equal(codes, oracle.record_codes(nxt)[want]), stride
    e2.close()
# one tick: selection and sweep enqueued together
e3 = rpk.Engine(1)
e3.upload_offers(offers)
pods = rpk.synth.make_pods(50_000, seed=3)
recs = rpk.synth.make_status_records(20_000, 0, stride=16)
tb, _, idx, codes = e3.tick(pods, recs)
ob, _ = oracle.select(offers, pods, want_top5=False, n_threads=8)
assert np.array_equal(tb, ob) and len(idx) == 20_000
e3.close()
# device entry points: two output vectors on one GPU (k_gather_push copies local -> local), twice on one scratch
import torch  # noqa: E402

eng.upload_offers(offers)
dev = torch.device("cuda", 0)
for P in (20_001, 70_003):
    pods = rpk.synth.make_pods(P, seed=P)
    d_pods = {k: torch.from_numpy(v).to(dev) for k, v in pods.items()}
    va, vb = torch.full((P + 3,), -9, dtype=torch.int32, device=dev), torch.full((P + 3,), -9, dtype=torch.int32, device=dev)
    ob, _ = oracle.select(offers, pods, want_top5=False, n_threads=8)
    for _ in range(2):
        eng.select_device_gather(d_pods, [va.data_ptr(), vb.data_ptr()], 3)  # slice starts 12 bytes into the vectors
        torch.cuda.synchronize()
        assert np.array_equal(va[3:].cpu().numpy(), ob) and np.array_equal(vb[3:].cpu().numpy(), ob), P
        assert int((va[:3] != -9).sum()) == 0 and int((vb[:3] != -9).sum()) == 0
# the device select over a slot list, whose entries nothing checks on the host: entries outside the table (a defined
# result, -1 and five -1) show that the gather stays inside it
if not ONLY_MULTI:  # the pod table was seeded above
    sl = np.random.default_rng(5).integers(0, 200_000, 30_001).astype(np.uint32)
    sl[[7, 30_000]] = [200_000, 0xFFFFFFFF]
    va, vb = torch.full((len(sl) + 3,), -9, dtype=torch.int32, device=dev), torch.full((len(sl) + 3,), -9, dtype=torch.int32, device=dev)
    t5 = torch.full((5 * len(sl),), -9, dtype=torch.int32, device=dev)
    eng.select_slots_device_gather(torch.from_numpy(sl.view(np.int32)).to(dev), [va.data_ptr(), vb.data_ptr()], 3, d_top5=t5)
    torch.cuda.synchronize()
    ok = sl < 200_000
    ob, ot = oracle.select(offers, {k: np.ascontiguousarray(v[sl[ok]]) for k, v in pods_t.items()}, n_threads=8)
    got, gt = va[3:].cpu().numpy(), t5.cpu().numpy().reshape(-1, 5)
    assert np.array_equal(got[ok], ob) and np.array_equal(gt[ok], ot) and (got[~ok] == -1).all() and (gt[~ok] == -1).all()
    assert np.array_equal(vb.cpu().numpy(), va.cpu().numpy())
eng.close()

# two GPUs: the fused push + signal + wait, and the sharded sweep's exchange (racecheck / memcheck see peer stores)
if torch.cuda.device_count() >= 2:
    e4 = rpk.Engine(2)
    e4.upload_offers(offers)
    pods = rpk.synth.make_pods(90_001, seed=9)
    ob, _ = oracle.select(offers, pods, want_top5=False, n_threads=8)
    for _ in range(2):
        b, _ = e4.select(pods)
        assert np.array_equal(b, ob)
    tab = oracle.StatusTable(50_001, 16)
    for sweep, frac in enumerate([0.0, 0.3]):
        recs = rpk.synth.make_status_records(50_001, sweep, frac, stride=16)
        got, codes, _ = e4.status_diff(recs, want_codes=True)
        want = tab.diff(recs)
        assert np.array_equal(got, want) and np.array_equal(codes, oracle.record_codes(recs)[want])
    e4.close()
    print("sanitize_smoke 2-GPU part ok")
print("sanitize_smoke ok")
