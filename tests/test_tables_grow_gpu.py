"""GPU tests of growing the pod table and the tracked status table in place (rpk_pods_grow, rpk_status_grow).

The contract: a ctx grown from N0 to N and a twin ctx reset at N from the start, given the same history of seeds, marks,
offer uploads and refreshes, return the same thing from every later call -- rpk_select_slots, rpk_select_pending and
rpk_select_pending_changed with its counts and rows.  Growth therefore reselects and reports nothing by itself: one extra
reselect means a stored result was lost.  The slots a grow adds read back, through the pod-table pointers of
rpk_test_capture_buffers, as the rows rpk_pods_reset writes, and the old slots as the twin's, bit for bit.  The
one-process-per-GPU forms clear their results on a grow (their peers' results live in other processes) and report every
pending slot of their new range once; the status table keeps its hashes across shard cuts."""
import ctypes as C

import numpy as np
import pytest

import oracle
import rpk
from test_graph_replay_across_calls_gpu import NAMES
from test_select_pending_changed_device_gather_gpu import Twins, make_rows, make_table
from test_select_pending_changed_gpu import call
from test_shared_device_ctx_gpu import shared_engine

pytestmark = pytest.mark.gpu

EINVAL, ENOMEM, ESTATE = rpk._ffi.RPK_EINVAL, rpk._ffi.RPK_ENOMEM, rpk._ffi.RPK_ESTATE
PT = ["pt_cols.mem", "pt_cols.vcpu", "pt_cols.ram", "pt_cols.max_price", "pt_cols.cloud", "pt_pending"]
PT_BYTES = [4, 4, 4, 8, 1, 1]
RESET_ROW = [np.int32(16), np.int32(0), np.int32(0), np.float64(0.5), np.uint8(0), np.uint8(0)]  # rpk_pods_reset's row
SCHEDULE = [15, 16, 17, 33, 1000, 100_003, 100_019, 110_000, 2**20 + 5]  # 110 000: inside the 25 % slack of 100 019
SHARD_SCHEDULE = [15, 33, 1000, 20_011, 100_003]  # one 16-slot unit, fewer than any shard count, to many per shard


def read_device(ptr, nbytes):
    """nbytes of device memory at ptr (a ctx-owned buffer) -> numpy uint8"""
    import torch

    torch.cuda.synchronize()
    out = np.empty(max(nbytes, 1), np.uint8)
    rc = C.CDLL("libcudart.so.12").cudaMemcpy(C.c_void_p(out.ctypes.data), C.c_void_p(ptr), C.c_size_t(nbytes), 2)
    assert rc == 0, f"cudaMemcpy D2H: {rc}"
    return out[:nbytes]


def pod_table(eng, shard, N):
    """the six columns of the pod table of shard `shard`, N slots, as numpy arrays of their element types"""
    bufs = eng.capture_buffers(shard)
    cols = []
    for name, b, proto in zip(PT, PT_BYTES, RESET_ROW):
        cols.append(read_device(bufs[NAMES.index(name)], N * b).view(np.asarray(proto).dtype))
    return cols


def check_table(what, grown, n_shards, twin, N0, N):
    """every replica of grown's table: [0, N0) equal to the twin's bit for bit, [N0, N) reset rows"""
    want = pod_table(twin, 0, N0)
    for s in range(n_shards):
        got = pod_table(grown, s, N)
        for name, g, w, proto in zip(PT, got, want, RESET_ROW):
            assert np.array_equal(g[:N0].view(np.uint8), w.view(np.uint8)), f"{what}: shard {s} {name} of [0, {N0}) changed"
            assert N == N0 or (g[N0:].view(np.uint8).reshape(N - N0, -1) == np.asarray(proto).reshape(1).view(np.uint8)).all(), \
                f"{what}: shard {s} {name} of [{N0}, {N}) is not the reset row"


def odd_rows(slots, seed):
    """pod rows for `slots` with NaN and -0.0 bounds and cloud bytes 2 and 255 among them"""
    pods = make_rows(max(len(slots), 1), seed)
    pods = {k: np.ascontiguousarray(v[:len(slots)]) for k, v in pods.items()}
    pods["max_price"][::11] = np.nan
    pods["max_price"][3::13] = -0.0
    pods["cloud"][::7] = 2
    pods["cloud"][1::9] = 255
    return pods


class PodTwins:
    """`grown` starts at N0 and grows; `twin` (one GPU) was reset at the last N of the schedule from the start"""

    def __init__(self, grown, n_shards, schedule, seed):
        self.grown, self.n_shards, self.twin = grown, n_shards, rpk.Engine(1)
        self.N, self.NF = schedule[0], schedule[-1]
        self.rng = np.random.default_rng(seed)
        self.offers = make_table(seed)
        self.history(lambda e: e.upload_offers(self.offers))
        self.grown.pods_reset(self.N)
        self.twin.pods_reset(self.NF)

    def history(self, fn):
        fn(self.grown)
        fn(self.twin)

    def close(self):
        self.grown.close()
        self.twin.close()

    def compare(self, what):
        """the three pending calls and a select over slots of the table, equal on both"""
        a, b = call(self.grown, self.NF), call(self.twin, self.NF)
        assert a[:2] == b[:2], f"{what}: (n_pending, n_reselected) {a[:2]} vs the twin's {b[:2]}"
        for x, y, name in zip(a[2:], b[2:], ("slots", "best", "top5")):
            assert np.array_equal(x, y), f"{what}: pending_changed {name} differ from the twin's"
        pa, pb = self.grown.select_pending(self.NF, want_top5=True), self.twin.select_pending(self.NF, want_top5=True)
        for x, y, name in zip(pa, pb, ("slots", "best", "top5")):
            assert np.array_equal(x, y), f"{what}: select_pending {name} differ from the twin's"
        sl = self.rng.integers(0, self.N, min(self.N, 5000)).astype(np.uint32)
        for x, y in zip(self.grown.select_slots(sl, want_top5=True), self.twin.select_slots(sl, want_top5=True)):
            assert np.array_equal(x, y), f"{what}: select_slots differ from the twin's"
        return a

    def stage(self, k):
        """seeds, marks, an offer change and the calls, over the slots [0, N) the grown table has"""
        N, rng = self.N, self.rng
        hit = np.unique(np.concatenate([rng.integers(0, N, max(1, N // 50)), [0, N - 1]])).astype(np.uint32)
        pods = odd_rows(hit, 100 + k)
        self.history(lambda e: e.pods_seed_slots(hit, pods))
        flip = np.unique(np.concatenate([rng.integers(0, N, max(1, N // 5)), [N - 1]])).astype(np.uint32)
        mark = (rng.random(len(flip)) < 0.6).astype(np.uint8)
        self.history(lambda e: e.pods_mark_pending(flip, mark))
        self.compare(f"stage {k} at N={N}: seeds and marks")
        if k % 3 == 1:  # a refresh the change window holds
            self.offers = {c: v.copy() for c, v in self.offers.items()}
            self.offers["secure_price"][[5, 700]] *= 0.5
            self.history(lambda e: e.refresh_offers(self.offers))
        elif k % 3 == 2:  # a refresh past the window: a wholesale invalidation
            self.offers = {c: v.copy() for c, v in self.offers.items()}
            self.offers["community_price"][::50] *= 1.5
            self.history(lambda e: e.refresh_offers(self.offers))
        elif k == 3:
            self.offers = make_table(k)
            self.history(lambda e: e.upload_offers(self.offers))
        self.compare(f"stage {k} at N={N}: after the offer change")
        got = self.compare(f"stage {k} at N={N}: steady")
        assert got[1] == 0, f"stage {k}: a steady call reselected {got[1]} slots"

    def grow(self, N):
        N0 = self.N
        self.grown.pods_grow(N)
        self.N = N
        check_table(f"grow {N0} -> {N}", self.grown, self.n_shards, self.twin, N0, N)
        got = self.compare(f"right after the grow {N0} -> {N}")
        assert got[1] == 0 and len(got[2]) == 0, f"grow {N0} -> {N}: reselected {got[1]}, reported {len(got[2])}"


def run_schedule(t, schedule):
    try:
        t.stage(0)
        for k, N in enumerate(schedule[1:], 1):
            t.grow(N)
            t.stage(k)
    finally:
        t.close()


def test_pod_table_one_gpu():
    """sizes off the 16-slot units, a partial last unit that becomes full (15 -> 16), a grow inside the slack"""
    run_schedule(PodTwins(rpk.Engine(1), 1, SCHEDULE, 1), SCHEDULE)


@pytest.mark.parametrize("n", [2, 3, 4, 8])
def test_pod_table_shards_of_one_gpu(n):
    """every owned range moves and the stored results change owner: from one 16-slot unit (fewer than the shards) up"""
    run_schedule(PodTwins(shared_engine(n), n, SHARD_SCHEDULE, n), SHARD_SCHEDULE)


def test_pod_table_two_gpus():
    """the same over real peer copies between two GPUs"""
    import torch

    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    run_schedule(PodTwins(rpk.Engine(2), 2, SHARD_SCHEDULE, 2), SHARD_SCHEDULE)


@pytest.mark.parametrize("R", [1, 2, 3])
def test_one_process_per_gpu_forms(R):
    """after a grow each rank's first call reports every pending slot of its new range, as a freshly reset ctx with the
    same rows and flags would (R = 1 keeps its results); later calls are steady, and a re-captured device form replays
    equal to the host-sync form"""
    N0, N1 = 1000, 100_003
    rng = np.random.default_rng(R)
    t = Twins(R, N1)  # exchange capacity for the grown ranges
    fresh = None
    try:
        offers = make_table(rpk.synth.SEED)
        pods = make_rows(N0, 5)
        every = np.arange(N0, dtype=np.uint32)
        flags = (rng.random(N0) < 0.4).astype(np.uint8)

        def setup(e):
            e.upload_offers(offers)
            e.pods_reset(N0)
            e.pods_seed_slots(every, pods)
            e.pods_mark_pending(every, flags)

        t.history(setup)
        t.step("first call")
        assert t.step("steady")[1] == 0
        t.history(lambda e: e.pods_grow(N1))
        new = np.arange(N0, N1, 7, dtype=np.uint32)
        t.history(lambda e: e.pods_mark_pending(new, np.ones(len(new), np.uint8)))
        if R > 1:  # the reference is a freshly reset ctx with the same rows and flags
            fresh = rpk.Engine(1)
            fresh.upload_offers(offers)
            fresh.pods_reset(N1)
            fresh.pods_seed_slots(every, pods)
            fresh.pods_mark_pending(every, flags)
            fresh.pods_mark_pending(new, np.ones(len(new), np.uint8))
            t.ref, fresh = fresh, t.ref
        n_p, n_r, _ = t.step("first call after the grow")
        assert n_p == int(flags.sum()) + len(new)
        assert n_r == (n_p if R > 1 else len(new)), f"R={R}: reselected {n_r} of {n_p} after the grow"
        assert t.step("steady after the grow")[1] == 0
        t.capture()
        hit = np.sort(rng.choice(N1, 500, replace=False)).astype(np.uint32)
        alt = make_rows(N1, 9)
        t.history(lambda e: e.pods_seed_slots(hit, {c: np.ascontiguousarray(v[hit]) for c, v in alt.items()}))
        assert t.step("replay after seeds", replay=True)[1] > 0
        assert t.step("steady replay", replay=True)[1] == 0
    finally:
        t.close()
        if fresh is not None:
            fresh.close()


def sweep_slots(table, slots, records):
    """oracle of rpk_status_diff_slots: the diff of the listed slots alone, against `table`'s state (updated)"""
    sub = oracle.StatusTable(len(slots), table.stride)
    sub.prev, sub.has_prev = table.prev[slots].copy(), table.has_prev[slots].copy()
    got = slots[sub.diff(records)]
    table.prev[slots], table.has_prev[slots] = sub.prev, sub.has_prev
    return got


def extend(table, N):
    """the oracle's table with never-seen slots up to N"""
    t = oracle.StatusTable(N, table.stride)
    t.prev[:table.N], t.has_prev[:table.N] = table.prev, table.has_prev
    return t


@pytest.mark.parametrize("stride", [16, 32, 64])
@pytest.mark.parametrize("n", [1, 2, 3, 4, 8])
def test_status_table(n, stride):
    """hashes kept across shard cuts; slot-list and whole-table sweeps after each grow equal the oracle; the old N is
    refused; no pointer of a device call moves"""
    eng = rpk.Engine(1) if n == 1 else shared_engine(n)
    try:
        sizes = [7, 40, 5003, 5100, 70_001]
        N0 = sizes[0]
        eng.status_reset(N0)
        table = oracle.StatusTable(N0, stride)
        recs = rpk.synth.make_status_records(N0, 0, stride=stride)
        assert np.array_equal(eng.status_diff(recs)[0], table.diff(recs))
        for k, N in enumerate(sizes[1:], 1):
            before = [eng.capture_buffers(s) for s in range(n)]
            eng.status_grow(N)
            assert [eng.capture_buffers(s) for s in range(n)] == before, "rpk_status_grow moved a device call's buffer"
            with pytest.raises(rpk.RpkError) as e:
                eng.status_diff(rpk.synth.make_status_records(N0, k, stride=stride))
            assert e.value.code == ESTATE
            table = extend(table, N)
            full = rpk.synth.make_status_records(N, k, 0.2, stride=stride)
            listed = np.unique(np.concatenate([np.arange(0, N, 3), [N0 - 1, N0, N - 1]])).astype(np.uint32)
            got, _ = eng.status_diff_slots(listed, np.ascontiguousarray(full[listed]))
            assert np.array_equal(got, sweep_slots(table, listed, np.ascontiguousarray(full[listed]))), f"slot sweep after grow to {N}"
            full = rpk.synth.make_status_records(N, k + 10, 0.3, stride=stride)
            assert np.array_equal(eng.status_diff(full)[0], table.diff(full)), f"whole-table sweep at N={N}"
            N0 = N
    finally:
        eng.close()


def test_status_grow_keeps_a_captured_device_sweep():
    """a captured rpk_status_diff_device replays correctly across rpk_status_grow (the sweep uses caller columns)"""
    import torch

    N, stride = 20_000, 32
    eng = rpk.Engine(1)
    try:
        eng.status_reset(100)
        recs = [torch.from_numpy(rpk.synth.make_status_records(N, k, 0.1, stride=stride)).cuda() for k in range(3)]
        d_rec = recs[0].clone()
        hashes = torch.zeros(N, dtype=torch.int64, device="cuda")
        idx = torch.empty(N, dtype=torch.int32, device="cuda")
        cnt = torch.zeros(1, dtype=torch.int32, device="cuda")
        eng.status_diff_device(d_rec, stride, hashes, idx, cnt)
        torch.cuda.synchronize()
        g = torch.cuda.CUDAGraph()
        s = torch.cuda.Stream()
        with torch.cuda.graph(g, stream=s, capture_error_mode="thread_local"):
            eng.status_diff_device(d_rec, stride, hashes, idx, cnt, stream=s.cuda_stream)
        table = oracle.StatusTable(N, stride)
        table.diff(recs[0].cpu().numpy())
        for k in (1, 2):
            eng.status_grow(100 + 5000 * k)
            d_rec.copy_(recs[k])
            torch.cuda.synchronize()
            g.replay()
            torch.cuda.synchronize()
            got = np.sort(idx[: int(cnt.item())].cpu().numpy().astype(np.uint32))
            assert np.array_equal(got, table.diff(recs[k].cpu().numpy())), f"replay {k} after a grow"
    finally:
        eng.close()


def refused(eng, code, fn, who):
    with pytest.raises(rpk.RpkError) as e:
        fn()
    assert e.value.code == code, str(e.value)
    assert who in str(e.value), f"the message does not name {who}: {e.value}"


def test_refusals():
    """every refusal names the entry point and leaves the ctx equal to its twin; N == N0 is a no-op; a pod table of
    2^32 - 1 slots (94 GB of columns) is more than one 80 GB card holds: RPK_ENOMEM with the ctx unchanged"""
    N = 3000
    eng = rpk.Engine(1)
    try:
        refused(eng, ESTATE, lambda: eng.pods_grow(10), "rpk_pods_grow")
        refused(eng, ESTATE, lambda: eng.status_grow(10), "rpk_status_grow")
    finally:
        eng.close()
    t = PodTwins(rpk.Engine(1), 1, [N, N], 5)
    try:
        t.stage(0)
        t.grown.status_reset(N)
        table = oracle.StatusTable(N, 32)
        recs = rpk.synth.make_status_records(N, 0, stride=32)
        assert np.array_equal(t.grown.status_diff(recs)[0], table.diff(recs))
        before = t.grown.capture_buffers()
        refused(t.grown, EINVAL, lambda: t.grown.pods_grow(N - 1), "rpk_pods_grow")
        refused(t.grown, EINVAL, lambda: t.grown.status_grow(N - 1), "rpk_status_grow")
        t.grown.pods_grow(N)
        t.grown.status_grow(N)
        assert t.grown.capture_buffers() == before, "a refused or empty grow moved a buffer"
        refused(t.grown, ENOMEM, lambda: t.grown.pods_grow(2**32 - 1), "rpk_pods_grow")
        assert t.grown.capture_buffers() == before, "a failed grow moved a buffer"
        check_table("after the refusals", t.grown, 1, t.twin, N, N)
        got = t.compare("after the refusals")
        assert got[1] == 0
        t.stage(1)
        recs = rpk.synth.make_status_records(N, 1, 0.3, stride=32)
        assert np.array_equal(t.grown.status_diff(recs)[0], table.diff(recs)), "tracked table after the refusals"
    finally:
        t.close()
