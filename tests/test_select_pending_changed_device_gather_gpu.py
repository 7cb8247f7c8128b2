"""GPU tests of the device form of the pending results for one process per GPU (rpk_select_pending_changed_device_gather):
the host-sync form's tick with the row count kept on the device, so it can be captured in a CUDA graph.

On one GPU the ranks of a group are separate one-GPU ctxs on device 0, each bound with its rank to the group's flag arrays,
called in turn with the inline wait off; then the device is synchronised.  Every rank has a twin ctx with the same history
that calls the host-sync form (rpk_select_pending_changed_gather) on buffers and flags of its own, and a reference ctx calls
rpk_select_pending_changed.  After each step the device form's buffers, flag words and counts must equal the twins' bit for
bit, the regions concatenated in rank order must equal the reference's output, and the reference's reported rows must equal
rpk_select_slots on the same ctx, which runs no reselect kernel.  Every buffer and count vector is sentinel-filled between
guard words before a call and compared whole.  The two-GPU case at the end runs the real group over NVLink (skipped on one
GPU)."""
import contextlib
import ctypes as C
import os

import numpy as np
import pytest

import rpk

pytestmark = pytest.mark.gpu

EINVAL, ESTATE = rpk._ffi.RPK_EINVAL, rpk._ffi.RPK_ESTATE
SENT = 0x5A5A5A5A
PADW = 16  # guard words before and after every exchange buffer; 64 bytes keeps the buffer 16-byte aligned
CPAD = 4   # guard words on each side of a rank's two count words
G = 3000
RESULTS_WORD0, RESULTS_CTR = 16, 34


def result_range(N, n, r):
    """the slots rank r of n owns: its share of the table's 16-slot units (rpk.h)"""
    units = (N + 15) // 16
    return min(units * r // n * 16, N), min(units * (r + 1) // n * 16, N)


@contextlib.contextmanager
def view_kind(kind):
    """RPK_FORCE_KERNEL is read by every offer upload and refresh: "generic" leaves the table without the bit-sliced view"""
    old = os.environ.pop("RPK_FORCE_KERNEL", None)
    if kind != "auto":
        os.environ["RPK_FORCE_KERNEL"] = kind
    try:
        yield
    finally:
        os.environ.pop("RPK_FORCE_KERNEL", None)
        if old is not None:
            os.environ["RPK_FORCE_KERNEL"] = old


class Side:
    """the exchange buffers and flag arrays of one group of n ranks on cuda:0"""

    def __init__(self, n, cap, engines):
        import torch

        self.words = engines[0].results_xchg_bytes(n, cap) // 4
        self.mem = [torch.full((self.words + 2 * PADW,), SENT, dtype=torch.int32, device="cuda") for _ in range(n)]
        self.ptrs = [m.data_ptr() + 4 * PADW for m in self.mem]
        self.flags = torch.zeros((n, 64), dtype=torch.int32, device="cuda")
        for r, e in enumerate(engines):
            e.peer_bind([self.flags[k].data_ptr() for k in range(n)], r)

    def fill(self):
        for m in self.mem:
            m.fill_(SENT)


class Twins:
    """n device-form ranks, their n host-sync twins and a reference ctx; every history call goes to all of them"""

    def __init__(self, n, N):
        import torch

        self.n, self.N = n, N
        self.dev = [rpk.Engine(1) for _ in range(n)]
        self.host = [rpk.Engine(1) for _ in range(n)]
        self.ref = rpk.Engine(1)
        self.cap = max(1, max(hi - lo for lo, hi in (result_range(N, n, r) for r in range(n))))
        self.d, self.h = Side(n, self.cap, self.dev), Side(n, self.cap, self.host)
        self.counts = torch.full((n, 2 + 2 * CPAD), SENT, dtype=torch.int32, device="cuda")
        self.graphs = None

    def d_counts(self, r):
        return self.counts[r, CPAD:CPAD + 2]

    def all(self):
        return self.dev + self.host + [self.ref]

    def history(self, fn):
        for e in self.all():
            fn(e)

    def close(self):
        self.graphs = None
        for e in self.all():
            e.close()

    def call(self, r):
        self.dev[r].select_pending_changed_device_gather(self.d.ptrs, self.cap, r, d_counts=self.d_counts(r))

    def capture(self):
        """one CUDA graph per rank of the device form's call (each rank has made one call of this shape before)"""
        import torch

        torch.cuda.synchronize()
        self.graphs = []
        stream = torch.cuda.Stream()
        for r in range(self.n):
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g, stream=stream, capture_error_mode="thread_local"):
                self.call(r)
            self.graphs.append(g)
        torch.cuda.synchronize()

    def step(self, what, replay=False):
        """one call of every rank (eager or a replay of its captured graph), of every twin and of the reference"""
        import torch

        self.d.fill()
        self.h.fill()
        self.counts.fill_(SENT)
        torch.cuda.synchronize()
        for r in range(self.n):
            if replay:
                self.graphs[r].replay()
            else:
                self.call(r)
        torch.cuda.synchronize()
        want_counts = [e.select_pending_changed_gather(self.h.ptrs, self.cap, r) for r, e in enumerate(self.host)]
        torch.cuda.synchronize()
        for o in range(self.n):
            if not torch.equal(self.d.mem[o], self.h.mem[o]):
                bad = torch.nonzero(self.d.mem[o] != self.h.mem[o]).flatten().cpu().numpy()
                raise AssertionError(f"{what}: buffer {o} differs from the host-sync form's at {len(bad)} words, first {bad[:8] - PADW}")
        assert torch.equal(self.d.flags, self.h.flags), f"{what}: flag words differ from the host-sync form's"
        cnt = self.counts.cpu().numpy()
        for r in range(self.n):
            assert tuple(int(x) for x in cnt[r, CPAD:CPAD + 2]) == want_counts[r], f"{what}: rank {r} counts {cnt[r]} vs {want_counts[r]}"
            assert (cnt[r, :CPAD] == SENT).all() and (cnt[r, CPAD + 2:] == SENT).all(), f"{what}: rank {r} wrote past its counts"
        n_p, n_r, slots, best, top5 = self.ref.select_pending_changed(max(self.N, 1))
        assert sum(c[0] for c in want_counts) == n_p and sum(c[1] for c in want_counts) == n_r, f"{what}: counts vs the host call"
        words = self.d.mem[0].cpu().numpy()[PADW:PADW + self.d.words]
        parts = [rpk.results_region(words, self.n, self.cap, r) for r in range(self.n)]
        got = [np.concatenate([p[i] for p in parts]) for i in range(3)]
        assert np.array_equal(got[0], slots), f"{what}: concatenated slots differ from rpk_select_pending_changed"
        assert np.array_equal(got[1], best) and np.array_equal(got[2], top5.reshape(-1, 5)), f"{what}: best / top5 differ"
        if len(slots):  # an independent reference: rpk_select_slots runs the gather, select and top-5 kernels, no reselect
            sb, st = self.ref.select_slots(slots, want_top5=True)
            assert np.array_equal(best, sb) and np.array_equal(top5.reshape(-1, 5), st), f"{what}: reported rows differ from rpk_select_slots"
        return n_p, n_r, slots


def changed_offers(offers, idx, seed):
    """offers with the prices of rows idx moved (a refresh that changes exactly those offers)"""
    rng = np.random.default_rng(seed)
    out = {k: v.copy() for k, v in offers.items()}
    for col in ("secure_price", "community_price"):
        out[col][idx] = np.round(rng.uniform(0.01, 0.6, len(idx)), 3)
    return out


def make_table(seed, rows64=False):
    """synth offers; rows64: 40 distinct mem values, so the bit-sliced view has 41 + 7 + 7 threshold words and rows
    of 64 words (synth alone gives 28 words, rows of 32)"""
    offers = rpk.synth.make_offers(G, seed=seed, correlated=True)
    if rows64:
        offers["mem_gb"] = (8 + 2 * (np.arange(G) * 7919 % 40)).astype(np.int32)
    return offers


def make_rows(N, seed):
    """synth pod rows with a few cloud bytes that are neither SECURE nor COMMUNITY (nothing is feasible: five -1)"""
    pods = rpk.synth.make_pods(N, seed=seed)
    pods["cloud"] = pods["cloud"].copy()
    pods["cloud"][::37] = 2
    pods["cloud"][5::101] = 255
    return pods


def history_steps(t, rng, step, kind="auto", rows64=False):
    """the call sequence every equality test runs; step(what) makes the calls and checks them"""
    N, n = t.N, t.n
    offers = make_table(rpk.synth.SEED, rows64)
    pods = make_rows(N, N)
    every = np.arange(N, dtype=np.uint32)
    flags = (rng.random(N) < 0.3).astype(np.uint8)
    for c in sorted({b for r in range(n) for b in result_range(N, n, r)}):  # both sides of every rank cut
        flags[[x for x in (c - 1, c) if 0 <= x < N]] = 1

    def setup(e):
        e.upload_offers(offers)
        e.pods_reset(N)
        e.pods_seed_slots(every, pods)
        e.pods_mark_pending(every, flags)

    with view_kind(kind):
        t.history(setup)
    if rows64:
        st = t.ref.stats()
        assert 32 < st["distinct_mem"] + st["distinct_vcpu"] + st["distinct_ram"] + 3 <= 64, st
    n_p, n_r, sl = step("first call")
    assert n_r == n_p == int(flags.sum())
    n_p, n_r, sl = step("steady call")
    assert n_r == 0 and len(sl) == 0
    hit = np.sort(rng.choice(N, max(1, N // 100), replace=False)).astype(np.uint32)
    alt = make_rows(N, N + 1)
    t.history(lambda e: e.pods_seed_slots(hit, {k: np.ascontiguousarray(v[hit]) for k, v in alt.items()}))
    step("1 % re-seeded")
    on = np.sort(rng.choice(N, max(1, N // 10), replace=False)).astype(np.uint32)
    off = np.flatnonzero(flags)[::3].astype(np.uint32)
    t.history(lambda e: e.pods_mark_pending(on, np.ones(len(on), np.uint8)))
    t.history(lambda e: e.pods_mark_pending(off, np.zeros(len(off), np.uint8)))
    step("marks set and cleared")
    few = changed_offers(offers, np.array([3, 500, 2000]), 1)
    with view_kind(kind):
        t.history(lambda e: e.refresh_offers(few))
    step("refresh within the window")
    many = changed_offers(few, np.arange(0, G, 97), 2)
    with view_kind(kind):
        t.history(lambda e: e.refresh_offers(many))
    step("refresh past the window")
    other = make_table(7, rows64)
    with view_kind(kind):
        t.history(lambda e: e.upload_offers(other))
    step("offer upload")
    with view_kind(kind):
        t.history(setup)
    n_p, n_r, sl = step("after a reset")
    assert n_r == n_p == int(flags.sum())
    step("steady after the reset")


CASES = [(n, N) for n in (1, 2, 3, 8) for N in sorted({15, 16 * n + 1, 100_003})]


@pytest.mark.parametrize("n,N", CASES)
def test_device_form_equals_the_host_sync_form(n, N):
    """the history of history_steps, with empty ranges at N = 15 and n > 1, on the bit-sliced view"""
    t = Twins(n, N)
    try:
        history_steps(t, np.random.default_rng(1000 * n + N), t.step)
    finally:
        t.close()


@pytest.mark.parametrize("n", [1, 3])
def test_device_form_on_the_wide_view(n):
    """the same history on tables without the bit-sliced view (one warp per row in the reselect)"""
    t = Twins(n, 100_003)
    try:
        history_steps(t, np.random.default_rng(7 + n), t.step, kind="generic")
    finally:
        t.close()


def test_device_form_on_64_word_rows():
    """the same history on a bit-sliced view of more than 32 threshold words (k_pod_reselect_top5<64>)"""
    t = Twins(3, 100_003)
    try:
        history_steps(t, np.random.default_rng(64), t.step, rows64=True)
    finally:
        t.close()


@pytest.mark.parametrize("kind", ["auto", "generic"])
def test_graph_replay(kind):
    """one call captured per rank; seeds and marks between replays are picked up, larger selects on the ctx leave the
    graph valid, and an offer refresh needs a re-capture"""
    import torch

    n, N = 2, 100_003
    rng = np.random.default_rng(11)
    t = Twins(n, N)
    try:
        offers = rpk.synth.make_offers(G, correlated=True)
        every = np.arange(N, dtype=np.uint32)
        with view_kind(kind):
            t.history(lambda e: e.upload_offers(offers))
        t.history(lambda e: e.pods_reset(N))
        pods = rpk.synth.make_pods(N, seed=3)
        half = (rng.random(N) < 0.5).astype(np.uint8)
        t.history(lambda e: e.pods_seed_slots(every, pods))
        t.history(lambda e: e.pods_mark_pending(every, half))
        t.step("first call (eager)")
        t.capture()
        n_p, n_r, _ = t.step("replay, nothing changed", replay=True)
        assert n_r == 0
        for k in range(3):
            hit = np.sort(rng.choice(N, 1000, replace=False)).astype(np.uint32)
            alt = rpk.synth.make_pods(N, seed=20 + k)
            t.history(lambda e: e.pods_seed_slots(hit, {c: np.ascontiguousarray(v[hit]) for c, v in alt.items()}))
            flip = np.sort(rng.choice(N, 2000, replace=False)).astype(np.uint32)
            mark = (rng.random(len(flip)) < 0.5).astype(np.uint8)
            t.history(lambda e: e.pods_mark_pending(flip, mark))
            n_p, n_r, _ = t.step(f"replay {k} after seeds and marks", replay=True)
            assert n_r > 0
        big = np.tile(every, 3)  # selects far larger than a rank's range grow and reallocate the select lanes
        for e in t.dev:
            e.select_slots(big, want_top5=True)
            e.select_slots_device(torch.from_numpy(big.astype(np.int32)).cuda(), torch.empty(len(big), dtype=torch.int32, device="cuda"),
                                  torch.empty(5 * len(big), dtype=torch.int32, device="cuda"))
        torch.cuda.synchronize()
        hit = np.sort(rng.choice(N, 1000, replace=False)).astype(np.uint32)
        alt = rpk.synth.make_pods(N, seed=30)
        t.history(lambda e: e.pods_seed_slots(hit, {c: np.ascontiguousarray(v[hit]) for c, v in alt.items()}))
        t.step("replay after larger selects on the same ctx", replay=True)
        with view_kind(kind):
            t.history(lambda e: e.refresh_offers(changed_offers(offers, np.array([10, 20]), 5)))
        t.capture()
        t.step("replay after a refresh and a re-capture", replay=True)
        t.step("steady replay", replay=True)
    finally:
        t.close()


def test_counts_stats_and_launches():
    """d_counts is optional; the call counts no select; a call with a non-empty range is three launches"""
    import torch

    N = 20_001
    t = Twins(1, N)
    try:
        t.history(lambda e: e.upload_offers(rpk.synth.make_offers(G, correlated=True)))
        t.history(lambda e: e.pods_reset(N))
        t.history(lambda e: e.pods_seed_slots(np.arange(N, dtype=np.uint32), rpk.synth.make_pods(N)))
        t.history(lambda e: e.pods_mark_pending(np.arange(0, N, 3, dtype=np.uint32), np.ones(len(range(0, N, 3)), np.uint8)))
        e = t.dev[0]
        s0, c0 = e.stats(), e.launch_count()
        e.select_pending_changed_device_gather(t.d.ptrs, t.cap, 0)  # no counts
        torch.cuda.synchronize()
        assert e.launch_count() == c0 + 3 and e.stats()["select_calls"] == s0["select_calls"]
        assert int(t.d.mem[0][PADW].item()) == len(range(0, N, 3))
        t.host[0].select_pending_changed_gather(t.h.ptrs, t.cap, 0)
        t.ref.select_pending_changed(N)
        t.step("steady with counts")
        assert e.stats()["select_calls"] == s0["select_calls"]
    finally:
        t.close()


# ---- refusals --------------------------------------------------------------------------------------------------------
def refused(side, eng, code, call, what):
    """call() raises RpkError(code) and moves no flag word, writes no buffer and launches nothing"""
    import torch

    torch.cuda.synchronize()
    flags, bufs, launches = side.flags.clone(), [m.clone() for m in side.mem], eng.launch_count()
    with pytest.raises(rpk.RpkError) as ei:
        call()
    assert ei.value.code == code, f"{what}: {ei.value}"
    assert "rpk_select_pending_changed_device_gather" in str(ei.value), f"{what}: the refusal names another call: {ei.value}"
    torch.cuda.synchronize()
    assert torch.equal(side.flags, flags), f"{what}: a flag word moved"
    assert all(torch.equal(a, b) for a, b in zip(side.mem, bufs)), f"{what}: a buffer was written"
    assert eng.launch_count() == launches, f"{what}: launched"


N_REF = 10_007


def ready_engine(N, offers=True, table=True):
    e = rpk.Engine(1)
    if offers:
        e.upload_offers(rpk.synth.make_offers(G, correlated=True))
    if table:
        e.pods_reset(N)
        e.pods_seed_slots(np.arange(N, dtype=np.uint32), rpk.synth.make_pods(N))
        e.pods_mark_pending(np.arange(0, N, 2, dtype=np.uint32), np.ones(len(range(0, N, 2)), np.uint8))
    return e


@pytest.fixture
def two_ranks():
    e = ready_engine(N_REF)
    cap = max(hi - lo for lo, hi in (result_range(N_REF, 2, r) for r in range(2)))
    side = Side(2, cap, [e])
    yield side, e, cap
    e.close()


@pytest.mark.parametrize("case", ["cap", "n_ranks 0", "n_ranks 9", "my_rank -1", "my_rank n", "NULL buffer", "misaligned buffer",
                                  "shard", "misaligned counts"])
def test_argument_refusals(two_ranks, case):
    import torch

    side, e, cap = two_ranks
    lo, hi = result_range(N_REF, 2, 0)
    counts = torch.zeros(4, dtype=torch.int32, device="cuda")
    args = dict(xchg_ptrs=side.ptrs, cap=cap, my_rank=0, d_counts=counts[:2])
    if case == "misaligned counts":  # the binding only passes whole int32 tensors: call the C-ABI with an odd address
        xchg = (C.c_void_p * 2)(*side.ptrs)
        refused(side, e, EINVAL, lambda: e._check(e._lib.rpk_select_pending_changed_device_gather(
            e._ctx, 0, 2, 0, xchg, cap, C.c_void_p(counts.data_ptr() + 2), None)), case)
    else:
        change = {"cap": dict(cap=hi - lo - 1), "n_ranks 0": dict(xchg_ptrs=[]), "n_ranks 9": dict(xchg_ptrs=side.ptrs * 4 + side.ptrs[:1]),
                  "my_rank -1": dict(my_rank=-1), "my_rank n": dict(my_rank=2), "NULL buffer": dict(xchg_ptrs=[side.ptrs[0], 0]),
                  "misaligned buffer": dict(xchg_ptrs=[side.ptrs[0], side.ptrs[1] + 4]), "shard": dict(shard=1, d_counts=None)}[case]
        refused(side, e, EINVAL, lambda: e.select_pending_changed_device_gather(**{**args, **change}), case)
    e.select_pending_changed_device_gather(**args)  # the valid call is accepted and signals
    torch.cuda.synchronize()
    assert int(side.flags[0, RESULTS_WORD0].item()) == 1 and int(side.flags[0, RESULTS_CTR].item()) == 1
    assert counts[:2].tolist() == [len(range(0, hi, 2)), len(range(0, hi, 2))]


def test_null_exchange_array(two_ranks):
    side, e, cap = two_ranks
    refused(side, e, EINVAL, lambda: e._check(e._lib.rpk_select_pending_changed_device_gather(e._ctx, 0, 2, 0, None, cap, None, None)),
            "d_xchg")


@pytest.mark.parametrize("missing", ["pod table", "offer table"])
def test_missing_tables(missing):
    e = ready_engine(N_REF, offers=missing != "offer table", table=missing != "pod table")
    try:
        side = Side(1, N_REF, [e])
        refused(side, e, ESTATE, lambda: e.select_pending_changed_device_gather(side.ptrs, N_REF, 0), missing)
    finally:
        e.close()


def test_range_mismatch():
    """stored results belong to the range of the first call after rpk_pods_reset, whichever form made it"""
    e = ready_engine(N_REF)
    try:
        cap = max(hi - lo for lo, hi in (result_range(N_REF, 2, r) for r in range(2)))
        side = Side(2, cap, [e])
        e.select_pending_changed_gather(side.ptrs, cap, 0)
        refused(side, e, ESTATE, lambda: e.select_pending_changed_device_gather(side.ptrs, cap, 1), "another my_rank")
        e.select_pending_changed_device_gather(side.ptrs, cap, 0)  # the host-sync form's range: accepted
        e.pods_reset(N_REF)
        e.select_pending_changed(N_REF)
        refused(side, e, ESTATE, lambda: e.select_pending_changed_device_gather(side.ptrs, cap, 0), "rank 0 of 2 after the host call")
    finally:
        e.close()


# ---- two GPUs ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("inline", [False, True])
def test_two_gpus(inline):
    """both shards of a 2-GPU ctx as the two ranks, IPC-allocated buffers on each GPU written over NVLink, closed by
    rpk_peer_wait(4) or by the inline wait (turned on after the first call, which sizes every buffer); each step equals the
    host-sync form of a twin 2-GPU ctx"""
    import torch

    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    peer = __import__("importlib").import_module("k8s-runpod-kubelet_b200.peer")
    n, N = 2, 100_003
    rng = np.random.default_rng(2 + inline)
    cap = max(hi - lo for lo, hi in (result_range(N, n, r) for r in range(n)))
    offers = rpk.synth.make_offers(G, correlated=True)
    pods = rpk.synth.make_pods(N)
    every = np.arange(N, dtype=np.uint32)
    with rpk.Engine(2) as eng, rpk.Engine(2) as twin:
        nbytes = eng.results_xchg_bytes(n, cap)
        sides = []
        for e in (eng, twin):
            xch = [e.ipc_alloc(nbytes, shard=s)[0] for s in range(n)]
            flags = [e.ipc_alloc(64 * 4, shard=s)[0] for s in range(n)]
            for s in range(n):
                e.peer_bind(flags, s, shard=s)
            sides.append((xch, flags))
        streams = []
        for s in range(n):
            with torch.cuda.device(s):
                streams.append(torch.cuda.Stream(device=torch.device("cuda", s)))
        counts = [torch.zeros(2, dtype=torch.int32, device=torch.device("cuda", s)) for s in range(n)]
        for e in (eng, twin):
            e.upload_offers(offers)
            e.pods_reset(N)
            e.pods_seed_slots(every, pods)
            e.pods_mark_pending(every, np.ones(N, np.uint8))
        for step in range(4):
            if step == 1:
                mark = (rng.random(N) < 0.5).astype(np.uint8)
                for e in (eng, twin):
                    e.pods_mark_pending(every, mark)
                    for s in range(n):
                        e.peer_inline_wait(inline, shard=s)
            if step == 2:
                hit = np.sort(rng.choice(N, N // 100, replace=False)).astype(np.uint32)
                alt = rpk.synth.make_pods(N, seed=5)
                for e in (eng, twin):
                    e.pods_seed_slots(hit, {k: np.ascontiguousarray(v[hit]) for k, v in alt.items()})
            want = []
            for e, (xch, _) in ((eng, sides[0]), (twin, sides[1])):
                for s in range(n):
                    with torch.cuda.device(s):
                        if e is eng:
                            e.select_pending_changed_device_gather(xch, cap, s, d_counts=counts[s], shard=s, stream=streams[s].cuda_stream)
                        else:
                            want.append(e.select_pending_changed_gather(xch, cap, s, shard=s, stream=streams[s].cuda_stream))
                        if not (inline and step >= 1):
                            e.peer_wait(4, shard=s, stream=streams[s].cuda_stream)
                for st in streams:
                    st.synchronize()
            for s in range(n):
                assert tuple(counts[s].tolist()) == want[s], f"step {step}: rank {s} counts"
                with torch.cuda.device(s):
                    got = peer.as_int32_tensor(sides[0][0][s], nbytes // 4, torch.device("cuda", s)).cpu().numpy()
                    ref = peer.as_int32_tensor(sides[1][0][s], nbytes // 4, torch.device("cuda", s)).cpu().numpy()
                for r in range(n):
                    a, b = rpk.results_region(got, n, cap, r), rpk.results_region(ref, n, cap, r)
                    assert all(np.array_equal(x, y) for x, y in zip(a, b)), f"step {step}: GPU {s} region {r}"
