"""GPU tests of the pending results for one process per GPU (rpk_select_pending_changed_gather): each rank reselects the
pending slots of its own range and writes its changed rows into its region of every rank's exchange buffer.

On one GPU the ranks of a group are separate one-GPU ctxs on device 0 with the same history, each bound with its rank to
the group's flag arrays; their exchange buffers and flag arrays are torch tensors on device 0.  No kernel here waits for
another rank: the ranks are called in turn with the inline wait off, then the device is synchronised.  A reference ctx
with the same history calls rpk_select_pending_changed, and the regions concatenated in rank order must equal its output
bit for bit; its reported rows must equal rpk_select_slots on the same ctx, which runs no reselect kernel.  Every buffer
is sentinel-filled between guard words before a call and compared whole, so a store past a region's count shows.  The two-GPU cases at the end run the real group over NVLink (skipped on one GPU)."""
import ctypes as C

import numpy as np
import pytest

import rpk

pytestmark = pytest.mark.gpu

EINVAL, ESTATE = rpk._ffi.RPK_EINVAL, rpk._ffi.RPK_ESTATE
SENT = 0x5A5A5A5A
PADW = 16  # guard words before and after every exchange buffer; 64 bytes keeps the buffer 16-byte aligned
G = 3000
RESULTS_WORD0, RESULTS_CTR = 16, 34


def result_range(N, n, r):
    """the slots rank r of n owns: its share of the table's 16-slot units (rpk.h)"""
    units = (N + 15) // 16
    return min(units * r // n * 16, N), min(units * (r + 1) // n * 16, N)


def cuts(N, n):
    return sorted({b for r in range(n) for b in result_range(N, n, r)})


def pending_set(N, n, rng, frac):
    """a random fraction of the slots, plus the slots on both sides of every rank cut and of the first unit cuts"""
    s = set(np.flatnonzero(rng.random(N) < frac).tolist())
    for c in cuts(N, n) + list(range(16, min(N, 80), 16)):
        s.update(x for x in (c - 1, c) if 0 <= x < N)
    return np.array(sorted(s), np.uint32)


class Group:
    """n ranks as one-GPU ctxs on cuda:0 plus a reference ctx; every history call goes to all of them"""

    def __init__(self, n, N, cap=None):
        import torch

        self.n, self.N = n, N
        self.ranks = [rpk.Engine(1) for _ in range(n)]
        self.ref = rpk.Engine(1)
        self.cap = max(hi - lo for lo, hi in (result_range(N, n, r) for r in range(n))) if cap is None else cap
        self.words = self.ranks[0].results_xchg_bytes(n, self.cap) // 4
        self.mem = [torch.full((self.words + 2 * PADW,), SENT, dtype=torch.int32, device="cuda") for _ in range(n)]
        self.ptrs = [m.data_ptr() + 4 * PADW for m in self.mem]
        self.flags = torch.zeros((n, 64), dtype=torch.int32, device="cuda")
        for r, e in enumerate(self.ranks):
            e.peer_bind([self.flags[k].data_ptr() for k in range(n)], r)
        self.epoch = 0

    def all(self):
        return self.ranks + [self.ref]

    def history(self, fn):
        for e in self.all():
            fn(e)

    def close(self):
        for e in self.all():
            e.close()

    def expected_flags(self):
        want = np.zeros((self.n, 64), np.int32)
        want[:, RESULTS_WORD0:RESULTS_WORD0 + self.n] = self.epoch
        want[:, RESULTS_CTR] = self.epoch
        return want

    def expected_buffer(self, slots, best, top5):
        e = np.full(self.words + 2 * PADW, SENT, np.int32)
        body = e[PADW:PADW + self.words]
        for r in range(self.n):
            lo, hi = result_range(self.N, self.n, r)
            m = (slots >= lo) & (slots < hi)
            k = int(m.sum())
            body[r] = k
            reg = body[8 + r * 7 * self.cap:]
            reg[:k] = slots[m].view(np.int32)
            reg[self.cap:self.cap + k] = best[m]
            reg[2 * self.cap:2 * self.cap + 5 * k] = top5[m].reshape(-1)
        return e

    def step(self, what):
        """one call of every rank and of the reference; every check of the contract"""
        import torch

        for m in self.mem:
            m.fill_(SENT)
        torch.cuda.synchronize()
        counts = [e.select_pending_changed_gather(self.ptrs, self.cap, r) for r, e in enumerate(self.ranks)]
        torch.cuda.synchronize()
        self.epoch += 1
        n_p, n_r, slots, best, top5 = self.ref.select_pending_changed(self.N)
        assert sum(c[0] for c in counts) == n_p and sum(c[1] for c in counts) == n_r, f"{what}: counts {counts} vs ({n_p}, {n_r})"
        for r, (cp, cr) in enumerate(counts):
            assert cr <= cp, f"{what}: rank {r} reselected more than it has pending"
        bufs = [m.cpu().numpy() for m in self.mem]
        parts = [rpk.results_region(bufs[0][PADW:PADW + self.words], self.n, self.cap, r) for r in range(self.n)]
        got = [np.concatenate([p[i] for p in parts]) for i in range(3)]
        assert np.array_equal(got[0], slots), f"{what}: concatenated slots differ from rpk_select_pending_changed"
        assert np.array_equal(got[1], best) and np.array_equal(got[2], top5.reshape(-1, 5)), f"{what}: best / top5 differ"
        if len(slots):  # an independent reference: rpk_select_slots runs the gather, select and top-5 kernels, no reselect
            sb, st = self.ref.select_slots(slots, want_top5=True)
            assert np.array_equal(best, sb) and np.array_equal(top5.reshape(-1, 5), st), f"{what}: reported rows differ from rpk_select_slots"
        want = self.expected_buffer(slots, best, top5)
        for o, b in enumerate(bufs):
            if not np.array_equal(b, want):
                bad = np.flatnonzero(b != want)
                raise AssertionError(f"{what}: buffer {o} differs at {len(bad)} words, first {bad[:8] - PADW}")
        assert np.array_equal(self.flags.cpu().numpy(), self.expected_flags()), f"{what}: flag words"
        return n_p, n_r, slots


CASES = [(n, N) for n in (1, 2, 3, 4, 8) for N in sorted({15, 16 * n - 1, 16 * n + 1, 100_003})]


@pytest.mark.parametrize("n,N", CASES)
def test_ranks_equal_the_host_call(n, N):
    """first call, steady call, 1 % re-seeded, marks set and cleared, an offer upload, an identical re-upload, and a
    reset: after each, the regions concatenated in rank order are rpk_select_pending_changed's output"""
    rng = np.random.default_rng(1000 * n + N)
    g = Group(n, N)
    try:
        offers = rpk.synth.make_offers(G, correlated=True)
        pods = rpk.synth.make_pods(N, seed=N)
        every = np.arange(N, dtype=np.uint32)
        pend = pending_set(N, n, rng, 0.3)
        flags = np.zeros(N, np.uint8)
        flags[pend] = 1

        def setup(e):
            e.upload_offers(offers)
            e.pods_reset(N)
            e.pods_seed_slots(every, pods)
            e.pods_mark_pending(every, flags)

        g.history(setup)
        n_p, n_r, sl = g.step("first call")
        assert n_r == n_p == len(pend) and np.array_equal(sl, pend), "the first call reports every pending slot"
        n_p, n_r, sl = g.step("steady call")
        assert n_r == 0 and len(sl) == 0
        hit = np.sort(rng.choice(N, max(1, N // 100), replace=False)).astype(np.uint32)
        alt = rpk.synth.make_pods(N, seed=N + 1)
        g.history(lambda e: e.pods_seed_slots(hit, {k: np.ascontiguousarray(v[hit]) for k, v in alt.items()}))
        g.step("1 % re-seeded")
        on = pending_set(N, n, rng, 0.1)
        off = np.sort(rng.choice(pend, len(pend) // 3, replace=False)).astype(np.uint32)
        g.history(lambda e: e.pods_mark_pending(on, np.ones(len(on), np.uint8)))
        g.history(lambda e: e.pods_mark_pending(off, np.zeros(len(off), np.uint8)))
        g.step("marks set and cleared")
        other = rpk.synth.make_offers(G, seed=7, correlated=True)
        g.history(lambda e: e.upload_offers(other))
        g.step("offer upload")
        g.history(lambda e: e.upload_offers(other))
        n_p, n_r, sl = g.step("identical re-upload")
        assert n_r == n_p and len(sl) == 0, "an identical table reselects every pending slot and reports none"
        g.history(setup)
        n_p, n_r, sl = g.step("after a reset")
        assert n_r == n_p == len(pend) and np.array_equal(sl, pend)
        g.step("steady after the reset")
    finally:
        g.close()


def test_stats_and_launches():
    """a call that reselects counts one select (offer_scores += n_reselected * G) and is three launches; a steady call
    counts none and is two launches (the stale step, and the diff that publishes the zero count and signals)"""
    N = 20_001
    g = Group(1, N)
    try:
        e = g.ranks[0]
        e.upload_offers(rpk.synth.make_offers(G, correlated=True))
        e.pods_reset(N)
        e.pods_seed_slots(np.arange(N, dtype=np.uint32), rpk.synth.make_pods(N))
        e.pods_mark_pending(np.arange(0, N, 3, dtype=np.uint32), np.ones(len(range(0, N, 3)), np.uint8))
        s0, c0 = e.stats(), e.launch_count()
        n_p, n_r = e.select_pending_changed_gather(g.ptrs, g.cap, 0)
        s1 = e.stats()
        assert n_r == n_p == len(range(0, N, 3))
        assert e.launch_count() == c0 + 3, "a reselecting call is three launches (stale step, reselect, diff)"
        assert s1["select_calls"] == s0["select_calls"] + 1 and s1["offer_scores"] == s0["offer_scores"] + n_r * G
        c0 = e.launch_count()
        assert e.select_pending_changed_gather(g.ptrs, g.cap, 0) == (n_p, 0)
        assert e.launch_count() == c0 + 2 and e.stats()["select_calls"] == s1["select_calls"]
    finally:
        g.close()


# ---- refusals --------------------------------------------------------------------------------------------------------
def refused(g, eng, code, call, what):
    """call() raises RpkError(code) and moves no flag word, writes no buffer and launches nothing"""
    import torch

    torch.cuda.synchronize()
    flags, bufs, launches = g.flags.clone(), [m.clone() for m in g.mem], eng.launch_count()
    with pytest.raises(rpk.RpkError) as ei:
        call()
    assert ei.value.code == code, f"{what}: {ei.value}"
    torch.cuda.synchronize()
    assert torch.equal(g.flags, flags), f"{what}: a flag word moved"
    assert all(torch.equal(a, b) for a, b in zip(g.mem, bufs)), f"{what}: a buffer was written"
    assert eng.launch_count() == launches, f"{what}: launched"


def ready_engine(N, offers=True, table=True):
    e = rpk.Engine(1)
    if offers:
        e.upload_offers(rpk.synth.make_offers(G, correlated=True))
    if table:
        e.pods_reset(N)
        e.pods_seed_slots(np.arange(N, dtype=np.uint32), rpk.synth.make_pods(N))
        e.pods_mark_pending(np.arange(0, N, 2, dtype=np.uint32), np.ones(len(range(0, N, 2)), np.uint8))
    return e


N_REF = 10_007


@pytest.fixture
def two_ranks():
    g = Group(2, N_REF)
    e = ready_engine(N_REF)
    e.peer_bind([g.flags[k].data_ptr() for k in range(2)], 0)
    yield g, e
    e.close()
    g.close()


@pytest.mark.parametrize("case", ["cap", "n_ranks 0", "n_ranks 9", "my_rank -1", "my_rank n", "NULL buffer", "misaligned buffer", "shard"])
def test_argument_refusals(two_ranks, case):
    g, e = two_ranks
    lo, hi = result_range(N_REF, 2, 0)
    args = dict(xchg_ptrs=g.ptrs, cap=g.cap, my_rank=0)
    change = {"cap": dict(cap=hi - lo - 1), "n_ranks 0": dict(xchg_ptrs=[]), "n_ranks 9": dict(xchg_ptrs=g.ptrs * 4 + g.ptrs[:1]),
              "my_rank -1": dict(my_rank=-1), "my_rank n": dict(my_rank=2), "NULL buffer": dict(xchg_ptrs=[g.ptrs[0], 0]),
              "misaligned buffer": dict(xchg_ptrs=[g.ptrs[0], g.ptrs[1] + 4]), "shard": dict(shard=1)}[case]
    refused(g, e, EINVAL, lambda: e.select_pending_changed_gather(**{**args, **change}), case)
    e.select_pending_changed_gather(**args)  # the valid call is accepted and signals
    import torch

    torch.cuda.synchronize()
    assert int(g.flags[0, RESULTS_WORD0].item()) == 1 and int(g.flags[0, RESULTS_CTR].item()) == 1


@pytest.mark.parametrize("which", ["n_pending", "n_reselected", "d_xchg"])
def test_null_pointer_refusals(two_ranks, which):
    g, e = two_ranks
    xchg = (C.c_void_p * 2)(*g.ptrs)
    n = C.c_uint32(0)
    p = C.cast(C.byref(n), C.c_void_p)
    args = {"d_xchg": xchg, "n_pending": p, "n_reselected": p, which: None}

    def call():
        rc = e._lib.rpk_select_pending_changed_gather(e._ctx, 0, 2, 0, args["d_xchg"], g.cap, args["n_pending"], args["n_reselected"], None)
        e._check(rc)

    refused(g, e, EINVAL, call, which)


@pytest.mark.parametrize("missing", ["pod table", "offer table"])
def test_missing_tables(missing):
    g = Group(1, N_REF)
    e = ready_engine(N_REF, offers=missing != "offer table", table=missing != "pod table")
    try:
        e.peer_bind([g.flags[0].data_ptr()], 0)
        refused(g, e, ESTATE, lambda: e.select_pending_changed_gather(g.ptrs, g.cap, 0), missing)
    finally:
        e.close()
        g.close()


def test_range_mismatch_against_another_rank_and_the_host_call():
    """stored results belong to the range of the first call after rpk_pods_reset: another my_rank or n_ranks, or the host
    call's range on the same ctx, is refused with RPK_ESTATE until the next reset"""
    g = Group(2, N_REF)
    e = ready_engine(N_REF)
    try:
        e.peer_bind([g.flags[k].data_ptr() for k in range(2)], 0)
        e.select_pending_changed_gather(g.ptrs, g.cap, 0)
        refused(g, e, ESTATE, lambda: e.select_pending_changed_gather(g.ptrs, g.cap, 1), "another my_rank")
        refused(g, e, ESTATE, lambda: e.select_pending_changed(N_REF), "the host call over [0, N)")
        e.pods_reset(N_REF)
        e.pods_mark_pending(np.arange(0, N_REF, 2, dtype=np.uint32), np.ones(len(range(0, N_REF, 2)), np.uint8))
        e.select_pending_changed_gather(g.ptrs, g.cap, 1)  # a reset frees the range
        e.pods_reset(N_REF)
        e.pods_mark_pending(np.arange(0, N_REF, 2, dtype=np.uint32), np.ones(len(range(0, N_REF, 2)), np.uint8))
        e.select_pending_changed(N_REF)
        refused(g, e, ESTATE, lambda: e.select_pending_changed_gather(g.ptrs, g.cap, 0), "rank 0 of 2 after the host call")
        g1 = Group(1, N_REF)
        try:  # one rank owns the whole table: the host call's range
            e.peer_bind([g1.flags[0].data_ptr()], 0)
            n_p, n_r = e.select_pending_changed_gather(g1.ptrs, g1.cap, 0)
            assert n_p == len(range(0, N_REF, 2)) and n_r == 0
        finally:
            g1.close()
    finally:
        e.close()
        g.close()


def test_results_region_refuses_a_bad_region():
    w = np.zeros(8 + 2 * 7 * 4, np.int32)
    w[1] = 5
    with pytest.raises(ValueError):
        rpk.results_region(w, 2, 4, 1)  # count above cap
    with pytest.raises(ValueError):
        rpk.results_region(w, 2, 4, 2)
    assert [len(x) for x in rpk.results_region(w, 2, 4, 0)] == [0, 0, 0]


# ---- two GPUs ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("inline", [False, True])
def test_two_gpus(inline):
    """both shards of a 2-GPU ctx as the two ranks, IPC-allocated buffers on each GPU written over NVLink; the step is
    closed by rpk_peer_wait(4) or by the inline wait (turned on after the first call, which reselects every slot, so no
    later call allocates)"""
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
    with rpk.Engine(2) as eng, rpk.Engine(1) as ref:
        nbytes = eng.results_xchg_bytes(n, cap)
        xch = [eng.ipc_alloc(nbytes, shard=s)[0] for s in range(n)]
        flags = [eng.ipc_alloc(64 * 4, shard=s)[0] for s in range(n)]
        streams = []
        for s in range(n):
            eng.peer_bind(flags, s, shard=s)
            with torch.cuda.device(s):
                streams.append(torch.cuda.Stream(device=torch.device("cuda", s)))
        for e in (eng, ref):
            e.upload_offers(offers)
            e.pods_reset(N)
            e.pods_seed_slots(every, pods)
            e.pods_mark_pending(every, np.ones(N, np.uint8))
        for step in range(4):
            if step == 1:
                for e in (eng, ref):
                    e.pods_mark_pending(every, (rng.random(N) < 0.5).astype(np.uint8))
                for s in range(n):
                    eng.peer_inline_wait(inline, shard=s)
            if step == 2:
                hit = np.sort(rng.choice(N, N // 100, replace=False)).astype(np.uint32)
                alt = rpk.synth.make_pods(N, seed=5)
                for e in (eng, ref):
                    e.pods_seed_slots(hit, {k: np.ascontiguousarray(v[hit]) for k, v in alt.items()})
            for s in range(n):
                with torch.cuda.device(s):
                    eng.select_pending_changed_gather(xch, cap, s, shard=s, stream=streams[s].cuda_stream)
                    if not (inline and step >= 1):
                        eng.peer_wait(4, shard=s, stream=streams[s].cuda_stream)
            for st in streams:
                st.synchronize()
            _, _, slots, best, top5 = ref.select_pending_changed(N)
            for s in range(n):
                with torch.cuda.device(s):
                    words = peer.as_int32_tensor(xch[s], nbytes // 4, torch.device("cuda", s)).cpu().numpy()
                parts = [rpk.results_region(words, n, cap, r) for r in range(n)]
                got = [np.concatenate([p[i] for p in parts]) for i in range(3)]
                assert np.array_equal(got[0], slots) and np.array_equal(got[1], best) and np.array_equal(got[2], top5), f"step {step}: GPU {s}"
                with torch.cuda.device(s):
                    fw = peer.as_int32_tensor(flags[s], 64, torch.device("cuda", s)).cpu().numpy()
                assert (fw[RESULTS_WORD0:RESULTS_WORD0 + n] == step + 1).all() and fw[RESULTS_CTR] == step + 1
