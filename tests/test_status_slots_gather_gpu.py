"""GPU tests of the sharded slot-list sweep with exchange (rpk_status_diff_slots_device_gather) and of the whole-table
gather at the wide strides, against the oracle's state model (status_slots_model.diff_slots over oracle.StatusTable)
and oracle.record_codes.

The ranks of a group are emulated on one GPU: every "rank" is one call with its own hash column, idx_base and my_rank,
and all of them write into the same set of local exchange buffers, so the regions, counts and codes can be checked
word by word.  Exchange buffers and columns are pre-filled with sentinels and surrounded by guard words; a test
compares the WHOLE buffer with what the call may write, so a store beyond a region's count shows.  The multi-GPU
cases at the end run the real group over NVLink (skipped below 2, 4 or 8 GPUs)."""
import ctypes as C
import importlib

import numpy as np
import pytest

import oracle
import rpk
import status_cases as sc
import status_slots_model as ssm

pytestmark = pytest.mark.gpu

BIG = 4 << 20
SENT = 0x5A5A5A5A
PADW = 16  # guard words (int32) before and after every exchange buffer; 64 bytes keeps the buffer 16-byte aligned
GUARD64 = 0x5A5A5A5A5A5A5A5A
EINVAL = rpk._ffi.RPK_EINVAL


def sm_count() -> int:
    import torch

    return torch.cuda.get_device_properties(0).multi_processor_count


def peer_mod():
    return importlib.import_module("k8s-runpod-kubelet_b200.peer")


class XBufs:
    """one exchange buffer per rank of an n-rank group of capacity cap, all on cuda:0, sentinel-filled between guards"""

    def __init__(self, eng, n: int, cap: int):
        import torch

        self.n, self.cap = n, cap
        self.words = eng.xchg_bytes(n, cap) // 4
        self.mem = [torch.full((self.words + 2 * PADW,), SENT, dtype=torch.int32, device="cuda") for _ in range(n)]
        self.ptrs = [m.data_ptr() + 4 * PADW for m in self.mem]

    def fill(self):
        for m in self.mem:
            m.fill_(SENT)

    def expected(self, regions) -> np.ndarray:
        """the buffer contents (guards included) after every rank r wrote regions[r] = (ids, codes); None: rank r did
        not write"""
        e = np.full(self.words + 2 * PADW, SENT, np.int32)
        body = e[PADW:PADW + self.words]
        c16 = body[8 + self.n * self.cap:].view(np.uint16)
        for r, reg in enumerate(regions):
            if reg is None:
                continue
            ids, codes = reg
            body[r] = len(ids)
            body[8 + r * self.cap: 8 + r * self.cap + len(ids)] = np.asarray(ids, np.uint32).view(np.int32)
            c16[r * self.cap: r * self.cap + len(codes)] = codes
        return e

    def check(self, regions, what):
        import torch

        torch.cuda.synchronize()
        want = self.expected(regions)
        for o, m in enumerate(self.mem):
            got = m.cpu().numpy()
            if not np.array_equal(got, want):
                bad = np.nonzero(got != want)[0]
                raise AssertionError(f"{what}: buffer {o} differs at {len(bad)} words, first {bad[:8] - PADW} "
                                     f"(got {got[bad[:8]]}, want {want[bad[:8]]})")

    def concat(self, o: int = 0):
        """buffer o's regions concatenated in rank order -> (ids, codes)"""
        import torch

        torch.cuda.synchronize()
        body = self.mem[o].cpu().numpy()[PADW:PADW + self.words]
        c16 = body[8 + self.n * self.cap:].view(np.uint16)
        cnt = body[:self.n].astype(np.int64)
        ids = np.concatenate([body[8 + r * self.cap: 8 + r * self.cap + cnt[r]] for r in range(self.n)]).astype(np.uint32)
        codes = np.concatenate([c16[r * self.cap: r * self.cap + cnt[r]] for r in range(self.n)])
        return ids, codes


class Columns:
    """the hash columns of an n-rank split of N slots at `bounds`, each between int64 guard words"""

    def __init__(self, bounds):
        import torch

        self.bounds = bounds
        self.n = len(bounds) - 1
        self.mem, self.cols = [], []
        for r in range(self.n):
            k = bounds[r + 1] - bounds[r]
            m = torch.full((k + 4,), GUARD64, dtype=torch.int64, device="cuda")
            m[2:2 + k] = 0
            self.mem.append(m)
            self.cols.append(m[2:2 + k])

    def check(self, tab, what):
        import torch

        torch.cuda.synchronize()
        for m in self.mem:
            h = m.cpu().numpy()
            assert (h[:2] == GUARD64).all() and (h[-2:] == GUARD64).all(), f"{what}: guard words around a column written"
        full = np.concatenate([c.cpu().numpy() for c in self.cols]).view(np.uint64)
        assert np.array_equal(full, tab.prev_hashes()), f"{what}: hash columns differ from the model"


def ragged_bounds(N: int, n: int, rng) -> list:
    """n columns over [0, N), of uneven sizes (none empty)"""
    if n == 1:
        return [0, N]
    cuts = np.sort(rng.choice(np.arange(1, N), n - 1, replace=False))
    return [0, *[int(c) for c in cuts], N]


def to_dev(a, dtype=None):
    import torch

    a = np.ascontiguousarray(a)
    if dtype is not None:
        a = a.astype(dtype).view(np.int32) if dtype == np.uint32 else a.astype(dtype)
    return torch.from_numpy(a).cuda()


def list_sweep(eng, xb, cols, slots, recs, stride, tab, own: bool, what: str):
    """one sweep of every emulated rank over `slots` (ascending; records of the whole table `recs`): rank r is handed
    its own part of the list (own) or the whole list.  Checks every buffer word by word, the regions against the
    unsharded slot diff, the hash columns and the per-rank counts."""
    import torch

    sub = np.ascontiguousarray(recs[slots])
    want = ssm.diff_slots(tab, slots, sub)
    wcodes = oracle.record_codes(recs)[want]
    b = cols.bounds
    regions, cnts = [], []
    for r in range(cols.n):
        lo, hi = b[r], b[r + 1]
        p0, p1 = (int(np.searchsorted(slots, lo)), int(np.searchsorted(slots, hi))) if own else (0, len(slots))
        d_n = torch.full((1,), -1, dtype=torch.int32, device="cuda")
        eng.status_diff_slots_device_gather(to_dev(slots[p0:p1], np.uint32), to_dev(sub[p0:p1].reshape(-1)), stride,
                                            cols.cols[r], lo, xb.ptrs, xb.cap, r, d_n)
        cnts.append(d_n)
        m = (want >= lo) & (want < hi)
        regions.append((want[m], wcodes[m]))
    xb.check(regions, what)
    ids, codes = xb.concat()
    assert np.array_equal(ids, want) and np.array_equal(codes, wcodes), f"{what}: concatenated regions"
    assert [int(c.item()) for c in cnts] == [len(r[0]) for r in regions], f"{what}: d_n_changed"
    cols.check(tab, what)
    return want


# ---- emulated ranks on one GPU ----------------------------------------------------------------------------------------
@pytest.mark.parametrize("n_ranks", [1, 2, 3, 8])
@pytest.mark.parametrize("stride", [16, 32, 48, 64, 128, 256])
def test_emulated_ranks(stride, n_ranks):
    N = 40_003
    rng = np.random.default_rng(1000 * stride + n_ranks)
    lt = sc.LogicalTable(N, rng)
    bounds = ragged_bounds(N, n_ranks, rng)
    tab = oracle.StatusTable(N, stride)
    with rpk.Engine(1) as eng:
        cols = Columns(bounds)
        # (fraction of slots that change, list): random subsets of several sizes, the whole table, and contiguous runs
        # that straddle every column boundary
        straddle = np.unique(np.concatenate([np.arange(max(0, c - 70), min(N, c + 70)) for c in bounds]))
        plan = [(1.0, N // 2), (0.2, N), (0.05, 1000), (0.5, "all"), (0.3, "straddle"), (0.0, N // 3), (0.7, 1)]
        for i, (frac, n) in enumerate(plan):
            lt.step(stride, frac)
            recs = lt.records(stride)
            if n == "all":
                slots = np.arange(N, dtype=np.uint32)
            elif n == "straddle":
                slots = straddle.astype(np.uint32)
            else:
                slots = np.sort(rng.choice(N, n, replace=False)).astype(np.uint32)
            for own in (True, False):
                if not own:  # the global list sweeps records that moved on once more
                    lt.step(stride, frac / 2)
                    recs = lt.records(stride)
                xb = XBufs(eng, n_ranks, len(slots))
                list_sweep(eng, xb, cols, slots, recs, stride, tab, own, f"stride {stride} ranks {n_ranks} sweep {i} own {own}")


def test_edge_lists():
    """an empty list, a list outside a column, lists on the launch boundaries (63/64/65 entries, the saturation point
    of the 256-thread shape +- 1) and a 4M + 37-entry list, which takes the 1024-thread shape"""
    import torch

    sat = sm_count() * 8 * 64
    N = BIG + 37 + 4096
    stride = 16
    rng = np.random.default_rng(77)
    lt = sc.LogicalTable(N, rng)
    bounds = [0, 1_000_003, N]
    tab = oracle.StatusTable(N, stride)
    with rpk.Engine(1) as eng:
        cols = Columns(bounds)
        recs = lt.records(stride)
        # n_slots = 0: both ranks publish a zero count
        xb = XBufs(eng, 2, 1)
        for r in range(2):
            d_n = torch.full((1,), -1, dtype=torch.int32, device="cuda")
            eng.status_diff_slots_device_gather(torch.zeros(0, dtype=torch.int32, device="cuda"),
                                                torch.zeros(0, dtype=torch.uint8, device="cuda"), stride, cols.cols[r],
                                                bounds[r], xb.ptrs, 1, r, d_n)
            assert int(d_n.item()) == 0
        xb.check([(np.zeros(0, np.uint32), np.zeros(0, np.uint16))] * 2, "empty list")
        cols.check(tab, "empty list")
        # a list entirely inside rank 1's column: rank 0 reads nothing, reports nothing, touches nothing
        slots = np.arange(bounds[1] + 5, bounds[1] + 600, 3, dtype=np.uint32)
        xb = XBufs(eng, 2, len(slots))
        list_sweep(eng, xb, cols, slots, recs, stride, tab, False, "list outside rank 0's column")
        for n in (63, 64, 65, sat - 1, sat, sat + 1, BIG + 37):
            lt.step(stride, 0.3)
            recs = lt.records(stride)
            slots = np.sort(rng.choice(N, n, replace=False)).astype(np.uint32)
            xb = XBufs(eng, 2, n)
            list_sweep(eng, xb, cols, slots, recs, stride, tab, False, f"global list of {n}")
        # nearly the whole table, each rank handed its own part
        lt.step(stride, 0.1)
        recs = lt.records(stride)
        slots = np.sort(rng.choice(N, N - 1000, replace=False)).astype(np.uint32)
        xb = XBufs(eng, 2, len(slots))
        list_sweep(eng, xb, cols, slots, recs, stride, tab, True, "own parts of a list of N - 1000")


# ---- whole-table gather at the wide strides --------------------------------------------------------------------------
@pytest.mark.parametrize("stride,N,n_ranks", [(48, 70_001, 2), (64, 3_001, 3), (128, 70_001, 2), (256, 40_003, 8), (48, BIG + 37, 1)])
def test_whole_table_gather_wide_strides(stride, N, n_ranks):
    import torch

    rng = np.random.default_rng(stride + N)
    lt = sc.LogicalTable(N, rng)
    bounds = ragged_bounds(N, n_ranks, rng)
    tab = oracle.StatusTable(N, stride)
    cap = max(bounds[r + 1] - bounds[r] for r in range(n_ranks))
    with rpk.Engine(1) as eng:
        cols = Columns(bounds)
        xb = XBufs(eng, n_ranks, cap)
        for i, frac in enumerate((1.0, 0.05, 0.0)):
            lt.step(stride, frac)
            recs = lt.records(stride)
            want = tab.diff(recs)
            wcodes = oracle.record_codes(recs)[want]
            xb.fill()
            regions = []
            for r in range(n_ranks):
                lo, hi = bounds[r], bounds[r + 1]
                d_n = torch.full((1,), -1, dtype=torch.int32, device="cuda")
                eng.status_diff_device_gather(to_dev(recs[lo:hi].reshape(-1)), stride, cols.cols[r], lo, xb.ptrs, cap, r, d_n)
                m = (want >= lo) & (want < hi)
                regions.append((want[m], wcodes[m]))
                assert int(d_n.item()) == int(m.sum())
            xb.check(regions, f"stride {stride} N {N} sweep {i}")
            cols.check(tab, f"stride {stride} N {N} sweep {i}")


# ---- the bound signal ------------------------------------------------------------------------------------------------
def delta(*idx):
    d = np.zeros(64, np.int64)
    d[list(idx)] = 1
    return d


def test_bound_signal_once_per_call():
    """bound to a fresh flag array: every call -- an empty list included -- adds exactly 1 to words 8 and 33; unbound
    calls leave the flags alone"""
    import torch

    peer = peer_mod()
    dev = torch.device("cuda", 0)
    N = 30_001
    rng = np.random.default_rng(5)
    lt = sc.LogicalTable(N, rng)
    with rpk.Engine(1) as eng:
        flags = eng.ipc_alloc(64 * 4)[0]

        def words():
            torch.cuda.synchronize()
            return peer.as_int32_tensor(flags, 64, dev).cpu().numpy().astype(np.int64)

        col = torch.zeros(N, dtype=torch.int64, device=dev)
        tab = oracle.StatusTable(N, 48)
        eng.peer_bind([flags], 0)
        for stride, n in ((16, 3_001), (48, 0), (48, 20_000), (32, 0), (256, 5)):
            lt.step(stride, 0.3)
            recs = lt.records(stride)
            slots = np.sort(rng.choice(N, n, replace=False)).astype(np.uint32)
            sub = np.ascontiguousarray(recs[slots])
            xb = XBufs(eng, 1, max(n, 1))
            d_n = torch.full((1,), -1, dtype=torch.int32, device=dev)
            before = words()
            eng.status_diff_slots_device_gather(to_dev(slots, np.uint32), to_dev(sub.reshape(-1)), stride, col, 0, xb.ptrs, xb.cap, 0, d_n)
            assert np.array_equal(words() - before, delta(8, 33)), (stride, n, words()[:40])
            want = ssm.diff_slots(tab, slots, sub)
            xb.check([(want, oracle.record_codes(recs)[want])], f"bound, stride {stride}, {n} slots")
            assert int(d_n.item()) == len(want)
        eng.peer_bind(None, 0)
        before = words()
        for n in (0, 4_000):
            lt.step(32, 0.3)
            recs = lt.records(32)
            slots = np.sort(rng.choice(N, n, replace=False)).astype(np.uint32)
            sub = np.ascontiguousarray(recs[slots])
            xb = XBufs(eng, 1, max(n, 1))
            eng.status_diff_slots_device_gather(to_dev(slots, np.uint32), to_dev(sub.reshape(-1)), 32, col, 0, xb.ptrs, xb.cap, 0,
                                                torch.zeros(1, dtype=torch.int32, device=dev))
            want = ssm.diff_slots(tab, slots, sub)
            xb.check([(want, oracle.record_codes(recs)[want])], f"unbound, {n} slots")
        assert np.array_equal(words(), before)


# ---- refusals --------------------------------------------------------------------------------------------------------
def test_refusals_launch_nothing_and_touch_nothing():
    import torch

    peer = peer_mod()
    dev = torch.device("cuda", 0)
    N, n, stride = 8_192, 1_000, 16
    rng = np.random.default_rng(9)
    recs = sc.LogicalTable(N, rng).records(stride)
    slots = np.sort(rng.choice(N, n, replace=False)).astype(np.uint32)
    d_slots = to_dev(slots, np.uint32)
    with rpk.Engine(1) as eng:
        flags = eng.ipc_alloc(64 * 4)[0]
        eng.peer_bind([flags], 0)
        colm = torch.zeros(N + 2, dtype=torch.int64, device=dev)
        col = colm[:N]
        d_n = torch.zeros(1, dtype=torch.int32, device=dev)

        def d_recs(s, off=0):  # n records of s bytes starting `off` bytes into a buffer (zeros unless s is the table's stride)
            buf = torch.zeros(n * s + 16, dtype=torch.uint8, device=dev)
            if s == stride:
                buf[off:off + n * s] = torch.from_numpy(np.ascontiguousarray(recs[slots]).reshape(-1)).to(dev)
            return buf[off:off + n * s]

        xb = XBufs(eng, 2, n)
        eng.status_diff_slots_device_gather(d_slots, d_recs(stride), stride, col, 0, xb.ptrs, n, 0, d_n)  # sizes the scratch
        torch.cuda.synchronize()
        good = dict(d_slots=d_slots, d_records=d_recs(stride), stride=stride, d_hash_prev=col, idx_base=0, xchg_ptrs=xb.ptrs,
                    cap=n, my_rank=0, d_n_changed=d_n)
        cases = {
            "n_slots > cap": dict(cap=n - 1),
            "my_rank = n_ranks": dict(my_rank=2),
            "my_rank < 0": dict(my_rank=-1),
            "n_ranks 0": dict(xchg_ptrs=[]),
            "n_ranks 9": dict(xchg_ptrs=xb.ptrs * 4 + xb.ptrs[:1]),
            "NULL buffer": dict(xchg_ptrs=[xb.ptrs[0], 0]),
            "misaligned records": dict(d_records=d_recs(stride, 8)),
            "misaligned column": dict(d_hash_prev=colm[1:N + 1]),
            "stride 8": dict(stride=8, d_records=d_recs(8)),
            "stride 24": dict(stride=24, d_records=d_recs(24)),
            "stride 272": dict(stride=272, d_records=d_recs(272)),
        }
        torch.cuda.synchronize()
        snap = lambda: ([m.clone() for m in xb.mem], colm.clone(), d_n.clone(), peer.as_int32_tensor(flags, 64, dev).clone())
        for name, change in cases.items():
            before, launches = snap(), eng.launch_count()
            with pytest.raises(rpk.RpkError) as e:
                eng.status_diff_slots_device_gather(**{**good, **change})
            assert e.value.code == EINVAL, name
            torch.cuda.synchronize()
            after = snap()
            assert eng.launch_count() == launches, name
            assert all(torch.equal(a, b) for a, b in zip(before[0], after[0])), f"{name}: exchange buffer written"
            assert all(torch.equal(a, b) for a, b in zip(before[1:], after[1:])), f"{name}: column, count or flags written"
        # NULL d_slots with n_slots > 0 (only the C-ABI can pass it)
        xchg = (C.c_void_p * 2)(*xb.ptrs)
        before, launches = snap(), eng.launch_count()
        rc = eng._lib.rpk_status_diff_slots_device_gather(eng._ctx, 0, N, 0, n, None, good["d_records"].data_ptr(), stride,
                                                          col.data_ptr(), 2, xchg, n, 0, d_n.data_ptr(), None)
        assert rc == EINVAL and eng.launch_count() == launches
        after = snap()
        assert all(torch.equal(a, b) for a, b in zip(before[0] + list(before[1:]), after[0] + list(after[1:])))
        # the valid call still works and signals once
        w0 = peer.as_int32_tensor(flags, 64, dev).cpu().numpy().astype(np.int64)
        eng.status_diff_slots_device_gather(**good)
        torch.cuda.synchronize()
        assert np.array_equal(peer.as_int32_tensor(flags, 64, dev).cpu().numpy().astype(np.int64) - w0, delta(8, 33))


# ---- bad tensors in Python -------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind", ["host", "dtype", "strided", "short"])
def test_bad_tensor_is_refused(kind):
    """each tensor argument in turn replaced by its `kind` of bad stand-in (test_engine_args_gpu's buffers): TypeError or
    ValueError, no launch, no store; then the valid call is accepted"""
    import torch

    from test_engine_args_gpu import N, N_SLOTS, STRIDE, Buf, bad

    dev = torch.device("cuda", 0)
    recs = rpk.synth.make_status_records(N, 0, stride=STRIDE)
    slots = np.arange(0, 3 * N_SLOTS, 3, dtype=np.int32)
    with rpk.Engine(1) as eng:
        args = {"d_hash_prev": Buf(N, "int64", dev), "d_slots": Buf(N_SLOTS, "int32", dev, slots),
                "d_records": Buf(N_SLOTS * STRIDE, "uint8", dev, recs[slots].reshape(-1)), "d_n_changed": Buf(1, "int32", dev)}
        defining = {"d_hash_prev", "d_slots"}
        xch = Buf(eng.xchg_bytes(1, N_SLOTS) // 4, "int32", dev)

        def call(a):
            eng.status_diff_slots_device_gather(a["d_slots"], a["d_records"], STRIDE, a["d_hash_prev"], 0, [xch.valid().data_ptr()],
                                                N_SLOTS, 0, a["d_n_changed"])

        tried = 0
        for name, buf in args.items():
            t = bad(kind, buf, name in defining, [])
            if t is None:
                continue
            tried += 1
            launches = eng.launch_count()
            with pytest.raises((TypeError, ValueError)):
                call({**{k: b.valid() for k, b in args.items()}, name: t})
            torch.cuda.synchronize()
            touched = [k for k, b in args.items() if b.touched()] + (["exchange buffer"] if xch.touched() else [])
            assert eng.launch_count() == launches and not touched, f"{name} ({kind}): launched or stored into {touched}"
        assert tried
        launches = eng.launch_count()
        call({k: b.valid() for k, b in args.items()})
        torch.cuda.synchronize()
        # the hash column holds guard words, so every listed slot reports changed
        assert eng.launch_count() == launches + 1 and int(args["d_n_changed"].valid().item()) == N_SLOTS


# ---- CUDA graph ------------------------------------------------------------------------------------------------------
def test_graph_capture_replay():
    """after one call of the size each rank's call only enqueues: two ranks' calls captured once (one launch each),
    replayed over changing records"""
    import torch as t

    N, stride = 60_001, 48
    rng = np.random.default_rng(21)
    lt = sc.LogicalTable(N, rng)
    bounds = [0, 25_000, N]
    slots = np.sort(rng.choice(N, 30_000, replace=False)).astype(np.uint32)
    parts = [(int(np.searchsorted(slots, bounds[r])), int(np.searchsorted(slots, bounds[r + 1]))) for r in range(2)]
    tab = oracle.StatusTable(N, stride)
    with rpk.Engine(1) as eng:
        cols = Columns(bounds)
        xb = XBufs(eng, 2, max(p1 - p0 for p0, p1 in parts))
        d_slots = [to_dev(slots[p0:p1], np.uint32) for p0, p1 in parts]
        d_recs = [t.from_numpy(lt.records(stride, slots[p0:p1]).reshape(-1)).cuda() for p0, p1 in parts]
        d_n = [t.zeros(1, dtype=t.int32, device="cuda") for _ in range(2)]
        side = t.cuda.Stream()

        def step():
            for r in range(2):
                eng.status_diff_slots_device_gather(d_slots[r], d_recs[r], stride, cols.cols[r], bounds[r], xb.ptrs, xb.cap, r, d_n[r],
                                                    stream=side.cuda_stream)

        t.cuda.synchronize()
        with t.cuda.stream(side):
            step()
        side.synchronize()
        ssm.diff_slots(tab, slots, lt.records(stride, slots))
        g = t.cuda.CUDAGraph()
        launches = eng.launch_count()
        with t.cuda.graph(g, stream=side):
            step()
        assert eng.launch_count() - launches == 2
        for k in range(4):
            lt.step(stride, 0.1 * (k + 1))
            recs = lt.records(stride)
            for r, (p0, p1) in enumerate(parts):
                d_recs[r].copy_(t.from_numpy(np.ascontiguousarray(recs[slots[p0:p1]]).reshape(-1)))
            xb.fill()
            t.cuda.synchronize()
            g.replay()
            t.cuda.synchronize()
            want = ssm.diff_slots(tab, slots, np.ascontiguousarray(recs[slots]))
            wcodes = oracle.record_codes(recs)[want]
            regions = [(want[(want >= bounds[r]) & (want < bounds[r + 1])], wcodes[(want >= bounds[r]) & (want < bounds[r + 1])])
                       for r in range(2)]
            xb.check(regions, f"replay {k}")
            cols.check(tab, f"replay {k}")


# ---- multi-GPU -------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n,inline", [(2, False), (2, True), (4, True), (8, False), (8, True)])
def test_multi_gpu_slot_gather(n, inline):
    """The one-process-per-GPU shape inside one process: every shard sweeps its slot list with
    rpk_status_diff_slots_device_gather into every shard's IPC-allocated exchange buffer, and rpk_peer_wait(2) closes
    the step -- or, with the inline wait, the signalling warp does.  Two buffer sets, issue order reversed every other
    step, ragged columns, stride 48; steps 0, 1 and 4 hand each rank its own sub-list, steps 2 and 3 the global list.
    Every GPU must end with the oracle's whole changed list and codes."""
    import torch

    if torch.cuda.device_count() < n:
        pytest.skip(f"needs {n} GPUs")
    peer = peer_mod()
    NS, stride = 70_001, 48
    rng = np.random.default_rng(n)
    lt = sc.LogicalTable(NS, rng)
    bounds = ragged_bounds(NS, n, rng)
    sizes = [NS // 2, NS, 777, NS // 3, 1]
    cap = max(sizes)
    with rpk.Engine(n) as eng:
        xb = eng.xchg_bytes(n, cap)
        xch = [[eng.ipc_alloc(xb, shard=s)[0] for s in range(n)] for _ in range(2)]   # [set][shard]
        flags = [eng.ipc_alloc(64 * 4, shard=s)[0] for s in range(n)]
        sides, d_hash, d_n = [], [], []
        for s in range(n):
            dev = torch.device("cuda", s)
            with torch.cuda.device(s):
                sides.append(torch.cuda.Stream(device=dev))
                d_hash.append(torch.zeros(bounds[s + 1] - bounds[s], dtype=torch.int64, device=dev))
                d_n.append(torch.zeros(1, dtype=torch.int32, device=dev))
            eng.peer_bind(flags, s, shard=s)
        tab = oracle.StatusTable(NS, stride)
        for step in range(5):
            par = step & 1
            own = (step // 2) & 1 == 0
            if step == 1:   # only after one call has sized the scratch (one host thread drives every shard)
                for s in range(n):
                    eng.peer_inline_wait(inline, shard=s)
            waits = not (inline and step >= 1)
            lt.step(stride, 0.3)
            recs = lt.records(stride)
            slots = np.sort(rng.choice(NS, sizes[step], replace=False)).astype(np.uint32)
            sub = np.ascontiguousarray(recs[slots])
            inputs = []
            for s in range(n):
                p0, p1 = (int(np.searchsorted(slots, bounds[s])), int(np.searchsorted(slots, bounds[s + 1]))) if own else (0, len(slots))
                with torch.cuda.device(s):
                    dev = torch.device("cuda", s)
                    inputs.append((torch.from_numpy(slots[p0:p1].view(np.int32)).to(dev), torch.from_numpy(sub[p0:p1].reshape(-1)).to(dev)))
            for s in range(n):
                torch.cuda.synchronize(s)
            for s in (range(n) if step & 1 else reversed(range(n))):   # issue order must not matter
                with torch.cuda.device(s):
                    eng.status_diff_slots_device_gather(inputs[s][0], inputs[s][1], stride, d_hash[s], bounds[s], xch[par], cap, s, d_n[s],
                                                        shard=s, stream=sides[s].cuda_stream)
                    if waits:
                        eng.peer_wait(2, shard=s, stream=sides[s].cuda_stream)
            for st in sides:
                st.synchronize()
            want = ssm.diff_slots(tab, slots, sub)
            wcodes = oracle.record_codes(recs)[want]
            for s in range(n):
                with torch.cuda.device(s):
                    xv = peer.as_int32_tensor(xch[par][s], xb // 4, torch.device("cuda", s)).cpu().numpy()
                counts = xv[:n].astype(np.int64)
                idx = np.concatenate([xv[8 + r * cap: 8 + r * cap + counts[r]] for r in range(n)]).astype(np.uint32)
                c16 = xv[8 + n * cap:].view(np.uint16)
                codes = np.concatenate([c16[r * cap: r * cap + counts[r]] for r in range(n)])
                assert np.array_equal(idx, want), f"step {step} (own lists: {own}): GPU {s} changed list"
                assert np.array_equal(codes, wcodes), f"step {step} (own lists: {own}): GPU {s} codes"
            hashes = np.concatenate([h.cpu().numpy() for h in d_hash]).view(np.uint64)
            assert np.array_equal(hashes, tab.prev_hashes()), f"step {step}: hash columns"
