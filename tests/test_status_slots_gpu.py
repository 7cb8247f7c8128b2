"""GPU tests of the slot-list status diff (rpk_status_diff_slots / rpk_status_diff_slots_device) against the oracle's
state model (status_slots_model.diff_slots over oracle.StatusTable) and oracle.record_codes.

List lengths sit on every boundary of the launch code, which picks its shape from the list length exactly as it does
from N for a whole table: the streaming unit (64 entries), the point where the small-shape streaming grid saturates
(one 8-warp CTA per SM, one 64-entry unit per warp) and the 1024-thread shape from 4M entries up (up to stride 64).
Wide strides also take lengths ragged against blocks of 512 entries (strides 48 / 64) or 256 (above): one block
± 1, and 34 and 1025 blocks + 1."""
import ctypes as C

import numpy as np
import pytest

import oracle
import rpk
import status_cases as sc
import status_slots_model as ssm

pytestmark = pytest.mark.gpu

BIG = 4 << 20


def sm_count() -> int:
    import torch

    return torch.cuda.get_device_properties(0).multi_processor_count


def list_lengths(stride: int) -> list:
    sat = sm_count() * 8 * 64
    lengths = [0, 1, 63, 64, 65, sat - 1, sat, sat + 1]
    if stride <= 64:  # a 4M-entry table of the widest records would take gigabytes of host memory
        lengths.append(BIG + 37)
    if stride > 32:
        block = 512 if stride <= 64 else 256
        lengths += [block - 1, block, block + 1, 34 * block + 1, 1025 * block + 1]
    return lengths


def check_codes(codes, recs, changed):
    if codes is not None:
        assert np.array_equal(codes, oracle.record_codes(recs)[changed]), "codes differ from record_codes"


@pytest.mark.parametrize("stride", sc.STRIDES)
def test_slots_every_stride(stride):
    lengths = list_lengths(stride)
    N = max(lengths) + 1000
    rng = np.random.default_rng(stride)
    lt = sc.LogicalTable(N, rng)
    lt.step(stride, 1.0)
    with rpk.Engine(1) as eng:
        eng.status_reset(N)
        tab = oracle.StatusTable(N, stride)
        recs = lt.records(stride)
        eng.status_seed(recs)
        tab.seed(recs)
        lists = [np.sort(rng.choice(N, n, replace=False)) for n in lengths]
        lists += [np.sort(rng.choice(N, max(1, N // 1000), replace=False)), np.sort(rng.choice(N, N // 2, replace=False)),
                  np.arange(N), np.array([0, N // 3, N - 1])]
        for i, slots in enumerate(lists):
            lt.step(stride, 0.3)
            recs = lt.records(stride)
            for codes in (False, True):
                sub = np.ascontiguousarray(recs[slots])
                got, gcodes = eng.status_diff_slots(slots, sub, want_codes=codes)
                want = ssm.diff_slots(tab, slots, sub)
                assert np.array_equal(got, want), (stride, len(slots), codes)
                check_codes(gcodes, recs, want)
        # never-seen slots (after reset): every listed slot reports, the others stay never seen
        eng.status_reset(N)
        tab.reset(N)
        slots = np.sort(rng.choice(N, 5000, replace=False))
        got, gcodes = eng.status_diff_slots(slots, np.ascontiguousarray(recs[slots]), want_codes=True)
        assert np.array_equal(got, slots)
        ssm.diff_slots(tab, slots, np.ascontiguousarray(recs[slots]))
        check_codes(gcodes, recs, got)
        # unlisted state untouched: a whole-table diff agrees with the model
        got, gcodes, _ = eng.status_diff(recs, want_codes=True)
        want = tab.diff(recs)
        assert np.array_equal(got, want) and len(got) == N - len(slots)
        assert eng.stats()["status_calls"] > 0


@pytest.mark.parametrize("stride", [16, 32, 64, 256])
def test_identity_list_equals_full_diff(stride):
    N = 100_003
    lt = sc.LogicalTable(N, np.random.default_rng(stride + 1))
    with rpk.Engine(1) as a, rpk.Engine(1) as b:
        a.status_reset(N)
        b.status_reset(N)
        ident = np.arange(N, dtype=np.uint32)
        for frac in (1.0, 0.0, 0.01, 0.5):
            lt.step(stride, frac)
            recs = lt.records(stride)
            want, wcodes, _ = a.status_diff(recs, want_codes=True)
            got, gcodes = b.status_diff_slots(ident, recs, want_codes=True)
            assert np.array_equal(got, want) and np.array_equal(gcodes, wcodes), frac
        sb = b.stats()
        assert sb["status_records"] == 4 * N


# ---- call sequences on one context ---------------------------------------------------------------------------------
class Program:
    """One engine, one logical table, the model of the engine's table and of a caller-owned device column swept
    through rpk_status_diff_slots_device."""

    def __init__(self, N: int, seed: int):
        import torch

        self.torch = torch
        self.N, self.seed = N, seed
        self.rng = np.random.default_rng(seed)
        self.lt = sc.LogicalTable(N, self.rng)
        self.eng = rpk.Engine(1)
        self.tab = oracle.StatusTable(N, 16)
        self.col = torch.zeros(N, dtype=torch.int64, device="cuda")
        self.ctab = oracle.StatusTable(N, 16)
        self.idx = torch.empty(max(N, 1), dtype=torch.int32, device="cuda")
        self.code = torch.empty(max(N, 1), dtype=torch.int16, device="cuda")
        self.n = torch.zeros(1, dtype=torch.int32, device="cuda")
        self.offers = rpk.synth.make_offers(300, correlated=True)
        self.pods = rpk.synth.make_pods(64, seed=seed)
        self.eng.upload_offers(self.offers)
        self.best = oracle.select(self.offers, self.pods)[0]
        self.log = []

    def close(self):
        self.eng.close()

    def check(self, ok, what):
        if not ok:
            raise AssertionError(f"{what}\nprogram seed {self.seed}, N {self.N}; operations:\n  " + "\n  ".join(self.log))

    def pick(self):
        n = int(self.rng.choice([0, 1, max(1, self.N // 100), self.N // 2, self.N]))
        return np.sort(self.rng.choice(self.N, n, replace=False)).astype(np.uint32)

    def run(self, op, stride, frac):
        t = self.torch
        self.lt.step(stride, frac)
        recs = self.lt.records(stride)
        eng, tab, N = self.eng, self.tab, self.N
        self.log.append(f"{op} stride {stride} frac {frac}")
        if op == "reset":
            eng.status_reset(N)
            tab.reset(N)
        elif op == "seed":
            eng.status_seed(recs)
            tab.seed(recs)
        elif op == "seed_slots":
            slots = self.pick()
            eng.status_seed_slots(slots, np.ascontiguousarray(recs[slots]))
            tab.seed_slots(slots, recs[slots])
        elif op in ("diff", "diff_codes"):
            got, codes, _ = eng.status_diff(recs, want_codes=True)
            want = tab.diff(recs)
            self.check(np.array_equal(got, want), f"{op}: changed list differs")
            self.check(np.array_equal(codes, oracle.record_codes(recs)[want]), f"{op}: codes differ")
        elif op in ("slots", "slots_codes"):
            slots = self.pick()
            sub = np.ascontiguousarray(recs[slots])
            got, codes = eng.status_diff_slots(slots, sub, want_codes=op == "slots_codes")
            want = ssm.diff_slots(tab, slots, sub)
            self.check(np.array_equal(got, want), f"{op}: changed list {len(got)} slots, model {len(want)}")
            if codes is not None:
                self.check(np.array_equal(codes, oracle.record_codes(recs)[want]), f"{op}: codes differ")
        elif op == "tick":
            best, _, got, codes = eng.tick(self.pods, recs)
            want = tab.diff(recs)
            self.check(np.array_equal(got, want) and np.array_equal(best, self.best), "tick differs")
        elif op == "dev_slots":
            slots = self.pick()
            sub = np.ascontiguousarray(recs[slots])
            d_slots = t.from_numpy(slots.view(np.int32)).cuda()
            eng.status_diff_slots_device(d_slots, t.from_numpy(sub).cuda(), stride, self.col, self.idx, self.n, d_changed_code=self.code)
            t.cuda.synchronize()
            k = int(self.n.item())
            got = self.idx[:k].cpu().numpy().view(np.uint32)
            want = ssm.diff_slots(self.ctab, slots, sub)
            self.check(np.array_equal(got, want), f"{op}: changed list differs")
            self.check(np.array_equal(self.code[:k].cpu().numpy().view(np.uint16), oracle.record_codes(recs)[want]), f"{op}: codes differ")
            self.check(np.array_equal(self.col.cpu().numpy().view(np.uint64), self.ctab.prev_hashes()), f"{op}: device column differs")
        else:
            raise ValueError(op)


RANDOM_OPS = ["diff_codes", "seed", "seed_slots", "reset", "slots", "slots_codes", "tick", "dev_slots"]


def program_ops(rng, extra):
    """every stride entered the way WidenRecords enters it (whole-table seed, then the sweep -- here a slot-list sweep --
    at the same stride), then random operations at random strides"""
    ops = [("reset", 16, 0.0), ("slots_codes", 16, 0.0)]
    for s in rng.permutation(sc.STRIDES):
        s = int(s)
        ops += [("seed", s, 0.3), ("slots_codes", s, 0.0), (str(rng.choice(["diff_codes", "dev_slots", "slots"])), int(rng.choice([16, 32, s])), 0.05)]
        for _ in range(int(rng.integers(0, extra + 1))):
            ops.append((str(rng.choice(RANDOM_OPS)), int(rng.choice(sc.STRIDES)), float(rng.choice([0.0, 0.01, 0.2, 1.0]))))
    return ops


@pytest.mark.parametrize("size", [1, 65, 513, 34 * 256 + 1, "sat+1"])
def test_slots_call_sequences(size):
    N = size if isinstance(size, int) else sm_count() * 8 * 64 + 1
    p = Program(N, 104729 * N + 3)
    try:
        for op, stride, frac in program_ops(p.rng, 3 if N < 10_000 else 1):
            p.run(op, stride, frac)
    finally:
        p.close()


# ---- device variant ------------------------------------------------------------------------------------------------
def _dev(eng, t, slots, recs, stride, col, idx_base, codes=True):
    n = len(slots)
    idx = t.empty(max(n, 1), dtype=t.int32, device="cuda")
    code = t.empty(max(n, 1), dtype=t.int16, device="cuda")
    cnt = t.zeros(1, dtype=t.int32, device="cuda")
    eng.status_diff_slots_device(t.from_numpy(np.ascontiguousarray(slots, np.uint32).view(np.int32)).cuda(),
                                 t.from_numpy(np.ascontiguousarray(recs)).cuda(), stride, col, idx, cnt, idx_base=idx_base,
                                 d_changed_code=code if codes else None)
    t.cuda.synchronize()
    k = int(cnt.item())
    return idx[:k].cpu().numpy().view(np.uint32), code[:k].cpu().numpy().view(np.uint16)


@pytest.mark.parametrize("stride", [16, 32, 48, 256])
def test_device_sharded_columns(stride):
    """two columns handed the same global list with different idx_base: each is updated only in its own range, and
    the concatenated outputs equal the unsharded result; guard words after a column are never written"""
    import torch as t

    N, N0 = 70_001, 33_333
    rng = np.random.default_rng(stride)
    lt = sc.LogicalTable(N, rng)
    with rpk.Engine(1) as eng:
        full = t.zeros(N, dtype=t.int64, device="cuda")
        buf0 = t.full((N0 + 16,), 0x5A5A5A5A5A5A5A5A, dtype=t.int64, device="cuda")
        buf0[:N0] = 0
        col0, col1 = buf0[:N0], t.zeros(N - N0, dtype=t.int64, device="cuda")
        tab = oracle.StatusTable(N, stride)
        for frac, n in ((1.0, N // 2), (0.2, N), (0.05, 1000), (0.5, N // 3)):
            lt.step(stride, frac)
            recs = lt.records(stride)
            slots = np.sort(rng.choice(N, n, replace=False)).astype(np.uint32)
            sub = recs[slots]
            g, gc = _dev(eng, t, slots, sub, stride, full, 0)
            a, ac = _dev(eng, t, slots, sub, stride, col0, 0)
            b, bc = _dev(eng, t, slots, sub, stride, col1, N0)
            want = ssm.diff_slots(tab, slots, np.ascontiguousarray(sub))
            assert np.array_equal(g, want) and np.array_equal(gc, oracle.record_codes(recs)[want])
            assert np.array_equal(np.concatenate([a, b]), g) and np.array_equal(np.concatenate([ac, bc]), gc)
            h = full.cpu()
            assert t.equal(col0.cpu(), h[:N0]) and t.equal(col1.cpu(), h[N0:])
            assert (buf0[N0:] == 0x5A5A5A5A5A5A5A5A).all().item(), "guard words after the column were written"
            assert np.array_equal(h.numpy().view(np.uint64), tab.prev_hashes())
        # a list entirely outside a column touches nothing and reports nothing
        before = col0.clone()
        out, _ = _dev(eng, t, np.arange(N0, N0 + 500, dtype=np.uint32), lt.records(stride, np.arange(N0, N0 + 500)), stride, col0, 0)
        assert len(out) == 0 and t.equal(col0, before)


def test_device_refusals_and_launch_count():
    import torch as t

    with rpk.Engine(1) as eng:
        N = 4096
        recs = sc.LogicalTable(N, np.random.default_rng(0)).records(16)
        slots = np.arange(0, N, 7, dtype=np.uint32)
        col = t.zeros(N + 2, dtype=t.int64, device="cuda")
        _dev(eng, t, slots, recs[slots], 16, col[:N], 0)  # sizes the scratch
        before = eng.launch_count()
        _dev(eng, t, slots, recs[slots], 16, col[:N], 0)
        assert eng.launch_count() - before == 1
        with pytest.raises(rpk.RpkError) as e:
            _dev(eng, t, slots, recs[slots], 16, col[1:N + 1], 0)  # 8-byte aligned column
        assert e.value.code == rpk._ffi.RPK_EINVAL
        d_recs = t.zeros(len(slots) * 16 + 8, dtype=t.uint8, device="cuda")
        n = t.zeros(1, dtype=t.int32, device="cuda")
        idx = t.empty(len(slots), dtype=t.int32, device="cuda")
        with pytest.raises(rpk.RpkError) as e:
            eng.status_diff_slots_device(t.from_numpy(slots.view(np.int32)).cuda(), d_recs[8:], 16, col[:N], idx, n)
        assert e.value.code == rpk._ffi.RPK_EINVAL
        with pytest.raises(rpk.RpkError):
            _dev(eng, t, slots, recs[slots], 16, col[:N], 0xFFFFFFFF)  # idx_base + N beyond the slot range


def test_device_graph_capture_replay():
    """after one call of the size the device variant only enqueues: captured once, replayed over changing records"""
    import torch as t

    N, stride = 50_000, 32
    rng = np.random.default_rng(11)
    lt = sc.LogicalTable(N, rng)
    slots = np.sort(rng.choice(N, 20_000, replace=False)).astype(np.uint32)
    with rpk.Engine(1) as eng:
        d_slots = t.from_numpy(slots.view(np.int32)).cuda()
        d_recs = t.from_numpy(lt.records(stride, slots)).cuda()
        col = t.zeros(N, dtype=t.int64, device="cuda")
        idx = t.empty(len(slots), dtype=t.int32, device="cuda")
        code = t.empty(len(slots), dtype=t.int16, device="cuda")
        cnt = t.zeros(1, dtype=t.int32, device="cuda")
        tab = oracle.StatusTable(N, stride)
        side = t.cuda.Stream()
        with t.cuda.stream(side):
            eng.status_diff_slots_device(d_slots, d_recs, stride, col, idx, cnt, d_changed_code=code, stream=side.cuda_stream)
        side.synchronize()
        ssm.diff_slots(tab, slots, lt.records(stride, slots))
        g = t.cuda.CUDAGraph()
        with t.cuda.graph(g, stream=side):
            eng.status_diff_slots_device(d_slots, d_recs, stride, col, idx, cnt, d_changed_code=code, stream=side.cuda_stream)
        for step in range(4):
            lt.step(stride, 0.1 * (step + 1))
            sub = lt.records(stride, slots)
            d_recs.copy_(t.from_numpy(sub))
            t.cuda.synchronize()
            g.replay()
            t.cuda.synchronize()
            k = int(cnt.item())
            want = ssm.diff_slots(tab, slots, sub)
            assert np.array_equal(idx[:k].cpu().numpy().view(np.uint32), want), step
            assert np.array_equal(code[:k].cpu().numpy().view(np.uint16), oracle.record_codes(lt.records(stride))[want])


# ---- host refusals -------------------------------------------------------------------------------------------------
def test_host_refusals_leave_state_unchanged():
    N = 3000
    lt = sc.LogicalTable(N, np.random.default_rng(3))
    recs = lt.records(16)
    with rpk.Engine(1) as fresh:
        with pytest.raises(rpk.RpkError) as e:
            fresh.status_diff_slots(np.array([1, 2], np.uint32), recs[:2])
        assert e.value.code == rpk._ffi.RPK_ESTATE
        assert len(fresh.status_diff_slots(np.zeros(0, np.uint32), recs[:0])[0]) == 0
    with rpk.Engine(1) as eng:
        eng.status_reset(N)
        tab = oracle.StatusTable(N, 16)
        eng.status_seed(recs)
        tab.seed(recs)
        lt.step(16, 0.5)
        recs = lt.records(16)
        bad = [np.array([5, 3, 9]), np.array([3, 5, 5, 9]), np.array([0, 1, N]), np.array([2**32 - 1])]
        for slots in bad:
            with pytest.raises(rpk.RpkError) as e:
                eng.status_diff_slots(slots.astype(np.uint32), np.ascontiguousarray(recs[np.minimum(slots, N - 1)]))
            assert e.value.code == rpk._ffi.RPK_EINVAL, slots
        with pytest.raises(rpk.RpkError) as e:
            eng.status_diff_slots(np.array([1, 2], np.uint32), np.zeros((2, 24), np.uint8))  # stride 24
        assert e.value.code == rpk._ffi.RPK_EINVAL
        L = eng._lib
        n = C.c_uint32(0)
        idx = np.empty(4, np.uint32)
        sl = np.array([1, 2], np.uint32)
        r2 = np.ascontiguousarray(recs[:2])
        for args in ((None, r2.ctypes.data, idx.ctypes.data, C.cast(C.byref(n), C.c_void_p)),
                     (sl.ctypes.data, None, idx.ctypes.data, C.cast(C.byref(n), C.c_void_p)),
                     (sl.ctypes.data, r2.ctypes.data, None, C.cast(C.byref(n), C.c_void_p)),
                     (sl.ctypes.data, r2.ctypes.data, idx.ctypes.data, None)):
            assert L.rpk_status_diff_slots(eng._ctx, 2, args[0], args[1], 16, args[2], None, args[3]) == rpk._ffi.RPK_EINVAL
        got, codes, _ = eng.status_diff(recs, want_codes=True)
        assert np.array_equal(got, tab.diff(recs))


def test_multi_gpu_host_split():
    import torch

    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    N = 200_001
    lt = sc.LogicalTable(N, np.random.default_rng(9))
    rng = np.random.default_rng(10)
    with rpk.Engine(2) as eng:
        eng.status_reset(N)
        tab = oracle.StatusTable(N, 16)
        for n in (N, 1, 777, N // 2, 0):
            lt.step(16, 0.3)
            recs = lt.records(16)
            slots = np.sort(rng.choice(N, n, replace=False)).astype(np.uint32)
            sub = np.ascontiguousarray(recs[slots])
            got, codes = eng.status_diff_slots(slots, sub, want_codes=True)
            want = ssm.diff_slots(tab, slots, sub)
            assert np.array_equal(got, want) and np.array_equal(codes, oracle.record_codes(recs)[want])
        got, _, _ = eng.status_diff(recs, want_codes=True)
        assert np.array_equal(got, tab.diff(recs))
