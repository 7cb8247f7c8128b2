"""GPU tests of the status sweep (K2) over sequences of calls on one context, against the oracle's state model.

Every status kernel of a context shares its scheduling ticket and look-back state, whichever entry point (host or
device) and whichever instantiation (strides 16 / 32, or the wide form for 48..256) runs it, so a call can go wrong
because of what the call before it left behind.  Each program below is a seeded random sequence of resets, seeds,
per-slot seeds, diffs (with and without codes and hashes), ticks and device-column diffs at every stride, with the
stride changing the way Provider::WidenRecords changes it (whole-table seed at the new stride, then the sweep at it),
checked against oracle.StatusTable after every step.  Sizes sit on the streaming unit (64 slots), on blocks of 512
slots (strides 48 / 64) and 256 (above) with more than 33 and more than 1024 of them, and past the point where the
small-table streaming grid saturates (four 8-warp CTAs per SM, one 64-slot unit per warp)."""
import numpy as np
import pytest

import oracle
import rpk
import status_cases as sc

pytestmark = pytest.mark.gpu


def sm_count() -> int:
    import torch

    return torch.cuda.get_device_properties(0).multi_processor_count


def resolve(size):
    """sizes that depend on the device are named at collection time (no GPU there) and resolved here"""
    if isinstance(size, int):
        return size
    sat = 4 * sm_count() * 8 * 64  # small-shape streaming grid: 4 CTAs / SM x 8 warps x one 64-slot unit
    return {"sat-1": sat - 1, "sat": sat, "sat+1": sat + 1}[size]


class DeviceColumn:
    """A caller-owned hash column (torch) swept with rpk_status_diff_device_codes, and its own oracle state."""

    def __init__(self, N: int):
        import torch

        self.torch = torch
        self.N = N
        self.hash = torch.zeros(N, dtype=torch.int64, device="cuda")
        self.idx = torch.empty(N, dtype=torch.int32, device="cuda")
        self.code = torch.empty(N, dtype=torch.int16, device="cuda")
        self.n = torch.zeros(1, dtype=torch.int32, device="cuda")
        self.tab = oracle.StatusTable(N, 16)

    def diff(self, eng, recs: np.ndarray, codes: bool):
        t = self.torch
        d_recs = t.from_numpy(recs).cuda()
        eng.status_diff_device(d_recs, recs.shape[1], self.hash, self.idx, self.n, d_changed_code=self.code if codes else None)
        t.cuda.synchronize()
        n = int(self.n.item())
        idx = self.idx[:n].cpu().numpy().view(np.uint32)
        code = self.code[:n].cpu().numpy().view(np.uint16) if codes else None
        return idx, code

    def column(self) -> np.ndarray:
        return self.hash.cpu().numpy().view(np.uint64)

    def set_column(self, h: np.ndarray):
        self.hash.copy_(self.torch.from_numpy(h.view(np.int64)))


class Program:
    """One engine, one logical table, the oracle's model of the engine's state (and of a device column)."""

    def __init__(self, N: int, seed: int):
        self.N, self.seed = N, seed
        self.rng = np.random.default_rng(seed)
        self.lt = sc.LogicalTable(N, self.rng)
        self.eng = rpk.Engine(1)
        self.tab = oracle.StatusTable(N, 16)
        self.dev = DeviceColumn(N)
        self.offers = rpk.synth.make_offers(300, correlated=True)
        self.pods = rpk.synth.make_pods(64, seed=seed)
        self.eng.upload_offers(self.offers)
        self.best = oracle.select(self.offers, self.pods)[0]
        self.log = []

    def close(self):
        self.eng.close()

    def check(self, ok: bool, what: str):
        if not ok:
            raise AssertionError(f"{what}\nprogram seed {self.seed}, N {self.N}; operations:\n  " + "\n  ".join(self.log))

    def check_changed(self, got, want, codes, recs, label):
        self.check(np.array_equal(got, want), f"{label}: changed list {len(got)} slots, model {len(want)}")
        if codes is not None:
            self.check(np.array_equal(codes, oracle.record_codes(recs)[want]), f"{label}: codes differ from record_codes")

    def run(self, op: str, stride: int, frac: float):
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
            slots = np.sort(self.rng.choice(N, int(self.rng.integers(1, min(N, 300) + 1)), replace=False)).astype(np.uint32)
            eng.status_seed_slots(slots, np.ascontiguousarray(recs[slots]))
            tab.seed_slots(slots, recs[slots])
        elif op in ("diff", "diff_codes", "diff_hashes"):
            want_codes, want_hashes = op != "diff", op == "diff_hashes"
            out = eng.status_diff(recs, want_hashes=want_hashes, want_codes=want_codes)
            got, codes, hashes = out if want_codes else (out[0], None, out[1])
            self.check_changed(got, tab.diff(recs), codes, recs, op)
            if want_hashes:
                self.check(np.array_equal(hashes, oracle.record_hashes(recs)), f"{op}: hash column differs from record_hashes")
        elif op in ("tick", "tick_p"):
            pods = self.pods if op == "tick_p" else None
            best, _, got, codes = eng.tick(pods, recs)
            self.check_changed(got, tab.diff(recs), codes, recs, op)
            if pods is not None:
                self.check(np.array_equal(best, self.best), "tick: selection differs from the oracle")
        elif op in ("dev", "dev_codes"):
            got, codes = self.dev.diff(eng, recs, op == "dev_codes")
            self.check_changed(got, self.dev.tab.diff(recs), codes, recs, op)
            self.check(np.array_equal(self.dev.column(), self.dev.tab.prev_hashes()), f"{op}: device hash column differs from the model")
        elif op == "dev_reset":  # the caller forgets its column
            self.dev.set_column(np.zeros(N, np.uint64))
            self.dev.tab.reset(N)
        elif op == "dev_seed":  # ... or fills it itself
            self.dev.set_column(oracle.record_hashes(recs))
            self.dev.tab.seed(recs)
        else:
            raise ValueError(op)


RANDOM_OPS = ["diff", "diff_codes", "diff_hashes", "seed", "seed_slots", "reset", "tick", "tick_p", "dev", "dev_codes",
              "dev_reset", "dev_seed"]


def program_ops(rng, extra: int):
    """Every stride, in a seeded order, is entered the way WidenRecords enters it -- a whole-table seed at the stride,
    then a sweep at the same stride -- followed by a sweep at that stride, 16 or 32, and up to `extra` random
    operations at random strides (device-column sweeps included)."""
    ops = [("reset", 16, 0.0), ("diff_codes", 16, 0.0)]
    for s in rng.permutation(sc.STRIDES):
        s = int(s)
        ops += [("seed", s, 0.3), ("diff_hashes", s, 0.0), (str(rng.choice(["diff_codes", "dev_codes"])), int(rng.choice([16, 32, s])), 0.05)]
        for _ in range(int(rng.integers(0, extra + 1))):
            ops.append((str(rng.choice(RANDOM_OPS)), int(rng.choice(sc.STRIDES)), float(rng.choice([0.0, 0.01, 0.2, 1.0]))))
    return ops


SIZES = [1, 63, 64, 65, 255, 256, 257, 511, 512, 513, 34 * 512 + 1, 1025 * 256 + 1, "sat-1", "sat", "sat+1"]


@pytest.mark.parametrize("size", SIZES)
def test_status_call_sequences(size):
    N = resolve(size)
    seed = 7919 * N + 17
    p = Program(N, seed)
    try:
        for op, stride, frac in program_ops(p.rng, 3 if N < 100_000 else 1):
            p.run(op, stride, frac)
    finally:
        p.close()


@pytest.mark.parametrize("stride", [s for s in sc.STRIDES if s > 32])
def test_seed_at_wide_stride_then_diff(stride):
    """A whole-table seed at a wide stride, then sweeps at that stride and at strides 16 and 32, then
    device-column sweeps on the same context: nothing is reported until something changes, and then exactly that."""
    N = 3 * 512 + 5
    p = Program(N, stride)
    try:
        p.lt.step(stride, 1.0)
        p.run("seed", stride, 0.0)
        got, codes, _ = p.eng.status_diff(p.lt.records(stride), want_codes=True)
        p.check(len(got) == 0, "the sweep right after the whole-table seed reported slots")
        p.run("diff_codes", stride, 0.0)
        p.run("diff_codes", 16, 0.0)  # statuses longer than 13 characters cannot stay: exactly those slots report
        p.run("seed", stride, 0.2)
        p.run("diff_codes", 32, 0.0)
        for op in ("diff_codes", "dev_codes", "dev_codes", "seed", "diff_hashes", "tick_p", "dev_codes", "seed_slots", "diff_codes"):
            p.run(op, stride, 0.1)
    finally:
        p.close()


@pytest.mark.parametrize("N", [513, 5000, 40_000])
def test_hash_does_not_depend_on_stride(N):
    """include/rpk.h: the slot hash covers the zero-padded prefix in whole 8-byte lanes, so the same logical records
    at 16, 64 and 256 bytes hash alike: state established at 16 reports nothing at 64 or 256 (host table and device
    column), and the hash columns are equal."""
    lt = sc.LogicalTable(N, np.random.default_rng(N))
    narrow = lt.records(16)
    p = Program(N, N)
    try:
        idx, hashes = p.eng.status_diff(narrow, want_hashes=True)
        assert len(idx) == N
        dev_idx, _ = p.dev.diff(p.eng, narrow, True)
        assert len(dev_idx) == N
        col = p.dev.column()
        assert np.array_equal(col, hashes)
        for stride in (64, 256, 48, 16):
            recs = lt.records(stride)
            idx, h = p.eng.status_diff(recs, want_hashes=True)
            assert len(idx) == 0 and np.array_equal(h, hashes), stride
            dev_idx, _ = p.dev.diff(p.eng, recs, False)
            assert len(dev_idx) == 0 and np.array_equal(p.dev.column(), col), stride
    finally:
        p.close()
