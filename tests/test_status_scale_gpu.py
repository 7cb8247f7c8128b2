"""GPU tests of the status sweep at the sizes the API accepts: every stride in the 1024-thread shape, final copies of
more than 1024 units per CTA, record tables past 4 GiB, slot lists over a 2^28-slot column up to slot id 2^32 - 1, a
table grown to 2^26 slots, a per-slot seed past 4 GiB, a sweep beside a select, and a 3-shard ctx on one GPU.

Tables are columns of keys (status_scale_model.py): the records are built on the GPU from the keys through the key
table, so host memory stays at a few bytes per slot except where a case uses a host entry point, and every result is
checked against the model, which test_status_scale_model.py holds to oracle.StatusTable.  Each case names the regime
it is for on this device (launch shape, units per CTA, final-copy rounds), fills its changed-list and code outputs with
a sentinel PAD entries past their capacity, checks every changed id, code and hash and that the sentinel survived,
runs on a context of its own, and skips with the bytes it needs when the device or the host does not have them free."""
import ctypes as C
import time

import numpy as np
import pytest

import oracle
import rpk
import status_scale_model as m

pytestmark = pytest.mark.gpu

BIG = 4 << 20  # kBigTable (status.cu): 1024-thread CTAs from here
UNIT = 64  # kUnit (status.cu): slots per warp per unit
PAD = 37
SENT32, SENT16, SENT64 = 0x5EA5_1DE5, 0x5EA5, 0x5EA5_1DE5_5EA5_1DE5
GIB = 1 << 30
CHUNK = 1 << 24  # keys per gather on the device


# ---- the device and the launch plan ----------------------------------------------------------------------------------
def sm_count() -> int:
    import torch

    return torch.cuda.get_device_properties(0).multi_processor_count


def regime(N: int) -> dict:
    """launch_status (status.cu) for a sweep of N slots or list entries: CTA size, grid, the units (64 slots) of the
    CTA that owns the most, and the rounds of THREADS units its final copy takes"""
    threads = 1024 if N >= BIG else 256
    n_units = (N + UNIT - 1) // UNIT
    grid = max(min((n_units + threads // 32 - 1) // (threads // 32), sm_count()), 1)
    upc = max(n_units * (c + 1) // grid - n_units * c // grid for c in range(grid))
    return {"threads": threads, "grid": grid, "units_per_cta": upc, "rounds": (upc + threads - 1) // threads}


def cta_edges(N: int) -> np.ndarray:
    """the first and the last slot of every CTA's unit range"""
    r = regime(N)
    n_units = (N + UNIT - 1) // UNIT
    lo = np.array([n_units * c // r["grid"] for c in range(r["grid"])], np.int64) * UNIT
    hi = np.minimum(np.array([n_units * (c + 1) // r["grid"] for c in range(r["grid"])], np.int64) * UNIT, N) - 1
    return np.unique(np.concatenate([lo, hi]))


def mem_available() -> int:
    with open("/proc/meminfo") as f:
        for line in f:
            if line.startswith("MemAvailable:"):
                return int(line.split()[1]) * 1024
    return 0


def need(name: str, device: int, host: int):
    """skip unless the device and the host have the bytes the case needs (other processes may share both)"""
    import torch

    free = torch.cuda.mem_get_info()[0]
    if free < device:
        pytest.skip(f"{name} needs {device} bytes of free device memory; {free} are free")
    avail = mem_available()
    if avail < host:
        pytest.skip(f"{name} needs {host} bytes of available host memory; {avail} are available")


class Case:
    """a context of the case's own, and the log line that records its regime, memory and time"""

    def __init__(self, name: str, N: int, device: int, host: int, n_shards: int = 1):
        import torch

        torch.cuda.empty_cache()  # what earlier cases left in torch's cache counts as free
        need(name, device, host)
        self.name, self.t0 = name, time.time()
        self.free0 = torch.cuda.mem_get_info()[0]
        if n_shards > 1:
            from test_shared_device_ctx_gpu import shared_engine

            self.eng = shared_engine(n_shards)
        else:
            self.eng = rpk.Engine(1)
        self.low = self.free0
        r = regime(N)
        print(f"\n[status-scale] {name}: N={N} {r['threads']}-thread CTAs x {r['grid']}, {r['units_per_cta']} units per CTA, "
              f"{r['rounds']} final-copy round(s)")

    def mark(self):
        import torch

        torch.cuda.synchronize()
        self.low = min(self.low, torch.cuda.mem_get_info()[0])

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.mark()
        self.eng.close()
        print(f"[status-scale] {self.name}: {self.free0 - self.low} bytes of device memory in use at the most (sampled "
              f"after its sweeps), {time.time() - self.t0:.1f} s")


# ---- keys and records on the device ----------------------------------------------------------------------------------
class Dev:
    """the key table of one stride on the device: records and hash columns are gathered from key columns"""

    def __init__(self, stride: int):
        import torch

        self.stride = stride
        self.lut = torch.from_numpy(m.lut(stride)).cuda()
        self.h = torch.from_numpy(m.hashes(256).view(np.int64)).cuda()  # a key's hash does not depend on the stride

        self.buf = None

    def records(self, d_keys):
        """the records of a key column, in a buffer the next call reuses"""
        import torch

        n = int(d_keys.numel())
        if self.buf is None or self.buf.numel() < n * self.stride:
            self.buf = None
            self.buf = torch.empty(max(n, 1) * self.stride, dtype=torch.uint8, device="cuda")
        rows = self.buf[: n * self.stride].view(n, self.stride)
        for a in range(0, n, CHUNK):
            torch.index_select(self.lut, 0, d_keys[a:a + CHUNK].long(), out=rows[a:a + CHUNK])
        return self.buf[: n * self.stride]

    def check_column(self, col, model: m.Model, what: str):
        """the column equals the model's state, row by row (compared on the device)"""
        import torch

        assert int(col.numel()) == model.N
        bad = 0
        for a in range(0, model.N, CHUNK):
            st = torch.from_numpy(model.state[a:a + CHUNK]).cuda()
            want = torch.where(st >= 0, self.h[(st.clamp(min=0) * 2).long()], torch.zeros((), dtype=torch.int64, device="cuda"))
            bad += int((col[a:a + CHUNK] != want).sum().item())
        assert bad == 0, f"{what}: {bad} rows of the hash column differ from the model"


def to_dev(a):
    import torch

    a = np.ascontiguousarray(a)
    return torch.from_numpy(a.view(np.int32) if a.dtype == np.uint32 else a).cuda()


class Outs:
    """a device changed list and code buffer of capacity cap, sentinel-filled PAD entries past it"""

    def __init__(self, cap: int):
        import torch

        self.cap = cap
        self.idx = torch.empty(cap + PAD, dtype=torch.int32, device="cuda")
        self.code = torch.empty(cap + PAD, dtype=torch.int16, device="cuda")
        self.n = torch.empty(1, dtype=torch.int32, device="cuda")

    def fill(self):
        self.idx.fill_(SENT32)  # both below 2^31 / 2^15: the same bits signed
        self.code.fill_(SENT16)
        self.n.fill_(-1)
        return self.idx[: self.cap], self.code[: self.cap], self.n

    def check(self, want_ids, want_codes, what: str):
        import torch

        torch.cuda.synchronize()
        n = int(self.n.item())
        tail_i = self.idx[self.cap:].cpu().numpy().view(np.uint32)
        tail_c = self.code[self.cap:].cpu().numpy().view(np.uint16)
        assert (tail_i == SENT32).all() and (tail_c == SENT16).all(), f"{what}: written past the capacity"
        check_list(what, self.idx[:max(n, 0)].cpu().numpy().view(np.uint32), self.code[:max(n, 0)].cpu().numpy().view(np.uint16),
                   want_ids, want_codes)


def check_list(what, ids, codes, want_ids, want_codes):
    if len(ids) != len(want_ids) or not np.array_equal(ids, want_ids):
        k = min(len(ids), len(want_ids))
        bad = np.nonzero(ids[:k] != want_ids[:k])[0]
        raise AssertionError(f"{what}: {len(ids)} changed ids, want {len(want_ids)}; {len(bad)} of the first {k} differ, "
                             f"first at {bad[:4]} (got {ids[bad[:4]]}, want {want_ids[bad[:4]]})")
    bad = np.nonzero(codes != want_codes)[0]
    assert len(bad) == 0, f"{what}: {len(bad)} codes differ, first at {bad[:4]}"


def device_sweep(eng, dev: Dev, outs: Outs, col, model: m.Model, keys, what: str):
    """rpk_status_diff_device_codes over the records of `keys` against the caller-owned column -> the changed ids"""
    recs = dev.records(to_dev(keys))
    idx, code, n = outs.fill()
    eng.status_diff_device(recs, dev.stride, col, idx, n, d_changed_code=code)
    want, wcodes, _ = model.diff(keys, dev.stride, want_hashes=False)
    outs.check(want, wcodes, what)
    dev.check_column(col, model, what)
    return want


def ptr(a):
    return None if a is None else C.c_void_p(a.ctypes.data)


def host_sweep(eng, model: m.Model, keys, stride: int, what: str, hashes: bool = True):
    """rpk_status_diff_codes with host records of `keys`, into host outputs with PAD sentinel entries"""
    N = len(keys)
    recs = m.records(keys, stride)
    idx = np.full(N + PAD, SENT32, np.uint32)
    code = np.full(N + PAD, SENT16, np.uint16)
    hout = np.full(N + PAD, SENT64, np.uint64) if hashes else None
    n = np.zeros(1, np.uint32)
    eng._check(eng._lib.rpk_status_diff_codes(eng._ctx, N, ptr(recs), stride, ptr(idx), ptr(code), ptr(n), ptr(hout)))
    del recs
    want, wcodes, wh = model.diff(keys, stride, want_hashes=hashes)
    assert (idx[N:] == SENT32).all() and (code[N:] == SENT16).all(), f"{what}: written past the capacity"
    check_list(what, idx[:n[0]], code[:n[0]], want, wcodes)
    if hashes:
        assert (hout[N:] == SENT64).all(), f"{what}: hashes written past N"
        bad = np.count_nonzero(hout[:N] != wh)
        assert bad == 0, f"{what}: {bad} hashes differ"
    return want


def host_sweep_slots(eng, model: m.Model, slots, keys, stride: int, what: str):
    """rpk_status_diff_slots (host records of the listed slots) with PAD sentinel entries"""
    n_s = len(slots)
    recs = m.records(keys, stride)
    slots = np.ascontiguousarray(slots, np.uint32)
    idx = np.full(n_s + PAD, SENT32, np.uint32)
    code = np.full(n_s + PAD, SENT16, np.uint16)
    n = np.zeros(1, np.uint32)
    eng._check(eng._lib.rpk_status_diff_slots(eng._ctx, n_s, ptr(slots), ptr(recs), stride, ptr(idx), ptr(code), ptr(n)))
    want, wcodes = model.diff_slots(slots, keys, stride)
    assert (idx[n_s:] == SENT32).all() and (code[n_s:] == SENT16).all(), f"{what}: written past the capacity"
    check_list(what, idx[:n[0]], code[:n[0]], want, wcodes)
    return want


def slot_list(rng, n: int, M: int) -> np.ndarray:
    """n strictly ascending slots of [0, M) with random gaps, M - 1 among them"""
    idx = np.flatnonzero(rng.random(M - 1, dtype=np.float32) < min((n - 1) / (M - 1) * 1.02 + 1e-3, 1.0))
    assert len(idx) >= n - 1
    idx = np.delete(idx, rng.choice(len(idx), len(idx) - (n - 1), replace=False))
    return np.r_[idx, M - 1].astype(np.uint32)


# ---- a. every stride in the 1024-thread shape ------------------------------------------------------------------------
N_A = BIG + 37
STRIDES = list(range(16, 257, 16))


@pytest.mark.parametrize("stride", STRIDES)
def test_every_stride_big(stride):
    """4M + 37 slots at every stride: the wide strides 64..256 run k_status_stream<0, 1024> with records of up to 125
    characters (the multi-stripe hash inside a 1024-thread CTA).  Device entry point: after a reset (every slot), after
    a step that changes ~20 % of the slots and flips the flag on a third, and unchanged; at strides 64, 128 and 256 the
    host entry point with codes and hashes runs the same three sweeps."""
    import torch

    N = N_A
    host = stride in (64, 128, 256)
    with Case(f"a stride {stride}", N, N * (stride + 40) + GIB, N * (24 + (stride + 8 if host else 0)) + GIB) as cs:
        assert regime(N)["threads"] == 1024
        rng = np.random.default_rng(stride)
        dev, outs = Dev(stride), Outs(N)
        col = torch.zeros(N, dtype=torch.int64, device="cuda")
        model = m.Model(N)
        keys = m.draw(rng, N, stride)
        assert (m.LENS[keys >> 2] > 45).any() or stride < 64
        for what in ("after reset", "changed", "unchanged"):
            if what == "changed":
                keys = m.step(rng, keys, stride)
            got = device_sweep(cs.eng, dev, outs, col, model, keys, f"stride {stride} device {what}")
            assert len(got) == {"after reset": N, "unchanged": 0}.get(what, len(got))
            if what == "changed":
                assert N // 10 < len(got) < N // 3
        cs.mark()
        del dev, outs, col
        if host:
            cs.eng.status_reset(N)
            model.reset(N)
            for what in ("after reset", "changed", "unchanged"):
                if what == "changed":
                    keys = m.step(rng, keys, stride)
                got = host_sweep(cs.eng, model, keys, stride, f"stride {stride} host {what}")
                assert len(got) == {"after reset": N, "unchanged": 0}.get(what, len(got))
            cs.mark()


# ---- b. final-copy rounds ----------------------------------------------------------------------------------------
def round_size(size: str) -> int:
    full = UNIT * 1024 * sm_count()  # every CTA owns exactly 1024 units
    return {"full-64": full - 64, "full": full, "full+64": full + 64, "2full+37": 2 * full + 37}[size]


SIZES_B = ["full-64", "full", "full+64", "2full+37"]
ROUNDS_B = {"full-64": 1, "full": 1, "full+64": 2, "2full+37": 3}


@pytest.mark.parametrize("stride", [16, 32, 48, 256])
@pytest.mark.parametrize("size", SIZES_B)
def test_final_copy_rounds(size, stride):
    """N around 64 x 1024 x SMs: one round of the final copy per CTA, then one CTA owning 1025 units (a second round),
    then three rounds.  Every slot changes (after a reset), then ~20 %, then only the first and the last slot of every
    CTA's unit range -- the entries a dropped or doubled carry between rounds would move."""
    import torch

    N = round_size(size)
    with Case(f"b {size} stride {stride}", N, N * (stride + 40) + GIB, N * 24 + GIB) as cs:
        r = regime(N)
        assert r["threads"] == 1024 and r["rounds"] == ROUNDS_B[size]
        rng = np.random.default_rng(N + stride)
        dev, outs = Dev(stride), Outs(N)
        col = torch.zeros(N, dtype=torch.int64, device="cuda")
        model = m.Model(N)
        keys = m.draw(rng, N, stride)
        for what in ("every slot", "~20 %", "sparse"):
            if what == "~20 %":
                keys = m.step(rng, keys, stride)
            elif what == "sparse":
                edges = cta_edges(N)
                keys = keys.copy()
                keys[edges] = m.other_class(keys[edges], stride)
            got = device_sweep(cs.eng, dev, outs, col, model, keys, f"{size} stride {stride} {what}")
            if what == "sparse":
                assert np.array_equal(got, edges.astype(np.uint32))
        cs.mark()


@pytest.mark.parametrize("stride", [16, 48])
@pytest.mark.parametrize("size", SIZES_B)
def test_final_copy_rounds_slots(size, stride):
    """the slot-list sweep with lists of the same lengths (the launch follows the list length) over a column 1/8
    longer: host entry point (the ctx's tracked table) and device entry point, each after a reset, after a ~20 % step
    and with only the list positions at the CTA edges changed"""
    import torch

    n = round_size(size)
    M = n + n // 8
    with Case(f"b slots {size} stride {stride}", n, n * (2 * stride + 40) + M * 8 + GIB,
              n * (stride + 40) + M * 8 + GIB) as cs:
        assert regime(n)["rounds"] == ROUNDS_B[size]
        rng = np.random.default_rng(n + stride + 1)
        slots = slot_list(rng, n, M)
        edges = cta_edges(n)
        dev, outs = Dev(stride), Outs(n)
        d_slots = to_dev(slots)
        for form in ("host", "device"):
            model = m.Model(M)
            col = torch.zeros(M, dtype=torch.int64, device="cuda") if form == "device" else None
            if form == "host":
                cs.eng.status_reset(M)
            keys = m.draw(rng, n, stride)
            for what in ("after reset", "~20 %", "sparse"):
                if what == "~20 %":
                    keys = m.step(rng, keys, stride)
                elif what == "sparse":
                    keys = keys.copy()
                    keys[edges] = m.other_class(keys[edges], stride)
                label = f"{size} stride {stride} {form} slots {what}"
                if form == "host":
                    got = host_sweep_slots(cs.eng, model, slots, keys, stride, label)
                else:
                    recs = dev.records(to_dev(keys))
                    idx, code, d_n = outs.fill()
                    cs.eng.status_diff_slots_device(d_slots, recs, stride, col, idx, d_n, d_changed_code=code)
                    want, wcodes = model.diff_slots(slots, keys, stride)
                    outs.check(want, wcodes, label)
                    dev.check_column(col, model, label)
                    got = want
                if what == "after reset":
                    assert len(got) == n
                if what == "sparse":
                    assert np.array_equal(got, slots[edges])
            cs.mark()


# ---- c. records past 4 GiB -----------------------------------------------------------------------------------------
N_C = {16: 2**28 + 37, 32: 2**27 + 37, 48: -(-2**32 // 48) + 37, 256: 2**24 + 37}


def check_aliasing(keys, changed, stride: int, what: str):
    """most changed slots at or past the 4 GiB byte offset hash differently from the bytes a 32-bit byte offset
    (s * stride mod 2^32) would read instead, so a wrapped address cannot match by chance"""
    past = changed[changed >= -(-2**32 // stride)].astype(np.int64)
    assert len(past) > 0, f"{what}: no changed slot past 4 GiB"
    off = past * stride % 2**32
    j, r = off // stride, off % stride
    lut = m.lut(stride)
    alias = np.empty((len(past), stride), np.uint8)
    for rr in np.unique(r):  # the wrapped offset may start inside a record
        sel = r == rr
        alias[sel] = np.concatenate([lut[keys[j[sel]]][:, rr:], lut[keys[j[sel] + 1]][:, :rr]], axis=1)
    same = oracle.record_hashes(alias) == m.hashes(256)[keys[past]]
    assert same.sum() <= len(past) // 5, f"{what}: {same.sum()} of {len(past)} slots past 4 GiB read alike at a 32-bit offset"
    return len(past)


@pytest.mark.parametrize("stride", list(N_C))
def test_records_past_4gib(stride):
    """2^28 + 37 slots at stride 16, 2^27 + 37 at 32, ceil(2^32 / 48) + 37 at 48 and 2^24 + 37 at 256, through the
    device entry point: reset, a sweep that reports every slot, a changed sweep and an unchanged one"""
    import torch

    N = N_C[stride]
    assert N * stride > 2**32
    with Case(f"c stride {stride}", N, N * (stride + 40) + GIB, N * 32 + GIB) as cs:
        rng = np.random.default_rng(stride + 4)
        dev, outs = Dev(stride), Outs(N)
        col = torch.zeros(N, dtype=torch.int64, device="cuda")
        model = m.Model(N)
        keys = m.draw(rng, N, stride)
        for what in ("after reset", "changed", "unchanged"):
            if what == "changed":
                keys = m.step(rng, keys, stride)
            got = device_sweep(cs.eng, dev, outs, col, model, keys, f"stride {stride} N {N} {what}")
            if what == "after reset":
                assert len(got) == N
                assert check_aliasing(keys, got, stride, what) == N - -(-2**32 // stride) == 37
            elif what == "changed":
                check_aliasing(keys, got, stride, what)
            else:
                assert len(got) == 0
        cs.mark()


def test_records_past_4gib_host():
    """the host entry point with codes and hashes over 2^24 + 37 records of 256 bytes (4.3 GB uploaded)"""
    stride, N = 256, N_C[256]
    with Case("c host stride 256", N, N * (stride + 40) + GIB, N * (2 * stride + 40) + GIB) as cs:
        rng = np.random.default_rng(5)
        model = m.Model(N)
        cs.eng.status_reset(N)
        keys = m.draw(rng, N, stride)
        for what in ("after reset", "changed", "unchanged"):
            if what == "changed":
                keys = m.step(rng, keys, stride)
            got = host_sweep(cs.eng, model, keys, stride, f"host stride 256 {what}")
            if what != "unchanged":
                check_aliasing(keys, got, stride, what)
            else:
                assert len(got) == 0
        cs.mark()


# ---- d. slot lists at scale and the top of the id range ------------------------------------------------------------
M_D, N_D = 2**28, 2**26 + 37


@pytest.mark.parametrize("base", ["zero", "top"])
def test_slot_list_at_scale(base):
    """a 2^26 + 37-entry ascending list with gaps over a 2^28-slot column (1 GiB of records at stride 16), with entries
    outside the column: the column at idx_base 0 (entries up to 0xFFFFFFFF above it), or at 2^32 - 2^28 (entries below
    it; the ids reported reach 0xFFFFFFFF).  rpk_status_diff_slots_device and rpk_status_diff_slots_device_gather with
    one rank take turns over one column"""
    import torch

    from test_status_slots_gather_gpu import XBufs

    stride = 16
    idx_base = 0 if base == "zero" else 2**32 - M_D
    with Case(f"d {base}", N_D, N_D * (stride + 40) + M_D * 16 + GIB, N_D * 32 + M_D * 8 + GIB) as cs:
        rng = np.random.default_rng(7 if base == "zero" else 8)
        n_out = 4096
        inside = slot_list(rng, N_D - n_out, M_D).astype(np.int64) + idx_base
        if base == "zero":
            outside = np.unique(np.r_[rng.integers(M_D, 2**32 - 1, 2 * n_out), 2**32 - 1])[-n_out:]
            slots = np.concatenate([inside, outside])
        else:
            outside = np.unique(np.r_[rng.integers(0, idx_base, 2 * n_out), 0, idx_base - 1])[:n_out]
            slots = np.concatenate([outside, inside])
        assert len(slots) == N_D and (np.diff(slots) > 0).all() and slots[-1] == 2**32 - 1
        slots = slots.astype(np.uint32)
        dev, outs = Dev(stride), Outs(N_D)
        xb = XBufs(cs.eng, 1, N_D)
        d_slots = to_dev(slots)
        col = torch.zeros(M_D, dtype=torch.int64, device="cuda")
        model = m.Model(M_D)
        keys = m.draw(rng, N_D, stride)
        for what, form in (("after reset", "device"), ("changed", "gather"), ("unchanged", "gather"), ("changed again", "device")):
            if what.startswith("changed"):
                keys = m.step(rng, keys, stride)
            recs = dev.records(to_dev(keys))
            want, wcodes = model.diff_slots(slots, keys, stride, idx_base=idx_base, col_n=M_D)
            label = f"{base} {what} {form}"
            if form == "device":
                idx, code, d_n = outs.fill()
                cs.eng.status_diff_slots_device(d_slots, recs, stride, col, idx, d_n, idx_base=idx_base, d_changed_code=code)
                outs.check(want, wcodes, label)
            else:
                xb.fill()
                d_n = torch.full((1,), -1, dtype=torch.int32, device="cuda")
                cs.eng.status_diff_slots_device_gather(d_slots, recs, stride, col, idx_base, xb.ptrs, xb.cap, 0, d_n)
                xb.check([(want, wcodes)], label)
                assert int(d_n.item()) == len(want), label
            dev.check_column(col, model, label)
            if what == "after reset":
                assert len(want) == N_D - n_out
                assert (want[-1] == 0xFFFFFFFF) == (base == "top")
            if what == "unchanged":
                assert len(want) == 0
        cs.mark()


# ---- e. grow and per-slot seed at scale ----------------------------------------------------------------------------
def test_grow_to_2_26():
    """rpk_status_grow from 4M - 1 slots to 2^26 + 37 at stride 32: the next sweep reports exactly the old slots that
    changed and every new slot"""
    stride, N0, N = 32, BIG - 1, 2**26 + 37
    with Case("e grow", N, N * (stride + 30) + GIB, N * (stride + 40) + GIB) as cs:
        assert regime(N0)["threads"] == 256 and regime(N)["threads"] == 1024
        rng = np.random.default_rng(26)
        model = m.Model(N0)
        cs.eng.status_reset(N0)
        keys = m.draw(rng, N0, stride)
        host_sweep(cs.eng, model, keys, stride, "before the grow")
        cs.eng.status_grow(N)
        model.grow(N)
        keys = np.concatenate([m.step(rng, keys, stride), m.draw(rng, N - N0, stride)])
        got = host_sweep(cs.eng, model, keys, stride, "after the grow")
        assert (got[got >= N0] == np.arange(N0, N)).all() and np.count_nonzero(got >= N0) == N - N0
        assert 0 < np.count_nonzero(got < N0) < N0 // 3
        assert len(host_sweep(cs.eng, model, keys, stride, "unchanged after the grow")) == 0
        cs.mark()


def test_seed_slots_past_4gib():
    """rpk_status_seed_slots of 2^24 + 37 records at stride 256 (the packed records pass 4 GiB) into a table of
    2^24 + 2^22 slots, then a whole-table sweep at stride 16: the seeded slots report only where the class moved"""
    stride, n = 256, 2**24 + 37
    N = 2**24 + 2**22
    with Case("e seed_slots", n, n * (2 * stride + 8) + GIB, n * (stride + 16) + N * 40 + GIB) as cs:
        rng = np.random.default_rng(24)
        slots = np.sort(rng.choice(N, n, replace=False)).astype(np.uint32)
        model = m.Model(N)
        cs.eng.status_reset(N)
        sk = m.draw(rng, n, stride)
        sk[2**24:] = m.draw(rng, n - 2**24, 16)  # the records past 4 GiB stay as seeded in the sweep at stride 16
        recs = m.records(sk, stride)
        cs.eng.status_seed_slots(slots, recs)
        del recs
        model.seed_slots(slots, sk)
        keys = m.draw(rng, N, 16)
        keep = np.zeros(N, bool)
        keep[slots] = (m.LENS[sk >> 2] <= 13) & (rng.random(n) < 0.8)  # seeded slots that stay as seeded
        late = slots[2**24:]  # their packed records start past 4 GiB
        keep[late] = True
        keys[slots[keep[slots]]] = sk[keep[slots]]
        # a 32-bit record offset would seed them with the records 2^24 places before theirs: other classes
        assert ((sk[2**24:] >> 1) != (sk[:n - 2**24] >> 1)).mean() > 0.8
        got = host_sweep(cs.eng, model, keys, 16, "sweep after the per-slot seed")
        assert not np.isin(late, got).any()
        cs.mark()


# ---- f. beside a select and across shards --------------------------------------------------------------------------
def test_tick_beside_select():
    """rpk_tick: 4096 pod rows (every row against oracle.select) and a sweep of 2^26 + 37 slots at stride 32"""
    stride, N, P = 32, 2**26 + 37, 4096
    with Case("f tick", N, N * (stride + 30) + 2 * GIB, N * (stride + 40) + GIB) as cs:
        rng = np.random.default_rng(32)
        offers = rpk.synth.make_offers(20_000, correlated=True)
        pods = rpk.synth.make_pods(P, seed=3)
        ob, _ = oracle.select(offers, pods, want_top5=False, n_threads=4)
        cs.eng.upload_offers(offers)
        model = m.Model(N)
        cs.eng.status_reset(N)
        keys = m.draw(rng, N, stride)
        host_sweep(cs.eng, model, keys, stride, "before the tick", hashes=False)
        keys = m.step(rng, keys, stride)
        recs = m.records(keys, stride)
        best = np.full(P + PAD, SENT32, np.uint32).view(np.int32)
        idx = np.full(N + PAD, SENT32, np.uint32)
        code = np.full(N + PAD, SENT16, np.uint16)
        n = np.zeros(1, np.uint32)
        cols = {k: np.ascontiguousarray(pods[k]) if pods.get(k) is not None else None
                for k in ("req_mem_gb", "req_vcpu", "req_ram_gb", "max_price", "cloud")}
        cs.eng._check(cs.eng._lib.rpk_tick(cs.eng._ctx, P, *[ptr(cols[k]) for k in cols], ptr(best), None, N, ptr(recs),
                                           stride, ptr(idx), ptr(code), ptr(n)))
        del recs
        want, wcodes, _ = model.diff(keys, stride, want_hashes=False)
        assert (idx[N:] == SENT32).all() and (code[N:] == SENT16).all() and (best[P:].view(np.uint32) == SENT32).all()
        check_list("tick sweep", idx[:n[0]], code[:n[0]], want, wcodes)
        bad = np.nonzero(best[:P] != ob)[0]
        assert len(bad) == 0, f"tick select: {len(bad)} rows differ from oracle.select, first {bad[:4]}"
        cs.mark()


def test_three_shards_one_gpu():
    """a 3-shard ctx on one GPU at 3 x 4M + 37 slots and stride 256: every shard takes the 1024-thread shape, and the
    shard cuts fall inside 64-slot units.  Host entry point with codes and hashes: reset, changed, unchanged"""
    from test_shared_device_ctx_gpu import cuts

    stride, N = 256, 3 * BIG + 37
    b = cuts(N, 3)
    assert all(b[s + 1] - b[s] >= BIG for s in range(3)) and all(c % UNIT for c in b[1:3])
    with Case("f 3 shards", N // 3, N * (stride + 40) + GIB, N * (2 * stride + 40) + GIB, n_shards=3) as cs:
        rng = np.random.default_rng(3)
        model = m.Model(N)
        cs.eng.status_reset(N)
        keys = m.draw(rng, N, stride)
        for what in ("after reset", "changed", "unchanged"):
            if what == "changed":
                keys = m.step(rng, keys, stride)
            got = host_sweep(cs.eng, model, keys, stride, f"3 shards {what}")
            assert len(got) == {"after reset": N, "unchanged": 0}.get(what, len(got))
        cs.mark()
