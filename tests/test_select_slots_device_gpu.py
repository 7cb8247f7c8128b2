"""GPU tests of the device select over a list of pod-table slots (rpk_select_slots_device and its gathers' shared path).

The pod table, its seeds and the oracle's result per slot come from test_select_slots_gpu.py (PodTable, tracked(),
slot_list()).  Every device call must return, row for row, what the host call rpk_select_slots returns for the same
list and what the oracle gives for the slot.  A list entry outside the table has a defined result on the device path:
-1 and five -1.  Every output tensor starts as SENTINEL, so a row the kernels never write shows up."""
import ctypes as C
import zlib

import numpy as np
import pytest

import rpk
import select_plan_cases as sc
from test_select_sequences_gpu import FORCE, MENU
from test_select_slots_gpu import R, SHAPES, SIZES, TRACKED, PodTable, run_slots, seeded_engine, slot_list, tracked

pytestmark = pytest.mark.gpu

EINVAL, ESTATE = rpk._ffi.RPK_EINVAL, rpk._ffi.RPK_ESTATE
OUTSIDE = (TRACKED, TRACKED + 1, TRACKED + 4097, 0x7FFFFFFF, 0xFFFFFFFE, 0xFFFFFFFF)


def d_list(sl):
    import torch

    return torch.from_numpy(np.ascontiguousarray(sl, np.uint32).view(np.int32)).cuda()


def run_slots_device(eng, sl, top5, stream=None):
    """rpk_select_slots_device on `stream` (a torch.cuda.Stream; None: the current stream), then a device synchronise"""
    import torch

    n = len(sl)
    d = d_list(sl)
    d_best = torch.full((n,), sc.SENTINEL, dtype=torch.int32, device="cuda")
    d_t5 = torch.full((n * 5,), sc.SENTINEL, dtype=torch.int32, device="cuda") if top5 else None
    torch.cuda.synchronize()  # inputs are written on the current stream; the call may run on another one
    eng.select_slots_device(d, d_best, d_t5, stream=stream.cuda_stream if stream is not None else None)
    torch.cuda.synchronize()
    return d_best.cpu().numpy(), d_t5.cpu().numpy().reshape(n, 5) if top5 else None


def with_outside(rng, sl, frac=0.05):
    """-> (list with about `frac` of its entries replaced by entries >= TRACKED, mask of those)"""
    sl = sl.copy()
    bad = rng.random(len(sl)) < frac
    bad[rng.integers(0, len(sl))] = True
    sl[bad] = rng.choice(np.array(OUTSIDE, np.uint32), int(bad.sum()))
    return sl, bad


@pytest.mark.parametrize("force", FORCE)
@pytest.mark.parametrize("name", MENU)
def test_select_slots_device_equals_host_and_oracle(name, force):
    """every list size (both sides of the fused kernel's size, a multi-sub-batch host size) and shape, with and without
    top-5, over rows seeded with and without optional columns and unseeded rows"""
    _, eb, et, _ = tracked(name)
    rng = np.random.default_rng(zlib.crc32(f"device/{name}/{force}".encode()))
    sizes = SIZES + ([TRACKED] if name == "synth100k" else [])
    eng = seeded_engine(name, force)
    try:
        for n in sizes:
            for shape in SHAPES:
                sl = slot_list(rng, n, shape)
                label = f"{name} force={force} n={n} {shape}"
                hb, ht = run_slots(eng, sl, True)
                for top5 in (False, True):
                    best, t5 = run_slots_device(eng, sl, top5)
                    sc.check(f"{label} top5={top5}: device vs oracle", best, t5, eb[sl], et[sl] if top5 else None)
                    sc.check(f"{label} top5={top5}: device vs select_slots", best, t5, hb, ht if top5 else None)
    finally:
        eng.close()


@pytest.mark.parametrize("force", FORCE)
def test_entries_outside_the_table(force):
    """entries >= N (0xFFFFFFFF included) give -1 and five -1; every other row is right, at the fused kernel's sizes
    and at sizes the persistent kernel takes"""
    _, eb, et, _ = tracked("synth20k")
    rng = np.random.default_rng(zlib.crc32(f"outside/{force}".encode()))
    eng = seeded_engine("synth20k", force)
    try:
        for n in (1, 4097, 16_384, 16_385, R):
            for shape in ("shuffled", "repeats"):
                sl, bad = with_outside(rng, slot_list(rng, n, shape))
                ok = np.where(bad, 0, sl)
                wb, wt = eb[ok].copy(), et[ok].copy()
                wb[bad], wt[bad] = -1, -1
                for top5 in (False, True):
                    best, t5 = run_slots_device(eng, sl, top5)
                    sc.check(f"force={force} n={n} {shape} top5={top5} ({int(bad.sum())} outside)", best, t5, wb,
                             wt if top5 else None)
        best, t5 = run_slots_device(eng, np.array(OUTSIDE, np.uint32), True)  # a list with nothing inside the table
        assert (best == -1).all() and (t5 == -1).all()
    finally:
        eng.close()


def test_launches_and_stats():
    """one gather on top of what the column call launches; one select in the stats"""
    m, eb, et, _ = tracked("synth20k")
    G = len(sc.table("synth20k")["mem_gb"])
    rng = np.random.default_rng(13)
    eng = seeded_engine("synth20k")
    try:
        for n in (1, 4097, 16_385, R):
            sl = slot_list(rng, n, "shuffled")
            run_slots_device(eng, sl, True)  # sizes the scratch
            sc.run_device(eng, m.rows(sl), True)
            s0, c0 = eng.stats(), eng.launch_count()
            best, t5 = run_slots_device(eng, sl, True)
            s1, c1 = eng.stats(), eng.launch_count()
            sc.run_device(eng, m.rows(sl), True)
            c2 = eng.launch_count()
            assert (c1 - c0) - (c2 - c1) == 1, n
            assert s1["select_calls"] == s0["select_calls"] + 1 and s1["offer_scores"] == s0["offer_scores"] + n * G
            sc.check(f"n={n}", best, t5, eb[sl], et[sl])
        c0 = eng.launch_count()
        eng.select_slots_device(d_list(np.zeros(0, np.uint32)), d_list(np.zeros(0, np.uint32)))  # empty: nothing
        assert eng.launch_count() == c0
    finally:
        eng.close()


def raw(eng, fn, *args, shard=0, stream=None):
    """an rpk_select_slots_device* call straight from the library (arguments the binding would refuse first)"""
    import torch

    st = C.c_void_p(stream if stream is not None else (torch.cuda.current_stream(0).cuda_stream or 1))
    return getattr(eng._lib, fn)(eng._ctx, shard, *args, st)


def arr(ptrs):
    return (C.c_void_p * max(len(ptrs), 1))(*ptrs)


def test_refusals_leave_the_launch_count():
    import torch

    _, eb, et, _ = tracked("synth20k")
    rng = np.random.default_rng(17)
    n = 40_001
    sl = slot_list(rng, n, "shuffled")
    d = d_list(sl)
    best = torch.full((n + 9,), sc.SENTINEL, dtype=torch.int32, device="cuda")
    t5 = [torch.full((5 * n + 9,), sc.SENTINEL, dtype=torch.int32, device="cuda") for _ in range(2)]
    S, B, T = d.data_ptr(), best.data_ptr(), [v.data_ptr() for v in t5]
    eng = seeded_engine("synth20k")
    try:
        run_slots_device(eng, sl, True)  # warm: sizes the scratch
        c0 = eng.launch_count()

        def refused(rc, code, what):
            assert rc == code, (what, rc, eng._lib.rpk_last_error(eng._ctx))
            assert eng.launch_count() == c0, f"{what}: launched"

        refused(raw(eng, "rpk_select_slots_device", n, None, B, None), EINVAL, "NULL list")
        refused(raw(eng, "rpk_select_slots_device", n, S, B, None, shard=1), EINVAL, "shard 1 of a 1-GPU ctx")
        refused(raw(eng, "rpk_select_slots_device", n, S, B, None, shard=-1), EINVAL, "shard -1")
        refused(raw(eng, "rpk_select_slots_device", n, S, None, None), EINVAL, "NULL d_best")
        refused(raw(eng, "rpk_select_slots_device_gather", n, None, 1, arr([B]), 0, None), EINVAL, "gather: NULL list")
        refused(raw(eng, "rpk_select_slots_device_gather", n, S, 0, arr([B]), 0, None), EINVAL, "gather: n_out 0")
        refused(raw(eng, "rpk_select_slots_device_gather", n, S, 9, arr([B] * 9), 0, None), EINVAL, "gather: n_out 9")
        refused(raw(eng, "rpk_select_slots_device_gather", n, S, 2, arr([B, 0]), 0, None), EINVAL, "gather: NULL vector")
        refused(raw(eng, "rpk_select_slots_device_gather", n, S, 1, None, 0, None), EINVAL, "gather: NULL vector array")
        G5 = "rpk_select_slots_device_gather_top5"
        refused(raw(eng, G5, n, None, 2, arr([B, B]), arr(T), 0), EINVAL, "top5: NULL list")
        refused(raw(eng, G5, n, S, 2, arr([B, B]), arr([T[0], T[1] + 4]), 0), EINVAL, "top5: phase")
        refused(raw(eng, G5, n, S, 2, arr([B, B]), arr([T[0], 0]), 0), EINVAL, "top5: NULL top-5 vector")
        refused(raw(eng, G5, n, S, 0, arr([B]), arr(T), 0), EINVAL, "top5: n_out 0")
        refused(raw(eng, G5, 858_993_460, S, 2, arr([B, B]), arr(T), 0), EINVAL, "top5: 5*n beyond uint32")
        host = [eng._lib.rpk_host_alloc(5 * n * 4) for _ in range(2)]
        try:
            refused(raw(eng, G5, n, S, 2, arr([B, B]), arr(host), 0), EINVAL, "top5: no top-5 vector on the GPU")
        finally:
            for h in host:
                eng._lib.rpk_host_free(h)
        assert eng._lib.rpk_select_slots_device(None, 0, n, S, B, None, None) == EINVAL
        with pytest.raises(TypeError):  # the binding's tensor checks
            eng.select_slots_device(d.to(torch.int64), best)
        with pytest.raises(ValueError):
            eng.select_slots_device(d, best[: n - 1])
        with pytest.raises(ValueError):
            eng.select_slots_device(d, best, t5[0][: 5 * n - 1])
        with pytest.raises(TypeError):
            eng.select_slots_device(d[::2], best)
        with pytest.raises(ValueError):
            eng.select_slots_device_gather(d, [B], 0, d_top5=t5[0], top5_ptrs=T[:1])
        with pytest.raises(ValueError):
            eng.select_slots_device_gather(d, [B], 0, top5_ptrs=T)
        assert eng.launch_count() == c0
        torch.cuda.synchronize()
        assert (best == sc.SENTINEL).all() and all((v == sc.SENTINEL).all() for v in t5)
        got = run_slots_device(eng, sl, True)  # the next valid call is right
        sc.check("after the refusals", *got, eb[sl], et[sl])
    finally:
        eng.close()
    # RPK_ESTATE: no pod table, no offer table; before anything is enqueued
    offers = sc.table("synth300")
    with rpk.Engine(1) as e:
        e.upload_offers(offers)
        c0 = e.launch_count()
        for top5 in (False, True):
            with pytest.raises(rpk.RpkError) as ei:
                e.select_slots_device(d[:5], best[:5], t5[0][:25] if top5 else None)
            assert ei.value.code == ESTATE
        with pytest.raises(rpk.RpkError) as ei:
            e.select_slots_device_gather(d[:5], [B], 0, top5_ptrs=[T[0]])
        assert ei.value.code == ESTATE and e.launch_count() == c0
    with rpk.Engine(1) as e:
        e.pods_reset(16)
        c0 = e.launch_count()
        with pytest.raises(rpk.RpkError) as ei:
            e.select_slots_device(d[:5], best[:5])
        assert ei.value.code == ESTATE and e.launch_count() == c0


def test_seeds_between_device_calls_without_a_synchronise():
    """device call, host seed of rows it listed, device call, all issued on a torch side stream without a synchronise:
    the first call sees the rows before the seed, the second the seeded ones"""
    import torch

    offers = sc.table("synth20k")
    N = 200_000
    rng = np.random.default_rng(23)
    side = torch.cuda.Stream(device="cuda:0")
    with rpk.Engine(1) as eng:
        eng.upload_offers(offers)
        eng.pods_reset(N)
        m = PodTable(N)
        pods = sc.pods_for("synth20k", N, seed=5)
        every = np.arange(N, dtype=np.uint32)
        eng.pods_seed_slots(every, pods)
        m.seed(every, pods)
        for step, n in enumerate((4097, 30_000, 150_000, 30_000)):
            sl = slot_list(rng, n, "shuffled", N)
            d = d_list(sl)
            outs = [(torch.full((n,), sc.SENTINEL, dtype=torch.int32, device="cuda"),
                     torch.full((5 * n,), sc.SENTINEL, dtype=torch.int32, device="cuda")) for _ in range(2)]
            torch.cuda.synchronize()
            want = [sc.expected(offers, m.rows(sl))]
            eng.select_slots_device(d, *outs[0], stream=side.cuda_stream)
            rows = np.unique(sl[rng.random(n) < 0.5])  # strictly ascending
            fresh = sc.pods_for("synth20k", len(rows), seed=100 + step)
            if step % 2:
                fresh = sc.without_optional(fresh)
            eng.pods_seed_slots(rows, fresh)
            m.seed(rows, fresh)
            want.append(sc.expected(offers, m.rows(sl)))
            eng.select_slots_device(d, *outs[1], stream=side.cuda_stream)
            side.synchronize()
            for k, ((b, t), (wb, wt)) in enumerate(zip(outs, want)):
                sc.check(f"step {step} call {k}", b.cpu().numpy(), t.cpu().numpy().reshape(n, 5), wb, wt)


def test_reset_to_a_larger_table_between_calls():
    import torch

    offers = sc.table("synth20k")
    db, _ = sc.expected(offers, {"req_mem_gb": np.array([16], np.int32), "req_vcpu": None, "req_ram_gb": None,
                                  "max_price": None, "cloud": None})
    rng = np.random.default_rng(29)
    side = torch.cuda.Stream(device="cuda:0")
    with rpk.Engine(1) as eng:
        eng.upload_offers(offers)
        N = 50_000
        eng.pods_reset(N)
        pods = sc.pods_for("synth20k", N, seed=9)
        eng.pods_seed_slots(np.arange(N, dtype=np.uint32), pods)
        sl = slot_list(rng, 40_000, "shuffled", 4 * N)  # entries of the larger table: a quarter inside the first one
        d = d_list(sl)
        b0 = torch.full((len(sl),), sc.SENTINEL, dtype=torch.int32, device="cuda")
        b1 = torch.full((len(sl),), sc.SENTINEL, dtype=torch.int32, device="cuda")
        torch.cuda.synchronize()
        eng.select_slots_device(d, b0, stream=side.cuda_stream)
        eng.pods_reset(4 * N)  # no synchronise in between: the reset waits for the call's gather
        m = PodTable(4 * N)
        late = np.sort(rng.choice(np.arange(N, 4 * N), 30_000, replace=False)).astype(np.uint32)
        lp = sc.pods_for("synth20k", len(late), seed=10)
        eng.pods_seed_slots(late, lp)
        m.seed(late, lp)
        eng.select_slots_device(d, b1, stream=side.cuda_stream)
        side.synchronize()
        inside = sl < N
        wb0 = np.full(len(sl), -1, np.int32)
        wb0[inside] = sc.expected(offers, {k: np.ascontiguousarray(v[sl[inside]]) for k, v in pods.items()})[0]
        sc.check("before the reset", b0.cpu().numpy(), None, wb0, None)
        sc.check("after the reset", b1.cpu().numpy(), None, sc.expected(offers, m.rows(sl))[0], None)
        assert (b1.cpu().numpy()[~np.isin(sl, late)] == db[0]).all()
        edge = np.array([0, 4 * N - 1], np.uint32)  # the first and last row of the larger table, and one past it
        best, t5 = run_slots_device(eng, np.append(edge, 4 * N), True)
        wb, wt = sc.expected(offers, m.rows(edge))
        sc.check("edge rows", best[:2], t5[:2], wb, wt)
        assert best[0] == db[0] and best[2] == -1 and (t5[2] == -1).all()


def test_device_and_column_calls_interleaved():
    """slot-list and column calls, plain and gathered, with and without top-5, on the current stream and on a side
    stream, at changing sizes on one ctx: every call is checked"""
    import torch

    m, eb, et, _ = tracked("synth100k")
    rng = np.random.default_rng(31)
    side = torch.cuda.Stream(device="cuda:0")
    steps = [("slots", 40_001), ("cols", 40_001), ("slots_gather", 5_003), ("cols_gather", 196_609), ("slots", 196_609),
             ("slots_side", 16_385), ("cols", 1), ("slots_gather", 70_003), ("slots_side", 4_096), ("cols_gather", 5_003),
             ("slots", 1)]
    eng = seeded_engine("synth100k")
    try:
        for i, (kind, n) in enumerate(steps):
            sl = slot_list(rng, n, str(rng.choice(SHAPES)))
            what = f"step {i} ({kind}, n={n})"
            if kind == "slots":
                got = run_slots_device(eng, sl, i % 2 == 0)
            elif kind == "slots_side":
                got = run_slots_device(eng, sl, True, stream=side)
            elif kind == "cols":
                got = sc.run_device(eng, m.rows(sl), True)
            elif kind == "cols_gather":
                got = sc.run_gather(eng, m.rows(sl), True, 3)
            else:
                vecs = [torch.full((n + 10,), sc.SENTINEL, dtype=torch.int32, device="cuda") for _ in range(2)]
                d_t5 = torch.full((5 * n,), sc.SENTINEL, dtype=torch.int32, device="cuda")
                d = d_list(sl)
                torch.cuda.synchronize()
                eng.select_slots_device_gather(d, [v.data_ptr() for v in vecs], 3, d_top5=d_t5)
                torch.cuda.synchronize()
                h = [v.cpu().numpy() for v in vecs]
                assert np.array_equal(h[0], h[1]), what
                assert (h[0][:3] == sc.SENTINEL).all() and (h[0][3 + n:] == sc.SENTINEL).all(), what
                got = (h[0][3:3 + n], d_t5.cpu().numpy().reshape(n, 5))
            sc.check(what, got[0], got[1], eb[sl], et[sl] if got[1] is not None else None)
    finally:
        eng.close()
