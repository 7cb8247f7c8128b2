"""GPU tests of the pending set of the pod table (rpk_pods_mark_pending, rpk_select_pending,
rpk_pods_pending_list_device).

A numpy vector of flags is the model: the list the device builds must be np.flatnonzero(flags), and the select over it
must equal, row for row, rpk_select_slots over that list and the oracle's result per slot (tracked() of
test_select_slots_gpu.py).  Every output starts as SENTINEL, so an entry the kernels never write shows up."""
import ctypes as C
import zlib

import numpy as np
import pytest

import rpk
import select_plan_cases as sc
from test_select_sequences_gpu import FORCE, MENU
from test_select_slots_gpu import R, TRACKED, PodTable, run_slots, seeded_engine, tracked

pytestmark = pytest.mark.gpu

EINVAL, ESTATE = rpk._ffi.RPK_EINVAL, rpk._ffi.RPK_ESTATE
TILE = 4096  # slots a CTA of k_pod_pending turns into list entries per round (256 threads x 16 slots)
SLOT_SENTINEL = 0xFFFFFFF7


def mark_all(eng, flags):
    """the whole flag column := flags"""
    eng.pods_mark_pending(np.arange(len(flags), dtype=np.uint32), flags)


def flags_with(rng, N, n):
    """exactly n of N flags set (values 1..255: any non-zero byte marks)"""
    f = np.zeros(N, np.uint8)
    f[rng.choice(N, n, replace=False)] = rng.integers(1, 256, n)
    return f


def run_pending(eng, cap, top5, want_slots=True):
    best = np.full(cap, sc.SENTINEL, np.int32)
    t5 = np.full((cap, 5), sc.SENTINEL, np.int32) if top5 else None
    slots = np.full(cap, SLOT_SENTINEL, np.uint32) if want_slots else None
    got = eng.select_pending(cap, want_top5=top5, want_slots=want_slots, out_best=best, out_top5=t5, out_slots=slots)
    n = len(got[1])
    assert (best[n:] == sc.SENTINEL).all() and (t5 is None or (t5[n:] == sc.SENTINEL).all()), "written beyond n_pending"
    assert slots is None or (slots[n:] == SLOT_SENTINEL).all(), "slots_out written beyond n_pending"
    return got


def list_device(eng, N, stream=None):
    """rpk_pods_pending_list_device -> (the whole d_slots_out of N entries, n)"""
    import torch

    d_out = torch.full((max(N, 1),), SLOT_SENTINEL - (1 << 32), dtype=torch.int32, device="cuda")
    d_n = torch.full((1,), -1, dtype=torch.int32, device="cuda")
    torch.cuda.synchronize()
    eng.pods_pending_list_device(d_out, d_n, stream=stream.cuda_stream if stream is not None else None)
    torch.cuda.synchronize()
    return d_out.cpu().numpy().view(np.uint32), int(d_n.item())


def check_list(label, out, n, flags):
    want = np.flatnonzero(flags).astype(np.uint32)
    assert n == len(want), f"{label}: n = {n}, {len(want)} flags are set"
    assert np.array_equal(out[:n], want), f"{label}: list differs at {np.nonzero(out[:n] != want)[0][:6].tolist()}"
    assert (out[n:] == SLOT_SENTINEL).all(), f"{label}: written beyond n"


def patterns(rng, name):
    """(label, flags) over the tracked table: every density and shape, and counts on both sides of the latency path, of
    the fused kernel's size and of one sub-batch of the host pipeline"""
    N = TRACKED
    one = lambda s: np.bincount([s], minlength=N).astype(np.uint8)  # noqa: E731
    yield "none", np.zeros(N, np.uint8)
    yield "first slot", one(0)
    yield "last slot", one(N - 1)
    yield "a middle slot", one(N // 2 + 7)
    for n in (4096, 4097, 10_486, 16_384, 16_385, R):
        yield f"{n} random slots", flags_with(rng, N, n)
    runs = np.zeros(N, np.uint8)
    for s in rng.choice(N - 3000, 40, replace=False):
        runs[s:s + rng.integers(1, 3000)] = 1
    yield "clustered runs", runs
    if name == "synth100k":
        yield "alternating slots", (np.arange(N) & 1).astype(np.uint8)
        yield "half", (rng.random(N) < 0.5).astype(np.uint8)
        yield "every slot", np.full(N, 255, np.uint8)


@pytest.mark.parametrize("force", FORCE)
@pytest.mark.parametrize("name", MENU)
def test_select_pending_equals_select_slots_and_oracle(name, force):
    _, eb, et, _ = tracked(name)
    rng = np.random.default_rng(zlib.crc32(f"pending/{name}/{force}".encode()))
    eng = seeded_engine(name, force)
    try:
        for k, (what, flags) in enumerate(patterns(rng, name)):
            label = f"{name} force={force} {what}"
            mark_all(eng, flags)
            sl = np.flatnonzero(flags).astype(np.uint32)
            cap = len(sl) + (k % 3)  # exact and roomier capacities
            hb, ht = run_slots(eng, sl, True) if len(sl) else (np.zeros(0, np.int32), np.zeros((0, 5), np.int32))
            for top5, want_slots in ((True, True), (False, True), (True, False), (False, False)):
                slots, best, t5 = run_pending(eng, cap, top5, want_slots)
                assert len(best) == len(sl), f"{label}: n_pending = {len(best)}, {len(sl)} flags are set"
                assert not want_slots or np.array_equal(slots, sl), f"{label}: slots_out is not flatnonzero(flags)"
                sc.check(f"{label} top5={top5}: pending vs oracle", best, t5, eb[sl], et[sl] if top5 else None)
                sc.check(f"{label} top5={top5}: pending vs select_slots", best, t5, hb, ht if top5 else None)
    finally:
        eng.close()


def test_compaction_boundaries():
    """table sizes around the 16-slot load, the CTA tile and one tile per SM, and large ones; random flags with the last
    slot set, and only the last slot set; the tail of the output stays untouched"""
    sms = sc.sm_count()
    sizes = [1, 15, 16, 17, 63, 64, 65, TILE - 1, TILE, TILE + 1, sms * TILE - 1, sms * TILE, sms * TILE + 1, 1 << 20, (4 << 20) + 37]
    rng = np.random.default_rng(41)
    with rpk.Engine(1) as eng:
        for N in sizes:
            eng.pods_reset(N)
            out, n = list_device(eng, N)
            check_list(f"N={N} after the reset", out, n, np.zeros(N, np.uint8))
            for density in (0.5, 0.01):
                flags = (rng.random(N) < density).astype(np.uint8)
                flags[N - 1] = 1
                mark_all(eng, flags)
                check_list(f"N={N} density {density}", *list_device(eng, N), flags)
            flags = np.zeros(N, np.uint8)
            flags[N - 1] = 1
            mark_all(eng, flags)
            check_list(f"N={N} last slot only", *list_device(eng, N), flags)
            mark_all(eng, np.ones(N, np.uint8))
            check_list(f"N={N} every slot", *list_device(eng, N), np.ones(N, np.uint8))
        eng.pods_reset(0)
        out, n = list_device(eng, 0)
        assert n == 0 and (out == SLOT_SENTINEL).all()


def test_mark_semantics_against_a_model():
    """seeded programs of mark / clear / re-mark / seed / reset / select against numpy flags and a PodTable"""
    offers = sc.table("synth300")
    pool, _, _ = sc.batch("synth300", R)
    for seed in range(3):
        rng = np.random.default_rng(100 + seed)
        with rpk.Engine(1) as eng:
            eng.upload_offers(offers)
            N = int(rng.integers(3000, 60_000))
            eng.pods_reset(N)
            m, flags = PodTable(N), np.zeros(N, np.uint8)
            for step in range(40):
                op = rng.choice(["mark", "clear", "mixed", "seed", "reset", "select", "select"])
                k = int(rng.integers(1, min(N, 5000)))
                sl = np.sort(rng.choice(N, k, replace=False)).astype(np.uint32)
                if op in ("mark", "clear", "mixed"):
                    v = {"mark": np.ones(k, np.uint8), "clear": np.zeros(k, np.uint8), "mixed": rng.integers(0, 2, k).astype(np.uint8)}[op]
                    eng.pods_mark_pending(sl, v)
                    if step % 3 == 0:
                        eng.pods_mark_pending(sl, v)  # idempotent
                    flags[sl] = v
                elif op == "seed":  # changes columns, no flag
                    at = int(rng.integers(0, R - k))
                    pods = {c: np.ascontiguousarray(x[at:at + k]) for c, x in pool.items()}
                    eng.pods_seed_slots(sl, pods)
                    m.seed(sl, pods)
                elif op == "reset":
                    N = int(rng.integers(3000, 60_000))
                    eng.pods_reset(N)
                    m, flags = PodTable(N), np.zeros(N, np.uint8)
                else:
                    want = np.flatnonzero(flags).astype(np.uint32)
                    slots, best, t5 = run_pending(eng, N, True)
                    assert np.array_equal(slots, want), f"seed {seed} step {step}: the pending list differs from the model"
                    if len(want):
                        wb, wt = sc.expected(offers, m.rows(want))
                        sc.check(f"seed {seed} step {step}", best, t5, wb, wt)
            out, n = list_device(eng, N)
            check_list(f"seed {seed}: final list", out, n, flags)


def test_mark_refusals_write_nothing():
    with rpk.Engine(1) as eng:
        with pytest.raises(rpk.RpkError) as ei:
            eng.pods_mark_pending(np.array([0], np.uint32), np.array([1], np.uint8))
        assert ei.value.code == ESTATE
        N = 1000
        eng.pods_reset(N)
        flags = np.zeros(N, np.uint8)
        flags[[3, 500, 999]] = 1
        mark_all(eng, flags)
        c0 = eng.launch_count()
        for bad in ([5, 4], [7, 7], [1, N], [0xFFFFFFFF], [2, 9, 8, 20]):
            with pytest.raises(rpk.RpkError) as ei:
                eng.pods_mark_pending(np.array(bad, np.uint32), np.ones(len(bad), np.uint8))
            assert ei.value.code == EINVAL, bad
        assert eng._lib.rpk_pods_mark_pending(eng._ctx, 1, None, None) == EINVAL
        assert eng.launch_count() == c0
        eng.pods_mark_pending(np.zeros(0, np.uint32), np.zeros(0, np.uint8))  # a no-op
        assert eng.launch_count() == c0
        check_list("after the refusals", *list_device(eng, N), flags)


def test_select_pending_refusals():
    _, eb, et, _ = tracked("synth20k")
    G = len(sc.table("synth20k")["mem_gb"])
    rng = np.random.default_rng(43)
    eng = seeded_engine("synth20k")
    try:
        for n in (5, 4097, 40_001):
            flags = flags_with(rng, TRACKED, n)
            mark_all(eng, flags)
            run_pending(eng, n, True)  # sizes the scratch
            s0 = eng.stats()
            best = np.full(n, sc.SENTINEL, np.int32)
            t5 = np.full((n, 5), sc.SENTINEL, np.int32)
            slots = np.full(n, SLOT_SENTINEL, np.uint32)
            with pytest.raises(rpk.RpkError) as ei:
                eng.select_pending(n - 1, want_top5=True, out_best=best[: n - 1], out_top5=t5[: n - 1], out_slots=slots[: n - 1])
            assert ei.value.code == EINVAL and ei.value.n_pending == n
            assert (best == sc.SENTINEL).all() and (t5 == sc.SENTINEL).all() and (slots == SLOT_SENTINEL).all()
            s1 = eng.stats()
            assert s1["select_calls"] == s0["select_calls"] and s1["offer_scores"] == s0["offer_scores"]
            sl = np.flatnonzero(flags)
            slots, best, t5 = run_pending(eng, n, True)  # the next valid call is right, and is counted once
            sc.check(f"n={n} after the refusal", best, t5, eb[sl], et[sl])
            s2 = eng.stats()
            assert s2["select_calls"] == s1["select_calls"] + 1 and s2["offer_scores"] == s1["offer_scores"] + n * G
        n = C.c_uint32(7)
        assert eng._lib.rpk_select_pending(eng._ctx, 0, None, None, None, None) == EINVAL  # n_pending is required
        assert eng._lib.rpk_select_pending(eng._ctx, 10, None, C.cast(C.byref(n), C.c_void_p), None, None) == EINVAL and n.value == 7
        mark_all(eng, np.zeros(TRACKED, np.uint8))
        s0 = eng.stats()
        assert eng._lib.rpk_select_pending(eng._ctx, 0, None, C.cast(C.byref(n), C.c_void_p), None, None) == 0 and n.value == 0
        assert eng.stats()["select_calls"] == s0["select_calls"]  # zero pending: not a select
    finally:
        eng.close()
    with rpk.Engine(1) as e:  # no pod table, then no offer table
        e.upload_offers(sc.table("synth300"))
        with pytest.raises(rpk.RpkError) as ei:
            e.select_pending(4)
        assert ei.value.code == ESTATE
        import torch

        with pytest.raises(rpk.RpkError) as ei:
            e.pods_pending_list_device(torch.zeros(4, dtype=torch.int32, device="cuda"), torch.zeros(1, dtype=torch.int32, device="cuda"))
        assert ei.value.code == ESTATE
    with rpk.Engine(1) as e:
        e.pods_reset(16)
        c0 = e.launch_count()
        with pytest.raises(rpk.RpkError) as ei:
            e.select_pending(4)
        assert ei.value.code == ESTATE and e.launch_count() == c0
        d_n = torch.zeros(1, dtype=torch.int32, device="cuda")
        assert e._lib.rpk_pods_pending_list_device(e._ctx, 0, None, C.c_void_p(d_n.data_ptr()), None) == EINVAL
        assert e._lib.rpk_pods_pending_list_device(e._ctx, 0, C.c_void_p(d_n.data_ptr()), None, None) == EINVAL
        assert e._lib.rpk_pods_pending_list_device(e._ctx, 1, C.c_void_p(d_n.data_ptr()), C.c_void_p(d_n.data_ptr()), None) == EINVAL
        with pytest.raises(ValueError):  # the binding: one entry per slot of the table
            e.pods_pending_list_device(torch.zeros(15, dtype=torch.int32, device="cuda"), d_n)
        assert e.launch_count() == c0


def test_host_calls_right_after_a_device_select():
    """a host mark and a host select_pending issued right after a device select on a side stream, no synchronise in
    between: the device call reads the table before them, and they see it finished"""
    import torch

    from test_select_slots_device_gpu import d_list

    _, eb, et, _ = tracked("synth100k")
    rng = np.random.default_rng(47)
    side = torch.cuda.Stream(device="cuda:0")
    eng = seeded_engine("synth100k")
    try:
        flags = flags_with(rng, TRACKED, 150_000)
        mark_all(eng, flags)
        for step in range(3):
            sl = np.sort(rng.choice(TRACKED, 300_000, replace=False)).astype(np.uint32)
            d = d_list(sl)
            d_best = torch.full((len(sl),), sc.SENTINEL, dtype=torch.int32, device="cuda")
            d_t5 = torch.full((5 * len(sl),), sc.SENTINEL, dtype=torch.int32, device="cuda")
            torch.cuda.synchronize()
            eng.select_slots_device(d, d_best, d_t5, stream=side.cuda_stream)
            flip = np.sort(rng.choice(TRACKED, 20_000, replace=False)).astype(np.uint32)
            flags[flip] ^= 1
            eng.pods_mark_pending(flip, flags[flip])
            slots, best, t5 = run_pending(eng, TRACKED, True)
            want = np.flatnonzero(flags)
            assert np.array_equal(slots, want), f"step {step}: the pending list"
            sc.check(f"step {step}: pending select", best, t5, eb[want], et[want])
            side.synchronize()
            sc.check(f"step {step}: device select", d_best.cpu().numpy(), d_t5.cpu().numpy().reshape(-1, 5), eb[sl], et[sl])
    finally:
        eng.close()


def test_captured_list_replays_read_the_current_flags():
    import torch

    N = 300_001
    rng = np.random.default_rng(53)
    st = torch.cuda.Stream(device="cuda:0")
    with rpk.Engine(1) as eng:
        eng.pods_reset(N)
        flags = (rng.random(N) < 0.1).astype(np.uint8)
        mark_all(eng, flags)
        d_out = torch.full((N,), SLOT_SENTINEL - (1 << 32), dtype=torch.int32, device="cuda")
        d_n = torch.full((1,), -1, dtype=torch.int32, device="cuda")
        torch.cuda.synchronize()
        eng.pods_pending_list_device(d_out, d_n, stream=st.cuda_stream)  # one call of the size before the capture
        st.synchronize()
        g = torch.cuda.CUDAGraph()
        c0 = eng.launch_count()
        with torch.cuda.graph(g, stream=st):
            eng.pods_pending_list_device(d_out, d_n, stream=torch.cuda.current_stream().cuda_stream)
        assert eng.launch_count() == c0 + 1  # one kernel, no memset
        for k in range(4):
            flip = np.sort(rng.choice(N, 5000 * (k + 1), replace=False)).astype(np.uint32)
            flags[flip] ^= 1
            eng.pods_mark_pending(flip, flags[flip])
            d_out.fill_(SLOT_SENTINEL - (1 << 32))
            torch.cuda.synchronize()
            g.replay()
            torch.cuda.synchronize()
            check_list(f"replay {k}", d_out.cpu().numpy().view(np.uint32), int(d_n.item()), flags)


def test_list_beside_a_device_select_and_a_sweep():
    """the list kernel on a stream of its own while a 1M-row device select and a 1M-slot sweep run on two others"""
    import torch

    from test_select_slots_device_gpu import d_list

    _, eb, _, _ = tracked("synth100k")
    rng = np.random.default_rng(59)
    s_sel, s_sweep, s_list = (torch.cuda.Stream(device="cuda:0") for _ in range(3))
    eng = seeded_engine("synth100k")
    try:
        flags = (rng.random(TRACKED) < 0.3).astype(np.uint8)
        mark_all(eng, flags)
        sl = np.arange(TRACKED, dtype=np.uint32)
        d = d_list(sl)
        d_best = torch.full((TRACKED,), sc.SENTINEL, dtype=torch.int32, device="cuda")
        recs = torch.from_numpy(rpk.synth.make_status_records(TRACKED, 0, 0.0, stride=16)).cuda()
        prev = torch.zeros(TRACKED, dtype=torch.int64, device="cuda")
        ch = torch.zeros(TRACKED, dtype=torch.int32, device="cuda")
        nch = torch.zeros(1, dtype=torch.int32, device="cuda")
        d_out = torch.full((TRACKED,), SLOT_SENTINEL - (1 << 32), dtype=torch.int32, device="cuda")
        d_n = torch.full((1,), -1, dtype=torch.int32, device="cuda")
        torch.cuda.synchronize()
        eng.status_diff_device(recs, 16, prev, ch, nch, stream=s_sweep.cuda_stream)
        eng.pods_pending_list_device(d_out, d_n, stream=s_list.cuda_stream)
        eng.select_slots_device(d, d_best, stream=s_sel.cuda_stream)
        torch.cuda.synchronize()
        check_list("beside a select and a sweep", d_out.cpu().numpy().view(np.uint32), int(d_n.item()), flags)
        sc.check("the select beside it", d_best.cpu().numpy(), None, eb, None)
        assert int(nch.item()) == TRACKED  # a first sweep reports every slot
    finally:
        eng.close()


def test_multi_gpu_ctx():
    import importlib

    import torch

    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    peer = importlib.import_module("k8s-runpod-kubelet_b200.peer")
    _, eb, et, _ = tracked("synth100k")
    rng = np.random.default_rng(61)
    eng = seeded_engine("synth100k", n_gpus=2)
    try:
        for n in (3, 4097, 400_001):
            flags = flags_with(rng, TRACKED, n)
            mark_all(eng, flags)
            sl = np.flatnonzero(flags).astype(np.uint32)
            hb, ht = run_slots(eng, sl, True)
            for top5 in (True, False):
                slots, best, t5 = run_pending(eng, n, top5)
                assert np.array_equal(slots, sl)
                sc.check(f"2 GPUs n={n} top5={top5}: vs oracle", best, t5, eb[sl], et[sl] if top5 else None)
                sc.check(f"2 GPUs n={n} top5={top5}: vs select_slots", best, t5, hb, ht if top5 else None)
            for s in range(2):
                with torch.cuda.device(s):
                    t = peer.as_int32_tensor(eng.best_device_ptr(s), n, torch.device("cuda", s))
                    assert np.array_equal(t.cpu().numpy(), eb[sl]), f"GPU {s} does not hold the whole vector"
    finally:
        eng.close()
