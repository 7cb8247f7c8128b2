"""GPU tests of the pending results (rpk_select_pending_changed): reselect only the pending slots whose columns or offer
table changed since their last report, and report only the lists that changed.

The model is a per-slot mirror that applies every report.  After every call, for every pending slot, the mirror must
equal rpk_select_slots over the pending list and the oracle; what a call reselects and reports is checked against the
rule of include/rpk.h where a test controls it (seeds, uploads, marks, resets)."""
import ctypes as C
import time
import zlib

import numpy as np
import pytest

import rpk
import select_plan_cases as sc
from test_select_sequences_gpu import FORCE, MENU
from test_select_slots_gpu import COLS, R, TRACKED, PodTable, run_slots, seeded_engine, tracked

pytestmark = pytest.mark.gpu

EINVAL, ESTATE = rpk._ffi.RPK_EINVAL, rpk._ffi.RPK_ESTATE
TILE = 4096  # slots a CTA of the compaction turns into list entries per round (256 threads x 16 slots)
SLOT_SENTINEL = 0xFFFFFFF7
SLEEP_CYCLES = 2_000_000_000  # about 1 s at the H100's SM clock


class Mirror:
    """the caller's per-slot copy of what the call reported"""

    def __init__(self, N):
        self.best = np.full(N, sc.SENTINEL, np.int32)
        self.top5 = np.full((N, 5), sc.SENTINEL, np.int32)

    def apply(self, slots, best, top5):
        assert np.all(np.diff(slots.astype(np.int64)) > 0), "reported slots are not strictly ascending"
        assert np.array_equal(best, top5[:, 0]), "best is not top5[:, 0] on a reported row"
        self.best[slots], self.top5[slots] = best, top5


def call(eng, cap):
    """rpk_select_pending_changed with sentinel-filled outputs of capacity cap -> (n_pending, n_reselected, slots, best,
    top5); nothing beyond the reported rows is written"""
    slots = np.full(cap, SLOT_SENTINEL, np.uint32)
    best = np.full(cap, sc.SENTINEL, np.int32)
    t5 = np.full((cap, 5), sc.SENTINEL, np.int32)
    got = eng.select_pending_changed(cap, out_slots=slots, out_best=best, out_top5=t5)
    n = len(got[2])
    assert n <= got[1] <= got[0], f"n_changed {n}, n_reselected {got[1]}, n_pending {got[0]}"
    assert (slots[n:] == SLOT_SENTINEL).all() and (best[n:] == sc.SENTINEL).all() and (t5[n:] == sc.SENTINEL).all(), "written beyond n_changed"
    return got


def step(eng, mirror, cap):
    got = call(eng, cap)
    mirror.apply(*got[2:])
    return got


def mark_only(eng, N, slots):
    f = np.zeros(N, np.uint8)
    f[slots] = 1
    eng.pods_mark_pending(np.arange(N, dtype=np.uint32), f)
    return np.flatnonzero(f).astype(np.uint32)


def check_mirror(label, eng, mirror, pending, want_best=None, want_top5=None):
    """mirror == rpk_select_slots over the pending list (== the oracle, when given)"""
    if not len(pending):
        return
    hb, ht = run_slots(eng, pending, True)
    sc.check(f"{label}: mirror vs select_slots", mirror.best[pending], mirror.top5[pending], hb, ht)
    if want_best is not None:
        sc.check(f"{label}: mirror vs oracle", mirror.best[pending], mirror.top5[pending], want_best, want_top5)


@pytest.mark.parametrize("force", FORCE)
@pytest.mark.parametrize("name", MENU)
def test_first_call_reports_every_pending_slot_then_nothing(name, force):
    _, eb, et, _ = tracked(name)
    rng = np.random.default_rng(zlib.crc32(f"changed/{name}/{force}".encode()))
    eng = seeded_engine(name, force)
    try:
        pend = np.union1d(rng.choice(TRACKED, 30_000, replace=False), [0, TRACKED - 1]).astype(np.uint32)
        if name == "synth100k":
            pend = np.arange(TRACKED, dtype=np.uint32)
        mark_only(eng, TRACKED, pend)
        m = Mirror(TRACKED)
        c0 = eng.launch_count()
        n_p, n_r, slots, _, _ = step(eng, m, len(pend))
        assert n_p == n_r == len(slots) == len(pend) and np.array_equal(slots, pend), f"{name} {force}: the first call reports every pending slot"
        assert eng.launch_count() == c0 + 3, "a reselecting call is three launches per GPU (stale step, reselect, diff)"
        check_mirror(f"{name} force={force}", eng, m, pend, eb[pend], et[pend])
        for cap in (len(pend), 0):  # a steady call needs no capacity
            s0, c0 = eng.stats(), eng.launch_count()
            n_p, n_r, slots, _, _ = call(eng, cap)
            assert (n_p, n_r, len(slots)) == (len(pend), 0, 0), f"{name} {force}: a steady call reselects nothing"
            assert eng.launch_count() == c0 + 1, "a steady call is one launch per GPU"
        assert eng.stats()["select_calls"] == s0["select_calls"] and eng.stats()["offer_scores"] == s0["offer_scores"]
    finally:
        eng.close()


def test_seeds_reselect_exactly_the_changed_pending_rows():
    name = "synth20k"
    offers = sc.table(name)
    m_tab, eb, et, seeds = tracked(name)
    rng = np.random.default_rng(71)
    eng = seeded_engine(name)
    try:
        pend = mark_only(eng, TRACKED, np.sort(rng.choice(TRACKED, 50_000, replace=False)))
        m = Mirror(TRACKED)
        step(eng, m, TRACKED)
        tab = PodTable(TRACKED)
        tab.cols = {k: v.copy() for k, v in m_tab.cols.items()}
        # identical columns, pending and not: nothing reselected
        same = np.sort(rng.choice(TRACKED, 20_000, replace=False)).astype(np.uint32)
        eng.pods_seed_slots(same, tab.rows(same))
        n_p, n_r, sl, _, _ = call(eng, TRACKED)
        assert (n_r, len(sl)) == (0, 0), "seeding identical columns reselects nothing"
        # new columns on 3000 pending and 3000 other slots: exactly the pending ones are reselected
        pool, _, _ = sc.batch(name, R, seed=5)
        on = np.sort(rng.choice(pend, 3000, replace=False))
        off = np.sort(rng.choice(np.setdiff1d(np.arange(TRACKED, dtype=np.uint32), pend), 3000, replace=False))
        sl_seed = np.union1d(on, off).astype(np.uint32)
        pods = {k: np.ascontiguousarray(v[:len(sl_seed)]) for k, v in pool.items()}
        before_b, before_t = m.best[sl_seed].copy(), m.top5[sl_seed].copy()
        eng.pods_seed_slots(sl_seed, pods)
        tab.seed(sl_seed, pods)
        n_p, n_r, sl, b, t = step(eng, m, TRACKED)
        old, new = m_tab.rows(on), tab.rows(on)
        changed_cols = np.any([(old[k].view(np.uint8).reshape(len(on), -1) != new[k].view(np.uint8).reshape(len(on), -1)).any(axis=1) for k in COLS], axis=0)
        assert n_p == len(pend) and n_r == int(changed_cols.sum()), f"reselected {n_r}, {int(changed_cols.sum())} pending rows changed"
        wb, wt = sc.expected(offers, tab.rows(on))
        was = np.isin(sl_seed, on)
        want = on[(wt != before_t[was]).any(axis=1)]
        assert np.array_equal(sl, want), "reported != the pending slots whose oracle list changed"
        sc.check("seeded pending rows", m.best[on], m.top5[on], wb, wt)
        check_mirror("after the seeds", eng, m, pend)
        assert call(eng, TRACKED)[1] == 0
    finally:
        eng.close()


def test_offer_uploads():
    name = "synth20k"
    offers = sc.table(name)
    m_tab, eb, et, _ = tracked(name)
    rng = np.random.default_rng(73)
    eng = seeded_engine(name)
    try:
        pend = mark_only(eng, TRACKED, np.sort(rng.choice(TRACKED, 40_000, replace=False)))
        m = Mirror(TRACKED)
        step(eng, m, TRACKED)
        G = len(offers["mem_gb"])
        # the identical table again: everything pending reselected, nothing reported
        eng.upload_offers(offers)
        s0 = eng.stats()
        n_p, n_r, sl, _, _ = step(eng, m, TRACKED)
        assert (n_r, len(sl)) == (len(pend), 0)
        s1 = eng.stats()
        assert s1["select_calls"] == s0["select_calls"] + 1 and s1["offer_scores"] == s0["offer_scores"] + len(pend) * G
        # one price changed: exactly the slots whose oracle list changed are reported
        rows = m_tab.rows(pend)
        old_b, old_t = m.best[pend].copy(), m.top5[pend].copy()
        used = np.bincount(old_t[old_t >= 0].ravel(), minlength=G)
        g = int(rng.choice(np.flatnonzero(used)))
        new = {k: v.copy() for k, v in offers.items()}
        for c in ("secure_price", "community_price"):
            if new[c][g] > 0:
                new[c][g] *= 1.7
        eng.upload_offers(new)
        n_p, n_r, sl, _, _ = step(eng, m, TRACKED)
        wb, wt = sc.expected(new, rows)
        assert n_r == len(pend) and np.array_equal(sl, pend[(wt != old_t).any(axis=1)]), "reported != slots whose list changed"
        assert len(sl) < len(pend)
        sc.check("after one price", m.best[pend], m.top5[pend], wb, wt)
        # permuted offers: the comparison is by index
        perm = rng.permutation(G)
        pt = {k: np.ascontiguousarray(v[perm]) for k, v in new.items()}
        eng.upload_offers(pt)
        n_p, n_r, sl, _, _ = step(eng, m, TRACKED)
        pb, ptt = sc.expected(pt, rows)
        assert np.array_equal(sl, pend[(ptt != wt).any(axis=1)])
        sc.check("after the permutation", m.best[pend], m.top5[pend], pb, ptt)
        check_mirror("after the uploads", eng, m, pend)
    finally:
        eng.close()


def test_mark_unmark_and_reset():
    name = "synth20k"
    offers = sc.table(name)
    m_tab, eb, et, _ = tracked(name)
    rng = np.random.default_rng(79)
    eng = seeded_engine(name)
    try:
        pend = mark_only(eng, TRACKED, np.sort(rng.choice(TRACKED, 20_000, replace=False)))
        m = Mirror(TRACKED)
        step(eng, m, TRACKED)
        away = np.sort(rng.choice(pend, 4000, replace=False))
        eng.pods_mark_pending(away, np.zeros(len(away), np.uint8))
        n_p, n_r, sl, _, _ = step(eng, m, TRACKED)
        assert (n_p, n_r, len(sl)) == (len(pend) - len(away), 0, 0)
        # back unchanged: not reported; back with new columns (a default row): reported where the list changes
        newcols = away[::2]
        eng.pods_seed_slots(newcols, {"req_mem_gb": np.full(len(newcols), 16, np.int32)})
        eng.pods_mark_pending(away, np.ones(len(away), np.uint8))
        n_p, n_r, sl, _, _ = step(eng, m, TRACKED)
        was_default = np.all([m_tab.rows(newcols)[k] == v for k, v in (("req_mem_gb", 16), ("req_vcpu", 0), ("req_ram_gb", 0), ("max_price", 0.5), ("cloud", 0))], axis=0)
        assert n_p == len(pend) and n_r == int((~was_default).sum())
        db, dt = sc.expected(offers, {"req_mem_gb": np.array([16], np.int32), "req_vcpu": None, "req_ram_gb": None, "max_price": None, "cloud": None})
        assert np.array_equal(sl, newcols[(et[newcols] != dt[0]).any(axis=1)])
        check_mirror("after mark / unmark", eng, m, pend)
        # reset: every pending slot reported again, at the same N and at another
        for N in (TRACKED, 70_001):
            eng.pods_reset(N)
            p2 = mark_only(eng, N, np.sort(rng.choice(N, 5000, replace=False)))
            m = Mirror(N)
            n_p, n_r, sl, _, _ = step(eng, m, N)
            assert n_p == n_r == 5000 and np.array_equal(sl, p2)
            sc.check(f"reset to {N}", m.best[p2], m.top5[p2], np.full(5000, db[0], np.int32), np.tile(dt[0], (5000, 1)))
    finally:
        eng.close()


def test_refusal_writes_and_counts_nothing():
    name = "synth20k"
    _, eb, et, _ = tracked(name)
    rng = np.random.default_rng(83)
    eng = seeded_engine(name)
    try:
        for n in (5, 4097, 40_001):
            eng.pods_reset(TRACKED)  # no stored result: every pending slot is to reselect
            pend = mark_only(eng, TRACKED, np.sort(rng.choice(TRACKED, n, replace=False)))
            s0, c0 = eng.stats(), eng.launch_count()
            slots = np.full(n - 1, SLOT_SENTINEL, np.uint32)
            best = np.full(n - 1, sc.SENTINEL, np.int32)
            t5 = np.full((n - 1, 5), sc.SENTINEL, np.int32)
            with pytest.raises(rpk.RpkError) as ei:
                eng.select_pending_changed(n - 1, out_slots=slots, out_best=best, out_top5=t5)
            assert ei.value.code == EINVAL and ei.value.n_pending == n and ei.value.n_reselected == n
            assert (slots == SLOT_SENTINEL).all() and (best == sc.SENTINEL).all() and (t5 == sc.SENTINEL).all()
            assert eng.stats() == s0 and eng.launch_count() == c0
            m = Mirror(TRACKED)
            n_p, n_r, sl, _, _ = step(eng, m, n)
            assert n_p == n_r == n and np.array_equal(sl, pend), "the next call reports what the refused one would have"
            check_mirror(f"n={n} after the refusal", eng, m, pend)
        v = C.c_uint32(7)
        p = C.cast(C.byref(v), C.c_void_p)
        lib, ctx = eng._lib, eng._ctx
        assert lib.rpk_select_pending_changed(ctx, 0, None, p, None, None, None, p) == EINVAL
        assert lib.rpk_select_pending_changed(ctx, 4, p, p, None, None, None, p) == EINVAL and v.value == 7
    finally:
        eng.close()
    with rpk.Engine(1) as e:
        e.upload_offers(sc.table("synth300"))
        with pytest.raises(rpk.RpkError) as ei:
            e.select_pending_changed(4)
        assert ei.value.code == ESTATE
    with rpk.Engine(1) as e:
        e.pods_reset(16)
        c0 = e.launch_count()
        with pytest.raises(rpk.RpkError) as ei:
            e.select_pending_changed(4)
        assert ei.value.code == ESTATE and e.launch_count() == c0


def test_interleaving_with_other_selects_a_sweep_and_a_device_call():
    import torch

    from test_select_slots_device_gpu import d_list

    name = "synth100k"
    eb, et = (x.copy() for x in tracked(name)[1:3])  # the oracle's cached arrays are shared: this test changes rows
    rng = np.random.default_rng(89)
    eng = seeded_engine(name)
    try:
        pend = mark_only(eng, TRACKED, np.sort(rng.choice(TRACKED, 100_000, replace=False)))
        m = Mirror(TRACKED)
        step(eng, m, TRACKED)
        eng.status_reset(TRACKED)
        for k in range(3):
            sl = np.sort(rng.choice(TRACKED, 200_000, replace=False)).astype(np.uint32)
            d = d_list(sl)
            d_best = torch.full((len(sl),), sc.SENTINEL, dtype=torch.int32, device="cuda")
            d_t5 = torch.full((5 * len(sl),), sc.SENTINEL, dtype=torch.int32, device="cuda")
            eng.select_slots_device(d, d_best, d_t5, stream=torch.cuda.current_stream().cuda_stream)  # sizes the call
            torch.cuda.synchronize()
            s = torch.cuda.Stream()
            ev = torch.cuda.Event()
            with torch.cuda.stream(s):
                torch.cuda._sleep(SLEEP_CYCLES)
                eng.select_slots_device(d, d_best, d_t5, stream=s.cuda_stream)
                ev.record(s)
            got = call(eng, TRACKED)
            t0 = time.monotonic()
            while not ev.query():
                assert time.monotonic() - t0 < 0.05, "the device select had not finished when the call returned"
                time.sleep(1e-4)
            assert got[1] == 0
            sc.check(f"round {k}: device select", d_best.cpu().numpy(), d_t5.cpu().numpy().reshape(-1, 5), eb[sl], et[sl])
            sp = run_slots(eng, pend, True)
            sc.check(f"round {k}: select_slots", *sp, eb[pend], et[pend])
            _, pb, pt = eng.select_pending(TRACKED, want_top5=True)
            sc.check(f"round {k}: select_pending", pb, pt, eb[pend], et[pend])
            recs = rpk.synth.make_status_records(TRACKED, k, 0.1, stride=16)
            eng.status_diff(recs)
            assert call(eng, TRACKED)[1] == 0, "other calls left the stored results alone"
            check_mirror(f"round {k}", eng, m, pend, eb[pend], et[pend])
            # columns change on some pending rows: only those are reselected
            hit = np.sort(rng.choice(pend, 1000, replace=False))
            eng.pods_seed_slots(hit, {"req_mem_gb": np.full(1000, 1 << 30, np.int32)})
            eb[hit], et[hit] = -1, -1
            n_p, n_r, sl2, _, _ = step(eng, m, TRACKED)
            assert n_r <= 1000 and np.isin(sl2, hit).all()
            check_mirror(f"round {k} after the seed", eng, m, pend, eb[pend], et[pend])
    finally:
        eng.close()


def test_compaction_boundaries():
    sms = sc.sm_count()
    sizes = [1, 15, 16, 17, TILE - 1, TILE + 1, sms * TILE - 1, sms * TILE + 1, 1 << 20, (4 << 20) + 37]
    offers = sc.table("synth300")
    db, dt = sc.expected(offers, {"req_mem_gb": np.array([16, 1 << 30], np.int32), "req_vcpu": None, "req_ram_gb": None, "max_price": None, "cloud": None})
    rng = np.random.default_rng(97)
    with rpk.Engine(1) as eng:
        eng.upload_offers(offers)
        for N in sizes:
            eng.pods_reset(N)
            m = Mirror(N)
            for what, sl in (("first", [0]), ("last", [N - 1]), ("first and last", [0, N - 1]), ("every", np.arange(N))):
                pend = mark_only(eng, N, np.asarray(sl, np.uint32))
                n_p, n_r, got, _, _ = step(eng, m, N)
                assert n_p == len(pend) and np.isin(got, pend).all(), f"N={N} {what}"
                want_b = np.full(len(pend), db[0], np.int32)
                sc.check(f"N={N} {what}", m.best[pend], m.top5[pend], want_b, np.tile(dt[0], (len(pend), 1)))
            # a random 1 % of the rows change to a pod nothing fits: exactly those are reselected and reported
            hit = np.sort(rng.choice(N, max(1, N // 100), replace=False)).astype(np.uint32)
            hit = np.union1d(hit, [N - 1]).astype(np.uint32)
            eng.pods_seed_slots(hit, {"req_mem_gb": np.full(len(hit), 1 << 30, np.int32)})
            n_p, n_r, got, _, _ = step(eng, m, N)
            want = hit if (dt[0] != dt[1]).any() else hit[:0]
            assert n_p == N and n_r == len(hit) and np.array_equal(got, want), f"N={N} 1 % changed"
            assert np.array_equal(m.top5[hit], np.tile(dt[1], (len(hit), 1)))
            assert call(eng, N)[1] == 0


def test_random_sequences_against_the_model():
    """several hundred steps of seeds, marks, offer uploads and resets, checked against the oracle after every call"""
    pool, _, _ = sc.batch("synth300", R)
    base = sc.table("synth300")
    G = len(base["mem_gb"])
    for seed in range(3):
        rng = np.random.default_rng(200 + seed)
        offers = {k: v.copy() for k, v in base.items()}
        with rpk.Engine(1) as eng:
            eng.upload_offers(offers)
            N = int(rng.integers(3000, 40_000))
            eng.pods_reset(N)
            tab, flags, m = PodTable(N), np.zeros(N, np.uint8), Mirror(N)
            stored = np.zeros(N, bool)  # the library holds a reported result for the slot
            fresh = np.zeros(N, bool)  # ... against the current offers and columns
            for stp in range(120):
                op = rng.choice(["mark", "mark", "seed", "seed", "offers", "reset", "call", "call", "call"])
                k = int(rng.integers(1, min(N, 3000)))
                sl = np.sort(rng.choice(N, k, replace=False)).astype(np.uint32)
                if op == "mark":
                    v = rng.integers(0, 2, k).astype(np.uint8)
                    eng.pods_mark_pending(sl, v)
                    flags[sl] = v
                elif op == "seed":
                    at = int(rng.integers(0, R - k))
                    pods = {c: np.ascontiguousarray(x[at:at + k]) for c, x in pool.items()}
                    if rng.random() < 0.3:
                        pods = tab.rows(sl)  # identical columns
                    before = tab.rows(sl)
                    eng.pods_seed_slots(sl, pods)
                    tab.seed(sl, pods)
                    same = np.all([(before[c].view(np.uint8).reshape(k, -1) == tab.rows(sl)[c].view(np.uint8).reshape(k, -1)).all(axis=1) for c in COLS], axis=0)
                    fresh[sl[~same]] = False
                elif op == "offers":
                    if rng.random() < 0.5:
                        g = rng.integers(0, G, 3)
                        offers["secure_price"][g] *= rng.uniform(0.5, 1.5, 3)
                    eng.upload_offers(offers)
                    fresh[:] = False
                elif op == "reset":
                    N = int(rng.integers(3000, 40_000))
                    eng.pods_reset(N)
                    tab, flags, m, stored, fresh = PodTable(N), np.zeros(N, np.uint8), Mirror(N), np.zeros(N, bool), np.zeros(N, bool)
                else:
                    pend = np.flatnonzero(flags).astype(np.uint32)
                    stale = pend[~(stored[pend] & fresh[pend])]
                    n_p, n_r, got, _, _ = step(eng, m, N)
                    assert n_p == len(pend) and n_r == len(stale), f"seed {seed} step {stp}: reselected {n_r}, the rule says {len(stale)}"
                    assert np.isin(got, stale).all()
                    stored[stale] = fresh[stale] = True
                    if len(pend):
                        wb, wt = sc.expected(offers, tab.rows(pend))
                        sc.check(f"seed {seed} step {stp}", m.best[pend], m.top5[pend], wb, wt)


def test_multi_gpu_ctx():
    import torch

    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    name = "synth100k"
    rng = np.random.default_rng(101)
    half = TRACKED // 2
    e1, e2 = seeded_engine(name), seeded_engine(name, n_gpus=2)
    try:
        for what, sl in (("first GPU only", rng.choice(half - 16, 3000, replace=False)),
                         ("second GPU only", half + 16 + rng.choice(half - 16, 3000, replace=False)),
                         ("straddling", np.arange(half - 2000, half + 2000)), ("random", rng.choice(TRACKED, 400_001, replace=False))):
            pend = np.sort(sl).astype(np.uint32)
            for e in (e1, e2):
                mark_only(e, TRACKED, pend)
            a, b = call(e1, TRACKED), call(e2, TRACKED)
            assert a[:2] == b[:2] and all(np.array_equal(x, y) for x, y in zip(a[2:], b[2:])), f"2 GPUs != 1 GPU: {what}"
            hit = np.sort(rng.choice(pend, 100, replace=False))
            for e in (e1, e2):
                e.pods_seed_slots(hit, {"req_mem_gb": np.full(100, 1 << 30, np.int32)})
            a, b = call(e1, TRACKED), call(e2, TRACKED)
            assert a[:2] == b[:2] and all(np.array_equal(x, y) for x, y in zip(a[2:], b[2:])), f"2 GPUs != 1 GPU after a seed: {what}"
    finally:
        e1.close()
        e2.close()
