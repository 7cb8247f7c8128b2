"""The one-process, several-shards ctx (rpk_create with n_gpus > 1) on ONE GPU.

RPK_TEST_SHARED_DEVICE=1 lets rpk_create accept a repeated device id, so `rpk.Engine(device_ids=[0] * n)` is an
n-shard ctx whose shards all live on GPU 0: each has its own streams, lanes, buffers and worker thread, and the shards
store into each other's vectors through plain device pointers, exactly as they do over NVLink.  Everything the host
entry points do per shard -- the row, slot, list and unit ranges, the worker threads, the in-ctx gather of the
assignment vector, the concatenation of the shards' changed lists -- runs here at n = 2, 3, 4 and 8 and is compared
bit for bit with the oracle and, where cheap, with the same call on a one-shard ctx.

Not covered here (these need several GPUs): peer stores over NVLink and cudaDeviceEnablePeerAccess itself,
rpk_peer_fence across devices and the bound / inline-wait gathers across devices -- a kernel of one shard that waits
for a kernel of another cannot be assumed to make progress when both share one GPU, so no test below queues one."""
import functools
import importlib
import os
import zlib
from contextlib import contextmanager

import numpy as np
import pytest

import oracle
import rpk
import select_plan_cases as sc
from status_slots_model import diff_slots
from test_host_after_device_gpu import SHARD_1_CASES, Rig, run_case
from test_select_pending_changed_gpu import SLOT_SENTINEL, Mirror, call, check_mirror, mark_only
from test_select_pending_gpu import run_pending
from test_select_sequences_gpu import FORCE
from test_select_slots_gpu import DEFAULT_POD, PodTable, run_slots

pytestmark = pytest.mark.gpu

EINVAL = rpk._ffi.RPK_EINVAL
NS = [2, 3, 4, 8]  # 3: total * s / n rounds unevenly; 8: RPK_MAX_GPUS
HOOK = "RPK_TEST_SHARED_DEVICE"
TABLES = ["synth20k", "many_queues", "packed_only", "full_int32", "stride64", "empty"]
P_MAX = 400_003  # two sub-batches per shard at n = 2: a cut inside a shard as well
POD_N = 100_003


@contextmanager
def shared_device(value="1"):
    old = os.environ.pop(HOOK, None)
    try:
        if value is not None:
            os.environ[HOOK] = value
        yield
    finally:
        os.environ.pop(HOOK, None)
        if old is not None:
            os.environ[HOOK] = old


def shared_engine(n):
    """an n-shard ctx with every shard on GPU 0 (the variable is read by rpk_create only)"""
    with shared_device():
        return rpk.Engine(device_ids=[0] * n)


def cuts(total, n):
    """shard_range of rpk_api.cu: shard s takes [cuts[s], cuts[s + 1])"""
    return [total * s // n for s in range(n + 1)]


def unit_cuts(N, n):
    """result_range of rpk_api.cu: the stored pending results are shared out by 16-slot units"""
    return [min(c * 16, N) for c in cuts((N + 15) // 16, n)]


def around(bounds, N):
    """the slots on both sides of every cut: lo - 1, lo, hi - 1, hi, inside [0, N)"""
    s = {b + d for b in bounds for d in (-1, 0)}
    return np.array(sorted(x for x in s if 0 <= x < N), np.uint32)


def shard_vectors(eng, rows):
    """every shard's copy of the full assignment vector, as torch views of `rows` elements"""
    import torch

    peer = importlib.import_module("k8s-runpod-kubelet_b200.peer")
    return [peer.as_int32_tensor(eng.best_device_ptr(s), rows, torch.device("cuda", 0)) for s in range(eng.n_gpus)]


def check_every_shard(label, eng, want, filled=None):
    """every shard holds `want` in rows [0, len(want)) and, where the views were filled before the call, SENTINEL after"""
    import torch

    torch.cuda.synchronize()
    for s, v in enumerate(shard_vectors(eng, filled or len(want))):
        h = v.cpu().numpy()
        sc.check(f"{label}: shard {s}'s vector", h[:len(want)], None, want, None)
        assert (h[len(want):] == sc.SENTINEL).all(), f"{label}: shard {s}'s vector written past row {len(want)}"


def fill_every_shard(eng, rows):
    import torch

    for v in shard_vectors(eng, rows):
        v.fill_(sc.SENTINEL)
    torch.cuda.synchronize()


# ---- rpk_create ---------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("value", [None, "0", ""])
def test_repeated_device_id_is_refused_without_the_hook(value):
    with shared_device(value):
        with pytest.raises(rpk.RpkError) as ei:
            rpk.Engine(device_ids=[0, 0])
    assert ei.value.code == EINVAL and "duplicate device id" in str(ei.value)
    with shared_device():
        for ids in ([0, -1], [0, 1 << 20]):  # the hook lifts that refusal only
            with pytest.raises(rpk.RpkError) as ei:
                rpk.Engine(device_ids=ids)
            assert ei.value.code == EINVAL and "out of range" in str(ei.value)
        with pytest.raises(rpk.RpkError):
            rpk.Engine(device_ids=[0] * 9)


# ---- select -------------------------------------------------------------------------------------------------------

def select_sizes(n):
    return sorted({0, 1, n - 1, n, n + 1, 3, 5, 50_001, 50_003, 300_007, P_MAX}, reverse=True)  # the largest first sizes the vectors


@pytest.mark.parametrize("name", TABLES)
@pytest.mark.parametrize("n", NS)
def test_sharded_select_gathers_into_every_shard(n, name):
    """shards with no rows, slices shorter than one 16-byte unit, shard and sub-batch cuts off the 16-byte grid: the
    caller's best / top5 and every shard's full vector equal the oracle, and no row past P is written"""
    pods, wb, wt = sc.batch(name, P_MAX)
    pods_n, nb, nt = sc.batch_without_optional(name, P_MAX)
    for force in FORCE:
        eng = shared_engine(n)
        try:
            with sc.forced(force):
                eng.upload_offers(sc.table(name))
            for k, P in enumerate(select_sizes(n)):
                for top5, nulls in ((True, False), (False, True)) if P > 50_000 else ((True, False), (False, False), (True, True), (False, True)):
                    label = f"{n} shards, {name} force={force} P={P} top5={top5} nulls={nulls}"
                    if k:
                        fill_every_shard(eng, P_MAX)
                    best, t5 = sc.run_host(eng, sc.head(pods_n if nulls else pods, P), top5)
                    eb, et = (nb, nt) if nulls else (wb, wt)
                    sc.check(label, best, t5, eb[:P], et[:P])
                    if k:
                        check_every_shard(label, eng, eb[:P], P_MAX)
                    else:
                        check_every_shard(label, eng, eb[:P])
        finally:
            eng.close()


@pytest.mark.parametrize("n", NS)
def test_small_batches_equal_the_one_shard_latency_path(n):
    """a one-shard ctx answers up to 4096 rows in one copy each way (select_small); a multi-shard ctx sends them down
    the pipeline: the results are the same"""
    for name, force in (("synth20k", None), ("packed_only", None), ("synth20k", "bitmap_grouped")):
        pods, wb, wt = sc.batch(name, P_MAX)
        e1, en = rpk.Engine(1), shared_engine(n)
        try:
            for e in (e1, en):
                with sc.forced(force):
                    e.upload_offers(sc.table(name))
            for P in (1, 2, n, 7, 100, 4095, 4096):
                for top5 in (False, True):
                    for rows in (sc.head(pods, P), sc.without_optional(sc.head(pods, P))):
                        a, b = sc.run_host(e1, rows, top5), sc.run_host(en, rows, top5)
                        sc.check(f"{n} shards vs one, {name} force={force} P={P}", b[0], b[1], a[0], a[1])
                    sc.check(f"{n} shards vs oracle, {name} P={P}", *sc.run_host(en, sc.head(pods, P), top5), wb[:P], wt[:P])
        finally:
            e1.close()
            en.close()


# ---- sweeps -------------------------------------------------------------------------------------------------------

def sweep_sizes(n):
    return sorted({0, 1, n - 1, n, 63 * n + 1, 30_001, 67_585})


@pytest.mark.parametrize("stride", [16, 32, 48, 64, 256])
@pytest.mark.parametrize("n", NS)
def test_sharded_sweeps(n, stride):
    """rpk_status_diff with codes and hashes over three sweeps (nothing, 5 % and everything changed), the table cut into
    n shards: the changed list comes back ascending over the shards"""
    synth = rpk.synth
    eng = shared_engine(n)
    try:
        for N in sweep_sizes(n):
            eng.status_reset(N)
            tab = oracle.StatusTable(N, stride) if N else None
            for sweep, frac in enumerate([0.0, 0.05, 1.0]):
                recs = synth.make_status_records(N, sweep, frac, stride=stride)
                idx, codes, hashes = eng.status_diff(recs, want_hashes=True, want_codes=True)
                label = f"{n} shards, stride {stride}, N={N}, sweep {sweep}"
                if not N:
                    assert len(idx) == 0 and len(codes) == 0, label
                    continue
                want = tab.diff(recs)
                assert np.array_equal(idx, want), f"{label}: changed list differs from the oracle"
                assert np.array_equal(codes, oracle.record_codes(recs)[want]), f"{label}: codes"
                assert np.array_equal(hashes, oracle.record_hashes(recs)), f"{label}: hashes"
    finally:
        eng.close()


@pytest.mark.parametrize("stride", [16, 48])
@pytest.mark.parametrize("n", NS)
def test_seeds_and_slot_sweeps_at_the_shard_cuts(n, stride):
    """rpk_status_seed, rpk_status_seed_slots and rpk_status_diff_slots with slots on both sides of every shard cut;
    lists inside one shard, lists that leave some shards empty, the cut slots alone, and every slot"""
    synth = rpk.synth
    rng = np.random.default_rng(zlib.crc32(f"slots/{n}/{stride}".encode()))
    eng = shared_engine(n)
    try:
        for N in (63 * n + 1, 30_001):
            c = cuts(N, n)
            edge = around(c, N)
            recs = [synth.make_status_records(N, s, 0.3 if s else 0.0, stride=stride) for s in range(8)]
            eng.status_reset(N)
            tab = oracle.StatusTable(N, stride)
            eng.status_seed(recs[0])
            tab.seed(recs[0])

            def whole(label, r):
                idx, got_codes, _ = eng.status_diff(r, want_codes=True)
                want = tab.diff(r)
                assert np.array_equal(idx, want), f"{n} shards, stride {stride}, N={N}, {label}: changed list"
                assert np.array_equal(got_codes, oracle.record_codes(r)[want]), f"{n} shards, N={N}, {label}: codes"

            def listed(label, sl, r):
                sl = np.asarray(sl, np.uint32)
                idx, got_codes = eng.status_diff_slots(sl, np.ascontiguousarray(r[sl]), want_codes=True)
                want = diff_slots(tab, sl, r[sl])
                assert np.array_equal(idx, want), f"{n} shards, stride {stride}, N={N}, {label}: changed list"
                assert np.array_equal(got_codes, oracle.record_codes(r)[want]), f"{n} shards, N={N}, {label}: codes"

            whole("after the seed", recs[0])  # nothing changed
            eng.status_seed_slots(edge, np.ascontiguousarray(recs[1][edge]))
            tab.seed_slots(edge, recs[1][edge])
            whole("after seeds at the cuts", recs[1])  # everything that changed but the seeded slots
            for s in range(n):  # wholly inside one shard: every other shard gets an empty part
                if c[s + 1] > c[s]:
                    listed(f"inside shard {s}", np.arange(c[s], c[s + 1]), recs[2])
            listed("every other shard", np.concatenate([np.arange(c[s], c[s + 1]) for s in range(0, n, 2)]), recs[3])
            listed("the cut slots", edge, recs[4])
            listed("one slot", [N - 1], recs[5])
            listed("a random tenth", np.sort(rng.choice(N, N // 10 + 1, replace=False)), recs[5])
            listed("every slot", np.arange(N), recs[6])
            whole("after the lists", recs[7])
    finally:
        eng.close()


@pytest.mark.parametrize("n", NS)
def test_tick(n):
    """rpk_tick without and with pods: the select on the lanes, the sweep on the status stream, on every shard"""
    synth = rpk.synth
    pods, wb, wt = sc.batch("synth20k", P_MAX)
    N = 30_001
    eng = shared_engine(n)
    try:
        eng.upload_offers(sc.table("synth20k"))
        tab = oracle.StatusTable(N, 16)
        for sweep, (P, frac) in enumerate([(0, 0.0), (50_003, 0.02), (5, 0.4), (0, 0.1), (P_MAX, 1.0), (n - 1, 0.05)]):
            recs = synth.make_status_records(N, sweep, frac, stride=16)
            best = np.full(P, sc.SENTINEL, np.int32)
            got = eng.tick(sc.head(pods, P) if P else None, recs, want_top5=True, out_best=best if P else None)
            want = tab.diff(recs)
            label = f"{n} shards, tick {sweep} with {P} pods"
            assert np.array_equal(got[2], want) and np.array_equal(got[3], oracle.record_codes(recs)[want]), f"{label}: sweep"
            if P:
                sc.check(label, got[0], got[1], wb[:P], wt[:P])
                check_every_shard(label, eng, wb[:P])
            else:
                assert got[0] is None and got[1] is None
    finally:
        eng.close()


# ---- pod table ----------------------------------------------------------------------------------------------------

@functools.lru_cache(maxsize=None)
def pod_rows():
    """(columns of POD_N pods, oracle best, oracle top5) on the synth20k table"""
    pods = sc.pods_for("synth20k", POD_N, seed=9)
    return (pods,) + tuple(sc.expected(sc.table("synth20k"), pods))


def pod_engine(eng, force=None):
    """offers uploaded, the pod table of POD_N slots seeded with pod_rows() in two lists that interleave"""
    pods = pod_rows()[0]
    with sc.forced(force):
        eng.upload_offers(sc.table("synth20k"))
    eng.pods_reset(POD_N)
    for part in (np.arange(0, POD_N, 2, dtype=np.uint32), np.arange(1, POD_N, 2, dtype=np.uint32)):
        eng.pods_seed_slots(part, {k: np.ascontiguousarray(v[part]) for k, v in pods.items()})
    return eng


@pytest.mark.parametrize("n", NS)
def test_slot_lists_are_cut_by_list_position(n):
    """the shards cut the LIST, whatever slots it names: lists shorter than the shard count, off the 16-byte grid,
    shuffled and with repeats; a slot outside the table in the first, a middle and the last shard's part is refused and
    the next call is right; rpk_pods_reset and a re-seed reach every replica"""
    _, eb, et = pod_rows()
    rng = np.random.default_rng(n)
    eng = pod_engine(shared_engine(n))
    try:
        for k in (n - 1, n, n + 1, 4097, 50_003, 150_001):
            for sl in (rng.permutation(POD_N)[:min(k, POD_N)].astype(np.uint32), rng.integers(0, POD_N, k).astype(np.uint32),
                       np.full(k, POD_N - 1, np.uint32)):
                for top5 in (False, True):
                    label = f"{n} shards, list of {len(sl)}, top5={top5}"
                    best, t5 = run_slots(eng, sl, top5)
                    sc.check(label, best, t5, eb[sl], et[sl])
                    check_every_shard(label, eng, eb[sl])
        good = rng.integers(0, POD_N, 50_003).astype(np.uint32)
        c = cuts(len(good), n)
        for s in sorted({0, n // 2, n - 1}):
            for where in sorted({c[s], (c[s] + c[s + 1]) // 2, c[s + 1] - 1}):
                bad = good.copy()
                bad[where] = POD_N + s
                s0 = eng.stats()
                with pytest.raises(rpk.RpkError) as ei:
                    eng.select_slots(bad, want_top5=True)
                assert ei.value.code == EINVAL and "outside the pod table" in str(ei.value), f"bad slot in shard {s}'s part"
                assert eng.stats() == s0
                best, t5 = run_slots(eng, good, True)
                sc.check(f"{n} shards, after a bad slot at {where} (shard {s}'s part)", best, t5, eb[good], et[good])
        # a re-seed that names one slot per shard of the list, then the reset: every replica follows
        sl = np.array(sorted(set(cuts(POD_N - 1, n))), np.uint32)
        eng.pods_seed_slots(sl, {"req_mem_gb": np.full(len(sl), 1 << 30, np.int32)})
        lst = np.concatenate([sl] * (2 * n))  # every shard's part of the list names re-seeded slots
        best, t5 = run_slots(eng, lst, True)
        assert (best == -1).all() and (t5 == -1).all(), "a replica did not take the re-seed"
        eng.pods_reset(1000)
        db, dt = sc.expected(sc.table("synth20k"), DEFAULT_POD)
        best, t5 = run_slots(eng, np.arange(1000, dtype=np.uint32)[::-1].copy(), True)
        sc.check("after pods_reset", best, t5, np.full(1000, db[0], np.int32), np.tile(dt[0], (1000, 1)))
        with pytest.raises(rpk.RpkError):
            eng.select_slots(np.array([5, 1000] * n, np.uint32))
    finally:
        eng.close()


@pytest.mark.parametrize("n", NS)
def test_pending_set(n):
    """every shard compacts its replica of the flags and takes its part of the list: pending sets that lie inside one
    shard's share of the TABLE (so the list's cuts fall elsewhere), then spread; cap refusals"""
    _, eb, et = pod_rows()
    rng = np.random.default_rng(100 + n)
    c = cuts(POD_N, n)
    sets = [("none", np.zeros(0, np.int64)), ("one slot", np.array([POD_N - 1])), (f"{n - 1} slots", rng.choice(POD_N, n - 1, replace=False)),
            (f"{n + 1} slots", rng.choice(POD_N, n + 1, replace=False))]
    sets += [(f"inside shard {s}'s rows", c[s] + rng.choice(c[s + 1] - c[s], 5000 + s, replace=False)) for s in sorted({0, n // 2, n - 1})]
    sets += [("at the cuts", around(c, POD_N)), ("spread", rng.choice(POD_N, 50_003, replace=False)), ("all", np.arange(POD_N))]
    eng = pod_engine(shared_engine(n))
    try:
        for what, sl in sets:
            pend = mark_only(eng, POD_N, np.sort(sl).astype(np.int64))
            k = len(pend)
            label = f"{n} shards, pending: {what}"
            hb, ht = run_slots(eng, pend, True) if k else (np.zeros(0, np.int32), np.zeros((0, 5), np.int32))
            for top5 in (True, False):
                for want_slots in (True, False):
                    slots, best, t5 = run_pending(eng, k + 3, top5, want_slots)
                    assert len(best) == k and (slots is None or np.array_equal(slots, pend)), f"{label}: the list"
                    sc.check(f"{label} top5={top5}: vs oracle", best, t5, eb[pend], et[pend])
                    sc.check(f"{label} top5={top5}: vs select_slots", best, t5, hb, ht)
            if k:
                check_every_shard(label, eng, eb[pend])
                run_pending(eng, k, True)  # exactly enough
                s0 = eng.stats()
                with pytest.raises(rpk.RpkError) as ei:
                    run_pending(eng, k - 1, True)
                assert ei.value.code == EINVAL and ei.value.n_pending == k and eng.stats() == s0, f"{label}: cap refusal"
    finally:
        eng.close()


# ---- pending results ------------------------------------------------------------------------------------------------

def changed_sizes(n):
    return [15, 16, 17, 16 * n - 1, 16 * n, 16 * n + 1, POD_N]


class Pair:
    """an n-shard and a one-shard ctx driven side by side through rpk_select_pending_changed: both must report the same
    rows, and the mirror of the n-shard one must equal rpk_select_slots and the oracle"""

    def __init__(self, n, N):
        self.N, self.n = N, n
        self.offers = {k: None if v is None else v.copy() for k, v in sc.table("synth20k").items()}
        self.pool = pod_rows()[0]
        self.engs = [shared_engine(n), rpk.Engine(1)]
        for e in self.engs:
            e.upload_offers(self.offers)
        self.reset(N)

    def close(self):
        for e in self.engs:
            e.close()

    def reset(self, N):
        self.N, self.tab, self.mirror, self.pend = N, PodTable(N), Mirror(N), np.zeros(0, np.uint32)
        for e in self.engs:
            e.pods_reset(N)

    def seed(self, slots, at=0):
        slots = np.asarray(slots, np.uint32)
        pods = {k: np.ascontiguousarray(v[at:at + len(slots)]) for k, v in self.pool.items()}
        for e in self.engs:
            e.pods_seed_slots(slots, pods)
        self.tab.seed(slots, pods)

    def mark(self, slots):
        for e in self.engs:
            self.pend = mark_only(e, self.N, np.asarray(slots, np.int64))

    def upload(self):
        for e in self.engs:
            e.upload_offers(self.offers)

    def call(self, label, cap=None, reselected=None):
        cap = self.N if cap is None else cap
        got, one = call(self.engs[0], cap), call(self.engs[1], cap)
        assert got[:2] == one[:2], f"{label}: (n_pending, n_reselected) {got[:2]}, one shard {one[:2]}"
        for what, a, b in zip(("slots", "best", "top5"), got[2:], one[2:]):
            assert np.array_equal(a, b), f"{label}: {what} differ from the one-shard ctx's"
        assert got[0] == len(self.pend), f"{label}: n_pending {got[0]}, {len(self.pend)} slots are pending"
        if reselected is not None:
            assert got[1] == reselected, f"{label}: reselected {got[1]}, expected {reselected}"
        assert np.isin(got[2], self.pend).all(), f"{label}: a slot that is not pending was reported"
        self.mirror.apply(*got[2:])
        if len(self.pend):
            wb, wt = sc.expected(self.offers, self.tab.rows(self.pend))
            check_mirror(label, self.engs[0], self.mirror, self.pend, wb, wt)
        return got


@pytest.mark.parametrize("n", NS)
def test_pending_results_are_stored_by_units_of_16_slots(n):
    """tables with fewer 16-slot units than shards, a ragged last unit, unit cuts that differ from the row cuts; pending
    slots in one shard's units only and on both sides of every unit cut; first and steady calls, seeds on slots a shard
    owns and on slots it does not, an offer upload, a refusal one row short of the capacity, and a reset"""
    rng = np.random.default_rng(300 + n)
    p = Pair(n, 16)
    try:
        for N in changed_sizes(n):
            what = f"{n} shards, N={N}"
            p.reset(N)
            p.seed(np.arange(N))
            u = unit_cuts(N, n)
            owners = [s for s in range(n) if u[s + 1] > u[s]]
            for s in sorted({owners[0], owners[len(owners) // 2], owners[-1]}):  # one shard's units only
                lo, hi = u[s], u[s + 1]
                sl = np.arange(lo, hi) if hi - lo <= 64 else np.sort(lo + rng.choice(hi - lo, (hi - lo) // 3, replace=False))
                fresh = np.setdiff1d(sl, p.pend)
                p.mark(np.union1d(sl, p.pend))
                p.call(f"{what}: pending in shard {s}'s units", reselected=len(fresh))
                p.call(f"{what}: steady after shard {s}", cap=0, reselected=0)
            p.reset(N)
            p.seed(np.arange(N))
            edge = around(u, N)
            p.mark(edge)
            got = p.call(f"{what}: both sides of every unit cut", reselected=len(edge))
            assert np.array_equal(got[2], edge), f"{what}: the first call reports every pending slot"
            p.call(f"{what}: steady", cap=0, reselected=0)
            # seeds: new columns on pending slots (every shard's and one shard's) and on slots that are not pending
            spread = np.sort(rng.choice(N, max(N // 7, 1), replace=False))
            p.mark(np.union1d(edge, spread))
            p.call(f"{what}: more pending")
            hit = np.union1d(np.union1d(edge[::2], spread[::3]), rng.choice(N, max(N // 9, 1), replace=False))
            before = p.tab.rows(hit)
            p.seed(hit, at=7)
            after = p.tab.rows(hit)
            moved = np.any([(before[k].view(np.uint8).reshape(len(hit), -1) != after[k].view(np.uint8).reshape(len(hit), -1)).any(axis=1) for k in before], axis=0)
            p.call(f"{what}: after seeds", reselected=int((moved & np.isin(hit, p.pend)).sum()))
            p.call(f"{what}: steady after seeds", cap=0, reselected=0)
            # every result is stale after an upload; one row short of the capacity is refused and nothing is lost
            p.offers["secure_price"][rng.integers(0, len(p.offers["secure_price"]), 200)] *= 1.3
            p.upload()
            k = len(p.pend)
            if k > 1:
                for e in p.engs:
                    out = np.full(k - 1, SLOT_SENTINEL, np.uint32), np.full(k - 1, sc.SENTINEL, np.int32), np.full((k - 1, 5), sc.SENTINEL, np.int32)
                    s0, c0 = e.stats(), e.launch_count()
                    with pytest.raises(rpk.RpkError) as ei:
                        e.select_pending_changed(k - 1, out_slots=out[0], out_best=out[1], out_top5=out[2])
                    assert ei.value.code == EINVAL and (ei.value.n_pending, ei.value.n_reselected) == (k, k), f"{what}: refusal counts"
                    assert (out[0] == SLOT_SENTINEL).all() and (out[1] == sc.SENTINEL).all() and (out[2] == sc.SENTINEL).all()
                    assert e.stats() == s0 and e.launch_count() == c0
            p.call(f"{what}: after the upload", cap=k, reselected=k)
            p.call(f"{what}: steady after the upload", cap=0, reselected=0)
    finally:
        p.close()


# ---- sequences ----------------------------------------------------------------------------------------------------

SEQ_N, SEQ_STATUS = 40_003, 9_001
SEQ_OPS = ["select", "select", "slots", "slots", "seed", "mark", "pending", "changed", "changed", "status_seed", "sweep",
           "sweep_slots", "tick", "upload"]


def same(label, a, b):
    assert len(a) == len(b), label
    for i, (x, y) in enumerate(zip(a, b)):
        assert (x is None and y is None) or np.array_equal(x, y), f"{label}: output {i} of the 3-shard ctx differs from the one-shard ctx's"


@pytest.mark.parametrize("seed", [1, 2, 3])
def test_call_sequences_three_shards_beside_one(seed):
    """a seeded sequence of uploads, selects, slot selects, seeds, marks, pending and pending-changed calls, status
    seeds, sweeps, slot sweeps and ticks on a 3-shard and a one-shard ctx: every output of every step is the same, and
    the selects equal the oracle"""
    synth = rpk.synth
    rng = np.random.default_rng(seed)
    pool = pod_rows()[0]
    engs = [shared_engine(3), rpk.Engine(1)]
    log = []
    try:
        tab, flags, sweep = PodTable(SEQ_N), np.zeros(SEQ_N, np.uint8), 0
        for e in engs:
            e.pods_reset(SEQ_N)
            e.status_reset(SEQ_STATUS)
        offers = None
        for stp in range(60):
            op = "upload" if offers is None else str(rng.choice(SEQ_OPS))
            k = int(rng.choice([1, 2, 3, 4, 47, 4097, 20_001]))
            top5 = bool(rng.integers(0, 2))
            log.append(f"{op} k={k} top5={top5}")
            label = f"seed {seed} step {stp} ({'; '.join(log[-8:])})"
            both = lambda f: [f(e) for e in engs]  # noqa: E731
            if op == "upload":
                name, force = str(rng.choice(["synth20k", "synth300", "packed_only", "stride64"])), FORCE[int(rng.integers(0, len(FORCE)))]
                offers = sc.table(name)
                with sc.forced(force):
                    both(lambda e: e.upload_offers(offers))
            elif op in ("select", "tick"):
                at = int(rng.integers(0, POD_N - k))
                rows = {c: np.ascontiguousarray(v[at:at + k]) for c, v in pool.items()}
                if rng.random() < 0.3:
                    rows = sc.without_optional(rows)
                if op == "select":
                    got = both(lambda e: sc.run_host(e, rows, top5))
                else:
                    sweep += 1
                    recs = synth.make_status_records(SEQ_STATUS, sweep, 0.2, seed=seed, stride=32)
                    got = both(lambda e: e.tick(rows, recs, want_top5=top5))
                same(label, *got)
                wb, wt = sc.expected(offers, rows)
                sc.check(label, got[0][0], got[0][1], wb, wt)
            elif op == "slots":
                sl = rng.integers(0, SEQ_N, k).astype(np.uint32)
                got = both(lambda e: run_slots(e, sl, top5))
                same(label, *got)
                wb, wt = sc.expected(offers, tab.rows(sl))
                sc.check(label, got[0][0], got[0][1], wb, wt)
            elif op == "seed":
                sl = np.sort(rng.choice(SEQ_N, k, replace=False)).astype(np.uint32)
                at = int(rng.integers(0, POD_N - k))
                rows = {c: np.ascontiguousarray(v[at:at + k]) for c, v in pool.items()}
                both(lambda e: e.pods_seed_slots(sl, rows))
                tab.seed(sl, rows)
            elif op == "mark":
                sl = np.sort(rng.choice(SEQ_N, k, replace=False)).astype(np.uint32)
                v = rng.integers(0, 2, k).astype(np.uint8)
                both(lambda e: e.pods_mark_pending(sl, v))
                flags[sl] = v
            elif op == "pending":
                pend = np.flatnonzero(flags).astype(np.uint32)
                got = both(lambda e: run_pending(e, len(pend) + 1, top5))
                same(label, *got)
                assert np.array_equal(got[0][0], pend), f"{label}: the pending list"
                if len(pend):
                    wb, wt = sc.expected(offers, tab.rows(pend))
                    sc.check(label, got[0][1], got[0][2], wb, wt)
            elif op == "changed":
                got = both(lambda e: call(e, SEQ_N))
                assert got[0][:2] == got[1][:2], f"{label}: counts {got[0][:2]} and {got[1][:2]}"
                same(label, got[0][2:], got[1][2:])
            elif op == "status_seed":
                sl = np.sort(rng.choice(SEQ_STATUS, min(k, 300), replace=False)).astype(np.uint32)
                recs = np.ascontiguousarray(synth.make_status_records(SEQ_STATUS, sweep + 100, 0.5, seed=seed, stride=32)[sl])
                both(lambda e: e.status_seed_slots(sl, recs))
            elif op == "sweep":
                sweep += 1
                recs = synth.make_status_records(SEQ_STATUS, sweep, 0.2, seed=seed, stride=32)
                same(label, *both(lambda e: e.status_diff(recs, want_hashes=True, want_codes=True)))
            else:
                sweep += 1
                sl = np.sort(rng.choice(SEQ_STATUS, min(k, SEQ_STATUS), replace=False)).astype(np.uint32)
                recs = np.ascontiguousarray(synth.make_status_records(SEQ_STATUS, sweep, 0.5, seed=seed, stride=32)[sl])
                same(label, *both(lambda e: e.status_diff_slots(sl, recs, want_codes=True)))
    finally:
        for e in engs:
            e.close()


# ---- ordering and lifetime -----------------------------------------------------------------------------------------

@pytest.mark.parametrize("name", SHARD_1_CASES)
def test_host_call_waits_for_device_call_on_shard_1(name):
    """a 2-shard ctx: the device call is queued behind a sleep on a plain stream of shard 1 (it waits for no other
    shard's kernel), and the host call spans both shards"""
    rig = Rig(2, 1, make_engine=shared_engine)
    try:
        run_case(rig, name)
    finally:
        rig.close()


def n_threads():
    return len(os.listdir("/proc/self/task"))


@pytest.mark.parametrize("n", NS)
def test_close_and_recreate(n):
    """create, use and close an n-shard ctx five times in one process: closing joins the shard workers and frees the
    shards' buffers, and a one-shard ctx works afterwards"""
    import torch

    pods, wb, wt = sc.batch("synth20k", P_MAX)
    rows = sc.head(pods, 50_003)
    recs = rpk.synth.make_status_records(30_001, 0, stride=16)
    threads, free = [], []
    torch.cuda.synchronize()
    for cycle in range(5):
        eng = shared_engine(n)
        eng.upload_offers(sc.table("synth20k"))
        sc.check(f"cycle {cycle}", *sc.run_host(eng, rows, True), wb[:50_003], wt[:50_003])
        assert len(eng.status_diff(recs)[0]) == 30_001
        eng.close()
        torch.cuda.synchronize()
        threads.append(n_threads())
        free.append(torch.cuda.mem_get_info()[0])
    assert threads[2:] == threads[1:-1], f"threads alive after each close: {threads}"
    assert free[1] - free[-1] < (64 << 20), f"free device memory after each close: {[f >> 20 for f in free]} MiB"
    with shared_engine(n) as eng:
        held = n_threads()
    assert held - n_threads() == n - 1, f"an {n}-shard ctx holds {n - 1} workers; closing it ended {held - n_threads()} threads"
    with rpk.Engine(1) as eng:
        eng.upload_offers(sc.table("synth20k"))
        sc.check("one shard afterwards", *sc.run_host(eng, rows, True), wb[:50_003], wt[:50_003])
