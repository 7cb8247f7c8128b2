"""GPU tests of the selection over a list of slots of the device pod table (rpk_pods_reset, rpk_pods_seed_slots,
rpk_select_slots).

A numpy model of the table (the five columns of every slot, the no-annotation defaults where nothing was seeded) gives
each list its pod columns: rpk_select_slots over the list must equal rpk_select over the model's rows of the list, and the
oracle on every row.  The tracked table has 1M slots; one region of it is seeded with a table's test batch, another with
the same batch without the optional columns (their defaults), and the rest holds the defaults.  Every output buffer
starts as SENTINEL, so a row the kernels never write shows up."""
import functools
import zlib

import numpy as np
import pytest

import oracle
import persist_plan_model as model
import rpk
import select_plan_cases as sc
from test_select_sequences_gpu import FORCE, MENU

pytestmark = pytest.mark.gpu

TRACKED = 1 << 20
R = 196_609  # rows of each seeded region: the test batch of test_select_sequences_gpu (shared oracle cache)
SIZES = [1, 4096, 4097, 16_384, 16_385, 196_609]
SHAPES = ["ascending", "shuffled", "repeats"]
COLS = ("req_mem_gb", "req_vcpu", "req_ram_gb", "max_price", "cloud")
DTYPES = {"req_mem_gb": np.int32, "req_vcpu": np.int32, "req_ram_gb": np.int32, "max_price": np.float64, "cloud": np.uint8}
DEFAULTS = {"req_mem_gb": 16, "req_vcpu": 0, "req_ram_gb": 0, "max_price": 0.5, "cloud": 0}  # a pod with no annotations
DEFAULT_POD = {"req_mem_gb": np.array([16], np.int32), "req_vcpu": None, "req_ram_gb": None, "max_price": None, "cloud": None}


class PodTable:
    """numpy model of the device pod table"""

    def __init__(self, N):
        self.N = N
        self.cols = {k: np.full(N, DEFAULTS[k], DTYPES[k]) for k in COLS}

    def seed(self, slots, pods):
        for k in COLS:
            v = pods.get(k)
            self.cols[k][slots] = DEFAULTS[k] if v is None else v

    def rows(self, slots):
        return {k: np.ascontiguousarray(c[slots]) for k, c in self.cols.items()}


def slot_list(rng, n, shape, N=TRACKED):
    if shape == "ascending":
        return np.arange(N, dtype=np.uint32) if n == N else np.sort(rng.choice(N, n, replace=False)).astype(np.uint32)
    if shape == "shuffled":
        return rng.permutation(N)[:n].astype(np.uint32)
    return rng.integers(0, min(N, max(2 * n // 3, 1)), n).astype(np.uint32)  # repeats


@functools.lru_cache(maxsize=None)
def tracked(name):
    """(model, oracle best per slot, oracle top5 per slot, [(slots, pods) of each seed]) for table `name`"""
    rng = np.random.default_rng(zlib.crc32(name.encode()))
    perm = rng.permutation(TRACKED)
    a, b = np.sort(perm[:R]).astype(np.uint32), np.sort(perm[R:2 * R]).astype(np.uint32)
    pods, wb, wt = sc.batch(name, R)
    pods_n, nb, nt = sc.batch_without_optional(name, R)
    db, dt = sc.expected(sc.table(name), DEFAULT_POD)
    eb = np.full(TRACKED, db[0], np.int32)
    et = np.tile(dt[0], (TRACKED, 1)).astype(np.int32)
    eb[a], et[a], eb[b], et[b] = wb, wt, nb, nt
    m = PodTable(TRACKED)
    m.seed(a, pods)
    m.seed(b, pods_n)
    return m, eb, et, [(a, pods), (b, pods_n)]


def seeded_engine(name, force=None, n_gpus=1):
    _, _, _, seeds = tracked(name)
    eng = rpk.Engine(n_gpus)
    with sc.forced(force):
        eng.upload_offers(sc.table(name))
    eng.pods_reset(TRACKED)
    for slots, pods in seeds:
        eng.pods_seed_slots(slots, pods)
    return eng


def run_slots(eng, sl, top5):
    n = len(sl)
    best = np.full(n, sc.SENTINEL, np.int32)
    t5 = np.full((n, 5), sc.SENTINEL, np.int32) if top5 else None
    eng.select_slots(sl, want_top5=top5, out_best=best, out_top5=t5)
    return best, t5


@pytest.mark.parametrize("force", FORCE)
@pytest.mark.parametrize("name", MENU)
def test_select_slots_equals_select_and_oracle(name, force):
    """every list size (both sides of the latency path, the fused kernel's size and the sub-batch size) and shape, with
    and without top-5, over rows seeded with and without optional columns and unseeded rows"""
    m, eb, et, _ = tracked(name)
    rng = np.random.default_rng(zlib.crc32(f"{name}/{force}".encode()))
    sizes = SIZES + ([TRACKED] if name == "synth100k" else [])
    eng = seeded_engine(name, force)
    try:
        k = 0
        for n in sizes:
            for shape in SHAPES:
                top5 = k % 2 == 0
                k += 1
                sl = slot_list(rng, n, shape)
                label = f"{name} force={force} n={n} {shape} top5={top5}"
                best, t5 = run_slots(eng, sl, top5)
                sc.check(label + ": select_slots vs oracle", best, t5, eb[sl], et[sl] if top5 else None)
                rb, rt = sc.run_host(eng, m.rows(sl), top5)
                sc.check(label + ": select_slots vs select of the model's rows", best, t5, rb, rt)
    finally:
        eng.close()


def test_table_state_defaults_reseed_and_reset():
    offers = sc.table("synth300")
    db, dt = sc.expected(offers, DEFAULT_POD)
    with rpk.Engine(1) as eng:
        eng.upload_offers(offers)
        N = 50_000
        eng.pods_reset(N)
        m = PodTable(N)
        sl = np.arange(N, dtype=np.uint32)
        best, t5 = run_slots(eng, sl, True)
        sc.check("unseeded rows", best, t5, np.full(N, db[0], np.int32), np.tile(dt[0], (N, 1)))
        pods, _, _ = sc.batch("synth300", R)
        rng = np.random.default_rng(5)
        first = np.sort(rng.choice(N, 20_000, replace=False)).astype(np.uint32)
        eng.pods_seed_slots(first, sc.head(pods, 20_000))
        m.seed(first, sc.head(pods, 20_000))
        again = np.sort(rng.choice(first, 3000, replace=False)).astype(np.uint32)  # a re-seed of part of the rows
        src = {k: np.ascontiguousarray(v[50_000:53_000]) for k, v in pods.items()}
        eng.pods_seed_slots(again, sc.without_optional(src))
        m.seed(again, sc.without_optional(src))
        best, t5 = run_slots(eng, sl, True)
        wb, wt = sc.expected(offers, m.rows(sl))
        sc.check("after a re-seed", best, t5, wb, wt)
        # reset: every row back to the defaults, at the new size
        eng.pods_reset(N // 2)
        best, t5 = run_slots(eng, sl[: N // 2], True)
        sc.check("after pods_reset", best, t5, np.full(N // 2, db[0], np.int32), np.tile(dt[0], (N // 2, 1)))
        with pytest.raises(rpk.RpkError) as ei:
            eng.select_slots(np.array([N // 2], np.uint32))
        assert ei.value.code == rpk._ffi.RPK_EINVAL
        eng.pods_reset(2 * N)  # grows
        best, _ = run_slots(eng, np.array([0, 2 * N - 1], np.uint32), False)
        assert best.tolist() == [db[0], db[0]]


def test_launches_stats_and_device_vector():
    """one gather per host sub-batch on top of what rpk_select launches; one select in the stats; the assignment vector
    on the device as after rpk_select"""
    import torch

    peer = __import__("k8s-runpod-kubelet_b200.peer", fromlist=["as_int32_tensor"])
    m, eb, _, _ = tracked("synth20k")
    rng = np.random.default_rng(11)
    G = len(sc.table("synth20k")["mem_gb"])
    eng = seeded_engine("synth20k")
    try:
        for n in (1, 4096, 4097, 196_609, 600_000):
            sl = rng.integers(0, TRACKED, n).astype(np.uint32)
            s0, c0 = eng.stats(), eng.launch_count()
            best, _ = eng.select_slots(sl, want_top5=True)
            s1, c1 = eng.stats(), eng.launch_count()
            if n > 4096:
                dev = peer.as_int32_tensor(eng.best_device_ptr(0), n, torch.device("cuda", 0)).cpu().numpy()
                assert np.array_equal(dev, best), f"n={n}: device assignment vector differs"
            eng.select(m.rows(sl), want_top5=True)
            c2 = eng.launch_count()
            assert (c1 - c0) - (c2 - c1) == len(model.host_sub_batches(n)), n
            assert s1["select_calls"] == s0["select_calls"] + 1 and s1["offer_scores"] == s0["offer_scores"] + n * G
            assert np.array_equal(best, eb[sl])
    finally:
        eng.close()


def test_errors():
    m, eb, et, _ = tracked("synth20k")
    lib = rpk._ffi.load()
    rng = np.random.default_rng(3)
    eng = seeded_engine("synth20k")
    try:
        good = rng.integers(0, TRACKED, 300_000).astype(np.uint32)
        for where in (0, 100, 250_000, 299_999):  # the first sub-batch, or only a later one
            bad = good.copy()
            bad[where] = TRACKED + where % 3
            with pytest.raises(rpk.RpkError) as ei:
                eng.select_slots(bad, want_top5=True)
            assert ei.value.code == rpk._ffi.RPK_EINVAL and "outside the pod table" in str(ei.value)
            best, t5 = run_slots(eng, good, True)  # the next valid call is right
            sc.check(f"after a bad entry at {where}", best, t5, eb[good], et[good])
        for bad in (np.array([5, TRACKED], np.uint32), np.array([0xFFFFFFFF], np.uint32)):  # latency path
            with pytest.raises(rpk.RpkError) as ei:
                eng.select_slots(bad)
            assert ei.value.code == rpk._ffi.RPK_EINVAL
        # a bad seed changes nothing
        probe = np.arange(0, 64, dtype=np.uint32)
        before = run_slots(eng, probe, True)
        cols = {"req_mem_gb": np.full(3, 4000, np.int32)}
        for bad in ([3, 2, 9], [3, 3, 9], [3, 9, TRACKED]):
            with pytest.raises(rpk.RpkError) as ei:
                eng.pods_seed_slots(np.array(bad, np.uint32), cols)
            assert ei.value.code == rpk._ffi.RPK_EINVAL
        after = run_slots(eng, probe, True)
        assert np.array_equal(before[0], after[0]) and np.array_equal(before[1], after[1])
        # n = 0 is a no-op; NULL pointers
        assert eng.select_slots(np.zeros(0, np.uint32))[0].size == 0
        eng.pods_seed_slots(np.zeros(0, np.uint32), {"req_mem_gb": np.zeros(0, np.int32)})
        out = np.empty(4, np.int32)
        sl = np.arange(4, dtype=np.uint32)
        E = rpk._ffi.RPK_EINVAL
        assert lib.rpk_select_slots(eng._ctx, 4, None, out.ctypes.data, None) == E
        assert lib.rpk_select_slots(eng._ctx, 4, sl.ctypes.data, None, None) == E
        assert lib.rpk_pods_seed_slots(eng._ctx, 4, None, out.ctypes.data, None, None, None, None) == E
        assert lib.rpk_pods_seed_slots(eng._ctx, 4, sl.ctypes.data, None, None, None, None, None) == E
        assert lib.rpk_select_slots(None, 4, sl.ctypes.data, out.ctypes.data, None) == E
        assert lib.rpk_pods_reset(None, 4) == E
        after = run_slots(eng, probe, True)
        assert np.array_equal(before[0], after[0])
    finally:
        eng.close()
    # RPK_ESTATE: no pod table, no offer table
    with rpk.Engine(1) as e:
        e.upload_offers(sc.table("synth300"))
        for call in (lambda: e.select_slots(np.array([0], np.uint32)),
                     lambda: e.pods_seed_slots(np.array([0], np.uint32), {"req_mem_gb": np.array([8], np.int32)})):
            with pytest.raises(rpk.RpkError) as ei:
                call()
            assert ei.value.code == rpk._ffi.RPK_ESTATE
    with rpk.Engine(1) as e:
        e.pods_reset(16)
        e.pods_seed_slots(np.array([1], np.uint32), {"req_mem_gb": np.array([8], np.int32)})
        with pytest.raises(rpk.RpkError) as ei:
            e.select_slots(np.array([1], np.uint32))
        assert ei.value.code == rpk._ffi.RPK_ESTATE


# ---- sequences: seed, select_slots, select, device selects and tick on one ctx --------------------------------------
SEQ_N = 300_000
SEQ_OPS = ["seed", "seed", "slots", "slots", "slots", "select", "device", "tick"]
SEQ_SIZES = [1, 4096, 4097, 30_000, 140_000]


class Program:
    def __init__(self, seed):
        self.seed = seed
        self.rng = np.random.default_rng(seed)
        self.eng = rpk.Engine(1)
        self.model = PodTable(SEQ_N)
        self.status = oracle.StatusTable(1000, 16)
        self.eng.status_reset(1000)
        self.eng.pods_reset(SEQ_N)
        self.sweep = 0
        self.log = []

    def fail(self, err):
        raise AssertionError(f"{err}\nprogram seed {self.seed}; operations:\n  " + "\n  ".join(self.log))

    def run(self, op, offers):
        rng = self.rng
        n = int(rng.choice(SEQ_SIZES))
        top5 = bool(rng.integers(0, 2))
        shape = str(rng.choice(SHAPES))
        self.log.append(f"{op} n={n} top5={top5} {shape}")
        try:
            if op == "seed":
                sl = np.sort(rng.choice(SEQ_N, n, replace=False)).astype(np.uint32)
                pods = sc.pods_for("synth20k", n, seed=int(rng.integers(0, 1 << 30)))
                if rng.random() < 0.3:
                    pods = sc.without_optional(pods)
                self.eng.pods_seed_slots(sl, pods)
                self.model.seed(sl, pods)
                return
            sl = slot_list(rng, n, shape, SEQ_N)
            rows = self.model.rows(sl)
            wb, wt = sc.expected(offers, rows)
            if op == "slots":
                got = run_slots(self.eng, sl, top5)
            elif op == "select":
                got = sc.run_host(self.eng, rows, top5)
            elif op == "device":
                got = sc.run_device(self.eng, rows, top5)
            else:
                self.sweep += 1
                recs = rpk.synth.make_status_records(1000, self.sweep, 0.2, seed=self.seed, stride=16)
                best, t5, idx, _ = self.eng.tick(rows, recs, want_top5=top5)
                if not np.array_equal(idx, self.status.diff(recs)):
                    raise AssertionError("tick: changed list differs from the model")
                got = (best, t5)
            sc.check(op, got[0], got[1], wb, wt if top5 else None)
        except AssertionError as e:
            self.fail(str(e))


@pytest.mark.parametrize("seed", [1, 2, 3])
def test_slot_select_call_sequences(seed):
    p = Program(seed)
    try:
        for name in ("synth20k", "synth300", "synth20k"):
            p.log.append(f"upload {name}")
            offers = sc.table(name)
            p.eng.upload_offers(offers)
            for _ in range(6):
                p.run(str(p.rng.choice(SEQ_OPS)), offers)
            p.log.append("slots (whole table)")
            sl = np.arange(SEQ_N, dtype=np.uint32)
            best, _ = run_slots(p.eng, sl, False)
            try:
                sc.check("whole table", best, None, sc.expected(offers, p.model.rows(sl))[0], None)
            except AssertionError as e:
                p.fail(str(e))
    finally:
        p.eng.close()


def test_multi_gpu_replicas():
    import torch

    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    m, eb, et, _ = tracked("synth100k")
    rng = np.random.default_rng(21)
    e1, e2 = seeded_engine("synth100k"), seeded_engine("synth100k", n_gpus=2)
    try:
        for n in (1, 4096, 4097, 196_609):
            sl = slot_list(rng, n, "shuffled")
            b1, t1 = run_slots(e1, sl, True)
            b2, t2 = run_slots(e2, sl, True)
            assert np.array_equal(b1, b2) and np.array_equal(t1, t2), n
            sc.check(f"Engine(2) n={n}", b2, t2, eb[sl], et[sl])
        # every replica holds every seed: each GPU takes one half of a list whose halves are the same slots
        rows = slot_list(rng, 100_000, "shuffled")
        fresh = {k: np.ascontiguousarray(v[::-1][:100_000]) for k, v in sc.batch("synth100k", R)[0].items()}
        srt = np.argsort(rows)
        e2.pods_seed_slots(rows[srt], {k: v[srt] for k, v in fresh.items()})
        m2 = PodTable(TRACKED)
        m2.cols = {k: v.copy() for k, v in m.cols.items()}
        m2.seed(rows[srt], {k: v[srt] for k, v in fresh.items()})
        sl = np.concatenate([rows, rows])
        b2, t2 = run_slots(e2, sl, True)
        wb, wt = sc.expected(sc.table("synth100k"), m2.rows(rows))
        sc.check("replica 0", b2[:100_000], t2[:100_000], wb, wt)
        sc.check("replica 1", b2[100_000:], t2[100_000:], wb, wt)
    finally:
        e1.close()
        e2.close()
