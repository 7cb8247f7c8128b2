"""GPU tests of rpk_explain and rpk_explain_slots (include/rpk.h): every output word of every row, bit for bit, against
the C reference of explain_model.py, with the outputs filled with a sentinel before each call.

Covered: the table shapes of select_plan_cases (and offer counts around the kernel's 1024-offer stage), row counts from 1
to 1M; the slot form against the column form on the gathered rows; every refusal, with no state changed after it;
explains after an offer-table refresh and a pod-table grow; a pending-results history that interleaves explains and
matches the same history without them; a captured _device select replayed after a larger explain; and 2-, 3-, 4- and
8-shard ctxs on one GPU, bit-identical to one shard."""
import os

import numpy as np
import pytest

import explain_model as em
import rpk
import select_plan_cases as sc

pytestmark = pytest.mark.gpu

SENT = 0xDEADBEEF
THREADS = os.cpu_count() or 1
CHUNK = 1024  # offers k_explain stages per pass (explain.cu kExplainChunk)


def sentinel(n):
    return np.full(n * em.WORDS, SENT, np.uint32)


def explain(eng, pods):
    out = sentinel(sc.nrows(pods))
    return eng.explain(pods, out=out)


def explain_slots(eng, slots):
    out = sentinel(len(slots))
    return eng.explain_slots(slots, out=out)


def gathered(pods, rows):
    return {k: None if v is None else np.ascontiguousarray(v[rows]) for k, v in pods.items()}


@pytest.mark.parametrize("name,P", [("synth20k", 1), ("synth20k", 20_000), ("many_queues", 2_000), ("packed_only", 50_000),
                                    ("full_int32", 50_000), ("stride64", 20_000), ("empty", 1_000), ("synth100k", 20_000)])
def test_table_shapes(name, P):
    offers, pods = sc.table(name), sc.pods_for(name, P)
    with rpk.Engine(1) as eng:
        eng.upload_offers(offers)
        em.assert_same(explain(eng, pods), em.explain(offers, pods, THREADS), f"{name} P={P}")
        bare = sc.without_optional(pods)
        em.assert_same(explain(eng, bare), em.explain(offers, bare, THREADS), f"{name} P={P} without optional columns")


@pytest.mark.parametrize("G", [1, 2, CHUNK - 1, CHUNK, CHUNK + 1, 2 * CHUNK - 1, 2 * CHUNK + 1, 5 * CHUNK + 3])
def test_offer_counts_around_the_stage(G):
    for tie_free in (False, True):
        offers = rpk.synth.make_offers(G, tie_free=tie_free, seed=rpk.synth.SEED + G)
        pods = rpk.synth.make_pods(3_001, seed=G)
        pods["max_price"] = np.random.default_rng(G).choice(sc.price_set(offers), 3_001)
        with rpk.Engine(1) as eng:
            eng.upload_offers(offers)
            em.assert_same(explain(eng, pods), em.explain(offers, pods, THREADS), f"G={G} tie_free={tie_free}")


def test_one_million_rows():
    offers = rpk.synth.make_offers(1_000, correlated=True)
    pods = sc.pods_for("synth20k", 1_000_000)
    with rpk.Engine(1) as eng:
        eng.upload_offers(offers)
        em.assert_same(explain(eng, pods), em.explain(offers, pods, THREADS), "G=1k P=1M")


def test_known_answers():
    with rpk.Engine(1) as eng:
        eng.upload_offers(em.kat_offers())
        em.assert_same(explain(eng, em.kat_pods()), em.kat_expected(), "KAT")


def test_slots_against_columns():
    offers = sc.table("synth20k")
    pool = sc.pods_for("synth20k", 30_000, seed=3)
    N = 30_000
    rng = np.random.default_rng(11)
    with rpk.Engine(1) as eng:
        eng.upload_offers(offers)
        eng.pods_reset(N)
        seeded = np.sort(rng.choice(N, 25_000, replace=False)).astype(np.uint32)
        eng.pods_seed_slots(seeded, gathered(pool, seeded))
        table = gathered(pool, np.arange(N))  # the pod table's rows: seeded slots from the pool, the others the defaults
        unseeded = np.setdiff1d(np.arange(N), seeded)
        for k, v in (("req_mem_gb", 16), ("req_vcpu", 0), ("req_ram_gb", 0), ("max_price", 0.5), ("cloud", 0)):
            table[k][unseeded] = v
        for n in (1, 7, 4_097, 60_000):  # repeats and any order
            slots = rng.integers(0, N, n).astype(np.uint32)
            got = explain_slots(eng, slots)
            em.assert_same(got, explain(eng, gathered(table, slots)), f"slots n={n} vs columns")
            em.assert_same(got, em.explain(offers, gathered(table, slots), THREADS), f"slots n={n} vs reference")


def rc_of(fn):
    with pytest.raises(rpk.RpkError) as ei:
        fn()
    return ei.value.code, str(ei.value)


def test_refusals_change_nothing():
    offers = sc.table("synth20k")
    pods = sc.pods_for("synth20k", 5_000)
    with rpk.Engine(1) as eng:
        code, msg = rc_of(lambda: eng.explain(pods))
        assert code == rpk._ffi.RPK_ESTATE and "rpk_explain:" in msg
        code, msg = rc_of(lambda: eng.explain_slots(np.arange(3, dtype=np.uint32)))
        assert code == rpk._ffi.RPK_ESTATE and "rpk_explain_slots" in msg
        eng.upload_offers(offers)
        code, msg = rc_of(lambda: eng.explain_slots(np.arange(3, dtype=np.uint32)))
        assert code == rpk._ffi.RPK_ESTATE and "rpk_explain_slots" in msg and "pod table" in msg
        N = 5_000
        eng.pods_reset(N)
        slots = np.arange(N, dtype=np.uint32)
        eng.pods_seed_slots(slots, pods)
        eng.pods_mark_pending(slots[::3], np.ones(len(slots[::3]), np.uint8))
        first = eng.select_pending_changed(N)
        before_rows = explain_slots(eng, slots)
        stats, launches = eng.stats(), eng.launch_count()
        for bad in ([N], [0, 1, N + 5], [2**32 - 1]):
            out = sentinel(len(bad))
            code, msg = rc_of(lambda: eng.explain_slots(np.array(bad, np.uint32), out=out))
            assert code == rpk._ffi.RPK_EINVAL and "rpk_explain_slots" in msg and "outside the pod table" in msg
            assert (out == SENT).all(), "a refused call writes no output"
        L = eng._lib
        assert L.rpk_explain(eng._ctx, 1, None, None, None, None, None, None) == rpk._ffi.RPK_EINVAL
        assert b"rpk_explain" in L.rpk_last_error(eng._ctx)
        assert L.rpk_explain_slots(eng._ctx, 1, None, None) == rpk._ffi.RPK_EINVAL
        assert L.rpk_explain(eng._ctx, 0, None, None, None, None, None, None) == rpk._ffi.RPK_OK  # P == 0: a no-op
        assert L.rpk_explain_slots(eng._ctx, 0, None, None) == rpk._ffi.RPK_OK
        assert eng.stats() == stats and eng.launch_count() == launches
        em.assert_same(explain_slots(eng, slots), before_rows, "pod rows after the refusals")
        n_p, n_r, s, b, t = eng.select_pending_changed(N)
        assert (n_p, n_r, len(s)) == (first[0], 0, 0), "no stored pending result changed"
        assert eng.stats()["select_calls"] == stats["select_calls"]


def test_after_refresh_and_grow():
    offers = rpk.synth.make_offers(9_000, correlated=True)
    pool = sc.pods_for("synth20k", 12_000, seed=5)
    with rpk.Engine(1) as eng:
        eng.upload_offers(offers)
        eng.pods_reset(8_000)
        eng.pods_seed_slots(np.arange(8_000, dtype=np.uint32), gathered(pool, np.arange(8_000)))
        changed = {k: None if v is None else v.copy() for k, v in offers.items()}
        changed["secure_price"][[3, 50, 4_000]] = [0.01, 0.0, 7.5]
        changed["flags"][[10, 11]] ^= 1
        assert 0 < eng.refresh_offers(changed) <= 5
        slots = np.random.default_rng(2).integers(0, 8_000, 9_000).astype(np.uint32)
        em.assert_same(explain_slots(eng, slots), em.explain(changed, gathered(pool, slots), THREADS), "after refresh")
        eng.pods_grow(12_000)
        eng.pods_seed_slots(np.arange(8_000, 11_000, dtype=np.uint32), gathered(pool, np.arange(8_000, 11_000)))
        table = gathered(pool, np.arange(12_000))
        for k, v in (("req_mem_gb", 16), ("req_vcpu", 0), ("req_ram_gb", 0), ("max_price", 0.5), ("cloud", 0)):
            table[k][11_000:] = v
        slots = np.random.default_rng(3).integers(0, 12_000, 20_000).astype(np.uint32)
        em.assert_same(explain_slots(eng, slots), em.explain(changed, gathered(table, slots), THREADS), "after grow")


def pending_history(eng, offers, pool, with_explain):
    """a tick history: seeds, marks, refreshes and pending-results calls; with_explain adds explains between them"""
    N = 20_000
    rng, ask = np.random.default_rng(17), np.random.default_rng(18)  # the history's draws do not depend on the explains
    log = []
    eng.upload_offers(offers)
    eng.pods_reset(N)
    all_slots = np.arange(N, dtype=np.uint32)
    eng.pods_seed_slots(all_slots, gathered(pool, all_slots))
    table = offers
    for step in range(6):
        marks = np.sort(rng.choice(N, 3_000, replace=False)).astype(np.uint32)
        eng.pods_mark_pending(marks, (rng.random(3_000) < 0.7).astype(np.uint8))
        if with_explain:
            explain_slots(eng, ask.integers(0, N, 50_000).astype(np.uint32))
        res = eng.select_pending_changed(N)
        log.append((res[0], res[1], res[2].copy(), res[3].copy(), res[4].copy()))
        if with_explain:
            explain(eng, gathered(pool, np.arange(40_000) % len(pool["req_mem_gb"])))
        reseed = np.sort(rng.choice(N, 500, replace=False)).astype(np.uint32)
        eng.pods_seed_slots(reseed, gathered(pool, rng.integers(0, N, 500)))
        if step % 2:
            table = {k: None if v is None else v.copy() for k, v in table.items()}
            table["secure_price"][rng.integers(0, len(table["mem_gb"]), 3)] *= 0.9
            eng.refresh_offers(table)
    log.append(eng.stats()["select_calls"])
    return log


def test_pending_results_unchanged_by_explains():
    offers = rpk.synth.make_offers(4_000, correlated=True)
    pool = sc.pods_for("synth20k", 20_000, seed=9)
    with rpk.Engine(1) as a, rpk.Engine(1) as b:
        la, lb = pending_history(a, offers, pool, True), pending_history(b, offers, pool, False)
    assert la[-1] == lb[-1]
    for i, (x, y) in enumerate(zip(la[:-1], lb[:-1])):
        assert x[:2] == y[:2], f"step {i}: (n_pending, n_reselected) {x[:2]} != {y[:2]}"
        for u, v in zip(x[2:], y[2:]):
            assert np.array_equal(u, v), f"step {i}: reported rows differ"


def test_captured_select_replays_after_a_larger_explain():
    import torch

    offers = sc.table("synth20k")
    P = 20_000
    pods, want_best, want_top5 = sc.batch("synth20k", P)
    with rpk.Engine(1) as eng:
        eng.upload_offers(offers)
        eng.pods_reset(1_000)  # before the capture: a reset invalidates captures of the calls that read the pod table
        cols = {k: None if v is None else torch.from_numpy(np.ascontiguousarray(v)).cuda() for k, v in pods.items()}
        d_best = torch.full((P,), sc.SENTINEL, dtype=torch.int32, device="cuda")
        d_top5 = torch.full((P * 5,), sc.SENTINEL, dtype=torch.int32, device="cuda")
        st = torch.cuda.Stream()
        with torch.cuda.stream(st):
            eng.select_device(cols, d_best, d_top5, stream=st.cuda_stream)
        st.synchronize()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=st, capture_error_mode="relaxed"):
            eng.select_device(cols, d_best, d_top5, stream=st.cuda_stream)
        torch.cuda.synchronize()
        before = eng.capture_buffers()
        big = sc.pods_for("synth20k", 200_000, seed=4)
        em.assert_same(explain(eng, big), em.explain(offers, big, THREADS), "explain between capture and replay")
        explain_slots(eng, np.arange(300_000, dtype=np.uint32) % 1_000)
        assert eng.capture_buffers() == before, "an explain moved a buffer the captured select points at"
        d_best.fill_(sc.SENTINEL)
        d_top5.fill_(sc.SENTINEL)
        g.replay()
        torch.cuda.synchronize()
        sc.check("replay after explain", d_best.cpu().numpy(), d_top5.cpu().numpy().reshape(P, 5), want_best, want_top5)


@pytest.mark.parametrize("n", [2, 3, 4, 8])
def test_shards_on_one_gpu_match_one_shard(n, monkeypatch):
    monkeypatch.setenv("RPK_TEST_SHARED_DEVICE", "1")
    offers = sc.table("synth20k")
    pods = sc.pods_for("synth20k", 50_001, seed=n)
    N = 10_007
    slots = np.random.default_rng(n).integers(0, N, 30_001).astype(np.uint32)
    with rpk.Engine(1) as one, rpk.Engine(device_ids=[0] * n) as many:
        for eng in (one, many):
            eng.upload_offers(offers)
            eng.pods_reset(N)
            eng.pods_seed_slots(np.arange(N, dtype=np.uint32), sc.head(pods, N))
        em.assert_same(explain(many, pods), explain(one, pods), f"{n} shards, columns")
        em.assert_same(explain_slots(many, slots), explain_slots(one, slots), f"{n} shards, slots")
        tiny = sc.head(pods, n - 1)  # fewer rows than shards: some shards get none
        em.assert_same(explain(many, tiny), explain(one, tiny), f"{n} shards, {n - 1} rows")
