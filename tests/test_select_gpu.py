"""GPU parity tests for the selection grid: the CUDA path through the C-ABI (host entry points) against the
C oracle on the same inputs -- bit-exact (integer / index work)."""
import json
import os

import numpy as np
import pytest

import oracle
import rpk
from test_oracle import CLOUD, kat_offers

pytestmark = pytest.mark.gpu


# "bitmap": the natural choice (fused kernel up to 16k rows, persistent kernel above); "bitmap_grouped": every size
# through the persistent kernel (an empty table: the fused kernel at every size)
KINDS = {"generic": 1, "packed": 2, "packed_pos": 3, "bitmap": 4, "bitmap_grouped": 4}


def upload_forced(engine, offers, force):
    """RPK_FORCE_KERNEL is read by rpk_offers_upload: run the same table through a chosen kernel."""
    old = os.environ.pop("RPK_FORCE_KERNEL", None)
    if force:
        os.environ["RPK_FORCE_KERNEL"] = force
    try:
        engine.upload_offers(offers)
    finally:
        os.environ.pop("RPK_FORCE_KERNEL", None)
        if old is not None:
            os.environ["RPK_FORCE_KERNEL"] = old


def check(engine, offers, pods, top5=True, expect_kind=None, all_kernels=True):
    """CUDA path vs oracle, bit-exact; by default through every kernel the table admits (the natural
    choice first, then each lower kind forced)."""
    ob, ot = oracle.select(offers, pods, want_top5=True, n_threads=8)
    best0 = None
    for force in ([None, "bitmap_grouped", "packed_pos", "packed", "generic"] if all_kernels else [None]):
        upload_forced(engine, offers, force)
        kind = engine.stats()["select_kernel_kind"]
        if force is None and expect_kind is not None:
            assert kind == expect_kind, (kind, expect_kind)
        if force is not None and kind > KINDS[force]:
            raise AssertionError(f"forcing {force} left kernel kind {kind}")
        best, t5 = engine.select(pods, want_top5=top5)
        assert np.array_equal(best, ob), f"[{force}/{kind}] best differs at rows {np.nonzero(best != ob)[0][:10]}"
        if top5:
            assert np.array_equal(t5, ot), f"[{force}/{kind}] top5 differs at rows {np.nonzero((t5 != ot).any(axis=1))[0][:10]}"
            assert np.array_equal(best, t5[:, 0])
        best0 = best if best0 is None else best0
    upload_forced(engine, offers, None)
    return best0


def test_kat_table(engine):
    kat, offers = kat_offers()
    engine.upload_offers(offers)
    for c in kat["cases"]:
        cloud = {"SECURE": 0, "COMMUNITY": 1}.get(c["cloud"], 7)
        pods = {"req_mem_gb": np.array([c["minMem"]], np.int32), "max_price": np.array([c["maxPrice"]], np.float64),
                "cloud": np.array([cloud], np.uint8)}
        best, t5 = engine.select(pods, want_top5=True)
        want = c["top5"] + [-1] * (5 - len(c["top5"]))
        assert t5[0].tolist() == want, c
        assert best[0] == want[0], c


def test_c1_reference_scale(engine):
    """BASELINE config 1: 100 pods x 50 GPU types, reference-exact profile."""
    check(engine, rpk.synth.make_offers(50, with_ext=False), rpk.synth.make_pods(100, reference_exact=True))


@pytest.mark.parametrize("tie_free,ref_exact,with_ext,corr", [
    (False, False, True, False), (False, False, True, True), (True, False, True, False),
    (False, True, False, True), (True, True, True, False)])
def test_c2_10k_by_1k(engine, tie_free, ref_exact, with_ext, corr):
    """BASELINE config 2: 10k pods x 1k offers, bit-exact assignments."""
    offers = rpk.synth.make_offers(1000, tie_free=tie_free, with_ext=with_ext, correlated=corr)
    pods = rpk.synth.make_pods(10_000, reference_exact=ref_exact)
    best = check(engine, offers, pods, expect_kind=4)
    assert len(np.unique(best)) >= 2


def test_nullable_columns_default_to_reference_behaviour(engine):
    offers = rpk.synth.make_offers(777, with_ext=False, correlated=True)
    pods = rpk.synth.make_pods(1234, reference_exact=True)
    engine.upload_offers(offers)
    full, _ = engine.select(pods)
    minimal, _ = engine.select({"req_mem_gb": pods["req_mem_gb"], "cloud": pods["cloud"]})
    assert np.array_equal(full, minimal)  # NULL max_price = 0.5, NULL vcpu/ram = 0
    sec, _ = engine.select({"req_mem_gb": pods["req_mem_gb"]})
    ob, _ = oracle.select(offers, {"req_mem_gb": pods["req_mem_gb"]})
    assert np.array_equal(sec, ob)  # NULL cloud = SECURE


def test_generic_kernel_full_int32_range(engine):
    """More distinct column values than the packed word can rank -> the int32-compare kernel."""
    G, P = 5000, 3000
    rng = np.random.default_rng(11)
    offers = rpk.synth.make_offers(G, correlated=True)
    offers["mem_gb"] = rng.integers(-2**31, 2**31 - 1, G, dtype=np.int64).astype(np.int32)
    offers["vcpu"] = rng.integers(-2**31, 2**31 - 1, G, dtype=np.int64).astype(np.int32)
    offers["ram_gb"] = rng.integers(0, 4000, G, dtype=np.int64).astype(np.int32)
    pods = rpk.synth.make_pods(P)
    pods["req_mem_gb"] = rng.integers(-2**31, 2**31, P, dtype=np.int64).astype(np.int32)
    pods["req_vcpu"] = rng.integers(-2**31, 2**31, P, dtype=np.int64).astype(np.int32)
    pods["req_ram_gb"] = rng.integers(0, 4000, P, dtype=np.int64).astype(np.int32)
    pods["req_mem_gb"][:8] = [2**31 - 1, -2**31, 0, -1, 2**31 - 2, 5, -2**31, 2**31 - 1]
    best = check(engine, offers, pods, expect_kind=1)
    assert (best >= 0).any() and (best < 0).any()


def test_bitmap_rows_of_33_to_64_thresholds(engine):
    """Column cardinalities that need more than 32 mask words per chunk: the bit-sliced kernel with 64-word
    rows (and, forced, every lower kernel on the same table)."""
    G, P = 9000, 5000
    rng = np.random.default_rng(9)
    offers = rpk.synth.make_offers(G, correlated=True)
    offers["mem_gb"] = (rng.integers(1, 31, G) * 8).astype(np.int32)      # 30 distinct
    offers["vcpu"] = (rng.integers(1, 13, G) * 4).astype(np.int32)        # 12 distinct
    offers["ram_gb"] = (rng.integers(1, 11, G) * 16).astype(np.int32)     # 10 distinct
    pods = rpk.synth.make_pods(P)
    pods["req_mem_gb"] = rng.integers(-8, 260, P).astype(np.int32)
    pods["req_vcpu"] = rng.integers(0, 56, P).astype(np.int32)
    pods["req_ram_gb"] = rng.integers(0, 180, P).astype(np.int32)
    pods["max_price"][:] = 10.0
    best = check(engine, offers, pods, expect_kind=4)
    st = engine.stats()
    assert st["distinct_mem"] + st["distinct_vcpu"] + st["distinct_ram"] + 3 > 32
    assert (best >= 0).any() and (best < 0).any()


def test_top5_sparse_feasibility(engine):
    """Rows with few or no feasible offers and no binding price bound: the top-5 walk has to cross most of the
    sorted view (worst case for the early-exit kernels)."""
    G, P = 50_000, 3000
    offers = rpk.synth.make_offers(G, correlated=True)
    pods = rpk.synth.make_pods(P)
    pods["req_mem_gb"][:] = 192
    pods["req_vcpu"][:] = 128
    pods["req_ram_gb"][:] = 512
    pods["req_mem_gb"][::7] = 10**6      # nothing feasible
    pods["max_price"][:] = 1e9
    pods["max_price"][::11] = np.nan     # NaN bound: nothing feasible
    best = check(engine, offers, pods)
    assert (best >= 0).any() and (best < 0).any()


def test_packed_select_layout_19_to_32_bits(engine):
    """Column cardinalities whose rank fields need more than 18 bits: the packed kernel without the
    embedded position (predicate + select form)."""
    G, P = 6000, 3000
    rng = np.random.default_rng(5)
    offers = rpk.synth.make_offers(G, correlated=True)
    offers["mem_gb"] = rng.integers(1, 900, G, dtype=np.int64).astype(np.int32)     # ~10 bits
    offers["vcpu"] = rng.integers(1, 400, G, dtype=np.int64).astype(np.int32)       # ~9 bits
    offers["ram_gb"] = rng.integers(1, 200, G, dtype=np.int64).astype(np.int32)     # ~8 bits
    pods = rpk.synth.make_pods(P)
    pods["req_mem_gb"] = rng.integers(-3, 950, P, dtype=np.int64).astype(np.int32)
    pods["req_vcpu"] = rng.integers(0, 420, P, dtype=np.int64).astype(np.int32)
    pods["req_ram_gb"] = rng.integers(0, 210, P, dtype=np.int64).astype(np.int32)
    pods["max_price"][:] = 10.0
    best = check(engine, offers, pods, expect_kind=2)
    assert (best >= 0).any() and (best < 0).any()


def test_packed_and_generic_agree(engine):
    """Same table through both kernels: force the generic one by adding high-cardinality noise to an
    offer that can never win, compare against the packed result on the untouched table."""
    G, P = 3000, 4000
    offers = rpk.synth.make_offers(G, correlated=True)
    pods = rpk.synth.make_pods(P)
    engine.upload_offers(offers)
    assert engine.stats()["select_kernel_kind"] == 4
    packed, _ = engine.select(pods)
    wide = {k: (v.copy() if v is not None else None) for k, v in offers.items()}
    # make the first 2500 offers unavailable and give them unique junk values: same feasible set, no packing
    wide_full = {k: (np.concatenate([v, v[:2500]]) if v is not None else None) for k, v in wide.items()}
    wide_full["flags"][G:] = 0
    wide_full["mem_gb"][G:] = np.arange(1000, 3500, dtype=np.int32) * 7
    wide_full["vcpu"][G:] = np.arange(1000, 3500, dtype=np.int32) * 11
    wide_full["ram_gb"][G:] = np.arange(1000, 3500, dtype=np.int32) * 13
    engine.upload_offers(wide_full)
    assert engine.stats()["select_kernel_kind"] == 1
    generic, _ = engine.select(pods)
    assert np.array_equal(packed, generic)


def test_edge_cases(engine):
    offers = rpk.synth.make_offers(64)
    offers["secure_price"][:4] = [np.nan, np.inf, -1.0, 5e-324]
    offers["flags"][:4] = 3
    pods = {
        "req_mem_gb": np.array([-5, 0, 2**31 - 1, -(2**31), 16, 16, 16], np.int32),
        "req_vcpu": np.zeros(7, np.int32), "req_ram_gb": np.zeros(7, np.int32),
        "max_price": np.array([0.5, np.inf, 0.5, 0.5, np.nan, -1.0, 1e308], np.float64),
        "cloud": np.array([0, 0, 0, 0, 0, 1, 7], np.uint8),
    }
    check(engine, offers, pods)
    # single pod, single offer
    one = {k: (v[:1].copy() if v is not None else None) for k, v in offers.items()}
    one["secure_price"][0] = 0.3
    check(engine, one, {k: v[:1].copy() for k, v in pods.items()})
    # empty offer table: every pod gets -1; P == 0 is a no-op
    empty = {k: (v[:0].copy() if v is not None else None) for k, v in offers.items()}
    engine.upload_offers(empty)
    best, t5 = engine.select(pods, want_top5=True)
    assert (best == -1).all() and (t5 == -1).all()
    b0, _ = engine.select({"req_mem_gb": np.zeros(0, np.int32)})
    assert b0.size == 0
    # empty offer table and a batch above the fused kernel's size, through every kernel
    best = check(engine, empty, rpk.synth.make_pods(20_000))
    assert (best == -1).all()
    # nothing feasible at all / everything tied
    offers2 = rpk.synth.make_offers(300)
    offers2["secure_price"][:] = 0.25
    offers2["community_price"][:] = 0.25
    check(engine, offers2, rpk.synth.make_pods(500))
    offers2["flags"][:] = 0
    best = check(engine, offers2, rpk.synth.make_pods(500))
    assert (best == -1).all()


def test_ragged_sizes(engine):
    """P and G around every tiling boundary (warp, chunk of 128, segment, row tile)."""
    for G in (1, 31, 32, 33, 127, 128, 129, 4095, 4097, 16383, 16385, 20000):
        offers = rpk.synth.make_offers(G, correlated=True, seed=G)
        for P in (1, 7, 8, 9, 127, 129, 255, 257, 1000):
            check(engine, offers, rpk.synth.make_pods(P, seed=P + G), top5=(P <= 129), all_kernels=(P in (7, 257, 1000)))


def test_rejects_bad_arguments(engine):
    offers = rpk.synth.make_offers(10)
    bad = dict(offers)
    bad["mem_gb"] = offers["mem_gb"].copy()
    bad["mem_gb"][3] = 2**31 - 1
    with pytest.raises(rpk.RpkError) as ei:
        engine.upload_offers(bad)
    assert ei.value.code == rpk._ffi.RPK_EINVAL
    fresh = rpk.Engine(1)
    with pytest.raises(rpk.RpkError) as ei:
        fresh.select(rpk.synth.make_pods(4))
    assert ei.value.code == rpk._ffi.RPK_ESTATE
    fresh.close()


def test_c3_100k_by_10k_sampled(engine):
    """BASELINE config 3 (10^9 offer-scores): full GPU run; oracle on a row sample plus size-independent
    properties (feasibility and minimality of every assignment, checked with numpy)."""
    G, P = 10_000, 100_000
    offers = rpk.synth.make_offers(G, correlated=True)
    pods = rpk.synth.make_pods(P)
    engine.upload_offers(offers)
    best, t5 = engine.select(pods, want_top5=True)
    verify_properties(offers, pods, best)
    rows = np.random.default_rng(3).choice(P, 1500, replace=False)
    sub = {k: np.ascontiguousarray(v[rows]) for k, v in pods.items()}
    ob, ot = oracle.select(offers, sub, n_threads=8)
    assert np.array_equal(best[rows], ob) and np.array_equal(t5[rows], ot)


def verify_properties(offers, pods, best):
    """Every assignment is feasible, and no strictly cheaper (or equal-price, lower-index) feasible offer
    exists: checked per distinct pod class so it stays O(classes x G)."""
    cols = np.stack([pods["req_mem_gb"].astype(np.float64), pods["req_vcpu"].astype(np.float64), pods["req_ram_gb"].astype(np.float64),
                     pods["max_price"], pods["cloud"].astype(np.float64)], axis=1)
    classes, inv = np.unique(cols, axis=0, return_inverse=True)
    inv = inv.reshape(-1)
    for ci, (m, v, r, mp, c) in enumerate(classes):
        ids = oracle.get_gpu_types(offers, int(m), float(mp), int(c) if c in (0, 1) else 2, int(v), int(r))
        want = ids[0] if ids else -1
        got = best[inv == ci]
        assert (got == want).all(), (m, v, r, mp, c, want, np.unique(got))


def test_c4_shape_1m_by_100k_properties(engine):
    """BASELINE config 4's full size on one GPU (10^11 offer-scores): checked through the class property
    (all pods of one (mem, vcpu, ram, max_price, cloud) class share the oracle's answer)."""
    G, P = 100_000, 1_000_000
    offers = rpk.synth.make_offers(G, correlated=True)
    pods = rpk.synth.make_pods(P)
    engine.upload_offers(offers)
    best, _ = engine.select(pods)
    verify_properties(offers, pods, best)


def test_random_small_tables_property(engine):
    """hypothesis: arbitrary small tables (NaN / inf / zero / negative prices, duplicated prices, extreme int32
    columns and requests, unknown cloud bytes, with and without extension columns) through every kernel."""
    from hypothesis import given, settings

    from test_oracle_property import tables

    @settings(max_examples=120, deadline=None)
    @given(tables())
    def run(t):
        offers, pods = t
        check(engine, offers, pods)

    run()
