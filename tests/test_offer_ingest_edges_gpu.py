"""GPU tests of the offer-table ingest (launch_offer_ingest, offers.cu) at its edges: the price keys, the bitonic sort
of (key, offer index) pairs across its block and global stages, the per-column distinct values k_unique carries from
one 1024-key round to the next, and every view layout the distinct counts select.

Each case first asserts through persist_plan_model.layout, and through rpk_stats (select_kernel_kind, packed_bits,
distinct_*), that the table reaches the layout the case is named for, so a change to a constant that moves a case off
its boundary fails it.  Then every row of best and of top-5 is compared with the oracle, through the host and the
device entry points, for pods with and without the optional columns (3 % with an unknown cloud byte), through every
kernel the table admits: the automatic choice, then RPK_FORCE_KERNEL packed_pos, packed and generic, and
bitmap_grouped / bitmap_price where a bit-sliced view exists.  Pods request below the smallest value, at every value
and one either side of it, above the largest, and at -2^31 and 2^31 - 1."""
import numpy as np
import pytest

import persist_plan_model as model
import select_plan_cases as sc

pytestmark = pytest.mark.gpu

FORCES = [None, "packed_pos", "packed", "generic", "bitmap_grouped", "bitmap_price"]
I32_MIN, I32_MAX = -2**31, 2**31 - 1
ROWS = 2048


# ---- pods and checks -----------------------------------------------------------------------------------------------
def requests(col):
    """below the smallest value, every value and one either side of it, above the largest, and both int32 ends"""
    v = np.unique(col).astype(np.int64)
    r = np.concatenate([v - 1, v, v + 1, [0, I32_MIN, I32_MAX]])
    return np.unique(np.clip(r, I32_MIN, I32_MAX)).astype(np.int32)


def pods_for(offers, P=ROWS, seed=0):
    """at least P rows; every request value of every column occurs (each column cycles through its own permutation)"""
    rng = np.random.default_rng(seed)
    req = {k: requests(offers[c] if offers[c] is not None else np.zeros(1, np.int32))
           for k, c in (("req_mem_gb", "mem_gb"), ("req_vcpu", "vcpu"), ("req_ram_gb", "ram_gb"))}
    P = max(P, max(len(r) for r in req.values()))
    pods = {k: np.resize(rng.permutation(r), P) for k, r in req.items()}
    pods["max_price"] = rng.choice(sc.price_set(offers), P).astype(np.float64)
    pods["cloud"] = rng.integers(0, 2, P).astype(np.uint8)
    odd = rng.random(P) < 0.03
    pods["cloud"][odd] = rng.choice(np.array([2, 7, 255], np.uint8), int(odd.sum()))
    return pods


def distinct_counts(offers):
    return [len(d) for d in model.distinct(offers)]


def assert_layout(engine, D, force, what):
    """rpk_stats after an upload equal persist_plan_model.layout(D, force)"""
    L = model.layout(D, force)
    st = engine.stats()
    got = (st["select_kernel_kind"], st["packed_bits"], [st["distinct_mem"], st["distinct_vcpu"], st["distinct_ram"]])
    assert got == (L.kind, L.packed_bits, list(D)), f"{what} [{force}]: stats {got}, the model says {L}"
    return L


def check_all(engine, offers, pod_sets, what, force):
    for i, (pods, wb, wt) in enumerate(pod_sets):
        sc.check(f"{what} [{force}] pods {i} host", *sc.run_host(engine, pods, True), wb, wt)
        sc.check(f"{what} [{force}] pods {i} device", *sc.run_device(engine, pods, True), wb, wt)


def oracle_sets(offers, P=ROWS, seed=0):
    pods = pods_for(offers, P, seed)
    return [(p,) + tuple(sc.expected(offers, p)) for p in (pods, sc.without_optional(pods))]


def run_case(engine, offers, what, want_kind=None, P=ROWS, seed=0):
    """the table's layout is `want_kind` (a KIND_NAMES value); every kernel it admits equals the oracle.  Forced
    choices that the model says build the same views as an earlier one are skipped."""
    D = distinct_counts(offers)
    natural = model.layout(D)
    if want_kind is not None:
        assert natural.name == want_kind, f"{what}: D = {D} gives {natural}, not {want_kind}"
    sets = oracle_sets(offers, P, seed)
    seen = set()
    for force in FORCES:
        L = model.layout(D, force)
        key = (L.kind, L.packed_bits, L.pos_bits, L.bm_words, L.no_fused, L.no_slice)
        if key in seen:
            continue
        seen.add(key)
        with sc.forced(force):
            engine.upload_offers(offers)
        assert_layout(engine, D, force, what)
        check_all(engine, offers, sets, what, force)
    return natural


# ---- layout boundaries ---------------------------------------------------------------------------------------------
# (dm, dv, dr) distinct mem / vcpu / ram values -> the automatic layout
LAYOUT_EDGES = {
    (62, 15, 31): "packed_pos",    # 6 + 4 + 5 + 3 = 18 bits: the position field fits
    (63, 15, 31): "packed",        # mem threshold 64 takes 7 bits: 19
    (62, 16, 31): "packed",        # vcpu threshold 16: 5 bits
    (62, 15, 32): "packed",        # ram threshold 32: 6 bits
    (64, 15, 31): "packed",        # 2^k + 1 thresholds
    (30, 64, 7): "packed_pos",     # vcpu at 2^6: 18 bits
    (14, 7, 128): "packed_pos",    # ram at 2^7: 18 bits
    (1022, 1023, 511): "packed",   # 10 + 10 + 9 + 3 = 32 bits
    (1023, 1023, 511): "generic",  # mem threshold 1024: 33
    (1022, 1024, 511): "generic",
    (1022, 1023, 512): "generic",
    (15, 7, 7): "bitmap",          # 32 mask words: 32-word rows
    (16, 7, 7): "bitmap",          # 33: 64-word rows
    (47, 7, 7): "bitmap",          # 64
    (48, 7, 7): "packed_pos",      # 65: no bit-sliced view
    (31, 7, 7): "bitmap",          # 2 x 32 x 8 x 8 = 4096 classes: per-mem-threshold slices
    (32, 7, 7): "bitmap",          # 4224: staged by price only
}


@pytest.mark.parametrize("D,kind", list(LAYOUT_EDGES.items()), ids=lambda x: "-".join(map(str, x)) if isinstance(x, tuple) else x)
def test_layout_boundary(engine, D, kind):
    G = 4099
    offers = sc.distinct_table(G, *D, seed=sum(D))
    assert distinct_counts(offers) == list(D)
    L = run_case(engine, offers, f"D={D}", kind)
    if kind == "bitmap":
        words = sum(D) + 3
        assert L.bm_words == words and L.bm_stride == (32 if words <= 32 else 64)
        assert L.slice == (2 * (D[0] + 1) * (D[1] + 1) * (D[2] + 1) <= model.MAX_CLASSES)


# ---- sort and distinct edges ---------------------------------------------------------------------------------------
SORT_G = [1023, 1024, 1025, 2047, 2048, 2049, 16385, 65537, 131073]
# offer indices where the mem step columns change value: the block (1024) and global stage boundaries of the sort
STEPS = [1, 511, 1022, 1023, 1024, 1025, 2046, 2047, 2048, 2049, 4095, 4096, 16383, 16384, 16385, 65535, 65536,
         65537, 131071, 131072]


def step_column(G, rising, scale=4):
    """mem by offer index, changing value at every STEPS index below G (rising: higher indices hold more memory)"""
    cuts = np.array([s for s in STEPS if s < G], np.int64)
    k = np.searchsorted(cuts, np.arange(G), side="right")
    return ((k if rising else len(cuts) - k) * scale + scale).astype(np.int32)


def pattern_table(G, pattern, seed):
    """prices by pattern; mem steps at the sort's stage boundaries, in the direction that puts the cheapest feasible
    offer of each mem threshold at a step (equal prices: the lowest feasible index, so rising mem; descending prices:
    the highest feasible index, so falling mem)"""
    rng = np.random.default_rng(seed)
    i = np.arange(G)
    flags = np.full(G, 3, np.uint8)
    vcpu = rng.choice(np.array([2, 4, 8], np.int32), G)
    ram = rng.choice(np.array([16, 32], np.int32), G)
    if pattern == "equal":
        sp, cp, mem = np.full(G, 1.25), np.full(G, 0.75), step_column(G, True)
    elif pattern == "descending":
        sp, cp, mem = (G - i) / 100.0, (G - i) / 200.0, step_column(G, False)
    elif pattern == "alternating":
        sp, cp, mem = np.where(i % 2, 2.0, 1.0), np.where(i % 2, 1.0, 2.0), step_column(G, True)
    elif pattern == "sparse":
        # only the first and the last offer have cloud flags, and the last has no secure price
        sp, cp, mem = np.full(G, 3.0), np.full(G, 0.0), step_column(G, True)
        flags[:] = 0
        flags[0], flags[-1] = 3, 3
        cp[-1], sp[-1] = 0.5, 0.0
        cp[0] = 0.25
    elif pattern == "special":
        # +Inf and the least subnormal next to NaN, 0.0 and -0.0, and two prices 2^-40 apart
        cyc = np.array([np.inf, 5e-324, np.nan, 0.0, -0.0, 1.0, 1.0 + 2**-40])
        sp = cyc[i % len(cyc)]
        cp = cyc[(i + 3) % len(cyc)]
        mem = step_column(G, True)
    else:
        raise ValueError(pattern)
    return {"mem_gb": mem, "vcpu": vcpu, "ram_gb": ram, "secure_price": sp.astype(np.float64),
            "community_price": cp.astype(np.float64), "flags": flags}


@pytest.mark.parametrize("pattern", ["equal", "descending", "alternating", "sparse", "special"])
@pytest.mark.parametrize("G", SORT_G)
def test_sort_edges(engine, G, pattern):
    """tables of 1023 .. 131073 offers (sort length n = 1024 .. 262144), whose price keys tie across the sort's block
    and global stages, run against it, alternate, or are almost all excluded"""
    offers = pattern_table(G, pattern, seed=G)
    P = 1024
    pods = pods_for(offers, P, seed=G)
    # the mem requests cover every step, so some rows' cheapest offer sits at each stage boundary below G
    assert set(np.unique(offers["mem_gb"])) <= set(pods["req_mem_gb"].tolist())
    run_case(engine, offers, f"{pattern} G={G}", P=P, seed=G)


def test_sort_over_eight_million_keys(engine):
    """2^22 + 1 offers: n = 2^23, merge stages k = 2^11 .. 2^23 across blocks.  Prices fall with the index in pairs
    of equal price and mem falls in 61 steps, so each mem threshold's cheapest feasible offer is the first of a tie
    pair at a different depth of the array; checked by row class."""
    G = 2**22 + 1
    rng = np.random.default_rng(22)
    i = np.arange(G, dtype=np.int64)
    mem = ((60 - (i * 61) // G) * 4 + 4).astype(np.int32)
    sp = ((G - i) // 2 + 1) / 100.0
    offers = {"mem_gb": mem, "vcpu": rng.choice(np.array([2, 4, 8], np.int32), G),
              "ram_gb": rng.choice(np.array([16, 32], np.int32), G), "secure_price": sp, "community_price": sp * 0.5,
              "flags": rng.integers(0, 4, G).astype(np.uint8)}
    D = distinct_counts(offers)
    assert D == [61, 3, 2] and model.layout(D).name == "packed_pos"
    assert len(pods_for(offers, 256)["req_mem_gb"]) * G > sc.ROW_ORACLE_LIMIT  # checked by row class
    run_case(engine, offers, "2^22 + 1 offers", "packed_pos", P=256, seed=22)


def heads_column(G, values, heads, rng):
    """a column whose sorted order starts values[k] at sorted position heads[k], shuffled over the offers"""
    counts = np.diff(np.append(heads, G))
    return rng.permutation(np.repeat(np.asarray(values, np.int64), counts)).astype(np.int32)


@pytest.mark.parametrize("G", [2049, 3073])
def test_distinct_round_edges(engine, G):
    """new distinct values first appear at sorted positions 1023, 1024 and 2048, where k_unique carries its count
    from one 1024-key round into the next, with -2^31 and 2^31 - 2 among the values"""
    rng = np.random.default_rng(G)
    heads = [0, 1023, 1024, 2048] + ([2500, 3072] if G > 3072 else [])
    top = 2**31 - 2
    mem = heads_column(G, [I32_MIN, 8, 16, 40, 2**31 - 3, top][:len(heads) - 1] + [top], heads, rng)
    vcpu = heads_column(G, [-5, 0, 3, 7, 100, top][:len(heads) - 1] + [top], heads, rng)
    ram = heads_column(G, [I32_MIN, I32_MIN + 1, 64, 65, 66, top][:len(heads) - 1] + [top], heads, rng)
    offers = sc._table(G, mem, vcpu, ram, rng)
    assert distinct_counts(offers) == [len(heads)] * 3
    for col in ("mem_gb", "vcpu", "ram_gb"):
        s = np.sort(offers[col])
        first = np.nonzero(np.r_[True, s[1:] != s[:-1]])[0].tolist()
        assert first == heads and s[0] < 0 < s[-1] == top, (col, first)
    run_case(engine, offers, f"distinct heads G={G}", P=1024, seed=G)


# ---- position segments ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("G", [16383, 16384, 16385, 32767, 32768, 32769])
def test_position_segments(engine, G):
    """packed_pos words carry the position inside 16384-offer segments.  Prices rise with the index in both clouds, so
    an offer's view position is its index, and the only offers with more memory than the base sizes sit at 16383,
    16384, 32767, 32768 and G - 1: rows that ask for one of those sizes win at a segment's last or first position, or
    at the table's last offer."""
    rng = np.random.default_rng(G)
    i = np.arange(G)
    mem = rng.choice(np.array([4, 8, 12], np.int32), G)
    vcpu = rng.choice(np.arange(1, 61, dtype=np.int32) * 2, G)
    ram = rng.choice(np.array([16, 32], np.int32), G)
    marks = {p: m for p, m in ((16383, 100), (16384, 200), (32767, 240), (32768, 260), (G - 1, 300)) if p < G}
    for p, m in marks.items():
        mem[p], vcpu[p], ram[p] = m, 120, 32
    offers = {"mem_gb": mem, "vcpu": vcpu, "ram_gb": ram, "secure_price": (i + 1) / 100.0,
              "community_price": (i + 1) / 200.0, "flags": np.full(G, 3, np.uint8)}
    D = distinct_counts(offers)
    assert D[1] == 60 and sum(D) + 3 > model.BM_MAX_STRIDE  # no bit-sliced view
    pods, wb, _ = oracle_sets(offers)[0]
    for p in marks:
        assert (wb == p).any(), f"no row wins at position {p}"
    run_case(engine, offers, f"segments G={G}", "packed_pos")


# ---- layout changes on one engine ----------------------------------------------------------------------------------
def checked(engine, offers, what, force=None):
    D = distinct_counts(offers)
    assert_layout(engine, D, force, what)
    check_all(engine, offers, oracle_sets(offers, seed=len(what)), what, force)
    return model.layout(D, force)


def test_layout_changes_by_upload(engine):
    """a large table with no rank layout, then small packed_pos and bit-sliced ones, then the large one again: the
    views of one table must not leak into the next one's select"""
    wide = sc.distinct_table(65_537, 1022, 1023, 512, 1)
    small = sc.distinct_table(3_000, 62, 15, 31, 2)
    bits = sc.distinct_table(3_000, 15, 7, 7, 3)
    kinds = []
    for name, offers in (("wide", wide), ("small", small), ("wide again", wide), ("bit-sliced", bits),
                         ("wide after bit-sliced", wide)):
        with sc.forced(None):
            engine.upload_offers(offers)
        kinds.append(checked(engine, offers, name).name)
    assert kinds == ["generic", "packed_pos", "generic", "bitmap", "generic"]


def new_value_edit(offers, col, rng):
    """a copy of `offers` where one offer whose value occurs more than once takes a value no offer has: the column
    gains one distinct value"""
    new = {k: (None if v is None else np.array(v, copy=True)) for k, v in offers.items()}
    vals, counts = np.unique(new[col], return_counts=True)
    g = int(rng.choice(np.nonzero(np.isin(new[col], vals[counts > 1]))[0]))
    new[col][g] = int(vals[-1]) + 1
    return new


@pytest.mark.parametrize("D,col,before,after", [
    ((62, 15, 31), "mem_gb", "packed_pos", "packed"),   # 18 -> 19 bits
    ((62, 15, 31), "vcpu", "packed_pos", "packed"),
    ((1022, 1023, 511), "ram_gb", "packed", "generic"),  # 32 -> 33 bits
    ((15, 7, 7), "mem_gb", "bitmap", "bitmap"),          # 32 -> 33 mask words: 32- to 64-word rows
    ((47, 7, 7), "ram_gb", "bitmap", "packed_pos"),      # 64 -> 65 mask words: no bit-sliced view
    ((31, 7, 7), "vcpu", "bitmap", "bitmap"),            # 4096 -> 4608 classes: the slices go
])
def test_layout_changes_by_refresh(engine, D, col, before, after):
    """rpk_offers_refresh of a table with the same G where one changed offer moves a distinct count across a layout
    boundary, and a second refresh that moves it back"""
    rng = np.random.default_rng(sum(D))
    offers = sc.distinct_table(4_099, *D, seed=sum(D) + 1)
    changed = new_value_edit(offers, col, rng)
    with sc.forced(None):
        engine.upload_offers(offers)
        L0 = checked(engine, offers, f"{D} uploaded")
        assert engine.refresh_offers(changed) == 1
        L1 = checked(engine, changed, f"{D} refreshed: {col} + 1")
        assert engine.refresh_offers(offers) == 1
        L2 = checked(engine, offers, f"{D} refreshed back")
    assert (L0.name, L1.name, L2.name) == (before, after, before)
    assert (L0.bm_stride, L0.slice, L0.packed_bits) != (L1.bm_stride, L1.slice, L1.packed_bits)
