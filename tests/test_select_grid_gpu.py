"""GPU tests of the grid kernels that tables without a bit-sliced view take -- k_select_packed<R, true> (kind 3,
packed_pos), k_select_packed<R, false> (kind 2, packed), k_select_wide<R> (kind 1, generic), with k_pod_prep,
finish_tile and k_select_top5 around them -- at every rows-per-warp instantiation R in {1, 2, 4, 8, 16} and at the
edges of their offer segments, against the oracle.

Sizes come from the device's SM count through persist_plan_model.py: P = b - 1 and b at every R boundary b, and 1M
rows.  Each case asserts its regime through the model (the kind and packed bits of layout(), R and the segment count
S), fills every output with SENTINEL, and checks every row of best and top-5 (select_plan_cases.check).  Pod rows are
drawn from a few request values per column (just below, at and above table values, so on kinds 3 and 2 all 8 row
groups of k_pod_prep occur; kind 1 puts every row in group 3 or 7), max_price from NaN, +-inf, -0.0, 0, a bound above every price and prices of the table, and 3 %
carry an unknown cloud byte; so the oracle runs once per row class (select_plan_cases.expected).

The segment-edge tables place offers at chosen positions of the price-sorted views: every offer is in both clouds
with a positive price, prices rise with the position in runs of 8 equal prices that straddle every multiple of 8, and
offer indices inside a run rise with the position, so an offer's position is known.  Edge classes are an antichain
of (mem, ram) requests, each met by its own offers only: one offer just below, at or just above a segment boundary
(or the last offer), or four offers of one equal-price run on both sides of a boundary.

The last test runs the wide kernel over 2^26 offers with batches whose grid has more than 2^31 - 1 CTAs."""
import functools
import os
import subprocess
import sys
import time

import numpy as np
import pytest

import persist_plan_model as model
import rpk
import select_plan_cases as sc
import select_scale_model as sm

pytestmark = pytest.mark.gpu
SENTINEL = sc.SENTINEL
P_1M = 1_000_000


# ---- tables ----------------------------------------------------------------------------------------------------------
# name: (builder, kind, RPK_FORCE_KERNEL); the natural kinds come from the distinct counts (layout())
TABLES = {
    "pos16384": (lambda: sc.distinct_table(16_384, 62, 15, 31, 1), 3, None),     # 18 layout bits; one segment
    "pos16385": (lambda: sc.distinct_table(16_385, 62, 15, 31, 2), 3, None),     # two segments, the second 128 offers
    "pos100k": (lambda: sc.distinct_table(100_000, 62, 15, 31, 3), 3, None),     # 7 segments
    "packed100k": (lambda: sc.distinct_table(100_000, 200, 60, 100, 4), 2, None),  # 8 + 6 + 7 + 3 = 24 bits; 7 x 14 336
    "wide20k": (lambda: sc.full_int32_table(20_000, 5), 1, None),                # 5 x 4096
    "wide100k": (lambda: sc.full_int32_table(100_000, 6), 1, None),              # 25 x 4096
    "synth_pos": (lambda: sc.table("synth100k"), 3, "packed_pos"),
    "synth_packed": (lambda: sc.table("synth100k"), 2, "packed"),
    "synth_generic": (lambda: sc.table("synth100k"), 1, "generic"),
}


@functools.lru_cache(maxsize=None)
def table(name):
    return TABLES[name][0]()


def upload(eng, offers, kind, force):
    """upload under `force` and assert the layout the model gives: kind, packed bits, no bit-sliced view"""
    D = [len(d) for d in model.distinct(offers)]
    L = model.layout(D, force)
    assert L.kind == kind and L.bm_words == 0, (D, force, L)
    with sc.forced(force):
        eng.upload_offers(offers)
    st = eng.stats()
    assert (st["select_kernel_kind"], st["packed_bits"]) == (L.kind, L.packed_bits), (st, L)
    return model.grid_segments(kind, len(offers["mem_gb"]))


# ---- pod rows --------------------------------------------------------------------------------------------------------
def _pool(col, n, rng):
    """n request values around a column's distinct values: below the smallest (meets every offer), at and just above
    values spread over the range, and above the largest (meets none)"""
    v = np.unique(col).astype(np.int64)
    picks = v[np.linspace(0, len(v) - 1, n - 2).astype(int)] + rng.integers(0, 2, n - 2)
    return np.unique(np.clip(np.r_[v[0] - 1, picks, v[-1] + 1], -2**31, 2**31 - 1)).astype(np.int32)


def price_pool(offers, rng):
    """NaN, +-inf, -0.0, 0, 1e9, and five prices of the table (the strict bound meets ties)"""
    p = np.concatenate([offers["secure_price"], offers["community_price"]])
    p = np.unique(p[np.isfinite(p) & (p > 0)])
    return np.r_[np.nan, np.inf, -np.inf, -0.0, 0.0, 1e9, rng.choice(p, 5)]


def pool_pods(offers, P, seed):
    """P rows: mem from 12 values, vcpu and ram from 4 each (half of them 0 or below every value, so the rows fall in
    all 8 row groups), max_price from price_pool, clouds 0 / 1 and 3 % unknown bytes (2, 7, 255)"""
    rng = np.random.default_rng(seed)
    pods = {}
    for req, col, n in (("req_mem_gb", "mem_gb", 12), ("req_vcpu", "vcpu", 4), ("req_ram_gb", "ram_gb", 4)):
        pods[req] = rng.choice(_pool(offers[col], n, rng), P).astype(np.int32)
        if req != "req_mem_gb":
            pods[req][rng.random(P) < 0.5] = min(0, int(np.min(offers[col])))
    pods["max_price"] = rng.choice(price_pool(offers, rng), P)
    pods["cloud"] = rng.integers(0, 2, P).astype(np.uint8)
    odd = rng.random(P) < 0.03
    pods["cloud"][odd] = rng.choice(np.array([2, 7, 255], np.uint8), int(odd.sum()))
    return pods


@functools.lru_cache(maxsize=None)
def batch(name, nulls=False):
    """(pods, oracle best, oracle top5) of P_1M rows for table `name`; nulls: only req_mem_gb is passed"""
    offers = table(name)
    pods = pool_pods(offers, P_1M, seed=len(name))
    if nulls:
        pods = sc.without_optional(pods)
    return (pods,) + tuple(sc.expected(offers, pods))


def rows(name, P, nulls=False):
    pods, wb, wt = batch(name, nulls)
    return sc.head(pods, P), wb[:P], wt[:P]


def sizes(sms):
    """[(P, R)]: b - 1 and b at every R boundary, then 1M rows"""
    out = []
    for b in model.rows_per_warp_bounds(sms):
        out += [(b - 1, model.rows_per_warp(b - 1, sms)), (b, model.rows_per_warp(b, sms))]
    out.append((P_1M, 16))
    assert [R for _, R in out] == [1, 2, 2, 4, 4, 8, 8, 16, 16]
    return out


@pytest.fixture(scope="module")
def eng():
    e = rpk.Engine(1)
    yield e
    e.close()


# ---- every R, every kind ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", list(TABLES))
def test_rows_per_warp(eng, name):
    """one device call per size (so the R in use is known), top-5 on every other size and on 1M rows; NULL optional
    columns at every boundary b; the host entry point at 1M rows (sub-batches of R = 8, 16, 16, 16)"""
    offers = table(name)
    _, kind, force = TABLES[name]
    S, seg_len = upload(eng, offers, kind, force)
    G = len(offers["mem_gb"])
    want_S = {16_384: 1, 16_385: 2, 20_000: 5}.get(G, 25 if kind == 1 else 7)
    assert S == want_S, (name, S, seg_len)
    sms = sc.sm_count()
    pods, _, _ = batch(name)
    # kinds 3 / 2 group rows by cloud and by whether the vcpu / ram thresholds constrain: all 8 groups occur; the
    # generic kernel has no thresholds and puts every row in group 3 or 7
    occupied = np.nonzero(model.row_groups(kind, model.distinct(offers), pods))[0].tolist()
    assert occupied == ([3, 7] if kind == 1 else list(range(8))), (name, occupied)
    for i, (P, R) in enumerate(sizes(sms)):
        assert model.rows_per_warp(P, sms) == R
        p, wb, wt = rows(name, P)
        top5 = i % 2 == 0 or P == P_1M
        sc.check(f"{name} P={P} R={R} S={S} device top5={top5}", *sc.run_device(eng, p, top5), wb, wt if top5 else None)
        if i % 2:
            p, wb, wt = rows(name, P, nulls=True)
            sc.check(f"{name} P={P} R={R} device, NULL optional columns", *sc.run_device(eng, p, R == 16), wb,
                     wt if R == 16 else None)
    assert [model.rows_per_warp(P, sms) for P in model.host_sub_batches(P_1M)] == [8, 16, 16, 16]
    p, wb, wt = rows(name, P_1M)
    sc.check(f"{name} host 1M rows top5", *sc.run_host(eng, p, True), wb, wt)
    p, wb, _ = rows(name, P_1M)
    sc.check(f"{name} device 1M rows", *sc.run_device(eng, p, False), wb, None)


# ---- segment edges ---------------------------------------------------------------------------------------------------
RUN = 8  # equal-price run length of the edge tables; runs cover positions [8k - 4, 8k + 4)


def edge_positions(kind, G):
    """the positions of each edge class's offers: one offer at b - 1, b and b + 1 of every segment boundary b (multiples
    of 16 384 for kind 3, whose words carry the position in the segment; of 14 336 for kind 2 at 100k offers; of 4096
    for kind 1), one at G - 1, and four of one equal-price run on both sides of the first and the last boundary"""
    S, seg_len = model.grid_segments(kind, G)
    bounds = [k * seg_len for k in range(1, S)]
    cls = []
    for b in bounds:
        cls += [[b - 1], [b], [b + 1]]
    cls.append([G - 1])
    for b in sorted({bounds[0], bounds[-1]}):
        cls.append([b - 4, b - 3, b + 2, b + 3])
    return cls


EDGE = {  # name: (kind, G, mem / vcpu / ram distinct counts of the whole table, or None: full int32 columns)
    "pos": (3, 100_000, (62, 15, 31)),
    "packed": (2, 100_000, (200, 60, 100)),
    "wide": (1, 20_000, None),
}


@functools.lru_cache(maxsize=None)
def edge_table(name):
    """(offers, classes [(mem request, ram request, positions, table indices of its offers, their price)]) of an edge
    table"""
    kind, G, D = EDGE[name]
    rng = np.random.default_rng(G + kind)
    cls = edge_positions(kind, G)
    K = len(cls)
    if D is None:  # full int32 columns, the K largest mem and ram values kept for the classes
        base = lambda: rng.integers(-2**31 + 1, 2**31 - 1 - 4 * K, G, dtype=np.int64)  # noqa: E731
        mem, vcpu, ram = base(), base(), base()
        mem_hi = 2**31 - 1 - 2 * K + np.arange(K)
        ram_hi = 2**31 - 1 - 2 * K + np.arange(K)
    else:
        dm, dv, dr = D
        assert dm > K and dr > K, (name, K)
        mem = sc._columns(G, np.arange(1, dm - K + 1) * 4, rng).astype(np.int64)
        vcpu = sc._columns(G, np.arange(1, dv + 1) * 3, rng).astype(np.int64)
        ram = sc._columns(G, np.arange(1, dr - K + 1) * 16, rng).astype(np.int64)
        mem_hi = (dm - K + 1 + np.arange(K)) * 4
        ram_hi = (dr - K + 1 + np.arange(K)) * 16
    # class j: mem_hi[j] and ram_hi[K - 1 - j], so a request for exactly that pair meets class j's offers only (the
    # arrays are indexed by price-sorted position here)
    for j, pos in enumerate(cls):
        mem[pos], ram[pos] = mem_hi[j], ram_hi[K - 1 - j]
    run = (np.arange(G) + RUN // 2) // RUN
    cents = 100 + run
    perm = rng.permutation(G)  # table index of each position: random runs, indices rising inside each run
    perm = perm[np.lexsort((perm, run))]
    offers = {}
    for k, col in (("mem_gb", mem), ("vcpu", vcpu), ("ram_gb", ram)):
        a = np.empty(G, np.int32)
        a[perm] = col
        offers[k] = a
    price = np.empty(G)
    price[perm] = cents / 100.0
    offers["secure_price"] = price
    offers["community_price"] = price / 2
    offers["flags"] = np.full(G, 3, np.uint8)
    if D is not None:
        assert [len(d) for d in model.distinct(offers)] == list(D), name
    classes = [(int(mem_hi[j]), int(ram_hi[K - 1 - j]), np.array(pos), perm[pos], cents[pos[0]] / 100.0)
               for j, pos in enumerate(cls)]
    return offers, classes


def edge_pods(offers, classes, P, seed):
    """P rows: half of them one edge class each (no vcpu constraint, cloud 0 or 1, max_price +inf, the class's price,
    the next run's price or NaN), the others pool_pods rows"""
    rng = np.random.default_rng(seed)
    pods = pool_pods(offers, P, seed)
    e = np.nonzero(rng.random(P) < 0.5)[0]
    j = rng.integers(0, len(classes), len(e))
    cm = np.array([c[0] for c in classes], np.int32)
    cr = np.array([c[1] for c in classes], np.int32)
    cp = np.array([c[4] for c in classes])
    pods["req_mem_gb"][e], pods["req_ram_gb"][e] = cm[j], cr[j]
    pods["req_vcpu"][e] = min(0, int(np.min(offers["vcpu"])))  # meets every offer
    c = rng.integers(0, 2, len(e)).astype(np.uint8)
    pods["cloud"][e] = c
    half = np.where(c == 1, 0.5, 1.0)  # community prices are half the secure ones
    pick = rng.integers(0, 4, len(e))
    pods["max_price"][e] = np.choose(pick, [np.full(len(e), np.inf), cp[j] * half, (cp[j] + 0.01) * half,
                                            np.full(len(e), np.nan)])
    return pods


@pytest.mark.parametrize("name", list(EDGE))
def test_segment_edges(eng, name):
    """each edge table at one size per R (4000 rows, then b for R = 2, 4, 8, 16), device calls with top-5: a class
    whose only offer sits at b - 1, b, b + 1 or G - 1 must get exactly that offer; the straddling runs must give the
    lowest index and a top-5 list that crosses the boundary in position order.  Above one k_select_top5 pass, the rows
    whose only offer is the last one walk the whole view."""
    kind, G, _ = EDGE[name]
    offers, classes = edge_table(name)
    S, seg_len = upload(eng, offers, kind, None)
    assert S == {3: 7, 2: 7, 1: 5}[kind] and seg_len == {3: 16_384, 2: 14_336, 1: 4_096}[kind]
    # every class meets its own offers only, and they sit at the intended positions of both views ((price, index) order)
    by_pos = np.lexsort((np.arange(G), offers["secure_price"]))
    assert np.array_equal(by_pos, np.lexsort((np.arange(G), offers["community_price"])))
    for mreq, rreq, pos, idx, _ in classes:
        meets = np.nonzero((offers["mem_gb"] >= mreq) & (offers["ram_gb"] >= rreq))[0]
        assert np.array_equal(meets, np.sort(idx)) and np.array_equal(by_pos[pos], idx), (mreq, rreq, pos)
        assert len(pos) == 1 or (len(set(offers["secure_price"][idx])) == 1 and np.all(np.diff(idx) > 0))
    sms = sc.sm_count()
    for P in [4000] + model.rows_per_warp_bounds(sms):
        pods = edge_pods(offers, classes, P, seed=P)
        wb, wt = sc.expected(offers, pods)
        hit = [int((wb == c[3][0]).sum()) for c in classes]
        assert min(hit) > 0, f"{name} P={P}: an edge class never wins: {hit}"
        R = model.rows_per_warp(P, sms)
        if R == 16:
            assert P > model.top5_rows_per_pass(P, sms)
        sc.check(f"edge {name} P={P} R={R} S={S} device top5", *sc.run_device(eng, pods, True), wb, wt)


# ---- gathers at R = 16 -----------------------------------------------------------------------------------------------
def run_gather(eng, pods, row0, skew, top5_vectors):
    """rpk_select_device_gather (or _top5 with top5_vectors) into 3 vectors at row0: skew 0 gives every vector the
    same 16-byte phase (the push kernel copies the slice), skew 1 starts vector i i elements later, so the select's
    epilogue stores every row into every vector.  Every vector must hold the slice and SENTINEL elsewhere."""
    import torch

    P = sc.nrows(pods)
    d = sc.to_device(pods)
    base = [torch.full((row0 + P + 16,), SENTINEL, dtype=torch.int32, device="cuda") for _ in range(3)]
    vecs = [b[i * skew:] for i, b in enumerate(base)]
    t5base = [torch.full((5 * (row0 + P) + 16,), SENTINEL, dtype=torch.int32, device="cuda") for _ in range(3)]
    t5vecs = [b[i * skew:] for i, b in enumerate(t5base)]
    torch.cuda.synchronize()
    if top5_vectors:
        eng.select_device_gather(d, [v.data_ptr() for v in vecs], row0, top5_ptrs=[v.data_ptr() for v in t5vecs])
    else:
        eng.select_device_gather(d, [v.data_ptr() for v in vecs], row0)
    torch.cuda.synchronize()
    n, n5 = row0 + P + 16 - 2 * skew, 5 * (row0 + P) + 16 - 2 * skew  # the length all three views share
    host = [v.cpu().numpy()[:n] for v in vecs]
    t5host = [v.cpu().numpy()[:n5] for v in t5vecs]
    for i in range(3):
        out = np.r_[host[i][:row0], host[i][row0 + P:]]
        assert (out == SENTINEL).all(), f"best vector {i} written outside [{row0}, {row0 + P})"
        assert np.array_equal(host[i], host[0]), f"best vector {i} differs from vector 0"
        if top5_vectors:
            out = np.r_[t5host[i][:5 * row0], t5host[i][5 * (row0 + P):]]
            assert (out == SENTINEL).all(), f"top5 vector {i} written outside its slice"
            assert np.array_equal(t5host[i], t5host[0]), f"top5 vector {i} differs from vector 0"
        else:
            assert (t5host[i] == SENTINEL).all()
    t5 = t5host[0][5 * row0:5 * (row0 + P)].reshape(P, 5) if top5_vectors else None
    return host[0][row0:row0 + P].copy(), t5


@pytest.mark.parametrize("name", ["pos100k", "packed100k", "wide100k"])
def test_gather_r16(eng, name):
    """at the R = 16 boundary: rpk_select_device_gather with equal and unequal 16-byte phases, and
    rpk_select_device_gather_top5, each at row0 = 1001"""
    offers = table(name)
    upload(eng, offers, TABLES[name][1], None)
    sms = sc.sm_count()
    P = model.rows_per_warp_bounds(sms)[-1]
    assert model.rows_per_warp(P, sms) == 16
    p, wb, wt = rows(name, P)
    for skew in (0, 1):
        got = run_gather(eng, p, 1001, skew, False)
        sc.check(f"{name} gather P={P} skew={skew}", got[0], None, wb, None)
    sc.check(f"{name} gather_top5 P={P}", *run_gather(eng, p, 1001, 0, True), wb, wt)


# ---- one context, every regime ---------------------------------------------------------------------------------------
def test_sequence_every_regime():
    """one context: the three kinds' 100k tables uploaded in turn, and on each device calls of descending then ascending
    P across every R (the tile count changes at every call): tile tickets, done and the group counts must be zero
    again after each call for the next to be right"""
    sms = sc.sm_count()
    b = model.rows_per_warp_bounds(sms)
    down = [P_1M, b[3], b[3] - 1, b[2] - 1, b[1] - 1, b[0] - 1, 3000]
    seq = down + down[::-1][1:]
    with rpk.Engine(1) as e:
        for name in ("wide100k", "pos100k", "packed100k", "wide100k"):
            upload(e, table(name), TABLES[name][1], None)
            for i, P in enumerate(seq):
                p, wb, wt = rows(name, P)
                top5 = i % 3 == 0
                sc.check(f"sequence {name} step {i} P={P} R={model.rows_per_warp(P, sms)}", *sc.run_device(e, p, top5),
                         wb, wt if top5 else None)


# ---- launches after the first -------------------------------------------------------------------------------------------
CHILD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "select_grid_child.py")


def test_capped_grid():
    """RPK_TUNE gridtiles=97 caps the row tiles per launch, so batches of 1000 to 250 000 rows on a 100k-offer table
    span 2 to 33 launches, with tiles that hold rows in each; each kind, every row (select_grid_child.py)"""
    setting = "gridtiles=97"
    env = dict(os.environ, RPK_TUNE=setting)
    env.pop("RPK_FORCE_KERNEL", None)
    out = subprocess.run([sys.executable, CHILD], env=env, capture_output=True, text=True, timeout=600)
    assert out.returncode == 0, out.stdout[-4000:] + out.stderr[-4000:]
    assert out.stdout.strip().splitlines()[-1] == f"ok {setting}"


# ---- grids past 2^31 - 1 CTAs ----------------------------------------------------------------------------------------
G_MAX = 1 << 26
P_HUGE = (2**24 + 2**20 + 37, 2**25 + 2**20)  # 2.28e9 CTAs; 4.43e9, 134 348 800 when wrapped to 32 bits
REAL = 2_100_000  # rows of cloud 0 / 1 per batch, spread over the whole range; the others carry cloud byte 255
GIB = 1 << 30
NEED = int(17.4 * GIB)  # measured on an H100 SXM 80 GB: 16.33 GiB in use at the lowest point, with 1 GiB to spare


def huge_batch(offers, idx, P, seed):
    """P rows, REAL of them scale_pods rows at sorted random positions, the others cloud 255; -> (pods, best)"""
    rng = np.random.default_rng(seed)
    at = np.sort(rng.choice(P, REAL, replace=False))
    real = sm.scale_pods(offers, REAL, seed)
    real["cloud"] = (real["cloud"] & 1).astype(np.uint8)
    pods = {"req_mem_gb": np.zeros(P, np.int32), "req_vcpu": np.zeros(P, np.int32), "req_ram_gb": np.zeros(P, np.int32),
            "max_price": np.zeros(P), "cloud": np.full(P, 255, np.uint8)}
    for k in pods:
        pods[k][at] = real[k]
    best = np.full(P, -1, np.int32)
    best[at] = idx.select(real, want_top5=False)[0]
    return pods, best


def test_grid_past_2_31_ctas():
    """2^26 offers with 3 / 2 / 2 distinct values under RPK_FORCE_KERNEL=generic: S = 16 384 segments of 4096 offers, so
    device selects of 2^24 + 2^20 + 37 and 2^25 + 2^20 rows (R = 16) need 2.28e9 and 4.43e9 CTAs, cut into 2 and 3
    launches.  Every row is checked, then a small select on the same context (the counters of the large grid are
    zero again)."""
    import torch

    free = torch.cuda.mem_get_info()[0]
    if free < NEED:
        pytest.skip(f"needs {NEED} bytes of free device memory; {free} are free")
    t0 = time.time()
    offers = sm.scale_table(G_MAX, 3, 2, 2, seed=31)
    idx = sm.Index(offers)
    sms = sc.sm_count()
    S = model.grid_segments(1, G_MAX)[0]
    low = free
    with rpk.Engine(1) as e:
        upload(e, offers, 1, "generic")
        for i, P in enumerate(P_HUGE):
            R = model.rows_per_warp(P, sms)
            n = len(model.grid_launches(P, R, S))
            assert R == 16 and model.tiles_max(P, R) * S > model.GRID_X_MAX and n == 2 + i
            pods, wb = huge_batch(offers, idx, P, seed=i)
            t1 = time.time()
            got, _ = sc.run_device(e, pods, False)
            low = min(low, torch.cuda.mem_get_info()[0])
            sc.check(f"2^26 offers, P={P} ({n} launches)", got, None, wb, None)
            print(f"\n[grid] 2^26 offers P={P}: {model.tiles_max(P, R) * S} CTAs in {n} launches, "
                  f"select + copies {time.time() - t1:.1f} s")
            del pods, wb, got
        small = sm.scale_pods(offers, 5000, seed=7)
        sb, st5 = idx.select(small)
        sc.check("2^26 offers, 5000 rows after the large grids", *sc.run_device(e, small, True), sb, st5)
        low = min(low, torch.cuda.mem_get_info()[0])
    print(f"[grid] 2^26 offers: {free - low} bytes of device memory in use at the lowest point, "
          f"{time.time() - t0:.1f} s")
