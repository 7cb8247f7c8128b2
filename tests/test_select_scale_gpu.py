"""GPU tests of the select at the sizes the API accepts: persistent-select CTAs that load dozens of stages in one call,
the 2^26-offer table limit, and one batch past 2^24 rows.  Results are checked against select_scale_model.py, an exact
restatement that stays cheap at these sizes (tests/test_select_scale_model.py holds it to oracle.select), and a few
rows of each table against the oracle itself.

Each case asserts through persist_plan_model.py the regime it is named for on this device (queues, stages each CTA
loads, copy groups of the last stage), fills its outputs with SENTINEL a few words past P, and checks every row of
best (and of top-5 where asked) and that nothing was written past P.  Each runs on a context of its own, closed
before the next case, and skips with the bytes it needs when the device does not have them free (other processes
may share it)."""
import functools
import time

import numpy as np
import pytest

import oracle
import persist_plan_model as model
import rpk
import select_plan_cases as sc
import select_scale_model as sm

pytestmark = pytest.mark.gpu
PAD = 37  # outputs run this many words past P, and must keep SENTINEL there
# free device memory each case needs: its use measured on an H100 SXM 80 GB (free memory before its context is created
# less free memory after its last select: 2.37 GB for the 4M-offer reload tables, 15.3 GB at 2^26 offers, 2.36 GB for
# the 17.8M-row batch), with 1 GiB to spare
GIB = 1 << 30
NEED = {"reload": int(3.3 * GIB), "limit": int(15.3 * GIB), "rows": int(3.3 * GIB)}


@pytest.fixture
def ctx(request):
    """a context of the case's own, after a check that the device has the memory the case needs"""
    import torch

    case = request.node.originalname.split("_")[1]
    free = torch.cuda.mem_get_info()[0]
    if free < NEED[case]:
        pytest.skip(f"{request.node.name} needs {NEED[case]} bytes of free device memory; {free} are free")
    t0 = time.time()
    eng = rpk.Engine(1)
    yield eng
    low = torch.cuda.mem_get_info()[0]
    eng.close()
    print(f"\n[scale] {request.node.name}: {free - low} bytes of device memory in use at the end, "
          f"{time.time() - t0:.1f} s")


# ---- entry points with outputs past P ---------------------------------------------------------------------------------
def run_host(eng, pods, top5):
    P = sc.nrows(pods)
    best = np.full(P + PAD, sc.SENTINEL, np.int32)
    t5 = np.full((P + PAD, 5), sc.SENTINEL, np.int32)
    eng.select(pods, want_top5=top5, out_best=best[:P], out_top5=t5[:P] if top5 else None)
    return past(best, t5, P, top5)


def run_device(eng, pods, top5):
    import torch

    P = sc.nrows(pods)
    d = sc.to_device(pods)
    d_best = torch.full((P + PAD,), sc.SENTINEL, dtype=torch.int32, device="cuda")
    d_t5 = torch.full(((P + PAD) * 5,), sc.SENTINEL, dtype=torch.int32, device="cuda")
    torch.cuda.synchronize()
    eng.select_device(d, d_best[:P], d_t5[:P * 5] if top5 else None)
    torch.cuda.synchronize()
    del d
    return past(d_best.cpu().numpy(), d_t5.cpu().numpy().reshape(P + PAD, 5), P, top5)


def past(best, t5, P, top5):
    assert (best[P:] == sc.SENTINEL).all(), "best was written past P"
    assert (t5[P:] == sc.SENTINEL).all() and (top5 or (t5 == sc.SENTINEL).all()), "top5 was written past P"
    return best[:P], t5[:P] if top5 else None


def check(label, got, want):
    sc.check(label, got[0], got[1], want[0], want[1])


def spot_check(offers, pods, want, rows):
    """the reference's lists for `rows` equal oracle.get_gpu_types (one O(G) scan each)"""
    for r in rows:
        r = int(r)
        got = oracle.get_gpu_types(offers, int(pods["req_mem_gb"][r]), float(pods["max_price"][r]), int(pods["cloud"][r]),
                                   int(pods["req_vcpu"][r]), int(pods["req_ram_gb"][r]))
        assert got + [-1] * (5 - len(got)) == want[1][r].tolist(), f"row {r}: oracle {got}, model {want[1][r].tolist()}"


def spot_rows(pods, idx, k=8):
    """k rows of different classes: both clouds at the top of the class grid (few offers), an unknown cloud byte, a
    NaN bound, and rows whose bound is a price of the table"""
    mp, cloud = pods["max_price"], pods["cloud"]
    th = np.stack(idx.thresholds(pods), 1)
    tops = np.nonzero((th == th.max(axis=0)).sum(axis=1) >= 2)[0]
    rows = [tops[cloud[tops] == 0][:1], tops[cloud[tops] == 1][:1], np.nonzero(cloud > 1)[0][:1],
            np.nonzero(np.isnan(mp))[0][:1]]
    priced = np.nonzero(np.isfinite(mp) & (mp > 0) & (mp < 1e9) & (mp != sm.DEFAULT_MAX_PRICE))[0]
    rows.append(priced[np.argsort(mp[priced], kind="stable")][:: max(len(priced) // (k - 4), 1)][: k - 4])
    return np.concatenate(rows)


# ---- stage reloads: more (row group, stage) queues than CTAs -----------------------------------------------------------
D_RELOAD = (20, 1, 39)  # 2 x 21 x 2 x 40 = 3360 classes: staged per mem threshold, 42 slice rows, 19 sub-ranges a stage
RELOAD_G = {"1M": 977_944,       # 478 sub-ranges: 26 stages of 19, the last of 3 (3 copy groups against 7)
            "1M-even": 1_011_707,  # 494 = 26 x 19: every stage full
            "4M": 3_978_487}     # 1943 sub-ranges: 103 stages, the last of 5; over 30 stages per CTA
RELOAD_P = 1_000_000


@functools.lru_cache(maxsize=None)
def reload_case(name):
    """(offers, pods, reference (best, top5)) of a reload table"""
    offers = sm.scale_table(RELOAD_G[name], *D_RELOAD, seed=RELOAD_G[name])
    pods = sm.scale_pods(offers, RELOAD_P, seed=RELOAD_G[name] + 1)
    idx = sm.Index(offers)
    want = idx.select(pods)
    spot_check(offers, pods, want, spot_rows(pods, idx))
    return offers, pods, want


@pytest.mark.parametrize("staging", [None, "bitmap_price"])
@pytest.mark.parametrize("G", list(RELOAD_G))
def test_reload_stages(ctx, G, staging):
    """1M rows over ~1M and ~4M offers with 20 / 1 / 39 distinct values: staged per mem threshold, 42 row groups x
    26 or 103 stages are more queues than CTAs, so each CTA loads 9-10 or 33-38 stages one after the other, and the
    last stage of a queue row takes fewer copy groups than the full ones (except on the even table).  Staged by price
    (RPK_FORCE_KERNEL=bitmap_price) the same tables are (cloud, stage) queues of bitmapT stages, 3 per CTA at 4M.
    Host entry point with top-5, device entry point with and without."""
    offers, pods, want = reload_case(G)
    Gn, D = len(offers["mem_gb"]), [len(d) for d in model.distinct(offers)]
    assert D == list(D_RELOAD)
    pl = model.plan(Gn, RELOAD_P, D, sc.sm_count(), no_slice=staging == "bitmap_price")
    nq = model.queues(pl, model.distinct(offers), pods)
    its = model.iterations_per_cta(pl, nq)
    last, full = model.copy_groups(pl, pl.S - 1), model.copy_groups(pl, 0)
    print(f"\n[scale] G={Gn} {staging}: slice={pl.slice} S={pl.S} per={pl.per} nsub={pl.nsub} queues={nq} "
          f"grid={pl.grid} stages per CTA={its} copy groups {full} full / {last} last")
    if staging is None:
        assert pl.slice and pl.per == 19 and nq == 42 * pl.S > pl.grid
        assert its >= (30 if G == "4M" else 8)
        if G == "1M-even":
            assert pl.nsub % pl.per == 0 and last == full
        else:
            assert pl.nsub % pl.per != 0 and last < full < 8
    else:
        assert not pl.slice and nq == 2 * pl.S
        assert (nq > pl.grid) == (G == "4M")
    with sc.forced(staging):
        ctx.upload_offers(offers)
    assert ctx.stats()["select_kernel_kind"] == 4
    check(f"[{staging}] G={Gn} host top-5", run_host(ctx, pods, True), want)
    check(f"[{staging}] G={Gn} device", run_device(ctx, pods, False), want)
    check(f"[{staging}] G={Gn} device top-5", run_device(ctx, pods, True), want)


# ---- the table limit: 2^26 offers --------------------------------------------------------------------------------------
G_MAX = 1 << 26
D_LIMIT = (3, 2, 2)


def test_limit_offers(ctx):
    """2^26 offers with 3 / 2 / 2 distinct values (the ingest sorts n = 2^27 keys; k_unique and the slice build run
    over the whole table): 2^26 + 1 is refused with RPK_EINVAL; the fused kernel (16 000 rows, top-5) and the
    persistent kernel (200 000 rows, and 1M with top-5: 238 stages of 138 sub-ranges, 8 row groups, 15-17 stages per
    CTA) walk all 2M chunks.  Then a small table replaces it and its selects must see nothing of the large views."""
    t0 = time.time()
    big = sm.scale_table(G_MAX + 1, *D_LIMIT, seed=26)
    with pytest.raises(rpk.RpkError) as ei:
        ctx.upload_offers(big)
    assert ei.value.code == rpk._ffi.RPK_EINVAL and "2^26" in str(ei.value)
    offers = {k: v[:G_MAX] for k, v in big.items()}
    del big
    idx = sm.Index(offers)
    pods = sm.scale_pods(offers, 1_000_000, seed=27)
    want = idx.select(pods)
    spot_check(offers, pods, want, spot_rows(pods, idx))
    print(f"\n[scale] 2^26 offers: table, reference and spot checks {time.time() - t0:.1f} s")
    D = [len(d) for d in idx.dist]
    assert D == list(D_LIMIT)
    for P in (200_000, 1_000_000):
        pl = model.plan(G_MAX, P, D, sc.sm_count())
        nq = model.queues(pl, idx.dist, sc.head(pods, P))
        its = model.iterations_per_cta(pl, nq)
        print(f"[scale] 2^26 offers, P={P}: S={pl.S} per={pl.per} queues={nq} stages per CTA={its} "
              f"copy groups {model.copy_groups(pl, 0)} full / {model.copy_groups(pl, pl.S - 1)} last")
        assert pl.slice and pl.S >= 200 and nq == 8 * pl.S and its >= 14
    assert not model.persistent(16_000) and model.persistent(200_000)
    ctx.upload_offers(offers)
    st = ctx.stats()
    assert st["select_kernel_kind"] == 4 and [st["distinct_mem"], st["distinct_vcpu"], st["distinct_ram"]] == D
    head = lambda P: (sc.head(pods, P), (want[0][:P], want[1][:P]))  # noqa: E731
    p16, w16 = head(16_000)
    check("2^26 offers, 16 000 rows host top-5", run_host(ctx, p16, True), w16)
    check("2^26 offers, 16 000 rows device top-5", run_device(ctx, p16, True), w16)
    p200, w200 = head(200_000)
    check("2^26 offers, 200 000 rows device", run_device(ctx, p200, False), w200)
    check("2^26 offers, 1M rows device top-5", run_device(ctx, pods, True), want)
    del offers, idx
    small = rpk.synth.make_offers(20_000, correlated=True)
    spods = rpk.synth.make_pods(200_000, seed=9)
    swant = sm.select(small, spods)
    ctx.upload_offers(small)
    check("small table after 2^26 offers, host top-5", run_host(ctx, spods, True), swant)
    check("small table after 2^26 offers, device 16 000 rows top-5",
          run_device(ctx, sc.head(spods, 16_000), True), (swant[0][:16_000], swant[1][:16_000]))


# ---- rows past 2^24 ------------------------------------------------------------------------------------------------------
P_BIG = 2**24 + 2**20 + 37


def test_rows_past_2_24(ctx):
    """the bench table (100 000 synth offers) and 2^24 + 2^20 + 37 synth rows: one device select over all of them (K0
    over 4 CTAs per SM, class totals, ord_rw and pos past 2^24 rows), then the host entry point, which cuts the batch
    into row sub-batches; every row against the reference, 20 000 sampled rows against the oracle"""
    offers = rpk.synth.make_offers(100_000, correlated=True)
    pods = rpk.synth.make_pods(P_BIG, seed=24)
    want = sm.select(offers, pods)
    rng = np.random.default_rng(24)
    sample = np.sort(rng.choice(P_BIG, 20_000, replace=False))
    spods = {k: v[sample] for k, v in pods.items()}
    ob, ot = sc.expected(offers, spods)
    assert np.array_equal(ob, want[0][sample]) and np.array_equal(ot, want[1][sample]), "reference != oracle"
    dist = model.distinct(offers)
    pl = model.plan(100_000, P_BIG, [len(d) for d in dist], sc.sm_count())
    assert model.persistent(P_BIG) and pl.k0_blocks == 4 * sc.sm_count() and 5 * P_BIG < 2**32
    subs = model.host_sub_batches(P_BIG)
    print(f"\n[scale] P={P_BIG}: queues={model.queues(pl, dist, pods)} K0 CTAs={pl.k0_blocks} "
          f"host sub-batches={len(subs)} of at most {max(subs)} rows")
    assert sum(subs) == P_BIG and len(subs) == 36 and max(subs) < 2**24
    ctx.upload_offers(offers)
    got = run_device(ctx, pods, True)
    check(f"{P_BIG} rows device top-5 (sampled rows)", (got[0][sample], got[1][sample]), (ob, ot))
    check(f"{P_BIG} rows device top-5", got, want)
    del got
    check(f"{P_BIG} rows host", run_host(ctx, pods, False), want)
