"""GPU parity tests of the persistent select's launch plans (select_persist.cu, persist_plan): the regimes the default
shapes of the other tests never reach.  Each case first asserts through persist_plan_model.py that it reaches the
regime it is named for on this device, then checks every row of best (and top-5) against the oracle, through the host
and the device entry points, and through both table stagings where both exist (RPK_FORCE_KERNEL=bitmap_grouped: per
mem threshold; bitmap_price: by price).

Regimes that only RPK_TUNE can put on a small table run in child processes (select_plan_child.py): RPK_TUNE is read
once per process."""
import os
import subprocess
import sys

import numpy as np
import pytest

import persist_plan_model as model
import select_plan_cases as sc

pytestmark = pytest.mark.gpu
CHILD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "select_plan_child.py")
STAGINGS = ["bitmap_grouped", "bitmap_price"]


BIG = 1_000_000       # rows of the synth batch the 100k-offer cases take their prefixes from
MQ_ROWS = 196_609     # ... and of the many-queue table's batch (test_select_sequences_gpu.py uses the same one)


def batch(name, P):
    """(offers, pods, oracle best, oracle top5): the first P rows of the table's shared batch"""
    pods, wb, wt = sc.batch(name, BIG if name == "synth100k" else MQ_ROWS)
    return sc.table(name), sc.head(pods, P), wb[:P], wt[:P]


def plan_of(name, P, staging):
    offers = sc.table(name)
    dist = model.distinct(offers)
    return model.plan(len(offers["mem_gb"]), P, [len(d) for d in dist], sc.sm_count(), no_slice=staging == "bitmap_price"), dist


def upload(engine, name, staging):
    with sc.forced(staging):
        engine.upload_offers(sc.table(name))
    assert engine.stats()["select_kernel_kind"] == 4


def host_and_device(engine, name, P, label):
    offers, pods, wb, wt = batch(name, P)
    sc.check(f"{label} host", *sc.run_host(engine, pods, True), wb, wt)
    sc.check(f"{label} device", *sc.run_device(engine, pods, True), wb, wt)


@pytest.mark.parametrize("staging", STAGINGS)
def test_more_queues_than_ctas(engine, staging):
    """40 mem sizes x 3 vcpu x 3 ram over 250k offers, pods just below, at and just above every value in both clouds:
    82 row groups x 2 stages = 164 queues per mem-threshold staging, more than one CTA per SM can hold, so CTA b serves
    queues b, b + grid, ... and reloads its stage for each (the price staging of the same table is the control)."""
    P = 150_000
    pl, dist = plan_of("many_queues", P, staging)
    assert [len(d) for d in dist] == [40, 3, 3]
    _, pods, _, _ = batch("many_queues", P)
    if staging == "bitmap_grouped":
        assert pl.slice and pl.S == 2 and model.queues(pl, dist, pods) == 164 > pl.grid
    else:
        assert not pl.slice and model.queues(pl, dist, pods) <= pl.grid
    assert model.host_sub_batches(P) == [P]
    upload(engine, "many_queues", staging)
    host_and_device(engine, "many_queues", P, f"[{staging}] many queues")


def direct_edge():
    """the least batch for which one item spans the whole table (tickets per row block = 1) on the 100k-offer table"""
    return (4 * sc.sm_count() * model.PWARPS - 1) * model.RPI + 1


@pytest.mark.parametrize("staging", STAGINGS)
@pytest.mark.parametrize("rows", ["edge-1", "edge", "1M"])
def test_direct_items_over_sub_ranges(engine, staging, rows):
    """The bench's device step: 1M rows on the 100k-offer synth table, where every item walks all 49 sub-ranges and
    stores its rows at once, and the two batch sizes on either side of the point where direct items begin
    (540 608 / 540 609 rows on 132 SMs).  Staged by price the table takes two stages and is never direct."""
    P = {"edge-1": direct_edge() - 1, "edge": direct_edge(), "1M": 1_000_000}[rows]
    pl, _ = plan_of("synth100k", P, staging)
    assert pl.nsub == 49
    if staging == "bitmap_grouped":
        assert pl.slice and pl.S == 1 and pl.direct == (rows != "edge-1")
        if rows == "edge-1":
            assert pl.tickets_per_block == 2
    else:
        assert not pl.slice and (pl.S, pl.per) == (2, 25) and not pl.direct
    offers, pods, wb, wt = batch("synth100k", P)
    upload(engine, "synth100k", staging)
    sc.check(f"[{staging}] {P} rows device", *sc.run_device(engine, pods, rows == "edge"), wb, wt)


@pytest.mark.parametrize("name,staging", [("classes4096", "bitmap_grouped"), ("classes4096", "bitmap_price"),
                                          ("classes4224", "bitmap_grouped")])
def test_class_key_limit(engine, name, staging):
    """31 / 7 / 7 distinct values: 2 x 32 x 8 x 8 = 4096 classes, exactly the class key's limit, with the mem threshold
    in the key and stages per mem threshold; 32 / 7 / 7: 4224, just past it, so the key drops the mem threshold and
    even the forced per-mem-threshold run stages by price."""
    P = 40_000
    pl, dist = plan_of(name, P, staging)
    D = [len(d) for d in dist]
    if name == "classes4096":
        assert D == [31, 7, 7] and pl.classes == model.MAX_CLASSES and pl.slice == (staging == "bitmap_grouped")
    else:
        assert D == [32, 7, 7] and 2 * 33 * 8 * 8 > model.MAX_CLASSES and pl.classes == 2 * 8 * 8 and not pl.slice
    upload(engine, name, staging)
    host_and_device(engine, name, P, f"[{staging}] {name}")


@pytest.mark.parametrize("P", [16_385, 200_000])
def test_unknown_cloud_only(engine, P):
    """Every row carries a cloud byte that is neither SECURE nor COMMUNITY: the scatter kernel finalises every row, the
    grid kernel has no queue at all, and with three output vectors the scatter kernel's own row count must release
    the push."""
    offers = sc.table("synth20k")
    pods = sc.pods_for("synth20k", P, seed=5)
    pods["cloud"] = np.array([2, 7, 255], np.uint8)[np.arange(P) % 3]
    dist = model.distinct(offers)
    pl = model.plan(len(offers["mem_gb"]), P, [len(d) for d in dist], sc.sm_count())
    assert model.persistent(P) and model.queues(pl, dist, pods) == 0
    wb, wt = sc.expected(offers, pods)
    assert (wb == -1).all()
    with sc.forced(None):
        engine.upload_offers(offers)
    sc.check(f"unknown cloud, {P} rows host", *sc.run_host(engine, pods, True), wb, wt)
    sc.check(f"unknown cloud, {P} rows device", *sc.run_device(engine, pods, True), wb, wt)
    sc.check(f"unknown cloud, {P} rows gather", *sc.run_gather(engine, pods, True, row0=13), wb, wt)


@pytest.mark.parametrize("P,n_sub", [(196_607, 1), (196_609, 2), (1_000_000, 4)])
def test_host_top5_over_sub_batches(engine, P, n_sub):
    """The host entry point cuts a batch into row sub-batches on up to four lanes, each with its own top-5 buffer
    copied back at row b0 x 5: one sub-batch just below the split, a ragged second one just above it, and all four
    lanes at 1M rows."""
    assert len(model.host_sub_batches(P)) == n_sub
    offers, pods, wb, wt = batch("synth100k", P)
    with sc.forced(None):
        engine.upload_offers(offers)
    sc.check(f"host top-5, {P} rows", *sc.run_host(engine, pods, True), wb, wt)


@pytest.mark.parametrize("setting", ["stagekb=4", "stagekb=1", "ipw=64", "ipw=1", "k0ctas=1", "k0ctas=3", "pdl=off"])
def test_tuned_plan(setting):
    """plans only RPK_TUNE reaches on a small table, one child process per setting (select_plan_child.py)"""
    env = dict(os.environ, RPK_TUNE=setting)
    env.pop("RPK_FORCE_KERNEL", None)
    out = subprocess.run([sys.executable, CHILD], env=env, capture_output=True, text=True, timeout=600)
    assert out.returncode == 0, out.stdout[-4000:] + out.stderr[-4000:]
    assert out.stdout.strip().splitlines()[-1] == f"ok {setting}"
