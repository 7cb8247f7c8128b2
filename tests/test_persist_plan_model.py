"""CPU tests of persist_plan_model.py: the restated plan gives the figures DESIGN §4 states for the bench table, and
the boundaries the GPU plan tests are built around."""
import numpy as np

import persist_plan_model as model
import rpk


def synth_d(G):
    return [len(d) for d in model.distinct(rpk.synth.make_offers(G, correlated=True))]


def test_bench_table_figures():
    """G = 100k: 49 sub-ranges; per mem threshold one 186 KB stage of (7 + 7) rows x 272 B x 49; by price two stages
    of 25 and 24 sub-ranges; 2 x 14 x 7 x 7 = 1372 classes"""
    D = synth_d(100_000)
    assert D == [13, 6, 6]
    pl = model.plan(100_000, 1_000_000, D, 132)
    assert pl.nsub == 49 and pl.slice and (pl.S, pl.per) == (1, 49)
    assert pl.smem_bytes == 14 * 272 * 49 == 186_592 and pl.classes == 1372
    assert pl.direct  # the bench's 1M-row device step
    pr = model.plan(100_000, 1_000_000, D, 132, no_slice=True)
    assert not pr.slice and (pr.S, pr.per) == (2, 25) and pr.nsub - pr.per == 24 and not pr.direct


def test_direct_items_boundary():
    """direct items need one item per row block: nblk >= 4 items x 132 SMs x 16 warps, i.e. more than 540 608 rows"""
    D = synth_d(100_000)
    below, at = (model.plan(100_000, P, D, 132) for P in (540_608, 540_609))
    assert not below.direct and below.tickets_per_block == 2 and at.direct
    assert not model.plan(100_000, 540_609, D, 132, items_per_warp=8).direct
    assert model.plan(100_000, 135_105, D, 132, items_per_warp=1).direct
    assert not model.plan(100_000, 135_104, D, 132, items_per_warp=1).direct


def test_tuned_stages():
    """stagekb=4: one sub-range per slice stage (1372 queues at most, 588 with synth pods); stagekb=1: price stages of
    one sub-range (148 queues at G = 150k); ipw=64: qspan 1"""
    D = synth_d(100_000)
    pl = model.plan(100_000, 40_000, D, 132, stage_kb=4)
    assert pl.slice and (pl.S, pl.per) == (49, 1) and 2 * pl.groups_per_cloud * pl.S == 1372
    pods = rpk.synth.make_pods(40_000)
    assert model.queues(pl, model.distinct(rpk.synth.make_offers(100_000, correlated=True)), pods) == 588
    pl = model.plan(150_000, 40_000, synth_d(150_000), 132, stage_kb=1)
    assert not pl.slice and (pl.S, pl.per) == (74, 1) and model.queues(pl, None, pods) == 148
    pl = model.plan(20_000, 40_000, synth_d(20_000), 132, items_per_warp=64)
    assert pl.qspan == 1 and pl.tickets_per_block == pl.nsub == 10


def test_class_key_limit():
    """2 x 32 x 8 x 8 = 4096 classes keep the mem threshold in the key; one more mem value drops it"""
    assert model.class_dims([31, 7, 7])[3:] == (True, 4096)
    assert model.class_dims([32, 7, 7])[3:] == (False, 128)
    assert model.plan(20_000, 40_000, [31, 7, 7], 132).slice
    assert not model.plan(20_000, 40_000, [32, 7, 7], 132).slice


def test_many_queue_table():
    """40 / 3 / 3 distinct values at 250k offers: 82 row groups x 2 stages = 164 queues, more than 132 CTAs"""
    pl = model.plan(250_000, 150_000, [40, 3, 3], 132)
    assert pl.slice and pl.S == 2 and 2 * pl.groups_per_cloud * pl.S == 164


def test_host_sub_batches():
    assert model.host_sub_batches(196_607) == [196_607]
    assert model.host_sub_batches(196_609) == [131_072, 65_537]
    assert model.host_sub_batches(1_000_000) == [131_072, 262_144, 393_216, 213_568]
    assert sum(model.host_sub_batches(12_345_678)) == 12_345_678


def test_unknown_cloud_has_no_queue():
    pods = rpk.synth.make_pods(1000)
    pods["cloud"][:] = 2
    pl = model.plan(20_000, 1000, [13, 6, 6], 132)
    assert model.queues(pl, [np.arange(13)] * 3, pods) == 0


def test_tune_parsing():
    assert model.tune_from_env("stagekb=4") == (4, 0, 0)
    assert model.tune_from_env("pdl=off,ipw=64,k0ctas=3") == (0, 64, 3)
