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


def test_layout_packed_boundaries():
    """field widths bitlen(D0 + 1), bitlen(D1), bitlen(D2) plus three guards: 18 bits keep the position field, 19 drop
    it, 32 are packed, 33 generic; each field steps where its highest threshold (D0 + 1 for mem, D for vcpu / ram)
    needs one more bit.  Every case has more than 64 mask words, so packed is the automatic choice."""
    cases = {  # D: (kind, packed_bits)
        (62, 15, 31): (3, 18),   # 6 + 4 + 5 + 3
        (63, 15, 31): (2, 19),   # mem threshold 64: 7 bits
        (62, 16, 31): (2, 19),   # vcpu threshold 16: 5 bits
        (62, 15, 32): (2, 19),   # ram threshold 32: 6 bits
        (64, 15, 31): (2, 19),
        (61, 15, 31): (3, 18),
        (30, 63, 7): (3, 17),
        (30, 64, 7): (3, 18),
        (14, 7, 127): (3, 17),
        (14, 7, 128): (3, 18),
        (1022, 1023, 511): (2, 32),  # 10 + 10 + 9 + 3
        (1023, 1023, 511): (1, 0),   # mem threshold 1024: 11 bits
        (1022, 1024, 511): (1, 0),
        (1022, 1023, 512): (1, 0),
        (1021, 1023, 511): (2, 32),
    }
    for D, (kind, bits) in cases.items():
        L = model.layout(list(D))
        assert sum(D) + 3 > model.BM_MAX_STRIDE and L.bm_words == 0 and L.bm_stride == 0, D
        assert (L.kind, L.packed_bits) == (kind, bits), (D, L)
        assert L.pos_bits == (model.POS_BITS if kind == 3 else 0), D


def test_layout_bitmap_boundaries():
    """mask words (D0 + 1) + (D1 + 1) + (D2 + 1): rows of 32 words up to 32, 64 up to 64, no bit-sliced view at 65;
    per-mem-threshold slices while 2 * Dm1 * Dv1 * Dr1 <= 4096"""
    L = model.layout([15, 7, 7])
    assert (L.kind, L.bm_words, L.bm_stride, L.slice, L.packed_bits, L.pos_bits) == (4, 32, 32, True, 14, 14)
    L = model.layout([16, 7, 7])
    assert (L.kind, L.bm_words, L.bm_stride, L.slice) == (4, 33, 64, True)
    L = model.layout([47, 7, 7])
    assert (L.kind, L.bm_words, L.bm_stride, L.slice) == (4, 64, 64, False)
    L = model.layout([48, 7, 7])
    assert (L.kind, L.bm_words, L.bm_stride, L.packed_bits) == (3, 0, 0, 6 + 3 + 3 + 3)
    assert model.layout([31, 7, 7]).slice and not model.layout([32, 7, 7]).slice
    assert model.layout([0, 0, 0]).kind == 4 and not model.layout([0, 0, 0]).slice  # empty table: no sub-range


def test_layout_forced():
    """RPK_FORCE_KERNEL removes views, never adds one: packed_pos drops the bit-sliced view, packed also the position,
    generic every rank view; bitmap_grouped / bitmap_price keep the views and route every batch through the
    persistent kernel (bitmap_price without the slices); an unknown value is the automatic choice"""
    bm, pos, packed, generic = [15, 7, 7], [62, 15, 31], [63, 15, 31], [1022, 1023, 512]
    want = {  # (D, force): kind
        (0, None): 4, (0, "packed_pos"): 3, (0, "packed"): 2, (0, "generic"): 1, (0, "bitmap"): 4,
        (0, "bitmap_grouped"): 4, (0, "bitmap_price"): 4, (0, "no-such-kernel"): 4,
        (1, None): 3, (1, "packed_pos"): 3, (1, "packed"): 2, (1, "generic"): 1, (1, "bitmap_grouped"): 3,
        (2, None): 2, (2, "packed_pos"): 2, (2, "packed"): 2, (2, "generic"): 1,
        (3, None): 1, (3, "packed_pos"): 1, (3, "packed"): 1, (3, "bitmap"): 1,
    }
    tables = [bm, pos, packed, generic]
    for (t, force), kind in want.items():
        assert model.layout(tables[t], force).kind == kind, (tables[t], force)
    assert model.layout(bm, "packed").packed_bits == 14 and model.layout(bm, "packed").pos_bits == 0
    assert model.layout(bm, "generic").packed_bits == 0
    g, p = model.layout(bm, "bitmap_grouped"), model.layout(bm, "bitmap_price")
    assert g.no_fused and not g.no_slice and p.no_fused and p.no_slice and g.slice and p.slice
    assert not model.layout(bm, "bitmap").no_fused


def test_tune_parsing():
    assert model.tune_from_env("stagekb=4") == (4, 0, 0)
    assert model.tune_from_env("pdl=off,ipw=64,k0ctas=3") == (0, 64, 3)
