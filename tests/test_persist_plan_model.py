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
    assert model.tune_value("gridtiles=97,pdl=off", "gridtiles=") == 97 and model.tune_value("ipw=4", "gridtiles=") == 0


def test_grid_tiles_cap():
    """gridtiles=97 on 100k synth offers: the last tile with rows lies in a later launch than the first one at every
    size of the capped-grid test (select_grid_child.py), for each kind's row groups"""
    offers = rpk.synth.make_offers(100_000, correlated=True)
    dist = model.distinct(offers)
    pods = rpk.synth.make_pods(50_000)
    for kind in (1, 2, 3):
        counts = model.row_groups(kind, dist, pods)
        assert counts.sum() == (pods["cloud"] <= 1).sum()
        assert (np.nonzero(counts)[0] % 4 == 3).all() if kind == 1 else len(np.nonzero(counts)[0]) > 2
        R = model.rows_per_warp(50_000, 132)
        launches = model.grid_launches(50_000, R, model.grid_segments(kind, 100_000)[0], grid_tiles=97)
        assert len(launches) == 33 and all(n == 97 * model.grid_segments(kind, 100_000)[0] for _, n in launches[:-1])
        assert model.valid_tiles(counts, R) > 97 * 30
    assert model.grid_launches(50_000, 2, 7) == [(0, model.tiles_max(50_000, 2) * 7)]


def test_rows_per_warp_boundaries():
    """R steps at ceil(P / (8 R)) = 12 x SMs row tiles: 25 329 / 50 657 / 101 313 / 202 625 rows with 132 SMs,
    21 873 / 43 745 / 87 489 / 174 977 with 114; the host entry point's 1M-row sub-batches take R = 8, 16, 16, 16"""
    for sm, bounds in ((132, [25_329, 50_657, 101_313, 202_625]), (114, [21_873, 43_745, 87_489, 174_977])):
        assert model.rows_per_warp_bounds(sm) == bounds
        for R, b in zip((2, 4, 8, 16), bounds):
            assert model.rows_per_warp(b - 1, sm) == R // 2 and model.rows_per_warp(b, sm) == R, (sm, b)
        assert [model.rows_per_warp(P, sm) for P in model.host_sub_batches(1_000_000)] == [8, 16, 16, 16]
        assert model.rows_per_warp(1, sm) == 1 and model.rows_per_warp(2**32 // 5, sm) == 16
    assert model.tiles_max(1, 1) == 9 and model.tiles_max(128, 16) == 9 and model.tiles_max(129, 16) == 10


def test_grid_segments():
    """packed_pos: 2^14-offer segments at any G; packed: seg_plan(G, 16 384), 7 x 14 336 at 100k; wide: seg_plan(G,
    4096); every table of a multiple of 4096 offers fills its segments"""
    assert model.grid_segments(3, 16_384) == (1, 16_384) and model.grid_segments(3, 16_385) == (2, 16_384)
    assert model.grid_segments(3, 100_000) == (7, 16_384) and model.grid_segments(3, 0) == (1, 16_384)
    assert model.grid_segments(2, 100_000) == (7, 14_336) and model.grid_segments(2, 16_384) == (1, 16_384)
    assert model.grid_segments(2, 16_385) == (2, 8_320)
    assert model.grid_segments(1, 100_000) == (25, 4_096) and model.grid_segments(1, 20_000) == (5, 4_096)
    assert model.grid_segments(1, 4_097) == (2, 2_176) and model.grid_segments(1, 2**26) == (16_384, 4_096)
    assert model.grid_segments(2, 2**26) == (4_096, 16_384)


def test_grid_launches():
    """2^26 offers in the wide kernel (S = 16 384) at R = 16: 2^24 + 2^20 + 37 rows need 2.28e9 CTAs, more than
    gridDim.x takes; 2^25 + 2^20 rows need 4.43e9, which wraps modulo 2^32 to 134 348 800 (8200 tiles) in 32 bits.
    They take two and three launches of whole tiles; the 1M-row bench step on 100k offers takes one."""
    P1, P2 = 2**24 + 2**20 + 37, 2**25 + 2**20
    S = model.grid_segments(1, 2**26)[0]
    assert model.rows_per_warp(P1, 132) == model.rows_per_warp(P2, 114) == 16
    t1, t2 = model.tiles_max(P1, 16), model.tiles_max(P2, 16)
    assert t1 * S == 2_281_848_832 > model.GRID_X_MAX and (t2 * S) % 2**32 == 134_348_800 == 8200 * S
    per = model.GRID_X_MAX // S
    assert model.grid_launches(P1, 16, S) == [(0, per * S), (per, (t1 - per) * S)]
    assert model.grid_launches(P2, 16, S) == [(0, per * S), (per, per * S), (2 * per, (t2 - 2 * per) * S)]
    assert all(n <= model.GRID_X_MAX for _, n in model.grid_launches(2**32 // 5, 1, S))
    assert sum(n for _, n in model.grid_launches(2**32 // 5, 1, S)) == model.tiles_max(2**32 // 5, 1) * S
    assert model.grid_launches(1_000_000, 16, 7) == [(0, model.tiles_max(1_000_000, 16) * 7)]


def test_top5_rows_per_pass():
    assert model.top5_rows_per_pass(1_000_000, 132) == 33_792 and model.top5_rows_per_pass(1_000_000, 114) == 29_184
    assert model.top5_rows_per_pass(5_003, 132) == 5_008 and model.top5_rows_per_pass(1, 132) == 8
