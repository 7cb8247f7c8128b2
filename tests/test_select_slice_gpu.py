"""GPU parity tests for the persistent select's two table stagings: per mem threshold (bitmapM, the default where the
view exists) and by price (bitmapT, RPK_FORCE_KERNEL=bitmap_price).  Both run every batch size through the persistent
kernel and must give the oracle's assignment vector and top-5 lists on the same inputs (the top-5 kernel reads the
row thresholds the class sort computes)."""
import os

import numpy as np
import pytest

import oracle
import rpk

pytestmark = pytest.mark.gpu


def both_stagings(engine, offers, pods):
    ob, ot = oracle.select(offers, pods, want_top5=True, n_threads=8)
    old = os.environ.pop("RPK_FORCE_KERNEL", None)
    try:
        for force in ("bitmap_grouped", "bitmap_price"):
            os.environ["RPK_FORCE_KERNEL"] = force
            engine.upload_offers(offers)
            assert engine.stats()["select_kernel_kind"] == 4
            best, t5 = engine.select(pods, want_top5=True)
            assert np.array_equal(best, ob), f"[{force}] best differs at rows {np.nonzero(best != ob)[0][:10]}"
            assert np.array_equal(t5, ot), f"[{force}] top5 differs at rows {np.nonzero((t5 != ot).any(axis=1))[0][:10]}"
    finally:
        os.environ.pop("RPK_FORCE_KERNEL", None)
        if old is not None:
            os.environ["RPK_FORCE_KERNEL"] = old
    return ob


@pytest.mark.parametrize("tie_free,ref_exact,with_ext,corr", [
    (False, False, True, False), (False, False, True, True), (True, False, True, False),
    (False, True, False, True), (True, True, True, False)])
def test_c2_flavours(engine, tie_free, ref_exact, with_ext, corr):
    """10k pods x 1k offers: the table is one 64-chunk sub-range, so every row block is final after one walk."""
    offers = rpk.synth.make_offers(1000, tie_free=tie_free, with_ext=with_ext, correlated=corr)
    best = both_stagings(engine, offers, rpk.synth.make_pods(10_000, reference_exact=ref_exact))
    assert len(np.unique(best)) >= 2


@pytest.mark.parametrize("P", [1, 63, 64, 65, 129, 16383, 16384, 16385, 16384 + 65])
def test_ragged_batches(engine, P):
    """Row counts around the 64-row item and the fused kernel's 16k-row limit, on a 20k-offer table (ten sub-ranges:
    row blocks are split over several items and merged)."""
    both_stagings(engine, rpk.synth.make_offers(20_000, correlated=True), rpk.synth.make_pods(P, row0=P))


def test_slice_larger_than_a_stage(engine):
    """300k offers: one mem threshold's slice needs several stages, so a row block is merged across them."""
    offers = rpk.synth.make_offers(300_000, correlated=True)
    best = both_stagings(engine, offers, rpk.synth.make_pods(30_000))
    assert (best >= 0).any() and (best < 0).any()


def test_class_key_without_mem_threshold(engine):
    """30 x 12 x 10 thresholds: the mem threshold does not fit the class key, so the per-mem-threshold view is not
    built and both runs stage by price."""
    G, P = 9000, 20_000
    rng = np.random.default_rng(9)
    offers = rpk.synth.make_offers(G, correlated=True)
    offers["mem_gb"] = (rng.integers(1, 31, G) * 8).astype(np.int32)
    offers["vcpu"] = (rng.integers(1, 13, G) * 4).astype(np.int32)
    offers["ram_gb"] = (rng.integers(1, 11, G) * 16).astype(np.int32)
    pods = rpk.synth.make_pods(P)
    pods["req_mem_gb"] = rng.integers(-8, 260, P).astype(np.int32)
    pods["req_vcpu"] = rng.integers(0, 56, P).astype(np.int32)
    pods["req_ram_gb"] = rng.integers(0, 180, P).astype(np.int32)
    pods["max_price"][:] = 10.0
    best = both_stagings(engine, offers, pods)
    assert (best >= 0).any() and (best < 0).any()


def test_one_mem_threshold(engine):
    """Every pod asks for the same memory: one row group per cloud takes every CTA."""
    offers = rpk.synth.make_offers(50_000, correlated=True)
    pods = rpk.synth.make_pods(40_000)
    pods["req_mem_gb"][:] = 48
    best = both_stagings(engine, offers, pods)
    assert (best >= 0).any()


def test_every_threshold(engine):
    """Pods spread over every (mem, vcpu, ram) threshold of the table, each just below, at and just above an offer
    value, with the price bound out of the way."""
    offers = rpk.synth.make_offers(50_000, correlated=True)
    rng = np.random.default_rng(3)
    P = 60_000

    def around(col):
        v = np.unique(col).astype(np.int64)
        return np.concatenate([v - 1, v, v + 1, [-1, 0]])

    pods = rpk.synth.make_pods(P)
    for req, col in (("req_mem_gb", "mem_gb"), ("req_vcpu", "vcpu"), ("req_ram_gb", "ram_gb")):
        pods[req] = rng.choice(around(offers[col]), P).astype(np.int32)
    pods["max_price"][:] = 1e9
    best = both_stagings(engine, offers, pods)
    assert (best >= 0).any() and (best < 0).any()


def test_community_rows_only(engine):
    """No SECURE rows: only the community cloud's row groups have queues."""
    offers = rpk.synth.make_offers(50_000, correlated=True)
    pods = rpk.synth.make_pods(40_000)
    pods["cloud"][:] = 1
    best = both_stagings(engine, offers, pods)
    assert (best >= 0).any()
