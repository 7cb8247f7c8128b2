"""GPU parity tests for the status sweep diff (K2) through the C-ABI against the oracle."""
import json
import os

import numpy as np
import pytest

import np_restatement as npr
import oracle
import rpk
import status_cases as sc

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def make_engine():
    return rpk.Engine(1)


def changed_rows(a, b):
    """rows whose compared fields differ (the flag bit of byte 0 is not one of them)"""
    ma, mb = a.copy(), b.copy()
    ma[:, 0] &= 0x7F
    mb[:, 0] &= 0x7F
    return np.nonzero((ma != mb).any(axis=1))[0].astype(np.uint32)


def test_device_xxh64_matches_golden_vectors():
    """The committed slot-prefix XXH64 vectors (python-xxhash; every len 0..127, 1..16 lanes incl. the 32-byte stripes)
    through the hash column of every kernel that can hold them, with and without the unhashed flag bit."""
    g = json.load(open(os.path.join(GOLD, "xxh64_kat.json")))
    for stride in (16, 32, 48, 64, 128, 256):
        vecs = [v for v in g["slot_vectors"] if v["len"] <= min(stride - 1, 127)]
        recs = np.zeros((len(vecs), stride), np.uint8)
        for i, v in enumerate(vecs):
            d = np.frombuffer(bytes.fromhex(v["hex"]), np.uint8)
            recs[i, : len(d)] = d[:stride]
        recs[1::2, 0] |= 0x80
        eng = make_engine()
        idx, hashes = eng.status_diff(recs, want_hashes=True)
        eng.close()
        for i, v in enumerate(vecs):
            assert format(int(hashes[i]), "016x") == v["xxh64"], (stride, v["len"])
        assert len(idx) == len(vecs)


@pytest.mark.parametrize("stride", [16, 32, 48, 64, 128, 256])
def test_hash_column_all_lengths(stride):
    rng = np.random.default_rng(stride)
    N = 3000
    recs = rng.integers(0, 256, (N, stride), dtype=np.uint8)
    recs[:, 0] = rng.integers(0, min(stride, 128), N)  # len in [0, min(stride-1, 127)]
    recs[: min(stride, 128), 0] = np.arange(min(stride, 128))
    recs[::3, 0] |= 0x80                               # flag bit: never hashed
    eng = make_engine()
    _, hashes = eng.status_diff(recs, want_hashes=True)
    eng.close()
    assert np.array_equal(hashes, oracle.record_hashes(recs))


@pytest.mark.parametrize("stride", [16, 32, 64])
@pytest.mark.parametrize("N", [1, 63, 64, 65, 255, 1024, 1025, 100_000])
def test_sweeps_match_reference_predicate(N, stride):
    """BASELINE config 3's reconcile: N tracked pods, sweeps with f = 0, 1 %, 10 %, 100 % mutation; the
    changed list must equal the reference's string/bool predicate (oracle) exactly, in ascending order, and the
    code emitted next to each changed slot must equal translateRunPodStatus (kubelet.go:1848-2024) of its record."""
    eng = make_engine()
    tab = oracle.StatusTable(N, stride)
    for sweep, frac in enumerate([0.0, 0.0, 0.01, 0.10, 1.0, 0.0]):
        recs = rpk.synth.make_status_records(N, sweep=sweep, mutate_frac=frac, stride=stride)
        got, codes, hashes = eng.status_diff(recs, want_hashes=True, want_codes=True)
        want = tab.diff(recs)
        assert np.array_equal(got, want), (N, sweep, len(got), len(want))
        assert np.array_equal(hashes, oracle.record_hashes(recs))
        assert np.array_equal(codes, oracle.record_codes(recs)[want]), (N, sweep)
        if sweep == 0:
            assert len(got) == N
        if sweep == 1:
            assert len(got) == 0
    eng.close()


def test_hash_column_large_tables():
    """Enough slots that every persistent CTA walks many tiles through both bulk-copy stages: heavy repetition
    of a small pool, fully random rows, and near-duplicates that differ only in one late byte."""
    N = 1_200_000
    rng = np.random.default_rng(21)
    pool = rng.integers(0, 256, (50, 32), dtype=np.uint8)
    pool[:, 0] = rng.integers(0, 32, 50) | (rng.integers(0, 2, 50) << 7)
    recs = pool[rng.integers(0, 50, N)]
    rnd = rng.random(N) < 0.2
    recs[rnd] = rng.integers(0, 256, (int(rnd.sum()), 32), dtype=np.uint8)
    near = rng.random(N) < 0.1
    recs[near, 31] ^= rng.integers(1, 256, int(near.sum())).astype(np.uint8)   # same head, different tail byte
    recs[:, 0] = np.minimum(recs[:, 0] & 0x7F, 31) | (recs[:, 0] & 0x80)
    recs = np.ascontiguousarray(recs)
    eng = make_engine()
    idx, hashes = eng.status_diff(recs, want_hashes=True)
    assert np.array_equal(hashes, oracle.record_hashes(recs))
    assert len(idx) == N
    recs2 = recs.copy()
    rows = rng.choice(N, 5000, replace=False)
    recs2[rows, 5] ^= 0x40
    idx2, hashes2 = eng.status_diff(recs2, want_hashes=True)
    assert np.array_equal(hashes2, oracle.record_hashes(recs2))
    want = np.sort(rows).astype(np.uint32)   # byte 5 of the slot is inside the first 8-byte lane: always hashed
    assert np.array_equal(idx2, want)
    eng.close()


def test_seed_reset_and_resize():
    N = 5000
    eng = make_engine()
    base = rpk.synth.make_status_records(N, 0)
    eng.status_seed(base)  # CreatePod / LoadRunning: fill state, report nothing
    got, _ = eng.status_diff(base)
    assert len(got) == 0
    nxt = rpk.synth.make_status_records(N, 3, 0.2)
    got, _ = eng.status_diff(nxt)
    want = changed_rows(base, nxt)
    assert np.array_equal(got, want)
    # per-slot seed (CreatePod writes ONE InstanceInfo): those slots stop reporting, nothing else is absorbed
    third = rpk.synth.make_status_records(N, 4, 0.3)
    moved = changed_rows(nxt, third)
    assert len(moved) > 100
    quiet = moved[::3]
    eng.status_seed_slots(quiet, np.ascontiguousarray(third[quiet]))
    got, _ = eng.status_diff(third)
    assert np.array_equal(got, np.setdiff1d(moved, quiet).astype(np.uint32))
    eng.status_seed_slots(np.array([7], np.uint32), np.ascontiguousarray(nxt[7:8]))  # slot 7 now "was" something else
    got, _ = eng.status_diff(third)
    assert got.tolist() == ([7] if (nxt[7, :] & np.r_[0x7F, [0xFF] * 31].astype(np.uint8) != third[7, :] & np.r_[0x7F, [0xFF] * 31].astype(np.uint8)).any() else [])
    nxt = third
    with pytest.raises(rpk.RpkError) as ei:
        eng.status_diff(nxt[:100].copy())
    assert ei.value.code == rpk._ffi.RPK_ESTATE
    eng.status_reset(100)
    got, _ = eng.status_diff(nxt[:100].copy())
    assert np.array_equal(got, np.arange(100, dtype=np.uint32))
    with pytest.raises(rpk.RpkError):
        eng.status_diff(np.zeros((4, 20), np.uint8))  # stride not a multiple of 16
    eng.close()


@pytest.mark.parametrize("stride", [32, 16])
@pytest.mark.parametrize("N", [1 << 22, (1 << 22) + 37])
def test_large_sweep_ordering_and_count(N, stride):
    """4M slots (the big-table build: per-warp rings of bulk-copied units; the ragged last unit is loaded the plain
    way): the single-pass look-back scan must emit every changed slot exactly once, ascending, with its code, and
    the hash column must be the reference hash of every record."""
    eng = make_engine()
    base = rpk.synth.make_status_records(N, 0, stride=stride)
    eng.status_seed(base)
    nxt = rpk.synth.make_status_records(N, 2, 0.37, stride=stride)
    got, codes, hashes = eng.status_diff(nxt, want_codes=True, want_hashes=True)
    want = changed_rows(base, nxt)
    assert np.array_equal(got, want)
    assert np.array_equal(codes, oracle.record_codes(nxt)[want])
    assert np.array_equal(hashes, oracle.record_hashes(nxt))
    got, _ = eng.status_diff(nxt)  # the state was replaced for exactly the changed slots
    assert len(got) == 0
    eng.close()


def test_tick_matches_separate_calls():
    """rpk_tick = rpk_select + rpk_status_diff_codes enqueued together: same results, with and without pending pods."""
    offers = rpk.synth.make_offers(20_000, correlated=True)
    N = 70_000
    for P in (0, 300, 200_000):
        eng = make_engine()
        eng.upload_offers(offers)
        tab = oracle.StatusTable(N, 16)
        pods = rpk.synth.make_pods(P, seed=P + 1) if P else None
        ob = oracle.select(offers, pods, n_threads=8) if P else (None, None)
        for sweep, frac in enumerate([0.0, 0.02, 0.5]):
            recs = rpk.synth.make_status_records(N, sweep, frac, stride=16)
            best, top5, idx, codes = eng.tick(pods, recs, want_top5=bool(P))
            want = tab.diff(recs)
            assert np.array_equal(idx, want) and np.array_equal(codes, oracle.record_codes(recs)[want])
            if P:
                assert np.array_equal(best, ob[0]) and np.array_equal(top5, ob[1])
        eng.close()


@pytest.mark.parametrize("stride", sc.STRIDES)
def test_code_corpus_every_stride(stride):
    """The adversarial corpus (each known status, each with one byte changed at every position, one byte short or
    long, lower-cased; unknown strings of a known status's length; empty and one-character statuses) x ports x
    message flag: the code of every slot equals translateRunPodStatus of the decoded string.  Every stride runs the
    corpus as it is (the 256-thread streaming shape); strides 16 / 32 also run it repeated past the 4M-slot big-table
    boundary (the 1024-thread shape)."""
    recs, sts, ports, flags = sc.corpus_records(stride)
    want = sc.translated_codes(sts, ports, flags)
    shapes = [1] + ([-(-(4 << 20) // len(recs))] if stride <= 32 else [])
    for reps in shapes:
        tab = np.ascontiguousarray(np.tile(recs, (reps, 1)))
        eng = make_engine()
        idx, codes, hashes = eng.status_diff(tab, want_hashes=True, want_codes=True)
        eng.close()
        assert len(idx) == len(tab)  # a fresh table: every slot reports, with its code
        assert np.array_equal(codes, np.tile(want, reps)), (stride, len(tab))
        assert np.array_equal(codes, oracle.record_codes(tab)), (stride, len(tab))
        assert np.array_equal(hashes, oracle.record_hashes(tab)), (stride, len(tab))
