"""CPU tests of status_scale_model.py, the one-int-per-slot restatement of the status sweep that the scale tests check
the GPU against: its key table against the oracle's hashes and codes, and seeded call programs against
oracle.StatusTable and status_slots_model.diff_slots at every stride."""
import numpy as np
import pytest

import oracle
import status_scale_model as m
import status_slots_model as ssm
from status_cases import STRIDES, capacity


@pytest.mark.parametrize("stride", STRIDES)
def test_key_table(stride):
    """every fitting key's record is canonical; its hash is the same at every stride it fits and does not depend on the
    flag; two keys hash alike exactly when their classes (pool id, ports) are equal; no hash is 0 (never seen)"""
    fit = m.fitting_keys(stride)
    assert len(fit) > 0 and len(fit) % 4 == 0
    assert np.array_equal(fit, np.nonzero(m.LENS[np.arange(m.K) >> 2] <= capacity(stride))[0])
    h, c = m.hashes(stride)[fit], m.codes(stride)[fit]
    assert np.array_equal(h, m.hashes(256)[fit]), "a key's hash depends on the stride"
    assert np.array_equal(c, m.codes(256)[fit]), "a key's code depends on the stride"
    assert np.array_equal(h[0::2], h[1::2]), "the flag is hashed"
    assert (h != 0).all()
    cls = fit >> 1
    assert len(np.unique(h)) == len(np.unique(cls)), "two classes share a hash"
    _, first = np.unique(cls, return_index=True)
    assert len(np.unique(h[first])) == len(first)
    # the record of a key decodes to its pool entry, ports and flag
    recs = m.lut(stride)[fit]
    pid, ports, flag = fit >> 2, (fit >> 1) & 1, fit & 1
    n = m.LENS[pid]
    assert np.array_equal(recs[:, 0], ((n + 2) | (flag << 7)).astype(np.uint8))
    assert np.array_equal(recs[np.arange(len(fit)), n + 2], ports.astype(np.uint8))


def test_pool_edges():
    """the pool has the pairs the GPU cases lean on: a known status at every stride, twins whose records differ only at
    a byte >= 32, >= 64 and at byte 125, and a status past the 32-byte stripe that fits only the wide strides"""
    twins = edge_twins()
    pos = sorted(p for _, _, p in twins)
    assert any(p >= 32 for p in pos) and any(p >= 64 for p in pos) and 125 in pos
    for s in STRIDES:
        assert len(m.fitting_keys(s)) >= 4 * 6
    assert (m.LENS > 45).any() and (m.LENS <= capacity(16)).any()


def edge_twins():
    """(pool id, pool id, byte): two statuses of one length whose records differ only at that byte"""
    out = []
    for i, a in enumerate(m.POOL):
        for j, b in enumerate(m.POOL):
            if i < j and len(a) == len(b) and len(a) > 0 and a[:-1] == b[:-1]:
                out.append((i, j, len(a)))  # the last character sits at byte 1 + len - 1
    return out


def check_diff(model, tab, keys, stride, what):
    ids, codes, col = model.diff(keys, stride)
    recs = m.records(keys, stride)
    want = tab.diff(recs)
    assert np.array_equal(ids, want), f"{what}: changed list"
    assert np.array_equal(codes, oracle.record_codes(recs)[want]), f"{what}: codes"
    assert np.array_equal(col, oracle.record_hashes(recs)), f"{what}: hash column"
    assert np.array_equal(model.column(), tab.prev_hashes()), f"{what}: state"
    return ids


@pytest.mark.parametrize("stride", STRIDES)
def test_edges(stride):
    """flag-only, ports-only and last-byte-only changes, with the twins at each byte position that fits the stride"""
    rng = np.random.default_rng(stride)
    fit = m.fitting_keys(stride)
    pairs = [(i, j) for i, j, _ in edge_twins() if m.LENS[i] <= capacity(stride)]
    lo, hi = [i for i, _ in pairs], [j for _, j in pairs]
    # flag only (not compared), ports only, then the twins with ports set and with the flag set
    a = np.concatenate([fit, fit, m.key(lo, 1, 0), m.key(lo, 0, 1)])
    b = np.concatenate([fit ^ 1, fit ^ 2, m.key(hi, 1, 0), m.key(hi, 0, 1)])
    model, tab = m.Model(len(a)), oracle.StatusTable(len(a), stride)
    assert len(check_diff(model, tab, a, stride, "first sweep")) == len(a)
    ids = check_diff(model, tab, b, stride, "edge changes")
    want = np.nonzero((a >> 1) != (b >> 1))[0]
    assert np.array_equal(ids, want)
    assert len(want) == len(a) - len(fit), "a flag-only change was reported, or a fields change was not"
    perm = rng.permutation(len(a))
    check_diff(model, tab, b[perm], stride, "permuted")


@pytest.mark.parametrize("stride", STRIDES)
def test_programs(stride):
    """seeded programs of reset / seed / per-slot seed / diff / slot diff / grow at N <= 100k"""
    rng = np.random.default_rng(1000 + stride)
    for prog in range(3):
        N = int(rng.integers(1, 100_000)) if prog else 100_000
        model, tab = m.Model(N), oracle.StatusTable(N, stride)
        keys = m.draw(rng, N, stride)
        for _ in range(12):
            op = rng.choice(["diff", "step", "seed", "seed_slots", "slots", "slots_base", "grow", "reset"])
            what = f"N {N} stride {stride} {op}"
            if op == "reset":
                N = int(rng.integers(1, 100_000))
                model.reset(N)
                tab.reset(N)
                keys = m.draw(rng, N, stride)
            elif op == "grow":
                N2 = N + int(rng.integers(0, 5000))
                model.grow(N2)
                tab.grow(N2)
                keys = np.concatenate([keys, m.draw(rng, N2 - N, stride)])
                N = N2
                assert np.array_equal(model.column(), tab.prev_hashes()), what
            elif op == "seed":
                keys = m.step(rng, keys, stride, 0.5)
                model.seed(keys)
                tab.seed(m.records(keys, stride))
                assert np.array_equal(model.column(), tab.prev_hashes()), what
            elif op == "seed_slots":
                slots = rng.choice(N, int(rng.integers(0, N + 1)), replace=False)
                sk = m.draw(rng, len(slots), stride)
                model.seed_slots(slots, sk)
                tab.seed_slots(slots, m.records(sk, stride))
                assert np.array_equal(model.column(), tab.prev_hashes()), what
            elif op in ("slots", "slots_base"):
                keys = m.step(rng, keys, stride, 0.3)
                slots = np.sort(rng.choice(N, int(rng.integers(0, N + 1)), replace=False)).astype(np.uint32)
                if op == "slots":
                    got, codes = model.diff_slots(slots, keys[slots], stride)
                    want = ssm.diff_slots(tab, slots, m.records(keys[slots], stride))
                else:
                    # a column of global slots [base, base + N), and a list that also holds slots on both sides of it
                    base = int(rng.integers(0, 2**32 - N + 1)) if prog != 1 else 2**32 - N
                    below = np.sort(rng.choice(base, min(base, 50), replace=False)) if base else np.zeros(0, np.int64)
                    top = 2**32 - base - N
                    above = base + N + np.sort(rng.choice(top, min(top, 50), replace=False)) if top else np.zeros(0, np.int64)
                    glob = np.concatenate([below, slots.astype(np.int64) + base, above]).astype(np.uint32)
                    gkeys = np.concatenate([m.draw(rng, len(below), stride), keys[slots], m.draw(rng, len(above), stride)])
                    got, codes = model.diff_slots(glob, gkeys, stride, idx_base=base, col_n=N)
                    want = ssm.diff_slots(tab, slots, m.records(keys[slots], stride)).astype(np.int64) + base
                    assert (want < 2**32).all()
                assert np.array_equal(got, want.astype(np.uint32)), f"{what}: changed list"
                local = (want - (base if op == "slots_base" else 0)).astype(np.int64)
                assert np.array_equal(codes, oracle.record_codes(m.records(keys[local], stride))), f"{what}: codes"
                assert np.array_equal(model.column(), tab.prev_hashes()), f"{what}: state"
            else:
                if op == "step":
                    keys = m.step(rng, keys, stride)
                check_diff(model, tab, keys, stride, what)


def test_diff_slots_list_order():
    """a list that is not ascending reports its changed entries in list order"""
    model = m.Model(1000)
    slots = np.array([7, 3, 999, 0], np.uint32)
    keys = m.draw(np.random.default_rng(0), 4, 16)
    got, _ = model.diff_slots(slots, keys, 16)
    assert got.tolist() == [7, 3, 999, 0]
    got, _ = model.diff_slots(slots, keys, 16)
    assert len(got) == 0
    got, _ = model.diff_slots(slots[::-1].copy(), m.other_class(keys[::-1].copy(), 16), 16)
    assert got.tolist() == [0, 999, 3, 7]


@pytest.mark.parametrize("stride", [16, 48, 256])
def test_other_class(stride):
    fit = m.fitting_keys(stride)
    o = m.other_class(fit, stride)
    assert np.isin(o, fit).all() and ((o >> 1) != (fit >> 1)).all() and np.array_equal(o & 1, fit & 1)
