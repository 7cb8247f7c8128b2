"""CPU tests of offers_refresh_model.py against the oracle: whenever the model says no changed offer reaches a row, the
oracle's list for the row under the new table is its list under the old one."""
import numpy as np
import pytest

import oracle
import offers_refresh_model as model

PRICES = np.array([0.1, 0.2, 0.25, 0.3, 0.3, 0.45, 0.5, 0.7, 0.0, -0.0, -0.2, np.nan, np.inf, -np.inf, 1e-300])


def table(rng, G):
    return {
        "mem_gb": rng.choice([8, 16, 24, 40, 80], G).astype(np.int32),
        "vcpu": rng.choice([0, 4, 8, 16], G).astype(np.int32),
        "ram_gb": rng.choice([0, 32, 64], G).astype(np.int32),
        "secure_price": rng.choice(PRICES, G),
        "community_price": rng.choice(PRICES, G),
        "flags": rng.integers(0, 4, G).astype(np.uint8),
    }


def rows(rng, P):
    return {
        "req_mem_gb": rng.choice([1, 8, 16, 24, 40, 80, 100], P).astype(np.int32),
        "req_vcpu": rng.choice([0, 4, 8], P).astype(np.int32),
        "req_ram_gb": rng.choice([0, 32], P).astype(np.int32),
        "max_price": rng.choice([0.5, 0.3, 0.25, 1.0, np.inf, np.nan, 0.0], P),
        "cloud": rng.choice([0, 1, 2], P, p=[0.45, 0.45, 0.1]).astype(np.uint8),
    }


def change(rng, offers, k):
    """k offers of a copy of the table get a new value in one random column"""
    new = {c: v.copy() for c, v in offers.items()}
    G = len(offers["mem_gb"])
    for g in rng.choice(G, k, replace=False):
        c = rng.choice(model.COLS)
        if c in ("secure_price", "community_price"):
            new[c][g] = rng.choice(PRICES) if rng.random() < 0.6 else new[c][g] * rng.choice([0.5, 0.999, 1.001, 2.0])
        elif c == "flags":
            new[c][g] ^= np.uint8(rng.integers(1, 4))
        else:
            new[c][g] = rng.choice(offers[c])
    return new


def check(offers, new, pods, changed):
    _, old5 = oracle.select(offers, pods)
    _, new5 = oracle.select(new, pods)
    hit = model.reached(new, pods, old5, changed)
    same = (old5 == new5).all(axis=1)
    assert same[~hit].all(), f"rows the model leaves alone changed: {np.flatnonzero(~hit & ~same)[:10]}"
    return hit, same


@pytest.mark.parametrize("seed", range(12))
def test_unreached_rows_keep_their_list(seed):
    rng = np.random.default_rng(1000 + seed)
    G = int(rng.integers(8, 80))
    offers = table(rng, G)
    pods = rows(rng, 3000)
    total_hit = total = 0
    for k in (1, 2, 5, min(16, G)):
        new = change(rng, offers, k)
        changed = model.changed_offers(offers, new)
        assert len(changed) <= k
        hit, _ = check(offers, new, pods, changed)
        total_hit += int(hit.sum())
        total += len(hit)
    assert total_hit < total, "the rule reaches every row: it would save nothing"


def test_an_offer_changed_twice_and_a_superset():
    rng = np.random.default_rng(7)
    offers = table(rng, 40)
    pods = rows(rng, 4000)
    mid = change(rng, offers, 3)
    new = change(rng, mid, 3)
    changed = np.union1d(model.changed_offers(offers, mid), model.changed_offers(mid, new))
    check(offers, new, pods, changed)
    check(offers, new, pods, np.union1d(changed, rng.choice(40, 5, replace=False)))  # any superset is safe


def test_ties_at_the_fifth_entry():
    """a changed offer priced exactly as L[4] reaches the row only when its index is below L[4]'s"""
    G = 12
    offers = {"mem_gb": np.full(G, 80, np.int32), "vcpu": None, "ram_gb": None,
              "secure_price": np.array([0.1, 0.1, 0.2, 0.2, 0.3, 0.3, 0.3, 0.4, 0.45, 0.45, 0.6, 0.6]),
              "community_price": np.zeros(G), "flags": np.ones(G, np.uint8)}
    pods = {"req_mem_gb": np.array([16], np.int32), "req_vcpu": None, "req_ram_gb": None, "max_price": None, "cloud": None}
    _, l = oracle.select(offers, pods)
    assert l[0].tolist() == [0, 1, 2, 3, 4]
    for g, want in ((5, False), (7, False), (9, False)):  # after L[4] = 4 at 0.3: not before it
        new = {k: (v.copy() if v is not None else None) for k, v in offers.items()}
        new["secure_price"][g] = 0.3
        assert model.reached(new, pods, l, [g])[0] == want
        check(offers, new, pods, [g])
    new = {k: (v.copy() if v is not None else None) for k, v in offers.items()}
    new["secure_price"][3] = 0.3  # in L: reached
    assert model.reached(new, pods, l, [3])[0]
    new = {k: (v.copy() if v is not None else None) for k, v in offers.items()}
    new["secure_price"][5] = 0.2999999  # just below L[4]'s price: reached, and the list changes
    assert model.reached(new, pods, l, [5])[0]
    assert not (check(offers, new, pods, [5])[1]).all()


def test_special_prices_flags_and_clouds():
    """NaN / Inf / 0 / negative prices, flags off and on, max_price NaN, cloud byte 2, rows with 0-4 feasible offers"""
    rng = np.random.default_rng(11)
    for G in (1, 3, 5, 9):
        offers = table(rng, G)
        pods = rows(rng, 2000)
        for g in range(G):
            for col, vals in (("secure_price", [np.nan, np.inf, 0.0, -0.0, -1.0, 0.05]),
                              ("community_price", [np.nan, np.inf, 0.0, -1.0, 0.05]), ("flags", [0, 1, 2, 3])):
                for v in vals:
                    new = {k: x.copy() for k, x in offers.items()}
                    new[col][g] = v
                    check(offers, new, pods, model.changed_offers(offers, new))
    pods = rows(rng, 100)
    pods["cloud"][:] = 2
    offers = table(rng, 10)
    _, l = oracle.select(offers, pods)
    assert (l == -1).all()
    assert not model.reached(change(rng, offers, 10), pods, l, np.arange(10)).any(), "nothing reaches a row of neither cloud"
