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


# ---- Generations: the rule over whole histories ----------------------------------------------------------------------
def seeded(rng, N, G):
    offers = table(rng, G)
    gm = model.Generations(N)
    gm.upload(offers)
    pods = rows(rng, N)
    gm.seed(np.arange(N), pods)
    return gm, offers


def test_window_arithmetic():
    rng = np.random.default_rng(3)
    gm, offers = seeded(rng, 10, 40)
    assert gm.refresh(offers) == 0 and gm.gen == 1, "an identical refresh bumps nothing"

    def bump(t, gs):
        new = {k: v.copy() for k, v in t.items()}
        new["mem_gb"][gs] += 1
        return new

    a = bump(offers, np.arange(8))
    assert gm.refresh(a) == 8
    b = bump(a, np.arange(8, 16))
    assert gm.refresh(b) == 8 and len(gm.window) == 16 and [e[1] for e in gm.window] == [3] * 8 + [2] * 8
    c = bump(b, [3])
    assert gm.refresh(c) == 1 and len(gm.window) == 16 and gm.window[0] == (3, 4), "an offer changed twice holds one entry"
    d = bump(c, [20])
    assert gm.refresh(d) == model.WHOLESALE and gm.window == [] and gm.floor == gm.gen == 5, "17 offers: wholesale"
    assert gm.refresh(bump(d, np.arange(17))) == model.WHOLESALE, "17 in one refresh: wholesale"
    assert gm.refresh({k: v[:39] for k, v in d.items()}) == model.WHOLESALE, "another G: wholesale"
    fresh = model.Generations(4)
    assert fresh.refresh(offers) == model.WHOLESALE and fresh.floor == 1, "no resident table: wholesale"


def oracle_lists(gm):
    pend = gm.pending_slots()
    return pend, oracle.select(gm.offers, gm.rows(pend))[1] if len(pend) else np.zeros((0, 5), np.int32)


@pytest.mark.parametrize("seed", range(8))
def test_random_histories_keep_every_unreselected_list(seed):
    """refreshes of 1-17 offers (some changed again), uploads, identical and changed seeds, marks and unmarks across
    refreshes, and ticks: after every tick each pending slot the model does not reselect holds the oracle's list"""
    rng = np.random.default_rng(2000 + seed)
    N, G = 3000, int(rng.integers(17, 60))
    gm, offers = seeded(rng, N, G)
    gm.mark(np.arange(N), rng.random(N) < 0.5)
    kept = hit_total = 0
    ops = {"refresh": 0, "wholesale": 0}
    for stp in range(60):
        op = rng.choice(["refresh", "refresh", "refresh", "upload", "seed", "mark", "tick", "tick", "tick"])
        if op == "refresh":
            k = int(rng.integers(1, 18))
            new = change(rng, gm.offers, k)
            if rng.random() < 0.3 and gm.window:  # one more change to an offer the window already holds
                g = gm.window[-1][0]
                new["mem_gb"][g] ^= np.int32(1)
            n = gm.refresh(new)
            ops["refresh"] += 1
            ops["wholesale"] += n == model.WHOLESALE
            assert n == model.WHOLESALE or n == len(model.changed_offers(offers, new))
            offers = new
        elif op == "upload":
            gm.upload(change(rng, gm.offers, 2) if rng.random() < 0.5 else gm.offers)
            offers = gm.offers
        elif op == "seed":
            sl = np.sort(rng.choice(N, int(rng.integers(1, 400)), replace=False))
            gm.seed(sl, gm.rows(sl) if rng.random() < 0.4 else rows(rng, len(sl)))
        elif op == "mark":
            sl = np.sort(rng.choice(N, int(rng.integers(1, 800)), replace=False))
            gm.mark(sl, rng.random(len(sl)) < 0.5)
        else:
            pend, want = oracle_lists(gm)
            before = gm.top5[pend].copy()
            hit = gm.tick(want)
            keep = ~np.isin(pend, hit)
            bad = np.flatnonzero(keep & (before != want).any(axis=1))
            assert not len(bad), f"step {stp}: slots {pend[bad[:8]].tolist()} keep a stale list"
            assert np.array_equal(gm.top5[pend], want)
            kept += int(keep.sum())
            hit_total += len(hit)
    assert kept and hit_total and ops["refresh"] > ops["wholesale"], (kept, hit_total, ops)
