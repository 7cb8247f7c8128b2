"""A model of one whole ctx, for call histories that cross offer refreshes, table grows, resets and sweeps.

It restates no rule: offers_refresh_model.Generations holds the offers, the generations and change window, the pod rows,
pending flags and stored pending results; oracle.StatusTable holds the tracked status table and
status_slots_model.diff_slots sweeps a slot list of it; every expected list is oracle.select's.  What this module adds
is the bookkeeping between them: which rows a pending tick reports, and the table edits the histories draw from."""
import os

import numpy as np

import offers_refresh_model as orm
import oracle
import status_slots_model


def lists(offers, rows):
    """oracle.select of the rows under the table -> (best[P], top5[P, 5])"""
    P = len(rows["req_mem_gb"])
    if P == 0:
        return np.zeros(0, np.int32), np.zeros((0, 5), np.int32)
    return oracle.select(offers, rows, want_top5=True, n_threads=os.cpu_count() or 1)


class Tick:
    """what one rpk_select_pending_changed must return: n_pending, the slots it reselects (the stale set) and the rows it
    reports -- the reselected slots with no stored result or a stored list other than the oracle's, ascending"""

    def __init__(self, pend, stale, slots, best, top5):
        self.pend, self.stale = pend, stale
        self.slots, self.best, self.top5 = slots, best, top5

    def in_range(self, lo, hi):
        """the part of the tick a rank whose slots are [lo, hi) returns: (n_pending, n_reselected, slots, best, top5)"""
        p = (self.pend >= lo) & (self.pend < hi)
        s = (self.stale >= lo) & (self.stale < hi)
        r = (self.slots >= lo) & (self.slots < hi)
        return int(p.sum()), int(s.sum()), self.slots[r], self.best[r], self.top5[r]


class Ctx:
    """The state of one ctx (or of every rank of a group, which share a history) after each call."""

    def __init__(self):
        self.gens = orm.Generations(0)
        self.status = None  # no tracked table before status_reset

    # -- offers ----------------------------------------------------------------------------------------------------
    @property
    def offers(self):
        return self.gens.offers

    def upload(self, offers):
        self.gens.upload(offers)

    def refresh(self, offers):
        """-> the expected *n_offers_changed (orm.WHOLESALE for a wholesale invalidation)"""
        return self.gens.refresh(offers)

    # -- pod table -------------------------------------------------------------------------------------------------
    @property
    def N(self):
        return self.gens.N

    def pods_reset(self, N):
        self.gens.reset(N)

    def pods_grow(self, N, keep_results=True):
        self.gens.grow(N, keep_results)

    def seed(self, slots, rows):
        self.gens.seed(slots, rows)

    def mark(self, slots, flags):
        self.gens.mark(slots, flags)

    def rows(self, slots):
        return self.gens.rows(np.asarray(slots, np.int64))

    def pending(self):
        return self.gens.pending_slots()

    def expected(self, slots):
        """oracle.select over the rows held at `slots` (any order, repeats allowed)"""
        return lists(self.offers, self.rows(slots))

    def stored_full_lists(self):
        """the stored lists of pending slots that hold five entries and are the slot's list under the current table"""
        g = self.gens
        pend = g.pending_slots()
        G = len(self.offers["mem_gb"])
        full = pend[(g.res_gen[pend] != 0) & (g.top5[pend] >= 0).all(axis=1) & (g.top5[pend] < G).all(axis=1)]
        return g.top5[full][(self.expected(full)[1] == g.top5[full]).all(axis=1)]

    def tick(self):
        """one rpk_select_pending_changed -> Tick.  Afterwards every pending slot's stored list is the oracle's; a slot
        the reach rule leaves alone must already hold it (AssertionError naming the slots otherwise)."""
        g = self.gens
        pend = g.pending_slots()
        best, top5 = lists(self.offers, g.rows(pend))
        had = g.res_gen[pend] != 0
        before = g.top5[pend].copy()
        stale = np.isin(pend, g.tick(top5))
        kept_bad = np.flatnonzero(~stale & (before != top5).any(axis=1))
        assert not len(kept_bad), f"the reach rule keeps a stale list at slots {pend[kept_bad[:8]].tolist()}"
        rep = stale & (~had | (before != top5).any(axis=1))
        return Tick(pend, pend[stale], pend[rep], best[rep], top5[rep])

    # -- status table ----------------------------------------------------------------------------------------------
    def status_reset(self, N, stride):
        if self.status is None:
            self.status = oracle.StatusTable(N, stride)
        else:
            self.status.reset(N)

    def status_grow(self, N):
        self.status.grow(N)

    def status_seed(self, records):
        self.status.seed(records)

    def status_seed_slots(self, slots, records):
        self.status.seed_slots(slots, records)

    def status_diff(self, records):
        return self.status.diff(records)

    def status_diff_slots(self, slots, records):
        return status_slots_model.diff_slots(self.status, slots, records)


# ---- table edits the histories draw from ----------------------------------------------------------------------------
def copy_table(offers):
    return {k: (None if v is None else np.array(v, copy=True)) for k, v in offers.items()}


def edit_offers(rng, offers, k):
    """k distinct offers of a copy of the table get a new value in one column each (a price scaled or redrawn, the flags
    flipped, or a requirement column set to another value the column holds)"""
    new = copy_table(offers)
    G = len(new["mem_gb"])
    for g in rng.choice(G, min(k, G), replace=False):
        col = str(rng.choice(["secure_price", "community_price", "flags", "mem_gb", "vcpu", "ram_gb"]))
        if new.get(col) is None:
            col = "secure_price"
        if col.endswith("price"):
            new[col][g] = new[col][g] * rng.choice([0.5, 0.97, 1.03, 2.0]) if rng.random() < 0.7 else rng.choice([0.0, 0.011, 0.3, 5.0])
        elif col == "flags":
            new[col][g] ^= np.uint8(rng.integers(1, 4))
        else:
            new[col][g] = new[col][int(rng.integers(0, G))] + (0 if rng.random() < 0.7 else 1)
    return new


def tie_edit(rng, offers, top5, n_pairs=3):
    """a refresh that moves offers onto the fifth entry L[4] of stored lists: offer c takes every column of L[4] (the
    same requirements, both prices and the flags), so the two tie on price and c comes first exactly when c < L[4].
    top5: stored lists with five entries.  Half the pairs take a c below L[4], the others one above it.
    -> (new table, [(c, L[4])])"""
    new = copy_table(offers)
    G = len(new["mem_gb"])
    pairs = []
    for i in rng.permutation(len(top5))[: 4 * n_pairs]:
        l4 = int(top5[i, 4])
        below = len(pairs) % 2 == 0
        pool = np.setdiff1d(np.arange(0, l4) if below else np.arange(l4 + 1, G), top5[i])
        pool = np.setdiff1d(pool, [x for p in pairs for x in p])
        if l4 in {x for p in pairs for x in p} or not len(pool):
            continue
        c = int(rng.choice(pool))
        for col in ("mem_gb", "vcpu", "ram_gb", "secure_price", "community_price", "flags"):
            if new.get(col) is not None:
                new[col][c] = new[col][l4]
        pairs.append((c, l4))
        if len(pairs) == n_pairs:
            break
    return new, pairs


def layout_edit(rng, offers, k):
    """k offers take mem values the table has never held, so the offer view gets k more threshold words"""
    new = copy_table(offers)
    G = len(new["mem_gb"])
    top = int(new["mem_gb"].max()) if G else 0
    for i, g in enumerate(rng.choice(G, min(k, G), replace=False)):
        new["mem_gb"][g] = top + 3 + 2 * i
    return new


def odd_rows(rng, offers, n):
    """n pod rows: requests around the table's values, max_price from the table's prices with NaN, -0.0, 0.0 and +inf
    among them, cloud bytes 0 and 1 and a few 2 and 255"""
    G = len(offers["mem_gb"])

    def around(col, fallback):
        v = offers.get(col)
        if v is None or not G:
            v = np.asarray(fallback)
        v = np.unique(np.asarray(v, np.int64))
        return np.clip(np.concatenate([v - 1, v, v + 1, [0]]), -2**31, 2**31 - 1)

    rows = {"req_mem_gb": rng.choice(around("mem_gb", [8, 16, 80]), n).astype(np.int32),
            "req_vcpu": rng.choice(around("vcpu", [0, 4]), n).astype(np.int32),
            "req_ram_gb": rng.choice(around("ram_gb", [0, 32]), n).astype(np.int32)}
    rows["req_vcpu"][rng.random(n) < 0.5] = 0
    rows["req_ram_gb"][rng.random(n) < 0.5] = 0
    prices = np.concatenate([offers["secure_price"], offers["community_price"]]) if G else np.zeros(0)
    prices = prices[prices > 0]
    mp = rng.choice(prices, n) * rng.choice([1.0, 1.0, 1.5, 3.0], n) if len(prices) else np.full(n, 0.5)
    odd = rng.random(n)
    mp[odd < 0.04] = np.nan
    mp[(odd >= 0.04) & (odd < 0.08)] = -0.0
    mp[(odd >= 0.08) & (odd < 0.10)] = 0.0
    mp[(odd >= 0.10) & (odd < 0.14)] = np.inf
    rows["max_price"] = mp.astype(np.float64)
    cloud = rng.choice(np.array([0, 1, 2, 255], np.uint8), n, p=[0.46, 0.46, 0.04, 0.04])
    rows["cloud"] = cloud
    return rows
