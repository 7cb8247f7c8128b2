"""The reach rule of rpk_offers_refresh (include/rpk.h, rpk_select_pending_changed) in numpy.

A row's stored list L was selected against an earlier table; the current table differs from it only at the offer
indices in `changed`.  The row's list under the current table is L unless a changed offer reaches the row: it is in L,
or it is feasible for the row now and L has fewer than five entries or (price(c), c) < (price(L[4]), L[4]).

Generations follows the rule over a whole history: the change window, the generations and the floor, and which pending
slots a tick reselects."""
import numpy as np

COLS = ("mem_gb", "vcpu", "ram_gb", "secure_price", "community_price", "flags")


def column(offers, name):
    G = len(offers["mem_gb"])
    v = offers.get(name)
    return np.zeros(G, np.int32) if v is None else np.asarray(v)


def changed_offers(old, new):
    """ascending indices of the offers whose six columns differ bit for bit (same G)"""
    diff = np.zeros(len(old["mem_gb"]), bool)
    for k in COLS:
        a, b = column(old, k), column(new, k)
        diff |= (a.view(np.uint8).reshape(len(a), a.itemsize) != b.view(np.uint8).reshape(len(b), b.itemsize)).any(axis=1)
    return np.flatnonzero(diff)


def reached(offers, pods, top5, changed):
    """bool[P]: some offer of `changed` reaches row p, whose stored list is top5[p], under the current table `offers`"""
    P = len(pods["req_mem_gb"])
    changed = np.asarray(changed, np.int64)
    if not len(changed) or not P:
        return np.zeros(P, bool)
    mem, vcpu, ram = (column(offers, k)[changed][None, :] for k in ("mem_gb", "vcpu", "ram_gb"))
    sp, cp = column(offers, "secure_price"), column(offers, "community_price")
    flags = column(offers, "flags")[changed][None, :]
    req_vcpu = pods.get("req_vcpu") if pods.get("req_vcpu") is not None else np.zeros(P, np.int32)
    req_ram = pods.get("req_ram_gb") if pods.get("req_ram_gb") is not None else np.zeros(P, np.int32)
    mx = pods.get("max_price") if pods.get("max_price") is not None else np.full(P, 0.5)
    cloud = pods.get("cloud") if pods.get("cloud") is not None else np.zeros(P, np.uint8)
    cloud = cloud.astype(np.int64)[:, None]
    in_list = (top5[:, :, None] == changed[None, None, :]).any(axis=1)
    price = np.where(cloud == 1, cp[changed][None, :], sp[changed][None, :])
    bit = np.where(cloud == 1, 2, 1)
    with np.errstate(invalid="ignore"):
        feasible = ((cloud <= 1) & ((flags & bit) != 0) & (price > 0) & (price < mx[:, None]) &
                    (mem >= pods["req_mem_gb"][:, None]) & (vcpu >= req_vcpu[:, None]) & (ram >= req_ram[:, None]))
        l4 = top5[:, 4].astype(np.int64)[:, None]
        p4 = np.where(cloud == 1, cp[np.maximum(l4, 0)], sp[np.maximum(l4, 0)])
        before = (l4 < 0) | (price < p4) | ((price == p4) & (changed[None, :] < l4))
    return in_list.any(axis=1) | (feasible & before).any(axis=1)


WHOLESALE = 2**32 - 1  # *n_offers_changed of a refresh that invalidated the stored results wholesale
DELTA_MAX = 16  # RPK_OFFERS_DELTA_MAX
POD_COLS = {"req_mem_gb": (np.int32, 16), "req_vcpu": (np.int32, 0), "req_ram_gb": (np.int32, 0),
            "max_price": (np.float64, 0.5), "cloud": (np.uint8, 0)}  # dtype and rpk_pods_reset's value


def _copy(offers):
    return {k: (None if v is None else np.array(v, copy=True)) for k, v in offers.items()}


class Generations:
    """The stored pending results of one ctx (rpk.h: rpk_offers_refresh, rpk_select_pending_changed) over a whole
    history of offer uploads and refreshes, pod-table resets, seeds and marks, and ticks.

    The ctx holds a generation, a floor (the generation of the last wholesale invalidation) and the change window: one
    entry per offer at the generation of its latest change, newest first, at most DELTA_MAX entries.  Each slot holds the
    generation of its stored result (0: none), the five columns the result came from and its top-5 list."""

    def __init__(self, N=0):
        self.offers = None
        self.gen = self.floor = 0
        self.window = []  # [(offer, generation)], newest first
        self.reset(N)

    def reset(self, N):
        self.N = N
        self.cols = {k: np.full(N, v, t) for k, (t, v) in POD_COLS.items()}
        self.res_cols = {k: np.zeros(N, t) for k, (t, _) in POD_COLS.items()}
        self.pending = np.zeros(N, bool)
        self.res_gen = np.zeros(N, np.int64)
        self.top5 = np.full((N, 5), -1, np.int32)

    def grow(self, N, keep_results=True):
        """rpk_pods_grow: slots [self.N, N) get reset rows, no flag and no stored result; every other slot keeps its row,
        flag and stored result.  keep_results=False drops every stored result, as a grow does on a ctx whose results
        were made for the range of a one-process-per-GPU rank."""
        assert N >= self.N
        N0, old = self.N, (self.cols, self.res_cols, self.pending, self.res_gen, self.top5)
        self.reset(N)
        for k in POD_COLS:
            self.cols[k][:N0], self.res_cols[k][:N0] = old[0][k], old[1][k]
        self.pending[:N0] = old[2]
        if keep_results:
            self.res_gen[:N0], self.top5[:N0] = old[3], old[4]

    def _wholesale(self):
        self.gen += 1
        self.floor = self.gen
        self.window = []

    def upload(self, offers):
        self.offers = _copy(offers)
        self._wholesale()

    def refresh(self, new):
        """-> the expected *n_offers_changed"""
        if self.offers is None or len(new["mem_gb"]) != len(self.offers["mem_gb"]):
            self.upload(new)
            return WHOLESALE
        changed = changed_offers(self.offers, new)
        self.offers = _copy(new)
        if not len(changed):
            return 0
        w = [(int(c), self.gen + 1) for c in changed] + [e for e in self.window if e[0] not in set(changed.tolist())]
        if len(w) > DELTA_MAX:
            self._wholesale()
            return WHOLESALE
        self.gen += 1
        self.window = w
        return len(changed)

    def seed(self, slots, pods):
        for k, (t, v) in POD_COLS.items():
            x = pods.get(k)
            self.cols[k][slots] = v if x is None else x

    def mark(self, slots, flags):
        self.pending[slots] = np.asarray(flags) != 0

    def rows(self, slots):
        return {k: np.ascontiguousarray(c[slots]) for k, c in self.cols.items()}

    def pending_slots(self):
        return np.flatnonzero(self.pending).astype(np.uint32)

    def tick(self, top5):
        """One rpk_select_pending_changed.  top5: the lists of the pending slots (ascending) under the current table.
        -> the slots it reselects: no stored result, columns that differ bit for bit, a result below the floor, or one
        that a window entry newer than it reaches.  Every pending slot's result is current afterwards."""
        pend = self.pending_slots()
        g = self.res_gen[pend]
        same = np.ones(len(pend), bool)
        for k, c in self.cols.items():
            a, b = c[pend], self.res_cols[k][pend]
            same &= (a.view(np.uint8).reshape(len(pend), a.itemsize) == b.view(np.uint8).reshape(len(pend), b.itemsize)).all(axis=1)
        stale = (g == 0) | ~same | (g < self.floor)
        test = ~stale & (g != self.gen)
        for rg in np.unique(g[test]):
            at = np.flatnonzero(test & (g == rg))
            newer = [c for c, cg in self.window if cg > rg]
            stale[at] |= reached(self.offers, self.rows(pend[at]), self.top5[pend[at]], newer)
        hit = pend[stale]
        self.top5[hit] = top5[stale]
        for k, c in self.cols.items():
            self.res_cols[k][hit] = c[hit]
        self.res_gen[pend] = self.gen
        return hit
