"""GPU tests of offer-table refreshes at the edges of prices, columns and views: k_offer_diff (which offers a refresh
changed), k_pod_stale_reach (which pending rows a changed offer can reach) and the device form's reselect
(k_pod_reselect_top5), each against offers_refresh_model.Generations and the oracle.

Every history runs on every path at once: the device form of 1 or 3 ranks, their host-sync twins and a reference ctx
that calls rpk_select_pending_changed (Twins), or one host ctx of one or three shards.  After every tick:
n_reselected is the model's count exactly (fewer is a stale list, more is a rule other than rpk.h's), the reported slots
are the pending slots whose oracle list changed, and a per-slot mirror of the reports equals the oracle and
rpk_select_slots on every pending slot."""
import numpy as np
import pytest

import offers_refresh_model as model
import rpk
import select_plan_cases as sc
from test_offers_refresh_gpu import shared_device
from test_select_pending_changed_device_gather_gpu import PADW, Twins, result_range, view_kind
from test_select_pending_changed_gpu import Mirror, check_mirror, step

pytestmark = pytest.mark.gpu

N = 100_003
N_PEND = 20_000
WHOLESALE = model.WHOLESALE
EINVAL = rpk._ffi.RPK_EINVAL


def copy(offers):
    return {k: (None if v is None else np.array(v, copy=True)) for k, v in offers.items()}


class Hist:
    """one history on the paths of `kind` ("twins" with n ranks, "host": a one-GPU ctx, "shards": an n-shard ctx on
    one GPU), the model and the per-slot mirror"""

    def __init__(self, offers, pods, kind="twins", n=1, seed=0, n_pend=N_PEND, force=None, N_slots=N):
        self.N = N_slots
        self.rng = np.random.default_rng(seed)
        self.t = self.eng = None
        if kind == "twins":
            self.t = Twins(n, self.N)
            self.engines = self.t.all()
            self.ref = self.t.ref
        else:
            if kind == "shards":
                with shared_device():
                    self.eng = rpk.Engine(device_ids=[0] * n)
            else:
                self.eng = rpk.Engine(1)
            self.engines = [self.eng]
            self.ref = self.eng
        self.gm = model.Generations(self.N)
        self.capture = False  # the next tick of the device form replays a graph captured after the table changed
        self.ticked = False
        self.upload(offers, force)
        self.history(lambda e: e.pods_reset(self.N))
        self.seed(np.arange(self.N, dtype=np.uint32), pods)
        pend = np.sort(self.rng.choice(self.N, min(n_pend, self.N), replace=False))
        cuts = [c for r in range(n) for c in result_range(self.N, n, r)]
        pend = np.union1d(pend, [x for c in cuts for x in (c - 1, c) if 0 <= x < self.N]).astype(np.uint32)
        self.mark(pend, np.ones(len(pend), np.uint8))
        self.m = Mirror(self.N)

    @property
    def offers(self):
        return self.gm.offers

    def history(self, fn):
        for e in self.engines:
            fn(e)

    def close(self):
        if self.t is not None:
            self.t.close()
        else:
            self.eng.close()

    def upload(self, offers, force=None):
        with view_kind(force or "auto"):
            self.history(lambda e: e.upload_offers(offers))
        self.gm.upload(offers)
        self.capture = True

    def refresh(self, new, force=None, what=""):
        ns = []
        with view_kind(force or "auto"):
            self.history(lambda e: ns.append(e.refresh_offers(new)))
        want = self.gm.refresh(new)
        assert set(ns) == {want}, f"{what}: n_offers_changed {ns}, the model says {want}"
        self.capture = True
        return want

    def edit(self, edits, what, force=None):
        """a refresh of the current table with (column, offer, value) edits"""
        new = copy(self.offers)
        for col, g, v in edits:
            new[col][g] = v
        return self.refresh(new, force, what)

    def seed(self, slots, pods):
        self.history(lambda e: e.pods_seed_slots(slots, pods))
        self.gm.seed(slots, pods)

    def mark(self, slots, flags):
        self.history(lambda e: e.pods_mark_pending(slots, flags))
        self.gm.mark(slots, flags)

    def call(self, what):
        """one call on every path -> (n_pending, n_reselected, slots, best, top5) of the whole table"""
        if self.t is None:
            return step(self.eng, self.m, self.N)
        replay = self.capture and self.ticked
        if replay:
            self.t.capture()
        n_p, n_r, slots = self.t.step(what, replay=replay)  # device form == host-sync twins == the reference, bit for bit
        words = self.t.d.mem[0].cpu().numpy()[PADW:PADW + self.t.d.words]
        parts = [rpk.results_region(words, self.t.n, self.t.cap, r) for r in range(self.t.n)]
        got = [np.concatenate([p[i] for p in parts]) for i in range(3)]
        self.m.apply(*got)
        return n_p, n_r, got[0], got[1], got[2]

    def tick(self, what):
        pend = self.gm.pending_slots()
        rows = self.gm.rows(pend)
        wb, wt = sc.expected(self.offers, rows) if len(pend) else (np.zeros(0, np.int32), np.zeros((0, 5), np.int32))
        old = self.m.top5[pend].copy()
        hit = self.gm.tick(wt)
        n_p, n_r, sl, _, _ = self.call(what)
        self.capture, self.ticked = False, True
        assert n_p == len(pend), f"{what}: n_pending {n_p}, {len(pend)} pending"
        assert n_r == len(hit), f"{what}: reselected {n_r}, the model says {len(hit)}" + (
            " (a stale list is kept)" if n_r < len(hit) else "")
        assert np.array_equal(sl, pend[(wt != old).any(axis=1)]), f"{what}: reported != the pending slots whose oracle list changed"
        if len(pend):
            sc.check(f"{what}: mirror vs oracle", self.m.best[pend], self.m.top5[pend], wb, wt)
            check_mirror(what, self.ref, self.m, pend)
        return n_r

    # ---- what the edits aim at ---------------------------------------------------------------------------------------
    def lists(self):
        pend = self.gm.pending_slots()
        return pend, self.gm.rows(pend), self.gm.top5[pend]

    def price_col(self, cloud):
        return "community_price" if cloud == 1 else "secure_price"

    def most_listed(self):
        _, _, t = self.lists()
        G = len(self.offers["mem_gb"])
        return int(np.bincount(t[t >= 0].ravel(), minlength=G).argmax())

    def unlisted(self, k=1):
        _, _, t = self.lists()
        free = np.setdiff1d(np.arange(len(self.offers["mem_gb"])), t[t >= 0])
        return [int(x) for x in free[:k]]

    def reachable(self, g, price=None):
        """offer g, fed the largest mem / vcpu / ram values of the table and both cloud bits: feasible for every row
        with a price bound above its price (the values already occur, so the view keeps its shape)"""
        o = self.offers
        e = [("mem_gb", g, o["mem_gb"].max()), ("flags", g, 3)]
        for col in ("vcpu", "ram_gb"):
            if o.get(col) is not None:
                e.append((col, g, o[col].max()))
        if price is not None:
            e += [("secure_price", g, price), ("community_price", g, price)]
        return e

    def fifth(self, cloud=0):
        """(L[4], its price) shared by the most pending rows of `cloud` with five entries"""
        _, rows, t = self.lists()
        sel = (rows["cloud"] == cloud) & (t[:, 4] > 0)
        if not sel.any():
            return None
        l4 = int(np.bincount(t[sel, 4]).argmax())
        return l4, float(self.offers[self.price_col(cloud)][l4])

    def make_room(self, k):
        """an identical upload when the window has no room for k more offers, so the next refreshes keep results"""
        if len(self.gm.window) + k > model.DELTA_MAX:
            self.upload(copy(self.offers))
            self.tick("an identical upload: every pending slot reselected")


# ---- (b) the reach pre-pass at the edges ----------------------------------------------------------------------------
def reach_history(h, label):
    """refreshes aimed at the reach rule's edges, each followed by a tick; slots unmarked across refreshes and marked
    again; slots re-seeded between a refresh and its tick"""
    G = len(h.offers["mem_gb"])
    h.tick(f"{label}: first call")
    assert h.tick(f"{label}: steady") == 0
    pend, _, _ = h.lists()
    away = np.sort(h.rng.choice(pend, min(2000, len(pend) // 4), replace=False)).astype(np.uint32)
    h.mark(away, np.zeros(len(away), np.uint8))
    for cloud in (0, 1):  # a price exactly at price(L[4]) of many rows, from an index below L[4] and one above
        f = h.fifth(cloud)
        if f is None:
            continue
        l4, p4 = f
        listed = set(h.lists()[2].ravel().tolist())
        below = [g for g in range(l4) if g not in listed][:1] or [0]
        above = [g for g in range(l4 + 1, G) if g not in listed][:1]
        for side, gs in (("below", below), ("above", above)):
            if gs:
                h.make_room(1)
                h.edit(h.reachable(gs[0]) + [(h.price_col(cloud), gs[0], p4)], f"{label}: tie {side} L[4]")
                h.tick(f"{label}: cloud {cloud}, a price equal to L[4]'s from {side}")
        if cloud == 0:  # back after one to three refresh + tick rounds
            h.mark(away, np.ones(len(away), np.uint8))
            h.tick(f"{label}: unmarked slots back")
    f = h.fifth(0)
    if f is not None:
        h.make_room(1)
        h.edit([("secure_price", f[0], f[1] * 1.25)], f"{label}: L[4] itself")
        h.tick(f"{label}: the L[4] offer changed")
    # a price exactly at rows' max_price (infeasible by the strict bound), then just below it (feasible)
    _, rows, _ = h.lists()
    mp = rows["max_price"]
    fin = np.unique(mp[np.isfinite(mp) & (mp > 0) & (mp < 1e9)])
    if len(fin) and h.unlisted():
        mx = float(fin[0])
        g = h.unlisted()[0]
        for p, what in ((mx, "equal to"), (float(np.nextafter(mx, 0)), "just below")):
            h.make_room(1)
            h.edit(h.reachable(g, p), f"{label}: price {what} max_price")
            h.tick(f"{label}: a price {what} rows' max_price")
    # the most-listed offer's price through NaN / Inf / 0 / -0.0 / negative and back
    g = h.most_listed()
    keep = (h.offers["secure_price"][g], h.offers["community_price"][g])
    for v in (np.nan, np.inf, 0.0, -0.0, -0.25):
        h.make_room(1)
        h.edit([("secure_price", g, v), ("community_price", g, v)], f"{label}: listed price {v}")
        h.tick(f"{label}: a listed offer's price {v}")
    h.make_room(1)
    h.edit([("secure_price", g, keep[0]), ("community_price", g, keep[1])], f"{label}: price back")
    # re-seeded between a refresh and its tick: identical columns, and columns of other rows
    pend, rows, _ = h.lists()
    same = np.sort(h.rng.choice(pend, 1000, replace=False)).astype(np.uint32)
    other = np.sort(h.rng.choice(np.setdiff1d(pend, same), 1000, replace=False)).astype(np.uint32)
    h.seed(same, h.gm.rows(same))
    donor = np.sort(h.rng.choice(h.N, 1000, replace=False))
    h.seed(other, h.gm.rows(donor))
    h.tick(f"{label}: price back, re-seeded rows")
    # a listed offer made infeasible by its flags, then by its mem
    g = h.most_listed()
    h.make_room(2)
    h.edit([("flags", g, 0)], f"{label}: flags off")
    h.tick(f"{label}: a listed offer's flags off")
    g2 = h.most_listed()
    h.edit([("mem_gb", g2, h.offers["mem_gb"].min())], f"{label}: mem down")
    h.tick(f"{label}: a listed offer's mem at the table's least")
    # an unlisted offer becomes feasible and cheap for rows with short lists
    pos = np.concatenate([h.offers["secure_price"], h.offers["community_price"]])
    pos = pos[np.isfinite(pos) & (pos > 0)]
    if len(pos) and h.unlisted():
        h.make_room(1)
        h.edit(h.reachable(h.unlisted()[-1], float(pos.min())), f"{label}: a far offer")
        h.tick(f"{label}: a far offer feasible and cheapest")
    # mem / vcpu / ram at req - 1, req and req + 1 of many rows
    _, rows, _ = h.lists()
    gs = h.unlisted(3) or [h.most_listed()] * 3
    for d in (-1, 0, 1):
        edits = []
        for (col, req), g in zip((("mem_gb", "req_mem_gb"), ("vcpu", "req_vcpu"), ("ram_gb", "req_ram_gb")), gs):
            if h.offers.get(col) is None:
                continue
            vals, cnt = np.unique(rows[req], return_counts=True)
            v = int(vals[cnt.argmax()])  # the request of the most rows
            edits.append((col, g, int(np.clip(v + d, -2**31, 2**31 - 2))))
        edits += [("flags", g, 3) for g in gs] + [(c, g, float(pos.min()) if len(pos) else 0.01) for g in gs
                                                   for c in ("secure_price", "community_price")]
        h.make_room(len(set(gs)))
        h.edit(edits, f"{label}: columns at req {d:+d}")
        h.tick(f"{label}: offer columns at req {d:+d} of many rows")
    assert h.tick(f"{label}: steady at the end") == 0


TABLES_B = ["synth300", "classes4224", "stride64", "packed_only", "full_int32"]


@pytest.mark.parametrize("n", [1, 3])
@pytest.mark.parametrize("name", TABLES_B)
def test_reach_edges(name, n):
    """(b) on the device form of n ranks, their host-sync twins and the reference ctx"""
    h = Hist(sc.table(name), sc.pods_for(name, N, seed=5), n=n, seed=n)
    try:
        reach_history(h, f"{name} n={n}")
    finally:
        h.close()


def test_reach_edges_on_three_shards_of_one_gpu():
    """(e) one history on a 3-shard ctx: each shard diffs its own replica and the host merges the lists"""
    h = Hist(sc.table("synth300"), sc.pods_for("synth300", N, seed=6), kind="shards", n=3, seed=33)
    try:
        reach_history(h, "3 shards")
    finally:
        h.close()


def test_empty_table():
    """G = 0: every list is five -1, a G = 0 refresh changes nothing, and a table after it reaches every row"""
    for n in (1, 3):
        h = Hist(sc.table("empty"), sc.pods_for("synth300", N, seed=7), n=n, seed=70 + n)
        try:
            h.tick(f"empty n={n}: first call")
            assert (h.m.top5[h.gm.pending_slots()] == -1).all()
            assert h.refresh(sc.table("empty")) == 0
            assert h.tick(f"empty n={n}: G = 0 refreshed") == 0
            assert h.refresh(sc.table("synth300")) == WHOLESALE
            h.tick(f"empty n={n}: a table after the empty one")
            assert h.refresh(sc.table("empty")) == WHOLESALE
            h.tick(f"empty n={n}: empty again")
        finally:
            h.close()


# ---- (c) refreshes that change the view -----------------------------------------------------------------------------
def words(eng):
    st = eng.stats()
    return st["distinct_mem"] + st["distinct_vcpu"] + st["distinct_ram"] + 3


@pytest.mark.parametrize("n", [1, 3])
def test_refreshes_that_change_the_view(n):
    """one-offer mem edits that take the bit-sliced rows from 32 to 33 words (stride 64), past 64 (no bit-sliced view:
    the wide reselect) and back, and RPK_FORCE_KERNEL differing between the upload and the refresh"""
    t32 = sc.distinct_table(4000, 15, 7, 7, 15)  # 16 + 8 + 8 = 32 threshold words
    pods = sc.pods_for("synth300", N, seed=8)
    pods["req_mem_gb"] = np.random.default_rng(8).choice(sc._around(t32["mem_gb"]), N).astype(np.int32)
    h = Hist(t32, pods, n=n, seed=80 + n)
    try:
        h.tick("32 words: first call")
        assert words(h.ref) == 32
        g = h.most_listed()
        was = int(h.offers["mem_gb"][g])
        h.edit([("mem_gb", g, 1000)], "33 words")
        assert words(h.ref) == 33
        h.tick("32 -> 33 words")
        h.edit([("mem_gb", g, was)], "back to 32")
        assert words(h.ref) == 32
        h.tick("33 -> 32 words")
        t64 = sc.distinct_table(4000, 47, 7, 7, 47)  # 48 + 8 + 8 = 64
        h.upload(t64)
        assert words(h.ref) == 64
        h.tick("64 words: upload")
        g = h.most_listed()
        was = int(h.offers["mem_gb"][g])
        h.edit([("mem_gb", g, 1001)], "65 words")
        assert words(h.ref) == 65 and h.ref.stats()["select_kernel_kind"] != 4
        h.tick("64 -> 65 words: no bit-sliced view")
        h.edit([("mem_gb", g, was)], "back to 64")
        assert words(h.ref) == 64 and h.ref.stats()["select_kernel_kind"] == 4
        h.tick("65 -> 64 words")
        h.upload(t32)
        h.tick("32 words again")
        for force in ("generic", "packed", None, "generic"):
            g = h.most_listed()
            h.edit([("secure_price", g, h.offers["secure_price"][g] * 1.5 + 0.01)], f"refreshed with {force}", force=force)
            h.tick(f"a refresh with RPK_FORCE_KERNEL={force}")
    finally:
        h.close()


# ---- (a) the diff ----------------------------------------------------------------------------------------------------
def test_diff_indices_and_table_sizes():
    """changed offers at warp and CTA edges of tables of 1 .. 20k offers; n_offers_changed is the model's"""
    pods = rpk.synth.make_pods(20_000, seed=9)
    for G in (1, 255, 257, 3000, 20_000):
        h = Hist(rpk.synth.make_offers(G, correlated=True), pods, kind="host", n_pend=5000, N_slots=20_000, seed=G)
        try:
            h.tick(f"G={G}: first call")
            idx = sorted({i for i in (0, 31, 32, 255, 256, G - 1) if i < G})
            assert h.edit([("mem_gb", i, h.offers["mem_gb"][i] + 1) for i in idx], f"G={G}: {idx}") == len(idx)
            h.tick(f"G={G}: offers {idx}")
            if G == 20_000:
                spread = list(range(0, 256 * 16, 256))  # one per CTA
                assert h.refresh(copy(h.offers)) == 0
                h.upload(copy(h.offers))
                h.tick("an upload")
                assert h.edit([("vcpu", i, h.offers["vcpu"][i] + 1) for i in spread], "16 spread") == 16
                h.tick("16 offers, one per CTA")
                assert h.edit([("vcpu", i, h.offers["vcpu"][i] + 1) for i in range(3, 256 * 17, 256)], "17 spread") == WHOLESALE
                h.tick("17 offers: wholesale")
                assert h.edit([("ram_gb", i, 7) for i in range(0, G, 37)], "hundreds") == WHOLESALE
                assert h.edit([("ram_gb", 5, 9)], "one after hundreds") == 1
                h.tick("one offer after several hundred: the state words were cleared")
        finally:
            h.close()


def test_diff_bit_patterns():
    """prices compared as bit patterns, absent vcpu / ram equal to explicit zeros, extreme mem values, a refused
    refresh, and several refreshes between ticks"""
    base = rpk.synth.make_offers(3000, correlated=True)
    base["vcpu"] = base["ram_gb"] = None
    h = Hist(base, rpk.synth.make_pods(20_000, seed=10), kind="host", n_pend=5000, N_slots=20_000, seed=10)
    try:
        h.tick("first call")
        g = h.most_listed()
        both = ("secure_price", "community_price")
        assert h.edit([(c, g, 0.0) for c in both], "0.0") == 1
        h.tick("a listed offer's prices to 0.0")
        assert h.edit([(c, g, -0.0) for c in both], "-0.0") == 1, "0.0 -> -0.0 is a change"
        assert h.tick("0.0 -> -0.0") == 0, "0.0 -> -0.0 reaches no row"
        assert h.edit([("secure_price", g, np.nan)], "NaN") == 1
        h.tick("NaN")
        assert h.refresh(copy(h.offers)) == 0, "the same NaN is no change"
        new = copy(h.offers)
        new["secure_price"].view(np.uint64)[g] = np.uint64(0x7FF8000000000001)
        assert h.refresh(new) == 1, "a NaN with another payload is a change"
        h.tick("another NaN payload")
        u = h.unlisted(4)
        assert h.edit([("secure_price", u[0], 5e-324), ("community_price", u[1], np.inf), ("secure_price", u[2], -np.inf),
                       ("community_price", u[3], -0.5)], "tiny / inf / negative") == 4
        h.tick("5e-324, +Inf, -Inf and a negative price")
        g = h.most_listed()
        assert h.edit([("flags", g, h.offers["flags"][g] ^ 2)], "the other cloud's bit") == 1
        h.tick("flags: the community bit toggled")
        zeros = copy(h.offers)
        zeros["vcpu"], zeros["ram_gb"] = np.zeros(3000, np.int32), np.zeros(3000, np.int32)
        assert h.refresh(zeros) == 0, "absent vcpu / ram and explicit zeros are the same table"
        zeros["ram_gb"][g] = 8
        assert h.refresh(zeros) == 1
        h.tick("ram from absent to 8")
        h.upload(copy(h.offers))
        h.tick("an upload")
        for v in (-2**31, 2**31 - 2):
            assert h.edit([("mem_gb", g, v)], f"mem {v}") == 1
            h.tick(f"mem at {v}")
        bad = copy(h.offers)
        bad["mem_gb"][7] = 2**31 - 1
        for e in h.engines:
            with pytest.raises(rpk.RpkError) as ei:
                e.refresh_offers(bad)
            assert ei.value.code == EINVAL
        h.tick("after a refused refresh")
        h.upload(copy(h.offers))
        h.tick("an upload")
        a = h.unlisted(16)
        assert h.edit([("vcpu", i, 1) for i in a[:8]], "8") == 8
        assert h.edit([("vcpu", i, 2) for i in a[7:15]], "8 more, one again") == 8
        assert len(h.gm.window) == 15
        assert h.edit([("vcpu", a[0], 3)], "the first again") == 1
        h.tick("three refreshes without a tick: 15 offers in the window")
        h.upload(copy(h.offers))
        h.tick("an upload")
        assert h.edit([("vcpu", i, 4) for i in a[:8]], "8") == 8
        assert h.edit([("vcpu", i, 5) for i in a[8:16]], "8 more") == 8
        h.tick("8 + 8: the window at capacity")
        assert h.edit([("vcpu", i, 6) for i in h.unlisted(40)[16:25]], "9 more") == WHOLESALE
        h.tick("8 + 8 + 9: wholesale")
    finally:
        h.close()
