"""GPU tests of rpk_offers_refresh: after a refresh, rpk_select_pending_changed[_gather] reselects exactly the pending
slots a changed offer reaches (offers_refresh_model.py), and the per-slot mirror stays equal to rpk_select_slots and to
the oracle after every call."""
import contextlib
import ctypes as C
import os

import numpy as np
import pytest

import offers_refresh_model as model
import rpk
import select_plan_cases as sc
from test_select_pending_changed_gather_gpu import Group, pending_set
from test_select_pending_changed_gpu import Mirror, call, check_mirror, mark_only, step
from test_select_slots_gpu import TRACKED, seeded_engine, tracked

pytestmark = pytest.mark.gpu

EINVAL = rpk._ffi.RPK_EINVAL
WHOLESALE = 0xFFFFFFFF
DELTA_MAX = 16  # RPK_OFFERS_DELTA_MAX


class Run:
    """a seeded ctx, its pending set and mirror, and the table as the library holds it"""

    def __init__(self, name="synth20k", n_pend=40_000, seed=1, eng=None):
        self.offers = {k: (v.copy() if v is not None else None) for k, v in sc.table(name).items()}
        self.tab = tracked(name)[0]
        self.rng = np.random.default_rng(seed)
        self.eng = eng if eng is not None else seeded_engine(name)
        self.pend = mark_only(self.eng, TRACKED, np.sort(self.rng.choice(TRACKED, n_pend, replace=False)))
        self.m = Mirror(TRACKED)
        step(self.eng, self.m, TRACKED)
        self.changed = np.zeros(0, np.int64)  # offers changed since the pending slots' results were made

    def new_table(self, edits):
        new = {k: (v.copy() if v is not None else None) for k, v in self.offers.items()}
        for col, g, v in edits:
            new[col][g] = v
        return new

    def refresh(self, new, want_n=None):
        n = self.eng.refresh_offers(new)
        same_g = len(new["mem_gb"]) == len(self.offers["mem_gb"])
        diff = model.changed_offers(self.offers, new) if same_g else np.zeros(0, np.int64)
        assert n == (len(diff) if want_n is None else want_n), f"n_offers_changed {n}, {len(diff)} offers differ"
        self.changed = np.union1d(self.changed, diff)
        self.offers = new
        return n

    def tick(self, label, stale=None):
        """one call: n_reselected is the model's stale set, the reported slots those whose oracle list changed"""
        rows = self.tab.rows(self.pend)
        old_t = self.m.top5[self.pend].copy()
        if stale is None:
            stale = model.reached(self.offers, rows, old_t, self.changed)
        n_p, n_r, sl, _, _ = step(self.eng, self.m, TRACKED)
        wb, wt = sc.expected(self.offers, rows)
        assert n_p == len(self.pend) and n_r == int(stale.sum()), f"{label}: reselected {n_r}, the rule says {int(stale.sum())}"
        assert np.array_equal(sl, self.pend[(wt != old_t).any(axis=1)]), f"{label}: reported != slots whose list changed"
        check_mirror(label, self.eng, self.m, self.pend, wb, wt)
        self.changed = np.zeros(0, np.int64)
        return n_r

    def most_listed(self):
        t = self.m.top5[self.pend]
        return int(np.bincount(t[t >= 0].ravel(), minlength=len(self.offers["mem_gb"])).argmax())

    def unlisted(self):
        t = self.m.top5[self.pend]
        return int(np.setdiff1d(np.arange(len(self.offers["mem_gb"])), t[t >= 0])[0])

    def steady(self, label):
        c0 = self.eng.launch_count()
        n_p, n_r, sl, _, _ = call(self.eng, TRACKED)
        assert (n_r, len(sl)) == (0, 0), f"{label}: a steady call reselects nothing"
        assert self.eng.launch_count() == c0 + 1, f"{label}: a steady call is one launch per GPU"


def test_identical_and_single_offer_refreshes():
    r = Run()
    try:
        r.steady("before any refresh")
        assert r.refresh({k: (v.copy() if v is not None else None) for k, v in r.offers.items()}) == 0
        assert r.tick("identical refresh") == 0, "an identical refresh reselects nothing"
        g = r.most_listed()
        n_r = 0
        for col in ("secure_price", "community_price"):
            if r.offers[col][g] > 0:
                r.refresh(r.new_table([(col, g, r.offers[col][g] * 1.5)]))
                n_r = r.tick(f"{col} of the most-listed offer up")
        assert 0 < n_r < len(r.pend)
        r.steady("after a refresh")
        u = r.unlisted()
        r.refresh(r.new_table([("secure_price", u, 0.001), ("community_price", u, 0.001)]))
        r.tick("an unlisted offer down")
        r.refresh(r.new_table([("flags", g, 0)]))
        r.tick("availability off")
        r.refresh(r.new_table([("flags", g, 3)]))
        r.tick("availability on")
        r.refresh(r.new_table([("mem_gb", g, 1)]))
        r.tick("mem down")
        r.steady("after the refreshes")
        # an identical upload still reselects every pending slot
        r.eng.upload_offers(r.offers)
        r.tick("identical upload", stale=np.ones(len(r.pend), bool))
    finally:
        r.eng.close()


def test_two_refreshes_with_and_without_a_tick():
    r = Run(seed=2)
    try:
        G = len(r.offers["mem_gb"])
        a, b = (int(x) for x in r.rng.choice(G, 2, replace=False))
        r.refresh(r.new_table([("secure_price", r.most_listed(), 0.011)]))
        r.refresh(r.new_table([("secure_price", a, 0.012), ("mem_gb", b, 4096)]))
        r.tick("two refreshes, one tick")
        r.refresh(r.new_table([("secure_price", a, 0.2)]))
        r.tick("first of two ticks")
        r.refresh(r.new_table([("secure_price", a, 0.013)]))  # the same offer again
        r.tick("the same offer changed twice")
        r.steady("after")
    finally:
        r.eng.close()


def test_a_slot_that_leaves_across_a_refresh():
    r = Run(seed=3)
    try:
        away = np.sort(r.rng.choice(r.pend, 5000, replace=False))
        r.eng.pods_mark_pending(away, np.zeros(len(away), np.uint8))
        full = r.pend
        r.pend = np.setdiff1d(full, away)
        g = r.most_listed()
        r.refresh(r.new_table([("secure_price", g, 0.0105), ("community_price", g, 0.0105)]))
        changed = r.changed.copy()
        r.tick("while away")
        r.refresh(r.new_table([("mem_gb", r.unlisted(), 10_000)]))
        changed = np.union1d(changed, r.changed)
        r.eng.pods_mark_pending(away, np.ones(len(away), np.uint8))
        r.pend = full
        stale = model.reached(r.offers, r.tab.rows(full), r.m.top5[full], r.changed)
        stale |= np.isin(full, away) & model.reached(r.offers, r.tab.rows(full), r.m.top5[full], changed)
        r.tick("back", stale=stale)
        r.steady("after")
    finally:
        r.eng.close()


def test_window_capacity_other_G_upload_and_reset():
    r = Run(seed=4)
    try:
        G = len(r.offers["mem_gb"])
        gs = r.rng.choice(G, DELTA_MAX + 1, replace=False)
        r.refresh(r.new_table([("secure_price", int(g), 0.0001 * (1 + k)) for k, g in enumerate(gs[:DELTA_MAX // 2])]))
        r.refresh(r.new_table([("ram_gb", int(g), 1 << 20) for g in gs[DELTA_MAX // 2:DELTA_MAX]]))
        assert len(r.changed) == DELTA_MAX
        r.tick("a window of exactly RPK_OFFERS_DELTA_MAX")
        r.refresh(r.new_table([("vcpu", int(gs[-1]), 99)]), want_n=WHOLESALE)
        r.tick("one more: wholesale", stale=np.ones(len(r.pend), bool))
        r.refresh(r.new_table([("secure_price", r.most_listed(), 0.0102)]))
        r.tick("a refresh after the wholesale one")
        r.eng.upload_offers(r.offers)
        r.tick("an upload after a refresh", stale=np.ones(len(r.pend), bool))
        r.refresh(r.new_table([("secure_price", r.most_listed(), 0.0103)]))
        r.tick("a refresh after an upload")
        short = {k: (v[:G - 1].copy() if v is not None else None) for k, v in r.offers.items()}
        r.refresh(short, want_n=WHOLESALE)
        r.tick("another G", stale=np.ones(len(r.pend), bool))
        r.refresh({k: (v.copy() if v is not None else None) for k, v in r.offers.items()}, want_n=0)
        r.refresh(r.new_table([("secure_price", r.most_listed(), 0.0104)]))
        r.eng.pods_reset(TRACKED)
        tab, seeds = tracked("synth20k")[0], tracked("synth20k")[3]
        for slots, pods in seeds:
            r.eng.pods_seed_slots(slots, pods)
        mark_only(r.eng, TRACKED, r.pend)
        r.m = Mirror(TRACKED)
        r.tick("rpk_pods_reset after a refresh", stale=np.ones(len(r.pend), bool))
    finally:
        r.eng.close()


def test_cap_refusal_and_refresh_refusals():
    r = Run(seed=5)
    try:
        g = r.most_listed()
        r.refresh(r.new_table([("secure_price", g, 0.0106), ("community_price", g, 0.0106)]))
        stale = model.reached(r.offers, r.tab.rows(r.pend), r.m.top5[r.pend], r.changed)
        k = int(stale.sum())
        assert k > 1
        with pytest.raises(rpk.RpkError) as ei:
            r.eng.select_pending_changed(k - 1)
        assert ei.value.code == EINVAL and ei.value.n_reselected == k
        # refused refreshes leave the window and the floor alone
        lib, ctx = r.eng._lib, r.eng._ctx
        n = C.c_uint32(7)
        assert lib.rpk_offers_refresh(ctx, 5, None, None, None, None, None, None, C.cast(C.byref(n), C.c_void_p)) == EINVAL
        assert b"rpk_offers_refresh" in lib.rpk_last_error(ctx) and n.value == 7
        bad = r.new_table([("mem_gb", 0, 2**31 - 1)])
        with pytest.raises(rpk.RpkError) as ei:
            r.eng.refresh_offers(bad)
        assert ei.value.code == EINVAL and "rpk_offers_refresh" in str(ei.value)
        r.tick("retry after the refusals", stale=stale)
        r.steady("after")
    finally:
        r.eng.close()


@contextlib.contextmanager
def shared_device():
    old = os.environ.get("RPK_TEST_SHARED_DEVICE")
    os.environ["RPK_TEST_SHARED_DEVICE"] = "1"
    try:
        yield
    finally:
        if old is None:
            os.environ.pop("RPK_TEST_SHARED_DEVICE", None)
        else:
            os.environ["RPK_TEST_SHARED_DEVICE"] = old


@pytest.mark.parametrize("n", [2, 3, 4, 8])
def test_shards_on_one_gpu(n):
    with shared_device():
        eng = rpk.Engine(device_ids=[0] * n)
    eng.upload_offers(sc.table("synth20k"))
    eng.pods_reset(TRACKED)
    for slots, pods in tracked("synth20k")[3]:
        eng.pods_seed_slots(slots, pods)
    r = Run(seed=10 + n, eng=eng)
    try:
        g = r.most_listed()
        r.refresh(r.new_table([("secure_price", g, 0.0107), ("community_price", g, 0.0107)]))
        r.tick(f"{n} shards: one offer")
        r.refresh(r.new_table([("flags", r.unlisted(), 3), ("mem_gb", g, 2)]))
        r.tick(f"{n} shards: two offers")
        c0 = eng.launch_count()
        assert call(eng, TRACKED)[1] == 0 and eng.launch_count() == c0 + n, "a steady call is one launch per GPU"
    finally:
        eng.close()


@pytest.mark.parametrize("n", [1, 2, 3, 4, 8])
def test_gather_ranks_equal_the_host_call(n):
    N = 100_003
    rng = np.random.default_rng(500 + n)
    g = Group(n, N)
    try:
        offers = rpk.synth.make_offers(3000, correlated=True)
        pods = rpk.synth.make_pods(N, seed=N)
        every = np.arange(N, dtype=np.uint32)
        flags = np.zeros(N, np.uint8)
        flags[pending_set(N, n, rng, 0.3)] = 1

        def setup(e):
            e.upload_offers(offers)
            e.pods_reset(N)
            e.pods_seed_slots(every, pods)
            e.pods_mark_pending(every, flags)

        g.history(setup)
        g.step("first call")
        _, _, t5 = g.ref.select_pending(N, want_top5=True)
        used = np.bincount(t5[t5 >= 0].ravel(), minlength=3000)
        top = int(used.argmax())
        for what, edits in (("one price", [("secure_price", top, 0.0101)]),
                            ("flag off and a mem change", [("flags", top, 0), ("mem_gb", int(used.argmin()), 1 << 16)])):
            new = {k: (v.copy() if v is not None else None) for k, v in offers.items()}
            for col, i, v in edits:
                new[col][i] = v
            ns = []
            g.history(lambda e: ns.append(e.refresh_offers(new)))
            assert len(set(ns)) == 1 and ns[0] == len(model.changed_offers(offers, new))
            offers = new
            n_p, n_r, _ = g.step(what)
            assert 0 < n_r < n_p, f"{what}: {n_r} of {n_p} reselected"
            assert g.step(f"steady after {what}")[1] == 0
    finally:
        g.close()
