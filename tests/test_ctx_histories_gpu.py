"""GPU tests of whole-ctx call histories against ctx_model.py: every call's output is checked against the model and the
oracle, across offer refreshes, pod-table grows and resets, status-table grows and sweeps.

Each program is a seeded sequence of about 150 steps drawn from one menu:
- offers: uploads of a synth table (rows of 32 threshold words), a 64-word bitmap table, a packed-only table, the synth
  table without its bit-sliced view ("wide"), an empty table and a table of another G; refreshes that change nothing, 1-16
  offers (inside the change window), 17 or more (wholesale), offers that take every column of the fifth entry L[4] of
  stored lists (so they tie with it on price, below or above it in index order), offers with mem values the view has
  never held (more threshold words) and a table of another G;
- pod table: rpk_pods_reset and rpk_pods_grow to sizes on and beside the 16-slot units and the shard cuts, inside the
  25 % spare capacity and past it; seeds with identical columns, NaN, -0.0, 0.0 and +inf max_price, cloud bytes 2 and
  255; marks;
- selects: host, _device, _slots, _slots_device and select_pending, row by row against the oracle over the model's
  rows; rpk_select_pending_changed in its host, _gather and _device_gather forms, where n_pending, n_reselected (the
  model's stale set), the reported slots (those whose oracle list differs from the stored one) and best and top-5 must
  equal the model's;
- status: reset, grow, seed, seed_slots, diff with codes and hashes, diff_slots, diff_device on a caller-owned column
  that grows with the table, and rpk_tick with no pods and with pods.

The programs run on a one-shard ctx (every pending form on one ctx), on 2- and 3-shard ctxs on one GPU, and on groups of
R = 1, 2, 3 one-GPU ctxs called as the ranks of the one-process-per-GPU forms (one group per form, the same history).
A failure names the step and prints the program's step log."""
import functools

import numpy as np
import pytest

import ctx_model
import offers_refresh_model as orm
import oracle
import rpk
import select_plan_cases as sc
from test_offers_refresh_gpu import shared_device
from test_select_pending_changed_device_gather_gpu import result_range, view_kind
from test_select_pending_changed_gpu import call

pytestmark = pytest.mark.gpu

N_MAX = 50_000
SENT = 0x5A5A5A5A

TABLES = {
    "synth": lambda: rpk.synth.make_offers(3000, correlated=True),  # 28 threshold words: rows of 32
    "bitmap64": lambda: sc.distinct_table(4000, 20, 10, 10, 20),   # 43 words: rows of 64
    "packed": lambda: sc.distinct_table(3000, 61, 10, 10, 61),     # 84 words: no bit-sliced view
    "wide": lambda: rpk.synth.make_offers(3000, correlated=True),  # uploaded under RPK_FORCE_KERNEL=generic
    "empty": sc.empty_table,
    "other_G": lambda: rpk.synth.make_offers(2999, seed=5, correlated=True),
}
FORCE = {"wide": "generic"}


@functools.cache
def base_table(name):
    return TABLES[name]()


def words(stats):
    """threshold words of the offer view"""
    return stats["distinct_mem"] + stats["distinct_vcpu"] + stats["distinct_ram"] + 3


class Group:
    """R one-GPU ctxs called as the ranks of one group through the _gather or the _device_gather form"""

    def __init__(self, form, engines, cap):
        import torch

        self.form, self.engines, self.cap, R = form, engines, cap, len(engines)
        self.words = engines[0].results_xchg_bytes(R, cap) // 4
        self.mem = [torch.full((self.words,), SENT, dtype=torch.int32, device="cuda") for _ in range(R)]
        self.ptrs = [m.data_ptr() for m in self.mem]
        self.flags = torch.zeros((R, 64), dtype=torch.int32, device="cuda")
        self.counts = torch.full((R, 2), SENT, dtype=torch.int32, device="cuda")
        for r, e in enumerate(engines):
            e.peer_bind([self.flags[k].data_ptr() for k in range(R)], r)

    def tick(self):
        """one call of every rank -> [(n_pending, n_reselected, slots, best, top5)] by rank"""
        import torch

        R = len(self.engines)
        for m in self.mem:
            m.fill_(SENT)
        self.counts.fill_(SENT)
        torch.cuda.synchronize()
        counts = []
        for r, e in enumerate(self.engines):
            if self.form == "gather":
                counts.append(e.select_pending_changed_gather(self.ptrs, self.cap, r))
            else:
                e.select_pending_changed_device_gather(self.ptrs, self.cap, r, d_counts=self.counts[r])
        torch.cuda.synchronize()
        if self.form != "gather":
            counts = [tuple(int(x) for x in c) for c in self.counts.cpu().numpy()]
        for o in range(1, R):
            assert torch.equal(self.mem[o], self.mem[0]), f"{self.form}: exchange buffer {o} differs from buffer 0"
        w = self.mem[0].cpu().numpy()
        return [counts[r] + rpk.results_region(w, R, self.cap, r) for r in range(R)]


class Program:
    """one seeded history on the ctxs of one configuration, checked against one ctx_model.Ctx"""

    def __init__(self, config, n, seed):
        self.config, self.n, self.seed = config, n, seed
        self.rng = np.random.default_rng(seed * 1000 + n * 10 + {"one": 1, "shards": 2, "ranks": 3}[config])
        self.log = []
        self.model = ctx_model.Ctx()
        self.groups = []
        if config == "one":
            self.engines = [rpk.Engine(1)]
            self.forms = ["host", "gather", "device_gather"]
            self.groups = [Group("gather", self.engines, N_MAX), Group("device_gather", self.engines, N_MAX)]
        elif config == "shards":
            with shared_device():
                self.engines = [rpk.Engine(device_ids=[0] * n)]
            self.forms = ["host"]
        else:
            cap = max(hi - lo for lo, hi in (result_range(N_MAX, n, r) for r in range(n)))
            self.engines = [rpk.Engine(1) for _ in range(2 * n)]
            self.groups = [Group("gather", self.engines[:n], cap), Group("device_gather", self.engines[n:], cap)]
            self.forms = ["ranks"]
        self.main = self.engines[0]  # the ctx the status table lives on
        self.units = n  # shards or ranks: the sizes around their cuts matter
        self.stride = (16, 32, 64)[seed % 3]
        self.sweep = 0
        self.table = None
        self.dev = None  # the caller-owned hash column of status_diff_device
        self.counted = dict.fromkeys(["window", "wholesale", "tie", "grow", "reported", "kept"], 0)

    def close(self):
        self.groups = []
        for e in self.engines:
            e.close()

    def history(self, fn):
        return [fn(e) for e in self.engines]

    def check(self, ok, what):
        if not ok:
            raise AssertionError(what)

    # -- offers --------------------------------------------------------------------------------------------------
    def upload(self, name):
        self.table = name
        offers = ctx_model.copy_table(base_table(name))
        with view_kind(FORCE.get(name, "auto")):
            self.history(lambda e: e.upload_offers(offers))
        self.model.upload(offers)
        self.log[-1] += f" {name} G={len(offers['mem_gb'])}"

    def refresh(self, kind):
        rng, offers = self.rng, self.model.offers
        G = len(offers["mem_gb"])
        if kind == "other_G" or G == 0:
            kind = "other_G"
            self.table = "other_G" if G == len(base_table("synth")["mem_gb"]) else "synth"
            new = ctx_model.copy_table(base_table(self.table))
        elif kind == "identical":
            new = ctx_model.copy_table(offers)
        elif kind == "window":
            new = ctx_model.edit_offers(rng, offers, int(rng.integers(1, 17)))
        elif kind == "wholesale":
            new = ctx_model.edit_offers(rng, offers, int(rng.integers(17, 41)))
        elif kind == "tie":
            new, pairs = ctx_model.tie_edit(rng, offers, self.model.stored_full_lists(), n_pairs=4)
            self.log[-1] += f" pairs (c, L[4]) {pairs}"
        else:  # layout
            new = ctx_model.layout_edit(rng, offers, int(rng.integers(1, 17)))
        before = words(self.main.stats())
        with view_kind(FORCE.get(self.table, "auto")):
            got = self.history(lambda e: e.refresh_offers(new))
        want = self.model.refresh(new)
        after = words(self.main.stats())
        self.log[-1] += f" {kind} -> {'wholesale' if want == orm.WHOLESALE else want} (view words {before} -> {after})"
        self.check(all(n == want for n in got), f"n_offers_changed {got}, the model says {want}")
        self.counted["wholesale" if want == orm.WHOLESALE else "window"] += 1
        self.counted["tie"] += kind == "tie"

    # -- pod table -----------------------------------------------------------------------------------------------
    def sizes_near(self, N):
        """sizes on and beside the 16-slot units, the shard cuts, and 25 % and 100 % above N"""
        k = N // 16
        out = {15, 16, 17, 16 * self.units - 1, 16 * self.units + 1, N + 1, 16 * (k + 1) - 1, 16 * (k + 1),
               16 * (k + 1) + 1, 16 * (k + 2), 16 * (k + self.units) + 1, N + N // 5, 2 * N + 1}
        return sorted(out)

    def pods_reset(self):
        """a reset to a size around the cuts or a random one, then every row seeded and about a third marked"""
        rng = self.rng
        small = [15, 16, 17, 16 * self.units - 1, 16 * self.units + 1]
        N = int(rng.choice(small)) if rng.random() < 0.4 else int(rng.integers(2000, 30_000))
        self.history(lambda e: e.pods_reset(N))
        self.model.pods_reset(N)
        every = np.arange(N, dtype=np.uint32)
        rows = ctx_model.odd_rows(rng, self.model.offers, N)
        flags = (rng.random(N) < 0.3).astype(np.uint8)
        self.history(lambda e: e.pods_seed_slots(every, rows))
        self.history(lambda e: e.pods_mark_pending(every, flags))
        self.model.seed(every, rows)
        self.model.mark(every, flags)
        self.log[-1] += f" N={N}, {int(flags.sum())} marked"

    def pods_grow(self):
        N0 = self.model.N
        grow = [c for c in self.sizes_near(N0) if N0 < c <= N_MAX]
        if not grow:
            return self.pods_reset()
        N = int(self.rng.choice(grow))
        self.history(lambda e: e.pods_grow(N))
        # the one-process-per-GPU ranks of a group of more than one clear their results
        self.model.pods_grow(N, keep_results=not (self.config == "ranks" and self.n > 1))
        self.counted["grow"] += 1
        self.log[-1] += f" {N0} -> {N}"

    def some_slots(self, most):
        N = self.model.N
        sl = self.rng.choice(N, int(self.rng.integers(1, min(N, most) + 1)), replace=False)
        return np.sort(sl).astype(np.uint32)

    def seed_rows(self):
        sl = self.some_slots(4000)
        same = self.rng.random() < 0.3
        rows = self.model.rows(sl) if same else ctx_model.odd_rows(self.rng, self.model.offers, len(sl))
        self.history(lambda e: e.pods_seed_slots(sl, rows))
        self.model.seed(sl, rows)
        self.log[-1] += f" {len(sl)} slots{' (identical columns)' if same else ''}"

    def mark(self):
        N = self.model.N
        sl = self.some_slots(N // 2 + 1)
        if self.rng.random() < 0.3:  # both sides of every cut between ranks and shards
            cuts = {b for r in range(self.units) for b in result_range(N, self.units, r)}
            sl = np.union1d(sl, [x for c in cuts for x in (c - 1, c) if 0 <= x < N]).astype(np.uint32)
        flags = (self.rng.random(len(sl)) < 0.5).astype(np.uint8)
        self.history(lambda e: e.pods_mark_pending(sl, flags))
        self.model.mark(sl, flags)
        self.log[-1] += f" {len(sl)} slots, {int(flags.sum())} set"

    # -- selects -------------------------------------------------------------------------------------------------
    def select(self, form):
        import torch

        rng, m, N = self.rng, self.model, self.model.N
        e = self.engines[int(rng.integers(0, len(self.engines)))]
        P = int(rng.choice([1, 17, 1000, 4097]))
        slots = rng.integers(0, N, P).astype(np.uint32)  # any order, repeats
        wb, wt = m.expected(slots)
        top5 = bool(rng.integers(0, 2)) or form in ("slots", "slots_device")
        self.log[-1] += f" P={P} top5={top5}"
        if form == "host":
            got = sc.run_host(e, m.rows(slots), top5)
        elif form == "device":
            got = sc.run_device(e, m.rows(slots), top5)
        elif form == "slots":
            got = e.select_slots(slots, want_top5=True, out_best=np.full(P, sc.SENTINEL, np.int32),
                                 out_top5=np.full((P, 5), sc.SENTINEL, np.int32))
        elif form == "slots_device":  # one entry outside the table: -1 and five -1
            d = torch.from_numpy(np.append(slots, N + 3).astype(np.int32)).cuda()
            d_best = torch.full((P + 1,), sc.SENTINEL, dtype=torch.int32, device="cuda")
            d_t5 = torch.full((5 * (P + 1),), sc.SENTINEL, dtype=torch.int32, device="cuda")
            torch.cuda.synchronize()
            e.select_slots_device(d, d_best, d_t5)
            torch.cuda.synchronize()
            b, t = d_best.cpu().numpy(), d_t5.cpu().numpy().reshape(-1, 5)
            self.check(b[P] == -1 and (t[P] == -1).all(), "select_slots_device: an entry outside the table is not -1")
            got = b[:P], t[:P]
        else:  # pending
            pend = m.pending()
            cap = max(N, 1)
            got_slots, b, t = e.select_pending(cap, want_top5=True)
            self.check(np.array_equal(got_slots, pend), f"select_pending: {len(got_slots)} slots, the model has {len(pend)} pending")
            wb, wt = m.expected(pend)
            got = b, t
        sc.check(f"select {form}", got[0], got[1] if top5 else None, wb, wt)

    def changed(self, form):
        """one pending tick in `form`, against the model's"""
        want = self.model.tick()
        N = self.model.N
        if form == "host":
            got = [call(e, max(N, 1)) for e in self.engines]
            ranks = [[g] for g in got]
            ranges = [[(0, N)]] * len(got)
        else:
            groups = self.groups if form == "ranks" else [g for g in self.groups if g.form == form]
            ranks = [g.tick() for g in groups]
            ranges = [[result_range(N, len(g.engines), r) for r in range(len(g.engines))] for g in groups]
        self.log[-1] += f" n_pending {len(want.pend)} stale {len(want.stale)} reported {len(want.slots)}"
        for got_group, rr, gname in zip(ranks, ranges, [form] * len(ranks) if form != "ranks" else [g.form for g in self.groups]):
            for r, (got, (lo, hi)) in enumerate(zip(got_group, rr)):
                n_p, n_r, slots, best, top5 = want.in_range(lo, hi)
                who = f"{gname} rank {r} of slots [{lo}, {hi})"
                self.check(int(got[0]) == n_p, f"{who}: n_pending {got[0]}, the model has {n_p}")
                if int(got[1]) != n_r:
                    st = want.stale[(want.stale >= lo) & (want.stale < hi)]
                    raise AssertionError(f"{who}: n_reselected {got[1]}, the model's stale set has {n_r} (first {st[:8].tolist()})")
                if not np.array_equal(np.asarray(got[2], np.uint32), slots):
                    extra, miss = np.setdiff1d(got[2], slots), np.setdiff1d(slots, got[2])
                    raise AssertionError(f"{who}: reported {len(got[2])} slots, the model {len(slots)}; "
                                         f"extra {extra[:8].tolist()}, missing {miss[:8].tolist()}")
                sc.check(f"{who}: reported rows", np.asarray(got[3]), np.asarray(got[4]).reshape(-1, 5), best, top5)
        self.counted["reported"] += len(want.slots)
        self.counted["kept"] += len(want.pend) - len(want.stale)

    # -- status --------------------------------------------------------------------------------------------------
    def records(self, N, frac):
        self.sweep += 1
        return rpk.synth.make_status_records(N, self.sweep, frac, seed=self.seed, stride=self.stride)

    def dev_column(self, N, keep):
        """the caller's hash column for status_diff_device: a new one of N slots, keeping the old one's hashes"""
        import torch

        col = torch.zeros(N, dtype=torch.int64, device="cuda")
        tab = oracle.StatusTable(N, self.stride)
        if keep and self.dev is not None:
            col[:self.dev["N"]] = self.dev["hash"]
            tab = self.dev["tab"]
            tab.grow(N)
        self.dev = {"N": N, "hash": col, "tab": tab, "idx": torch.empty(N, dtype=torch.int32, device="cuda"),
                    "code": torch.empty(N, dtype=torch.int16, device="cuda"), "n": torch.zeros(1, dtype=torch.int32, device="cuda")}

    def status(self, op):
        import torch

        rng, e, m = self.rng, self.main, self.model
        if op == "reset" or m.status is None:
            N = int(rng.choice([1, 15, 17, 16 * self.units + 1, 4096, int(rng.integers(100, 30_000))]))
            e.status_reset(N)
            m.status_reset(N, self.stride)
            self.dev_column(N, keep=False)
            self.log[-1] += f" reset N={N}"
            return
        N = m.status.N
        if op == "grow":
            grow = [c for c in self.sizes_near(N) if N < c <= N_MAX]
            N = int(rng.choice(grow)) if grow else N
            e.status_grow(N)
            m.status_grow(N)
            self.dev_column(N, keep=True)
            self.log[-1] += f" -> N={N}"
            return
        frac = float(rng.choice([0.0, 0.01, 0.2, 1.0]))
        recs = self.records(N, frac)
        self.log[-1] += f" N={N} frac={frac}"
        if op == "seed":
            e.status_seed(recs)
            m.status_seed(recs)
        elif op in ("seed_slots", "diff_slots"):
            sl = np.sort(rng.choice(N, int(rng.integers(1, N + 1)), replace=False)).astype(np.uint32)
            sub = np.ascontiguousarray(recs[sl])
            if op == "seed_slots":
                e.status_seed_slots(sl, sub)
                m.status_seed_slots(sl, sub)
            else:
                got, codes = e.status_diff_slots(sl, sub, want_codes=True)
                want = m.status_diff_slots(sl, sub)
                self.check(np.array_equal(got, want), f"status_diff_slots: {len(got)} changed, the oracle {len(want)}")
                self.check(np.array_equal(codes, oracle.record_codes(sub)[np.searchsorted(sl, want)]), "status_diff_slots: codes")
        elif op == "diff":
            got, codes, hashes = e.status_diff(recs, want_hashes=True, want_codes=True)
            want = m.status_diff(recs)
            self.check(np.array_equal(got, want), f"status_diff: {len(got)} changed, the oracle {len(want)}")
            self.check(np.array_equal(codes, oracle.record_codes(recs)[want]), "status_diff: codes")
            self.check(np.array_equal(hashes, oracle.record_hashes(recs)), "status_diff: hashes")
        elif op == "diff_device":
            d = self.dev
            d_recs = torch.from_numpy(recs).cuda()
            torch.cuda.synchronize()
            e.status_diff_device(d_recs, self.stride, d["hash"], d["idx"], d["n"], d_changed_code=d["code"])
            torch.cuda.synchronize()
            k = int(d["n"].item())
            got = d["idx"][:k].cpu().numpy().view(np.uint32)
            want = d["tab"].diff(recs)
            self.check(np.array_equal(got, want), f"status_diff_device: {k} changed, the oracle {len(want)}")
            self.check(np.array_equal(d["code"][:k].cpu().numpy().view(np.uint16), oracle.record_codes(recs)[want]), "status_diff_device: codes")
            self.check(np.array_equal(d["hash"].cpu().numpy().view(np.uint64), d["tab"].prev_hashes()), "status_diff_device: hash column")
        else:  # tick, tick_pods
            pods, wb, wt = None, None, None
            if op == "tick_pods":
                slots = rng.integers(0, self.model.N, int(rng.choice([1, 300, 5000]))).astype(np.uint32)
                pods = self.model.rows(slots)
                wb, wt = self.model.expected(slots)
            best, t5, got, codes = e.tick(pods, recs, want_top5=True)
            want = m.status_diff(recs)
            self.check(np.array_equal(got, want), f"rpk_tick: {len(got)} changed, the oracle {len(want)}")
            self.check(np.array_equal(codes, oracle.record_codes(recs)[want]), "rpk_tick: codes")
            if pods is not None:
                sc.check("rpk_tick: select", best, t5, wb, wt)

    # -- the program ---------------------------------------------------------------------------------------------
    def do(self, op, arg=None):
        self.log.append(f"{len(self.log):3d} {op}" + (f" {arg}" if arg else ""))
        try:
            {"upload": lambda: self.upload(arg), "refresh": lambda: self.refresh(arg), "pods_reset": self.pods_reset,
             "pods_grow": self.pods_grow, "seed": self.seed_rows, "mark": self.mark, "select": lambda: self.select(arg),
             "changed": lambda: self.changed(arg), "status": lambda: self.status(arg)}[op]()
        except AssertionError as err:
            raise AssertionError(f"step {len(self.log) - 1} ({op} {arg or ''}): {err}\n{self.config} n={self.n} seed={self.seed}; "
                                 "steps:\n  " + "\n  ".join(self.log)) from None

    def draw(self):
        """one step of the menu"""
        rng = self.rng
        op = str(rng.choice(["upload", "refresh", "refresh", "refresh", "refresh", "refresh", "pods_reset", "pods_grow",
                             "pods_grow", "pods_grow", "seed", "seed", "seed", "mark", "mark", "select", "select", "changed",
                             "changed", "changed", "changed", "changed", "changed", "status", "status", "status"]))
        arg = {"upload": lambda: str(rng.choice(list(TABLES))),
               "refresh": lambda: str(rng.choice(["identical", "window", "window", "window", "wholesale", "tie", "tie",
                                                  "layout", "other_G"])),
               "select": lambda: str(rng.choice(["host", "device", "slots", "slots_device", "pending"])),
               "changed": lambda: str(rng.choice(self.forms)),
               "status": lambda: str(rng.choice(["reset", "grow", "grow", "seed", "seed_slots", "diff", "diff", "diff_slots",
                                                 "diff_device", "tick", "tick_pods"]))}.get(op, lambda: None)()
        return op, arg

    def run(self, steps):
        self.do("upload", "synth")
        self.do("pods_reset")
        self.do("status", "reset")
        self.do("changed", self.forms[0])
        for _ in range(steps):
            self.do(*self.draw())
        self.do("changed", self.forms[-1])
        c = self.counted
        assert c["window"] and c["wholesale"] and c["grow"] and c["reported"] and c["kept"], (c, self.log)


def run_program(config, n, seed, steps=150):
    p = Program(config, n, seed)
    try:
        p.run(steps)
    finally:
        p.close()


@pytest.mark.parametrize("seed", range(1, 13))
def test_one_shard(seed):
    """every pending form on one ctx"""
    run_program("one", 1, seed)


@pytest.mark.parametrize("seed", range(1, 7))
@pytest.mark.parametrize("n", [2, 3])
def test_shards_on_one_gpu(n, seed):
    run_program("shards", n, seed)


@pytest.mark.parametrize("seed", range(1, 7))
@pytest.mark.parametrize("R", [1, 2, 3])
def test_ranks_of_the_device_form(R, seed):
    """R one-GPU ctxs through _device_gather, and R more through _gather, with one history"""
    run_program("ranks", R, seed)
