"""GPU tests of CUDA-graph captures of the device entry points while the other calls of their ctx run between replays.

include/rpk.h ("Graph capture") lists which calls keep a capture of a _device call valid and which invalidate it.  A
capture holds every ctx-owned device pointer the call handed its kernels, so a call on the valid side must leave all of
them where they were: rpk_test_capture_buffers lists them, and the first test checks that no call of the valid side
moves one, without replaying anything.  The other tests replay captures between those calls and compare every output
with the oracle or a model: the select results row by row (select_plan_cases.check), the sweeps against
oracle.StatusTable, the pending list against the flags, the pending results through a per-slot mirror, the fence through
its flag words, with SENTINEL past every count and outside every gathered slice.  After a call of the invalid side the
seeded programs capture again, as the contract asks; no test replays a capture the contract calls invalid.

Captures and replays on one ctx share the device scratch, so every replay's stream is synchronised before the next host
call or replay of another entry point, as rpk.h requires."""
import contextlib

import numpy as np
import pytest

import oracle
import rpk
import select_plan_cases as sc
import status_slots_model

pytestmark = pytest.mark.gpu

# rpk_test_capture_buffers' order
POD_COLS = ("mem", "vcpu", "ram", "max_price", "cloud")
LANE = ["cols.mem", "cols.vcpu", "cols.ram", "cols.max_price", "cols.cloud", "p_slots", "top5", "rw", "order", "pos", "ctrs",
        "key", "ord_rw", "hist", "k0_base", "hdr"]
NAMES = ([f"dev_lane.{b}" for b in LANE] + [f"dev_sweep.{b}" for b in ("tile_state", "misc", "stage_idx", "stage_code", "unit_cnt")]
         + [f"view{c}.{b}" for c in (0, 1) for b in ("packed", "bitmap", "bitmapT", "bitmapM", "wide", "price", "perm")]
         + ["distinct_mem", "distinct_vcpu", "distinct_ram", "raw.mem", "raw.vcpu", "raw.ram", "raw.secure_price",
            "raw.community_price", "raw.flags", "win"]
         + [f"pt_cols.{c}" for c in POD_COLS] + ["pt_pending", "pt_state", "pt_ticket"]
         + [f"r_cols.{c}" for c in POD_COLS] + ["r_gen", "r_top5", "r_list", "r_mask", "r_dn"]
         + [f"r_lane.{b}" for b in LANE])

C = 20_000         # rows of a captured select: above the fused kernel's 16 384, so the persistent path's buffers exist
POOL = 3 * C       # pod rows the tests draw from; the larger host selects take all of them
BIG = 196_609      # a host select past the first sub-batch edge
N = 40_000         # pod-table slots
ND = 30_000        # records of a captured sweep
NL = 8_000         # entries of a captured slot-list sweep
NS = 3 * ND + 7    # the host sweeps' tracked table: larger than any captured sweep
STRIDE = 32
ROW0 = 5
SLOT_SENT = 0x5A5A5A5A
ENTRIES = ["select", "select_gather", "select_gather_top5", "slots", "slots_gather", "slots_gather_top5", "pending_list",
           "status", "status_codes", "status_gather", "status_slots", "status_slots_gather", "pending_changed", "fence"]
UNBOUND = ["select", "select_gather", "slots", "slots_gather", "pending_list", "status", "status_codes", "status_gather",
           "status_slots", "pending_changed"]


def test_hook_names_every_buffer(engine):
    assert len(engine.capture_buffers()) == len(NAMES)


def moved(before, after):
    """the buffers a capture taken at `before` held that are elsewhere at `after` (a buffer allocated since is not one)"""
    return [NAMES[i] for i, (b, a) in enumerate(zip(before, after)) if b and b != a]


def t(a, dtype=None):
    import torch

    return torch.from_numpy(np.ascontiguousarray(a if dtype is None else a.astype(dtype))).cuda()


def full(n, v, dtype):
    import torch

    return torch.full((n,), v, dtype=dtype, device="cuda")


class World:
    """One ctx (shard `shard` of it) holding a capture of every entry point in `entries`, its inputs, outputs and models.
    The pod table holds rows of the pool (idx[s]: the pool row of slot s); the flags mirror is `flags`."""

    def __init__(self, eng, name, shard=0, entries=ENTRIES, n_ranks=1, my_rank=0, seed=0):
        import torch

        self.eng, self.shard, self.entries, self.n_ranks, self.my_rank = eng, shard, list(entries), n_ranks, my_rank
        self.rng = np.random.default_rng(seed)
        self.log = []
        self.set_table(name, sc.table(name), upload=True)
        eng.pods_reset(N)
        self.pods_n = N
        self.seed_all()
        eng.status_reset(NS)
        self.host_tab = oracle.StatusTable(NS, STRIDE)
        self.sweep = 0
        self.streams = {e: torch.cuda.Stream() for e in self.entries}
        self.other = torch.cuda.Stream()
        self.graphs = {}
        # outputs and caller-owned state of each entry point
        self.best = full(C + 8, sc.SENTINEL, torch.int32)
        self.top5 = full(5 * C + 8, sc.SENTINEL, torch.int32)
        self.vecs = [full(ROW0 + C + 7, sc.SENTINEL, torch.int32) for _ in range(3)]
        self.t5vecs = [full(5 * (ROW0 + C) + 9, sc.SENTINEL, torch.int32) for _ in range(3)]
        self.d_pods = {k: t(v) for k, v in self.pool_rows(0).items()}
        self.d_slots = t(np.zeros(C, np.uint32), np.int32)
        self.pl_out, self.pl_n = full(N + 8, SLOT_SENT, torch.int32), full(1, -1, torch.int32)
        self.sw = {}
        for e in ("status", "status_codes", "status_gather", "status_slots", "status_slots_gather"):
            n = NL if "slots" in e else ND
            self.sw[e] = dict(tab=oracle.StatusTable(ND, STRIDE), hash=full(ND, 0, torch.int64), n=n,
                              recs=full(n * STRIDE, 0, torch.uint8), idx=full(n + 8, SLOT_SENT, torch.int32),
                              code=full(n + 8, -1, torch.int16), cnt=full(1, -1, torch.int32),
                              slots=t(np.zeros(NL, np.uint32), np.int32), xchg=full(eng.xchg_bytes(1, n) // 4, SLOT_SENT, torch.int32),
                              sweep=0, list=None, host_recs=None)
        cap = self.pc_cap = N
        self.pc_xchg = [full(eng.results_xchg_bytes(n_ranks, cap) // 4, SLOT_SENT, torch.int32) for _ in range(n_ranks)]
        self.pc_counts = full(4, -1, torch.int32)
        self.mirror_best = np.full(N, sc.SENTINEL, np.int32)
        self.mirror_top5 = np.full((N, 5), sc.SENTINEL, np.int32)
        self.fence_flags = full(64, 0, torch.int32)
        self.fences = 0
        for e in self.entries:
            self.load(e)
        self.capture_all()

    # ---- the tables ----------------------------------------------------------------------------------------------
    def set_table(self, name, offers, upload=False, refresh=False):
        self.name, self.offers = name, offers
        self.pool = sc.pods_for(name, POOL, 0)
        self.pool_best, self.pool_top5 = sc.expected(offers, self.pool)
        self.cache = {}
        if upload:
            self.eng.upload_offers(offers)
        if refresh:
            self.eng.refresh_offers(offers)

    def pool_rows(self, k, n=C):
        return sc.head({c: None if v is None else v[k * C:] for c, v in self.pool.items()}, n)

    def seed_all(self):
        """every slot := a random pool row, and a random third of the slots pending"""
        self.idx = self.rng.integers(0, POOL, N)
        self.eng.pods_seed_slots(np.arange(N, dtype=np.uint32), {c: v[self.idx] for c, v in self.pool.items()})
        self.flags = (self.rng.random(N) < 0.33).astype(np.uint8)
        self.eng.pods_mark_pending(np.arange(N, dtype=np.uint32), self.flags)

    def slot_expect(self, slots):
        return self.pool_best[self.idx[slots]], self.pool_top5[self.idx[slots]]

    def fail(self, err):
        raise AssertionError(f"{err}\noperations on table {self.name}:\n  " + "\n  ".join(self.log[-60:]))

    # ---- the entry points: inputs, one call, checks ----------------------------------------------------------------
    def load(self, e):
        """new inputs for entry point e, written into the buffers its capture reads"""
        rng = self.rng
        if e.startswith("select"):
            k = int(rng.integers(0, 3))
            for c, v in self.pool_rows(k).items():
                self.d_pods[c].copy_(t(v))
            self.sel_k = k
        elif e.startswith("slots"):
            self.slot_list = rng.integers(0, self.pods_n, C).astype(np.uint32)
            self.d_slots.copy_(t(self.slot_list, np.int32))
        elif e in self.sw:
            s = self.sw[e]
            s["sweep"] += 1
            recs = rpk.synth.make_status_records(ND, s["sweep"], 0.3, seed=len(e), stride=STRIDE)
            if "slots" in e:
                s["list"] = np.sort(rng.choice(ND, NL, replace=False)).astype(np.uint32)
                s["slots"].copy_(t(s["list"], np.int32))
                recs = recs[s["list"]]
            s["host_recs"] = recs
            s["recs"].copy_(t(recs.reshape(-1)))
        import torch

        torch.cuda.synchronize()

    def call(self, e, stream):
        eng, sh, st = self.eng, self.shard, stream.cuda_stream
        if e == "select":
            eng.select_device(self.d_pods, self.best[:C], self.top5[:5 * C], shard=sh, stream=st)
        elif e == "select_gather":
            eng.select_device_gather(self.d_pods, [v.data_ptr() for v in self.vecs], ROW0, self.top5[:5 * C], shard=sh, stream=st)
        elif e == "select_gather_top5":
            eng.select_device_gather(self.d_pods, [v.data_ptr() for v in self.vecs], ROW0, shard=sh, stream=st,
                                     top5_ptrs=[v.data_ptr() for v in self.t5vecs])
        elif e == "slots":
            eng.select_slots_device(self.d_slots, self.best[:C], self.top5[:5 * C], shard=sh, stream=st)
        elif e == "slots_gather":
            eng.select_slots_device_gather(self.d_slots, [v.data_ptr() for v in self.vecs], ROW0, self.top5[:5 * C], shard=sh, stream=st)
        elif e == "slots_gather_top5":
            eng.select_slots_device_gather(self.d_slots, [v.data_ptr() for v in self.vecs], ROW0, shard=sh, stream=st,
                                           top5_ptrs=[v.data_ptr() for v in self.t5vecs])
        elif e == "pending_list":
            eng.pods_pending_list_device(self.pl_out, self.pl_n, shard=sh, stream=st)
        elif e == "status":  # the call without codes, straight through the C-ABI
            s = self.sw[e]
            eng._check(eng._lib.rpk_status_diff_device(eng._ctx, sh, ND, s["recs"].data_ptr(), STRIDE, s["hash"].data_ptr(),
                                                       s["idx"].data_ptr(), s["cnt"].data_ptr(), st))
        elif e == "status_codes":
            s = self.sw[e]
            eng.status_diff_device(s["recs"], STRIDE, s["hash"], s["idx"][:ND], s["cnt"], shard=sh, stream=st, d_changed_code=s["code"][:ND])
        elif e == "status_gather":
            s = self.sw[e]
            eng.status_diff_device_gather(s["recs"], STRIDE, s["hash"], 0, [s["xchg"].data_ptr()], ND, 0, s["cnt"], shard=sh, stream=st)
        elif e == "status_slots":
            s = self.sw[e]
            eng.status_diff_slots_device(s["slots"], s["recs"], STRIDE, s["hash"], s["idx"][:NL], s["cnt"], 0,
                                         d_changed_code=s["code"][:NL], shard=sh, stream=st)
        elif e == "status_slots_gather":
            s = self.sw[e]
            eng.status_diff_slots_device_gather(s["slots"], s["recs"], STRIDE, s["hash"], 0, [s["xchg"].data_ptr()], NL, 0, s["cnt"],
                                                shard=sh, stream=st)
        elif e == "pending_changed":
            eng.select_pending_changed_device_gather([x.data_ptr() for x in self.pc_xchg], self.pc_cap, self.my_rank,
                                                     d_counts=self.pc_counts[:2], shard=sh, stream=st)
        elif e == "fence":
            eng.peer_fence([self.fence_flags.data_ptr()], 0, 0, shard=sh, stream=st)
        else:
            raise ValueError(e)

    def reset_outputs(self, e):
        if e.startswith(("select", "slots")):
            for b in [self.best, self.top5] + self.vecs + self.t5vecs:
                b.fill_(sc.SENTINEL)
        elif e == "pending_list":
            self.pl_out.fill_(SLOT_SENT)
            self.pl_n.fill_(-1)
        elif e in self.sw:
            s = self.sw[e]
            for b in ("idx", "xchg"):
                s[b].fill_(SLOT_SENT)
            s["code"].fill_(-1)
            s["cnt"].fill_(-1)
        elif e == "pending_changed":
            for x in self.pc_xchg:
                x.fill_(SLOT_SENT)
            self.pc_counts.fill_(-1)

    def check(self, e, label):
        """the outputs of one execution of e (its replay or its eager call) against the oracle or the model"""
        if e.startswith(("select", "slots")):
            wb, wt = ((self.pool_best[self.sel_k * C:(self.sel_k + 1) * C], self.pool_top5[self.sel_k * C:(self.sel_k + 1) * C])
                      if e.startswith("select") else self.slot_expect(self.slot_list))
            if "gather" in e:
                host = [v.cpu().numpy() for v in self.vecs]
                for i, h in enumerate(host):
                    if not ((h[:ROW0] == sc.SENTINEL).all() and (h[ROW0 + C:] == sc.SENTINEL).all()):
                        self.fail(f"{label}: gather vector {i} written outside its slice")
                    sc.check(f"{label} vector {i}", h[ROW0:ROW0 + C], None, wb, wt)
            else:
                b = self.best.cpu().numpy()
                if not (b[C:] == sc.SENTINEL).all():
                    self.fail(f"{label}: best written past row {C}")
                sc.check(label, b[:C], None, wb, wt)
            if e.endswith("top5"):
                for i, v in enumerate(self.t5vecs):
                    h = v.cpu().numpy()
                    if not ((h[:5 * ROW0] == sc.SENTINEL).all() and (h[5 * (ROW0 + C):] == sc.SENTINEL).all()):
                        self.fail(f"{label}: top-5 vector {i} written outside its slice")
                    sc.check(f"{label} top-5 vector {i}", wb, h[5 * ROW0:5 * (ROW0 + C)].reshape(C, 5), wb, wt)
                if not (self.top5.cpu().numpy() == sc.SENTINEL).all():
                    self.fail(f"{label}: the local top-5 vector was written")
            else:
                t5 = self.top5.cpu().numpy()
                if not (t5[5 * C:] == sc.SENTINEL).all():
                    self.fail(f"{label}: top5 written past row {C}")
                sc.check(label, wb, t5[:5 * C].reshape(C, 5), wb, wt)
        elif e == "pending_list":
            out, n = self.pl_out.cpu().numpy().view(np.uint32), int(self.pl_n.item())
            want = np.flatnonzero(self.flags[:self.pods_n]).astype(np.uint32)
            if n != len(want) or not np.array_equal(out[:n], want) or not (out[n:] == SLOT_SENT).all():
                self.fail(f"{label}: pending list of {n} slots, flags hold {len(want)}")
        elif e in self.sw:
            s = self.sw[e]
            recs = s["host_recs"]
            want = (status_slots_model.diff_slots(s["tab"], s["list"], recs) if "slots" in e else s["tab"].diff(recs))
            codes = oracle.record_codes(recs)
            want_codes = codes[np.searchsorted(s["list"], want)] if "slots" in e else codes[want]
            n = int(s["cnt"].item())
            if "gather" in e:
                w = s["xchg"].cpu().numpy()
                cap = s["n"]
                got = w[8:8 + cap].view(np.uint32)
                got_codes = w[8 + cap:].view(np.uint16)[:cap]
                if int(w[0]) != n or not (w[1:8] == SLOT_SENT).all():
                    self.fail(f"{label}: exchange count {int(w[0])}, d_n_changed {n}, or a foreign count word written")
            else:
                got, got_codes = s["idx"].cpu().numpy().view(np.uint32), s["code"].cpu().numpy().view(np.uint16)
            if n != len(want) or not np.array_equal(got[:n], want):
                self.fail(f"{label}: {n} changed slots, model {len(want)}")
            if not (got[n:s["n"]] == SLOT_SENT).all():
                self.fail(f"{label}: changed list written past its count")
            if e != "status" and not np.array_equal(got_codes[:n], want_codes):
                self.fail(f"{label}: codes differ from record_codes")
        elif e == "pending_changed":
            w = self.pc_xchg[0].cpu().numpy()
            r = self.my_rank
            slots, best, top5 = rpk.results_region(w, self.n_ranks, self.pc_cap, r)
            counts = self.pc_counts.cpu().numpy()
            lo, hi = self.result_range()
            n_pend = int(self.flags[lo:hi].sum())
            if int(counts[0]) != n_pend or not len(slots) <= counts[1] <= counts[0] or (counts[2:] != -1).any():
                self.fail(f"{label}: counts {counts.tolist()}, {n_pend} pending, {len(slots)} reported")
            if len(slots) and (slots.min() < lo or slots.max() >= hi):
                self.fail(f"{label}: a reported slot outside [{lo}, {hi})")
            for x in self.pc_xchg[1:]:
                if not np.array_equal(x.cpu().numpy(), w):
                    self.fail(f"{label}: exchange buffers differ")
            self.apply(slots, best, top5, label)
            self.check_mirror(label, lo, hi)
        elif e == "fence":
            f = self.fence_flags.cpu().numpy()
            if int(f[32]) != self.fences or int(f[0]) != self.fences:
                self.fail(f"{label}: fence words {int(f[0])}, {int(f[32])} after {self.fences} fences")

    def result_range(self):
        units = (self.pods_n + 15) // 16
        lo = min(units * self.my_rank // self.n_ranks * 16, self.pods_n)
        hi = min(units * (self.my_rank + 1) // self.n_ranks * 16, self.pods_n)
        return lo, hi

    def apply(self, slots, best, top5, label):
        if np.any(np.diff(slots.astype(np.int64)) <= 0) or not np.array_equal(best, top5[:, 0]):
            self.fail(f"{label}: reported rows not ascending, or best is not top5[:, 0]")
        self.mirror_best[slots], self.mirror_top5[slots] = best, top5

    def check_mirror(self, label, lo=0, hi=None):
        pend = lo + np.flatnonzero(self.flags[lo:hi if hi is not None else self.pods_n])
        wb, wt = self.slot_expect(pend)
        sc.check(f"{label}: pending results mirror", self.mirror_best[pend], self.mirror_top5[pend], wb, wt)

    def execute(self, e, how):
        """one execution of e -- its graph's replay or an eager call on its stream -- checked"""
        import torch

        self.reset_outputs(e)
        torch.cuda.synchronize()
        if how == "replay":
            self.graphs[e].replay()
        else:
            self.call(e, self.streams[e])
        self.fences += e == "fence"
        torch.cuda.synchronize()
        self.check(e, f"{e} {how}")

    def capture(self, e):
        """one eager call (checked), then the capture of the same call on e's own stream"""
        import torch

        self.load(e)
        self.execute(e, "eager")
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=self.streams[e], capture_error_mode="relaxed"):
            self.call(e, self.streams[e])
        torch.cuda.synchronize()
        self.graphs[e] = g
        self.log.append(f"capture {e}")

    def capture_all(self):
        for e in self.entries:
            self.capture(e)

    def replay_all(self, step):
        """new inputs into every capture, two replays and one eager call of each, every one checked"""
        for e in self.entries:
            self.load(e)
            for how in ("replay", "replay", "eager"):
                try:
                    self.execute(e, how)
                except AssertionError as err:
                    self.fail(f"after {step}: {err}")

    # ---- the calls that keep a capture valid, each checked ----------------------------------------------------
    def batch(self, P, nulls=False):
        """(pods, oracle best, oracle top5) of P rows under the resident offers: the pool's first rows, or the table's
        shared batch of select_plan_cases above the pool's size"""
        if (P, nulls) not in self.cache:
            if P <= POOL and not nulls:
                self.cache[P, nulls] = (sc.head(self.pool, P), self.pool_best[:P], self.pool_top5[:P])
            else:
                pods = sc.head(self.pool, P) if P <= POOL else sc.batch(self.name, P)[0]
                pods = sc.without_optional(pods) if nulls else pods
                self.cache[P, nulls] = (pods,) + tuple(sc.expected(self.offers, pods))
        return self.cache[P, nulls]

    def host_select(self, P, top5, nulls):
        pods, wb, wt = self.batch(P, nulls)
        sc.check(f"host select P={P}", *sc.run_host(self.eng, pods, top5), wb, wt if top5 else None)

    def host_slots(self, n, top5):
        slots = self.rng.integers(0, self.pods_n, n).astype(np.uint32)
        best = np.full(n, sc.SENTINEL, np.int32)
        t5 = np.full((n, 5), sc.SENTINEL, np.int32) if top5 else None
        self.eng.select_slots(slots, want_top5=top5, out_best=best, out_top5=t5)
        wb, wt = self.slot_expect(slots)
        sc.check(f"select_slots n={n}", best, t5, wb, wt if top5 else None)

    def host_pending(self):
        got_slots, best, t5 = self.eng.select_pending(self.pods_n, want_top5=True)
        want = np.flatnonzero(self.flags).astype(np.uint32)
        if not np.array_equal(got_slots, want):
            self.fail("select_pending: the pending list differs from the flags")
        sc.check("select_pending", best, t5, *self.slot_expect(want))

    def host_pending_changed(self):
        n_p, n_r, slots, best, t5 = self.eng.select_pending_changed(self.pods_n)
        if n_p != int(self.flags.sum()) or not len(slots) <= n_r <= n_p:
            self.fail(f"select_pending_changed: n_pending {n_p}, n_reselected {n_r}, {len(slots)} reported")
        self.apply(slots, best, t5, "select_pending_changed")
        self.check_mirror("select_pending_changed")

    def host_records(self, frac=0.2):
        self.sweep += 1
        return rpk.synth.make_status_records(NS, self.sweep, frac, seed=11, stride=STRIDE)

    def host_sweep(self):
        recs = self.host_records()
        idx, codes, _ = self.eng.status_diff(recs, want_codes=True)
        want = self.host_tab.diff(recs)
        if not np.array_equal(idx, want) or not np.array_equal(codes, oracle.record_codes(recs)[want]):
            self.fail(f"status_diff: {len(idx)} changed slots, model {len(want)}, or codes differ")

    def host_seed(self):
        recs = self.host_records()
        self.eng.status_seed(recs)
        self.host_tab.seed(recs)

    def host_slot_sweeps(self):
        slots = np.sort(self.rng.choice(NS, 3 * NL, replace=False)).astype(np.uint32)
        recs = self.host_records(0.5)[slots]
        half = slots[::2]
        half_recs = np.ascontiguousarray(recs[::2])
        self.eng.status_seed_slots(half, half_recs)
        self.host_tab.seed_slots(half, half_recs)
        recs = self.host_records(0.5)[slots]
        idx, codes = self.eng.status_diff_slots(slots, recs, want_codes=True)
        want = status_slots_model.diff_slots(self.host_tab, slots, recs)
        if not np.array_equal(idx, want) or not np.array_equal(codes, oracle.record_codes(recs)[np.searchsorted(slots, want)]):
            self.fail(f"status_diff_slots: {len(idx)} changed slots, model {len(want)}, or codes differ")

    def host_tick(self, P):
        recs = self.host_records()
        pods, wb, wt = self.batch(P) if P else (None, None, None)
        best, t5, idx, codes = self.eng.tick(pods, recs, want_top5=bool(P))
        want = self.host_tab.diff(recs)
        if not np.array_equal(idx, want) or not np.array_equal(codes, oracle.record_codes(recs)[want]):
            self.fail(f"tick P={P}: {len(idx)} changed slots, model {len(want)}, or codes differ")
        if P:
            sc.check(f"tick P={P}", best, t5, wb[:P], wt[:P])

    def pods_seed(self):
        slots = np.sort(self.rng.choice(self.pods_n, 2000, replace=False)).astype(np.uint32)
        rows = self.rng.integers(0, POOL, len(slots))
        self.eng.pods_seed_slots(slots, {c: None if v is None else v[rows] for c, v in self.pool.items()})
        self.idx[slots] = rows

    def pods_mark(self):
        slots = np.sort(self.rng.choice(self.pods_n, 3000, replace=False)).astype(np.uint32)
        f = (self.rng.random(len(slots)) < 0.5).astype(np.uint8)
        self.eng.pods_mark_pending(slots, f)
        self.flags[slots] = f

    def smaller_device_calls(self):
        """a device select and a device sweep, both smaller than the captured ones, on another stream"""
        import torch

        P = C // 2
        d = sc.to_device(self.pool_rows(1, P))
        best, t5 = full(P, sc.SENTINEL, torch.int32), full(5 * P, sc.SENTINEL, torch.int32)
        torch.cuda.synchronize()
        self.eng.select_device(d, best, t5, shard=self.shard, stream=self.other.cuda_stream)
        torch.cuda.synchronize()
        sc.check("smaller device select", best.cpu().numpy(), t5.cpu().numpy().reshape(P, 5), self.pool_best[C:C + P],
                 self.pool_top5[C:C + P])
        n = ND // 2
        recs = rpk.synth.make_status_records(n, 1, 0.0, seed=5, stride=STRIDE)
        hp, idx, cnt = full(n, 0, torch.int64), full(n, 0, torch.int32), full(1, 0, torch.int32)
        d_recs = t(recs.reshape(-1))
        torch.cuda.synchronize()
        self.eng.status_diff_device(d_recs, STRIDE, hp, idx, cnt, shard=self.shard, stream=self.other.cuda_stream)
        torch.cuda.synchronize()
        if int(cnt.item()) != n:  # a fresh column: every slot changed
            self.fail("smaller device sweep: not every slot of a fresh column reported")

    def menu(self):
        """(label, call) of every call the contract says keeps a capture valid"""
        return [
            ("host select 1x top5", lambda: self.host_select(C, True, False)),
            ("host select 3x NULL columns", lambda: self.host_select(POOL, False, True)),
            ("host select 2x top5", lambda: self.host_select(2 * C, True, False)),
            (f"host select {BIG} top5", lambda: self.host_select(BIG, True, False)),
            ("select_slots 3x", lambda: self.host_slots(3 * C, True)),
            ("select_pending", self.host_pending),
            ("select_pending_changed", self.host_pending_changed),
            ("tick P=0", lambda: self.host_tick(0)),
            ("tick P=3x", lambda: self.host_tick(POOL)),
            ("status_diff", self.host_sweep),
            ("status_seed", self.host_seed),
            ("status seeds and slot sweeps", self.host_slot_sweeps),
            ("pods_seed_slots", self.pods_seed),
            ("pods_mark_pending", self.pods_mark),
            ("smaller device calls", self.smaller_device_calls),
        ]


@contextlib.contextmanager
def world(name, **kw):
    eng = rpk.Engine(kw.pop("n_gpus", 1), device_ids=kw.pop("device_ids", None))
    try:
        yield World(eng, name, **kw)
    finally:
        import torch

        torch.cuda.synchronize()
        eng.close()


def check_allocated(w, ptrs):
    """Every buffer the eager calls of w's entry points must have used is listed, not NULL: the hook reports the scratch
    the device calls really run on (a device call moved back onto a host lane would leave these entries NULL, and the
    moves of the host lane would go unseen)"""
    need = ["dev_lane.rw", "dev_lane.order", "dev_lane.pos", "dev_lane.ctrs"]
    need += [f"dev_sweep.{b}" for b in ("tile_state", "misc", "stage_idx", "stage_code", "unit_cnt")]
    need += [f"view{c}.{b}" for c in (0, 1) for b in ("price", "perm")]
    need += [f"pt_cols.{c}" for c in POD_COLS] + ["pt_pending", "pt_state", "pt_ticket", "r_gen", "r_list", "r_dn",
                                                   "r_lane.cols.mem", "r_lane.top5"]
    if any(e.startswith("slots") for e in w.entries):  # the slot selects gather all five pod columns into the lane
        need += [f"dev_lane.{b}" for b in LANE[:5]]
    if w.eng.stats()["select_kernel_kind"] == 4:  # bit-sliced view: the captured C rows take the persistent path
        need += [f"dev_lane.{b}" for b in ("key", "ord_rw", "hist", "k0_base", "hdr")]
    missing = [n for n in need if not ptrs[NAMES.index(n)]]
    assert not missing, f"table {w.name}: the device calls ran without allocating {missing}"


def check_larger_device_calls_move(w):
    """The positive control, with no replay after it (these calls invalidate every capture): a device select of BIG rows
    and a device sweep of 2^20 records with codes, both checked, must move the device select lane and the device sweep
    scratch the hook lists.  cudaMalloc may hand a grown buffer the address it freed (harmless for a graph: the new block
    is larger), so each scratch must show one moved buffer, not a fixed set"""
    import torch

    before = w.eng.capture_buffers(w.shard)
    pods, wb, _ = w.batch(BIG)
    d = sc.to_device(pods)
    best = full(BIG, sc.SENTINEL, torch.int32)
    n = 1 << 20
    recs = rpk.synth.make_status_records(n, 0, 0.0, seed=9, stride=STRIDE)
    hp, idx, cnt = full(n, 0, torch.int64), full(n, 0, torch.int32), full(1, 0, torch.int32)
    code = full(n, 0, torch.int16)
    d_recs = t(recs.reshape(-1))
    torch.cuda.synchronize()
    w.eng.select_device(d, best, shard=w.shard, stream=w.other.cuda_stream)
    w.eng.status_diff_device(d_recs, STRIDE, hp, idx, cnt, shard=w.shard, stream=w.other.cuda_stream, d_changed_code=code)
    torch.cuda.synchronize()
    sc.check("larger device select", best.cpu().numpy(), None, wb, None)
    assert int(cnt.item()) == n, "larger device sweep: not every slot of a fresh column reported"
    got = moved(before, w.eng.capture_buffers(w.shard))
    lane = [f"dev_lane.{b}" for b in ("rw", "order", "pos", "ctrs", "key", "ord_rw", "k0_base")]
    sweep = [f"dev_sweep.{b}" for b in ("stage_idx", "stage_code", "unit_cnt")]
    assert set(lane) & set(got) and set(sweep) & set(got), \
        f"table {w.name}: larger device calls moved only {got}; expected one of {lane} and one of {sweep}"


@pytest.mark.parametrize("name", ["synth20k", "stride64", "packed_only", "full_int32"])
def test_valid_calls_leave_every_captured_buffer_in_place(name):
    """No replay: after one eager call of every capturable entry point, every call of the valid side, at up to 10x the
    captured size, leaves each buffer those calls handed their kernels where it was.  The listed buffers are shown to be
    the ones in use first (allocated by the eager calls) and last (moved by larger device calls)."""
    with world(name) as w:
        before = w.eng.capture_buffers()
        check_allocated(w, before)
        problems = []
        for label, fn in w.menu():
            fn()
            after = w.eng.capture_buffers()
            if moved(before, after):
                problems.append(f"{label} moved {', '.join(moved(before, after))}")
            before = after
        assert not problems, f"table {name}:\n  " + "\n  ".join(problems)
        check_larger_device_calls_move(w)


def test_replays_between_every_valid_call():
    """The replay matrix: after each call of the valid side (checked), every entry point's capture gets new inputs,
    is replayed twice and called once, and every output is checked."""
    with world("synth20k") as w:
        for label, fn in w.menu():
            w.log.append(label)
            fn()
            w.replay_all(label)


INVALID = ["upload", "refresh", "pods_reset", "peer_bind"]


@pytest.mark.parametrize("seed", [1, 2, 3])
def test_seeded_programs(seed):
    """A random sequence of valid calls, replays and eager device calls over tables whose view is bit-sliced at both
    row strides, packed only or wide; after every call of the invalid side every entry point is captured again."""
    rng = np.random.default_rng(seed)
    tables = ["synth20k", "stride64", "packed_only", "full_int32"]
    with world(str(rng.choice(tables)), seed=seed) as w:
        menu = dict(w.menu())
        bound = None
        # 30 random steps (valid calls twice as likely as a bare replay round), with every call of the invalid side
        # inserted once at a random place
        ops = [str(o) for o in rng.choice(list(menu) * 2 + ["replay"] * 8, 30)]
        for op in INVALID:
            ops.insert(int(rng.integers(0, len(ops) + 1)), op)
        for op in ops:
            w.log.append(op)
            if op == "replay":
                w.replay_all(op)
                continue
            if op not in INVALID:
                menu[op]()
                if rng.random() < 0.6:  # most valid calls are followed by a replay round before the next call
                    w.replay_all(op)
                continue
            if op == "upload":
                name = str(rng.choice(tables))
                w.set_table(name, sc.table(name), upload=True)
                w.seed_all()
            elif op == "refresh":
                offers = {k: None if v is None else v.copy() for k, v in w.offers.items()}
                ch = rng.choice(len(offers["mem_gb"]), 3, replace=False)
                offers["secure_price"][ch] *= 0.5
                offers["community_price"][ch] += 0.01
                w.set_table(w.name, offers, refresh=True)
            elif op == "pods_reset":  # the stored results go too: the next call reports every pending slot
                w.eng.pods_reset(N)
                w.seed_all()
                w.mirror_best[:], w.mirror_top5[:] = sc.SENTINEL, sc.SENTINEL
            else:  # a fresh one-rank group, or none: the gathers' signals go there from now on
                import torch

                bound = None if bound is not None else full(64, 0, torch.int32)
                w.eng.peer_bind([bound.data_ptr()] if bound is not None else [], 0)
            w.log.append(f"  table {w.name}")
            w.capture_all()
            w.replay_all(op)


def test_shard1_of_a_three_shard_ctx_on_one_gpu(monkeypatch):
    """Captures on shard 1 of a three-shard ctx (every shard on GPU 0) stay valid while host calls run over all
    shards.  Unbound calls only: shards that share a GPU may not wait on each other."""
    monkeypatch.setenv("RPK_TEST_SHARED_DEVICE", "1")
    with world("synth20k", n_gpus=3, device_ids=[0, 0, 0], shard=1, entries=UNBOUND, n_ranks=3, my_rank=1) as w:
        before = w.eng.capture_buffers(1)
        check_allocated(w, before)
        for label, fn in w.menu():
            w.log.append(label)
            fn()
            after = w.eng.capture_buffers(1)
            assert not moved(before, after), f"{label} moved {moved(before, after)} on shard 1"
            before = after
            w.replay_all(label)
        check_larger_device_calls_move(w)
