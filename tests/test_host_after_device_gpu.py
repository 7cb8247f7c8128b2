"""Host entry points called right behind a device call that is still queued on another stream of the same shard.

A one-process-per-GPU caller mixes the two kinds of call on one ctx: it refreshes offers, seeds the pod table or runs
a host sweep between device calls, without a synchronise.  include/rpk.h ("Ordering") promises that a host call first
waits for the shard's last device call on the buffers the two share.  Each case puts ~1 s of sleep ahead of the device
call on a fresh stream, makes the host call at once, and then checks

  - that the device call had completed when the host call returned (an event recorded behind it), and
  - that both calls computed what the oracle computes: the device call on the state before the host call, the host
    call (or the call that reads what it wrote) on the state after it.

Every size a case uses runs once before the sleep, so no call allocates: an allocation would synchronise the device
by itself and hide a missing wait.  Without the wait the host call finishes while the device call is still queued
behind the sleep, so the two never overlap."""
import time

import numpy as np
import pytest

import oracle
import rpk
import select_plan_cases as sc
from status_slots_model import diff_slots

pytestmark = pytest.mark.gpu

synth = rpk.synth
G, P_SMALL, P_PIPE, N_POD, N_ST, STRIDE = 3000, 1000, 6000, 8192, 8192, 16  # P_PIPE > 4096: the sub-batch pipeline
SLEEP_CYCLES = 2_000_000_000  # about 1 s at the H100's SM clock
GRACE_S = 0.05  # an event behind a finished device call completes within this of the host call's return
DEFAULT_POD = {"req_mem_gb": 16, "req_vcpu": 0, "req_ram_gb": 0, "max_price": 0.5, "cloud": 0}  # rpk_pods_reset's row


def finished(ev) -> bool:
    t0 = time.monotonic()
    while not ev.query():
        if time.monotonic() - t0 > GRACE_S:
            return False
        time.sleep(1e-4)
    return True


def table_rows(table: dict, slots) -> dict:
    return {k: np.ascontiguousarray(v[slots]) for k, v in table.items()}


class Rig:
    """One ctx with offers, a seeded pod table and a tracked status table, the oracle's copy of each, and a caller-owned
    hash column for the device sweep on GPU `shard`."""

    def __init__(self, n_gpus: int, shard: int, make_engine=None):
        """make_engine(n_gpus) -> the ctx; None: one shard per GPU (skipped where there are fewer GPUs than that)"""
        import torch

        if make_engine is None:
            if torch.cuda.device_count() < n_gpus:
                pytest.skip(f"needs {n_gpus} GPUs")
            make_engine = rpk.Engine
        self.eng = make_engine(n_gpus)
        self.shard = shard
        self.dev = torch.device("cuda", self.eng.device_ids[shard])
        self.offers = synth.make_offers(G, correlated=True)
        self.eng.upload_offers(self.offers)
        self.table = synth.make_pods(N_POD, seed=7)
        self.eng.pods_reset(N_POD)
        self.eng.pods_seed_slots(np.arange(N_POD, dtype=np.uint32), self.table)
        self.rng = np.random.default_rng(2026)
        self.host_tab, self.dev_tab = oracle.StatusTable(N_ST, STRIDE), oracle.StatusTable(N_ST, STRIDE)
        self.eng.status_reset(N_ST)
        self.d_hash = torch.zeros(N_ST, dtype=torch.int64, device=self.dev)
        self.sweep = 0
        self.warm_up()

    def close(self):
        self.eng.close()

    # -- inputs and the oracle ----------------------------------------------------------------------------------
    def records(self):
        self.sweep += 1
        return synth.make_status_records(N_ST, self.sweep, 0.1, stride=STRIDE)

    def slot_list(self, n):
        return self.rng.integers(0, N_POD, n).astype(np.uint32)

    def sweep_slots(self):
        return np.sort(self.rng.choice(N_ST, N_ST // 8, replace=False)).astype(np.uint32)

    def check_select(self, label, got, pods):
        want_best, want_top5 = oracle.select(self.offers, pods, want_top5=True, n_threads=4)
        sc.check(label, got[0], got[1], want_best, want_top5)

    def check_host_sweep(self, label, got_idx, got_codes, want, recs_of_want):
        assert np.array_equal(got_idx, want), f"{label}: changed list differs from the oracle"
        if got_codes is not None:
            assert np.array_equal(got_codes, oracle.record_codes(recs_of_want)), f"{label}: codes differ from the oracle"

    # -- calls --------------------------------------------------------------------------------------------------
    def host_sweep(self):
        recs = self.records()
        want = self.host_tab.diff(recs)
        idx, codes, _ = self.eng.status_diff(recs, want_codes=True)
        self.check_host_sweep("status_diff", idx, codes, want, recs[want])

    def host_sweep_slots(self):
        recs, sl = self.records(), self.sweep_slots()
        want = diff_slots(self.host_tab, sl, recs[sl])
        idx, codes = self.eng.status_diff_slots(sl, recs[sl], want_codes=True)
        self.check_host_sweep("status_diff_slots", idx, codes, want, recs[want])

    def host_seed(self):
        recs = self.records()
        self.eng.status_seed(recs)
        self.host_tab.seed(recs)

    def host_tick(self, P):
        pods = synth.make_pods(P, seed=13) if P else None
        recs = self.records()
        want = self.host_tab.diff(recs)
        best, top5, idx, codes = self.eng.tick(pods, recs, want_top5=True)
        self.check_host_sweep("tick", idx, codes, want, recs[want])
        if P:
            self.check_select("tick select", (best, top5), pods)

    def behind_sleep(self, enqueue):
        """On a new stream of the shard's GPU: the sleep, then enqueue(stream) -> a torch event recorded behind it"""
        import torch

        torch.cuda.synchronize(self.dev)  # the device call's inputs were written on the current stream
        with torch.cuda.device(self.dev):
            s = torch.cuda.Stream()
            ev = torch.cuda.Event()
            with torch.cuda.stream(s):
                torch.cuda._sleep(SLEEP_CYCLES)
                enqueue(s.cuda_stream)
                ev.record(s)
        return ev

    def device_select(self, sleep=True):
        """rpk_select_device of P_SMALL rows -> (event, check)"""
        import torch

        pods = synth.make_pods(P_SMALL, seed=11)
        cols = {k: torch.from_numpy(v).to(self.dev) for k, v in pods.items()}
        best = torch.full((P_SMALL,), sc.SENTINEL, dtype=torch.int32, device=self.dev)
        top5 = torch.full((P_SMALL * 5,), sc.SENTINEL, dtype=torch.int32, device=self.dev)
        offers = self.offers  # the table the call must see, whatever the host call uploads next
        call = lambda st: self.eng.select_device(cols, best, top5, shard=self.shard, stream=st)  # noqa: E731
        ev = self.behind_sleep(call) if sleep else call(None)

        def check():
            torch.cuda.synchronize(self.dev)
            want_best, want_top5 = oracle.select(offers, pods, want_top5=True, n_threads=4)
            sc.check("select_device", best.cpu().numpy(), top5.cpu().numpy().reshape(-1, 5), want_best, want_top5)
        return ev, check

    def device_select_slots(self, sleep=True):
        """rpk_select_slots_device of P_SMALL slots -> (event, check)"""
        import torch

        sl = self.slot_list(P_SMALL)
        d_slots = torch.from_numpy(sl.view(np.int32)).to(self.dev)
        best = torch.full((P_SMALL,), sc.SENTINEL, dtype=torch.int32, device=self.dev)
        top5 = torch.full((P_SMALL * 5,), sc.SENTINEL, dtype=torch.int32, device=self.dev)
        rows = table_rows(self.table, sl)  # the rows the call must see, whatever the host call writes next
        call = lambda st: self.eng.select_slots_device(d_slots, best, top5, shard=self.shard, stream=st)  # noqa: E731
        ev = self.behind_sleep(call) if sleep else call(None)

        def check():
            torch.cuda.synchronize(self.dev)
            self.check_select("select_slots_device", (best.cpu().numpy(), top5.cpu().numpy().reshape(-1, 5)), rows)
        return ev, check

    def device_sweep(self, sleep=True):
        """rpk_status_diff_device_codes over the caller's column -> (event, check)"""
        import torch

        recs = self.records()
        want = self.dev_tab.diff(recs)
        d_recs = torch.from_numpy(recs.reshape(-1)).to(self.dev)
        idx = torch.full((N_ST,), -1, dtype=torch.int32, device=self.dev)
        codes = torch.zeros(N_ST, dtype=torch.int16, device=self.dev)
        cnt = torch.zeros(1, dtype=torch.int32, device=self.dev)
        call = lambda st: self.eng.status_diff_device(d_recs, STRIDE, self.d_hash, idx, cnt, shard=self.shard,  # noqa: E731
                                                      stream=st, d_changed_code=codes)
        ev = self.behind_sleep(call) if sleep else call(None)

        def check():
            torch.cuda.synchronize(self.dev)
            k = int(cnt.item())
            self.check_host_sweep("status_diff_device", idx[:k].cpu().numpy().view(np.uint32),
                                  codes[:k].cpu().numpy().view(np.uint16), want, recs[want])
        return ev, check

    def warm_up(self):
        """every call of every size below once, so that none of them allocates"""
        for dev_call in (self.device_select, self.device_select_slots, self.device_sweep):
            dev_call(sleep=False)[1]()
        for P in (P_SMALL, P_PIPE):
            self.check_select(f"select {P}", self.eng.select(synth.make_pods(P, seed=11), want_top5=True), synth.make_pods(P, seed=11))
            sl = self.slot_list(P)
            self.check_select(f"select_slots {P}", self.eng.select_slots(sl, want_top5=True), table_rows(self.table, sl))
        self.eng.pods_seed_slots(np.arange(0, N_POD, 97, dtype=np.uint32), table_rows(self.table, np.arange(0, N_POD, 97)))
        self.host_sweep()
        self.host_sweep_slots()
        self.host_seed()
        self.host_tick(P_PIPE)
        self.host_tick(0)


# -- the cases: (the device call ahead of the host call, the host call with its checks) -----------------------------

def host_select(P):
    def run(rig):
        pods = synth.make_pods(P, seed=11)
        rig.check_select(f"select {P}", rig.eng.select(pods, want_top5=True), pods)
    return run


def host_select_slots(P):
    def run(rig):
        sl = rig.slot_list(P)
        rig.check_select(f"select_slots {P}", rig.eng.select_slots(sl, want_top5=True), table_rows(rig.table, sl))
    return run


def host_upload_offers(rig):
    """same G and the same distinct mem / vcpu / ram values, new prices and availability: the table's layout and every
    buffer stay, so the queued launch is valid for either table, and only its order decides which one it reads"""
    new = synth.make_offers(G, seed=99, correlated=True)
    for k in ("mem_gb", "vcpu", "ram_gb"):
        new[k] = rig.offers[k]
    rig.eng.upload_offers(new)
    rig.offers = new
    host_select(P_SMALL)(rig)


def host_pods_reset(rig):
    rig.eng.pods_reset(N_POD)
    rig.table = {k: np.full(N_POD, v, dtype=rig.table[k].dtype) for k, v in DEFAULT_POD.items()}
    host_select_slots(P_SMALL)(rig)


def host_pods_seed_slots(rig):
    sl = np.arange(0, N_POD, 97, dtype=np.uint32)
    new = synth.make_pods(len(sl), seed=23)
    rig.eng.pods_seed_slots(sl, new)
    for k in rig.table:
        rig.table[k][sl] = new[k]
    host_select_slots(P_SMALL)(rig)


CASES = {
    "select_small": ("select", host_select(P_SMALL)),
    "select_pipelined": ("select", host_select(P_PIPE)),
    "select_slots_small": ("select_slots", host_select_slots(P_SMALL)),
    "select_slots_pipelined": ("select_slots", host_select_slots(P_PIPE)),
    "upload_offers": ("select", host_upload_offers),
    "pods_reset": ("select_slots", host_pods_reset),
    "pods_seed_slots": ("select_slots", host_pods_seed_slots),
    "status_diff_codes": ("sweep", Rig.host_sweep),
    "status_seed": ("sweep", lambda rig: (rig.host_seed(), rig.host_sweep())),
    "status_diff_slots": ("sweep", Rig.host_sweep_slots),
    "tick_behind_select": ("select", lambda rig: rig.host_tick(P_PIPE)),
    "tick_behind_sweep": ("sweep", lambda rig: rig.host_tick(P_PIPE)),
    "tick_no_pods_behind_sweep": ("sweep", lambda rig: rig.host_tick(0)),
}
DEVICE = {"select": Rig.device_select, "select_slots": Rig.device_select_slots, "sweep": Rig.device_sweep}


def run_case(rig, name):
    device, host = CASES[name]
    ev, check_device = DEVICE[device](rig)
    try:
        host(rig)
        done = finished(ev)
    finally:
        ev.synchronize()  # whatever happened, the device call ends before the ctx it uses can be destroyed
    assert done, f"{name}: the host call returned while the {device} device call ahead of it was still queued"
    check_device()


@pytest.mark.parametrize("name", list(CASES))
def test_host_call_waits_for_device_call(name):
    rig = Rig(1, 0)
    try:
        run_case(rig, name)
    finally:
        rig.close()


# every device call of these cases is queued on a plain stream of one shard, and none waits for another shard's kernel
SHARD_1_CASES = ["select_pipelined", "select_slots_pipelined", "upload_offers", "pods_seed_slots", "status_diff_codes",
                 "tick_behind_sweep"]


@pytest.mark.parametrize("name", SHARD_1_CASES)
def test_host_call_waits_for_device_call_on_shard_1(name):
    """a 2-GPU ctx: the device call runs on shard 1, and the host call spans both shards"""
    rig = Rig(2, 1)
    try:
        run_case(rig, name)
    finally:
        rig.close()
