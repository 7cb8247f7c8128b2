"""GPU tests of the select over sequences of calls on one context, against the oracle.

Every select of a context relies on state that cleans itself between calls: row-block tickets, queue cursors, the
class counts and cursors (zeroed by the grid kernel's block 0), the push counters, and the control block regrown when
a table needs more queue cursors.  Each program below is a seeded sequence on a fresh rpk.Engine(1) that visits every
table of a menu (synth tables of 300 / 20k / 100k offers, the many-queue table, both class-limit tables, a 64-word
bitmap table, a packed-only table, a full-int32 table and an empty table), each uploaded under a random forced kernel,
and runs host selects (with and without top-5, optional columns NULL or not), device selects on two streams, device
gathers into three vectors at row0 != 0 and rpk_tick with a small status table.  Every step is checked (the checker of
select_plan_cases.py, oracle.StatusTable) and a failure prints the operation log.  Device calls are synchronised before the next host
call: the host entry points do not order themselves after unsynchronised device calls on the same shard."""
import numpy as np
import pytest

import oracle
import rpk
import select_plan_cases as sc

pytestmark = pytest.mark.gpu

MENU = ["synth300", "synth20k", "synth100k", "many_queues", "classes4096", "classes4224", "stride64", "packed_only",
        "full_int32", "empty"]
FORCE = [None, "bitmap_grouped", "bitmap_price", "packed_pos", "packed", "generic"]
SIZES = [1, 4096, 4097, 16_384, 16_385, 196_609]
ROWS = max(SIZES)
STATUS_N = 1000
OPS = ["host", "host", "dev_a", "dev_b", "gather", "tick"]


def batch(name, P, nulls):
    """the first P rows of the table's shared batch and their oracle results; nulls: only req_mem_gb is passed"""
    pods, wb, wt = sc.batch(name, ROWS)
    if nulls:
        pods, wb, wt = sc.batch_without_optional(name, ROWS)
    return sc.head(pods, P), wb[:P], wt[:P]


class Program:
    def __init__(self, seed: int):
        import torch

        self.seed = seed
        self.rng = np.random.default_rng(seed)
        self.eng = rpk.Engine(1)
        self.stream_b = torch.cuda.Stream()
        self.status = oracle.StatusTable(STATUS_N, 16)
        self.eng.status_reset(STATUS_N)
        self.sweep = 0
        self.table = None
        self.log = []

    def close(self):
        self.eng.close()

    def fail(self, err):
        raise AssertionError(f"{err}\nprogram seed {self.seed}; operations:\n  " + "\n  ".join(self.log))

    def upload(self, name, force):
        self.log.append(f"upload {name} force={force}")
        with sc.forced(force):
            self.eng.upload_offers(sc.table(name))
        self.table = name

    def run(self, op):
        rng = self.rng
        P = int(rng.choice(SIZES))
        top5 = bool(rng.integers(0, 2))
        nulls = op == "host" and rng.random() < 0.3
        row0 = int(rng.integers(1, 1000))
        self.log.append(f"{op} P={P} top5={top5}" + (" nulls" if nulls else "") + (f" row0={row0}" if op == "gather" else ""))
        pods, wb, wt = batch(self.table, P, nulls)
        try:
            if op == "host":
                got = sc.run_host(self.eng, pods, top5)
            elif op == "dev_a":
                got = sc.run_device(self.eng, pods, top5)
            elif op == "dev_b":  # the select scope moves to the other stream
                got = sc.run_device(self.eng, pods, top5, stream=self.stream_b)
            elif op == "gather":
                got = sc.run_gather(self.eng, pods, top5, row0)
            else:
                self.sweep += 1
                recs = rpk.synth.make_status_records(STATUS_N, self.sweep, 0.2, seed=self.seed, stride=16)
                best, t5, idx, codes = self.eng.tick(pods, recs, want_top5=top5)
                want = self.status.diff(recs)
                if not np.array_equal(idx, want):
                    raise AssertionError(f"tick: changed list {len(idx)} slots, model {len(want)}")
                if not np.array_equal(codes, oracle.record_codes(recs)[want]):
                    raise AssertionError("tick: codes differ from record_codes")
                got = (best, t5)
            sc.check(op, got[0], got[1], wb, wt)
        except AssertionError as e:
            self.fail(str(e))


@pytest.mark.parametrize("seed", [1, 2, 3])
def test_select_call_sequences(seed):
    """every table once in a seeded order, each under a random forced kernel, followed by two or three random calls"""
    p = Program(seed)
    try:
        for name in p.rng.permutation(MENU):
            p.upload(str(name), FORCE[int(p.rng.integers(0, len(FORCE)))])
            for _ in range(int(p.rng.integers(2, 4))):
                p.run(str(p.rng.choice(OPS)))
    finally:
        p.close()
