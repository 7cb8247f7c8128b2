"""CPU tests of ctx_model.py: random whole-ctx histories -- offer uploads of several G, refreshes inside and past the
change window and onto the fifth entry of stored lists, seeds, marks, pod-table resets and grows (with and without their
stored results) -- run through the model alone.  After every tick each pending slot the reach rule did not reselect
holds exactly oracle.select's list under the current table (Ctx.tick asserts it)."""
import numpy as np
import pytest

import ctx_model
import offers_refresh_model as orm
import oracle
from test_offers_refresh_model import table

OPS = ["refresh", "refresh", "tie", "upload", "seed", "seed", "mark", "mark", "grow", "reset", "tick", "tick", "tick"]


@pytest.mark.parametrize("seed", range(10))
def test_random_histories_keep_every_unreselected_list(seed):
    rng = np.random.default_rng(4000 + seed)
    ctx = ctx_model.Ctx()
    G = int(rng.integers(20, 60))
    ctx.upload(table(rng, G))
    N = int(rng.integers(15, 40))
    ctx.pods_reset(N)
    seen = dict.fromkeys(["window", "wholesale", "tie", "grow kept", "grow dropped", "kept", "reselected"], 0)
    for stp in range(150):
        op = str(rng.choice(OPS))
        if op == "refresh":
            k = int(rng.choice([0, 1, 2, 5, 16, 17, 30]))
            n = ctx.refresh(ctx_model.edit_offers(rng, ctx.offers, k) if k else ctx_model.copy_table(ctx.offers))
            seen["wholesale" if n == orm.WHOLESALE else "window"] += 1
        elif op == "tie":
            new, pairs = ctx_model.tie_edit(rng, ctx.offers, ctx.stored_full_lists(), n_pairs=1)
            ctx.refresh(new)
            if pairs:  # one c below its L[4]: c takes the place of L[4] in the list of the pair's row
                ctx.tick()
                lists = ctx.gens.top5[ctx.pending()]
                assert all((lists == c).any() for c, _ in pairs), f"step {stp}: an offer tied below an L[4] is in no list"
                seen["tie"] += 1
        elif op == "upload":
            ctx.upload(table(rng, int(rng.integers(20, 60))) if rng.random() < 0.5 else ctx.offers)
        elif op == "seed":
            sl = np.sort(rng.choice(ctx.N, int(rng.integers(1, ctx.N + 1)), replace=False))
            ctx.seed(sl, ctx.rows(sl) if rng.random() < 0.3 else ctx_model.odd_rows(rng, ctx.offers, len(sl)))
        elif op == "mark":
            sl = np.sort(rng.choice(ctx.N, int(rng.integers(1, ctx.N + 1)), replace=False))
            ctx.mark(sl, rng.random(len(sl)) < 0.6)
        elif op == "grow":
            keep = rng.random() < 0.6
            N0 = ctx.N
            before = ctx.gens.res_gen.copy(), ctx.gens.top5.copy(), ctx.rows(np.arange(N0))
            ctx.pods_grow(N0 + int(rng.choice([0, 1, 15, 16, 17, N0 // 4, N0])), keep)
            assert np.array_equal(ctx.gens.res_gen[:N0], before[0] if keep else np.zeros(N0, np.int64))
            assert not keep or np.array_equal(ctx.gens.top5[:N0], before[1])
            assert all(np.array_equal(ctx.rows(np.arange(N0))[k].view(np.uint8), v.view(np.uint8)) for k, v in before[2].items())
            assert not ctx.gens.pending[N0:].any() and not ctx.gens.res_gen[N0:].any()
            seen["grow kept" if keep else "grow dropped"] += 1
        elif op == "reset":
            ctx.pods_reset(int(rng.integers(15, 200)))
        else:
            n_kept = len(ctx.pending())
            t = ctx.tick()
            seen["kept"] += n_kept - len(t.stale)
            seen["reselected"] += len(t.stale)
            assert np.array_equal(t.top5, ctx.expected(t.slots)[1]) and np.array_equal(t.best, t.top5[:, 0])
    assert all(seen.values()), seen


def test_grown_status_table_reports_only_the_new_slots():
    """a grown table keeps every seen slot's state, and its new slots report on the next diff"""
    rng = np.random.default_rng(5)
    recs = rng.integers(0, 256, (40, 32)).astype(np.uint8)
    t = oracle.StatusTable(17, 32)
    t.seed(recs[:17])
    t.grow(40)
    assert np.array_equal(t.diff(recs), np.arange(17, 40, dtype=np.uint32))
    assert len(t.diff(recs)) == 0
