"""CPU test of the slot-list model (status_slots_model.diff_slots): for random tables and lists it equals a whole-table
diff in which every unlisted slot carries its previous record, and it leaves the state of unlisted slots untouched."""
import numpy as np
import pytest

import oracle
import status_cases as sc
import status_slots_model as ssm


@pytest.mark.parametrize("stride", [16, 32, 48, 128, 256])
@pytest.mark.parametrize("seed", [1, 2, 3])
def test_diff_slots_equals_whole_table_diff(stride, seed):
    rng = np.random.default_rng(1000 * seed + stride)
    N = int(rng.integers(1, 3000))
    lt = sc.LogicalTable(N, rng)
    tab = oracle.StatusTable(N, stride)
    seen = np.sort(rng.choice(N, int(rng.integers(0, N + 1)), replace=False))  # the rest stays never seen
    tab.seed_slots(seen, lt.records(stride, seen))
    for step in range(4):
        lt.step(stride, float(rng.choice([0.0, 0.05, 0.5, 1.0])))
        recs = lt.records(stride)
        n = int(rng.choice([0, 1, N, int(rng.integers(0, N + 1))]))
        slots = np.sort(rng.choice(N, n, replace=False))
        listed = np.zeros(N, bool)
        listed[slots] = True
        # whole-table twin: an unlisted slot carries its previous record, so only a never-seen one can report there
        twin = oracle.StatusTable(N, tab.stride)
        twin.prev[:], twin.has_prev[:] = tab.prev, tab.has_prev
        whole = np.where(listed[:, None], tab._fit(recs), tab.prev)
        want = twin.diff(whole)
        before_prev, before_has = tab.prev.copy(), tab.has_prev.copy()
        got = ssm.diff_slots(tab, slots, np.ascontiguousarray(recs[slots]))
        assert np.array_equal(got, want[listed[want]]), (stride, seed, step)
        assert np.array_equal(tab.prev[~listed], before_prev[~listed]) and np.array_equal(tab.has_prev[~listed], before_has[~listed])
        assert np.array_equal(tab.prev[listed], twin.prev[listed]) and np.array_equal(tab.has_prev[listed], twin.has_prev[listed])


def test_diff_slots_widens_the_table():
    """records wider than the table widen it, exactly as a whole-table diff does"""
    rng = np.random.default_rng(5)
    lt = sc.LogicalTable(200, rng)
    tab = oracle.StatusTable(200, 16)
    tab.seed(lt.records(16))
    slots = np.arange(0, 200, 3)
    assert len(ssm.diff_slots(tab, slots, lt.records(64, slots))) == 0 and tab.stride == 64
