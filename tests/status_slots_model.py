"""The reference's per-slot compare restricted to a list of slots, on top of oracle.StatusTable: the listed rows of the
table are gathered, diffed by the oracle's C compare (rpk_oracle_status_diff) and scattered back.  This is what
rpk_status_diff_slots must compute; the CPU test pins it to a whole-table diff."""
import numpy as np

import oracle


def diff_slots(tab: oracle.StatusTable, slots, records: np.ndarray) -> np.ndarray:
    """records[i] is this sweep's state of slot slots[i] (distinct slots < tab.N) -> changed slot ids, ascending.
    The state of the listed slots that changed is replaced; no other slot is touched."""
    slots = np.asarray(slots, np.int64)
    assert records.shape[0] == len(slots) and len(np.unique(slots)) == len(slots)
    if len(slots) == 0:
        return np.empty(0, np.uint32)
    assert slots.min() >= 0 and slots.max() < tab.N
    recs = tab._fit(records)  # widens the table first when the records are wider
    sub = oracle.StatusTable(len(slots), tab.stride)
    sub.prev[:] = tab.prev[slots]
    sub.has_prev[:] = tab.has_prev[slots]
    pos = sub.diff(recs)
    tab.prev[slots] = sub.prev
    tab.has_prev[slots] = sub.has_prev
    return np.sort(slots[pos]).astype(np.uint32)
