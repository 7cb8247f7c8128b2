"""GPU tests of the streaming status sweep on both sides of its two launch boundaries, each call checked against
oracle.StatusTable.

Below the big-table threshold the sweep runs one 8-warp CTA per SM (so that it fits beside the persistent select), and
every warp takes one 64-slot unit until SMs * 8 * 64 slots; past that point the warps take longer runs.  At 4M slots
the sweep switches to 1024-thread CTAs.  The boundaries are the same at every stride; they are crossed at strides 16
and 32, and at the wide strides 48, 64 and 256, whose sweep takes the stride from its arguments (the 4M boundary at 48
only, which keeps host memory modest; test_status_scale_gpu.py runs every stride 16..256 at 4M + 37 slots, with keys
instead of host records).  Each size runs a host-entry sequence (seed, diff with codes and hashes, an unchanged diff,
reset, diff), a device-entry diff of a caller-owned hash column, and an rpk_tick."""
import numpy as np
import pytest

import oracle
import rpk

pytestmark = pytest.mark.gpu

BIG = 4 << 20  # kBigTable (status.cu)


def sm_count() -> int:
    import torch

    return torch.cuda.get_device_properties(0).multi_processor_count


def resolve(size: str) -> int:
    """sizes that depend on the device are named at collection time (no GPU there) and resolved here"""
    sat = sm_count() * 8 * 64  # one CTA per SM x 8 warps x one 64-slot unit
    base, _, off = size.partition("+") if "+" in size else size.partition("-")
    n = {"sat": sat, "big": BIG}[base]
    return n + int(off) if "+" in size else n - int(off or 0)


SAT_SIZES, BIG_SIZES = ["sat-1", "sat", "sat+1"], ["big-1", "big", "big+1"]
BOUNDARY_CASES = ([(size, stride) for size in SAT_SIZES + BIG_SIZES for stride in (16, 32)]
                  + [(size, stride) for size in SAT_SIZES for stride in (48, 64, 256)])


@pytest.mark.parametrize("size,stride", BOUNDARY_CASES)
def test_sweep_at_launch_boundary(size, stride):
    import torch

    N = resolve(size)
    base = rpk.synth.make_status_records(N, 0, stride=stride)
    nxt = rpk.synth.make_status_records(N, 3, 0.2, stride=stride)
    tab = oracle.StatusTable(N, stride)
    with rpk.Engine(1) as eng:
        eng.status_reset(N)
        eng.status_seed(base)
        tab.seed(base)
        got, codes, hashes = eng.status_diff(nxt, want_codes=True, want_hashes=True)
        want = tab.diff(nxt)
        assert len(want) > N // 20
        assert np.array_equal(got, want), f"N {N}: changed list"
        assert np.array_equal(codes, oracle.record_codes(nxt)[want]), f"N {N}: codes"
        assert np.array_equal(hashes, oracle.record_hashes(nxt)), f"N {N}: hash column"
        got, _ = eng.status_diff(nxt)
        assert np.array_equal(got, tab.diff(nxt)) and len(got) == 0, f"N {N}: unchanged sweep"
        eng.status_reset(N)
        tab.reset(N)
        got, codes, _ = eng.status_diff(base, want_codes=True)
        want = tab.diff(base)
        assert len(want) == N and np.array_equal(got, want), f"N {N}: sweep after reset"
        assert np.array_equal(codes, oracle.record_codes(base)), f"N {N}: codes after reset"

        # device entry point: a caller-owned column holding the hashes of `base`
        col_tab = oracle.StatusTable(N, stride)
        col_tab.seed(base)
        col = torch.from_numpy(oracle.record_hashes(base).view(np.int64)).cuda()
        d_idx = torch.empty(N, dtype=torch.int32, device="cuda")
        d_code = torch.empty(N, dtype=torch.int16, device="cuda")
        d_n = torch.zeros(1, dtype=torch.int32, device="cuda")
        eng.status_diff_device(torch.from_numpy(nxt).cuda(), stride, col, d_idx, d_n, d_changed_code=d_code)
        torch.cuda.synchronize()
        n = int(d_n.item())
        want = col_tab.diff(nxt)
        assert np.array_equal(d_idx[:n].cpu().numpy().view(np.uint32), want), f"N {N}: device changed list"
        assert np.array_equal(d_code[:n].cpu().numpy().view(np.uint16), oracle.record_codes(nxt)[want]), f"N {N}: device codes"
        assert np.array_equal(col.cpu().numpy().view(np.uint64), col_tab.prev_hashes()), f"N {N}: device column"

        # rpk_tick (P = 0): the same kernel behind the tick entry point
        _, _, got, codes = eng.tick(None, nxt)
        want = tab.diff(nxt)
        assert np.array_equal(got, want), f"N {N}: tick changed list"
        assert np.array_equal(codes, oracle.record_codes(nxt)[want]), f"N {N}: tick codes"


@pytest.mark.parametrize("stride", [16, 32, 48])
def test_big_table_boundary(stride):
    """One context over the big-table boundary (4M - 1 slots: the largest 256-thread table; 4M; 4M + 37: a ragged last
    unit), host entry point; then the device entry point on a caller-owned column, and a misaligned column refused."""
    import torch

    M = BIG + 37
    base_all = rpk.synth.make_status_records(M, 0, stride=stride)
    next_all = rpk.synth.make_status_records(M, 2, 0.37, stride=stride)
    with rpk.Engine(1) as eng:
        for N in (BIG - 1, BIG, BIG + 37):
            base, nxt = base_all[:N], next_all[:N]
            tab = oracle.StatusTable(N, stride)
            eng.status_reset(N)
            eng.status_seed(base)
            tab.seed(base)
            got, codes, hashes = eng.status_diff(nxt, want_codes=True, want_hashes=True)
            want = tab.diff(nxt)
            assert len(want) > N // 10, f"N {N}: the tables barely differ"
            assert np.array_equal(got, want), f"N {N}: changed list"
            assert np.array_equal(codes, oracle.record_codes(nxt)[want]), f"N {N}: codes"
            assert np.array_equal(hashes, oracle.record_hashes(nxt)), f"N {N}: hash column"
            got, _ = eng.status_diff(nxt)
            assert len(got) == 0, f"N {N}: second sweep reported {len(got)} slots"
        # device entry point, caller-owned column seeded by the caller with the reference hashes of `base_all`
        col_tab = oracle.StatusTable(M, stride)
        col_tab.seed(base_all)
        d_recs = torch.from_numpy(next_all).cuda()
        col = torch.from_numpy(oracle.record_hashes(base_all).view(np.int64)).cuda()
        d_idx = torch.empty(M, dtype=torch.int32, device="cuda")
        d_code = torch.empty(M, dtype=torch.int16, device="cuda")
        d_n = torch.zeros(1, dtype=torch.int32, device="cuda")
        eng.status_diff_device(d_recs, stride, col, d_idx, d_n, d_changed_code=d_code)
        torch.cuda.synchronize()
        n = int(d_n.item())
        want = col_tab.diff(next_all)
        assert np.array_equal(d_idx[:n].cpu().numpy().view(np.uint32), want), "device changed list"
        assert np.array_equal(d_code[:n].cpu().numpy().view(np.uint16), oracle.record_codes(next_all)[want]), "device codes"
        assert np.array_equal(col.cpu().numpy().view(np.uint64), oracle.record_hashes(next_all)), "device column"
        # a column that starts 8 bytes off a 16-byte boundary is refused before anything is launched
        buf = torch.zeros(M + 1, dtype=torch.int64, device="cuda")
        with pytest.raises(rpk.RpkError) as ei:
            eng.status_diff_device(d_recs, stride, buf[1:], d_idx, d_n)
        assert ei.value.code == rpk._ffi.RPK_EINVAL
        torch.cuda.synchronize()
        assert int(buf.count_nonzero().item()) == 0, "the refused call wrote the column"
