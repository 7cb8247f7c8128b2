"""Child process of test_status_modes_gpu.py.  The big-table streaming loop mode (RPK_TUNE k2=units|beats|beats4|ring)
is read once per process, so every mode runs in a process of its own: this script sweeps the big-table boundary
(4M - 1 slots: the largest small-shape table; 4M; 4M + 37: a ragged last unit) at strides 16 and 32 through the host
and the device entry points and exits non-zero on the first difference from the oracle."""
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
for p in (ROOT, HERE):
    if p not in sys.path:
        sys.path.insert(0, p)

import numpy as np  # noqa: E402

import oracle  # noqa: E402
import rpk  # noqa: E402

BIG = 4 << 20  # kBigTable (status.cu): tables from here on take the 1024-thread shape and the selected loop mode


def changed_rows(a, b):
    """rows whose compared fields differ (the flag bit of byte 0 is not one of them)"""
    ma, mb = a.copy(), b.copy()
    ma[:, 0] &= 0x7F
    mb[:, 0] &= 0x7F
    return np.nonzero((ma != mb).any(axis=1))[0].astype(np.uint32)


def check(ok, what):
    if not ok:
        print("FAIL", os.environ.get("RPK_TUNE"), what, flush=True)
        sys.exit(1)


def main():
    import torch

    M = BIG + 37
    for stride in (16, 32):
        base_all = rpk.synth.make_status_records(M, 0, stride=stride)
        next_all = rpk.synth.make_status_records(M, 2, 0.37, stride=stride)
        with rpk.Engine(1) as eng:
            for N in (BIG - 1, BIG, BIG + 37):
                base, nxt = base_all[:N], next_all[:N]
                eng.status_reset(N)
                eng.status_seed(base)
                got, codes, hashes = eng.status_diff(nxt, want_codes=True, want_hashes=True)
                want = changed_rows(base, nxt)
                check(len(want) > N // 10, f"stride {stride} N {N}: the tables barely differ")
                check(np.array_equal(got, want), f"stride {stride} N {N}: changed list")
                check(np.array_equal(codes, oracle.record_codes(nxt)[want]), f"stride {stride} N {N}: codes")
                check(np.array_equal(hashes, oracle.record_hashes(nxt)), f"stride {stride} N {N}: hash column")
                got, _ = eng.status_diff(nxt)
                check(len(got) == 0, f"stride {stride} N {N}: second sweep reported {len(got)} slots")
            # device entry point, caller-owned column seeded by the caller with the reference hashes of `base`
            N = BIG + 37
            d_recs = torch.from_numpy(next_all).cuda()
            col = torch.from_numpy(oracle.record_hashes(base_all).view(np.int64)).cuda()
            d_idx = torch.empty(N, dtype=torch.int32, device="cuda")
            d_code = torch.empty(N, dtype=torch.int16, device="cuda")
            d_n = torch.zeros(1, dtype=torch.int32, device="cuda")
            eng.status_diff_device(d_recs, stride, col, d_idx, d_n, d_changed_code=d_code)
            torch.cuda.synchronize()
            n = int(d_n.item())
            want = changed_rows(base_all, next_all)
            check(np.array_equal(d_idx[:n].cpu().numpy().view(np.uint32), want), f"device stride {stride}: changed list")
            check(np.array_equal(d_code[:n].cpu().numpy().view(np.uint16), oracle.record_codes(next_all)[want]), f"device stride {stride}: codes")
            check(np.array_equal(col.cpu().numpy().view(np.uint64), oracle.record_hashes(next_all)), f"device stride {stride}: column")
            # a column that starts 8 bytes off a 16-byte boundary is refused before anything is launched
            buf = torch.zeros(N + 1, dtype=torch.int64, device="cuda")
            try:
                eng.status_diff_device(d_recs, stride, buf[1:], d_idx, d_n)
                check(False, "a misaligned hash column was accepted")
            except rpk.RpkError as e:
                check(e.code == rpk._ffi.RPK_EINVAL, f"misaligned column: error {e.code}")
            torch.cuda.synchronize()
            check(int(buf.count_nonzero().item()) == 0, "the refused call wrote the column")
            del d_recs, col, d_idx, d_code, d_n, buf
    print("ok", os.environ.get("RPK_TUNE"), flush=True)


if __name__ == "__main__":
    main()
