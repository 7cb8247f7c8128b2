"""rpk_select_slots_device_gather and rpk_select_slots_device_gather_top5: the sharded select over a device list of
pod-table slots.  Rank r takes list entries [lo_r, hi_r) at row0 = lo_r; its results land at [row0, row0 + n_r) of every
assignment vector and its lists at [5*row0, 5*(row0 + n_r)) of every top-5 vector, so after every rank's call each vector
holds the whole list's results in list order.  With flags bound the call signals the select epoch once.

On one GPU the ranks are emulated: every "rank" is one call on the same ctx, and the "peers" are local vectors (the push
kernel is the one that stores over NVLink); the cross-GPU case is the last test.  Every output starts as SENTINEL and
must keep it outside the slices written."""
import importlib
import zlib

import numpy as np
import pytest

import rpk
import select_plan_cases as sc
from test_select_slots_gpu import PodTable, seeded_engine, slot_list, tracked

pytestmark = pytest.mark.gpu

N_OUT = 3   # vectors of each kind per call: the local one and two that receive the push
SPARE = 9   # elements past the list in every vector
OUTSIDE = np.array([1 << 20, 0xFFFFFFFF], np.uint32)


def delta(*idx):
    d = np.zeros(64, np.int64)
    d[list(idx)] = 1
    return d


def d_list(sl):
    import torch

    return torch.from_numpy(np.ascontiguousarray(sl, np.uint32).view(np.int32)).cuda()


def vectors(n, top5):
    import torch

    best = [torch.full((n + SPARE,), sc.SENTINEL, dtype=torch.int32, device="cuda:0") for _ in range(N_OUT)]
    lists = [torch.full((5 * n + SPARE,), sc.SENTINEL, dtype=torch.int32, device="cuda:0") for _ in range(N_OUT)] if top5 else []
    return best, lists


def reset(vecs):
    for v in vecs:
        v.fill_(sc.SENTINEL)


def gather(eng, d, lo, hi, best, lists, stream=None):
    """rank's call: entries [lo, hi) of the device list at row0 = lo"""
    eng.select_slots_device_gather(d[lo:hi], [v.data_ptr() for v in best], lo, stream=stream,
                                   top5_ptrs=[v.data_ptr() for v in lists] if lists else None)


def expect(eb, et, sl):
    """oracle rows of a list; entries outside the table: -1 and five -1"""
    bad = sl >= len(eb)
    ok = np.where(bad, 0, sl)
    wb, wt = eb[ok].copy(), et[ok].copy()
    wb[bad], wt[bad] = -1, -1
    return wb, wt


def with_head(wb, wt, k=3):
    """expected vectors of a call at row0 = k: k SENTINEL rows first"""
    return (np.concatenate([np.full(k, sc.SENTINEL, np.int32), wb]),
            np.concatenate([np.full((k, 5), sc.SENTINEL, np.int32), wt]))


def check(best, lists, wb, wt, upto, what):
    """every vector holds rows [0, upto) of the expected results and SENTINEL after them"""
    import torch

    torch.cuda.synchronize()
    for k, v in enumerate(best):
        h = v.cpu().numpy()
        sc.check(f"{what}: best vector {k}", h[:upto], None, wb[:upto], None)
        assert (h[upto:] == sc.SENTINEL).all(), f"{what}: best vector {k} written past row {upto}"
    for k, v in enumerate(lists):
        h = v.cpu().numpy()
        got = h[:5 * upto].reshape(upto, 5)
        assert np.array_equal(got, wt[:upto]), f"{what}: top-5 vector {k} differs at rows {np.nonzero((got != wt[:upto]).any(axis=1))[0][:6]}"
        assert (h[5 * upto:] == sc.SENTINEL).all(), f"{what}: top-5 vector {k} written past row {5 * upto}"


@pytest.fixture(scope="module")
def group():
    """-> (engine seeded as test_select_slots_gpu's synth20k table, oracle best / top5 per slot, flag array pointer,
    read_words())"""
    import torch

    peer = importlib.import_module("k8s-runpod-kubelet_b200.peer")
    _, eb, et, _ = tracked("synth20k")
    eng = seeded_engine("synth20k")
    flags = eng.ipc_alloc(64 * 4)[0]

    def words():
        torch.cuda.synchronize()
        return peer.as_int32_tensor(flags, 64, torch.device("cuda", 0)).cpu().numpy().astype(np.int64)

    try:
        yield eng, eb, et, flags, words
    finally:
        eng.close()


@pytest.mark.parametrize("top5", [False, True])
@pytest.mark.parametrize("ranks", [1, 2, 3, 8])
def test_emulated_ranks_assemble_the_whole_list(group, ranks, top5):
    """ragged parts of one list (shuffled, repeats and entries outside the table), each rank at its row0; 40 001 / 3
    puts rank 1's lists 13 333 * 20 bytes in, off the 16-byte grid"""
    eng, eb, et, flags, words = group
    eng.peer_bind([flags], 0)
    rng = np.random.default_rng(zlib.crc32(f"ranks/{ranks}/{top5}".encode()))
    for n in (40_001, 262_147):
        sl = slot_list(rng, n, "repeats" if n % 2 else "shuffled")
        sl[rng.integers(0, n, 5)] = OUTSIDE[rng.integers(0, 2, 5)]
        wb, wt = expect(eb, et, sl)
        d = d_list(sl)
        best, lists = vectors(n, top5)
        for rep in range(2):
            reset(best + lists)
            for r in range(ranks):
                lo, hi = n * r // ranks, n * (r + 1) // ranks
                before = words()
                gather(eng, d, lo, hi, best, lists)
                what = f"{ranks} ranks, n={n}, top5={top5}, call {rep}, rank {r}"
                check(best, lists, wb, wt, hi, what)
                assert np.array_equal(words() - before, delta(0, 32)), what


@pytest.mark.parametrize("n", [5_003, 40_001])
@pytest.mark.parametrize("inline", [False, True])
def test_flag_words_with_and_without_the_inline_wait(group, n, inline):
    eng, eb, et, flags, words = group
    eng.peer_bind([flags], 0)
    rng = np.random.default_rng(n)
    sl = slot_list(rng, n, "shuffled")
    wb, wt = expect(eb, et, sl)
    d = d_list(sl)
    wb, wt = with_head(wb, wt)
    best, lists = vectors(n + 3, True)
    bp, tp = [v.data_ptr() for v in best], [v.data_ptr() for v in lists]
    eng.select_slots_device_gather(d, bp, 3, top5_ptrs=tp)  # sizes the scratch before the inline wait is on
    eng.select_slots_device_gather(d, bp, 3)
    words()
    eng.peer_inline_wait(inline)
    try:
        for _ in range(2):
            reset(best + lists)
            before = words()
            eng.select_slots_device_gather(d, bp, 3, top5_ptrs=tp)
            check(best, lists, wb, wt, n + 3, f"inline={inline}")
            assert np.array_equal(words() - before, delta(0, 32)), words()[:40]
            before = words()
            eng.select_slots_device_gather(d, bp, 3)  # assignments only: the same signal
            assert np.array_equal(words() - before, delta(0, 32)), words()[:40]
    finally:
        eng.peer_inline_wait(False)


def test_empty_list_signals_and_launches_only_the_signal(group):
    import torch

    eng, eb, et, flags, words = group
    best, lists = vectors(4, True)
    empty = torch.zeros(0, dtype=torch.int32, device="cuda:0")
    for bound in (True, False):
        eng.peer_bind([flags] if bound else None, 0)
        for top5 in (False, True):
            before, c0 = words(), eng.launch_count()
            gather(eng, empty, 0, 0, best, lists if top5 else [])
            assert eng.launch_count() == c0 + (1 if bound else 0), (bound, top5)
            assert np.array_equal(words() - before, delta(0, 32) if bound else np.zeros(64, np.int64)), (bound, top5)
            check(best, lists, np.zeros(0, np.int32), np.zeros((0, 5), np.int32), 0, f"empty, bound={bound}")
    eng.peer_bind([flags], 0)


@pytest.mark.parametrize("n", [5_003, 40_001])
def test_replay_from_a_cuda_graph_picks_up_new_seeds(n):
    """one warm call, the next captured; between replays the host re-seeds rows the list names and writes a new list
    into the captured tensor: every replay reads the table and the list as they are then"""
    import torch

    offers = sc.table("synth20k")
    N = 100_000
    rng = np.random.default_rng(n)
    with rpk.Engine(1) as eng:
        eng.upload_offers(offers)
        eng.pods_reset(N)
        m = PodTable(N)
        flags = eng.ipc_alloc(64 * 4)[0]
        eng.peer_bind([flags], 0)
        sl = slot_list(rng, n, "shuffled", N)
        dd = d_list(np.concatenate([sl[:3], sl]))  # the call takes dd[3:]: the list starts 12 bytes in
        best, lists = vectors(n + 3, True)
        s = torch.cuda.Stream(device="cuda:0")
        torch.cuda.synchronize()
        with torch.cuda.stream(s):
            gather(eng, dd, 3, n + 3, best, lists)
        s.synchronize()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=s, capture_error_mode="relaxed"):
            gather(eng, dd, 3, n + 3, best, lists)
        for it in range(3):
            rows = np.sort(rng.choice(N, N // 4, replace=False)).astype(np.uint32)
            pods = sc.pods_for("synth20k", len(rows), seed=200 + it)
            eng.pods_seed_slots(rows, pods)
            m.seed(rows, pods)
            if it == 2:  # a new list in the captured tensor
                sl = slot_list(rng, n, "repeats", N)
                dd[3:].copy_(d_list(sl))
            torch.cuda.synchronize()
            reset(best + lists)
            wb, wt = with_head(*sc.expected(offers, m.rows(sl)))
            g.replay()
            s.synchronize()
            check(best, lists, wb, wt, n + 3, f"replay {it}")


@pytest.mark.parametrize("n", [2, 4, 8])
def test_every_gpu_holds_every_pending_pods_results(n):
    """One ctx over n GPUs, every GPU with the whole pod table seeded alike, one stream per shard: each shard takes its
    part of one list and gathers the assignments and lists into every GPU's vectors (NVLink peer stores), the bound
    group's rpk_peer_wait closes the step; two steps on two vector sets, with a seed in between."""
    import torch

    if torch.cuda.device_count() < n:
        pytest.skip(f"needs {n} GPUs")
    peer = importlib.import_module("k8s-runpod-kubelet_b200.peer")
    offers = sc.table("synth20k")
    N, P = 400_000, 150_003
    rng = np.random.default_rng(n)
    m = PodTable(N)
    with rpk.Engine(n) as eng:
        eng.upload_offers(offers)
        eng.pods_reset(N)
        every = np.arange(N, dtype=np.uint32)
        pods = sc.pods_for("synth20k", N, seed=3)
        eng.pods_seed_slots(every, pods)
        m.seed(every, pods)
        sl = slot_list(rng, P, "shuffled", N)
        vec = [[eng.ipc_alloc(P * 4, shard=s)[0] for s in range(n)] for _ in range(2)]   # [set][shard]
        lists = [[eng.ipc_alloc(P * 20, shard=s)[0] for s in range(n)] for _ in range(2)]
        flags = [eng.ipc_alloc(64 * 4, shard=s)[0] for s in range(n)]
        streams, d_sl = [], []
        for s in range(n):
            dev = torch.device("cuda", s)
            lo, hi = P * s // n, P * (s + 1) // n
            with torch.cuda.device(s):
                streams.append(torch.cuda.Stream(device=dev))
                d_sl.append(torch.from_numpy(np.ascontiguousarray(sl[lo:hi]).view(np.int32)).to(dev))
            eng.peer_bind(flags, s, shard=s)
        for s in range(n):
            torch.cuda.synchronize(s)
        for step in range(2):
            if step:
                rows = np.sort(rng.choice(N, N // 3, replace=False)).astype(np.uint32)
                fresh = sc.pods_for("synth20k", len(rows), seed=4)
                eng.pods_seed_slots(rows, fresh)
                m.seed(rows, fresh)
            ob, ot = sc.expected(offers, m.rows(sl))
            par = step & 1
            for s in (range(n) if par else reversed(range(n))):   # issue order must not matter
                with torch.cuda.device(s):
                    eng.select_slots_device_gather(d_sl[s], vec[par], P * s // n, shard=s, stream=streams[s].cuda_stream,
                                                   top5_ptrs=lists[par])
                    eng.peer_wait(1, shard=s, stream=streams[s].cuda_stream)
            for st in streams:
                st.synchronize()
            for s in range(n):
                with torch.cuda.device(s):
                    dev = torch.device("cuda", s)
                    b = peer.as_int32_tensor(vec[par][s], P, dev).cpu().numpy()
                    t = peer.as_int32_tensor(lists[par][s], 5 * P, dev).cpu().numpy().reshape(P, 5)
                    sc.check(f"step {step}: GPU {s}", b, t, ob, ot)
