"""The peer-flag words on ONE GPU: a one-rank group bound to a 64-word array (rpk_peer_bind), gathers into two local
vectors.  Every signalling path -- the persistent select's last pusher, k_peer_signal behind the other select paths
and behind an empty shard, the status sweep's last CTA, rpk_peer_fence -- must move exactly the words include/rpk.h
documents: a select gather adds 1 to words 0 (epoch seen by rank 0) and 32 (own select counter), a status gather to
words 8 and 33.  The multi-GPU protocol itself is tests/test_multi_gpu.py; these checks need no peer."""
import importlib

import numpy as np
import pytest

import oracle
import rpk

pytestmark = pytest.mark.gpu

ROW0 = 3  # off the 16-byte grid: head and tail of the slice copy


@pytest.fixture(scope="module")
def group():
    """-> (engine, device pointer of the rank's zeroed 64-word flag array, read_words())"""
    import torch

    peer = importlib.import_module("k8s-runpod-kubelet_b200.peer")
    dev = torch.device("cuda", 0)
    with rpk.Engine(1) as eng:
        flags = eng.ipc_alloc(64 * 4)[0]

        def words(ptr=flags):
            torch.cuda.synchronize()
            return peer.as_int32_tensor(ptr, 64, dev).cpu().numpy().astype(np.int64)

        yield eng, flags, words


def delta(*idx):
    d = np.zeros(64, np.int64)
    d[list(idx)] = 1
    return d


def gather(eng, offers, pods, P):
    """one rpk_select_device_gather of P rows into two local vectors at ROW0; checked against the oracle"""
    import torch

    dev = torch.device("cuda", 0)
    d_pods = {k: torch.from_numpy(np.ascontiguousarray(v[:P])).to(dev) for k, v in pods.items()}
    vecs = [torch.full((ROW0 + P + 9,), -9, dtype=torch.int32, device=dev) for _ in range(2)]
    eng.select_device_gather(d_pods, [v.data_ptr() for v in vecs], ROW0)
    torch.cuda.synchronize()
    if P:
        ob, _ = oracle.select(offers, {k: v[:P] for k, v in pods.items()}, want_top5=False, n_threads=4)
        for k, v in enumerate(vecs):
            h = v.cpu().numpy()
            assert np.array_equal(h[ROW0:ROW0 + P], ob), f"vector {k}"
            assert (h[:ROW0] == -9).all() and (h[ROW0 + P:] == -9).all(), f"vector {k}: written outside the slice"


# (forced kernel, rows, expected select_kernel_kind): the fused kernel, the persistent kernel (its last pusher signals),
# the packed and generic grids (k_peer_signal behind k_gather_push), and an empty shard (k_peer_signal alone)
PATHS = {"fused": (None, 5_003, 4), "persistent": (None, 40_001, 4), "packed": ("packed", 5_003, 2),
         "generic": ("generic", 5_003, 1), "empty": (None, 0, 4)}


@pytest.mark.parametrize("path", list(PATHS))
def test_bound_gather_signals_once(group, path):
    from test_select_gpu import upload_forced

    eng, flags, words = group
    force, P, kind = PATHS[path]
    offers = rpk.synth.make_offers(20_000, correlated=True)
    upload_forced(eng, offers, force)
    assert eng.stats()["select_kernel_kind"] == kind
    eng.peer_bind([flags], 0)
    pods = rpk.synth.make_pods(max(P, 1), row0=ROW0)
    for _ in range(2):
        before, launches = words(), eng.launch_count()
        gather(eng, offers, pods, P)
        assert np.array_equal(words() - before, delta(0, 32)), (path, words()[:40])
        if P == 0:
            assert eng.launch_count() == launches + 1  # the signal and nothing else
    upload_forced(eng, offers, None)


@pytest.mark.parametrize("stride,N", [(16, 3_001), (32, 3_001), (32, 0)])
def test_bound_status_gather_signals_once(group, stride, N):
    import torch

    eng, flags, words = group
    dev = torch.device("cuda", 0)
    eng.peer_bind([flags], 0)
    cap = max(N, 1)
    xch = torch.zeros(eng.xchg_bytes(1, cap) // 4 + 4, dtype=torch.int32, device=dev)
    hash_prev = torch.zeros(N, dtype=torch.int64, device=dev)
    n_changed = torch.zeros(1, dtype=torch.int32, device=dev)
    tab = oracle.StatusTable(N, stride) if N else None
    for sweep, frac in enumerate([0.0, 0.05]):
        recs = rpk.synth.make_status_records(N, sweep, frac, stride=stride)
        d_recs = torch.from_numpy(recs.reshape(-1).copy()).to(dev)
        xch.fill_(-1)
        before = words()
        eng.status_diff_device_gather(d_recs, stride, hash_prev, 0, [xch.data_ptr()], cap, 0, n_changed)
        assert np.array_equal(words() - before, delta(8, 33)), (stride, N, words()[:40])
        xv = xch.cpu().numpy()
        want = tab.diff(recs) if N else np.zeros(0, np.uint32)
        assert xv[0] == len(want) and int(n_changed.item()) == len(want)
        assert np.array_equal(xv[8:8 + len(want)].astype(np.uint32), want)


def test_unbound_calls_leave_the_flags_alone(group):
    import torch

    eng, flags, words = group
    dev = torch.device("cuda", 0)
    offers = rpk.synth.make_offers(20_000, correlated=True)
    eng.upload_offers(offers)
    pods = rpk.synth.make_pods(40_001, row0=ROW0)
    eng.peer_bind(None, 0)
    try:
        before = words()
        for P in (5_003, 40_001):
            gather(eng, offers, pods, P)
        launches = eng.launch_count()
        gather(eng, offers, pods, 0)
        assert eng.launch_count() == launches  # an empty shard with nothing bound launches nothing
        N = 3_001
        recs = rpk.synth.make_status_records(N, 0, 0.0)
        xch = torch.zeros(eng.xchg_bytes(1, N) // 4 + 4, dtype=torch.int32, device=dev)
        eng.status_diff_device_gather(torch.from_numpy(recs.reshape(-1).copy()).to(dev), 32, torch.zeros(N, dtype=torch.int64, device=dev),
                                      0, [xch.data_ptr()], N, 0, torch.zeros(1, dtype=torch.int32, device=dev))
        assert xch[0].item() == N
        assert np.array_equal(words(), before)
    finally:
        eng.peer_bind([flags], 0)


def test_peer_fence_words(group):
    """rpk_peer_fence with one rank: self-counting moves words 0 and 32; an explicit epoch sets word 0 and leaves 32"""
    eng, _, words = group
    f = eng.ipc_alloc(64 * 4)[0]
    for k in (1, 2):
        eng.peer_fence([f], 0, 0)
        w = words(f)
        assert w[0] == k and w[32] == k and not w[1:32].any() and not w[33:].any(), w[:40]
    eng.peer_fence([f], 0, 7)
    w = words(f)
    assert w[0] == 7 and w[32] == 2 and not w[1:32].any() and not w[33:].any(), w[:40]


def test_waits_on_the_rank_own_words(group):
    """rpk_peer_wait(3) and an inline-wait gather, once each.  With one rank both wait on words this rank has already
    stored (asserted first), so they return at once."""
    eng, flags, words = group
    offers = rpk.synth.make_offers(20_000, correlated=True)
    eng.upload_offers(offers)
    eng.peer_bind([flags], 0)
    w = words()
    assert w[0] == w[32] and w[8] == w[33], w[:40]  # every epoch the counters name has been signalled
    eng.peer_wait(3)
    assert np.array_equal(words(), w)
    eng.peer_inline_wait(True)
    try:
        gather(eng, offers, rpk.synth.make_pods(5_003, row0=ROW0), 5_003)
        assert np.array_equal(words() - w, delta(0, 32))
    finally:
        eng.peer_inline_wait(False)
