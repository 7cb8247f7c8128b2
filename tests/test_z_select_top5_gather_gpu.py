"""rpk_select_device_gather_top5: the sharded select's all-gather carrying the gpuTypeIds lists.  A shard's results land
at [row0, row0+P) of every assignment vector and its lists at [5*row0, 5*(row0+P)) of every top-5 vector; with flags
bound the call signals the select epoch once, after both slices have landed.  On one GPU the "peers" are local vectors
(the push kernel is the same one that stores over NVLink); the cross-GPU case is the last test.  Every output is
pre-filled with -9 and compared with the oracle on the slice and with -9 outside it."""
import ctypes as C
import importlib

import numpy as np
import pytest

import oracle
import rpk

pytestmark = pytest.mark.gpu

EINVAL = rpk._ffi.RPK_EINVAL
N_OUT = 3   # vectors of each kind per call: the local one and two that receive the push
G = 20_000
COLS = ("req_mem_gb", "req_vcpu", "req_ram_gb", "max_price", "cloud")


@pytest.fixture(scope="module")
def group():
    """-> (engine, offers, device pointer of the rank's zeroed 64-word flag array, read_words())"""
    import torch

    peer = importlib.import_module("k8s-runpod-kubelet_b200.peer")
    dev = torch.device("cuda", 0)
    offers = rpk.synth.make_offers(G, correlated=True)
    with rpk.Engine(1) as eng:
        eng.upload_offers(offers)
        flags = eng.ipc_alloc(64 * 4)[0]

        def words():
            torch.cuda.synchronize()
            return peer.as_int32_tensor(flags, 64, dev).cpu().numpy().astype(np.int64)

        yield eng, offers, flags, words


def delta(*idx):
    d = np.zeros(64, np.int64)
    d[list(idx)] = 1
    return d


def device_pods(pods, P):
    import torch

    return {k: torch.from_numpy(np.ascontiguousarray(v[:P])).to("cuda:0") for k, v in pods.items()}


def outputs(row0, P):
    """N_OUT assignment and N_OUT top-5 vectors, -9 everywhere, 9 spare elements past the slice"""
    import torch

    best = [torch.full((row0 + P + 9,), -9, dtype=torch.int32, device="cuda:0") for _ in range(N_OUT)]
    top5 = [torch.full((5 * (row0 + P) + 9,), -9, dtype=torch.int32, device="cuda:0") for _ in range(N_OUT)]
    return best, top5


def reset(vecs):
    for v in vecs:
        v.fill_(-9)


def check(offers, pods, P, row0, best, top5, what=""):
    import torch

    torch.cuda.synchronize()
    if P:
        ob, ot = oracle.select(offers, {k: v[:P] for k, v in pods.items()}, want_top5=True, n_threads=8)
    for k, v in enumerate(best):
        h = v.cpu().numpy()
        if P:
            assert np.array_equal(h[row0:row0 + P], ob), f"{what}: best vector {k}"
        assert (h[:row0] == -9).all() and (h[row0 + P:] == -9).all(), f"{what}: best vector {k} written outside the slice"
    for k, v in enumerate(top5):
        h = v.cpu().numpy()
        if P:
            assert np.array_equal(h[5 * row0:5 * (row0 + P)].reshape(P, 5), ot), f"{what}: top-5 vector {k}"
        assert (h[:5 * row0] == -9).all() and (h[5 * (row0 + P):] == -9).all(), f"{what}: top-5 vector {k} written outside the slice"


def gather_top5(eng, d_pods, best, top5, row0, stream=None):
    eng.select_device_gather(d_pods, [v.data_ptr() for v in best], row0, top5_ptrs=[v.data_ptr() for v in top5], stream=stream)


def raw_call(eng, d_pods, P, best_ptrs, top5_ptrs, row0, n_out=None):
    """rpk_select_device_gather_top5 straight from the library (arguments the Python binding would refuse first)"""
    import torch

    n_out = len(best_ptrs) if n_out is None else n_out
    arr = lambda ptrs: (C.c_void_p * max(len(ptrs), 1))(*ptrs)
    cols = [C.c_void_p(d_pods[k].data_ptr()) if k in d_pods else None for k in COLS]
    return eng._lib.rpk_select_device_gather_top5(eng._ctx, 0, P, *cols, n_out, arr(best_ptrs), arr(top5_ptrs), row0,
                                                   C.c_void_p(torch.cuda.current_stream(0).cuda_stream or 1))


# (forced kernel, rows, expected select_kernel_kind): the fused kernel, the persistent kernel at two sizes (it pushes
# the assignments itself and must leave the signal to the call), the packed and generic grids, and an empty shard
PATHS = {"fused": (None, 5_003, 4), "persistent": (None, 40_001, 4), "persistent_large": (None, 262_147, 4),
         "packed": ("packed", 5_003, 2), "generic": ("generic", 5_003, 1), "empty": (None, 0, 4)}


@pytest.mark.parametrize("row0", [0, 3])   # 3: the lists' slice starts 60 bytes in, the push copies a head and a tail
@pytest.mark.parametrize("path", list(PATHS))
def test_every_select_path_gathers_both_slices_and_signals_once(group, path, row0):
    from test_select_gpu import upload_forced

    eng, offers, flags, words = group
    force, P, kind = PATHS[path]
    upload_forced(eng, offers, force)
    try:
        assert eng.stats()["select_kernel_kind"] == kind
        eng.peer_bind([flags], 0)
        pods = rpk.synth.make_pods(max(P, 1), row0=row0 + 11)
        d_pods = device_pods(pods, P)
        best, top5 = outputs(row0, P)
        for _ in range(2):
            reset(best + top5)
            before, launches = words(), eng.launch_count()
            gather_top5(eng, d_pods, best, top5, row0)
            check(offers, pods, P, row0, best, top5, path)
            assert np.array_equal(words() - before, delta(0, 32)), (path, words()[:40])
            if P == 0:
                assert eng.launch_count() == launches + 1  # the signal and nothing else
    finally:
        upload_forced(eng, offers, None)


@pytest.mark.parametrize("P", [5_003, 40_001])
@pytest.mark.parametrize("inline", [False, True])
def test_flag_words_with_and_without_the_inline_wait(group, P, inline):
    eng, offers, flags, words = group
    eng.peer_bind([flags], 0)
    pods = rpk.synth.make_pods(P, row0=5)
    d_pods = device_pods(pods, P)
    best, top5 = outputs(3, P)
    gather_top5(eng, d_pods, best, top5, 3)   # sizes the scratch before the inline wait is on
    words()
    eng.peer_inline_wait(inline)
    try:
        for _ in range(2):
            reset(best + top5)
            before = words()
            gather_top5(eng, d_pods, best, top5, 3)
            check(offers, pods, P, 3, best, top5, f"inline={inline}")
            assert np.array_equal(words() - before, delta(0, 32)), words()[:40]
    finally:
        eng.peer_inline_wait(False)


def test_unbound_calls_leave_the_flags_alone(group):
    eng, offers, flags, words = group
    eng.peer_bind(None, 0)
    try:
        before = words()
        for P in (5_003, 40_001, 0):
            pods = rpk.synth.make_pods(max(P, 1), row0=P)
            d_pods = device_pods(pods, P)
            best, top5 = outputs(3, P)
            launches = eng.launch_count()
            gather_top5(eng, d_pods, best, top5, 3)
            check(offers, pods, P, 3, best, top5, f"P={P}")
            if P == 0:
                assert eng.launch_count() == launches  # an empty shard with nothing bound launches nothing
        assert np.array_equal(words(), before)
    finally:
        eng.peer_bind([flags], 0)


def test_refusals_enqueue_nothing_and_signal_nothing(group):
    import torch

    eng, offers, flags, words = group
    eng.peer_bind([flags], 0)
    P, row0 = 40_001, 3
    pods = rpk.synth.make_pods(P, row0=row0)
    d_pods = device_pods(pods, P)
    best, top5 = outputs(row0, P)
    bp, tp = [v.data_ptr() for v in best], [v.data_ptr() for v in top5]
    gather_top5(eng, d_pods, best, top5, row0)   # a warm call: the scratch is sized
    reset(best + top5)
    before = words()

    def refused(rc, what):
        assert rc == EINVAL, (what, rc, eng._lib.rpk_last_error(eng._ctx))
        torch.cuda.synchronize()
        for k, v in enumerate(best + top5):
            assert (v == -9).all(), f"{what}: vector {k} written"
        assert np.array_equal(words(), before), f"{what}: flag words moved"

    with pytest.raises(rpk.RpkError) as ei:   # top-5 vectors of different 16-byte phase
        eng.select_device_gather(d_pods, bp, row0, top5_ptrs=[tp[0], tp[1] + 4, tp[2]])
    refused(ei.value.code, "phase")
    host = [eng._lib.rpk_host_alloc(5 * (row0 + P) * 4) for _ in range(N_OUT)]
    try:   # pinned host memory: no top-5 vector lives on the shard's GPU
        assert all(host)
        refused(raw_call(eng, d_pods, P, bp, host, row0), "host vectors")
        refused(raw_call(eng, d_pods, P, bp[:1], host[:1], row0), "one host vector")
    finally:
        for h in host:
            eng._lib.rpk_host_free(h)
    refused(raw_call(eng, d_pods, P, bp, [tp[0], None, tp[2]], row0), "NULL top-5 vector")
    refused(raw_call(eng, d_pods, P, [bp[0], None, bp[2]], tp, row0), "NULL best vector")
    refused(raw_call(eng, d_pods, P, bp * 3, tp * 3, row0, n_out=9), "n_out = 9")
    refused(raw_call(eng, d_pods, P, bp, tp, row0, n_out=0), "n_out = 0")
    refused(raw_call(eng, d_pods, 858_993_460, bp, tp, row0), "5*P beyond uint32")
    with pytest.raises(ValueError):   # the binding refuses a local list and a gathered one together
        eng.select_device_gather(d_pods, bp, row0, d_top5=top5[0][:5 * P], top5_ptrs=tp)
    assert np.array_equal(words(), before)

    gather_top5(eng, d_pods, best, top5, row0)   # the next valid call is correct and signals once
    check(offers, pods, P, row0, best, top5, "after the refusals")
    assert np.array_equal(words() - before, delta(0, 32))


@pytest.mark.parametrize("P", [5_003, 40_001])
def test_replay_from_a_cuda_graph(group, P):
    """one warm call, the next captured, three replays over new pod columns copied into the captured tensors"""
    import torch

    eng, offers, flags, words = group
    eng.peer_bind([flags], 0)
    row0 = 3
    pods = [rpk.synth.make_pods(P, row0=r) for r in (0, 1_000_000, 2_000_000, 3_000_000)]
    d_pods = device_pods(pods[0], P)
    best, top5 = outputs(row0, P)
    s = torch.cuda.Stream(device="cuda:0")
    with torch.cuda.stream(s):
        gather_top5(eng, d_pods, best, top5, row0)
    s.synchronize()
    check(offers, pods[0], P, row0, best, top5, "warm call")
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=s, capture_error_mode="relaxed"):
        gather_top5(eng, d_pods, best, top5, row0)
    for it in (1, 2, 3):
        for k, v in pods[it].items():
            d_pods[k].copy_(torch.from_numpy(v))
        reset(best + top5)
        before = words()
        g.replay()
        check(offers, pods[it], P, row0, best, top5, f"replay {it}")
        assert np.array_equal(words() - before, delta(0, 32)), f"replay {it}"


def test_sequences_on_one_context(group):
    """the lists' gather interleaved with the plain gather, the host select with top5 and the lists' gather on a second
    stream, at changing sizes on one ctx: every step is checked (the select scope orders the two streams)"""
    import torch

    eng, offers, flags, words = group
    eng.peer_bind([flags], 0)
    side = torch.cuda.Stream(device="cuda:0")
    steps = [("top5", 40_001, 3), ("plain", 40_001, 0), ("host", 20_001, 0), ("top5", 5_003, 0),
             ("side", 70_003, 3), ("plain", 5_003, 3), ("top5", 70_003, 3), ("host", 3_001, 0), ("side", 40_001, 0),
             ("top5", 40_001, 3)]
    for i, (kind, P, row0) in enumerate(steps):
        pods = rpk.synth.make_pods(P, row0=1_000 * i)
        what = f"step {i} ({kind}, P={P})"
        if kind == "host":
            b, t = eng.select(pods, want_top5=True)
            ob, ot = oracle.select(offers, pods, want_top5=True, n_threads=8)
            assert np.array_equal(b, ob) and np.array_equal(t, ot), what
            continue
        d_pods = device_pods(pods, P)
        best, top5 = outputs(row0, P)
        before = words()
        if kind == "plain":
            eng.select_device_gather(d_pods, [v.data_ptr() for v in best], row0)
            check(offers, pods, P, row0, best, [], what)
        elif kind == "side":
            torch.cuda.current_stream(0).synchronize()   # the tensors above were filled on the current stream
            gather_top5(eng, d_pods, best, top5, row0, stream=side.cuda_stream)
            side.synchronize()
            check(offers, pods, P, row0, best, top5, what)
        else:
            gather_top5(eng, d_pods, best, top5, row0)
            check(offers, pods, P, row0, best, top5, what)
        assert np.array_equal(words() - before, delta(0, 32)), what


@pytest.mark.parametrize("n", [2, 4, 8])
def test_every_gpu_holds_every_list(n):
    """One ctx over n GPUs, one stream per shard: each shard gathers its rows' assignments and lists into every GPU's
    vectors (NVLink peer stores), the bound group's rpk_peer_wait closes the step; two steps on two vector sets,
    ragged shards whose slices sit off the 16-byte grid."""
    import torch

    if torch.cuda.device_count() < n:
        pytest.skip(f"needs {n} GPUs")
    peer = importlib.import_module("k8s-runpod-kubelet_b200.peer")
    offers = rpk.synth.make_offers(G, correlated=True)
    P = 150_003
    pods = rpk.synth.make_pods(P)
    ob, ot = oracle.select(offers, pods, want_top5=True, n_threads=8)
    with rpk.Engine(n) as eng:
        eng.upload_offers(offers)
        vec = [[eng.ipc_alloc(P * 4, shard=s)[0] for s in range(n)] for _ in range(2)]   # [set][shard]
        lists = [[eng.ipc_alloc(P * 20, shard=s)[0] for s in range(n)] for _ in range(2)]
        flags = [eng.ipc_alloc(64 * 4, shard=s)[0] for s in range(n)]
        streams, d_pods = [], []
        for s in range(n):
            dev = torch.device("cuda", s)
            lo, hi = P * s // n, P * (s + 1) // n
            with torch.cuda.device(s):
                streams.append(torch.cuda.Stream(device=dev))
                d_pods.append({k: torch.from_numpy(np.ascontiguousarray(v[lo:hi])).to(dev) for k, v in pods.items()})
            eng.peer_bind(flags, s, shard=s)
        for s in range(n):
            torch.cuda.synchronize(s)
        for step in range(2):
            par = step & 1
            for s in (range(n) if par else reversed(range(n))):   # issue order must not matter
                with torch.cuda.device(s):
                    eng.select_device_gather(d_pods[s], vec[par], P * s // n, shard=s, stream=streams[s].cuda_stream,
                                             top5_ptrs=lists[par])
                    eng.peer_wait(1, shard=s, stream=streams[s].cuda_stream)
            for st in streams:
                st.synchronize()
            for s in range(n):
                with torch.cuda.device(s):
                    dev = torch.device("cuda", s)
                    b = peer.as_int32_tensor(vec[par][s], P, dev).cpu().numpy()
                    t = peer.as_int32_tensor(lists[par][s], 5 * P, dev).cpu().numpy().reshape(P, 5)
                    assert np.array_equal(b, ob), f"step {step}: GPU {s} does not hold the oracle's vector"
                    assert np.array_equal(t, ot), f"step {step}: GPU {s} does not hold the oracle's lists"
