"""The device entry points refuse, in Python and before anything is launched, every tensor the C side cannot check behind
its pointer: a host tensor, a tensor on another GPU than the shard's, a wrong dtype, a non-contiguous view, and a
buffer with fewer elements than the call needs.

Every bad input here is harmless even if it slipped through.  Host tensors are pinned, so the GPU can reach them.
Wrong-dtype, strided and short views start at the front of a buffer with room for the valid call, and guard words
surround that buffer.  The other-GPU case runs only in a two-GPU context, where rpk_create has enabled peer access.
An input that slipped through would therefore show up as a launch and as stores into a guarded buffer, and the tests
check both."""
import numpy as np
import pytest

import oracle
import rpk

pytestmark = pytest.mark.gpu

P, N, N_SLOTS, STRIDE = 1000, 1000, 300, 16
PAD = 64  # guard words (int64) before and after every buffer
GUARD = 0x5A5A5A5A5A5A5A5A
WRONG = {"int32": "float32", "int64": "float64", "float64": "int64", "uint8": "int8", "int16": "float16"}
POD_COLS = [("req_mem_gb", "int32"), ("req_vcpu", "int32"), ("req_ram_gb", "int32"), ("max_price", "float64"), ("cloud", "uint8")]


def n_devices():
    import torch

    return torch.cuda.device_count()


class Buf:
    """n elements of `dtype` at the front of a body of 16 bytes per element (room for every view bad() takes), between
    guard words.  Apart from the input data it holds, the body is guard words too, so any store into it shows."""

    def __init__(self, n, dtype, device, data=None):
        import torch

        self.n, self.dtype = n, dtype
        self.mem = torch.full((2 * PAD + 2 * n,), GUARD, dtype=torch.int64, device=device)
        self.body = self.mem[PAD:PAD + 2 * n]
        if data is not None:
            self.valid().copy_(torch.as_tensor(data))
        self.before = self.mem.clone()

    def view(self, dtype, stop, step=1):
        import torch

        return self.body.view(getattr(torch, dtype))[:stop:step]

    def valid(self):
        return self.view(self.dtype, self.n)

    def touched(self):
        import torch

        return not torch.equal(self.mem, self.before)


def bad(kind, buf, defines_size, others):
    """the `kind` of bad stand-in for buf's valid tensor, or None where that kind does not apply"""
    if kind == "host":
        return buf.valid().cpu().pin_memory()
    if kind == "dtype":
        return buf.view(WRONG[buf.dtype], buf.n)
    if kind == "strided":  # a one-element view is contiguous whatever its stride
        return buf.view(buf.dtype, 2 * buf.n, 2) if buf.n > 1 else None
    if kind == "short":  # a shorter size-defining tensor is just a smaller call
        return None if defines_size else buf.view(buf.dtype, buf.n - 1)
    assert kind == "other_gpu", kind
    other = Buf(buf.n, buf.dtype, "cuda:1", buf.valid())
    others.append(other)
    return other.valid()


def select_case(offers, dev, gather):
    """-> (arguments {name: Buf}, size-defining names, buffers reached through raw pointers, call(eng, tensors),
    check of the valid call's result)"""
    pods = rpk.synth.make_pods(P)
    args = {k: Buf(P, dt, dev, pods[k]) for k, dt in POD_COLS}
    args["d_top5"] = Buf(5 * P, "int32", dev)
    want = oracle.select(offers, pods, want_top5=False)[0]

    def cols(a):
        return {k: a[k] for k, _ in POD_COLS}

    if gather:
        vec = Buf(P, "int32", dev)
        return (args, {"req_mem_gb"}, [vec],
                lambda eng, a: eng.select_device_gather(cols(a), [vec.valid().data_ptr()], 0, a["d_top5"]),
                lambda: np.array_equal(vec.valid().cpu().numpy(), want))
    args["d_best"] = Buf(P, "int32", dev)
    return (args, {"req_mem_gb"}, [], lambda eng, a: eng.select_device(cols(a), a["d_best"], a["d_top5"]),
            lambda: np.array_equal(args["d_best"].valid().cpu().numpy(), want))


def status_case(eng, dev, method):
    """the same for the status sweeps; the hash column holds guard words, so every compared slot reports changed"""
    recs = rpk.synth.make_status_records(N, 0, stride=STRIDE)
    n = N_SLOTS if method == "status_diff_slots_device" else N
    args = {"d_hash_prev": Buf(N, "int64", dev)}
    defining, raw = {"d_hash_prev"}, []
    if method == "status_diff_slots_device":
        slots = np.arange(0, 3 * N_SLOTS, 3, dtype=np.int32)
        args["d_slots"] = Buf(n, "int32", dev, slots)
        args["d_records"] = Buf(n * STRIDE, "uint8", dev, recs[slots].reshape(-1))
        defining.add("d_slots")
    else:
        args["d_records"] = Buf(n * STRIDE, "uint8", dev, recs.reshape(-1))
    if method == "status_diff_device_gather":
        xch = Buf(eng.xchg_bytes(1, N) // 4, "int32", dev)
        raw.append(xch)

        def call(eng, a):
            eng.status_diff_device_gather(a["d_records"], STRIDE, a["d_hash_prev"], 0, [xch.valid().data_ptr()], N, 0,
                                          a["d_n_changed"])
    else:
        args["d_changed_idx"] = Buf(n, "int32", dev)
        args["d_changed_code"] = Buf(n, "int16", dev)
        if method == "status_diff_device":
            def call(eng, a):
                eng.status_diff_device(a["d_records"], STRIDE, a["d_hash_prev"], a["d_changed_idx"], a["d_n_changed"],
                                       d_changed_code=a["d_changed_code"])
        else:
            def call(eng, a):
                eng.status_diff_slots_device(a["d_slots"], a["d_records"], STRIDE, a["d_hash_prev"], a["d_changed_idx"],
                                             a["d_n_changed"], d_changed_code=a["d_changed_code"])
    args["d_n_changed"] = Buf(1, "int32", dev)
    return args, defining, raw, call, lambda: int(args["d_n_changed"].valid().item()) == n


METHODS = ["select_device", "select_device_gather", "status_diff_device", "status_diff_slots_device", "status_diff_device_gather"]


@pytest.fixture(scope="module")
def ctx():
    """a two-GPU context where there are two GPUs (peer access enabled), else one; offers uploaded"""
    offers = rpk.synth.make_offers(2000, correlated=True)
    with rpk.Engine(min(n_devices(), 2)) as eng:
        eng.upload_offers(offers)
        yield eng, offers


@pytest.mark.parametrize("kind", ["host", "dtype", "strided", "short", "other_gpu"])
@pytest.mark.parametrize("method", METHODS)
def test_bad_device_argument_is_refused(ctx, method, kind):
    """each argument of `method` in turn replaced by its `kind` of bad stand-in, the others valid: TypeError or
    ValueError, no launch, no store; then the all-valid call is accepted and computes the right result"""
    import torch

    eng, offers = ctx
    if kind == "other_gpu" and eng.n_gpus < 2:
        pytest.skip("needs 2 GPUs")
    dev = torch.device("cuda", 0)
    if method.startswith("select"):
        args, defining, raw, call, result_ok = select_case(offers, dev, method == "select_device_gather")
    else:
        args, defining, raw, call, result_ok = status_case(eng, dev, method)
    others, tried = [], 0
    for name, buf in args.items():
        t = bad(kind, buf, name in defining, others)
        if t is None:
            continue
        tried += 1
        launches = eng.launch_count()
        try:
            call(eng, {**{k: b.valid() for k, b in args.items()}, name: t})
            refused = None
        except (TypeError, ValueError) as e:
            refused = e
        torch.cuda.synchronize()
        launched = eng.launch_count() - launches
        touched = [k for k, b in args.items() if b.touched()] + ["raw-pointer buffer" for b in raw + others if b.touched()]
        assert not launched and not touched, f"{name} ({kind}): {launched} kernels launched, stores into {touched}"
        assert refused is not None, f"{name} ({kind}): accepted"
    assert tried, "no argument takes this kind of bad input"
    launches = eng.launch_count()
    call(eng, {k: b.valid() for k, b in args.items()})
    torch.cuda.synchronize()
    assert eng.launch_count() > launches and result_ok(), "the valid arguments were not accepted"


def test_default_stream_is_the_shard_gpu():
    """Engine(2), torch's current device 0 running a stream of its own: select_device on shard 1 without a stream
    enqueues on GPU 1's current stream, not on the current device's."""
    import torch

    if n_devices() < 2:
        pytest.skip("needs 2 GPUs")
    offers = rpk.synth.make_offers(2000, correlated=True)
    pods = rpk.synth.make_pods(P)
    with rpk.Engine(2) as eng:
        eng.upload_offers(offers)
        d_pods = {k: torch.from_numpy(v).to("cuda:1") for k, v in pods.items()}
        d_best = torch.full((P,), -7, dtype=torch.int32, device="cuda:1")
        torch.cuda.synchronize(1)
        with torch.cuda.device(0), torch.cuda.stream(torch.cuda.Stream(device=0)):
            eng.select_device(d_pods, d_best, shard=1)
        torch.cuda.synchronize(1)
        assert np.array_equal(d_best.cpu().numpy(), oracle.select(offers, pods, want_top5=False)[0])
