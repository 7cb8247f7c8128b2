"""Tables, pod batches and the one result checker of the persistent-select plan tests (test_select_plans_gpu.py,
select_plan_child.py, test_select_sequences_gpu.py).

Every output buffer is filled with SENTINEL before a call, so a row the kernels never write shows up, and every row of
`best` (and of `top5` when requested) is compared with the oracle.  Where P x G is too large for a row-by-row oracle
run, rows are grouped by their class -- (mem, vcpu, ram threshold from searchsorted on the table's distinct values,
max_price, cloud) -- and the oracle runs on one representative row per class: rows of one class meet exactly the same
offers under the same price bound, so their results are equal (the class property, extended to top-5)."""
import functools
import os
from contextlib import contextmanager

import numpy as np

import oracle
import persist_plan_model as model
import rpk

SENTINEL = -9
ROW_ORACLE_LIMIT = 5 * 10**8  # P x G up to this: oracle.select on every row


def _table(G, mem, vcpu, ram, rng, price_scale=1.0):
    """offers with the given columns; prices in cents grow with the row's ranks (plus noise), 2 % of them are 0
    (never feasible), and many prices repeat, so the tie rule and the strict price bound both matter"""
    rank = sum(np.searchsorted(np.unique(c), c) for c in (mem, vcpu, ram) if c is not None)
    cents = 5 + (rank * 7 * price_scale).astype(np.int64) + rng.integers(0, 40, G)
    cents[rng.random(G) < 0.02] = 0
    return {"mem_gb": mem.astype(np.int32), "vcpu": None if vcpu is None else vcpu.astype(np.int32),
            "ram_gb": None if ram is None else ram.astype(np.int32),
            "secure_price": cents.astype(np.float64) / 100.0,
            "community_price": ((cents * 6) // 10).astype(np.float64) / 100.0,
            "flags": rng.integers(0, 4, G).astype(np.uint8)}


def _columns(G, values, rng):
    """one column over G rows that takes every value of `values` (the first len(values) rows hold one each)"""
    col = rng.choice(values, G)
    col[: len(values)] = values
    return rng.permutation(col)


def distinct_table(G, dm, dv, dr, seed):
    """a table with exactly dm / dv / dr distinct mem / vcpu / ram values"""
    rng = np.random.default_rng(seed)
    return _table(G, _columns(G, np.arange(1, dm + 1) * 4, rng), _columns(G, np.arange(1, dv + 1) * 3, rng),
                  _columns(G, np.arange(1, dr + 1) * 16, rng), rng)


def full_int32_table(G, seed):
    """columns over the whole int32 range: no rank layout fits, the generic kernel runs"""
    rng = np.random.default_rng(seed)
    col = lambda: rng.integers(-2**31 + 1, 2**31 - 1, G, dtype=np.int64)  # noqa: E731
    return _table(G, col(), col(), col(), rng, price_scale=0.0)


def empty_table():
    return {"mem_gb": np.zeros(0, np.int32), "vcpu": np.zeros(0, np.int32), "ram_gb": np.zeros(0, np.int32),
            "secure_price": np.zeros(0), "community_price": np.zeros(0), "flags": np.zeros(0, np.uint8)}


# the named tables (built on first use)
TABLES = {
    "synth300": lambda: rpk.synth.make_offers(300, correlated=True),
    "synth20k": lambda: rpk.synth.make_offers(20_000, correlated=True),
    "synth100k": lambda: rpk.synth.make_offers(100_000, correlated=True),
    "synth150k": lambda: rpk.synth.make_offers(150_000, correlated=True),
    # 40 mem sizes x 3 x 3: 2 clouds x 41 mem thresholds = 82 row groups, 2 stages each at 250k offers
    "many_queues": lambda: distinct_table(250_000, 40, 3, 3, 40),
    # 2 x 32 x 8 x 8 = 4096 classes exactly (per-mem-threshold view), and 2 x 33 x 8 x 8 = 4224 (staged by price)
    "classes4096": lambda: distinct_table(20_000, 31, 7, 7, 31),
    "classes4224": lambda: distinct_table(20_000, 32, 7, 7, 32),
    "stride64": lambda: distinct_table(30_000, 20, 10, 10, 20),    # 43 mask words: 64-word bitmap rows
    "packed_only": lambda: distinct_table(8_000, 61, 10, 10, 61),  # 84 mask words: no bit-sliced view
    "full_int32": lambda: full_int32_table(3_000, 7),
    "empty": empty_table,
}
_table_cache = {}


def table(name):
    if name not in _table_cache:
        _table_cache[name] = TABLES[name]()
    return _table_cache[name]


def _around(col):
    v = np.unique(col).astype(np.int64)
    return np.clip(np.concatenate([v - 1, v, v + 1, [-1, 0]]), -2**31, 2**31 - 2)


def price_set(offers):
    """max_price values: NaN, a bound above every price, and prices that occur in the table (ties on the winner
    meet the strict price < maxPrice there)"""
    prices = np.concatenate([offers["secure_price"], offers["community_price"]])
    prices = np.unique(prices[prices > 0])
    picks = prices[np.linspace(0, len(prices) - 1, 3).astype(int)] if len(prices) else np.array([0.5])
    return np.concatenate([[np.nan, 1e9], picks])


def pods_for(name, P, seed=0):
    """P pod rows for table `name`: synth pods on the synth tables, else requests just below, at and just above every
    value of the table; max_price from price_set; 3 % of the rows carry an unknown cloud byte"""
    offers = table(name)
    rng = np.random.default_rng(seed * 7919 + P)
    if name.startswith("synth"):
        pods = rpk.synth.make_pods(P, seed=rpk.synth.SEED + seed)
    else:
        pods = {"cloud": rng.integers(0, 2, P).astype(np.uint8)}
        for req, col in (("req_mem_gb", "mem_gb"), ("req_vcpu", "vcpu"), ("req_ram_gb", "ram_gb")):
            vals = _around(offers[col]) if len(offers[col]) else np.array([0, 8, 16])
            pods[req] = rng.choice(vals, P).astype(np.int32)
    pods["max_price"] = rng.choice(price_set(offers), P).astype(np.float64)
    odd = rng.random(P) < 0.03
    pods["cloud"][odd] = rng.choice(np.array([2, 7, 255], np.uint8), int(odd.sum()))
    return pods


def nrows(pods):
    return len(pods["req_mem_gb"])


def head(pods, P):
    """the first P rows (results of a select are per row, so the expected result is the same prefix)"""
    return {k: None if v is None else np.ascontiguousarray(v[:P]) for k, v in pods.items()}


def without_optional(pods):
    """only req_mem_gb: vcpu / ram requests 0, max_price 0.5 and SECURE by default"""
    return {"req_mem_gb": pods["req_mem_gb"], "req_vcpu": None, "req_ram_gb": None, "max_price": None, "cloud": None}


def class_keys(offers, pods):
    P = nrows(pods)
    dist = model.distinct(offers) if len(offers["mem_gb"]) else [np.zeros(0, np.int32)] * 3
    cols = []
    for d, req in zip(dist, ("req_mem_gb", "req_vcpu", "req_ram_gb")):
        v = pods.get(req)
        cols.append(np.searchsorted(d, np.zeros(P, np.int32) if v is None else v, side="left"))
    cloud = pods.get("cloud")
    cols.append(np.zeros(P, np.int64) if cloud is None else np.minimum(cloud, 2).astype(np.int64))
    mp = pods.get("max_price")
    cols.append(np.zeros(P, np.int64) if mp is None else np.ascontiguousarray(mp).view(np.int64))
    return np.stack([c.astype(np.int64) for c in cols], axis=1)


def expected(offers, pods):
    """oracle (best, top5) for every row: row by row when P x G is small, else once per row class"""
    threads = os.cpu_count() or 1
    P, G = nrows(pods), len(offers["mem_gb"])
    if P * max(G, 1) <= ROW_ORACLE_LIMIT:
        return oracle.select(offers, pods, want_top5=True, n_threads=threads)
    _, first, inv = np.unique(class_keys(offers, pods), axis=0, return_index=True, return_inverse=True)
    rep = {k: None if v is None else np.ascontiguousarray(v[first]) for k, v in pods.items()}
    b, t = oracle.select(offers, rep, want_top5=True, n_threads=threads)
    inv = inv.reshape(-1)
    return b[inv], t[inv]


@functools.lru_cache(maxsize=None)
def batch(name, P, seed=0):
    """(pods, oracle best, oracle top5) of P rows for table `name`, computed once per process (callers must not
    modify the arrays; take rows with head())"""
    pods = pods_for(name, P, seed)
    return (pods,) + tuple(expected(table(name), pods))


@functools.lru_cache(maxsize=None)
def batch_without_optional(name, P, seed=0):
    """batch() with only req_mem_gb passed"""
    pods = without_optional(batch(name, P, seed)[0])
    return (pods,) + tuple(expected(table(name), pods))


def check(label, got_best, got_top5, want_best, want_top5):
    """every row of best (and top5 when it was asked for) equals the oracle; sentinel rows are named"""
    bad = np.nonzero(got_best != want_best)[0]
    if len(bad):
        r = bad[:6]
        raise AssertionError(f"{label}: best differs at {len(bad)} of {len(want_best)} rows "
                             f"({int((got_best == SENTINEL).sum())} never written); rows {r.tolist()}: "
                             f"got {got_best[r].tolist()}, oracle {want_best[r].tolist()}")
    if got_top5 is not None:
        bad = np.nonzero((got_top5 != want_top5).any(axis=1))[0]
        if len(bad):
            r = bad[:4]
            raise AssertionError(f"{label}: top5 differs at {len(bad)} rows "
                                 f"({int((got_top5 == SENTINEL).all(axis=1).sum())} never written); rows {r.tolist()}: "
                                 f"got {got_top5[r].tolist()}, oracle {want_top5[r].tolist()}")


@contextmanager
def forced(kind):
    """RPK_FORCE_KERNEL for the uploads inside the block (None: the automatic choice)"""
    old = os.environ.pop("RPK_FORCE_KERNEL", None)
    try:
        if kind is not None:
            os.environ["RPK_FORCE_KERNEL"] = kind
        yield
    finally:
        os.environ.pop("RPK_FORCE_KERNEL", None)
        if old is not None:
            os.environ["RPK_FORCE_KERNEL"] = old


# ---- entry points: outputs start as SENTINEL -------------------------------------------------------------------
def run_host(eng, pods, top5):
    P = nrows(pods)
    best = np.full(P, SENTINEL, np.int32)
    t5 = np.full((P, 5), SENTINEL, np.int32) if top5 else None
    eng.select(pods, want_top5=top5, out_best=best, out_top5=t5)
    return best, t5


def to_device(pods):
    import torch

    return {k: None if v is None else torch.from_numpy(np.ascontiguousarray(v)).cuda() for k, v in pods.items()}


def run_device(eng, pods, top5, stream=None):
    """rpk_select_device on `stream` (a torch.cuda.Stream; None: the current stream), then a device synchronise"""
    import torch

    P = nrows(pods)
    d = to_device(pods)
    d_best = torch.full((P,), SENTINEL, dtype=torch.int32, device="cuda")
    d_t5 = torch.full((P * 5,), SENTINEL, dtype=torch.int32, device="cuda") if top5 else None
    torch.cuda.synchronize()  # inputs are written on the current stream; the call may run on another one
    eng.select_device(d, d_best, d_t5, stream=stream.cuda_stream if stream is not None else None)
    torch.cuda.synchronize()
    return d_best.cpu().numpy(), d_t5.cpu().numpy().reshape(P, 5) if top5 else None


def run_gather(eng, pods, top5, row0):
    """rpk_select_device_gather into three local vectors: each must hold the slice at [row0, row0 + P) and keep
    SENTINEL everywhere else.  Returns (best of the first vector's slice, top5)."""
    import torch

    P = nrows(pods)
    d = to_device(pods)
    vecs = [torch.full((row0 + P + 7,), SENTINEL, dtype=torch.int32, device="cuda") for _ in range(3)]
    d_t5 = torch.full((P * 5,), SENTINEL, dtype=torch.int32, device="cuda") if top5 else None
    torch.cuda.synchronize()
    eng.select_device_gather(d, [v.data_ptr() for v in vecs], row0, d_t5)
    torch.cuda.synchronize()
    host = [v.cpu().numpy() for v in vecs]
    for i, h in enumerate(host):
        outside = np.concatenate([h[:row0], h[row0 + P:]])
        if not (outside == SENTINEL).all():
            raise AssertionError(f"gather: vector {i} was written outside [row0, row0 + P) = [{row0}, {row0 + P})")
        if i and not np.array_equal(h, host[0]):
            raise AssertionError(f"gather: vector {i} differs from vector 0 at "
                                 f"{np.nonzero(h != host[0])[0][:8].tolist()}")
    return host[0][row0:row0 + P].copy(), d_t5.cpu().numpy().reshape(P, 5) if top5 else None


def sm_count():
    import torch

    return torch.cuda.get_device_properties(0).multi_processor_count
