"""A restatement of the select that stays exact and cheap on tables of up to 2^26 offers with few distinct
(mem, vcpu, ram) values, for the scale tests (test_select_scale_gpu.py).  oracle.select costs O(P x G); this costs
O(G log G) once per table and O(log G) per row.

Per cloud, the feasible offers (the cloud's flag set, price > 0, so NaN never) are put in (price, offer index) order,
the tie contract of DESIGN section 2, and numbered by position in that order.  Rows that request at most a
(mem, vcpu, ram) triple meet exactly the offers of the triples that dominate it, and `price < max_price` keeps a
prefix of the positions (NaN keeps none).  So a row's top-5 is the five smallest positions over its dominating triples
that fall inside its prefix, and those are among the first five positions of each such triple.  `Index` keeps, for
every request threshold (searchsorted on the table's distinct values), the five smallest positions over the triples
that dominate it; a row then takes the ones below its price cut.  NULL columns and unknown cloud bytes are read as
oracle.get_gpu_types reads them: vcpu / ram 0, max_price 0.5, SECURE; a cloud byte other than 0 / 1 meets no offer."""
import numpy as np

DEFAULT_MAX_PRICE = 0.5
MAX_TRIPLES = 1 << 22  # the dense threshold grid: tables with this many distinct triples are not what it is for
_NONE = np.iinfo(np.int64).max


def _distinct(v):
    """(the distinct values of v, the rank of each value among them), v without NaN, exact; O(n log U) for U distinct
    values, which beats sorting n values when U is small (they are collected from a sample, then from the misses)"""
    u = np.unique(v[:: max(len(v) // 65536, 1)])
    while True:
        r = np.searchsorted(u, v)
        miss = (r == len(u)) | (u[np.minimum(r, len(u) - 1)] != v) if len(u) else np.ones(len(v), bool)
        if not miss.any():
            return u, r
        u = np.union1d(u, v[miss])


def _stable_argsort(keys):
    """stable argsort of non-negative integer keys (a radix sort when they fit 16 bits)"""
    if len(keys) and keys.max() < 2**15:
        keys = keys.astype(np.int16)
    return np.argsort(keys, kind="stable")


def _column(offers, name, G):
    v = offers.get(name)
    return np.zeros(G, np.int32) if v is None else np.asarray(v)


class Index:
    def __init__(self, offers):
        G = len(offers["mem_gb"])
        cols = [_column(offers, k, G) for k in ("mem_gb", "vcpu", "ram_gb")]
        dist = [_distinct(c) for c in cols]
        self.dist = [d for d, _ in dist]
        D = [len(d) for d in self.dist]
        assert np.prod([d + 1 for d in D], dtype=np.int64) <= MAX_TRIPLES, f"{D} distinct values: too many triples"
        triple = np.zeros(G, np.int64)
        for d, rank in dist:
            triple = triple * len(d) + rank
        self.order, self.price, self.top = [], [], []
        for cloud, key in ((0, "secure_price"), (1, "community_price")):
            price = np.asarray(offers[key], np.float64)
            ok = np.nonzero(((offers["flags"] & (1 << cloud)) != 0) & (price > 0))[0]
            order = ok[_stable_argsort(_distinct(price[ok])[1])]  # ascending index within a price: (price, index)
            self.order.append(order)
            self.price.append(price[order])
            self.top.append(self._first5(triple[order], D))

    @staticmethod
    def _first5(tri, D):
        """[D0 + 1, D1 + 1, D2 + 1, 5]: at (i, j, k), the five smallest positions over triples >= (i, j, k)"""
        n = len(tri)
        T = int(np.prod(D, dtype=np.int64))
        top = np.full((T, 5), _NONE, np.int64)
        if n:
            by = _stable_argsort(tri)  # positions ascending within each triple
            t = tri[by]
            start = np.r_[0, np.nonzero(t[1:] != t[:-1])[0] + 1]
            rank = np.arange(n) - np.repeat(start, np.diff(np.r_[start, n]))
            keep = rank < 5
            top[t[keep], rank[keep]] = by[keep]
        grid = np.full((D[0] + 1, D[1] + 1, D[2] + 1, 5), _NONE, np.int64)
        grid[: D[0], : D[1], : D[2]] = top.reshape(D[0], D[1], D[2], 5)
        for axis in range(3):  # suffix merges: the triples each step adds are disjoint from those already in
            g = np.moveaxis(grid, axis, 0)
            for i in range(g.shape[0] - 2, -1, -1):
                g[i] = np.sort(np.concatenate([g[i], g[i + 1]], axis=-1), axis=-1)[..., :5]
        return grid

    def thresholds(self, pods):
        """per row the searchsorted threshold of each request on the table's distinct values"""
        P = len(pods["req_mem_gb"])
        out = []
        for d, k in zip(self.dist, ("req_mem_gb", "req_vcpu", "req_ram_gb")):
            v = pods.get(k)
            out.append(np.searchsorted(d, np.zeros(P, np.int32) if v is None else v, side="left"))
        return out

    def select(self, pods, want_top5=True):
        """(best[P], top5[P, 5] | None), as oracle.select returns them"""
        P = len(pods["req_mem_gb"])
        cloud = pods.get("cloud")
        cloud = np.zeros(P, np.int64) if cloud is None else np.asarray(cloud).astype(np.int64)
        mp = pods.get("max_price")
        mp = np.full(P, DEFAULT_MAX_PRICE) if mp is None else np.asarray(mp, np.float64)
        ti, tj, tk = self.thresholds(pods)
        top5 = np.full((P, 5), -1, np.int32)
        for c in (0, 1):
            rows = np.nonzero(cloud == c)[0]
            if not len(rows) or not len(self.order[c]):
                continue
            pos = self.top[c][ti[rows], tj[rows], tk[rows]]
            cut = np.searchsorted(self.price[c], mp[rows], side="left")  # prices < max_price
            cut[np.isnan(mp[rows])] = 0
            hit = pos < cut[:, None]
            top5[rows] = np.where(hit, self.order[c][np.where(hit, pos, 0)], -1)
        return top5[:, 0].copy(), top5 if want_top5 else None


def select(offers, pods, want_top5=True):
    return Index(offers).select(pods, want_top5)


# ---- the scale tables and their pod batches --------------------------------------------------------------------------
def scale_table(G, dm, dv, dr, seed):
    """G offers with exactly dm / dv / dr distinct mem / vcpu / ram values (the first max(dm, dv, dr) offers take each
    once).  Prices in cents grow with the offer's value ranks, so the cheapest offer a request meets lies deeper in
    price order the more it asks; noise of 40 cents makes long runs of equal prices, and 3 % of the offers copy the
    columns of the offer before them (tie pairs: equal price and triple, the lower index wins).  2 % cost 0, and 0.1 %
    each are NaN or +inf (never feasible)."""
    rng = np.random.default_rng(seed)
    k = [rng.integers(0, d, G, dtype=np.int32) for d in (dm, dv, dr)]
    for c, d in zip(k, (dm, dv, dr)):
        c[:d] = np.arange(d)
    cents = 5 + (k[0] + k[1] + k[2]).astype(np.int64) * 7 + rng.integers(0, 40, G)
    cents[rng.random(G) < 0.02] = 0
    flags = rng.integers(0, 4, G).astype(np.uint8)
    cols = [(k[0] + 1) * 4, (k[1] + 1) * 3, (k[2] + 1) * 16]
    tie = np.nonzero(rng.random(G) < 0.03)[0]
    tie = tie[tie >= max(dm, dv, dr) + 1]
    for a in cols + [cents, flags]:
        a[tie] = a[tie - 1]
    secure = cents.astype(np.float64) / 100.0
    secure[rng.random(G) < 0.001] = np.nan
    secure[rng.random(G) < 0.001] = np.inf
    return {"mem_gb": cols[0].astype(np.int32), "vcpu": cols[1].astype(np.int32), "ram_gb": cols[2].astype(np.int32),
            "secure_price": secure, "community_price": ((cents * 6) // 10).astype(np.float64) / 100.0, "flags": flags}


def _around(d):
    v = d.astype(np.int64)
    return np.unique(np.clip(np.concatenate([v - 1, v, v + 1, [0, -2**31, 2**31 - 1]]), -2**31, 2**31 - 1))


def price_bounds(offers, rng, n=6):
    """max_price values: NaN, +-inf, 0, a bound above every price and n prices of the table (ties at the bound)"""
    p = np.concatenate([offers["secure_price"][:200_000], offers["community_price"][:200_000]])
    p = np.unique(p[np.isfinite(p) & (p > 0)])
    return np.concatenate([[np.nan, np.inf, -np.inf, 0.0, 1e9], rng.choice(p, n) if len(p) else []])


def scale_pods(offers, P, seed):
    """P rows that cover every class: the first rows take each (mem, vcpu, ram threshold, cloud) once, at one value
    of the threshold and with an unbounded price, the others draw each request from just below, at and just above
    every distinct value (or 0, 70 % of the vcpu / ram requests, as in the synth pods), max_price from price_bounds or
    the default 0.5, and 3 % an unknown cloud byte (2, 7, 255)"""
    rng = np.random.default_rng(seed)
    G = len(offers["mem_gb"])
    dist = [np.unique(_column(offers, k, G)) for k in ("mem_gb", "vcpu", "ram_gb")]
    pods = {}
    for d, k in zip(dist, ("req_mem_gb", "req_vcpu", "req_ram_gb")):
        pods[k] = rng.choice(_around(d), P).astype(np.int32)
    for k in ("req_vcpu", "req_ram_gb"):
        pods[k][rng.random(P) < 0.7] = 0
    pods["max_price"] = rng.choice(price_bounds(offers, rng), P)
    pods["max_price"][rng.random(P) < 0.3] = DEFAULT_MAX_PRICE
    pods["cloud"] = rng.integers(0, 2, P).astype(np.uint8)
    odd = rng.random(P) < 0.03
    pods["cloud"][odd] = rng.choice(np.array([2, 7, 255], np.uint8), int(odd.sum()))
    reps = [np.r_[d, d[-1] + 1].astype(np.int32) for d in dist]  # one request per threshold, the last above them all
    grid = np.stack(np.meshgrid(*reps, np.arange(2), indexing="ij"), -1).reshape(-1, 4)
    n = min(len(grid), P)
    for i, k in enumerate(("req_mem_gb", "req_vcpu", "req_ram_gb")):
        pods[k][:n] = grid[:n, i]
    pods["cloud"][:n] = grid[:n, 3]
    pods["max_price"][:n] = np.inf
    return pods
