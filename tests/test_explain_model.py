"""CPU tests of the explain references (explain_model.py): the C loop and the numpy restatement agree on the known
answers, on random tables and at the edges of every column, and both keep the invariants rpk.h states against
oracle.select."""
import numpy as np
import pytest

import explain_model as em
import oracle
import rpk

INT32_MIN, INT32_MAX = -2**31, 2**31 - 1


def check_invariants(offers, pods, ex):
    G = len(offers["mem_gb"])
    best, top5 = oracle.select(offers, pods, want_top5=True)
    # an offer failing at least one requirement counts once under n_fail[r] for each r it fails: bound it by its parts
    failing = G - ex["n_unoffered"].astype(np.int64) - ex["n_feasible"]
    assert (failing >= 0).all()
    assert (failing <= ex["n_fail"].sum(axis=1)).all()
    assert (failing >= ex["n_fail"].max(axis=1, initial=0)).all()
    assert (failing >= ex["n_only"].sum(axis=1)).all()
    assert np.array_equal(ex["n_feasible"] > 0, best != -1)
    assert np.array_equal(np.minimum(ex["n_feasible"], 5), (top5 != -1).sum(axis=1))
    assert ((ex["nearest"] >= 0) == (ex["n_only"] > 0)).all()
    assert (ex["n_only"] <= ex["n_fail"]).all()


def exact_failing(offers, pods):
    """#{offered offers failing at least one requirement} per row, counted directly from rpk_select's predicate"""
    G, P = len(offers["mem_gb"]), len(pods["req_mem_gb"])
    opt = lambda d, k, n, v: d[k] if d.get(k) is not None else np.full(n, v)  # noqa: E731
    out = np.zeros(P, np.int64)
    for c, (bit, col) in enumerate(((1, "secure_price"), (2, "community_price"))):
        price = offers[col]
        offered = ((offers["flags"] & bit) != 0) & (price > 0)
        r = opt(pods, "cloud", P, 0) == c
        ok = ((price[None, :] < opt(pods, "max_price", P, 0.5)[r, None]) & (offers["mem_gb"][None, :] >= pods["req_mem_gb"][r, None])
              & (opt(offers, "vcpu", G, 0)[None, :] >= opt(pods, "req_vcpu", P, 0)[r, None])
              & (opt(offers, "ram_gb", G, 0)[None, :] >= opt(pods, "req_ram_gb", P, 0)[r, None]))
        out[r] = (offered[None, :] & ~ok).sum(axis=1)
    return out


def both(offers, pods, n_threads=1):
    got = em.explain(offers, pods, n_threads=n_threads)
    em.assert_same(got, em.explain_np(offers, pods), "C reference vs numpy")
    return got


def test_known_answers():
    offers, pods = em.kat_offers(), em.kat_pods()
    got = both(offers, pods)
    em.assert_same(got, em.kat_expected(), "KAT")
    check_invariants(offers, pods, got)


def test_known_answers_first_row_by_hand():
    """offer 6 (A100, $1.64) alone fails only the price; offer 0 (A4000, $0.32) is the cheapest failing only memory"""
    got = em.explain(em.kat_offers(), em.kat_pods())
    assert em.KAT_IDS[got["nearest"][0, 0]] == "A100" and em.KAT_IDS[got["nearest"][0, 1]] == "A4000"


@pytest.mark.parametrize("tie_free", [False, True])
@pytest.mark.parametrize("G,P", [(1, 300), (37, 500), (1000, 700), (3000, 200)])
def test_random_tables(tie_free, G, P):
    offers = rpk.synth.make_offers(G, tie_free=tie_free)
    pods = rpk.synth.make_pods(P, seed=G + P)
    got = both(offers, pods)
    check_invariants(offers, pods, got)
    assert np.array_equal(G - got["n_unoffered"].astype(np.int64) - got["n_feasible"], exact_failing(offers, pods))


def test_threads_split_rows_identically():
    offers = rpk.synth.make_offers(2000, correlated=True)
    pods = rpk.synth.make_pods(3001)
    em.assert_same(em.explain(offers, pods, n_threads=7), em.explain(offers, pods, n_threads=1), "7 threads vs 1")


def edge_offers():
    """prices 0, -0.0, NaN, negative, +inf and ties; columns at INT32_MIN and INT32_MAX - 1 (the upload's limit)"""
    sp = np.array([0.0, -0.0, np.nan, -1.0, 0.25, 0.25, 0.5, np.inf, 1e-300, 0.25, 3.0, 0.5], np.float64)
    cp = np.array([0.25, 0.0, 0.1, np.nan, -0.0, 0.25, 0.25, 0.5, 0.1, 1e300, 0.25, 0.5], np.float64)
    G = len(sp)
    mem = np.array([INT32_MIN, -1, 0, 1, 16, 16, 80, INT32_MAX - 1, 24, 24, 0, INT32_MAX - 1], np.int32)
    vcpu = np.array([0, INT32_MAX - 1, INT32_MIN, 4, 8, 8, 16, 0, -5, 32, INT32_MIN, 64], np.int32)
    ram = np.array([16, 0, INT32_MAX - 1, INT32_MIN, 32, 64, 64, 128, 0, -1, 7, INT32_MAX - 1], np.int32)
    flags = np.array([3, 3, 3, 3, 1, 3, 2, 3, 3, 3, 0, 3], np.uint8)
    return {"mem_gb": mem, "vcpu": vcpu, "ram_gb": ram, "secure_price": sp, "community_price": cp, "flags": flags}, G


def edge_pods(offers, P=4000, seed=5):
    rng = np.random.default_rng(seed)
    vals = np.array([INT32_MIN, INT32_MIN + 1, -1, 0, 1, 8, 16, 24, 80, INT32_MAX - 1, INT32_MAX], np.int64)
    prices = np.concatenate([[np.nan, -np.nan, 0.0, -0.0, -1.0, np.inf, -np.inf, 1e-300],
                             offers["secure_price"], offers["community_price"]])
    return {"req_mem_gb": rng.choice(vals, P).astype(np.int32), "req_vcpu": rng.choice(vals, P).astype(np.int32),
            "req_ram_gb": rng.choice(vals, P).astype(np.int32), "max_price": rng.choice(prices, P).astype(np.float64),
            "cloud": rng.choice(np.array([0, 1, 2, 255], np.uint8), P)}


def test_edge_values():
    offers, _ = edge_offers()
    pods = edge_pods(offers)
    got = both(offers, pods)
    check_invariants(offers, pods, got)
    assert np.array_equal(len(offers["mem_gb"]) - got["n_unoffered"].astype(np.int64) - got["n_feasible"], exact_failing(offers, pods))
    nan = np.isnan(pods["max_price"]) & (pods["cloud"] < 2)
    assert (got["n_fail"][nan, 0] == len(offers["mem_gb"]) - got["n_unoffered"][nan]).all(), "a NaN bound fails every offered offer"
    other = pods["cloud"] >= 2
    assert (got["n_unoffered"][other] == len(offers["mem_gb"])).all() and (got["nearest"][other] == -1).all()


def test_bound_equal_to_a_price_fails_it():
    offers, _ = edge_offers()
    pods = {"req_mem_gb": np.array([INT32_MIN], np.int32), "req_vcpu": np.array([INT32_MIN], np.int32),
            "req_ram_gb": np.array([INT32_MIN], np.int32), "max_price": np.array([0.25]), "cloud": np.array([0], np.uint8)}
    got = both(offers, pods)
    # SECURE offered: 4, 5, 7, 8, 9, 11 (flag and price > 0); below 0.25 only offer 8 (1e-300)
    assert got["n_unoffered"][0] == 6 and got["n_feasible"][0] == 1 and got["n_fail"][0, 0] == 5
    assert got["nearest"][0, 0] == 4, "ties at 0.25 go to the lowest offer index"


def test_without_optional_columns():
    offers = rpk.synth.make_offers(500)
    pods = rpk.synth.make_pods(400)
    pods = {"req_mem_gb": pods["req_mem_gb"], "req_vcpu": None, "req_ram_gb": None, "max_price": None, "cloud": None}
    got = both(offers, pods)
    check_invariants(offers, pods, got)
    assert (got["n_fail"][:, 2:] == 0).all(), "vcpu and ram requests default to 0, which every offer meets"


@pytest.mark.parametrize("G", [0, 1])
def test_tiny_tables(G):
    offers, _ = edge_offers()
    offers = {k: v[5:5 + G] if v is not None else None for k, v in offers.items()}
    pods = edge_pods(offers, P=300, seed=G)
    got = both(offers, pods)
    check_invariants(offers, pods, got)
    if G == 0:
        assert (got["n_unoffered"] == 0).all() and (got["nearest"] == -1).all() and (got["n_feasible"] == 0).all()
