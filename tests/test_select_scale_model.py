"""The scale tests' reference (select_scale_model.py) against oracle.select, row by row, on the CPU: every scale-table
shape the GPU file uploads, at G <= 20 000, and the synth and plan-test tables, with NaN / +-inf / 0 / tied
max_price, cloud bytes 2, 7 and 255, and NULL optional columns."""
import numpy as np
import pytest

import oracle
import rpk
import select_plan_cases as sc
import select_scale_model as sm

TABLES = {
    "reload-20x1x39": lambda: sm.scale_table(20_000, 20, 1, 39, 1),
    "limit-3x2x2": lambda: sm.scale_table(20_000, 3, 2, 2, 2),
    "tiny-3x2x2": lambda: sm.scale_table(64, 3, 2, 2, 3),
    "one-value": lambda: sm.scale_table(5_000, 1, 1, 1, 4),
    "synth20k": lambda: rpk.synth.make_offers(20_000, correlated=True),
    "synth-no-ext": lambda: rpk.synth.make_offers(10_000, with_ext=False),
    "synth-tie-free": lambda: rpk.synth.make_offers(10_000, tie_free=True),
    "stride64": lambda: sc.distinct_table(20_000, 20, 10, 10, 20),
    "empty": sc.empty_table,
}


def compare(offers, pods, what):
    want_b, want_t = oracle.select(offers, pods, want_top5=True, n_threads=4)
    got_b, got_t = sm.select(offers, pods)
    bad = np.nonzero((got_t != want_t).any(axis=1) | (got_b != want_b))[0]
    assert not len(bad), (f"{what}: {len(bad)} of {len(want_b)} rows differ; rows {bad[:4].tolist()}: "
                          f"model {got_t[bad[:4]].tolist()}, oracle {want_t[bad[:4]].tolist()}")


@pytest.mark.parametrize("name", list(TABLES))
def test_model_equals_oracle(name):
    offers = TABLES[name]()
    P = 4000
    pods = sm.scale_pods(offers, P, seed=len(name)) if len(offers["mem_gb"]) else sc.pods_for("empty", P)
    compare(offers, pods, name)
    compare(offers, sc.without_optional(pods), f"{name} (NULL columns)")
    if name.startswith("synth"):
        compare(offers, rpk.synth.make_pods(P), f"{name} (synth pods)")


def test_edges_are_present():
    """the scale pods and tables carry the edges the model must read like the oracle"""
    offers = TABLES["reload-20x1x39"]()
    pods = sm.scale_pods(offers, 4000, seed=1)
    mp = pods["max_price"]
    assert np.isnan(mp).any() and (mp == np.inf).any() and (mp == -np.inf).any() and (mp == 0).any()
    assert {2, 255} <= set(pods["cloud"].tolist())
    sp = offers["secure_price"]
    assert (sp == 0).any() and np.isnan(sp).any() and (sp == np.inf).any()
    # tie pairs: equal price and triple on neighbouring offers
    same = np.ones(len(sp) - 1, bool)
    for k in ("mem_gb", "vcpu", "ram_gb", "secure_price"):
        same &= offers[k][1:] == offers[k][:-1]
    assert same.sum() > 100
    # every (threshold triple, cloud) class appears
    ti, tj, tk = sm.Index(offers).thresholds(pods)
    assert len(np.unique(np.stack([ti, tj, tk, pods["cloud"]])[:, pods["cloud"] <= 1], axis=1).T) == 21 * 2 * 40 * 2


def test_max_price_is_a_strict_bound_on_ties():
    """a max_price equal to a tied price excludes both offers of the pair; one ulp above includes both, lower index
    first"""
    offers = {"mem_gb": np.array([8, 8, 8], np.int32), "vcpu": None, "ram_gb": None,
              "secure_price": np.array([0.5, 0.25, 0.25]), "community_price": np.array([0.1, 0.1, 0.0]),
              "flags": np.array([3, 3, 3], np.uint8)}
    pods = {"req_mem_gb": np.array([8, 8, 8, 9, 8], np.int32), "req_vcpu": None, "req_ram_gb": None,
            "max_price": np.array([0.25, np.nextafter(0.25, 1), np.nan, 1.0, 0.2]),
            "cloud": np.array([0, 0, 0, 0, 1], np.uint8)}
    b, t = sm.select(offers, pods)
    assert b.tolist() == [-1, 1, -1, -1, 0]
    assert t[1].tolist() == [1, 2, -1, -1, -1] and t[4].tolist() == [0, 1, -1, -1, -1]
    compare(offers, pods, "ties")
