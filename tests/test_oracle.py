"""CPU tests: the oracle against the reference-derived golden vectors and against the independent numpy
restatement.  No GPU, no product code on the compute path."""
import json
import os

import numpy as np
import pytest

import np_restatement as npr
import oracle
import rpk
import status_cases as sc

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
CLOUD = {"SECURE": oracle.CLOUD_SECURE, "COMMUNITY": oracle.CLOUD_COMMUNITY}


def kat_offers():
    kat = json.load(open(os.path.join(GOLD, "select_kat.json")))
    o = kat["offers"]
    offers = {
        "mem_gb": np.array([x["memGb"] for x in o], np.int32),
        "secure_price": np.array([x["securePrice"] for x in o], np.float64),
        "community_price": np.array([x["communityPrice"] for x in o], np.float64),
        "flags": np.array([(1 if x["secureCloud"] else 0) | (2 if x["communityCloud"] else 0) for x in o], np.uint8),
        "vcpu": None,
        "ram_gb": None,
    }
    return kat, offers


def test_column_producers_golden():
    g = json.load(open(os.path.join(GOLD, "column_producers.json")))
    for c in g["annotation_fallback"]:
        assert oracle.annotation_with_fallback(c["pod"], c["job"], c["default"]) == c["want"], c
    for c in g["extract_gpu_memory"]:
        assert oracle.extract_gpu_memory(c["in"]) == c["want"], c
    names = {0: "SECURE", 1: "COMMUNITY"}
    for c in g["validate_cloud_type"]:
        assert names[oracle.validate_cloud_type(c["in"])] == c["want"], c


def test_reference_test_scenarios():
    """The three PrepareRunPodParameters scenarios the reference asserts (annotations_test.go:106-143,
    216-238): job annotations, pod-overrides-job, job fallback."""
    job = {"runpod.io/required-gpu-memory": "8", "runpod.io/cloud-type": "SECURE"}
    pod = {}
    mem = oracle.extract_gpu_memory(oracle.annotation_with_fallback(pod.get("runpod.io/required-gpu-memory"), job.get("runpod.io/required-gpu-memory"), ""))
    assert mem == 8
    assert oracle.validate_cloud_type(oracle.annotation_with_fallback(pod.get("runpod.io/cloud-type"), job.get("runpod.io/cloud-type"), "")) == 0
    pod = {"runpod.io/required-gpu-memory": "16"}
    mem = oracle.extract_gpu_memory(oracle.annotation_with_fallback(pod.get("runpod.io/required-gpu-memory"), job.get("runpod.io/required-gpu-memory"), ""))
    assert mem == 16
    job2 = {"runpod.io/required-gpu-memory": "24", "runpod.io/cloud-type": "COMMUNITY"}
    pod2 = {"runpod.io/cloud-type": "SECURE"}
    assert oracle.extract_gpu_memory(oracle.annotation_with_fallback(pod2.get("runpod.io/required-gpu-memory"), job2.get("runpod.io/required-gpu-memory"), "")) == 24
    assert oracle.validate_cloud_type(oracle.annotation_with_fallback(pod2.get("runpod.io/cloud-type"), job2.get("runpod.io/cloud-type"), "")) == 0


def test_clamp_i32():
    assert oracle.clamp_i32(2**40) == 2**31 - 1
    assert oracle.clamp_i32(-(2**40)) == -(2**31)
    assert oracle.clamp_i32(24) == 24


def test_select_kat_oracle_and_numpy():
    kat, offers = kat_offers()
    for c in kat["cases"]:
        cloud = CLOUD.get(c["cloud"], oracle.CLOUD_OTHER)
        assert oracle.get_gpu_types(offers, c["minMem"], c["maxPrice"], cloud) == c["top5"], c
        assert npr.get_gpu_types(offers, c["minMem"], c["maxPrice"], c["cloud"]) == c["top5"], c


@pytest.mark.parametrize("tie_free,ref_exact,with_ext", [(False, False, True), (True, False, True), (False, True, False), (True, True, True)])
def test_oracle_matches_numpy_restatement(tie_free, ref_exact, with_ext):
    offers = rpk.synth.make_offers(700, tie_free=tie_free, with_ext=with_ext, correlated=not tie_free)
    pods = rpk.synth.make_pods(300, reference_exact=ref_exact)
    b0, t0 = oracle.select(offers, pods)
    b1, t1 = npr.select(offers, pods)
    assert np.array_equal(b0, b1) and np.array_equal(t0, t1)
    assert len(np.unique(b0)) >= 3


def test_oracle_c1_config():
    """BASELINE config 1: 100 pending pods x 50 GPU types, the reference's own scale."""
    offers = rpk.synth.make_offers(50, with_ext=False)
    pods = rpk.synth.make_pods(100, reference_exact=True)
    b0, t0 = oracle.select(offers, pods)
    b1, t1 = npr.select(offers, pods)
    assert np.array_equal(b0, b1) and np.array_equal(t0, t1)
    assert np.array_equal(b0, t0[:, 0])


def test_oracle_threads_agree():
    offers = rpk.synth.make_offers(500)
    pods = rpk.synth.make_pods(257)
    b1, t1 = oracle.select(offers, pods, n_threads=1)
    b4, t4 = oracle.select(offers, pods, n_threads=4)
    assert np.array_equal(b1, b4) and np.array_equal(t1, t4)


def test_oracle_edge_cases():
    offers = rpk.synth.make_offers(64)
    # NaN / inf prices, negative and extreme requests, unknown cloud byte
    offers["secure_price"][:4] = [np.nan, np.inf, -1.0, 5e-324]
    offers["flags"][:4] = 3
    pods = {
        "req_mem_gb": np.array([-5, 0, 2**31 - 1, -(2**31), 16, 16, 16], np.int32),
        "req_vcpu": np.zeros(7, np.int32), "req_ram_gb": np.zeros(7, np.int32),
        "max_price": np.array([0.5, np.inf, 0.5, 0.5, np.nan, -1.0, 1e308], np.float64),
        "cloud": np.array([0, 0, 0, 0, 0, 1, 7], np.uint8),
    }
    b0, t0 = oracle.select(offers, pods)
    b1, t1 = npr.select(offers, pods)
    assert np.array_equal(b0, b1) and np.array_equal(t0, t1)
    assert b0[2] == -1 and b0[4] == -1 and b0[5] == -1 and b0[6] == -1
    assert b0[1] == 3  # the denormal price 5e-324 is > 0 and the cheapest; +inf is never < +inf
    # empty table / no pods
    empty = {k: (v[:0] if v is not None else None) for k, v in offers.items()}
    b, t = oracle.select(empty, pods)
    assert (b == -1).all() and (t == -1).all()


def test_xxh64_golden():
    g = json.load(open(os.path.join(GOLD, "xxh64_kat.json")))
    for v in g["vectors"]:
        assert format(oracle.xxh64(bytes.fromhex(v["hex"]), v["seed"]), "016x") == v["xxh64"], v
    try:
        import xxhash
    except ImportError:
        return
    rng = np.random.default_rng(7)
    for n in (0, 1, 5, 31, 32, 33, 63, 64, 200, 1000):
        d = rng.integers(0, 256, n, dtype=np.uint8).tobytes()
        assert oracle.xxh64(d) == xxhash.xxh64(d).intdigest()


def test_status_states_collision_free():
    """The known state space (6 enum strings + unknowns) x ports must hash to distinct values, so the
    hash changed-set equals the reference's string/bool changed-set (SURVEY.md 8d)."""
    recs = [rpk.synth.encode_record(s, p) for s in rpk.synth.STATUS_SET + rpk.synth.UNKNOWN_STATUS for p in (False, True)]
    h = oracle.record_hashes(np.stack(recs))
    assert len(set(h.tolist())) == len(recs) and 0 not in set(h.tolist())


def test_status_diff_oracle_vs_numpy():
    N = 3000
    tab = oracle.StatusTable(N)
    prev = [None] * N
    for sweep, frac in enumerate([0.0, 0.01, 0.10, 1.0, 0.0]):
        recs = rpk.synth.make_status_records(N, sweep=sweep, mutate_frac=frac)
        a = tab.diff(recs)
        b = npr.status_changed_set(recs, prev)
        assert np.array_equal(a, b), sweep
        if sweep == 0:
            assert len(a) == N  # never seen -> all changed
    # hash equality <=> decoded equality on these tables
    r0 = rpk.synth.make_status_records(N, 0)
    r1 = rpk.synth.make_status_records(N, 2, 0.5)
    same_hash = oracle.record_hashes(r0) == oracle.record_hashes(r1)
    m0, m1 = r0.copy(), r1.copy()
    m0[:, 0] &= 0x7F  # the message flag moves between sweeps; it is neither compared nor hashed
    m1[:, 0] &= 0x7F
    same_rec = (m0 == m1).all(axis=1)
    assert np.array_equal(same_hash, same_rec)
    assert (r0[:, 0] != r1[:, 0]).sum() > (~same_rec).sum()  # ... and it really does move on unchanged rows


def test_record_hash_matches_python_xxhash():
    recs = rpk.synth.make_status_records(500, 1, 0.3)
    h = oracle.record_hashes(recs)
    try:
        import xxhash
    except ImportError:
        pytest.skip("python-xxhash not installed")
    for i in range(0, 500, 37):
        ln = int(recs[i, 0]) & 0x7F
        d = bytearray(recs[i, : 8 * ((1 + ln + 7) // 8)].tobytes())  # zero-padded prefix in whole 8-byte lanes
        d[0] &= 0x7F
        assert int(h[i]) == xxhash.xxh64(bytes(d)).intdigest()


def test_slot_prefix_golden_vectors():
    """oracle.record_hashes against the committed slot-prefix vectors (python-xxhash): every len 0..127, strides 128/256."""
    g = json.load(open(os.path.join(GOLD, "xxh64_kat.json")))
    for stride in (128, 256):
        recs = np.zeros((len(g["slot_vectors"]), stride), np.uint8)
        for i, v in enumerate(g["slot_vectors"]):
            d = np.frombuffer(bytes.fromhex(v["hex"]), np.uint8)
            recs[i, : len(d)] = d
        flagged = recs.copy()
        flagged[:, 0] |= 0x80
        for tab in (recs, flagged):
            h = oracle.record_hashes(tab)
            for i, v in enumerate(g["slot_vectors"]):
                assert format(int(h[i]), "016x") == v["xxh64"], (stride, v["len"])


def test_translate_run_pod_status_table():
    """kubelet.go:1866-1985 by hand: (status, message, ports) -> phase / ready / started / state / exit / reason / message."""
    PH = {"Unknown": 0, "Pending": 1, "Running": 2, "Succeeded": 3, "Failed": 4}
    ST = {"Waiting": 0, "Running": 1, "Terminated": 2}
    RS = {"": 0, "ContainerCreating": 1, "Completed": 2, "Error": 3, "Terminated": 4, "PodDeleted": 5, "ContainerStatusUnknown": 6}
    rows = [  # status, message, ports -> phase, ready, started, state, exit, reason, message kind
        ("RUNNING", "", True, "Running", 1, 1, "Running", 0, "", 0),                           # :1868-1879
        ("RUNNING", "", False, "Pending", 0, 0, "Waiting", 0, "ContainerCreating", 1),         # :1880-1891
        ("STARTING", "pulling image", True, "Pending", 0, 0, "Waiting", 0, "ContainerCreating", 0),  # :1893-1903
        ("EXITED", "done", True, "Succeeded", 0, 0, "Terminated", 0, "Completed", 0),          # :1914-1916
        ("EXITED", "Container FAILED to start", False, "Failed", 0, 0, "Terminated", 1, "Error", 0),  # :1907-1913 (case fold)
        ("EXITED", "some ERROR", True, "Failed", 0, 0, "Terminated", 1, "Error", 0),
        ("TERMINATING", "", False, "Running", 1, 1, "Running", 0, "", 0),                      # :1931-1941
        ("TERMINATED", "", True, "Succeeded", 0, 0, "Terminated", 0, "Terminated", 0),         # :1943-1955
        ("NOT_FOUND", "", True, "Failed", 0, 0, "Terminated", 1, "PodDeleted", 2),             # :1957-1969
        ("PAUSED", "", True, "Unknown", 0, 0, "Waiting", 0, "ContainerStatusUnknown", 3),      # :1971-1979
        ("running", "", True, "Unknown", 0, 0, "Waiting", 0, "ContainerStatusUnknown", 3),     # the switch is case sensitive
        ("", "", True, "Unknown", 0, 0, "Waiting", 0, "ContainerStatusUnknown", 3),
    ]
    for st, msg, ports, ph, ready, started, state, ex, reason, mk in rows:
        want = PH[ph] | ready << 3 | started << 4 | ST[state] << 5 | ex << 7 | RS[reason] << 8 | mk << 11
        assert oracle.translate(st, msg, ports) == want, (st, msg, ports)
    # record form: flag bit = "message contains error/fail"
    for s in rpk.synth.STATUS_SET + rpk.synth.UNKNOWN_STATUS:
        for p in (False, True):
            for f in (False, True):
                rec = rpk.synth.encode_record(s, p, 16, f)[None, :]
                assert int(oracle.record_codes(rec)[0]) == oracle.translate(s.decode(), "it FAILed" if f else "", p)


# ---- the sweep-state model (oracle.StatusTable) across calls and strides ----------------------------------------

def _decoded(records):
    return [npr.decode_record(r) for r in records]


def test_status_table_seed_then_diff_reports_nothing():
    lt = sc.LogicalTable(700, np.random.default_rng(1))
    for stride in (16, 48, 256):
        lt.step(stride, 0.5)
        recs = lt.records(stride)
        tab = oracle.StatusTable(700, stride)
        tab.seed(recs)
        assert len(tab.diff(recs)) == 0
        lt.step(stride, 0.1)
        nxt = lt.records(stride)
        prev = _decoded(recs)
        assert np.array_equal(tab.diff(nxt), npr.status_changed_set(nxt, prev))


def test_status_table_seed_slots_touches_only_named_slots():
    N = 500
    lt = sc.LogicalTable(N, np.random.default_rng(2))
    base = lt.records(32)
    tab = oracle.StatusTable(N, 32)
    tab.diff(base)
    lt.step(32, 0.6)
    nxt = lt.records(32)
    moved = npr.status_changed_set(nxt, _decoded(base))
    assert len(moved) > 100
    quiet = moved[::4]
    tab.seed_slots(quiet, nxt[quiet])
    assert np.array_equal(tab.diff(nxt), np.setdiff1d(moved, quiet).astype(np.uint32))
    # a seeded slot takes the seeded record as its state, whatever it held before
    tab.seed_slots(np.array([3]), base[3:4])
    assert tab.diff(nxt).tolist() == ([3] if npr.decode_record(base[3]) != npr.decode_record(nxt[3]) else [])
    tab.seed_slots(np.array([], np.int64), nxt[:0])
    assert len(tab.diff(nxt)) == 0


def test_status_table_reset_makes_every_slot_report():
    recs = rpk.synth.make_status_records(300, 0)
    tab = oracle.StatusTable(300)
    tab.seed(recs)
    tab.reset(300)
    assert np.array_equal(tab.diff(recs), np.arange(300, dtype=np.uint32))
    tab.reset(120)
    assert tab.N == 120 and (tab.prev_hashes() == 0).all()
    assert np.array_equal(tab.diff(np.ascontiguousarray(recs[:120])), np.arange(120, dtype=np.uint32))
    assert np.array_equal(tab.prev_hashes(), oracle.record_hashes(np.ascontiguousarray(recs[:120])))


def test_status_table_restride_keeps_state():
    """The same logical records at another stride are the same state: seeded at 16, they report nothing at 64 or 256,
    and a long status seeded at 256 still differs from everything a 16-byte slot can hold -- until it is replaced."""
    N = 400
    lt = sc.LogicalTable(N, np.random.default_rng(3))
    tab = oracle.StatusTable(N, 16)
    tab.seed(lt.records(16))
    for stride in (64, 256, 32, 16):
        assert len(tab.diff(lt.records(stride))) == 0, stride
    lt.step(256, 0.5)
    wide = lt.records(256)
    long_rows = np.nonzero(lt.lens[lt.ids] > sc.capacity(16))[0]
    assert len(long_rows) > 20
    tab.seed(wide)
    assert tab.stride == 256 and len(tab.diff(lt.records(256))) == 0
    assert np.array_equal(tab.prev_hashes(), oracle.record_hashes(wide))
    lt.step(16, 0.0)  # only the slots whose status does not fit 16 bytes change
    got = tab.diff(lt.records(16))
    assert np.array_equal(got, long_rows.astype(np.uint32))
    assert len(tab.diff(lt.records(128))) == 0


def test_status_table_program_matches_numpy_restatement():
    """Seeded programs of reset / seed / seed_slots / diff at every stride: the oracle's table equals the decoded
    (status, ports) bookkeeping of np_restatement after every step."""
    for seed in range(6):
        rng = np.random.default_rng(100 + seed)
        N = int(rng.choice([1, 63, 200, 513]))
        lt = sc.LogicalTable(N, rng)
        tab = oracle.StatusTable(N, 16)
        prev = [None] * N
        log = []
        for step in range(40):
            stride = int(rng.choice(sc.STRIDES))
            lt.step(stride, float(rng.choice([0.0, 0.05, 0.5])))
            recs = lt.records(stride)
            op = rng.choice(["diff", "diff", "seed", "seed_slots", "reset"])
            log.append((str(op), stride))
            if op == "diff":
                assert np.array_equal(tab.diff(recs), npr.status_changed_set(recs, prev)), (seed, log)
            elif op == "seed":
                tab.seed(recs)
                prev = _decoded(recs)
            elif op == "seed_slots":
                slots = rng.choice(N, int(rng.integers(1, N + 1)), replace=False)
                tab.seed_slots(slots, recs[slots])
                for s in slots:
                    prev[s] = npr.decode_record(recs[s])
            else:
                tab.reset(N)
                prev = [None] * N
            want = np.array([0 if p is None else 1 for p in prev], np.uint8)
            assert np.array_equal(tab.has_prev, want), (seed, log)


@pytest.mark.parametrize("stride", sc.STRIDES)
def test_status_code_corpus_oracles_agree(stride):
    """The adversarial corpus (near-misses of every known status) x ports x message flag: the record decoder of the
    oracle (record_codes) and translateRunPodStatus on the decoded string agree -- so either can pin the kernels."""
    recs, sts, ports, flags = sc.corpus_records(stride)
    want = sc.translated_codes(sts, ports, flags)
    assert np.array_equal(oracle.record_codes(recs), want)
    # the corpus really reaches every branch: all six known statuses, both RUNNING forms, both EXITED forms, unknown
    assert len(set(want.tolist())) == 8
