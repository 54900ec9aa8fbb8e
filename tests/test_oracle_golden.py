"""Pins the CPU oracle (oracle/kta_oracle.c) to every golden vector available for this path:
FNV known-answer vectors (src/fnv32.rs:92-101 followed by hand) and the one real output of the
reference, demo_output.png.  Then the quirk list of SURVEY.md §8(c), each quirk one test, each
citing the reference lines it comes from."""
import json
import os

import numpy as np
import pytest

import np_oracle
from oracle_lib import Oracle, fnv32, hll_estimate, olib
from parity import replay_demo_row

GOLD = os.path.join(os.path.dirname(__file__), "golden")


def _kat():
    return json.load(open(os.path.join(GOLD, "fnv_kat.json")))["vectors"]


def _demo():
    return json.load(open(os.path.join(GOLD, "demo_output.json")))


def test_fnv_kat_oracle():
    for v in _kat():
        assert fnv32(bytes.fromhex(v["key_hex"])) == v["reference_fnv32"], v


def test_fnv_is_not_standard_fnv1a():
    # Q1: the multiplier is the offset basis 0x811c9dc5 (fnv32.rs:97), so everything but "" differs
    for v in _kat():
        if v["key_hex"]:
            assert v["reference_fnv32"] != v["standard_fnv1a32"]
        else:
            assert v["reference_fnv32"] == 0x811C9DC5


def test_fnv_numpy_oracle_agrees():
    keys = [bytes.fromhex(v["key_hex"]) for v in _kat()]
    kl = np.array([len(k) for k in keys], dtype=np.int32)
    kb = np.frombuffer(b"".join(keys), dtype=np.uint8)
    got = np_oracle.fnv32_many(kl, kb)
    assert got.tolist() == [v["reference_fnv32"] for v in _kat()]


def test_demo_output_table_getters():
    """All 10 rows of demo_output.png: set the 7 counters, read every column the report prints
    (src/main.rs:153-171) through the oracle's getters / derived metrics (metric.rs:104-167)."""
    demo = _demo()
    o = Oracle()
    for r in demo["rows"]:
        p = r["P"]
        o.set_counter("total", p, r["total"])
        o.set_counter("alive", p, r["alive"])
        o.set_counter("tombstones", p, r["tombstones"])
        o.set_counter("key_null", p, r["key_null"])
        o.set_counter("key_non_null", p, r["key_non_null"])
        o.set_counter("key_size_sum", p, r["k_bytes"])
        o.set_counter("value_size_sum", p, r["v_bytes"])
    for r in demo["rows"]:
        p = r["P"]
        assert o.counter("key_size_sum", p) + o.counter("value_size_sum", p) == r["p_bytes"]  # main.rs:165
        assert o.avg("key_size_avg", p) == r["key_size_avg"]
        assert o.avg("value_size_avg", p) == r["value_size_avg"]
        assert o.avg("message_size_avg", p) == r["message_size_avg"]
        assert "%.4f" % o.dirty_ratio(p) == r["dirty_ratio"]


def test_demo_output_replay_row8():
    """Row 8 (the one whose averages differ: 262 / 271) replayed record by record through
    MessageMetrics::handle_message (metric.rs:206-253)."""
    demo = _demo()
    row = demo["rows"][8]
    o = Oracle(no_hist=True)

    def feed(part, ts, kl, vl):
        o.handle_batch(part, ts, kl, vl, np.zeros(0, dtype=np.uint8))

    replay_demo_row(row, demo, feed)
    p = 8
    assert o.counter("total", p) == row["total"] and o.counter("alive", p) == row["alive"]
    assert o.counter("key_non_null", p) == row["key_non_null"] and o.counter("key_null", p) == 0
    assert o.counter("key_size_sum", p) == row["k_bytes"] and o.counter("value_size_sum", p) == row["v_bytes"]
    assert (o.avg("key_size_avg", p), o.avg("value_size_avg", p), o.avg("message_size_avg", p)) == (9, 262, 271)
    assert o.scalar("largest_message") == 750 and o.scalar("smallest_message") == 139
    assert o.earliest() == (demo["earliest_message_s"], 0) and o.latest() == demo["latest_message_s"]
    assert o.scalar("overall_size") == row["p_bytes"] and o.scalar("overall_count") == row["total"]


# ------------------------------ quirks (SURVEY.md §8 c, Q2..Q11) ------------------------------

def test_q2_avg_divides_by_alive_and_panics():
    o = Oracle()
    o.handle_message(0, 1000, b"abc", None)  # keyed tombstone only: key_size_sum 3, alive 0
    with pytest.raises(ZeroDivisionError):
        o.avg("key_size_avg", 0)             # metric.rs:132-139
    with pytest.raises(ZeroDivisionError):
        o.avg("message_size_avg", 0)         # metric.rs:150-157
    assert o.avg("value_size_avg", 0) == 0   # sum == 0 → guarded
    o.handle_message(0, 1000, b"abcd", 10)
    assert o.avg("key_size_avg", 0) == 7     # (3+4)/alive(=1), NOT / key_non_null(=2)


def test_q3_q4_min_max_size_skip_tombstones():
    o = Oracle()
    assert o.scalar("smallest_message") == 0          # Q4 metric.rs:177-183
    o.handle_message(0, 0, b"k" * 100, None)           # tombstone: not a size sample (metric.rs:249-251)
    assert o.scalar("largest_message") == 0 and o.scalar("smallest_message") == 0
    o.handle_message(0, 0, None, 7)                    # null key + value: size = 7
    o.handle_message(0, 0, b"kk", 20)
    assert o.scalar("largest_message") == 22 and o.scalar("smallest_message") == 7
    o.handle_message(0, 0, b"", 0)                     # Q10: empty key + empty value → size 0 sample
    assert o.scalar("smallest_message") == 0 and o.counter("alive", 0) == 3


def test_q5_q6_timestamps():
    now = (2_000_000_000, 5)
    o = Oracle(now=now)
    assert o.earliest() == now and o.latest() == 0     # Q6 metric.rs:39-40
    o.handle_message(0, 2_000_000_000_999, b"a", 1)     # same second as `now`, but now has ns > 0
    assert o.earliest() == (2_000_000_000, 0)
    o.handle_message(0, None, b"a", 1)                  # Q5: missing → 0 → 1970-01-01 (metric.rs:209)
    assert o.earliest() == (0, 0)
    o.handle_message(0, -1500, b"a", 1)                 # truncating division: -1500/1000 == -1
    assert o.earliest() == (-1, 0)
    o.handle_message(0, -999, b"a", 1)                  # -999/1000 == 0 (toward zero), not -1
    assert o.earliest() == (-1, 0)
    assert o.latest() == 2_000_000_000
    o2 = Oracle(now=now)
    o2.handle_message(0, 2_000_000_001_000, b"a", 1)    # later than now: earliest stays the construction clock
    assert o2.earliest() == now and o2.latest() == 2_000_000_001


def test_q7_alive_counts_messages_not_keys():
    o = Oracle()
    for _ in range(5):
        o.handle_message(3, 0, b"same", 1)
    assert o.counter("alive", 3) == 5                   # metric.rs:239


def test_q8_dirty_ratio_f32():
    o = Oracle()
    assert o.dirty_ratio(0) == 0.0
    for i in range(3):
        o.handle_message(0, 0, b"k", None if i == 0 else 1)
    want = np.float32(1) / (np.float32(3) / np.float32(100.0))   # metric.rs:163 operation order
    assert o.dirty_ratio(0) == float(want)
    o.handle_message(1, 0, b"k", 1)
    assert o.dirty_ratio(1) == 0.0                       # tombstones == 0


def test_q9_alive_keys_global_last_writer_wins():
    o = Oracle(count_alive_keys=True)
    o.handle_message(0, 0, b"a", 1)
    o.handle_message(1, 0, b"a", None)       # same key, other partition: one global set (metric.rs:262-264)
    assert o.scalar("sum_all_alive") == 0
    o.handle_message(2, 0, b"a", 1)
    o.handle_message(0, 0, b"b", None)       # remove of a never-inserted key is a no-op
    o.handle_message(0, 0, None, 1)          # null key ignored (metric.rs:302)
    o.handle_message(0, 0, b"", 1)           # Q10: empty key is a key; hashes to the basis
    assert o.scalar("sum_all_alive") == 2
    assert olib().kto_alive_contains(o.o, 0x811C9DC5) == 1
    assert olib().kto_alive_contains(o.o, fnv32(b"a")) == 1
    assert olib().kto_alive_contains(o.o, fnv32(b"b")) == 0


def test_q11_unseen_partition_reads_zero():
    o = Oracle()
    o.handle_message(5, 0, b"k", 1)
    for name in ("total", "alive", "tombstones", "key_null", "key_non_null", "key_size_sum", "value_size_sum"):
        assert o.counter(name, 4) == 0 and o.counter(name, -7) == 0     # metric.rs:198-203
    assert o.avg("key_size_avg", 4) == 0 and o.dirty_ratio(4) == 0.0


def test_any_partition_id_is_a_key():
    o = Oracle()
    o.handle_message(-3, 0, b"k", 1)
    o.handle_message(2_000_000_000, 0, None, None)
    assert o.counter("total", -3) == 1 and o.counter("tombstones", 2_000_000_000) == 1


# ------------------------------ extensions ------------------------------

def test_hist_invariants_tie_to_reference_counters():
    rng = np.random.default_rng(1)
    o = Oracle()
    for _ in range(2000):
        kl = int(rng.integers(-1, 70))
        vl = int(rng.choice([-1, 0, 1, 2, 3, 255, 256, 257, 65535, 65536, 1 << 20]))
        o.handle_message(int(rng.integers(0, 3)), 0, None if kl < 0 else b"x" * kl, None if vl < 0 else vl)
    for p in range(3):
        kh, vh = o.hist(0, p), o.hist(1, p)
        assert int(kh.sum()) == o.counter("key_non_null", p)
        assert int(vh.sum()) == o.counter("alive", p)
        lo = sum(int(c) * (0 if b == 0 else 1 << (b - 1)) for b, c in enumerate(vh))
        hi = sum(int(c) * (0 if b == 0 else (1 << b) - 1) for b, c in enumerate(vh))
        assert lo <= o.counter("value_size_sum", p) <= hi


def test_hll_estimator_accuracy():
    rng = np.random.default_rng(7)
    for p, n in ((14, 1000), (14, 50_000), (14, 400_000), (16, 200_000), (12, 30)):
        hashes = rng.choice(1 << 32, size=n, replace=False).astype(np.uint32)
        regs = np.zeros(1 << p, dtype=np.uint8)
        for h in hashes.tolist():
            olib().kto_hll_insert(regs.ctypes.data, p, h)
        est = hll_estimate(regs, p)
        sigma = 1.04 / np.sqrt(1 << p)
        assert abs(est - n) <= max(4 * sigma * n, 3), (p, n, est)


# ------------------------------------------------------------------------------------------------
# property test: the two independent restatements (C, record at a time; numpy, vectorised) agree on arbitrary
# batches — nulls, empties, negative / missing timestamps, colliding and repeated keys, any partition layout
# ------------------------------------------------------------------------------------------------
from hypothesis import given, settings, strategies as st
from oracle_lib import COUNTERS

_key = st.one_of(st.none(), st.binary(min_size=0, max_size=24), st.sampled_from([b"a", b"b", b"key-0", b"key-1", b""]))
_val = st.one_of(st.none(), st.integers(min_value=0, max_value=70_000), st.sampled_from([0, 1, 65535, 65536, 2**31 - 1]))
_ts = st.one_of(st.none(), st.integers(min_value=-10**7, max_value=2 * 10**12), st.sampled_from([0, 999, 1000, -999, -1000, -1]))
_rec = st.tuples(st.integers(min_value=0, max_value=6), _ts, _key, _val)


@settings(max_examples=60, deadline=None)
@given(st.lists(_rec, min_size=0, max_size=60))
def test_c_and_numpy_restatements_agree_on_arbitrary_batches(records):
    import np_oracle
    P = 7
    o = Oracle(count_alive_keys=True, now=(4102444800, 7))
    for p, ts, key, vl in records:
        o.handle_message(p, ts, key, vl)
    n = len(records)
    part = np.array([r[0] for r in records], dtype=np.int32)
    ts = np.array([-1 if r[1] is None else r[1] for r in records], dtype=np.int64)   # None -> "not available" (-1)
    kl = np.array([-1 if r[2] is None else len(r[2]) for r in records], dtype=np.int32)
    vl = np.array([-1 if r[3] is None else r[3] for r in records], dtype=np.int32)
    kb = np.frombuffer(b"".join(r[2] or b"" for r in records), dtype=np.uint8)
    m = np_oracle.message_metrics(P, part, ts, kl, vl)
    for p in range(P):
        for name in COUNTERS:
            assert o.counter(name, p) == int(m[name][p]), (name, p)
        assert o.hist(0, p).tolist() == m["khist"][p].tolist() and o.hist(1, p).tolist() == m["vhist"][p].tolist()
    assert o.scalar("overall_count") == n and o.scalar("overall_size") == m["overall_size"]
    assert o.scalar("largest_message") == m["largest"] and o.scalar("smallest_message") == m["smallest"]
    if n:
        # an explicit -1 and a missing timestamp are the same thing at this boundary (rdkafka: to_millis() == None)
        assert o.earliest() == (min(m["min_ts_s"], 4102444800), 0 if m["min_ts_s"] <= 4102444800 else 7)
        assert o.latest() == max(m["max_ts_s"], 0)
    else:
        assert o.earliest() == (4102444800, 7) and o.latest() == 0
    h = np_oracle.fnv32_many(kl, kb)
    assert o.scalar("sum_all_alive") == len(np_oracle.alive_set(kl, vl, h))
