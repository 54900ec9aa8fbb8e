"""GPU parity tests: the CUDA path, called through the C ABI (include/kta.h), against the CPU oracle on
the same seeded inputs — bit-exact for every counter, sum, histogram bucket, extremum, the alive-key
count and the HLL registers; HLL *estimate* within 4 sigma of the exact count (sigma = 1.04/sqrt(m)).
At the full BASELINE sizes parity is checked through size-independent invariants."""
import json
import os

import numpy as np
import pytest

from kafka_topic_analyzer_b200 import KtaEngine, KtaError, Message, TopicAnalyzer, synth
from kafka_topic_analyzer_b200 import _native as N
from kafka_topic_analyzer_b200.synth import HostTopic, tile_base_from_key_len
from feed import (Topic, capture_hashes, device, feed, fixed_width_topic, push_host, push_records, random_topic, scan,
                  settle, take, to_device)
from oracle_lib import Oracle
from parity import assert_parity, expected, oracle_for, replay_demo_row
import np_oracle

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(__file__), "golden")
NOW = (4102444800, 123456789)  # 2100-01-01: later than every synthetic record


# ------------------------------------------------------------------------------------------------
def test_fnv_kat_on_device():
    """src/fnv32.rs:92-101 known answers, computed by the device hash."""
    vec = json.load(open(os.path.join(GOLD, "fnv_kat.json")))["vectors"]
    with KtaEngine(1) as e:
        got = e.fnv32([bytes.fromhex(v["key_hex"]) for v in vec] + [None])
    assert got[:-1].tolist() == [v["reference_fnv32"] for v in vec]
    assert got[-1] == 0
    assert all(g != v["standard_fnv1a32"] for g, v in zip(got.tolist(), vec) if v["key_hex"])


@pytest.mark.parametrize("mode", ["device", "device_no_tile_base", "host_batch", "push"])
def test_config0_counters(mode):
    """BASELINE configs[0]: 4 partitions, 100k messages, counters + histograms, no -c."""
    spec = synth.make_spec(100_000, 4, ts_missing_per_10k=10, empty_value_per_10k=20)
    t = synth.fill_host(spec)
    o = oracle_for(t, now=NOW)
    with KtaEngine(4, now=NOW, ring_records=16384) as e:
        if mode == "push":
            push_records(e, t, 30_000)
            o = Oracle(now=NOW)
            o.handle_batch(t.partition[:30000], t.ts_ms[:30000], t.key_len[:30000], t.value_len[:30000], t.key_bytes)
        else:
            feed(e, t, mode)
        e.finalize()
        assert_parity(e, o, 4)


@pytest.mark.parametrize("key_mode,run_len,P", [(0, 1, 64), (1, 64, 16), (2, 7, 5), (0, 500, 256), (2, 1, 700)])
def test_fused_alive_exact_and_hll(key_mode, run_len, P):
    """-c path: FNV per key from staged shared memory + exact alive-key table, vs the BitSet replay."""
    n = P * run_len * max(1, 120_000 // (P * run_len))
    spec = synth.make_spec(n, P, run_len=run_len, key_mode=key_mode, distinct_keys=max(P, n // 20),
                           tombstone_per_10k=2500, null_key_per_10k=300, ts_missing_per_10k=5)
    t = synth.fill_host(spec)
    o = oracle_for(t, count_alive_keys=True, now=NOW)
    with KtaEngine(P, count_alive_keys=True, hll_precision=12, now=NOW) as e:
        scan(e, t)
        e.finalize()
        assert_parity(e, o, P, check_alive=True, hll_regs=o.hll_alive_regs(12))
        exact = e.alive_keys()
        assert abs(e.alive_keys_hll() - exact) <= max(4 * 1.04 / 64 * exact, 3)


@pytest.mark.parametrize("key_mode,P", [(0, 8), (1, 64)])
def test_stress_distributions_hot_keys_and_value_tail(key_mode, P):
    """SURVEY.md §8 d stress cases: log-uniform key ids (the hottest key of a partition carries ~8 % of its records, so
    many stamps of one hash are in flight at once) and geometric-tailed value lengths (lanes below and above 2^16 in
    the same warp: both byte-sum paths inside one tile)."""
    n = P * 20_000
    spec = synth.make_spec(n, P, key_mode=key_mode, distinct_keys=P * 4096, value_mean=2048, tombstone_per_10k=2000,
                           null_key_per_10k=200, zipf_keys=True, geometric_values=True)
    t = synth.fill_host(spec)
    assert int(t.value_len.max()) > (1 << 16) and int((t.value_len < (1 << 16)).sum()) > n // 2
    for mode in ("exact", "hll"):                                # hll: the in-stream sketch (no -c), the fused bench mode
        o, kw = expected(mode, t, 12)
        with KtaEngine(P, count_alive_keys=mode == "exact", hll_precision=12, now=NOW) as e:
            scan(e, t)
            e.finalize()
            assert_parity(e, o, P, **kw)


@pytest.mark.parametrize("seed", [1, 2, 3])
def test_random_ragged_batches(seed):
    """Adversarial inputs: ragged keys 0..40 B, null/empty keys and values, missing and negative
    timestamps, i32-max value length, several batches through different entry points."""
    rng = np.random.default_rng(seed)
    P = 9
    o = Oracle(count_alive_keys=True, now=NOW)
    with KtaEngine(P, count_alive_keys=True, hll_precision=10, now=NOW, ring_records=4096) as e:
        base = 0
        for b in range(4):
            t = random_topic(rng, int(rng.integers(1, 9000)), P, big=True)
            o.handle_batch(t.partition, t.ts_ms, t.key_len, t.value_len, t.key_bytes)
            if b % 2 == 0:
                push_host(e, t, tile_base=b == 0, seq_base=base)
            else:
                scan(e, t, tile_base=False, seq_base=base)
            base += t.n
        e.finalize()
        assert_parity(e, o, P, check_alive=True, hll_regs=o.hll_alive_regs(10))


@pytest.mark.parametrize("L", [1, 9, 16, 17, 40, 100, 200])
def test_fixed_width_keys(L):
    """Fixed-width keys of any length take the ballot-offset path (16-byte aligned ones the LDS.128 path)."""
    t = fixed_width_topic(np.random.default_rng(L), 20_000, 5, L, 0.03, 500)
    o = oracle_for(t, count_alive_keys=True, now=NOW)
    with KtaEngine(5, count_alive_keys=True, hll_precision=9, now=NOW) as e:
        scan(e, t)
        e.finalize()
        assert_parity(e, o, 5, check_alive=True, hll_regs=o.hll_alive_regs(9))


def test_hash_capture_matches_oracle_per_record():
    """Every per-record hash computed inside the fused kernel (bulk-copy staged path, all alignments)."""
    import torch
    rng = np.random.default_rng(11)
    t = random_topic(rng, 50_000, 3)
    want = np_oracle.fnv32_many(t.key_len, t.key_bytes)
    with KtaEngine(3, hll_precision=8, now=NOW) as e:
        out = torch.full((t.n,), 0xFFFFFFFF, dtype=torch.int64, device="cuda").to(torch.int32)
        capture_hashes(e, out)
        scan(e, t)
        e.finalize()
        capture_hashes(e, None)
        got = out.cpu().numpy().view(np.uint32)
    assert np.array_equal(got, want)


def test_hll_in_stream_registers():
    """Extension: without -c the sketch is fed in-stream by every (key, value) record."""
    spec = synth.make_spec(64 * 2000, 64, distinct_keys=20_000, tombstone_per_10k=0, null_key_per_10k=50)
    t = synth.fill_host(spec)
    o = oracle_for(t, track_stream=True, now=NOW)
    with KtaEngine(64, hll_precision=14, now=NOW) as e:
        scan(e, t)
        e.finalize()
        assert_parity(e, o, 64, hll_regs=o.hll_stream_regs(14))
        distinct = len(set(np_oracle.fnv32_many(t.key_len, t.key_bytes)[(t.key_len >= 0) & (t.value_len >= 0)].tolist()))
        assert abs(e.alive_keys_hll() - distinct) <= 4 * 1.04 / 128 * distinct
        with pytest.raises(KtaError):
            e.alive_keys()   # -c was not given


def test_edge_cases():
    with KtaEngine(2, count_alive_keys=True, now=NOW) as e:
        e.finalize()                                    # empty topic
        o = Oracle(count_alive_keys=True, now=NOW)
        assert_parity(e, o, 2, check_alive=True)
        assert e.message_metrics.earliest_message() == NOW and e.message_metrics.latest_message() == 0
        # keyed tombstone only → the averages panic in the reference (metric.rs:132-157)
        e.push(0, 0, 1000, b"abc", -1)
        o.handle_message(0, 1000, b"abc", None)
        # null key tombstone, empty key, empty value
        e.push(1, 0, -1, None, -1)
        o.handle_message(1, None, None, None)
        e.push(1, 1, 5, b"", 0)
        o.handle_message(1, 5, b"", 0)
        e.finalize()
        assert_parity(e, o, 2, check_alive=True)
        with pytest.raises(ZeroDivisionError):
            e.message_metrics.key_size_avg(0)
        e.reset()
        e.finalize()
        assert e.message_metrics.overall_count() == 0 and e.alive_keys() == 0


def test_reset_forgets_the_alive_table():
    """kta_reset wipes the alive-key table: stamps of the previous topic must not leak."""
    sa = synth.make_spec(8 * 4000, 8, distinct_keys=800, tombstone_per_10k=1000, key_mode=1)
    sb = synth.make_spec(8 * 3000, 8, distinct_keys=800, tombstone_per_10k=6000, key_mode=1, seed=77)   # same key space
    ta, tb = synth.fill_host(sa), synth.fill_host(sb)
    with KtaEngine(8, count_alive_keys=True, hll_precision=10, now=NOW) as e:
        for t in (ta, tb, ta):
            e.reset()
            scan(e, t)
            e.finalize()
            o = oracle_for(t, count_alive_keys=True, now=NOW)
            assert_parity(e, o, 8, check_alive=True, hll_regs=o.hll_alive_regs(10))
        # and without a reset the second topic continues the first (seq keeps counting)
        e.reset()
        push_host(e, ta, seq_base=0)
        push_host(e, tb, seq_base=ta.n)
        e.finalize()
        o = Oracle(count_alive_keys=True, now=NOW)
        o.handle_batch(ta.partition, ta.ts_ms, ta.key_len, ta.value_len, ta.key_bytes)
        o.handle_batch(tb.partition, tb.ts_ms, tb.key_len, tb.value_len, tb.key_bytes)
        assert_parity(e, o, 8, check_alive=True, hll_regs=o.hll_alive_regs(10))


@pytest.mark.parametrize("layout", ["runs", "interleaved"])
def test_byte_sums_survive_u32_wraparound(layout):
    """Every CTA adds far more than 2^32 to its 16-bit-split shared-memory sums, so the result is only exact if the
    fold logic drains them in time.  "runs": two long runs, lengths 0x1ffff / 0xffff (warp-reduced rows, high halves in
    use).  "interleaved": three partitions round-robin, every length 0xffff (the per-lane path whose fast branch adds
    the whole length to the low word: the largest value that branch can add, 48 M times)."""
    import torch
    if layout == "runs":
        n, P, klv, vlv = 16_000_000, 2, 0x1FFFF, 0xFFFF
        part = torch.zeros(n, dtype=torch.int32, device="cuda")
        part[n // 2:] = 1
    else:
        n, P, klv, vlv = 48_000_000, 3, 0xFFFF, 0xFFFF
        part = (torch.arange(n, dtype=torch.int64, device="cuda") % 3).to(torch.int32)
    ts = torch.full((n,), 1_600_000_000_000, dtype=torch.int64, device="cuda")
    kl = torch.full((n,), klv, dtype=torch.int32, device="cuda")
    vl = torch.full((n,), vlv, dtype=torch.int32, device="cuda")
    with KtaEngine(P, now=NOW) as e:
        scan(e, Topic(part, ts, kl, vl, None, 0), tile_base=False)
        e.finalize()
        mm = e.message_metrics
        for p in range(P):
            assert mm.total(p) == n // P and mm.key_size_sum(p) == (n // P) * klv and mm.value_size_sum(p) == (n // P) * vlv
        assert mm.overall_size() == n * (klv + vlv)
        assert mm.largest_message() == klv + vlv == mm.smallest_message()
        assert mm.earliest_message() == (1_600_000_000, 0) and mm.latest_message() == 1_600_000_000


@pytest.mark.parametrize("case", ["crossing", "missing_late", "negative_early"])
def test_timestamp_extrema_across_high_word_boundaries(case):
    """The scan compares timestamps on their low 32 bits while every high word it has seen agrees and falls back to
    the 64-bit comparison otherwise (metric.rs:65-72, :209-211).  Topics whose timestamps cross a multiple of 2^32 ms,
    carry a late "not available" (-1 -> 0) or start negative must report the reference's earliest / latest."""
    n, P = 1 << 20, 4
    i = np.arange(n, dtype=np.int64)
    ts = (350 << 32) - 500_000_000 + i * 1000          # crosses 350 * 2^32 at record 500 000
    if case == "missing_late":
        ts = ts.copy()
        ts[900_001] = -1
        ts[n - 1] = -1
    elif case == "negative_early":
        ts = ts - (350 << 32)                             # -5e8 .. +5.5e8: the high word flips 0xffffffff -> 0
    part = (i % P).astype(np.int32)
    kl = np.full(n, -1, dtype=np.int32)
    vl = np.full(n, 10, dtype=np.int32)
    o = Oracle(now=NOW)
    o.handle_batch(part, ts, kl, vl, np.zeros(0, dtype=np.uint8))
    with KtaEngine(P, now=NOW) as e:
        scan(e, Topic(*(device(c) for c in (part, ts, kl, vl)), None, 0), tile_base=False)
        e.finalize()
        assert_parity(e, o, P)
        mm = e.message_metrics
        want_min = 0 if case == "missing_late" else int(ts.min())
        assert mm.earliest_message() == (int(np.trunc(want_min / 1000)), 0)
        assert mm.latest_message() == max(0, int(ts.max()) // 1000)


def test_partition_out_of_range_is_an_error():
    with KtaEngine(2, now=NOW) as e:
        e.push(2, 0, 0, b"k", 1)
        with pytest.raises(KtaError) as ei:
            e.finalize()
        assert ei.value.code == 4


def test_out_of_range_partitions_are_left_out_of_every_metric():
    """A record whose partition is outside [0, P) takes part in nothing — counters, sums, extrema, alive keys — so the
    state stays consistent and equals the reference fed with the in-range records only; finalize says how many."""
    rng = np.random.default_rng(21)
    P = 6
    t = random_topic(rng, 40_000, P)
    badp = rng.random(t.n) < 0.07
    part = t.partition.copy()
    part[badp] = rng.choice(np.array([-1, -5, P, P + 1, 1 << 30], dtype=np.int32), size=int(badp.sum()))
    # the bad records carry the extreme timestamps and sizes: they must not show up in the extrema either
    ts, vl = t.ts_ms.copy(), t.value_len.copy()
    ts[badp] = np.where(rng.random(int(badp.sum())) < 0.5, 1, 4_000_000_000_000)
    vl[badp] = (1 << 31) - 1
    tb = HostTopic(part, t.offset, ts, t.key_len, vl, t.seq, t.key_bytes, t.key_tile_base)
    # oracle: the in-range records only, in order
    o = oracle_for(take(tb, np.nonzero(~badp)[0]), count_alive_keys=True, now=NOW)
    for mode in ("device", "host"):
        with KtaEngine(P, count_alive_keys=True, hll_precision=10, now=NOW, ring_records=8192) as e:
            with pytest.raises(KtaError) as ei:
                if mode == "device":
                    scan(e, tb)
                else:
                    push_host(e, tb, tile_base=False)
                e.finalize()
            assert ei.value.code == 4
            assert e.bad_partition_records() == int(badp.sum())
            assert e.finalize(strict=False) == int(badp.sum())     # the same as a warning: the count, no exception
            assert_parity(e, o, P, check_alive=True, hll_regs=o.hll_alive_regs(10), extra_partitions=())


# ------------------------------------------------------------------------------------------------
# the alive-key table itself: growth + re-run, seq window (rebase), ordering contract
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("mode", ["device", "host_batch", "push", "device_batches"])
def test_alive_table_grows_and_restamps(mode):
    """A table that starts far too small (1 KiB = 128 slots for 6000 keys) drops stamps, is grown (rehash) and the pending
    batches are re-run stamps-only: the result must equal the BitSet replay, counters must not be counted twice."""
    P, n = 8, 120_000
    spec = synth.make_spec(n, P, key_mode=1, distinct_keys=6000, tombstone_per_10k=3000, null_key_per_10k=200)
    t = synth.fill_host(spec)
    o = oracle_for(t, count_alive_keys=True, now=NOW)
    with KtaEngine(P, count_alive_keys=True, hll_precision=11, now=NOW, ring_records=4096, alive_table_kib=1) as e:
        assert e.alive_table_stats()[0] == 128
        if mode != "device_batches":
            feed(e, t, mode)                                # host_batch: 30 ring chunks
        else:
            # several device batches queued before the first confirmation: all of them are re-run
            T = N.KTA_KEY_TILE
            d = to_device(t)
            cuts = [0, 40 * T, 300 * T, 301 * T, n]
            for lo, hi in zip(cuts[:-1], cuts[1:]):
                scan(e, Topic(*(c[lo:hi] for c in (d.partition, d.ts_ms, d.key_len, d.value_len)), d.key_bytes, d.kbl,
                              key_tile_base=d.key_tile_base[lo // T:]))
        e.finalize()
        slots, occupied, grows, reruns = e.alive_table_stats()
        assert grows >= 1 and reruns >= 1 and occupied * 10 <= slots * 7
        distinct = len(set(np_oracle.fnv32_many(t.key_len, t.key_bytes)[t.key_len >= 0].tolist()))
        assert occupied == distinct
        assert_parity(e, o, P, check_alive=True, hll_regs=o.hll_alive_regs(11))
        # and the grown table keeps working: the same topic again (new sequence numbers) changes nothing but the counters
        before = e.alive_keys()
        push_host(e, t)
        e.finalize()
        assert e.alive_keys() == before and e.message_metrics.overall_count() == 2 * n


def test_alive_table_rebase_keeps_last_writer_across_the_seq_window():
    """The table keeps 31 bits of seq.  Batches whose sequence numbers leave the window force a rebase (every entry
    becomes 'older than anything that follows'); the result is still the BitSet replay in batch order."""
    rng = np.random.default_rng(3)
    P = 4
    o = Oracle(count_alive_keys=True, now=NOW)
    bases = [0, (1 << 31) - 1000, (1 << 31) + 10_000, (1 << 33) + 5, (1 << 33) + 20_000, (1 << 40)]
    with KtaEngine(P, count_alive_keys=True, hll_precision=9, now=NOW, alive_table_kib=64) as e:
        for b, base in enumerate(bases):
            t = random_topic(rng, 6000, P, max_key=6)      # short keys: plenty of overwrites between batches
            o.handle_batch(t.partition, t.ts_ms, t.key_len, t.value_len, t.key_bytes)
            if b % 2:
                push_host(e, t, seq_base=base)
            else:
                scan(e, t, tile_base=False, seq_base=base)
            e.finalize()
            assert_parity(e, o, P, check_alive=True, hll_regs=o.hll_alive_regs(9))
        # a batch that goes back before the window: refused, state untouched
        t = random_topic(rng, 100, P)
        with pytest.raises(KtaError) as ei:
            push_host(e, t, seq_base=5)
        assert ei.value.code == 1
        e.finalize()
        assert_parity(e, o, P, check_alive=True)
        # exports need absolute sequence numbers, which a rebase forgets
        with pytest.raises(KtaError):
            e.alive_export_count()


def test_seq_contract():
    """Last-writer-wins is decided by seq (src/kafka.rs:99).  Default = the handle's running count across every entry
    point; re-using sequence numbers without a seq column is refused; explicit seq columns must fit the 31-bit window."""
    rng = np.random.default_rng(9)
    P = 3
    o = Oracle(count_alive_keys=True, now=NOW)
    with KtaEngine(P, count_alive_keys=True, now=NOW) as e:
        for b in range(4):
            t = random_topic(rng, 3000, P, max_key=5)
            o.handle_batch(t.partition, t.ts_ms, t.key_len, t.value_len, t.key_bytes)
            if b == 1:     # per-record pushes in between: the batches after them must count on from there
                push_records(e, t)
            else:
                push_host(e, t)                             # seq_base=None
        e.finalize()
        assert_parity(e, o, P, check_alive=True)
        t = random_topic(rng, 500, P)
        with pytest.raises(KtaError) as ei:
            push_host(e, t, seq_base=0)
        assert ei.value.code == 1 and "seq_base" in str(ei.value)
        # explicit seq outside the window: reported by finalize, the offending records are left out of the table
        seq = np.arange(t.n, dtype=np.uint64) + np.uint64((1 << 31) + 10)
        push_host(e, t, seq=seq)
        with pytest.raises(KtaError) as ei:
            e.finalize()
        assert ei.value.code == 1 and "window" in str(ei.value)


@pytest.mark.parametrize("L,with_tile_base", [(150, False), (150, True), (1000, False), (40_000, False)])
def test_host_batch_whose_keys_exceed_the_staging_ring(L, with_tile_base):
    """kta_push_batch_host splits a batch into chunks whose key bytes fit ring_key_bytes; tiles heavier than 64 B per
    record used to trip the split (ADVICE r1).  Fixed-length L-byte keys, total far above the ring's key capacity."""
    t = fixed_width_topic(np.random.default_rng(L), 40_000 if L < 10_000 else 1500, 4, L, 0.02, 300)
    o = oracle_for(t, count_alive_keys=True, now=NOW)
    ring_kb = 1 << 20 if L < 10_000 else 6 << 20       # one 128-record tile of 40 KB keys is 5 MB
    assert t.key_bytes.size > 4 * ring_kb
    with KtaEngine(4, count_alive_keys=True, now=NOW, ring_records=16384, ring_key_bytes=ring_kb) as e:
        push_host(e, t, tile_base=with_tile_base)
        e.finalize()
        assert_parity(e, o, 4, check_alive=True)
    # a single tile that cannot fit is the one case that is refused, and it says so
    with KtaEngine(4, count_alive_keys=True, now=NOW, ring_records=16384, ring_key_bytes=100 * L) as e:
        with pytest.raises(KtaError) as ei:
            push_host(e, t, tile_base=False)
        assert ei.value.code == 1 and "ring_key_bytes" in str(ei.value)


def test_long_keys_fall_back_to_global_reads():
    """A tile whose keys exceed the 20 KiB staging buffer takes the direct-global path; results equal."""
    rng = np.random.default_rng(5)
    n = 3000
    kl = rng.integers(0, 300, size=n).astype(np.int32)
    kl[100] = 70_000
    kb = rng.integers(0, 256, size=int(np.maximum(kl, 0).sum()), dtype=np.uint8)
    t = HostTopic(rng.integers(0, 3, size=n).astype(np.int32), np.zeros(n, dtype=np.int64),
                  np.full(n, 1_600_000_000_000, dtype=np.int64), kl, rng.integers(-1, 50, size=n).astype(np.int32),
                  np.arange(n, dtype=np.uint64), kb, tile_base_from_key_len(kl))
    o = oracle_for(t, count_alive_keys=True, now=NOW)
    with KtaEngine(3, count_alive_keys=True, now=NOW, ring_key_bytes=1 << 20) as e:
        scan(e, t)
        e.finalize()
        assert_parity(e, o, 3, check_alive=True)
        e.reset()
        push_host(e, t, tile_base=False)
        e.finalize()
        assert_parity(e, o, 3, check_alive=True)


def test_topic_analyzer_interface():
    """The reference's own call shape: two handlers registered, one pass (src/main.rs:108-117)."""
    e = KtaEngine(2, count_alive_keys=True, now=NOW)
    ta = TopicAnalyzer()
    ta.add_metric_handler(e.message_metrics)
    ta.add_metric_handler(e.log_compaction_metrics)
    msgs = [Message(0, 0, 1_600_000_000_000, b"a", 10), Message(1, 0, None, None, 3), Message(0, 1, 1_600_000_001_000, b"a", None),
            Message(1, 1, 1_600_000_002_000, b"b", 5), Message(0, 2, 1_600_000_003_000, b"never-read", 1)]
    seen = ta.read_topic_into_metrics(msgs, {0: 2, 1: 2})
    assert seen == 4                                    # stops when every partition reached its end offset
    assert e.message_metrics.total(0) == 2 and e.message_metrics.total(1) == 2
    assert e.log_compaction_metrics.sum_all_alive() == 1
    e.close()


def test_demo_output_row8_replay_on_gpu():
    """Row 8 of demo_output.png replayed through the GPU path: 20 021 871 records."""
    demo = json.load(open(os.path.join(GOLD, "demo_output.json")))
    row = demo["rows"][8]
    with KtaEngine(10, now=NOW) as e:
        replay_demo_row(row, demo, lambda part, ts, kl, vl: e.push_batch_host(part, ts, kl, vl))
        e.finalize()
        mm = e.message_metrics
        assert (mm.total(8), mm.alive(8), mm.tombstones(8), mm.key_null(8)) == (row["total"], row["alive"], 0, 0)
        assert mm.key_size_sum(8) == row["k_bytes"] and mm.value_size_sum(8) == row["v_bytes"]
        assert (mm.key_size_avg(8), mm.value_size_avg(8), mm.message_size_avg(8)) == (9, 262, 271)
        assert mm.largest_message() == 750 and mm.smallest_message() == 139
        assert mm.earliest_message() == (demo["earliest_message_s"], 0) and mm.latest_message() == demo["latest_message_s"]
        assert "%.4f" % mm.dirty_ratio(8) == "0.0000"


# ------------------------------------------------------------------------------------------------
# full BASELINE sizes: size-independent properties (the oracle would take minutes here)
# ------------------------------------------------------------------------------------------------
def test_config1_full_size_properties():
    """configs[1]: 64 partitions, 1e8 messages, 256 B mean value, generated in HBM.
    (i) closed-form totals; (ii) histogram/counter identities; (iii) scanning the topic in two halves
    equals scanning it whole (associativity); (iv) a 2^20-record prefix equals the oracle bit-exactly."""
    P, n = 64, 100_000_000
    spec = synth.make_spec(n, P, distinct_keys=10_000_000)
    topic = synth.DeviceTopic(spec)
    with KtaEngine(P, hll_precision=14, now=NOW) as e:
        e.scan_batch_device(topic.partition, topic.ts_ms, topic.key_len, topic.value_len, key_bytes=topic.key_bytes,
                            key_bytes_len=topic.key_bytes_len, key_tile_base=topic.key_tile_base)
        e.finalize()
        mm = e.message_metrics
        whole = {p: [e.counter(i, p) for i in range(7)] + e.hist(0, p).tolist() + e.hist(1, p).tolist() for p in range(P)}
        regs = e.hll_registers()
        glob = (mm.smallest_message(), mm.largest_message(), mm.overall_size(), mm.overall_count(),
                mm.earliest_message(), mm.latest_message())
        assert mm.overall_count() == n
        for p in range(P):
            assert mm.total(p) == n // P                                  # generator: equal shares
            assert mm.key_null(p) + mm.key_non_null(p) == mm.total(p)
            assert mm.alive(p) + mm.tombstones(p) == mm.total(p)
            assert mm.key_size_sum(p) == 16 * mm.key_non_null(p)           # key_mode 0: 16-byte keys
            assert 128 * mm.alive(p) <= mm.value_size_sum(p) <= 384 * mm.alive(p)
        assert mm.smallest_message() == 128 and mm.largest_message() == 16 + 384
        # generator: ts = 1.5e12 + 7 i + jitter(0..999); the true extrema come from the column itself (torch reduction)
        assert mm.earliest_message() == (int(topic.ts_ms.min().item()) // 1000, 0) == (1_500_000_000, 0)
        assert mm.latest_message() == int(topic.ts_ms.max().item()) // 1000
        assert (1_500_000_000_000 + (n - 1) * 7) // 1000 <= mm.latest_message() <= (1_500_000_000_000 + (n - 1) * 7 + 999) // 1000
        # halves
        e.reset()
        T = N.KTA_KEY_TILE
        h = (n // 2) // T * T
        for lo, hi in ((0, h), (h, n)):
            e.scan_batch_device(topic.partition[lo:hi], topic.ts_ms[lo:hi], topic.key_len[lo:hi], topic.value_len[lo:hi],
                                key_bytes=topic.key_bytes, key_bytes_len=topic.key_bytes_len,
                                key_tile_base=topic.key_tile_base[lo // T:], seq_base=lo)
        e.finalize()
        assert whole == {p: [e.counter(i, p) for i in range(7)] + e.hist(0, p).tolist() + e.hist(1, p).tolist() for p in range(P)}
        assert np.array_equal(regs, e.hll_registers())
        assert glob == (mm.smallest_message(), mm.largest_message(), mm.overall_size(), mm.overall_count(),
                        mm.earliest_message(), mm.latest_message())
        # prefix vs oracle
        m = 1 << 20
        e.reset()
        e.scan_batch_device(topic.partition[:m], topic.ts_ms[:m], topic.key_len[:m], topic.value_len[:m],
                            key_bytes=topic.key_bytes, key_bytes_len=topic.key_bytes_len, key_tile_base=topic.key_tile_base)
        e.finalize()
        th = synth.fill_host(spec, count=m)
        assert np.array_equal(topic.key_len[:m].cpu().numpy(), th.key_len)     # host and device generators agree
        o = oracle_for(th, track_stream=True, now=NOW)
        assert_parity(e, o, P, hll_regs=o.hll_stream_regs(14))


def test_alive_keys_large_vs_exact_set():
    """configs[2] shape at 1/10 scale on the test box: 1e8 messages, 1e6 distinct keys, 25% tombstones.
    Exact count vs an independent device computation (sort by (hash, seq), take the last of each run)."""
    import torch
    P, n = 64, 100_000_000
    spec = synth.make_spec(n, P, distinct_keys=1_000_000, tombstone_per_10k=2500, null_key_per_10k=0)
    topic = synth.DeviceTopic(spec)
    hashes = torch.empty(n, dtype=torch.int32, device="cuda")
    with KtaEngine(P, count_alive_keys=True, hll_precision=14, now=NOW) as e:
        capture_hashes(e, hashes)
        e.scan_batch_device(topic.partition, topic.ts_ms, topic.key_len, topic.value_len, key_bytes=topic.key_bytes,
                            key_bytes_len=topic.key_bytes_len, key_tile_base=topic.key_tile_base)
        e.finalize()
        capture_hashes(e, None)
        got = e.alive_keys()
        est = e.alive_keys_hll()
    want, _ = _alive_by_sort(hashes, topic.value_len, None)
    assert got == want
    assert abs(est - want) <= 4 * 1.04 / 128 * want


def _alive_by_sort(hashes_i32, value_len, keyed):
    """Independent statement of metric.rs:288-305 on the device: composite (hash, seq, alive) keys sorted; the last
    element of every hash run is that hash's last writer.  torch is plumbing for the CHECK here, not the product."""
    import torch
    n = hashes_i32.shape[0]
    assert n < (1 << 30)
    comp = ((hashes_i32.to(torch.int64) & 0xFFFFFFFF) << 31) | (torch.arange(n, device="cuda", dtype=torch.int64) << 1)
    comp |= (value_len >= 0).to(torch.int64)
    if keyed is not None:
        comp = comp[keyed]
    comp = torch.sort(comp)[0]
    last = torch.ones(comp.shape[0], dtype=torch.bool, device="cuda")
    last[:-1] = (comp[1:] >> 31) != (comp[:-1] >> 31)
    return int((last & ((comp & 1) == 1)).sum().item()), int(last.sum().item())


def test_config2_full_size_alive_exact():
    """BASELINE configs[2] at its stated size: 64 partitions, 1e9 messages, 1e7 distinct keys, -c.  The exact alive count
    of the compact table vs the sort-based statement over all 1e9 (hash, seq, alive) triples; the table must hold exactly
    the distinct hashes; HLL over the resolved set within 4 sigma."""
    import torch
    free, _ = torch.cuda.mem_get_info()
    # peak: 40 GB of columns + hashes during the scan, then ~56 GB while sorting 1e9 composite keys (columns freed)
    if free < 64e9:
        pytest.skip("needs ~60 GB of HBM")
    P, n = 64, 1_000_000_000
    spec = synth.make_spec(n, P, distinct_keys=10_000_000, null_key_per_10k=0)     # compacted topic: every record keyed, 5 % tombstones
    topic = synth.DeviceTopic(spec)
    hashes = torch.empty(n, dtype=torch.int32, device="cuda")
    with KtaEngine(P, count_alive_keys=True, hll_precision=14, now=NOW) as e:
        capture_hashes(e, hashes)
        e.scan_batch_device(topic.partition, topic.ts_ms, topic.key_len, topic.value_len, key_bytes=topic.key_bytes,
                            key_bytes_len=topic.key_bytes_len, key_tile_base=topic.key_tile_base)
        e.finalize()
        capture_hashes(e, None)
        got, est = e.alive_keys(), e.alive_keys_hll()
        slots, occupied, grows, reruns = e.alive_table_stats()
        assert e.message_metrics.overall_count() == n
        # the timed configuration of bench.py --config C2: no capture
        e.reset()
        e.scan_batch_device(topic.partition, topic.ts_ms, topic.key_len, topic.value_len, key_bytes=topic.key_bytes,
                            key_bytes_len=topic.key_bytes_len, key_tile_base=topic.key_tile_base)
        e.finalize()
        assert e.alive_keys() == got
    vl = topic.value_len
    del topic.partition, topic.ts_ms, topic.key_bytes
    want, distinct = _alive_by_sort(hashes, vl, None)
    assert got == want
    assert occupied == distinct and 9_900_000 < distinct <= 10_000_000      # FNV32 collisions merge a few keys (SURVEY a9)
    assert abs(est - want) <= 4 * 1.04 / 128 * want


def test_config3_rank_shape_256_partitions():
    """BASELINE configs[3] as ONE of its 8 ranks sees it: 256 partitions of which only p = r (mod 8) occur, 1 KiB mean
    values, 5e7 of the rank's 5e8 records (the bench runs the full 5e8).  Closed-form shares, identities, and the first
    2^20 records bit-exact against the oracle (which also checks the shard enumeration of the generator)."""
    P, world, rank = 256, 8, 5
    n_total = 400_000_000
    spec = synth.make_spec(n_total, P, distinct_keys=8_000_000, value_mean=1024)
    topic = synth.DeviceTopic(spec, rank=rank, world=world)
    n = topic.n
    assert n == n_total // world
    with KtaEngine(P, hll_precision=14, now=NOW) as e:
        e.scan_batch_device(topic.partition, topic.ts_ms, topic.key_len, topic.value_len, key_bytes=topic.key_bytes,
                            key_bytes_len=topic.key_bytes_len, key_tile_base=topic.key_tile_base)
        e.finalize()
        mm = e.message_metrics
        assert mm.overall_count() == n
        for p in range(P):
            assert mm.total(p) == (n_total // P if p % world == rank else 0)
            assert mm.key_null(p) + mm.key_non_null(p) == mm.total(p) == mm.alive(p) + mm.tombstones(p)
            assert mm.key_size_sum(p) == 16 * mm.key_non_null(p)
            assert 512 * mm.alive(p) <= mm.value_size_sum(p) <= 1536 * mm.alive(p)
            assert int(e.hist(0, p).sum()) == mm.key_non_null(p) and int(e.hist(1, p).sum()) == mm.alive(p)
        assert mm.smallest_message() == 512 and mm.largest_message() == 16 + 1536
        assert mm.earliest_message() == (int(topic.ts_ms.min().item()) // 1000, 0)
        assert mm.latest_message() == int(topic.ts_ms.max().item()) // 1000
        m = 1 << 20
        e.reset()
        e.scan_batch_device(topic.partition[:m], topic.ts_ms[:m], topic.key_len[:m], topic.value_len[:m],
                            key_bytes=topic.key_bytes, key_bytes_len=topic.key_bytes_len, key_tile_base=topic.key_tile_base)
        e.finalize()
        th = synth.fill_host(spec, rank=rank, world=world, count=m)
        assert np.array_equal(topic.partition[:m].cpu().numpy(), th.partition) and set(th.partition.tolist()) <= set(range(rank, P, world))
        o = oracle_for(th, track_stream=True, now=NOW)
        assert_parity(e, o, P, hll_regs=o.hll_stream_regs(14))


@pytest.mark.parametrize("P,world,run_len", [(16, 4, 3), (256, 8, 1), (10, 3, 1)])
def test_partition_sharded_engines_merge_to_the_whole_topic(P, world, run_len):
    """SURVEY.md §8 e on one device: `world` engines, engine r scanning only the partitions p = r (mod world) with counter
    columns carved for those alone (kta_config.shard_*); their exported merge buffers summed (what the ONE all-reduce does)
    and imported give the whole topic's state, bit for bit the oracle's.  A record of a foreign partition is left out."""
    import torch
    n = P * run_len * max(1, 60_000 // (P * run_len))
    spec = synth.make_spec(n, P, run_len=run_len, key_mode=1, distinct_keys=max(P, n // 10), tombstone_per_10k=2000,
                           null_key_per_10k=300, ts_missing_per_10k=10)
    whole = synth.fill_host(spec)
    o = oracle_for(whole, track_stream=True, now=NOW)
    engines = [KtaEngine(P, hll_precision=11, now=NOW, shard=(r, world)) for r in range(world)]
    try:
        words = engines[0].merge_words(world)
        total = torch.zeros(words, dtype=torch.int64, device="cuda")
        for r, e in enumerate(engines):
            # shard r of the topic = the records whose partition is r mod world, in seq order
            scan(e, take(whole, np.nonzero(whole.partition % world == r)[0]))
            e.finalize()
            # the shard alone: its own partitions as the oracle sees them, the others untouched
            mm = e.message_metrics
            for p in range(P):
                assert mm.total(p) == (o.counter("total", p) if p % world == r else 0)
            buf = torch.zeros(words, dtype=torch.int64, device="cuda")
            settle()
            e.merge_export(r, world, buf)                   # returns once the engine's stream has written buf
            total += buf
        settle()
        engines[0].merge_import(world, total)
        engines[0].finalize()
        assert_parity(engines[0], o, P, hll_regs=o.hll_stream_regs(11))
        # a foreign partition's record on a sharded handle is left out and reported
        e = engines[1 % world]
        e.reset()
        foreign = (1 % world + 1) % world if world > 1 else 0
        e.push(foreign, 0, 1000, b"k", 5)
        with pytest.raises(KtaError) as ei:
            e.finalize()
        assert ei.value.code == 4 and e.bad_partition_records() == 1 and e.message_metrics.overall_count() == 0
    finally:
        for e in engines:
            e.close()
