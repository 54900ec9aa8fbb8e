"""The timeline extension (include/kta.h, kta_set_timeline / kta_timeline): per partition and time bucket, the records,
tombstones and bytes the counters count.

CPU: the numpy restatement against the record-at-a-time one over the edge seconds (hypothesis), the kernel's bucket
quotient and correction step against exact division (hypothesis), the shard rule against brute force, and the merge
buffer's timeline segment (distributed.py).  GPU: every entry point against the numpy restatement fed the delivered
records, with the invariants against kta_counter; the edge seconds and shapes; the bucket edges that need the correction
step; warp aggregation; sharded handles at their limit shapes; both bin paths; the byte carry and a row's high word;
full tiles read row by row; the depth of a launch; the multi-GPU merge; the handle's lifecycle; and that nothing else
changes."""
import ctypes as C
import datetime
import os
import shutil
import subprocess
import sys
import types

import numpy as np
import pytest
import torch
from hypothesis import given, settings, strategies as st

import feed
import kafka_codec as kc
import timeline_ref as TR
from parity import exported
from kafka_topic_analyzer_b200 import KtaEngine, KtaError, lib, distributed
from kafka_topic_analyzer_b200 import _native as N
from kafka_topic_analyzer_b200 import metrics as M

I64_MIN, I64_MAX = -(1 << 63), (1 << 63) - 1
SPECIAL_MS = (-1, 0, -999, -1000, -1001, I64_MIN, I64_MAX)
T0 = 1_500_000_000   # seconds: 2017-07-14


def edge_ms(rng, n, origin, width, buckets):
    """timestamps around every edge of the range (O - 1, O, O + W - 1, O + W, O + B W - 1, O + B W seconds, each at
    a random millisecond), the special values, and uniform ones inside the range"""
    secs = [origin - 1, origin, origin + width - 1, origin + width, origin + buckets * width - 1, origin + buckets * width]
    out = []
    for _ in range(n):
        r = rng.random()
        if r < 0.5:
            s = secs[int(rng.integers(0, len(secs)))]
            ms = int(rng.integers(0, 1000))
            v = s * 1000 + (ms if s >= 0 else -ms)   # truncation: -ms keeps a negative second
        elif r < 0.65:
            v = SPECIAL_MS[int(rng.integers(0, len(SPECIAL_MS)))]
        else:
            v = (origin + int(rng.integers(0, max(buckets * width, 1)))) * 1000 + int(rng.integers(0, 1000))
        out.append(min(max(v, I64_MIN), I64_MAX))
    return np.array(out, dtype=np.int64)


# Ranges whose bucket edges need timeline_index's correction step, as (O, W, B, needs q--, needs q++).  The quotient
# (double)d * (1/W) lands one too low at some edges of 30-day buckets (the first edge among them: d = W gives 0.99999...)
# and of W = 999 999 937; it lands one too high only where d passes 2^53, which takes an origin near the most negative
# second an int64 millisecond value reaches.  B = 2048 fits shared memory up to P = 7, B = 65536 does not fit it at all.
CORRECTION_RANGES = {
    "30d": (1_498_176_000, 2_592_000, 1000, False, True),
    "w999999937": (T0, 999_999_937, 65536, False, True),
    "w2^43-1": (-TR.SMAX, (1 << 43) - 1, 2048, True, True),
    "w2^38-1": (-TR.SMAX, (1 << 38) - 1, 65536, True, True),
}


# ---- CPU ------------------------------------------------------------------------------------------------------------
@settings(max_examples=100, deadline=None)
@given(st.data())
def test_numpy_restatement_matches_record_at_a_time(data):
    origin = data.draw(st.one_of(st.integers(-10 ** 6, 10 ** 6), st.just(0), st.integers(-(1 << 62), 1 << 62)))
    width = data.draw(st.one_of(st.just(1), st.just(1 << 40), st.integers(1, 10 ** 5)))
    buckets = data.draw(st.one_of(st.just(1), st.just(65536), st.integers(1, 300)))
    if origin + buckets * width > I64_MAX:
        origin = I64_MAX - buckets * width
    seed = data.draw(st.integers(0, 2 ** 32 - 1))
    rng = np.random.default_rng(seed)
    n, P = 200, 3
    ts = edge_ms(rng, n, origin, width, buckets)
    p = rng.integers(-1, P + 1, size=n)
    kl = rng.integers(-1, 40, size=n)
    vl = rng.choice([-1, 0, 5, (1 << 31) - 1], size=n)
    recs = list(zip(p.tolist(), ts.tolist(), kl.tolist(), vl.tolist()))
    want = TR.record_counts(P, origin, width, buckets, recs)
    assert np.array_equal(TR.timeline_np(P, origin, width, buckets, p, ts, kl, vl), want)


@pytest.mark.parametrize("origin,width,buckets", [
    (T0, 3600, 197), (-5000, 7, 100), (0, 1, 1), (-(1 << 62), 1 << 40, 2000), (I64_MIN, 1, 1), (I64_MAX - 65536 * 3, 3, 65536),
])
def test_torch_restatement_matches_numpy(origin, width, buckets):
    """timeline_torch (used for depth-sized batches) against timeline_np on CPU tensors, over the edge seconds"""
    rng = np.random.default_rng(buckets)
    n, P = 20_000, 5
    ts = edge_ms(rng, n, origin, width, buckets)
    p = rng.integers(-1, P + 1, size=n).astype(np.int32)
    kl = rng.integers(-1, 40, size=n).astype(np.int32)
    vl = rng.choice([-1, 0, 5, (1 << 31) - 1], size=n).astype(np.int32)
    for shard in (None, (1, 2)):
        want = TR.timeline_np(P, origin, width, buckets, p, ts, kl, vl, shard=shard)
        got = TR.timeline_torch(P, origin, width, buckets, *(torch.from_numpy(a) for a in (p, ts, kl, vl)), shard=shard)
        assert np.array_equal(got.numpy().astype(np.uint64), want)


def test_edge_seconds_by_hand():
    assert [TR.second(v) for v in (-1, 0, -999, -1000, -1001, 1999, -1999)] == [0, 0, 0, -1, -1, 1, -1]
    assert TR.second(I64_MIN) == -9223372036854775 and TR.second(I64_MAX) == 9223372036854775
    O, W, B = -10, 3, 4
    got = [TR.record_index(s * 1000, O, W, B) for s in (O - 1, O, O + W - 1, O + W, O + B * W - 1, O + B * W)]
    assert got == [0, 1, 1, 2, B, B + 1]
    assert list(TR.index_np(np.array([s * 1000 for s in (O - 1, O, O + W - 1, O + W, O + B * W - 1, O + B * W)]), O, W, B)) == got


@settings(max_examples=1000, deadline=None)
@given(st.data())
def test_kernel_index_matches_exact_division(data):
    """the kernel's bucket index (its double-precision quotient and one correction step) equals the exact one, for W up
    to (2^63 - 1) / B, seconds at and beside multiples of W, and origins at the reachable extremes; and the quotient
    before the correction is never off by more than one, for every d below B W (reachable or not)"""
    B = data.draw(st.one_of(st.just(1), st.just(65536), st.integers(1, 65536)), label="B")
    wmax = I64_MAX // B
    W = data.draw(st.one_of(st.integers(1, wmax), st.integers(max(1, wmax - 4096), wmax),
                            st.sampled_from([1, 3, 3600, 2_592_000, 999_999_937, (1 << 38) - 1, 1 << 40, (1 << 43) - 1])),
                  label="W")
    top = I64_MAX - B * W                                   # the largest origin kta_set_timeline accepts
    O = data.draw(st.one_of(st.just(-TR.SMAX), st.integers(-TR.SMAX - 4096, -TR.SMAX + 4096), st.just(I64_MIN),
                            st.just(top), st.just(TR.SMAX - B * W), st.just(0), st.integers(I64_MIN, top)), label="O")
    q = data.draw(st.one_of(st.integers(0, B), st.sampled_from([0, 1, B - 1, B])), label="q")
    delta = data.draw(st.one_of(st.integers(-2, 2), st.integers(-W, W)), label="delta")
    s = min(max(O + q * W + delta, -TR.SMAX), TR.SMAX)
    ms = data.draw(st.sampled_from([0, 1, 999]), label="ms")
    ts = min(max(s * 1000 + (ms if s >= 0 else -ms), I64_MIN), I64_MAX)
    assert TR.second(ts) == s
    assert TR.kernel_index(ts, O, W, B)[0] == TR.record_index(ts, O, W, B)
    d = min(max(q * W + delta, 0), B * W - 1)
    assert abs(TR.kernel_quotient(d, W, B) - d // W) <= 1


def test_boundary_ms_by_hand():
    O, W, B = -3, 5, 2
    want_s = [O - 1, O, O + 1, O + W - 1, O + W, O + W + 1, O + 2 * W - 1, O + 2 * W, O + 2 * W + 1]
    got = TR.boundary_ms(O, W, B)
    assert [TR.second(int(v)) for v in got] == [s for s in want_s for _ in (0, 999)]
    assert list(got[:4]) == [-4000, -4999, -3000, -3999] and list(got[-2:]) == [8000, 8999]
    # the ends of the int64 range keep their second, seconds past them are left out
    low = TR.boundary_ms(-TR.SMAX, 1, 1)
    assert [TR.second(int(v)) for v in low[::2]] == [-TR.SMAX, 1 - TR.SMAX, -TR.SMAX, 1 - TR.SMAX, 2 - TR.SMAX]
    assert low[1] == I64_MIN and TR.boundary_ms(TR.SMAX - 1, 1, 1)[-1] == I64_MAX
    # a large B: every q within `ends` of both ends, `sample` between
    qs = {(TR.second(int(v)) - T0 + 1) // 7 for v in TR.boundary_ms(T0, 7, 65536)}
    assert len(qs) == 2 * 1024 + 4096 and set(range(1024)) <= qs and set(range(65537 - 1024, 65537)) <= qs


@pytest.mark.parametrize("name", list(CORRECTION_RANGES))
def test_correction_ranges_need_their_corrections(name):
    """each range test_bucket_boundaries runs on the GPU has records that need the correction step it is there for"""
    O, W, B, down, up = CORRECTION_RANGES[name]
    steps = {-1: 0, 0: 0, 1: 0}
    for v in TR.boundary_ms(O, W, B).tolist():
        i, step = TR.kernel_index(v, O, W, B)
        assert i == TR.record_index(v, O, W, B)
        steps[step] += 1
    assert (steps[-1] > 0, steps[1] > 0) == (down, up), "%s: %d records need q--, %d need q++" % (name, steps[-1], steps[1])


def shard_division_exact(P, G):
    """the scan's column mulhi(p, ceil(2^32 / G)) is p / G for every p < P: checked at p = kG - 1 (the largest remainder
    of each quotient, where the rounded-up multiplier errs first) and at P - 1"""
    p = np.append(np.arange(G - 1, P, G), P - 1).astype(np.uint64)
    return bool(np.array_equal(TR.shard_column_mulhi(p, G), p // np.uint64(G)))


def test_shard_rule_against_brute_force():
    """kta_create's shard rule accepts only shapes whose every partition the scan divides exactly: all G <= 4096 at
    P = 2^20, every G at P <= 65536, and a seeded sample of larger G; the shapes it refuses include ones the division
    gets wrong"""
    P = 1 << 20
    for G in range(2, 4097):
        assert TR.shard_accepted(P, G) and shard_division_exact(P, G), G
    assert all(TR.shard_accepted(65536, G) for G in range(2, 65537))
    rng = np.random.default_rng(20)
    refused = 0
    for G in rng.integers(4097, P + 1, size=3000).tolist():
        for PP in (G, min(G, 65536), int(rng.integers(G, P + 1)), P):
            PP = max(PP, G)
            if TR.shard_accepted(PP, G):
                assert shard_division_exact(PP, G), (PP, G)
            else:
                refused += 1
    assert refused > 0
    # where the division is wrong: column 1 for partition 65 536 of 65 537 shards; partition 1 031 965 of rank 4177
    for P_, G, p in ((65537, 65537, 65536), (1_031_966, 4178, 1_031_965)):
        assert not TR.shard_accepted(P_, G) and not shard_division_exact(P_, G)
        assert int(TR.shard_column_mulhi([p], G)[0]) == p // G + 1


@pytest.mark.parametrize("world", [1, 4])
def test_merge_buffer_timeline_segment(world):
    rng = np.random.default_rng(world)
    nsums, nhll, tw = 37, 64, 3 * 5 * 7
    assert distributed.merge_words(nsums, nhll, world) == nsums + 4 * world + world * 8
    assert distributed.merge_words(nsums, nhll, world, tw) == distributed.merge_words(nsums, nhll, world) + tw
    tls, bufs = [], []
    for r in range(world):
        tl = rng.integers(0, 1 << 40, size=(3, 5, 7)).astype(np.uint64)
        tls.append(tl)
        sums = rng.integers(0, 1000, size=nsums).astype(np.uint64)
        hll = rng.integers(0, 20, size=nhll).astype(np.uint8)
        plain = distributed.pack_merge_buffer(sums, (5, 9, 1, 2), hll, r, world)
        b = distributed.pack_merge_buffer(sums, (5, 9, 1, 2), hll, r, world, timeline=tl)
        assert np.array_equal(b[:plain.size], plain) and b.size == plain.size + tw
        bufs.append(b)
    total = np.sum(bufs, axis=0, dtype=np.uint64)
    out = distributed.fold_merge_buffer(total, nsums, nhll, world, timeline_words=tw)
    assert len(out) == 4 and np.array_equal(out[3], np.sum(tls, axis=0, dtype=np.uint64).ravel())
    plain3 = distributed.fold_merge_buffer(total[:distributed.merge_words(nsums, nhll, world)], nsums, nhll, world)
    assert len(plain3) == 3 and all(np.array_equal(a, b) for a, b in zip(plain3[0:1] + plain3[2:], out[0:1] + out[2:3]))


# ---- GPU helpers ----------------------------------------------------------------------------------------------------
def engine_tl(P, origin, width, buckets, **kw):
    kw.setdefault("now", feed.NOW)
    e = KtaEngine(P, **kw)
    e.set_timeline(origin, width, buckets)
    return e


def got_arrays(e, P):
    return np.stack([np.stack([e.timeline(w, p) for p in range(P)]) for w in range(3)])


def assert_timeline(e, P, origin, width, buckets, partition, ts_ms, key_len, value_len, shard=None):
    """the engine's three arrays equal the restatement over the given (delivered) records, and each row sums to the
    engine's own counters"""
    want = TR.timeline_np(P, origin, width, buckets, partition, ts_ms, key_len, value_len, shard=shard)
    got = got_arrays(e, P)
    if not np.array_equal(got, want):
        w, p, i = (int(x[0]) for x in np.nonzero(got != want))
        raise AssertionError("counter %d, partition %d, index %d: got %d, want %d" % (w, p, i, got[w, p, i], want[w, p, i]))
    assert_invariants(e, P, got)


def assert_invariants(e, P, got):
    for p in range(P):
        assert int(got[0, p].sum()) == e.counter(M.TOTAL, p)
        assert int(got[1, p].sum()) == e.counter(M.TOMBSTONES, p)
        assert int(got[2, p].sum()) == e.counter(M.KEY_SIZE_SUM, p) + e.counter(M.VALUE_SIZE_SUM, p)


def cols_topic(rng, n, P, origin, width, buckets, bad=False):
    """host columns: partitions (some outside [0, P) when bad), edge timestamps, ragged keys, tombstones"""
    part = rng.integers(-2 if bad else 0, P + (2 if bad else 0), size=n).astype(np.int32)
    ts = edge_ms(rng, n, origin, width, buckets)
    kl = rng.integers(-1, 24, size=n).astype(np.int32)
    vl = rng.choice(np.array([-1, 0, 1, 300, 65535, 65536, 1 << 20], dtype=np.int32), size=n)
    kb = rng.integers(0, 256, size=int(np.maximum(kl, 0).sum()), dtype=np.uint8)
    return part, ts, kl, vl, kb


def scan_cols(e, part, ts, kl, vl, kb=None):
    d = [torch.from_numpy(np.ascontiguousarray(a)).cuda() for a in (part, ts, kl, vl)]
    kbd = None if kb is None else torch.from_numpy(np.concatenate([kb, np.zeros(64, np.uint8)])).cuda()
    feed.settle()
    e.scan_batch_device(*d, key_bytes=kbd, key_bytes_len=0 if kb is None else kb.size)
    return d


# ---- GPU: entry points ----------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("entry", ["push", "host_batch", "device"])
def test_entry_points(entry):
    rng = np.random.default_rng(7)
    P, O, W, B = 6, T0, 3600, 50
    n = 50_000
    part, ts, kl, vl, kb = cols_topic(rng, n, P, O, W, B, bad=True)
    t = feed.HostTopic(part, np.arange(n, dtype=np.int64), ts, kl, vl, np.arange(n, dtype=np.uint64), kb,
                       feed.tile_base_from_key_len(kl))
    with engine_tl(P, O, W, B, count_alive_keys=True, hll_precision=10, ring_records=4096 if entry == "push" else 8192) as e:
        if entry == "push":
            feed.push_records(e, t)            # 13 ring chunks: more than four turns of the three-chunk ring
        elif entry == "host_batch":
            feed.push_host(e, t)
        else:
            feed.scan(e, t)
        assert e.finalize(strict=False) == int(((part < 0) | (part >= P)).sum())
        assert_timeline(e, P, O, W, B, part, ts, kl, vl)


@pytest.mark.gpu
@pytest.mark.parametrize("entry", feed.LOG_ENTRIES)
def test_log_entry_points(entry):
    """every codec, a failed CRC under check.crcs, a window that cuts a batch, and an aborted transaction under
    read_committed: the timeline counts only the delivered records"""
    rng = np.random.default_rng(11)
    P, O, W, B = 4, T0, 60, 30
    codecs = [None, "gzip", "snappy", "snappy-xerial", "lz4", "zstd"]
    parts, delivered = {}, []
    for p in range(P):
        recs = [(T0 * 1000 + 7000 * j + int(rng.integers(0, 900)), None if j % 9 == 0 else b"k%d" % (j % 13),
                 None if j % 5 == 0 else int(rng.integers(0, 300))) for j in range(240)]
        seg = kc.set_crcs(kc.encode_partition(recs, rng, max_batch=30, compression=codecs))
        batches = kc.split_batches(seg)
        # partition 1: one batch's CRC broken; partition 2: an aborted transaction and its marker at the end
        keep = [True] * len(batches)
        if p == 1:
            b = bytearray(batches[2]); b[17:21] = b"\xde\xad\xbe\xef"; batches[2] = bytes(b); keep[2] = False
        recs_by_batch = [kc.delivered(b) if k else [] for b, k in zip(batches, keep)]
        raws = list(batches)
        if p == 2:
            end = max(o for r in recs_by_batch for o, *_ in r) + 1
            raws.append(kc.set_crcs(kc.txn_batch(end, T0 * 1000, [(0, 5, b"x", 10), (1, 6, None, None)], pid=7)))
            raws.append(kc.set_crcs(kc.marker(end + 2, 7, 0, False, T0 * 1000)))
        parts[p] = [types.SimpleNamespace(p=p, raw=r) for r in raws]
        delivered += [(p, ts, k, v) for r in recs_by_batch for (_, ts, k, v) in r]
    # partition 3: a window that starts inside its second batch
    start3 = kc.read_segment(parts[3][1].raw)[0].base_offset + 1
    rec3 = [(o, ts, k, v) for b in parts[3] for (o, ts, k, v) in kc.delivered(b.raw)]
    delivered = [d for d in delivered if d[0] != 3] + [(3, ts, k, v) for (o, ts, k, v) in rec3 if o >= start3]
    with engine_tl(P, O, W, B, count_alive_keys=True, isolation_level="read_committed", check_crcs=True) as e:
        e.set_log_offsets(3, start3, None)
        n, _ = feed.scan_log(e, entry, parts)
        e.finalize()
        assert n == len(delivered)
        assert e.log_crc_stats()[1] == 1 and e.log_txn_stats()[0] == 1
        p_, ts_, k_, v_ = (np.array(x) for x in zip(*[(p, ts, -1 if k is None else len(k), -1 if v is None else v)
                                                    for p, ts, k, v in delivered]))
        assert_timeline(e, P, O, W, B, p_, ts_, k_, v_)


# ---- GPU: edge seconds and shapes -----------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("origin,width,buckets", [
    (T0, 3600, 197), (-5000, 7, 100), (0, 1, 1), (T0, 1, 1000), (-(1 << 50), 1 << 40, 2000), (T0, 1 << 40, 65536),
    (I64_MAX - 65536 * 3, 3, 65536), (I64_MIN, 1, 1),
])
def test_edge_seconds(origin, width, buckets):
    rng = np.random.default_rng(buckets)
    P = 3
    part, ts, kl, vl, _ = cols_topic(rng, 20_000, P, origin, width, buckets)
    with engine_tl(P, origin, width, buckets) as e:
        scan_cols(e, part, ts, kl, vl)
        e.finalize()
        assert_timeline(e, P, origin, width, buckets, part, ts, kl, vl)


BOUNDARY_CASES = [("30d", True), ("30d", False), ("w999999937", False), ("w2^43-1", True), ("w2^43-1", False),
                  ("w2^38-1", False)]


@pytest.mark.gpu
@pytest.mark.parametrize("name,smem", BOUNDARY_CASES,
                         ids=["%s-%s" % (n, "smem" if s else "global") for n, s in BOUNDARY_CASES])
def test_bucket_boundaries(name, smem):
    """every bucket edge (sampled between the ends for B = 65536) of a range whose quotients need the correction step,
    three seconds at each, at ms 0 and 999, on the given bin path"""
    O, W, B = CORRECTION_RANGES[name][:3]
    P = 3 if smem else max(3, smem_max_bins() // (B + 2) + 1)
    ts = TR.boundary_ms(O, W, B)
    n = ts.size
    rng = np.random.default_rng(B)
    part = rng.integers(0, P, size=n).astype(np.int32)
    kl = rng.integers(-1, 24, size=n).astype(np.int32)
    vl = rng.choice(np.array([-1, 0, 7, 65536], dtype=np.int32), size=n)
    with engine_tl(P, O, W, B) as e:
        assert e.timeline_shape(n)[2] == smem
        scan_cols(e, part, ts, kl, vl)
        e.finalize()
        assert_timeline(e, P, O, W, B, part, ts, kl, vl)


@pytest.mark.gpu
def test_setter_refusals_and_the_largest_range():
    with KtaEngine(2, now=feed.NOW) as e:
        e.set_timeline(I64_MAX - 65536 * 5, 5, 65536)              # ends exactly at INT64_MAX: accepted
        for args in ((I64_MAX - 65536 * 5 + 1, 5, 65536), (0, 0, 1), (0, -1, 1), (0, 1, -1), (0, 1, 65537)):
            with pytest.raises(KtaError) as ex:
                e.set_timeline(*args)
            assert ex.value.code == N.ERR_INVALID
    with KtaEngine(1 << 20, now=feed.NOW) as e:
        e.set_timeline(0, 1, (1 << 24) // (1 << 20) - 2)            # P (B + 2) = 2^24: accepted
        with pytest.raises(KtaError):
            e.set_timeline(0, 1, (1 << 24) // (1 << 20) - 1)


# ---- GPU: warp aggregation, bad and foreign partitions --------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("shape", ["one_bin", "distinct", "alternating", "across_31_0", "tail"])
def test_warp_aggregation(shape):
    P, O, W, B = 64, 0, 10, 40
    n = 128 * 50 + (37 if shape == "tail" else 0)
    i = np.arange(n)
    lane = i % 32
    if shape == "one_bin":
        part, sec = np.full(n, 5), np.full(n, 123)
    elif shape == "distinct":
        part, sec = lane * 2, (lane % 7) * 10 + 3
    elif shape == "alternating":
        part, sec = np.where(i % 2, 3, 9), np.where(i % 2, 15, 395)
    elif shape == "across_31_0":
        g = (lane + 1) // 2 % 16                         # groups {31, 0}, {1, 2}, ... straddle the row boundary
        part, sec = g * 3, np.full(n, 55)
    else:
        part, sec = (i // 300) % P, i // 17
    ts = sec.astype(np.int64) * 1000 + (i % 1000)
    kl = (i % 30 - 1).astype(np.int32)
    vl = np.where(i % 11 == 0, -1, i % 5000).astype(np.int32)
    part = part.astype(np.int32)
    with engine_tl(P, O, W, B) as e:
        scan_cols(e, part, ts, kl, vl)
        e.finalize()
        assert_timeline(e, P, O, W, B, part, ts, kl, vl)


@pytest.mark.gpu
@pytest.mark.parametrize("rank", [0, 1, 2])
def test_bad_and_foreign_partitions(rank):
    rng = np.random.default_rng(rank)
    P, O, W, B = 9, T0, 600, 20
    part, ts, kl, vl, _ = cols_topic(rng, 30_000, P, O, W, B, bad=True)
    with engine_tl(P, O, W, B, shard=(rank, 3)) as e:
        scan_cols(e, part, ts, kl, vl)
        e.finalize(strict=False)
        assert_timeline(e, P, O, W, B, part, ts, kl, vl, shard=(rank, 3))


@pytest.mark.gpu
@pytest.mark.parametrize("P,G,rank", [(65537, 65537, 65536), (1_031_966, 4178, 4177)])
def test_shard_shapes_the_scan_cannot_divide_are_refused(P, G, rank):
    """the scan would put partition P - 1 (65 536) in column 1 instead of 0, or partition 1 031 965 of rank 4177 in the
    wrong column, leaving the handle's own records out as foreign: kta_create refuses both shapes"""
    assert not TR.shard_accepted(P, G)
    with pytest.raises(KtaError) as ex:
        KtaEngine(P, now=feed.NOW, shard=(rank, G)).close()
    assert ex.value.code == N.ERR_INVALID


# accepted shard shapes at the limits: P = 2^20 with G = 4096 (rank 4095 owns partition 2^20 - 1) and G = 4095 (rank
# 4094's largest partition is one below a multiple of G, where (P - 1) e is closest to 2^32); 65 536 partitions over
# 65 536 and 65 535 shards
SHARD_LIMITS = [(1 << 20, 4096, 4095), (1 << 20, 4095, 4094), (65536, 65536, 65535), (65536, 65535, 65534)]


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["counters", "hll", "exact"])
@pytest.mark.parametrize("P,G,rank", SHARD_LIMITS, ids=["P%d-G%d-r%d" % s for s in SHARD_LIMITS])
def test_shard_limit_shapes_count_their_own_partitions(P, G, rank, mode):
    """a handle fed only its own partitions, up to the largest, counts every record: no record is reported out of range,
    and each own partition's counters and timeline row (P (B + 2) <= 2^24) agree with the restatement"""
    assert TR.shard_accepted(P, G)
    O, W, B = T0, 600, 14
    assert P * (B + 2) <= 1 << 24
    own = np.arange(rank, P, G)
    rng = np.random.default_rng(G)
    n = 30_000
    part = rng.choice(own, size=n).astype(np.int32)
    part[: own.size] = own[::-1]                         # every own partition, the largest first
    ts = edge_ms(rng, n, O, W, B)
    kl = rng.integers(-1, 24, size=n).astype(np.int32)
    vl = rng.choice(np.array([-1, 0, 1, 300, 65536], dtype=np.int32), size=n)
    kb = rng.integers(0, 256, size=int(np.maximum(kl, 0).sum()), dtype=np.uint8)
    t = feed.HostTopic(part, np.arange(n, dtype=np.int64), ts, kl, vl, np.arange(n, dtype=np.uint64), kb,
                       feed.tile_base_from_key_len(kl))
    kw = {"counters": {}, "hll": dict(hll_precision=10), "exact": dict(count_alive_keys=True)}[mode]
    with engine_tl(P, O, W, B, shard=(rank, G), **kw) as e:
        feed.scan(e, t)
        assert e.finalize(strict=False) == 0 and e.bad_partition_records() == 0
        # the own partitions renumbered 0 .. len(own) - 1 for the restatement (a whole [3][P][B + 2] would be 400 MB)
        want = TR.timeline_np(own.size, O, W, B, (part - rank) // G, ts, kl, vl)
        got = np.stack([np.stack([e.timeline(w, int(p)) for p in own]) for w in range(3)])
        assert np.array_equal(got, want)
        for j, p in enumerate(own.tolist()):
            mine = part == p
            assert e.counter(M.TOTAL, p) == int(mine.sum()) == int(got[0, j].sum())
            assert e.counter(M.TOMBSTONES, p) == int((vl[mine] < 0).sum()) == int(got[1, j].sum())
            assert (e.counter(M.KEY_SIZE_SUM, p) + e.counter(M.VALUE_SIZE_SUM, p) == int(got[2, j].sum())
                    == int(np.maximum(kl[mine], 0).sum() + np.maximum(vl[mine], 0).sum()))
        for p in (0, rank - 1, P - 1 if (P - 1) % G != rank else P - 2):   # foreign partitions read as zeros
            assert p % G != rank and not e.timeline(0, p).any() and e.counter(M.TOTAL, p) == 0


# ---- GPU: both bin paths, byte carry, depth -------------------------------------------------------------------------
def smem_max_bins():
    return torch.cuda.get_device_properties(0).shared_memory_per_block_optin // 16


@pytest.mark.gpu
def test_both_bin_paths_agree():
    P = 64
    B = smem_max_bins() // P - 2                       # P (B + 2) fits shared memory ...
    rng = np.random.default_rng(3)
    part, ts, kl, vl, _ = cols_topic(rng, 200_000, P, T0, 60, B)
    ts = np.sort(ts)                                  # time-ordered, as a topic is written
    out = []
    for b in (B, B + 1):                              # ... one bucket more is P bins more: global
        with engine_tl(P, T0, 60, b) as e:
            assert e.timeline_shape(len(part))[2] == (b == B)
            scan_cols(e, part, ts, kl, vl)
            e.finalize()
            assert_timeline(e, P, T0, 60, b, part, ts, kl, vl)
            out.append(got_arrays(e, P))
    # the same records: indices 0..B agree, and the wider range splits the first one's "after" index in two
    assert np.array_equal(out[0][:, :, :B + 1], out[1][:, :, :B + 1])
    assert np.array_equal(out[0][:, :, B + 1], out[1][:, :, B + 1] + out[1][:, :, B + 2])


@pytest.mark.gpu
def test_exact_smem_edge_and_many_partitions():
    nb = smem_max_bins()
    for P in (nb // 3, nb // 3 + 1):                     # one bucket: P (B + 2) = 3 P bins, the last that fits and one more
        with engine_tl(P, 0, 1, 1) as e:
            assert e.timeline_shape(1000)[2] == (P * 3 <= nb)
    P = 100_000
    rng = np.random.default_rng(5)
    part, ts, kl, vl, _ = cols_topic(rng, 300_000, P, T0, 3600, 10)
    with engine_tl(P, T0, 3600, 10) as e:
        assert not e.timeline_shape(len(part))[2]
        scan_cols(e, part, ts, kl, vl)
        e.finalize()
        want = TR.timeline_np(P, T0, 3600, 10, part, ts, kl, vl)
        got = got_arrays(e, P)
        assert np.array_equal(got, want)
        assert_invariants(e, P, got)


BYTE_ROWS = [(True, "mixed"), (False, "mixed"), (True, "one_bin"), (False, "one_bin"), (True, "alternating"),
             (False, "alternating")]


@pytest.mark.gpu
@pytest.mark.parametrize("smem,rows", BYTE_ROWS, ids=["%s%s" % (s, "" if r == "mixed" else "-" + r) for s, r in BYTE_ROWS])
def test_bytes_past_2_32_in_one_cta(smem, rows):
    """bins take more than 2^32 bytes from a single CTA (32 full tiles), records of 2^31 - 1 + 20 bytes; lane l reads
    records 4 l .. 4 l + 3.  "mixed": two bins, neighbouring lanes differ, so every row is mixed and in shared memory each
    record's add carries from the low word into the high word (in global memory the group sums are 64-bit).
    "one_bin": every row lies in one bin, so the warp's sum of a row passes 2^36 and its own high word is nonzero.
    "alternating": the first two rows of a tile lie in one bin and the last two alternate between two, so the rows' high
    words and the per-record carries meet in the same bin"""
    P = 64
    B = 4 if smem else smem_max_bins() // P
    n = 128 * 32
    i = np.arange(n)
    part = {"mixed": i // 4 % 2, "one_bin": np.zeros(n, np.int64), "alternating": np.where(i % 4 < 2, 0, i // 4 % 2)}[rows]
    part = part.astype(np.int32)
    ts = np.full(n, (T0 + 5) * 1000, np.int64) + i % 1000
    kl = np.full(n, 20, np.int32)
    vl = np.full(n, (1 << 31) - 1, np.int32)
    with engine_tl(P, T0, 10, B) as e:
        assert e.timeline_shape(n)[0] == 1 and e.timeline_shape(n)[2] == smem
        scan_cols(e, part, ts, kl, vl)
        e.finalize()
        for p in (0, 1):
            assert int(e.timeline(N.TIMELINE_BYTES, p)[1]) == int((part == p).sum()) * ((1 << 31) - 1 + 20)
        assert int(e.timeline(N.TIMELINE_BYTES, 0)[1]) > 1 << 32
        assert_timeline(e, P, T0, 10, B, part, ts, kl, vl)


@pytest.mark.gpu
@pytest.mark.parametrize("smem", [True, False])
@pytest.mark.parametrize("column", ["partition", "ts_ms", "key_len", "value_len", "all"])
def test_full_tiles_row_by_row(column, smem):
    """a column that starts one element past a 16-byte boundary sends every tile, the full ones too, down the row-by-row
    path: each column on its own, then all four.  Half the records are edge timestamps over random partitions (mixed
    rows), half time-ordered runs of one partition (rows in one bin)"""
    P = 64
    B = 40 if smem else smem_max_bins() // P
    rng = np.random.default_rng(17)
    n = 128 * 400
    part, ts, kl, vl, _ = cols_topic(rng, n, P, T0, 60, B)
    i = np.arange(n // 2)
    part[n // 2:] = i // 200 % P
    ts[n // 2:] = T0 * 1000 + i * 71
    names = ("partition", "ts_ms", "key_len", "value_len")
    d = [feed.device(a, shift=1 if column in (name, "all") else 0) for name, a in zip(names, (part, ts, kl, vl))]
    assert sum(c.data_ptr() % 16 != 0 for c in d) == (4 if column == "all" else 1)
    with engine_tl(P, T0, 60, B) as e:
        assert e.timeline_shape(n)[2] == smem
        feed.settle()
        e.scan_batch_device(*d)
        e.finalize()
        assert_timeline(e, P, T0, 60, B, part, ts, kl, vl)


DEPTH_CASES = [(197, "spread"), (20_000, "spread"), (197, "one_bin"), (20_000, "one_bin"), (197, "offset"),
               (20_000, "offset")]


@pytest.mark.gpu
@pytest.mark.parametrize("buckets,layout", DEPTH_CASES,
                         ids=["%d%s" % (b, "" if l == "spread" else "-" + l) for b, l in DEPTH_CASES])
def test_depth(buckets, layout):
    """every warp of the launch takes at least 64 tiles, and the last tile is partial; "one_bin": every record in one
    bin, so every CTA adds to and flushes into the same bins; "offset": every column one element past a 16-byte
    boundary, so every tile is read row by row"""
    P, O, W = 64, T0, 3600
    with engine_tl(P, O, W, buckets) as e:
        grid, threads, _ = e.timeline_shape(1 << 33)     # the full grid
        n = grid * (threads // 32) * 64 * 128 + 77
        assert e.timeline_shape(n)[:2] == (grid, threads)
        ntiles = -(-n // 128)
        assert ntiles // grid // (threads // 32) >= 64
        # built and restated on the device (timeline_torch): the host holds no column of the 3.5e7 records
        i = torch.arange(n, dtype=torch.int64, device="cuda")
        if layout == "one_bin":
            part = torch.full((n,), 5, dtype=torch.int32, device="cuda")
            ts = (T0 + 100) * 1000 + i % 1000
        else:
            part = ((i // 512) % P).to(torch.int32)
            ts = T0 * 1000 + i * 7 + (i * 2654435761 % 5)
        kl = torch.full((n,), 16, dtype=torch.int32, device="cuda")
        vl = torch.where(i % 20 == 0, -1, 100 + i % 300).to(torch.int32)
        del i
        if layout == "offset":
            part, ts, kl, vl = (feed.device(c, shift=1) for c in (part, ts, kl, vl))
        feed.settle()
        e.scan_batch_device(part, ts, kl, vl)
        e.finalize()
        want = TR.timeline_torch(P, O, W, buckets, part, ts, kl, vl).cpu().numpy().astype(np.uint64)
        got = got_arrays(e, P)
        assert np.array_equal(got, want)
        assert_invariants(e, P, got)
        if layout == "one_bin":
            assert int(got[0, 5, 1]) == n and int(got[2, 5, 1]) > 1 << 32


# ---- GPU: merge -----------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_merge_of_four_shards_equals_one_handle():
    rng = np.random.default_rng(9)
    P, O, W, B, G = 12, T0, 300, 40, 4
    part, ts, kl, vl, kb = cols_topic(rng, 40_000, P, O, W, B)
    with engine_tl(P, O, W, B, hll_precision=8) as one:
        scan_cols(one, part, ts, kl, vl, kb)
        one.finalize()
        want = got_arrays(one, P)
    shards = [engine_tl(P, O, W, B, hll_precision=8, shard=(r, G)) for r in range(G)]
    try:
        bufs = []
        for r, e in enumerate(shards):
            scan_cols(e, part, ts, kl, vl, kb)
            words = e.merge_words(G)
            with KtaEngine(P, hll_precision=8, shard=(r, G)) as plain:
                assert words == plain.merge_words(G) + 3 * P * (B + 2)
            b = torch.zeros(words, dtype=torch.int64, device="cuda")
            e.merge_export(r, G, b)
            bufs.append(b)
        total = torch.stack(bufs).sum(0)
        for e in shards:
            e.merge_import(G, total)
            e.finalize(strict=False)
            assert np.array_equal(got_arrays(e, P), want)
            assert_invariants(e, P, want)
    finally:
        for e in shards:
            e.close()


# ---- GPU: lifecycle and non-interference ----------------------------------------------------------------------------
@pytest.mark.gpu
def test_lifecycle():
    P = 3
    with KtaEngine(P, now=feed.NOW) as e:
        with pytest.raises(KtaError) as ex:
            e.timeline(0, 0)
        assert ex.value.code == N.ERR_NOT_ENABLED
        e.set_timeline(T0, 60, 10)
        with pytest.raises(KtaError) as ex:
            e.timeline(0, 0)
        assert ex.value.code == N.ERR_NOT_FINALIZED
        e.push(1, 0, (T0 + 65) * 1000, b"ab", 7)                   # in the ring, not yet scanned
        with pytest.raises(KtaError):
            e.set_timeline(T0, 60, 11)
        e.finalize()
        assert list(e.timeline(0, 1)) == [0, 0, 1] + [0] * 9
        assert list(e.timeline(2, 1)) == [0, 0, 9] + [0] * 9
        assert list(e.timeline(0, 7)) == [0] * 12 and list(e.timeline(0, -1)) == [0] * 12
        short = np.full(4, 99, np.uint64)
        N.check(lib().kta_timeline(e.handle, 0, 1, short.ctypes.data_as(C.POINTER(C.c_uint64)), 2))
        assert list(short) == [0, 0, 99, 99]
        with pytest.raises(KtaError):
            e.set_timeline(T0, 60, 11)                             # after a scan
        e.reset()
        e.push(2, 0, (T0 + 1) * 1000, None, -1)
        e.finalize()
        assert list(e.timeline(0, 1)) == [0] * 12 and list(e.timeline(1, 2)) == [0, 1] + [0] * 10
        e.reset()
        e.set_timeline(0, 1, 0)                                    # off
        e.push(2, 0, 5, None, 3)
        e.finalize()
        with pytest.raises(KtaError) as ex:
            e.timeline(0, 0)
        assert ex.value.code == N.ERR_NOT_ENABLED


@pytest.mark.gpu
@pytest.mark.parametrize("entry", ["device", "host_batch"])
def test_nothing_else_changes(entry):
    """a twin without the timeline gives the same counters, histograms, HLL registers and alive set; launches differ by
    one per counted scan; and the re-runs of a grown alive-key table add no counts"""
    rng = np.random.default_rng(21)
    P, O, W, B = 8, T0, 900, 64
    n = 1 << 20
    part, ts, kl, vl, kb = cols_topic(rng, n, P, O, W, B)
    kl = np.maximum(kl, 4).astype(np.int32)
    kb = rng.integers(0, 256, size=int(kl.sum()), dtype=np.uint8)
    t = feed.HostTopic(part, np.arange(n, dtype=np.int64), ts, kl, vl, np.arange(n, dtype=np.uint64), kb,
                       feed.tile_base_from_key_len(kl))
    res = []
    for on in (False, True):
        e = KtaEngine(P, count_alive_keys=True, hll_precision=12, now=feed.NOW, alive_table_kib=1, ring_records=1 << 18)
        if on:
            e.set_timeline(O, W, B)
        feed.feed(e, t, entry)
        e.finalize()
        launches = e.stats()[0]
        grows, reruns = e.alive_table_stats()[2:]
        assert grows > 0 and reruns > 0
        res.append(dict(
            counters=[[e.counter(w, p) for w in range(7)] for p in range(P)],
            hist=[[e.hist(w, p).tolist() for w in (0, 1)] for p in range(P)],
            regs=e.hll_registers().tolist(), alive=e.alive_keys(), table=[a.tolist() for a in exported(e)],
            launches=launches))
        if on:
            assert_timeline(e, P, O, W, B, part, ts, kl, vl)
        e.close()
    scans = 1 if entry == "device" else -(-n // (1 << 18))
    assert res[1].pop("launches") - res[0].pop("launches") == scans
    assert res[0] == res[1]


# ---- the CLI: --timeline W[,ORIGIN,BUCKETS] -------------------------------------------------------------------------
def _cli():
    from test_report import CLI_DIR, _build
    _build()
    return os.path.join(CLI_DIR, "kafka-topic-analyzer")


@pytest.mark.parametrize("arg,msg", [("0", "W[,ORIGIN,BUCKETS]"), ("-60", "W[,ORIGIN,BUCKETS]"), ("x", "W[,ORIGIN,BUCKETS]"),
                                     ("60,5", "W[,ORIGIN,BUCKETS]"), ("60,0,0", "BUCKETS at least 1"),
                                     ("60,x,3", "ORIGIN must be an integer"), ("1,0,10001", "use a wider W")])
def test_cli_timeline_argument_errors(arg, msg):
    r = subprocess.run([_cli(), "-t", "t", "-b", "x", "--synthetic", "n=1000", "--timeline", arg], capture_output=True, text=True)
    assert r.returncode == 2 and msg in r.stderr and r.stdout == "", r.stderr


def test_cli_timeline_refuses_more_than_10000_derived_buckets():
    """2e7 synthetic records span about 39 hours: 1-second buckets are refused (before any device work), 15-second ones
    are not refused for their number"""
    r = subprocess.run([_cli(), "-t", "t", "-b", "x", "--synthetic", "n=20000000", "--timeline", "1"], capture_output=True, text=True)
    assert r.returncode == 2 and "more than 10000: use a wider W" in r.stderr, r.stderr


def utc(sec):
    return datetime.datetime.fromtimestamp(sec, datetime.timezone.utc).strftime("%Y-%m-%d %H:%M:%S UTC")


def expected_rows(P, origin, width, buckets, part, ts, kl, vl, partitions):
    a = TR.timeline_np(P, origin, width, buckets, part, ts, kl, vl)[:, partitions, :].sum(axis=1)
    rows = []
    for i in range(buckets + 2):
        if a[0, i]:
            start = ("before " + utc(origin) if i == 0 else utc(origin + buckets * width) + " and later" if i == buckets + 1
                     else utc(origin + (i - 1) * width))
            rows.append([start, str(a[0, i]), str(a[1, i]), str(a[2, i])])
    return rows


def cli_rows(out):
    """the timeline's header line and table rows printed after the report"""
    lines = out.splitlines()
    k = next(j for j, l in enumerate(lines) if l.startswith("| extension: timeline"))
    rows = [[c.strip() for c in l.strip("|").split("|")] for l in lines[k + 1:] if l.startswith("|")]
    assert rows[0] == ["Bucket start", "Records", "Tmb", "Bytes"]
    return lines[k], rows[1:], "\n".join(lines[:k])


def report_part(out):
    """the report without the lines that carry the run's duration"""
    return [l for l in out.splitlines() if not l.startswith(("Scanning took", "Estimated Msg/s"))]


@pytest.mark.gpu
@pytest.mark.parametrize("feed_", ["batch", "push", "device"])
def test_cli_timeline_synthetic(feed_):
    from kafka_topic_analyzer_b200 import synth
    P, n, W = 4, 200_000, 60
    args = [_cli(), "-t", "demo", "-b", "x", "--feed", feed_, "--synthetic", "n=%d,partitions=%d,distinct_keys=20000" % (n, P)]
    r = subprocess.run(args + ["--timeline", str(W)], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr
    plain = subprocess.run(args, capture_output=True, text=True, timeout=600)
    assert plain.returncode == 0, plain.stderr
    head, rows, report = cli_rows(r.stdout)
    assert report_part(report + "\n") == report_part(plain.stdout)          # the report itself is unchanged
    t = synth.fill_host(synth.make_spec(n, P, distinct_keys=20_000))
    lo, hi = (min(TR.second(int(t.ts_ms[0])), TR.second(int(t.ts_ms[-1]))), max(TR.second(int(t.ts_ms[0])), TR.second(int(t.ts_ms[-1]))))
    origin = lo // W * W
    buckets = (hi - origin) // W + 1
    assert head == "| extension: timeline, %d buckets of %d s from %s" % (buckets, W, utc(origin))
    assert rows == expected_rows(P, origin, W, buckets, t.partition, t.ts_ms, t.key_len, t.value_len, list(range(P)))
    # an explicit range: records before and after it get their rows
    r = subprocess.run(args + ["--timeline", "%d,%d,%d" % (W, origin + 2 * W, 3)], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr
    _, rows, _ = cli_rows(r.stdout)
    assert rows == expected_rows(P, origin + 2 * W, W, 3, t.partition, t.ts_ms, t.key_len, t.value_len, list(range(P)))
    assert rows[0][0].startswith("before") and rows[-1][0].endswith("and later")


@pytest.mark.gpu
def test_cli_timeline_log_dir(tmp_path):
    """segments of three partitions (partition 1 has no directory) in a broker's data directory; the range from the
    batch headers' baseTimestamp / maxTimestamp, the rows from the delivered records of the report's partitions"""
    rng = np.random.default_rng(4)
    W, recs_all = 30, []
    for p in (0, 2, 3):
        recs = [(T0 * 1000 + 3000 * j + int(rng.integers(0, 2000)) - (600_000 if j % 50 == 7 else 0),
                 None if j % 9 == 0 else b"k%d" % (j % 17), None if j % 6 == 0 else int(rng.integers(0, 500))) for j in range(600)]
        seg = kc.encode_partition(recs, rng, max_batch=25, compression=[None, "gzip", "lz4"])
        d = tmp_path / ("orders-%d" % p)
        d.mkdir()
        (d / "00000000000000000000.log").write_bytes(seg)
        batches = kc.read_segment(seg)
        recs_all += [(p, ts, k, v, b) for b in batches for (_, ts, k, v) in kc.delivered([b])]
    args = [_cli(), "-t", "orders", "-b", "x", "--log-dir", str(tmp_path)]
    r = subprocess.run(args + ["--timeline", str(W)], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr
    plain = subprocess.run(args, capture_output=True, text=True, timeout=600)
    head, rows, report = cli_rows(r.stdout)
    assert report_part(report + "\n") == report_part(plain.stdout)
    secs = [TR.second(x) for b in {id(x[4]): x[4] for x in recs_all}.values() for x in (b.base_ts, b.max_ts)]
    origin = min(secs) // W * W
    buckets = (max(secs) - origin) // W + 1
    assert head == "| extension: timeline, %d buckets of %d s from %s" % (buckets, W, utc(origin))
    part = np.array([x[0] for x in recs_all], np.int32)
    ts = np.array([x[1] for x in recs_all], np.int64)
    kl = np.array([-1 if x[2] is None else len(x[2]) for x in recs_all], np.int32)
    vl = np.array([-1 if x[3] is None else x[3] for x in recs_all], np.int32)
    assert rows == expected_rows(4, origin, W, buckets, part, ts, kl, vl, [0, 2, 3])


# ---- compute-sanitizer --------------------------------------------------------------------------------------------------
SANITIZED_CASE = """
import sys
sys.path.insert(0, {tests!r})
import numpy as np, torch
import timeline_ref as TR
from kafka_topic_analyzer_b200 import KtaEngine
rng = np.random.default_rng(0)
n, P = 5000, 8
part = rng.integers(-1, P + 1, size=n).astype(np.int32)
ts = (1_500_000_000_000 + rng.integers(-100_000, 10_000_000, size=n)).astype(np.int64)
kl = rng.integers(-1, 20, size=n).astype(np.int32)
vl = rng.choice([-1, 0, 9, 1 << 30], size=n).astype(np.int32)
for B in (20, 14528 // P):            # shared-memory bins, then global bins (P (B + 2) > 14528)
    e = KtaEngine(P, now=(4102444800, 0))
    e.set_timeline(1_500_000_000 - 50, 60, B)
    cols = [torch.from_numpy(a).cuda() for a in (part, ts, kl, vl)]
    torch.cuda.synchronize()
    e.scan_batch_device(*cols)
    e.finalize(strict=False)
    got = np.stack([np.stack([e.timeline(w, p) for p in range(P)]) for w in range(3)])
    assert np.array_equal(got, TR.timeline_np(P, 1_500_000_000 - 50, 60, B, part, ts, kl, vl)), B
    e.close()
print("timeline sanitized case ok")
"""


@pytest.mark.gpu
@pytest.mark.parametrize("tool", ["memcheck", "racecheck"])
def test_sanitizer_over_a_small_case(tool):
    here = os.path.dirname(os.path.abspath(__file__))
    san = shutil.which("compute-sanitizer") or os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin", "compute-sanitizer")
    env = dict(os.environ, KTA_NO_BUILD="1", PYTHONPATH=os.path.dirname(here))
    code = SANITIZED_CASE.format(tests=here)
    plain = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, env=env, timeout=600)
    assert plain.returncode == 0 and "ok" in plain.stdout, plain.stdout + plain.stderr
    if not os.path.exists(san):
        pytest.skip("compute-sanitizer not found")
    probe = subprocess.run([san, "--tool", "memcheck", sys.executable, "-c",
                            "from kafka_topic_analyzer_b200 import KtaEngine; KtaEngine(1, device=0).close()"],
                           capture_output=True, text=True, env=env, timeout=300)
    if probe.returncode != 0:   # the sanitizer cannot run CUDA work on this machine (the plain run above has passed)
        pytest.skip("compute-sanitizer cannot create a handle here: " + (probe.stdout + probe.stderr)[-300:])
    r = subprocess.run([san, "--tool", tool, "--error-exitcode", "77", sys.executable, "-c", code], capture_output=True,
                       text=True, env=env, timeout=1800)
    out = r.stdout + r.stderr
    assert r.returncode == 0 and "timeline sanitized case ok" in out, out[-4000:]
    assert "0 errors" in out or "0 hazards" in out or "ERROR SUMMARY: 0" in out, out[-2000:]
