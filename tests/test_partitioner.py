"""The partitioner check (include/kta.h, kta_set_partitioner_check; csrc/kta_partitioner.cuh).

CPU: the restatements (partitioner_ref.py) against Kafka's published murmur2 vectors, zlib's CRC-32 check value and
each other; the kernel's modulus restated; the merge segment of distributed.py; the CLI's argument errors and the
report golden.  GPU: the device hash functions value for value, per-record verdicts, every entry point, placed and grown
topics, a twin handle with the check off, partition handling and sharded merges, both counter paths at their edges and at
depth, refusals, the handle's lifetime, the CLI, and compute-sanitizer."""
import ctypes as C
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
import partitioner_ref as R
from parity import exported
from kafka_topic_analyzer_b200 import KtaEngine, KtaError, lib, distributed
from kafka_topic_analyzer_b200 import _native as N
from kafka_topic_analyzer_b200 import metrics as M

HERE = os.path.dirname(os.path.abspath(__file__))
N_EDGES = [1, 2, 3, 7, 12, 24, 64, 100, 255, 256, 1 << 16, (1 << 16) + 1, 999_999_937, (1 << 30), (1 << 31) - 2, (1 << 31) - 1]


# ---- CPU: the restatements --------------------------------------------------------------------------------------------
KAFKA_MURMUR2 = [(b"21", -973932308), (b"foobar", -790332482), (b"a-little-bit-long-string", -985981536),
                 (b"a-little-bit-longer-string", -1486304829),
                 (b"lkjh234lh9fiuh90y23oiuhsafujhadof229phr9h19h89h8", -58897971), (b"abc", 479470107)]


@pytest.mark.parametrize("key,want", KAFKA_MURMUR2)
def test_murmur2_kafka_vectors(key, want):
    """Kafka's UtilsTest.testMurmur2"""
    assert R.signed(R.murmur2(key)) == want
    kl = np.array([len(key)], np.int32)
    assert R.signed(int(R.murmur2_np(kl, np.frombuffer(key, np.uint8))[0])) == want
    assert R.signed(int(R.hashes_torch(torch.tensor([list(key)], dtype=torch.uint8))[0][0])) == want


def test_crc32_check_value():
    assert R.crc32(b"123456789") == 0xCBF43926 and R.crc32(b"") == 0
    assert int(R.crc32_np(np.array([9], np.int32), np.frombuffer(b"123456789", np.uint8))[0]) == 0xCBF43926
    assert int(R.hashes_torch(torch.tensor([list(b"123456789")], dtype=torch.uint8))[1][0]) == 0xCBF43926


@settings(max_examples=60, deadline=None)
@given(st.data())
def test_numpy_and_torch_match_record_at_a_time(data):
    lens = data.draw(st.lists(st.integers(-1, 70), min_size=1, max_size=40))
    keys = [None if L < 0 else bytes(data.draw(st.lists(st.integers(0, 255), min_size=L, max_size=L))) for L in lens]
    kl = np.array(lens, np.int32)
    kb = np.frombuffer(b"".join(k for k in keys if k), np.uint8)
    mm, cc = R.murmur2_np(kl, kb), R.crc32_np(kl, kb)
    for i, k in enumerate(keys):
        assert int(mm[i]) == (0 if k is None else R.murmur2(k)) and int(cc[i]) == (0 if k is None else R.crc32(k))
    for L in set(x for x in lens if x >= 0):
        same = [k for k in keys if k is not None and len(k) == L]
        h, c = R.hashes_torch(torch.tensor([list(k) for k in same], dtype=torch.uint8).reshape(len(same), L))
        assert h.tolist() == [R.murmur2(k) for k in same] and c.tolist() == [R.crc32(k) for k in same]
    counts = data.draw(st.lists(st.sampled_from(N_EDGES), min_size=1, max_size=8, unique=True))
    P = data.draw(st.integers(1, 30))
    part = np.array([data.draw(st.integers(-1, P)) for _ in lens], np.int32)
    want = R.record_counts(P, counts, list(zip(part.tolist(), keys)))
    assert np.array_equal(R.counts_np(P, counts, part, kl, kb), want)
    t = R.counts_torch(P, counts, torch.from_numpy(part).long(), torch.from_numpy(kl).long(),
                       torch.from_numpy(mm.astype(np.int64)), torch.from_numpy(cc.astype(np.int64)))
    assert np.array_equal(t.numpy().astype(np.uint64), want)


def kernel_mod(x, N_):
    """pc_mod (csrc/kta_partitioner.cuh): c = floor((2^64 - 1) / N) + 1 mod 2^64, the high word of (c x mod 2^64) N"""
    c = ((1 << 64) - 1) // N_ + 1 & ((1 << 64) - 1)
    return ((c * x & ((1 << 64) - 1)) * N_) >> 64


@settings(max_examples=400, deadline=None)
@given(st.one_of(st.integers(0, (1 << 32) - 1), st.sampled_from([0, 1, (1 << 31) - 1, 1 << 31, (1 << 32) - 1, (1 << 32) - 2])),
       st.one_of(st.integers(1, (1 << 31) - 1), st.sampled_from(N_EDGES)))
def test_kernel_modulus_is_exact(x, N_):
    assert kernel_mod(x, N_) == x % N_


def test_kernel_modulus_at_the_edges():
    for N_ in N_EDGES + [3 * 5 * 7 * 11 * 13 * 17 * 19 * 23]:
        for q in (0, 1, 2, ((1 << 32) - 1) // N_ - 1, ((1 << 32) - 1) // N_):
            for d in (-1, 0, 1, N_ - 1):
                x = q * N_ + d
                if 0 <= x < 1 << 32:
                    assert kernel_mod(x, N_) == x % N_, (x, N_)


@pytest.mark.parametrize("world", [1, 3])
def test_merge_buffer_partitioner_segment(world):
    rng = np.random.default_rng(world)
    nsums, nhll, tw, pw = 37, 64, 3 * 5 * 7, 5 * 9
    assert distributed.merge_words(nsums, nhll, world, tw, pw) == distributed.merge_words(nsums, nhll, world) + tw + pw
    pts, tls, bufs = [], [], []
    for r in range(world):
        pt = rng.integers(0, 1 << 40, size=(5, 9)).astype(np.uint64)
        tl = rng.integers(0, 1 << 40, size=(3, 5, 7)).astype(np.uint64)
        pts.append(pt)
        tls.append(tl)
        sums = rng.integers(0, 1000, size=nsums).astype(np.uint64)
        hll = rng.integers(0, 20, size=nhll).astype(np.uint8)
        with_tl = distributed.pack_merge_buffer(sums, (5, 9, 1, 2), hll, r, world, timeline=tl)
        b = distributed.pack_merge_buffer(sums, (5, 9, 1, 2), hll, r, world, timeline=tl, partitioner=pt)
        assert np.array_equal(b[:with_tl.size], with_tl) and b.size == with_tl.size + pw
        only = distributed.pack_merge_buffer(sums, (5, 9, 1, 2), hll, r, world, partitioner=pt)
        assert np.array_equal(only[-pw:], pt.ravel())
        bufs.append(b)
    total = np.sum(bufs, axis=0, dtype=np.uint64)
    out = distributed.fold_merge_buffer(total, nsums, nhll, world, timeline_words=tw, partitioner_words=pw)
    assert len(out) == 5
    assert np.array_equal(out[3], np.sum(tls, axis=0, dtype=np.uint64).ravel())
    assert np.array_equal(out[4], np.sum(pts, axis=0, dtype=np.uint64).ravel())
    assert len(distributed.fold_merge_buffer(total, nsums, nhll, world, timeline_words=tw)) == 4


# ---- CPU: the CLI -------------------------------------------------------------------------------------------------------
def _cli_dir():
    from test_report import CLI_DIR, _build
    _build()
    return CLI_DIR


@pytest.mark.parametrize("arg,msg", [("0", "N[,N...]"), ("-3", "N[,N...]"), ("x", "N[,N...]"), ("12,", "N[,N...]"),
                                     ("2147483648", "N[,N...]"), ("12,24,12", "given twice"),
                                     ("1,2,3,4,5,6,7,8,9", "more than 8")])
def test_cli_partitioner_check_argument_errors(arg, msg):
    r = subprocess.run([os.path.join(_cli_dir(), "kafka-topic-analyzer"), "-t", "t", "-b", "x", "--synthetic", "n=1000",
                        "--partitioner-check", arg], capture_output=True, text=True)
    assert r.returncode == 2 and msg in r.stderr and r.stdout == "", r.stderr


def test_partitioner_report_golden():
    out = subprocess.run([os.path.join(_cli_dir(), "partitioner_golden")], input="2 12 24\n3\n0 10 4 6 5 5 0\n1 7 7 0 0 7 0\n2 0 0 0 0 0 0\n",
                         text=True, capture_output=True, check=True).stdout
    assert out == open(os.path.join(HERE, "golden", "partitioner_report.txt")).read()


# ---- GPU helpers --------------------------------------------------------------------------------------------------------
def engine_pc(P, counts, **kw):
    kw.setdefault("now", feed.NOW)
    e = KtaEngine(P, **kw)
    e.set_partitioner_check(counts)
    return e


def got(e, P):
    return np.stack([e.partitioner_check(p) for p in range(P)], axis=1)


def assert_counts(e, P, counts, part, kl, kb, shard=None):
    want = R.counts_np(P, counts, part, kl, kb, shard=shard)
    g = got(e, P)
    if not np.array_equal(g, want):
        b, p = (int(x[0]) for x in np.nonzero(g != want))
        raise AssertionError("counter %d, partition %d: got %d, want %d" % (b, p, g[b, p], want[b, p]))
    for p in range(P):   # no counter exceeds the partition's keyed records
        assert int(g[:, p].max(initial=0)) <= e.counter(M.KEY_NON_NULL, p)


def ragged_topic(rng, n, P, max_key=40, bad=False):
    part = rng.integers(-2 if bad else 0, P + (2 if bad else 0), size=n).astype(np.int32)
    kl = rng.integers(-1, max_key + 1, size=n).astype(np.int32)
    vl = rng.integers(-1, 300, size=n).astype(np.int32)
    ts = (feed.NOW[0] * 1000 - rng.integers(0, 10 ** 9, size=n)).astype(np.int64)
    kb = rng.integers(0, 256, size=int(np.maximum(kl, 0).sum()), dtype=np.uint8)
    return feed.HostTopic(part, np.arange(n, dtype=np.int64), ts, kl, vl, np.arange(n, dtype=np.uint64), kb,
                          feed.tile_base_from_key_len(kl))


def packed(keys):
    kl = np.array([-1 if k is None else len(k) for k in keys], np.int32)
    kb = np.frombuffer(b"".join(k for k in keys if k), np.uint8).copy()
    return kl, kb


def scan_keys(e, part, keys):
    kl, kb = packed(keys)
    n = len(keys)
    t = feed.HostTopic(np.asarray(part, np.int32), np.arange(n, dtype=np.int64), np.zeros(n, np.int64), kl,
                       np.zeros(n, np.int32), np.arange(n, dtype=np.uint64), kb, feed.tile_base_from_key_len(kl))
    feed.scan(e, t)
    return kl, kb


# ---- GPU: the device hash functions --------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_device_hashes_every_length_and_alignment():
    rng = np.random.default_rng(1)
    lens = list(range(71)) + list(range(4093, 4100)) + [(1 << 20) - 1, (1 << 20) + 1]
    keys, off = [], 0
    for L in lens:
        for a in range(16):
            pad = (a - off) % 16
            if pad:                                    # a filler key that moves the next one to offset a (mod 16)
                keys.append(rng.integers(0, 256, pad, dtype=np.uint8).tobytes())
                off += pad
            keys.append(rng.integers(0, 256, L, dtype=np.uint8).tobytes())
            off += L
    keys.append(None)
    kl, kb = packed(keys)
    with KtaEngine(1, now=feed.NOW) as e:
        mm, cc = e.partitioner_hashes(kl, kb)
    assert np.array_equal(mm, R.murmur2_np(kl, kb)) and np.array_equal(cc, R.crc32_np(kl, kb))
    for i in list(range(0, len(keys), 97)) + [len(keys) - 2]:
        if keys[i] is not None:
            assert int(mm[i]) == R.murmur2(keys[i]) and int(cc[i]) == R.crc32(keys[i])
    assert mm[-1] == 0 and cc[-1] == 0


# ---- GPU: counter widths ----------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("path", ["smem", "global"])
def test_counters_carry_past_2_32(path):
    """every counter is seeded a little below 2^32 (and one partition's at 2^40 - 1) through the merge import, then a scan
    adds more than the headroom wherever it adds anything: the pass's adds (the shared-memory flush, or the global REDs)
    must carry into the high word"""
    rng = np.random.default_rng(12)
    P, counts = (16, [16, 8, 5]) if path == "smem" else (smem_limit_P(3) + 1, [16, 8, 5])
    nv = 2 * len(counts) + 1
    part = np.repeat(np.arange(P, dtype=np.int32), 200)               # rows of one partition and mixed rows
    part = np.concatenate([part, rng.integers(0, P, size=20 * P).astype(np.int32)])
    keys = [b""] * (P // 2) + [rng.integers(0, 256, int(rng.integers(0, 24)), dtype=np.uint8).tobytes()
                               for _ in range(part.size - P // 2)]
    kl, kb = packed(keys)
    add = R.counts_np(P, counts, part, kl, kb)
    seed = np.where(add > 0, (1 << 32) - np.maximum(add // 2, 1), (1 << 32) - 1).astype(np.uint64)
    seed[:, 1] = (1 << 40) - 1
    assert ((add + seed >= np.uint64(1 << 32)) & (seed < np.uint64(1 << 32))).sum() >= P - 1   # every neither counter at least
    with engine_pc(P, counts) as e:
        assert e.partitioner_shape(part.size, kb.size)[2] == (path == "smem")
        words = e.merge_words(1)
        buf = torch.zeros(words, dtype=torch.int64, device="cuda")
        e.merge_export(0, 1, buf)
        buf[words - nv * P:] = torch.from_numpy(seed.ravel().view(np.int64)).cuda()
        feed.settle()
        e.merge_import(1, buf)
        scan_keys(e, part, keys)
        e.finalize()
        assert np.array_equal(got(e, P), seed + add)


@pytest.mark.gpu
def test_one_cta_at_its_tile_cap():
    """one CTA takes 2^24 tiles (2^31 empty keys of partition 0): its u32 shared-memory counters reach 2^31 and are
    flushed exactly; one tile more raises the grid to two CTAs"""
    n, counts = 1 << 31, [1, 2]
    torch.cuda.empty_cache()
    with engine_pc(2, counts) as e:
        e.partitioner_limit_grid(1)
        assert e.partitioner_shape(n, 0) == (1, e.partitioner_shape(n, 0)[1], True)
        assert e.partitioner_shape(n + N.KTA_KEY_TILE, 0)[0] == 2
        zeros = torch.zeros(n, dtype=torch.int32, device="cuda")      # partition 0, empty key, empty value
        ts = torch.zeros(n, dtype=torch.int64, device="cuda")
        feed.settle()
        e.scan_batch_device(zeros, ts, zeros, zeros)
        e.finalize()
        assert e.counter(M.KEY_NON_NULL, 0) == n
        assert e.partitioner_check(0).tolist() == [n * int(b) for b in R.verdict(b"", 0, counts)]
        assert e.partitioner_check(1).tolist() == [0] * 5
        del zeros, ts
    torch.cuda.empty_cache()


# ---- GPU: per-record verdicts --------------------------------------------------------------------------------------------
def high_bit_keys(rng, n):
    """n keys, most of them with bit 31 of their murmur2 or CRC-32 set"""
    out = []
    while len(out) < n:
        k = rng.integers(0, 256, int(rng.integers(0, 24)), dtype=np.uint8).tobytes()
        if (R.murmur2(k) | R.crc32(k)) & 0x80000000 or rng.random() < 0.1:
            out.append(k)
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("P", [1, 3, 1000, 100_000])
def test_one_record_per_partition(P):
    rng = np.random.default_rng(P)
    counts = sorted({1, 2, 3, P, 1 << 10, (1 << 31) - 1, P + 1, 2 * P + 7})[:8]
    n = min(P, 20_000) if P > 20_000 else P
    parts = np.sort(rng.choice(P, size=n, replace=False)).astype(np.int32)
    keys = high_bit_keys(rng, n)
    with engine_pc(P, counts) as e:
        kl, kb = scan_keys(e, parts, keys)
        e.finalize()
        g = got(e, P)
    for i, (p, k) in enumerate(zip(parts.tolist(), keys)):
        assert g[:, p].tolist() == [int(b) for b in R.verdict(k, p, counts)], (p, k)
    assert np.array_equal(g, R.counts_np(P, counts, parts, kl, kb))


# ---- GPU: entry points ----------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["counters", "hll", "exact"])
@pytest.mark.parametrize("entry", ["push", "host_batch", "device", "device_no_tile_base"])
def test_entry_points(entry, mode):
    rng = np.random.default_rng(3)
    P, counts = 6, [6, 12, 1]
    t = ragged_topic(rng, 30_000, P, bad=True)
    kw = dict(counters={}, hll=dict(hll_precision=10), exact=dict(count_alive_keys=True))[mode]
    with engine_pc(P, counts, ring_records=4096 if entry == "push" else 8192, **kw) as e:
        feed.feed(e, t, entry)
        assert e.finalize(strict=False) == int(((t.partition < 0) | (t.partition >= P)).sum())
        assert_counts(e, P, counts, t.partition, t.key_len, t.key_bytes)


@pytest.mark.gpu
@pytest.mark.parametrize("entry", feed.LOG_ENTRIES)
def test_log_entry_points(entry):
    """every codec, a failed CRC under check.crcs, a window that cuts a batch, and an aborted transaction under
    read_committed: only the delivered keyed records are checked"""
    rng = np.random.default_rng(11)
    P, counts = 4, [4, 8]
    codecs = [None, "gzip", "snappy", "snappy-xerial", "lz4", "zstd"]
    parts, delivered = {}, []
    for p in range(P):
        recs = [(10 ** 12 + 7000 * j, None if j % 9 == 0 else (b"" if j % 11 == 0 else b"k%d" % (j % 13)),
                 None if j % 5 == 0 else int(rng.integers(0, 300))) for j in range(240)]
        seg = kc.set_crcs(kc.encode_partition(recs, rng, max_batch=30, compression=codecs))
        batches = kc.split_batches(seg)
        keep = [True] * len(batches)
        if p == 1:
            b = bytearray(batches[2]); b[17:21] = b"\xde\xad\xbe\xef"; batches[2] = bytes(b); keep[2] = False
        recs_by_batch = [kc.delivered(b) if k else [] for b, k in zip(batches, keep)]
        raws = list(batches)
        if p == 2:
            end = max(o for r in recs_by_batch for o, *_ in r) + 1
            raws.append(kc.set_crcs(kc.txn_batch(end, 10 ** 12, [(0, 5, b"x", 10), (1, 6, b"yy", None)], pid=7)))
            raws.append(kc.set_crcs(kc.marker(end + 2, 7, 0, False, 10 ** 12)))
        parts[p] = [types.SimpleNamespace(p=p, raw=r) for r in raws]
        delivered += [(p, k) for r in recs_by_batch for (_, ts, k, v) in r]
    start3 = kc.read_segment(parts[3][1].raw)[0].base_offset + 1
    rec3 = [(o, k) for b in parts[3] for (o, ts, k, v) in kc.delivered(b.raw)]
    delivered = [d for d in delivered if d[0] != 3] + [(3, k) for (o, k) in rec3 if o >= start3]
    for mode in ({}, dict(count_alive_keys=True)):
        with engine_pc(P, counts, isolation_level="read_committed", check_crcs=True, **mode) as e:
            e.set_log_offsets(3, start3, None)
            n, _ = feed.scan_log(e, entry, parts)
            e.finalize()
            assert n == len(delivered)
            assert e.log_crc_stats()[1] == 1 and e.log_txn_stats()[0] == 1
            assert np.array_equal(got(e, P), R.record_counts(P, counts, delivered))


# ---- GPU: placed and grown topics ---------------------------------------------------------------------------------------
def ascii_keys(n, rng):
    return [b"user-%d-%s" % (i, b"x" * int(rng.integers(0, 30))) for i in range(n)]


@pytest.mark.gpu
@pytest.mark.parametrize("fn", ["murmur2", "crc32"])
def test_placed_topic(fn):
    rng = np.random.default_rng(5)
    P, counts = 24, [12, 24, 48]
    keys = ascii_keys(60_000, rng) + [b""] * 7
    parts = np.array(R.place(keys, P, fn), np.int32)
    with engine_pc(P, counts, hll_precision=8) as e:
        kl, kb = scan_keys(e, parts, keys)
        e.finalize()
        g = got(e, P)
        col = 1 if fn == "murmur2" else len(counts) + 1
        for p in range(P):
            assert int(g[col, p]) == e.counter(M.KEY_NON_NULL, p) and int(g[-1, p]) == 0
    assert np.array_equal(g, R.counts_np(P, counts, parts, kl, kb))


@pytest.mark.gpu
def test_grown_topic_splits_between_the_murmur2_columns():
    """keys written at 12 partitions, then (other keys and some of the same) at 24"""
    rng = np.random.default_rng(6)
    keys_old, keys_new = ascii_keys(40_000, rng), ascii_keys(60_000, rng)[20_000:] + ascii_keys(5_000, rng)
    parts = np.array(R.place(keys_old, 12, "murmur2") + R.place(keys_new, 24, "murmur2"), np.int32)
    keys = keys_old + keys_new
    with engine_pc(24, [12, 24]) as e:
        kl, kb = scan_keys(e, parts, keys)
        e.finalize()
        g = got(e, 24)
    old_hits = np.bincount(parts[:40_000], minlength=24)
    assert np.array_equal(g, R.counts_np(24, [12, 24], parts, kl, kb))
    assert (g[0] >= old_hits).all() and int(g[4].sum()) == 0   # every old record matches murmur2@12; nothing is neither
    assert int(g[0].sum() + g[1].sum()) >= len(keys)


# ---- GPU: the twin handle -------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("entry", ["device", "host_batch"])
def test_nothing_else_changes(entry):
    rng = np.random.default_rng(21)
    P, n = 8, 1 << 20
    t = ragged_topic(rng, n, P)
    kl = np.maximum(t.key_len, 4).astype(np.int32)
    kb = rng.integers(0, 256, size=int(kl.sum()), dtype=np.uint8)
    t = feed.HostTopic(t.partition, t.offset, t.ts_ms, kl, t.value_len, t.seq, kb, feed.tile_base_from_key_len(kl))
    res = []
    for on in (False, True):
        e = KtaEngine(P, count_alive_keys=True, hll_precision=12, now=feed.NOW, alive_table_kib=1, ring_records=1 << 18)
        if on:
            e.set_partitioner_check([8, 16])
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
            assert_counts(e, P, [8, 16], t.partition, kl, kb)
        e.close()
    scans = 1 if entry == "device" else -(-n // (1 << 18))
    assert res[1].pop("launches") - res[0].pop("launches") == scans
    assert res[0] == res[1]


# ---- GPU: partition handling ----------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_merge_of_four_shards_equals_one_handle():
    rng = np.random.default_rng(9)
    P, G, counts = 12, 4, [12, 6]
    t = ragged_topic(rng, 40_000, P, bad=True)
    with engine_pc(P, counts, hll_precision=8) as one:
        feed.scan(one, t)
        one.finalize(strict=False)
        want = got(one, P)
    assert np.array_equal(want, R.counts_np(P, counts, t.partition, t.key_len, t.key_bytes))
    shards = [engine_pc(P, counts, hll_precision=8, shard=(r, G)) for r in range(G)]
    try:
        bufs = []
        for r, e in enumerate(shards):
            feed.scan(e, t)
            e.finalize(strict=False)
            assert np.array_equal(got(e, P), R.counts_np(P, counts, t.partition, t.key_len, t.key_bytes, shard=(r, G)))
            words = e.merge_words(G)
            with KtaEngine(P, hll_precision=8, shard=(r, G)) as plain:
                assert words == plain.merge_words(G) + (2 * len(counts) + 1) * P
            b = torch.zeros(words, dtype=torch.int64, device="cuda")
            e.merge_export(r, G, b)
            bufs.append(b)
        total = torch.stack(bufs).sum(0)
        for e in shards:
            e.merge_import(G, total)
            e.finalize(strict=False)
            assert np.array_equal(got(e, P), want)
    finally:
        for e in shards:
            e.close()


# ---- GPU: counter paths, stage edges, depth --------------------------------------------------------------------------------
def smem_limit_P(C_):
    """the largest P whose (2C + 1) P counters the handle keeps in shared memory"""
    lo, hi = 1, 1 << 20
    while lo < hi:
        mid = (lo + hi + 1) // 2
        with engine_pc(mid, list(range(1, C_ + 1))) as e:
            smem = e.partitioner_shape(1, 0)[2]
        lo, hi = (mid, hi) if smem else (lo, mid - 1)
    return lo


@pytest.mark.gpu
@pytest.mark.parametrize("C_", [1, 8])
def test_counter_path_edge(C_):
    """the last P with shared-memory counters and the next one, on a topic whose rows mix partitions"""
    Pl = smem_limit_P(C_)
    counts = list(range(1, C_ + 1))
    rng = np.random.default_rng(C_)
    for P, smem in ((Pl, True), (Pl + 1, False)):
        t = ragged_topic(rng, 200_000, P)
        with engine_pc(P, counts) as e:
            assert e.partitioner_shape(t.partition.size, t.key_bytes.size)[2] == smem
            feed.scan(e, t)
            e.finalize()
            assert_counts(e, P, counts, t.partition, t.key_len, t.key_bytes)


@pytest.mark.gpu
@pytest.mark.parametrize("shape", ["fixed16", "long_ragged", "over_stage", "wide_key", "uniform_rows"])
def test_key_spans(shape):
    """staged and unstaged tiles: 16-byte keys, ragged keys up to 300 bytes (spans past the stage), keys of 1 MiB and
    more (64-bit offsets) and fetch-shaped rows of one partition"""
    rng = np.random.default_rng(len(shape))
    P, counts, n = 16, [16, 8, 3], 40_000
    part = rng.integers(0, P, size=n).astype(np.int32)
    if shape == "fixed16":
        kl = np.full(n, 16, np.int32)
    elif shape == "long_ragged":
        kl = rng.integers(-1, 301, size=n).astype(np.int32)
    elif shape == "over_stage":
        kl = rng.integers(100, 200, size=n).astype(np.int32)
    elif shape == "wide_key":
        n = 1000
        part, kl = part[:n], rng.integers(-1, 20, size=n).astype(np.int32)
        kl[[3, 130, 500]] = [1 << 20, (1 << 20) + 1, (1 << 21) + 3]
    else:
        part = np.repeat(np.arange(P, dtype=np.int32), n // P)
        kl = rng.integers(0, 30, size=n).astype(np.int32)
    kb = rng.integers(0, 256, size=int(np.maximum(kl, 0).sum()), dtype=np.uint8)
    t = feed.HostTopic(part, np.arange(n, dtype=np.int64), np.zeros(n, np.int64), kl, np.zeros(n, np.int32),
                       np.arange(n, dtype=np.uint64), kb, feed.tile_base_from_key_len(kl))
    for Pe in (P, smem_limit_P(3) + 1 if shape == "uniform_rows" else P):
        with engine_pc(Pe, counts) as e:
            feed.scan(e, t)
            e.finalize()
            assert_counts(e, Pe, counts, part, kl, kb)


@pytest.mark.gpu
@pytest.mark.parametrize("path", ["smem", "global"])
def test_depth(path):
    """every warp of the grid takes at least 64 tiles; compared with the torch restatement on the device"""
    P, counts = (64, [64, 32, 7]) if path == "smem" else (6000, [6000, 3000, 128, 7, 1, 2, 3, (1 << 31) - 1])
    with engine_pc(P, counts) as e:
        grid, _, smem = e.partitioner_shape(1 << 30, 16 << 30)
        assert smem == (path == "smem")
        n = grid * 16 * 64 * 128
        grid2, _, _ = e.partitioner_shape(n, 16 * n)
        assert grid2 * 16 * 64 * 128 <= n
        g = torch.Generator(device="cuda").manual_seed(1)
        part = torch.randint(0, P, (n,), device="cuda", dtype=torch.int32, generator=g)
        keys = torch.randint(0, 256, (n, 16), device="cuda", dtype=torch.uint8, generator=g)
        kl = torch.full((n,), 16, device="cuda", dtype=torch.int32)
        z = torch.zeros(n, device="cuda", dtype=torch.int64)
        feed.settle()
        e.scan_batch_device(part, z, kl, kl, key_bytes=keys.reshape(-1), key_bytes_len=16 * n)
        e.finalize()
        mm, cc = R.hashes_torch(keys)
        want = R.counts_torch(P, counts, part.long(), kl.long(), mm, cc).cpu().numpy().astype(np.uint64)
        del keys, mm, cc
        assert np.array_equal(got(e, P), want)


# ---- GPU: refusals and lifetime --------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_setter_refusals():
    with KtaEngine(4, now=feed.NOW) as e:
        for bad in ([0], [-1], [-(1 << 31)], [3, 3], [1, 2, 1], list(range(1, 10))):
            assert lib().kta_set_partitioner_check(e.handle, (C.c_int32 * len(bad))(*bad), len(bad)) == N.ERR_INVALID
        assert lib().kta_set_partitioner_check(e.handle, None, 1) == N.ERR_INVALID
        assert lib().kta_set_partitioner_check(e.handle, None, -1) == N.ERR_INVALID
        for bad in ([(1 << 32) + 5], [1 << 31], [0]):                # refused in Python before ctypes could wrap them
            with pytest.raises(KtaError) as ex:
                e.set_partitioner_check(bad)
            assert ex.value.code == N.ERR_INVALID
        e.set_partitioner_check([4, 8])
        assert lib().kta_set_partitioner_check(e.handle, (C.c_int32 * 2)(5, 5), 2) == N.ERR_INVALID
        assert e.partitioner_shape(1, 0)[0] >= 1          # the failed call kept the configuration
        e.push(1, 0, 0, b"ab", 3)                            # in the ring, not yet scanned
        with pytest.raises(KtaError):
            e.set_partitioner_check([4])
        e.finalize()
        assert e.partitioner_check(1).tolist() == [int(b) for b in R.verdict(b"ab", 1, [4, 8])]


@pytest.mark.gpu
def test_batch_without_key_bytes_is_refused():
    kl = np.array([3, -1, 0], np.int32)
    z32, z64 = np.zeros(3, np.int32), np.zeros(3, np.int64)
    with engine_pc(2, [2]) as e:
        with pytest.raises(KtaError) as ex:
            e.push_batch_host(z32, z64, kl, z32)
        assert ex.value.code == N.ERR_INVALID
        with pytest.raises(KtaError) as ex:
            e.scan_batch_device(*[torch.from_numpy(a).cuda() for a in (z32, z64, kl, z32)])
        assert ex.value.code == N.ERR_INVALID
        e.push_batch_host(z32, z64, np.array([-1, 0, -1], np.int32), z32)   # null and empty keys need no bytes
        e.finalize()
        assert e.partitioner_check(0).tolist() == [int(b) for b in R.verdict(b"", 0, [2])]
        assert e.stats()[1] == 3


@pytest.mark.gpu
def test_lifetime():
    with KtaEngine(3, now=feed.NOW) as e:
        with pytest.raises(KtaError) as ex:
            e.partitioner_check(0)
        assert ex.value.code == N.ERR_NOT_ENABLED
        e.set_partitioner_check([3, 1])
        with pytest.raises(KtaError) as ex:
            e.partitioner_check(0)
        assert ex.value.code == N.ERR_NOT_FINALIZED
        e.push(2, 0, 0, b"key", 1)
        e.finalize()
        assert e.partitioner_check(2).tolist() == [int(b) for b in R.verdict(b"key", 2, [3, 1])]
        assert e.partitioner_check(7).tolist() == [0] * 5 and e.partitioner_check(-1).tolist() == [0] * 5
        short = np.full(4, 99, np.uint64)
        N.check(lib().kta_partitioner_check(e.handle, 2, short.ctypes.data_as(C.POINTER(C.c_uint64)), 2))
        assert short.tolist()[2:] == [99, 99]
        e.reset()
        e.push(1, 0, 0, None, 1)
        e.finalize()
        assert got(e, 3).sum() == 0
        e.reset()
        e.set_partitioner_check([])
        e.push(1, 0, 0, b"k", 1)
        e.finalize()
        with pytest.raises(KtaError) as ex:
            e.partitioner_check(0)
        assert ex.value.code == N.ERR_NOT_ENABLED


# ---- GPU: the CLI ---------------------------------------------------------------------------------------------------------
def cli_table(out):
    lines = out.splitlines()
    k = next(j for j, l in enumerate(lines) if l.startswith("| extension: partitioner check"))
    rows = [[c.strip() for c in l.strip("|").split("|")] for l in lines[k + 1:] if l.startswith("|")]
    return lines[k], rows, "\n".join(lines[:k])


def report_part(out):
    return [l for l in out.splitlines() if not l.startswith(("Scanning took", "Estimated Msg/s"))]


@pytest.mark.gpu
@pytest.mark.parametrize("feed_", ["batch", "push", "device"])
def test_cli_synthetic(feed_):
    from kafka_topic_analyzer_b200 import synth
    P, n = 4, 100_000
    args = [os.path.join(_cli_dir(), "kafka-topic-analyzer"), "-t", "demo", "-b", "x", "--feed", feed_, "--synthetic",
            "n=%d,partitions=%d,distinct_keys=20000" % (n, P)]
    r = subprocess.run(args + ["--partitioner-check", "4,2"], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr
    plain = subprocess.run(args, capture_output=True, text=True, timeout=600)
    head, rows, report = cli_table(r.stdout)
    assert report_part(report + "\n") == report_part(plain.stdout)
    assert rows[0] == ["P", "Keyed", "murmur2@4", "murmur2@2", "crc32@4", "crc32@2", "Neither"]
    t = synth.fill_host(synth.make_spec(n, P, distinct_keys=20_000))
    want = R.counts_np(P, [4, 2], t.partition, t.key_len, t.key_bytes)
    keyed = np.bincount(t.partition[t.key_len >= 0], minlength=P)
    for p in range(P):
        assert rows[1 + p] == [str(p), str(keyed[p])] + [str(v) for v in want[:, p]]
    assert rows[-1] == ["total", str(keyed.sum())] + [str(v) for v in want.sum(axis=1)]


@pytest.mark.gpu
def test_cli_log_dir(tmp_path):
    rng = np.random.default_rng(4)
    recs_all = []
    for p in (0, 2, 3):
        keys = [None if j % 9 == 0 else b"k%d" % (j % 17) for j in range(300)]
        recs = [(10 ** 12 + 3000 * j, k, int(rng.integers(0, 500))) for j, k in enumerate(keys)]
        seg = kc.encode_partition(recs, rng, max_batch=25, compression=[None, "gzip", "lz4"])
        d = tmp_path / ("orders-%d" % p)
        d.mkdir()
        (d / "00000000000000000000.log").write_bytes(seg)
        recs_all += [(p, k) for (_, ts, k, v) in kc.delivered(seg)]
    args = [os.path.join(_cli_dir(), "kafka-topic-analyzer"), "-t", "orders", "-b", "x", "--log-dir", str(tmp_path)]
    r = subprocess.run(args + ["--partitioner-check", "4"], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr
    _, rows, _ = cli_table(r.stdout)
    want = R.record_counts(4, [4], recs_all)
    assert [row[0] for row in rows[1:]] == ["0", "2", "3", "total"]
    for row, p in zip(rows[1:4], (0, 2, 3)):
        assert row[2:] == [str(v) for v in want[:, p]]


# ---- compute-sanitizer --------------------------------------------------------------------------------------------------
SANITIZED_CASE = """
import sys
sys.path.insert(0, {tests!r})
import numpy as np, torch
import partitioner_ref as R
from kafka_topic_analyzer_b200 import KtaEngine
rng = np.random.default_rng(0)
n = 5000
for P, C in ((8, 3), (4000, 8)):      # shared-memory counters, then global counters
    counts = list(range(P, P + C))
    part = rng.integers(-1, P + 1, size=n).astype(np.int32)
    kl = rng.integers(-1, 40, size=n).astype(np.int32)
    kb = rng.integers(0, 256, size=int(np.maximum(kl, 0).sum()), dtype=np.uint8)
    e = KtaEngine(P, now=(4102444800, 0))
    e.set_partitioner_check(counts)
    z = np.zeros(n, np.int32)
    cols = [torch.from_numpy(a).cuda() for a in (part, z.astype(np.int64), kl, z)]
    kbd = torch.from_numpy(kb).cuda()
    torch.cuda.synchronize()
    e.scan_batch_device(*cols, key_bytes=kbd, key_bytes_len=kb.size)
    e.finalize(strict=False)
    assert e.partitioner_shape(n, kb.size)[2] == (P == 8)
    got = np.stack([e.partitioner_check(p) for p in range(P)], axis=1)
    assert np.array_equal(got, R.counts_np(P, counts, part, kl, kb)), P
    e.close()
print("partitioner sanitized case ok")
"""


@pytest.mark.gpu
@pytest.mark.parametrize("tool", ["memcheck", "racecheck"])
def test_sanitizer_over_a_small_case(tool):
    san = shutil.which("compute-sanitizer") or os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin", "compute-sanitizer")
    env = dict(os.environ, KTA_NO_BUILD="1", PYTHONPATH=os.path.dirname(HERE))
    code = SANITIZED_CASE.format(tests=HERE)
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
    assert r.returncode == 0 and "partitioner sanitized case ok" in out, out[-4000:]
