"""Hot keys (include/kta.h, kta_set_hot_keys; csrc/kta_hotkeys.cuh).

CPU: the three restatements of hotkeys_ref.py pinned to each other, the top-K order and truncation, kta_hot_key's size
and offsets against kta.h, and the host's growth policy restated.  GPU: every case compares the whole exported table, entry
by entry after sorting by id, with the restatement fed the delivered records, and the top-K list; it checks that the
records sum to the partitions' KTA_KEY_NON_NULL and the bytes to the counters.  Entry points, log entry points, warp
aggregation, key shapes, growth and its out-of-memory state, import (wrap-around, the empty marker's id, counters past 2^32
and 2^63, refusals), sharded merges, a twin handle without the table, the handle's lifetime, and depth."""
import ctypes as C
import os
import subprocess
import types
import zlib

import numpy as np
import pytest
import torch
from hypothesis import given, settings, strategies as st

import feed
import hotkeys_ref as R
import kafka_codec as kc
import partitioner_ref as PR
from parity import exported
from kafka_topic_analyzer_b200 import KtaEngine, KtaError, lib
from kafka_topic_analyzer_b200 import _native as N
from kafka_topic_analyzer_b200 import metrics as M
from kafka_topic_analyzer_b200 import synth

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
T = N.KTA_KEY_TILE
EDGE_TS = [-1, 0, 999, 1000, -999, -1000, -1001, 1001, (1 << 62), -(1 << 62), 10 ** 12 + 999]


# ---- CPU: the restatements ------------------------------------------------------------------------------------------
def packed(keys):
    kl = np.array([-1 if k is None else len(k) for k in keys], np.int32)
    kb = np.frombuffer(b"".join(k for k in keys if k), np.uint8).copy()
    return kl, kb


@settings(max_examples=80, deadline=None)
@given(st.data())
def test_restatements_agree(data):
    pool = data.draw(st.lists(st.one_of(st.none(), st.binary(min_size=0, max_size=70)), min_size=1, max_size=6))
    n = data.draw(st.integers(1, 60))
    P = data.draw(st.integers(1, 6))
    recs = [(data.draw(st.integers(-1, P)), data.draw(st.sampled_from(pool)), data.draw(st.sampled_from([-1, 0, 5, 300])),
             data.draw(st.sampled_from(EDGE_TS))) for _ in range(n)]
    part = np.array([r[0] for r in recs], np.int32)
    kl, kb = packed([r[1] for r in recs])
    vl = np.array([r[2] for r in recs], np.int32)
    ts = np.array([r[3] for r in recs], np.int64)
    want = R.record_table(P, recs)
    got = R.table_np(P, part, kl, vl, ts, kb)
    assert got.tobytes() == want.tobytes()
    # torch (on the CPU here), from the per-length hashes
    by_len = {}
    for L in set(int(x) for x in kl if x >= 0):
        rows = np.nonzero(kl == L)[0]
        keys = [recs[i][1] for i in rows]
        by_len[L] = (torch.from_numpy(rows), torch.tensor([list(k) for k in keys], dtype=torch.uint8).reshape(len(keys), L))
    ids = R.ids_torch(torch.from_numpy(kl), by_len)
    u, rec, tomb, byt, lat, lo, hi = R.table_torch(P, torch.from_numpy(part), torch.from_numpy(kl), torch.from_numpy(vl),
                                                   torch.from_numpy(ts), ids)
    assert u.numpy().view(np.uint64).tolist() == want["id"].tolist()
    for f, v in (("records", rec), ("tombstones", tomb), ("bytes", byt), ("latest_s", lat), ("min_partition", lo),
                 ("max_partition", hi)):
        assert v.numpy().tolist() == want[f].astype(np.int64).tolist(), f


def test_key_id_is_the_partitioner_checks_hashes():
    for k in (b"", b"21", b"foobar", b"a-little-bit-long-string"):
        assert R.key_id(k) == zlib.crc32(k) << 32 | PR.murmur2(k)
    assert R.key_id(b"123456789") >> 32 == 0xCBF43926


def test_top_order_and_truncation():
    t = np.zeros(6, N.HOT_KEY_DTYPE)
    t["id"] = [9, 3, 7, 1, (1 << 64) - 1, 0]
    t["records"] = [5, 5, 8, 1, 5, 1]
    assert R.top(t, 10)["id"].tolist() == [7, 3, 9, (1 << 64) - 1, 0, 1]
    assert R.top(t, 2)["id"].tolist() == [7, 3]
    assert R.top(t, 0).size == 0


def test_struct_layout_matches_kta_h(tmp_path):
    fields = [f for f, *_ in N.HotKey._fields_]
    src = tmp_path / "layout.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "kta.h"\nint main(void) {\n printf("%zu\\n", sizeof(kta_hot_key));\n' +
                   "".join(' printf("%%zu\\n", offsetof(kta_hot_key, %s));\n' % f for f in fields) + " return 0;\n}\n")
    exe = tmp_path / "layout"
    subprocess.run(["gcc", "-I", os.path.join(ROOT, "include"), "-o", str(exe), str(src)], check=True)
    out = [int(x) for x in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split()]
    assert out[0] == C.sizeof(N.HotKey) == N.HOT_KEY_DTYPE.itemsize == 88
    assert out[1:] == [getattr(N.HotKey, f).offset for f in fields] == [N.HOT_KEY_DTYPE.fields[f][1] for f in fields]


def growth_model(slots, batches, bound=0):
    """kta_api.cu launch_hot_keys restated: (slots, grows, slices) after batches, each a list of ids (None: not counted)"""
    grows = slices = 0
    seen = set()
    for ids in batches:
        n = len(ids)
        ntiles, t = -(-n // T), 0
        while t < ntiles:
            t1 = ntiles
            if bound + (n - t * T) > slots // 2:
                bound = len(seen)
                while bound * 4 > slots or slots // 2 - bound < T:
                    slots, grows = slots * 2, grows + 1
                t1 = min(ntiles, t + (slots // 2 - bound) // T)
            if t1 - t < ntiles:
                slices += 1
            seen.update(i for i in ids[t * T:t1 * T] if i is not None)
            bound += min(n, t1 * T) - t * T
            t = t1
    return slots, grows, slices


def test_growth_model_keeps_the_table_at_most_half_full():
    rng = np.random.default_rng(0)
    for _ in range(200):
        slots = 1 << int(rng.integers(4, 10))
        batches = [list(rng.integers(0, int(rng.integers(1, 5000)), size=int(rng.integers(1, 3000)))) for _ in range(3)]
        final, grows, _ = growth_model(slots, batches)
        assert len(set().union(*map(set, batches))) <= final // 2 and final == slots << grows


def home(i, n):
    """kta_hotkeys.cuh hk_home: the multiply-high of murmur3's fmix64 by n"""
    m = (1 << 64) - 1
    i ^= i >> 33
    i = i * 0xff51afd7ed558ccd & m
    i ^= i >> 33
    i = i * 0xc4ceb9fe1a85ec53 & m
    i ^= i >> 33
    return i * n >> 64


# ---- GPU helpers --------------------------------------------------------------------------------------------------------
def engine_hk(P, top_k=16, slots=0, **kw):
    kw.setdefault("now", feed.NOW)
    e = KtaEngine(P, **kw)
    e.set_hot_keys(top_k, slots)
    return e


def table_of(e):
    """the engine's whole table (kta_hot_keys_export_device), sorted by id"""
    n = e.hot_keys_export_count()
    buf = torch.zeros(max(n, 1) * 88, dtype=torch.uint8, device="cuda")
    feed.settle()
    assert e.hot_keys_export(buf, n) == n
    return R.by_id(buf[:n * 88].cpu().numpy().view(N.HOT_KEY_DTYPE).copy())


def import_entries(e, entries):
    buf = torch.from_numpy(np.ascontiguousarray(entries).view(np.uint8).copy()).cuda()
    feed.settle()
    e.hot_keys_import(buf, len(entries))


def want_of(P, t, shard=None):
    return R.table_np(P, t.partition, t.key_len, t.value_len, t.ts_ms, t.key_bytes, shard=shard)


def first_diff(got, want):
    if got.size != want.size:
        return "entries: got %d, want %d" % (got.size, want.size)
    for i in range(got.size):
        if got[i].tobytes() != want[i].tobytes():
            return "entry %d: got %r, want %r" % (i, got[i], want[i])
    return None


def assert_hot(e, P, want, vsum_keyed=None):
    """whole table, top-K, stats against the counters (after finalize)"""
    got = table_of(e)
    d = first_diff(got, want)
    assert d is None, d
    top = e.hot_keys()
    assert top.tobytes() == R.top(want, e.hot_keys_top_k).tobytes()
    distinct, keyed, slots, grows, slices = e.hot_key_stats()
    assert distinct == want.size and keyed == int(want["records"].sum()) == sum(e.counter(M.KEY_NON_NULL, p) for p in range(P))
    assert distinct <= slots // 2
    key_sum = sum(e.counter(M.KEY_SIZE_SUM, p) for p in range(P))
    if vsum_keyed is not None:
        assert int(want["bytes"].sum()) == key_sum + vsum_keyed
    assert int(want["bytes"].sum()) <= key_sum + sum(e.counter(M.VALUE_SIZE_SUM, p) for p in range(P))
    return distinct, keyed, slots, grows, slices


def keyed_values(t, P):
    ok = (t.key_len >= 0) & (t.partition >= 0) & (t.partition < P)
    return int(np.maximum(t.value_len[ok], 0).astype(np.int64).sum())


def ragged_topic(rng, n, P, max_key=40, bad=False, pool=None):
    part = rng.integers(-2 if bad else 0, P + (2 if bad else 0), size=n).astype(np.int32)
    if pool is None:
        kl = rng.integers(-1, max_key + 1, size=n).astype(np.int32)
        kb = rng.integers(0, 256, size=int(np.maximum(kl, 0).sum()), dtype=np.uint8)
    else:
        keys = [pool[i] for i in rng.integers(0, len(pool), size=n)]
        kl, kb = packed(keys)
    vl = rng.integers(-1, 300, size=n).astype(np.int32)
    ts = rng.choice(np.array(EDGE_TS[:9] + [feed.NOW[0] * 1000 - 5], np.int64), size=n)
    return feed.HostTopic(part, np.arange(n, dtype=np.int64), ts, kl, vl, np.arange(n, dtype=np.uint64), kb,
                          feed.tile_base_from_key_len(kl))


def topic_of(part, keys, vl=None, ts=None):
    kl, kb = packed(keys)
    n = len(keys)
    vl = np.zeros(n, np.int32) if vl is None else np.asarray(vl, np.int32)
    ts = np.zeros(n, np.int64) if ts is None else np.asarray(ts, np.int64)
    return feed.HostTopic(np.asarray(part, np.int32), np.arange(n, dtype=np.int64), ts, kl, vl, np.arange(n, dtype=np.uint64),
                          kb, feed.tile_base_from_key_len(kl))


def ids_of(t, P):
    ids = R.ids_np(t.key_len, t.key_bytes)
    ok = (t.key_len >= 0) & (t.partition >= 0) & (t.partition < P)
    return [int(i) if o else None for i, o in zip(ids, ok)]


# ---- GPU: entry points ----------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["counters", "hll", "exact"])
@pytest.mark.parametrize("entry", ["push", "host_batch", "device", "device_no_tile_base"])
def test_entry_points(entry, mode):
    rng = np.random.default_rng(3)
    P = 6
    pool = [None, b""] + [rng.integers(0, 256, int(rng.integers(0, 41)), dtype=np.uint8).tobytes() for _ in range(3000)]
    t = ragged_topic(rng, 30_000, P, bad=True, pool=pool)
    kw = dict(counters={}, hll=dict(hll_precision=10), exact=dict(count_alive_keys=True))[mode]
    with engine_hk(P, 50, ring_records=4096 if entry == "push" else 8192, **kw) as e:
        feed.feed(e, t, entry)
        assert e.finalize(strict=False) == int(((t.partition < 0) | (t.partition >= P)).sum())
        assert_hot(e, P, want_of(P, t), keyed_values(t, P))


@pytest.mark.gpu
@pytest.mark.parametrize("entry", feed.LOG_ENTRIES)
def test_log_entry_points(entry):
    """every codec, a failed CRC under check.crcs, a window that cuts a batch, and an aborted transaction under
    read_committed: only the delivered keyed records are counted"""
    rng = np.random.default_rng(11)
    P = 4
    codecs = [None, "gzip", "snappy", "snappy-xerial", "lz4", "zstd"]
    parts, delivered = {}, []
    for p in range(P):
        recs = [(10 ** 12 + 7000 * j - (5 * 10 ** 5 if j % 7 == 0 else 0), None if j % 9 == 0 else (b"" if j % 11 == 0 else b"k%d" % (j % 13)),
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
        delivered += [(p, o, k, -1 if v is None else v, ts) for r in recs_by_batch for (o, ts, k, v) in r]
    start3 = kc.read_segment(parts[3][1].raw)[0].base_offset + 1
    delivered = [d for d in delivered if d[0] != 3 or d[1] >= start3]
    want = R.record_table(P, [(p, k, v, ts) for (p, o, k, v, ts) in delivered])
    for mode in ({}, dict(count_alive_keys=True)):
        with engine_hk(P, 7, isolation_level="read_committed", check_crcs=True, **mode) as e:
            e.set_log_offsets(3, start3, None)
            n, _ = feed.scan_log(e, entry, parts)
            e.finalize()
            assert n == len(delivered)
            assert e.log_crc_stats()[1] == 1 and e.log_txn_stats()[0] == 1
            assert_hot(e, P, want)


# ---- GPU: warp aggregation --------------------------------------------------------------------------------------------------
def aggregation_topic(shape, rng):
    n = 32 * 4 * 40 + 77
    if shape == "one_key":
        keys, part = [b"hot"] * n, np.zeros(n, np.int32)
    elif shape == "distinct32":
        keys, part = [b"k%02d" % (i % 32) for i in range(n)], rng.integers(0, 4, size=n)
    elif shape == "alternating":
        keys, part = [(b"a", b"bb")[i % 2] for i in range(n)], rng.integers(0, 4, size=n)
    elif shape == "lanes_31_0":   # a group across lanes 31 and 0 of the next row, others distinct
        keys = [b"edge" if i % 32 in (31, 0) else b"u%d" % i for i in range(n)]
        part = rng.integers(0, 4, size=n)
    elif shape == "partitions_in_a_row":   # one key in several partitions within a row, nulls between
        keys = [None if i % 5 == 0 else b"multi" for i in range(n)]
        part = np.arange(n) % 4
    vl = rng.choice(np.array([-1, 0, 7, 1 << 30], np.int32), size=n)
    ts = rng.choice(np.array(EDGE_TS, np.int64), size=n)
    return topic_of(part, keys, vl, ts)


@pytest.mark.gpu
@pytest.mark.parametrize("shape", ["one_key", "distinct32", "alternating", "lanes_31_0", "partitions_in_a_row"])
def test_warp_aggregation(shape):
    rng = np.random.default_rng(5)
    t = aggregation_topic(shape, rng)
    with engine_hk(4, 40) as e:
        feed.scan(e, t)
        e.finalize()
        assert_hot(e, 4, want_of(4, t), keyed_values(t, 4))


@pytest.mark.gpu
@pytest.mark.parametrize("key_mode", [0, 1, 2])
def test_loguniform_synthetic_keys(key_mode):
    P, n = 8, 1 << 20
    spec = synth.make_spec(n, P, distinct_keys=50_000, key_mode=key_mode, zipf_keys=True, run_len=16)
    h = synth.fill_host(spec)
    with engine_hk(P, 100, slots=1 << 18) as e:
        feed.scan(e, h)
        e.finalize()
        assert_hot(e, P, want_of(P, h), keyed_values(h, P))
        top = e.hot_keys()
        assert top["records"][0] > 4 * top["records"][-1]   # a few hot keys


# ---- GPU: key shapes -----------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("shape", ["k16", "ascii", "ragged", "over_stage", "wide", "all_null_tiles", "empty"])
def test_key_shapes(shape):
    rng = np.random.default_rng(8)
    if shape == "k16":
        keys = [rng.integers(0, 256, 16, dtype=np.uint8).tobytes() for _ in range(500)] * 20
    elif shape == "ascii":
        keys = [b"user-%d" % int(i) for i in rng.integers(0, 3000, size=20000)]
    elif shape == "ragged":
        pool = [rng.integers(0, 256, int(rng.integers(0, 41)), dtype=np.uint8).tobytes() for _ in range(2000)]
        keys = [pool[i] for i in rng.integers(0, 2000, size=20000)]
    elif shape == "over_stage":   # tiles whose key spans exceed the stage (hashed from global memory) next to short ones
        keys = [rng.integers(0, 256, int(rng.integers(200, 400)), dtype=np.uint8).tobytes() for _ in range(60)] * 10 + \
               [b"s%d" % i for i in range(3000)]
    elif shape == "wide":
        big = rng.integers(0, 256, (1 << 20) + 1, dtype=np.uint8).tobytes()
        keys = [big, big[:-2], b"x", big, None, big[:(1 << 20) - 1]] + [b"y"] * 200
    elif shape == "all_null_tiles":
        keys = [None] * (3 * T) + [b"a", b"b"] * T + [None] * (5 * T + 3)
    elif shape == "empty":
        keys = [b"" if i % 3 else None for i in range(5000)]
    n = len(keys)
    t = topic_of(rng.integers(0, 5, size=n), keys, rng.integers(-1, 100, size=n), rng.integers(0, 10 ** 13, size=n))
    with engine_hk(5, 64) as e:
        feed.scan(e, t)
        e.finalize()
        want = want_of(5, t)
        assert_hot(e, 5, want, keyed_values(t, 5))
        if shape == "wide":
            top = e.hot_keys(as_dicts=True)
            assert top[1]["key_len"] == (1 << 20) + 1 and top[1]["key_prefix"] == big[:32]


# ---- GPU: growth ---------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("case", ["doublings", "exact_room", "one_more", "few_distinct"])
def test_growth(case):
    rng = np.random.default_rng(13)
    if case == "doublings":
        slots, keys = 16, [b"d%d" % i for i in rng.permutation(40_000)]
    elif case == "exact_room":
        slots, keys = 1024, [b"r%d" % i for i in range(512)]
    elif case == "one_more":
        slots, keys = 1024, [b"r%d" % i for i in range(513)]
    else:
        slots, keys = 1024, [b"f%d" % (i % 10) for i in range(10_000)]
    t = topic_of(rng.integers(0, 3, size=len(keys)), keys)
    with engine_hk(3, 20, slots=slots) as e:
        feed.scan(e, t)
        e.finalize()
        _, _, got_slots, grows, slices = assert_hot(e, 3, want_of(3, t), 0)
    assert (got_slots, grows, slices) == growth_model(slots, [ids_of(t, 3)])
    want = {"doublings": lambda: grows >= 10 and slices >= 10, "exact_room": lambda: grows == 0 and slices == 0,
            "one_more": lambda: grows == 1 and slices == 2, "few_distinct": lambda: grows == 0 and slices > 1}[case]
    assert want(), (grows, slices)


@pytest.mark.gpu
def test_out_of_memory_then_reset():
    rng = np.random.default_rng(14)
    P = 4
    t = topic_of(rng.integers(0, P, size=5000), [b"m%d" % i for i in range(5000)], rng.integers(-1, 50, size=5000))
    with engine_hk(P, 8, slots=16, hll_precision=10) as e:
        e.hot_keys_limit_slots(256)
        with pytest.raises(KtaError) as ex:
            feed.scan(e, t)
        assert ex.value.code == N.ERR_NOMEM and "hot-key table" in str(ex.value)
        e.finalize()   # reported once; every other metric counted the batch
        assert sum(e.counter(M.TOTAL, p) for p in range(P)) == 5000
        for p in range(P):
            assert e.counter(M.KEY_NON_NULL, p) == int((t.partition == p).sum())
        for call in (e.hot_keys, e.hot_key_stats, e.hot_keys_export_count):
            with pytest.raises(KtaError) as ex:
                call()
            assert ex.value.code == N.ERR_NOMEM
        e.reset()
        small = topic_of(np.zeros(50, np.int32), [b"s%d" % (i % 7) for i in range(50)])
        feed.scan(e, small)
        e.finalize()
        assert_hot(e, P, want_of(P, small), 0)


# ---- GPU: import ------------------------------------------------------------------------------------------------------------------
def entry(i, records, p=(0, 0), key=b"", tomb=0, byt=0, latest=0, reserved=0, key_len=None):
    e = np.zeros(1, N.HOT_KEY_DTYPE)
    e["id"], e["records"], e["tombstones"], e["bytes"], e["latest_s"] = i, records, tomb, byt, latest
    e["min_partition"], e["max_partition"] = p
    e["key_len"] = len(key) if key_len is None else key_len
    e["reserved"] = reserved
    e["key_prefix"][0, :min(len(key), 32)] = np.frombuffer(key[:32], np.uint8)
    return e


@pytest.mark.gpu
def test_import_wraps_and_keeps_the_empty_marker():
    slots = 16
    ids = [i for i in range(1, 200000) if home(i, slots) == slots - 1][:3]
    assert len(ids) == 3
    es = np.concatenate([entry(i, 2, (1, 2), b"w%d" % i, tomb=1, byt=9, latest=-5) for i in ids] +
                        [entry(0, 3, (0, 3), b"zero", latest=7)])
    with engine_hk(4, 10, slots=slots) as e:
        import_entries(e, es)
        import_entries(e, es[:2])
        e.finalize()
        got = table_of(e)
        want = R.by_id(np.concatenate([es, es[:2]]))
        assert got["id"].tolist() == sorted(set(want["id"].tolist()))
        g = {int(x["id"]): x for x in got}
        assert int(g[0]["records"]) == 3 and bytes(g[0]["key_prefix"][:4]) == b"zero"
        assert int(g[ids[0]]["records"]) == 4 and int(g[ids[0]]["tombstones"]) == 2 and int(g[ids[2]]["records"]) == 2
        assert e.hot_key_stats()[0] == 4 and e.hot_keys()["id"].tolist() == [ids[0], ids[1], 0, ids[2]]


@pytest.mark.gpu
def test_import_counters_carry_past_2_32_and_2_63():
    key = b"carry"
    P = 3
    seed = entry(R.key_id(key), (1 << 32) - 1, (1, 1), key, tomb=(1 << 32) - 2, byt=(1 << 63) - 3, latest=-(1 << 40))
    n = 300
    t = topic_of(np.full(n, 2, np.int32), [key] * n, np.full(n, -1, np.int32), np.full(n, 5000, np.int64))
    with engine_hk(P, 4) as e:
        import_entries(e, seed)
        feed.scan(e, t)
        e.finalize(strict=False)
        got = table_of(e)
    assert got.size == 1
    assert int(got["records"][0]) == (1 << 32) - 1 + n and int(got["tombstones"][0]) == (1 << 32) - 2 + n
    assert int(got["bytes"][0]) == (1 << 63) - 3 + n * len(key)
    assert int(got["latest_s"][0]) == 5 and (int(got["min_partition"][0]), int(got["max_partition"][0])) == (1, 2)


@pytest.mark.gpu
@pytest.mark.parametrize("bad", ["records0", "tombstones", "key_len", "reserved", "pmin", "pmax", "range"])
def test_import_refusals_apply_nothing(bad):
    good = entry(R.key_id(b"g"), 2, (0, 1), b"g")
    e_ = dict(records0=entry(5, 0), tombstones=entry(5, 1, tomb=2), key_len=entry(5, 1, key_len=-1),
              reserved=entry(5, 1, reserved=1), pmin=entry(5, 1, (-1, 0)), pmax=entry(5, 1, (0, 3)), range=entry(5, 1, (2, 1)))[bad]
    with engine_hk(3, 4) as e:
        import_entries(e, good)
        with pytest.raises(KtaError) as ex:
            import_entries(e, np.concatenate([good, e_]))
        assert ex.value.code == N.ERR_INVALID
        e.finalize()
        assert table_of(e).tobytes() == good.tobytes()


# ---- GPU: merges, twin handle, lifecycle --------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_merge_of_four_shards_equals_one_handle():
    rng = np.random.default_rng(9)
    P, G = 12, 4
    pool = [None] + [b"s%d" % i for i in range(4000)]
    t = ragged_topic(rng, 40_000, P, bad=True, pool=pool)
    want = want_of(P, t)
    shards = [engine_hk(P, 30, slots=1 << 12, shard=(r, G)) for r in range(G)]
    try:
        bufs = []
        for r, e in enumerate(shards):
            feed.scan(e, t)
            e.finalize(strict=False)
            assert table_of(e).tobytes() == want_of(P, t, shard=(r, G)).tobytes()
            n = e.hot_keys_export_count()
            b = torch.zeros(max(n, 1) * 88, dtype=torch.uint8, device="cuda")
            feed.settle()
            assert e.hot_keys_export(b, n) == n
            bufs.append((b, n))
        for r, e in enumerate(shards):
            for q, (b, n) in enumerate(bufs):
                if q != r and n:
                    e.hot_keys_import(b, n)
            e.finalize(strict=False)
            got = table_of(e)
            assert got[["id", "records", "tombstones", "bytes", "latest_s", "min_partition", "max_partition", "key_len"]].tobytes() == \
                want[["id", "records", "tombstones", "bytes", "latest_s", "min_partition", "max_partition", "key_len"]].tobytes()
            assert e.hot_keys().tobytes() == R.top(want, 30).tobytes()
    finally:
        for e in shards:
            e.close()


@pytest.mark.gpu
@pytest.mark.parametrize("entry_", ["device", "host_batch"])
def test_twin_handle_without_the_table(entry_):
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
            e.set_hot_keys(100, 1 << 22)
        feed.feed(e, t, entry_)
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
            assert assert_hot(e, P, want_of(P, t), keyed_values(t, P))[3:] == (0, 0)
        e.close()
    scans = 1 if entry_ == "device" else -(-n // (1 << 18))
    assert res[1].pop("launches") - res[0].pop("launches") == scans + 4   # the passes; export, sort keys, sort, gather
    assert res[0] == res[1]


@pytest.mark.gpu
def test_setter_refusals_reset_and_lifetime():
    with KtaEngine(4, now=feed.NOW) as e:
        with pytest.raises(KtaError) as ex:
            e.hot_keys()
        assert ex.value.code == N.ERR_NOT_ENABLED
        for k, s in ((-1, 0), (N.HOT_KEYS_MAX + 1, 0), (1, 8), (1, 17), (1, (1 << 31) + 1), (1, 1 << 32), (1, -16)):
            assert lib().kta_set_hot_keys(e.handle, k, s) == N.ERR_INVALID, (k, s)
        e.set_hot_keys(3, 64)
        assert lib().kta_set_hot_keys(e.handle, 3, 100) == N.ERR_INVALID
        with pytest.raises(KtaError) as ex:
            e.hot_keys()
        assert ex.value.code == N.ERR_NOT_FINALIZED
        e.push(1, 0, 2500, b"ab", 3)   # in the ring, not yet scanned
        with pytest.raises(KtaError):
            e.set_hot_keys(5)
        e.push(2, 0, -1, b"ab", -1)
        e.push(3, 0, 0, None, 1)
        e.push(0, 0, 0, b"", 1)
        e.finalize()
        top = e.hot_keys(as_dicts=True)
        assert [d["key_prefix"] for d in top] == [b"ab", b""]
        assert top[0]["records"] == 2 and top[0]["tombstones"] == 1 and top[0]["bytes"] == 7 and top[0]["latest_s"] == 2
        assert (top[0]["min_partition"], top[0]["max_partition"]) == (1, 2)
        assert e.hot_key_stats()[:3] == (2, 3, 64)
        e.reset()
        assert e.hot_keys_export_count() == 0
        e.push(1, 0, 0, b"q", 1)
        e.finalize()
        assert [d["key_prefix"] for d in e.hot_keys(as_dicts=True)] == [b"q"] and e.hot_key_stats()[2] == 64
        e.reset()
        e.set_hot_keys(0)
        e.push(1, 0, 0, b"k", 1)
        e.finalize()
        with pytest.raises(KtaError) as ex:
            e.hot_keys()
        assert ex.value.code == N.ERR_NOT_ENABLED


@pytest.mark.gpu
def test_batch_without_key_bytes_is_refused():
    kl = np.array([3, -1, 0], np.int32)
    z32, z64 = np.zeros(3, np.int32), np.zeros(3, np.int64)
    with engine_hk(2, 4) as e:
        with pytest.raises(KtaError) as ex:
            e.push_batch_host(z32, z64, kl, z32)
        assert ex.value.code == N.ERR_INVALID
        with pytest.raises(KtaError) as ex:
            e.scan_batch_device(*[torch.from_numpy(a).cuda() for a in (z32, z64, kl, z32)])
        assert ex.value.code == N.ERR_INVALID
        e.push_batch_host(z32, z64, np.array([-1, 0, -1], np.int32), z32)
        e.finalize()
        assert e.hot_keys()["id"].tolist() == [R.key_id(b"")] and e.stats()[1] == 3


# ---- GPU: depth --------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_depth():
    """one launch in which every warp takes at least 64 tiles, against the torch restatement on the device"""
    P = 16
    props = torch.cuda.get_device_properties(0)
    warps = props.multi_processor_count * 2 * 16            # two CTAs of 16 warps per SM (hot_keys_kernel's bounds)
    n = warps * 64 * T + 1024   # (a multiple of P * run_len)
    spec = synth.make_spec(n, P, distinct_keys=2_000_000, run_len=4)
    torch.cuda.empty_cache()   # the table takes 12 GiB: what earlier tests left in torch's cache goes back first
    topic = synth.DeviceTopic(spec, device=0)
    with engine_hk(P, 1000, slots=1 << 27) as e:
        feed.settle()
        e.scan_batch_device(topic.partition, topic.ts_ms, topic.key_len, topic.value_len, key_bytes=topic.key_bytes,
                            key_bytes_len=topic.key_bytes_len, key_tile_base=topic.key_tile_base)
        e.finalize()
        assert e.hot_key_stats()[3:] == (0, 0)
        got = table_of(e)
        kl = topic.key_len
        rows = torch.nonzero(kl >= 0).squeeze(1)
        assert bool((kl[rows] == 16).all())
        keys = topic.key_bytes[:rows.numel() * 16].view(-1, 16)
        ids = R.ids_torch(kl, {16: (rows, keys)})
        u, rec, tomb, byt, lat, lo, hi = R.table_torch(P, topic.partition, kl, topic.value_len, topic.ts_ms, ids)
        assert np.array_equal(got["id"], u.cpu().numpy().view(np.uint64))
        for f, v in (("records", rec), ("tombstones", tomb), ("bytes", byt), ("latest_s", lat), ("min_partition", lo),
                     ("max_partition", hi)):
            assert np.array_equal(got[f].astype(np.int64), v.cpu().numpy()), f
        assert int(rec.sum()) == sum(e.counter(M.KEY_NON_NULL, p) for p in range(P))
        top = e.hot_keys()
        assert top.tobytes() == R.top(got, 1000).tobytes()
    del topic
    torch.cuda.empty_cache()


# ---- CPU: the CLI -----------------------------------------------------------------------------------------------------------
def _cli_dir():
    from test_report import CLI_DIR, _build
    _build()
    return CLI_DIR


GOLDEN_INPUT = ("7 4\n500 3 12000 1700000000 2 2 5 6b65792d31\n500 0 9 0 0 63 0 -\n"
                "12 12 999 -1 1 3 40 000102030405060708090a0b0c0d0e0f101112131415161718191a1b1c1d1e1f\n"
                "3 0 300 86399 4 4 33 " + "6b" * 32 + "\n")


@pytest.mark.parametrize("arg", ["0", "-3", "x", "65537", "1.5", ""])
def test_cli_hot_keys_argument_errors(arg):
    r = subprocess.run([os.path.join(_cli_dir(), "kafka-topic-analyzer"), "-t", "t", "-b", "x", "--synthetic", "n=1000",
                        "--hot-keys", arg], capture_output=True, text=True)
    assert r.returncode == 2 and "--hot-keys takes K" in r.stderr and r.stdout == "", r.stderr


def test_hot_keys_report_golden():
    """text, empty, hex and long keys, a partition range, a second before the epoch"""
    out = subprocess.run([os.path.join(_cli_dir(), "hot_keys_golden")], input=GOLDEN_INPUT, text=True, capture_output=True,
                         check=True).stdout
    assert out == open(os.path.join(HERE, "golden", "hot_keys_report.txt"), encoding="utf-8").read()


def render_key(prefix, key_len):
    """kta_report.hpp render_key restated"""
    if key_len == 0:
        return "(empty)"
    s = prefix.decode("latin1") if all(0x20 <= c < 0x7F for c in prefix) else "0x" + prefix.hex()
    return s + ("…" if key_len > len(prefix) else "")


def cli_rows(want, k):
    import datetime
    rows = []
    for i, e in enumerate(R.top(want, k)):
        lo, hi = int(e["min_partition"]), int(e["max_partition"])
        kl = int(e["key_len"])
        when = datetime.datetime.fromtimestamp(int(e["latest_s"]), datetime.timezone.utc).strftime("%Y-%m-%d %H:%M:%S UTC")
        rows.append([str(i + 1), str(int(e["records"])), str(int(e["tombstones"])), str(int(e["bytes"])),
                     str(lo) if lo == hi else "%d–%d" % (lo, hi), when, render_key(bytes(e["key_prefix"][:min(kl, 32)]), kl)])
    return rows


def cli_hot(out):
    lines = out.splitlines()
    k = next(j for j, l in enumerate(lines) if l.startswith("| extension: hot keys"))
    rows = [[c.strip() for c in l.strip("|").split("|")] for l in lines[k + 2:] if l.startswith("|")]
    return lines[k + 1], rows, "\n".join(lines[:k])


def report_part(out):
    return [l for l in out.splitlines() if not l.startswith(("Scanning took", "Estimated Msg/s"))]


# ---- GPU: the CLI -----------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("feed_", ["batch", "push", "device"])
@pytest.mark.parametrize("key_mode", [0, 1])
def test_cli_synthetic(feed_, key_mode):
    P, n, K = 4, 100_000, 12
    args = [os.path.join(_cli_dir(), "kafka-topic-analyzer"), "-t", "demo", "-b", "x", "--feed", feed_, "--synthetic",
            "n=%d,partitions=%d,distinct_keys=20000,key_mode=%d" % (n, P, key_mode)]
    r = subprocess.run(args + ["--hot-keys", str(K)], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr
    plain = subprocess.run(args, capture_output=True, text=True, timeout=600)
    distinct, rows, report = cli_hot(r.stdout)
    assert report_part(report + "\n") == report_part(plain.stdout)   # without the flag the output is the same
    t = synth.fill_host(synth.make_spec(n, P, distinct_keys=20_000, key_mode=key_mode))
    want = want_of(P, t)
    assert distinct == "Distinct keys: %d (by 64-bit id)" % want.size
    assert rows[0] == ["#", "Records", "Tombstones", "Bytes", "Partitions", "Latest write", "Key"]
    assert rows[1:] == cli_rows(want, K)


@pytest.mark.gpu
def test_cli_log_dir(tmp_path):
    rng = np.random.default_rng(4)
    recs_all = []
    for p in (0, 2, 3):
        keys = [None if j % 9 == 0 else (b"" if j % 10 == 0 else b"k%d" % (j % 17)) for j in range(300)]
        keys[5] = bytes(range(40))
        recs = [(10 ** 12 + 3000 * j, k, None if j % 7 == 0 else int(rng.integers(0, 500))) for j, k in enumerate(keys)]
        seg = kc.encode_partition(recs, rng, max_batch=25, compression=[None, "gzip", "lz4"])
        d = tmp_path / ("orders-%d" % p)
        d.mkdir()
        (d / "00000000000000000000.log").write_bytes(seg)
        recs_all += [(p, k, -1 if v is None else v, ts) for (_, ts, k, v) in kc.delivered(seg)]
    args = [os.path.join(_cli_dir(), "kafka-topic-analyzer"), "-t", "orders", "-b", "x", "--log-dir", str(tmp_path)]
    r = subprocess.run(args + ["--hot-keys", "30"], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr
    distinct, rows, _ = cli_hot(r.stdout)
    want = R.record_table(4, recs_all)
    assert distinct == "Distinct keys: %d (by 64-bit id)" % want.size
    assert rows[1:] == cli_rows(want, 30)


# ---- GPU: the multi-GPU helper --------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_allgather_hot_keys_as_rank_0_of_2(monkeypatch):
    """distributed.allgather_hot_keys on rank 0 of a two-rank world, the collectives standing in for rank 1's engine:
    its count and entries land where the helper slices them"""
    import torch.distributed as dist
    from kafka_topic_analyzer_b200 import distributed
    rng = np.random.default_rng(31)
    P = 6
    pool = [None, b""] + [b"g%d" % i for i in range(700)]
    t = ragged_topic(rng, 8000, P, pool=pool)
    half = np.arange(8000) < 3000
    with engine_hk(P, 20) as e0, engine_hk(P, 20) as e1:
        feed.scan(e0, feed.take(t, np.nonzero(half)[0]))
        feed.scan(e1, feed.take(t, np.nonzero(~half)[0]))
        n1 = e1.hot_keys_export_count()

        def all_reduce(x, op=None, group=None):
            x[1] += n1

        def all_gather_into_tensor(out, inp, group=None):
            cap = inp.numel()
            out[:cap].copy_(inp)
            assert e1.hot_keys_export(out[cap:], cap // N.HOT_KEY_DTYPE.itemsize) == n1
            feed.settle()

        monkeypatch.setattr(dist, "get_world_size", lambda group=None: 2)
        monkeypatch.setattr(dist, "get_rank", lambda group=None: 0)
        monkeypatch.setattr(dist, "all_reduce", all_reduce)
        monkeypatch.setattr(dist, "all_gather_into_tensor", all_gather_into_tensor)
        distributed.allgather_hot_keys(e0)
        e0.finalize()
        want = want_of(P, t)
        assert table_of(e0)[["id", "records", "tombstones", "bytes", "latest_s", "min_partition", "max_partition"]].tobytes() == \
            want[["id", "records", "tombstones", "bytes", "latest_s", "min_partition", "max_partition"]].tobytes()
        assert e0.hot_keys()["id"].tolist() == R.top(want, 20)["id"].tolist()


# ---- compute-sanitizer ------------------------------------------------------------------------------------------------------
SANITIZED_CASE = """
import sys
sys.path.insert(0, {tests!r})
import numpy as np, torch
import hotkeys_ref as R
from kafka_topic_analyzer_b200 import KtaEngine
from kafka_topic_analyzer_b200._native import HOT_KEY_DTYPE
rng = np.random.default_rng(0)
n, P = 5000, 8
part = rng.integers(-1, P + 1, size=n).astype(np.int32)
kl = rng.integers(-1, 40, size=n).astype(np.int32)
kl[::3] = 3
kb = rng.integers(0, 4, size=int(np.maximum(kl, 0).sum()), dtype=np.uint8)
vl = rng.integers(-1, 100, size=n).astype(np.int32)
ts = rng.integers(-5000, 5000, size=n).astype(np.int64)
e = KtaEngine(P, now=(4102444800, 0))
e.set_hot_keys(10, 16)                # grows through several rehashes
cols = [torch.from_numpy(a).cuda() for a in (part, ts, kl, vl)]
kbd = torch.from_numpy(kb).cuda()
torch.cuda.synchronize()
e.scan_batch_device(*cols, key_bytes=kbd, key_bytes_len=kb.size)
e.finalize(strict=False)
m = e.hot_keys_export_count()
buf = torch.zeros(m * 88, dtype=torch.uint8, device="cuda")
e.hot_keys_export(buf, m)
e.hot_keys_import(buf, m)             # every entry once more
e.finalize(strict=False)
want = R.table_np(P, part, kl, vl, ts, kb)
got = e.hot_keys()
top = R.top(want, 10)
assert got["id"].tolist() == top["id"].tolist() and (got["records"] == 2 * top["records"]).all()
e.close()
print("hot keys sanitized case ok")
"""


@pytest.mark.gpu
@pytest.mark.parametrize("tool", ["memcheck", "racecheck"])
def test_sanitizer_over_a_small_case(tool):
    import shutil
    import sys
    san = shutil.which("compute-sanitizer") or os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin", "compute-sanitizer")
    env = dict(os.environ, KTA_NO_BUILD="1", PYTHONPATH=ROOT)
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
    assert r.returncode == 0 and "hot keys sanitized case ok" in out, out[-4000:]
