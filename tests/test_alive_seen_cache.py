"""Exact alive keys (-c) with the seen cache on: every batch here has at least 2^20 records, so it goes through the
32 MiB cache of (mixed hash -> newest wave) before the table (ALIVE_CACHE_MIN_RECORDS, csrc/kta_api.cu).

Every GPU case checks the whole table, entry by entry, not just the alive count:
  * the exported (reference hash, (seq + 1) << 1 | alive) pairs equal an independent last-writer map of the records;
  * the report matches the C oracle fed in seq order, HLL registers of the alive set included;
  * the table holds exactly one entry per distinct hash.
Keys are crafted where a case needs a chosen mixed hash x = fmix32(fnv32(key)): the same cache set, the table's empty
pattern, or a run of consecutive x that share a home pair at every table size."""
import numpy as np
import pytest

from kafka_topic_analyzer_b200 import KtaError, synth
from kafka_topic_analyzer_b200.synth import HostTopic, tile_base_from_key_len
from feed import (MASK32, NOW, alive_import, engine, fmix32, gather, keys_for_mixed, last_writer_map, push_host, scan, settle,
                  take, unmix32)
from oracle_lib import Oracle, fnv32, olib
from parity import assert_parity, assert_same_map, exported
import np_oracle

HLL_P = 12                      # feed.engine's
P = 8                           # feed.engine's default
M20 = 1 << 20


# ------------------------------------------------------------------------------------------------
# topics
# ------------------------------------------------------------------------------------------------
def pool_topic(rng, ids, pool, alive):
    """Records whose key is pool[ids[i]] (ids < 0: null key); alive[i] False = tombstone."""
    n = ids.size
    plen = np.array([len(k) for k in pool], dtype=np.int64)
    poff = np.cumsum(plen) - plen
    blob = np.frombuffer(b"".join(pool) or b"\0", dtype=np.uint8)
    keyed = ids >= 0
    kl = np.where(keyed, plen[np.maximum(ids, 0)], -1).astype(np.int32)
    kb = gather(blob, poff[np.maximum(ids, 0)], np.maximum(kl, 0)).copy()
    vl = np.where(alive, rng.integers(0, 300, size=n), -1).astype(np.int32)
    part = rng.integers(0, P, size=n).astype(np.int32)
    ts = (1_600_000_000_000 + rng.integers(-10**6, 10**6, size=n)).astype(np.int64)
    return HostTopic(part, np.zeros(n, dtype=np.int64), ts, kl, vl, np.arange(n, dtype=np.uint64), kb, tile_base_from_key_len(kl))


def filler_pool(rng, count, length=8):
    return [bytes(r) for r in rng.integers(0, 256, size=(count, length), dtype=np.uint8)]


# ------------------------------------------------------------------------------------------------
# expected and observed tables
# ------------------------------------------------------------------------------------------------
def oracle_of(*topics):
    o = Oracle(count_alive_keys=True, now=NOW)
    for t in topics:
        o.handle_batch(t.partition, t.ts_ms, t.key_len, t.value_len, t.key_bytes)
    return o


def check_exact(e, o, want, parts=P):
    """finalize, then the three statements every case makes."""
    e.finalize()
    assert_same_map(exported(e), want)
    assert_parity(e, o, parts, check_alive=True, hll_regs=o.hll_alive_regs(HLL_P))
    _, occupied, _, _ = e.alive_table_stats()
    assert occupied == want[0].size


def wave_shift(n):
    """The host's wave rule for a batch spanning n sequence numbers (at most 127 waves)."""
    sh = 0
    while ((n - 1) >> sh) + 1 > 127:
        sh += 1
    return sh


# ------------------------------------------------------------------------------------------------
# CPU: the key crafting itself
# ------------------------------------------------------------------------------------------------
def test_keys_for_mixed_hit_their_targets():
    rng = np.random.default_rng(5)
    xs = [0, MASK32, 1, 0x80000000, 0x7FFFFFFF] + [int(v) for v in rng.integers(0, 1 << 32, size=40, dtype=np.uint64)]
    xs += list(range(0x12345678, 0x12345678 + 8))
    keys = keys_for_mixed(xs)
    mix = olib().kto_hll_mix
    for k, x in zip(keys, xs):
        assert len(k) == 5
        h = fnv32(k)
        assert mix(h) == x and fmix32(h) == x and unmix32(x) == h, (k.hex(), hex(x))
    assert len(set(keys)) == len(keys)
    # the vectorised hash of the parity tests agrees
    kl = np.full(len(keys), 5, dtype=np.int32)
    got = np_oracle.fnv32_many(kl, np.frombuffer(b"".join(keys), dtype=np.uint8))
    assert [fmix32(int(h)) for h in got] == xs


def test_last_writer_map_is_the_replay():
    """The expected-table helper against the BitSet replay of the numpy restatement, on a ragged topic."""
    rng = np.random.default_rng(6)
    pool = filler_pool(rng, 50, 3) + [b""]
    ids = rng.integers(-1, len(pool), size=5000)
    t = pool_topic(rng, ids, pool, rng.random(5000) < 0.6)
    seq = rng.permutation(5000).astype(np.uint64) + np.uint64(7)
    h, s = last_writer_map(t, seq)
    assert np.all(np.diff(h.astype(np.int64)) > 0)
    hashes = np_oracle.fnv32_many(t.key_len, t.key_bytes)
    assert set(h[(s & np.uint64(1)) == 1].tolist()) == np_oracle.alive_set(t.key_len, t.value_len, hashes, seq)
    assert set(h.tolist()) == set(hashes[t.key_len >= 0].tolist())


# ------------------------------------------------------------------------------------------------
# GPU cases
# ------------------------------------------------------------------------------------------------
def wave_edge_topic(n, rng):
    """Filler plus keys at the wave boundaries of an n-record batch:
      * periodic keys written once per wave at phases 0, 1, -2, -1 of the wave;
      * for every other boundary: one key written by the last record of the wave before it and the first after it;
      * 'burst' keys written 40 times inside one wave, alive and tombstone interleaved; the last write of
        half of them is a tombstone, of the other half a value.
    Returns (topic, burst keys whose last write is alive, burst keys whose last write is a tombstone)."""
    sh = wave_shift(n)
    W = 1 << sh
    nfill = 100_000
    pool = filler_pool(rng, nfill)
    ids = rng.integers(0, nfill, size=n)
    ids[rng.random(n) < 0.01] = -1
    alive = rng.random(n) < 0.7
    for ph in (0, 1, W - 2, W - 1):
        pos = np.arange(ph, n, W)
        ids[pos] = len(pool)
        alive[pos] = rng.random(pos.size) < 0.5
        pool += filler_pool(rng, 1, 7)
    bounds = np.arange(2 * W, n, 2 * W)              # every other boundary (the periodic keys keep the rest)
    base = len(pool)
    pool += filler_pool(rng, bounds.size, 6)
    ids[bounds - 1] = base + np.arange(bounds.size)
    ids[bounds] = base + np.arange(bounds.size)
    burst_alive, burst_dead = [], []
    nwaves = (n + W - 1) // W
    for j in range(16):
        w = int(rng.integers(0, nwaves))
        lo, hi = w * W, min(n, (w + 1) * W)
        pos = np.sort(rng.choice(np.arange(lo, hi), size=40, replace=False))
        ids[pos] = len(pool)
        alive[pos] = np.arange(40) % 2 == (j % 2)      # interleaved; the last write (index 39) is alive iff j is odd
        key = filler_pool(rng, 1, 9)[0]
        pool.append(key)
        (burst_alive if j % 2 else burst_dead).append(key)
    return pool_topic(rng, ids, pool, alive), burst_alive, burst_dead


@pytest.mark.gpu
@pytest.mark.parametrize("n", [M20 - 128, M20, 127 << 14, (127 << 14) + 1])
def test_wave_edges(n):
    """64 waves (2^20), 127 full waves (127 * 2^14) and the step back to 64 waves one record later; 2^20 - 128 records
    go straight to the table and pin the boundary of the cache."""
    rng = np.random.default_rng(n)
    t, burst_alive, burst_dead = wave_edge_topic(n, rng)
    seq_base = 1_000_000_007
    seq = np.arange(n, dtype=np.uint64) + np.uint64(seq_base)
    want = last_writer_map(t, seq)
    with engine() as e:
        scan(e, t, seq_base=seq_base)
        check_exact(e, oracle_of(t), want)
    # the bursts' outcome, stated directly
    wh, ws = want
    for keys, bit in ((burst_alive, 1), (burst_dead, 0)):
        for k in keys:
            i = np.searchsorted(wh, fnv32(k))
            assert wh[i] == fnv32(k) and int(ws[i]) & 1 == bit


@pytest.mark.gpu
@pytest.mark.parametrize("ways", [3, 8, 32])
def test_keys_that_share_one_cache_set(ways):
    """`ways` keys with one cache set (x >> 9) and different tags, tag 0 among them, each written in every wave with a
    random last write, next to 200k ordinary keys."""
    rng = np.random.default_rng(ways)
    n = M20
    W = 1 << wave_shift(n)
    s = int(rng.integers(0, 1 << 23))
    # tag 0, and tags 0 and 256 agree in their low 8 bits: a tag one bit short would merge them
    tags = [0, 256] + [int(v) for v in rng.choice(np.setdiff1d(np.arange(1, 512), [256]), size=ways - 2, replace=False)]
    crafted = keys_for_mixed([(s << 9) | tg for tg in tags])
    nfill = 200_000
    pool = filler_pool(rng, nfill) + crafted
    ids = rng.integers(0, nfill, size=n)
    alive = rng.random(n) < 0.6
    for w0 in range(0, n, W):
        for j in range(ways):
            pos = w0 + rng.choice(W, size=3, replace=False)
            ids[pos] = nfill + j
    last = {}
    for j in range(ways):
        pos = np.nonzero(ids == nfill + j)[0]
        last[j] = bool(rng.random() < 0.5)
        alive[pos[-1]] = last[j]
    t = pool_topic(rng, ids, pool, alive)
    want = last_writer_map(t, np.arange(n, dtype=np.uint64))
    with engine() as e:
        scan(e, t)
        check_exact(e, oracle_of(t), want)
    wh, ws = want
    for j, k in enumerate(crafted):
        i = np.searchsorted(wh, fnv32(k))
        assert int(ws[i]) & 1 == int(last[j])


@pytest.mark.gpu
@pytest.mark.parametrize("last_alive", [False, True])
def test_table_edge_hashes(last_alive):
    """x = 0xffffffff (the empty slot's hash word) and x = 0, written in many waves; the last write decides."""
    rng = np.random.default_rng(11 + last_alive)
    n = M20 + 4096
    crafted = keys_for_mixed([MASK32, 0])
    nfill = 50_000
    pool = filler_pool(rng, nfill) + crafted
    ids = rng.integers(0, nfill, size=n)
    alive = rng.random(n) < 0.7
    for j in range(2):
        pos = np.sort(rng.choice(n - 10, size=300, replace=False))
        ids[pos] = nfill + j
        alive[pos] = rng.random(pos.size) < 0.5
        ids[n - 5 + j] = nfill + j                # the very last writes
        alive[n - 5 + j] = last_alive
    t = pool_topic(rng, ids, pool, alive)
    want = last_writer_map(t, np.arange(n, dtype=np.uint64))
    with engine() as e:
        scan(e, t)
        check_exact(e, oracle_of(t), want)
        assert e.alive_keys() == int((want[1] & np.uint64(1)).sum())
    for k in crafted:
        i = np.searchsorted(want[0], fnv32(k))
        assert int(want[1][i]) & 1 == int(last_alive)


@pytest.mark.gpu
@pytest.mark.parametrize("key_mode,n", [(0, 2 * M20), (1, 3 * M20), (2, 4 * M20)])
def test_skewed_keys(key_mode, n):
    """Log-uniform (Zipf-like) key ids: a few keys carry most records, so many stamps of one hash meet in one wave.
    16-byte, ASCII and ragged 0..40-byte keys, with null keys and tombstones."""
    spec = synth.make_spec(n, P, key_mode=key_mode, distinct_keys=P * 20_000, zipf_keys=True, tombstone_per_10k=3000,
                           null_key_per_10k=200)
    t = synth.fill_host(spec)
    want = last_writer_map(t, np.arange(n, dtype=np.uint64))
    with engine() as e:
        scan(e, t)
        check_exact(e, oracle_of(t), want)


def seq_topic(n, seed):
    spec = synth.make_spec(n, P, key_mode=2, seed=seed, distinct_keys=P * 25_000, tombstone_per_10k=2500,
                           null_key_per_10k=100)
    return synth.fill_host(spec)


@pytest.mark.gpu
@pytest.mark.parametrize("entry", ["device", "host"])
@pytest.mark.parametrize("shape", ["gapped", "permuted"])
def test_explicit_seq_with_the_cache(shape, entry):
    """An explicit seq column: gapped and increasing (what a shard of a partition-sharded job sees), or permuted within
    the batch so that its ends are neither its minimum nor its maximum (waves are then read off the wrong range: records
    outside it fall into the first or last wave).  The host entry point splits the batch into 2^22-record ring chunks,
    each cached, with seq ends taken from the host column."""
    n = (1 << 22) + M20 if entry == "host" else M20 + 776
    rng = np.random.default_rng(n + len(shape))
    t = seq_topic(n, 21 + len(shape))
    if shape == "gapped":
        seq = np.uint64(1000) + np.cumsum(rng.integers(1, 6, size=n)).astype(np.uint64)
    else:
        seq = rng.permutation(n).astype(np.uint64) + np.uint64(50)
        lo, hi = int(seq.min()), int(seq.max())
        if int(seq[0]) in (lo, hi) or int(seq[-1]) in (lo, hi):
            seq[[0, 1]] = seq[[1, 0]]
            seq[[-1, -2]] = seq[[-2, -1]]
        assert int(seq[0]) not in (lo, hi) and int(seq[-1]) not in (lo, hi)
    want = last_writer_map(t, seq)
    with engine() as e:
        (scan if entry == "device" else push_host)(e, t, seq=seq)
        check_exact(e, oracle_of(take(t, np.argsort(seq, kind="stable"))), want)


@pytest.mark.gpu
@pytest.mark.parametrize("entry", ["device", "host"])
def test_explicit_seq_outside_the_window(entry):
    """A seq column whose ends lie in the table's 31-bit window but some middle records outside it: those are left out of
    the table (and only of the table) and reported by finalize."""
    n = M20 + 4096
    rng = np.random.default_rng(31)
    t = seq_topic(n, 31)
    seq = np.arange(n, dtype=np.uint64) + np.uint64(10)
    out = np.zeros(n, dtype=bool)
    out[rng.choice(np.arange(1000, n - 1000), size=5000, replace=False)] = True
    seq[out] = np.uint64((1 << 31) + 5) + np.arange(int(out.sum()), dtype=np.uint64)
    want = last_writer_map(t, seq, keep=~out)
    with engine() as e:
        (scan if entry == "device" else push_host)(e, t, seq=seq)
        with pytest.raises(KtaError) as ei:
            e.finalize()
        assert ei.value.code == 1 and "window" in str(ei.value)
        assert_same_map(exported(e), want)
        assert e.alive_keys() == int((want[1] & np.uint64(1)).sum())
        assert e.alive_table_stats()[1] == want[0].size
        # everything but the table counts every record
        assert_parity(e, oracle_of(t), P)


@pytest.mark.gpu
@pytest.mark.parametrize("entry", ["device", "device_batches", "host"])
def test_growth_and_stamps_only_rerun_under_the_cache(entry):
    """A 64 KiB table (8192 slots) and ~200k distinct keys: stamps are dropped, the table grows and the batches are
    re-run stamps-only through the cached scan.  Counters must not be counted twice."""
    n = 3 * M20 + 5000 if entry == "device_batches" else 2 * M20
    spec = synth.make_spec(n, P, key_mode=1, seed=41, distinct_keys=P * 25_000, tombstone_per_10k=3000,
                           null_key_per_10k=100)
    t = synth.fill_host(spec)
    want = last_writer_map(t, np.arange(n, dtype=np.uint64))
    with engine(alive_table_kib=64) as e:
        assert e.alive_table_stats()[0] == 8192
        if entry == "device":
            scan(e, t)
        elif entry == "device_batches":
            # three cached batches queued before the first confirmation: all of them are re-run
            cuts = [0, M20, 2 * M20, n]
            for lo, hi in zip(cuts[:-1], cuts[1:]):
                scan(e, take(t, np.arange(lo, hi)))
        else:
            push_host(e, t)
        check_exact(e, oracle_of(t), want)
        slots, occupied, grows, reruns = e.alive_table_stats()
        assert grows >= 1 and reruns >= 1 and occupied * 10 <= slots * 6
        assert e.message_metrics.overall_count() == n


@pytest.mark.gpu
def test_rebase_under_the_cache():
    """2^20-record batches whose implicit seq straddles 2^31 and 2^32 force rebases between cached scans; the count and
    the HLL registers of the alive set stay the oracle's, and the export is refused afterwards."""
    rng = np.random.default_rng(51)
    bases = [0, (1 << 31) - (1 << 19), (1 << 31) + (1 << 20) + 7, (1 << 32) + 3]
    pool = filler_pool(rng, 60_000, 4)
    o = Oracle(count_alive_keys=True, now=NOW)
    seen = set()
    with engine() as e:
        for b, base in enumerate(bases):
            ids = rng.integers(0, len(pool), size=M20)
            ids[rng.random(M20) < 0.01] = -1
            t = pool_topic(rng, ids, pool, rng.random(M20) < 0.5)
            o.handle_batch(t.partition, t.ts_ms, t.key_len, t.value_len, t.key_bytes)
            seen |= set(np_oracle.fnv32_many(t.key_len, t.key_bytes)[t.key_len >= 0].tolist())
            (scan if b % 2 == 0 else push_host)(e, t, seq_base=base)
            e.finalize()
            assert_parity(e, o, P, check_alive=True, hll_regs=o.hll_alive_regs(HLL_P))
            assert e.alive_table_stats()[1] == len(seen)
        with pytest.raises(KtaError):
            e.alive_export_count()


@pytest.mark.gpu
def test_sharded_exact_handles_merge_to_the_whole_topic():
    """world = 4 partition-sharded engines on one device, each scanning its shard (>= 2^20 records) with the global seq
    column; every table exported and imported into engine 0 (the all-gather of distributed.py, without NCCL) and the
    counters merged: engine 0 then holds the whole topic's table, entry by entry."""
    import torch
    world, P16 = 4, 16
    n = 4 * M20 + 8 * 1024
    spec = synth.make_spec(n, P16, key_mode=2, seed=61, distinct_keys=P16 * 8000, tombstone_per_10k=3000,
                           null_key_per_10k=100)
    whole = synth.fill_host(spec)
    o = Oracle(count_alive_keys=True, now=NOW)
    o.handle_batch(whole.partition, whole.ts_ms, whole.key_len, whole.value_len, whole.key_bytes)
    engines = [engine(P16, shard=(r, world)) for r in range(world)]
    try:
        words = engines[0].merge_words(world)
        total = torch.zeros(words, dtype=torch.int64, device="cuda")
        lists = []
        for r, e in enumerate(engines):
            idx = np.nonzero(whole.partition % world == r)[0]
            assert idx.size >= M20
            t = take(whole, idx)
            scan(e, t, seq=whole.seq[idx])
            buf = torch.zeros(words, dtype=torch.int64, device="cuda")
            settle()
            e.merge_export(r, world, buf)                   # returns once the engine's stream has written buf
            total += buf
            cnt = e.alive_export_count()
            h = torch.zeros(cnt, dtype=torch.int32, device="cuda")
            s = torch.zeros(cnt, dtype=torch.int64, device="cuda")
            settle()
            assert e.alive_export(h, s, cnt) == cnt
            lists.append((h, s, cnt))
        e0 = engines[0]
        settle()
        e0.merge_import(world, total)
        for h, s, cnt in lists[1:]:
            alive_import(e0, h, s, cnt)
        check_exact(e0, o, last_writer_map(whole, whole.seq, parts=P16), parts=P16)
    finally:
        for e in engines:
            e.close()


@pytest.mark.gpu
@pytest.mark.parametrize("table_kib", [0, 64])
@pytest.mark.parametrize("cluster", [200, 400])
def test_clustered_home_pairs_do_not_grow_the_table(cluster, table_kib):
    """`cluster` keys with consecutive mixed hashes share a home pair at every table size, so a run of them outlasts the
    96-pair probe limit however large the table is.  A table that has room for them must keep its size; the table must
    still be exact."""
    rng = np.random.default_rng(cluster + table_kib)
    n = M20
    x0 = int(rng.integers(0, (1 << 32) - 4096)) & ~0xFFF
    crafted = keys_for_mixed(range(x0, x0 + cluster))
    nfill = 2500
    pool = filler_pool(rng, nfill) + crafted
    ids = rng.integers(0, nfill, size=n)
    pos = rng.choice(n, size=3 * cluster, replace=False)
    ids[pos] = nfill + np.arange(3 * cluster) % cluster
    t = pool_topic(rng, ids, pool, rng.random(n) < 0.6)
    want = last_writer_map(t, np.arange(n, dtype=np.uint64))
    with engine(alive_table_kib=table_kib) as e:
        slots0 = e.alive_table_stats()[0]
        scan(e, t)
        check_exact(e, oracle_of(t), want)
        slots, occupied, grows, reruns = e.alive_table_stats()
        assert occupied * 10 <= slots0 * 6
        assert (slots, grows) == (slots0, 0), "table grew from %d to %d slots (%d grows) for %d distinct keys" % (
            slots0, slots, grows, occupied)
