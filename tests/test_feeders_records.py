"""The host feeders, record by record: the landing ring behind kta_push and kta_push_batch_host (csrc/kta_api.cu).

The host decides where a chunk ends (a tile boundary chosen by key bytes), where its keys land (d_keys + (k0 & 15) under
the virtual base d_keys + shift - k0), which sequence numbers it gets, when its ring slot may be overwritten and whether
its exact-mode stamps are confirmed or re-run.  A wrong decision moves a few records' key bytes or sequence numbers, which
the alive count usually survives.  So every case here checks, with -c:
  * the exported table (hash, (seq + 1) << 1 | alive) against last_writer_map over the records in the order they were
    fed, with the seq each should have received; a failure names the first bad record by chunk, row, tile and k0 & 15;
  * counters, histograms, extrema, the alive count and the alive set's HLL registers against the C oracle;
  * the edge the case names, asserted as reached: chunk scans counted by kta_stats on a twin handle without -c (whose
    launches are the create's state reset plus one per chunk scan), and grows and re-runs by kta_alive_table_stats.
Keys carry their record's index in their first 8 bytes (fewer for shorter keys), then a tail made from that index, so
they are distinct unless a case repeats one on purpose.  `host_chunks` and `push_chunks` restate where the two feeders
cut a batch."""
import re

import numpy as np
import pytest

from kafka_topic_analyzer_b200 import KtaEngine, KtaError
from kafka_topic_analyzer_b200 import _native as N
from kafka_topic_analyzer_b200.synth import HostTopic, tile_base_from_key_len
from feed import (NOW, T, engine, keys_for_mixed, last_writer_map, made_byte, push_host, push_records, scan, take)
from oracle_lib import Oracle
from parity import assert_parity, assert_same_map, exported
import kafka_codec as kc
import np_oracle

P = 8
HLL_P = 12                      # feed.engine's
M20 = 1 << 20
STAGE_MAX = 128 * T             # a tile with more key bytes than this is hashed from global memory (KEYBUF_MAX - slack)


# ------------------------------------------------------------------------------------------------
# topics
# ------------------------------------------------------------------------------------------------
def make_topic(rng, kl, *, ids=None, ascii=False, alive=0.7, parts=None, block=1 << 18):
    """Records with key lengths kl (< 0: null key).  Record i's key is made from ids[i] (default i): its first min(len, 8)
    bytes are ids[i] little-endian (ASCII: 8 decimal digits), the rest a tail made from ids[i] and the position.  Two
    records with the same id and length have the same key."""
    kl = np.asarray(kl, dtype=np.int32)
    n = kl.size
    ids = np.arange(n, dtype=np.int64) if ids is None else np.asarray(ids, dtype=np.int64)
    lens = np.maximum(kl, 0).astype(np.int64)
    parts_kb = []
    for a in range(0, n, block):                      # bounded temporaries on deep topics
        b = min(n, a + block)
        ln = lens[a:b]
        total = int(ln.sum())
        r = np.repeat(ids[a:b], ln)
        pos = np.arange(total, dtype=np.int64) - np.repeat(np.cumsum(ln) - ln, ln)
        byte = made_byte(r, pos)
        if ascii:
            byte = 97 + byte % 26
            head = (r // 10 ** (7 - np.minimum(pos, 7))) % 10 + 48
        else:
            head = (r >> (8 * np.minimum(pos, 7))) & 0xFF
        parts_kb.append(np.where(pos < 8, head, byte).astype(np.uint8))
    kb = np.concatenate(parts_kb) if parts_kb else np.zeros(0, dtype=np.uint8)
    part = rng.integers(0, P, size=n).astype(np.int32) if parts is None else np.asarray(parts, dtype=np.int32)
    vl = np.where(rng.random(n) < alive, rng.integers(0, 300, size=n), -1).astype(np.int32)
    ts = (1_600_000_000_000 + rng.integers(-10**6, 10**6, size=n)).astype(np.int64)
    return HostTopic(part, np.arange(n, dtype=np.int64), ts, kl, vl, np.arange(n, dtype=np.uint64), kb,
                     tile_base_from_key_len(kl))


def ragged(rng, n, lo=0, hi=40, null=0.05):
    kl = rng.integers(lo, hi + 1, size=n).astype(np.int32)
    kl[rng.random(n) < null] = -1
    return kl


def equal_tiles(rng, ntiles, B):
    """ntiles tiles of ragged keys (nulls and empties among them) whose key bytes are exactly B each: the last key of every
    tile makes up the rest"""
    kl = ragged(rng, ntiles * T, 0, 30).reshape(ntiles, T)
    kl[:, -1] = B - np.maximum(kl[:, :-1], 0).sum(1)
    assert (kl[:, -1] >= 0).all()
    return kl.reshape(-1)


def concat(*ts):
    """the records of several topics in this order"""
    cat = lambda f: np.concatenate([getattr(t, f) for t in ts])
    kl = cat("key_len")
    return HostTopic(cat("partition"), cat("offset"), cat("ts_ms"), kl, cat("value_len"), np.arange(kl.size, dtype=np.uint64),
                     cat("key_bytes"), tile_base_from_key_len(kl))


def oracle_of(t, order=None):
    o = Oracle(count_alive_keys=True, now=NOW)
    if order is not None:
        t = take(t, order)
    o.handle_batch(t.partition, t.ts_ms, t.key_len, t.value_len, t.key_bytes)
    return o


# ------------------------------------------------------------------------------------------------
# where the feeders cut (restated)
# ------------------------------------------------------------------------------------------------
def host_chunks(kl, R, KB):
    """kta_push_batch_host's chunks of a batch with key lengths kl, ring_records R (a multiple of T) and ring_key_bytes KB:
    ([(r0, r1, k0)], None), or (the chunks scanned, r0) when the tile at r0 alone has more than KB key bytes (refused)"""
    tb = tile_base_from_key_len(np.asarray(kl)).astype(np.int64)
    n, out, r0 = len(kl), [], 0
    while r0 < n:
        tiles_max = -(-min(R, n - r0) // T)
        t0 = r0 // T
        k0 = int(tb[t0])
        tiles = min(int(np.searchsorted(tb[t0:t0 + tiles_max + 1], k0 + KB, side="right")) - 1, tiles_max)
        if tiles < 1:
            return out, r0
        r1 = min(r0 + tiles * T, n, r0 + R)
        out.append((r0, r1, k0))
        r0 = r1
    return out, None


def push_chunks(kl, R, KB):
    """kta_push's chunks of a run of records: one closes when it holds R records or the next key would pass KB bytes;
    every chunk's keys start at 0 of its landing area.  [(r0, r1, 0)]"""
    lens = np.maximum(np.asarray(kl, dtype=np.int64), 0)
    assert (lens <= KB).all()
    cs = np.concatenate([[0], np.cumsum(lens)])
    n, out, r0 = lens.size, [], 0
    while r0 < n:
        by_bytes = int(np.searchsorted(cs, cs[r0] + KB, side="right")) - 1   # records r0..by_bytes-1 fit KB
        r1 = min(r0 + R, by_bytes, n)
        out.append((r0, r1, 0))
        r0 = r1
    return out


def shifted(chunks, by):
    """chunks of a batch fed after `by` other records (their key offsets are the batch's own)"""
    return [(a + by, b + by, k) for a, b, k in chunks]


# ------------------------------------------------------------------------------------------------
# the three checks
# ------------------------------------------------------------------------------------------------
def where(i, chunks):
    for j, (r0, r1, k0) in enumerate(chunks or ()):
        if r0 <= i < r1:
            return "chunk %d, row %d, tile %d, k0 & 15 = %d" % (j, i - r0, (i - r0) // T, k0 & 15)
    return "no chunk"


def assert_table(e, t, seq, chunks=None, keep=None):
    """the export equals last_writer_map(t, seq); otherwise the first record whose hash entry is wrong is named"""
    got, want = exported(e), last_writer_map(t, seq, keep=keep, parts=P)
    try:
        assert_same_map(got, want)
    except AssertionError as err:
        # the records behind the wrong entries: the one whose stamp was expected and the one whose stamp was exported
        gh, gs = got
        wh, ws = want
        stamps = np.concatenate([gs[~np.isin(gh, wh)], ws[~np.isin(wh, gh)]])
        common, gi, wi = np.intersect1d(gh, wh, return_indices=True)
        differ = gs[gi] != ws[wi]
        stamps = np.concatenate([stamps, gs[gi][differ], ws[wi][differ]])
        recs = np.nonzero(np.isin(np.asarray(seq, dtype=np.uint64), (stamps >> np.uint64(1)) - np.uint64(1)))[0]
        if keep is not None:
            recs = recs[keep[recs]]
        if not recs.size:
            raise
        i = int(recs[0])
        k = int(np.maximum(t.key_len[:i], 0).sum())
        raise AssertionError("first bad record %d (%s; seq %d, key %s): %s"
                             % (i, where(i, chunks), int(seq[i]), t.key_bytes[k:k + max(int(t.key_len[i]), 0)].tobytes().hex(),
                                err)) from None


def assert_exact(e, t, seq, chunks=None, order=None):
    """finalize, then the table, entry by entry, and the report against the oracle fed in seq order"""
    e.finalize()
    assert_table(e, t, seq, chunks)
    o = oracle_of(t, np.argsort(seq, kind="stable") if order is None else order)
    assert_parity(e, o, P, check_alive=True, hll_regs=o.hll_alive_regs(HLL_P))


def twin(R, KB):
    """a handle whose keys travel like an -c handle's (it hashes them for its HLL sketch) but which has no alive-key table:
    its launches are the create's state reset plus one per scan"""
    return KtaEngine(P, hll_precision=HLL_P, now=NOW, ring_records=R, ring_key_bytes=KB)


def chunk_scans(R, KB, feed_fn):
    with twin(R, KB) as tw:
        feed_fn(tw)
        tw.finalize()
        return tw.stats()[0] - 1


# ------------------------------------------------------------------------------------------------
# CPU: the restated cuts
# ------------------------------------------------------------------------------------------------
def test_host_chunks_cut_on_tile_bounds_by_key_bytes():
    B = 1000
    kl = np.full(10 * T, -1, dtype=np.int32)
    kl[::T] = B                                           # one B-byte key per tile
    assert host_chunks(kl, 64 * T, 5 * B) == ([(0, 5 * T, 0), (5 * T, 10 * T, 5 * B)], None)
    kl[4 * T + 1] = 1                                     # one byte more in the first five tiles
    assert [c[:2] for c in host_chunks(kl, 64 * T, 5 * B)[0]] == [(0, 4 * T), (4 * T, 8 * T), (8 * T, 10 * T)]
    assert host_chunks(kl, 3 * T, 100 * B)[0][:2] == [(0, 3 * T, 0), (3 * T, 6 * T, 3 * B)]
    kl[4 * T + 1] = -1
    kl[6 * T + 1] = 1                                     # tile 6 alone holds B + 1 bytes
    assert host_chunks(kl, 64 * T, B) == ([(i * T, (i + 1) * T, i * B) for i in range(6)], 6 * T)
    assert host_chunks(np.zeros(T + 1, dtype=np.int32), 64 * T, 1) == ([(0, T + 1, 0)], None)


def test_push_chunks_close_on_count_and_key_bytes():
    assert push_chunks([5] * 10, 4, 100) == [(0, 4, 0), (4, 8, 0), (8, 10, 0)]
    assert push_chunks([30, 30, 40, 0, -1, 1, 100, 0, 7], 64, 100) == [(0, 5, 0), (5, 6, 0), (6, 8, 0), (8, 9, 0)]


def test_made_keys_are_distinct_and_carry_their_index():
    rng = np.random.default_rng(1)
    for ascii in (False, True):
        t = make_topic(rng, np.full(3000, 12, dtype=np.int32), ascii=ascii)
        keys = t.key_bytes.reshape(-1, 12)
        assert len({k.tobytes() for k in keys}) == 3000
        if ascii:
            assert ((keys >= 48) & (keys < 123)).all() and keys[1234, :8].tobytes() == b"00001234"
        else:
            assert int(keys[1234, :8].view(np.uint64)[0]) == 1234
    ids = np.array([0, 1, 0, 1], dtype=np.int64)
    t = make_topic(rng, np.array([20, 20, 20, 3], dtype=np.int32), ids=ids)
    assert t.key_bytes[:20].tobytes() == t.key_bytes[40:60].tobytes()


# ------------------------------------------------------------------------------------------------
# 1. chunk cuts by key bytes (kta_push_batch_host)
# ------------------------------------------------------------------------------------------------
B = 2560                        # key bytes of one tile in the equal-tile topics


def cut_shape(rng, shape):
    """(key lengths, ring_records, ring_key_bytes, what the cuts must show)"""
    if shape == "fills_exactly":
        return equal_tiles(rng, 10, B), 64 * T, 5 * B, lambda c: c[0][:2] == (0, 5 * T) and len(c) == 2
    if shape == "one_byte_heavier":
        kl = equal_tiles(rng, 10, B)
        kl[5 * T - 1] += 1                                # tiles 0..4 now hold 5B + 1 bytes: cut one tile earlier
        return kl, 64 * T, 5 * B, lambda c: c[0][:2] == (0, 4 * T) and len(c) == 3
    if shape == "one_tile":
        return equal_tiles(rng, 6, B), 64 * T, B + B // 2, lambda c: all(r1 - r0 == T for r0, r1, _ in c)
    if shape == "one_tile_fills_exactly":
        return equal_tiles(rng, 6, B), 64 * T, B, lambda c: all(r1 - r0 == T for r0, r1, _ in c) and len(c) == 6
    if shape == "tail_1":
        return np.concatenate([equal_tiles(rng, 6, B), ragged(rng, 1)]), 64 * T, 2 * B, lambda c: (c[-1][1] - c[-1][0]) % T == 1
    if shape == "tail_127":
        return (np.concatenate([equal_tiles(rng, 7, B), ragged(rng, 127, 0, 8)]), 64 * T, 2 * B,
                lambda c: c[-1][1] - c[-1][0] == T + 127)
    if shape == "records_first":
        return equal_tiles(rng, 10, B), 3 * T, 8 * B, lambda c: [r1 - r0 for r0, r1, _ in c] == [3 * T] * 3 + [T]
    raise ValueError(shape)


@pytest.mark.gpu
@pytest.mark.parametrize("tile_base", [True, False])
@pytest.mark.parametrize("shape", ["fills_exactly", "one_byte_heavier", "one_tile", "one_tile_fills_exactly", "tail_1",
                                   "tail_127", "records_first"])
def test_chunk_cuts_by_key_bytes(shape, tile_base):
    """Chunks of kta_push_batch_host end where host_chunks says, with and without the caller's tile bases: a chunk whose
    keys fill ring_key_bytes exactly next to the same batch one byte heavier, one-tile chunks (one filling it exactly),
    a partial last tile of 1 and 127 records, and ring_records reached before ring_key_bytes."""
    rng = np.random.default_rng(len(shape))
    kl, R, KB, edge = cut_shape(rng, shape)
    t = make_topic(rng, kl)
    chunks, refused = host_chunks(kl, R, KB)
    assert refused is None and edge(chunks), chunks
    with engine(ring_records=R, ring_key_bytes=KB) as e:
        push_host(e, t, tile_base=tile_base)
        assert_exact(e, t, t.seq, chunks)
    assert chunk_scans(R, KB, lambda tw: push_host(tw, t, tile_base=tile_base)) == len(chunks)


@pytest.mark.gpu
@pytest.mark.parametrize("tile_base", [True, False])
def test_one_tile_over_the_key_ring_is_refused_after_the_prefix(tile_base):
    """A tile of exactly ring_key_bytes is taken; the next one, one byte heavier, refuses the call.  The error says how
    many records were scanned, and the engine holds exactly that prefix."""
    rng = np.random.default_rng(7)
    kl = equal_tiles(rng, 9, B)
    kl[6 * T + 5] += 1
    t = make_topic(rng, kl)
    chunks, refused = host_chunks(kl, 64 * T, B)
    assert refused == 6 * T and len(chunks) == 6
    keep = np.arange(t.n) < refused
    for e in (engine(ring_records=64 * T, ring_key_bytes=B), twin(64 * T, B)):
        with e:
            with pytest.raises(KtaError) as ei:
                push_host(e, t, tile_base=tile_base)
            assert ei.value.code == N.ERR_INVALID and "ring_key_bytes" in str(ei.value)
            assert int(re.search(r"(\d+) earlier record\(s\)", str(ei.value)).group(1)) == refused
            e.finalize()
            if e.count_alive_keys:
                assert_table(e, t, t.seq, chunks, keep=keep)
                o = oracle_of(t, np.arange(refused))
                assert_parity(e, o, P, check_alive=True, hll_regs=o.hll_alive_regs(HLL_P))
            else:
                assert e.stats() == (1 + len(chunks), refused)


# ------------------------------------------------------------------------------------------------
# 2. key placement: chunk starts at every k0 mod 16
# ------------------------------------------------------------------------------------------------
def placement_lengths(rng, shape, ntiles):
    """key lengths whose every tile holds 1 mod 16 key bytes, so that one-tile chunks start at k0 mod 16 = 0, 1, ..., 15"""
    n = ntiles * T + 77
    if shape == "fixed16":
        kl = np.full(n, 16, dtype=np.int32)
    else:
        kl = ragged(rng, n, 0, 40, null=0.1)
    if shape == "global_read":
        kl[21 * T] = STAGE_MAX + 700                    # chunk 21's first tile is hashed from global memory
    for t in range(ntiles):
        last = t * T + T - 1
        kl[last] = max(kl[last], 0) + (1 - int(np.maximum(kl[t * T:last + 1], 0).sum())) % 16
    return kl


@pytest.mark.gpu
@pytest.mark.parametrize("tile_base", [True, False])
@pytest.mark.parametrize("shape", ["fixed16", "ragged", "ascii", "global_read"])
def test_key_placement_at_every_residue(shape, tile_base):
    """One-tile chunks whose keys start at every k0 mod 16 (the shift under the chunk's virtual base): 16-byte keys,
    ragged keys with nulls and empty keys, ASCII keys, and a chunk whose first tile's keys exceed the scan's stage."""
    rng = np.random.default_rng(20 + len(shape))
    kl = placement_lengths(rng, shape, 40)
    t = make_topic(rng, kl, ascii=shape == "ascii")
    R, KB = T, 1 << 16
    chunks, _ = host_chunks(kl, R, KB)
    assert {k0 & 15 for _, _, k0 in chunks} == set(range(16))
    if shape == "global_read":
        j = 21
        assert chunks[j][:2] == (21 * T, 22 * T) and chunks[j][2] & 15 and t.key_tile_base[22] - t.key_tile_base[21] > STAGE_MAX
    with engine(ring_records=R, ring_key_bytes=KB) as e:
        push_host(e, t, tile_base=tile_base)
        assert_exact(e, t, t.seq, chunks)
    assert chunk_scans(R, KB, lambda tw: push_host(tw, t, tile_base=tile_base)) == len(chunks)


# ------------------------------------------------------------------------------------------------
# 3. kta_push, record by record
# ------------------------------------------------------------------------------------------------
def at_the_end(KB):
    """keys of 8, 9, 16 and 17 bytes that end exactly at the landing area's end (kta_push's three copy branches), a key that
    fills it alone, with nulls and empty keys between"""
    kl = [30] * 20                                      # 600 bytes: the first chunk is exactly full
    for L in (8, 9, 16, 17):
        kl += [KB - L, 0, -1, L]
    kl += [KB, 0, 5]
    return np.array(kl, dtype=np.int32)


@pytest.mark.gpu
@pytest.mark.parametrize("shape", ["by_count", "by_key_bytes"])
def test_push_closes_chunks(shape):
    """kta_push closes a chunk when it holds ring_records records, or when the next key would pass ring_key_bytes; keys
    written at the very end of the landing area."""
    rng = np.random.default_rng(30 + len(shape))
    if shape == "by_count":
        R, KB = 2 * T, 1 << 20
        kl = ragged(rng, 5 * R + 3)
    else:
        R, KB = 64 * T, 600
        kl = np.concatenate([at_the_end(KB), ragged(rng, 700), at_the_end(KB)])
    t = make_topic(rng, kl)
    chunks = push_chunks(kl, R, KB)
    if shape == "by_count":
        assert [b - a for a, b, _ in chunks] == [R] * 5 + [3]
    else:
        assert chunks[0][:2] == (0, 20) and len(chunks) > 20
    with engine(ring_records=R, ring_key_bytes=KB) as e:
        push_records(e, t)
        assert_exact(e, t, t.seq, chunks)
    assert chunk_scans(R, KB, lambda tw: push_records(tw, t)) == len(chunks)


@pytest.mark.gpu
def test_push_refuses_a_key_over_the_key_ring_and_takes_nothing():
    """A key of ring_key_bytes bytes is taken; one byte more is refused, nothing of it is taken, and the next record gets
    the next sequence number."""
    rng = np.random.default_rng(33)
    R, KB = 4 * T, 600
    kl = ragged(rng, 900)
    kl[300], kl[301] = KB, KB + 1
    t = make_topic(rng, kl)
    idx = np.delete(np.arange(t.n), 301)
    kept = take(t, idx)
    chunks = push_chunks(kept.key_len, R, KB)
    seq = np.zeros(t.n, dtype=np.uint64)
    seq[idx] = np.arange(idx.size, dtype=np.uint64)
    for e in (engine(ring_records=R, ring_key_bytes=KB), twin(R, KB)):
        with e:
            push_records(e, t, count=301)
            with pytest.raises(KtaError) as ei:
                push_records(e, t, start=301, count=1)
            assert ei.value.code == N.ERR_INVALID and "exceeds ring_key_bytes" in str(ei.value)
            push_records(e, t, start=302)
            e.finalize()
            if e.count_alive_keys:
                assert_table(e, t, seq, [(idx[a], idx[b - 1] + 1, k) for a, b, k in chunks], keep=np.arange(t.n) != 301)
                o = oracle_of(kept)
                assert_parity(e, o, P, check_alive=True, hll_regs=o.hll_alive_regs(HLL_P))
            else:
                assert e.stats() == (1 + len(chunks), idx.size)


@pytest.mark.gpu
def test_push_negative_lengths_are_minus_one():
    """key_len and value_len of -1 and below -1 give the state of -1."""
    rng = np.random.default_rng(34)
    n = 700
    t = make_topic(rng, ragged(rng, n, null=0.2))
    raw_k, raw_v = t.key_len.copy(), t.value_len.copy()
    neg = t.key_len < 0
    raw_k[neg] = rng.choice(np.array([-1, -2, -40, -(1 << 31)], dtype=np.int32), size=int(neg.sum()))
    deadv = t.value_len < 0
    raw_v[deadv] = rng.choice(np.array([-1, -3, -1000, -(1 << 31)], dtype=np.int32), size=int(deadv.sum()))
    assert (raw_k < -1).sum() > 50 and (raw_v < -1).sum() > 50
    raw = HostTopic(t.partition, t.offset, t.ts_ms, raw_k, raw_v, t.seq, t.key_bytes, t.key_tile_base)
    with engine(ring_records=2 * T) as e:
        push_records(e, raw)
        assert_exact(e, t, t.seq, push_chunks(t.key_len, 2 * T, 2 * T * 24))


# ------------------------------------------------------------------------------------------------
# 4. ring turns at depth
# ------------------------------------------------------------------------------------------------
def repeating_topic(rng, n, lo, hi, repeat=0.3, **kw):
    """ragged keys; a `repeat` share of the keyed records re-writes the key of an earlier record"""
    kl = ragged(rng, n, lo, hi)
    ids = np.arange(n, dtype=np.int64)
    again = np.nonzero(rng.random(n) < repeat)[0][1:]
    ids[again] = (rng.random(again.size) * again).astype(np.int64)
    ids[again] = ids[ids[again]]                       # (an earlier record may itself repeat one)
    kl[again] = kl[ids[again]]
    return make_topic(rng, kl, ids=ids, **kw)


@pytest.mark.gpu
@pytest.mark.parametrize("entry", ["host", "push"])
def test_ring_turns(entry):
    """65 turns of the three-chunk ring in one call, with repeated keys."""
    rng = np.random.default_rng(40 + len(entry))
    R, KB = 2 * T, 1 << 16
    n = 3 * 65 * R + 37
    t = repeating_topic(rng, n, 0, 40)
    chunks = host_chunks(t.key_len, R, KB)[0] if entry == "host" else push_chunks(t.key_len, R, KB)
    assert len(chunks) >= 3 * 64
    feed_fn = (lambda e: push_host(e, t, tile_base=False)) if entry == "host" else (lambda e: push_records(e, t))
    with engine(ring_records=R, ring_key_bytes=KB) as e:
        feed_fn(e)
        assert_exact(e, t, t.seq, chunks)
    assert chunk_scans(R, KB, feed_fn) == len(chunks)


@pytest.mark.gpu
@pytest.mark.parametrize("entry", ["host_gapped_seq", "host", "push"])
def test_ring_turns_with_the_seen_cache(entry):
    """ring_records = 2^20: every chunk scan goes through the seen cache, with waves from the chunk's own seq range,
    through kta_push_batch_host with a gapped, increasing seq column and without one, and through kta_push."""
    rng = np.random.default_rng(50 + len(entry))
    R = M20
    n = 3 * R
    t = repeating_topic(rng, n, 4, 16, repeat=0.4)
    seq = t.seq
    if entry == "host_gapped_seq":
        seq = np.uint64(77) + np.cumsum(rng.integers(1, 4, size=n)).astype(np.uint64)
    KB = R * 24
    chunks = host_chunks(t.key_len, R, KB)[0] if entry != "push" else push_chunks(t.key_len, R, KB)
    assert [b - a for a, b, _ in chunks] == [R] * 3
    if entry == "push":
        feed_fn = lambda e: push_records(e, t)
    else:
        feed_fn = lambda e: push_host(e, t, seq=seq if entry == "host_gapped_seq" else None)
    with engine(ring_records=R) as e:
        feed_fn(e)
        assert_exact(e, t, seq, chunks, order=np.arange(n))
    assert chunk_scans(R, KB, feed_fn) == 3


# ------------------------------------------------------------------------------------------------
# 5. exact-mode confirmations across the ring
# ------------------------------------------------------------------------------------------------
def burst_topic(rng, nchunks, R, burst_chunks, nfill=24):
    """nchunks chunks of R records over `nfill` repeated 8-byte keys, except that the records of the burst chunks all
    carry new keys"""
    n = nchunks * R
    ids = rng.integers(0, nfill, size=n)
    for c in burst_chunks:
        ids[c * R:(c + 1) * R] = nfill + np.arange(c * R, (c + 1) * R)
    kl = np.full(n, 8, dtype=np.int32)
    kl[rng.random(n) < 0.03] = -1
    return make_topic(rng, kl, ids=ids)


@pytest.mark.gpu
@pytest.mark.parametrize("where_", ["first", "last"])
def test_stamps_dropped_in_one_chunk_of_a_turn(where_):
    """A 1 KiB table (128 slots) and one chunk of 256 new keys, the first (ring slot 0) or the last (slot 2) chunk of the
    ring's second turn: its dropped stamps are found in its status snapshot when its slot is reused, the table grows and
    the pending chunks are re-run."""
    rng = np.random.default_rng(60 + len(where_))
    R = 2 * T
    burst = 3 if where_ == "first" else 5
    t = burst_topic(rng, 9, R, [burst])
    chunks = host_chunks(t.key_len, R, 1 << 20)[0]
    assert len(chunks) == 9
    with engine(ring_records=R, alive_table_kib=1) as e:
        assert e.alive_table_stats()[0] == 128
        push_host(e, t)
        assert_exact(e, t, t.seq, chunks)
        slots, occupied, grows, reruns = e.alive_table_stats()
        assert grows >= 1 and reruns >= 1


@pytest.mark.gpu
def test_stamps_dropped_only_by_a_device_batch_between_two_host_batches():
    """kta_push_batch_host (two chunks, no drops), kta_scan_batch_device (the only drops), kta_push_batch_host again (five
    chunks): when the third ring slot is reused, ring entries and the device batch's entry are both pending, and the
    snapshot behind it must see the device batch's drops."""
    rng = np.random.default_rng(61)
    R = 2 * T
    a = burst_topic(rng, 2, R, [])
    b = make_topic(rng, np.full(300, 9, dtype=np.int32), ids=np.arange(10**6, 10**6 + 300))
    c = burst_topic(rng, 5, R, [])
    t = concat(a, b, c)
    ca = host_chunks(a.key_len, R, 1 << 20)[0]
    cc = shifted(host_chunks(c.key_len, R, 1 << 20)[0], a.n + b.n)
    with engine(ring_records=R, alive_table_kib=1) as e:
        push_host(e, a)
        assert e.alive_table_stats()[2:] == (0, 0)
        scan(e, b)
        push_host(e, c)
        assert_exact(e, t, t.seq, ca + [(a.n, a.n + b.n, 0)] + cc)
        slots, occupied, grows, reruns = e.alive_table_stats()
        assert grows >= 1 and reruns >= 1


@pytest.mark.gpu
def test_wide_rerun_over_ring_chunks_mid_turn():
    """300 keys whose mixed hashes are consecutive, in the middle chunk of the ring's second turn, next to 2500 filler
    keys, in a 64 KiB table with room for all: the re-run probes the whole table over the pending ring chunks, and the
    table keeps its size."""
    rng = np.random.default_rng(62)
    R = 8 * T
    nfill, cluster = 2500, 300
    t0 = burst_topic(rng, 9, R, [], nfill=nfill)
    x0 = int(rng.integers(0, (1 << 32) - 4096)) & ~0xFFF
    crafted = keys_for_mixed(range(x0, x0 + cluster))
    # chunk 4 carries the crafted keys (5 bytes) among its filler
    pos = 4 * R + np.sort(rng.choice(R, size=cluster, replace=False))
    kl = t0.key_len.copy()
    kl[pos] = 5
    t = make_topic(rng, kl, ids=np.where(np.isin(np.arange(t0.n), pos), -1, rng.integers(0, nfill, size=t0.n)))
    koff = np.cumsum(np.maximum(kl, 0)) - np.maximum(kl, 0)
    for p, k in zip(pos, crafted):
        t.key_bytes[koff[p]:koff[p] + 5] = np.frombuffer(k, dtype=np.uint8)
    chunks = host_chunks(t.key_len, R, 1 << 20)[0]
    with engine(ring_records=R, alive_table_kib=64) as e:
        slots0 = e.alive_table_stats()[0]
        push_host(e, t)
        assert_exact(e, t, t.seq, chunks)
        slots, occupied, grows, reruns = e.alive_table_stats()
        assert reruns >= 1 and (slots, grows) == (slots0, 0)


@pytest.mark.gpu
def test_rebase_between_two_chunks_of_one_call():
    """A seq_base that puts the second chunk of one kta_push_batch_host call across origin + 2^31 - 2: the first chunk's
    stamps (some dropped: a 4 KiB table) are settled and the table rebased between the two chunks.  The export is refused
    after a rebase, so the alive count and the alive set's HLL registers are checked."""
    rng = np.random.default_rng(63)
    R = 2 * T
    t = burst_topic(rng, 6, R, [0, 4], nfill=200)
    base = (1 << 31) - 2 - R - R // 2
    chunks = host_chunks(t.key_len, R, 1 << 20)[0]
    with engine(ring_records=R, alive_table_kib=4) as e:
        push_host(e, t, seq_base=base)
        e.finalize()
        o = oracle_of(t)
        assert_parity(e, o, P, check_alive=True, hll_regs=o.hll_alive_regs(HLL_P))
        slots, occupied, grows, reruns = e.alive_table_stats()
        assert grows >= 1 and reruns >= 1
        assert occupied == len(set(np_oracle.fnv32_many(t.key_len, t.key_bytes)[t.key_len >= 0].tolist()))
        with pytest.raises(KtaError) as ei:
            e.alive_export_count()
        assert "rebased" in str(ei.value)
    assert chunk_scans(R, 1 << 20, lambda tw: push_host(tw, t, seq_base=base)) == len(chunks)


# ------------------------------------------------------------------------------------------------
# 6. entry points interleaved in one stream
# ------------------------------------------------------------------------------------------------
def log_segments(rng, t):
    """t's records, which lie partition by partition in increasing partition order, as one segment per partition"""
    segs = []
    for p in np.unique(t.partition):
        idx = np.nonzero(t.partition == p)[0]
        koff = np.cumsum(np.maximum(t.key_len, 0)) - np.maximum(t.key_len, 0)
        recs = [(int(t.ts_ms[i]), None if t.key_len[i] < 0 else t.key_bytes[koff[i]:koff[i] + t.key_len[i]].tobytes(),
                 None if t.value_len[i] < 0 else int(t.value_len[i])) for i in idx]
        segs.append((int(p), kc.encode_partition(recs, rng, max_batch=50)))
    return segs


@pytest.mark.gpu
def test_entry_points_interleaved_then_reset():
    """kta_push leaving a chunk open, kta_push_batch_host (KTA_SEQ_AUTO), kta_scan_batch_device without tile bases over
    1025 tiles (tile_base_scan_kernel carries between its chunks), kta_push_log_segments_host, kta_push again, and
    kta_push_batch_host at an explicit seq_base above the running count: every record's seq is its place in that order.
    Then kta_reset with a chunk open and earlier chunks in flight, and a second topic: the table holds only it, from seq 0."""
    rng = np.random.default_rng(70)
    R, KB = 4 * T, 1 << 14
    sizes = [700, 1500, 1025 * T - 50, 0, 300, 900]
    parts = []
    for i, n in enumerate(sizes):
        if i == 3:
            kl = ragged(rng, 400)
            tl = make_topic(rng, kl, ids=np.arange(400) + 10**7, parts=np.sort(rng.integers(0, P, size=400)))
            parts.append(tl)
        else:
            parts.append(make_topic(rng, ragged(rng, n), ids=np.arange(n) + (i + 1) * 10**7))
    t = concat(*parts)
    ends = np.cumsum([p.n for p in parts])
    gap = 1000
    seq = t.seq.copy()
    seq[ends[4]:] += np.uint64(gap)
    with engine(ring_records=R, ring_key_bytes=KB) as e:
        push_records(e, parts[0])
        push_host(e, parts[1])
        scan(e, parts[2], tile_base=False)
        assert e.push_log_segments(log_segments(rng, parts[3])) == parts[3].n
        push_records(e, parts[4])
        push_host(e, parts[5], seq_base=int(ends[4]) + gap)
        assert_exact(e, t, seq, order=np.arange(t.n))
        assert e.stats()[1] == t.n

        # reset with chunks in flight and one open, then a second topic
        first = make_topic(rng, ragged(rng, 3000), ids=np.arange(3000) + 9 * 10**7)
        push_records(e, first)
        e.reset()
        a = make_topic(rng, ragged(rng, 1000), ids=np.arange(1000) + 11 * 10**7)
        b = make_topic(rng, ragged(rng, 800), ids=np.arange(800) + 12 * 10**7)
        push_records(e, a)
        push_host(e, b)
        second = concat(a, b)
        assert_exact(e, second, second.seq)
        assert e.stats()[1] == second.n
