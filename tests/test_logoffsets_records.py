"""The offset windows of the RecordBatch decoder (kta_logoffsets.cuh) checked record by record: the window test of the header
pass, log_cut_count_kernel (warp per cut batch: how many rows each cut batch gets) and log_decode_window_kernel (the kept
records ranked by a ballot and a popcount, plus a carry across lane rounds).

tests/native/log_probe.cu, given a window table, runs scan_log_batches' steps (kta_logscan.cuh) for a handle with windows
and returns every decoded column, every batch's flags after the header pass, the count
pass's drops and the header pass's window words.  Each case compares them with window_contract(), a plain restatement on top
of test_logdecode_records.contract(): a batch's verdict (not served / served / cut) comes from baseOffset and the stored
lastOffsetDelta alone; records below the log start offset S are dropped only from cut batches (baseOffset < S); offsets are
computed in 64-bit two's complement.  The hand-built cases also compare it with offsets_codec.fetched / fetch_stats.  The
scan's metrics would hide most of these errors (rows moved inside a partition, a row left unwritten)."""
import struct
from collections import namedtuple

import numpy as np
import pytest

import kafka_codec as kc
import log_probe
import offsets_codec as oc
from test_logdecode_records import (TS0, Case, Cols, batch_of_length, check, columns, contract, decode, decode_shape, i64,
                                    key)

LOGB_BAD, LOGB_SKIP_OFFSET = 2, 512
CODECS = (None, "gzip", "snappy", "snappy-xerial", "lz4", "zstd", "zstd-stream")   # test_log_offsets.CODECS
# what window_contract gives for an accepted call: the delivered records [(partition, ts, key|None, value_len)], per batch the
# rows it gets, whether it is not served, whether it is cut and how many records it drops; the header pass's words [6..9]
# as (cut batches, batches not served, their data records)
WinWant = namedtuple("WinWant", "recs counts skip cut drops words")


# ------------------------------------------------------------------------------------------------
# the restatement
# ------------------------------------------------------------------------------------------------
def window_contract(data, offs, parts, win):
    """None when the call is refused, else a WinWant.  win: [(S, H)] of partitions [0, len(win)), -1 = that side unbounded;
    any other partition has no window.  A framed batch (magic 2, batchLength >= 49, inside the buffer) with last = baseOffset
    + lastOffsetDelta outside [S, H) is not served: none of its other fields is read, and its recordsCount counts as left out
    when it is a data batch.  A served batch is read as contract() reads it (a compressed one in its uncompressed image); a
    served data batch with records and baseOffset < S is cut, and only there a record whose offset is below S is dropped."""
    n = len(data)
    recs, counts, skip, cut, drops = [], [], [], [], []
    ncut = not_served = left = 0
    for i, off in enumerate(offs):
        p = parts[i] if parts else 0
        lo, hi = win[p] if 0 <= p < len(win) else (-1, -1)
        if off + 61 > n:
            return None
        base, bl = struct.unpack_from(">qi", data, off)
        magic, = struct.unpack_from(">b", data, off + 16)
        attrs, last_delta = struct.unpack_from(">hi", data, off + 21)
        cnt, = struct.unpack_from(">i", data, off + 57)
        if not (magic == 2 and bl >= 49 and off + 12 + bl <= n):
            return None
        last = i64(base + last_delta)
        out = (lo >= 0 and last < lo) or (hi >= 0 and last >= hi)
        skip.append(out)
        is_cut = not out and lo >= 0 and base < lo and not attrs & 0x20 and cnt > 0
        cut.append(is_cut)
        if out:
            not_served += 1
            left += cnt if not attrs & 0x20 and cnt > 0 else 0
            counts.append(0)
            drops.append(0)
            continue
        if attrs & 7 > 4:
            return None
        image, at = data, off
        if attrs & 7 and not attrs & 0x20:
            if cnt < 0:
                return None
            image, at = kc.with_section(data[off:off + 61], kc._decompress(attrs & 7, data[off + 61:off + 12 + bl]), 0), 0
        got = contract(image, [at], len(image), with_offsets=True)
        if got is None:
            return None
        kept = [r for r in got if r[4] >= lo] if is_cut else got
        ncut += is_cut
        drops.append(len(got) - len(kept))
        counts.append(len(kept))
        recs += [(p,) + r[1:4] for r in kept]
    return WinWant(recs, counts, skip, cut, drops, (ncut, not_served, left))


def oc_expect(c):
    """what offsets_codec gives for the case: per partition (in batch order) the fetched records, and over all partitions
    fetch_stats' (batches not served, records left out)"""
    segs = {}
    for p, raw in zip(c.parts, c.raw):
        segs[p] = segs.get(p, b"") + raw
    recs, nb, left = {}, 0, 0
    for p, seg in segs.items():
        lo, hi = c.win[p] if 0 <= p < len(c.win) else (-1, -1)
        recs[p] = [(p, ts, k, -1 if vl is None else vl) for _, ts, k, vl in oc.fetched(seg, lo, hi)]
        st = oc.fetch_stats(seg, lo, hi)
        nb, left = nb + st[0], left + st[1]
    return recs, (nb, left)


# ------------------------------------------------------------------------------------------------
# cases
# ------------------------------------------------------------------------------------------------
def wb(base, deltas, codec=None, last=None, seed=0, attributes=0, value=None):
    """one batch at `base` with a record per offset delta (keys, nulls and value lengths drawn from the record's index);
    last: the stored lastOffsetDelta, when it is not the largest delta"""
    recs = [(d, j * 3 - 7, None if (j + seed) % 7 == 5 else key(j + seed, (j + seed) % 13),
             None if (j + seed) % 9 == 4 else (j * 5 + seed) % 40) for j, d in enumerate(deltas)]
    if value:
        recs[0] = recs[0][:3] + (None, (), value)
    b = kc.encode_batch(base, TS0 + seed, recs, attributes=attributes, compression=codec)
    return b if last is None else oc.with_last_offset_delta(b, last)


def wcase(name, batches, parts, win, slack=0, oc_check=True):
    """batches back to back, batch i in partition parts[i]; win: the window table"""
    c = Case.__new__(Case)
    c.name, c.slack, c.parts, c.win, c.raw, c.oc_check = name, slack, list(parts), list(win), list(batches), oc_check
    c.offs = np.concatenate([[0], np.cumsum([len(b) for b in batches])[:-1]]).astype(int).tolist()
    c.data = b"".join(batches)
    c.want = window_contract(c.data, c.offs, c.parts, c.win)
    if c.want is not None:
        c.cols, c.counts = columns(c.want.recs), c.want.counts
    return c


def rank_cases():
    """recordsCount around the lane rounds; for the smaller ones S at every record (and one past the last), each in a
    partition of its own, so every rank carry is met"""
    batches, parts, win = [], [], []
    for n in (1, 31, 32, 33, 63, 64, 65, 97):
        for s in range(n + 1):
            batches.append(wb(0, range(n), seed=n + s))
            parts.append(len(win))
            win.append((s, -1))
    out = [wcase("rank-every-start", batches, parts, win)]
    batches, parts, win = [], [], []
    for n in (1000, 4097):
        for s in (0, 1, 31, 32, 33, 64, 500, 999, 1000, 4000, 4096, 4097):
            if s <= n:
                batches.append(wb(0, range(n), seed=s))
                parts.append(len(win))
                win.append((s, -1))
    out.append(wcase("rank-long", batches, parts, win))
    return out


def mask_cases():
    """cut batches whose kept records form no suffix inside a lane round: offset deltas that are a random permutation, that
    alternate above and below S, or that are drawn above or below S independently"""
    rng = np.random.default_rng(101)
    batches, parts, win = [], [], []
    for n in (2, 31, 32, 33, 64, 65, 100, 1000):
        batches.append(wb(0, rng.permutation(n).tolist(), seed=n))
        win.append(((n + 1) // 2, -1))
        batches.append(wb(0, [j // 2 if j % 2 else n + j for j in range(n)], seed=n + 1))    # below, above, below, ...
        win.append((n, -1))
        batches.append(wb(0, [n + j if j % 2 else j // 2 for j in range(n)], seed=n + 2))    # above, below, above, ...
        win.append((n, -1))
        pick = rng.choice(2 * n, n, replace=False)
        batches.append(wb(0, pick.tolist(), seed=n + 3))                                   # each record kept by a coin
        win.append((n, -1))
    parts = list(range(len(win)))
    return [wcase("any-keep-mask", batches, parts, win)]


def compacted_cases():
    """offset gaps with S in a gap, at a record, and between the last record and the stored last (served, keeps nothing)"""
    gaps = [0, 1, 4, 9, 10, 11, 20, 33, 34, 40]
    batches, win = [], []
    for s in (2, 4, 5, 12, 19, 21, 34, 35, 40, 41, 44, 45, 46):
        batches.append(wb(100, gaps, last=45, seed=s))
        win.append((100 + s, -1))
    batches.append(wb(100, gaps, last=45, seed=99))
    win.append((100 + 41, 100 + 46))                                                      # cut, and H past last
    parts = list(range(len(win)))
    return [wcase("compacted", batches, parts, win)]


def header_edge_cases():
    """lastOffsetDelta at -2^31, -1, 0 and 2^31 - 1; S and H at last - 1, last, last + 1; S = 0, H = 0; baseOffsets up to 2^62"""
    batches, win = [], []
    for base in (0, 1, 2 ** 31, 2 ** 62):
        for ld in (-2 ** 31, -1, 0, 2 ** 31 - 1):
            last = base + ld
            for s, h in ((last - 1, -1), (last, -1), (last + 1, -1), (-1, last - 1), (-1, last), (-1, last + 1),
                         (0, -1), (-1, 0), (0, 0), (last, last + 1), (base + 1, -1)):
                if s < -1 or h < -1 or (s >= 0 and h >= 0 and s > h):
                    continue
                batches.append(wb(base, range(5), last=ld, seed=len(win)))
                win.append((s, h))
    parts = list(range(len(win)))
    out = [wcase("header-edges", batches, parts, win)]
    # a batch whose records' offsets wrap past 2^63: in 64-bit two's complement they lie below S and are dropped
    base = 2 ** 63 - 10
    out.append(wcase("offset-wraps-past-2^63", [wb(base, range(20), last=5), wb(0, range(3))], [0, 1], [(base + 3, -1)],
                     oc_check=False))
    return out


def outside_cases():
    """batches of partitions outside [0, nwin) that would be cut or not served with a window: they get none"""
    parts = [-1, 0, 3, 2 ** 31 - 1, 1, -2 ** 31, 2]
    batches = [wb(0, range(40), seed=i) for i in range(len(parts))]
    return [wcase("outside-the-table", batches, parts, [(10, -1), (50, -1), (5, 100)])]


def codec_cases():
    """cut batches in every codec, in a staged launch and in an in-place one (a batch past 48 KiB), with images longer
    than the stage"""
    out = []
    for in_place in (False, True):
        batches, parts, win = [], [], []
        for i, codec in enumerate(CODECS):
            p = 3 * i
            batches += [wb(0, range(40), codec, seed=i), wb(40, range(10), codec, seed=i + 1)]
            parts += [p, p]
            win.append((17, -1))
            batches.append(wb(0, [0, 1, 4, 9, 10, 11, 20, 33, 34, 40], codec, last=45, seed=i + 2))   # compacted, S in a gap
            parts.append(p + 1)
            win.append((5, 48))
            batches.append(wb(0, range(4), codec, seed=i + 3, value=bytes(30_000 + 1000 * i)))     # image past the stage
            parts.append(p + 2)
            win.append((2, -1))
        if in_place:
            batches.append(wb(0, range(2), seed=7, value=bytes(60_000)))
            parts.append(len(win))
            win.append((1, -1))
        out.append(wcase("codecs-" + ("in-place" if in_place else "staged"), batches, parts, win))
    return out


def damaged_cut_cases():
    """a cut batch that keeps nothing (S past its last record, not past last) whose first record's key runs past the record
    (the count pass, which reads no key lengths, walks it): refused, alone and with other batches"""
    bad = bytearray(wb(0, range(20), last=30))
    _, _, at, n = record_fields(bad)[0]
    bad[at + n] = 0x7E                                  # key length 63 in a record of a few bytes
    return [wcase("damaged-cut-alone", [bytes(bad)], [0], [(25, -1)], oc_check=False),
            wcase("damaged-cut-with-others", [wb(0, range(8)), bytes(bad), wb(0, range(8), seed=3)], [1, 0, 2],
                  [(25, -1), (3, -1)], oc_check=False)]


def negative_delta_cases():
    """the batch at S = 10 with offset deltas [0, -3, 1] (partition 1) keeps its three records, whether or not a batch of
    partition 0 is cut in the same call"""
    neg = wb(10, [0, -3, 1], seed=5)
    cut = wb(0, range(10), seed=6)
    return [wcase("negative-delta-with-cut", [cut, neg], [0, 1], [(5, -1), (10, -1)]),
            wcase("negative-delta-alone", [cut, neg], [0, 1], [(0, -1), (10, -1)])]


def hand_built():
    return (rank_cases() + mask_cases() + compacted_cases() + header_edge_cases() + outside_cases() + codec_cases() +
            damaged_cut_cases() + negative_delta_cases())


# ------------------------------------------------------------------------------------------------
# the checks
# ------------------------------------------------------------------------------------------------
def refused(r):
    return bool(r.hdr & LOGB_BAD or r.unc_err or r.dec_err)


def check_window(c, r):
    """the window words, every batch's flag, every cut batch's drops, which decode ran, then every column, the tile bases
    and the key bytes (test_logdecode_records.check)"""
    w = c.want
    assert not refused(r), (c.name, r.hdr, r.unc_err, r.dec_err)
    assert r.words == w.words, (c.name, "words [6..9]", r.words, w.words)
    skip = r.flags == LOGB_SKIP_OFFSET
    if not np.array_equal(skip, w.skip):
        b = int(np.argmax(skip != np.asarray(w.skip)))
        pytest.fail("%s: batch %d is %sLOGB_SKIP_OFFSET (flags %d)" % (c.name, b, "" if skip[b] else "not ", r.flags[b]))
    drops = np.diff(r.drop.astype(np.int64))
    if not np.array_equal(drops, w.drops):
        b = int(np.argmax(drops != np.asarray(w.drops)))
        pytest.fail("%s: cut batch %d drops %d records, want %d" % (c.name, b, drops[b], w.drops[b]))
    if r.ran:
        assert r.windowed == (w.words[0] > 0), (c.name, "windowed", r.windowed)
    check(c, r)


def by_partition(recs):
    out = {}
    for rec in recs:
        out.setdefault(rec[0], []).append(rec)
    return out


# ---- CPU: the restatement against offsets_codec -----------------------------------------------------------------------
def test_restatement_and_offsets_codec_agree_on_the_hand_built_cases():
    """window_contract (the decoder's rules) and offsets_codec (a consumer's) give the same records per partition and the
    same totals on every hand-built case; the offset that wraps past 2^63 and the damaged cases are the restatement's own"""
    for c in hand_built():
        if not c.oc_check:
            continue
        assert c.want is not None, c.name
        recs, stats = oc_expect(c)
        got = by_partition(c.want.recs)
        assert {p: v for p, v in got.items()} == {p: v for p, v in recs.items() if v}, c.name
        assert (c.want.words[1], c.want.words[2] + sum(c.want.drops)) == stats, c.name


def test_hand_built_cases_reach_their_edges():
    by = {c.name: c for c in hand_built()}
    # keep masks that are no suffix of a lane round
    c = by["any-keep-mask"]
    nonsuffix = 0
    for i, (raw, cut) in enumerate(zip(c.raw, c.want.cut)):
        assert cut or i % 4 == 3                          # (a coin batch may have drawn every delta below S)
        b = kc.read_segment(raw)[0]
        for i0 in range(0, len(b.records), 32):
            m = [r[0] >= c.win[i][0] for r in b.records[i0:i0 + 32]]
            nonsuffix += m != sorted(m)
    assert nonsuffix > 30
    assert sum(by["rank-every-start"].want.cut) == sum(n - 1 for n in (1, 31, 32, 33, 63, 64, 65, 97))
    assert by["damaged-cut-alone"].want is None and by["damaged-cut-with-others"].want is None
    assert by["offset-wraps-past-2^63"].want.counts == [7, 3]
    h = by["header-edges"].want
    assert 0 < sum(h.skip) < len(h.skip) and 0 < sum(h.cut)


def test_negative_delta_rule():
    """the rule: records are dropped only from cut batches.  The batch at S with a record at S - 3 keeps it (offsets_codec and
    the restatement); the same record in a cut batch is dropped"""
    neg = wb(10, [0, -3, 1], seed=5)
    assert [r[0] for r in oc.fetched(neg, 10)] == [10, 7, 11]
    assert oc.fetch_stats(neg, 10) == (0, 0)
    w = window_contract(neg, [0], [0], [(10, -1)])
    assert w.counts == [3] and w.cut == [False] and w.drops == [0]
    cut = wb(9, [1, -2, 2], seed=5)                     # offsets 10, 7, 11 in a batch that starts below S
    assert [r[0] for r in oc.fetched(cut, 10)] == [10, 11]
    w = window_contract(cut, [0], [0], [(10, -1)])
    assert w.counts == [2] and w.cut == [True] and w.drops == [1]
    a, b = negative_delta_cases()
    assert by_partition(a.want.recs)[1] == by_partition(b.want.recs)[1]
    assert a.want.words[0] == 1 and b.want.words[0] == 0


# ---- GPU: the hand-built cases -------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_hand_built_window_cases_decode_record_by_record():
    cases = hand_built()
    (sm, optin), res = decode(cases)
    for c, r in zip(cases, res):
        staged, stage, _, grid = decode_shape(r.longest, len(c.offs), sm, optin)
        assert (r.staged, r.stage, r.grid) == (staged, stage, grid), c.name
        if c.want is None:
            assert refused(r), (c.name, "accepted")
            continue
        check_window(c, r)
        if c.oc_check:
            assert (r.words[1], r.words[2] + int(r.drop[-1])) == oc_expect(c)[1], c.name
    by = {c.name: r for c, r in zip(cases, res)}
    assert by["codecs-staged"].staged and not by["codecs-in-place"].staged
    a, b = by["negative-delta-with-cut"], by["negative-delta-alone"]
    assert a.windowed and not b.windowed
    for name in ("part", "ts", "klen", "vlen"):                # partition 1's three rows
        assert np.array_equal(getattr(a, name)[-3:], getattr(b, name)[-3:]), name


# ---- depth ------------------------------------------------------------------------------------------------------------
def depth_pool(rng, big=None):
    """templates (kind, bytes, window relative to baseOffset 0, or None: a partition outside the table): cut batches,
    uncompressed ('C') and compressed ('Z'), batches not served ('U'), served whole ('W'), control and empty ones ('-');
    `big`: one more served batch of that length ('B')"""
    pool = []
    for i in range(40):
        n = int(rng.choice([1, 2, 3, 5, 8, 12, 33, 40, 65], p=[.2, .15, .15, .15, .1, .1, .05, .05, .05]))
        deltas = rng.permutation(n).tolist() if i % 2 else sorted(rng.choice(2 * n + 3, n, replace=False).tolist())
        pool.append(("C", wb(0, deltas, seed=i), (int(rng.integers(1, max(deltas) + 1)) if max(deltas) else 0, -1)))
    pool = [p if p[2][0] > 0 else ("W",) + p[1:] for p in pool]
    for i, codec in enumerate(["gzip", "lz4", "snappy", "zstd"] * 2):
        n = int(rng.integers(2, 12))
        pool.append(("Z", wb(0, rng.permutation(n).tolist(), codec, seed=50 + i), (n // 2, -1)))
    for i in range(6):
        pool.append(("U", wb(0, range(5), seed=60 + i), (7, -1) if i % 2 else (-1, 3)))
    for i in range(6):
        pool.append(("W", wb(0, range(1 + i), seed=70 + i), None if i % 2 else (0, 100)))
    pool += [("-", kc.encode_batch(0, TS0, [(0, 0, kc.marker_record_key(True), None)], attributes=0x30), (1, -1)),
             ("-", kc.encode_batch(0, TS0, []), (0, -1)), ("-", kc.encode_batch(0, TS0, []), None)]
    order = rng.permutation(len(pool))
    pool = [pool[i] for i in order]
    if big:
        pool.append(("B", batch_of_length(big, 5)[0], (1, -1)))
    return pool


def depth_case(pool, idx, name):
    """batch i: pool[idx[i]] at baseOffset 2^40 + 1000 i, in partition i (its window moved with it) or, without a window, in
    partition nb + i"""
    nb = len(idx)
    raws = [pool[t][1] for t in idx]
    lens = np.array([len(b) for b in raws], np.int64)
    offs = np.concatenate([[0], np.cumsum(lens)[:-1]])
    data = bytearray(b"".join(raws))
    bases = (2 ** 40 + 1000 * np.arange(nb, dtype=np.int64))
    arr = np.frombuffer(data, np.uint8)
    arr[(offs[:, None] + np.arange(8)).ravel()] = bases.astype(">i8").view(np.uint8)
    has = np.array([pool[t][2] is not None for t in range(len(pool))])
    rel = np.array([pool[t][2] or (-1, -1) for t in range(len(pool))], np.int64)
    parts = np.where(has[idx], np.arange(nb), nb + np.arange(nb)).astype(np.int32)
    w = rel[idx]
    win = np.where(w >= 0, w + bases[:, None], -1)
    tw = [window_contract(pool[t][1], [0], [0], [pool[t][2]] if pool[t][2] else []) for t in range(len(pool))]
    tc = [columns(t.recs) for t in tw]
    c = Case.__new__(Case)
    c.name, c.slack, c.parts, c.data, c.offs = name, 48, parts.tolist(), bytes(data), offs.tolist()
    c.win = win
    counts = np.array([tw[t].counts[0] for t in range(len(pool))])[idx]
    c.counts = counts.tolist()
    c.cols = Cols(np.repeat(parts, counts), np.concatenate([tc[t].ts for t in idx]), np.concatenate([tc[t].klen for t in idx]),
                  np.concatenate([tc[t].vlen for t in idx]), b"".join(tc[t].keys for t in idx))
    words = np.array([tw[t].words for t in range(len(pool))], np.int64)[idx].sum(0)
    c.want = WinWant(None, c.counts, np.array([tw[t].skip[0] for t in range(len(pool))])[idx],
                     np.array([tw[t].cut[0] for t in range(len(pool))])[idx],
                     np.array([tw[t].drops[0] for t in range(len(pool))])[idx], tuple(int(x) for x in words))
    return c


@pytest.mark.gpu
@pytest.mark.parametrize("shape", ["small-batches", "stage-48k"])
def test_every_warp_counts_and_decodes_many_cut_batches(shape):
    """Every warp of the count pass takes >= 64 cut batches (one per partition, next to batches not served and batches
    served whole), and every warp of the window decode >= 64 batches, going staged -> in place -> staged."""
    rng = np.random.default_rng(103 if shape == "small-batches" else 107)
    pool = depth_pool(rng, 49136 if shape == "stage-48k" else None)
    sm, optin = log_probe.device()
    k = len(pool) - (1 if shape == "stage-48k" else 0)
    cut_per = sum(p[0] in "CZ" for p in pool[:k])
    count_warps = 4 * sm * 16
    nb = -(-(64 * count_warps + 17) // cut_per) * k + 5
    idx = np.arange(nb) % k
    if shape == "stage-48k":
        idx[np.arange(3, nb, 50_000)] = k                  # the 48 KiB batch, a few times
    case = depth_case(pool, idx, "depth-" + shape)
    longest = max(len(pool[t][1]) for t in set(idx.tolist()) if pool[t][0] in "CWB")
    staged, stage, per_sm, grid = decode_shape(longest, nb, sm, optin)
    assert staged and per_sm == (16 if shape == "small-batches" else 1)
    warps = 4 * grid
    kinds = np.array([{"C": "S", "W": "S", "B": "S", "Z": "P"}.get(pool[t][0], "-") for t in range(len(pool))])[idx]
    seqs = ["".join(k for k in kinds[w::warps][:64] if k != "-") for w in range(warps)]
    assert sum("SPS" in s for s in seqs) > warps // 4
    _, (r,) = decode([case])
    assert (r.staged, r.stage, r.grid) == (staged, stage, grid)
    ncut = r.words[0]
    cgrid = min((ncut + 3) // 4, sm * 16)
    assert ncut >= 64 * 4 * cgrid and nb >= 64 * warps, (ncut, cgrid, nb, warps)
    print("%s: %d batches, %d cut, %d records; count pass %.1f cut batches per warp, decode %.1f batches per warp"
          % (shape, nb, ncut, r.nrec, ncut / (4 * cgrid), nb / warps))
    check_window(case, r)


# ---- damage -----------------------------------------------------------------------------------------------------------
def record_fields(b):
    """per record of an uncompressed batch: (where its length varint starts, its bytes, where its offset delta starts, its
    bytes)"""
    def vlen(p):
        k = 0
        while b[p + k] & 0x80:
            k += 1
        return k + 1
    out, pos = [], 61
    for _ in range(struct.unpack_from(">i", b, 57)[0]):
        k = vlen(pos)
        ln = kc._read_varint(b, pos)[0]
        t = vlen(pos + k + 1)
        out.append((pos, k, pos + k + 1 + t, vlen(pos + k + 1 + t)))
        pos += k + ln
    return out


def damaged_cases():
    """about 3000 single-byte mutations of cut batches, each between intact batches: offset-delta varints and their
    continuation bits, record lengths, recordsCount, and the low bytes of baseOffset and lastOffsetDelta (which flip the
    verdict)"""
    rng = np.random.default_rng(109)
    bases = [(wb(1000, sorted(rng.choice(300, 40, replace=False).tolist()), seed=1), 1150),
             (wb(5000, rng.permutation(100)[:33].tolist(), seed=2), 5050),
             (wb(2 ** 40, [j // 2 if j % 2 else 200 + j for j in range(70)], seed=3), 2 ** 40 + 100),
             (wb(0, range(20), last=30, seed=4), 25)]
    fields = [record_fields(b) for b, _ in bases]
    before, after = wb(7, range(5), seed=8), wb(50, range(70), seed=9)
    cases = []
    for i in range(3000):
        t = i % len(bases)
        b, lo = bytearray(bases[t][0]), bases[t][1]
        f = fields[t]
        kind = (i // len(bases)) % 6
        if kind == 0:                                          # an offset-delta varint
            r = f[int(rng.integers(0, len(f)))]
            at = r[2] + int(rng.integers(0, r[3]))
            b[at] = int(rng.integers(0, 256)) if i % 2 else b[at] ^ (1 << int(rng.integers(0, 8)))
        elif kind == 1:                                        # a continuation bit: offset delta or record length
            r = f[int(rng.integers(0, len(f)))]
            at = r[2] + int(rng.integers(0, r[3])) if i % 2 else r[0] + int(rng.integers(0, r[1]))
            b[at] ^= 0x80
        elif kind == 2:                                        # a record length
            r = f[int(rng.integers(0, len(f)))]
            b[r[0] + int(rng.integers(0, r[1]))] = int(rng.integers(0, 256))
        elif kind == 3:                                        # recordsCount
            cnt = len(f)
            new = [0, 1, cnt - 1, cnt + 1, cnt - 32, cnt + 32, 2 ** 31 - 1, -1][(i // 24) % 8]
            b[57:61] = (new & 0xFFFFFFFF).to_bytes(4, "big")
        elif kind == 4:                                        # the low byte of baseOffset
            b[7] = int(rng.integers(0, 256))
        else:                                                  # the low byte of lastOffsetDelta
            b[26] = int(rng.integers(0, 256))
        cut_neighbour = i % 2                                  # half the calls have a second cut batch
        c = wcase("damaged-%d" % i, [before, bytes(b), after], [1, 0, 2],
                  [(lo, -1), (10 if cut_neighbour else -1, -1)], oc_check=False)
        cases.append(c)
    return cases


@pytest.mark.gpu
def test_damaged_cut_batches_agree_with_the_contract():
    """Each mutated cut batch is refused exactly when window_contract refuses it, and otherwise decodes to its columns,
    flags, drops and words.  One probe run carries every case."""
    cases = damaged_cases()
    _, res = decode(cases)
    disagree = []
    for c, r in zip(cases, res):
        if refused(r) != (c.want is None):
            disagree.append((c.name, "refused" if refused(r) else "accepted", r.hdr, r.dec_err))
        elif c.want is not None:
            check_window(c, r)
    assert not disagree, "%d of %d cases: %s" % (len(disagree), len(cases), disagree[:20])
    nref = sum(c.want is None for c in cases)
    still_cut = sum(c.want is not None and c.want.cut[1] for c in cases)
    print("%d refused, %d accepted with the mutated batch still cut" % (nref, still_cut))
    assert 300 < nref < 2700 and still_cut > 800
