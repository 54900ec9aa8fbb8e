"""Offsets for the log entry points (include/kta.h kta_log_set_offsets, kta_logoffsets.cuh): a consumer that starts at a
partition's log start offset S and reads up to its high watermark H is served only the batches with S <= last < H
(last = baseOffset + the stored lastOffsetDelta) and drops the records below S inside them.

Each GPU case compares the engine with the oracle fed exactly offsets_codec.fetched()'s records, in scan order, and checks
records_out and log_offset_stats exactly."""
import os
import struct
import subprocess
from dataclasses import dataclass

import numpy as np
import pytest

import kafka_codec as kc
import offsets_codec as oc
from feed import LOG_ENTRIES, scan_log
from kafka_topic_analyzer_b200 import KtaEngine, KtaError
from parity import assert_parity, oracle_in_order

NOW = (4102444800, 123456789)
TS0 = 1_700_000_000_000
CODECS = (None, "gzip", "snappy", "snappy-xerial", "lz4", "zstd", "zstd-stream")   # test_log_crc.CODECS


@dataclass
class B:
    p: int
    raw: bytes
    bad: bool = False   # its CRC fails


def mk(p, base, recs, codec=None, last_delta=None, attributes=0, crc=True):
    """recs [(offset, ts, key, value_len)] (absolute offsets, gaps allowed) as one batch at `base` with its real CRC (0
    without crc); last_delta: the stored lastOffsetDelta, when it is to exceed the last record's (a compacted batch)"""
    ts0 = recs[0][1] if recs else TS0 + base
    raw = kc.encode_batch(base, ts0, [(o - base, t - ts0, k, v) for o, t, k, v in recs], attributes=attributes, compression=codec)
    if last_delta is not None:
        raw = oc.with_last_offset_delta(raw, last_delta)
    return B(p, kc.set_crcs(raw) if crc else raw)


def recs_at(offsets, rng, keys=40, max_value=200):
    out = []
    for o in offsets:
        k = None if rng.random() < 0.05 else b"key-%d" % int(rng.integers(0, keys))
        vl = None if rng.random() < 0.15 else int(rng.integers(0, max_value))
        out.append((int(o), TS0 + 10 * int(o) + int(rng.integers(0, 7)), k, vl))
    return out


def gen_partition(rng, p, nb, codecs=CODECS, max_n=60):
    """nb batches at increasing offsets, every batch its own codec; one in four compacted (offset gaps, and a stored
    lastOffsetDelta past its last record)"""
    out, off = [], 0
    for _ in range(nb):
        n = int(rng.integers(1, max_n))
        codec = codecs[int(rng.integers(0, len(codecs)))]
        if rng.random() < 0.25:
            span = n + int(rng.integers(1, 20))
            offs = np.sort(rng.choice(span, size=n, replace=False)) + off
            out.append(mk(p, off, recs_at(offs, rng), codec, last_delta=span - 1 + int(rng.integers(0, 3))))
            off += span + 3
        else:
            out.append(mk(p, off, recs_at(range(off, off + n), rng), codec))
            off += n
    return out, off


def expect(order, win):
    """(partition, ts, key, value_len) records a consumer is served, in scan order, and (batches not served, records left
    out) — batches whose CRC fails deliver nothing and, being served or not, are not counted as left out"""
    recs, nb, left = [], 0, 0
    for b in order:
        lo, hi = win.get(b.p, (None, None))
        st = oc.fetch_stats(b.raw, lo, hi)
        if b.bad and st[0] == 0:
            continue                     # served but failed its CRC: skipped by check.crcs
        recs += [(b.p, ts, k, vl) for _, ts, k, vl in oc.fetched(b.raw, lo, hi)]
        nb, left = nb + st[0], left + st[1]
    return recs, (nb, left)


def engine(P, **kw):
    return KtaEngine(P, count_alive_keys=True, hll_precision=10, now=NOW, **kw)


def set_windows(e, win):
    for p, (lo, hi) in win.items():
        e.set_log_offsets(p, lo, hi)


def check(e, order, win, P, n):
    e.finalize()
    recs, stats = expect(order, win)
    assert n == len(recs)
    o = oracle_in_order(recs)
    assert_parity(e, o, P, check_alive=True, hll_regs=o.hll_alive_regs(10))
    assert e.log_offset_stats() == stats
    return recs


# ---- CPU: fetched() on hand-built batches ----------------------------------------------------------------------------
def _offs(seg, lo=None, hi=None):
    return [r[0] for r in oc.fetched(seg, lo, hi)]


def test_fetched_log_start():
    # batch A: offsets 0-4; batch B (compacted): records 5, 7, 9, stored lastOffsetDelta 6 (last = 11); batch C: 12-13
    a = mk(0, 0, [(o, TS0 + o, b"k", 1) for o in range(5)]).raw
    b = mk(0, 5, [(o, TS0 + o, b"k", 1) for o in (5, 7, 9)], last_delta=6).raw
    c = mk(0, 12, [(o, TS0 + o, b"k", 1) for o in (12, 13)]).raw
    seg = a + b + c
    assert _offs(seg) == [0, 1, 2, 3, 4, 5, 7, 9, 12, 13] == _offs(seg, -1, -1)
    assert _offs(seg, 0) == _offs(seg)
    assert _offs(seg, 5) == [5, 7, 9, 12, 13]                       # S at a batch's first record
    assert _offs(seg, 4) == [4, 5, 7, 9, 12, 13]                    # S at a batch's last record
    assert _offs(seg, 6) == [7, 9, 12, 13]                          # S inside an offset gap
    assert _offs(seg, 10) == [12, 13]                               # between the last record and `last`: served, empty
    assert _offs(seg, 11) == [12, 13]
    assert _offs(seg, 12) == [12, 13]
    assert _offs(seg, 14) == []
    assert oc.fetch_stats(seg, 6) == (1, 5 + 1)                     # A not served; 5 dropped inside B
    assert oc.fetch_stats(seg, 10) == (1, 5 + 3)                    # B served, every record dropped
    assert oc.fetch_stats(seg, 12) == (2, 8)
    assert oc.fetch_stats(seg) == (0, 0)


def test_fetched_high_watermark():
    a = mk(0, 0, [(o, TS0 + o, b"k", 1) for o in range(5)]).raw
    b = mk(0, 5, [(o, TS0 + o, b"k", 1) for o in (5, 7, 9)], last_delta=6).raw
    seg = a + b
    assert _offs(seg, None, 5) == [0, 1, 2, 3, 4]                   # H at a batch boundary
    assert _offs(seg, None, 3) == []                                # H inside a batch: the batch goes whole
    assert _offs(seg, None, 11) == [0, 1, 2, 3, 4]                  # H at `last` of the compacted batch
    assert _offs(seg, None, 12) == [0, 1, 2, 3, 4, 5, 7, 9]
    assert _offs(seg, 2, 5) == [2, 3, 4]
    assert oc.fetch_stats(seg, None, 3) == (2, 8)
    assert oc.fetch_stats(seg, 2, 5) == (1, 3 + 2)


def test_fetched_empty_and_control_batches_at_the_edges():
    empty = mk(0, 0, []).raw                                          # last = 0, no records
    ctrl = mk(0, 1, [(1, TS0, kc.marker_record_key(True), None)], attributes=0x30).raw
    data = mk(0, 2, [(o, TS0 + o, b"k", 1) for o in (2, 3)]).raw
    seg = empty + ctrl + data
    assert _offs(seg) == [2, 3]
    assert oc.fetch_stats(seg, 2) == (2, 0)                          # the empty and the control batch: no data records
    assert oc.fetch_stats(seg, 1) == (1, 0)
    assert oc.fetch_stats(seg, None, 2) == (1, 2)
    assert oc.fetch_stats(seg, None, 1) == (2, 2)
    assert _offs(seg, 3) == [3]


def test_with_last_offset_delta_changes_only_that_field():
    raw = mk(0, 100, [(100, TS0, b"k", 3), (104, TS0 + 1, None, None)]).raw
    assert struct.unpack(">i", raw[23:27])[0] == 4
    patched = oc.with_last_offset_delta(raw, 9)
    assert struct.unpack(">i", patched[23:27])[0] == 9 and patched[:23] == raw[:23] and patched[27:] == raw[27:]
    assert kc.read_segment(patched)[0].records == kc.read_segment(raw)[0].records


# ---- CPU: checkpoint files of the CLI --------------------------------------------------------------------------------
def _cli():
    from test_report import CLI_DIR, _build
    _build()
    return os.path.join(CLI_DIR, "kafka-topic-analyzer")


def _log_dir(tmp_path, topic="orders", parts=(0,)):
    for p in parts:
        d = tmp_path / ("%s-%d" % (topic, p))
        d.mkdir()
        (d / ("%020d.log" % 0)).write_bytes(mk(p, 0, [(o, TS0 + o, b"k", 1) for o in range(3)]).raw)
    return tmp_path


@pytest.mark.parametrize("name,text", [
    ("log-start-offset-checkpoint", "1\n1\norders 0 0\n"),                    # bad version
    ("log-start-offset-checkpoint", "0\n2\norders 0 0\n"),                    # count mismatch
    ("replication-offset-checkpoint", "0\n1\norders 0 0\norders 1 0\n"),     # count mismatch
    ("replication-offset-checkpoint", "0\n1\norders x 0\n"),                  # non-numeric partition
    ("replication-offset-checkpoint", "0\n1\norders 0 1x\n"),                 # non-numeric offset
    ("log-start-offset-checkpoint", "0\nfour\n"),                             # non-numeric count
    ("log-start-offset-checkpoint", ""),                                      # empty
])
def test_cli_rejects_a_malformed_checkpoint(tmp_path, name, text):
    cli = _cli()
    d = _log_dir(tmp_path)
    (d / name).write_text(text)
    r = subprocess.run([cli, "-t", "orders", "-b", "x", "--log-dir", str(d)], capture_output=True, text=True)
    assert r.returncode == 1 and name in r.stderr, (r.returncode, r.stderr)


def test_cli_help_names_the_checkpoint_files():
    r = subprocess.run([_cli(), "--help"], capture_output=True, text=True)
    assert "log-start-offset-checkpoint" in r.stdout + r.stderr and "replication-offset-checkpoint" in r.stdout + r.stderr


# ---- GPU ------------------------------------------------------------------------------------------------------------
def gen(seed, P=4, nb=30, codecs=CODECS):
    """P partitions with windows: partition 0 none, 1 a start only, 2 a watermark only, 3.. both, each drawn inside"""
    rng = np.random.default_rng(seed)
    parts, win = {}, {}
    for p in range(P):
        parts[p], end = gen_partition(rng, p, nb, codecs)
        lo, hi = int(rng.integers(0, end // 2)), int(rng.integers(end // 2, end + 1))
        if p == 1:
            win[p] = (lo, None)
        elif p == 2:
            win[p] = (None, hi)
        elif p >= 3:
            win[p] = (lo, hi)
    return parts, win


@pytest.mark.gpu
@pytest.mark.parametrize("entry", LOG_ENTRIES)
def test_entry_points(entry):
    parts, win = gen(21, P=5)
    with engine(5) as e:
        set_windows(e, win)
        n, order = scan_log(e, entry, parts)
        recs = check(e, order, win, 5, n)
        assert 0 < len(recs) < sum(len(kc.delivered(b.raw)) for b in order)


@pytest.mark.gpu
@pytest.mark.parametrize("entry", ["segments_host", "batches_device"])
@pytest.mark.parametrize("n", [1, 31, 32, 33, 100])
def test_start_at_every_record(entry, n):
    """partition p: batch A (offsets 0-6), batch B (n records from 7), batch C (3 records); S = 6 + p walks from inside A
    over every record of B to past it — every rank carry of the decode's lane rounds"""
    rng = np.random.default_rng(n)
    P = n + 3
    parts, win = {}, {}
    for p in range(P):
        parts[p] = [mk(p, 0, recs_at(range(0, 7), rng)), mk(p, 7, recs_at(range(7, 7 + n), rng)),
                    mk(p, 7 + n, recs_at(range(7 + n, 10 + n), rng))]
        win[p] = (6 + p, None)
    with engine(P) as e:
        set_windows(e, win)
        n_out, order = scan_log(e, entry, parts)
        check(e, order, win, P, n_out)


@pytest.mark.gpu
@pytest.mark.parametrize("in_place", [False, True], ids=["staged", "in_place"])
@pytest.mark.parametrize("codec", CODECS)
def test_cut_batches_in_every_codec(codec, in_place):
    rng = np.random.default_rng(CODECS.index(codec) * 2 + in_place)
    parts, win = {}, {}
    # 0: a plain cut batch; 1: a compacted cut batch, S in a gap; 2: a cut batch that keeps nothing (S past its last
    # record, not past `last`); 3: a cut batch of 100 records, S in its third lane round
    parts[0] = [mk(0, 0, recs_at(range(0, 40), rng), codec), mk(0, 40, recs_at(range(40, 50), rng), codec)]
    win[0] = (17, None)
    gaps = [0, 1, 4, 9, 10, 11, 20, 33, 34, 40]
    parts[1] = [mk(1, 0, recs_at(gaps, rng), codec, last_delta=45), mk(1, 46, recs_at(range(46, 50), rng), codec)]
    win[1] = (5, 48)
    parts[2] = [mk(2, 0, recs_at(range(0, 20), rng), codec, last_delta=25), mk(2, 26, recs_at(range(26, 30), rng), codec)]
    win[2] = (22, None)
    parts[3] = [mk(3, 0, recs_at(range(0, 100), rng), codec)]
    win[3] = (70, None)
    if in_place:   # an uncompressed batch past 48 KiB puts the whole decode in place
        parts[4] = [mk(4, 0, [(0, TS0, b"big", 60000), (1, TS0 + 1, b"k", 3)]), mk(4, 2, recs_at(range(2, 9), rng), codec)]
        win[4] = (1, None)
    P = len(parts)
    for entry in ("segments_host", "batches_device"):
        with engine(P) as e:
            set_windows(e, win)
            n, order = scan_log(e, entry, parts)
            check(e, order, win, P, n)


@pytest.mark.gpu
def test_high_watermark_at_and_inside_batches():
    rng = np.random.default_rng(5)
    parts, win = {}, {}
    for p, hi in enumerate((10, 5, 11, 0, 1)):
        parts[p] = [mk(p, 0, recs_at(range(0, 5), rng), "lz4"), mk(p, 5, recs_at(range(5, 10), rng)),
                    mk(p, 10, recs_at(range(10, 20), rng), "zstd")]
        win[p] = (None, hi)
    with engine(5) as e:
        set_windows(e, win)
        n, order = scan_log(e, "segments_host", parts)
        check(e, order, win, 5, n)


@pytest.mark.gpu
@pytest.mark.parametrize("entry", ["segment_host", "batches_device"])
def test_window_that_excludes_the_whole_call(entry):
    parts, _ = gen(7, P=2, nb=10)
    win = {0: (10 ** 6, None), 1: (None, 0)}
    with engine(2) as e:
        set_windows(e, win)
        n, order = scan_log(e, entry, parts)
        assert n == 0
        check(e, order, win, 2, n)
        assert e.message_metrics.overall_count() == 0


@pytest.mark.gpu
@pytest.mark.parametrize("in_place", [False, True], ids=["staged", "in_place"])
def test_many_partitions_each_cut(in_place):
    """about 20 000 partitions, each cut inside its first batch: every warp of the count pass and of the decode takes
    many cut batches"""
    rng = np.random.default_rng(9)
    P = 20000
    parts, win = {}, {}
    for p in range(P):
        n = 3 + p % 37
        parts[p] = [mk(p, 0, recs_at(range(0, n), rng, 5000, 20), crc=False),
                    mk(p, n, recs_at(range(n, n + 4), rng, 5000, 20), crc=False)]
        win[p] = (1 + p % n, None)
    if in_place:
        parts[0].append(mk(0, 100, [(100, TS0, b"big", 60000)], crc=False))
    with engine(P) as e:
        set_windows(e, win)
        n_out, order = scan_log(e, "batches_device", parts)
        check(e, order, win, P, n_out)


@pytest.mark.gpu
@pytest.mark.parametrize("entry", ["segments_host", "batches_device"])
@pytest.mark.parametrize("with_cut", [False, True], ids=["alone", "beside-a-cut-batch"])
def test_negative_offset_delta_at_the_log_start(entry, with_cut):
    """partition 1: S = 10 and a batch at baseOffset 10 with offset deltas [0, -3, 1] (no broker writes a negative delta).
    It is served and not cut, so it keeps all three records, whether or not partition 0 has a cut batch in the same call
    (records are dropped only from cut batches, kta_log_set_offsets)"""
    rng = np.random.default_rng(13)
    parts = {0: [mk(0, 0, recs_at(range(0, 10), rng))], 1: [mk(1, 10, recs_at([10, 7, 11], rng))]}
    win = {0: (5 if with_cut else 0, None), 1: (10, None)}
    with engine(2) as e:
        set_windows(e, win)
        n, order = scan_log(e, entry, parts)
        recs = check(e, order, win, 2, n)
        assert sum(r[0] == 1 for r in recs) == 3 and n == (8 if with_cut else 13)


@pytest.mark.gpu
def test_compaction_below_the_log_start():
    """-c: a key whose only live write lies below S is not alive; a tombstone inside the window over a live write below
    S leaves its key dead"""
    recs = [(0, TS0, b"only-below", 5), (1, TS0 + 1, b"tomb", 7), (2, TS0 + 2, b"x", 1), (3, TS0 + 3, b"tomb", None),
            (4, TS0 + 4, b"y", 2)]
    for codec in (None, "zstd"):
        parts = {0: [mk(0, 0, recs, codec)]}
        win = {0: (2, None)}
        with engine(1) as e:
            set_windows(e, win)
            n, order = scan_log(e, "segment_host", parts)
            check(e, order, win, 1, n)
            assert e.alive_keys() == 2                                  # x and y


@pytest.mark.gpu
@pytest.mark.parametrize("with_index", [False, True])
def test_abort_marker_above_the_watermark(with_index):
    txn = B(0, kc.set_crcs(kc.txn_batch(0, TS0, [(j, j, b"t%d" % j, 4) for j in range(5)], pid=7)))
    abort = B(0, kc.set_crcs(kc.marker(5, 7, 0, False, TS0 + 9)))
    plain = mk(0, 6, [(6, TS0 + 6, b"p", 1)])
    parts, win = {0: [txn, abort, plain]}, {0: (None, 5)}
    with engine(1, isolation_level="read_committed") as e:
        set_windows(e, win)
        if with_index:
            e.push_txn_index(0, kc.txn_index([(7, 0, 5)]))
        n, order = scan_log(e, "segment_host", parts)
        e.finalize()
        want = [] if with_index else [(0, ts, k, vl) for _, ts, k, vl in oc.fetched(txn.raw)]
        assert n == len(want)
        o = oracle_in_order(want)
        assert_parity(e, o, 1, check_alive=True, hll_regs=o.hll_alive_regs(10))
        assert e.log_offset_stats() == (2, 1)                          # the marker and `plain`; plain's record
        assert e.log_txn_stats() == ((1, 5, 0) if with_index else (0, 0, 5))


@pytest.mark.gpu
def test_aborted_transaction_that_starts_below_the_log_start():
    t1 = B(0, kc.set_crcs(kc.txn_batch(0, TS0, [(j, j, b"a%d" % j, 4) for j in range(5)], pid=9)))
    t2 = B(0, kc.set_crcs(kc.txn_batch(5, TS0, [(j, j, b"b%d" % j, 4) for j in range(5)], pid=9, base_seq=5)))
    abort = B(0, kc.set_crcs(kc.marker(10, 9, 0, False, TS0 + 20)))
    plain = mk(0, 11, [(o, TS0 + o, b"p%d" % o, 2) for o in (11, 12, 13)])
    parts, win = {0: [t1, t2, abort, plain]}, {0: (7, None)}
    with engine(1, isolation_level="read_committed") as e:
        set_windows(e, win)
        n, order = scan_log(e, "batches_device", parts)
        e.finalize()
        want = [(0, ts, k, vl) for _, ts, k, vl in oc.fetched(plain.raw, 7)]
        assert n == 3
        o = oracle_in_order(want)
        assert_parity(e, o, 1, check_alive=True, hll_regs=o.hll_alive_regs(10))
        assert e.log_offset_stats() == (1, 5)                          # t1; t2 is aborted whole, not cut
        assert e.log_txn_stats() == (1, 5, 0)


def damaged(b: B, at=17):
    raw = bytearray(b.raw)
    raw[at] ^= 1
    return B(b.p, bytes(raw), True)


@pytest.mark.gpu
@pytest.mark.parametrize("entry", ["segments_host", "batches_device"])
def test_check_crcs_counts_served_batches_only(entry):
    rng = np.random.default_rng(3)
    below = damaged(mk(0, 0, recs_at(range(0, 10), rng), "gzip"), at=70)     # not served: neither reported nor counted
    cut = damaged(mk(0, 10, recs_at(range(10, 20), rng)))                    # served and cut: skipped and listed
    ok = mk(0, 20, recs_at(range(20, 30), rng), "lz4")
    at_h = damaged(mk(0, 30, recs_at(range(30, 40), rng)))                   # at H: not served
    above = damaged(mk(0, 40, recs_at(range(40, 45), rng), "zstd"), at=64)
    p1 = [mk(1, 0, recs_at(range(0, 8), rng)), damaged(mk(1, 8, recs_at(range(8, 12), rng)))]
    parts = {0: [below, cut, ok, at_h, above], 1: p1}
    win = {0: (15, 39), 1: (4, None)}
    with engine(2, check_crcs=True) as e:
        set_windows(e, win)
        n, order = scan_log(e, entry, parts)
        check(e, order, win, 2, n)
        fails = e.log_crc_failures()
        assert sorted((f[0], f[2]) for f in fails) == [(0, 10), (1, 8)]
        assert e.log_crc_stats()[:2] == (4, 2)                          # cut, ok, and partition 1's two


def _one_call(e, entry, order):
    """the batches in the given order in one call: every partition's segment to kta_push_log_segments_host, or every batch
    (not interleaved) to kta_scan_log_batches_device"""
    from feed import scan_log_batches, stage_batches
    if entry == "segments_host":
        segs = {}
        for b in order:
            segs[b.p] = segs.get(b.p, b"") + b.raw
        return e.push_log_segments(list(segs.items()))
    return scan_log_batches(e, stage_batches([(b.p, b.raw) for b in order]))


def _check_crcs_call(entry, P, order, win):
    with engine(P, check_crcs=True) as e:
        set_windows(e, win)
        n = _one_call(e, entry, order)
        check(e, order, win, P, n)
        assert e.log_crc_failures() == []
        assert e.log_crc_stats() == (len(order) - e.log_offset_stats()[0], 0, 0)


@pytest.mark.gpu
@pytest.mark.parametrize("entry", ["segments_host", "batches_device"])
def test_check_crcs_across_a_partition_seam(entry):
    """check.crcs, one call: partition 0's 100 batches, then partition 1's 40 below its log start offset (no CRC spans) and
    its 100 served ones.  The span pass's warps each take 7 spans; the warp over the seam looks past the 32 batch ends behind
    its current batch (partition 1's first, empty ones) for the first five served batches of partition 1."""
    rng = np.random.default_rng(40)
    order = [mk(0, i, recs_at([i], rng)) for i in range(100)] + [mk(1, i, recs_at([i], rng)) for i in range(140)]
    _check_crcs_call(entry, 2, order, {1: (40, None)})


@pytest.mark.gpu
@pytest.mark.parametrize("entry", ["segments_host", "batches_device"])
def test_check_crcs_on_a_saturated_grid(entry):
    """check.crcs, one call of ~150 000 one-record batches in 1024 partitions, each partition's first two below its log start
    offset: the span pass's grid is capped at the SM count (more than 32 spans per warp), and gaps of two batches without
    spans sit at every partition seam.  The batches are tiled from 64 templates: baseOffset lies outside the CRC."""
    rng = np.random.default_rng(41)
    tmpl = [mk(0, 0, recs_at([0], rng)).raw for _ in range(64)]
    P, per_part = 1024, 150
    order = [B(p, struct.pack(">q", i) + tmpl[(p * 7 + i) % 64][8:]) for p in range(P) for i in range(per_part)]
    _check_crcs_call(entry, P, order, {p: (2, None) for p in range(P)})


@pytest.mark.gpu
def test_damage_inside_a_batch_that_is_not_served():
    rng = np.random.default_rng(4)
    for codec in ("gzip", "zstd", "lz4", None):
        bad = mk(0, 0, recs_at(range(0, 30), rng), codec)
        raw = bytearray(bad.raw)
        raw[61:len(raw) - 2] = bytes(len(raw) - 63)                     # the records section wiped
        parts = {0: [B(0, bytes(raw)), mk(0, 30, recs_at(range(30, 40), rng))]}
        win = {0: (35, None)}
        with engine(1) as e:
            set_windows(e, win)
            n, order = scan_log(e, "segment_device", parts)
            check(e, order, win, 1, n)
            e.reset()
            with pytest.raises(KtaError):                               # without the window the damage refuses the call
                scan_log(e, "segment_device", parts)


@pytest.mark.gpu
def test_reset_clears_windows_and_totals():
    parts, win = gen(8, P=4, nb=12)
    with engine(4) as e:
        set_windows(e, win)
        n, order = scan_log(e, "segments_host", parts)
        check(e, order, win, 4, n)
        assert e.log_offset_stats() != (0, 0)
        e.reset()
        assert e.log_offset_stats() == (0, 0)
        n, order = scan_log(e, "segments_host", parts)
        check(e, order, {}, 4, n)


@pytest.mark.gpu
def test_bad_arguments():
    with engine(3) as e:
        for args in ((-1, 0, 5), (3, 0, 5), (0, -2, 5), (0, 0, -2), (0, 6, 5)):
            with pytest.raises(KtaError) as ei:
                e.set_log_offsets(*args)
            assert ei.value.code == 1
        e.set_log_offsets(0, 5, 5)
        e.set_log_offsets(1, None, None)
        e.set_log_offsets(2, -1, 0)
        assert e.log_offset_stats() == (0, 0)


@pytest.mark.gpu
def test_windows_replaced_between_calls():
    parts, _ = gen(10, P=3, nb=15)
    wins = [{0: (5, None), 1: (None, 40)}, {0: (None, None), 1: (20, 60), 2: (3, 4)}, {}]
    with engine(3) as e:
        got, want, stats = 0, [], (0, 0)
        for w in wins:
            for p in range(3):
                lo, hi = w.get(p, (None, None))
                e.set_log_offsets(p, lo, hi)
            n, order = scan_log(e, "batches_device", parts)
            r, s = expect(order, w)
            got, want, stats = got + n, want + r, (stats[0] + s[0], stats[1] + s[1])
        e.finalize()
        assert got == len(want)
        o = oracle_in_order(want)
        assert_parity(e, o, 3, check_alive=True, hll_regs=o.hll_alive_regs(10))
        assert e.log_offset_stats() == stats


# ---- GPU: the CLI over a data directory with checkpoint files --------------------------------------------------------
def _write_topic(tmp_path, parts, topic="orders"):
    """each partition's batches as two segments named by their base offsets, as a broker names them"""
    for p, batches in parts.items():
        d = tmp_path / ("%s-%d" % (topic, p))
        d.mkdir()
        half = len(batches) // 2
        for chunk in (batches[:half], batches[half:]):
            if chunk:
                base = struct.unpack(">q", chunk[0].raw[:8])[0]
                (d / ("%020d.log" % base)).write_bytes(b"".join(b.raw for b in chunk))


def _checkpoint(path, entries):
    path.write_text("0\n%d\n" % len(entries) + "".join("%s %d %d\n" % e for e in entries))


def _run(cli, d, *opts):
    return subprocess.run([cli, "-t", "orders", "-b", "unused:9092", "-c", "--log-dir", str(d), *opts], capture_output=True, text=True)


def _rows(stdout):
    return {int(c[0]): c for c in ([x.strip() for x in l.strip("|").split("|")] for l in stdout.splitlines()
                                   if l.startswith("| ") and l[2].isdigit())}


def _without_duration(stdout):
    return [l for l in stdout.splitlines() if not l.startswith(("Scanning took", "Estimated Msg/s"))]


@pytest.mark.gpu
def test_cli_reads_the_checkpointed_window(tmp_path):
    rng = np.random.default_rng(17)
    P = 3
    parts = {}
    for p in range(P):
        parts[p], _ = gen_partition(rng, p, 12, codecs=(None, "lz4", "zstd"), max_n=30)
    _write_topic(tmp_path, parts)
    ends = {p: struct.unpack(">q", parts[p][-1].raw[:8])[0] + struct.unpack(">i", parts[p][-1].raw[23:27])[0] + 1 for p in parts}
    cli = _cli()
    plain = _run(cli, tmp_path)
    assert plain.returncode == 0, plain.stderr
    # a checkpoint that lists only another topic changes nothing
    _checkpoint(tmp_path / "log-start-offset-checkpoint", [("other", 0, 50), ("orders-x", 1, 9)])
    other = _run(cli, tmp_path)
    assert other.returncode == 0 and _without_duration(other.stdout) == _without_duration(plain.stdout)
    # partition 0: start inside its first segment; 1: a start below the first segment's base and a watermark past the
    # log end (clamped); 2: not listed, as before
    second = {p: struct.unpack(">q", parts[p][len(parts[p]) // 2].raw[:8])[0] for p in parts}
    _checkpoint(tmp_path / "log-start-offset-checkpoint", [("orders", 0, 7), ("orders", 1, 0), ("other", 2, 3)])
    _checkpoint(tmp_path / "replication-offset-checkpoint", [("orders", 0, ends[0] - 5), ("orders", 1, ends[1] + 100)])
    # move partition 1's first segment away: its log start is then raised to the second segment's base offset
    first1 = tmp_path / "orders-1" / ("%020d.log" % 0)
    first1.unlink()
    parts[1] = parts[1][len(parts[1]) // 2:]
    win = {0: (7, ends[0] - 5), 1: (second[1], ends[1])}
    r = _run(cli, tmp_path)
    assert r.returncode == 0, r.stderr
    order = [b for p in sorted(parts) for b in parts[p]]
    recs, _ = expect(order, win)
    o = oracle_in_order(recs)
    rows = _rows(r.stdout)
    assert sorted(rows) == [0, 1, 2]
    assert [int(rows[0][1]), int(rows[0][2])] == [7, ends[0] - 5]
    assert [int(rows[1][1]), int(rows[1][2])] == [second[1], ends[1]]
    assert [int(rows[2][1]), int(rows[2][2])] == [0, ends[2]]
    for p, c in rows.items():
        assert [int(c[3]), int(c[4]), int(c[5])] == [o.counter("total", p), o.counter("alive", p), o.counter("tombstones", p)]
        assert [int(c[7]), int(c[8]), int(c[10]), int(c[11])] == [o.counter("key_null", p), o.counter("key_non_null", p),
                                                                  o.counter("key_size_sum", p), o.counter("value_size_sum", p)]
    lines = r.stdout.splitlines()
    assert "Alive keys: %d" % o.scalar("sum_all_alive") in lines
    assert "Topic Size: %d bytes" % o.scalar("overall_size") in lines


@pytest.mark.gpu
def test_cli_watermarks_all_zero_is_no_content(tmp_path):
    rng = np.random.default_rng(18)
    parts = {p: gen_partition(rng, p, 4, codecs=(None,))[0] for p in range(2)}
    _write_topic(tmp_path, parts)
    _checkpoint(tmp_path / "replication-offset-checkpoint", [("orders", 0, 0), ("orders", 1, 0)])
    r = _run(_cli(), tmp_path)
    assert r.returncode == 254 and "no content" in r.stderr


@pytest.mark.gpu
def test_cli_check_crcs_across_a_partition_seam(tmp_path):
    """--log-dir with check.crcs=true: partition 0's 100 batches and partition 1's 140, the first 40 below the log start
    offset its checkpoint gives; every segment goes to the library in one call.  No batch fails its check."""
    rng = np.random.default_rng(19)
    parts = {0: [mk(0, i, recs_at([i], rng)) for i in range(100)], 1: [mk(1, i, recs_at([i], rng)) for i in range(140)]}
    _write_topic(tmp_path, parts)
    _checkpoint(tmp_path / "log-start-offset-checkpoint", [("orders", 1, 40)])
    r = _run(_cli(), tmp_path, "--librdkafka", "check.crcs=true")
    assert r.returncode == 0, r.stderr
    assert not [l for l in r.stderr.splitlines() if "CRC32C" in l]
    order = [b for p in sorted(parts) for b in parts[p]]
    recs, _ = expect(order, {1: (40, None)})
    assert len(recs) == 200
    o = oracle_in_order(recs)
    rows = _rows(r.stdout)
    for p, c in rows.items():
        assert [int(c[3]), int(c[4]), int(c[5])] == [o.counter("total", p), o.counter("alive", p), o.counter("tombstones", p)]
    assert "Alive keys: %d" % o.scalar("sum_all_alive") in r.stdout.splitlines()
