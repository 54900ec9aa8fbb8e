"""read_committed isolation of the log entry points (include/kta.h, kta_logtxn.cuh): records of aborted transactions are
left out, decided from the control markers in the same call and from the broker's .txnindex ranges.

The generator below writes transactional topics whose delivered records are known by construction (each transaction is
decided commit, abort or open before its batches are written).  A CPU test checks that set against a second model that
walks the encoded bytes as librdkafka does, driven by the aborted-transaction list; the GPU tests compare the engine
with the oracle fed only the delivered records."""
import struct
from dataclasses import dataclass, field
from typing import Optional

import numpy as np
import pytest

import kafka_codec as kc
from feed import LOG_ENTRIES, scan_log, scan_log_batches, stage_batches
from kafka_codec import marker, marker_record_key, txn_batch, txn_index, with_producer
from kafka_topic_analyzer_b200 import KtaEngine, KtaError
from parity import assert_parity, oracle_in_order

NOW = (4102444800, 123456789)
TS0 = 1_700_000_000_000


# ---- generator: topics with transactions decided by construction ----------------------------------------------------
@dataclass
class Bt:
    p: int
    off: int
    pid: int
    epoch: int
    txn: Optional[int]                         # transaction id, None = not transactional
    recs: list = field(default_factory=list)   # (ts, key, value_len)
    commit: Optional[bool] = None              # a marker: True COMMIT, False ABORT; None = data batch
    codec: Optional[str] = None
    raw: bytes = b""

    @property
    def is_marker(self):
        return self.commit is not None


@dataclass
class Topic:
    batches: dict            # partition -> [Bt] in offset order
    outcome: dict            # txn id -> "commit" | "abort" | "open"
    aborted: dict            # partition -> [(pid, firstOffset, lastOffset)] (the .txnindex entries)

    def truth(self, p):
        """partition p's delivered records: everything but control batches and the batches of aborted transactions"""
        return [r for b in self.batches[p] if not b.is_marker and (b.txn is None or self.outcome[b.txn] != "abort") for r in b.recs]

    def segment(self, p, lo=0, hi=None):
        return b"".join(b.raw for b in self.batches[p][lo:hi])


def _encode(b: Bt) -> bytes:
    if b.is_marker:
        return marker(b.off, b.pid, b.epoch, b.commit, TS0 + b.off)
    if not b.recs:
        return txn_batch(b.off, TS0 + b.off, [], b.pid, b.epoch, transactional=b.txn is not None)
    base = b.recs[0][0]
    return txn_batch(b.off, base, [(j, ts - base, k, vl) for j, (ts, k, vl) in enumerate(b.recs)], b.pid, b.epoch,
                     compression=b.codec, transactional=b.txn is not None)


def gen_topic(seed, P=3, pids=(11, 12, 13, 14, 15), steps=250, keys=40, codecs=("gzip", "lz4", "snappy")):
    """Every partition interleaves transactions of the same producer ids (so one id has different outcomes in different
    partitions) with non-transactional batches (producerId -1, or an id of the pool without the transactional bit).
    Transactions: 0..5 data batches (some without records), then a marker; aborts sometimes bump the epoch; some never
    get a marker (open)."""
    rng = np.random.default_rng(seed)
    batches, outcome, aborted = {}, {}, {}
    tid = 0
    for p in range(P):
        out, ab, off = [], [], 0
        epoch = {q: 0 for q in pids}
        cur = {}   # pid -> [txn id, fate, batches left, first data offset]

        def data(pid, txn, ep):
            nonlocal off
            n = 0 if rng.random() < 0.06 else int(rng.integers(1, 6))
            recs = []
            for j in range(n):
                k = None if rng.random() < 0.05 else b"key-%d" % int(rng.integers(0, keys))
                vl = None if rng.random() < 0.2 else int(rng.integers(0, 300))
                recs.append((TS0 + 10 * (off + j) + int(rng.integers(0, 7)), k, vl))
            codec = codecs[int(rng.integers(0, len(codecs)))] if (n and codecs and rng.random() < 0.25) else None
            b = Bt(p, off, pid, ep, txn, recs, None, codec)
            off += max(n, 1)
            out.append(b)
            return b

        for _ in range(steps):
            r = rng.random()
            if r < 0.15:
                data(-1 if rng.random() < 0.7 else int(rng.choice(pids)), None, 0)
                continue
            pid = int(rng.choice(pids))
            if pid not in cur:
                fate = rng.choice(["commit", "abort", "open"], p=[0.55, 0.35, 0.10])
                cur[pid] = [tid, str(fate), int(rng.integers(0, 6)), None]
                outcome[tid] = "open"   # until its marker is written
                tid += 1
            t = cur[pid]
            if t[2] > 0:
                b = data(pid, t[0], epoch[pid])
                t[3] = b.off if t[3] is None else t[3]
                t[2] -= 1
            elif t[1] == "open":
                data(-1, None, 0)       # an open transaction stays open: something else is written instead
            else:
                commit = t[1] == "commit"
                ep = epoch[pid]
                if not commit and rng.random() < 0.3:   # fenced: the coordinator aborts under a bumped epoch
                    ep += 1
                    epoch[pid] = ep
                out.append(Bt(p, off, pid, ep, t[0], [], commit))
                outcome[t[0]] = t[1]
                if not commit and t[3] is not None:
                    ab.append((pid, t[3], off))
                off += 1
                del cur[pid]
        for b in out:
            b.raw = _encode(b)
        batches[p], aborted[p] = out, ab
    return Topic(batches, outcome, aborted)


def rule_model(calls, ranges):
    """The rule of include/kta.h over calls (lists of Bt in call order) with the registered ranges {p: [(pid, first,
    last)]}: (delivered [(p, record)] in call order, (aborted batches, aborted records, undecided records))."""
    out, ab_b, ab_r, und = [], 0, 0, 0
    for call in calls:
        for i, b in enumerate(call):
            if b.is_marker:
                continue
            if b.txn is None or b.pid == -1:
                out += [(b.p, r) for r in b.recs]
                continue
            nxt = next((c for c in call[i + 1:] if c.is_marker and c.p == b.p and c.pid == b.pid), None)
            covered = any(q == b.pid and f <= b.off <= l for q, f, l in ranges.get(b.p, ()))
            if (nxt is not None and not nxt.commit) or covered:
                ab_b += 1
                ab_r += len(b.recs)
                continue
            if nxt is None:
                und += len(b.recs)
            out += [(b.p, r) for r in b.recs]
    return out, (ab_b, ab_r, und)


# ---- a second model: the bytes walked as librdkafka's read_committed consumer walks them ----------------------------
def librdkafka_walk(seg: bytes, aborted_txns):
    """A read_committed consumer over one partition's bytes, given the fetch response's aborted transactions [(pid,
    firstOffset)]: a transactional batch whose producer has a pending aborted transaction starting at or before it is
    skipped; that producer's next ABORT marker retires the transaction.  Returns the delivered (ts, key, value_len)."""
    pending = {}
    for pid, first in sorted(aborted_txns, key=lambda e: e[1]):
        pending.setdefault(pid, []).append(first)
    out = []
    for b in kc.read_segment(seg):
        waiting = pending.get(b.producer_id)
        if b.attributes & 0x20:
            # an ABORT marker retires the producer's pending aborted transaction that started before it
            if b.records and struct.unpack(">hh", b.records[0][2])[1] == 0 and waiting and waiting[0] <= b.base_offset:
                waiting.pop(0)
            continue
        if b.attributes & 0x10 and waiting and waiting[0] <= b.base_offset:
            continue
        out += [(ts, key, vl) for _, ts, key, vl in b.records]
    return out


# ---- CPU tests --------------------------------------------------------------------------------------------------------
def test_encoder_fields_and_index_image():
    plain = kc.encode_batch(7, TS0, [(0, 0, b"k", 3)])
    b = txn_batch(7, TS0, [(0, 0, b"k", 3)], pid=0x0102030405060708, epoch=9, base_seq=44)
    assert b[:21] == plain[:21] and b[23:43] == plain[23:43] and b[57:] == plain[57:]
    assert b[21:23] == b"\x00\x10" and struct.unpack(">qhi", b[43:57]) == (0x0102030405060708, 9, 44)
    m = marker(20, 5, 2, commit=False, ts=TS0)
    assert m[21:23] == b"\x00\x30" and struct.unpack(">qh", m[43:53]) == (5, 2)
    assert librdkafka_walk(m, []) == []
    img = txn_index([(5, 10, 20, 21), (6, 1, 2)])
    assert len(img) == 68 and struct.unpack(">hqqqq", img[:34]) == (0, 5, 10, 20, 21)


@pytest.mark.parametrize("seed", [1, 2, 3])
def test_generated_truth_matches_a_librdkafka_walk_of_the_bytes(seed):
    t = gen_topic(seed)
    assert set(t.outcome.values()) == {"commit", "abort", "open"}
    for p in t.batches:
        got = librdkafka_walk(t.segment(p), [(q, f) for q, f, _ in t.aborted[p]])
        assert got == t.truth(p)
        # and the rule of kta.h, one call per partition with every marker in it, delivers the same records
        assert [r for _, r in rule_model([t.batches[p]], {})[0]] == got


# ---- GPU tests --------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("entry", LOG_ENTRIES)
def test_four_entry_points(entry):
    """every marker in the call: the engine equals the oracle over the delivered records, for read_committed; the same
    bytes on a read_uncommitted handle deliver every data record, as before"""
    t = gen_topic(7, P=4)
    P = 4
    for level in ("read_committed", "read_uncommitted"):
        with KtaEngine(P, count_alive_keys=True, hll_precision=10, now=NOW, isolation_level=level) as e:
            total, order = scan_log(e, entry, t.batches)
            e.finalize()
            # the rule decides a batch by the later markers of its own partition in its call, so one call over `order`
            # stands for the one call per partition of segment_host and segment_device too
            want, stats = rule_model([order], {})
            assert sorted(map(repr, want)) == sorted(repr((p, r)) for p in range(P) for r in t.truth(p))
            assert stats[0] > 0 and stats[2] > 0
            exp = want if level == "read_committed" else [(b.p, r) for b in order if not b.is_marker for r in b.recs]
            o = oracle_in_order((p, *r) for p, r in exp)
            assert total == len(exp)
            assert_parity(e, o, P, check_alive=True, hll_regs=o.hll_alive_regs(10))
            if level == "read_committed":
                assert e.log_txn_stats() == stats
            else:
                with pytest.raises(KtaError):
                    e.log_txn_stats()


@pytest.mark.gpu
def test_markers_in_a_later_call_need_the_index():
    """each partition's log cut in two calls: transactions whose marker lies in the second call are undecided in the first
    (delivered: the result is wrong) unless the .txnindex ranges are registered (then it is exact)"""
    t = gen_topic(8, P=3, steps=300)
    P = 3
    cut = {p: len(t.batches[p]) // 2 for p in range(P)}
    calls = [[b for p in range(P) for b in t.batches[p][:cut[p]]], [b for p in range(P) for b in t.batches[p][cut[p]:]]]
    truth = [(p, r) for p in range(P) for r in t.truth(p)]
    for with_index in (False, True):
        ranges = t.aborted if with_index else {}
        want, stats = rule_model(calls, ranges)
        with KtaEngine(P, count_alive_keys=True, now=NOW, isolation_level="read_committed") as e:
            if with_index:
                for p in range(P):
                    e.push_txn_index(p, txn_index(t.aborted[p]))
            n = e.push_log_segments([(p, t.segment(p, 0, cut[p])) for p in range(P)])
            n += e.push_log_segments([(p, t.segment(p, cut[p])) for p in range(P)])
            e.finalize()
            o = oracle_in_order((p, *r) for p, r in want)
            assert n == len(want)
            assert_parity(e, o, P, check_alive=True)
            assert e.log_txn_stats() == stats
        if with_index:
            assert sorted(map(repr, want)) == sorted(map(repr, truth))
        else:
            assert len(want) > len(truth)          # aborted records of the first half were delivered
        assert stats[2] > 0


@pytest.mark.gpu
def test_same_producer_id_in_two_partitions_and_epoch_bump():
    """producer 77 aborts (under a bumped epoch) in partition 0 and commits in partition 1 in one call; a later transaction
    of the bumped epoch commits; an empty transaction and a zero-record batch change nothing"""
    seg0 = (txn_batch(0, TS0, [(0, 0, b"a", 1), (1, 1, b"b", 2)], pid=77, epoch=3)
            + txn_batch(2, TS0, [(0, 0, b"n", 5)], pid=-1, transactional=False)
            + marker(3, 77, 4, commit=False, ts=TS0)
            + txn_batch(4, TS0 + 4, [(0, 0, b"c", 3)], pid=77, epoch=4)
            + marker(5, 77, 4, commit=True, ts=TS0)
            + marker(6, 78, 0, commit=True, ts=TS0)                             # empty transaction
            + txn_batch(7, TS0 + 7, [], pid=78)                                 # zero records, then aborted
            + marker(8, 78, 0, commit=False, ts=TS0))
    seg1 = (txn_batch(0, TS0, [(0, 0, b"a", 7)], pid=77, epoch=3)
            + marker(1, 77, 3, commit=True, ts=TS0))
    want = [(0, TS0, b"n", 5), (0, TS0 + 4, b"c", 3), (1, TS0, b"a", 7)]
    with KtaEngine(2, count_alive_keys=True, now=NOW, isolation_level="read_committed") as e:
        assert e.push_log_segments([(0, seg0), (1, seg1)]) == 3
        e.finalize()
        assert_parity(e, oracle_in_order(want), 2, check_alive=True)
        assert e.log_txn_stats() == (2, 2, 0)


@pytest.mark.gpu
def test_aborted_overwrite_and_tombstone_do_not_win_the_alive_table():
    seg = (txn_batch(0, TS0, [(0, 0, b"k1", 5), (1, 1, b"k2", 5)], pid=-1, transactional=False)
           + txn_batch(2, TS0, [(0, 0, b"k1", None), (1, 0, b"k3", 4)], pid=9)      # tombstone of k1, new key k3: aborted
           + txn_batch(4, TS0, [(0, 0, b"k2", None)], pid=10)                      # tombstone of k2: committed
           + marker(5, 9, 0, commit=False, ts=TS0) + marker(6, 10, 0, commit=True, ts=TS0))
    with KtaEngine(1, count_alive_keys=True, now=NOW, isolation_level="read_committed") as e:
        assert e.push_log_segment(0, seg) == 3
        e.finalize()
        assert e.alive_keys() == 1                                                  # k1 only
        assert_parity(e, oracle_in_order([(0, TS0, b"k1", 5), (0, TS0 + 1, b"k2", 5), (0, TS0, b"k2", None)]), 1, check_alive=True)
    with KtaEngine(1, count_alive_keys=True, now=NOW) as e:
        assert e.push_log_segment(0, seg) == 5
        e.finalize()
        assert e.alive_keys() == 1                                                  # k3 only


@pytest.mark.gpu
def test_damaged_aborted_compressed_batch_is_left_out_unread():
    recs = [(i, i, b"key-%d" % i, 30) for i in range(40)]
    bad = bytearray(txn_batch(0, TS0, recs, pid=5, compression="gzip"))
    bad[75] ^= 0xFF                                                                 # inside the deflate stream
    seg = (bytes(bad) + txn_batch(40, TS0, recs[:3], pid=6, compression="lz4") + marker(43, 5, 0, False, ts=TS0)
           + marker(44, 6, 0, True, ts=TS0))
    with KtaEngine(1, now=NOW, isolation_level="read_committed") as e:
        assert e.push_log_segment(0, seg) == 3
        e.finalize()
        assert e.log_txn_stats() == (1, 40, 0)
    with KtaEngine(1, now=NOW) as e:
        with pytest.raises(KtaError):
            e.push_log_segment(0, seg)


@pytest.mark.gpu
def test_malformed_markers_order_and_indexes_are_refused():
    d = txn_batch(0, TS0, [(0, 0, b"k", 1)], pid=5)
    good = d + marker(1, 5, 0, True, ts=TS0)
    comp = bytearray(marker(1, 5, 0, True, ts=TS0))
    comp[22] |= 1                                                                   # a "gzip" control batch
    bad_markers = [
        bytes(comp),
        marker(1, 5, 0, True, ts=TS0, key=b"\x00\x00\x01"),                         # key length 3
        marker(1, 5, 0, True, ts=TS0, key=marker_record_key(True, version=1)),      # version 1
        with_producer(kc.encode_batch(1, TS0, [], attributes=0x30), 5),             # no record
    ]
    trunc = bytearray(marker(1, 5, 0, True, ts=TS0))
    trunc[61] = 0x7E                                                                # record length past the batch
    bad_markers.append(bytes(trunc))
    with KtaEngine(1, now=NOW, isolation_level="read_committed") as e:
        for m in bad_markers:
            with pytest.raises(KtaError):
                e.push_log_segment(0, d + m)
        with pytest.raises(KtaError):                                               # (5) offsets 10 then 0
            e.push_log_segment(0, txn_batch(10, TS0, [(0, 0, b"k", 1)], pid=5) + txn_batch(0, TS0, [(0, 0, b"k", 1)], pid=5))
        for img in (txn_index([(5, 0, 1)])[:-1], b"\x00\x01" + txn_index([(5, 0, 1)])[2:], txn_index([(5, 3, 1)])):
            with pytest.raises(KtaError):
                e.push_txn_index(0, img)
        e.push_txn_index(0, b"")                                                    # no aborted transaction: fine
        assert e.log_txn_stats() == (0, 0, 0)
        assert e.push_log_segment(0, good) == 1                                     # nothing of the refusals was kept
        e.finalize()
        assert e.message_metrics.overall_count() == 1
        # other producers, or the same producer in other partitions, may interleave freely
        assert e.push_log_segment(0, txn_batch(10, TS0, [(0, 0, b"k", 1)], pid=6) + txn_batch(0, TS0, [(0, 0, b"k", 1)], pid=5)) == 2
    with KtaEngine(1, now=NOW) as e:
        with pytest.raises(KtaError):
            e.push_txn_index(0, txn_index([(5, 0, 1)]))                              # read_uncommitted handle
        assert e.push_log_segment(0, d + bad_markers[1]) == 1                       # markers are not read there
    with pytest.raises(ValueError):
        KtaEngine(1, isolation_level="serializable")


@pytest.mark.gpu
def test_reset_clears_ranges_and_counters():
    seg = txn_batch(0, TS0, [(0, 0, b"k", 1), (1, 0, b"j", 2)], pid=5)              # its ABORT marker is elsewhere
    with KtaEngine(1, now=NOW, isolation_level="read_committed") as e:
        e.push_txn_index(0, txn_index([(5, 0, 2)]))
        assert e.push_log_segment(0, seg) == 0
        assert e.log_txn_stats() == (1, 2, 0)
        e.reset()
        assert e.log_txn_stats() == (0, 0, 0)
        assert e.push_log_segment(0, seg) == 2                                      # undecided now
        assert e.log_txn_stats() == (0, 0, 2)


@pytest.mark.gpu
def test_many_transactional_batches_in_one_call():
    """16 partitions x 256 producers, 8 transactions each of 4 single-record batches + marker, interleaved across producers
    (every producer has a transaction open at once): 2^17 transactional batches in one call, 1 in 10 transactions aborted;
    the sort, resolve and carry passes run over hundreds of tiles.  Its chains are at most 4 keys long and it stays inside
    one carry chunk; long transactions, chains across warps, tiles and carry chunks, and every array of the passes key by key
    are in tests/test_logtxn_passes.py"""
    P, PR, T = 16, 256, 8
    rng = np.random.default_rng(5)
    keys = [b"key-%d" % i for i in range(5000)]
    per, n_ab = [], 0
    for p in range(P):
        out, off = [], 0                       # (raw batch, delivered record or None)
        for t in range(T):
            abort = rng.random(PR) < 0.1
            kidx = rng.integers(0, len(keys), size=(4, PR))
            for step in range(5):
                for q in range(PR):
                    pid = ((q + 1) * 0x9E3779B97F4A7C15) & ((1 << 63) - 1)           # ids that use all 63 bits
                    if step < 4:
                        rec = (TS0 + off, keys[kidx[step, q]], int(kidx[step, q] % 97))
                        out.append((txn_batch(off, rec[0], [(0, 0, rec[1], rec[2])], pid=pid, epoch=t), None if abort[q] else rec))
                    else:
                        out.append((marker(off, pid, t, commit=not abort[q], ts=TS0), None))
                        n_ab += 4 * int(abort[q])
                    off += 1
        per.append(out)
    order = rng.permutation(P)                 # the partitions interleaved batch by batch, in a shuffled order
    inter = [(int(p), per[p][i]) for i in range(len(per[0])) for p in order]
    assert sum(1 for _, (raw, _r) in inter if raw[22] == 0x10) == 1 << 17
    want = [(p, *rec) for p, (_, rec) in inter if rec is not None]
    with KtaEngine(P, count_alive_keys=True, now=NOW, isolation_level="read_committed") as e:
        n = scan_log_batches(e, stage_batches([(p, raw) for p, (raw, _) in inter]))
        e.finalize()
        assert n == len(want)
        assert e.log_txn_stats() == (n_ab, n_ab, 0)
        assert_parity(e, oracle_in_order(want), P, check_alive=True)


@pytest.mark.gpu
def test_cli_isolation_level(tmp_path):
    """--log-dir over <topic>-<p>/ with .log and .txnindex files, two segments per partition (markers of the first
    segment's transactions partly in the second): read_committed prints the oracle over the committed records, the default
    the oracle over all records"""
    import os
    import subprocess
    from test_report import CLI_DIR, _build
    _build()
    P = 3
    t = gen_topic(12, P=P, steps=200)
    for p in range(P):
        d = tmp_path / ("orders-%d" % p)
        d.mkdir()
        half = len(t.batches[p]) // 2
        first_off = t.batches[p][half].off
        (d / "00000000000000000000.log").write_bytes(t.segment(p, 0, half))
        (d / ("%020d.log" % first_off)).write_bytes(t.segment(p, half))
        # the broker writes an aborted transaction into the index of the segment that holds its marker
        (d / "00000000000000000000.txnindex").write_bytes(txn_index([a for a in t.aborted[p] if a[2] < first_off]))
        (d / ("%020d.txnindex" % first_off)).write_bytes(txn_index([a for a in t.aborted[p] if a[2] >= first_off]))
    cli = os.path.join(CLI_DIR, "kafka-topic-analyzer")
    for opts, recs in (([], lambda p: [r for b in t.batches[p] if not b.is_marker for r in b.recs]),
                       (["--librdkafka", "isolation.level=read_committed"], t.truth)):
        r = subprocess.run([cli, "-t", "orders", "-b", "unused:9092", "-c", "--log-dir", str(tmp_path)] + opts,
                           capture_output=True, text=True)
        assert r.returncode == 0, r.stderr
        o = oracle_in_order([(p, *x) for p in range(P) for x in recs(p)])
        lines = r.stdout.splitlines()
        assert "Alive keys: %d" % o.scalar("sum_all_alive") in lines
        assert "Topic Size: %d bytes" % o.scalar("overall_size") in lines
        rows = [l for l in lines if l.startswith("| ") and l[2].isdigit()]
        assert len(rows) == P
        for l in rows:
            c = [x.strip() for x in l.strip("|").split("|")]
            p = int(c[0])
            assert [int(c[3]), int(c[4]), int(c[5])] == [o.counter("total", p), o.counter("alive", p), o.counter("tombstones", p)]
            assert [int(c[10]), int(c[11])] == [o.counter("key_size_sum", p), o.counter("value_size_sum", p)]
        assert ("warning:" in r.stderr) == bool(opts)                                # open transactions were counted
    r = subprocess.run([cli, "-t", "orders", "-b", "x", "--log-dir", str(tmp_path), "--librdkafka", "isolation.level=snapshot"],
                       capture_output=True, text=True)
    assert r.returncode != 0
