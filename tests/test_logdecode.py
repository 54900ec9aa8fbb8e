"""SURVEY.md §8 f2: Kafka RecordBatch v2 log segments decoded on the GPU and scanned, against the CPU oracle fed
with the same records (what librdkafka would have delivered message by message)."""
import numpy as np
import pytest

from feed import partition_lists, scan_log_batches, scan_log_segment, stage_batches
from kafka_topic_analyzer_b200 import KtaEngine, KtaError, synth
from oracle_lib import Oracle
from parity import assert_parity, expected, oracle_over
import kafka_codec as kc

NOW = (4102444800, 123456789)


def test_codec_varints_roundtrip():
    for n in (0, 1, -1, 63, 64, -64, -65, 300, -300, 2**31 - 1, -2**31, 2**40, -2**40):
        b = kc.varint(n)
        u, shift = 0, 0
        for x in b:
            u |= (x & 0x7F) << shift
            shift += 7
        assert ((u >> 1) ^ -(u & 1)) == n
    assert kc.varint(-1) == b"\x01" and kc.varint(0) == b"\x00" and kc.varint(1) == b"\x02"


def test_smallest_record_is_seven_bytes():
    """log_header_kernel bounds recordsCount by (batchLength - 49) / 7 before the output columns are sized."""
    assert len(kc.encode_record(0, 0, None, None)) == 7
    b = kc.encode_batch(5, 1000, [(i % 64, 0, None, None) for i in range(100)])      # one-byte varints only
    batch_len = int.from_bytes(b[8:12], "big")
    count = int.from_bytes(b[57:61], "big")
    assert count == 100 and count * 7 + 49 == batch_len == len(b) - 12


@pytest.mark.gpu
@pytest.mark.parametrize("key_mode,exact", [(0, True), (2, True), (1, False)])
def test_segments_decode_and_scan(key_mode, exact):
    rng = np.random.default_rng(3 + key_mode)
    P = 6
    spec = synth.make_spec(P * 1500, P, key_mode=key_mode, distinct_keys=600, tombstone_per_10k=2000, null_key_per_10k=400,
                           ts_missing_per_10k=300, empty_value_per_10k=200, value_mean=40)
    per = partition_lists(synth.fill_host(spec))
    o, kw = expected("exact" if exact else "hll", per, 10)
    with KtaEngine(P, count_alive_keys=exact, hll_precision=10, now=NOW) as e:
        total = 0
        for p in sorted(per):
            seg = kc.encode_partition(per[p], rng)
            total += e.push_log_segment(p, seg + b"\x00" * 17)      # + a truncated tail, as in a partial fetch
        e.finalize()
        assert total == spec.n_total
        assert_parity(e, o, P, **kw)


@pytest.mark.gpu
def test_log_append_time_control_batches_and_big_fields():
    rng = np.random.default_rng(9)
    big_key = bytes(rng.integers(0, 256, size=70_000, dtype=np.uint8))
    recs = [(1_700_000_000_123, b"a", 10), (1_700_000_000_456, None, None), (1_700_000_001_000, b"", 0),
            (1_700_000_002_000, big_key, 300_000), (1_600_000_000_000, b"a", None)]
    seg = kc.encode_batch(0, 1_700_000_000_000, [(i, r[0] - 1_700_000_000_000, r[1], r[2]) for i, r in enumerate(recs)])
    # a control batch (transaction marker) is never delivered to the application
    seg += kc.encode_batch(5, 1_700_000_003_000, [(0, 0, b"\x00\x00\x00\x01", 6)], attributes=0x20)
    # LogAppendTime: every record carries the batch's maxTimestamp
    seg += kc.encode_batch(6, 1_500_000_000_000, [(0, 5, b"b", 1), (1, 9, b"c", 2)], attributes=0x08, max_ts=1_800_000_000_999)
    o = Oracle(count_alive_keys=True, now=NOW)
    for ts, key, vl in recs:
        o.handle_message(2, ts, key, vl)
    o.handle_message(2, 1_800_000_000_999, b"b", 1)
    o.handle_message(2, 1_800_000_000_999, b"c", 2)
    with KtaEngine(4, count_alive_keys=True, now=NOW) as e:
        assert e.push_log_segment(2, seg) == 7
        e.finalize()
        assert_parity(e, o, 4, check_alive=True)
        assert e.message_metrics.latest_message() == 1_800_000_000


@pytest.mark.gpu
def test_compressed_and_malformed_batches_are_rejected():
    good = kc.encode_batch(0, 1000, [(0, 0, b"k", 1)])
    with KtaEngine(1, now=NOW) as e:
        with pytest.raises(KtaError):
            e.push_log_segment(0, kc.encode_batch(0, 1000, [(0, 0, b"k", 1)], attributes=0x04))   # zstd: no decompressor
        with pytest.raises(KtaError):
            e.push_log_segment(0, kc.encode_batch(0, 1000, [(0, 0, b"k", 1)], attributes=0x01))   # "gzip" that is not a gzip member
        bad = bytearray(good)
        bad[16] = 1                                                                              # magic 1
        with pytest.raises(KtaError):
            e.push_log_segment(0, bytes(bad))
        bad = bytearray(good)
        bad[61] = 0x7F                                                                           # record length beyond the batch
        with pytest.raises(KtaError):
            e.push_log_segment(0, bytes(bad))
        bad = bytearray(good)
        bad[57:61] = (0x7FFFFFFF).to_bytes(4, "big")                                             # recordsCount the batch cannot hold:
        with pytest.raises(KtaError):                                                            # rejected before any column is sized by it
            e.push_log_segment(0, bytes(bad))
        assert e.push_log_segment(0, good[:30]) == 0                                             # only a truncated header


@pytest.mark.gpu
def test_cli_log_dir(tmp_path):
    """The C++ CLI over a broker-style data directory: <topic>-<partition>/<base offset>.log, two segments per
    partition, -c.  The printed table must equal the oracle over the same records."""
    import os
    import subprocess
    from test_report import CLI_DIR, _build
    _build()
    rng = np.random.default_rng(21)
    P = 3
    spec = synth.make_spec(P * 2000, P, key_mode=1, distinct_keys=300, tombstone_per_10k=3000, value_mean=30)
    per = partition_lists(synth.fill_host(spec))
    for p, recs in per.items():
        d = tmp_path / ("orders-%d" % p)
        d.mkdir()
        half = len(recs) // 2
        (d / "00000000000000000000.log").write_bytes(kc.encode_partition(recs[:half], rng))
        second = bytearray()
        # second segment continues the offsets
        i = half
        while i < len(recs):
            chunk = recs[i:i + 25]
            second += kc.encode_batch(i, chunk[0][0], [(j, r[0] - chunk[0][0], r[1], r[2]) for j, r in enumerate(chunk)])
            i += len(chunk)
        (d / ("%020d.log" % half)).write_bytes(bytes(second))
        (d / "00000000000000000000.index").write_bytes(b"\x00" * 8)   # ignored
    (tmp_path / "other-0").mkdir()
    r = subprocess.run([os.path.join(CLI_DIR, "kafka-topic-analyzer"), "-t", "orders", "-b", "unused:9092", "-c", "--log-dir",
                        str(tmp_path)], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    o = oracle_over(per, count_alive_keys=True)
    lines = r.stdout.splitlines()
    assert "Alive keys: %d" % o.scalar("sum_all_alive") in lines
    assert "Topic Size: %d bytes" % o.scalar("overall_size") in lines
    rows = [l for l in lines if l.startswith("| ") and l[2].isdigit()]
    assert len(rows) == P
    for l in rows:
        c = [x.strip() for x in l.strip("|").split("|")]
        p = int(c[0])
        assert (int(c[1]), int(c[2])) == (0, len(per[p]))                     # start / end offsets from the batch headers
        assert [int(c[3]), int(c[4]), int(c[5])] == [o.counter("total", p), o.counter("alive", p), o.counter("tombstones", p)]
        assert [int(c[10]), int(c[11])] == [o.counter("key_size_sum", p), o.counter("value_size_sum", p)]


def test_cpp_segment_encoder_matches_the_topic():
    """kta_synth_encode_segment_host (the broker-format face of the synthetic topic) against fill_host.  Records without a
    timestamp, alone and inside batches that have one, read back as -1 (baseTimestamp + timestampDelta = -1)."""
    P = 8
    spec = synth.make_spec(P * 700, P, key_mode=2, distinct_keys=400, tombstone_per_10k=1500, null_key_per_10k=500,
                           ts_missing_per_10k=800)
    for p in (0, 5):
        got = [r for b in kc.read_segment(synth.encode_segment(spec, p, batch_records=33)) for r in b.records]
        t = synth.fill_host(spec, rank=p, world=P)              # partition p's records in offset order
        koff = np.concatenate([[0], np.cumsum(np.maximum(t.key_len, 0))])
        assert len(got) == t.n
        for i, (off, ts, key, vl) in enumerate(got):
            assert off == t.offset[i] and ts == t.ts_ms[i]
            assert key == (None if t.key_len[i] < 0 else t.key_bytes[koff[i]:koff[i] + t.key_len[i]].tobytes())
            assert vl == (None if t.value_len[i] < 0 else t.value_len[i])
        assert 0 < int((t.ts_ms == -1).sum()) < t.n


@pytest.mark.gpu
def test_synthetic_topic_with_missing_timestamps_as_log_segments():
    """A topic whose records lack timestamps here and there, encoded broker-style by kta_synth_encode_segment_host: the
    decoded log gives the oracle's answer over fill_host, its earliest message (-1 ms: a record without a timestamp)
    included."""
    P = 3
    spec = synth.make_spec(P * 3000, P, key_mode=2, distinct_keys=500, tombstone_per_10k=1500, ts_missing_per_10k=30)
    o = Oracle(count_alive_keys=True, now=NOW)
    with KtaEngine(P, count_alive_keys=True, now=NOW) as e:
        for p in range(P):
            t = synth.fill_host(spec, rank=p, world=P)
            o.handle_batch(t.partition, t.ts_ms, t.key_len, t.value_len, t.key_bytes)
            assert e.push_log_segment(p, synth.encode_segment(spec, p, batch_records=100)) == t.n
        e.finalize()
        assert e.message_metrics.earliest_message() == o.earliest()
        assert_parity(e, o, P, check_alive=True)


@pytest.mark.gpu
def test_synthetic_topic_as_log_segments_full_path():
    """configs[0]-sized topic stored broker-style (one segment per partition), decoded + scanned on the GPU with -c."""
    P = 4
    spec = synth.make_spec(100_000, P, distinct_keys=5000, tombstone_per_10k=1500)
    o = Oracle(count_alive_keys=True, now=NOW)
    with KtaEngine(P, count_alive_keys=True, hll_precision=11, now=NOW) as e:
        for p in range(P):
            t = synth.fill_host(spec, rank=p, world=P)
            o.handle_batch(t.partition, t.ts_ms, t.key_len, t.value_len, t.key_bytes)
            assert e.push_log_segment(p, synth.encode_segment(spec, p, batch_records=200)) == t.n
        e.finalize()
        assert_parity(e, o, P, check_alive=True, hll_regs=o.hll_alive_regs(11))
        # the same topic again, all partitions (two segments each) in ONE call
        e.reset()
        half = spec.n_total // P // 2
        segs = []
        for p in range(P):
            segs.append((p, synth.encode_segment(spec, p, 0, half, batch_records=57)))
            segs.append((p, synth.encode_segment(spec, p, half, None, batch_records=57)))
        assert e.push_log_segments(segs) == spec.n_total
        e.finalize()
        assert_parity(e, o, P, check_alive=True, hll_regs=o.hll_alive_regs(11))


@pytest.mark.gpu
@pytest.mark.parametrize("batch_records", [40, 300])
def test_device_entry_points_one_buffer_many_partitions(batch_records):
    """kta_scan_log_batches_device: the batches of all partitions in ONE device buffer, decoded and scanned in one go; and
    kta_scan_log_segment_device per partition.  40 records per batch (≈ 12 KB: staged in shared memory by a bulk copy) and 300
    (≈ 90 KB: read in place); the buffer has no slack behind its last byte, so the last batch is read in place too."""
    P = 5
    spec = synth.make_spec(P * 12_000, P, distinct_keys=3000, tombstone_per_10k=2000, key_mode=1)
    o = Oracle(count_alive_keys=True, now=NOW)
    segs = []
    for p in range(P):
        t = synth.fill_host(spec, rank=p, world=P)
        o.handle_batch(t.partition, t.ts_ms, t.key_len, t.value_len, t.key_bytes)
        segs.append((p, synth.encode_segment(spec, p, batch_records=batch_records)))
    staged = stage_batches(segs)              # packed back to back: batches start at arbitrary alignments
    assert staged[0].numel() == staged[1] == sum(s.size for _, s in segs)
    with KtaEngine(P, count_alive_keys=True, hll_precision=10, now=NOW) as e:
        assert scan_log_batches(e, staged) == spec.n_total
        e.finalize()
        assert_parity(e, o, P, check_alive=True, hll_regs=o.hll_alive_regs(10))
        # partition by partition through the single-partition entry point: the result is the same
        e.reset()
        for p, s in segs:
            assert scan_log_segment(e, p, s) == spec.n_total // P
        e.finalize()
        assert_parity(e, o, P, check_alive=True, hll_regs=o.hll_alive_regs(10))


def test_codec_compression_roundtrips_on_the_host():
    """The test encoder's compressed sections are what they claim (pyarrow decompresses them back): LZ4 frame magic, raw
    Snappy, xerial framing."""
    import pyarrow as pa
    recs = b"".join(kc.encode_record(i, i, b"key-%d" % (i % 7), 40 + i % 5) for i in range(300))
    lz = kc.compress_records(recs, "lz4")
    assert lz[:4] == bytes([0x04, 0x22, 0x4D, 0x18]) and len(lz) < len(recs)
    assert pa.decompress(lz, decompressed_size=len(recs), codec="lz4", asbytes=True) == recs
    gz = kc.compress_records(recs, "gzip")
    import gzip
    assert gz[:3] == b"\x1f\x8b\x08" and gzip.decompress(gz) == recs and len(gz) < len(recs)
    sn = kc.compress_records(recs, "snappy")
    assert pa.decompress(sn, decompressed_size=len(recs), codec="snappy", asbytes=True) == recs
    xe = kc.compress_records(recs, "snappy-xerial")
    assert xe[:8] == b"\x82SNAPPY\x00"
    b = kc.encode_batch(5, 1000, [(0, 0, b"k", 3)], compression="lz4")
    assert b[22] & 7 == 3 and int.from_bytes(b[8:12], "big") == len(b) - 12


@pytest.mark.gpu
@pytest.mark.parametrize("codec", ["gzip", "lz4", "snappy", "snappy-xerial", "mixed"])
def test_compressed_segments_decode_and_scan(codec):
    """gzip, LZ4 (frame) and Snappy (raw / xerial) batches — what producers with compression.type set write and librdkafka
    decompresses inside poll (src/kafka.rs:93) — are decompressed on the GPU and then give the reference's answer.
    'mixed': every batch picks its own codec, uncompressed ones included, in one segment."""
    rng = np.random.default_rng(11)
    P = 5
    spec = synth.make_spec(P * 4000, P, key_mode=1, distinct_keys=900, tombstone_per_10k=2000, null_key_per_10k=300,
                           empty_value_per_10k=100, value_mean=120)
    per = partition_lists(synth.fill_host(spec))
    o = oracle_over(per, count_alive_keys=True)
    comp = ["gzip", "lz4", "snappy", "snappy-xerial", None] if codec == "mixed" else codec
    with KtaEngine(P, count_alive_keys=True, hll_precision=10, now=NOW) as e:
        total = 0
        raw = comp_bytes = 0
        for p in sorted(per):
            seg = kc.encode_partition(per[p], rng, max_batch=200, compression=comp)
            raw += len(kc.encode_partition(per[p], np.random.default_rng(1), max_batch=200))
            comp_bytes += len(seg)
            total += e.push_log_segment(p, seg)
        e.finalize()
        assert total == spec.n_total and comp_bytes < raw            # it really was compressed
        assert_parity(e, o, P, check_alive=True, hll_regs=o.hll_alive_regs(10))
        # all partitions in one call too
        e.reset()
        rng = np.random.default_rng(12)
        assert e.push_log_segments([(p, kc.encode_partition(per[p], rng, max_batch=64, compression=comp)) for p in sorted(per)]) == spec.n_total
        e.finalize()
        assert_parity(e, o, P, check_alive=True, hll_regs=o.hll_alive_regs(10))


@pytest.mark.gpu
def test_corrupt_compressed_batches_are_rejected():
    recs = [(i, i, b"key-%d" % (i % 5), 30) for i in range(50)]
    with KtaEngine(1, now=NOW) as e:
        for codec in ("gzip", "lz4", "snappy"):
            good = kc.encode_batch(0, 1000, recs, compression=codec)
            assert e.push_log_segment(0, good) == 50
            bad = bytearray(good)
            bad[61] ^= 0x15                          # gzip / LZ4: the magic; Snappy: the uncompressed-length preamble
            with pytest.raises(KtaError):
                e.push_log_segment(0, bytes(bad))
            cut = bytearray(good[:-7])               # shorter section under an adjusted batchLength
            cut[8:12] = (len(cut) - 12).to_bytes(4, "big")
            with pytest.raises(KtaError):
                e.push_log_segment(0, bytes(cut))
        with pytest.raises(KtaError):                # zstd: no decompressor
            e.push_log_segment(0, kc.encode_batch(0, 1000, recs[:2], attributes=kc.CODEC_BITS["zstd"]))
        # gzip: damage inside the deflate stream or a wrong ISIZE must be caught, not written past the scratch slot
        good = kc.encode_batch(0, 1000, recs, compression="gzip")
        for at, x in ((75, 0xFF), (len(good) - 1, 0x01), (len(good) - 4, 0x40)):
            bad = bytearray(good)
            bad[at] ^= x
            with pytest.raises(KtaError):
                e.push_log_segment(0, bytes(bad))
        assert e.push_log_segment(0, good) == 50
