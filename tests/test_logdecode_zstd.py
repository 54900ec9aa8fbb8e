"""zstd record batches (codec 4) decompressed on the GPU (csrc/kta_zstd.cuh) and then decoded and scanned: against the CPU
oracle fed with the same records, through every log-segment entry point, from ~16 KB batches up to one of about 1 MiB."""
import os
import subprocess
from types import SimpleNamespace

import numpy as np
import pytest

from feed import partition_lists, scan_log
from kafka_topic_analyzer_b200 import KtaEngine, KtaError, synth
from parity import assert_parity, oracle_over
import kafka_codec as kc

NOW = (4102444800, 123456789)
MIXED = ["zstd", "zstd-stream", "gzip", "lz4", "snappy", None]


def _check_all_entry_points(P, per, segs, hll_p=10):
    """push_log_segment per partition, push_log_segments in one call, scan_log_batches_device over one device buffer"""
    o = oracle_over(per, count_alive_keys=True)
    n = sum(len(v) for v in per.values())
    parts = {p: [SimpleNamespace(p=p, raw=s)] for p, s in segs}      # each segment as it is
    with KtaEngine(P, count_alive_keys=True, hll_precision=hll_p, now=NOW) as e:
        for entry in ("segment_host", "segments_host", "batches_device"):
            e.reset()
            assert scan_log(e, entry, parts)[0] == n
            e.finalize()
            assert_parity(e, o, P, check_alive=True, hll_regs=o.hll_alive_regs(hll_p))


@pytest.mark.gpu
@pytest.mark.parametrize("codec", ["zstd", "zstd-stream", "mixed"])
def test_zstd_segments_decode_and_scan(codec):
    """one-shot frames (with Frame_Content_Size), streaming frames (without), and a mix in which every batch picks zstd,
    gzip, LZ4, Snappy or none"""
    rng = np.random.default_rng(31)
    P = 5
    spec = synth.make_spec(P * 4000, P, key_mode=1, distinct_keys=900, tombstone_per_10k=2000, null_key_per_10k=300,
                           empty_value_per_10k=100, value_mean=120)
    per = partition_lists(synth.fill_host(spec))
    # every partition's batch sizes are drawn before their codecs
    pick = (lambda: MIXED[int(rng.integers(0, len(MIXED)))]) if codec == "mixed" else (lambda: codec)
    segs = [(p, kc.recompress(kc.encode_partition(per[p], rng, max_batch=200), pick)) for p in sorted(per)]
    raw = sum(len(kc.encode_partition(per[p], np.random.default_rng(1), max_batch=200)) for p in per)
    assert sum(len(s) for _, s in segs) < raw                       # it really was compressed
    if codec != "mixed":
        assert all(s[22] & 7 == 4 for _, s in segs)
    _check_all_entry_points(P, per, segs)


def _fixed_batches(recs, per_batch, codec):
    out, i = bytearray(), 0
    while i < len(recs):
        chunk = recs[i:i + per_batch]
        base_ts = chunk[0][0]
        out += kc.encode_batch(i, base_ts, [(j, r[0] - base_ts, r[1], r[2]) for j, r in enumerate(chunk)], compression=codec)
        i += len(chunk)
    return bytes(out)


@pytest.mark.gpu
@pytest.mark.parametrize("codec", ["zstd", "zstd-stream"])
def test_large_zstd_batches(codec):
    """batches whose records exceed 48 KiB (decoded unstaged), 128 KiB (several zstd blocks) and one of about 1 MiB (Kafka's
    default message.max.bytes)"""
    P = 3
    spec = synth.make_spec(P * 9000, P, key_mode=1, distinct_keys=4000, tombstone_per_10k=1500, value_mean=120)
    per = partition_lists(synth.fill_host(spec))
    sizes = {0: 450, 1: 1100, 2: 9000}                             # records per batch: ~60 KB, ~150 KB, ~1.1 MB
    segs = []
    for p in sorted(per):
        seg = _fixed_batches(per[p], sizes[p], codec)
        segs.append((p, seg))
    big = _fixed_batches(per[2], sizes[2], None)
    assert len(big) > 1_000_000 and len(kc.batch_offsets(big)) == 1
    assert len(_fixed_batches(per[0][:450], 450, None)) > 48 * 1024
    assert len(_fixed_batches(per[1][:1100], 1100, None)) > 128 * 1024
    _check_all_entry_points(P, per, segs)


@pytest.mark.gpu
def test_corrupt_zstd_batches_are_rejected():
    recs = [(i, i, b"key-%d" % (i % 5), 30) for i in range(50)]
    with KtaEngine(1, now=NOW) as e:
        good = kc.encode_batch(0, 1000, recs, compression="zstd")
        assert good[61:65] == b"\x28\xb5\x2f\xfd" and good[65] >> 6 == 1          # one-shot: a 2-byte Frame_Content_Size
        assert e.push_log_segment(0, good) == 50
        bad = bytearray(good)
        bad[61] ^= 0x15                                                           # the magic
        with pytest.raises(KtaError):
            e.push_log_segment(0, bytes(bad))
        for codec in ("zstd", "zstd-stream"):
            g = kc.encode_batch(0, 1000, recs, compression=codec)
            cut = bytearray(g[:-7])                                               # shorter section under an adjusted batchLength
            cut[8:12] = (len(cut) - 12).to_bytes(4, "big")
            with pytest.raises(KtaError):
                e.push_log_segment(0, bytes(cut))
        for d in (1, -1):                                                         # Frame_Content_Size off by one
            bad = bytearray(good)
            fcs = int.from_bytes(bad[66:68], "little") + d
            bad[66:68] = fcs.to_bytes(2, "little")
            with pytest.raises(KtaError):
                e.push_log_segment(0, bytes(bad))
        for codec in ("zstd", "zstd-stream"):                                     # recordsCount the section cannot hold
            bad = bytearray(kc.encode_batch(0, 1000, recs, compression=codec))
            bad[57:61] = (0x7FFFFFFF).to_bytes(4, "big")
            with pytest.raises(KtaError):
                e.push_log_segment(0, bytes(bad))
        with pytest.raises(KtaError):                                             # zstd bits over uncompressed records
            e.push_log_segment(0, kc.encode_batch(0, 1000, recs, attributes=4))
        with pytest.raises(KtaError):                                             # an unassigned codec
            e.push_log_segment(0, kc.encode_batch(0, 1000, recs, attributes=5))
        e.reset()
        assert e.push_log_segment(0, good) == 50                                  # the handle still works
        e.finalize()
        assert e.message_metrics.overall_count() == 50


@pytest.mark.gpu
def test_cli_log_dir_zstd(tmp_path):
    """The C++ CLI over a broker-style data directory of zstd segments (one-shot and streaming batches) prints the same
    report as over the same topic uncompressed."""
    from test_report import CLI_DIR, _build
    _build()
    rng = np.random.default_rng(23)
    P = 3
    spec = synth.make_spec(P * 2000, P, key_mode=1, distinct_keys=300, tombstone_per_10k=3000, value_mean=30)
    per = partition_lists(synth.fill_host(spec))
    reports = []
    for comp in (None, ["zstd", "zstd-stream"]):
        root = tmp_path / ("zstd" if comp else "plain")
        for p, recs in per.items():
            d = root / ("orders-%d" % p)
            d.mkdir(parents=True)
            rng = np.random.default_rng(p)
            seg = kc.encode_partition(recs, rng)
            if comp:
                seg = kc.recompress(seg, lambda: comp[int(rng.integers(0, len(comp)))])
            (d / "00000000000000000000.log").write_bytes(seg)
        r = subprocess.run([os.path.join(CLI_DIR, "kafka-topic-analyzer"), "-t", "orders", "-b", "unused:9092", "-c", "--log-dir",
                            str(root)], capture_output=True, text=True)
        assert r.returncode == 0, r.stderr
        reports.append(r.stdout.splitlines())
    plain, zstd = reports
    o = oracle_over(per, count_alive_keys=True)
    assert "Alive keys: %d" % o.scalar("sum_all_alive") in zstd
    rows = [l for l in zstd if l.startswith("| ") and l[2].isdigit()]
    assert len(rows) == P
    for l in rows:
        c = [x.strip() for x in l.strip("|").split("|")]
        p = int(c[0])
        assert [int(c[3]), int(c[4]), int(c[5])] == [o.counter("total", p), o.counter("alive", p), o.counter("tombstones", p)]
    assert zstd == plain
