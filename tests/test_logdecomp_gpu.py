"""The GPU decompression stage of the RecordBatch decoder (log_decompress_kernel: gzip, LZ4, Snappy, zstd; one warp per batch,
32 lanes sharing the copies, the Huffman table fill and the Huffman streams) against the reference codecs, byte for byte.

tests/native/log_probe.cu runs scan_log_batches' steps (kta_logscan.cuh) through the size and copy steps, and returns every
batch's rewritten image.  For every batch that image must equal the same batch encoded
uncompressed (kafka_codec: byte-identical apart from batchLength and the codec bits), and its scratch slot must be that
length rounded up to 16.  The host tests run the same walks with one lane; the scan afterwards never reads value bytes,
header bytes or offset deltas, so this is where the lane-split output is checked.  Damaged sections must be accepted or
rejected as the host walks (one lane) accept or reject them, with the same bytes.  One more test sends batches whose every
decompressed byte the scan sees is a key byte through the product's entry points and compares the per-record key hashes."""
import gzip
import zlib

import numpy as np
import pytest

import codec_harness as ch
import kafka_codec as kc
import log_probe
import native_build
import np_oracle
import test_inflate_host as ih
import test_lzwalk_host as lh
import test_zstd_host as zh
from feed import capture_hashes, scan_log_batches, stage_batches
from kafka_codec import with_section
from parity import assert_parity, oracle_over

NOW = (4102444800, 123456789)
LOGB_OK, LOGB_BAD = 0, 2
STRATEGIES = (zlib.Z_DEFAULT_STRATEGY, zlib.Z_FIXED, zlib.Z_HUFFMAN_ONLY, zlib.Z_RLE, zlib.Z_FILTERED)


def decompress(segments):
    """segments: list of bytes (whole record batches each, found by the host walk; one call per segment, in a buffer with 64
    bytes of slack), the size and copy steps run even where the library stops before or between them → per segment, per
    batch (flags, slot size, image)"""
    res = []
    for seg, r in zip(segments, log_probe.run([log_probe.inputs(s, slack=64, decompress=True) for s in segments])):
        assert r.get("info") is not None, (r.rc, r.msg)
        slot, unc_at = np.diff(r.slot.astype(np.int64)), int(r.unc_at[0])
        batches = []
        for bi, size in zip(r.info, slot):
            n = int(bi["len"]) if bi["flags"] == LOGB_OK else 0
            at = (int(bi["off"]) - unc_at) % (1 << 64) if size else int(bi["off"])   # (a decompressed image lies in the scratch)
            batches.append((int(bi["flags"]), int(size), bytes((r.unc if size else np.frombuffer(seg, np.uint8))[at:at + n])))
        res.append(batches)
    return res


# ------------------------------------------------------------------------------------------------
# batches
# ------------------------------------------------------------------------------------------------
def payload_batch(data):
    """a batch whose records section is `data` as it is, recordsCount 0 (the decompression stage does not parse records)"""
    return with_section(kc.encode_batch(0, 1000, []), data, 0)


def records_batch(records, base_offset=0, base_ts=1_700_000_000_000):
    """records: (key, value, headers) → kafka_codec.encode_batch with explicit value bytes"""
    return kc.encode_batch(base_offset, base_ts, [(i, i * 3, k, None, h, v) for i, (k, v, h) in enumerate(records)])


def gz(data, level=6, strategy=zlib.Z_DEFAULT_STRATEGY):
    return ih.gz(data, level, strategy)


def compressors(data, zstd_levels=range(-5, 23)):
    """(name, codec bits, section) for every codec and setting the corpus uses"""
    out = [("gzip-%d-%d" % (lvl, st), 1, gz(data, lvl, st)) for lvl in (0, 1, 6, 9) for st in STRATEGIES]
    out.append(("gzip-python", 1, gzip.compress(data, mtime=0)))
    if data:                                           # (pyarrow's LZ4 and Snappy writers take no empty input)
        out += [("lz4", 3, kc.compress_records(data, "lz4")), ("snappy", 2, kc.compress_records(data, "snappy")),
                ("snappy-xerial", 2, kc.compress_records(data, "snappy-xerial"))]
    for lvl in zstd_levels:
        f = zh.one_shot(data, lvl)
        out.append(("zstd-%d" % lvl, 4, f))
        if lvl in zh.LEVELS:
            out.append(("zstd-%d-no-fcs" % lvl, 4, zh.without_content_size(f)))
    out.append(("zstd-stream", 4, kc.compress_records(data, "zstd-stream")))
    return out


def all_codecs(name, unc, zstd_levels=range(-5, 23)):
    """(name, compressed batch, expected image) for every codec and setting, from one uncompressed batch"""
    section = unc[61:]
    return [("%s/%s" % (name, cname), with_section(unc, c, bits), unc) for cname, bits, c in compressors(section, zstd_levels)]


def text_bytes(rng, n):
    words = [b"customer", b"order", b"status", b"shipped", b"\"id\":", b"{", b"}", b", ", b"2026-10-15T", b"EUR", b"\n"]
    out = bytearray()
    while len(out) < n:
        out += words[int(rng.integers(0, len(words)))] + b"%d" % int(rng.integers(0, 10 ** int(rng.integers(1, 7))))
    return bytes(out[:n])


def run_bytes(rng, n):
    out = bytearray()
    while len(out) < n:
        out += bytes([int(rng.integers(0, 256))]) * int(rng.integers(1, 200))
    return bytes(out[:n])


def record_corpus():
    """record sections whose values and headers carry real bytes: random, text-like, run-heavy"""
    rng = np.random.default_rng(41)
    kinds = {"random": lambda n: rng.integers(0, 256, n, dtype=np.uint8).tobytes(), "text": lambda n: text_bytes(rng, n),
             "runs": lambda n: run_bytes(rng, n)}
    out = []
    for kname, make in kinds.items():
        recs = []
        for i in range(200):
            hdrs = tuple((make(int(rng.integers(1, 12))), None if i % 5 == 0 else make(int(rng.integers(0, 40))))
                         for _ in range(int(rng.integers(0, 3))))
            key = None if i % 11 == 0 else make(int(rng.integers(0, 30)))
            out_v = None if i % 13 == 0 else make(int(rng.integers(0, 600)))
            recs.append((key, out_v, hdrs))
        out += all_codecs("records-" + kname, records_batch(recs))
    return out


def lane_corpus():
    """periodic data (matches with offset k, shorter than the warp for k < 32), literal runs around 32 and 64 bytes between
    matches, long zero runs, incompressible data (stored / raw blocks)"""
    rng = np.random.default_rng(43)
    out = []
    for k in list(range(1, 41)) + [63, 64, 65, 200]:
        data = (rng.integers(0, 256, k, dtype=np.uint8).tobytes() * (3000 // k + 2))[:3000 + k]
        out += all_codecs("period-%d" % k, records_batch([(b"k", data, ())]), zstd_levels=(-5, 1, 3, 19))
    marker = b"<<--kafka-topic-analyzer-marker-->>"
    for run in (31, 32, 33, 63, 64, 65):
        data = b"".join(rng.integers(0, 256, run, dtype=np.uint8).tobytes() + marker for _ in range(120))
        out += all_codecs("literals-%d" % run, records_batch([(b"k", data, ())]), zstd_levels=(-5, 1, 3, 19))
    out += all_codecs("zeros", records_batch([(b"z", bytes(300_000), ()), (None, b"x" + bytes(70_000) + b"y", ())]),
                      zstd_levels=(-5, 3, 19))
    out += all_codecs("random", records_batch([(b"r", rng.integers(0, 256, 100_000, dtype=np.uint8).tobytes(), ())]),
                      zstd_levels=(-5, 3, 19))
    return out


def size_corpus():
    """zstd over several 128 KiB blocks with matches across block boundaries, LZ4 over several 64 KiB blocks, gzip distances
    near 32 KiB, a batch of about 1 MiB, an empty and a one-byte records section"""
    rng = np.random.default_rng(47)
    out = []
    chunk = rng.integers(0, 256, 50_000, dtype=np.uint8).tobytes()
    blocks = records_batch([(b"b", chunk * 9, ())])                                 # 450 KB: offset 50 000 across blocks
    out += all_codecs("blocks", blocks, zstd_levels=(-5, 1, 3, 9, 19))
    for dist in (32_700, 32_767, 32_768):
        data = rng.integers(0, 256, dist, dtype=np.uint8).tobytes()
        unc = records_batch([(b"d", data * 3, ())])
        out += [("distance-%d/gzip-%d" % (dist, lvl), with_section(unc, gz(unc[61:], lvl), 1), unc) for lvl in (1, 6, 9)]
    big = records_batch([(b"key-%d" % i, text_bytes(rng, int(rng.integers(500, 1500))), ()) for i in range(1000)])
    assert 900_000 < len(big) < 1_400_000
    out += all_codecs("1mib", big, zstd_levels=(-5, 1, 3, 19))
    out += all_codecs("empty", payload_batch(b""))
    out += all_codecs("one-byte", payload_batch(b"\x00"))
    return out


def host_corpus():
    """the inputs of the host tests (one lane there, 32 lanes here) and the hand-assembled zstd frames"""
    out = [("zstd-host-%d" % i, with_section(payload_batch(b""), f, 4), payload_batch(want)) for i, (f, want) in enumerate(zh.corpus())]
    for name, data in ih.payloads().items():
        unc = payload_batch(data)
        out += [("inflate-%s/%d-%d" % (name, lvl, st), with_section(unc, gz(data, lvl, st), 1), unc) for lvl in (0, 1, 6, 9) for st in STRATEGIES]
        out.append(("inflate-%s/python" % name, with_section(unc, gzip.compress(data, mtime=0), 1), unc))
        out.append(("inflate-%s/memlevel1" % name, with_section(unc, ih.gz(data, 9, memlevel=1), 1), unc))
    for name, data in lh.sections().items():
        unc = payload_batch(data)
        for codec in ("gzip", "lz4", "snappy", "snappy-xerial"):
            if codec != "gzip" and not data:
                continue
            out.append(("lzwalk-%s/%s" % (name, codec), with_section(unc, kc.compress_records(data, codec), kc.CODEC_BITS[codec]), unc))
    return out


CORPORA = {"records": record_corpus, "lane_shapes": lane_corpus, "sizes": size_corpus, "host_inputs": host_corpus}


def check_images(items, got):
    """every batch decoded, its image equal to the uncompressed batch, its slot the image's length rounded up to 16"""
    assert len(got) == len(items)
    bad = []
    for (name, comp, want), (flags, slot, img) in zip(items, got):
        if flags != LOGB_OK or img != want or slot != (len(want) + 15) & ~15:
            first = next((i for i in range(min(len(img), len(want))) if img[i] != want[i]), min(len(img), len(want)))
            bad.append("%s: flags %d, slot %d (want %d), %d bytes (want %d), first difference at %d" %
                       (name, flags, slot, (len(want) + 15) & ~15, len(img), len(want), first))
    assert not bad, "%d of %d batches differ:\n%s" % (len(bad), len(items), "\n".join(bad[:30]))


@pytest.mark.gpu
@pytest.mark.parametrize("corpus", sorted(CORPORA))
def test_decompressed_images_match_the_reference_codecs(corpus):
    items = CORPORA[corpus]()
    assert all(c[22] & 7 for _, c, _ in items)
    got = decompress([b"".join(c for _, c, _ in items)])[0]   # every batch of the corpus in one launch group
    check_images(items, got)


@pytest.mark.gpu
def test_many_batches_per_launch():
    """more small batches than the warps of the decompression grid (132 SMs x 16 CTAs x 4 warps), every codec interleaved
    (uncompressed ones too): the grid-stride loop wraps, and the warps of one CTA run different codecs side by side"""
    rng = np.random.default_rng(53)
    codecs = ["gzip", "lz4", "snappy", "snappy-xerial", "zstd", "zstd-stream", None]
    items = []
    for b in range(132 * 16 * 4 + 700):
        recs = [(b"key-%d" % int(rng.integers(0, 1000)), text_bytes(rng, int(rng.integers(0, 120))), ())
                for _ in range(int(rng.integers(1, 5)))]
        unc = records_batch(recs, base_offset=b * 10)
        codec = codecs[b % len(codecs)]
        comp = kc.recompress(unc, lambda: codec)
        items.append(("batch-%d/%s" % (b, codec), comp, unc, codec))
    got = decompress([b"".join(c for _, c, _, _ in items)])[0]
    assert len(got) == len(items)
    bad = [name for (name, _, unc, codec), (flags, slot, img) in zip(items, got)
           if flags != LOGB_OK or img != unc or slot != (0 if codec is None else (len(unc) + 15) & ~15)]
    assert not bad, "%d of %d batches differ: %s" % (len(bad), len(items), bad[:30])


@pytest.mark.gpu
def test_damaged_sections_agree_with_the_host_walks():
    """The damaged sections of the host tests (900 zstd frames, 1200 gzip / LZ4 / Snappy sections), once, in one launch: the
    GPU accepts exactly the ones the host walk accepts, with the same bytes.  recordsCount is 0, so that only the walks decide."""
    cases = [(kc.CODEC_BITS["zstd"], f) for f in zh.damaged_frames()] + lh.damaged_sections()
    host = ch.run_cases(native_build.build("codec_harness"), cases)
    base = payload_batch(b"")
    got = decompress([b"".join(with_section(base, s, c) for c, s in cases)])[0]
    assert len(got) == len(cases)
    disagree = []
    for i, ((ok, _, out), (flags, slot, img)) in enumerate(zip(host, got)):
        assert flags in (LOGB_OK, LOGB_BAD), (i, flags)
        if ok != (flags == LOGB_OK) or (ok and (img[61:] != out or slot != (61 + len(out) + 15) & ~15)):
            disagree.append((i, "codec %d" % cases[i][0], ok, flags, len(out), len(img)))
    assert not disagree, disagree[:20]
    assert sum(ok for ok, _, _ in host) > 50          # both outcomes are exercised
    assert sum(not ok for ok, _, _ in host) > 500


@pytest.mark.gpu
def test_every_decompressed_byte_is_a_key_byte():
    """Records with random, long (up to ~2 KiB) and run-heavy keys, null or empty values and no headers, every codec mixed:
    what the scan hashes is all the decompressed records carry besides lengths, so the per-record key hashes (captured
    inside the fused scan) check the decompression through the product's own entry points and buffers."""
    import torch
    from kafka_topic_analyzer_b200 import KtaEngine
    rng = np.random.default_rng(59)
    codecs = ["gzip", "lz4", "snappy", "snappy-xerial", "zstd", "zstd-stream", None]
    P = 4
    segs, order, per = [], [], {p: [] for p in range(P)}
    for p in range(P):
        seg, off = bytearray(), 0
        for b in range(60):
            recs = []
            for j in range(int(rng.integers(1, 40))):
                kind = int(rng.integers(0, 4))
                n = int(rng.integers(0, 2048)) if kind else int(rng.integers(0, 40))
                key = (None if j % 17 == 5 else rng.integers(0, 256, n, dtype=np.uint8).tobytes() if kind < 2
                       else run_bytes(rng, n) if kind == 2 else bytes(n))
                value = None if rng.integers(0, 2) else 0
                ts = 1_700_000_000_000 + int(rng.integers(0, 10 ** 6))
                recs.append((j, ts - 1_700_000_000_000, key, value))
                per[p].append((ts, key, value))
                order.append(key)
            seg += kc.encode_batch(off, 1_700_000_000_000, recs, compression=codecs[(p + b) % len(codecs)])
            off += len(recs)
        segs.append((p, bytes(seg)))
    kl = np.array([-1 if k is None else len(k) for k in order], dtype=np.int32)
    want = np_oracle.fnv32_many(kl, np.frombuffer(b"".join(k for k in order if k), dtype=np.uint8))
    o = oracle_over(per, count_alive_keys=True)
    n = len(order)
    with KtaEngine(P, count_alive_keys=True, hll_precision=10, now=NOW) as e:
        cap = torch.zeros(n, dtype=torch.int32, device="cuda")
        capture_hashes(e, cap)
        assert e.push_log_segments(segs) == n
        capture_hashes(e, None)
        e.finalize()
        assert np.array_equal(cap.cpu().numpy().view(np.uint32), want)
        assert_parity(e, o, P, check_alive=True, hll_regs=o.hll_alive_regs(10))
        # the same batches in one device buffer, through kta_scan_log_batches_device
        e.reset()
        cap.fill_(0)
        capture_hashes(e, cap)
        assert scan_log_batches(e, stage_batches(segs)) == n
        capture_hashes(e, None)
        e.finalize()
        assert np.array_equal(cap.cpu().numpy().view(np.uint32), want)
        assert_parity(e, o, P, check_alive=True, hll_regs=o.hll_alive_regs(10))
