"""The gzip / DEFLATE decoder of the RecordBatch path (csrc/kta_inflate.cuh) against zlib, on the host: the product's
gzip_size and gzip_walk, the same __host__ __device__ statements log_unc_size_kernel and log_decompress_kernel run on the GPU,
compiled by nvcc as a plain host program with the address sanitizer (tests/native/codec_harness.cu, one lane, exact-size
buffers).  The lane split (lane 0's literals, the 32-lane matches) runs only on the GPU: test_logdecomp_gpu.py compares its
output with zlib's, over these payloads among others."""
import gzip
import struct
import zlib

import numpy as np
import pytest

import codec_harness as ch
import kafka_codec as kc


@pytest.fixture(scope="module")
def harness(tmp_path_factory):
    return ch.sanitized(tmp_path_factory)


def run_cases(exe, cases):
    """gzip members → per case (ok, size-pass length, output)"""
    return ch.run_cases(exe, [(kc.CODEC_BITS["gzip"], c) for c in cases])


def gz(data, level=6, strategy=zlib.Z_DEFAULT_STRATEGY, memlevel=8):
    c = zlib.compressobj(level, zlib.DEFLATED, 31, memlevel, strategy)
    return c.compress(data) + c.flush()


def payloads():
    rng = np.random.default_rng(7)
    text = b" ".join(b"key-%d value-%d" % (i % 97, i * i) for i in range(4000))
    records = b"".join(bytes([40 + i % 5, 0, i % 7, i & 0xff]) + b"key-%07d" % (i % 5000) + bytes(60) for i in range(3000))
    return {
        "empty": b"",
        "one": b"x",
        "text": text,
        "records": records,                                      # what a batch's records section looks like
        "zeros": bytes(100_000),                                 # long self-overlapping matches (distance 1)
        "random": rng.integers(0, 256, 70_000, dtype=np.uint8).tobytes(),   # incompressible: stored blocks (> 65535: several)
        "period3": b"abc" * 20_000,
        "bytes": bytes(range(256)) * 40,
        "mixed": text[:5000] + rng.integers(0, 256, 3000, dtype=np.uint8).tobytes() + bytes(5000) + text[5000:9000],
    }


def test_inflate_matches_zlib(harness):
    cases, want = [], []
    for name, data in payloads().items():
        for level in (0, 1, 6, 9):
            for strategy in (zlib.Z_DEFAULT_STRATEGY, zlib.Z_FIXED, zlib.Z_HUFFMAN_ONLY, zlib.Z_RLE, zlib.Z_FILTERED):
                cases.append(gz(data, level, strategy))
                want.append(data)
        cases.append(gzip.compress(data, mtime=0))              # Python's writer (header with flags / extra fields as it writes them)
        want.append(data)
        cases.append(gz(data, 9, memlevel=1))                   # tiny hash table: many small dynamic blocks
        want.append(data)
    got = run_cases(harness, cases)
    for i, ((ok, size_len, out), w) in enumerate(zip(got, want)):
        assert ok and size_len == len(w) and out == w, i


def test_gzip_header_fields(harness):
    """FEXTRA / FNAME / FCOMMENT / FHCRC are skipped (RFC 1952 2.3.1)."""
    data = b"kafka " * 500
    raw = zlib.compress(data, 6)[2:-4]                           # the bare deflate stream
    trailer = struct.pack("<II", zlib.crc32(data), len(data))
    plain = b"\x1f\x8b\x08\x00" + bytes(6)
    cases = [
        plain + raw + trailer,
        b"\x1f\x8b\x08\x04" + bytes(6) + struct.pack("<H", 5) + b"extra" + raw + trailer,
        b"\x1f\x8b\x08\x08" + bytes(6) + b"name.log\x00" + raw + trailer,
        b"\x1f\x8b\x08\x1e" + bytes(6) + struct.pack("<H", 2) + b"xy" + b"n\x00" + b"comment\x00" + b"\x12\x34" + raw + trailer,
    ]
    for ok, size_len, out in run_cases(harness, cases):
        assert ok and size_len == len(data) and out == data


def test_corrupt_streams_fail_cleanly(harness):
    data = b" ".join(b"key-%d" % (i % 50) for i in range(3000))
    good = gz(data)
    cases = [
        b"",                                                    # nothing
        good[:10],                                              # header only
        b"\x1f\x8b\x07" + good[3:],                             # not deflate
        good[:len(good) // 2] + good[-8:],                      # truncated stream under an intact trailer
        good[:-4] + struct.pack("<I", len(data) + 1),           # ISIZE disagrees
        good[:-4] + struct.pack("<I", len(data) - 1),
        good[:10] + b"\x07" + good[11:],                        # block type 3
        good[:10] + bytes([good[10] ^ 0x10]) + good[11:],       # a flipped bit in the dynamic header
    ]
    rng = np.random.default_rng(3)
    for _ in range(200):                                        # random single-byte damage inside the stream: never a crash
        b = bytearray(good)
        b[int(rng.integers(10, len(good) - 8))] ^= 1 << int(rng.integers(0, 8))
        cases.append(bytes(b))
    res = run_cases(harness, cases)
    for ok, _, out in res[:8]:
        assert not ok
    for ok, _, out in res[8:]:                                     # damage may survive as different bytes; what matters is that the
        if ok:                                                  # walk terminates inside its bounds and still honours ISIZE
            assert len(out) == len(data)
