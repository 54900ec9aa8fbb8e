"""The decompressor walks of the RecordBatch decoder (LZ4 frame, Snappy raw / xerial: csrc/kta_lz4_snappy.cuh; gzip:
csrc/kta_inflate.cuh) on the host, through the product's section_size / section_copy (csrc/kta_logdecode.cuh), compiled by
nvcc with the address sanitizer (tests/native/codec_harness.cu): the same statements the GPU runs per warp, against pyarrow's /
zlib's compressors, and under random damage — a damaged batch must be rejected or decode to SOMETHING of the announced size,
never read or write outside its buffers (the harness allocates them at their exact sizes)."""
import numpy as np
import pytest

import codec_harness as ch
import kafka_codec as kc


@pytest.fixture(scope="module")
def harness(tmp_path_factory):
    return ch.sanitized(tmp_path_factory)


def sections():
    rng = np.random.default_rng(5)
    recs = b"".join(kc.encode_record(i, i, b"key-%d" % (i % 50), 30 + i % 9) for i in range(400))
    big = b"".join(kc.encode_record(i, i, bytes(rng.integers(0, 256, 16, dtype=np.uint8)), 200) for i in range(3000))   # > one 64 KiB LZ4 block
    return {"records": recs, "big": big, "empty": b"", "one": b"\x00", "zeros": bytes(70_000),
            "random": rng.integers(0, 256, 20_000, dtype=np.uint8).tobytes()}


def test_walks_match_the_compressors(harness):
    cases, want = [], []
    for name, data in sections().items():
        for codec in ("gzip", "lz4", "snappy", "snappy-xerial"):
            if codec != "gzip" and not data:
                continue
            cases.append((kc.CODEC_BITS[codec], kc.compress_records(data, codec)))
            want.append(data)
    for (ok, size_len, out), w in zip(ch.run_cases(harness, cases), want):
        assert ok and size_len == len(w) and out == w


def test_damaged_sections_never_leave_their_buffers(harness):
    """Bit flips, truncations and spliced garbage: the harness runs under the address sanitizer with exact-size buffers, so
    any read past the input or write past the size pass's length ends the process with a report."""
    cases = damaged_sections()
    res = ch.run_cases(harness, cases)                 # returncode 0 = no sanitizer report, no crash
    assert len(res) == len(cases)
    for ok, size_len, out in res:
        if ok:
            assert len(out) == size_len


def damaged_sections():
    """(codec, section): 300 damaged sections per codec (test_logdecomp_gpu.py runs the same ones on the GPU)"""
    rng = np.random.default_rng(9)
    data = sections()["records"]
    cases = []
    for codec in ("gzip", "lz4", "snappy", "snappy-xerial"):
        good = kc.compress_records(data, codec)
        for _ in range(300):
            b = bytearray(good)
            kind = int(rng.integers(0, 4))
            if kind == 0:
                b[int(rng.integers(0, len(b)))] ^= 1 << int(rng.integers(0, 8))
            elif kind == 1:
                b = b[: int(rng.integers(0, len(b)))]
            elif kind == 2:
                at = int(rng.integers(0, len(b)))
                b[at:at + 4] = bytes(rng.integers(0, 256, 4, dtype=np.uint8))
            else:
                b += bytes(rng.integers(0, 256, int(rng.integers(1, 9)), dtype=np.uint8))
            cases.append((kc.CODEC_BITS[codec], bytes(b)))
    return cases
