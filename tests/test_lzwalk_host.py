"""The decompressor walks of the RecordBatch decoder (LZ4 frame, Snappy raw / xerial, gzip: csrc/kta_logdecode.cuh,
csrc/kta_inflate.cuh) on the host, compiled by nvcc with the address sanitizer: the same statements the GPU runs per warp,
against pyarrow's / zlib's compressors, and under random damage — a damaged batch must be rejected or decode to SOMETHING
of the announced size, never read or write outside its buffers (the harness allocates them at their exact sizes)."""
import os
import shutil
import struct
import subprocess
import zlib

import numpy as np
import pytest

import kafka_codec as kc

HERE = os.path.dirname(os.path.abspath(__file__))
NVCC = os.environ.get("NVCC") or "/usr/local/cuda/bin/nvcc"
CODEC = {"gzip": 1, "snappy": 2, "snappy-xerial": 2, "lz4": 3}


@pytest.fixture(scope="module")
def harness(tmp_path_factory):
    nvcc = NVCC if os.path.exists(NVCC) else shutil.which("nvcc")
    if not nvcc:
        pytest.skip("nvcc not available")
    exe = str(tmp_path_factory.mktemp("lzwalk") / "lzwalk_harness")
    src = os.path.join(HERE, "native", "lzwalk_harness.cu")
    r = subprocess.run([nvcc, "-O1", "-g", "-std=c++17", "-Xcompiler", "-fsanitize=address,-fno-omit-frame-pointer", "-o", exe, src],
                       capture_output=True, text=True)
    if r.returncode != 0:        # no sanitizer runtime in this toolchain: the plain build still checks the results
        subprocess.run([nvcc, "-O1", "-std=c++17", "-o", exe, src], check=True, capture_output=True)
    return exe


def run_cases(exe, cases):
    blob = b"".join(struct.pack("<BI", c, len(d)) + d for c, d in cases)
    env = dict(os.environ, ASAN_OPTIONS="detect_leaks=0:protect_shadow_gap=0")
    r = subprocess.run([exe], input=blob, capture_output=True, env=env)
    assert r.returncode == 0, r.stderr.decode("utf-8", "replace")[-2000:]
    out, res, at = r.stdout, [], 0
    for _ in cases:
        ok, size_len, n = out[at], *struct.unpack_from("<II", out, at + 1)
        res.append((bool(ok), size_len, out[at + 9:at + 9 + n]))
        at += 9 + n
    assert at == len(out)
    return res


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
            cases.append((CODEC[codec], kc.compress_records(data, codec)))
            want.append(data)
    for (ok, size_len, out), w in zip(run_cases(harness, cases), want):
        assert ok and size_len == len(w) and out == w


def test_damaged_sections_never_leave_their_buffers(harness):
    """Bit flips, truncations and spliced garbage: the harness runs under the address sanitizer with exact-size buffers, so
    any read past the input or write past the size pass's length ends the process with a report."""
    cases = damaged_sections()
    res = run_cases(harness, cases)                 # returncode 0 = no sanitizer report, no crash
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
            cases.append((CODEC[codec], bytes(b)))
    return cases
