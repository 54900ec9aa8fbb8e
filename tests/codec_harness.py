"""Runs tests/native/codec_harness.cu — TEST INFRASTRUCTURE: the codec walks of the RecordBatch decoder as a plain host program,
one "lane".  stdin: per case u8 Kafka codec id (kafka_codec.CODEC_BITS) | u32 length | bytes; stdout: per case u8 ok | u32
size-pass length | u32 length | bytes."""
import os
import struct
import subprocess
import warnings

import pytest

import native_build

ASAN_OPTIONS = "detect_leaks=0:protect_shadow_gap=0"


def sanitized(tmp_path_factory):
    """the host tests' build: with the address sanitizer where the toolchain has it (shared by the modules of one session)"""
    if not native_build.nvcc():
        pytest.skip("nvcc not available")
    exe, how = native_build.build_sanitized("codec_harness", str(tmp_path_factory.getbasetemp()))
    print(how)
    if not exe.endswith("_asan"):
        warnings.warn(how)
    return exe


def run_cases(exe, cases):
    """cases: (codec id, section) → per case (ok, size-pass length, output)"""
    blob = b"".join(struct.pack("<BI", c, len(d)) + d for c, d in cases)
    r = subprocess.run([exe], input=blob, capture_output=True, env=dict(os.environ, ASAN_OPTIONS=ASAN_OPTIONS))
    assert r.returncode == 0, r.stderr.decode("utf-8", "replace")[-3000:]
    out, res, at = r.stdout, [], 0
    for _ in cases:
        ok, size_len, n = out[at], *struct.unpack_from("<II", out, at + 1)
        res.append((bool(ok), size_len, out[at + 9:at + 9 + n]))
        at += 9 + n
    assert at == len(out)
    return res
