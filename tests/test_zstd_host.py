"""The zstd walk of the RecordBatch decoder (csrc/kta_zstd.cuh) on the host, compiled by nvcc with the address sanitizer: the
same statements the GPU runs per warp, against pyarrow's zstd, over hand-assembled frames, and under random damage — a
damaged section must be rejected or decode to SOMETHING of the size the size pass announced, never read or write outside
its buffers (the harness allocates input, output and literal buffers at their exact sizes)."""
import collections
import os
import shutil
import struct
import subprocess

import numpy as np
import pytest

import kafka_codec as kc
import zstd_codec as zc

HERE = os.path.dirname(os.path.abspath(__file__))
NVCC = os.environ.get("NVCC") or "/usr/local/cuda/bin/nvcc"
LEVELS = (-5, 1, 3, 9, 19, 22)
MAGIC = b"\x28\xb5\x2f\xfd"


@pytest.fixture(scope="module")
def harness(tmp_path_factory):
    nvcc = NVCC if os.path.exists(NVCC) else shutil.which("nvcc")
    if not nvcc:
        pytest.skip("nvcc not available")
    exe = str(tmp_path_factory.mktemp("zstd") / "zstd_harness")
    src = os.path.join(HERE, "native", "zstd_harness.cu")
    r = subprocess.run([nvcc, "-O1", "-g", "-std=c++17", "-Xcompiler", "-fsanitize=address,-fno-omit-frame-pointer", "-o", exe, src],
                       capture_output=True, text=True)
    if r.returncode != 0:        # no sanitizer runtime in this toolchain: the plain build still checks the results
        subprocess.run([nvcc, "-O1", "-std=c++17", "-o", exe, src], check=True, capture_output=True)
    return exe


def run_cases(exe, cases):
    blob = b"".join(struct.pack("<I", len(d)) + d for d in cases)
    env = dict(os.environ, ASAN_OPTIONS="detect_leaks=0:protect_shadow_gap=0")
    r = subprocess.run([exe], input=blob, capture_output=True, env=env)
    assert r.returncode == 0, r.stderr.decode("utf-8", "replace")[-3000:]
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
    big = b"".join(kc.encode_record(i, i, bytes(rng.integers(0, 256, 16, dtype=np.uint8)), 200) for i in range(3000))
    text = b"".join(b"customer-%d:order-%d;" % (int(a), int(b)) for a, b in rng.integers(0, 10**6, (150_000, 2)))
    return {"records": recs, "big": big, "empty": b"", "one": b"\x00", "zeros": bytes(300_000),
            "random": rng.integers(0, 256, 20_000, dtype=np.uint8).tobytes(), "text": text,
            "alphabet16": rng.integers(0, 16, 2000, dtype=np.uint8).tobytes(),          # Huffman literals, no sequences
            "alphabet16_small": rng.integers(0, 16, 200, dtype=np.uint8).tobytes()}     # the same in one stream


def one_shot(data, level):
    import pyarrow as pa
    return pa.Codec("zstd", compression_level=level).compress(data, asbytes=True)


def header_len(f):
    """bytes of a zstd frame header (magic included)"""
    fhd = f[4]
    single = (fhd >> 5) & 1
    return 5 + (0 if single else 1) + (0, 1, 2, 4)[fhd & 3] + ((1 if single else 0), 2, 4, 8)[fhd >> 6]


def without_content_size(f):
    """the same blocks behind a streaming-style header: no Frame_Content_Size, a window descriptor of 8 MiB (pyarrow's
    streaming compressor takes no level, so this gives the no-content-size path every level's blocks)"""
    return MAGIC + bytes([0x00, (23 - 10) << 3]) + f[header_len(f):]


def raw_block(data, last):
    return struct.pack("<I", (len(data) << 3) | last)[:3] + data


def inspect(f, seen):
    """headers-only frame inspector: block types, literals-section types and stream counts, the Huffman description's
    first byte, sequence counts and modes.  No entropy decoding."""
    p = 0
    while p < len(f):
        magic = int.from_bytes(f[p:p + 4], "little")
        if magic & 0xFFFFFFF0 == 0x184D2A50:
            seen["skippable"] += 1
            p += 8 + int.from_bytes(f[p + 4:p + 8], "little")
            continue
        assert magic == 0xFD2FB528
        fhd = f[p + 4]
        seen["fcs" if fhd >> 6 or (fhd >> 5) & 1 else "no_fcs"] += 1
        q = p + header_len(f[p:])
        while True:
            bh = int.from_bytes(f[q:q + 3], "little")
            q += 3
            last, bt, bs = bh & 1, (bh >> 1) & 3, bh >> 3
            seen["block_" + ("raw", "rle", "compressed", "reserved")[bt]] += 1
            if bt == 2:
                b = f[q:q + bs]
                lt, sf = b[0] & 3, (b[0] >> 2) & 3
                if lt < 2:
                    hl = {0: 1, 2: 1, 1: 2, 3: 3}[sf]
                    o = hl + (int.from_bytes(b[:hl], "little") >> (3 if hl == 1 else 4) if lt == 0 else 1)
                    name = ("lit_raw", "lit_rle")[lt]
                else:
                    hl, bits = {0: (3, 10), 1: (3, 10), 2: (4, 14), 3: (5, 18)}[sf]
                    o = hl + ((int.from_bytes(b[:hl], "little") >> (4 + bits)) & ((1 << bits) - 1))
                    name = ("lit_huffman", "lit_treeless")[lt - 2] + ("_1stream" if sf == 0 else "_4streams")
                    if lt == 2:
                        seen["weights_" + ("fse" if b[hl] < 128 else "direct")] += 1
                seen[name] += 1
                n = b[o]
                if n == 0:
                    seen["seq_none"] += 1
                    seen[name + "+seq_none"] += 1
                else:
                    seen[name + "+sequences"] += 1
                    o += 1 if n < 128 else 2 if n < 255 else 3
                    for nm, sh in (("LL", 6), ("OF", 4), ("ML", 2)):
                        seen[nm + "_" + ("predefined", "rle", "fse", "repeat")[(b[o] >> sh) & 3]] += 1
            q += 1 if bt == 1 else bs
            if last:
                break
        if fhd & 4:
            seen["checksum"] += 1
            q += 4
        p = q


def rle_literals_block(byte, n, last=1):
    """a compressed block built from header bytes alone: an RLE literals section of n copies of `byte` and a sequences
    section that is the single byte 0 (no sequences)"""
    assert n < 4096
    body = bytes([(1 | 4) | ((n & 15) << 4), n >> 4, byte, 0])   # Size_Format 01: 2-byte header, 12-bit size
    return struct.pack("<I", (len(body) << 3) | (2 << 1) | last)[:3] + body


def corpus():
    """(frame, expected output) pairs covering the format's shapes"""
    out = []
    for data in sections().values():
        for lvl in LEVELS:
            f = one_shot(data, lvl)
            out.append((f, data))
            out.append((without_content_size(f), data))
        out.append((zc.compress_records(data, "zstd-stream"), data))
    recs, text = sections()["records"], sections()["text"]
    a, b = one_shot(recs, 3), zc.compress_records(text[:50_000], "zstd-stream")
    skip = struct.pack("<II", 0x184D2A53, 5) + b"hello"
    out.append((a + b, recs + text[:50_000]))                                   # two frames
    out.append((skip + a + skip + b, recs + text[:50_000]))                     # skippable frames before and between
    out.append((skip + a + struct.pack("<II", 0x184D2A5F, 0), recs))            # and an empty one after
    ck = bytearray(a)
    ck[4] |= 4                                                                  # Content_Checksum flag: 4 bytes follow
    out.append((bytes(ck) + b"\x01\x02\x03\x04", recs))
    rle = MAGIC + bytes([0x20, 100]) + rle_literals_block(0x41, 60, last=0) + raw_block(b"xyz", 0) + rle_literals_block(0x7A, 37)
    out.append((rle, b"A" * 60 + b"xyz" + b"z" * 37))                          # RLE literals, one-byte FCS
    out.append((MAGIC + bytes([0x00, 0x00]) + rle_literals_block(0x00, 5), bytes(5)))   # no FCS, 1 KiB window
    return out


def test_walk_matches_pyarrow(harness):
    cases = corpus()
    res = run_cases(harness, [f for f, _ in cases])
    for i, ((ok, size_len, out), (f, want)) in enumerate(zip(res, cases)):
        assert ok and size_len == len(want) and out == want, (i, len(f), ok, size_len, len(want))


def test_corpus_reaches_every_mode():
    """The corpus above reaches every block type, literals type and stream count, weight encoding and sequence mode except
    the ones named in NOT_REACHED: pyarrow never writes them for these inputs, and entropy-coded streams are not hand-built."""
    seen = collections.Counter()
    for f, _ in corpus():
        inspect(f, seen)
    want = {"fcs", "no_fcs", "skippable", "checksum", "block_raw", "block_rle", "block_compressed",
            "lit_raw", "lit_rle", "lit_huffman_1stream", "lit_huffman_4streams", "lit_treeless_4streams",
            "weights_direct", "weights_fse", "seq_none", "lit_huffman_1stream+seq_none", "lit_raw+sequences"}
    want |= {"%s_%s" % (t, m) for t in ("LL", "OF", "ML") for m in ("predefined", "rle", "fse", "repeat")}
    missing = sorted(k for k in want if not seen[k])
    assert not missing, (missing, dict(seen))
    NOT_REACHED = {"lit_treeless_1stream", "lit_rle+sequences"}
    assert not any(seen[k] for k in NOT_REACHED), "now reached: move it into `want`"


def test_rejections(harness):
    recs = sections()["records"]
    good = one_shot(recs, 3)
    assert good[4] == 0x60 or good[4] >> 6            # one-shot frames carry Frame_Content_Size
    hl = header_len(good)
    fcs_at, fcs_len = hl - (1, 2, 4, 8)[good[4] >> 6] if good[4] >> 6 else hl - 1, (1, 2, 4, 8)[good[4] >> 6] if good[4] >> 6 else 1
    fcs = int.from_bytes(good[fcs_at:fcs_at + fcs_len], "little") + (256 if fcs_len == 2 else 0)
    assert fcs == len(recs)

    def with_fcs(v):
        b = bytearray(good)
        b[fcs_at:fcs_at + fcs_len] = (v - (256 if fcs_len == 2 else 0)).to_bytes(fcs_len, "little")
        return bytes(b)

    did = bytearray(good[:4]) + bytes([good[4] | 1, 7]) + good[5:]     # Dictionary_ID (1 byte) = 7
    reserved = bytearray(good)
    reserved[hl] |= 6                                                    # block type 3
    big_raw = MAGIC + bytes([0x00, (23 - 10) << 3]) + struct.pack("<I", ((ZSTD_BLOCK_MAX + 1) << 3) | 1)[:3] + bytes(ZSTD_BLOCK_MAX + 1)
    bad = {
        "magic": b"\x29" + good[1:],
        "dictionary id": bytes(did),
        "reserved block type": bytes(reserved),
        "content size + 1": with_fcs(fcs + 1),
        "content size - 1": with_fcs(fcs - 1),
        "trailing byte": good + b"\x00",
        "truncated": good[:-1],
        "truncated header": good[:hl],
        "raw block over 128 KiB": big_raw,
        "empty section": b"",
        "reserved frame header bit": good[:4] + bytes([good[4] | 8]) + good[5:],
        "uncompressed records": recs,
    }
    for name, (ok, _, _) in zip(bad, run_cases(harness, list(bad.values()))):
        assert not ok, name
    # the same frame as it was decodes
    assert run_cases(harness, [good])[0][0]


ZSTD_BLOCK_MAX = 128 * 1024


def test_damaged_frames_never_leave_their_buffers(harness):
    """Bit flips, truncations, spliced garbage and appended bytes, 300 each for one-shot, streaming and level-19 frames: the
    harness runs under the address sanitizer with exact-size buffers, so any read past the input or write past the size
    pass's length ends the process with a report.  A damaged frame that still decodes has the size the size pass gave."""
    rng = np.random.default_rng(9)
    s = sections()
    data = s["records"] + s["text"][:20_000]
    goods = (one_shot(data, 3), zc.compress_records(data, "zstd-stream"), one_shot(data, 19))
    cases = []
    for good in goods:
        for i in range(300):
            b = bytearray(good)
            kind = i % 4
            if kind == 0:
                b[int(rng.integers(0, len(b)))] ^= 1 << int(rng.integers(0, 8))
            elif kind == 1:
                b = b[: int(rng.integers(0, len(b)))]
            elif kind == 2:
                at = int(rng.integers(0, len(b)))
                b[at:at + 4] = bytes(rng.integers(0, 256, 4, dtype=np.uint8))
            else:
                b += bytes(rng.integers(0, 256, int(rng.integers(1, 9)), dtype=np.uint8))
            cases.append(bytes(b))
    res = run_cases(harness, cases)                 # returncode 0 = no sanitizer report, no crash
    assert len(res) == len(cases)
    for ok, size_len, out in res:
        if ok:
            assert len(out) == size_len
    assert sum(not ok for ok, _, _ in res) > len(cases) // 2
