"""The zstd walk of the RecordBatch decoder (csrc/kta_zstd.cuh) on the host, compiled by nvcc with the address sanitizer
(tests/native/codec_harness.cu): the same statements the GPU runs per warp, against pyarrow's zstd, over hand-assembled frames,
and under random damage — a damaged section must be rejected or decode to SOMETHING of the size the size pass announced, never
read or write outside its buffers (the harness allocates input, output and literal buffers at their exact sizes)."""
import collections
import struct

import numpy as np
import pytest

import codec_harness as ch
import kafka_codec as kc

LEVELS = (-5, 1, 3, 9, 19, 22)
MAGIC = b"\x28\xb5\x2f\xfd"


@pytest.fixture(scope="module")
def harness(tmp_path_factory):
    return ch.sanitized(tmp_path_factory)


def run_cases(exe, frames):
    """zstd sections → per case (ok, size-pass length, output)"""
    return ch.run_cases(exe, [(kc.CODEC_BITS["zstd"], f) for f in frames])


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


class BackwardBits:
    """the writing side of a zstd backward bitstream (RFC 8878 4.1): values go in low bits first and are read back last
    first, from the top; finish() adds the padding marker"""

    def __init__(self):
        self.v, self.n = 0, 0

    def add(self, value, nbits):
        assert 0 <= value < (1 << nbits) or (value == 0 and nbits == 0)
        self.v |= value << self.n
        self.n += nbits

    def finish(self):
        return (self.v | (1 << self.n)).to_bytes(self.n // 8 + 1, "little")


def huffman_codes(weights):
    """canonical prefix codes from Huffman weights (RFC 8878 4.2.1.3), the last symbol's weight included: symbols sorted by
    weight, in symbol order within a weight, codes handed out in sequence from the lowest weight.  {symbol: (code, bits)}"""
    total = sum(1 << (w - 1) for w in weights if w)
    log = total.bit_length() - 1
    assert total == 1 << log
    codes, at = {}, 0
    for w in range(1, log + 1):
        for sym, x in enumerate(weights):
            if x == w:
                codes[sym] = (at >> (w - 1), log + 1 - w)
                at += 1 << (w - 1)
    return codes


def huffman_stream(data, codes):
    """one Huffman stream: the first literal is read first, so it is written last"""
    bw = BackwardBits()
    for b in reversed(data):
        bw.add(*codes[b])
    return bw.finish()


def block(body, bt, last):
    return struct.pack("<I", (len(body) << 3) | (bt << 1) | last)[:3] + body


def rle_mode_sequences(seqs, ll_code, of_code, ml_code):
    """a sequences section with RLE mode for all three codes (one symbol each, no state bits): the bitstream holds only the
    extra bits.  seqs: (ll extra, of extra, ml extra) per sequence → (section, [(literal length, offset value, match length)])"""
    assert len(seqs) < 128
    bw = BackwardBits()
    for lle, ofe, mle in reversed(seqs):                  # read per sequence as OF, ML, LL: written the other way round
        bw.add(lle, ZSTD_LL_BITS[ll_code])
        bw.add(mle, ZSTD_ML_BITS[ml_code])
        bw.add(ofe, of_code)
    decoded = [(ZSTD_LL_BASE[ll_code] + lle, (1 << of_code) + ofe, ZSTD_ML_BASE[ml_code] + mle) for lle, ofe, mle in seqs]
    return bytes([len(seqs), 0x54, ll_code, of_code, ml_code]) + bw.finish(), decoded


# the few literal-length / match-length codes used below (RFC 8878 3.1.1.3.2.1.1): code → baseline, extra bits
ZSTD_LL_BASE, ZSTD_LL_BITS = {5: 5, 16: 16, 18: 20}, {5: 0, 16: 1, 18: 1}
ZSTD_ML_BASE, ZSTD_ML_BITS = {32: 35, 33: 37}, {32: 1, 33: 1}


def execute(out, lits, seqs):
    """RFC 8878 3.1.1.4 for sequences whose offset values are all > 3 (no repeat offsets)"""
    out, lp = bytearray(out), 0
    for ll, ov, ml in seqs:
        assert ov > 3
        out += lits[lp:lp + ll]
        lp += ll
        for _ in range(ml):
            out.append(out[-(ov - 3)])
    return bytes(out + lits[lp:])


def rle_literals_with_sequences():
    """a raw block, then a compressed block whose RLE literals are followed by sequences (RLE mode for LL, OF and ML) that
    reach back into the raw block; single segment, one-byte Frame_Content_Size"""
    raw = b"0123456789abcdefghijklmnopqrstuvwxyzABCD"
    seqs = [(1, 5, 0), (0, 13, 1), (1, 0, 1)]
    section, decoded = rle_mode_sequences(seqs, 16, 4, 32)
    body = bytes([1 | 4 | ((60 & 15) << 4), 60 >> 4, ord("Z")]) + section   # RLE literals, Size_Format 01: 60 x 'Z'
    want = execute(raw, b"Z" * 60, decoded)
    assert len(want) < 256
    return MAGIC + bytes([0x20, len(want)]) + block(raw, 0, 0) + block(body, 2, 1), want


def treeless_one_stream():
    """a block of Huffman literals in one stream, its table in direct 4-bit weights (header byte >= 128), no sequences; then a
    block of Treeless literals in one stream that reuses the table, followed by sequences.  No Frame_Content_Size, 4 KiB
    window."""
    rng = np.random.default_rng(17)
    weights = [0] * 103
    for ch, w in zip(b"abcdef", (5, 4, 3, 2, 1, 1)):      # 16 + 8 + 4 + 2 + 1 + 1 = 32: a complete code, 5-bit table
        weights[ch] = w
    codes = huffman_codes(weights)
    alphabet = np.frombuffer(b"abcdef", dtype=np.uint8)
    lits_a = rng.choice(alphabet, 200, p=[0.5, 0.25, 0.125, 0.0625, 0.03125, 0.03125]).tobytes()
    lits_b = rng.choice(alphabet, 150).tobytes()
    desc = bytes([127 + 102]) + bytes((weights[i] << 4) | weights[i + 1] for i in range(0, 102, 2))   # weights of 0..101; 'f' implied
    stream_a, stream_b = huffman_stream(lits_a, codes), huffman_stream(lits_b, codes)
    cs_a = len(desc) + len(stream_a)
    body_a = struct.pack("<I", 2 | (len(lits_a) << 4) | (cs_a << 14))[:3] + desc + stream_a + b"\x00"
    section, decoded = rle_mode_sequences([(0, 7, 1), (1, 30, 0)], 16, 5, 33)
    body_b = struct.pack("<I", 3 | (len(lits_b) << 4) | (len(stream_b) << 14))[:3] + stream_b + section
    want = execute(execute(b"", lits_a, []), lits_b, decoded)
    return MAGIC + bytes([0x00, (12 - 10) << 3]) + block(body_a, 2, 0) + block(body_b, 2, 1), want


def hand_assembled():
    return [rle_literals_with_sequences(), treeless_one_stream()]


def test_hand_assembled_frames_are_valid_zstd():
    """the two hand-assembled frames decode with pyarrow's zstd (the reference library) to what they are built to hold, so
    the walk is measured against the format, not against the encoder above; the code assignment is RFC 8878's example"""
    import pyarrow as pa
    assert huffman_codes([4, 3, 2, 0, 1, 1]) == {0: (1, 1), 1: (1, 2), 2: (1, 3), 4: (0, 4), 5: (1, 4)}
    for f, want in hand_assembled():
        assert pa.decompress(f, decompressed_size=len(want), codec="zstd", asbytes=True) == want


def corpus():
    """(frame, expected output) pairs covering the format's shapes"""
    out = []
    for data in sections().values():
        for lvl in LEVELS:
            f = one_shot(data, lvl)
            out.append((f, data))
            out.append((without_content_size(f), data))
        out.append((kc.compress_records(data, "zstd-stream"), data))
    recs, text = sections()["records"], sections()["text"]
    a, b = one_shot(recs, 3), kc.compress_records(text[:50_000], "zstd-stream")
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
    out += hand_assembled()                                                     # modes pyarrow does not write here
    return out


def test_walk_matches_pyarrow(harness):
    cases = corpus()
    res = run_cases(harness, [f for f, _ in cases])
    for i, ((ok, size_len, out), (f, want)) in enumerate(zip(res, cases)):
        assert ok and size_len == len(want) and out == want, (i, len(f), ok, size_len, len(want))


def test_corpus_reaches_every_mode():
    """The corpus above reaches every block type, literals type and stream count, weight encoding and sequence mode; the
    hand-assembled frames supply the two that pyarrow never writes for these inputs (one-stream Treeless literals, RLE
    literals followed by sequences)."""
    seen = collections.Counter()
    for f, _ in corpus():
        inspect(f, seen)
    want = {"fcs", "no_fcs", "skippable", "checksum", "block_raw", "block_rle", "block_compressed",
            "lit_raw", "lit_rle", "lit_huffman_1stream", "lit_huffman_4streams", "lit_treeless_4streams",
            "weights_direct", "weights_fse", "seq_none", "lit_huffman_1stream+seq_none", "lit_raw+sequences",
            "lit_treeless_1stream", "lit_treeless_1stream+sequences", "lit_rle+sequences"}
    want |= {"%s_%s" % (t, m) for t in ("LL", "OF", "ML") for m in ("predefined", "rle", "fse", "repeat")}
    missing = sorted(k for k in want if not seen[k])
    assert not missing, (missing, dict(seen))
    NOT_REACHED = set()
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
    cases = damaged_frames()
    res = run_cases(harness, cases)                 # returncode 0 = no sanitizer report, no crash
    assert len(res) == len(cases)
    for ok, size_len, out in res:
        if ok:
            assert len(out) == size_len
    assert sum(not ok for ok, _, _ in res) > len(cases) // 2


def damaged_frames():
    """900 damaged frames (test_logdecomp_gpu.py runs the same ones on the GPU)"""
    rng = np.random.default_rng(9)
    s = sections()
    data = s["records"] + s["text"][:20_000]
    goods = (one_shot(data, 3), kc.compress_records(data, "zstd-stream"), one_shot(data, 19))
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
    return cases
