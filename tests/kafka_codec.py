"""Kafka RecordBatch v2 (magic 2) log codec — TEST INFRASTRUCTURE for the GPU decoder (kta_logdecode.cuh) and its
decompression, read_committed and check.crcs passes.  Follows the Kafka protocol documentation for the record batch /
record layout (KIP-98) and the transaction log formats; independent of the decoder's code.

Writing: records and batches, their records sections compressed by every codec the decoder takes (zlib's gzip; pyarrow's
LZ4 frame, raw and xerial-framed Snappy, one-shot and streaming zstd), transactional batches, control markers and
.txnindex images.  The encoders write the CRC field as 0, which librdkafka by default (check.crcs=false) and the decoder
with its check off never read; set_crcs gives a segment the CRC-32C a broker stores, with a plain byte-at-a-time CRC-32C
that is independent of the GPU pass (kta_logcrc.cuh).

Reading: read_segment walks a segment's bytes back into batch headers and records.  It has its own varint decoding and
decompresses with zlib and pyarrow, so that a walk of the bytes checks the encoders instead of restating them."""
import struct
import zlib
from collections import namedtuple


# ---- records and batches --------------------------------------------------------------------------------------------
def zigzag(n: int) -> int:
    return (n << 1) ^ (n >> 63) if n < 0 else n << 1


def uvarint(u: int) -> bytes:
    out = bytearray()
    while True:
        b = u & 0x7F
        u >>= 7
        if u:
            out.append(b | 0x80)
        else:
            out.append(b)
            return bytes(out)


def varint(n: int, width: int = 0) -> bytes:
    """n zig-zag encoded; width > 0 pads it to that many bytes (up to 10) with empty continuation groups, as a writer that
    reserves a fixed-width length field may — a non-minimal encoding that readers take as the same value"""
    b = uvarint(zigzag(n) & 0xFFFFFFFFFFFFFFFF)
    if width > len(b):
        assert width <= 10
        b = b[:-1] + bytes([b[-1] | 0x80]) + b"\x80" * (width - len(b) - 1) + b"\x00"
    return b


def encode_record(offset_delta, ts_delta, key, value_len, headers=(), value=None, widths=None):
    """value bytes are synthesised (the metric path never reads them) unless `value` gives them; value_len None (and no
    value) = tombstone.  widths: {"len", "ts", "key", "value"} → the byte width of the record-length, timestamp-delta,
    key-length and value-length varints (padded; see varint)"""
    w = widths or {}
    body = bytearray(b"\x00")                      # record attributes
    body += varint(ts_delta, w.get("ts", 0)) + varint(offset_delta)
    if key is None:
        body += varint(-1, w.get("key", 0))
    else:
        body += varint(len(key), w.get("key", 0)) + key
    if value is not None:
        assert value_len is None or value_len == len(value)
        body += varint(len(value), w.get("value", 0)) + value
    elif value_len is None:
        body += varint(-1, w.get("value", 0))
    else:
        body += varint(value_len, w.get("value", 0)) + bytes((i * 31 + 7) & 0xFF for i in range(value_len))
    body += varint(len(headers))
    for hk, hv in headers:
        body += varint(len(hk)) + hk
        body += varint(-1) if hv is None else varint(len(hv)) + hv
    return varint(len(body), w.get("len", 0)) + bytes(body)


def compress_records(recs: bytes, codec: str) -> bytes:
    """The records section as a producer with compression.type=<codec> writes it.  'snappy-xerial' adds the framing of
    the Java client's snappy-java stream (magic, two version words, chunks of u32 BE length + raw snappy); 'zstd' is a
    one-shot frame, which carries Frame_Content_Size, and 'zstd-stream' pyarrow's CompressedOutputStream, which does not
    (as streaming compressors such as the Java client's write it)."""
    import pyarrow as pa
    if codec == "gzip":                                  # zlib's gzip wrapper (what librdkafka and the Java client write)
        c = zlib.compressobj(6, zlib.DEFLATED, 31)
        return c.compress(recs) + c.flush()
    if codec in ("lz4", "snappy", "zstd"):
        return pa.compress(recs, codec=codec, asbytes=True)
    if codec == "snappy-xerial":
        out = bytearray(b"\x82SNAPPY\x00" + struct.pack(">ii", 1, 1))
        step = max(1, len(recs) // 3 + 1)              # several chunks per batch
        for i in range(0, len(recs), step):
            c = pa.compress(recs[i:i + step], codec="snappy", asbytes=True)
            out += struct.pack(">i", len(c)) + c
        return bytes(out)
    if codec == "zstd-stream":
        sink = pa.BufferOutputStream()
        with pa.CompressedOutputStream(sink, "zstd") as s:
            s.write(recs)
        return sink.getvalue().to_pybytes()
    raise ValueError(codec)


# Kafka's compression codec ids (attributes & 7), by the names these encoders take
CODEC_BITS = {None: 0, "gzip": 1, "snappy": 2, "snappy-xerial": 2, "lz4": 3, "zstd": 4, "zstd-stream": 4}


def _int32(x):
    return (x + (1 << 31)) % (1 << 32) - (1 << 31)


def _int64(x):
    return (x + (1 << 63)) % (1 << 64) - (1 << 63)


def encode_batch(base_offset, base_ts, records, attributes=0, max_ts=None, compression=None):
    """records: list of (offset_delta, ts_delta, key|None, value_len|None[, headers[, value[, widths]]])"""
    recs = b"".join(encode_record(*r) for r in records)
    if compression:
        recs = compress_records(recs, compression)
        attributes |= CODEC_BITS[compression]
    last_delta = _int32(max((r[0] for r in records), default=0))
    if max_ts is None:
        max_ts = _int64(max((base_ts + r[1] for r in records), default=base_ts))
    after_len = struct.pack(">iBIhiqqqhii", 0, 2, 0, attributes, last_delta, base_ts, max_ts, -1, -1, -1, len(records)) + recs
    return struct.pack(">qi", base_offset, len(after_len)) + after_len


def encode_partition(partition_records, rng, max_batch=40, log_append_time=False, compression=None):
    """partition_records: list of (ts_ms, key|None, value_len|None) in offset order → one log segment (bytes).
    ts_ms == -1 (not available) forces a batch with base timestamp -1.  A list of codecs: every batch draws its own, right
    after drawing its size (recompress over the uncompressed segment draws every size first)."""
    out = bytearray()
    i, n = 0, len(partition_records)
    while i < n:
        m = int(rng.integers(1, max_batch + 1))
        chunk = partition_records[i:i + m]
        # records without a timestamp can only be expressed with baseTimestamp == -1 (whole batch)
        if chunk[0][0] == -1:
            k = 1
            while k < len(chunk) and chunk[k][0] == -1:
                k += 1
            chunk = chunk[:k]
            base_ts = -1
        else:
            k = 1
            while k < len(chunk) and chunk[k][0] != -1:
                k += 1
            chunk = chunk[:k]
            base_ts = chunk[0][0] - int(rng.integers(0, 1000))
        recs = []
        for j, (ts, key, vl) in enumerate(chunk):
            hdrs = ((b"h", b"v"), (b"trace", None)) if (i + j) % 7 == 0 else ()
            recs.append((j, 0 if base_ts == -1 else ts - base_ts, key, vl, hdrs))
        attrs = 0x08 if log_append_time else 0
        codec = compression
        if isinstance(compression, (list, tuple)):          # a mix: every batch picks its own codec
            codec = compression[int(rng.integers(0, len(compression)))]
        out += encode_batch(i, base_ts, recs, attributes=attrs, compression=codec)
        i += len(chunk)
    return bytes(out)


# ---- segments -------------------------------------------------------------------------------------------------------
def batch_offsets(seg):
    """where every batch of a segment starts: the walk from batch header to batch header by batchLength"""
    seg, offs, pos = bytes(seg), [], 0
    while pos + 61 <= len(seg):
        offs.append(pos)
        pos += 12 + int.from_bytes(seg[pos + 8:pos + 12], "big", signed=True)
    return offs


def split_batches(seg):
    """the bytes of every batch of a segment, each up to where the next begins (the last one up to the segment's end)"""
    seg = bytes(seg)
    offs = batch_offsets(seg)
    return [seg[a:b] for a, b in zip(offs, offs[1:] + [len(seg)])]


def with_section(batch, section, codec_bits):
    """the batch with its records section replaced; batchLength and the codec bits follow"""
    hdr = bytearray(batch[:61])
    hdr[8:12] = struct.pack(">i", 49 + len(section))
    hdr[22] = (hdr[22] & 0xF8) | codec_bits
    return bytes(hdr) + section


def recompress(seg, pick) -> bytes:
    """every batch of an uncompressed segment with its records section compressed by pick() (a codec name, or None to
    leave the batch as it is), one call per batch in order"""
    out = bytearray()
    for b in split_batches(seg):
        codec = pick()
        out += with_section(b, compress_records(b[61:], codec), CODEC_BITS[codec]) if codec else b
    return bytes(out)


# ---- CRC-32C (check.crcs) -------------------------------------------------------------------------------------------
def _crc32c_table():
    t = []
    for i in range(256):
        c = i
        for _ in range(8):
            c = (c >> 1) ^ (0x82F63B78 if c & 1 else 0)
        t.append(c)
    return t


_CRC32C = _crc32c_table()


def crc32c(data) -> int:
    """CRC-32C (Castagnoli: reflected polynomial 0x82F63B78, init and xorout 0xFFFFFFFF), one byte at a time"""
    crc, t = 0xFFFFFFFF, _CRC32C
    for b in bytes(data):
        crc = t[(crc ^ b) & 0xFF] ^ (crc >> 8)
    return crc ^ 0xFFFFFFFF


def batch_crc(seg, off) -> int:
    """the CRC a broker stores for the batch at `off`: over its bytes from attributes (21) to its end"""
    end = off + 12 + int.from_bytes(bytes(seg[off + 8:off + 12]), "big", signed=True)
    return crc32c(bytes(seg[off + 21:end]))


def set_crcs(seg) -> bytes:
    """seg with every batch's CRC field (bytes 17-20) set to the CRC-32C of the batch as it stands"""
    out = bytearray(seg)
    for o in batch_offsets(out):
        out[o + 17:o + 21] = batch_crc(out, o).to_bytes(4, "big")
    return bytes(out)


# ---- transactions (read_committed) ----------------------------------------------------------------------------------
def with_producer(batch: bytes, pid: int, epoch: int = 0, base_seq: int = 0) -> bytes:
    """a batch of encode_batch with its producerId / producerEpoch / baseSequence set (header bytes 43-56)"""
    b = bytearray(batch)
    b[43:57] = struct.pack(">qhi", pid, epoch, base_seq)
    return bytes(b)


def txn_batch(base_offset, base_ts, records, pid, epoch=0, base_seq=0, compression=None, transactional=True):
    """records as for encode_batch; attributes bit 4 = transactional"""
    return with_producer(encode_batch(base_offset, base_ts, records, attributes=0x10 if transactional else 0,
                                      compression=compression), pid, epoch, base_seq)


def marker_record_key(commit: bool, version: int = 0) -> bytes:
    return struct.pack(">hh", version, 1 if commit else 0)


def marker(offset, pid, epoch, commit, ts, key=None):
    """a control batch (attributes bits 4 and 5) holding one ABORT / COMMIT marker record: key version | type, value
    version | coordinatorEpoch"""
    key = marker_record_key(commit) if key is None else key
    return with_producer(encode_batch(offset, ts, [(0, 0, key, None, (), struct.pack(">hi", 0, 3))], attributes=0x30),
                         pid, epoch)


def txn_index(entries) -> bytes:
    """.txnindex image: (pid, firstOffset, lastOffset[, lastStableOffset]) → 34-byte big-endian entries, version 0"""
    return b"".join(struct.pack(">hqqqq", 0, e[0], e[1], e[2], e[3] if len(e) > 3 else e[2] + 1) for e in entries)


# ---- reading ----------------------------------------------------------------------------------------------------------
# one batch as read back: its header fields and its records [(offset, ts, key|None, value_len|None)]
Batch = namedtuple("Batch", "base_offset attributes base_ts producer_id count records max_ts")


def _read_varint(b, p):
    u, sh = 0, 0
    while True:
        x = b[p]
        p += 1
        u |= (x & 0x7F) << sh
        sh += 7
        if not x & 0x80:
            return (u >> 1) ^ -(u & 1), p


def _decompress(codec_bits, data):
    import pyarrow as pa
    if codec_bits == 0:
        return data
    if codec_bits == 1:
        return zlib.decompress(data, 31)
    if codec_bits == 2:
        if data[:8] == b"\x82SNAPPY\x00":             # xerial framing: chunks of u32 BE length + raw snappy
            out, p = bytearray(), 16
            while p < len(data):
                n = int.from_bytes(data[p:p + 4], "big")
                out += _decompress(2, data[p + 4:p + 4 + n])
                p += 4 + n
            return bytes(out)
        n, p = 0, 0
        for sh in range(0, 35, 7):                    # raw snappy: uncompressed length first
            n |= (data[p] & 0x7F) << sh
            p += 1
            if not data[p - 1] & 0x80:
                break
        return pa.decompress(data, decompressed_size=n, codec="snappy", asbytes=True)
    if codec_bits in (3, 4):
        return pa.CompressedInputStream(pa.BufferReader(data), "lz4" if codec_bits == 3 else "zstd").read()
    raise ValueError(codec_bits)


def read_segment(seg):
    """every batch of a segment as a Batch, its records as the consumer computes them: a record's timestamp is
    baseTimestamp + timestampDelta (in 64-bit arithmetic), and it is -1 ("not available") only when that sum is.  Every
    batch is read, control and LogAppendTime batches as they are stored (delivered() applies the consumer's rules)."""
    seg, out, pos = bytes(seg), [], 0
    while pos + 61 <= len(seg):
        base_off, bl = struct.unpack(">qi", seg[pos:pos + 12])
        attrs, = struct.unpack(">h", seg[pos + 21:pos + 23])
        base_ts, max_ts, pid = struct.unpack(">qqq", seg[pos + 27:pos + 51])
        cnt, = struct.unpack(">i", seg[pos + 57:pos + 61])
        body = _decompress(attrs & 7, seg[pos + 61:pos + 12 + bl])
        recs, p = [], 0
        for _ in range(cnt):
            ln, p = _read_varint(body, p)
            end = p + ln
            p += 1                                    # record attributes
            tsd, p = _read_varint(body, p)
            od, p = _read_varint(body, p)
            kl, p = _read_varint(body, p)
            key = None if kl < 0 else bytes(body[p:p + kl])
            p += max(kl, 0)
            vl, p = _read_varint(body, p)
            recs.append((base_off + od, _int64(base_ts + tsd), key, None if vl < 0 else vl))
            p = end
        out.append(Batch(base_off, attrs, base_ts, pid, cnt, recs, max_ts))
        pos += 12 + bl
    return out


def delivered(seg):
    """the records a consumer delivers from a segment (bytes, or read_segment's batches): control batches (attributes bit 5)
    and batches without records are not delivered, and a LogAppendTime batch (bit 3) stamps every record with its
    maxTimestamp"""
    batches = read_segment(seg) if isinstance(seg, (bytes, bytearray, memoryview)) else seg
    out = []
    for b in batches:
        if b.attributes & 0x20 or not b.records:
            continue
        out += [(off, b.max_ts, key, vl) for off, _, key, vl in b.records] if b.attributes & 0x08 else b.records
    return out
