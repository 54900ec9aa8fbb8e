"""Kafka RecordBatch v2 (magic 2) ENCODER — TEST INFRASTRUCTURE for the GPU decoder (kta_logdecode.cuh).
Follows the Kafka protocol documentation for the record batch / record layout (KIP-98); independent of the
decoder's code.  CRC is written as 0: neither librdkafka by default (check.crcs=false) nor the decoder verify it."""
import struct


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


def varint(n: int) -> bytes:
    return uvarint(zigzag(n) & 0xFFFFFFFFFFFFFFFF)


def encode_record(offset_delta, ts_delta, key, value_len, headers=(), value=None):
    """value bytes are synthesised (the metric path never reads them) unless `value` gives them; value_len None (and no
    value) = tombstone"""
    body = bytearray(b"\x00")                      # record attributes
    body += varint(ts_delta) + varint(offset_delta)
    if key is None:
        body += varint(-1)
    else:
        body += varint(len(key)) + key
    if value is not None:
        assert value_len is None or value_len == len(value)
        body += varint(len(value)) + value
    elif value_len is None:
        body += varint(-1)
    else:
        body += varint(value_len) + bytes((i * 31 + 7) & 0xFF for i in range(value_len))
    body += varint(len(headers))
    for hk, hv in headers:
        body += varint(len(hk)) + hk
        body += varint(-1) if hv is None else varint(len(hv)) + hv
    return varint(len(body)) + bytes(body)


def compress_records(recs: bytes, codec: str) -> bytes:
    """The records section as a producer with compression.type=<codec> writes it.  The compressors are zlib's (gzip) and
    pyarrow's (LZ4 frame format, raw Snappy): independent of the GPU decompressor under test.  'snappy-xerial' adds the framing of the Java
    client's snappy-java stream (magic, two version words, chunks of u32 BE length + raw snappy)."""
    import pyarrow as pa
    if codec == "gzip":                                  # zlib's gzip wrapper (what librdkafka and the Java client write)
        import zlib
        c = zlib.compressobj(6, zlib.DEFLATED, 31)
        return c.compress(recs) + c.flush()
    if codec == "lz4":
        return pa.compress(recs, codec="lz4", asbytes=True)
    if codec == "snappy":
        return pa.compress(recs, codec="snappy", asbytes=True)
    if codec == "snappy-xerial":
        out = bytearray(b"\x82SNAPPY\x00" + struct.pack(">ii", 1, 1))
        step = max(1, len(recs) // 3 + 1)              # several chunks per batch
        for i in range(0, len(recs), step):
            c = pa.compress(recs[i:i + step], codec="snappy", asbytes=True)
            out += struct.pack(">i", len(c)) + c
        return bytes(out)
    raise ValueError(codec)


# Kafka's compression codec ids (attributes & 7), by the names these encoders take
CODEC_BITS = {None: 0, "gzip": 1, "snappy": 2, "snappy-xerial": 2, "lz4": 3, "zstd": 4, "zstd-stream": 4}


def encode_batch(base_offset, base_ts, records, attributes=0, max_ts=None, compression=None):
    """records: list of (offset_delta, ts_delta, key|None, value_len|None[, headers[, value]])"""
    recs = b"".join(encode_record(*r) for r in records)
    if compression:
        recs = compress_records(recs, compression)
        attributes |= CODEC_BITS[compression]
    last_delta = max((r[0] for r in records), default=0)
    if max_ts is None:
        max_ts = max((base_ts + r[1] for r in records), default=base_ts)
    after_len = struct.pack(">iBIhiqqqhii", 0, 2, 0, attributes, last_delta, base_ts, max_ts, -1, -1, -1, len(records)) + recs
    return struct.pack(">qi", base_offset, len(after_len)) + after_len


def batch_offsets(seg):
    """where every batch of a segment starts: the walk from batch header to batch header by batchLength"""
    seg, offs, pos = bytes(seg), [], 0
    while pos + 61 <= len(seg):
        offs.append(pos)
        pos += 12 + int.from_bytes(seg[pos + 8:pos + 12], "big", signed=True)
    return offs


def encode_partition(partition_records, rng, max_batch=40, log_append_time=False, compression=None):
    """partition_records: list of (ts_ms, key|None, value_len|None) in offset order → one log segment (bytes).
    ts_ms == -1 (not available) forces a batch with base timestamp -1."""
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
