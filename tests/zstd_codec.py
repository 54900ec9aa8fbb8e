"""zstd record batches — TEST INFRASTRUCTURE for the GPU decoder's zstd walk (kta_zstd.cuh), on top of kafka_codec's
RecordBatch v2 encoder: a batch is encoded uncompressed by kafka_codec, then its records section is re-written compressed.
The compressor is pyarrow's zstd, independent of the decoder under test:
  'zstd'         one-shot, the frame carries Frame_Content_Size;
  'zstd-stream'  pyarrow's CompressedOutputStream, no Frame_Content_Size (as streaming compressors such as the Java
                 client's write it).
Any other codec name is handed to kafka_codec.compress_records."""
import struct

import kafka_codec as kc

def compress_records(recs: bytes, codec: str) -> bytes:
    import pyarrow as pa
    if codec == "zstd":
        return pa.compress(recs, codec="zstd", asbytes=True)
    if codec == "zstd-stream":
        sink = pa.BufferOutputStream()
        with pa.CompressedOutputStream(sink, "zstd") as s:
            s.write(recs)
        return sink.getvalue().to_pybytes()
    return kc.compress_records(recs, codec)


def recompress(seg: bytes, pick) -> bytes:
    """every batch of an uncompressed segment with its records section compressed by pick() (a codec name, or None to
    leave the batch as it is); batchLength and the attributes' codec bits follow"""
    out, offs = bytearray(), kc.batch_offsets(seg)
    for pos, end in zip(offs, offs[1:] + [len(seg)]):
        hdr, body = bytearray(seg[pos:pos + 61]), seg[pos + 61:end]
        codec = pick()
        if codec:
            body = compress_records(body, codec)
            hdr[8:12] = struct.pack(">i", 49 + len(body))
            hdr[22] |= kc.CODEC_BITS[codec]
        out += hdr + body
    return bytes(out)


def encode_batch(base_offset, base_ts, records, attributes=0, compression=None):
    """kafka_codec.encode_batch, with the zstd codecs too"""
    return recompress(kc.encode_batch(base_offset, base_ts, records, attributes=attributes), lambda: compression)


def encode_partition(partition_records, rng, max_batch=40, compression=None):
    """kafka_codec.encode_partition, with the zstd codecs too; a list of codecs: every batch picks its own"""
    seg = kc.encode_partition(partition_records, rng, max_batch=max_batch)
    if isinstance(compression, (list, tuple)):
        return recompress(seg, lambda: compression[int(rng.integers(0, len(compression)))])
    return recompress(seg, lambda: compression)
