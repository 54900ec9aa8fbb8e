"""The RecordBatch v2 CRC as a broker writes it (TEST INFRASTRUCTURE for check.crcs, kta_logcrc.cuh): a plain
byte-at-a-time CRC-32C, and the rewrite of every batch's CRC field in a segment.  kafka_codec's encoders write the field
as 0 (neither librdkafka by default nor the decoder with its check off read it); set_crcs gives such a segment the real
values.  Independent of the GPU pass under test: one table, one byte per step."""
import kafka_codec as kc


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
    """seg with every batch's CRC field (bytes 17-20) set to the CRC-32C of the batch as it stands (batches found by
    kafka_codec.batch_offsets)"""
    out = bytearray(seg)
    for o in kc.batch_offsets(out):
        out[o + 17:o + 21] = batch_crc(out, o).to_bytes(4, "big")
    return bytes(out)
