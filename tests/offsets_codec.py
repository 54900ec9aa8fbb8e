"""The offsets a Kafka consumer fetches, over kafka_codec's RecordBatch v2 reader — TEST INFRASTRUCTURE for the offset
windows of the GPU decoder (kta_logoffsets.cuh).  Follows the broker's fetch rules and librdkafka's v2 reader;
independent of the decoder's code.

A consumer that starts at a partition's log start offset S and reads up to its high watermark H is served only the
batches with S <= last < H, last being baseOffset + the lastOffsetDelta stored in the batch (which can lie past the last
record of a compacted batch), and drops the records whose offset is below S inside the served batches that start below S
(the cut ones).  A batch that is not served is
known by its header alone: its records section is never read, as a consumer never receives it."""
import struct

import kafka_codec as kc


def with_last_offset_delta(batch, delta) -> bytes:
    """the batch with its stored lastOffsetDelta (header bytes 23-26) set: a compacted batch keeps the delta of the last
    record it had before compaction, which can exceed its last remaining record's (offset gaps come from the records'
    own offset deltas, which kafka_codec.encode_batch takes as given)"""
    b = bytearray(batch)
    b[23:27] = struct.pack(">i", delta)
    return bytes(b)


def _bound(x):
    return None if x is None or x == -1 else x


def fetched(seg, log_start=None, high_watermark=None):
    """the records a consumer delivers when it fetches from log_start up to high_watermark (None or -1: no bound), on top
    of kafka_codec.delivered(): a batch is served only when log_start <= last < high_watermark, last being baseOffset +
    the lastOffsetDelta stored in the batch's bytes; inside a served batch with baseOffset < log_start a record whose
    offset is below log_start is dropped"""
    return kc.delivered(_served(seg, _bound(log_start), _bound(high_watermark))[0])


def fetch_stats(seg, log_start=None, high_watermark=None):
    """(batches not served, records left out) of fetched(): the recordsCount of the data batches not served, plus the
    records dropped below log_start inside served data batches"""
    _, skipped, dropped = _served(seg, _bound(log_start), _bound(high_watermark))
    return len(skipped), sum(max(b.count, 0) for b in skipped if not b.attributes & 0x20) + dropped


def _served(seg, lo, hi):
    """(the served batches with their records below lo removed, the batches not served, the data records removed).  Records
    are removed only from cut batches, those with baseOffset < lo: a served batch at or past lo keeps every record, even one
    that a negative offset delta (which no broker writes) puts below lo"""
    served, skipped, dropped = [], [], 0
    for raw in kc.split_batches(bytes(seg)):
        base, = struct.unpack(">q", raw[:8])
        last = base + struct.unpack(">i", raw[23:27])[0]
        if (lo is not None and last < lo) or (hi is not None and last >= hi):
            attrs, = struct.unpack(">h", raw[21:23])
            skipped.append(kc.Batch(base, attrs, None, None, struct.unpack(">i", raw[57:61])[0], None, None))
            continue
        b = kc.read_segment(raw)[0]
        if lo is not None and base < lo:
            kept = [r for r in b.records if r[0] >= lo]
            if not b.attributes & 0x20:
                dropped += len(b.records) - len(kept)
            b = b._replace(records=kept)
        served.append(b)
    return served, skipped, dropped
