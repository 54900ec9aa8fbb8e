"""Host-side mirror of the reference's metric interface over libkta_gpu.so.

Names, argument meaning and error behaviour follow the reference so parity tests read like tests of
the reference itself:

    MessageMetrics                 /root/reference/src/metric.rs:11-204  (getters :104-195)
    LogCompactionInMemoryMetrics   /root/reference/src/metric.rs:262-285
    MetricHandler.handle_message   /root/reference/src/kafka.rs:18-20
    TopicAnalyzer.add_metric_handler / read_topic_into_metrics   src/kafka.rs:56-58, 74-137

All arithmetic happens on the GPU (and, for the O(P) derived getters, in the C library); this file
only marshals arguments.  Nothing here computes a metric in Python.
"""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass
from typing import Iterable, Optional

import numpy as np

from . import _native as N
from ._native import Batch, Config, KtaError, check, lib

TOTAL, TOMBSTONES, ALIVE, KEY_NULL, KEY_NON_NULL, KEY_SIZE_SUM, VALUE_SIZE_SUM = range(7)
KEY_SIZE_AVG, VALUE_SIZE_AVG, MESSAGE_SIZE_AVG = range(3)
SMALLEST_MESSAGE, LARGEST_MESSAGE, OVERALL_SIZE, OVERALL_COUNT = range(4)


@dataclass
class Message:
    """What the handlers read from rdkafka's BorrowedMessage (src/metric.rs:208-209,218,233)."""
    partition: int
    offset: int = 0
    timestamp_ms: Optional[int] = None   # None == Timestamp::NotAvailable
    key: Optional[bytes] = None          # None == null key; b"" == empty key
    payload_len: Optional[int] = None    # None == tombstone; 0 == empty value (bytes are never read)


def _ptr(a) -> Optional[int]:
    """Raw address of a numpy array / torch tensor / int / None."""
    if a is None:
        return None
    if isinstance(a, int):
        return a
    if isinstance(a, np.ndarray):
        return a.ctypes.data
    return a.data_ptr()  # torch.Tensor


class KtaEngine:
    """One kta_handle: MessageMetrics plus (optionally) LogCompactionInMemoryMetrics in one scan."""

    def __init__(self, num_partitions: int, count_alive_keys: bool = False, hll_precision: int = 0,
                 device: int = -1, ring_records: int = 0, ring_key_bytes: int = 0,
                 now: Optional[tuple] = None, alive_table_kib: int = 0, shard: Optional[tuple] = None,
                 isolation_level: str = "read_uncommitted", check_crcs: bool = False):
        """shard = (rank, world): this engine scans only partitions p with p % world == rank (a partition-sharded job).
        isolation_level: "read_uncommitted" (every data batch of a log segment is delivered) or "read_committed" (records
        of aborted transactions are left out, include/kta.h).  check_crcs: verify every record batch's CRC-32C and skip
        the batches that fail it (librdkafka's check.crcs; see set_check_crcs)."""
        levels = {"read_uncommitted": N.READ_UNCOMMITTED, "read_committed": N.READ_COMMITTED}
        if isolation_level not in levels:
            raise ValueError("isolation_level must be 'read_uncommitted' or 'read_committed', not %r" % (isolation_level,))
        cfg = Config()
        cfg.isolation_level = levels[isolation_level]
        cfg.struct_size = C.sizeof(Config)
        cfg.device = device
        cfg.num_partitions = num_partitions
        cfg.count_alive_keys = 1 if count_alive_keys else 0
        cfg.hll_precision = hll_precision
        cfg.alive_table_kib = alive_table_kib   # initial size of the alive-key table (0 = 256 MiB); it grows on demand
        cfg.ring_records = ring_records
        cfg.ring_key_bytes = ring_key_bytes
        if shard is not None:
            cfg.shard_rank, cfg.shard_world = shard
        if now is None:
            cfg.now_s, cfg.now_ns = N.INT64_MIN, 0
        else:
            cfg.now_s, cfg.now_ns = now
        self._h = C.c_void_p()
        self._keep = []  # device buffers that must outlive queued scans
        check(lib().kta_create(C.byref(cfg), C.byref(self._h)))
        if check_crcs:
            self.set_check_crcs(True)
        self.num_partitions = num_partitions
        self.count_alive_keys = bool(count_alive_keys)
        self.hll_precision = hll_precision
        self.shares_caller_stream = False   # True after set_stream(): work is ordered by the caller's stream
        self.timeline_buckets = 0           # set_timeline
        self.partitioner_counts = ()        # set_partitioner_check
        self.hot_keys_top_k = 0             # set_hot_keys
        self.message_metrics = MessageMetrics(self)
        self.log_compaction_metrics = LogCompactionInMemoryMetrics(self) if count_alive_keys else None

    # -- lifetime ---------------------------------------------------------------------------------
    def close(self) -> None:
        if getattr(self, "_h", None) is not None and self._h:
            lib().kta_destroy(self._h)
            self._h = C.c_void_p()
        self._keep = []

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()

    @property
    def handle(self):
        return self._h

    # -- ingest -----------------------------------------------------------------------------------
    def push(self, partition: int, offset: int, ts_ms: int, key: Optional[bytes], value_len: int) -> None:
        """MetricHandler::handle_message for one record (src/kafka.rs:107-109)."""
        if key is None:
            check(lib().kta_push(self._h, partition, offset, ts_ms, None, -1, value_len))
        else:
            buf = (C.c_char * max(len(key), 1)).from_buffer_copy(key or b"\0")
            check(lib().kta_push(self._h, partition, offset, ts_ms, C.cast(buf, C.c_void_p), len(key), value_len))

    def handle_message(self, m: Message) -> None:
        self.push(m.partition, m.offset, -1 if m.timestamp_ms is None else m.timestamp_ms, m.key,
                  -1 if m.payload_len is None else m.payload_len)

    def _batch(self, n, partition, ts_ms, key_len, value_len, key_bytes, key_bytes_len, key_tile_base, seq,
               seq_base, offset) -> Batch:
        b = Batch()
        b.n = n
        b.seq_base = N.SEQ_AUTO if seq_base is None else seq_base   # None: continue the handle's running count
        b.partition, b.offset, b.ts_ms = _ptr(partition), _ptr(offset), _ptr(ts_ms)
        b.key_len, b.value_len, b.key_bytes = _ptr(key_len), _ptr(value_len), _ptr(key_bytes)
        b.key_bytes_len = key_bytes_len
        b.key_tile_base, b.seq = _ptr(key_tile_base), _ptr(seq)
        return b

    def push_batch_host(self, partition, ts_ms, key_len, value_len, key_bytes=None, key_tile_base=None, seq=None,
                        seq_base: Optional[int] = None, offset=None) -> None:
        """SoA batch in host memory (numpy arrays, or pinned torch CPU tensors).  seq_base None = the records follow
        everything this engine has seen so far (src/kafka.rs:99: `seq += 1` per polled message)."""
        n = int(partition.shape[0])
        kbl = 0 if key_bytes is None else int(key_bytes.shape[0])
        b = self._batch(n, partition, ts_ms, key_len, value_len, key_bytes, kbl, key_tile_base, seq, seq_base, offset)
        check(lib().kta_push_batch_host(self._h, C.byref(b)))

    def scan_batch_device(self, partition, ts_ms, key_len, value_len, key_bytes=None, key_bytes_len: int = 0,
                          key_tile_base=None, seq=None, seq_base: Optional[int] = None, n: Optional[int] = None) -> None:
        """SoA batch already in HBM (torch CUDA tensors or raw device addresses).  Asynchronous."""
        if n is None:
            n = int(partition.shape[0])
        b = self._batch(n, partition, ts_ms, key_len, value_len, key_bytes, key_bytes_len, key_tile_base, seq,
                        seq_base, None)
        self._keep.append((partition, ts_ms, key_len, value_len, key_bytes, key_tile_base, seq))
        check(lib().kta_scan_batch_device(self._h, C.byref(b)))

    def push_log_segment(self, partition: int, data) -> int:
        """Decode + scan one Kafka log segment (RecordBatch v2 bytes of one partition, host memory).  Returns the
        number of records delivered to the handlers."""
        buf = np.frombuffer(data, dtype=np.uint8) if not isinstance(data, np.ndarray) else data
        n = C.c_int64()
        check(lib().kta_push_log_segment_host(self._h, partition, buf.ctypes.data, buf.size, C.byref(n)))
        return n.value

    def scan_log_batches_device(self, dev_bytes, length: int, dev_batch_off, dev_batch_partition, nbatches: int) -> int:
        """RecordBatch v2 batches of any partitions lying in ONE device buffer (torch CUDA tensors / raw addresses): one
        decode + one scan.  Returns the number of records delivered to the handlers."""
        n = C.c_int64()
        self._keep.append((dev_bytes, dev_batch_off, dev_batch_partition))
        check(lib().kta_scan_log_batches_device(self._h, _ptr(dev_bytes), length, _ptr(dev_batch_off), _ptr(dev_batch_partition),
                                                nbatches, C.byref(n)))
        return n.value

    def push_log_segments(self, segments) -> int:
        """segments: iterable of (partition, bytes-like).  One decode + one scan for all of them."""
        segs = [(int(p), np.frombuffer(d, dtype=np.uint8) if not isinstance(d, np.ndarray) else d) for p, d in segments]
        k = len(segs)
        parts = (C.c_int32 * k)(*[p for p, _ in segs])
        ptrs = (C.c_void_p * k)(*[d.ctypes.data for _, d in segs])
        lens = (C.c_int64 * k)(*[d.size for _, d in segs])
        n = C.c_int64()
        check(lib().kta_push_log_segments_host(self._h, k, parts, ptrs, lens, C.byref(n)))
        return n.value

    def push_txn_index(self, partition: int, data) -> None:
        """Register the aborted transactions of one .txnindex image of `partition` for every later log call
        (read_committed engines only)."""
        buf = np.frombuffer(data, dtype=np.uint8) if not isinstance(data, np.ndarray) else data
        check(lib().kta_log_add_txn_index_host(self._h, partition, buf.ctypes.data if buf.size else None, buf.size))

    def log_txn_stats(self):
        """(aborted batches, aborted records, undecided records) since create / reset (read_committed engines only)."""
        v = [C.c_uint64() for _ in range(3)]
        check(lib().kta_log_txn_stats(self._h, *[C.byref(x) for x in v]))
        return tuple(x.value for x in v)

    def set_check_crcs(self, enabled: bool) -> None:
        """check.crcs for every later log call: a record batch whose CRC-32C does not match is skipped unread and
        listed (log_crc_failures) instead of being decoded.  Off by default; reset() keeps the setting."""
        check(lib().kta_log_set_check_crcs(self._h, 1 if enabled else 0))

    def log_crc_stats(self):
        """(checked batches, failed batches, failed bytes) over the successful log calls since create / reset."""
        v = [C.c_uint64() for _ in range(3)]
        check(lib().kta_log_crc_stats(self._h, *[C.byref(x) for x in v]))
        return tuple(x.value for x in v)

    def log_crc_failures(self):
        """The kept failures (the first N.LOG_CRC_KEEP since create / reset), in call order and, within a call, in batch
        order: [(partition, batch bytes, base offset, stored crc, computed crc)]."""
        n = C.c_int64()
        check(lib().kta_log_crc_failures(self._h, None, 0, C.byref(n)))
        buf = (N.CrcFailure * max(n.value, 1))()
        check(lib().kta_log_crc_failures(self._h, buf, n.value, C.byref(n)))
        return [(f.partition, f.batch_bytes, f.base_offset, f.stored_crc, f.computed_crc) for f in buf[:n.value]]

    def set_log_offsets(self, partition: int, log_start_offset: Optional[int] = None,
                        high_watermark: Optional[int] = None) -> None:
        """The offsets a consumer of `partition` fetches, for every later log call: from its log start offset up to its
        high watermark (None = no bound on that side).  Batches outside are skipped unread, and records below the log
        start offset inside a served batch are dropped (include/kta.h).  A later call replaces the window; reset()
        clears every window."""
        check(lib().kta_log_set_offsets(self._h, partition, -1 if log_start_offset is None else log_start_offset,
                                        -1 if high_watermark is None else high_watermark))

    def log_offset_stats(self):
        """(batches not served, records left out) over the successful log calls since create / reset."""
        v = [C.c_uint64() for _ in range(2)]
        check(lib().kta_log_offset_stats(self._h, *[C.byref(x) for x in v]))
        return tuple(x.value for x in v)

    def set_timeline(self, origin_s: int, width_s: int, buckets: int) -> None:
        """Count each partition's records, tombstones and bytes per time bucket: index 0 before origin_s, index
        1 + (t - origin_s) // width_s for the `buckets` buckets of width_s seconds, index buckets + 1 after them
        (include/kta.h).  Only before the first record (after create or reset); buckets = 0 turns it off; reset()
        keeps the setting."""
        check(lib().kta_set_timeline(self._h, origin_s, width_s, buckets))
        self.timeline_buckets = buckets

    def timeline(self, which: int, p: int) -> np.ndarray:
        """One partition's row of a timeline counter (N.TIMELINE_RECORDS / _TOMBSTONES / _BYTES): buckets + 2 u64,
        after finalize()."""
        n = self.timeline_buckets + 2
        out = np.zeros(n, dtype=np.uint64)
        check(lib().kta_timeline(self._h, which, p, out.ctypes.data_as(C.POINTER(C.c_uint64)), n))
        return out

    def timeline_shape(self, n: int):
        """(grid, threads, bins in shared memory) of the timeline pass over a scan of n records (test hook)."""
        g, t, s = C.c_int32(), C.c_int32(), C.c_int32()
        check(lib().kta_timeline_shape(self._h, n, C.byref(g), C.byref(t), C.byref(s)))
        return g.value, t.value, bool(s.value)

    def set_partitioner_check(self, counts) -> None:
        """Per partition, count the keyed records that Kafka's murmur2 partitioner and librdkafka's CRC-32 partitioner
        would place there at each partition count in `counts` (at most 8, distinct, each in [1, 2^31 - 1];
        include/kta.h).  Only before the first record (after create or reset); an empty list turns it off; reset() keeps
        the setting."""
        counts = [int(c) for c in counts]
        bad = [c for c in counts if not 1 <= c < 1 << 31]
        if bad:   # (ctypes would wrap them into int32 silently)
            raise KtaError(N.ERR_INVALID, "partition count %d outside [1, 2^31 - 1]" % bad[0])
        arr = (C.c_int32 * max(len(counts), 1))(*counts)
        check(lib().kta_set_partitioner_check(self._h, arr, len(counts)))
        self.partitioner_counts = tuple(counts)

    def partitioner_check(self, p: int) -> np.ndarray:
        """One partition's 2C + 1 u64 after finalize(): murmur2 matches per count, CRC-32 matches per count, neither."""
        n = 2 * len(self.partitioner_counts) + 1
        out = np.zeros(n, dtype=np.uint64)
        check(lib().kta_partitioner_check(self._h, p, out.ctypes.data_as(C.POINTER(C.c_uint64)), n))
        return out

    def partitioner_limit_grid(self, max_ctas: int) -> None:
        """at most max_ctas CTAs per partitioner pass, 0 = no limit (test hook)."""
        check(lib().kta_partitioner_limit_grid(self._h, max_ctas))

    def partitioner_shape(self, n: int, key_bytes: int):
        """(grid, stage bytes per warp, counters in shared memory) of the partitioner pass over a scan of n records with
        key_bytes key bytes (test hook)."""
        g, s, m = C.c_int32(), C.c_int32(), C.c_int32()
        check(lib().kta_partitioner_shape(self._h, n, key_bytes, C.byref(g), C.byref(s), C.byref(m)))
        return g.value, s.value, bool(m.value)

    def partitioner_hashes(self, key_len, key_bytes):
        """(murmur2, crc32) u32 arrays of the check's device hash functions over packed host keys (test hook)."""
        kl = np.ascontiguousarray(key_len, dtype=np.int32)
        kb = np.ascontiguousarray(key_bytes, dtype=np.uint8)
        mm, cc = np.zeros(kl.size, np.uint32), np.zeros(kl.size, np.uint32)
        check(lib().kta_partitioner_hash_host(self._h, kl.size, kl.ctypes.data, kb.ctypes.data if kb.size else None, kb.size,
                                              mm.ctypes.data, cc.ctypes.data))
        return mm, cc

    def set_hot_keys(self, top_k: int, table_slots: int = 0) -> None:
        """Count every key's records, tombstones and bytes in an exact table on the GPU and keep the top_k keys with the
        most records (include/kta.h).  top_k in [1, 65536], 0 turns it off; table_slots 0 (2^20) or a power of two in
        [16, 2^31].  Only before the first record (after create or reset); reset() keeps the setting."""
        top_k, table_slots = int(top_k), int(table_slots)
        if not 0 <= top_k < 1 << 31 or not 0 <= table_slots < 1 << 63:   # (ctypes would wrap them silently)
            raise KtaError(N.ERR_INVALID, "top_k %d / table_slots %d out of range" % (top_k, table_slots))
        check(lib().kta_set_hot_keys(self._h, top_k, table_slots))
        self.hot_keys_top_k = top_k

    def hot_keys(self, as_dicts: bool = False):
        """The top keys after finalize(), by records descending then id ascending: a numpy structured array of
        _native.HOT_KEY_DTYPE, or (as_dicts) a list of dicts whose key_prefix is the key's first min(key_len, 32) bytes."""
        out = np.zeros(max(self.hot_keys_top_k, 1), dtype=N.HOT_KEY_DTYPE)
        n = C.c_int64()
        check(lib().kta_hot_keys(self._h, out.ctypes.data, out.size, C.byref(n)))
        out = out[:n.value]
        if not as_dicts:
            return out
        return [dict({f: int(r[f]) for f in N.HOT_KEY_DTYPE.names if f != "key_prefix"},
                     key_prefix=bytes(r["key_prefix"][:min(int(r["key_len"]), N.HOT_KEY_PREFIX)])) for r in out]

    def hot_key_stats(self):
        """(distinct keys, keyed records, slots, grows, slices) after finalize()."""
        v = [C.c_uint64() for _ in range(5)]
        check(lib().kta_hot_key_stats(self._h, *[C.byref(x) for x in v]))
        return tuple(x.value for x in v)

    def hot_keys_export_count(self) -> int:
        n = C.c_int64()
        check(lib().kta_hot_keys_export_count(self._h, C.byref(n)))
        return n.value

    def hot_keys_export(self, dev_out, cap: int) -> int:
        """every entry into a device buffer of cap 88-byte entries; returns how many"""
        n = C.c_int64()
        check(lib().kta_hot_keys_export_device(self._h, _ptr(dev_out), cap, C.byref(n)))
        return n.value

    def hot_keys_import(self, dev_in, count: int) -> None:
        check(lib().kta_hot_keys_import_device(self._h, _ptr(dev_in), count))

    def hot_keys_limit_slots(self, max_slots: int) -> None:
        """the table may not grow beyond max_slots slots, 0 = no cap (test hook)."""
        check(lib().kta_hot_keys_limit_slots(self._h, max_slots))

    def sync(self) -> None:
        check(lib().kta_sync(self._h))
        self._keep = []

    def reset(self) -> None:
        check(lib().kta_reset(self._h))

    def finalize(self, strict: bool = True) -> int:
        """kta_sync + state to the host.  Records whose partition lies outside [0, num_partitions) are left out of every
        metric: with strict (default) that raises KtaError(ERR_PARTITION) — the getters are valid nevertheless —, without
        it the number of such records is returned."""
        try:
            rc = lib().kta_finalize(self._h)
        finally:
            self._keep = []
        if rc == N.ERR_PARTITION and not strict:
            return self.bad_partition_records()
        check(rc)
        return 0

    # -- read-back --------------------------------------------------------------------------------
    def counter(self, which: int, p: int) -> int:
        out = C.c_uint64()
        check(lib().kta_counter(self._h, which, p, C.byref(out)))
        return out.value

    def avg(self, which: int, p: int) -> int:
        out = C.c_uint64()
        rc = lib().kta_avg(self._h, which, p, C.byref(out))
        if rc == N.ERR_DIV_BY_ZERO:
            # the reference panics: "attempt to divide by zero" (src/metric.rs:135,144,153)
            raise ZeroDivisionError((lib().kta_last_error() or b"").decode())
        check(rc)
        return out.value

    def global_(self, which: int) -> int:
        out = C.c_uint64()
        check(lib().kta_global(self._h, which, C.byref(out)))
        return out.value

    def timestamps(self):
        es, ens, ls = C.c_int64(), C.c_int32(), C.c_int64()
        check(lib().kta_timestamps(self._h, C.byref(es), C.byref(ens), C.byref(ls)))
        return es.value, ens.value, ls.value

    def hist(self, which: int, p: int) -> np.ndarray:
        out = (C.c_uint64 * N.KTA_HIST_BUCKETS)()
        check(lib().kta_hist(self._h, which, p, out))
        return np.frombuffer(out, dtype=np.uint64).copy()

    def alive_keys(self) -> int:
        out = C.c_uint64()
        check(lib().kta_alive_keys(self._h, C.byref(out)))
        return out.value

    def bad_partition_records(self) -> int:
        out = C.c_uint64()
        check(lib().kta_bad_partition_records(self._h, C.byref(out)))
        return out.value

    def alive_table_stats(self):
        """(slots, occupied, grows, reruns) of the alive-key table."""
        v = [C.c_uint64() for _ in range(4)]
        check(lib().kta_alive_table_stats(self._h, *[C.byref(x) for x in v]))
        return tuple(x.value for x in v)

    def alive_keys_hll(self) -> float:
        out = C.c_double()
        check(lib().kta_alive_keys_hll(self._h, C.byref(out)))
        return out.value

    def hll_registers(self) -> np.ndarray:
        regs = np.zeros(1 << self.hll_precision, dtype=np.uint8)
        check(lib().kta_hll_registers(self._h, regs.ctypes.data, regs.size))
        return regs

    def fnv32(self, keys: Iterable[Optional[bytes]]) -> np.ndarray:
        """The reference hash (src/fnv32.rs:92-101) of each key, computed on the device."""
        keys = list(keys)
        lens = np.array([-1 if k is None else len(k) for k in keys], dtype=np.int32)
        blob = np.frombuffer(b"".join(k for k in keys if k) or b"\0", dtype=np.uint8)
        out = np.zeros(len(keys), dtype=np.uint32)
        total = int(sum(len(k) for k in keys if k))
        check(lib().kta_fnv32_host(self._h, len(keys), lens.ctypes.data, blob.ctypes.data, total, out.ctypes.data))
        return out

    def set_stream(self, cuda_stream: int) -> None:
        """Run on a caller-owned CUDA stream (e.g. torch.cuda.current_stream().cuda_stream)."""
        check(lib().kta_set_stream(self._h, cuda_stream))
        self.shares_caller_stream = True

    def merge_words(self, world: int) -> int:
        return lib().kta_merge_words(self._h, world)

    def merge_export(self, rank: int, world: int, dev_buf) -> None:
        check(lib().kta_merge_export_device(self._h, rank, world, _ptr(dev_buf)))

    def merge_import(self, world: int, dev_buf) -> None:
        check(lib().kta_merge_import_device(self._h, world, _ptr(dev_buf)))

    def alive_export_count(self) -> int:
        n = C.c_int64()
        check(lib().kta_alive_export_count(self._h, C.byref(n)))
        return n.value

    def alive_export(self, dev_hash, dev_stamp, cap: int) -> int:
        n = C.c_int64()
        check(lib().kta_alive_export_device(self._h, _ptr(dev_hash), _ptr(dev_stamp), cap, C.byref(n)))
        return n.value

    def alive_import(self, dev_hash, dev_stamp, count: int) -> None:
        check(lib().kta_alive_import_device(self._h, _ptr(dev_hash), _ptr(dev_stamp), count))

    def stats(self):
        a, b = C.c_uint64(), C.c_uint64()
        check(lib().kta_stats(self._h, C.byref(a), C.byref(b)))
        return a.value, b.value

    def set_timing(self, on: bool) -> None:
        check(lib().kta_set_timing(self._h, 1 if on else 0))

    def scan_time_ms(self):
        ms, n = C.c_double(), C.c_uint64()
        check(lib().kta_scan_time_ms(self._h, C.byref(ms), C.byref(n)))
        return ms.value, n.value


class MessageMetrics:
    """Getter surface of the reference's MessageMetrics (src/metric.rs:104-195)."""

    def __init__(self, engine: KtaEngine):
        self.engine = engine

    def handle_message(self, m: Message) -> None:  # impl MetricHandler, src/metric.rs:206-253
        self.engine.handle_message(m)

    def total(self, p): return self.engine.counter(TOTAL, p)
    def tombstones(self, p): return self.engine.counter(TOMBSTONES, p)
    def alive(self, p): return self.engine.counter(ALIVE, p)
    def key_null(self, p): return self.engine.counter(KEY_NULL, p)
    def key_non_null(self, p): return self.engine.counter(KEY_NON_NULL, p)
    def key_size_sum(self, p): return self.engine.counter(KEY_SIZE_SUM, p)
    def value_size_sum(self, p): return self.engine.counter(VALUE_SIZE_SUM, p)
    def key_size_avg(self, p): return self.engine.avg(KEY_SIZE_AVG, p)
    def value_size_avg(self, p): return self.engine.avg(VALUE_SIZE_AVG, p)
    def message_size_avg(self, p): return self.engine.avg(MESSAGE_SIZE_AVG, p)

    def dirty_ratio(self, p) -> float:
        out = C.c_float()
        check(lib().kta_dirty_ratio(self.engine.handle, p, C.byref(out)))
        return out.value

    def earliest_message(self):
        """(seconds, nanoseconds) since the epoch, UTC."""
        es, ens, _ = self.engine.timestamps()
        return es, ens

    def latest_message(self) -> int:
        return self.engine.timestamps()[2]

    def smallest_message(self): return self.engine.global_(SMALLEST_MESSAGE)
    def largest_message(self): return self.engine.global_(LARGEST_MESSAGE)
    def overall_size(self): return self.engine.global_(OVERALL_SIZE)
    def overall_count(self): return self.engine.global_(OVERALL_COUNT)


class LogCompactionInMemoryMetrics:
    """src/metric.rs:262-305: alive keys of a log-compacted topic (exact, keyed by the 32-bit hash)."""

    def __init__(self, engine: KtaEngine):
        self.engine = engine

    def handle_message(self, m: Message) -> None:
        self.engine.handle_message(m)

    def sum_all_alive(self) -> int:  # src/metric.rs:282-284
        return self.engine.alive_keys()


class TopicAnalyzer:
    """The driver of src/kafka.rs:74-137 over an in-memory message source instead of librdkafka."""

    def __init__(self):
        self.metric_handlers = []

    def add_metric_handler(self, handler) -> None:  # src/kafka.rs:56-58
        self.metric_handlers.append(handler)

    def read_topic_into_metrics(self, messages: Iterable[Message], end_offsets: dict) -> int:
        """Feeds every message to every registered handler once, in order, until every partition has
        reached its end offset (src/kafka.rs:119-132).  Handlers that share one engine are fed once."""
        engines = []
        for mh in self.metric_handlers:
            if mh.engine not in engines:
                engines.append(mh.engine)
        still_running = {p: True for p in end_offsets}
        seq = 0
        for m in messages:
            seq += 1
            for e in engines:
                e.handle_message(m)
            if m.offset + 1 >= end_offsets[m.partition]:
                still_running[m.partition] = False
            if not any(still_running.values()):
                break
        for e in engines:
            e.finalize()
        return seq


__all__ = ["KtaEngine", "MessageMetrics", "LogCompactionInMemoryMetrics", "TopicAnalyzer", "Message", "KtaError"]
