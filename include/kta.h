/*
 * kta.h — C ABI of libkta_gpu.so: the H100-native (sm_90a) replacement for the per-message
 * metric-aggregation path of xenji/kafka-topic-analyzer.
 *
 * Boundary being replaced (reference, Rust):
 *   trait MetricHandler { fn handle_message(&mut self, m: &BorrowedMessage) }    src/kafka.rs:18-20
 *   TopicAnalyzer::add_metric_handler                                            src/kafka.rs:56-58
 *   call site, once per handler per polled message                               src/kafka.rs:107-109
 *   impl MetricHandler for MessageMetrics                                        src/metric.rs:206-253
 *   impl MetricHandler for LogCompactionInMemoryMetrics                          src/metric.rs:288-305
 *   read-back: getters src/metric.rs:104-195, sum_all_alive :282-284, used at    src/main.rs:130-170
 *
 * One kta_handle is BOTH handlers (MessageMetrics always; LogCompactionInMemoryMetrics when
 * cfg.count_alive_keys == 1, mirroring `-c`, src/main.rs:77-80).
 *
 * Rules of the boundary
 *   - plain C types only; no exceptions or unwinding cross it; every entry point returns a status
 *     (KTA_OK == 0) and kta_last_error() gives the text for the last failure on the calling thread.
 *   - single-producer: all calls on one handle come from one host thread, as in the reference
 *     (handlers are `&mut`, src/kafka.rs:15).  Different handles are independent.
 *   - the library copies what it needs before a push returns; caller buffers are never retained
 *     (BorrowedMessage is only borrowed for the call, src/kafka.rs:107-109).
 *   - there is NO CPU fallback: without a usable CUDA device kta_create fails with KTA_ERR_CUDA.
 *
 * Record encoding (rdkafka 0.25.0 accessor semantics, call sites src/metric.rs:208-209,218,233):
 *   key_len   == -1  key() is None            key_len   == 0  Some(&[])  (hashes to 0x811c9dc5)
 *   value_len == -1  payload() is None (tombstone)             value_len == 0  Some(&[])  (alive)
 *   ts_ms     == -1  timestamp().to_millis() is None → treated as 0 (src/metric.rs:209)
 *   partition must lie in [0, cfg.num_partitions)
 *   value BYTES never cross the boundary: the reference only reads v.len() (src/metric.rs:235).
 */
#ifndef KTA_H
#define KTA_H
#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define KTA_ABI_VERSION 2
#define KTA_KEY_TILE 128      /* records per key tile (granularity of kta_batch.key_tile_base) */
#define KTA_HIST_BUCKETS 32   /* bucket(len) = len == 0 ? 0 : 1 + floor(log2(len)) */

enum {
    KTA_OK = 0,
    KTA_ERR_INVALID = 1,       /* bad argument / bad state */
    KTA_ERR_CUDA = 2,          /* CUDA runtime failure (including: no device) */
    KTA_ERR_NOMEM = 3,
    KTA_ERR_PARTITION = 4,     /* a record's partition was outside [0, num_partitions) */
    KTA_ERR_DIV_BY_ZERO = 5,   /* the reference would panic here: avg with sum > 0 && alive == 0
                                  (src/metric.rs:132-157) */
    KTA_ERR_NOT_ENABLED = 6,   /* getter for a feature that was not enabled at create */
    KTA_ERR_NOT_FINALIZED = 7
};

typedef struct kta_handle kta_handle;

/* kta_config.isolation_level (librdkafka's isolation.level) */
#define KTA_READ_UNCOMMITTED 0
#define KTA_READ_COMMITTED 1

typedef struct kta_config {
    int32_t struct_size;       /* = sizeof(kta_config) */
    int32_t device;            /* CUDA device ordinal, -1 = current device */
    int32_t num_partitions;    /* P; partition ids are 0..P-1 (metadata, src/kafka.rs:60-72) */
    int32_t count_alive_keys;  /* 1 = exact alive-key table, i.e. `-c` given once (src/main.rs:77-80) */
    int32_t hll_precision;     /* EXTENSION: 0 = off, else 4..18 HyperLogLog index bits */
    int32_t alive_table_kib;   /* initial size of the alive-key table in KiB (8 bytes per distinct key hash, kept at
                                  load <= 0.6 and grown on demand); 0 = default (262144 = 256 MiB: 1e7 keys) */
    int64_t ring_records;      /* records per landing-ring chunk for kta_push / host batches; 0 = default */
    int64_t ring_key_bytes;    /* key bytes per landing-ring chunk; 0 = default */
    int64_t now_s;             /* construction wall clock for earliest_message (Utc::now(), */
    int32_t now_ns;            /*   src/metric.rs:39); now_s == INT64_MIN → library reads the clock */
    int32_t isolation_level;   /* log entry points: KTA_READ_UNCOMMITTED (0, every data batch is delivered) or
                                  KTA_READ_COMMITTED (records of aborted transactions are left out, see below) */
    int32_t shard_world;       /* partition-sharded job (one handle per GPU, gpu = partition mod G, SURVEY.md §8 e): this */
    int32_t shard_rank;        /*   handle scans only partitions p with p % shard_world == shard_rank; records of other
                                    partitions are left out like out-of-range ones.  0 or 1 = not sharded.  The handle
                                    still holds (and, after kta_merge_import_device, reports) all num_partitions.
                                    Shapes are limited by the scan's division p / G = mulhi(p, ceil(2^32 / G)): with
                                    e = ceil(2^32 / G) * G - 2^32, kta_create refuses (KTA_ERR_INVALID) unless
                                    (num_partitions - 1) * e < 2^32.  Every num_partitions <= 65536 and every
                                    shard_world <= 4096 is accepted. */
} kta_config;

/* kta_batch.seq_base value that means "continue this handle's running count" (what kta_push does: the consumer's
 * `seq += 1`, src/kafka.rs:99) */
#define KTA_SEQ_AUTO UINT64_MAX

/* SoA record batch.  Pointers are all host or all device (see the two scan entry points). */
typedef struct kta_batch {
    int64_t n;                     /* records */
    uint64_t seq_base;             /* seq of record 0; record i has seq_base + i (src/kafka.rs:99), or KTA_SEQ_AUTO.
                                      With count_alive_keys the LAST record of a key decides (src/metric.rs:295,298) and
                                      "last" is by seq: a batch without a seq column whose seq_base lies below the
                                      handle's running count is refused (it would let older records win silently). */
    const int32_t *partition;      /* [n] */
    const int64_t *offset;         /* [n] carried for the caller; never read by a metric (may be NULL) */
    const int64_t *ts_ms;          /* [n] */
    const int32_t *key_len;        /* [n] */
    const int32_t *value_len;      /* [n] */
    const uint8_t *key_bytes;      /* keys packed back to back in record order (null/empty keys take
                                      0 bytes); may be NULL when neither -c nor HLL is enabled */
    int64_t key_bytes_len;         /* = sum(max(key_len, 0)) */
    const uint64_t *key_tile_base; /* optional [ceil(n/KTA_KEY_TILE)+1]: byte offset into key_bytes
                                      of the first key of each tile (+ total at the end).  NULL →
                                      the library derives it with one extra pass over key_len. */
    const uint64_t *seq;           /* optional [n] explicit sequence numbers (partition-sharded
                                      scans, where the global order is not base+i); NULL → seq_base+i.
                                      The alive-key table keeps 31 bits of seq: explicit sequence numbers must stay
                                      below 2^31 - 2 between kta_reset calls (kta_finalize reports violations);
                                      implicit ones are unlimited (the table is rebased as the stream advances). */
} kta_batch;

enum kta_counter_id { /* per-partition counters, src/metric.rs:13-19 / getters :104-130 */
    KTA_TOTAL = 0,
    KTA_TOMBSTONES = 1,
    KTA_ALIVE = 2,
    KTA_KEY_NULL = 3,
    KTA_KEY_NON_NULL = 4,
    KTA_KEY_SIZE_SUM = 5,
    KTA_VALUE_SIZE_SUM = 6
};
enum kta_avg_id { KTA_KEY_SIZE_AVG = 0, KTA_VALUE_SIZE_AVG = 1, KTA_MESSAGE_SIZE_AVG = 2 };
enum kta_global_id { /* src/metric.rs:22-25 / getters :177-195 */
    KTA_SMALLEST_MESSAGE = 0,
    KTA_LARGEST_MESSAGE = 1,
    KTA_OVERALL_SIZE = 2,
    KTA_OVERALL_COUNT = 3
};

const char *kta_last_error(void);
int kta_abi_version(void);
/* number of CUDA devices visible, or -1 if the runtime cannot initialise (no throw, no abort) */
int kta_device_count(void);

/* MessageMetrics::new + (cfg.count_alive_keys) LogCompactionInMemoryMetrics::new
 * src/metric.rs:30-46, 267-271; registration src/main.rs:108-115 */
int kta_create(const kta_config *cfg, kta_handle **out);
int kta_destroy(kta_handle *h);
/* back to the just-constructed state (keeps device allocations) */
int kta_reset(kta_handle *h);

/* MetricHandler::handle_message for one record (src/kafka.rs:107-109).  Lands the record in a
 * pinned ring chunk; full chunks are staged to HBM with cudaMemcpyAsync and scanned asynchronously.
 * `offset` is accepted for interface parity and ignored.  `key` may be NULL iff key_len <= 0. */
int kta_push(kta_handle *h, int32_t partition, int64_t offset, int64_t ts_ms, const uint8_t *key,
             int32_t key_len, int32_t value_len);

/* The same for a whole SoA batch in HOST memory (pinned or pageable): chunked host→device copies
 * overlapped with the scan kernels.  Returns once the caller's buffers may be reused. */
int kta_push_batch_host(kta_handle *h, const kta_batch *b);

/* The same for an SoA batch already resident in DEVICE memory (asynchronous on the handle's
 * stream; the buffers must stay valid until kta_sync / kta_finalize). */
int kta_scan_batch_device(kta_handle *h, const kta_batch *b);

/* drain the ring and wait for all queued scans */
int kta_sync(kta_handle *h);
/* kta_sync + resolve the alive-key table + bring the metric state to the host.  Getters below are
 * valid after this.  More records may be pushed afterwards; finalize again to refresh. */
int kta_finalize(kta_handle *h);

/* getters — src/metric.rs:104-130 */
int kta_counter(const kta_handle *h, int which, int32_t partition, uint64_t *out);
/* src/metric.rs:132-157; KTA_ERR_DIV_BY_ZERO where the reference panics */
int kta_avg(const kta_handle *h, int which, int32_t partition, uint64_t *out);
/* src/metric.rs:159-167 (f32 arithmetic, same operation order) */
int kta_dirty_ratio(const kta_handle *h, int32_t partition, float *out);
/* src/metric.rs:177-195 */
int kta_global(const kta_handle *h, int which, uint64_t *out);
/* earliest_message / latest_message, src/metric.rs:169-175, as UTC seconds (+ ns of the
 * construction clock when no record was earlier than it) */
int kta_timestamps(const kta_handle *h, int64_t *earliest_s, int32_t *earliest_ns, int64_t *latest_s);
/* LogCompactionInMemoryMetrics::sum_all_alive, src/metric.rs:282-284 (exact) */
int kta_alive_keys(const kta_handle *h, uint64_t *out);
/* records whose partition was outside [0, num_partitions): they are left out of EVERY metric (kta_finalize returns
 * KTA_ERR_PARTITION to say so; the getters stay valid and describe the in-range records) */
int kta_bad_partition_records(const kta_handle *h, uint64_t *out);

/* ---- EXTENSIONS: not in the reference (SURVEY.md D2, D3) ---- */
/* per-partition log2 size histogram: which = 0 key sizes, 1 value sizes */
int kta_hist(const kta_handle *h, int which, int32_t partition, uint64_t out[KTA_HIST_BUCKETS]);
/* HyperLogLog estimate of distinct alive key hashes.  With count_alive_keys the sketch is built
 * from the resolved alive set; otherwise it is the in-stream sketch of every (key, value) insert,
 * which equals the alive count only on tombstone-free topics. */
int kta_alive_keys_hll(const kta_handle *h, double *out);
/* raw registers (one byte each, 1 << hll_precision of them) */
int kta_hll_registers(const kta_handle *h, uint8_t *out, size_t cap);
/* the hash itself, computed on the device for n packed keys given in HOST memory (test hook for
 * src/fnv32.rs:92-101 known-answer vectors).  key_len[i] < 0 yields 0. */
int kta_fnv32_host(kta_handle *h, int64_t n, const int32_t *key_len, const uint8_t *key_bytes,
                   int64_t key_bytes_len, uint32_t *out);

/* Timeline: per partition, the records, tombstones and bytes written in each time bucket (when a partition's data was
 * written: how much of it is older than retention.ms, which tombstones are older than delete.retention.ms, whether a
 * partition has stopped receiving data, whether the topic was filled in bursts).  Off by default.
 *   Records counted: exactly the records the counters count.  A record whose partition lies outside [0, P), a record of
 *   a foreign partition on a sharded handle, and log records never delivered (aborted, CRC-failed, outside a window,
 *   dropped below the log start) are left out; stamps-only re-runs of the alive-key table are not counted again.
 *   Second of a record: t = (ts_ms == -1 ? 0 : ts_ms) / 1000, truncating toward zero, as earliest / latest
 *   (src/metric.rs:209-211).  A record without a timestamp lands at 1970-01-01; other negative ms are real times:
 *   -999 gives 0, -1000 gives -1, -1001 gives -1.
 *   Buckets: origin O (s), width W >= 1 (s), B buckets.  Index 0 counts t < O; index 1 + (t - O) / W counts
 *   O <= t < O + B*W; index B + 1 counts everything later.
 *   Counters per (partition, index): KTA_TIMELINE_RECORDS (sums to KTA_TOTAL over the B + 2 indices),
 *   KTA_TIMELINE_TOMBSTONES (value_len < 0; sums to KTA_TOMBSTONES), KTA_TIMELINE_BYTES (max(key_len, 0) +
 *   max(value_len, 0); sums to KTA_KEY_SIZE_SUM + KTA_VALUE_SIZE_SUM).
 * kta_set_timeline: buckets == 0 turns the timeline off.  KTA_ERR_INVALID when a record has been pushed or scanned since
 * create or the last kta_reset (records still in the landing ring included), when width_s < 1, buckets lies outside
 * [0, 65536], origin_s + buckets * width_s overflows int64, or num_partitions * (buckets + 2) > 2^24.  The arrays take
 * 3 * num_partitions * (buckets + 2) u64 of device memory; kta_reset zeroes them and keeps the configuration.  Every
 * counted scan is followed by one more kernel (kta_stats counts it) that reads the four header columns again.
 * kta_timeline: valid after kta_finalize; copies min(cap, buckets + 2) words of one partition's row.
 * KTA_ERR_NOT_ENABLED when the timeline is off, KTA_ERR_NOT_FINALIZED before kta_finalize; a partition outside [0, P)
 * reads as zeros (like kta_counter).  A sharded handle keeps all P rows; foreign rows stay zero. */
enum { KTA_TIMELINE_RECORDS = 0, KTA_TIMELINE_TOMBSTONES = 1, KTA_TIMELINE_BYTES = 2 };
int kta_set_timeline(kta_handle *h, int64_t origin_s, int64_t width_s, int32_t buckets);
int kta_timeline(const kta_handle *h, int which, int32_t partition, uint64_t *out, int64_t cap);

/* Partitioner check: per partition, how many keyed records sit where the common producers' partitioners would put them,
 * so that a key written to two partitions (the partition count was raised, or producers with different partitioners
 * wrote the topic) shows up: log compaction works per partition, and such a key keeps a live value in each.  Off by
 * default.
 *   Records checked: exactly the records the counters count (as the timeline's), and only those with a non-null key
 *   (key_len >= 0; an empty key is hashed like any other).  Stamps-only re-runs of the alive-key table are not counted
 *   again.
 *   For a record with key bytes k in partition p and each j < C:
 *     murmur2 at N_j: (murmur2(k) & 0x7fffffff) % N_j == p, with Kafka's Utils.murmur2 (seed 0x9747b28c, m 0x5bd1e995,
 *       r 24, little-endian 4-byte words, tail bytes folded high to low before one multiply): the Java producer's
 *       partitioner for keyed records, and librdkafka's murmur2 / murmur2_random;
 *     CRC-32 at N_j: crc32(k) % N_j == p, unsigned, with zlib's CRC-32 (reflected 0xEDB88320, init and xorout
 *       0xFFFFFFFF): librdkafka's consistent / consistent_random (its default) for non-empty keys;
 *     neither: the record matched no (function, count) pair.
 *   Not claimed: librdkafka's *_random variants may send an EMPTY key to a random partition (it is counted as hashed
 *   here); fnv1a (librdkafka, Sarama) and custom partitioners are not modelled.
 * kta_set_partitioner_check: ncounts = C in [0, KTA_PARTITIONER_MAX_COUNTS]; 0 turns the check off.  Every count lies in
 * [1, 2^31 - 1] and the counts are distinct.  KTA_ERR_INVALID, with nothing changed, on any violation and when a record
 * has been pushed or scanned since create or the last kta_reset (records still in the landing ring included).  The
 * counters take (2C + 1) * num_partitions u64 of device memory; kta_reset zeroes them and keeps the configuration.  Every
 * counted scan is followed by one more kernel (kta_stats counts it) that reads partition, key_len and the key bytes.
 * With the check on, key bytes reach the device on every handle, a counters-only one included: a batch with keyed
 * records must then carry key_bytes (KTA_ERR_INVALID otherwise), and kta_push copies each key.
 * kta_partitioner_check: valid after kta_finalize; copies min(cap, 2C + 1) words of one partition: murmur2 matches for
 * counts[0..C), CRC-32 matches for counts[0..C), neither.  KTA_ERR_NOT_ENABLED when the check is off,
 * KTA_ERR_NOT_FINALIZED before kta_finalize; a partition outside [0, P) reads as zeros.  A sharded handle keeps all P
 * rows; foreign rows stay zero.
 * kta_partitioner_hash_host: the check's own device hash functions over n packed keys given in HOST memory (test hook,
 * like kta_fnv32_host); key_len[i] < 0 yields 0 for both. */
#define KTA_PARTITIONER_MAX_COUNTS 8
int kta_set_partitioner_check(kta_handle *h, const int32_t *counts, int32_t ncounts);
int kta_partitioner_check(const kta_handle *h, int32_t partition, uint64_t *out, int64_t cap);
int kta_partitioner_hash_host(kta_handle *h, int64_t n, const int32_t *key_len, const uint8_t *key_bytes,
                              int64_t key_bytes_len, uint32_t *murmur2, uint32_t *crc32);

/* Hot keys: an exact, topic-wide table of per-key counters, filled on the GPU, and the top_k keys with the most records
 * (which keys a compacted topic is made of: a high dirty ratio or a hot partition usually comes from a few keys rewritten
 * constantly).  Off by default.
 *   Records counted: exactly the records the counters count (as the timeline's), and only those with a non-null key
 *   (key_len >= 0; an empty key is a key).  Stamps-only re-runs of the alive-key table are not counted again.
 *   Key identity: a key is its 64-bit id, (uint64_t)crc32(key) << 32 | murmur2(key) with the partitioner check's two
 *   hashes (zlib's CRC-32 and Kafka's murmur2, unmasked).  Two distinct keys with equal ids are merged into one entry; with
 *   D distinct keys about D^2 / 2^65 pairs collide (3e-6 expected pairs at 1e7 keys).  The prefix and key_len of a merged
 *   entry then come from whichever key claimed its slot.
 *   Per key: records; tombstones (value_len < 0); bytes, the sum of key_len + max(value_len, 0); latest_s, the largest
 *   (ts_ms == -1 ? 0 : ts_ms) / 1000 over its records (truncating, the timeline's second); the smallest and largest
 *   partition it was written to; key_len and the first min(key_len, 32) bytes of the key, zeros after.
 * kta_set_hot_keys: top_k = 0 turns the table off; otherwise top_k lies in [1, KTA_HOT_KEYS_MAX].  table_slots = 0 means
 * 2^20; otherwise it is a power of two in [16, 2^31].  KTA_ERR_INVALID, with nothing changed, on any violation and when a
 * record has been pushed or scanned since create or the last kta_reset (records still in the landing ring included).  The
 * table takes 96 bytes per slot (plus one) of device memory and is grown by rehash, doubling, so that it stays at most half
 * full: before a launch the library keeps an upper bound on the occupancy; when a batch could take it past half the slots it
 * reads the occupancy back (one copy to the host and a stream synchronisation), grows the table while it is more than a
 * quarter full, and scans the batch in slices that cannot overfill it, reading the occupancy back between slices.  With the
 * table on, a device batch may therefore wait for the device.  kta_reset zeroes the table and keeps its configuration and
 * its allocation.  Every counted scan is followed by at least one more kernel (kta_stats counts them) that reads partition,
 * key_len, value_len, ts_ms and the key bytes.  With the table on, key bytes reach the device on every handle: a batch with
 * keyed records must carry key_bytes (KTA_ERR_INVALID otherwise), and kta_push copies each key.
 * Out of memory: when the table cannot grow (cudaMalloc fails, or the kta_hot_keys_limit_slots cap), the call that scanned
 * returns KTA_ERR_NOMEM and kta_last_error names the hot-key table.  Every other metric has counted the batch; the table
 * stops counting, and kta_hot_keys, kta_hot_key_stats and the export return KTA_ERR_NOMEM until kta_reset.  The status is
 * returned once, by the call whose scan hit it; a kta_push that returns it HAS taken its record (do not push it again).
 * kta_finalize returns it only when it has no other status to return (KTA_ERR_INVALID for sequence numbers outside the
 * window, KTA_ERR_PARTITION); the getters return it regardless.
 * kta_hot_keys: valid after kta_finalize; copies min(cap, top_k, distinct) entries ordered by records descending, then id
 * ascending; *count (may be NULL) = min(top_k, distinct).  KTA_ERR_NOT_ENABLED when the table is off, KTA_ERR_NOT_FINALIZED
 * before kta_finalize.
 * kta_hot_key_stats: valid after kta_finalize (any pointer may be NULL): the distinct keys (the table's occupancy), the keyed
 * records (the sum of the entries' records, equal to the sum over partitions of KTA_KEY_NON_NULL), the slots, how often the
 * table grew, and how many pass launches covered only part of a batch (slices) since create.
 * Multi-GPU merge: the table does not travel in the merge buffer (kta_merge_words is unchanged).  kta_hot_keys_export_count
 * gives the number of entries; kta_hot_keys_export_device writes every entry, in no particular order, to a device buffer
 * of cap entries (KTA_ERR_INVALID if cap is smaller; *count gets the number either way).  kta_hot_keys_import_device adds
 * count entries from device memory into the table: records, tombstones and bytes are summed, the partition range and
 * latest_s are folded, the prefix and key_len come from the entry that claims the slot.  The table grows first, so an
 * import never runs out of room.  The whole list is refused (KTA_ERR_INVALID, nothing applied) when an entry has
 * records == 0, tombstones > records, key_len < 0, reserved != 0, or a partition outside [0, num_partitions) or
 * min_partition > max_partition.  On a sharded handle the table holds the handle's own partitions' records; exporting every
 * rank's entries and importing the others' on each rank makes it topic-wide.
 * kta_hot_keys_limit_slots: test hook; the table may not grow beyond max_slots slots (0 = no cap). */
#define KTA_HOT_KEYS_MAX 65536
#define KTA_HOT_KEY_PREFIX 32
typedef struct kta_hot_key {
    uint64_t id;                 /* (uint64_t)crc32(key) << 32 | murmur2(key) */
    uint64_t records;            /* delivered records with this key (key_len >= 0) */
    uint64_t tombstones;         /* of which value_len < 0 */
    uint64_t bytes;              /* sum of key_len + max(value_len, 0) */
    int64_t latest_s;            /* max over its records of (ts_ms == -1 ? 0 : ts_ms) / 1000, truncating */
    int32_t min_partition, max_partition;
    int32_t key_len;
    uint32_t reserved;           /* 0; keeps the struct at 88 bytes with no implicit padding */
    uint8_t key_prefix[KTA_HOT_KEY_PREFIX];   /* first min(key_len, 32) bytes, zeros after */
} kta_hot_key;                   /* 88 bytes */
int kta_set_hot_keys(kta_handle *h, int32_t top_k, int64_t table_slots);
int kta_hot_keys(const kta_handle *h, kta_hot_key *out, int64_t cap, int64_t *count);
int kta_hot_key_stats(const kta_handle *h, uint64_t *distinct_keys, uint64_t *keyed_records, uint64_t *slots, uint64_t *grows,
                      uint64_t *slices);
int kta_hot_keys_export_count(kta_handle *h, int64_t *count);
int kta_hot_keys_export_device(kta_handle *h, kta_hot_key *dev_out, int64_t cap, int64_t *count);
int kta_hot_keys_import_device(kta_handle *h, const kta_hot_key *dev_in, int64_t count);
int kta_hot_keys_limit_slots(kta_handle *h, int64_t max_slots);

/* ---- multi-GPU merge (one process per GPU; the collective itself is the caller's: NCCL via
 * torch.distributed, or ncclAllReduce directly) ----
 * The mergeable state is exported as ONE array of u64 laid out so that a single SUM all-reduce
 * merges everything: sums as they are; min/max scalars and HLL registers in per-rank slots
 * (zero elsewhere) that the import folds with min/max.  words = kta_merge_words(h, world).
 * With the timeline on, its 3 * P * (B + 2) words follow, summed as they are: every rank must use the same
 * timeline configuration (origin, width, buckets).  With the partitioner check on, its (2C + 1) * P words follow at
 * the end (after the timeline's), summed as they are: every rank must check the same counts. */
int64_t kta_merge_words(const kta_handle *h, int32_t world);
int kta_merge_export_device(kta_handle *h, int32_t rank, int32_t world, uint64_t *dev_buf);
int kta_merge_import_device(kta_handle *h, int32_t world, const uint64_t *dev_buf);
/* exact alive-key exchange: compact (hash, stamp) entries of the local table, to be all-gathered
 * and re-applied on every rank (last-writer-wins by global seq is associative/commutative). */
int kta_alive_export_count(kta_handle *h, int64_t *count);
int kta_alive_export_device(kta_handle *h, uint32_t *dev_hash, uint64_t *dev_stamp, int64_t cap,
                            int64_t *count);
int kta_alive_import_device(kta_handle *h, const uint32_t *dev_hash, const uint64_t *dev_stamp,
                            int64_t count);

/* ---- Kafka log segments (SURVEY.md §8 f2): the step before the handlers ----
 * A segment is the concatenation of RecordBatch v2 (magic 2) batches of ONE partition — what a broker stores in
 * <topic>-<partition>/NNN.log and returns in a fetch response.  The library decodes it on the GPU into the SoA
 * columns above (what librdkafka's parser + BorrowedMessage accessors do per message, src/kafka.rs:93,
 * src/metric.rs:208-209,218,233) and scans it.  Control batches are skipped, LogAppendTime batches use
 * maxTimestamp, a record's timestamp is baseTimestamp + timestampDelta (only a result of -1 is "not available"),
 * CRCs are verified only when check.crcs is switched on (kta_log_set_check_crcs; off by default, like librdkafka's
 * check.crcs=false).  gzip, LZ4 (frame format), Snappy (raw or
 * xerial-framed) and zstd batches are decompressed on the GPU; the checksums inside a compressed section (gzip's
 * CRC32, zstd's Content_Checksum) are skipped, not verified, like the batch CRC.  zstd frames with a Dictionary_ID and
 * the unassigned codecs 5-7 are rejected (KTA_ERR_INVALID).
 * Isolation (cfg.isolation_level).  KTA_READ_UNCOMMITTED delivers every data batch.  KTA_READ_COMMITTED (librdkafka's
 * default) leaves out the records of aborted transactions.  A transactional batch (attributes bit 4) of partition p and
 * producerId q is aborted when the first control batch of the same (p, q) that follows it in the same call is an ABORT
 * marker, or when its baseOffset lies in an aborted range of (p, q) registered with kta_log_add_txn_index_host.  Matching
 * ignores producerEpoch.  Non-transactional batches, committed transactions and producerId -1 are delivered as with
 * read_uncommitted; control batches never are.  Aborted batches are not decompressed or decoded, so damage inside them is
 * no error.  A control batch whose marker cannot be read (compressed, no record, key length != 4, version != 0) and a call
 * in which the batches of one (p, q) do not have increasing baseOffsets are KTA_ERR_INVALID.
 * Differences from a librdkafka consumer: under read_committed, a transactional batch that has no following marker in its
 * call and no registered range (a transaction still open at the end of what was read, or closed in a later call) is
 * delivered and counted as undecided (kta_log_txn_stats); a consumer would stop at the last stable offset and wait.
 * Legacy magic 0/1 message sets are reported as malformed.
 * records_out of every log entry point counts the records delivered. */
/* raw bytes already in device memory; batch_off[nbatches] = byte offset of every batch header (device memory) */
int kta_scan_log_segment_device(kta_handle *h, int32_t partition, const uint8_t *dev_bytes, int64_t len,
                                const uint64_t *dev_batch_off, int64_t nbatches, int64_t *records_out);
/* the same for batches of SEVERAL partitions lying in one device buffer (e.g. a whole fetch response, or many segments
 * staged back to back): dev_batch_partition[nbatches] names each batch's partition.  One decode and one scan. */
int kta_scan_log_batches_device(kta_handle *h, const uint8_t *dev_bytes, int64_t len, const uint64_t *dev_batch_off,
                                const int32_t *dev_batch_partition, int64_t nbatches, int64_t *records_out);
/* raw bytes in host memory (e.g. an mmap of a .log file); returns when `bytes` may be reused */
int kta_push_log_segment_host(kta_handle *h, int32_t partition, const uint8_t *bytes, int64_t len, int64_t *records_out);
/* several segments (any partitions) in one go: one staging copy per segment, ONE decode and ONE scan for all of them */
int kta_push_log_segments_host(kta_handle *h, int32_t nsegs, const int32_t *partitions, const uint8_t *const *bytes,
                               const int64_t *lens, int64_t *records_out);
/* read_committed only: parse one .txnindex image of `partition` (34-byte big-endian entries version i16 = 0 |
 * producerId i64 | firstOffset i64 | lastOffset i64 | lastStableOffset i64) and register its aborted ranges
 * [firstOffset, lastOffset] for every later log call on this handle (until kta_reset).  KTA_ERR_INVALID on a
 * read_uncommitted handle and on a malformed image (length not a multiple of 34, version != 0, firstOffset > lastOffset);
 * nothing of a malformed image is registered.  An empty image is fine (the broker writes the file lazily). */
int kta_log_add_txn_index_host(kta_handle *h, int32_t partition, const uint8_t *bytes, int64_t len);
/* read_committed only (KTA_ERR_NOT_ENABLED otherwise): totals over the successful log calls since create / reset of
 * the batches and records left out as aborted, and the records of undecided transactional batches that were delivered
 * (any pointer may be NULL) */
int kta_log_txn_stats(kta_handle *h, uint64_t *aborted_batches, uint64_t *aborted_records, uint64_t *undecided_records);

/* check.crcs: verify every record batch's CRC-32C and skip the batches that fail it.
 * The checksum is CRC-32C (Castagnoli, reflected polynomial 0x82F63B78, init and xorout 0xFFFFFFFF) over the batch from
 * `attributes` (byte 21) to its end (byte 12 + batchLength), computed over the bytes as stored (the compressed ones for a
 * compressed batch), compared with the big-endian u32 at bytes 17-20.
 * Off (the default, as librdkafka's check.crcs=false): nothing changes.  On: the check runs on the GPU before anything
 * reads a CRC-covered field.  A batch that fails it is not decompressed, decoded, or classified as transactional data or
 * as a marker: it delivers no records, takes no sequence numbers and raises no error, so an unknown codec, an implausible
 * recordsCount, a section that does not decompress, a malformed record, an unreadable marker or a producer's baseOffset
 * order inside it no longer refuse the call.  It is counted as a CRC failure only, never as aborted; under
 * read_committed a failed marker is not seen (its transaction is decided by the registered ranges, or is undecided).
 * The fields outside the CRC frame the batch and still refuse the call as before: the batch must fit the buffer,
 * batchLength >= 49 and magic == 2.  A batch that passes goes through every other check unchanged (a valid CRC over a
 * malformed record is a producer bug, not damage: KTA_ERR_INVALID).  librdkafka reports such a batch as a consumer error
 * (RD_KAFKA_RESP_ERR__BAD_MSG, "failed CRC32C check") and goes on with the next one; kta_log_crc_failures lists them. */
#define KTA_LOG_CRC_KEEP 4096   /* failures kept per handle (kta_log_crc_failures) */
typedef struct kta_log_crc_failure {
    int32_t partition;
    uint32_t batch_bytes;        /* 12 + batchLength */
    int64_t base_offset;
    uint32_t stored_crc;         /* bytes 17-20 of the batch */
    uint32_t computed_crc;
} kta_log_crc_failure;           /* 24 bytes */
/* enabled: 0 or 1 (anything else is KTA_ERR_INVALID); applies to every later log call; kta_reset keeps it */
int kta_log_set_check_crcs(kta_handle *h, int enabled);
/* totals over the successful log calls since create / reset: batches checked (while the switch was on), batches that
 * failed, and their bytes (12 + batchLength each).  Any pointer may be NULL; valid whether the switch is on or off. */
int kta_log_crc_stats(kta_handle *h, uint64_t *checked_batches, uint64_t *failed_batches, uint64_t *failed_bytes);
/* the first KTA_LOG_CRC_KEEP failures of successful calls since create / reset, in call order and, within a call, in
 * batch order: min(cap, kept) of them are copied to out; *count (may be NULL) = the number kept.  kta_reset clears them. */
int kta_log_crc_failures(kta_handle *h, kta_log_crc_failure *out, int64_t cap, int64_t *count);

/* Offsets: read only what a consumer would fetch, from a partition's log start offset S up to its high watermark H.
 * A broker keeps both in its data directory (log-start-offset-checkpoint, replication-offset-checkpoint); records below S
 * (DeleteRecords, purged repartition topics) and at or above H (appends not yet committed) stay in the .log files, and a
 * consumer that starts at S (auto.offset.reset=earliest) and reads up to H never sees them.
 * Unset (the default): nothing changes.  Set for partition p: with last = baseOffset + lastOffsetDelta (the stored field,
 * which can lie past the last record of a compacted batch), a batch is served only when S <= last < H: a fetch from S
 * starts at the first batch whose last offset is >= S, and a fetch bounded by H stops before the batch that holds H.  A
 * batch that is not served is skipped unread: it is not CRC-checked, decompressed, decoded, or classified as transactional
 * data or as a marker; it delivers no records, takes no sequence numbers and raises no error, so damage inside it does
 * not refuse the call.  Within a served batch with baseOffset < S (a cut batch) a record with baseOffset + offsetDelta < S
 * is dropped, as librdkafka's reader drops messages older than the fetch offset; offsets are read from the decompressed
 * records, so a compressed batch may be cut.  A served batch with baseOffset >= S keeps all its records, so a forged
 * negative offsetDelta cannot drop one: a batch's records depend only on its bytes and its partition's window.  On every
 * log a broker writes this equals librdkafka's rule, because stored offset deltas are never negative.  With check.crcs
 * only served batches are checked and counted; a served batch that fails is skipped and listed as before, cut or not.  Under read_committed a marker outside the window is not seen (its transaction is
 * decided by the registered ranges, or is undecided), and the producers' baseOffset order is checked over served batches
 * only.  The fields that frame a batch still refuse the call as before: it must fit the buffer, batchLength >= 49, magic 2.
 * Windows apply to the log entry points only; kta_push and the batch entry points ignore them.
 * log_start_offset, high_watermark: -1 = no bound on that side.  KTA_ERR_INVALID when the partition lies outside
 * [0, num_partitions), when a value is below -1, or when both are set and log_start_offset > high_watermark.  A later
 * call replaces the partition's window; it applies to every later log call; kta_reset clears every window. */
int kta_log_set_offsets(kta_handle *h, int32_t partition, int64_t log_start_offset, int64_t high_watermark);
/* totals over the successful log calls since create / reset: the batches that were not served, and the records left out
 * (the recordsCount of the data batches not served, plus the records dropped below the log start offset).  Either pointer
 * may be NULL. */
int kta_log_offset_stats(kta_handle *h, uint64_t *batches_not_served, uint64_t *records_left_out);

/* ---- introspection for benchmarks ---- */
/* kernels launched by this handle since create/reset, and device time of the scan kernels (ms,
 * CUDA events on the handle's stream; only collected when enabled) */
int kta_stats(const kta_handle *h, uint64_t *kernel_launches, uint64_t *records_scanned);
int kta_set_timing(kta_handle *h, int enabled);
int kta_scan_time_ms(kta_handle *h, double *total_ms, uint64_t *launches);
/* alive-key table: slots allocated, slots occupied (= distinct key hashes seen), how often it was grown and how many
 * batches had to be re-stamped because it was too small when they were scanned (any pointer may be NULL) */
int kta_alive_table_stats(kta_handle *h, uint64_t *slots, uint64_t *occupied, uint64_t *grows, uint64_t *reruns);
/* raw cudaStream_t of the handle (so a torch caller can order against it) */
void *kta_stream(kta_handle *h);
/* adopt a caller-owned cudaStream_t (e.g. torch's current stream) for all further work of this handle */
int kta_set_stream(kta_handle *h, void *stream);

/* ---- synthetic in-memory topic (configs[0..4] of BASELINE.json; SURVEY.md §8 d) ----
 * Counter-based: every field of record i is a pure function of (seed, i); the same code runs on
 * host and device.  Partition p of record i: runs of run_len records, runs dealt round-robin with a
 * per-cycle pseudo-random rotation, so per-partition offsets are closed-form and a rank that owns
 * partitions {p : p % world == rank} can enumerate exactly its records. */
/* key_mode flags.  Both are integer-only so that host and device generate identical topics.
 * KEYS_LOGUNIFORM: key ids are drawn log-uniformly (a staircase approximation of Zipf s = 1: id k of a partition
 *   is about as likely as 1/(k+1)) instead of uniformly — a few hot keys, a long tail of cold ones.
 * VALUES_GEOMETRIC: the uniform value length is multiplied by 2^g, P(g = k) = 2^-(k+1), g <= 6 — a geometric tail. */
#define KTA_SYNTH_KEYS_LOGUNIFORM 0x100
#define KTA_SYNTH_VALUES_GEOMETRIC 0x200
/* The largest value_mean a spec may ask for: the largest uniform value length, floor(mean/2) + mean, is then exactly
 * INT32_MAX.  Every entry point refuses a larger mean as an invalid spec (kta_synth_shard_records returns -1). */
#define KTA_SYNTH_MAX_VALUE_MEAN 1431655765

typedef struct kta_synth_spec {
    uint64_t seed;               /* default 0x4B544131 ("KTA1") */
    int64_t n_total;             /* records in the whole topic; multiple of num_partitions*run_len */
    int32_t num_partitions;
    int32_t run_len;             /* >= 1 */
    uint64_t distinct_keys;      /* D; rounded down to a multiple of num_partitions, >= P */
    int32_t key_mode;            /* low byte: 0 = 16-byte binary (id, id*phi64) LE; 1 = ASCII "key-<id>";
                                    2 = variable-length binary, 0..40 bytes.  Optional flags (stress cases):
                                    KTA_SYNTH_KEYS_LOGUNIFORM, KTA_SYNTH_VALUES_GEOMETRIC */
    int32_t value_mean;          /* value_len uniform in [mean/2, 3*mean/2]; at most KTA_SYNTH_MAX_VALUE_MEAN */
    int32_t null_key_per_10k;
    int32_t tombstone_per_10k;
    int32_t ts_missing_per_10k;
    int32_t empty_value_per_10k;
} kta_synth_spec;

/* number of records of the topic owned by `rank` of `world` (partitions p % world == rank) */
int64_t kta_synth_shard_records(const kta_synth_spec *s, int32_t rank, int32_t world);
/* Fill host SoA columns for local records [start, start+count) of the shard.  Any output pointer
 * may be NULL.  key_bytes_cap bounds key_bytes; *key_bytes_len receives the bytes written. */
int kta_synth_fill_host(const kta_synth_spec *s, int32_t rank, int32_t world, int64_t start,
                        int64_t count, int32_t *partition, int64_t *offset, int64_t *ts_ms,
                        int32_t *key_len, int32_t *value_len, uint64_t *seq, uint8_t *key_bytes,
                        int64_t key_bytes_cap, int64_t *key_bytes_len);
/* Same on the device (pointers are device memory; key_tile_base must hold
 * ceil(count/KTA_KEY_TILE)+1 words).  Synchronous.  The key bytes are placed by the tile bases, so a call
 * that asks for key_bytes or key_bytes_len without key_tile_base is refused with KTA_ERR_INVALID before
 * anything is written.  key_bytes_cap smaller than the slice's key bytes: KTA_ERR_NOMEM, no key byte written. */
int kta_synth_fill_device(const kta_synth_spec *s, int32_t device, int32_t rank, int32_t world,
                          int64_t start, int64_t count, int32_t *partition, int64_t *offset,
                          int64_t *ts_ms, int32_t *key_len, int32_t *value_len, uint64_t *seq,
                          uint8_t *key_bytes, int64_t key_bytes_cap, uint64_t *key_tile_base,
                          int64_t *key_bytes_len);

/* The same topic as a broker stores it: records [start, start+count) (offset order) of one partition as an
 * uncompressed RecordBatch v2 log segment, `batch_records` records per batch (feeds kta_push_log_segment_host). */
int kta_synth_encode_segment_host(const kta_synth_spec *s, int32_t partition, int64_t start, int64_t count,
                                  int32_t batch_records, uint8_t *out, int64_t cap, int64_t *len);

#ifdef __cplusplus
}
#endif
#endif
