// kafka-topic-analyzer (H100 build) — the reference's CLI surface (src/main.rs:32-67) over libkta_gpu.so.
//
//   -t/--topic TOPIC  -b/--bootstrap-server HOSTS  [--librdkafka k=v,...]  [-c/--count-alive-keys]
//   --synthetic n=...,partitions=...,value_mean=...,run_len=...,distinct_keys=...,key_mode=...,seed=...,
//               tombstone_per_10k=...,null_key_per_10k=...,zipf_keys=1,geometric_values=1
//                                                                (the in-memory topic of BASELINE.json configs)
//   --log-dir DIR              read Kafka log segments from DIR/<topic>-<partition>/*.log (a broker's data directory)
//                              and decode them on the GPU (RecordBatch v2, magic 2; uncompressed, gzip, LZ4, Snappy or
//                              zstd batches; compressed sections' checksums are not verified).  Isolation follows
//                              --librdkafka isolation.level=read_committed|read_uncommitted; the default here is
//                              read_uncommitted (every record counted), the reference's librdkafka default is read_committed.
//                              Under read_committed the *.txnindex files of every partition directory are read first and the
//                              records of aborted transactions are left out (include/kta.h).  Differences from a librdkafka
//                              consumer: records of transactions still open at the end of the files are counted (with a
//                              warning) instead of waiting at the last stable offset, and legacy magic 0/1 message sets are
//                              reported as malformed.
//                              --librdkafka check.crcs=true (default false, as librdkafka's) verifies every batch's
//                              CRC-32C on the GPU: a batch that fails it is skipped, and reported on stderr in librdkafka's
//                              words ("... failed CRC32C check ..."); the report covers the rest and the exit status stays
//                              0, as the reference logs a failed poll and goes on (src/kafka.rs:95-97).
//                              DIR/log-start-offset-checkpoint and DIR/replication-offset-checkpoint, when present, give each
//                              partition they list the offsets a consumer reads: from the log start offset (raised to the
//                              first segment's base offset) up to the high watermark (clamped into [start, log end offset]),
//                              as the reference reads from the earliest offset up to the high watermark (src/kafka.rs:28-31,
//                              60-72).  Records outside are left out, and the two offsets are the report's < OS and > OS.
//   --feed push|batch|device   how records reach the handlers: kta_push per record (the reference's call shape),
//                              kta_push_batch_host, or generated and scanned in HBM
//   --timeline W[,ORIGIN,BUCKETS]  extension: after the report, one row per non-empty W-second bucket (start time in UTC,
//                              records, tombstones, bytes, summed over the report's partitions), plus "before" and "after"
//                              rows when records fall outside.  Without ORIGIN and BUCKETS the range is what can be seen
//                              before the first record: under --log-dir every batch's baseTimestamp and maxTimestamp (a
//                              header-only walk of the segments), under --synthetic the timestamps of the first and last
//                              record; the origin is rounded down to a multiple of W.  More than 10 000 buckets are refused.
//   --partitioner-check N[,N...]  extension: after the report (and the timeline), one row per partition: its keyed records,
//                              how many of them sit where Kafka's murmur2 partitioner would put them at each N, where
//                              librdkafka's CRC-32 partitioner would, and where neither would; then a total row.  At most 8
//                              distinct counts, each in [1, 2^31 - 1].
//   --hot-keys K               extension: after the report (and the partitioner check), the number of distinct keys (by
//                              their 64-bit id) and the K keys with the most records, ranked: records, tombstones, bytes,
//                              the partition or partition range, the latest write (UTC) and the key (as text when its
//                              first 32 bytes are printable, else as hex; "…" when it is longer).  K in [1, 65536].
//
// There is no librdkafka and no broker in this build (SURVEY.md D9): without --synthetic the program explains
// that and exits, like the reference does when it cannot fetch metadata.  Everything numeric comes from the
// GPU library; this file only feeds records and prints.
#include <cuda_runtime_api.h>

#include <dirent.h>
#include <sys/stat.h>

#include <algorithm>
#include <cerrno>
#include <chrono>
#include <fstream>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <map>
#include <string>
#include <vector>

#include "../../../include/kta.h"
#include "kta_report.hpp"

static void die(const char *what) {
    fprintf(stderr, "error: %s: %s\n", what, kta_last_error());
    exit(1);
}
#define KTA(call) do { if ((call) != KTA_OK) die(#call); } while (0)

// kta_finalize reports records whose partition lies outside the topic's metadata with KTA_ERR_PARTITION; the state is
// valid (those records were left out of every metric), so the report is still printed — with a warning, like the
// reference's warn!() for a failed poll (src/kafka.rs:95-97).
static void finalize_or_warn(kta_handle *h) {
    const int rc = kta_finalize(h);
    if (rc == KTA_ERR_PARTITION) fprintf(stderr, "warning: %s\n", kta_last_error());
    else if (rc != KTA_OK) die("kta_finalize");
}


// ---- --log-dir: a broker's data directory instead of a live cluster ------------------------------------------------
static bool read_file(const std::string &path, std::vector<uint8_t> &out) {
    std::ifstream f(path, std::ios::binary | std::ios::ate);
    if (!f) return false;
    const std::streamsize n = f.tellg();
    f.seekg(0);
    out.resize((size_t)n);
    return n == 0 || (bool)f.read(reinterpret_cast<char *>(out.data()), n);
}

// --timeline: the bucket width and, once known, the range (kta_set_timeline)
struct TimelineOpt {
    bool on = false, ranged = false;   // ranged: ORIGIN and BUCKETS were given (or have been derived)
    int64_t width = 0, origin = 0, buckets = 0;
};
static constexpr int64_t TIMELINE_MAX_BUCKETS = 10000;

static bool parse_i64(const std::string &t, int64_t &v) {
    if (t.empty() || t.size() > 20 || t.find_first_not_of("0123456789", t[0] == '-' ? 1 : 0) != std::string::npos || t == "-") return false;
    errno = 0;
    v = strtoll(t.c_str(), nullptr, 10);
    return errno == 0;
}

// "W" or "W,ORIGIN,BUCKETS"; false (with a message) when it does not parse
static bool parse_timeline(const std::string &arg, TimelineOpt &t) {
    std::vector<std::string> f;
    for (size_t p = 0;;) {
        const size_t e = arg.find(',', p);
        f.push_back(arg.substr(p, e == std::string::npos ? std::string::npos : e - p));
        if (e == std::string::npos) break;
        p = e + 1;
    }
    if ((f.size() != 1 && f.size() != 3) || !parse_i64(f[0], t.width) || t.width < 1) {
        fprintf(stderr, "error: --timeline takes W[,ORIGIN,BUCKETS]: a bucket width of at least 1 second, optionally the first "
                "bucket's start (UTC seconds) and the number of buckets, not '%s'\n", arg.c_str());
        return false;
    }
    t.on = true;
    if (f.size() == 3) {
        if (!parse_i64(f[1], t.origin) || !parse_i64(f[2], t.buckets) || t.buckets < 1) {
            fprintf(stderr, "error: --timeline: ORIGIN must be an integer and BUCKETS at least 1, not '%s'\n", arg.c_str());
            return false;
        }
        if (t.buckets > TIMELINE_MAX_BUCKETS) {
            fprintf(stderr, "error: --timeline: %lld buckets is more than %lld: use a wider W or fewer buckets\n",
                    (long long)t.buckets, (long long)TIMELINE_MAX_BUCKETS);
            return false;
        }
        t.ranged = true;
    }
    return true;
}

// the second a record's timestamp counts in (include/kta.h): -1 = not available = 0, truncating toward zero
static int64_t ts_second(int64_t ts_ms) { return (ts_ms == -1 ? 0 : ts_ms) / 1000; }

// the range from the earliest and latest second seen: origin rounded down to a multiple of W, enough buckets to reach the
// latest second; false (with a message) beyond TIMELINE_MAX_BUCKETS
static bool timeline_range(TimelineOpt &t, int64_t lo_s, int64_t hi_s) {
    if (t.ranged) return true;
    if (lo_s > hi_s) lo_s = hi_s = 0;   // nothing seen
    const int64_t W = t.width;
    t.origin = lo_s / W * W - ((lo_s % W) < 0 ? W : 0);   // floor
    const __int128 n = ((__int128)hi_s - t.origin) / W + 1;
    if (n > TIMELINE_MAX_BUCKETS) {
        fprintf(stderr, "error: --timeline: the records span %s to %s, %lld buckets of %lld s, more than %lld: use a wider W\n",
                kta_report::format_utc(lo_s, 0).c_str(), kta_report::format_utc(hi_s, 0).c_str(), (long long)n, (long long)W,
                (long long)TIMELINE_MAX_BUCKETS);
        return false;
    }
    t.buckets = (int64_t)n;
    t.ranged = true;
    return true;
}

// one row per non-empty bucket, summed over the report's partitions, with "before" and "after" rows when nonzero
static void print_timeline(kta_handle *h, const std::vector<int> &partitions, const TimelineOpt &t) {
    const size_t row = (size_t)t.buckets + 2;
    std::vector<uint64_t> sum[3], one(row);
    for (int w = 0; w < 3; w++) {
        sum[w].assign(row, 0);
        for (int p : partitions) {
            KTA(kta_timeline(h, w, p, one.data(), (int64_t)row));
            for (size_t i = 0; i < row; i++) sum[w][i] += one[i];
        }
    }
    std::vector<kta_report::TimelineRow> rows;
    for (size_t i = 0; i < row; i++) {
        if (!sum[KTA_TIMELINE_RECORDS][i]) continue;
        kta_report::TimelineRow r{};
        r.index = (int64_t)i;
        r.start_s = t.origin + ((int64_t)i - 1) * t.width;
        r.records = sum[KTA_TIMELINE_RECORDS][i];
        r.tombstones = sum[KTA_TIMELINE_TOMBSTONES][i];
        r.bytes = sum[KTA_TIMELINE_BYTES][i];
        rows.push_back(r);
    }
    fputs(kta_report::render_timeline(t.origin, t.width, t.buckets, rows).c_str(), stdout);
}

// "N[,N...]": at most KTA_PARTITIONER_MAX_COUNTS distinct counts in [1, 2^31 - 1]; false (with a message) otherwise
static bool parse_partitioner_check(const std::string &arg, std::vector<int32_t> &counts) {
    counts.clear();
    for (size_t p = 0;;) {
        const size_t e = arg.find(',', p);
        const std::string f = arg.substr(p, e == std::string::npos ? std::string::npos : e - p);
        int64_t v = 0;
        if (!parse_i64(f, v) || v < 1 || v > INT32_MAX) {
            fprintf(stderr, "error: --partitioner-check takes N[,N...]: partition counts in [1, 2147483647], not '%s'\n", arg.c_str());
            return false;
        }
        if (std::find(counts.begin(), counts.end(), (int32_t)v) != counts.end()) {
            fprintf(stderr, "error: --partitioner-check: the count %lld is given twice\n", (long long)v);
            return false;
        }
        counts.push_back((int32_t)v);
        if (e == std::string::npos) break;
        p = e + 1;
    }
    if (counts.size() > KTA_PARTITIONER_MAX_COUNTS) {
        fprintf(stderr, "error: --partitioner-check: %zu counts is more than %d\n", counts.size(), KTA_PARTITIONER_MAX_COUNTS);
        return false;
    }
    return true;
}

// one row per report partition: keyed records (KTA_KEY_NON_NULL) and the check's 2C + 1 counters, then their total
static void print_partitioner_check(kta_handle *h, const std::vector<int> &partitions, const std::vector<int32_t> &counts) {
    const size_t nv = 2 * counts.size() + 1;
    std::vector<kta_report::PartitionerRow> rows;
    for (int p : partitions) {
        kta_report::PartitionerRow r{};
        r.partition = p;
        KTA(kta_counter(h, KTA_KEY_NON_NULL, p, &r.keyed));
        r.counts.resize(nv);
        KTA(kta_partitioner_check(h, p, r.counts.data(), (int64_t)nv));
        rows.push_back(r);
    }
    fputs(kta_report::render_partitioner_check(counts, rows).c_str(), stdout);
}

// --hot-keys K: 0 = off.  Read by both analysis paths (the table is switched on right after kta_create) and by print_report.
static int32_t g_hot_keys = 0;

static bool parse_hot_keys(const std::string &arg) {
    int64_t v = 0;
    if (!parse_i64(arg, v) || v < 1 || v > KTA_HOT_KEYS_MAX) {
        fprintf(stderr, "error: --hot-keys takes K: a number of keys in [1, %d], not '%s'\n", KTA_HOT_KEYS_MAX, arg.c_str());
        return false;
    }
    g_hot_keys = (int32_t)v;
    return true;
}

// the distinct keys, then the g_hot_keys keys with the most records
static void print_hot_keys(kta_handle *h) {
    std::vector<kta_hot_key> top((size_t)g_hot_keys);
    int64_t n = 0;
    uint64_t distinct = 0;
    KTA(kta_hot_keys(h, top.data(), g_hot_keys, &n));
    KTA(kta_hot_key_stats(h, &distinct, nullptr, nullptr, nullptr, nullptr));
    std::vector<kta_report::HotKeyRow> rows;
    for (int64_t i = 0; i < n; i++) {
        const kta_hot_key &k = top[(size_t)i];
        rows.push_back({k.records, k.tombstones, k.bytes, k.latest_s, k.min_partition, k.max_partition, k.key_len,
                        std::string((const char *)k.key_prefix, (size_t)std::min(k.key_len, KTA_HOT_KEY_PREFIX))});
    }
    fputs(kta_report::render_hot_keys(distinct, rows).c_str(), stdout);
}

static int print_report(kta_handle *h, const std::string &topic, const std::vector<int> &partitions, const std::vector<int64_t> &start_offsets,
                        const std::vector<int64_t> &end_offsets, bool alive, int hll, uint64_t duration_secs, const TimelineOpt &tl,
                        const std::vector<int32_t> &pcounts);

// check.crcs: every kept failure as librdkafka words the consumer error it raises (RD_KAFKA_RESP_ERR__BAD_MSG), logged as
// the reference logs a failed poll; the failures beyond those kept in one line
static void warn_crc_failures(kta_handle *h) {
    uint64_t failed = 0;
    KTA(kta_log_crc_stats(h, nullptr, &failed, nullptr));
    if (!failed) return;
    std::vector<kta_log_crc_failure> f(KTA_LOG_CRC_KEEP);
    int64_t kept = 0;
    KTA(kta_log_crc_failures(h, f.data(), (int64_t)f.size(), &kept));
    for (int64_t i = 0; i < kept; i++)
        fprintf(stderr, "warning: Kafka error: MessageSet at offset %lld (%u bytes) of partition %d failed CRC32C check (original 0x%08x != calculated 0x%08x)\n",
                (long long)f[(size_t)i].base_offset, f[(size_t)i].batch_bytes, f[(size_t)i].partition, f[(size_t)i].stored_crc, f[(size_t)i].computed_crc);
    if (failed > (uint64_t)kept)
        fprintf(stderr, "warning: %llu more record batch(es) failed CRC32C check and were skipped\n", (unsigned long long)(failed - (uint64_t)kept));
}

// A broker's offset checkpoint file (log-start-offset-checkpoint, replication-offset-checkpoint): a version line "0", a
// count line, then `count` lines "topic partition offset".  The entries of `topic` go to out[partition].  false (and a
// message naming the file) when it does not parse; true without entries when the file does not exist.
static bool read_checkpoint(const std::string &path, const std::string &topic, std::map<int, int64_t> &out) {
    std::ifstream f(path);
    if (!f) return true;
    auto bad = [&](const char *why) { fprintf(stderr, "error: %s: %s\n", path.c_str(), why); return false; };
    auto number = [](const std::string &t, int64_t &v) {
        if (t.empty() || t.size() > 19 || t.find_first_not_of("0123456789", t[0] == '-' ? 1 : 0) != std::string::npos || t == "-") return false;
        v = strtoll(t.c_str(), nullptr, 10);
        return true;
    };
    std::string line;
    int64_t version = -1, count = -1;
    if (!std::getline(f, line) || !number(line, version) || version != 0) return bad("not version 0");
    if (!std::getline(f, line) || !number(line, count) || count < 0) return bad("no entry count");
    for (int64_t i = 0; i < count; i++) {
        if (!std::getline(f, line)) return bad("fewer entries than its count");
        const size_t a = line.find(' '), b = a == std::string::npos ? a : line.find(' ', a + 1);
        int64_t part = -1, off = 0;
        if (b == std::string::npos || line.find(' ', b + 1) != std::string::npos || !number(line.substr(a + 1, b - a - 1), part) ||
            part < 0 || part > INT32_MAX || !number(line.substr(b + 1), off))
            return bad("an entry is not \"topic partition offset\"");
        if (line.compare(0, a, topic) == 0 && a == topic.size()) out[(int)part] = off;
    }
    while (std::getline(f, line))
        if (!line.empty()) return bad("more entries than its count");
    return true;
}

// --timeline under --log-dir: the earliest and latest second of every batch's baseTimestamp (bytes 27-34) and maxTimestamp
// (bytes 35-42), read from the batch headers alone
static bool log_dir_seconds(const std::map<int, std::vector<std::string>> &segs, int64_t &lo_s, int64_t &hi_s) {
    lo_s = INT64_MAX; hi_s = INT64_MIN;
    uint8_t hdr[43];
    for (const auto &kv : segs)
        for (const auto &path : kv.second) {
            std::ifstream f(path, std::ios::binary);
            if (!f) { fprintf(stderr, "cannot read %s\n", path.c_str()); return false; }
            f.seekg(0, std::ios::end);
            const int64_t size = (int64_t)f.tellg();
            for (int64_t pos = 0; pos + 61 <= size;) {
                f.seekg(pos);
                if (!f.read(reinterpret_cast<char *>(hdr), sizeof hdr)) break;
                int64_t bl = 0, base = 0, mx = 0;
                for (int i = 8; i < 12; i++) bl = (bl << 8) | hdr[i];
                bl = (int32_t)bl;
                for (int i = 27; i < 35; i++) base = (int64_t)(((uint64_t)base << 8) | hdr[i]);
                for (int i = 35; i < 43; i++) mx = (int64_t)(((uint64_t)mx << 8) | hdr[i]);
                if (bl < 49 || pos + 12 + bl > size) break;
                for (int64_t ts : {base, mx}) {
                    lo_s = std::min(lo_s, ts_second(ts));
                    hi_s = std::max(hi_s, ts_second(ts));
                }
                pos += 12 + bl;
            }
        }
    return true;
}

static int analyze_log_dir(const std::string &topic, const std::string &dir, bool alive, int hll, bool read_committed, bool check_crcs,
                           std::chrono::steady_clock::time_point start_time, TimelineOpt tl, const std::vector<int32_t> &pcounts) {
    // get_topic_offsets (src/kafka.rs:60-72) from the files: partitions = <topic>-<n> directories, low watermark =
    // first batch's baseOffset, high watermark = last batch's baseOffset + lastOffsetDelta + 1; for the partitions the
    // broker's checkpoint files list, its log start offset and high watermark instead (and only what lies between is read)
    std::map<int, int64_t> log_start, high_watermark;
    if (!read_checkpoint(dir + "/log-start-offset-checkpoint", topic, log_start) ||
        !read_checkpoint(dir + "/replication-offset-checkpoint", topic, high_watermark))
        return 1;
    std::map<int, std::vector<std::string>> segs, txn_indexes;
    DIR *d = opendir(dir.c_str());
    if (!d) { fprintf(stderr, "Error fetching metadata: cannot open %s\n", dir.c_str()); return 101; }
    while (dirent *e = readdir(d)) {
        const std::string name = e->d_name;
        if (name.size() <= topic.size() + 1 || name.compare(0, topic.size() + 1, topic + "-") != 0) continue;
        const std::string num = name.substr(topic.size() + 1);
        if (num.empty() || num.find_first_not_of("0123456789") != std::string::npos) continue;
        const int p = atoi(num.c_str());
        DIR *pd = opendir((dir + "/" + name).c_str());
        if (!pd) continue;
        std::vector<std::string> files;
        while (dirent *fe = readdir(pd)) {
            const std::string fn = fe->d_name;
            if (fn.size() > 4 && fn.substr(fn.size() - 4) == ".log") files.push_back(dir + "/" + name + "/" + fn);
            if (fn.size() > 9 && fn.substr(fn.size() - 9) == ".txnindex") txn_indexes[p].push_back(dir + "/" + name + "/" + fn);
        }
        closedir(pd);
        std::sort(files.begin(), files.end());
        segs[p] = files;
    }
    closedir(d);
    if (segs.empty()) { fprintf(stderr, "Topic not found!\n"); return 101; }  // src/kafka.rs:62
    const int P = segs.rbegin()->first + 1;
    std::vector<int64_t> start_offsets(P, 0), end_offsets(P, 0);
    kta_config cfg{};
    cfg.struct_size = sizeof cfg;
    cfg.device = -1;
    cfg.num_partitions = P;
    cfg.count_alive_keys = alive ? 1 : 0;
    cfg.hll_precision = hll;
    cfg.now_s = INT64_MIN;
    cfg.isolation_level = read_committed ? KTA_READ_COMMITTED : KTA_READ_UNCOMMITTED;
    if (tl.on && !tl.ranged) {
        int64_t lo = 0, hi = 0;
        if (!log_dir_seconds(segs, lo, hi)) return 1;
        if (!timeline_range(tl, lo, hi)) return 2;
    }
    kta_handle *h = nullptr;
    KTA(kta_create(&cfg, &h));
    if (check_crcs) KTA(kta_log_set_check_crcs(h, 1));
    if (tl.on) KTA(kta_set_timeline(h, tl.origin, tl.width, (int32_t)tl.buckets));
    if (!pcounts.empty()) KTA(kta_set_partitioner_check(h, pcounts.data(), (int32_t)pcounts.size()));
    if (g_hot_keys) KTA(kta_set_hot_keys(h, g_hot_keys, 0));
    // the window of every partition the checkpoints list: the log start offset raised to the first segment's base offset
    // (its 20-digit file name, as the broker loads a log), the high watermark no lower than that (it is clamped to the log
    // end offset once the files are read: no batch lies beyond it, so the window reads the same either way)
    std::map<int, int64_t> win_start;
    for (auto &kv : segs) {
        const int p = kv.first;
        if (!log_start.count(p) && !high_watermark.count(p)) continue;
        int64_t s = -1;
        if (log_start.count(p)) {
            s = std::max<int64_t>(log_start[p], 0);
            if (!kv.second.empty()) {
                const std::string &f = kv.second.front();
                const std::string base = f.substr(f.rfind('/') + 1, f.size() - 4 - (f.rfind('/') + 1));
                if (base.size() == 20 && base.find_first_not_of("0123456789") == std::string::npos)
                    s = std::max<int64_t>(s, strtoll(base.c_str(), nullptr, 10));
            }
        }
        const int64_t hw = high_watermark.count(p) ? std::max<int64_t>(std::max<int64_t>(high_watermark[p], 0), s) : -1;
        KTA(kta_log_set_offsets(h, p, s, hw));
        win_start[p] = s;
    }
    // read_committed: every partition's aborted transactions are known before any segment is decoded, so a transaction
    // whose marker lies in a later group of segments is decided exactly
    if (read_committed)
        for (auto &kv : txn_indexes)
            if (segs.count(kv.first))
                for (const auto &path : kv.second) {
                    std::vector<uint8_t> buf;
                    if (!read_file(path, buf)) { fprintf(stderr, "cannot read %s\n", path.c_str()); return 1; }
                    if (kta_log_add_txn_index_host(h, kv.first, buf.data(), (int64_t)buf.size()) != KTA_OK) {
                        fprintf(stderr, "error: %s: %s\n", path.c_str(), kta_last_error());
                        return 1;
                    }
                }
    printf("Subscribing to %s\n", topic.c_str());
    printf("Starting message consumption...\n");
    auto be64 = [](const uint8_t *p) { uint64_t v = 0; for (int i = 0; i < 8; i++) v = (v << 8) | p[i]; return (int64_t)v; };
    auto be32 = [](const uint8_t *p) { return (int32_t)(((uint32_t)p[0] << 24) | ((uint32_t)p[1] << 16) | ((uint32_t)p[2] << 8) | p[3]); };
    // segments are handed over in groups of up to 512 MiB: one staging copy each, one GPU decode + scan per group
    std::vector<std::vector<uint8_t>> bufs;
    std::vector<int32_t> parts;
    int64_t total = 0, pending = 0;
    auto flush = [&]() {
        if (bufs.empty()) return;
        std::vector<const uint8_t *> ptrs;
        std::vector<int64_t> lens;
        for (auto &b : bufs) { ptrs.push_back(b.data()); lens.push_back((int64_t)b.size()); }
        int64_t nrec = 0;
        KTA(kta_push_log_segments_host(h, (int32_t)bufs.size(), parts.data(), ptrs.data(), lens.data(), &nrec));
        total += nrec;
        bufs.clear(); parts.clear(); pending = 0;
    };
    for (auto &kv : segs) {
        bool first = true;
        for (const auto &path : kv.second) {
            std::vector<uint8_t> buf;
            if (!read_file(path, buf)) { fprintf(stderr, "cannot read %s\n", path.c_str()); return 1; }
            for (int64_t pos = 0; pos + 61 <= (int64_t)buf.size();) {
                const int64_t bl = be32(buf.data() + pos + 8);
                if (bl < 49 || pos + 12 + bl > (int64_t)buf.size()) break;
                if (first) { start_offsets[kv.first] = be64(buf.data() + pos); first = false; }
                end_offsets[kv.first] = be64(buf.data() + pos) + be32(buf.data() + pos + 23) + 1;
                pos += 12 + bl;
            }
            pending += (int64_t)buf.size();
            parts.push_back(kv.first);
            bufs.push_back(std::move(buf));
            if (pending >= ((int64_t)512 << 20)) flush();
        }
    }
    flush();
    for (auto &kv : win_start) {   // < OS and > OS of the partitions with a window
        const int p = kv.first;
        if (kv.second >= 0) start_offsets[p] = kv.second;
        if (high_watermark.count(p))   // clamped into [start, log end offset]
            end_offsets[p] = std::max(start_offsets[p], std::min(std::max<int64_t>(high_watermark[p], 0), end_offsets[p]));
    }
    if (check_crcs) warn_crc_failures(h);
    if (std::all_of(end_offsets.begin(), end_offsets.end(), [](int64_t v) { return v == 0; })) {
        fprintf(stderr, "Given topic has no content, no analysis possible. Exiting.\n");  // main.rs:98-101
        return 254;
    }
    finalize_or_warn(h);
    if (read_committed) {
        uint64_t undecided = 0;
        KTA(kta_log_txn_stats(h, nullptr, nullptr, &undecided));
        if (undecided)
            fprintf(stderr, "warning: %llu record(s) of transactions without a commit or abort marker in the files were counted "
                    "(a read_committed consumer would wait for them to be decided)\n", (unsigned long long)undecided);
    }
    const uint64_t secs = (uint64_t)std::chrono::duration_cast<std::chrono::seconds>(std::chrono::steady_clock::now() - start_time).count();
    // the report has one row per partition of the topic's metadata (main.rs:103-106): the <topic>-<n> directories found
    std::vector<int> present;
    for (auto &kv : segs) present.push_back(kv.first);
    const int rc = print_report(h, topic, present, start_offsets, end_offsets, alive, hll, secs, tl, pcounts);
    kta_destroy(h);
    return rc;
}

int main(int argc, char **argv) {
    std::string topic, bootstrap, librdkafka, synthetic, log_dir, feed = "batch";
    int count_alive_occurrences = 0, hll = 0;
    TimelineOpt tl;
    std::vector<int32_t> pcounts;
    for (int i = 1; i < argc; i++) {
        const std::string a = argv[i];
        auto val = [&]() -> std::string { if (i + 1 >= argc) { fprintf(stderr, "error: %s needs a value\n", a.c_str()); exit(2); } return argv[++i]; };
        if (a == "-t" || a == "--topic") topic = val();
        else if (a == "-b" || a == "--bootstrap-server") bootstrap = val();
        else if (a == "--librdkafka") librdkafka = val();
        else if (a == "-c" || a == "--count-alive-keys") count_alive_occurrences++;
        else if (a == "-cc") count_alive_occurrences += 2;
        else if (a == "--synthetic") synthetic = val();
        else if (a == "--log-dir") log_dir = val();
        else if (a == "--feed") feed = val();
        else if (a == "--hll") hll = atoi(val().c_str());
        else if (a == "--timeline") { if (!parse_timeline(val(), tl)) return 2; }
        else if (a == "--partitioner-check") { if (!parse_partitioner_check(val(), pcounts)) return 2; }
        else if (a == "--hot-keys") { if (!parse_hot_keys(val())) return 2; }
        else if (a == "-V" || a == "--version") { puts("Kafka Topic Analyzer 0.4.1"); return 0; }  // main.rs:35
        else if (a == "-h" || a == "--help") {
            puts("Kafka Topic Analyzer 0.4.1\n\nUSAGE:\n    kafka-topic-analyzer [FLAGS] [OPTIONS] --bootstrap-server <BOOTSTRAP_SERVER> --topic <TOPIC>\n\n"
                 "FLAGS:\n    -c, --count-alive-keys    Counts the effective number of alive keys in a log compacted topic\n\n"
                 "OPTIONS:\n    -b, --bootstrap-server <BOOTSTRAP_SERVER>    Bootstrap server(s) to work with, comma separated\n"
                 "        --librdkafka <LIBRDKAFKA>                Options to pass into the underlying librdkafka\n"
                 "                                                 (this build reads isolation.level=read_committed|read_uncommitted\n"
                 "                                                 for --log-dir; its default is read_uncommitted, librdkafka's is\n"
                 "                                                 read_committed: pass isolation.level=read_committed to match it)\n"
                 "                                                 and check.crcs=true|false for --log-dir (default false, as\n"
                 "                                                 librdkafka's): true verifies every batch's CRC-32C, skips and\n"
                 "                                                 reports the batches that fail it, and reports the rest\n"
                 "        --log-dir <DIR>                          read <DIR>/<TOPIC>-<partition>/*.log (and, read_committed,\n"
                 "                                                 *.txnindex) instead of a broker; for the partitions that\n"
                 "                                                 <DIR>/log-start-offset-checkpoint and\n"
                 "                                                 <DIR>/replication-offset-checkpoint list, only the records\n"
                 "                                                 from the log start offset up to the high watermark\n"
                 "    -t, --topic <TOPIC>                          The topic to analyze\n"
                 "        --synthetic <k=v,...>                    in-memory synthetic topic (this build has no Kafka client)\n"
                 "        --feed <push|batch|device>               how records are handed to the metric handlers\n"
                 "        --timeline <W[,ORIGIN,BUCKETS]>          extension: records, tombstones and bytes per W-second bucket\n"
                 "                                                 (UTC), printed after the report; without ORIGIN and BUCKETS\n"
                 "                                                 the range covers the records' timestamps (at most 10000\n"
                 "                                                 buckets)\n"
                 "        --partitioner-check <N[,N...]>           extension: per partition, the keyed records that murmur2\n"
                 "                                                 (Java) and CRC-32 (librdkafka) would place there at each\n"
                 "                                                 partition count N, printed after the report\n"
                 "        --hot-keys <K>                           extension: the number of distinct keys and the K keys with\n"
                 "                                                 the most records, printed after the report");
            return 0;
        } else { fprintf(stderr, "error: Found argument '%s' which wasn't expected\n", a.c_str()); return 2; }
    }
    if (topic.empty() || bootstrap.empty()) {
        fprintf(stderr, "error: The following required arguments were not provided:\n    --bootstrap-server <BOOTSTRAP_SERVER>\n    --topic <TOPIC>\n");
        return 2;
    }
    if (synthetic.empty() && log_dir.empty()) {
        fprintf(stderr, "Error fetching metadata: this build has no librdkafka client (no broker access); pass --log-dir DIR or --synthetic n=...,partitions=...\n");
        return 101;  // the reference panics here (src/kafka.rs:61)
    }
    // --librdkafka k=v,k=v (src/main.rs:84-93).  Without a client only isolation.level and check.crcs have a meaning here.
    bool read_committed = false, check_crcs = false;
    for (size_t p = 0; !librdkafka.empty() && p <= librdkafka.size();) {
        size_t e = librdkafka.find(',', p);
        if (e == std::string::npos) e = librdkafka.size();
        const std::string item = librdkafka.substr(p, e - p);
        const size_t q = item.find('=');
        if (q == std::string::npos) { fprintf(stderr, "error: --librdkafka: '%s' is not key=value\n", item.c_str()); return 2; }
        if (item.substr(0, q) == "isolation.level") {
            const std::string v = item.substr(q + 1);
            if (v != "read_committed" && v != "read_uncommitted") {
                fprintf(stderr, "error: --librdkafka: isolation.level must be read_committed or read_uncommitted, not '%s'\n", v.c_str());
                return 2;
            }
            read_committed = v == "read_committed";
        } else if (item.substr(0, q) == "check.crcs") {
            const std::string v = item.substr(q + 1);
            if (v != "true" && v != "false") {
                fprintf(stderr, "error: --librdkafka: check.crcs must be true or false, not '%s'\n", v.c_str());
                return 2;
            }
            check_crcs = v == "true";
        }
        p = e + 1;
    }
    const auto start_time = std::chrono::steady_clock::now();  // main.rs:69
    if (!log_dir.empty())
        return analyze_log_dir(topic, log_dir, count_alive_occurrences == 1, hll, read_committed, check_crcs, start_time, tl, pcounts);

    std::map<std::string, std::string> kv;
    for (size_t p = 0; p < synthetic.size();) {
        size_t e = synthetic.find(',', p);
        if (e == std::string::npos) e = synthetic.size();
        const std::string item = synthetic.substr(p, e - p);
        const size_t q = item.find('=');
        if (q != std::string::npos) kv[item.substr(0, q)] = item.substr(q + 1);
        p = e + 1;
    }
    auto geti = [&](const char *k, long long d) { return kv.count(k) ? atoll(kv[k].c_str()) : d; };
    kta_synth_spec spec{};
    spec.seed = (uint64_t)geti("seed", 0x4B544131);
    spec.num_partitions = (int32_t)geti("partitions", 4);
    spec.run_len = (int32_t)geti("run_len", 1);
    spec.n_total = geti("n", 100000);
    spec.n_total -= spec.n_total % ((int64_t)spec.num_partitions * spec.run_len);
    spec.distinct_keys = (uint64_t)geti("distinct_keys", spec.n_total / 10 > spec.num_partitions ? spec.n_total / 10 : spec.num_partitions);
    spec.key_mode = (int32_t)geti("key_mode", 0) | (geti("zipf_keys", 0) ? KTA_SYNTH_KEYS_LOGUNIFORM : 0) |
                    (geti("geometric_values", 0) ? KTA_SYNTH_VALUES_GEOMETRIC : 0);
    spec.value_mean = (int32_t)geti("value_mean", 256);
    spec.null_key_per_10k = (int32_t)geti("null_key_per_10k", 100);
    spec.tombstone_per_10k = (int32_t)geti("tombstone_per_10k", 500);
    spec.ts_missing_per_10k = (int32_t)geti("ts_missing_per_10k", 0);
    spec.empty_value_per_10k = (int32_t)geti("empty_value_per_10k", 0);
    const int P = spec.num_partitions;
    const int64_t n = spec.n_total;

    // get_topic_offsets (src/kafka.rs:60-72): synthetic watermarks
    std::vector<int64_t> start_offsets(P, 0), end_offsets(P, n / P);
    if (n == 0) { fprintf(stderr, "Given topic has no content, no analysis possible. Exiting.\n"); return 254; }  // main.rs:98-101
    if (tl.on && !tl.ranged) {   // the range from the first and the last record of the topic
        int64_t ts0 = 0, ts1 = 0;
        if (kta_synth_fill_host(&spec, 0, 1, 0, 1, nullptr, nullptr, &ts0, nullptr, nullptr, nullptr, nullptr, 0, nullptr) ||
            kta_synth_fill_host(&spec, 0, 1, n - 1, 1, nullptr, nullptr, &ts1, nullptr, nullptr, nullptr, nullptr, 0, nullptr)) {
            fprintf(stderr, "synthetic fill failed\n");
            return 1;
        }
        if (!timeline_range(tl, std::min(ts_second(ts0), ts_second(ts1)), std::max(ts_second(ts0), ts_second(ts1)))) return 2;
    }

    kta_config cfg{};
    cfg.struct_size = sizeof cfg;
    cfg.device = -1;
    cfg.num_partitions = P;
    cfg.count_alive_keys = count_alive_occurrences == 1 ? 1 : 0;  // occurrences_of == 1, main.rs:77-80
    cfg.hll_precision = hll;
    cfg.now_s = INT64_MIN;
    kta_handle *h = nullptr;
    KTA(kta_create(&cfg, &h));
    if (tl.on) KTA(kta_set_timeline(h, tl.origin, tl.width, (int32_t)tl.buckets));
    if (!pcounts.empty()) KTA(kta_set_partitioner_check(h, pcounts.data(), (int32_t)pcounts.size()));
    if (g_hot_keys) KTA(kta_set_hot_keys(h, g_hot_keys, 0));

    printf("Subscribing to %s\n", topic.c_str());          // src/kafka.rs:88
    printf("Starting message consumption...\n");            // src/kafka.rs:91
    const int64_t CH = 1 << 20;
    double feed_s = 0;   // time spent inside the library's entry points only (not in the synthetic generator)
    auto now = [] { return std::chrono::duration<double>(std::chrono::steady_clock::now().time_since_epoch()).count(); };
    if (feed == "device") {
        const int64_t ntiles = (n + KTA_KEY_TILE - 1) / KTA_KEY_TILE;
        int32_t *dp, *dk, *dv; int64_t *dt; uint8_t *dkb; uint64_t *dtb;
        const int64_t cap = n * 40 + 64;
        if (cudaMalloc((void **)&dp, n * 4) || cudaMalloc((void **)&dk, n * 4) || cudaMalloc((void **)&dv, n * 4) || cudaMalloc((void **)&dt, n * 8) ||
            cudaMalloc((void **)&dkb, cap) || cudaMalloc((void **)&dtb, (ntiles + 1) * 8)) { fprintf(stderr, "cudaMalloc failed\n"); return 1; }
        int64_t kbl = 0;
        if (kta_synth_fill_device(&spec, -1, 0, 1, 0, n, dp, nullptr, dt, dk, dv, nullptr, dkb, cap, dtb, &kbl)) { fprintf(stderr, "synthetic fill failed\n"); return 1; }
        kta_batch b{};
        b.n = n; b.partition = dp; b.ts_ms = dt; b.key_len = dk; b.value_len = dv; b.key_bytes = dkb; b.key_bytes_len = kbl; b.key_tile_base = dtb;
        const double t0 = now();
        KTA(kta_scan_batch_device(h, &b));
        KTA(kta_sync(h));
        feed_s += now() - t0;
    } else {
        if (feed == "push") {
            // the pinned landing ring (3 chunks, ~0.5 GB) is allocated by the first push: do that outside the timed feed —
            // a real run amortises it over the whole topic, a 2e7-record measurement would be dominated by it
            KTA(kta_push(h, 0, 0, 0, nullptr, -1, 0));
            KTA(kta_sync(h));
            KTA(kta_reset(h));   // (keeps the timeline's configuration)
        }
        std::vector<int32_t> part(CH), kl(CH), vl(CH);
        std::vector<int64_t> off(CH), ts(CH);
        std::vector<uint8_t> kb((size_t)CH * 40 + 16);
        for (int64_t s0 = 0; s0 < n; s0 += CH) {
            const int64_t c = std::min(CH, n - s0);
            int64_t kbl = 0;
            if (kta_synth_fill_host(&spec, 0, 1, s0, c, part.data(), off.data(), ts.data(), kl.data(), vl.data(), nullptr,
                                    kb.data(), (int64_t)kb.size(), &kbl)) { fprintf(stderr, "synthetic fill failed\n"); return 1; }
            const double t0 = now();
            if (feed == "push") {
                // the reference's shape: one handle_message per polled message (src/kafka.rs:107-109)
                int64_t ko = 0;
                for (int64_t i = 0; i < c; i++) {
                    KTA(kta_push(h, part[i], off[i], ts[i], kl[i] > 0 ? kb.data() + ko : (kl[i] == 0 ? kb.data() : nullptr), kl[i], vl[i]));
                    if (kl[i] > 0) ko += kl[i];
                }
            } else {
                kta_batch b{};
                b.n = c; b.seq_base = (uint64_t)s0; b.partition = part.data(); b.offset = off.data(); b.ts_ms = ts.data();
                b.key_len = kl.data(); b.value_len = vl.data(); b.key_bytes = kb.data(); b.key_bytes_len = kbl;
                KTA(kta_push_batch_host(h, &b));
            }
            feed_s += now() - t0;
        }
    }
    {
        const double t0 = now();
        finalize_or_warn(h);
        feed_s += now() - t0;
    }
    fprintf(stderr, "[kta] feed=%s: %lld records through the handlers in %.4f s = %.3e msg/s (generator excluded)\n", feed.c_str(),
            (long long)n, feed_s, feed_s > 0 ? (double)n / feed_s : 0.0);
    const uint64_t duration_secs = (uint64_t)std::chrono::duration_cast<std::chrono::seconds>(std::chrono::steady_clock::now() - start_time).count();

    std::vector<int> all_partitions(P);
    for (int p = 0; p < P; p++) all_partitions[p] = p;
    const int rc = print_report(h, topic, all_partitions, start_offsets, end_offsets, cfg.count_alive_keys == 1, hll, duration_secs, tl,
                                pcounts);
    kta_destroy(h);
    return rc;
}

static int print_report(kta_handle *h, const std::string &topic, const std::vector<int> &partitions, const std::vector<int64_t> &start_offsets,
                        const std::vector<int64_t> &end_offsets, bool alive, int hll, uint64_t duration_secs, const TimelineOpt &tl,
                        const std::vector<int32_t> &pcounts) {
    kta_report::Summary s{};
    s.topic = topic;
    s.duration_secs = duration_secs;
    KTA(kta_global(h, KTA_OVERALL_COUNT, &s.overall_count));
    KTA(kta_timestamps(h, &s.earliest_s, &s.earliest_ns, &s.latest_s));
    KTA(kta_global(h, KTA_LARGEST_MESSAGE, &s.largest_message));
    KTA(kta_global(h, KTA_SMALLEST_MESSAGE, &s.smallest_message));
    KTA(kta_global(h, KTA_OVERALL_SIZE, &s.overall_size));
    s.has_alive_keys = alive;
    if (s.has_alive_keys) KTA(kta_alive_keys(h, &s.alive_keys));
    std::vector<kta_report::PartitionRow> rows;
    for (int p : partitions) {  // partitions of the metadata, sorted ascending, main.rs:103-106
        kta_report::PartitionRow r{};
        r.partition = p; r.start_offset = start_offsets[p]; r.end_offset = end_offsets[p];
        KTA(kta_counter(h, KTA_TOTAL, p, &r.total)); KTA(kta_counter(h, KTA_ALIVE, p, &r.alive));
        KTA(kta_counter(h, KTA_TOMBSTONES, p, &r.tombstones)); KTA(kta_dirty_ratio(h, p, &r.dirty_ratio));
        KTA(kta_counter(h, KTA_KEY_NULL, p, &r.key_null)); KTA(kta_counter(h, KTA_KEY_NON_NULL, p, &r.key_non_null));
        KTA(kta_counter(h, KTA_KEY_SIZE_SUM, p, &r.key_size_sum)); KTA(kta_counter(h, KTA_VALUE_SIZE_SUM, p, &r.value_size_sum));
        // the reference panics ("attempt to divide by zero") when sum > 0 && alive == 0 (metric.rs:132-157)
        int rc = kta_avg(h, KTA_KEY_SIZE_AVG, p, &r.key_size_avg);
        if (rc == KTA_OK) rc = kta_avg(h, KTA_VALUE_SIZE_AVG, p, &r.value_size_avg);
        if (rc == KTA_OK) rc = kta_avg(h, KTA_MESSAGE_SIZE_AVG, p, &r.message_size_avg);
        if (rc == KTA_ERR_DIV_BY_ZERO) { fprintf(stderr, "thread 'main' panicked at 'attempt to divide by zero', src/metric.rs\n"); return 101; }
        if (rc != KTA_OK) die("kta_avg");
        rows.push_back(r);
    }
    fputs(kta_report::render(s, rows).c_str(), stdout);
    if (hll) { double e = 0; KTA(kta_alive_keys_hll(h, &e)); printf("| extension: HyperLogLog(p=%d) alive-key estimate: %.0f\n", hll, e); }
    if (tl.on) print_timeline(h, partitions, tl);
    if (!pcounts.empty()) print_partitioner_check(h, partitions, pcounts);
    if (g_hot_keys) print_hot_keys(h);
    return 0;
}
