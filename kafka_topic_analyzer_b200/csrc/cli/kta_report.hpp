// kta_report.hpp — the reference's report (src/main.rs:123-179) over the C ABI getters: header block,
// then the 15-column table in prettytable-rs' default format (borders + a separator after every row,
// cells left-aligned with one space of padding), `{:.4}` dirty ratio, chrono's `Display` for DateTime<Utc>.
#pragma once
#include <cstdint>
#include <cstdio>
#include <string>
#include <vector>

namespace kta_report {

struct PartitionRow {  // one table row, src/main.rs:153-171
    int32_t partition;
    int64_t start_offset, end_offset;
    uint64_t total, alive, tombstones;
    float dirty_ratio;
    uint64_t key_null, key_non_null, key_size_sum, value_size_sum, key_size_avg, value_size_avg, message_size_avg;
};

struct Summary {  // src/main.rs:125-143
    std::string topic;
    uint64_t duration_secs, overall_count;
    int64_t earliest_s;
    int32_t earliest_ns;
    int64_t latest_s;
    uint64_t largest_message, smallest_message, overall_size;
    bool has_alive_keys;
    uint64_t alive_keys;
};

// chrono 0.4 `impl Display for DateTime<Utc>`: "YYYY-MM-DD HH:MM:SS[.fff[fff[fff]]] UTC"
inline std::string format_utc(int64_t secs, int32_t nanos) {
    int64_t days = secs / 86400, rem = secs % 86400;
    if (rem < 0) { rem += 86400; days -= 1; }
    // civil-from-days (H. Hinnant), proleptic Gregorian
    int64_t z = days + 719468;
    const int64_t era = (z >= 0 ? z : z - 146096) / 146097;
    const unsigned doe = (unsigned)(z - era * 146097);
    const unsigned yoe = (doe - doe / 1460 + doe / 36524 - doe / 146096) / 365;
    int64_t y = (int64_t)yoe + era * 400;
    const unsigned doy = doe - (365 * yoe + yoe / 4 - yoe / 100);
    const unsigned mp = (5 * doy + 2) / 153;
    const unsigned d = doy - (153 * mp + 2) / 5 + 1;
    const unsigned m = mp < 10 ? mp + 3 : mp - 9;
    if (m <= 2) y += 1;
    char buf[96];
    int n = snprintf(buf, sizeof buf, "%04lld-%02u-%02u %02lld:%02lld:%02lld", (long long)y, m, d, (long long)(rem / 3600),
                     (long long)(rem % 3600 / 60), (long long)(rem % 60));
    if (nanos != 0) {
        if (nanos % 1000000 == 0) n += snprintf(buf + n, sizeof buf - n, ".%03d", nanos / 1000000);
        else if (nanos % 1000 == 0) n += snprintf(buf + n, sizeof buf - n, ".%06d", nanos / 1000);
        else n += snprintf(buf + n, sizeof buf - n, ".%09d", nanos);
    }
    snprintf(buf + n, sizeof buf - n, " UTC");
    return buf;
}

// columns a UTF-8 cell takes: its bytes that do not continue a character (ASCII cells: their size)
inline size_t cell_width(const std::string &s) {
    size_t n = 0;
    for (unsigned char c : s) n += (c & 0xc0) != 0x80;
    return n;
}

inline std::string render_table(const std::vector<std::vector<std::string>> &rows) {
    std::vector<size_t> w;
    for (const auto &r : rows) {
        if (w.size() < r.size()) w.resize(r.size(), 0);
        for (size_t c = 0; c < r.size(); c++) w[c] = std::max(w[c], cell_width(r[c]));
    }
    std::string sep = "+";
    for (size_t c = 0; c < w.size(); c++) sep += std::string(w[c] + 2, '-') + "+";
    sep += "\n";
    std::string out = sep;
    for (const auto &r : rows) {
        out += "|";
        for (size_t c = 0; c < w.size(); c++) {
            const std::string &cell = c < r.size() ? r[c] : std::string();
            out += " " + cell + std::string(w[c] - cell_width(cell), ' ') + " |";
        }
        out += "\n" + sep;
    }
    return out;
}

inline std::string render(const Summary &s, const std::vector<PartitionRow> &parts) {
    auto u = [](uint64_t v) { return std::to_string(v); };
    const std::string eq(120, '='), dash(120, '-');
    std::string o = "\n" + eq + "\nCalculating statistics...\n";
    o += "Topic " + s.topic + "\n";
    o += "Scanning took: " + u(s.duration_secs) + " seconds\n";
    o += "Estimated Msg/s: " + u(s.overall_count / (s.duration_secs > 1 ? s.duration_secs : 1)) + "\n";  // main.rs:130
    o += dash + "\nEarliest Message: " + format_utc(s.earliest_s, s.earliest_ns) + "\n";
    o += "Latest Message: " + format_utc(s.latest_s, 0) + "\n" + dash + "\n";
    o += "Largest Message: " + u(s.largest_message) + " bytes\n";
    o += "Smallest Message: " + u(s.smallest_message) + " bytes\n";
    o += "Topic Size: " + u(s.overall_size) + " bytes\n";
    if (s.has_alive_keys) o += dash + "\nAlive keys: " + u(s.alive_keys) + "\n" + dash + "\n";  // main.rs:139-146
    o += eq + "\n";
    std::vector<std::vector<std::string>> rows;
    rows.push_back({"P", "< OS", "> OS", "Total", "Alive", "Tmb", "DR", "K Null", "K !Null", "P-Bytes", "K-Bytes", "V-Bytes",
                    "A K-Sz", "A V-Sz", "A M-Sz"});  // main.rs:150
    for (const auto &p : parts) {
        char dr[64];
        snprintf(dr, sizeof dr, "%.4f", (double)p.dirty_ratio);  // {0:.4}
        rows.push_back({std::to_string(p.partition), std::to_string(p.start_offset), std::to_string(p.end_offset), u(p.total),
                        u(p.alive), u(p.tombstones), dr, u(p.key_null), u(p.key_non_null),
                        u(p.key_size_sum + p.value_size_sum), u(p.key_size_sum), u(p.value_size_sum), u(p.key_size_avg),
                        u(p.value_size_avg), u(p.message_size_avg)});
    }
    o += "| K = Key, V = Value, P = Partition, Tmb = Tombstone(s), Sz = Size\n";
    o += "| DR = Dirty Ratio, A = Average, Lst = last, < OS = start offset, > OS = end offset\n";
    o += render_table(rows);
    o += "\n" + eq + "\n";
    return o;
}

// extension (--timeline): one table row per non-empty index of the summed timeline (include/kta.h kta_timeline)
struct TimelineRow {
    int64_t index;       // 0 = before the range, 1..B = bucket index - 1, B + 1 = after it
    int64_t start_s;     // start of the bucket (index 1..B)
    uint64_t records, tombstones, bytes;
};

inline std::string render_timeline(int64_t origin, int64_t width, int64_t buckets, const std::vector<TimelineRow> &rows) {
    auto u = [](uint64_t v) { return std::to_string(v); };
    std::string o = "| extension: timeline, " + std::to_string(buckets) + " buckets of " + std::to_string(width) + " s from " +
                    format_utc(origin, 0) + "\n";
    std::vector<std::vector<std::string>> t;
    t.push_back({"Bucket start", "Records", "Tmb", "Bytes"});
    for (const auto &r : rows) {
        const std::string start = r.index == 0 ? "before " + format_utc(origin, 0)
                                  : r.index == buckets + 1 ? format_utc(origin + buckets * width, 0) + " and later"
                                                           : format_utc(r.start_s, 0);
        t.push_back({start, u(r.records), u(r.tombstones), u(r.bytes)});
    }
    return o + render_table(t);
}

// extension (--partitioner-check): per partition, its keyed records and where the partitioners would put them
// (include/kta.h kta_partitioner_check), then the total over the rows
struct PartitionerRow {
    int32_t partition;
    uint64_t keyed;                  // KTA_KEY_NON_NULL
    std::vector<uint64_t> counts;    // murmur2 per count | CRC-32 per count | neither
};

inline std::string render_partitioner_check(const std::vector<int32_t> &counts, const std::vector<PartitionerRow> &rows) {
    std::string o = "| extension: partitioner check, keyed records placed as murmur2 (Java) or CRC-32 (librdkafka) would place "
                    "them at";
    for (size_t j = 0; j < counts.size(); j++) o += (j ? ", " : " ") + std::to_string(counts[j]);
    o += " partitions\n";
    std::vector<std::vector<std::string>> t;
    std::vector<std::string> head = {"P", "Keyed"};
    for (int32_t n : counts) head.push_back("murmur2@" + std::to_string(n));
    for (int32_t n : counts) head.push_back("crc32@" + std::to_string(n));
    head.push_back("Neither");
    t.push_back(head);
    PartitionerRow total{};
    total.counts.assign(2 * counts.size() + 1, 0);
    for (const auto &r : rows) {
        std::vector<std::string> cells = {std::to_string(r.partition), std::to_string(r.keyed)};
        for (size_t b = 0; b < total.counts.size(); b++) {
            cells.push_back(std::to_string(r.counts[b]));
            total.counts[b] += r.counts[b];
        }
        total.keyed += r.keyed;
        t.push_back(cells);
    }
    std::vector<std::string> cells = {"total", std::to_string(total.keyed)};
    for (uint64_t v : total.counts) cells.push_back(std::to_string(v));
    t.push_back(cells);
    return o + render_table(t);
}

// extension (--hot-keys): the keys with the most records (include/kta.h kta_hot_keys), ranked
struct HotKeyRow {
    uint64_t records, tombstones, bytes;
    int64_t latest_s;
    int32_t min_partition, max_partition, key_len;
    std::string prefix;              // the first min(key_len, 32) bytes
};

// a key as text when every byte of its prefix is printable ASCII, else as 0x-prefixed hex; "…" when the key is longer
// than its prefix; an empty key as (empty)
inline std::string render_key(const std::string &prefix, int32_t key_len) {
    if (key_len == 0) return "(empty)";
    bool text = true;
    for (unsigned char c : prefix) text = text && c >= 0x20 && c < 0x7f;
    std::string o;
    if (text) {
        o = prefix;
    } else {
        static const char *hex = "0123456789abcdef";
        o = "0x";
        for (unsigned char c : prefix) { o += hex[c >> 4]; o += hex[c & 15]; }
    }
    if ((size_t)key_len > prefix.size()) o += "\u2026";
    return o;
}

inline std::string render_hot_keys(uint64_t distinct, const std::vector<HotKeyRow> &rows) {
    std::string o = "| extension: hot keys, the keys with the most records\nDistinct keys: " + std::to_string(distinct) +
                    " (by 64-bit id)\n";
    std::vector<std::vector<std::string>> t = {{"#", "Records", "Tombstones", "Bytes", "Partitions", "Latest write", "Key"}};
    for (size_t i = 0; i < rows.size(); i++) {
        const HotKeyRow &r = rows[i];
        const std::string parts = r.min_partition == r.max_partition
                                      ? std::to_string(r.min_partition)
                                      : std::to_string(r.min_partition) + "\u2013" + std::to_string(r.max_partition);
        t.push_back({std::to_string(i + 1), std::to_string(r.records), std::to_string(r.tombstones), std::to_string(r.bytes), parts,
                     format_utc(r.latest_s, 0), render_key(r.prefix, r.key_len)});
    }
    return o + render_table(t);
}

}  // namespace kta_report
