// kta_synth_host.cpp — the HOST half of the synthetic topic (kta_synth.h): slices of the topic as SoA columns in
// host memory and as RecordBatch v2 log segments.  Plain C++ (no CUDA): compiled into libkta_gpu.so (kta_synth.cu
// includes it) and, on its own, into libkta_synth.so, so that CPU-only users — the oracle tests and bench.py's
// reference arm — generate the same topic without mapping the GPU library.
#include <algorithm>
#include <array>
#include <cstdio>
#include <cstring>
#include <vector>

#include "kta_synth.h"

static int synth_check(const kta_synth_spec *s, int32_t rank, int32_t world) {
    if (!s || s->num_partitions < 1 || s->run_len < 1 || s->n_total < 0 || world < 1 || rank < 0 || rank >= world)
        return KTA_ERR_INVALID;
    if (s->key_mode < 0 || (s->key_mode & 0xff) > 2 || (s->key_mode & ~0x3ff) || s->value_mean < 0) return KTA_ERR_INVALID;
    // the largest uniform value length, mean/2 + mean, must fit value_len's int32 (KTA_SYNTH_MAX_VALUE_MEAN)
    if (s->value_mean > KTA_SYNTH_MAX_VALUE_MEAN) return KTA_ERR_INVALID;
    if (s->n_total % ((int64_t)s->num_partitions * s->run_len) != 0) return KTA_ERR_INVALID;
    if (world > 1 && s->num_partitions % world != 0) return KTA_ERR_INVALID;
    return KTA_OK;
}

extern "C" int64_t kta_synth_shard_records(const kta_synth_spec *s, int32_t rank, int32_t world) {
    if (synth_check(s, rank, world)) return -1;
    return s->n_total / world;  // every partition holds n_total / P records
}

extern "C" int kta_synth_fill_host(const kta_synth_spec *s, int32_t rank, int32_t world, int64_t start, int64_t count,
                                   int32_t *partition, int64_t *offset, int64_t *ts_ms, int32_t *key_len,
                                   int32_t *value_len, uint64_t *seq, uint8_t *key_bytes, int64_t key_bytes_cap,
                                   int64_t *key_bytes_len) {
    if (synth_check(s, rank, world) || start < 0 || count < 0 || start + count > s->n_total / world) return KTA_ERR_INVALID;
    int64_t kb = 0;
    uint8_t tmp[KTA_SYNTH_MAX_KEY];
    for (int64_t j = 0; j < count; j++) {
        kta_synth_record r;
        kta_synth_record_at(*s, kta_synth_local_to_global(*s, rank, world, (uint64_t)(start + j)), r);
        if (partition) partition[j] = r.partition;
        if (offset) offset[j] = r.offset;
        if (ts_ms) ts_ms[j] = r.ts_ms;
        if (key_len) key_len[j] = r.key_len;
        if (value_len) value_len[j] = r.value_len;
        if (seq) seq[j] = r.seq;
        if (r.key_len > 0) {
            if (key_bytes) {
                if (kb + r.key_len > key_bytes_cap) return KTA_ERR_NOMEM;
                kta_synth_key_bytes(*s, r.key_id, tmp);
                memcpy(key_bytes + kb, tmp, (size_t)r.key_len);
            }
            kb += r.key_len;
        }
    }
    if (key_bytes_len) *key_bytes_len = kb;
    return KTA_OK;
}

// ---- the same topic as a broker would store it: one RecordBatch v2 log segment per partition (uncompressed) ----
static inline void put_be(std::vector<uint8_t> &o, uint64_t v, int bytes) {
    for (int i = bytes - 1; i >= 0; i--) o.push_back((uint8_t)(v >> (8 * i)));
}
static inline void put_varint(std::vector<uint8_t> &o, int64_t n) {
    uint64_t u = ((uint64_t)n << 1) ^ (uint64_t)(n >> 63);   // zig-zag
    while (u >= 0x80) { o.push_back((uint8_t)(u | 0x80)); u >>= 7; }
    o.push_back((uint8_t)u);
}

// CRC-32C (Castagnoli, reflected polynomial 0x82F63B78), byte at a time: the register after [p, p + n) from `crc`
static uint32_t crc32c_update(uint32_t crc, const uint8_t *p, size_t n) {
    static const std::array<uint32_t, 256> table = [] {
        std::array<uint32_t, 256> t{};
        for (uint32_t i = 0; i < 256; i++) {
            uint32_t c = i;
            for (int k = 0; k < 8; k++) c = (c >> 1) ^ ((c & 1u) ? 0x82F63B78u : 0u);
            t[i] = c;
        }
        return t;
    }();
    for (size_t i = 0; i < n; i++) crc = table[(crc ^ p[i]) & 0xffu] ^ (crc >> 8);
    return crc;
}

// Encodes records [start, start+count) (offset order) of partition `partition` as record batches of
// `batch_records` records.  *len receives the bytes needed; nothing is written beyond cap (call twice to size).
extern "C" int kta_synth_encode_segment_host(const kta_synth_spec *s, int32_t partition, int64_t start, int64_t count,
                                             int32_t batch_records, uint8_t *out, int64_t cap, int64_t *len) {
    if (!s || !len || batch_records < 1 || partition < 0 || partition >= s->num_partitions) return KTA_ERR_INVALID;
    if (synth_check(s, 0, 1) || start < 0 || count < 0 || start + count > s->n_total / s->num_partitions) return KTA_ERR_INVALID;
    std::vector<uint8_t> batch, recs, rec;
    uint8_t key[KTA_SYNTH_MAX_KEY];
    int64_t total = 0;
    for (int64_t b0 = 0; b0 < count; b0 += batch_records) {
        const int64_t nb = std::min<int64_t>(batch_records, count - b0);
        recs.clear();
        int64_t base_ts = 0, max_ts = 0;
        bool have_ts = false;
        std::vector<kta_synth_record> rr((size_t)nb);
        for (int64_t i = 0; i < nb; i++) {
            // partition p's records in offset order = shard `p` of a world of P ranks
            kta_synth_record_at(*s, kta_synth_local_to_global(*s, partition, s->num_partitions, (uint64_t)(start + b0 + i)), rr[(size_t)i]);
            if (rr[(size_t)i].ts_ms != -1) {
                if (!have_ts) { base_ts = rr[(size_t)i].ts_ms; max_ts = base_ts; have_ts = true; }
                max_ts = std::max(max_ts, rr[(size_t)i].ts_ms);
            }
        }
        if (!have_ts) base_ts = max_ts = -1;
        for (int64_t i = 0; i < nb; i++) {
            const kta_synth_record &r = rr[(size_t)i];
            rec.clear();
            rec.push_back(0);
            // the consumer's timestamp is baseTimestamp + timestampDelta, and only a result of -1 means "not available": a
            // record without a timestamp inside a batch that has one gets the delta -1 - baseTimestamp
            put_varint(rec, !have_ts ? 0 : r.ts_ms != -1 ? r.ts_ms - base_ts : -1 - base_ts);
            put_varint(rec, i);
            if (r.key_len < 0) put_varint(rec, -1);
            else {
                put_varint(rec, r.key_len);
                const int32_t kl = kta_synth_key_bytes(*s, r.key_id, key);
                rec.insert(rec.end(), key, key + kl);
            }
            if (r.value_len < 0) put_varint(rec, -1);
            else {
                put_varint(rec, r.value_len);
                rec.insert(rec.end(), (size_t)r.value_len, (uint8_t)0x5a);
            }
            put_varint(rec, 0);
            put_varint(recs, (int64_t)rec.size());
            recs.insert(recs.end(), rec.begin(), rec.end());
        }
        batch.clear();
        put_be(batch, (uint64_t)rr[0].offset, 8);
        put_be(batch, (uint64_t)(49 + recs.size()), 4);
        put_be(batch, 0, 4);            // partitionLeaderEpoch
        batch.push_back(2);             // magic
        put_be(batch, 0, 4);            // crc: written below, once the bytes it covers are known
        put_be(batch, 0, 2);            // attributes: uncompressed, CreateTime
        put_be(batch, (uint64_t)(nb - 1), 4);
        put_be(batch, (uint64_t)base_ts, 8);
        put_be(batch, (uint64_t)max_ts, 8);
        put_be(batch, ~0ull, 8);        // producerId -1
        put_be(batch, 0xffff, 2);       // producerEpoch -1
        put_be(batch, 0xffffffffu, 4);  // baseSequence -1
        put_be(batch, (uint64_t)nb, 4);
        // the CRC-32C a broker stores: from attributes (byte 21) to the end of the batch
        const uint32_t crc = ~crc32c_update(crc32c_update(0xffffffffu, batch.data() + 21, batch.size() - 21), recs.data(), recs.size());
        for (int i = 0; i < 4; i++) batch[17 + i] = (uint8_t)(crc >> (24 - 8 * i));
        if (out && total + (int64_t)(batch.size() + recs.size()) <= cap) {
            memcpy(out + total, batch.data(), batch.size());
            memcpy(out + total + batch.size(), recs.data(), recs.size());
        }
        total += (int64_t)(batch.size() + recs.size());
    }
    *len = total;
    return (out && total > cap) ? KTA_ERR_NOMEM : KTA_OK;
}

