// kta_logdecode.cuh — Kafka RecordBatch v2 (magic 2) → SoA columns, on the GPU (SURVEY.md §8 f2).
//
// This is the step BEFORE the metric path: in the reference it happens inside librdkafka's fetch parser, which
// hands one BorrowedMessage per record to the handlers (src/kafka.rs:93,107-109).  Here a whole log segment
// (the concatenated record batches of one partition, exactly what a broker stores in <topic>-<p>/*.log and
// sends in a fetch response) is decoded where it lies in HBM:
//   batch header (61 bytes, big-endian): baseOffset i64 | batchLength i32 | partitionLeaderEpoch i32 | magic i8 |
//     crc u32 | attributes i16 | lastOffsetDelta i32 | baseTimestamp i64 | maxTimestamp i64 | producerId i64 |
//     producerEpoch i16 | baseSequence i32 | recordsCount i32
//   record: length varint | attributes i8 | timestampDelta varlong | offsetDelta varint | keyLength varint | key |
//     valueLength varint | value | headersCount varint | headers…          (varints are zig-zag, LSB group first)
// Semantics kept from the consumer: control batches (attributes bit 5) are not delivered to the application;
// LogAppendTime batches (attributes bit 3) stamp every record with maxTimestamp; a record's timestamp is baseTimestamp +
// timestampDelta as the consumer computes it, and only a RESULT of -1 means "not available"; key/value length -1 means
// null.  CRCs are verified only when the handle's check.crcs switch is on (kta_logcrc.cuh; off by default, like librdkafka's
// check.crcs=false).
// Compression (attributes bits 0-2, librdkafka decompresses inside poll, src/kafka.rs:93): gzip (kta_inflate.cuh), LZ4 (frame
// format), Snappy (raw or xerial-framed; both kta_lz4_snappy.cuh) and zstd (kta_zstd.cuh) batches are decompressed on the GPU
// into a scratch buffer and then decoded like the others; the unassigned codes 5-7 are rejected.  Checksums inside the
// compressed sections (gzip's CRC32, zstd's Content_Checksum) are skipped, not verified, like the batch CRC.
// Isolation: on a read_committed handle the passes of kta_logtxn.cuh mark the batches of aborted transactions
// LOGB_SKIP_ABORTED before anything here decompresses or decodes them; on a read_uncommitted handle (the default) every
// data batch is delivered, as before.  Not handled: legacy magic 0/1 message sets are flagged as malformed.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include <cstddef>
#include <type_traits>

#include "kta_codec.cuh"
#include "kta_inflate.cuh"
#include "kta_lz4_snappy.cuh"
#include "kta_zstd.cuh"

namespace kta {

constexpr int LOG_HEADER_BYTES = 61;
// LOGB_COMPRESSED: an unknown compression codec (the unassigned codes 5-7).  LOGB_LZ4 / LOGB_SNAPPY / LOGB_GZIP / LOGB_ZSTD: the
// records section must be decompressed first (log_unc_size_kernel, log_zstd_size_kernel for zstd, and log_decompress_kernel
// turn such a batch into LOGB_OK).  LOGB_SKIP_ABORTED: a batch of an aborted transaction (read_committed only,
// kta_logtxn.cuh); it replaces any codec flag, so no later pass touches the batch.  LOGB_SKIP_CRC: a batch whose CRC-32C
// failed (check.crcs only, kta_logcrc.cuh); nothing CRC-covered of it is read, by the header pass or any later one.
// LOGB_SKIP_OFFSET: a batch a consumer is not served, wholly outside its partition's [log start offset, high watermark)
// window (kta_logoffsets.cuh); like LOGB_SKIP_CRC it is neither checked nor read further.
enum LogBatchFlags { LOGB_OK = 0, LOGB_SKIP_CONTROL = 1, LOGB_BAD = 2, LOGB_COMPRESSED = 4, LOGB_LZ4 = 8, LOGB_SNAPPY = 16, LOGB_GZIP = 32,
                     LOGB_ZSTD = 64, LOGB_SKIP_ABORTED = 128, LOGB_SKIP_CRC = 256, LOGB_SKIP_OFFSET = 512 };
constexpr uint32_t LOGB_CODECS = LOGB_LZ4 | LOGB_SNAPPY | LOGB_GZIP | LOGB_ZSTD;   // batches log_decompress_kernel turns into LOGB_OK

// the flag of Kafka's compression codec id 0-4 (attributes & 7: none, gzip, Snappy, LZ4, zstd)
__host__ __device__ __forceinline__ uint32_t log_codec_flag(uint32_t codec) {
    return codec == 0 ? LOGB_OK : codec == 1 ? LOGB_GZIP : codec == 2 ? LOGB_SNAPPY : codec == 3 ? LOGB_LZ4 : LOGB_ZSTD;
}

__device__ __forceinline__ uint64_t be_u64(const uint8_t *p) {
    uint64_t v = 0;
#pragma unroll
    for (int i = 0; i < 8; i++) v = (v << 8) | __ldg(p + i);
    return v;
}
__device__ __forceinline__ uint32_t be_u32(const uint8_t *p) {
    return ((uint32_t)__ldg(p) << 24) | ((uint32_t)__ldg(p + 1) << 16) | ((uint32_t)__ldg(p + 2) << 8) | __ldg(p + 3);
}
__device__ __forceinline__ uint32_t be_u16(const uint8_t *p) { return ((uint32_t)__ldg(p) << 8) | __ldg(p + 1); }

__device__ __forceinline__ int64_t unzigzag(uint64_t u) { return (int64_t)(u >> 1) ^ -(int64_t)(u & 1); }

struct LogBatchInfo {      // one per record batch, filled by log_header_kernel
    uint64_t off;          // byte offset of the batch in the segment buffer
    uint32_t len;          // 12 + batchLength
    uint32_t flags;        // LogBatchFlags
    int32_t partition;
    int32_t records;       // records delivered to the handlers (0 for skipped batches)
    int64_t base_offset, base_ts, max_ts;
    uint32_t log_append_time;
    uint32_t pad;
};

// The header pass's error word: zeroed before the pass and read back whole.  The decompression and decode passes that
// follow use `flags` as their own flag word.
struct LogHeaderWord {
    uint32_t flags;                            // LOGB_* bits of batches that refuse the call or are to be decompressed
    uint32_t longest;                          // the longest LOGB_OK batch (sizes the decode stage)
    uint32_t crc_failed;                       // check.crcs: batches whose CRC failed
    uint32_t pad;
    unsigned long long crc_failed_bytes;       // check.crcs: their bytes
    uint32_t cut;                              // windows: cut batches (on the cut list)
    uint32_t not_served;                       // windows: batches not served
    unsigned long long not_served_records;     // windows: their data records
};
static_assert(sizeof(LogHeaderWord) == 40 && offsetof(LogHeaderWord, longest) == 4 && offsetof(LogHeaderWord, crc_failed) == 8 &&
                  offsetof(LogHeaderWord, crc_failed_bytes) == 16 && offsetof(LogHeaderWord, cut) == 24 &&
                  offsetof(LogHeaderWord, not_served) == 28 && offsetof(LogHeaderWord, not_served_records) == 32,
              "the probes write the header word out as ten u32 words");

// The header pass, thread per batch: validate + read the header.  crc_failed(p, len, b, partition) is asked first for a
// framed batch (magic 2, batchLength >= 49, inside the buffer); when it says so, the batch is LOGB_SKIP_CRC and none of
// its CRC-covered fields is read (check.crcs, kta_logcrc.cuh).  Without the check it is NoCrcCheck, which never says so.
// Before that, a Window with `on` set is asked whether the framed batch is served at all (window.test(p, partition):
// LOG_WIN_SKIP makes it LOGB_SKIP_OFFSET, counted by window.skipped; LOG_WIN_CUT puts a data batch with records on the
// window's cut list, kta_logoffsets.cuh).  NoWindow is off: the pass compiles to what it was without the question.
// log_header_kernel (kta_logoffsets.cuh) runs the pass with either switch.
struct NoCrcCheck {
    __device__ __forceinline__ bool operator()(const uint8_t *, uint32_t, int64_t, int32_t) const { return false; }
};
enum LogWinVerdict { LOG_WIN_SERVED = 0, LOG_WIN_CUT = 1, LOG_WIN_SKIP = 2 };
struct NoWindow {
    static constexpr bool on = false;
    __device__ __forceinline__ int test(const uint8_t *, int32_t) const { return LOG_WIN_SERVED; }
    __device__ __forceinline__ void skipped(uint32_t, int32_t) const {}
    __device__ __forceinline__ void cut(int64_t) const {}
};
template <typename CrcCheck, typename Window>
__device__ __forceinline__ void log_header_pass(const uint8_t *bytes, int64_t nbytes, const uint64_t *batch_off, int64_t nbatches,
                                                int32_t partition, const int32_t *batch_partition, LogBatchInfo *info,
                                                uint64_t *rec_count, LogHeaderWord *word, const CrcCheck &crc_failed,
                                                const Window &window) {
    for (int64_t b = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; b < nbatches; b += (int64_t)gridDim.x * blockDim.x) {
        LogBatchInfo bi{};
        bi.off = batch_off[b];
        bi.partition = batch_partition ? batch_partition[b] : partition;
        bi.flags = LOGB_BAD;
        if (bi.off + LOG_HEADER_BYTES <= (uint64_t)nbytes) {
            const uint8_t *p = bytes + bi.off;
            const int32_t batch_len = (int32_t)be_u32(p + 8);
            const int magic = (int8_t)__ldg(p + 16);
            const uint32_t attrs = be_u16(p + 21);
            const int32_t count = (int32_t)be_u32(p + 57);
            // recordsCount sizes the output columns, so it must be plausible before anything is allocated for it: the
            // smallest record is 7 bytes (length, attributes, two deltas, key length, value length, header count)
            const uint32_t codec = attrs & 0x7u;
            const bool framed = magic == 2 && batch_len >= LOG_HEADER_BYTES - 12 && bi.off + 12 + (uint64_t)batch_len <= (uint64_t)nbytes;
            int verdict = LOG_WIN_SERVED;
            if constexpr (Window::on) verdict = framed ? window.test(p, bi.partition) : LOG_WIN_SERVED;
            if (Window::on && verdict == LOG_WIN_SKIP) {
                bi.flags = LOGB_SKIP_OFFSET;
                bi.len = 12u + (uint32_t)batch_len;
                bi.base_offset = (int64_t)be_u64(p);
                window.skipped(attrs, count);
            } else if (framed && crc_failed(p, 12u + (uint32_t)batch_len, b, bi.partition)) {
                bi.flags = LOGB_SKIP_CRC;
                bi.len = 12u + (uint32_t)batch_len;
                bi.base_offset = (int64_t)be_u64(p);
            } else if (framed && count >= 0 &&   // (for a compressed batch the bound is checked against its uncompressed size later)
                       (codec != 0 || (uint64_t)count * 7u + (uint64_t)(LOG_HEADER_BYTES - 12) <= (uint64_t)batch_len)) {
                bi.len = 12u + (uint32_t)batch_len;
                bi.base_offset = (int64_t)be_u64(p);
                bi.base_ts = (int64_t)be_u64(p + 27);
                bi.max_ts = (int64_t)be_u64(p + 35);
                bi.log_append_time = (attrs >> 3) & 1u;
                if (attrs & 0x20u) bi.flags = LOGB_SKIP_CONTROL;
                else if (codec <= 4) {
                    bi.flags = log_codec_flag(codec);
                    bi.records = count;
                    if (Window::on && verdict == LOG_WIN_CUT && count > 0) window.cut(b);
                } else bi.flags = LOGB_COMPRESSED;   // unassigned codes
            }
        }
        if (bi.flags & (LOGB_BAD | LOGB_COMPRESSED | LOGB_CODECS)) atomicOr(&word->flags, bi.flags);
        else if (bi.flags == LOGB_OK) atomicMax(&word->longest, bi.len);
        info[b] = bi;
        rec_count[b + 1] = (uint64_t)bi.records;
    }
    if (blockIdx.x == 0 && threadIdx.x == 0) rec_count[0] = 0;
}

// The records section in[0, n) of a gzip, LZ4 or Snappy batch (flags: its LOGB_GZIP / LOGB_LZ4 / LOGB_SNAPPY): its uncompressed
// size (thread per batch), then its copy to out + at, out_cap bytes (the whole warp; work: the warp's inflate tables).  The
// copy kernel passes its image and the header's length as `at`: with the offset added in each branch it compiles to the same
// code as with the walks called in place.  zstd batches have a size kernel and a copy instance of their own (zstd_walk).
__host__ __device__ __forceinline__ LzWalk section_size(uint32_t flags, const uint8_t *in, uint32_t n) {
    return flags == LOGB_GZIP  ? gzip_size(in, n)
           : flags == LOGB_LZ4 ? lz4_frame_walk<false>(in, n, nullptr, 0, 0)
                               : snappy_walk<false>(in, n, nullptr, 0, 0);
}
__host__ __device__ __forceinline__ LzWalk section_copy(uint32_t flags, const uint8_t *in, uint32_t n, uint8_t *out, uint32_t at,
                                                        uint64_t out_cap, InfWork &work, int lane) {
    return flags == LOGB_LZ4    ? lz4_frame_walk<true>(in, n, out + at, out_cap, lane)
           : flags == LOGB_GZIP ? gzip_walk(in, n, out + at, out_cap, work, lane)
                                : snappy_walk<true>(in, n, out + at, out_cap, lane);
}

// the scratch bytes a batch's uncompressed image (header + records, rounded up to 16) needs, or 0 (and LOGB_BAD) when the walk
// failed or recordsCount is implausible for the uncompressed size (it sizes the output columns: 7 bytes per record at least)
__device__ __forceinline__ uint64_t unc_need(const LogBatchInfo &bi, const LzWalk &w, uint32_t *error_flags) {
    if (!w.ok || w.out_len > 0x7fffff00ull || (uint64_t)bi.records * 7u > w.out_len) {
        atomicOr(error_flags, (uint32_t)LOGB_BAD);
        return 0;
    }
    return ((uint64_t)LOG_HEADER_BYTES + w.out_len + 15u) & ~15ull;
}

// thread per batch: the uncompressed size of a compressed batch's records section → slot[b + 1] = bytes its uncompressed
// image needs in the scratch buffer (0 for batches that are not compressed; zstd batches are log_zstd_size_kernel's)
__global__ void log_unc_size_kernel(const uint8_t *bytes, const LogBatchInfo *info, int64_t nbatches, uint64_t *slot, uint32_t *error_flags) {
    for (int64_t b = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; b < nbatches; b += (int64_t)gridDim.x * blockDim.x) {
        const LogBatchInfo bi = info[b];
        uint64_t need = 0;
        if ((bi.flags & LOGB_CODECS) && bi.flags != LOGB_ZSTD)
            need = unc_need(bi, section_size(bi.flags, bytes + bi.off + LOG_HEADER_BYTES, bi.len - LOG_HEADER_BYTES), error_flags);
        slot[b + 1] = need;
    }
    if (blockIdx.x == 0 && threadIdx.x == 0) slot[0] = 0;
}

// warp per zstd batch, after log_unc_size_kernel (launched only when the header pass saw zstd): slot[b + 1] as above.  A frame
// without Frame_Content_Size is sized by decoding its sequences, which needs the FSE tables: they are in shared memory here,
// not in the local memory of a thread-per-batch kernel (CUDA reserves a kernel's local memory for every resident thread).
__global__ void __launch_bounds__(128) log_zstd_size_kernel(const uint8_t *bytes, const LogBatchInfo *info, int64_t nbatches, uint64_t *slot,
                                                            uint32_t *error_flags) {
    __shared__ ZstdWork zstd_work[4];
    const int lane = threadIdx.x & 31;
    const int64_t gw = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5, gs = ((int64_t)gridDim.x * blockDim.x) >> 5;
    for (int64_t b = gw; b < nbatches; b += gs) {
        const LogBatchInfo bi = info[b];
        if (bi.flags != LOGB_ZSTD) continue;
        const LzWalk w = zstd_walk<false>(bytes + bi.off + LOG_HEADER_BYTES, bi.len - LOG_HEADER_BYTES, nullptr, nullptr, 0, zstd_work[threadIdx.x >> 5], lane);
        if (lane == 0) slot[b + 1] = unc_need(bi, w, error_flags);
    }
}

// warp per compressed batch: header copy (compression bits cleared, batchLength = uncompressed) + decompressed records into
// scratch + slot[b]; the batch's info then points there (offsets are relative to `bytes`: the scratch buffer is simply
// another place in the same address space) and it is an ordinary LOGB_OK batch for the decoder.
// ZSTD = false: the gzip, LZ4 and Snappy batches; ZSTD = true: the zstd batches, launched only when there are some.  Two
// instances rather than one branch, because the zstd walk's tables (41 KiB of shared memory for 4 warps) and registers would
// lower the occupancy of the other codecs' decompression too.  lit_scratch (zstd only): the Huffman-decoded literals of a
// block go to the same offset in this buffer as the block's output has in `scratch`.
template <bool ZSTD>
__global__ void __launch_bounds__(128) log_decompress_kernel(const uint8_t *bytes, LogBatchInfo *info, int64_t nbatches, const uint64_t *slot,
                                                             uint8_t *scratch, uint8_t *lit_scratch, uint32_t *error_flags) {
    using Work = typename std::conditional<ZSTD, ZstdWork, InfWork>::type;   // the warp's entropy tables
    __shared__ Work work[4];
    const int lane = threadIdx.x & 31;
    const int64_t gw = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5, gs = ((int64_t)gridDim.x * blockDim.x) >> 5;
    for (int64_t b = gw; b < nbatches; b += gs) {
        const LogBatchInfo bi = info[b];
        if (!(bi.flags & LOGB_CODECS) || (bi.flags == LOGB_ZSTD) != ZSTD) continue;
        const uint64_t need = slot[b + 1] - slot[b];
        uint8_t *dst = scratch + slot[b];
        if (need < (uint64_t)LOG_HEADER_BYTES) {             // the size pass rejected it
            if (lane == 0) info[b].flags = LOGB_BAD;
            continue;
        }
        const uint8_t *src = bytes + bi.off;
        const uint64_t cap = need - LOG_HEADER_BYTES;
        const uint8_t *in = src + LOG_HEADER_BYTES;
        const uint32_t n = bi.len - LOG_HEADER_BYTES;
        LzWalk w;
        if constexpr (ZSTD) w = zstd_walk<true>(in, n, dst + LOG_HEADER_BYTES, lit_scratch + slot[b] + LOG_HEADER_BYTES, cap, work[threadIdx.x >> 5], lane);
        else w = section_copy(bi.flags, in, n, dst, LOG_HEADER_BYTES, cap, work[threadIdx.x >> 5], lane);
        for (int i = lane; i < LOG_HEADER_BYTES; i += 32) dst[i] = src[i];
        __syncwarp();
        if (lane == 0) {
            const uint32_t ulen = LOG_HEADER_BYTES + (uint32_t)w.out_len, bl = ulen - 12u;
            dst[8] = (uint8_t)(bl >> 24); dst[9] = (uint8_t)(bl >> 16); dst[10] = (uint8_t)(bl >> 8); dst[11] = (uint8_t)bl;   // batchLength
            dst[22] &= 0xf8;                                  // attributes: no compression
            if (!w.ok) atomicOr(error_flags, (uint32_t)LOGB_BAD);
            info[b].off = (uint64_t)(dst - bytes);            // relative to `bytes` (may wrap: one address space)
            info[b].len = ulen;
            info[b].flags = w.ok ? LOGB_OK : LOGB_BAD;
        }
    }
}

// One WARP per batch.  Records are length-prefixed, so finding where record i starts is a serial chain: lane 0 hops through
// 32 record-length varints at a time and publishes the 32 start positions; then the 32 lanes parse their records in
// parallel and write the columns coalesced.
// STAGED: the whole batch (what a producer's batch.size bounds: 16 KiB by default) is first brought global→shared by ONE
// bulk async copy per batch per warp (cp.async.bulk → UBLKCP, mbarrier completion), so every hop of the chain is a
// shared-memory read instead of a dependent global access to a new line (the chain of hops is the decoder's
// critical path).  Batches that do not fit the stage, or whose 16-byte-aligned copy would run past the readable
// bytes, are read in place.
// Output: the header columns and, per record, the position of its key bytes in the segment buffer (key_src, only when the
// keys will be hashed) — the keys themselves are packed afterwards by log_gather_keys_kernel, without a second walk.
constexpr int LOG_DECODE_THREADS = 128;
constexpr int LOG_WARP_HEADER = 192;   // per warp: mbarrier (8 B) + 33 record starts (132 B), padded

// WINDOW (launched only for a call with cut batches, kta_logoffsets.cuh): a record of a cut batch (baseOffset below its
// partition's log start offset window[p].x, -1 = none) whose own offset lies below that start is walked but not written;
// every other batch keeps all its records, whatever their offset deltas.  The kept records of a batch are written densely
// from rec_base[b]: each one's rank is the popcount of the lanes below it that keep theirs, plus the records the batch kept
// in the rounds before (rec_base already counts only the kept records, log_cut_count_kernel).  Without WINDOW, window and
// num_partitions are not read.
template <bool STAGED, bool WINDOW>
__global__ void __launch_bounds__(LOG_DECODE_THREADS) log_decode_kernel(
    const uint8_t *bytes, uint64_t readable /* bytes that may be read from `bytes` */, const LogBatchInfo *info, int64_t nbatches,
    const uint64_t *rec_base, int32_t *partition, int64_t *ts_ms, int32_t *key_len, int32_t *value_len, uint64_t *key_src,
    uint32_t stage_bytes /* per warp, multiple of 16 */, uint32_t *error_flags, const longlong2 *window, int32_t num_partitions) {
    extern __shared__ __align__(128) unsigned char log_smem[];
    const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5;
    const unsigned full = 0xffffffffu;
    unsigned char *wsm = log_smem + (size_t)wib * (LOG_WARP_HEADER + (STAGED ? stage_bytes : 0u));
    uint32_t *s_start = reinterpret_cast<uint32_t *>(wsm + 16);
    unsigned char *stage = wsm + LOG_WARP_HEADER;
    const uint32_t bar = (uint32_t)__cvta_generic_to_shared(wsm);
    uint32_t phase = 0;
    if (STAGED && lane == 0) {
        asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(bar));
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncwarp();
    const int64_t gw = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5, gs = ((int64_t)gridDim.x * blockDim.x) >> 5;
    for (int64_t b = gw; b < nbatches; b += gs) {
        const LogBatchInfo bi = info[b];
        if (bi.flags == LOGB_OK && bi.records > 0) {
            const uint8_t *base = bytes + bi.off;
            if (STAGED) {
                const uint32_t lead = (uint32_t)(bi.off & 15u), span = (lead + bi.len + 15u) & ~15u;
                if (span <= stage_bytes && (bi.off - lead) + span <= readable) {
                    if (lane == 0) {
                        asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(span) : "memory");
                        asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                                     ::"r"((uint32_t)__cvta_generic_to_shared(stage)), "l"(bytes + (bi.off - lead)), "r"(span), "r"(bar)
                                     : "memory");
                    }
                    asm volatile(
                        "{\n\t.reg .pred p;\n\t"
                        "LOGW_%=:\n\t"
                        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
                        "@p bra LOGD_%=;\n\t"
                        "bra LOGW_%=;\n\t"
                        "LOGD_%=:\n\t}" ::"r"(bar), "r"(phase) : "memory");
                    phase ^= 1u;
                    base = stage + lead;
                }
            }
            const uint8_t *end = base + bi.len;
            uint32_t pos = LOG_HEADER_BYTES;          // offset of the next record inside the batch
            const uint64_t r0 = rec_base[b];
            bool ok = true;
            int64_t lo = -1;      // WINDOW: the partition's log start offset
            uint64_t room = 0;    // WINDOW: the records rec_base gives the batch
            uint32_t kept = 0;    // WINDOW: the records it kept in the rounds before
            if constexpr (WINDOW) {
                lo = (uint32_t)bi.partition < (uint32_t)num_partitions ? window[bi.partition].x : -1;
                room = rec_base[b + 1] - r0;
            }
            for (int32_t i0 = 0; i0 < bi.records && ok; i0 += 32) {
                const int cnt = min(32, bi.records - i0);
                if (lane == 0) {
                    for (int j = 0; j < cnt; j++) {
                        s_start[j] = pos;
                        uint64_t u;
                        const int n = uvarint_g(base + pos, end, u);
                        const int64_t rec_len = unzigzag(u);
                        if (n <= 0 || rec_len < 0 || (uint64_t)pos + n + rec_len > bi.len) { ok = false; break; }
                        pos += (uint32_t)n + (uint32_t)rec_len;
                    }
                    s_start[32] = ok ? pos : 0xffffffffu;
                }
                __syncwarp();
                pos = s_start[32];
                ok = pos != 0xffffffffu;
                if (!ok) break;
                int64_t klen = -1, vlen = -1, ts_delta = 0, off_delta = 0;
                uint32_t key_at = 0;
                bool lane_ok = true;
                if (lane < cnt) {
                    const uint8_t *q = base + s_start[lane];
                    const uint8_t *rec_end = lane + 1 < cnt ? base + s_start[lane + 1] : base + pos;
                    uint64_t u;
                    int n = uvarint_g(q, rec_end, u); q += n;            // record length (validated by lane 0)
                    q += 1;                                               // record attributes (unused)
                    n = uvarint_g(q, rec_end, u); lane_ok = lane_ok && n > 0; q += n;
                    ts_delta = unzigzag(u);
                    n = uvarint_g(q, rec_end, u); lane_ok = lane_ok && n > 0; q += n;
                    off_delta = unzigzag(u);
                    n = uvarint_g(q, rec_end, u); lane_ok = lane_ok && n > 0; q += n;
                    klen = unzigzag(u);
                    lane_ok = lane_ok && klen >= -1 && klen <= 0x7fffffff && (klen <= 0 || q + klen <= rec_end);
                    key_at = (uint32_t)(q - base);
                    if (lane_ok && klen > 0) q += klen;
                    n = lane_ok ? uvarint_g(q, rec_end, u) : 0; lane_ok = lane_ok && n > 0; q += n;
                    vlen = unzigzag(u);
                    lane_ok = lane_ok && vlen >= -1 && vlen <= 0x7fffffff && (vlen <= 0 || q + vlen <= rec_end);
                }
                __syncwarp();   // every lane has read its start before lane 0 overwrites them
                ok = __all_sync(full, lane_ok);
                if (!ok) break;
                if constexpr (WINDOW) {
                    // only a cut batch (baseOffset < S, the header pass's test) drops records, as the count pass counts
                    const bool below = lo >= 0 && bi.base_offset < lo && (int64_t)((uint64_t)bi.base_offset + (uint64_t)off_delta) < lo;
                    const unsigned mask = __ballot_sync(full, lane < cnt && !below);
                    const uint32_t rank = kept + (uint32_t)__popc(mask & ((1u << lane) - 1u));
                    kept += (uint32_t)__popc(mask);
                    if (lane < cnt && !below && rank < room) {
                        const uint64_t r = r0 + rank;
                        partition[r] = bi.partition;
                        ts_ms[r] = bi.log_append_time ? bi.max_ts : bi.base_ts + ts_delta;
                        key_len[r] = (int32_t)klen;
                        value_len[r] = (int32_t)vlen;
                        if (key_src) key_src[r] = bi.off + key_at;
                    }
                } else if (lane < cnt) {
                    const uint64_t r = r0 + (uint64_t)i0 + lane;
                    partition[r] = bi.partition;
                    ts_ms[r] = bi.log_append_time ? bi.max_ts : bi.base_ts + ts_delta;
                    key_len[r] = (int32_t)klen;
                    value_len[r] = (int32_t)vlen;
                    if (key_src) key_src[r] = bi.off + key_at;
                }
            }
            if (!ok && lane == 0) atomicOr(error_flags, (uint32_t)LOGB_BAD);
            __syncwarp();   // the stage is free for the next batch's copy
        }
    }
}

// Packs the key bytes in record order (what the scan kernel hashes): one warp per 128-record tile, a lane owns four
// consecutive records; byte offsets from the tile base (key_tile_base, derived from key_len beforehand) plus an in-tile scan.
__global__ void __launch_bounds__(256) log_gather_keys_kernel(const uint8_t *bytes, const uint64_t *key_src, const int32_t *key_len,
                                                              int64_t n, const uint64_t *tile_base, uint8_t *key_out) {
    const int lane = threadIdx.x & 31;
    const int64_t ntiles = (n + 127) / 128;
    const int64_t gw = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5, gs = ((int64_t)gridDim.x * blockDim.x) >> 5;
    for (int64_t tile = gw; tile < ntiles; tile += gs) {
        int32_t len[4];
        uint64_t src[4];
        uint32_t mine = 0;
#pragma unroll
        for (int k = 0; k < 4; k++) {
            const int64_t r = tile * 128 + (int64_t)lane * 4 + k;
            len[k] = r < n ? key_len[r] : -1;
            src[k] = len[k] > 0 ? key_src[r] : 0;
            mine += len[k] > 0 ? (uint32_t)len[k] : 0u;
        }
        uint32_t inc = mine;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
            const uint32_t t = __shfl_up_sync(0xffffffffu, inc, d);
            if (lane >= d) inc += t;
        }
        uint8_t *o = key_out + tile_base[tile] + (inc - mine);
#pragma unroll
        for (int k = 0; k < 4; k++) {
            if (len[k] > 0) {
                const uint8_t *sp = bytes + src[k];
                int j = 0;
                if ((reinterpret_cast<uintptr_t>(o) & 3u) == 0) {
                    // word-aligned destination (always, for keys whose lengths are multiples of 4: ids, hashes, UUIDs): whole
                    // words, from aligned source words put together with a funnel shift
                    const uintptr_t a = reinterpret_cast<uintptr_t>(sp);
                    const uint32_t *wp = reinterpret_cast<const uint32_t *>(a & ~(uintptr_t)3);
                    const uint32_t sh = (uint32_t)(a & 3u) * 8u;
                    const int nw = len[k] >> 2;
                    uint32_t *ow = reinterpret_cast<uint32_t *>(o);
                    if (sh == 0) {
                        for (int w = 0; w < nw; w++) ow[w] = __ldg(wp + w);
                        j = nw * 4;
                    } else {
                        // the aligned word behind the last full one may reach past the key (and past the buffer): the last
                        // word is left to the byte loop
                        uint32_t lo = __ldg(wp);
                        for (int w = 0; w + 1 < nw; w++) {
                            const uint32_t hi = __ldg(wp + w + 1);
                            ow[w] = __funnelshift_r(lo, hi, sh);
                            lo = hi;
                        }
                        j = nw > 0 ? (nw - 1) * 4 : 0;
                    }
                }
                for (; j < len[k]; j++) o[j] = __ldg(sp + j);
                o += len[k];
            }
        }
    }
}

}  // namespace kta
