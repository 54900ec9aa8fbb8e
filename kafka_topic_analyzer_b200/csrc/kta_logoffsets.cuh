// kta_logoffsets.cuh — the offsets a consumer fetches, for the RecordBatch v2 decoder (kta_logdecode.cuh): per partition p a
// window [S, H) of log start offset and high watermark (kta_log_set_offsets; -1 = no bound on that side).
//
// A consumer that starts at S (auto.offset.reset=earliest) and reads up to H sees exactly this:
//   1. the batches the broker serves: last = baseOffset + lastOffsetDelta (the stored field, which can lie past the last
//      record of a compacted batch) with S <= last < H.  The broker places a fetch from S at the first batch whose last
//      offset is >= S, and bounds it at H by the position of the batch that holds H, so that batch goes whole.  A batch
//      that is not served is LOGB_SKIP_OFFSET: not CRC-checked, decompressed, decoded or classified, and no error.
//   2. the records librdkafka keeps: inside a served batch, a record with baseOffset + offsetDelta < S is dropped (the
//      v2 reader skips messages older than the fetch offset).  Only a served batch with baseOffset < S can hold such
//      records in a log a broker writes; the header pass lists these CUT batches, and records are dropped from cut batches
//      only (the count pass and the window decode both apply this rule).  A served batch with baseOffset >= S keeps every
//      record even when a forged negative offsetDelta puts one below S: its rows then depend on its own bytes and its
//      partition's window alone, not on whether another batch of the call is cut.
//
// The passes, on a handle with at least one window (a handle without one launches none of this):
//   header   (log_header_kernel<C, true>)  the header pass with LogOffsetWindow: one 16-byte load of [S, H) per batch; not
//            served → LOGB_SKIP_OFFSET, counted in the header word's not_served and not_served_records; cut data batches
//            with records → cut list, counted in its cut
//   crc      (log_crc_count_kernel<true>)  check.crcs: batches that are not served get no spans
//   count    (log_cut_count_kernel, warp per cut batch, after decompression)  walks the batch's records as the decode does
//            and stores how many it drops at drop[b + 1]; then the drops are scanned (tile_base_scan_kernel) and taken off
//            the record-count scan (log_cut_fix_kernel), so rec_base counts kept records only
//   decode   (log_decode_kernel<S, true>, only when the call has cut batches)  writes the kept records densely
// The header pass and the CRC span count are one kernel each, with check.crcs and the window as template switches; their
// launches (log_launch_header, log_launch_crc_spans) are at the end of this file.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "kta_logcrc.cuh"
#include "kta_logdecode.cuh"
#include "kta_logdecode_launch.cuh"

namespace kta {

// [S, H) of a partition inside [0, num_partitions) (-1: that side unbounded); any other partition has no window
__device__ __forceinline__ longlong2 log_window(const longlong2 *window, int32_t num_partitions, int32_t p) {
    return (uint32_t)p < (uint32_t)num_partitions ? window[p] : make_longlong2(-1, -1);
}

// The window question of the header pass (and of the CRC span count) for the framed batch at p
struct LogOffsetWindow {
    static constexpr bool on = true;
    const longlong2 *window;
    int32_t num_partitions;
    uint32_t *cut_list;        // the cut batches, in the order the pass met them (capacity: the call's batches)
    LogHeaderWord *word;
    __device__ __forceinline__ int test(const uint8_t *p, int32_t partition) const {
        const longlong2 w = log_window(window, num_partitions, partition);
        const int64_t base = (int64_t)be_u64(p);
        const int64_t last = (int64_t)((uint64_t)base + (uint64_t)(int64_t)(int32_t)be_u32(p + 23));   // + lastOffsetDelta
        if ((w.x >= 0 && last < w.x) || (w.y >= 0 && last >= w.y)) return LOG_WIN_SKIP;
        return w.x >= 0 && base < w.x ? LOG_WIN_CUT : LOG_WIN_SERVED;
    }
    // a batch that is not served: its records count as left out when it is a data batch
    __device__ __forceinline__ void skipped(uint32_t attrs, int32_t count) const {
        atomicAdd(&word->not_served, 1u);
        if (!(attrs & 0x20u) && count > 0) atomicAdd(&word->not_served_records, (unsigned long long)count);
    }
    __device__ __forceinline__ void cut(int64_t b) const { cut_list[atomicAdd(&word->cut, 1u)] = (uint32_t)b; }
};

// the header pass's questions with a switch on (the CRC check, the window) or off (NoCrcCheck, NoWindow)
template <bool CRC>
__device__ __forceinline__ auto log_crc_check(const uint32_t *acc, LogCrcFail *fails, LogHeaderWord *word) {
    if constexpr (CRC) return CrcAccCheck{acc, fails, word};
    else return NoCrcCheck{};
}
template <bool WIN>
__device__ __forceinline__ auto log_offset_window(const longlong2 *window, int32_t num_partitions, uint32_t *cut_list, LogHeaderWord *word) {
    if constexpr (WIN) return LogOffsetWindow{window, num_partitions, cut_list, word};
    else return NoWindow{};
}

// The header pass, with check.crcs (CRC: acc, the span pass's registers; fails, room for the call's batches) and with a
// window table (WIN: window of num_partitions; cut_list, room for the call's batches); a switch that is off leaves its
// parameters unread.
template <bool CRC, bool WIN>
__global__ void log_header_kernel(const uint8_t *bytes, int64_t nbytes, const uint64_t *batch_off, int64_t nbatches, int32_t partition,
                                  const int32_t *batch_partition /* per batch, or NULL = `partition` */, LogBatchInfo *info,
                                  uint64_t *rec_count /*[nbatches+1], [b+1]*/, LogHeaderWord *word, const uint32_t *acc,
                                  LogCrcFail *fails, const longlong2 *window, int32_t num_partitions, uint32_t *cut_list) {
    log_header_pass(bytes, nbytes, batch_off, nbatches, partition, batch_partition, info, rec_count, word,
                    log_crc_check<CRC>(acc, fails, word), log_offset_window<WIN>(window, num_partitions, cut_list, word));
}

// check.crcs: the span count (kta_logcrc.cuh), with a window table (WIN) for batches that are not served
template <bool WIN>
__global__ void log_crc_count_kernel(const uint8_t *bytes, int64_t nbytes, const uint64_t *batch_off, int64_t nbatches, uint64_t *spans,
                                     uint32_t *acc, int32_t partition, const int32_t *batch_partition, const longlong2 *window,
                                     int32_t num_partitions) {
    log_crc_count_pass(bytes, nbytes, batch_off, nbatches, spans, acc, partition, batch_partition,
                       log_offset_window<WIN>(window, num_partitions, nullptr, nullptr));
}

// Warp per cut batch (cut[0, ncut)), after the decompression, so a compressed batch is walked in its uncompressed image.
// The records are walked as log_decode_kernel walks them (lane 0 hops the record lengths 32 at a time, each lane reads
// its record's deltas) and those with offset < S are counted: drop[b + 1] = their number (drop: zeroed, nbatches + 1).
// A batch that the walk cannot read keeps drop 0; the decode refuses the call for it.  Aborted batches (LOGB_SKIP_ABORTED)
// and batches that failed to decompress are not walked.
__global__ void __launch_bounds__(128) log_cut_count_kernel(const uint8_t *bytes, const LogBatchInfo *info, const uint32_t *cut, int64_t ncut,
                                                            const longlong2 *window, int32_t num_partitions, uint64_t *drop) {
    __shared__ uint32_t starts[4][33];
    const int lane = threadIdx.x & 31;
    uint32_t *s_start = starts[threadIdx.x >> 5];
    const unsigned full = 0xffffffffu;
    const int64_t gw = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5, gs = ((int64_t)gridDim.x * blockDim.x) >> 5;
    for (int64_t k = gw; k < ncut; k += gs) {
        const uint32_t b = cut[k];
        const LogBatchInfo bi = info[b];
        if (bi.flags != LOGB_OK || bi.records <= 0) continue;
        const int64_t lo = log_window(window, num_partitions, bi.partition).x;
        const uint8_t *base = bytes + bi.off, *end = base + bi.len;
        uint32_t pos = LOG_HEADER_BYTES, kept = 0;
        bool ok = true;
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
            bool lane_ok = true, keep = false;
            if (lane < cnt) {
                const uint8_t *q = base + s_start[lane];
                const uint8_t *rec_end = lane + 1 < cnt ? base + s_start[lane + 1] : base + pos;
                uint64_t u;
                int n = uvarint_g(q, rec_end, u); q += n;            // record length (validated by lane 0)
                q += 1;                                               // record attributes
                n = uvarint_g(q, rec_end, u); lane_ok = n > 0; q += n;   // timestampDelta
                n = uvarint_g(q, rec_end, u); lane_ok = lane_ok && n > 0;
                keep = (int64_t)((uint64_t)bi.base_offset + (uint64_t)unzigzag(u)) >= lo;
            }
            __syncwarp();   // every lane has read its start before lane 0 overwrites them
            ok = __all_sync(full, lane_ok);
            kept += (uint32_t)__popc(__ballot_sync(full, keep && lane_ok));
        }
        if (lane == 0 && ok) drop[b + 1] = (uint64_t)bi.records - kept;
        __syncwarp();
    }
}

// rec_count[b] -= drop[b] for b in [0, nbatches]: the record-count scan without the dropped records (drop: scanned)
__global__ void log_cut_fix_kernel(uint64_t *rec_count, const uint64_t *drop, int64_t nbatches) {
    for (int64_t b = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; b <= nbatches; b += (int64_t)gridDim.x * blockDim.x)
        rec_count[b] -= drop[b];
}

// the count pass and the scan correction of a call with ncut cut batches (drop: nbatches + 1 words, zeroed here).  After
// it rec_count[nbatches] is the call's record count and drop[nbatches] the records dropped.
inline cudaError_t log_launch_cut_count(const uint8_t *bytes, const LogBatchInfo *info, int64_t nbatches, const uint32_t *cut, int64_t ncut,
                                        const longlong2 *window, int32_t num_partitions, uint64_t *rec_count, uint64_t *drop, int sm_count,
                                        cudaStream_t s) {
    cudaError_t e = cudaMemsetAsync(drop, 0, (size_t)(nbatches + 1) * sizeof(uint64_t), s);
    if (e != cudaSuccess) return e;
    log_cut_count_kernel<<<log_warp_grid(ncut, sm_count), 128, 0, s>>>(bytes, info, cut, ncut, window, num_partitions, drop);
    tile_base_scan_kernel<<<1, 1024, 0, s>>>(drop, nbatches);
    log_cut_fix_kernel<<<log_thread_grid(nbatches + 1, sm_count), 128, 0, s>>>(rec_count, drop, nbatches);
    return cudaGetLastError();
}

// check.crcs: the span pass's grid.  A call has at most nbytes / S + nbatches spans, one per thread at least, so a small
// call gets a small grid; at most one block per SM (the pass's 128 KiB of tables leave room for one).
inline int log_crc_span_grid(int64_t nbytes, int64_t nbatches, int sm_count) {
    const int64_t max_spans = nbytes / LOG_CRC_SPAN + nbatches;
    return (int)std::max<int64_t>(1, std::min<int64_t>((max_spans + LOG_CRC_THREADS - 1) / LOG_CRC_THREADS, sm_count));
}

// check.crcs: the passes of kta_logcrc.cuh that precede the header pass: the span counts (with a window table, batches that
// are not served get none), their scan into spans[0, nbatches], and the span pass on `grid` blocks (log_crc_span_grid; the
// span pass needs LOG_CRC_SMEM of dynamic shared memory allowed).  No host round trip: the span pass reads the total from
// the scan.
inline cudaError_t log_launch_crc_spans(const uint8_t *bytes, int64_t nbytes, const uint64_t *batch_off, int64_t nbatches, int32_t partition,
                                        const int32_t *batch_partition, const longlong2 *window, int32_t num_partitions,
                                        const LogCrcTables *tables, uint64_t *spans, uint32_t *acc, int grid, int sm_count, cudaStream_t s) {
    const auto count = window ? log_crc_count_kernel<true> : log_crc_count_kernel<false>;
    count<<<log_thread_grid(nbatches, sm_count), 128, 0, s>>>(bytes, nbytes, batch_off, nbatches, spans, acc, partition, batch_partition,
                                                              window, num_partitions);
    tile_base_scan_kernel<<<1, 1024, 0, s>>>(spans, nbatches);
    log_crc_span_kernel<<<grid, LOG_CRC_THREADS, LOG_CRC_SMEM, s>>>(bytes, batch_off, nbatches, spans, tables, acc);
    return cudaGetLastError();
}

// The header pass of a call: with check.crcs when acc is given (the span pass's registers; fails: room for the call's
// batches) and with windows when the window table is (cut_list: room for the call's batches), either, both or neither.
// word: zeroed by the caller.
inline cudaError_t log_launch_header(const uint8_t *bytes, int64_t nbytes, const uint64_t *batch_off, int64_t nbatches, int32_t partition,
                                     const int32_t *batch_partition, LogBatchInfo *info, uint64_t *rec_count, LogHeaderWord *word,
                                     const uint32_t *acc, LogCrcFail *fails, const longlong2 *window, int32_t num_partitions,
                                     uint32_t *cut_list, int sm_count, cudaStream_t s) {
    const auto header = acc ? (window ? log_header_kernel<true, true> : log_header_kernel<true, false>)
                            : (window ? log_header_kernel<false, true> : log_header_kernel<false, false>);
    header<<<log_thread_grid(nbatches, sm_count), 128, 0, s>>>(bytes, nbytes, batch_off, nbatches, partition, batch_partition, info,
                                                               rec_count, word, acc, fails, window, num_partitions, cut_list);
    return cudaGetLastError();
}

}  // namespace kta
