// kta_logscan.cuh — the host steps of the log entry points (Kafka RecordBatch v2 segments → SoA; kernels in kta_logdecode.cuh,
// kta_logcrc.cuh, kta_logoffsets.cuh and kta_logtxn.cuh).  LogScan owns everything only the log path uses; each step takes it
// and a LogEnv, never the handle.  scan_log_batches (kta_api.cu) calls the steps in order, between the handle's own work
// (the ring flush before, the scan after), and tests/native/log_probe.cu calls the same steps in the same order, so the
// tests that check the log path record by record run the library's sequencing.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include <algorithm>
#include <vector>

#include "kta_host.cuh"
#include "kta_kernels.cuh"
#include "kta_logcrc.cuh"
#include "kta_logdecode.cuh"
#include "kta_logdecode_launch.cuh"
#include "kta_logoffsets.cuh"
#include "kta_logtxn.cuh"

using namespace kta;

// read_committed isolation of the log entry points (kta_logtxn.cuh); allocated only on a read_committed handle
struct TxnState {
    DevBuf<TxnKey> d_keys, d_sorted;                 // classify's keys / sorted by (partition, producerId, batch)
    DevBuf<uint8_t> d_kind;                          // per batch: TxnKind of transactional data batches and markers
    DevBuf<uint8_t> d_res;                           // per sorted key: next marker within its resolve tile
    DevBuf<uint8_t> d_tile;                          // tile heads, then the carries behind each tile
    DevBuf<uint8_t> d_sort_tmp;
    DevBuf<uint32_t> d_word;                         // [0] keys classified, [1] TxnErr bits
    DevBuf<unsigned long long> d_stats;              // this call: aborted batches, aborted records, undecided records
    std::vector<TxnRange> ranges;                    // registered aborted ranges, sorted and merged; mirrored in d_ranges
    DevBuf<TxnRange> d_ranges;
    uint64_t totals[3] = {0, 0, 0};                  // the stats of every successful call since create / reset
};

// check.crcs of the log entry points (kta_logcrc.cuh): the switch, the passes' buffers, and what successful calls found
struct CrcState {
    bool on = false;
    int span_grid = 0;                               // test hook: the span pass's blocks (0: log_crc_span_grid)
    DevBuf<uint64_t> d_spans;                        // per batch: spans of its CRC region, then their inclusive scan
    DevBuf<uint32_t> d_acc;                          // per batch: the xor of its spans' shares of the register
    DevBuf<LogCrcFail> d_fails;                      // the call's failures, in the order the header pass met them
    DevBuf<LogCrcTables> d_tables;                   // built on the first call with the switch on
    uint64_t totals[3] = {0, 0, 0};                  // checked batches, failed batches, failed bytes
    std::vector<kta_log_crc_failure> kept;           // the first KTA_LOG_CRC_KEEP failures
};

// The log start offset and high watermark of each partition (kta_log_set_offsets, kta_logoffsets.cuh): the table, the
// passes' buffers, and what successful calls left out
struct OffsetState {
    std::vector<longlong2> win;                      // per partition: x log start offset, y high watermark (-1: unbounded);
                                                     // empty until a window is set
    int64_t set = 0;                                 // partitions with a bound: the window passes run only while > 0
    bool dirty = false;                              // win changed since it was last copied to d_win
    DevBuf<longlong2> d_win;                         // win on the device
    DevBuf<uint32_t> d_cut;                          // the call's cut batches (served, with records below the start)
    DevBuf<uint64_t> d_drop;                         // per batch: records the count pass drops, then their scan
    uint64_t totals[2] = {0, 0};                     // batches not served, records left out
};

// State of the log entry points (Kafka RecordBatch v2 segments → SoA → scan), reused from call to call
struct LogScan {
    DevBuf<uint8_t> bytes;                   // segments staged from the host (kta_push_log_segments_host)
    DevBuf<uint64_t> off;                    // their batch offsets
    DevBuf<int32_t> part;                    // and each batch's partition
    DevBuf<LogBatchInfo> info;               // per batch, from the header pass
    DevBuf<uint64_t> cnt;                    // records per batch, then their inclusive scan
    DevBuf<LogHeaderWord> err;               // the header pass's error word; its flags, the later passes' flag word
    DevBuf<int32_t> dec_part, dec_klen, dec_vlen;   // the decoded columns
    DevBuf<int64_t> dec_ts;
    DevBuf<uint64_t> dec_ksrc;               // per decoded record: where its key bytes lie in the segment buffer
    DevBuf<uint8_t> dec_keys;                // the keys gathered in record order
    DevBuf<uint8_t> unc;                     // uncompressed images of compressed batches
    DevBuf<uint8_t> unc_lit;                 // zstd: Huffman-decoded literals, at the offsets of unc
    DevBuf<uint64_t> unc_slot;               // per compressed batch: offset of its image in unc
    bool read_committed = false;
    TxnState txn;
    CrcState crc;
    OffsetState offsets;
};

// What a step needs of its caller: the stream and the device, the partitions of the window table, the buffer the decoded
// records' key tile bases go to (the handle's scratch for them), and the launch counter kta_stats reports.
struct LogEnv {
    cudaStream_t stream;
    int sm_count;
    size_t smem_optin;
    int32_t num_partitions;
    DevBuf<uint64_t> &tile_base;
    uint64_t &launches;
};

// What the header pass (and read_committed's passes and the CRC check) found in one call's batches
struct LogHeaders {
    uint64_t nrec = 0;                               // records in all
    LogHeaderWord word{};                            // the header pass's error word
    bool txn_ran = false;                            // read_committed's passes ran (the call has transactional batches)
    unsigned long long txn_stats[3] = {0, 0, 0};     // this call's aborted batches, aborted records, undecided records
    std::vector<kta_log_crc_failure> crc_fails;      // check.crcs: this call's failures, in batch order, as many as are kept
};

// ------------------------------------------------------------------------------------------------
// what create and the setters do to LogScan
// ------------------------------------------------------------------------------------------------
// read_committed's words, and the staged record decoder's shared memory: it stages a batch of up to 48 KiB per warp
// (log_decode); attributes belong to the device
static int log_scan_create(LogScan &L, bool read_committed, size_t smem_optin) {
    L.read_committed = read_committed;
    int rc;
    if (read_committed && ((rc = L.txn.d_word.alloc(2)) || (rc = L.txn.d_stats.alloc(3)))) return rc;
    CU(cudaFuncSetAttribute(log_decode_kernel<true, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_optin));
    CU(cudaFuncSetAttribute(log_decode_kernel<true, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_optin));
    return KTA_OK;
}

// windows: partition's [log_start_offset, high_watermark) (checked by the caller); the table goes to the device on the next call
static void log_set_window(LogScan &L, int32_t num_partitions, int32_t partition, int64_t log_start_offset, int64_t high_watermark) {
    OffsetState &o = L.offsets;
    if (o.win.empty()) o.win.assign((size_t)num_partitions, make_longlong2(-1, -1));
    longlong2 &w = o.win[(size_t)partition];
    o.set -= (w.x != -1 || w.y != -1);
    w = make_longlong2(log_start_offset, high_watermark);
    o.set += (w.x != -1 || w.y != -1);
    o.dirty = true;
}

// read_committed: checked ranges join the registered ones, sorted by (partition, producerId, firstOffset) with overlapping
// ranges of one producer merged (the apply pass's binary search then has one candidate per offset), and go to the device
static int log_add_txn_ranges(LogScan &L, const LogEnv &e, const std::vector<TxnRange> &add) {
    TxnState &t = L.txn;
    std::vector<TxnRange> &v = t.ranges;
    v.insert(v.end(), add.begin(), add.end());
    std::sort(v.begin(), v.end(), [](const TxnRange &a, const TxnRange &b) {
        return a.part != b.part ? a.part < b.part : a.pid != b.pid ? a.pid < b.pid : a.first < b.first;
    });
    size_t out = 0;
    for (size_t i = 0; i < v.size(); i++) {
        if (out && v[out - 1].part == v[i].part && v[out - 1].pid == v[i].pid && v[i].first <= v[out - 1].last)
            v[out - 1].last = std::max(v[out - 1].last, v[i].last);
        else v[out++] = v[i];
    }
    v.resize(out);
    int rc;
    if ((rc = t.d_ranges.grow(e.stream, (int64_t)v.size()))) return rc;
    CU(cudaStreamSynchronize(e.stream));   // no queued pass reads the ranges while they are replaced
    CU(cudaMemcpyAsync(t.d_ranges, v.data(), v.size() * sizeof(TxnRange), cudaMemcpyHostToDevice, e.stream));
    CU(cudaStreamSynchronize(e.stream));
    return KTA_OK;
}

// ------------------------------------------------------------------------------------------------
// the steps of one call, in the order scan_log_batches runs them
// ------------------------------------------------------------------------------------------------

// the key_tile_base column of n records' key lengths, into e.tile_base ([ntiles] = the key bytes in all)
static int log_tile_base(const LogEnv &e, const int32_t *d_klen, int64_t n) {
    const int64_t ntiles = (n + TILE - 1) / TILE;
    int rc;
    if ((rc = e.tile_base.grow(e.stream, ntiles + 1))) return rc;
    CU(log_launch_tile_base(d_klen, n, e.tile_base, e.sm_count, e.stream));
    e.launches += 2;
    return KTA_OK;
}

// read_committed: the passes of kta_logtxn.cuh over the batches log_header_kernel has read, before the record count is
// scanned.  Classify always; sort, resolve, carry and apply only when the call has transactional batches.  One host round
// trip (the classify count).  *ran: the apply pass was launched, so its error word and counters are to be read back.
static int txn_passes(LogScan &L, const LogEnv &e, int32_t partition, const uint8_t *dev_bytes, int64_t nbatches, bool *ran) {
    TxnState &t = L.txn;
    cudaStream_t s = e.stream;
    *ran = false;
    if (nbatches > (int64_t)UINT32_MAX) return fail(KTA_ERR_INVALID, "%lld batches in one read_committed call: split them", (long long)nbatches);
    int rc;
    if ((rc = t.d_keys.grow(s, nbatches)) || (rc = t.d_sorted.grow(s, nbatches)) || (rc = t.d_kind.grow(s, nbatches)) ||
        (rc = t.d_res.grow(s, nbatches)))
        return rc;
    CU(cudaMemsetAsync(t.d_word, 0, 8, s));
    CU(log_launch_txn_classify(dev_bytes, L.info, nbatches, t.d_keys, t.d_kind, t.d_word, e.sm_count, s));
    e.launches++;
    uint32_t w[3] = {0, 0, 0};   // keys, TxnErr bits, header flags
    CU(cudaMemcpyAsync(w, t.d_word, 8, cudaMemcpyDeviceToHost, s));
    CU(cudaMemcpyAsync(w + 2, &L.err.get()->flags, 4, cudaMemcpyDeviceToHost, s));
    CU(cudaStreamSynchronize(s));
    if (w[2] & (LOGB_BAD | LOGB_COMPRESSED)) return KTA_OK;   // the call is refused for its headers (log_headers says so)
    if (w[1] & TXN_ERR_MARKER)
        return fail(KTA_ERR_INVALID, "unreadable transaction marker in partition %d (control batch compressed, without a record, "
                    "truncated, or with a key that is not version 0 | type)", partition);
    const int64_t m = w[0];
    if (m == 0) return KTA_OK;
    const int64_t nranges = (int64_t)t.ranges.size();
    size_t tmp = 0;   // first the sort's scratch size, then the passes
    CU(log_launch_txn_passes(t.d_keys, t.d_sorted, m, t.d_kind, L.info, t.d_res, nullptr, nullptr, tmp, t.d_ranges, nranges, L.cnt,
                             t.d_word, t.d_stats, e.sm_count, s));
    if ((rc = t.d_sort_tmp.grow(s, (int64_t)tmp)) || (rc = t.d_tile.grow(s, 2 * log_txn_tiles(m)))) return rc;
    tmp = (size_t)t.d_sort_tmp.cap;
    CU(log_launch_txn_passes(t.d_keys, t.d_sorted, m, t.d_kind, L.info, t.d_res, t.d_tile, t.d_sort_tmp.get(), tmp, t.d_ranges, nranges,
                             L.cnt, t.d_word, t.d_stats, e.sm_count, s));
    e.launches += 4;   // (the sort counted as one)
    *ran = true;
    return KTA_OK;
}

// windows: the table the window passes read (on the device once log_offsets_upload ran), or null while the handle has none
static const longlong2 *log_window_table(const LogScan &L) {
    return L.offsets.set > 0 ? L.offsets.d_win.get() : nullptr;
}

// check.crcs: the span pass's blocks for a call of nbytes bytes in nbatches batches
static int log_crc_grid(const CrcState &c, int64_t nbytes, int64_t nbatches, int sm_count) {
    return c.span_grid ? c.span_grid : log_crc_span_grid(nbytes, nbatches, sm_count);
}

// check.crcs: the passes of kta_logcrc.cuh that precede the header pass (span counts, their scan, the spans' CRCs), through
// log_launch_crc_spans.  No host round trip; the span kernel's grid is bounded by the call's bytes.  Batches that are not
// served are not checked (the window table goes to the device first, log_offsets_upload).
static int log_crc_spans(LogScan &L, const LogEnv &e, int32_t partition, const int32_t *dev_batch_partition, const uint8_t *dev_bytes,
                         int64_t len, const uint64_t *dev_batch_off, int64_t nbatches) {
    CrcState &c = L.crc;
    cudaStream_t s = e.stream;
    int rc;
    if (!c.d_tables) {
        LogCrcTables t;
        log_crc_tables_host(t);
        if ((rc = c.d_tables.alloc(1))) return rc;
        CU(cudaMemcpyAsync(c.d_tables, &t, sizeof t, cudaMemcpyHostToDevice, s));
        CU(cudaStreamSynchronize(s));   // `t` lives on this stack frame
        CU(cudaFuncSetAttribute(log_crc_span_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)LOG_CRC_SMEM));
    }
    if ((rc = c.d_spans.grow(s, nbatches + 1)) || (rc = c.d_acc.grow(s, nbatches)) || (rc = c.d_fails.grow(s, nbatches))) return rc;
    CU(log_launch_crc_spans(dev_bytes, len, dev_batch_off, nbatches, partition, dev_batch_partition, log_window_table(L), e.num_partitions,
                            c.d_tables, c.d_spans, c.d_acc, log_crc_grid(c, len, nbatches, e.sm_count), e.sm_count, s));
    e.launches += 3;
    return KTA_OK;
}

// windows: the window table goes to the device when it changed since the last call (two host synchronisations, only then)
static int log_offsets_upload(LogScan &L, const LogEnv &e) {
    OffsetState &o = L.offsets;
    if (!o.dirty) return KTA_OK;
    int rc;
    if (!o.d_win && (rc = o.d_win.alloc((int64_t)o.win.size()))) return rc;
    CU(cudaStreamSynchronize(e.stream));   // no queued pass reads the table while it is replaced
    CU(cudaMemcpyAsync(o.d_win, o.win.data(), o.win.size() * sizeof(longlong2), cudaMemcpyHostToDevice, e.stream));
    CU(cudaStreamSynchronize(e.stream));
    o.dirty = false;
    return KTA_OK;
}

// The header pass, read_committed's passes and the scan of the record counts.  One host round trip (two under
// read_committed); refuses the call for its headers and for the order of a producer's batches.  With check.crcs the CRC
// passes come first and the failures are counted in the same round trip; only a call with failures makes one more, for
// their list.  With windows the header pass also skips the batches that are not served and lists the cut ones; their
// counts come back in the same round trip.
static int log_headers(LogScan &L, const LogEnv &e, int32_t partition, const int32_t *dev_batch_partition, const uint8_t *dev_bytes,
                       int64_t len, const uint64_t *dev_batch_off, int64_t nbatches, LogHeaders &out) {
    cudaStream_t s = e.stream;
    int rc;
    if ((rc = L.info.grow(s, nbatches + 1)) || (rc = L.cnt.grow(s, nbatches + 1))) return rc;
    if (!L.err && (rc = L.err.alloc(1))) return rc;
    const bool crc = L.crc.on;
    if (L.offsets.set > 0 && ((rc = log_offsets_upload(L, e)) || (rc = L.offsets.d_cut.grow(s, nbatches)))) return rc;
    if (crc && (rc = log_crc_spans(L, e, partition, dev_batch_partition, dev_bytes, len, dev_batch_off, nbatches))) return rc;
    CU(cudaMemsetAsync(L.err, 0, sizeof(LogHeaderWord), s));
    CU(log_launch_header(dev_bytes, len, dev_batch_off, nbatches, partition, dev_batch_partition, L.info, L.cnt, L.err,
                         crc ? L.crc.d_acc.get() : nullptr, L.crc.d_fails, log_window_table(L), e.num_partitions, L.offsets.d_cut,
                         e.sm_count, s));
    if (L.read_committed && (rc = txn_passes(L, e, partition, dev_bytes, nbatches, &out.txn_ran))) return rc;
    tile_base_scan_kernel<<<1, 1024, 0, s>>>(L.cnt, nbatches);   // inclusive scan of [1..nbatches] in place
    CU(cudaGetLastError());
    e.launches += 2;
    uint32_t txn_word[2] = {0, 0};
    CU(cudaMemcpyAsync(&out.nrec, L.cnt + nbatches, 8, cudaMemcpyDeviceToHost, s));
    CU(cudaMemcpyAsync(&out.word, L.err, sizeof(LogHeaderWord), cudaMemcpyDeviceToHost, s));
    if (out.txn_ran) {
        CU(cudaMemcpyAsync(txn_word, L.txn.d_word, 8, cudaMemcpyDeviceToHost, s));
        CU(cudaMemcpyAsync(out.txn_stats, L.txn.d_stats, 24, cudaMemcpyDeviceToHost, s));
    }
    CU(cudaStreamSynchronize(s));
    if (out.word.flags & LOGB_COMPRESSED)
        return fail(KTA_ERR_INVALID, "unknown compression codec (attributes bits 0-2 = 5..7) in partition %d", partition);
    if (out.word.flags & LOGB_BAD) return fail(KTA_ERR_INVALID, "malformed record batch header in partition %d", partition);
    if (txn_word[1] & TXN_ERR_ORDER)
        return fail(KTA_ERR_INVALID, "the batches of one producer in partition %d are not in increasing baseOffset order", partition);
    // the failures to keep: the first ones in batch order, as many as the handle's list still has room for
    const uint32_t nfail = out.word.crc_failed;
    const size_t room = KTA_LOG_CRC_KEEP - L.crc.kept.size();
    if (nfail && room) {
        std::vector<LogCrcFail> f(nfail);
        CU(cudaMemcpyAsync(f.data(), L.crc.d_fails, (size_t)nfail * sizeof(LogCrcFail), cudaMemcpyDeviceToHost, s));
        CU(cudaStreamSynchronize(s));
        std::sort(f.begin(), f.end(), [](const LogCrcFail &a, const LogCrcFail &b) { return a.batch < b.batch; });
        for (size_t i = 0; i < std::min<size_t>(room, f.size()); i++)
            out.crc_fails.push_back(kta_log_crc_failure{f[i].partition, f[i].batch_bytes, f[i].base_offset, f[i].stored, f[i].computed});
    }
    return KTA_OK;
}

// Compressed batches (codecs: the LOGB_CODECS bits the header pass saw), first step: the size pass.  One host round trip:
// *unc_total = the scratch bytes the images need, *bad = the size pass's flags (nonzero: some batch is malformed).
static int log_unc_size(LogScan &L, const LogEnv &e, const uint8_t *dev_bytes, int64_t nbatches, uint32_t codecs, uint64_t *unc_total,
                        uint32_t *bad) {
    cudaStream_t s = e.stream;
    int rc;
    if ((rc = L.unc_slot.grow(s, nbatches + 2))) return rc;
    uint32_t *flags = &L.err.get()->flags;
    CU(cudaMemsetAsync(flags, 0, 4, s));
    const bool zstd = (codecs & LOGB_ZSTD) != 0;
    CU(log_launch_size_pass(dev_bytes, L.info, nbatches, L.unc_slot, flags, zstd, e.sm_count, s));
    e.launches += zstd ? 3 : 2;
    CU(cudaMemcpyAsync(unc_total, L.unc_slot + nbatches, 8, cudaMemcpyDeviceToHost, s));
    CU(cudaMemcpyAsync(bad, flags, 4, cudaMemcpyDeviceToHost, s));
    CU(cudaStreamSynchronize(s));
    return KTA_OK;
}

// Second step: scratch allocation and decompression.  Afterwards the compressed batches are ordinary batches that happen to
// lie in the scratch buffer.
static int log_unc_copy(LogScan &L, const LogEnv &e, const uint8_t *dev_bytes, int64_t nbatches, uint32_t codecs, uint64_t unc_total) {
    cudaStream_t s = e.stream;
    const bool zstd = (codecs & LOGB_ZSTD) != 0;
    int rc;
    if ((rc = L.unc.grow(s, (int64_t)unc_total + 64))) return rc;
    // zstd's literal buffer has the size of the scratch buffer (a block's literals go at its output's offset); it is
    // only allocated once zstd batches are seen
    if (zstd && (rc = L.unc_lit.grow(s, (int64_t)unc_total + 64))) return rc;
    CU(log_launch_copy_pass(dev_bytes, L.info, nbatches, L.unc_slot, L.unc, L.unc_lit, &L.err.get()->flags, codecs, e.sm_count, s));
    e.launches += ((codecs & ~(uint32_t)LOGB_ZSTD) ? 1 : 0) + (zstd ? 1 : 0);
    return KTA_OK;
}

// windows: the call's cut batches (ncut of them, after the decompression) are walked and their records below the log
// start offset counted; the record-count scan is corrected for them.  One host round trip: *nrec = the records kept,
// *dropped = the records dropped.
static int log_cut_count(LogScan &L, const LogEnv &e, const uint8_t *dev_bytes, int64_t nbatches, int64_t ncut, uint64_t *nrec,
                         uint64_t *dropped) {
    cudaStream_t s = e.stream;
    int rc;
    if ((rc = L.offsets.d_drop.grow(s, nbatches + 1))) return rc;
    CU(log_launch_cut_count(dev_bytes, L.info, nbatches, L.offsets.d_cut, ncut, log_window_table(L), e.num_partitions, L.cnt,
                            L.offsets.d_drop, e.sm_count, s));
    e.launches += 3;
    CU(cudaMemcpyAsync(nrec, L.cnt + nbatches, 8, cudaMemcpyDeviceToHost, s));
    CU(cudaMemcpyAsync(dropped, L.offsets.d_drop + nbatches, 8, cudaMemcpyDeviceToHost, s));
    CU(cudaStreamSynchronize(s));
    return KTA_OK;
}

// The records of every batch into the decoded columns, which b then names; with keys, where each record's key bytes lie.
// One warp per batch; the batch is staged in shared memory when the longest one fits a stage of <= 48 KiB.  A call with
// cut batches (ncut > 0) runs the window decode, which leaves out their records below the log start offset.
static int log_decode(LogScan &L, const LogEnv &e, const uint8_t *dev_bytes, int64_t readable, int64_t nbatches, uint64_t nrec,
                      uint32_t longest, bool keys, int64_t ncut, kta_batch &b) {
    cudaStream_t s = e.stream;
    if ((int64_t)nrec >= ((int64_t)1 << 31) - 2) return fail(KTA_ERR_INVALID, "%llu records in one call: split the segments", (unsigned long long)nrec);
    int rc;
    if ((rc = L.dec_part.grow(s, (int64_t)nrec)) || (rc = L.dec_klen.grow(s, (int64_t)nrec)) || (rc = L.dec_vlen.grow(s, (int64_t)nrec)) ||
        (rc = L.dec_ts.grow(s, (int64_t)nrec)) || (rc = L.dec_ksrc.grow(s, (int64_t)nrec)))
        return rc;
    const LogDecodeShape shape = log_decode_shape(longest, nbatches, e.sm_count, e.smem_optin);
    CU(log_launch_decode(shape, dev_bytes, (uint64_t)readable, L.info, nbatches, L.cnt, L.dec_part, L.dec_ts, L.dec_klen, L.dec_vlen,
                         keys ? L.dec_ksrc.get() : nullptr, &L.err.get()->flags, ncut ? log_window_table(L) : nullptr, e.num_partitions, s));
    e.launches++;
    b = kta_batch{};
    b.n = (int64_t)nrec;
    b.seq_base = KTA_SEQ_AUTO;
    b.partition = L.dec_part;
    b.ts_ms = L.dec_ts;
    b.key_len = L.dec_klen;
    b.value_len = L.dec_vlen;
    return KTA_OK;
}

// Reads the decode's error word back (one host round trip).  With keys, first packs them in record order into b's key
// columns: tile bases from the key_len column, then one gather pass (no second walk of the log).
static int log_gather_keys(LogScan &L, const LogEnv &e, int32_t partition, const uint8_t *dev_bytes, bool keys, kta_batch &b) {
    cudaStream_t s = e.stream;
    int rc;
    uint32_t flags = 0;
    uint64_t nkey = 0;
    const int64_t ntiles = (b.n + TILE - 1) / TILE;
    if (keys) {
        if ((rc = log_tile_base(e, b.key_len, b.n))) return rc;
        CU(cudaMemcpyAsync(&nkey, e.tile_base + ntiles, 8, cudaMemcpyDeviceToHost, s));
    }
    CU(cudaMemcpyAsync(&flags, &L.err.get()->flags, 4, cudaMemcpyDeviceToHost, s));
    CU(cudaStreamSynchronize(s));
    if (flags) return fail(KTA_ERR_INVALID, "malformed record inside a batch of partition %d", partition);
    if (!keys) return KTA_OK;
    if ((rc = L.dec_keys.grow(s, (int64_t)nkey + 64))) return rc;
    CU(log_launch_gather_keys(dev_bytes, L.dec_ksrc, L.dec_klen, b.n, e.tile_base, L.dec_keys, e.sm_count, s));
    e.launches++;
    b.key_bytes = L.dec_keys;
    b.key_bytes_len = (int64_t)nkey;
    b.key_tile_base = e.tile_base;
    return KTA_OK;
}
