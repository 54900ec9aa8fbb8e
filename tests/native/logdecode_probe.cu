// TEST INFRASTRUCTURE: the record stage of the RecordBatch decoder on the GPU, with its output made visible.  It launches what
// scan_log_batches (csrc/kta_api.cu) launches up to the scan — the header pass, its record-count scan, the size and copy passes
// when there are compressed batches, the record decode, the key-length tile bases and the key gather — through the same launch
// functions (log_launch_header in csrc/kta_logoffsets.cuh, the others in csrc/kta_logdecode_launch.cuh), and writes out every
// decoded column, so that tests/test_logdecode_records.py can compare them record by record with the records a case was built
// from.
// With a window table (tests/test_logoffsets_records.py) it launches what scan_log_batches launches for a handle with offset
// windows (kta_logoffsets.cuh): the header pass with the window and the record-count scan, the size and copy passes, the count
// pass and its correction of the scan when the header pass cut batches, the record decode (given the window table, so the
// window decode runs, only when some batch is cut), the tile bases and the gather.
// stdin, per case (little-endian): u32 nbytes, the bytes; u32 nbatches, u64 batch offsets; u32 with_partitions, then i32 per
// batch partitions when it is 1 (else every batch is partition 0); u32 slack: the bytes behind nbytes that may be read (0 as
// the device entry points pass, 48 as kta_push_log_segments_host passes); u32 nwin, then nwin x (i64 S, i64 H): the window
// table of partitions [0, nwin) (-1: that side unbounded; nwin 0: no windows, the plain header pass and decode).  The device
// buffer is exactly nbytes + slack long.
// stdout: u32 SM count and u32 opt-in shared memory per block of the device; then per case: u32 header flags, u32 longest
// batch, u32 size-pass flags, u32 decode flags, u64 records (with windows: after the count pass), u32 staged, u32 stage,
// u32 grid, u32 ran (the decode was launched: the header and size passes accepted the call and the header pass found
// records); with windows then u32 header words [6..9] (cut batches, batches not served, their records as u64), u32 windowed
// (the window decode ran), u32 flags of every batch after the header pass, u64 drop[nbatches + 1] (the count pass's drops,
// scanned: [b] = the records dropped before batch b; zeros when it did not run); when ran: per record i32 partition, i64
// ts_ms, i32 key_len, i32 value_len (column by column); when ran, the decode flags are 0 and there are records: u64 tile
// base[ntiles + 1], then the key buffer (tile base[ntiles] packed key bytes and the 64 bytes behind them).
// The decoded columns and the key buffer are filled with 0xA5 first: an entry the decoder does not write shows up (its
// key_len is then negative, so the gather skips it).
#include "../../kafka_topic_analyzer_b200/csrc/kta_logoffsets.cuh"
#include "probe.h"

using namespace kta;

int main() {
    int sm_count = 0, optin = 0;
    CK(cudaDeviceGetAttribute(&sm_count, cudaDevAttrMultiProcessorCount, 0));
    CK(cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, 0));
    // as create_impl does: the staged decoder may take the device's opt-in shared memory
    CK(cudaFuncSetAttribute(log_decode_kernel<true, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, optin));
    CK(cudaFuncSetAttribute(log_decode_kernel<true, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, optin));
    const uint32_t device[2] = {(uint32_t)sm_count, (uint32_t)optin};
    put(device, 8);
    cudaStream_t s;
    CK(cudaStreamCreate(&s));
    uint32_t n;
    while (fread(&n, 4, 1, stdin) == 1) {
        std::vector<uint8_t> seg(n);
        get(seg.data(), n);
        uint32_t nb32 = 0, with_part = 0, slack = 0;
        get(&nb32, 4);
        const int64_t nb = nb32;
        std::vector<uint64_t> offs((size_t)nb);
        get(offs.data(), (size_t)nb * 8);
        get(&with_part, 4);
        std::vector<int32_t> parts(with_part ? (size_t)nb : 0);
        get(parts.data(), parts.size() * 4);
        get(&slack, 4);
        uint32_t nwin = 0;
        get(&nwin, 4);
        std::vector<longlong2> win(nwin);
        get(win.data(), (size_t)nwin * sizeof(longlong2));
        const uint64_t readable = (uint64_t)n + slack;

        uint8_t *d_bytes = dev_alloc<uint8_t>(readable, 0, s);
        uint64_t *d_off = dev_alloc<uint64_t>((size_t)nb, 0, s), *d_cnt = dev_alloc<uint64_t>((size_t)nb + 1, 0, s);
        int32_t *d_part = with_part ? dev_alloc<int32_t>((size_t)nb, 0, s) : nullptr;
        LogBatchInfo *d_info = dev_alloc<LogBatchInfo>((size_t)nb, 0, s);
        LogHeaderWord *d_word = dev_alloc<LogHeaderWord>(1, 0, s);
        uint32_t *d_flags = &d_word->flags;
        longlong2 *d_win = nwin ? dev_alloc<longlong2>(nwin, 0, s) : nullptr;
        uint32_t *d_cut = nwin ? dev_alloc<uint32_t>((size_t)nb, 0, s) : nullptr;
        uint64_t *d_drop = nwin ? dev_alloc<uint64_t>((size_t)nb + 1, 0, s) : nullptr;
        CK(cudaMemcpyAsync(d_bytes, seg.data(), n, cudaMemcpyHostToDevice, s));
        CK(cudaMemcpyAsync(d_off, offs.data(), (size_t)nb * 8, cudaMemcpyHostToDevice, s));
        if (d_part) CK(cudaMemcpyAsync(d_part, parts.data(), (size_t)nb * 4, cudaMemcpyHostToDevice, s));
        if (d_win) CK(cudaMemcpyAsync(d_win, win.data(), (size_t)nwin * sizeof(longlong2), cudaMemcpyHostToDevice, s));
        if (nb) {
            CK(log_launch_header(d_bytes, (int64_t)n, d_off, nb, 0, d_part, d_info, d_cnt, d_word, nullptr, nullptr, d_win, (int32_t)nwin,
                                 d_cut, sm_count, s));
            tile_base_scan_kernel<<<1, 1024, 0, s>>>(d_cnt, nb);
            CK(cudaGetLastError());
        }
        LogHeaderWord hdr{};
        uint32_t unc_err = 0, dec_err = 0;
        uint64_t nrec = 0;
        std::vector<LogBatchInfo> info(nwin ? (size_t)nb : 0);
        CK(cudaMemcpyAsync(&hdr, d_word, sizeof hdr, cudaMemcpyDeviceToHost, s));
        CK(cudaMemcpyAsync(&nrec, d_cnt + nb, 8, cudaMemcpyDeviceToHost, s));
        if (nwin && nb) CK(cudaMemcpyAsync(info.data(), d_info, (size_t)nb * sizeof(LogBatchInfo), cudaMemcpyDeviceToHost, s));
        CK(cudaStreamSynchronize(s));
        const int64_t ncut = nwin ? hdr.cut : 0;
        bool ran = nb > 0 && !(hdr.flags & (LOGB_BAD | LOGB_COMPRESSED)) && nrec > 0;
        uint8_t *d_unc = nullptr, *d_lit = nullptr;
        uint64_t *d_slot = nullptr;
        const uint32_t codecs = hdr.flags & LOGB_CODECS;
        if (ran && codecs) {
            const bool zstd = (codecs & LOGB_ZSTD) != 0;
            d_slot = dev_alloc<uint64_t>((size_t)nb + 2, 0, s);
            CK(cudaMemsetAsync(d_flags, 0, 4, s));
            CK(log_launch_size_pass(d_bytes, d_info, nb, d_slot, d_flags, zstd, sm_count, s));
            uint64_t unc_total = 0;
            CK(cudaMemcpyAsync(&unc_total, d_slot + nb, 8, cudaMemcpyDeviceToHost, s));
            CK(cudaMemcpyAsync(&unc_err, d_flags, 4, cudaMemcpyDeviceToHost, s));
            CK(cudaStreamSynchronize(s));
            if (unc_err) ran = false;
            else {
                d_unc = dev_alloc<uint8_t>(unc_total + 64, 0, s);
                if (zstd) d_lit = dev_alloc<uint8_t>(unc_total + 64, 0, s);
                CK(log_launch_copy_pass(d_bytes, d_info, nb, d_slot, d_unc, d_lit, d_flags, codecs, sm_count, s));
            }
        }
        if (ran && ncut) {   // as log_cut_count: the records kept, after the count pass's correction of the scan
            CK(log_launch_cut_count(d_bytes, d_info, nb, d_cut, ncut, d_win, (int32_t)nwin, d_cnt, d_drop, sm_count, s));
            CK(cudaMemcpyAsync(&nrec, d_cnt + nb, 8, cudaMemcpyDeviceToHost, s));
            CK(cudaStreamSynchronize(s));
        }
        const LogDecodeShape shape = log_decode_shape(hdr.longest, nb, sm_count, (size_t)optin);
        int32_t *d_dpart = nullptr, *d_klen = nullptr, *d_vlen = nullptr;
        int64_t *d_ts = nullptr;
        uint64_t *d_ksrc = nullptr, *d_tb = nullptr;
        uint8_t *d_keys = nullptr;
        const int64_t ntiles = ((int64_t)nrec + TILE - 1) / TILE;
        uint64_t nkey = 0;
        if (ran) {
            d_dpart = dev_alloc<int32_t>(nrec, 0xA5, s);
            d_ts = dev_alloc<int64_t>(nrec, 0xA5, s);
            d_klen = dev_alloc<int32_t>(nrec, 0xA5, s);
            d_vlen = dev_alloc<int32_t>(nrec, 0xA5, s);
            d_ksrc = dev_alloc<uint64_t>(nrec, 0xA5, s);
            d_tb = dev_alloc<uint64_t>((size_t)ntiles + 1, 0xA5, s);
            // (*d_flags is 0 here, or holds what the copy pass found, as in scan_log_batches)
            // (a call whose cut batches keep no record is still decoded, so damage in them refuses it, as in scan_log_batches)
            CK(log_launch_decode(shape, d_bytes, readable, d_info, nb, d_cnt, d_dpart, d_ts, d_klen, d_vlen, d_ksrc, d_flags,
                                 ncut ? d_win : nullptr, (int32_t)nwin, s));
            if (nrec) {
                CK(log_launch_tile_base(d_klen, (int64_t)nrec, d_tb, sm_count, s));
                CK(cudaMemcpyAsync(&nkey, d_tb + ntiles, 8, cudaMemcpyDeviceToHost, s));
            }
            CK(cudaMemcpyAsync(&dec_err, d_flags, 4, cudaMemcpyDeviceToHost, s));
            CK(cudaStreamSynchronize(s));
            if (!dec_err && nrec) {
                d_keys = dev_alloc<uint8_t>(nkey + 64, 0xA5, s);
                CK(log_launch_gather_keys(d_bytes, d_ksrc, d_klen, (int64_t)nrec, d_tb, d_keys, sm_count, s));
            }
            CK(cudaStreamSynchronize(s));
        }
        const uint32_t staged = shape.staged ? 1u : 0u, stage = shape.stage, grid = (uint32_t)shape.grid, ran32 = ran ? 1u : 0u;
        put(&hdr.flags, 4);
        put(&hdr.longest, 4);
        put(&unc_err, 4);
        put(&dec_err, 4);
        put(&nrec, 8);
        put(&staged, 4);
        put(&stage, 4);
        put(&grid, 4);
        put(&ran32, 4);
        if (nwin) {
            const uint32_t windowed = ran && ncut ? 1u : 0u;
            put(&hdr.cut, 4);
            put(&hdr.not_served, 4);
            put(&hdr.not_served_records, 8);
            put(&windowed, 4);
            for (const LogBatchInfo &bi : info) put(&bi.flags, 4);
            put_dev(d_drop, (size_t)nb + 1);
        }
        if (ran) {
            put_dev(d_dpart, nrec);
            put_dev(d_ts, nrec);
            put_dev(d_klen, nrec);
            put_dev(d_vlen, nrec);
            if (!dec_err && nrec) {
                put_dev(d_tb, (size_t)ntiles + 1);
                put_dev(d_keys, nkey + 64);
            }
        }
        for (void *p : {(void *)d_bytes, (void *)d_off, (void *)d_cnt, (void *)d_part, (void *)d_info, (void *)d_word, (void *)d_unc,
                        (void *)d_lit, (void *)d_slot, (void *)d_dpart, (void *)d_ts, (void *)d_klen, (void *)d_vlen, (void *)d_ksrc,
                        (void *)d_tb, (void *)d_keys, (void *)d_win, (void *)d_cut, (void *)d_drop})
            if (p) CK(cudaFree(p));
    }
    CK(cudaStreamDestroy(s));
    fflush(stdout);
    return 0;
}
