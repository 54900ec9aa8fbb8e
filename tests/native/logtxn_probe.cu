// TEST INFRASTRUCTURE: the read_committed passes of the RecordBatch decoder (csrc/kta_logtxn.cuh) on the GPU, with everything
// they produce made visible.  It launches what log_headers (csrc/kta_api.cu) launches for a read_committed handle —
// the header pass, the classify pass, the host round trip for the key count, the sort, resolve, carry and apply passes, then
// the record-count scan — through the same launch functions (log_launch_header, log_launch_txn_classify,
// log_launch_txn_passes), and writes out every array, so that tests/test_logtxn_passes.py can compare them key by key with a
// plain restatement of the rule.
// stdin, per case (little-endian): u32 nbytes, the bytes; u32 nbatches, u64 batch offsets, i32 batch partitions; u32 nranges,
// then nranges TxnRange images (i32 partition, u32 0, u64 producerId, i64 first, i64 last), sorted by (partition, producerId,
// first) and disjoint within a (partition, producerId): the table as the handle keeps it (the host's sort and merge are not run
// here).
// stdout: u32 SM count of the device; then per case: u32 header flags, u32 keys classified (word[0]), u32 TxnErr bits (word[1],
// after the passes), u32 ran (the sort, resolve, carry and apply passes were launched: the headers and markers were accepted
// and there are keys; m = keys when ran, else 0), u64 stats[3], u64 records after the record-count scan; u8 kind[nbatches];
// u32 flags[nbatches], i32 records[nbatches], u64 rec_count[nbatches + 1] as the apply pass leaves it (before the scan:
// [b + 1] = the rows of batch b); when ran: TxnKey sorted[m] (u64 producerId, u32 partition, u32 batch), u8 res[m], u8
// tile_head[ntiles], u8 carry[ntiles].
// kind, res, tile_head and carry are filled with 0xA5 first: an entry the passes do not write shows up.
#include "../../kafka_topic_analyzer_b200/csrc/kta_logoffsets.cuh"
#include "../../kafka_topic_analyzer_b200/csrc/kta_logtxn.cuh"
#include "probe.h"

using namespace kta;

int main() {
    int sm_count = 0;
    CK(cudaDeviceGetAttribute(&sm_count, cudaDevAttrMultiProcessorCount, 0));
    const uint32_t device = (uint32_t)sm_count;
    put(&device, 4);
    cudaStream_t s;
    CK(cudaStreamCreate(&s));
    uint32_t n;
    while (fread(&n, 4, 1, stdin) == 1) {
        std::vector<uint8_t> seg(n);
        get(seg.data(), n);
        uint32_t nb32 = 0, nranges = 0;
        get(&nb32, 4);
        const int64_t nb = nb32;
        std::vector<uint64_t> offs((size_t)nb);
        get(offs.data(), (size_t)nb * 8);
        std::vector<int32_t> parts((size_t)nb);
        get(parts.data(), (size_t)nb * 4);
        get(&nranges, 4);
        std::vector<TxnRange> ranges(nranges);
        get(ranges.data(), (size_t)nranges * sizeof(TxnRange));

        uint8_t *d_bytes = dev_alloc<uint8_t>(n, 0, s);
        uint64_t *d_off = dev_alloc<uint64_t>((size_t)nb, 0, s), *d_cnt = dev_alloc<uint64_t>((size_t)nb + 1, 0, s);
        int32_t *d_part = dev_alloc<int32_t>((size_t)nb, 0, s);
        LogBatchInfo *d_info = dev_alloc<LogBatchInfo>((size_t)nb + 1, 0, s);
        LogHeaderWord *d_hdr = dev_alloc<LogHeaderWord>(1, 0, s);
        uint32_t *d_word = dev_alloc<uint32_t>(2, 0, s);
        TxnKey *d_keys = dev_alloc<TxnKey>((size_t)nb, 0, s), *d_sorted = dev_alloc<TxnKey>((size_t)nb, 0, s);
        uint8_t *d_kind = dev_alloc<uint8_t>((size_t)nb, 0xA5, s), *d_res = dev_alloc<uint8_t>((size_t)nb, 0xA5, s);
        unsigned long long *d_stats = dev_alloc<unsigned long long>(3, 0, s);
        TxnRange *d_ranges = nranges ? dev_alloc<TxnRange>(nranges, 0, s) : nullptr;
        CK(cudaMemcpyAsync(d_bytes, seg.data(), n, cudaMemcpyHostToDevice, s));
        CK(cudaMemcpyAsync(d_off, offs.data(), (size_t)nb * 8, cudaMemcpyHostToDevice, s));
        CK(cudaMemcpyAsync(d_part, parts.data(), (size_t)nb * 4, cudaMemcpyHostToDevice, s));
        if (nranges) CK(cudaMemcpyAsync(d_ranges, ranges.data(), (size_t)nranges * sizeof(TxnRange), cudaMemcpyHostToDevice, s));
        uint32_t w[3] = {0, 0, 0};   // keys, TxnErr bits, header flags (as txn_passes reads them back)
        if (nb) {
            CK(log_launch_header(d_bytes, (int64_t)n, d_off, nb, 0, d_part, d_info, d_cnt, d_hdr, nullptr, nullptr, nullptr, 0, nullptr,
                                 sm_count, s));
            CK(log_launch_txn_classify(d_bytes, d_info, nb, d_keys, d_kind, d_word, sm_count, s));
        }
        CK(cudaMemcpyAsync(w, d_word, 8, cudaMemcpyDeviceToHost, s));
        CK(cudaMemcpyAsync(w + 2, &d_hdr->flags, 4, cudaMemcpyDeviceToHost, s));
        CK(cudaStreamSynchronize(s));
        const bool ran = !(w[2] & (LOGB_BAD | LOGB_COMPRESSED)) && !(w[1] & TXN_ERR_MARKER) && w[0] > 0;
        const int64_t m = ran ? w[0] : 0, tiles = log_txn_tiles(m);
        uint8_t *d_tile = nullptr, *d_tmp = nullptr;
        if (ran) {
            size_t tmp = 0;
            CK(log_launch_txn_passes(d_keys, d_sorted, m, d_kind, d_info, d_res, nullptr, nullptr, tmp, d_ranges, nranges, d_cnt, d_word,
                                     d_stats, sm_count, s));
            d_tmp = dev_alloc<uint8_t>(tmp, 0, s);
            d_tile = dev_alloc<uint8_t>((size_t)(2 * tiles), 0xA5, s);
            CK(log_launch_txn_passes(d_keys, d_sorted, m, d_kind, d_info, d_res, d_tile, d_tmp, tmp, d_ranges, nranges, d_cnt, d_word,
                                     d_stats, sm_count, s));
            CK(cudaMemcpyAsync(w, d_word, 8, cudaMemcpyDeviceToHost, s));
            CK(cudaStreamSynchronize(s));
        }
        const std::vector<uint64_t> cnt = from_dev(d_cnt, (size_t)nb + 1);
        uint64_t nrec = 0;
        if (nb) {
            tile_base_scan_kernel<<<1, 1024, 0, s>>>(d_cnt, nb);
            CK(cudaGetLastError());
            CK(cudaMemcpyAsync(&nrec, d_cnt + nb, 8, cudaMemcpyDeviceToHost, s));
            CK(cudaStreamSynchronize(s));
        }
        const uint32_t head[4] = {w[2], w[0], w[1], ran ? 1u : 0u};
        put(head, 16);
        put_dev(d_stats, 3);
        put(&nrec, 8);
        put_dev(d_kind, (size_t)nb);
        const std::vector<LogBatchInfo> info = from_dev(d_info, (size_t)nb);
        std::vector<uint32_t> flags((size_t)nb);
        std::vector<int32_t> records((size_t)nb);
        for (size_t b = 0; b < (size_t)nb; b++) flags[b] = info[b].flags, records[b] = info[b].records;
        put(flags.data(), (size_t)nb * 4);
        put(records.data(), (size_t)nb * 4);
        put(cnt.data(), ((size_t)nb + 1) * 8);
        if (ran) {
            put_dev(d_sorted, (size_t)m);
            put_dev(d_res, (size_t)m);
            put_dev(d_tile, (size_t)(2 * tiles));
        }
        for (void *p : {(void *)d_bytes, (void *)d_off, (void *)d_cnt, (void *)d_part, (void *)d_info, (void *)d_hdr, (void *)d_word,
                        (void *)d_keys, (void *)d_sorted, (void *)d_kind, (void *)d_res, (void *)d_stats, (void *)d_ranges, (void *)d_tile,
                        (void *)d_tmp})
            if (p) CK(cudaFree(p));
    }
    CK(cudaStreamDestroy(s));
    fflush(stdout);
    return 0;
}
