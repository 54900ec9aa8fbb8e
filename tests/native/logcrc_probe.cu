// TEST INFRASTRUCTURE: the check.crcs passes of the RecordBatch decoder (csrc/kta_logcrc.cuh) on the GPU, with everything they
// produce made visible.  It launches what log_headers (csrc/kta_api.cu) launches for a handle with check.crcs on — the span
// counts (windowed when a window table is given), their scan, the span pass, then the header pass with the CRC check — through
// the same launch functions (log_launch_crc_spans, log_launch_header in csrc/kta_logoffsets.cuh), and writes out every array,
// so that tests/test_logcrc_passes.py can compare them batch by batch with a plain CRC-32C.
// stdin, per case (little-endian): u64 nbytes, the bytes; u32 nbatches, u64 batch offsets; u32 with_partitions, then i32 per
// batch partitions when it is 1 (else every batch is partition 0); u32 slack: the bytes behind nbytes that may be read; u32
// nwin, then nwin x (i64 S, i64 H): the window table of partitions [0, nwin) (nwin 0: no windows); u32 grid: the span pass's
// blocks, 0 for the library's rule (log_crc_span_grid).  The span pass's body does not depend on its grid, so a small grid
// gives every warp many rounds with few spans.
// stdout: u32 SM count of the device; then per case: u32 the span pass's grid, u64 spans[nbatches + 1] after the scan, u32
// acc[nbatches], u32 flags[nbatches] after the header pass, the header pass's error word (LogHeaderWord: ten u32 words), then
// its crc_failed LogCrcFail records (u32 batch, u32 batch bytes, i64 baseOffset, i32 partition, u32 stored, u32 computed,
// u32 0), sorted by batch.
// acc is filled with 0xA5 first: an entry the count pass does not write shows up.
//
// `logcrc_probe host` is a plain reference instead, which touches no CUDA: stdin, per region, u64 n and n bytes; stdout the
// u32 CRC-32C of each, one byte at a time with a table of its own.
#include <cstring>

#include "../../kafka_topic_analyzer_b200/csrc/kta_logoffsets.cuh"
#include "probe.h"

using namespace kta;

// CRC-32C (reflected 0x82F63B78, init and xorout 0xFFFFFFFF), one byte at a time
static int host_mode() {
    uint32_t t[256];
    for (uint32_t i = 0; i < 256; i++) {
        uint32_t c = i;
        for (int k = 0; k < 8; k++) c = (c & 1u) ? (c >> 1) ^ 0x82F63B78u : c >> 1;
        t[i] = c;
    }
    std::vector<uint8_t> buf;
    uint64_t n;
    while (fread(&n, 8, 1, stdin) == 1) {
        buf.resize(n);
        get(buf.data(), n);
        uint32_t crc = 0xFFFFFFFFu;
        for (uint64_t i = 0; i < n; i++) crc = t[(crc ^ buf[i]) & 0xFFu] ^ (crc >> 8);
        crc ^= 0xFFFFFFFFu;
        put(&crc, 4);
    }
    fflush(stdout);
    return 0;
}

int main(int argc, char **argv) {
    if (argc > 1 && !strcmp(argv[1], "host")) return host_mode();
    int sm_count = 0;
    CK(cudaDeviceGetAttribute(&sm_count, cudaDevAttrMultiProcessorCount, 0));
    const uint32_t device = (uint32_t)sm_count;
    put(&device, 4);
    cudaStream_t s;
    CK(cudaStreamCreate(&s));
    // as log_crc_spans does on a handle's first call with the switch on
    LogCrcTables tables;
    log_crc_tables_host(tables);
    LogCrcTables *d_tables = dev_alloc<LogCrcTables>(1, 0, s);
    CK(cudaMemcpyAsync(d_tables, &tables, sizeof tables, cudaMemcpyHostToDevice, s));
    CK(cudaFuncSetAttribute(log_crc_span_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)LOG_CRC_SMEM));
    uint64_t n;
    while (fread(&n, 8, 1, stdin) == 1) {
        std::vector<uint8_t> seg(n);
        get(seg.data(), n);
        uint32_t nb32 = 0, with_part = 0, slack = 0, nwin = 0, grid_in = 0;
        get(&nb32, 4);
        const int64_t nb = nb32;
        std::vector<uint64_t> offs((size_t)nb);
        get(offs.data(), (size_t)nb * 8);
        get(&with_part, 4);
        std::vector<int32_t> parts(with_part ? (size_t)nb : 0);
        get(parts.data(), parts.size() * 4);
        get(&slack, 4);
        get(&nwin, 4);
        std::vector<longlong2> win(nwin);
        get(win.data(), (size_t)nwin * sizeof(longlong2));
        get(&grid_in, 4);

        uint8_t *d_bytes = dev_alloc<uint8_t>(n + slack, 0, s);
        uint64_t *d_off = dev_alloc<uint64_t>((size_t)nb, 0, s), *d_cnt = dev_alloc<uint64_t>((size_t)nb + 1, 0, s);
        uint64_t *d_spans = dev_alloc<uint64_t>((size_t)nb + 1, 0, s);
        uint32_t *d_acc = dev_alloc<uint32_t>((size_t)nb, 0xA5, s);
        LogCrcFail *d_fails = dev_alloc<LogCrcFail>((size_t)nb, 0, s);
        int32_t *d_part = with_part ? dev_alloc<int32_t>((size_t)nb, 0, s) : nullptr;
        LogBatchInfo *d_info = dev_alloc<LogBatchInfo>((size_t)nb, 0, s);
        LogHeaderWord *d_word = dev_alloc<LogHeaderWord>(1, 0, s);
        longlong2 *d_win = nwin ? dev_alloc<longlong2>(nwin, 0, s) : nullptr;
        uint32_t *d_cut = nwin ? dev_alloc<uint32_t>((size_t)nb, 0, s) : nullptr;
        CK(cudaMemcpyAsync(d_bytes, seg.data(), n, cudaMemcpyHostToDevice, s));
        CK(cudaMemcpyAsync(d_off, offs.data(), (size_t)nb * 8, cudaMemcpyHostToDevice, s));
        if (d_part) CK(cudaMemcpyAsync(d_part, parts.data(), (size_t)nb * 4, cudaMemcpyHostToDevice, s));
        if (d_win) CK(cudaMemcpyAsync(d_win, win.data(), (size_t)nwin * sizeof(longlong2), cudaMemcpyHostToDevice, s));
        const int grid = grid_in ? (int)grid_in : log_crc_span_grid((int64_t)n, nb, sm_count);
        if (nb) {
            CK(log_launch_crc_spans(d_bytes, (int64_t)n, d_off, nb, 0, d_part, d_win, (int32_t)nwin, d_tables, d_spans, d_acc, grid,
                                    sm_count, s));
            CK(log_launch_header(d_bytes, (int64_t)n, d_off, nb, 0, d_part, d_info, d_cnt, d_word, d_acc, d_fails, d_win, (int32_t)nwin,
                                 d_cut, sm_count, s));
        }
        CK(cudaStreamSynchronize(s));
        const uint32_t grid32 = (uint32_t)grid;
        put(&grid32, 4);
        put(from_dev(d_spans, (size_t)nb + 1).data(), ((size_t)nb + 1) * 8);
        put(from_dev(d_acc, (size_t)nb).data(), (size_t)nb * 4);
        const std::vector<LogBatchInfo> info = from_dev(d_info, (size_t)nb);
        std::vector<uint32_t> flags((size_t)nb);
        for (size_t b = 0; b < (size_t)nb; b++) flags[b] = info[b].flags;
        put(flags.data(), (size_t)nb * 4);
        const LogHeaderWord word = from_dev(d_word, 1)[0];
        put(&word, sizeof word);
        std::vector<LogCrcFail> fails = from_dev(d_fails, std::min<size_t>(word.crc_failed, (size_t)nb));
        std::sort(fails.begin(), fails.end(), [](const LogCrcFail &a, const LogCrcFail &b) { return a.batch < b.batch; });
        put(fails.data(), fails.size() * sizeof(LogCrcFail));
        for (void *p : {(void *)d_bytes, (void *)d_off, (void *)d_cnt, (void *)d_spans, (void *)d_acc, (void *)d_fails, (void *)d_part,
                        (void *)d_info, (void *)d_word, (void *)d_win, (void *)d_cut})
            if (p) CK(cudaFree(p));
    }
    CK(cudaFree(d_tables));
    CK(cudaStreamDestroy(s));
    fflush(stdout);
    return 0;
}
