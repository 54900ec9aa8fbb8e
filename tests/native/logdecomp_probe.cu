// TEST INFRASTRUCTURE: the decompression stage of the RecordBatch decoder on the GPU, with its output made visible.  It launches
// what scan_log_batches (csrc/kta_api.cu) launches up to the record decode — log_header_kernel, its record-count scan, the size
// pass and the copy pass (csrc/kta_logdecode_launch.cuh: the same functions, grids and blocks) — and writes out every batch's
// result, so that tests/test_logdecomp_gpu.py can compare the 32-lane output with the reference codecs byte for byte.
// stdin: cases of u32 length + a segment of whole record batches.  stdout per case: u32 batch count, then per batch u32 final
// LogBatchInfo.flags, u64 slot size (slot[b + 1] - slot[b], 0 for a batch that was not compressed), u32 image length and the
// image the decoder would read (61-byte header + records section; length 0 unless the flags are LOGB_OK).
// Unlike scan_log_batches, the copy pass also runs when the size pass rejected some batches (they come out LOGB_BAD), so that
// one launch can carry many damaged batches.  The scratch buffers are filled with 0xA5 first: a byte the copy pass does not
// write shows up as a wrong byte.
#include <cuda_runtime.h>

#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <vector>

#include "../../kafka_topic_analyzer_b200/csrc/kta_logdecode_launch.cuh"

using namespace kta;

#define CK(call)                                                                                           \
    do {                                                                                                   \
        cudaError_t e_ = (call);                                                                           \
        if (e_ != cudaSuccess) {                                                                           \
            fprintf(stderr, "%s: %s (%s:%d)\n", #call, cudaGetErrorString(e_), __FILE__, __LINE__);        \
            exit(3);                                                                                       \
        }                                                                                                  \
    } while (0)

static void put(const void *p, size_t n) {
    if (n && fwrite(p, 1, n, stdout) != n) exit(4);
}

int main() {
    int sm_count = 0;
    CK(cudaDeviceGetAttribute(&sm_count, cudaDevAttrMultiProcessorCount, 0));
    cudaStream_t s;
    CK(cudaStreamCreate(&s));
    uint32_t n;
    while (fread(&n, 4, 1, stdin) == 1) {
        std::vector<uint8_t> seg(n);
        if (n && fread(seg.data(), 1, n, stdin) != n) return 2;
        // batch offsets: hop from header to header as kta_push_log_segments_host does
        std::vector<uint64_t> offs;
        for (uint64_t pos = 0; pos + LOG_HEADER_BYTES <= n;) {
            const int64_t bl = (int32_t)(((uint32_t)seg[pos + 8] << 24) | ((uint32_t)seg[pos + 9] << 16) | ((uint32_t)seg[pos + 10] << 8) | seg[pos + 11]);
            if (bl < LOG_HEADER_BYTES - 12 || pos + 12 + (uint64_t)bl > n) break;
            offs.push_back(pos);
            pos += 12 + (uint64_t)bl;
        }
        const int64_t nb = (int64_t)offs.size();
        const uint32_t nb32 = (uint32_t)nb;
        put(&nb32, 4);
        if (nb == 0) continue;
        uint8_t *d_bytes;
        uint64_t *d_off, *d_cnt, *d_slot;
        LogBatchInfo *d_info;
        uint32_t *d_err;
        CK(cudaMalloc(&d_bytes, (size_t)n + 64));   // 64 bytes of slack, like the product's staging buffer
        CK(cudaMalloc(&d_off, (size_t)nb * 8));
        CK(cudaMalloc(&d_cnt, (size_t)(nb + 1) * 8));
        CK(cudaMalloc(&d_slot, (size_t)(nb + 2) * 8));
        CK(cudaMalloc(&d_info, (size_t)nb * sizeof(LogBatchInfo)));
        CK(cudaMalloc(&d_err, 8));
        CK(cudaMemsetAsync(d_bytes, 0, (size_t)n + 64, s));
        CK(cudaMemcpyAsync(d_bytes, seg.data(), n, cudaMemcpyHostToDevice, s));
        CK(cudaMemcpyAsync(d_off, offs.data(), (size_t)nb * 8, cudaMemcpyHostToDevice, s));
        CK(cudaMemsetAsync(d_slot, 0, (size_t)(nb + 2) * 8, s));
        CK(cudaMemsetAsync(d_err, 0, 8, s));
        log_header_kernel<<<log_thread_grid(nb, sm_count), 128, 0, s>>>(d_bytes, (int64_t)n, d_off, nb, 0, nullptr, d_info, d_cnt, d_err);
        tile_base_scan_kernel<<<1, 1024, 0, s>>>(d_cnt, nb);
        CK(cudaGetLastError());
        uint32_t err[2] = {0, 0};
        CK(cudaMemcpyAsync(err, d_err, 8, cudaMemcpyDeviceToHost, s));
        CK(cudaStreamSynchronize(s));
        uint8_t *d_unc = nullptr, *d_lit = nullptr;
        if (err[0] & LOGB_CODECS) {
            const uint32_t codecs = err[0] & LOGB_CODECS;
            const bool zstd = (codecs & LOGB_ZSTD) != 0;
            CK(cudaMemsetAsync(d_err, 0, 4, s));
            CK(log_launch_size_pass(d_bytes, d_info, nb, d_slot, d_err, zstd, sm_count, s));
            uint64_t unc_total = 0;
            CK(cudaMemcpyAsync(&unc_total, d_slot + nb, 8, cudaMemcpyDeviceToHost, s));
            CK(cudaStreamSynchronize(s));
            CK(cudaMalloc(&d_unc, unc_total + 64));
            CK(cudaMemsetAsync(d_unc, 0xA5, unc_total + 64, s));
            if (zstd) {
                CK(cudaMalloc(&d_lit, unc_total + 64));
                CK(cudaMemsetAsync(d_lit, 0xA5, unc_total + 64, s));
            }
            CK(log_launch_copy_pass(d_bytes, d_info, nb, d_slot, d_unc, d_lit, d_err, codecs, sm_count, s));
        }
        std::vector<LogBatchInfo> info((size_t)nb);
        std::vector<uint64_t> slot((size_t)nb + 1, 0);
        CK(cudaMemcpyAsync(info.data(), d_info, (size_t)nb * sizeof(LogBatchInfo), cudaMemcpyDeviceToHost, s));
        if (d_unc) CK(cudaMemcpyAsync(slot.data(), d_slot, (size_t)(nb + 1) * 8, cudaMemcpyDeviceToHost, s));
        CK(cudaStreamSynchronize(s));
        std::vector<uint8_t> img;
        for (int64_t b = 0; b < nb; b++) {
            const LogBatchInfo &bi = info[(size_t)b];
            const uint64_t slot_size = slot[(size_t)b + 1] - slot[(size_t)b];
            const uint32_t len = bi.flags == LOGB_OK ? bi.len : 0u;
            put(&bi.flags, 4);
            put(&slot_size, 8);
            put(&len, 4);
            if (len) {
                img.resize(len);
                CK(cudaMemcpy(img.data(), (const void *)((uintptr_t)d_bytes + bi.off), len, cudaMemcpyDeviceToHost));   // (off may lead into the scratch buffer)
                put(img.data(), len);
            }
        }
        CK(cudaFree(d_bytes));
        CK(cudaFree(d_off));
        CK(cudaFree(d_cnt));
        CK(cudaFree(d_slot));
        CK(cudaFree(d_info));
        CK(cudaFree(d_err));
        if (d_unc) CK(cudaFree(d_unc));
        if (d_lit) CK(cudaFree(d_lit));
    }
    CK(cudaStreamDestroy(s));
    fflush(stdout);
    return 0;
}
