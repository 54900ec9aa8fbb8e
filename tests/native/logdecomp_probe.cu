// TEST INFRASTRUCTURE: the decompression stage of the RecordBatch decoder on the GPU, with its output made visible.  It finds a
// segment's batches with the host walk of kta_push_log_segments_host (log_walk_batches) and launches what scan_log_batches
// (csrc/kta_api.cu) launches up to the record decode — the header pass (log_launch_header), its record-count scan, the size
// pass and the copy pass (csrc/kta_logdecode_launch.cuh: the same functions, grids and blocks) — and writes out every batch's
// result, so that tests/test_logdecomp_gpu.py can compare the 32-lane output with the reference codecs byte for byte.
// stdin: cases of u32 length + a segment of whole record batches.  stdout per case: u32 batch count, then per batch u32 final
// LogBatchInfo.flags, u64 slot size (slot[b + 1] - slot[b], 0 for a batch that was not compressed), u32 image length and the
// image the decoder would read (61-byte header + records section; length 0 unless the flags are LOGB_OK).
// Unlike scan_log_batches, the copy pass also runs when the size pass rejected some batches (they come out LOGB_BAD), so that
// one launch can carry many damaged batches.  The scratch buffers are filled with 0xA5 first: a byte the copy pass does not
// write shows up as a wrong byte.
#include "../../kafka_topic_analyzer_b200/csrc/kta_logoffsets.cuh"
#include "probe.h"

using namespace kta;

int main() {
    int sm_count = 0;
    CK(cudaDeviceGetAttribute(&sm_count, cudaDevAttrMultiProcessorCount, 0));
    cudaStream_t s;
    CK(cudaStreamCreate(&s));
    uint32_t n;
    while (fread(&n, 4, 1, stdin) == 1) {
        std::vector<uint8_t> seg(n);
        get(seg.data(), n);
        std::vector<uint64_t> offs;
        log_walk_batches(seg.data(), n, 0, offs);
        const int64_t nb = (int64_t)offs.size();
        const uint32_t nb32 = (uint32_t)nb;
        put(&nb32, 4);
        if (nb == 0) continue;
        uint8_t *d_bytes = dev_alloc<uint8_t>((size_t)n + 64, 0, s);   // 64 bytes of slack, like the product's staging buffer
        uint64_t *d_off = dev_alloc<uint64_t>((size_t)nb, 0, s), *d_cnt = dev_alloc<uint64_t>((size_t)nb + 1, 0, s);
        uint64_t *d_slot = dev_alloc<uint64_t>((size_t)nb + 2, 0, s);
        LogBatchInfo *d_info = dev_alloc<LogBatchInfo>((size_t)nb, 0, s);
        LogHeaderWord *d_word = dev_alloc<LogHeaderWord>(1, 0, s);
        uint32_t *d_flags = &d_word->flags;
        CK(cudaMemcpyAsync(d_bytes, seg.data(), n, cudaMemcpyHostToDevice, s));
        CK(cudaMemcpyAsync(d_off, offs.data(), (size_t)nb * 8, cudaMemcpyHostToDevice, s));
        CK(log_launch_header(d_bytes, (int64_t)n, d_off, nb, 0, nullptr, d_info, d_cnt, d_word, nullptr, nullptr, nullptr, 0, nullptr,
                             sm_count, s));
        tile_base_scan_kernel<<<1, 1024, 0, s>>>(d_cnt, nb);
        CK(cudaGetLastError());
        uint32_t flags = 0;
        CK(cudaMemcpyAsync(&flags, d_flags, 4, cudaMemcpyDeviceToHost, s));
        CK(cudaStreamSynchronize(s));
        uint8_t *d_unc = nullptr, *d_lit = nullptr;
        if (flags & LOGB_CODECS) {
            const uint32_t codecs = flags & LOGB_CODECS;
            const bool zstd = (codecs & LOGB_ZSTD) != 0;
            CK(cudaMemsetAsync(d_flags, 0, 4, s));
            CK(log_launch_size_pass(d_bytes, d_info, nb, d_slot, d_flags, zstd, sm_count, s));
            uint64_t unc_total = 0;
            CK(cudaMemcpyAsync(&unc_total, d_slot + nb, 8, cudaMemcpyDeviceToHost, s));
            CK(cudaStreamSynchronize(s));
            d_unc = dev_alloc<uint8_t>(unc_total + 64, 0xA5, s);
            if (zstd) d_lit = dev_alloc<uint8_t>(unc_total + 64, 0xA5, s);
            CK(log_launch_copy_pass(d_bytes, d_info, nb, d_slot, d_unc, d_lit, d_flags, codecs, sm_count, s));
        }
        CK(cudaStreamSynchronize(s));
        const std::vector<LogBatchInfo> info = from_dev(d_info, (size_t)nb);
        const std::vector<uint64_t> slot = d_unc ? from_dev(d_slot, (size_t)nb + 1) : std::vector<uint64_t>((size_t)nb + 1, 0);
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
        for (void *p : {(void *)d_bytes, (void *)d_off, (void *)d_cnt, (void *)d_slot, (void *)d_info, (void *)d_word, (void *)d_unc,
                        (void *)d_lit})
            if (p) CK(cudaFree(p));
    }
    CK(cudaStreamDestroy(s));
    fflush(stdout);
    return 0;
}
