// kta_logdecode_launch.cuh — the launch groups that turn compressed record batches into ordinary ones (kta_logdecode.cuh):
// the size pass, then, once the caller has sized the scratch buffers from its result, the copy pass.  scan_log_batches
// (kta_api.cu) and tests/native/logdecomp_probe.cu both launch through these, so the probe runs what the product runs.
// Allocation, error reporting and launch counting stay with the caller.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include <algorithm>

#include "kta_kernels.cuh"
#include "kta_logdecode.cuh"

namespace kta {

// thread per batch (log_header_kernel, log_unc_size_kernel) and warp per batch (the zstd size pass, the copies), 128 threads
inline int log_thread_grid(int64_t nbatches, int sm_count) { return (int)std::min<int64_t>((nbatches + 127) / 128, (int64_t)sm_count * 16); }
inline int log_warp_grid(int64_t nbatches, int sm_count) { return (int)std::min<int64_t>((nbatches + 3) / 4, (int64_t)sm_count * 16); }

// slot[b + 1] = scratch bytes of compressed batch b's uncompressed image, then scanned in place: slot[b] = its offset and
// slot[nbatches] = the total.  zstd: the header pass saw zstd batches (log_zstd_size_kernel sizes those).
inline cudaError_t log_launch_size_pass(const uint8_t *bytes, const LogBatchInfo *info, int64_t nbatches, uint64_t *slot,
                                        uint32_t *error_flags, bool zstd, int sm_count, cudaStream_t s) {
    log_unc_size_kernel<<<log_thread_grid(nbatches, sm_count), 128, 0, s>>>(bytes, info, nbatches, slot, error_flags);
    if (zstd) log_zstd_size_kernel<<<log_warp_grid(nbatches, sm_count), 128, 0, s>>>(bytes, info, nbatches, slot, error_flags);
    tile_base_scan_kernel<<<1, 1024, 0, s>>>(slot, nbatches);
    return cudaGetLastError();
}

// the decompression of every compressed batch into scratch + slot[b] (and zstd's literals into lit_scratch, a buffer of the
// scratch buffer's size); codecs: the LOGB_CODECS bits the header pass saw.  Afterwards info[b] describes the image.
inline cudaError_t log_launch_copy_pass(const uint8_t *bytes, LogBatchInfo *info, int64_t nbatches, const uint64_t *slot, uint8_t *scratch,
                                        uint8_t *lit_scratch, uint32_t *error_flags, uint32_t codecs, int sm_count, cudaStream_t s) {
    const int wgrid = log_warp_grid(nbatches, sm_count);
    if (codecs & ~(uint32_t)LOGB_ZSTD)
        log_decompress_kernel<false><<<wgrid, 128, 0, s>>>(bytes, info, nbatches, slot, scratch, nullptr, error_flags);
    if (codecs & LOGB_ZSTD)
        log_decompress_kernel<true><<<wgrid, 128, 0, s>>>(bytes, info, nbatches, slot, scratch, lit_scratch, error_flags);
    return cudaGetLastError();
}

}  // namespace kta
