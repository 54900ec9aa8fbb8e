// kta_logdecode_launch.cuh — the launch groups of the RecordBatch decoder (kta_logdecode.cuh): the ones that turn compressed
// record batches into ordinary ones (the size pass, then, once the caller has sized the scratch buffers from its result, the
// copy pass), the record decode with its shape (plain, or with offset windows), the key-length tile bases and the key
// gather; and the host walk that finds a segment's batches.  The header pass is launched by log_launch_header
// (kta_logoffsets.cuh).  The steps of kta_logscan.cuh launch through these; allocation, the host round trips, error reporting
// and launch counting are theirs.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include <algorithm>
#include <vector>

#include "kta_kernels.cuh"
#include "kta_logdecode.cuh"

namespace kta {

// The record batches of a segment of n bytes, found on the host: hops from batch header to batch header (12 + batchLength
// bytes each) and appends base + each batch's offset to offs.  A truncated tail is ignored, as a consumer ignores a
// partially fetched batch.  Returns the bytes the whole batches take.
inline int64_t log_walk_batches(const uint8_t *seg, int64_t n, int64_t base, std::vector<uint64_t> &offs) {
    int64_t pos = 0;
    while (pos + LOG_HEADER_BYTES <= n) {
        const uint8_t *p = seg + pos;
        const int64_t bl = (int64_t)(int32_t)(((uint32_t)p[8] << 24) | ((uint32_t)p[9] << 16) | ((uint32_t)p[10] << 8) | p[11]);
        if (bl < LOG_HEADER_BYTES - 12 || pos + 12 + bl > n) break;
        offs.push_back((uint64_t)(base + pos));
        pos += 12 + bl;
    }
    return pos;
}

// thread per batch (the header pass, log_unc_size_kernel) and warp per batch (the zstd size pass, the copies), 128 threads
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

// The shape of one record decode (log_decode_kernel, one warp per batch).  The stage holds the call's longest batch and the
// up to 15 bytes that lead it to a 16-byte boundary, rounded up to 1 KiB; the launch is staged only when that stage is at
// most 48 KiB, else every batch is read in place.  As many blocks per SM as the opt-in shared memory holds, 1 to 16.
struct LogDecodeShape {
    uint32_t stage;   // per warp, bytes (0 when not staged)
    bool staged;
    size_t smem;      // dynamic shared memory per block
    int per_sm;       // blocks per SM
    int grid;         // blocks; warp w decodes batches w, w + 4 * grid, ...
};
inline LogDecodeShape log_decode_shape(uint32_t longest, int64_t nbatches, int sm_count, size_t smem_optin) {
    LogDecodeShape d;
    const uint32_t stage = (uint32_t)(((size_t)longest + 16 + 1023) / 1024 * 1024);
    d.staged = stage <= 48u * 1024u;
    d.stage = d.staged ? stage : 0u;
    d.smem = (size_t)(LOG_DECODE_THREADS / 32) * (LOG_WARP_HEADER + d.stage);
    d.per_sm = (int)std::max<size_t>(1, std::min<size_t>(16, smem_optin / std::max<size_t>(d.smem, 1)));
    d.grid = (int)std::min<int64_t>((nbatches + 3) / 4, (int64_t)sm_count * d.per_sm);
    return d;
}

// the record decode in that shape: the columns of record rec_base[b] + i of batch b; key_src only when keys are gathered.
// With a window table (given only for a call with cut batches) the window decode runs, which leaves out the records of cut
// batches below their partition's log start offset; a call whose windows cut nothing keeps every record of its served
// batches, which is what the plain decode writes.
inline cudaError_t log_launch_decode(const LogDecodeShape &d, const uint8_t *bytes, uint64_t readable, const LogBatchInfo *info,
                                     int64_t nbatches, const uint64_t *rec_base, int32_t *partition, int64_t *ts_ms, int32_t *key_len,
                                     int32_t *value_len, uint64_t *key_src, uint32_t *error_flags, const longlong2 *window,
                                     int32_t num_partitions, cudaStream_t s) {
    const auto decode = window ? (d.staged ? log_decode_kernel<true, true> : log_decode_kernel<false, true>)
                               : (d.staged ? log_decode_kernel<true, false> : log_decode_kernel<false, false>);
    decode<<<d.grid, LOG_DECODE_THREADS, d.smem, s>>>(bytes, readable, info, nbatches, rec_base, partition, ts_ms, key_len, value_len,
                                                      key_src, d.stage, error_flags, window, num_partitions);
    return cudaGetLastError();
}

// the key_tile_base column of n records' key lengths: tile_base[t] = key bytes of the 128-record tiles before t, [ntiles] =
// the key bytes in all (two launches)
inline cudaError_t log_launch_tile_base(const int32_t *key_len, int64_t n, uint64_t *tile_base, int sm_count, cudaStream_t s) {
    const int64_t ntiles = (n + TILE - 1) / TILE;
    tile_key_bytes_kernel<<<(int)std::min<int64_t>((ntiles + 7) / 8, (int64_t)sm_count * 8), 256, 0, s>>>(key_len, n, ntiles, tile_base);
    tile_base_scan_kernel<<<1, 1024, 0, s>>>(tile_base, ntiles);
    return cudaGetLastError();
}

// the keys of n decoded records packed in record order into key_out, at the offsets tile_base gives
inline cudaError_t log_launch_gather_keys(const uint8_t *bytes, const uint64_t *key_src, const int32_t *key_len, int64_t n,
                                          const uint64_t *tile_base, uint8_t *key_out, int sm_count, cudaStream_t s) {
    const int64_t ntiles = (n + TILE - 1) / TILE;
    log_gather_keys_kernel<<<(int)std::min<int64_t>((ntiles + 7) / 8, (int64_t)sm_count * 8), 256, 0, s>>>(bytes, key_src, key_len, n,
                                                                                                            tile_base, key_out);
    return cudaGetLastError();
}

}  // namespace kta
