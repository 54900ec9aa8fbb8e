// kta_synth.cu — materialises slices of the synthetic topic (kta_synth.h) into SoA columns, on the
// host (configs[0], CPU checks) or directly in HBM (configs[1..4]: the 1e8–4e9 record topics are
// generated where they are scanned).  Stands in for the Kafka fetch path (src/kafka.rs:93), which
// needs librdkafka + a broker and is out of scope (SURVEY.md §8 f3).
#include <cuda_runtime.h>

#include <algorithm>
#include <cstdio>
#include <cstring>
#include <vector>

#include "kta_kernels.cuh"
#include "kta_synth.h"

using namespace kta;

#include "kta_synth_host.cpp"   // synth_check, kta_synth_shard_records, kta_synth_fill_host, kta_synth_encode_segment_host

__global__ void __launch_bounds__(256) synth_columns_kernel(kta_synth_spec s, int rank, int world, int64_t start,
                                                            int64_t count, int32_t *partition, int64_t *offset,
                                                            int64_t *ts_ms, int32_t *key_len, int32_t *value_len,
                                                            uint64_t *seq) {
    for (int64_t j = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; j < count; j += (int64_t)gridDim.x * blockDim.x) {
        kta_synth_record r;
        kta_synth_record_at(s, kta_synth_local_to_global(s, rank, world, (uint64_t)(start + j)), r);
        if (partition) partition[j] = r.partition;
        if (offset) offset[j] = r.offset;
        if (ts_ms) ts_ms[j] = r.ts_ms;
        if (key_len) key_len[j] = r.key_len;
        if (value_len) value_len[j] = r.value_len;
        if (seq) seq[j] = r.seq;
    }
}

// one warp per 128-record tile: exclusive scan of key_len inside the tile, then every lane writes its keys
__global__ void __launch_bounds__(256) synth_keys_kernel(kta_synth_spec s, int rank, int world, int64_t start,
                                                         int64_t count, const uint64_t *tile_base, uint8_t *key_bytes,
                                                         int64_t cap) {
    const int lane = threadIdx.x & 31;
    const int64_t ntiles = (count + TILE - 1) / TILE;
    const int64_t gw = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5, gs = ((int64_t)gridDim.x * blockDim.x) >> 5;
    for (int64_t tile = gw; tile < ntiles; tile += gs) {
        uint64_t ids[ROWS];
        int32_t len[ROWS];
        uint64_t mine = 0;
#pragma unroll
        for (int k = 0; k < ROWS; k++) {
            const int64_t j = tile * TILE + (int64_t)lane * ROWS + k;  // a lane owns ROWS consecutive records
            len[k] = -1;
            ids[k] = 0;
            if (j < count) {
                kta_synth_record r;
                kta_synth_record_at(s, kta_synth_local_to_global(s, rank, world, (uint64_t)(start + j)), r);
                len[k] = r.key_len;
                ids[k] = r.key_id;
            }
            mine += len[k] > 0 ? (uint64_t)len[k] : 0;
        }
        uint64_t inc = mine;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
            const uint64_t t = __shfl_up_sync(0xffffffffu, inc, d);
            if (lane >= d) inc += t;
        }
        uint64_t o = tile_base[tile] + inc - mine;
        uint8_t tmp[KTA_SYNTH_MAX_KEY];
#pragma unroll
        for (int k = 0; k < ROWS; k++) {
            if (len[k] > 0) {
                kta_synth_key_bytes(s, ids[k], tmp);
                if ((int64_t)(o + (uint64_t)len[k]) <= cap)
                    for (int b = 0; b < len[k]; b++) key_bytes[o + b] = tmp[b];
                o += (uint64_t)len[k];
            }
        }
    }
}

extern "C" int kta_synth_fill_device(const kta_synth_spec *s, int32_t device, int32_t rank, int32_t world, int64_t start,
                                     int64_t count, int32_t *partition, int64_t *offset, int64_t *ts_ms,
                                     int32_t *key_len, int32_t *value_len, uint64_t *seq, uint8_t *key_bytes,
                                     int64_t key_bytes_cap, uint64_t *key_tile_base, int64_t *key_bytes_len) {
    if (synth_check(s, rank, world) || start < 0 || count < 0 || start + count > s->n_total / world) return KTA_ERR_INVALID;
    if (!key_len && (key_bytes || key_tile_base)) return KTA_ERR_INVALID;
    // the key bytes are placed by the tile bases: without them no key could be written (refused before any launch)
    if (!key_tile_base && (key_bytes || key_bytes_len)) return KTA_ERR_INVALID;
    if (device >= 0 && cudaSetDevice(device) != cudaSuccess) return KTA_ERR_CUDA;
    if (count == 0) {
        if (key_bytes_len) *key_bytes_len = 0;
        return KTA_OK;
    }
    int sms = 132;
    int dev = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    synth_columns_kernel<<<sms * 8, 256>>>(*s, rank, world, start, count, partition, offset, ts_ms, key_len, value_len, seq);
    if (cudaGetLastError() != cudaSuccess) return KTA_ERR_CUDA;
    uint64_t total = 0;
    if (key_tile_base) {
        const int64_t ntiles = (count + TILE - 1) / TILE;
        tile_key_bytes_kernel<<<(int)std::min<int64_t>((ntiles + 7) / 8, (int64_t)sms * 8), 256>>>(key_len, count, ntiles, key_tile_base);
        tile_base_scan_kernel<<<1, 1024>>>(key_tile_base, ntiles);
        if (cudaMemcpy(&total, key_tile_base + ntiles, 8, cudaMemcpyDeviceToHost) != cudaSuccess) return KTA_ERR_CUDA;
        if (key_bytes) {
            if ((int64_t)total > key_bytes_cap) return KTA_ERR_NOMEM;
            synth_keys_kernel<<<(int)std::min<int64_t>((ntiles + 7) / 8, (int64_t)sms * 8), 256>>>(*s, rank, world, start, count,
                                                                                          key_tile_base, key_bytes, key_bytes_cap);
        }
    }
    if (cudaDeviceSynchronize() != cudaSuccess || cudaGetLastError() != cudaSuccess) return KTA_ERR_CUDA;
    if (key_bytes_len) *key_bytes_len = (int64_t)total;
    return KTA_OK;
}
