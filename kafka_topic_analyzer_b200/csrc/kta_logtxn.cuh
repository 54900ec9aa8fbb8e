// kta_logtxn.cuh — read_committed isolation for the RecordBatch v2 decoder (kta_logdecode.cuh): records of aborted
// transactions are left out, as a consumer with isolation.level=read_committed (librdkafka's default) leaves them out.
//
// Batch attributes bit 4 = transactional, bit 5 = control.  A control batch holds one record whose key is
// version i16 (= 0) | type i16 (0 = ABORT, 1 = COMMIT).  A transactional data batch of partition p and producerId q is
// ABORTED (none of its records are delivered) when
//   1. the first control batch of the same (p, q) that follows it among the batches of the same call is an ABORT marker, or
//   2. its baseOffset lies in a registered aborted range [firstOffset, lastOffset] of the same (p, q) (the broker's
//      .txnindex files, kta_log_add_txn_index_host): exact when the marker lands in a later call.
// Matching is on (p, q) only, never on producerEpoch (a fenced producer's transaction is aborted under a bumped epoch).  A
// transactional batch with no following marker in its call and no covering range is UNDECIDED: delivered and counted.
//
// The passes, run on a read_committed handle between log_header_kernel and the record-count scan:
//   classify  (thread per batch)   transactional data batches and ABORT / COMMIT markers → a TxnKey each (+ kind per batch)
//   sort      (CUB radix sort)     TxnKeys by (partition, producerId, batch index): call order within each (p, q)
//   resolve   (thread per key)     per 256-key tile, the kind of the next marker of each key's (p, q); baseOffset order
//   carry     (one block)          the next marker behind each tile, for chains that run past a tile's end
//   apply     (thread per key)     marker decision | registered range → LOGB_SKIP_ABORTED, records = 0, counters
// Aborted batches are never decompressed or decoded (the size, copy and decode passes skip LOGB_SKIP_ABORTED).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include <algorithm>

#include <cub/device/device_radix_sort.cuh>
#include <cuda/std/tuple>

#include "kta_codec.cuh"
#include "kta_logdecode.cuh"
#include "kta_logdecode_launch.cuh"

namespace kta {

// per-batch kinds (TxnState::d_kind) and the resolved "next marker" of a key.  TXN_PASS: the answer lies behind the tile.
enum TxnKind : uint8_t { TXN_UNDECIDED = 0, TXN_ABORT = 1, TXN_COMMIT = 2, TXN_DATA = 3, TXN_PASS = 4 };
// error word bits (TxnState::d_word[1])
enum TxnErr : uint32_t { TXN_ERR_MARKER = 1, TXN_ERR_ORDER = 2 };
constexpr int TXN_TILE = 256;   // keys per resolve block

// sort key: (partition, producerId) groups a transaction's batches with its markers; the batch index keeps call order
struct TxnKey {
    uint64_t pid;
    uint32_t part;   // partition id, as its bit pattern
    uint32_t batch;  // index of the batch in the call
};
struct TxnKeyDecomposer {   // most significant first
    __host__ __device__ ::cuda::std::tuple<uint32_t &, uint64_t &, uint32_t &> operator()(TxnKey &k) const {
        return {k.part, k.pid, k.batch};
    }
};

// a registered aborted range; the handle keeps them sorted by (partition, pid, first) and merged where they overlap
struct TxnRange {
    int32_t part;
    uint32_t pad;
    uint64_t pid;
    int64_t first, last;
};

__device__ __forceinline__ bool same_group(const TxnKey &a, const TxnKey &b) { return a.part == b.part && a.pid == b.pid; }

// The marker of a control batch: kind (TXN_ABORT / TXN_COMMIT), TXN_UNDECIDED for a control type that is not a transaction
// marker, or 0xff when the marker cannot be read (compressed, no record, truncated record, key length != 4, version != 0).
__device__ __forceinline__ uint32_t read_marker(const uint8_t *p, uint32_t len) {
    if ((be_u16(p + 21) & 0x7u) != 0 || (int32_t)be_u32(p + 57) < 1) return 0xff;
    const uint8_t *q = p + LOG_HEADER_BYTES, *end = p + len;
    uint64_t u;
    int n = uvarint_g(q, end, u);
    const int64_t rec_len = unzigzag(u);
    if (n <= 0 || rec_len < 0 || rec_len > end - (q + n)) return 0xff;
    q += n;
    end = q + rec_len;
    q += 1;                                                   // record attributes
    if (q > end) return 0xff;
    for (int f = 0; f < 3; f++) {                             // timestampDelta, offsetDelta, keyLength
        n = uvarint_g(q, end, u);
        if (n <= 0) return 0xff;
        q += n;
    }
    if (unzigzag(u) != 4 || end - q < 4) return 0xff;
    if (be_u16(q) != 0) return 0xff;                          // version
    const uint32_t type = be_u16(q + 2);
    return type == 0 ? TXN_ABORT : type == 1 ? TXN_COMMIT : TXN_UNDECIDED;
}

// thread per batch.  word[0]: TxnKeys written, word[1]: TxnErr bits.
__global__ void txn_classify_kernel(const uint8_t *bytes, const LogBatchInfo *info, int64_t nbatches, TxnKey *keys, uint8_t *kind,
                                    uint32_t *word) {
    for (int64_t b = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; b < nbatches; b += (int64_t)gridDim.x * blockDim.x) {
        const LogBatchInfo bi = info[b];
        if (bi.flags & (LOGB_BAD | LOGB_COMPRESSED)) continue;   // refused by the header pass: the call fails
        if (bi.flags & (LOGB_SKIP_CRC | LOGB_SKIP_OFFSET)) continue;   // failed its CRC (check.crcs) or not served: not read
        const uint8_t *p = bytes + bi.off;
        uint32_t k;
        if (bi.flags == LOGB_SKIP_CONTROL) {
            k = read_marker(p, bi.len);
            if (k == 0xff) { atomicOr(word + 1, (uint32_t)TXN_ERR_MARKER); continue; }
            if (k == TXN_UNDECIDED) continue;                  // another control type: not a transaction marker
        } else {
            if (!(be_u16(p + 21) & 0x10u)) continue;           // not transactional
            k = TXN_DATA;
        }
        const uint64_t pid = be_u64(p + 43);
        if (pid == ~0ull) continue;                            // producerId -1: no transaction to belong to
        const uint32_t slot = atomicAdd(word, 1u);
        keys[slot] = TxnKey{pid, (uint32_t)bi.partition, (uint32_t)b};
        kind[b] = (uint8_t)k;
    }
}

// block per TXN_TILE sorted keys.  res[i] = kind of the first marker at or after key i within its (p, q) group, looking
// only inside the tile: TXN_UNDECIDED when the group ends first, TXN_PASS when the tile ends first.  tile_head[t] = res of the
// tile's first key (what a chain that runs into tile t finds).  A group whose baseOffsets do not increase is flagged.
__global__ void __launch_bounds__(TXN_TILE) txn_resolve_kernel(const TxnKey *keys, int64_t m, const uint8_t *kind, const LogBatchInfo *info,
                                                               uint8_t *res, uint8_t *tile_head, uint32_t *word) {
    __shared__ uint8_t warp_head[TXN_TILE / 32];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int64_t i = (int64_t)blockIdx.x * TXN_TILE + threadIdx.x;
    uint32_t s = TXN_PASS;
    bool cont = false;   // key i + 1 belongs to the same group
    if (i < m) {
        const TxnKey k = keys[i];
        const uint32_t kd = kind[k.batch];
        if (i + 1 < m) {
            const TxnKey nk = keys[i + 1];
            cont = same_group(k, nk);
            if (cont && info[nk.batch].base_offset <= info[k.batch].base_offset) atomicOr(word + 1, (uint32_t)TXN_ERR_ORDER);
        }
        s = kd != TXN_DATA ? kd : cont ? (uint32_t)TXN_PASS : (uint32_t)TXN_UNDECIDED;
    }
    // first non-PASS value at or after each position: within the warp, then across the warps of the tile
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
        const uint32_t t = __shfl_down_sync(0xffffffffu, s, d);
        if (s == TXN_PASS && lane + d < 32) s = t;
    }
    if (lane == 0) warp_head[warp] = (uint8_t)s;
    __syncthreads();
    for (int w = warp + 1; w < TXN_TILE / 32 && s == TXN_PASS; w++) s = warp_head[w];
    if (i < m) res[i] = (uint8_t)s;
    if (threadIdx.x == 0) tile_head[blockIdx.x] = (uint8_t)s;
}

// one block: carry[t] = first non-PASS tile_head of the tiles behind t (what a chain that reaches the end of tile t finds).
// The last key of all is never PASS, so every chain ends.
__global__ void __launch_bounds__(1024) txn_carry_kernel(const uint8_t *tile_head, int64_t ntiles, uint8_t *carry) {
    __shared__ uint8_t warp_head[32];
    __shared__ uint8_t next_s;   // first non-PASS head behind the chunk being done
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    if (threadIdx.x == 0) next_s = TXN_PASS;
    __syncthreads();
    // chunks of 1024 tiles from the last one down; within a chunk, position j holds tile (base + j)
    for (int64_t base = ((ntiles - 1) / 1024) * 1024; base >= 0; base -= 1024) {
        const int64_t t = base + threadIdx.x;
        uint32_t s = t + 1 < ntiles ? tile_head[t + 1] : (uint32_t)TXN_PASS;   // exclusive: the tiles behind t
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
            const uint32_t x = __shfl_down_sync(0xffffffffu, s, d);
            if (s == TXN_PASS && lane + d < 32) s = x;
        }
        if (lane == 0) warp_head[warp] = (uint8_t)s;
        __syncthreads();
        for (int w = warp + 1; w < 32 && s == TXN_PASS; w++) s = warp_head[w];
        if (s == TXN_PASS) s = next_s;
        if (t < ntiles) carry[t] = (uint8_t)s;
        __syncthreads();   // every thread has read next_s and warp_head
        if (threadIdx.x == 0) {
            const uint32_t h0 = tile_head[base];              // the chunk's first tile, inclusive
            next_s = (uint8_t)(h0 != TXN_PASS ? h0 : s);
        }
        __syncthreads();
    }
}

// is (part, pid, off) inside a registered range?  ranges: sorted by (part, pid, first), disjoint within a (part, pid)
__device__ __forceinline__ bool in_aborted_range(const TxnRange *ranges, int64_t nranges, int32_t part, uint64_t pid, int64_t off) {
    int64_t lo = 0, hi = nranges;   // first range whose (part, pid, first) > (part, pid, off)
    while (lo < hi) {
        const int64_t mid = (lo + hi) >> 1;
        const TxnRange r = ranges[mid];
        const bool le = r.part != part ? r.part < part : r.pid != pid ? r.pid < pid : r.first <= off;
        if (le) lo = mid + 1;
        else hi = mid;
    }
    if (lo == 0) return false;
    const TxnRange r = ranges[lo - 1];
    return r.part == part && r.pid == pid && r.last >= off;
}

// thread per sorted key.  stats[0] aborted batches, [1] aborted records, [2] undecided records (this call).
__global__ void txn_apply_kernel(const TxnKey *keys, int64_t m, const uint8_t *kind, const uint8_t *res, const uint8_t *carry,
                                 const TxnRange *ranges, int64_t nranges, LogBatchInfo *info, uint64_t *rec_count,
                                 const uint32_t *word, unsigned long long *stats) {
    if (word[1]) return;   // the call is refused: nothing is applied
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < m; i += (int64_t)gridDim.x * blockDim.x) {
        const TxnKey k = keys[i];
        if (kind[k.batch] != TXN_DATA) continue;
        uint32_t s = res[i];
        if (s == TXN_PASS) s = carry[i / TXN_TILE];
        LogBatchInfo &bi = info[k.batch];
        const int32_t part = (int32_t)k.part;
        const bool aborted = s == TXN_ABORT || (nranges && in_aborted_range(ranges, nranges, part, k.pid, bi.base_offset));
        const int32_t records = bi.records;
        if (aborted) {
            bi.flags = LOGB_SKIP_ABORTED;
            bi.records = 0;
            rec_count[k.batch + 1] = 0;
            atomicAdd(stats, 1ull);
            if (records) atomicAdd(stats + 1, (unsigned long long)records);
        } else if (s == TXN_UNDECIDED && records) atomicAdd(stats + 2, (unsigned long long)records);
    }
}

// The launch groups of the passes, launched by txn_passes (kta_logscan.cuh), which does the allocation, the host round trip,
// error reporting and launch counting.  (They live here and not in kta_logdecode_launch.cuh: a translation unit that includes
// them compiles the radix sort's kernels.)

// the classify pass over the batches log_header_kernel has read; word[0..1] zeroed by the caller
inline cudaError_t log_launch_txn_classify(const uint8_t *bytes, const LogBatchInfo *info, int64_t nbatches, TxnKey *keys, uint8_t *kind,
                                           uint32_t *word, int sm_count, cudaStream_t s) {
    txn_classify_kernel<<<log_thread_grid(nbatches, sm_count), 128, 0, s>>>(bytes, info, nbatches, keys, kind, word);
    return cudaGetLastError();
}

inline int64_t log_txn_tiles(int64_t m) { return (m + TXN_TILE - 1) / TXN_TILE; }

// sort, resolve, carry and apply over the m > 0 keys the classify pass wrote.  tile: 2 * log_txn_tiles(m) bytes, the tile
// heads, then the carries.  With sort_tmp == nullptr nothing is launched and tmp_bytes becomes the sort's scratch size, as
// with CUB; else tmp_bytes is the size of sort_tmp.  stats[0..2] are zeroed here.
inline cudaError_t log_launch_txn_passes(TxnKey *keys, TxnKey *sorted, int64_t m, const uint8_t *kind, LogBatchInfo *info, uint8_t *res,
                                         uint8_t *tile, void *sort_tmp, size_t &tmp_bytes, const TxnRange *ranges, int64_t nranges,
                                         uint64_t *rec_count, uint32_t *word, unsigned long long *stats, int sm_count, cudaStream_t s) {
    cudaError_t e = cub::DeviceRadixSort::SortKeys(sort_tmp, tmp_bytes, keys, sorted, m, TxnKeyDecomposer{}, s);
    if (e != cudaSuccess || !sort_tmp) return e;
    const int64_t tiles = log_txn_tiles(m);
    if ((e = cudaMemsetAsync(stats, 0, 24, s)) != cudaSuccess) return e;
    txn_resolve_kernel<<<(unsigned)tiles, TXN_TILE, 0, s>>>(sorted, m, kind, info, res, tile, word);
    txn_carry_kernel<<<1, 1024, 0, s>>>(tile, tiles, tile + tiles);
    txn_apply_kernel<<<(int)std::min<int64_t>((m + 255) / 256, (int64_t)sm_count * 16), 256, 0, s>>>(
        sorted, m, kind, res, tile + tiles, ranges, nranges, info, rec_count, word, stats);
    return cudaGetLastError();
}

}  // namespace kta
