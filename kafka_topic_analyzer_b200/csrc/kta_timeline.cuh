// kta_timeline.cuh — the timeline extension (include/kta.h, kta_set_timeline): per partition and time bucket, the records,
// tombstones and bytes of every counted scan.
//
// A separate pass behind scan_kernel on the same stream, over the same four header columns (20 B per record); the scan
// kernels are not touched.  Each CTA takes a contiguous range of 128-record tiles, so on time-ordered input (a Kafka
// partition is written in time order) it touches few buckets.  A warp reads a tile as coalesced streaming loads
// (16-byte vectors when the columns are aligned and the tile is full).  A row of 32 records that lies in one bin (a
// fetch: runs of one partition, near-monotone time) is summed in the warp and added once per counter.  Two places to add
// to, chosen per handle from the shape:
//   * shared memory (P * (B + 2) bins fit the opt-in shared memory): CTA-private u32 bins, laid out bucket-major
//     (b * P + p) like the scan's counter rows, flushed to the global u64 arrays once at the end, nonzero bins only.
//     A row of mixed bins adds record by record (shared-memory adds to distinct bins run in parallel);
//   * global memory otherwise: a row of mixed bins is grouped by bin first (__match_any_sync), and each group's first
//     lane adds the group's warp-reduced sums with one 64-bit RED.ADD per counter straight into the arrays.
#pragma once
#include "kta_kernels.cuh"

namespace kta {

constexpr int TL_THREADS = 1024;
// A CTA takes at most 2^24 tiles (2^31 records) of one launch: the host raises the grid for larger scans.  This bounds
// the CTA-private shared-memory bins (see timeline_add).
constexpr int64_t TL_MAX_CTA_TILES = (int64_t)1 << 24;
constexpr uint32_t TL_NONE = 0xffffffffu;   // bin key of a record that is not counted (no bin index reaches 2^24)
constexpr int TL_MAX_BUCKETS = 65536;
constexpr int64_t TL_MAX_BINS = (int64_t)1 << 24;

struct TimelineParams {
    int64_t n, ntiles;
    const int32_t *partition;
    const int64_t *ts_ms;
    const int32_t *key_len;
    const int32_t *value_len;
    int32_t P;                       // partitions (ids 0..P-1); every one has a row, foreign ones stay zero
    int32_t shard_world, shard_rank; // only partitions p % shard_world == shard_rank are counted (world 1: all)
    int32_t B;                       // buckets inside the range; index 0 = before it, B + 1 = after it
    int64_t origin;                  // O, seconds
    uint64_t width;                  // W >= 1, seconds
    uint64_t span;                   // B * W (fits: O + B * W does not overflow int64, so B * W < 2^64)
    double inv_width;                // 1.0 / W
    unsigned long long *out;         // [3][P][B + 2]: records | tombstones | bytes
};

__device__ __forceinline__ int4 tl_ld_v4(const int32_t *p) {
    int4 v;
    asm volatile("ld.global.nc.L1::no_allocate.v4.s32 {%0, %1, %2, %3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(p));
    return v;
}
__device__ __forceinline__ longlong2 tl_ld_v2(const int64_t *p) {
    longlong2 v;
    asm volatile("ld.global.nc.L1::no_allocate.v2.s64 {%0, %1}, [%2];" : "=l"(v.x), "=l"(v.y) : "l"(p));
    return v;
}

// bucket index of a record's timestamp: t = (ts_ms == -1 ? 0 : ts_ms) / 1000 truncating toward zero (src/metric.rs:209-211),
// 0 for t < O, 1 + (t - O) / W inside the range, B + 1 after it
__device__ __forceinline__ uint32_t timeline_index(const TimelineParams &t, int64_t ts) {
    const int64_t s = (ts == -1 ? 0 : ts) / 1000;
    if (s < t.origin) return 0;
    const uint64_t d = (uint64_t)s - (uint64_t)t.origin;
    if (d >= t.span) return (uint32_t)t.B + 1;
    // d / W without a 64-bit division: the quotient is below B <= 2^16, and d * (1/W) in double is within 2^-35 of it,
    // so its floor is off by at most one either way; one exact step against q * W (< B * W, no overflow) settles it
    uint64_t q = min((uint64_t)((double)d * t.inv_width), (uint64_t)t.B - 1);
    const uint64_t lo = q * t.width;
    if (lo > d) q--;
    else if (d - lo >= t.width) q++;
    return 1u + (uint32_t)q;
}

// CTA-private u32 bins [records | tombstones | bytes low word | bytes high word], each nbins long.  A CTA counts at most
// 2^31 records (TL_MAX_CTA_TILES), so records and tombstones cannot overflow.  Bytes are a 64-bit sum in two words: the
// low word's carry goes to the high word with the same add, and the high word stays below 2^31 (< 2^31 records of
// < 2^32 bytes each).
__device__ __forceinline__ void timeline_smem_add(uint32_t smem, int nbins, uint32_t key, uint32_t nrec, uint32_t ntomb,
                                                  unsigned long long nbytes) {
    const uint32_t a = smem + 4u * key, nb4 = 4u * (uint32_t)nbins;
    red_shared_add(a, nrec);
    red_shared_add_nz(a + nb4, ntomb);
    const uint32_t add_lo = (uint32_t)nbytes;
    uint32_t old;
    asm volatile("atom.shared.add.u32 %0, [%1], %2;" : "=r"(old) : "r"(a + 2u * nb4), "r"(add_lo) : "memory");
    const uint32_t add_hi = (uint32_t)(nbytes >> 32) + (old + add_lo < old ? 1u : 0u);
    red_shared_add_nz(a + 3u * nb4, add_hi);
}

// one row of 32 records, one per lane: key = the record's bin (TL_NONE: not counted)
template <bool SMEM>
__device__ __forceinline__ void timeline_add(const TimelineParams &t, uint32_t smem, int nbins, int lane, uint32_t key,
                                             uint32_t bytes, bool tomb) {
    const unsigned full = 0xffffffffu;
    const uint32_t k0 = __shfl_sync(full, key, 0);
    const bool uniform = __all_sync(full, key == k0);
    if (SMEM && !uniform) {
        // shared-memory adds to distinct bins proceed in parallel: on mixed rows each lane adds its own record, which is
        // cheaper than forming the groups first (on C1's 64 interleaved partitions a row has ~32 of them)
        if (key != TL_NONE) timeline_smem_add(smem, nbins, key, 1u, tomb ? 1u : 0u, bytes);
        return;
    }
    const unsigned grp = uniform ? full : __match_any_sync(full, key);
    const unsigned tombs = __ballot_sync(full, tomb);
    // a record's bytes are below 2^32: its 16-bit halves summed over <= 32 lanes stay below 2^21
    const uint32_t lo16 = __reduce_add_sync(grp, bytes & 0xffffu), hi16 = __reduce_add_sync(grp, bytes >> 16);
    if (key == TL_NONE || lane != __ffs(grp) - 1) return;
    const uint32_t nrec = __popc(grp), ntomb = __popc(grp & tombs);
    const unsigned long long nbytes = (unsigned long long)lo16 + ((unsigned long long)hi16 << 16);   // < 2^37
    if (SMEM) {
        timeline_smem_add(smem, nbins, key, nrec, ntomb, nbytes);
    } else {
        const size_t words = (size_t)t.P * (size_t)(t.B + 2);
        atomicAdd(t.out + key, (unsigned long long)nrec);
        if (ntomb) atomicAdd(t.out + words + key, (unsigned long long)ntomb);
        if (nbytes) atomicAdd(t.out + 2 * words + key, nbytes);
    }
}

template <bool SMEM>
__device__ __forceinline__ void timeline_record(const TimelineParams &t, uint32_t smem, int nbins, int lane, bool valid, int p,
                                                int64_t ts, int kl, int vl) {
    bool ok = valid && (unsigned)p < (unsigned)t.P;
    if (t.shard_world > 1) ok = ok && p % t.shard_world == t.shard_rank;
    const uint32_t idx = timeline_index(t, ts);
    const uint32_t key = !ok ? TL_NONE : SMEM ? idx * (uint32_t)t.P + (uint32_t)p : (uint32_t)p * (uint32_t)(t.B + 2) + idx;
    const uint32_t bytes = (uint32_t)max(kl, 0) + (uint32_t)max(vl, 0);
    timeline_add<SMEM>(t, smem, nbins, lane, key, ok ? bytes : 0u, ok && vl < 0);
}

template <bool SMEM>
__global__ void __launch_bounds__(TL_THREADS) timeline_kernel(const TimelineParams t) {
    extern __shared__ __align__(16) uint32_t tl_bins[];
    const int nbins = SMEM ? t.P * (t.B + 2) : 0;
    const uint32_t smem = SMEM ? smem_u32(tl_bins) : 0u;
    if (SMEM) {
        for (int i = threadIdx.x; i < 4 * nbins; i += blockDim.x) tl_bins[i] = 0;
        __syncthreads();
    }
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = blockDim.x >> 5;
    const int64_t t0 = t.ntiles * blockIdx.x / gridDim.x, t1 = t.ntiles * (blockIdx.x + 1) / gridDim.x;
    const bool vec = (((uintptr_t)t.partition | (uintptr_t)t.ts_ms | (uintptr_t)t.key_len | (uintptr_t)t.value_len) & 15u) == 0;
    for (int64_t tile = t0 + warp; tile < t1; tile += nwarps) {
        const int64_t base = tile * TILE;
        if (vec && base + TILE <= t.n) {
            // a full tile: lane l reads records 4 l .. 4 l + 3 of every column as one 16-byte vector (two for ts_ms)
            const int64_t r = base + 4 * lane;
            const int4 p4 = tl_ld_v4(t.partition + r), k4 = tl_ld_v4(t.key_len + r), v4 = tl_ld_v4(t.value_len + r);
            const longlong2 ta = tl_ld_v2(t.ts_ms + r), tb = tl_ld_v2(t.ts_ms + r + 2);
            timeline_record<SMEM>(t, smem, nbins, lane, true, p4.x, ta.x, k4.x, v4.x);
            timeline_record<SMEM>(t, smem, nbins, lane, true, p4.y, ta.y, k4.y, v4.y);
            timeline_record<SMEM>(t, smem, nbins, lane, true, p4.z, tb.x, k4.z, v4.z);
            timeline_record<SMEM>(t, smem, nbins, lane, true, p4.w, tb.y, k4.w, v4.w);
        } else {
#pragma unroll
            for (int k = 0; k < ROWS; k++) {
                const int64_t r = base + 32 * k + lane;
                const bool valid = r < t.n;
                timeline_record<SMEM>(t, smem, nbins, lane, valid, valid ? ld_stream_s32(t.partition + r) : 0,
                                      valid ? ld_stream_s64(t.ts_ms + r) : 0, valid ? ld_stream_s32(t.key_len + r) : 0,
                                      valid ? ld_stream_s32(t.value_len + r) : 0);
            }
        }
    }
    if (SMEM) {
        __syncthreads();
        const size_t words = (size_t)t.P * (size_t)(t.B + 2);
        for (int i = threadIdx.x; i < nbins; i += blockDim.x) {
            const uint32_t nrec = tl_bins[i];
            if (!nrec) continue;   // a bin without records has no tombstones or bytes either
            const int b = i / t.P, p = i - b * t.P;
            const size_t g = (size_t)p * (size_t)(t.B + 2) + (size_t)b;
            atomicAdd(t.out + g, (unsigned long long)nrec);
            const uint32_t ntomb = tl_bins[nbins + i];
            if (ntomb) atomicAdd(t.out + words + g, (unsigned long long)ntomb);
            const unsigned long long nbytes = (unsigned long long)tl_bins[2 * nbins + i] | ((unsigned long long)tl_bins[3 * nbins + i] << 32);
            if (nbytes) atomicAdd(t.out + 2 * words + g, nbytes);
        }
    }
}

}  // namespace kta
