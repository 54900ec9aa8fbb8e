// kta_hotkeys.cuh — hot keys (include/kta.h, kta_set_hot_keys): an exact, topic-wide table of per-key counters (records,
// tombstones, bytes, latest second, partition range, key prefix), filled by a pass behind the counted scans; finalize picks
// the keys with the most records.
//
// A separate pass behind scan_kernel (and the timeline and partitioner passes) on the same stream; the scan kernels are not
// touched.  It reads partition, key_len, value_len and ts_ms, the tile bases and the key bytes: 20 B per record plus the
// keys, as the hashing scan does, plus its table traffic.  Each CTA takes a contiguous range of 128-record tiles, one warp
// per tile, as the partitioner pass does, with that pass's own pieces: the key span staged by pc_stage_copy, offsets from
// key_offsets (pc_wide_offsets for keys of 1 MiB and more), and a key's id from pc_hashes, (crc32 << 32) | murmur2.
//   * Table: open addressing over `slots` (a power of two) slots of HK_SLOT_BYTES.  The home slot is the multiply-high of
//     a 64-bit finalizer of the id by `slots`; the probe is linear and wraps at the end.  Id 0 marks an empty slot, so the
//     entry whose id is 0 lives in one side slot behind the table.  A slot is claimed once, by CAS on its id word (on its
//     claim word for the side slot); the claimant writes key_len and the prefix and counts the claim.  Counters are REDs:
//     ADD for records, tombstones and bytes, MAX for the latest second and the partition range (both kept so that zero is
//     the identity of MAX, so a zeroed table is an empty one).
//   * The probe is bounded by the table size: a probe that finds neither its id nor an empty slot raises the failure word
//     (the host reports it as an internal error).  The host keeps the table at most half full (kta_api.cu, launch_hot_keys),
//     so it never fires.
//   * Warp aggregation: a row of 32 records is grouped by id (__match_any_sync); each group's sums are gathered by shuffles
//     from the lanes of groups with more than one member, and the group's lowest lane updates the slot once.
//   * Layout: one record's update reads the id and adds to records, bytes and the latest second in the slot's first 32-byte
//     sector, and raises the partition range (and adds the tombstone) in its second.  Two sectors is the least: the id and
//     the six counters take 48 bytes.  The prefix sits in a third sector that only the claimant writes.
// Rehash (growth) and import insert through the same routine (hk_insert).  Finalize compacts the occupied slots into
// kta_hot_key entries, sorts them by (records descending, id ascending) with CUB's radix sort, and gathers the first top_k.
#pragma once
#include <cub/device/device_radix_sort.cuh>

#include "kta_partitioner.cuh"

namespace kta {

constexpr int HK_THREADS = 512;   // 16 warps
constexpr int HK_WARPS = HK_THREADS / 32;
constexpr int HK_PREFIX = KTA_HOT_KEY_PREFIX;
constexpr uint32_t HK_PMIN_BASE = 0x7fffffffu;   // pmin_inv = HK_PMIN_BASE - min partition
constexpr unsigned long long HK_TS_BIAS = 1ull << 63;   // latest = latest_s ^ 2^63: unsigned order = signed order

struct __align__(32) HkSlot {
    // sector 0: read and updated by every record's update
    unsigned long long id;           // 0 = empty (in the side slot: the entry whose id is 0)
    unsigned long long records;
    unsigned long long bytes;
    unsigned long long latest;       // latest_s ^ HK_TS_BIAS
    // sector 1
    unsigned long long tombstones;
    uint32_t pmin_inv;               // HK_PMIN_BASE - min partition
    uint32_t pmax1;                  // max partition + 1
    int32_t key_len;                 // written by the claimant
    uint32_t claim;                  // side slot only: 1 once claimed
    unsigned long long pad;
    // sector 2: written by the claimant
    uint8_t prefix[HK_PREFIX];
};
constexpr int HK_SLOT_BYTES = (int)sizeof(HkSlot);
static_assert(sizeof(HkSlot) == 96, "three 32-byte sectors");
static_assert(sizeof(kta_hot_key) == 88, "kta_hot_key is 88 bytes");

// the table as the kernels see it: slots [0, n) and the side slot at [n]
struct HkTable {
    HkSlot *slot;
    uint64_t n;                          // power of two
    unsigned long long *occupied;        // claims (exact occupancy)
    unsigned int *failed;                // a probe found no slot
};

// a 64-bit finalizer (murmur3's fmix64): ids with close values land far apart
__host__ __device__ __forceinline__ uint64_t hk_mix(uint64_t x) {
    x ^= x >> 33;
    x *= 0xff51afd7ed558ccdull;
    x ^= x >> 33;
    x *= 0xc4ceb9fe1a85ec53ull;
    x ^= x >> 33;
    return x;
}

__host__ __device__ __forceinline__ uint64_t hk_home(uint64_t id, uint64_t n) {
#ifdef __CUDA_ARCH__
    return __umul64hi(hk_mix(id), n);
#else
    return (uint64_t)(((unsigned __int128)hk_mix(id) * n) >> 64);
#endif
}

// One entry's contribution: `records` records with the counters given, the prefix written by `pf(dst)` if this call claims
// the slot.  Returns false (and raises the failure word) only if the probe ran over every slot.
template <class Prefix>
__device__ __noinline__ bool hk_insert(const HkTable &t, uint64_t id, unsigned long long records, unsigned long long tombstones,
                                          unsigned long long bytes, unsigned long long latest, uint32_t pmin_inv, uint32_t pmax1,
                                          int32_t key_len, const Prefix &pf) {
    HkSlot *s = nullptr;
    bool claimed = false;
    if (id == 0) {
        s = t.slot + t.n;
        claimed = atomicCAS(&s->claim, 0u, 1u) == 0u;
    } else {
        uint64_t j = hk_home(id, t.n);
        for (uint64_t i = 0; i < t.n; i++) {
            HkSlot *c = t.slot + j;
            unsigned long long cur = *reinterpret_cast<volatile unsigned long long *>(&c->id);
            if (cur == 0ull) {
                cur = atomicCAS(&c->id, 0ull, (unsigned long long)id);
                if (cur == 0ull) { s = c; claimed = true; break; }
            }
            if (cur == (unsigned long long)id) { s = c; break; }
            if (++j == t.n) j = 0;
        }
        if (!s) {
            atomicExch(t.failed, 1u);
            return false;
        }
    }
    if (claimed) {
        s->key_len = key_len;
        pf(s->prefix);
        atomicAdd(t.occupied, 1ull);
    }
    atomicAdd(&s->records, records);
    atomicAdd(&s->bytes, bytes);
    atomicMax(&s->latest, latest);
    if (tombstones) atomicAdd(&s->tombstones, tombstones);
    atomicMax(&s->pmin_inv, pmin_inv);
    atomicMax(&s->pmax1, pmax1);
    return true;
}

// the first min(len, 32) bytes of a key at address a of source src, zeros after
template <class Src>
struct HkKeyPrefix {
    Src src;
    uint64_t a;
    uint32_t len;
    __device__ __forceinline__ void operator()(uint8_t *dst) const {
        for (uint32_t i = 0; i < (uint32_t)HK_PREFIX; i++) dst[i] = i < len ? (uint8_t)src.byte(a + i) : (uint8_t)0;
    }
};
// a prefix copied as it is (rehash, import)
struct HkCopyPrefix {
    const uint8_t *p;
    __device__ __forceinline__ void operator()(uint8_t *dst) const {
        for (int i = 0; i < HK_PREFIX; i++) dst[i] = p[i];
    }
};

struct HotKeysParams {
    int64_t n;                        // records of the batch
    int64_t tile_lo, tile_hi;         // the tiles of this launch (a slice of the batch)
    const int32_t *partition;
    const int32_t *key_len;
    const int32_t *value_len;
    const int64_t *ts_ms;
    const uint8_t *key_bytes;         // may be an offset pointer; only [tile_base[tile_lo], tile_base[tile_hi]) is read
    const uint64_t *key_tile_base;    // [ntiles + 1]
    int32_t P;
    int32_t shard_world, shard_rank;  // only partitions p % shard_world == shard_rank are counted (world 1: all)
    int32_t stage;                    // bytes of a warp's stage (multiple of 16)
    const uint32_t *tables;           // zlib CRC-32 slicing tables [4][256]
    HkTable table;
};

// one row of 32 records, one per lane: ok = the record is counted, with its id and counters.  Lanes of one id are summed
// in the warp and the group's lowest lane updates the slot.
template <class Src>
__device__ __forceinline__ void hk_row(const HkTable &t, int lane, bool ok, uint64_t id, uint64_t bytes, uint64_t latest, uint32_t p,
                                       bool tomb, int32_t kl, const Src &src, uint64_t ka) {
    const unsigned full = 0xffffffffu;
    const unsigned valid = __ballot_sync(full, ok);
    if (!valid) return;
    unsigned grp = 0;
    if (ok) grp = __match_any_sync(valid, id);
    const unsigned tombs = __ballot_sync(full, ok && tomb);
    // lanes whose group has other members: only their values are exchanged
    const unsigned multi = __ballot_sync(full, ok && (grp & (grp - 1)) != 0);
    unsigned long long b = bytes, lt = latest;
    uint32_t pmin_inv = HK_PMIN_BASE - p, pmax1 = p + 1;
    for (unsigned m = multi; m; m &= m - 1) {
        const int j = __ffs(m) - 1;
        const unsigned long long bj = __shfl_sync(full, bytes, j), lj = __shfl_sync(full, latest, j);   // (the lane's own values)
        const uint32_t pj = __shfl_sync(full, p, j);
        if (j != lane && ((grp >> j) & 1u)) {
            b += bj;
            lt = max(lt, lj);
            pmin_inv = max(pmin_inv, HK_PMIN_BASE - pj);
            pmax1 = max(pmax1, pj + 1);
        }
    }
    if (ok && lane == __ffs(grp) - 1)
        hk_insert(t, id, (unsigned long long)__popc(grp), (unsigned long long)__popc(grp & tombs), b, lt, pmin_inv, pmax1, kl,
                  HkKeyPrefix<Src>{src, ka, (uint32_t)kl});
}

__global__ void __launch_bounds__(HK_THREADS, 2) hot_keys_kernel(const HotKeysParams t) {
    extern __shared__ __align__(16) uint32_t hk_smem[];
    uint32_t *tl = hk_smem;   // [4][256]
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = blockDim.x >> 5;
    const uint32_t stage = smem_u32(hk_smem) + 4u * PC_TABLE_WORDS + (uint32_t)warp * (uint32_t)(t.stage + PC_STAGE_PAD);
    for (int i = threadIdx.x; i < PC_TABLE_WORDS; i += blockDim.x) tl[i] = __ldg(t.tables + i);
    __syncthreads();
    const int64_t span = t.tile_hi - t.tile_lo;
    const int64_t t0 = t.tile_lo + span * blockIdx.x / gridDim.x, t1 = t.tile_lo + span * (blockIdx.x + 1) / gridDim.x;
    for (int64_t tile = t0 + warp; tile < t1; tile += nwarps) {
        const int64_t base = tile * TILE;
        int p[ROWS], kl[ROWS], vl[ROWS];
        int64_t ts[ROWS];
#pragma unroll
        for (int k = 0; k < ROWS; k++) {
            const int64_t r = base + 32 * k + lane;
            const bool valid = r < t.n;
            p[k] = valid ? ld_stream_s32(t.partition + r) : -1;
            kl[k] = valid ? ld_stream_s32(t.key_len + r) : -1;   // (a record past the end is not keyed)
            vl[k] = valid ? ld_stream_s32(t.value_len + r) : -1;
            ts[k] = valid ? ld_stream_s64(t.ts_ms + r) : 0;
        }
        const uint64_t g0 = __ldg(t.key_tile_base + tile), g1 = __ldg(t.key_tile_base + tile + 1);
        const KeyOffsets o = key_offsets(kl, lane);
        const uint8_t *gk = t.key_bytes + g0;
        const bool staged = o.small && g1 - g0 <= (uint64_t)t.stage;
        uint64_t off[ROWS];
        if (o.small) {
#pragma unroll
            for (int k = 0; k < ROWS; k++) off[k] = o.off[k];
        } else {
            pc_wide_offsets(kl, lane, off);
        }
        const uint32_t sbase = stage + (uint32_t)((uintptr_t)gk & 15u);
        if (staged) {
            pc_stage_copy(sbase, gk, (uint32_t)(g1 - g0), lane);
            __syncwarp();
        }
#pragma unroll
        for (int k = 0; k < ROWS; k++) {
            bool ok = kl[k] >= 0 && (unsigned)p[k] < (unsigned)t.P;
            if (t.shard_world > 1) ok = ok && p[k] % t.shard_world == t.shard_rank;
            uint32_t mm = 0, cc = 0;
            const uint64_t ka = staged ? (uint64_t)sbase + off[k] : reinterpret_cast<uint64_t>(gk) + off[k];
            if (ok) {
                if (staged) pc_hashes(PcSmem{}, ka, (uint32_t)kl[k], tl, mm, cc);
                else pc_hashes(PcGlobal{}, ka, (uint32_t)kl[k], tl, mm, cc);
            }
            const uint64_t id = ((uint64_t)cc << 32) | mm;
            const uint64_t bytes = (uint64_t)max(kl[k], 0) + (uint64_t)max(vl[k], 0);
            const int64_t sec = (ts[k] == -1 ? 0 : ts[k]) / 1000;
            const uint64_t latest = (uint64_t)sec ^ HK_TS_BIAS;
            if (staged) hk_row(t.table, lane, ok, id, bytes, latest, (uint32_t)p[k], vl[k] < 0, kl[k], PcSmem{}, ka);
            else hk_row(t.table, lane, ok, id, bytes, latest, (uint32_t)p[k], vl[k] < 0, kl[k], PcGlobal{}, ka);
        }
        __syncwarp();   // the stage is read before the next tile's copy overwrites it
    }
}

__device__ __forceinline__ bool hk_occupied(const HkSlot &s, bool side) { return side ? s.claim != 0u : s.id != 0ull; }

// the slot as a public entry
__device__ __forceinline__ void hk_entry(const HkSlot &s, kta_hot_key &e) {
    e.id = s.id;
    e.records = s.records;
    e.tombstones = s.tombstones;
    e.bytes = s.bytes;
    e.latest_s = (int64_t)(s.latest ^ HK_TS_BIAS);
    e.min_partition = (int32_t)(HK_PMIN_BASE - s.pmin_inv);
    e.max_partition = (int32_t)s.pmax1 - 1;
    e.key_len = s.key_len;
    e.reserved = 0;
    for (int i = 0; i < HK_PREFIX; i++) e.key_prefix[i] = s.prefix[i];
}

// every occupied slot of `from` into `to` (growth)
__global__ void hot_keys_rehash_kernel(const HkSlot *from, uint64_t nfrom, HkTable to) {
    for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i <= nfrom; i += (uint64_t)gridDim.x * blockDim.x) {
        const HkSlot &s = from[i];
        if (!hk_occupied(s, i == nfrom)) continue;
        hk_insert(to, s.id, s.records, s.tombstones, s.bytes, s.latest, s.pmin_inv, s.pmax1, s.key_len, HkCopyPrefix{s.prefix});
    }
}

// every occupied slot as a kta_hot_key at out[cursor++] (while cursor < cap); `records` gets the sum of their records
__global__ void hot_keys_export_kernel(const HkSlot *slot, uint64_t n, unsigned long long *cursor, unsigned long long *records,
                                       kta_hot_key *out, unsigned long long cap) {
    for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i <= n; i += (uint64_t)gridDim.x * blockDim.x) {
        const HkSlot &s = slot[i];
        if (!hk_occupied(s, i == n)) continue;
        const unsigned long long at = atomicAdd(cursor, 1ull);
        if (records) atomicAdd(records, s.records);
        if (at < cap) hk_entry(s, out[at]);
    }
}

// an imported list's entries that break kta.h's rules raise *bad
__global__ void hot_keys_validate_kernel(const kta_hot_key *in, int64_t count, int32_t P, unsigned int *bad) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < count; i += (int64_t)gridDim.x * blockDim.x) {
        const kta_hot_key &e = in[i];
        if (e.records == 0 || e.tombstones > e.records || e.key_len < 0 || e.reserved != 0 || e.min_partition < 0 ||
            e.max_partition >= P || e.min_partition > e.max_partition)
            atomicExch(bad, 1u);
    }
}

__global__ void hot_keys_import_kernel(const kta_hot_key *in, int64_t count, HkTable t) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < count; i += (int64_t)gridDim.x * blockDim.x) {
        const kta_hot_key &e = in[i];
        hk_insert(t, e.id, e.records, e.tombstones, e.bytes, (unsigned long long)e.latest_s ^ HK_TS_BIAS,
                  HK_PMIN_BASE - (uint32_t)e.min_partition, (uint32_t)e.max_partition + 1u, e.key_len, HkCopyPrefix{e.key_prefix});
    }
}

// sort key of an entry: records descending, then id ascending
struct HkSortKey {
    unsigned long long inv_records, id;
};
struct HkSortKeyDecomposer {   // most significant first
    __host__ __device__ ::cuda::std::tuple<unsigned long long &, unsigned long long &> operator()(HkSortKey &k) const {
        return {k.inv_records, k.id};
    }
};

__global__ void hot_keys_sort_keys_kernel(const kta_hot_key *e, int64_t n, HkSortKey *keys, uint32_t *idx) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        keys[i] = HkSortKey{~(unsigned long long)e[i].records, (unsigned long long)e[i].id};
        idx[i] = (uint32_t)i;
    }
}

__global__ void hot_keys_gather_kernel(const kta_hot_key *e, const uint32_t *idx, int64_t k, kta_hot_key *out) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < k; i += (int64_t)gridDim.x * blockDim.x) out[i] = e[idx[i]];
}

inline cudaError_t hot_keys_sort(void *tmp, size_t &tmp_bytes, HkSortKey *keys, HkSortKey *keys_out, uint32_t *idx, uint32_t *idx_out,
                                 int64_t n, cudaStream_t s) {
    return cub::DeviceRadixSort::SortPairs(tmp, tmp_bytes, keys, keys_out, idx, idx_out, n, HkSortKeyDecomposer{}, s);
}

}  // namespace kta
