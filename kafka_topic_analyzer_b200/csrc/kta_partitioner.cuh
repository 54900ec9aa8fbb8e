// kta_partitioner.cuh — the partitioner check (include/kta.h, kta_set_partitioner_check): per partition, how many keyed
// records sit where Kafka's murmur2 partitioner, and where librdkafka's CRC-32 partitioner, would put them at each of up
// to KTA_PARTITIONER_MAX_COUNTS partition counts.
//
// A separate pass behind scan_kernel (and the timeline pass) on the same stream; the scan kernels are not touched.  It
// reads the partition and key_len columns, the tile bases and the key bytes: 8 B per record plus the keys.  Each CTA
// takes a contiguous range of 128-record tiles, one warp per tile:
//   * the warp copies the tile's key span [tile_base[t], tile_base[t + 1]) into its shared-memory stage with coalesced
//     loads (16-byte vectors between byte-wise ends, so nothing outside the span is read), and each lane hashes its four
//     keys from there.  A span larger than the stage (or a key of 1 MiB and more, whose offsets need 64 bits) is hashed
//     straight from global memory;
//   * murmur2 and CRC-32 are computed in one walk over the key's 4-byte words (assembled from aligned words by funnel
//     shifts), CRC-32 by slicing-by-4 from one shared copy of the tables (the steps and the table build are
//     kta_logcrc.cuh's, with zlib's polynomial);
//   * x mod N by Lemire's multiply-high with a precomputed 64-bit reciprocal, exact for every 32-bit x and N < 2^32;
//   * a record's verdict is a (2C + 1)-bit word: bit j murmur2 at counts[j], bit C + j CRC-32 at counts[j], bit 2C
//     neither.  A row of 32 records in one partition (a fetch) is reduced with one ballot per bit and one add per nonzero
//     counter.  Two places to add to, chosen per handle from the shape:
//       - shared memory ((2C + 1) P words fit beside the table and the stages): CTA-private u32 counters, flushed as
//         nonzero u64 adds at the end; a mixed row adds record by record;
//       - global memory otherwise: a mixed row is grouped by partition (__match_any_sync) and each group's counts go out
//         as one 64-bit RED.ADD per nonzero counter.
#pragma once
#include "kta_kernels.cuh"
#include "kta_logcrc.cuh"

namespace kta {

constexpr int PC_THREADS = 512;                        // 16 warps
constexpr int PC_WARPS = PC_THREADS / 32;
constexpr int PC_MAX_COUNTS = KTA_PARTITIONER_MAX_COUNTS;
// A CTA takes at most 2^24 tiles (2^31 records) of one launch, so its u32 counters cannot overflow; the host raises the
// grid for larger scans
constexpr int64_t PC_MAX_CTA_TILES = (int64_t)1 << 24;
constexpr int PC_STAGE_MIN = 1024, PC_STAGE_MAX = 16384;   // key bytes of one warp's stage (multiple of 16)
constexpr int PC_STAGE_PAD = 32;                           // alignment shift (< 16) + the aligned word past the end
constexpr uint32_t PC_NONE = 0xffffffffu;                  // partition key of a record that is not checked
constexpr uint32_t ZLIB_CRC32_POLY = 0xEDB88320u;          // reflected
constexpr uint32_t MURMUR2_SEED = 0x9747b28cu, MURMUR2_M = 0x5bd1e995u;
constexpr int PC_TABLE_WORDS = 4 * 256;

struct PartitionerParams {
    int64_t n, ntiles;
    const int32_t *partition;
    const int32_t *key_len;
    const uint8_t *key_bytes;        // may be an offset pointer; only [tile_base[0], tile_base[ntiles]) is read
    const uint64_t *key_tile_base;   // [ntiles + 1]
    int32_t P;
    int32_t shard_world, shard_rank; // only partitions p % shard_world == shard_rank are counted (world 1: all)
    int32_t C;                       // partition counts checked, 1..PC_MAX_COUNTS
    int32_t stage;                   // bytes of a warp's stage (multiple of 16)
    uint32_t count[PC_MAX_COUNTS];   // N_j
    uint64_t recip[PC_MAX_COUNTS];   // floor((2^64 - 1) / N_j) + 1 (mod 2^64)
    const uint32_t *tables;          // zlib CRC-32 slicing tables [4][256]
    unsigned long long *out;         // [2C + 1][P]
};

// x mod N for any 32-bit x and 1 <= N < 2^32 (Lemire, Kaser, Kurz 2019, "Faster remainder by direct computation"):
// with c = ceil(2^64 / N), the low 64 bits of c x times N, high word.  N = 1 has c = 2^64 = 0 (mod 2^64): 0, as it must.
__host__ __device__ __forceinline__ uint32_t pc_mod(uint32_t x, uint64_t c, uint32_t N) {
    const uint64_t low = c * (uint64_t)x;
#ifdef __CUDA_ARCH__
    return (uint32_t)__umul64hi(low, (uint64_t)N);
#else
    return (uint32_t)(((unsigned __int128)low * N) >> 64);
#endif
}

// a key's bytes from the stage (shared-window addresses)
struct PcSmem {
    __device__ __forceinline__ uint32_t word(uint64_t a) const { return lds32((uint32_t)a); }   // a is 4-aligned
    __device__ __forceinline__ uint32_t byte(uint64_t a) const {
        uint32_t v;
        asm volatile("ld.shared.u8 %0, [%1];" : "=r"(v) : "r"((uint32_t)a));
        return v;
    }
};
// a key's bytes straight from global memory (generic addresses).  An aligned word that holds one of the key's bytes lies
// inside the key's allocation.
struct PcGlobal {
    __device__ __forceinline__ uint32_t word(uint64_t a) const { return __ldg(reinterpret_cast<const uint32_t *>(a)); }
    __device__ __forceinline__ uint32_t byte(uint64_t a) const { return __ldg(reinterpret_cast<const uint8_t *>(a)); }
};

// Kafka's Utils.murmur2 and zlib's CRC-32 of the len bytes at address a, in one walk over the key's 4-byte words.  The
// words are read aligned and joined by a funnel shift; only aligned words that hold a key byte are read.
template <class Src>
__device__ __forceinline__ void pc_hashes(const Src &src, uint64_t a, uint32_t len, const uint32_t *tl, uint32_t &mm, uint32_t &cc) {
    uint32_t h = MURMUR2_SEED ^ len, c = 0xffffffffu;
    const uint32_t sh = 8u * (uint32_t)(a & 3u);
    uint64_t w = a & ~(uint64_t)3;
    const uint32_t n4 = len >> 2;
    uint32_t lo = (sh && n4) ? src.word(w) : 0u;
    for (uint32_t i = 0; i < n4; i++, w += 4) {
        uint32_t k;
        if (sh) {
            const uint32_t hi = src.word(w + 4);
            k = __funnelshift_r(lo, hi, sh);
            lo = hi;
        } else {
            k = src.word(w);
        }
        c = crc_word<1>(c, k, tl);
        k *= MURMUR2_M;
        k ^= k >> 24;
        k *= MURMUR2_M;
        h *= MURMUR2_M;
        h ^= k;
    }
    const uint32_t rest = len & 3u;
    if (rest) {
        // Java's switch (length % 4): case 3 folds byte 2 << 16, case 2 byte 1 << 8, case 1 byte 0, then one multiply
        const uint64_t t = a + (uint64_t)(len & ~3u);
        const uint32_t b0 = src.byte(t), b1 = rest > 1 ? src.byte(t + 1) : 0u, b2 = rest > 2 ? src.byte(t + 2) : 0u;
        h ^= (b2 << 16) ^ (b1 << 8) ^ b0;
        h *= MURMUR2_M;
        c = crc_byte<1>(c, b0, tl);
        if (rest > 1) c = crc_byte<1>(c, b1, tl);
        if (rest > 2) c = crc_byte<1>(c, b2, tl);
    }
    h ^= h >> 13;
    h *= MURMUR2_M;
    h ^= h >> 15;
    mm = h;
    cc = c ^ 0xffffffffu;
}

// the verdict of one keyed record of partition p
__device__ __forceinline__ uint32_t pc_verdict(const PartitionerParams &t, uint32_t p, uint32_t mm, uint32_t cc) {
    const uint32_t pos = mm & 0x7fffffffu;   // Utils.toPositive
    uint32_t v = 0;
#pragma unroll
    for (int j = 0; j < PC_MAX_COUNTS; j++) {
        if (j < t.C) {
            v |= (pc_mod(pos, t.recip[j], t.count[j]) == p ? 1u : 0u) << j;
            v |= (pc_mod(cc, t.recip[j], t.count[j]) == p ? 1u : 0u) << (t.C + j);
        }
    }
    return v ? v : 1u << (2 * t.C);
}

// one row of 32 records, one per lane: key = the record's partition (PC_NONE: not checked), v its verdict
template <bool SMEM>
__device__ __forceinline__ void pc_add(const PartitionerParams &t, uint32_t cnt_smem, int lane, uint32_t key, uint32_t v) {
    const unsigned full = 0xffffffffu;
    const uint32_t k0 = __shfl_sync(full, key, 0);
    const bool uniform = __all_sync(full, key == k0);
    if (uniform && k0 == PC_NONE) return;
    const int nv = 2 * t.C + 1;
    if (SMEM && !uniform) {
        // shared-memory adds to distinct counters proceed in parallel: each lane adds its own record's bits
        if (key != PC_NONE)
            for (uint32_t m = v; m; m &= m - 1) red_shared_add(cnt_smem + 4u * ((uint32_t)(__ffs(m) - 1) * (uint32_t)t.P + key), 1u);
        return;
    }
    const unsigned grp = uniform ? full : __match_any_sync(full, key);
    const int leader = __ffs(grp) - 1;
    for (int b = 0; b < nv; b++) {
        const uint32_t c = __popc(__ballot_sync(full, (v >> b) & 1u) & grp);
        // a uniform row spreads its adds over the lanes (lane b adds counter b); a mixed row's group leader adds them all
        if (c && key != PC_NONE && lane == (uniform ? (b & 31) : leader)) {
            if (SMEM) red_shared_add(cnt_smem + 4u * ((uint32_t)b * (uint32_t)t.P + key), c);
            else atomicAdd(t.out + (size_t)b * (size_t)t.P + key, (unsigned long long)c);
        }
    }
}

// byte offsets of the lane's four keys inside a tile whose longest key is 1 MiB or more (64-bit exclusive scan)
__device__ __noinline__ void pc_wide_offsets(const int (&kl)[ROWS], int lane, uint64_t (&off)[ROWS]) {
    uint64_t before = 0;
#pragma unroll
    for (int k = 0; k < ROWS; k++) {
        const uint64_t v = (uint64_t)max(kl[k], 0);
        uint64_t inc = v;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
            const uint64_t x = __shfl_up_sync(0xffffffffu, inc, d);
            if (lane >= d) inc += x;
        }
        off[k] = before + inc - v;
        before += __shfl_sync(0xffffffffu, inc, 31);
    }
}

// copies the n bytes at global address g to the stage at shared address s, where s = g (mod 16): byte-wise up to the
// first 16-byte boundary and after the last one, 16-byte vectors between; nothing outside [g, g + n) is read
__device__ __forceinline__ void pc_stage_copy(uint32_t s, const uint8_t *g, uint32_t n, int lane) {
    const uint32_t head = min(n, (uint32_t)((16u - ((uintptr_t)g & 15u)) & 15u));
    const uint32_t nv = (n - head) >> 4, tail = n - head - 16u * nv;
    if ((uint32_t)lane < head) asm volatile("st.shared.u8 [%0], %1;" ::"r"(s + lane), "r"((uint32_t)__ldg(g + lane)));
    const uint4 *gv = reinterpret_cast<const uint4 *>(g + head);
    for (uint32_t i = lane; i < nv; i += 32) {
        const uint4 q = __ldg(gv + i);
        asm volatile("st.shared.v4.u32 [%0], {%1, %2, %3, %4};" ::"r"(s + head + 16u * i), "r"(q.x), "r"(q.y), "r"(q.z), "r"(q.w));
    }
    const uint32_t t0 = head + 16u * nv;
    if ((uint32_t)lane < tail) asm volatile("st.shared.u8 [%0], %1;" ::"r"(s + t0 + lane), "r"((uint32_t)__ldg(g + t0 + lane)));
}

template <bool SMEM>
__global__ void __launch_bounds__(PC_THREADS) partitioner_kernel(const PartitionerParams t) {
    extern __shared__ __align__(16) uint32_t pc_smem[];
    uint32_t *tl = pc_smem;                                         // [4][256]
    uint32_t *cnt = pc_smem + PC_TABLE_WORDS;                       // [2C + 1][P] (SMEM)
    const int ncnt = SMEM ? (2 * t.C + 1) * t.P : 0;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = blockDim.x >> 5;
    const uint32_t cnt_smem = smem_u32(cnt);
    const uint32_t stage0 = smem_u32(pc_smem) + 4u * (uint32_t)((PC_TABLE_WORDS + ncnt + 3) & ~3);
    const uint32_t stage = stage0 + (uint32_t)warp * (uint32_t)(t.stage + PC_STAGE_PAD);
    for (int i = threadIdx.x; i < PC_TABLE_WORDS; i += blockDim.x) tl[i] = __ldg(t.tables + i);
    for (int i = threadIdx.x; i < ncnt; i += blockDim.x) cnt[i] = 0;
    __syncthreads();
    const int64_t t0 = t.ntiles * blockIdx.x / gridDim.x, t1 = t.ntiles * (blockIdx.x + 1) / gridDim.x;
    for (int64_t tile = t0 + warp; tile < t1; tile += nwarps) {
        const int64_t base = tile * TILE;
        int p[ROWS], kl[ROWS];
#pragma unroll
        for (int k = 0; k < ROWS; k++) {
            const int64_t r = base + 32 * k + lane;
            const bool valid = r < t.n;
            p[k] = valid ? ld_stream_s32(t.partition + r) : -1;
            kl[k] = valid ? ld_stream_s32(t.key_len + r) : -1;   // (a record past the end is not keyed)
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
            uint32_t v = 0;
            if (ok) {
                uint32_t mm, cc;
                if (staged) pc_hashes(PcSmem{}, (uint64_t)sbase + off[k], (uint32_t)kl[k], tl, mm, cc);
                else pc_hashes(PcGlobal{}, reinterpret_cast<uint64_t>(gk) + off[k], (uint32_t)kl[k], tl, mm, cc);
                v = pc_verdict(t, (uint32_t)p[k], mm, cc);
            }
            pc_add<SMEM>(t, cnt_smem, lane, ok ? (uint32_t)p[k] : PC_NONE, v);
        }
        __syncwarp();   // the stage is read before the next tile's copy overwrites it
    }
    if (SMEM) {
        __syncthreads();
        for (int i = threadIdx.x; i < ncnt; i += blockDim.x) {
            const uint32_t c = cnt[i];
            if (c) atomicAdd(t.out + i, (unsigned long long)c);   // [b][P] in both layouts
        }
    }
}

// test hook (kta_partitioner_hash_host): the pass's own hash functions over n keys in global memory, thread per key
__global__ void partitioner_hash_kernel(int64_t n, const int32_t *key_len, const uint64_t *key_off, const uint8_t *key_bytes,
                                        const uint32_t *tables, uint32_t *murmur2, uint32_t *crc32) {
    __shared__ uint32_t tl[PC_TABLE_WORDS];
    for (int i = threadIdx.x; i < PC_TABLE_WORDS; i += blockDim.x) tl[i] = tables[i];
    __syncthreads();
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        uint32_t mm = 0, cc = 0;
        if (key_len[i] >= 0)
            pc_hashes(PcGlobal{}, reinterpret_cast<uint64_t>(key_bytes + key_off[i]), (uint32_t)key_len[i], tl, mm, cc);
        murmur2[i] = mm;
        crc32[i] = cc;
    }
}

}  // namespace kta
