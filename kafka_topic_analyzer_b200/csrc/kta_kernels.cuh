// kta_kernels.cuh — sm_90a (H100) device code for the message-scan metric path.
//
// What the kernels compute is exactly what the reference computes once per polled message
// (src/kafka.rs:107-109) in MessageMetrics::handle_message (src/metric.rs:206-253) and
// LogCompactionInMemoryMetrics::handle_message (src/metric.rs:288-305, hash src/fnv32.rs:92-101),
// restructured for an H100: records arrive as SoA columns resident in HBM, one CTA walks 1024-record
// tiles, per-partition counters live in shared memory (u32 + carry word, native ATOMS), the tile's
// packed key bytes are staged global→shared with one bulk async copy (cp.async.bulk / UBLKCP, mbarrier
// completion, double buffered), keys are hashed from shared memory, and the alive-key state is a
// compact open-addressed table of 64-bit last-writer stamps (hash | seq | alive) sized by the number
// of distinct key hashes (8 bytes each: 80 MB of entries for 1e7 keys) rather than by the 2^32 possible hashes, with a
// 32 MiB seen cache in front of it that fits the 50 MB L2, so that most records need one L2 hit, not a DRAM sector.
// No tensor cores: there is no dense contraction anywhere on this path.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include <type_traits>

#include "../../include/kta.h"

namespace kta {

#ifndef KTA_SCAN_THREADS
#define KTA_SCAN_THREADS 1024
#endif
constexpr int MAX_THREADS = KTA_SCAN_THREADS;  // one persistent CTA per SM, up to 32 autonomous warps
constexpr int TILE = KTA_KEY_TILE;        // records per warp tile (128)
constexpr int ROWS = TILE / 32;           // records per lane per tile
constexpr int NB = KTA_HIST_BUCKETS;      // 32 log2 buckets
// Per warp: 128 bytes (2 mbarriers + scratch) and a double-buffered key stage.  The stage size is chosen per launch
// from the batch's mean key length (ScanParams::keybuf): 18 B/record for the 16-byte-key benchmark, up to 128 B/record
// for long keys, trading warps per SM for stage bytes when shared memory runs out.  A stage has 32 bytes of slack for
// the (harmless, <= 23 byte) over-read of the last words.
constexpr int KEYBUF_MIN = TILE * 18 + 32, KEYBUF_MAX = TILE * 128 + 32, KEYBUF_SLACK = 32;
__host__ __device__ inline size_t warp_smem_bytes(bool hash, int keybuf, bool exact = false) {
    (void)exact;   // MODE_EXACT's queue of table-bound records lives in the key stage the tile has just finished with
    return hash ? 128 + 2 * (size_t)keybuf : 128;
}
constexpr uint32_t FNV_BASIS = 0x811c9dc5u;  // src/fnv32.rs:80
constexpr uint32_t FNV_MULT = 0x811c9dc5u;   // src/fnv32.rs:97 (NOT the FNV prime — kept for parity)
constexpr int FOLD_TILES = 8;             // every warp checks the CTA's 16-bit-split sums after every 8th tile of its own

// shared-memory counter rows (each row = P u32 words):
//   0..31 key-size buckets, 32 null keys | 33..64 value-size buckets, 65 tombstones |
//   66 Σ(key_len & 0xffff), 67 Σ(key_len >> 16), 68 Σ(value_len & 0xffff), 69 Σ(value_len >> 16)
// bucket(len) = bfind(len) + 1: 0 for len 0, 1 + floor(log2 len) otherwise, and 32 for len = -1 (null),
// so "null" needs neither a branch nor a select.
constexpr int ROW_V = NB + 1, ROW_KSUM = 2 * NB + 2, ROW_VSUM = 2 * NB + 4, SMEM_ROWS = 2 * NB + 6;
enum ScanMode { MODE_COUNTERS = 0, MODE_HLL = 1, MODE_EXACT = 2 };

// words of the u64 "sums" state: khist[P][32] | vhist[P][32] | ksum[P] | vsum[P] | knull[P] | bad
__host__ __device__ inline size_t sums_words(int P) { return (size_t)P * (2 * NB + 3) + 1; }
// counter rows, then the CTA scratch: one 128-byte line (word 0: the CTA's cached copy of the HLL floor, word 1:
// tiles finished CTA-wide)
constexpr int CTA_SCRATCH = 128;
__host__ __device__ inline size_t smem_counter_bytes(int P) { return (((size_t)P * SMEM_ROWS * 4 + 127) & ~(size_t)127) + CTA_SCRATCH; }

struct ScanParams {
    int64_t n;
    uint64_t seq_base;
    const int32_t *partition;
    const int64_t *ts_ms;
    const int32_t *key_len;
    const int32_t *value_len;
    const uint8_t *key_bytes;        // may be an offset pointer; only [tile_base..] is dereferenced
    const uint64_t *key_tile_base;   // [ntiles+1] absolute byte offsets relative to key_bytes
    const uint64_t *seq;             // optional explicit seq column
    int64_t ntiles;
    int32_t P;                       // partitions of the topic (ids 0..P-1)
    int32_t shard_world, shard_rank; // this handle scans only partitions p with p % shard_world == shard_rank (1, 0 = all)
    int32_t Pc;                      // counter columns = owned partitions; column c holds partition c * shard_world + shard_rank
    uint32_t shard_magic;            // ceil(2^32 / shard_world): p / shard_world = mulhi(p, magic) for p < 2^20
    int32_t hll_p;                   // HLL index bits (MODE_HLL)
    uint64_t stage_limit;            // bytes readable from key_bytes by 16-byte bulk copies, rounded DOWN to 16; 0 = staging not allowed
    int32_t keybuf;                  // bytes of one key stage (multiple of 16, incl. KEYBUF_SLACK)
    int32_t pad0;
    unsigned long long *sums;        // [sums_words(P)]
    long long *minmax;               // [0] min raw ts_ms, [1] max raw ts_ms, [2] min size, [3] max size (as u64)
    uint32_t *hll;                   // [1 << hll_p] registers (one u32 each so that RED.MAX applies)
    uint32_t *hll_floor;             // [0] lower bound of every register (monotone; lets most records skip the
                                     // table), [1..HLL_SLICES] per-slice minima it is derived from
    unsigned long long *alive_table; // [2 * alive_pairs] stamps: hash(32) | seq - alive_origin + 1 (31) | alive(1); ~0 = empty
    uint32_t alive_pairs;            // table size in 16-byte pairs of slots (any value >= 1, not only powers of two)
    int32_t alive_only;              // 1: MODE_EXACT re-run after the table grew — stamps only, no counters / extrema
    uint64_t alive_origin;           // seq that field value 1 stands for (moved forward by a rebase)
    uint64_t alive_fbase;            // seq_base - alive_origin + 1: the field of record 0 when seq is implicit
    unsigned long long *alive_count; // scratch u64 words: [0] alive entries, [1] export cursor, [2] occupied slots (count kernels)
    uint32_t *alive_cache;           // [2^ALIVE_CACHE_SET_BITS] seen cache of this batch (cleared by the host before the launch), or NULL
    int32_t alive_wave_shift;        // wave of a record = 1 + min((field - alive_wave_base) >> alive_wave_shift, 126): a monotone
    uint32_t alive_wave_base;        //   function of seq (field = seq - origin + 1); base = the field of the batch's first record
    uint32_t *alive_status;          // [0] stamps that found no slot (table too full: host grows it and re-runs the
                                     //     batch), [1] records whose seq lies outside the 31-bit window of the table
    uint32_t *hash_out;              // per-record hash capture (CAPTURE kernels only; test hook), 0 for null keys
};

// ------------------------------------------------------------------------------------------------
// small PTX wrappers
// ------------------------------------------------------------------------------------------------
// shared-window address of a generic pointer; volatile so that it is computed once and kept, not rematerialised
// (S2UR + ULEA) in front of every shared-memory reduction
__device__ __forceinline__ uint32_t smem_u32(const void *p) {
    uint32_t a;
    asm volatile("{ .reg .u64 t; cvta.to.shared.u64 t, %1; cvt.u32.u64 %0, t; }" : "=r"(a) : "l"(p));
    return a;
}

__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count));
}
__device__ __forceinline__ void fence_mbar_init() {
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint32_t bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "KTA_WAIT_%=:\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
        "@p bra KTA_DONE_%=;\n\t"
        "bra KTA_WAIT_%=;\n\t"
        "KTA_DONE_%=:\n\t}"
        ::"r"(bar), "r"(parity)
        : "memory");
}
// 1-D bulk async copy global → shared (TMA engine, no tensor map), completion on an mbarrier
__device__ __forceinline__ void bulk_g2s(uint32_t dst_smem, const void *src_gmem, uint32_t bytes, uint32_t bar) {
    asm volatile(
        "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
        ::"r"(dst_smem), "l"(src_gmem), "r"(bytes), "r"(bar)
        : "memory");
}
__device__ __forceinline__ void bulk_g2s(uint32_t dst_smem, const void *src_gmem, uint32_t bytes, uint32_t bar, uint64_t pol) {
    asm volatile(
        "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1], %2, [%3], %4;"
        ::"r"(dst_smem), "l"(src_gmem), "r"(bytes), "r"(bar), "l"(pol)
        : "memory");
}
// shared-memory reductions on 32-bit shared-window addresses (no generic→shared conversion in the loop)
__device__ __forceinline__ void red_shared_add(uint32_t addr, uint32_t v) {
    asm volatile("red.shared.add.u32 [%0], %1;" ::"r"(addr), "r"(v) : "memory");
}
// [addr] += v unless v == 0, as ONE predicated instruction (no branch, no reconvergence bookkeeping)
__device__ __forceinline__ uint32_t hi32(long long v) {   // the high word, without a 64-bit shift the compiler then carries around
    uint32_t hi;
    asm("{ .reg .b32 lo; mov.b64 {lo, %0}, %1; }" : "=r"(hi) : "l"(v));
    return hi;
}
__device__ __forceinline__ long long pack64(uint32_t lo, uint32_t hi) {
    long long v;
    asm("mov.b64 %0, {%1, %2};" : "=l"(v) : "r"(lo), "r"(hi));
    return v;
}
__device__ __forceinline__ void red_shared_add_nz(uint32_t addr, uint32_t v) {
    asm volatile("{ .reg .pred p; setp.ne.u32 p, %1, 0; @p red.shared.add.u32 [%0], %1; }" ::"r"(addr), "r"(v) : "memory");
}
__device__ __forceinline__ uint4 lds128(uint32_t addr) {
    uint4 v;
    asm volatile("ld.shared.v4.u32 {%0, %1, %2, %3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "r"(addr));
    return v;
}
__device__ __forceinline__ uint32_t lds32(uint32_t addr) {
    uint32_t v;
    asm volatile("ld.shared.u32 %0, [%1];" : "=r"(v) : "r"(addr));
    return v;
}
__device__ __forceinline__ uint32_t bfind_u32(uint32_t x) {  // index of the most significant set bit, 0xffffffff for 0
    uint32_t r;
    asm("bfind.u32 %0, %1;" : "=r"(r) : "r"(x));
    return r;
}
// streaming loads: read once, do not allocate in L1
__device__ __forceinline__ int32_t ld_stream_s32(const int32_t *p) {
    int32_t v;
    asm volatile("ld.global.nc.L1::no_allocate.s32 %0, [%1];" : "=r"(v) : "l"(p));
    return v;
}
__device__ __forceinline__ int64_t ld_stream_s64(const int64_t *p) {
    int64_t v;
    asm volatile("ld.global.nc.L1::no_allocate.s64 %0, [%1];" : "=l"(v) : "l"(p));
    return v;
}
__device__ __forceinline__ uint64_t ld_stream_u64(const uint64_t *p) {
    uint64_t v;
    asm volatile("ld.global.nc.L1::no_allocate.u64 %0, [%1];" : "=l"(v) : "l"(p));
    return v;
}
// the same with an L2 eviction policy (MODE_EXACT: the stream must not push the alive table out of L2)
__device__ __forceinline__ int32_t ld_stream_s32(const int32_t *p, uint64_t pol) {
    int32_t v;
    asm volatile("ld.global.nc.L1::no_allocate.L2::cache_hint.s32 %0, [%1], %2;" : "=r"(v) : "l"(p), "l"(pol));
    return v;
}
__device__ __forceinline__ int64_t ld_stream_s64(const int64_t *p, uint64_t pol) {
    int64_t v;
    asm volatile("ld.global.nc.L1::no_allocate.L2::cache_hint.s64 %0, [%1], %2;" : "=l"(v) : "l"(p), "l"(pol));
    return v;
}
__device__ __forceinline__ uint32_t ld_cg_u32(const uint32_t *p) {  // L2-coherent read
    uint32_t v;
    asm volatile("ld.global.cg.u32 %0, [%1];" : "=r"(v) : "l"(p));
    return v;
}
__device__ __forceinline__ void red_global_max(uint32_t *p, uint32_t v) {  // fire-and-forget, never stalls the warp
    asm volatile("red.global.max.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}

// ------------------------------------------------------------------------------------------------
// the reference hash, src/fnv32.rs:92-101: for each byte { hash ^= byte; hash *= 0x811c9dc5 }
// The integer ALU pipe is the busiest pipe of the fused kernel (ncu, profiles/), so bytes 1..3 of a
// word are brought down with a multiply-high on the FMA pipe instead of a shift on the ALU pipe;
// the byte mask is folded into the xor (one LOP3: h ^ (w & 0xff)).
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t fnv_step(uint32_t h, uint32_t byte) { return (h ^ byte) * FNV_MULT; }

__device__ __forceinline__ uint32_t shr_fma(uint32_t w, uint32_t two_pow_32_minus_s) {
    uint32_t r;
    asm("mul.hi.u32 %0, %1, %2;" : "=r"(r) : "r"(w), "r"(two_pow_32_minus_s));
    return r;
}

__device__ __forceinline__ uint32_t fnv_word(uint32_t h, uint32_t w) {
    h = fnv_step(h, w & 0xffu);
    h = fnv_step(h, shr_fma(w, 1u << 24) & 0xffu);
    h = fnv_step(h, shr_fma(w, 1u << 16) & 0xffu);
    h = fnv_step(h, shr_fma(w, 1u << 8));
    return h;
}

// key at byte offset `a` of the warp's staged key buffer (aligned word loads + funnel shift)
__device__ __forceinline__ uint32_t fnv_smem(uint32_t buf_addr, uint32_t a, int len) {
    uint32_t h = FNV_BASIS;
    const uint32_t wp = buf_addr + (a & ~3u);
    const uint32_t sh = (a & 3u) * 8u;
    uint32_t lo = lds32(wp);
    int j = 0;
    for (; j + 4 <= len; j += 4) {
        const uint32_t hi = lds32(wp + j + 4);
        h = fnv_word(h, __funnelshift_r(lo, hi, sh));
        lo = hi;
    }
    const int rem = len - j;
    if (rem > 0) {
        const uint32_t hi = lds32(wp + j + 4);
        uint32_t w = __funnelshift_r(lo, hi, sh);
        for (int r = 0; r < rem; r++) {
            h = fnv_step(h, w & 0xffu);
            w >>= 8;
        }
    }
    return h;
}

// key read straight from global memory (tiles whose key span does not fit the staging buffer,
// misaligned key buffers, and the kta_fnv32 test hook)
__device__ __forceinline__ uint32_t fnv_global(const uint8_t *key, int len) {
    uint32_t h = FNV_BASIS;
    for (int j = 0; j < len; j++) h = fnv_step(h, (uint32_t)__ldg(key + j));
    return h;
}

// ------------------------------------------------------------------------------------------------
// EXTENSION (not in the reference): HyperLogLog over the 32-bit reference hash, remixed by murmur3
// fmix32 (a bijection, so distinct reference hashes stay distinct).  Registers live in global memory
// (L2 resident) and are raised with RED.MAX — fire and forget, the warp never waits for L2.
// `floor` is a lower bound of every register, so a record whose rho <= floor cannot change anything
// and never touches the table — after warm-up that is all but 2^-floor of them.
// rho <= floor  ⇔  the top `floor` bits below the index bits are not all zero  ⇔  (x & skip_mask) != 0.
// ------------------------------------------------------------------------------------------------
__host__ __device__ __forceinline__ uint32_t hll_mix(uint32_t h) {
#ifdef __CUDA_ARCH__
    // same function; the three right shifts ride the FMA pipe (mul.hi by 2^(32-s)) because the integer ALU pipe is
    // the busiest pipe of the fused kernel
    h ^= shr_fma(h, 1u << 16);
    h *= 0x85ebca6bu;
    h ^= shr_fma(h, 1u << 19);
    h *= 0xc2b2ae35u;
    h ^= shr_fma(h, 1u << 16);
    return h;
#else
    h ^= h >> 16;
    h *= 0x85ebca6bu;
    h ^= h >> 13;
    h *= 0xc2b2ae35u;
    h ^= h >> 16;
    return h;
#endif
}

// the inverse bijection (the alive-key table stores mixed hashes; exports and the tests want the reference hash back)
__host__ __device__ __forceinline__ uint32_t hll_unmix(uint32_t h) {
    h ^= h >> 16;
    h *= 0x7ed1b41du;              // 0xc2b2ae35^-1 mod 2^32
    h ^= (h >> 13) ^ (h >> 26);
    h *= 0xa5cb9243u;              // 0x85ebca6b^-1 mod 2^32
    h ^= h >> 16;
    return h;
}

__device__ __forceinline__ uint32_t hll_skip_mask(int p, uint32_t floor) {
    const uint32_t f = min(floor, (uint32_t)(32 - p));
    return f ? (((1u << f) - 1u) << (32 - p - f)) : 0u;
}

__device__ __forceinline__ void hll_raise(uint32_t *regs, int p, uint32_t x) {
    const uint32_t rest = x << p;
    const uint32_t rho = min((uint32_t)__clz((int)rest) + 1u, (uint32_t)(32 - p + 1));
    red_global_max(regs + (x >> (32 - p)), rho);
}

__device__ __forceinline__ void hll_update(uint32_t *regs, int p, uint32_t skip_mask, uint32_t hash) {
    const uint32_t x = hll_mix(hash);
    if ((x & skip_mask) == 0) hll_raise(regs, p, x);
}

// Keeping the floor fresh: the register file is cut into HLL_SLICES slices; now and then a warp takes the min
// of ONE slice (a few independent L2 loads per lane), publishes it, and re-derives floor = min over the
// published slice minima.  The min over a snapshot of monotone registers is a valid lower bound for every
// later moment, so the filter stays exact.  aux[0] = floor, aux[1 + s] = min of slice s.
constexpr int HLL_SLICES = 64;
__device__ __noinline__ void hll_refresh_slice(const uint32_t *regs, int p, uint32_t *aux, uint32_t slice, int lane) {
    const uint32_t n = 1u << p;
    const uint32_t per = n >= HLL_SLICES ? n / HLL_SLICES : n;   // tiny sketches: every slice is the whole file
    const uint32_t base = n >= HLL_SLICES ? slice * per : 0u;
    uint32_t m = 255;
    for (uint32_t i = lane; i < per; i += 32) m = min(m, ld_cg_u32(regs + base + i));
    m = __reduce_min_sync(0xffffffffu, m);
    if (lane == 0 && m) atomicMax(aux + 1 + slice, m);
    uint32_t f;
    {
        const uint32_t s0 = (uint32_t)lane, s1 = (uint32_t)lane + 32u;
        const uint32_t v0 = s0 == slice ? m : ld_cg_u32(aux + 1 + s0);
        const uint32_t v1 = s1 == slice ? m : ld_cg_u32(aux + 1 + s1);
        f = min(v0, v1);
    }
    f = __reduce_min_sync(0xffffffffu, f);
    if (lane == 0 && f) atomicMax(aux, f);
}

// ------------------------------------------------------------------------------------------------
// per-partition counters (src/metric.rs:74-100, inc_*).  Derived at read-back: key_non_null = Σ key buckets,
// alive = Σ value buckets, total = key_non_null + key_null, tombstones = total − alive.
//
// SMEM = true: CTA-private u32 rows in shared memory (layout above), updated with RED.SHARED (no return
// value, nothing to wait for), branch-free per record.  64-bit byte sums are kept as two u32 words —
// Σ(len & 0xffff) and Σ(len >> 16) — that every warp checks after every FOLD_TILES-th tile of its own and drains into
// the global u64 sums with an atomic exchange before they can overflow (exact).
// SMEM = false: straight 64-bit global atomics (P too large for shared memory).
// ------------------------------------------------------------------------------------------------
template <bool SMEM>
struct Counters {
    uint32_t sbase;            // shared-window address of row 0
    uint32_t *s;               // the same, as a generic pointer (flush / fold)
    unsigned long long *g;
    int P;                     // counter COLUMNS (= partitions, or the owned ones of a partition-sharded scan)
    int Pg, G, R;              // partitions of the topic; column c is partition c * G + R
    __device__ __forceinline__ int part(int c) const { return c * G + R; }
    // row r of column p += c (uniform-row path, flush)
    __device__ __forceinline__ void row_add(int r, int p, uint32_t c) const {
        if (SMEM) red_shared_add(sbase + 4u * (uint32_t)(r * P + p), c);
        else if (r < NB) atomicAdd(&g[(size_t)part(p) * NB + r], (unsigned long long)c);                       // khist
        else if (r == NB) atomicAdd(&g[(size_t)Pg * (2 * NB + 2) + part(p)], (unsigned long long)c);          // knull
        else if (r < ROW_V + NB) atomicAdd(&g[(size_t)(Pg + part(p)) * NB + (r - ROW_V)], (unsigned long long)c);  // vhist
        // r == ROW_V + NB (tombstones) is derived, nothing to store
    }
    __device__ __forceinline__ void sum_add(int which /*0 key, 1 value*/, int p, uint32_t v) const {
        if (SMEM) {
            const uint32_t a = sbase + 4u * (uint32_t)((ROW_KSUM + 2 * which) * P + p);
            red_shared_add(a, v & 0xffffu);
            red_shared_add_nz(a + 4u * (uint32_t)P, v >> 16);
        } else if (v) atomicAdd(&g[(size_t)Pg * (2 * NB + which) + part(p)], (unsigned long long)v);
    }
    // one record, partition already validated; MessageMetrics::handle_message's increments (metric.rs:215-244).
    // buckets(): the two counting increments.  Lanes that hit the same counter are merged by the hardware
    // (ATOMS.POPC.INC), so rows of one partition cost no more than scattered rows.
    __device__ __forceinline__ void buckets(int p, int kl, int vl) const {
        const int kb = (int)bfind_u32((uint32_t)kl) + 1;   // 32 = null key (metric.rs:228), else its size bucket (:220)
        const int vb = (int)bfind_u32((uint32_t)vl) + 1;   // 32 = tombstone (:243), else its size bucket (:239)
        if (SMEM) {
            const uint32_t P4 = 4u * (uint32_t)P, pa = sbase + 4u * (uint32_t)p;
            red_shared_add(pa + (uint32_t)kb * P4, 1u);
            red_shared_add(pa + (uint32_t)(ROW_V + vb) * P4, 1u);
        } else {
            row_add(kb, p, 1u);
            row_add(ROW_V + vb, p, 1u);
        }
    }
    // sums(): the two byte sums (metric.rs:223, :237)
    __device__ __forceinline__ void sums(int p, int kl, int vl) const {
        if (SMEM) {
            const uint32_t P4 = 4u * (uint32_t)P, pa = sbase + 4u * (uint32_t)p;
            const uint32_t ks = (uint32_t)max(kl, 0), vs = (uint32_t)max(vl, 0);
            red_shared_add(pa + ROW_KSUM * P4, ks & 0xffffu);
            red_shared_add_nz(pa + (ROW_KSUM + 1) * P4, ks >> 16);
            red_shared_add(pa + ROW_VSUM * P4, vs & 0xffffu);
            red_shared_add_nz(pa + (ROW_VSUM + 1) * P4, vs >> 16);
        } else {
            sum_add(0, p, (uint32_t)max(kl, 0));
            sum_add(1, p, (uint32_t)max(vl, 0));
        }
    }
    __device__ __forceinline__ void record(int p, int kl, int vl) const {
        buckets(p, kl, vl);
        sums(p, kl, vl);
    }
    // the four records of one lane.  When every length of the lane fits 16 bits (one OR chain and one branch for
    // the lane's eight lengths) the high halves are zero and the low half IS the length: two adds per record
    // instead of two adds, two shifts, two masks and two guarded adds.
    __device__ __forceinline__ void record_rows(const int (&p)[ROWS], const int (&kl)[ROWS], const int (&vl)[ROWS]) const {
        if (SMEM) {
            uint32_t ks[ROWS], vs[ROWS], any = 0;
#pragma unroll
            for (int k = 0; k < ROWS; k++) {
                ks[k] = (uint32_t)max(kl[k], 0);
                vs[k] = (uint32_t)max(vl[k], 0);
                any |= ks[k] | vs[k];
                buckets(p[k], kl[k], vl[k]);
            }
            if (any < 0x10000u) {
                const uint32_t P4 = 4u * (uint32_t)P;
#pragma unroll
                for (int k = 0; k < ROWS; k++) {
                    const uint32_t pa = sbase + 4u * (uint32_t)p[k];
                    red_shared_add(pa + ROW_KSUM * P4, ks[k]);
                    red_shared_add(pa + ROW_VSUM * P4, vs[k]);
                }
            } else {
#pragma unroll
                for (int k = 0; k < ROWS; k++) sums(p[k], kl[k], vl[k]);
            }
        } else {
#pragma unroll
            for (int k = 0; k < ROWS; k++) record(p[k], kl[k], vl[k]);
        }
    }
    // One warp drains split sums that reached `threshold` into the global u64 sums; safe against concurrent
    // adds (atomicExch takes exactly what it zeroes).  Overflow bound: every warp runs the check after every
    // FOLD_TILES-th tile of its own (after that tile's adds; no CTA-wide counter, no synchronisation).  Take two
    // consecutive examinations of a word, by whichever warps: after the first, each warp reaches its own next check
    // within FOLD_TILES tiles, so until the second one every warp has finished fewer than FOLD_TILES tiles and has
    // at most one more in flight: at most 32 x 9 tiles x 128 records x (2^16 - 1) < 2.42e9 is added to a word that
    // was < 2^30 after the first examination — it stays below 3.5e9 < 2^32.
    __device__ __noinline__ void fold_sums(int lane, uint32_t threshold) const {
        if constexpr (SMEM) {
            for (int i = lane; i < 2 * P; i += 32) {
                const int which = i >= P, p = which ? i - P : i;
                uint32_t *lo = &s[(ROW_KSUM + 2 * which) * P + p];
                if (*(volatile uint32_t *)lo >= threshold || *(volatile uint32_t *)(lo + P) >= threshold) {
                    const unsigned long long v = (unsigned long long)atomicExch(lo, 0u) +
                                                 ((unsigned long long)atomicExch(lo + P, 0u) << 16);
                    if (v) atomicAdd(&g[(size_t)Pg * (2 * NB + which) + part(p)], v);
                }
            }
        }
    }
};

// ------------------------------------------------------------------------------------------------
// alive-key table (LogCompactionInMemoryMetrics, metric.rs:262-305): an open-addressed table with one 64-bit entry per
// distinct key hash,
//     x (32 bits) | seq - origin + 1 (31 bits) | alive (1 bit),          ~0 = empty,        x = fmix32(hash),
// holding the stamp of the LAST record that carried this hash (fmix32 is a bijection: x names the hash exactly, and it
// is what the table, the seen cache and the HLL sketch all index by, so it is computed once per record).  The reference's BitSet (metric.rs:273-280) is indexed by
// the hash itself — 2^32 bits, one random DRAM sector per record wherever the state lives; keyed by hash but SIZED by
// the number of distinct hashes, the same state is 80 MB of entries for 1e7 keys, and the seen cache below keeps most records in L2.
//   * A slot is claimed once (CAS from empty) and keeps its hash for ever; linear probing over 16-byte PAIRS of slots
//     from home = mulhi(x, pairs), so any table size works, not only powers of two.
//   * On a slot that holds the record's hash, atomicMax makes "last" mean highest seq regardless of execution order
//     (the hash sits in the top bits, so max over equal-hash stamps is max over seq).  Entries only grow, so a plain
//     read is a safe filter: a record that is not the newest for its hash stops after one 16-byte read.  The scan walks
//     each batch from its newest tile to its oldest, so for a key written k times about (k-1)/k of its records take
//     that exit.
//   * sum_all_alive (metric.rs:282-284) is a count over the table at finalize (a pass over ~128 MiB: tens of µs), so
//     the stamps themselves need no return value: raising an existing entry is a fire-and-forget RED.MAX.
//   * 31 bits of seq: when a batch would not fit the window the host REBASES (every entry keeps hash and alive bit, its
//     seq field drops to 0: older than everything that follows, which is all a later record needs to know).
//   * A stamp that finds neither its hash nor an empty slot within ALIVE_MAX_PROBES pairs is counted in status[0] and
//     dropped; the host then grows the table (rehash) and re-runs the batch stamps-only — stamping is idempotent.
//
// The SEEN CACHE in front of it.  A table of 128 MiB or more does not stay in L2 next to a multi-GB record stream, so
// a table probe per record is a random DRAM sector per record.  But 90–99 % of the
// records of a compacted topic are superseded by a newer record of the same key, and all they need to learn is that
// fact.  So each batch keeps a 32 MiB, 2-way set-associative, EXACT cache of (hash → newest wave seen), where a wave is
// 1/127 of the batch in seq order: set = top 23 bits of fmix32(hash) (a bijection), way = 9-bit tag (the other bits) +
// 7-bit wave.  A record that finds its own tag with a wave NEWER than its own is superseded by construction (waves are
// a monotone function of seq — no timing assumption) and is done after one L2 hit.  Everything else — the first record
// seen of each key, same-wave siblings, conflict misses — is compacted across the tile into one dense queue and takes
// the exact path through the table; whatever the table knows afterwards is written back to the cache.  The cache holds
// only true facts ("a record of this hash with this wave exists and is being stamped"), so a lost or stale entry costs a
// table probe, never correctness.
// ------------------------------------------------------------------------------------------------
constexpr unsigned long long ALIVE_EMPTY = ~0ull;
constexpr uint32_t ALIVE_FIELD_MAX = 0x7ffffffeu;   // largest seq field: a stamp's low word is <= 0xfffffffd, never ~0
constexpr int ALIVE_MAX_PROBES = 96;                // pairs examined before a stamp gives up

#ifndef KTA_L2_HINTS
#define KTA_L2_HINTS 1
#endif
#ifndef KTA_EXP_ALIVE_STAGE   // ablation knob: 0 = hashes only, 1 = + seen-cache probe and queue, 2 = everything (the product)
#define KTA_EXP_ALIVE_STAGE 2
#endif
// L2 residency control for MODE_EXACT: the table should stay in L2, the record stream should leave it at once.
__device__ __forceinline__ uint64_t l2_policy_evict_last() {
    uint64_t pol;
    asm volatile("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(pol));
    return pol;
}
__device__ __forceinline__ uint64_t l2_policy_evict_first() {
    uint64_t pol;
    asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(pol));
    return pol;
}
__device__ __forceinline__ ulonglong2 alive_ld_pair(const unsigned long long *p, uint64_t pol) {
    ulonglong2 v;
#if KTA_L2_HINTS
    asm volatile("ld.global.cg.L2::cache_hint.v2.u64 {%0, %1}, [%2], %3;" : "=l"(v.x), "=l"(v.y) : "l"(p), "l"(pol));
#else
    asm volatile("ld.global.cg.v2.u64 {%0, %1}, [%2];" : "=l"(v.x), "=l"(v.y) : "l"(p));
#endif
    return v;
}
__device__ __forceinline__ unsigned long long alive_atom_max(unsigned long long *p, unsigned long long v, uint64_t pol) {
    unsigned long long old;
#if KTA_L2_HINTS
    asm volatile("atom.global.max.L2::cache_hint.u64 %0, [%1], %2, %3;" : "=l"(old) : "l"(p), "l"(v), "l"(pol) : "memory");
#else
    old = atomicMax(p, v);
#endif
    return old;
}
// (atom.cas takes no cache-policy operand in PTX: a claim is a plain compare-and-swap)
__device__ __forceinline__ unsigned long long alive_atom_cas(unsigned long long *p, unsigned long long cmp, unsigned long long v,
                                                             uint64_t) {
    return atomicCAS(p, cmp, v);
}

__host__ __device__ __forceinline__ uint32_t alive_home(uint32_t x /* mixed hash */, uint32_t npairs) {
#ifdef __CUDA_ARCH__
    return __umulhi(x, npairs);
#else
    return (uint32_t)(((uint64_t)x * npairs) >> 32);
#endif
}

struct AliveTable {
    unsigned long long *slots;
    uint32_t npairs;
    uint32_t *status;
    uint64_t pol;       // L2 evict_last policy for the table's lines
};

// raise an entry that holds this stamp's hash: no return value, the warp does not wait
__device__ __forceinline__ void alive_red_max(unsigned long long *p, unsigned long long v, uint64_t pol) {
#if KTA_L2_HINTS
    asm volatile("red.global.max.L2::cache_hint.u64 [%0], %1, %2;" ::"l"(p), "l"(v), "l"(pol) : "memory");
#else
    asm volatile("red.global.max.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
#endif
}

// The general stamp: probe from `pair` until the hash or an empty slot is found.  Returns the low word of the newest
// stamp known for this hash afterwards (the record's own if it won).
__device__ __noinline__ uint32_t alive_stamp_slow(const AliveTable t, uint32_t pair, uint32_t hash, uint32_t low) {
    const unsigned long long stamp = ((unsigned long long)hash << 32) | low;
    for (int probe = 0; probe < ALIVE_MAX_PROBES; probe++) {
        unsigned long long *slot = t.slots + 2 * (size_t)pair;
        const ulonglong2 e = alive_ld_pair(slot, t.pol);
#pragma unroll
        for (int s = 0; s < 2; s++) {
            unsigned long long v = s ? e.y : e.x;
            if (v == ALIVE_EMPTY) {
                v = atomicCAS(slot + s, ALIVE_EMPTY, stamp);
                if (v == ALIVE_EMPTY) return low;                   // first record of this hash: mark_key_alive / _dead on a fresh bit
            }
            if ((uint32_t)(v >> 32) == hash) {                      // v is a real entry here (never ALIVE_EMPTY)
                if (v >= stamp) return (uint32_t)v;                 // a later record already spoke for this hash
                alive_red_max(slot + s, stamp, t.pol);
                return low;
            }
        }
        pair = pair + 1 == t.npairs ? 0 : pair + 1;
    }
    atomicAdd(t.status, 1u);   // table too full: the host grows it and re-runs this batch's stamps
    return low;
}

// One stamp with the home pair already loaded (`e`): the common cases need no second look at memory.
// (`hash` is the mixed hash x throughout the table code.)
__device__ __forceinline__ uint32_t alive_stamp(const AliveTable t, uint32_t pair, const ulonglong2 e, uint32_t hash, uint32_t low) {
    const bool hx = (uint32_t)(e.x >> 32) == hash, hy = (uint32_t)(e.y >> 32) == hash;
    const uint32_t seen = hx ? (uint32_t)e.x : (uint32_t)e.y;
    // equal hash ⇒ the stamps compare like their low words.  A real low word is <= 0xfffffffd and the empty pattern's is
    // 0xffffffff, so "seen + 1 > low" is "seen >= low" for real entries and false for an empty slot under hash 0xffffffff
    if ((hx || hy) && seen + 1u > low) return seen;                 // a later record already spoke for this hash
    unsigned long long *slot = t.slots + 2 * (size_t)pair;
    const unsigned long long stamp = ((unsigned long long)hash << 32) | low;
    const bool ex = e.x == ALIVE_EMPTY, ey = e.y == ALIVE_EMPTY;
    if ((hx && !ex) || (!hx && hy && !ey)) {                        // the hash is here with an older stamp: raise it
        alive_red_max(slot + (hx ? 0 : 1), stamp, t.pol);
        return low;
    }
    if (ex || ey) {                                                 // first record of this hash: claim the free slot
        unsigned long long *sl = slot + (ex ? 0 : 1);
        const unsigned long long old = atomicCAS(sl, ALIVE_EMPTY, stamp);
        if (old == ALIVE_EMPTY) return low;
        if ((uint32_t)(old >> 32) == hash) {                        // a sibling claimed it in the meantime
            if (old >= stamp) return (uint32_t)old;
            alive_red_max(sl, stamp, t.pol);
            return low;
        }
    }
    return alive_stamp_slow(t, pair, hash, low);                    // displaced: probe on
}

// ---- seen cache: nsets = 2^ALIVE_CACHE_SET_BITS sets of two 16-bit ways: tag (9 bits) << 7 | wave (7 bits), 0 = empty ----
constexpr int ALIVE_CACHE_SET_BITS = 23, ALIVE_CACHE_TAG_BITS = 32 - ALIVE_CACHE_SET_BITS, ALIVE_CACHE_WAVE_BITS = 16 - ALIVE_CACHE_TAG_BITS;
constexpr uint32_t ALIVE_CACHE_WAVES = (1u << ALIVE_CACHE_WAVE_BITS) - 1;   // waves 1..127 (0 = empty way)
static_assert(ALIVE_CACHE_TAG_BITS == 9 && ALIVE_CACHE_WAVE_BITS == 7, "16-bit ways");
__device__ __forceinline__ uint32_t alive_cache_ld(const uint32_t *p, uint64_t pol) {
    uint32_t v;
#if KTA_L2_HINTS
    asm volatile("ld.global.cg.L2::cache_hint.u32 %0, [%1], %2;" : "=r"(v) : "l"(p), "l"(pol));
#else
    asm volatile("ld.global.cg.u32 %0, [%1];" : "=r"(v) : "l"(p));
#endif
    return v;
}
// is a record of mixed hash x and wave `wv` superseded according to set word c?
__device__ __forceinline__ bool alive_cache_newer(uint32_t c, uint32_t x, uint32_t wv) {
    const uint32_t tag = x & ((1u << ALIVE_CACHE_TAG_BITS) - 1u);
    const uint32_t w0 = c & 0xffffu, w1 = c >> 16;
    // same tag and a larger wave  ⇔  way in (tag << 7 | wv, tag << 7 | 127]
    const uint32_t lo = (tag << ALIVE_CACHE_WAVE_BITS) | wv;
    return (w0 - lo - 1u < ALIVE_CACHE_WAVES - wv) || (w1 - lo - 1u < ALIVE_CACHE_WAVES - wv);
}
// record the fact "hash x has a record of wave wv" (wv >= 1) in its set; c = the set word as read by the probe.
// The tag's own way if it has one (and only if that improves on it), else an empty way, else either.  (Picking the way by
// a bit of the hash instead — nothing to carry from the probe — lets two keys that share a set evict each other for
// ever, and every such eviction is one more table probe.)
__device__ __forceinline__ void alive_cache_put(uint32_t *cache, uint32_t c, uint32_t x, uint32_t wv, uint32_t pick) {
    const uint32_t tag = x & ((1u << ALIVE_CACHE_TAG_BITS) - 1u);
    const uint32_t mine = (tag << ALIVE_CACHE_WAVE_BITS) | wv;
    const uint32_t w0 = c & 0xffffu, w1 = c >> 16;
    int way;
    if ((w0 >> ALIVE_CACHE_WAVE_BITS) == tag && w0) way = w0 >= mine ? -1 : 0;          // already known at least as new
    else if ((w1 >> ALIVE_CACHE_WAVE_BITS) == tag && w1) way = w1 >= mine ? -1 : 1;
    else way = w0 == 0 ? 0 : w1 == 0 ? 1 : (int)(pick & 1u);
    if (way >= 0) reinterpret_cast<unsigned short *>(cache + (x >> ALIVE_CACHE_TAG_BITS))[way] = (unsigned short)mine;   // way 0 = low half
}

// plain insert of an entry whose hash is known to be absent (rehash into a fresh table)
__device__ __forceinline__ bool alive_insert_unique(unsigned long long *slots, uint32_t npairs, unsigned long long entry) {
    uint32_t pair = alive_home((uint32_t)(entry >> 32), npairs);
    for (uint32_t probe = 0; probe < npairs; probe++) {
        unsigned long long *slot = slots + 2 * (size_t)pair;
#pragma unroll
        for (int s = 0; s < 2; s++)
            if (__ldcg(slot + s) == ALIVE_EMPTY && atomicCAS(slot + s, ALIVE_EMPTY, entry) == ALIVE_EMPTY) return true;
        pair = pair + 1 == npairs ? 0 : pair + 1;
    }
    return false;
}

// rare path: a tile with a key of >= 1 MiB — 64-bit offsets, keys read straight from global memory.
// Out of line and self-contained (re-reads key_len, hands the hashes back through the warp's shared
// scratch) so that it costs the hot path no registers.
__device__ __noinline__ void wide_tile_hashes(const int32_t *key_len, int64_t n, const uint8_t *tile_keys, int64_t tile,
                                              uint32_t *out /*[TILE]*/, int lane) {
    uint64_t carry = 0;
    for (int k = 0; k < ROWS; k++) {
        const int64_t r = tile * TILE + 32 * k + lane;
        const int kl = r < n ? key_len[r] : -1;
        const uint64_t v = (uint64_t)max(kl, 0);
        uint64_t inc = v;
        for (int d = 1; d < 32; d <<= 1) {
            const uint64_t t = __shfl_up_sync(0xffffffffu, inc, d);
            if (lane >= d) inc += t;
        }
        out[32 * k + lane] = kl >= 0 ? fnv_global(tile_keys + carry + inc - v, kl) : 0u;
        carry += __shfl_sync(0xffffffffu, inc, 31);
    }
    __syncwarp();
}

// wave of a stamp field (seq - origin + 1) within the batch being scanned: 0 = older than the batch, else 1..127, a monotone
// function of seq
struct AliveWaves {
    uint32_t *cache;   // the seen cache, or NULL
    uint32_t base;     // field of the batch's first record
    int shift;
};
__device__ __forceinline__ uint32_t alive_wave(uint32_t field, const AliveWaves w) {
    const uint32_t d = field - w.base;
    return (int32_t)d < 0 ? 0u : 1u + min(d >> w.shift, ALIVE_CACHE_WAVES - 1u);
}

// ------------------------------------------------------------------------------------------------
// the fused scan kernel.
//   MODE_COUNTERS: counters + histograms + extrema only (20 B/record, no key bytes touched — the reference
//                  without -c).
//   MODE_HLL:      + FNV per key from staged shared memory + the in-stream HLL sketch (20 + key bytes).
//   MODE_EXACT:    + FNV per key + alive-table stamps (the reference with -c).
//   CAPTURE (tests only) also writes every record's hash to prm.hash_out.
//
// One persistent CTA per SM; every WARP is an autonomous worker: it walks its own 128-record tiles
// (tile t belongs to global warp t % total_warps), stages each tile's packed key bytes with its own
// bulk async copy (cp.async.bulk → UBLKCP) on its own pair of mbarriers, and never waits for another
// warp — there is no __syncthreads in the loop, so the load phase of one warp overlaps the hash phase of
// the others.  Only the per-partition counters are shared (shared-memory reductions).
// ------------------------------------------------------------------------------------------------
template <int MODE, bool SMEM, bool CAPTURE, bool SHARD = false>
__global__ void __launch_bounds__(MAX_THREADS, 1) scan_kernel(const ScanParams prm) {
    constexpr bool HASH = MODE != MODE_COUNTERS;
    extern __shared__ __align__(128) unsigned char smem_raw[];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, nwarps = blockDim.x >> 5;
    const unsigned full = 0xffffffffu;
    const unsigned lt_mask = (1u << lane) - 1u;
    // SHARD: a partition-sharded scan (SURVEY.md §8 e: gpu = partition mod G) carves counter columns only for the
    // partitions it owns — a rank of BASELINE configs[3] holds 32 columns, not 256
    const int P = SHARD ? prm.Pc : prm.P;
    // layout: counter rows (SMEM) | per warp: mbar[2] + 112 B scratch | keybuf[2]
    uint32_t *scnt = reinterpret_cast<uint32_t *>(smem_raw);
    const size_t cta_bytes = SMEM ? smem_counter_bytes(P) : CTA_SCRATCH;
    const uint32_t KEYBUF = (uint32_t)prm.keybuf;
    const size_t warp_bytes = warp_smem_bytes(HASH, prm.keybuf, MODE == MODE_EXACT);
    unsigned char *wsm = smem_raw + cta_bytes + (size_t)warp * warp_bytes;
    const uint32_t mbar = smem_u32(wsm);            // two 8-byte mbarriers at +0, +8
    const uint32_t keybuf = smem_u32(wsm) + 128;    // two KEYBUF-byte stages
    const Counters<SMEM> C{smem_u32(scnt), scnt, prm.sums, P, prm.P, SHARD ? prm.shard_world : 1, SHARD ? prm.shard_rank : 0};
    // MODE_EXACT: the alive table's lines are asked to stay in L2 (evict_last), the record stream to leave first
    constexpr bool HINTS = MODE == MODE_EXACT && KTA_L2_HINTS;
    const uint64_t pol_stream = HINTS ? l2_policy_evict_first() : 0;
    const AliveTable AT{prm.alive_table, prm.alive_pairs, prm.alive_status, HINTS ? l2_policy_evict_last() : 0};
    const AliveWaves AW{prm.alive_cache, prm.alive_wave_base, prm.alive_wave_shift};
    const bool count_it = !(MODE == MODE_EXACT && prm.alive_only);   // false: a stamps-only re-run after the table grew

    if (SMEM) {
        const int nw = P * SMEM_ROWS;
        for (int i = tid; i < nw; i += blockDim.x) scnt[i] = 0;
    }
    if (HASH && lane == 0) {
        mbar_init(mbar, 1);
        mbar_init(mbar + 8, 1);
        fence_mbar_init();
    }
    __syncthreads();

    // lane 0: start the bulk copy of a tile's packed key bytes into stage b.
    // Returns the span descriptor: bit 0 staged, bits 1..4 = first key's offset inside its 16-byte line.
    auto issue = [&](int tile, int b) -> uint32_t {
        const uint64_t g0 = prm.key_tile_base[tile], g1 = prm.key_tile_base[tile + 1];
        const uint32_t a = (uint32_t)g0 & 15u;
        // the copy covers [g0 - a, roundup16(g1)).  Staged iff the tile has key bytes, the copy fits the stage
        // (KEYBUF and the slack are multiples of 16, so roundup16(g1 - g0 + a) + slack <= KEYBUF ⇔ g1 - g0 <= cap - a)
        // and it ends inside the readable bytes (stage_limit is a multiple of 16, so roundup16(g1) <= limit ⇔ g1 <= limit)
        const bool ok = (g1 - g0) - 1ull < (uint64_t)(KEYBUF - (uint32_t)KEYBUF_SLACK - a) && g1 <= prm.stage_limit;
        if (ok) {
            const uint32_t bytes = ((uint32_t)(g1 - g0) + a + 15u) & ~15u;
            mbar_arrive_expect_tx(mbar + 8u * b, bytes);
            if (HINTS) bulk_g2s(keybuf + (uint32_t)b * KEYBUF, prm.key_bytes + (g0 - a), bytes, mbar + 8u * b, pol_stream);
            else bulk_g2s(keybuf + (uint32_t)b * KEYBUF, prm.key_bytes + (g0 - a), bytes, mbar + 8u * b);
        }
        return (ok ? 1u : 0u) | (a << 1);
    };

    long long tmin = INT64_MAX, tmax = INT64_MIN;         // raw ts_ms extrema (None → 0 applied at read-back)
    uint32_t smin = 0xffffffffu, smax = 0;                // message size extrema (non-tombstones); sizes < 2^32 - 1
    uint32_t bad = 0;
    uint32_t phase = 0;       // bit b = parity to wait for on mbar[b]
    bool try_uni = true;      // probe rows for "one partition" only while that keeps paying off
    // MODE_HLL: the warp's copy of the sketch floor (a lower bound of every register: monotone, so a stale copy only
    // filters less).  Re-read from its global word after the first tiles and then every 16th tile — one global word read by
    // every warp for EVERY tile makes a single L2 line the bottleneck of the whole kernel.
    uint32_t floor_reg = MODE == MODE_HLL ? ld_cg_u32(prm.hll_floor) : 0u;
    uint32_t nxt_info = 0;

    // MODE_EXACT walks the batch from its newest tile to its oldest (see alive_stamp); the other modes ascend
    // tile indices fit 32 bits (the host refuses batches of 2^31 tiles = 2.7e11 records): the loop control stays out of
    // 64-bit arithmetic and out of local memory
    const int ntiles = (int)prm.ntiles;
    auto phys = [&](int t) { return MODE == MODE_EXACT ? ntiles - 1 - t : t; };
    const int gstride = (int)gridDim.x * nwarps;
    int tile = (int)blockIdx.x * nwarps + warp;
    if (HASH && lane == 0 && tile < ntiles) nxt_info = issue(phys(tile), 0);

    // the body of one tile; FULL = every record of the tile exists (no tail predicates)
    auto body = [&](auto full_tag, int tile, int buf, uint32_t info, bool has_next) {
        constexpr bool FULL = decltype(full_tag)::value;
        // ---- header columns: 4 rows of 32 consecutive records, fully coalesced ----
        const int64_t rbase = (int64_t)tile * TILE + lane;
        int p[ROWS], kl[ROWS], vl[ROWS];
        long long ts[ROWS];
        bool valid[ROWS];
#pragma unroll
        for (int k = 0; k < ROWS; k++) {
            const int64_t r = rbase + 32 * k;
            valid[k] = FULL || r < prm.n;
            if (valid[k]) {
                if (HINTS) {
                    p[k] = ld_stream_s32(prm.partition + r, pol_stream);
                    ts[k] = ld_stream_s64(prm.ts_ms + r, pol_stream);
                    kl[k] = ld_stream_s32(prm.key_len + r, pol_stream);
                    vl[k] = ld_stream_s32(prm.value_len + r, pol_stream);
                } else {
                    p[k] = ld_stream_s32(prm.partition + r);
                    ts[k] = ld_stream_s64(prm.ts_ms + r);
                    kl[k] = ld_stream_s32(prm.key_len + r);
                    vl[k] = ld_stream_s32(prm.value_len + r);
                }
            } else {
                p[k] = 0; ts[k] = INT64_MAX; kl[k] = -1; vl[k] = -1;
            }
        }
        // ---- MessageMetrics::handle_message (metric.rs:206-253) ----
        // A record whose partition lies outside [0, P) is counted in `bad` and takes part in NOTHING else (counters, extrema,
        // alive keys, sketch), so the state stays consistent; its key bytes still occupy their place in the packed keys.
        bool use[ROWS];
        bool inrange = true;
#pragma unroll
        for (int k = 0; k < ROWS; k++) {
            bool ok = (unsigned)p[k] < (unsigned)prm.P;
            if (SHARD) {
                // partition → column: c = p / G, and the partition must be one of this shard's (p - c G == rank);
                // others are left out like out-of-range ones.  From here on p[k] is the column.
                const int c = (int)__umulhi((uint32_t)p[k], prm.shard_magic);
                ok = ok && p[k] - c * prm.shard_world == prm.shard_rank;
                p[k] = ok ? c : 0;
            }
            use[k] = valid[k] && ok;
            inrange = inrange && ok;
        }
        const bool clean = FULL && __all_sync(full, inrange);   // warp-uniform: every record of the tile exists and counts
        uint32_t h[ROWS] = {0u, 0u, 0u, 0u};   // the reference hash of each of the lane's four keys (0 for null keys)
        // The two halves of the per-record work are independent of each other: MODE_EXACT runs the hashes FIRST, sends the
        // seen-cache probes off, and counts while they are in flight; the other modes count first (the key bytes arrive later).
        auto count_records = [&]() {
            if (!count_it) {
                // stamps-only re-run: the counters and extrema of this batch were taken by the first pass
            } else if (clean) {
                if (try_uni) {
                    // run-structured input (a Kafka fetch delivers long runs of one partition).
                    // A whole tile inside one run (3 of 4 tiles at run length 500): one vote, the lane's four lengths added up
                    // first, two warp reductions and two adds for the tile
                    const int p0t = __shfl_sync(full, p[0], 0);
                    uint32_t kv4 = 0, vv4 = 0, big = 0;
                    bool one = true;
#pragma unroll
                    for (int k = 0; k < ROWS; k++) {
                        const uint32_t kv = (uint32_t)max(kl[k], 0), vv = (uint32_t)max(vl[k], 0);
                        one = one && p[k] == p0t;
                        kv4 += kv; vv4 += vv; big |= kv | vv;
                    }
                    if (__all_sync(full, one && big < (1u << 24))) {
#pragma unroll
                        for (int k = 0; k < ROWS; k++) C.buckets(p0t, kl[k], vl[k]);
                        const uint32_t ks = __reduce_add_sync(full, kv4);   // 128 lengths < 2^24: no overflow
                        const uint32_t vs = __reduce_add_sync(full, vv4);
                        if (lane == 0) {
                            C.sum_add(0, p0t, ks);
                            C.sum_add(1, p0t, vs);
                        }
                    } else {
                    // otherwise row by row: the byte sums of a row that lies inside one run are reduced in the warp (2 REDUX)
                    // and added once, instead of 32 same-address adds
                    bool any_uni = false;
#pragma unroll
                    for (int k = 0; k < ROWS; k++) {
                        C.buckets(p[k], kl[k], vl[k]);
                        const int p0 = __shfl_sync(full, p[k], 0);
                        const unsigned m0 = __ballot_sync(full, p[k] == p0);
                        const bool small_row = __all_sync(full, (kl[k] | vl[k]) < (1 << 26));
                        const uint32_t kv = (uint32_t)max(kl[k], 0), vv = (uint32_t)max(vl[k], 0);
                        if (m0 == full && small_row) {
                            const uint32_t ks = __reduce_add_sync(full, kv);   // each < 2^26: no overflow
                            const uint32_t vs = __reduce_add_sync(full, vv);
                            if (lane == 0) {
                                C.sum_add(0, p0, ks);
                                C.sum_add(1, p0, vs);
                            }
                            any_uni = true;
                        } else {
                            // a row that straddles a run boundary holds two partitions: left to per-lane adds, its two
                            // counters would be hit 32 times each, serialised in the shared-memory pipe.  Reduce the two groups separately instead.
                            const int l1 = __ffs(~m0) - 1;                     // first lane of the second group
                            const int p1 = __shfl_sync(full, p[k], l1 & 31);
                            const unsigned m1 = __ballot_sync(full, p[k] == p1);
                            if (small_row && (m0 | m1) == full) {
                                const bool in0 = (m0 >> lane) & 1u;
                                const uint32_t ks0 = __reduce_add_sync(full, in0 ? kv : 0u), vs0 = __reduce_add_sync(full, in0 ? vv : 0u);
                                const uint32_t ks1 = __reduce_add_sync(full, in0 ? 0u : kv), vs1 = __reduce_add_sync(full, in0 ? 0u : vv);
                                if (lane == 0) {
                                    C.sum_add(0, p0, ks0);
                                    C.sum_add(1, p0, vs0);
                                } else if (lane == l1) {
                                    C.sum_add(0, p1, ks1);
                                    C.sum_add(1, p1, vs1);
                                }
                                any_uni = true;
                            } else {
                                C.sums(p[k], kl[k], vl[k]);
                            }
                        }
                    }
                    try_uni = any_uni;
                    }
                } else {
                    C.record_rows(p, kl, vl);
                }
            } else {
                // tail tile, or a record with a partition outside [0, P): per-record checks
#pragma unroll
                for (int k = 0; k < ROWS; k++) {
                    if (use[k]) C.record(p[k], kl[k], vl[k]);
                    else if (valid[k]) bad++;
                }
            }
            // metric.rs:209,247: None → 0 and ms → s are monotone maps, applied once at read-back: the raw
            // extrema determine the mapped extrema (raw == -1 ⇔ mapped 0, see kta_timestamps).
            // Timestamps of one topic share their high word for 49 days at a time: when the lane's four and its running
            // extrema do, the signed 64-bit order is the unsigned order of the low words (2 + 2 three-input min/max).
            bool ts_fast = false;
            if (clean && count_it) {
                const uint32_t hw = hi32(tmin);
                uint32_t x = hi32(tmax) ^ hw;
#pragma unroll
                for (int k = 0; k < ROWS; k++) x |= hi32(ts[k]) ^ hw;
                ts_fast = x == 0;
            }
            if (ts_fast) {
                const uint32_t hw = hi32(tmin);
                const uint32_t l0 = (uint32_t)ts[0], l1 = (uint32_t)ts[1], l2 = (uint32_t)ts[2], l3 = (uint32_t)ts[3];
                const uint32_t lo = min(min(min(l0, l1), l2), min(l3, (uint32_t)tmin));
                const uint32_t hi = max(max(max(l0, l1), l2), max(l3, (uint32_t)tmax));
                tmin = pack64(lo, hw);
                tmax = pack64(hi, hw);
            } else if (count_it) {
                asm volatile("");   // keep this a real branch: if-converted, the 64-bit chain runs every tile
#pragma unroll
                for (int k = 0; k < ROWS; k++) {
                    const bool u = clean || use[k];
                    const long long t0 = u ? ts[k] : INT64_MAX, t1 = u ? ts[k] : INT64_MIN;
                    tmin = t0 < tmin ? t0 : tmin;
                    tmax = t1 > tmax ? t1 : tmax;
                }
            }
            if (count_it) {
#pragma unroll
                for (int k = 0; k < ROWS; k++) {
                    // metric.rs:249-251: size extrema, not for tombstones (rows that do not exist carry vl = -1)
                    const uint32_t sz = (uint32_t)max(kl[k], 0) + (uint32_t)vl[k];
                    if (vl[k] >= 0 && (clean || use[k])) {
                        smin = min(smin, sz);
                        smax = max(smax, sz);
                    }
                }
            }

        };
        auto hash_keys = [&]() {
            // ---- byte offset of each key inside the tile: exclusive scan of max(key_len, 0) ----
            uint32_t off[ROWS];
            // do all keys of this tile that are not null have ONE length L?  L = the longest; read as unsigned, null (-1)
            // is the largest value, so the unsigned minimum is the shortest non-null key (or "null" if there is none):
            // one length ⇔ the two agree.  Two three-input min/max per lane and two warp reductions.
            const int lmax = max(max(kl[0], kl[1]), max(kl[2], kl[3]));
            const uint32_t lmin = min(min((uint32_t)kl[0], (uint32_t)kl[1]), min((uint32_t)kl[2], (uint32_t)kl[3]));
            static_assert(ROWS == 4, "written out for four rows");
            const int L = __reduce_max_sync(full, lmax);   // -1 when every key is null
            const bool fixL = __reduce_min_sync(full, lmin) == (uint32_t)L && L < (1 << 16);
            const bool small = L < (1 << 20);              // warp-uniform
            const bool fix16 = fixL && L == 16;
            if (fixL) {
                // fixed-width keys (the common case: ids, hashes, UUIDs)
                const uint32_t Lu = (uint32_t)max(L, 0);
                if (!__any_sync(full, (kl[0] | kl[1] | kl[2] | kl[3]) < 0)) {
                    // no null key in the tile (every tile of a keyed / compacted topic): record r's key is the r-th
#pragma unroll
                    for (int k = 0; k < ROWS; k++) off[k] = Lu * (uint32_t)(32 * k + lane);
                } else {
                    // offsets from ballots, no shuffle scan
                    uint32_t before = 0;
#pragma unroll
                    for (int k = 0; k < ROWS; k++) {
                        const unsigned m = __ballot_sync(full, kl[k] >= 0);
                        off[k] = Lu * (before + __popc(m & lt_mask));
                        before += __popc(m);
                    }
                }
            } else {
                static_assert(ROWS == 4, "the packed scan below handles exactly four rows");
                uint32_t mxl = 0;
#pragma unroll
                for (int k = 0; k < ROWS; k++) mxl = max(mxl, (uint32_t)max(kl[k], 0));
                if (__all_sync(full, mxl < 2048u)) {
                    // short keys (every row sums to < 2^16): scan two rows per 32-bit word, 10 shuffles instead of 20
                    const uint32_t v0 = (uint32_t)max(kl[0], 0), v1 = (uint32_t)max(kl[1], 0);
                    const uint32_t v2 = (uint32_t)max(kl[2], 0), v3 = (uint32_t)max(kl[3], 0);
                    uint32_t a = v0 | (v1 << 16), b = v2 | (v3 << 16);
#pragma unroll
                    for (int d = 1; d < 32; d <<= 1) {
                        const uint32_t ta = __shfl_up_sync(full, a, d), tb = __shfl_up_sync(full, b, d);
                        if (lane >= d) { a += ta; b += tb; }
                    }
                    const uint32_t ea = __shfl_sync(full, a, 31), eb = __shfl_sync(full, b, 31);
                    const uint32_t t0 = ea & 0xffffu, t1 = ea >> 16, t2 = eb & 0xffffu;
                    off[0] = (a & 0xffffu) - v0;
                    off[1] = t0 + (a >> 16) - v1;
                    off[2] = t0 + t1 + (b & 0xffffu) - v2;
                    off[3] = t0 + t1 + t2 + (b >> 16) - v3;
                } else if (small) {
                    uint32_t c32 = 0;
#pragma unroll
                    for (int k = 0; k < ROWS; k++) {
                        const uint32_t v = (uint32_t)max(kl[k], 0);
                        uint32_t inc = v;
#pragma unroll
                        for (int d = 1; d < 32; d <<= 1) {
                            const uint32_t t = __shfl_up_sync(full, inc, d);
                            if (lane >= d) inc += t;
                        }
                        off[k] = c32 + inc - v;
                        c32 += __shfl_sync(full, inc, 31);
                    }
                }
            }
            const uint32_t kb = keybuf + (uint32_t)buf * KEYBUF;

            if (info & 1u) {   // staged ⇒ the tile's keys fit one stage (<= 16 KiB) ⇒ small
                const uint32_t a0 = (info >> 1) & 15u;
                mbar_wait(mbar + 8u * buf, (phase >> buf) & 1u);
                phase ^= 1u << buf;
#ifdef KTA_EXP_NO_FNV
                if (fix16 && a0 == 0) {
#pragma unroll
                    for (int k = 0; k < ROWS; k++) h[k] = lds32(kb + off[k]);
                } else
#endif
                if (fix16 && a0 == 0) {
                    // two independent FNV chains at a time per lane, one LDS.128 per key (null keys hash
                    // garbage that is never used); the other warps of the SM sub-partition supply the rest of the ILP
#pragma unroll
                    for (int k = 0; k < ROWS; k += 2) {
                        const uint4 qa = lds128(kb + off[k]);
                        const uint4 qb = lds128(kb + off[k + 1]);
                        uint32_t ha = FNV_BASIS, hb = FNV_BASIS;
                        ha = fnv_word(ha, qa.x); hb = fnv_word(hb, qb.x);
                        ha = fnv_word(ha, qa.y); hb = fnv_word(hb, qb.y);
                        ha = fnv_word(ha, qa.z); hb = fnv_word(hb, qb.z);
                        ha = fnv_word(ha, qa.w); hb = fnv_word(hb, qb.w);
                        h[k] = ha;
                        h[k + 1] = hb;
                    }
                } else {
#pragma unroll
                    for (int k = 0; k < ROWS; k++) h[k] = kl[k] >= 0 ? fnv_smem(kb, a0 + off[k], kl[k]) : 0u;
                }
            } else if (fixL || small) {
                const uint64_t g0 = prm.key_tile_base[tile];
#pragma unroll
                for (int k = 0; k < ROWS; k++)
                    h[k] = (valid[k] && kl[k] >= 0) ? fnv_global(prm.key_bytes + g0 + off[k], kl[k]) : 0u;
            } else {
                uint32_t *scratch = reinterpret_cast<uint32_t *>(wsm + 128 + (size_t)buf * KEYBUF);  // not staged: free
                wide_tile_hashes(prm.key_len, prm.n, prm.key_bytes + prm.key_tile_base[tile], tile, scratch, lane);
#pragma unroll
                for (int k = 0; k < ROWS; k++) h[k] = scratch[32 * k + lane];
            }


            // ---- LogCompactionInMemoryMetrics::handle_message, metric.rs:288-305 ----
            if (CAPTURE) {
#pragma unroll
                for (int k = 0; k < ROWS; k++)
                    if (valid[k]) prm.hash_out[rbase + 32 * k] = kl[k] >= 0 ? h[k] : 0u;
            }
        };
        if (MODE != MODE_EXACT) count_records();
        if (HASH) hash_keys();
        if (MODE == MODE_EXACT) {
            // metric.rs:291-302: Some(key) → insert (value) / remove (tombstone); None → nothing.
            // Last-writer-wins per hash in seq order IS the BitSet insert/remove sequence replayed in order
            // (metric.rs:295 mark_key_alive, :298 mark_key_dead).
            // What limits this mode is the L1 pipe — a divergent 32-lane global access costs it ~2 cycles per lane — and
            // latency, not DRAM.  So: exactly ONE random access per record (the seen cache, in flight while the records
            // are counted); the ~12 % that survive it are compacted across the tile into one dense queue (in the key stage
            // the tile has just finished with) and take the exact path through the table, usually in a single pass.
            uint4 *queue = reinterpret_cast<uint4 *>(wsm + 128 + (size_t)buf * KEYBUF);   // (x, low word, set word, -) x TILE <= stage
            const bool cached = AW.cache != nullptr;
            const uint32_t r32 = (uint32_t)rbase;   // index in the batch (< 2^31: host-checked)
            uint32_t x[ROWS], low[ROWS], cw[ROWS];
            bool live[ROWS];
#pragma unroll
            for (int k = 0; k < ROWS; k++) {
                live[k] = (clean || use[k]) && kl[k] >= 0;
                uint32_t field;
                if (prm.seq) {
                    // explicit global sequence numbers (partition-sharded scans): must fall into the table's window
                    const uint64_t f = live[k] ? ld_stream_u64(prm.seq + rbase + 32 * k) - prm.alive_origin + 1ull : 1ull;
                    if (f - 1ull >= (uint64_t)ALIVE_FIELD_MAX) {
                        atomicAdd(prm.alive_status + 1, 1u);
                        live[k] = false;
                    }
                    field = (uint32_t)f;
                } else {
                    field = (uint32_t)prm.alive_fbase + r32 + 32u * k;   // host-checked: seq_base + n fits the window
                }
                low[k] = (field << 1) | (vl[k] >= 0 ? 1u : 0u);
                x[k] = hll_mix(h[k]);
                cw[k] = 0;
                if (cached && live[k]) cw[k] = alive_cache_ld(AW.cache + (x[k] >> ALIVE_CACHE_TAG_BITS), AT.pol);
            }
            count_records();   // ~250 instructions while the probes are in flight
#if KTA_EXP_ALIVE_STAGE >= 1
            __syncwarp();      // every lane is done reading its keys from this stage before any lane overwrites it
            uint32_t qn = 0;   // warp-uniform
#pragma unroll
            for (int k = 0; k < ROWS; k++) {
                const bool go = live[k] && !(cached && alive_cache_newer(cw[k], x[k], alive_wave(low[k] >> 1, AW)));
                const unsigned m = __ballot_sync(full, go);
                if (go) queue[qn + __popc(m & lt_mask)] = make_uint4(x[k], low[k], cw[k], 0u);
                qn += __popc(m);
            }
            __syncwarp();
#if KTA_EXP_ALIVE_STAGE >= 2
            for (uint32_t q0 = 0; q0 < qn; q0 += 32) {
                if (q0 + lane < qn) {
                    const uint4 item = queue[q0 + lane];
#if KTA_EXP_ALIVE_STAGE == 3   // ablation: the survivors update the seen cache but never go to the table
                    const uint32_t newest = item.y;
#else
                    const uint32_t pr = alive_home(item.x, AT.npairs);
                    const ulonglong2 e = alive_ld_pair(AT.slots + 2 * (size_t)pr, AT.pol);
                    const uint32_t newest = alive_stamp(AT, pr, e, item.x, item.y);
#endif
                    // tell the cache what the table knows now: the newest stamp of this hash as a wave of THIS batch (0 =
                    // older than the batch: says nothing), or the record's own wave
                    if (cached)
                        alive_cache_put(AW.cache, item.z, item.x, max(alive_wave(item.y >> 1, AW), alive_wave(newest >> 1, AW)), newest >> 1);
                }
            }
#endif
            // the queue lives in a key stage that the TMA engine refills next iteration: order these generic-proxy
            // accesses before that async-proxy write
            asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
            __syncwarp();
#endif
        }
#ifndef KTA_EXP_NO_HLL
        if (MODE == MODE_HLL) {
            const uint32_t skip_mask = hll_skip_mask(prm.hll_p, floor_reg);
#pragma unroll
            for (int k = 0; k < ROWS; k++) {
                // in-stream sketch: every record with a key and a value (invalid rows carry kl = vl = -1)
                const uint32_t x = hll_mix(h[k]);
                if (((x & skip_mask) | (uint32_t)((kl[k] | vl[k]) >> 31)) == 0 && (clean || use[k])) hll_raise(prm.hll, prm.hll_p, x);
            }
        }
#else
        if (MODE == MODE_HLL) {   // experiment: keep the hashes alive without the sketch
            if ((h[0] ^ h[1] ^ h[2] ^ h[3]) == 0x12345678u) prm.hll[0] = 1;
        }
#endif
    };

    for (int it = 0; tile < ntiles; tile += gstride, ++it) {
        const int buf = it & 1;
        uint32_t info = 0;
        if (HASH) {
            info = __shfl_sync(full, nxt_info, 0);   // also: every lane is done with stage buf^1 before it is refilled
        }
        const bool has_next = tile < ntiles - gstride;   // no overflow: gstride <= SMs * 32
        if (HASH && has_next && lane == 0) nxt_info = issue(phys(tile + gstride), buf ^ 1);
        const int pt = phys(tile);
        if ((int64_t)(pt + 1) * TILE <= prm.n) body(std::true_type{}, pt, buf, info, has_next);
        else body(std::false_type{}, pt, buf, info, has_next);
        // every warp examines the CTA's split sums after every 8th tile of its own (bound: see fold_sums)
        if (SMEM && (it & (FOLD_TILES - 1)) == FOLD_TILES - 1) C.fold_sums(lane, 1u << 30);
        try_uni = try_uni || (it & 15) == 15;   // re-probe for run-structured input now and then
        // HLL floor upkeep: every 4th tile ONE warp of each CTA (the role rotates, so no warp falls behind)
        // refreshes one slice — the 132 CTAs of an H100 cover all 64 slices about every two tile-times — and republishes
        // the floor (plus two early refreshes after the first and second tile, so that a cold sketch stops taking every
        // record); every warp picks the published floor up after its first tiles and then every 16th
        if (MODE == MODE_HLL) {
            if (((it & 3) == 3 && ((it >> 2) & 31) == (warp & 31)) || (it < 2 && warp == it + 1))
                hll_refresh_slice(prm.hll, prm.hll_p, prm.hll_floor, (blockIdx.x + (uint32_t)(it >> 2) * 37u) & (HLL_SLICES - 1), lane);
            if (it < 4 || (it & 15) == 15) floor_reg = ld_cg_u32(prm.hll_floor);
        }
    }

    // ---- flush CTA-private state ----
    __syncthreads();
    if (SMEM) {
        // bucket rows → global [which][p][bucket]; row 32 → knull; row 65 (tombstones) is derived, not stored
        const int nh = (ROW_V + NB) * P;
        for (int i = tid; i < nh; i += blockDim.x) {
            const uint32_t v = scnt[i];
            if (v) {
                const int row = i / P, pp = C.part(i - row * P);
                if (row < NB) atomicAdd(&prm.sums[(size_t)pp * NB + row], (unsigned long long)v);
                else if (row == NB) atomicAdd(&prm.sums[(size_t)prm.P * (2 * NB + 2) + pp], (unsigned long long)v);
                else atomicAdd(&prm.sums[(size_t)(prm.P + pp) * NB + (row - ROW_V)], (unsigned long long)v);
            }
        }
        if (warp == 0) C.fold_sums(lane, 1u);
    }
    // extrema + bad-partition count: warp shuffle, then one lane per warp, then one thread per CTA
    long long smin64 = smin != 0xffffffffu ? (long long)smin : INT64_MAX;
    long long smax64 = smin != 0xffffffffu ? (long long)smax : -1;
#pragma unroll
    for (int d = 16; d; d >>= 1) {
        const long long a = __shfl_xor_sync(full, tmin, d), b = __shfl_xor_sync(full, tmax, d);
        const long long c = __shfl_xor_sync(full, smin64, d), e = __shfl_xor_sync(full, smax64, d);
        tmin = a < tmin ? a : tmin;
        tmax = b > tmax ? b : tmax;
        smin64 = c < smin64 ? c : smin64;
        smax64 = e > smax64 ? e : smax64;
        bad += __shfl_xor_sync(full, bad, d);
    }
    long long *red = reinterpret_cast<long long *>(wsm + 64);   // per-warp scratch (4 × i64)
    if (lane == 0) {
        red[0] = tmin; red[1] = tmax; red[2] = smin64; red[3] = smax64;
        if (bad) atomicAdd(&prm.sums[sums_words(prm.P) - 1], (unsigned long long)bad);
    }
    __syncthreads();
    if (tid == 0) {
        for (int w = 1; w < nwarps; w++) {
            const long long *rw = reinterpret_cast<const long long *>(wsm + (size_t)w * warp_bytes + 64);
            tmin = rw[0] < tmin ? rw[0] : tmin;
            tmax = rw[1] > tmax ? rw[1] : tmax;
            smin64 = rw[2] < smin64 ? rw[2] : smin64;
            smax64 = rw[3] > smax64 ? rw[3] : smax64;
        }
        if (tmin != INT64_MAX) {
            atomicMin(&prm.minmax[0], tmin);
            atomicMax(&prm.minmax[1], tmax);
        }
        if (smax64 >= 0) {
            atomicMin(reinterpret_cast<unsigned long long *>(&prm.minmax[2]), (unsigned long long)smin64);
            atomicMax(reinterpret_cast<unsigned long long *>(&prm.minmax[3]), (unsigned long long)smax64);
        }
    }
}

// ------------------------------------------------------------------------------------------------
// key_tile_base derivation when the caller did not supply it: per-tile byte totals (one warp per
// 128-record tile), then one single-CTA exclusive scan over the tile totals.
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) tile_key_bytes_kernel(const int32_t *key_len, int64_t n, int64_t ntiles,
                                                             uint64_t *tile_base /*[ntiles+1], [t+1] = bytes of tile t*/) {
    const int lane = threadIdx.x & 31;
    const int64_t gw = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5, gs = ((int64_t)gridDim.x * blockDim.x) >> 5;
    for (int64_t tile = gw; tile < ntiles; tile += gs) {
        uint64_t s = 0;
#pragma unroll
        for (int k = 0; k < ROWS; k++) {
            const int64_t r = tile * TILE + k * 32 + lane;
            if (r < n) {
                const int32_t v = key_len[r];
                s += v > 0 ? (uint64_t)v : 0;
            }
        }
#pragma unroll
        for (int d = 16; d; d >>= 1) s += __shfl_xor_sync(0xffffffffu, s, d);
        if (lane == 0) tile_base[tile + 1] = s;
    }
    if (blockIdx.x == 0 && threadIdx.x == 0) tile_base[0] = 0;
}

__global__ void __launch_bounds__(1024) tile_base_scan_kernel(uint64_t *tile_base, int64_t ntiles) {
    // inclusive scan of tile_base[1..ntiles] in place (tile_base[0] == 0), one CTA, chunks of 1024
    __shared__ uint64_t wsum[32];
    __shared__ uint64_t carry_s;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    if (tid == 0) carry_s = 0;
    __syncthreads();
    for (int64_t base = 1; base <= ntiles; base += 1024) {
        const int64_t i = base + tid;
        const uint64_t v = i <= ntiles ? tile_base[i] : 0;
        uint64_t inc = v;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
            const uint64_t t = __shfl_up_sync(0xffffffffu, inc, d);
            if (lane >= d) inc += t;
        }
        if (lane == 31) wsum[warp] = inc;
        __syncthreads();
        uint64_t wb = 0;
        for (int w = 0; w < warp; w++) wb += wsum[w];
        const uint64_t out = carry_s + wb + inc;
        if (i <= ntiles) tile_base[i] = out;
        __syncthreads();
        if (tid == 1023) carry_s = out;
        __syncthreads();
    }
}

// ------------------------------------------------------------------------------------------------
// alive-key table: HLL over the alive set, export / import, rehash (growth), rebase (seq window)
// ------------------------------------------------------------------------------------------------
constexpr int THREADS = 256;  // block size of the table / utility kernels below
// EXTENSION: HyperLogLog over the resolved alive set (only when an HLL precision was asked for together with -c)
__global__ void __launch_bounds__(THREADS) alive_hll_kernel(const unsigned long long *table, size_t nslots, uint32_t *hll, int hll_p) {
    const size_t stride = (size_t)gridDim.x * THREADS;
    for (size_t i = (size_t)blockIdx.x * THREADS + threadIdx.x; i < nslots; i += stride) {
        const unsigned long long v = table[i];
        if (v != ALIVE_EMPTY && (v & 1ull)) hll_raise(hll, hll_p, (uint32_t)(v >> 32));   // the table holds x = fmix32(hash)
    }
}

// mode 0: count the entries; mode 1: append them as (hash, ((seq + 1) << 1) | alive) with absolute sequence numbers
__global__ void __launch_bounds__(THREADS) alive_export_kernel(const unsigned long long *table, size_t nslots, uint64_t origin, int mode,
                                                               unsigned long long *counter, uint32_t *out_hash,
                                                               unsigned long long *out_stamp, unsigned long long cap) {
    const int lane = threadIdx.x & 31;
    const size_t stride = (size_t)gridDim.x * THREADS;
    const size_t rounds = (nslots + stride - 1) / stride;   // every thread runs the same number of rounds (warp votes inside)
    for (size_t it = 0; it < rounds; it++) {
        const size_t i = it * stride + (size_t)blockIdx.x * THREADS + threadIdx.x;
        const unsigned long long v = i < nslots ? table[i] : ALIVE_EMPTY;
        const bool live = v != ALIVE_EMPTY;
        const unsigned m = __ballot_sync(0xffffffffu, live);
        if (!m) continue;
        unsigned long long base = 0;
        if (lane == 0) base = atomicAdd(counter, (unsigned long long)__popc(m));
        base = __shfl_sync(0xffffffffu, base, 0);
        if (mode == 1 && live) {
            const unsigned long long slot = base + __popc(m & ((1u << lane) - 1u));
            if (slot < cap) {
                const unsigned long long field = (v >> 1) & 0x7fffffffull;
                out_hash[slot] = hll_unmix((uint32_t)(v >> 32));   // back to the reference hash
                out_stamp[slot] = ((origin + field) << 1) | (v & 1ull);   // seq + 1 = origin + field
            }
        }
    }
}

__global__ void __launch_bounds__(THREADS) alive_import_kernel(const AliveTable t, uint64_t origin, const uint32_t *hash,
                                                               const unsigned long long *stamp, int64_t count) {
    AliveTable tt = t;
    tt.pol = KTA_L2_HINTS ? l2_policy_evict_last() : 0;
    const int64_t stride = (int64_t)gridDim.x * THREADS;
    for (int64_t i = (int64_t)blockIdx.x * THREADS + threadIdx.x; i < count; i += stride) {
        const unsigned long long st = stamp[i];
        const unsigned long long field = (st >> 1) - origin;        // seq + 1 - origin
        if (field - 1ull >= (unsigned long long)ALIVE_FIELD_MAX) {   // outside the table's 31-bit window
            atomicAdd(t.status + 1, 1u);
            continue;
        }
        const uint32_t x = hll_mix(hash[i]);
        alive_stamp_slow(tt, alive_home(x, t.npairs), x, ((uint32_t)field << 1) | (uint32_t)(st & 1ull));
    }
}

// sum_all_alive (metric.rs:282-284): out[0] += entries whose last writer carried a value, out[2] += occupied slots
__global__ void __launch_bounds__(THREADS) alive_count_kernel(const unsigned long long *table, size_t nslots, unsigned long long *out) {
    const size_t stride = (size_t)gridDim.x * THREADS;
    unsigned alive = 0, occ = 0;
    for (size_t i = (size_t)blockIdx.x * THREADS + threadIdx.x; i < nslots; i += stride) {
        const unsigned long long v = table[i];
        occ += v != ALIVE_EMPTY;
        alive += v != ALIVE_EMPTY && (v & 1ull);
    }
    alive = __reduce_add_sync(0xffffffffu, alive);
    occ = __reduce_add_sync(0xffffffffu, occ);
    if ((threadIdx.x & 31) == 0) {
        if (alive) atomicAdd(out, (unsigned long long)alive);
        if (occ) atomicAdd(out + 2, (unsigned long long)occ);
    }
}

// growth: every entry of the old table moves to its place in the new one (hashes are unique, so plain claims)
__global__ void __launch_bounds__(THREADS) alive_rehash_kernel(const unsigned long long *old_slots, size_t old_nslots,
                                                               unsigned long long *new_slots, uint32_t new_npairs, uint32_t *status) {
    const size_t stride = (size_t)gridDim.x * THREADS;
    for (size_t i = (size_t)blockIdx.x * THREADS + threadIdx.x; i < old_nslots; i += stride) {
        const unsigned long long v = old_slots[i];
        if (v != ALIVE_EMPTY && !alive_insert_unique(new_slots, new_npairs, v)) atomicAdd(status, 1u);
    }
}

// rebase: all entries become "older than anything that follows" (seq field 0), keeping hash and alive bit
__global__ void __launch_bounds__(THREADS) alive_rebase_kernel(unsigned long long *slots, size_t nslots) {
    const size_t stride = (size_t)gridDim.x * THREADS;
    for (size_t i = (size_t)blockIdx.x * THREADS + threadIdx.x; i < nslots; i += stride) {
        const unsigned long long v = slots[i];
        if (v != ALIVE_EMPTY) slots[i] = v & 0xffffffff00000001ull;
    }
}

// state (re)initialisation: sums = 0, minmax = {+inf, -inf, u64 max, 0}, hll = 0, hll floor = 0
__global__ void state_init_kernel(unsigned long long *sums, size_t nsums, long long *minmax, uint32_t *hll, size_t nhll,
                                  uint32_t *hll_floor) {
    const size_t stride = (size_t)gridDim.x * blockDim.x;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < nsums; i += stride) sums[i] = 0;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < nhll; i += stride) hll[i] = 0;
    if (blockIdx.x == 0 && threadIdx.x == 0) {
        minmax[0] = INT64_MAX;
        minmax[1] = INT64_MIN;
        reinterpret_cast<unsigned long long *>(minmax)[2] = ~0ull;
        reinterpret_cast<unsigned long long *>(minmax)[3] = 0ull;
        for (int i = 0; i <= HLL_SLICES; i++) hll_floor[i] = 0;
    }
}

// test hook: the reference hash of n packed keys (src/fnv32.rs:92-101)
__global__ void fnv32_kernel(int64_t n, const int32_t *key_len, const uint64_t *key_off, const uint8_t *key_bytes,
                             uint32_t *out) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
        out[i] = key_len[i] < 0 ? 0u : fnv_global(key_bytes + key_off[i], key_len[i]);
}

// ---- multi-GPU merge buffer (see kta.h): [sums | G×4 minmax slots | G×(nhll/8) register words] ----
// Every rank writes its min/max scalars and HLL registers (one byte each, eight per word) into its own slot and
// zeros elsewhere, so ONE SUM all-reduce over u64 delivers every rank's values to every rank; the import folds them.
__global__ void merge_export_kernel(const unsigned long long *sums, size_t nsums, const long long *minmax,
                                    const uint32_t *hll, size_t nhll, int rank, int world, unsigned long long *buf) {
    const size_t stride = (size_t)gridDim.x * blockDim.x, t0 = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    const size_t nmm = (size_t)world * 4, hw = nhll / 8, total = nsums + nmm + (size_t)world * hw;
    for (size_t i = t0; i < total; i += stride) {
        unsigned long long v = 0;
        if (i < nsums) v = sums[i];
        else if (i < nsums + nmm) {
            const size_t j = i - nsums;
            if ((int)(j / 4) == rank) v = (unsigned long long)minmax[j % 4];
        } else {
            const size_t j = i - nsums - nmm;
            if ((int)(j / hw) == rank) {
                const uint32_t *r = hll + (j % hw) * 8;
#pragma unroll
                for (int k = 0; k < 8; k++) v |= (unsigned long long)(r[k] & 0xffu) << (8 * k);
            }
        }
        buf[i] = v;
    }
}

__global__ void merge_import_kernel(unsigned long long *sums, size_t nsums, long long *minmax, uint32_t *hll,
                                    size_t nhll, uint32_t *hll_floor, int world, const unsigned long long *buf) {
    const size_t stride = (size_t)gridDim.x * blockDim.x, t0 = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    for (size_t i = t0; i < nsums; i += stride) sums[i] = buf[i];
    const unsigned long long *mm = buf + nsums;
    const size_t hw = nhll / 8;
    const unsigned long long *hb = mm + (size_t)world * 4;
    for (size_t i = t0; i < nhll; i += stride) {
        uint32_t m = 0;
        for (int r = 0; r < world; r++) m = max(m, (uint32_t)(hb[(size_t)r * hw + i / 8] >> (8 * (i % 8))) & 0xffu);
        hll[i] = m;
    }
    if (t0 == 0) {
        long long tmin = INT64_MAX, tmax = INT64_MIN;
        unsigned long long smin = ~0ull, smax = 0;
        for (int r = 0; r < world; r++) {
            tmin = min(tmin, (long long)mm[r * 4 + 0]);
            tmax = max(tmax, (long long)mm[r * 4 + 1]);
            smin = min(smin, mm[r * 4 + 2]);
            smax = max(smax, mm[r * 4 + 3]);
        }
        minmax[0] = tmin;
        minmax[1] = tmax;
        reinterpret_cast<unsigned long long *>(minmax)[2] = smin;
        reinterpret_cast<unsigned long long *>(minmax)[3] = smax;
        for (int i = 0; i <= HLL_SLICES; i++) hll_floor[i] = 0;
    }
}

}  // namespace kta
