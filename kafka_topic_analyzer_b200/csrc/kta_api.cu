// kta_api.cu — host side of libkta_gpu.so: the C ABI of include/kta.h over the sm_90a kernels.
//
// Mirrors, for this one path, what the reference's host does around the handlers:
//   MessageMetrics::new / LogCompactionInMemoryMetrics::new      src/metric.rs:30-46, 267-271
//   one handle_message per polled record                         src/kafka.rs:107-109
//   getters + derived values read by the report                  src/metric.rs:104-203, src/main.rs:130-170
// There is deliberately no CPU implementation of the scan in this file: if CUDA is unusable every
// compute entry point fails with KTA_ERR_CUDA.
#include <cuda_runtime.h>

#include <algorithm>
#include <chrono>
#include <climits>
#include <cmath>
#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <new>
#include <vector>

#include "kta_host.cuh"
#include "kta_hotkeys.cuh"
#include "kta_kernels.cuh"
#include "kta_logscan.cuh"
#include "kta_partitioner.cuh"
#include "kta_synth.h"
#include "kta_timeline.cuh"

using namespace kta;

// ------------------------------------------------------------------------------------------------
// errors
// ------------------------------------------------------------------------------------------------
extern "C" const char *kta_last_error(void) { return g_err; }
extern "C" int kta_abi_version(void) { return KTA_ABI_VERSION; }
extern "C" int kta_device_count(void) {
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess) {
        cudaGetLastError();
        return -1;
    }
    return n;
}

// ------------------------------------------------------------------------------------------------
// handle
// ------------------------------------------------------------------------------------------------
static constexpr int NCHUNK = 3;
static constexpr int32_t ALIVE_DEFAULT_KIB = 256 * 1024;       // initial alive-key table: 256 MiB = 2^25 slots
static constexpr int32_t ALIVE_MAX_KIB = 32 * 1024 * 1024;     // 32 GiB = one slot per possible 32-bit hash
static constexpr int64_t ALIVE_CACHE_MIN_RECORDS = 1 << 20;    // smaller batches go straight to the table
static constexpr int64_t DEFAULT_RING_RECORDS = 1 << 22;  // 4 Mi records per chunk

struct Chunk {
    // device staging (shared by kta_push and kta_push_batch_host)
    DevBuf<int32_t> d_partition, d_klen, d_vlen;
    DevBuf<int64_t> d_ts;
    DevBuf<uint64_t> d_seq;
    DevBuf<uint8_t> d_keys;
    DevBuf<uint64_t> d_tile_base;
    cudaEvent_t free_ev = nullptr;  // recorded after the scan that reads this chunk
    // pinned landing area for kta_push
    PinnedBuf<int32_t> h_partition, h_klen, h_vlen;
    PinnedBuf<int64_t> h_ts;
    PinnedBuf<uint8_t> h_keys;
    PinnedBuf<uint64_t> h_tile_base;
};

// Stamps the alive-key table has not confirmed yet (it may turn out too small: then they are applied again, which is
// idempotent).  Their inputs are still valid: caller buffers until kta_sync / kta_finalize by contract, ring chunks
// until they are reused, an imported list until kta_alive_import_device returns.
struct AlivePending {
    ScanParams prm;   // a MODE_EXACT scan (count == 0) as first launched, seen-cache waves included
    int64_t key_readable, key_bytes;
    int chunk;        // ring chunk the columns live in, -1 = caller-owned / scratch device buffers
    const uint32_t *hash; const uint64_t *stamp; int64_t count;   // an import (count > 0) of exported pairs
};

// Host side of the exact alive-key table (-c); only the alive_* functions read the status words or the pending list
struct AliveKeys {
    DevBuf<unsigned long long> d_table;      // open-addressed last-writer table, 2 * pairs slots
    uint32_t pairs = 0;
    uint64_t origin = 0;                     // seq that a stamp's field value 1 stands for
    bool rebased = false;                    // a rebase dropped absolute sequence numbers (exports are refused then)
    DevBuf<uint32_t> d_cache;                // seen cache of the batch being scanned (32 MiB, cleared per launch)
    DevBuf<uint32_t> d_status;               // [0] stamps that found no slot, [1] records outside the seq window, [2] wide re-run
    PinnedBuf<uint32_t> h_status;            // [0..1] read by alive_settle, [2c + 2..] snapshot behind ring chunk c's scan
    DevBuf<unsigned long long> d_count;      // [0] alive entries, [1] export cursor, [2] occupied slots
    uint64_t window_errors = 0;              // sticky until reset: reported by kta_finalize
    uint64_t grows = 0, reruns = 0;
    uint64_t now = 0, occupied = 0;          // counted by the last alive_settle
    std::vector<AlivePending> pending;
};

// The timeline extension (kta_set_timeline): its configuration and its three [P][B + 2] u64 arrays
struct Timeline {
    int32_t buckets = 0;                     // B; 0 = off
    int64_t origin = 0, width = 1;           // O, W (seconds)
    bool smem = false;                       // bins in shared memory (P * (B + 2) of them fit the opt-in shared memory)
    int blocks_per_sm = 0;                   // CTAs of timeline_kernel per SM (occupancy of the chosen instance)
    DevBuf<unsigned long long> d_bins;       // [3][P][B + 2]: records | tombstones | bytes
    std::vector<uint64_t> h_bins;            // host mirror, valid after finalize
    size_t words() const { return d_bins.cap > 0 ? (size_t)d_bins.cap : 0; }
};

// The partitioner check (kta_set_partitioner_check): its counts and its [2C + 1][P] u64 counters
struct Partitioner {
    int32_t ncounts = 0;                     // C; 0 = off
    int32_t counts[KTA_PARTITIONER_MAX_COUNTS] = {};
    bool smem = false;                       // counters in shared memory ((2C + 1) P of them fit beside the table and stages)
    int32_t max_grid = 0;                    // test hook (kta_partitioner_limit_grid): at most this many CTAs; 0 = no limit
    DevBuf<unsigned long long> d_counts;     // [2C + 1][P]: murmur2 per count | CRC-32 per count | neither
    std::vector<uint64_t> h_counts;          // host mirror, valid after finalize
    size_t words() const { return d_counts.cap > 0 ? (size_t)d_counts.cap : 0; }
};

// The hot-key table (kta_set_hot_keys): its configuration, the table, the occupancy bound and the host mirror; only the
// hk_* functions and the hot-key entry points touch them
struct HotKeys {
    int32_t top_k = 0;                       // 0 = off
    uint64_t slots = 0;                      // power of two; the side slot (id 0) follows them
    uint64_t max_slots = 0;                  // test hook (kta_hot_keys_limit_slots): 0 = no cap
    DevBuf<HkSlot> d_table;                  // [slots + 1]
    DevBuf<unsigned long long> d_word;       // [0] occupancy, [1] probe failure (u32), [2] export cursor, [3] records, [4] refusal
    uint64_t bound = 0;                      // U: the occupancy is at most this
    uint64_t grows = 0, slices = 0;
    bool nomem = false;                      // growth failed: nothing is counted until kta_reset
    bool unreported = false;                 // ... and the entry point that scanned has not returned KTA_ERR_NOMEM yet
    char nomem_msg[256] = "";
    // finalize's scratch and the host mirror (valid after finalize)
    DevBuf<kta_hot_key> d_entries, d_top;
    DevBuf<HkSortKey> d_keys;                // [2][distinct]
    DevBuf<uint32_t> d_idx;                  // [2][distinct]
    DevBuf<uint8_t> d_sort_tmp;
    std::vector<kta_hot_key> h_top;
    uint64_t h_distinct = 0, h_keyed = 0;
    HkTable table() { return HkTable{d_table, slots, d_word, reinterpret_cast<unsigned int *>(d_word.get() + 1)}; }
};

struct kta_handle {
    kta_config cfg{};
    int device = 0;
    int sm_count = 0;
    cudaStream_t stream = nullptr;
    bool own_stream = true;
    bool need_hash = false;
    // device state
    DevBuf<unsigned long long> d_sums;
    DevBuf<long long> d_minmax;
    DevBuf<uint32_t> d_hll;
    DevBuf<uint32_t> d_hll_floor;            // hll floor + slice minima
    AliveKeys alive;                         // count_alive_keys only
    uint32_t *d_hash_out = nullptr;          // test hook (the caller's buffer)
    DevBuf<uint64_t> d_tb_scratch;           // key_tile_base scratch for device batches and decoded segments
    LogScan log;
    Timeline tl;
    Partitioner pt;
    HotKeys hk;
    DevBuf<uint32_t> d_crc32_tables;         // zlib CRC-32 slicing tables of the partitioner check and the hot-key table (made on first use)
    size_t nsums = 0, nhll = 0;
    // landing ring
    Chunk chunks[NCHUNK];
    bool ring_dev_ready = false, ring_host_ready = false;
    int64_t ring_records = 0, ring_key_bytes = 0;
    int cur = 0;          // chunk being filled by kta_push
    // kta_push's hot state: raw cursors into that chunk's pinned landing area (one cache line, no indirection per call)
    struct PushCursor {
        int32_t *part = nullptr, *klen = nullptr, *vlen = nullptr;
        int64_t *ts = nullptr;
        uint8_t *keys = nullptr;
        uint64_t *tile_base = nullptr;
        int64_t n = 0, cap = 0;     // records in the chunk / its capacity (0 until the ring exists: first push takes the slow path)
        int64_t kb = 0, kcap = 0;   // key bytes in the chunk / capacity
        bool hash = false;          // key bytes travel only when they are hashed
    } pc;
    uint64_t next_seq = 0;   // seq of the first record not yet handed to a scan (records in the open chunk follow it)
    // host mirror (valid after finalize)
    bool finalized = false;
    std::vector<uint64_t> h_sums;
    long long h_minmax[4] = {0, 0, 0, 0};
    std::vector<uint32_t> h_hll;
    uint64_t h_alive = 0;
    // occupancy-derived grids
    int shard_world = 1, shard_rank = 0;     // partition-sharded scan: only partitions p % world == rank reach this handle
    int columns = 0;                         // counter columns the scan kernel carves = partitions this handle owns
    bool smem_counters = true;               // per-partition counters fit in shared memory
    size_t smem_optin = 0;
    // stats / timing
    uint64_t launches = 0, records = 0;
    bool timing = false;
    std::vector<std::pair<cudaEvent_t, cudaEvent_t>> ev_pool;
    size_t ev_used = 0;
    double scan_ms = 0;
    uint64_t scan_launches_timed = 0;
};

static int set_device(const kta_handle *h) {
    CU(cudaSetDevice(h->device));
    return KTA_OK;
}

// key bytes travel to the device only when they are hashed, by the scan, the partitioner check or the hot-key table
// (kta_push reads the copy in pc.hash)
static bool keys_travel(const kta_handle *h) { return h->need_hash || h->d_hash_out || h->pt.ncounts || h->hk.top_k; }

static size_t scan_smem_bytes(bool hash, bool smem, int P, int threads, int keybuf, int stages, bool hdr) {
    return (smem ? smem_counter_bytes(P) : CTA_SCRATCH) + (size_t)(threads / 32) * warp_smem_bytes(hash, keybuf, stages, hdr);
}

// Launch shape for one scan.  Counters mode: 32 warps, nothing staged.  Hashing modes: the key part of a stage from the
// batch's mean key length, then the first shape that fits the shared memory left next to the counter rows:
//   with headers staged (only if the columns are aligned): SCAN_STAGES (3) stages with 12..10 warps, else 2 stages with
//   12..10 warps.  12 x 3 is the fastest shape measured at C1 (16-byte keys, 64 partitions);
//   keys only: 2 stages with 16..8 warps.  With fewer than 10 warps, staging the headers as well was measured slower
//   than keys alone at more warps (512 or 692 partitions, 36- or 64-byte keys: profiles/h100_shapes.log);
//   the smallest key part at 2 stages (keys that do not fit it are hashed from global memory).
static void scan_shape(const kta_handle *h, bool hash, bool hdr_ok, int64_t n, int64_t key_bytes, int &threads, int &keybuf,
                       int &stages, bool &hdr, size_t &smem) {
    const int P = h->columns;
    keybuf = KEYBUF_MIN;
    stages = 0;
    hdr = false;
    if (!hash) {
        threads = MAX_THREADS;
        smem = scan_smem_bytes(false, h->smem_counters, P, threads, keybuf, stages, hdr);
        return;
    }
    if (n > 0) {
        const int64_t per_tile = (key_bytes * TILE + n - 1) / n;           // mean key bytes per 128-record tile
        int64_t want = per_tile + per_tile / 8 + 64 + KEYBUF_SLACK;       // 12.5 % headroom for ragged tiles (~2.4 sigma for 0..40 B keys)
        want = (want + 127) / 128 * 128;
        keybuf = (int)std::min<int64_t>(std::max<int64_t>(want, KEYBUF_MIN), KEYBUF_MAX);
        keybuf = (keybuf + 15) / 16 * 16;
    }
    auto fits = [&](bool with_hdr, int st, int max_warps, int min_warps) {
        hdr = with_hdr;
        stages = st;
        for (threads = std::min(max_warps * 32, HASH_MAX_THREADS); threads >= min_warps * 32; threads -= 32) {
            smem = scan_smem_bytes(true, h->smem_counters, P, threads, keybuf, stages, hdr);
            if (smem <= h->smem_optin) return true;
        }
        return false;
    };
    if (hdr_ok && (fits(true, SCAN_STAGES, 12, 10) || fits(true, 2, 12, 10))) return;
    if (fits(false, 2, 16, 8)) return;
    keybuf = KEYBUF_MIN;
    fits(false, 2, 16, 1);
}

// Every scan_kernel instance the library launches, [counters in shared memory][partition-sharded][mode][capture].
// Hash capture is a test hook of unsharded hashing handles; the other slots are empty.  One persistent CTA per SM;
// every instance may use the whole opt-in shared memory (the shape is chosen per launch).
using ScanFn = void (*)(ScanParams);
static const ScanFn SCAN_KERNELS[2][2][3][2] = {
    {{{scan_kernel<MODE_COUNTERS, false, false, false>, nullptr},
      {scan_kernel<MODE_HLL, false, false, false>, scan_kernel<MODE_HLL, false, true, false>},
      {scan_kernel<MODE_EXACT, false, false, false>, scan_kernel<MODE_EXACT, false, true, false>}},
     {{scan_kernel<MODE_COUNTERS, false, false, true>, nullptr},
      {scan_kernel<MODE_HLL, false, false, true>, nullptr},
      {scan_kernel<MODE_EXACT, false, false, true>, nullptr}}},
    {{{scan_kernel<MODE_COUNTERS, true, false, false>, nullptr},
      {scan_kernel<MODE_HLL, true, false, false>, scan_kernel<MODE_HLL, true, true, false>},
      {scan_kernel<MODE_EXACT, true, false, false>, scan_kernel<MODE_EXACT, true, true, false>}},
     {{scan_kernel<MODE_COUNTERS, true, false, true>, nullptr},
      {scan_kernel<MODE_HLL, true, false, true>, nullptr},
      {scan_kernel<MODE_EXACT, true, false, true>, nullptr}}},
};

// ------------------------------------------------------------------------------------------------
// alive-key table (-c): seq window (rebase), confirmation of pending stamps, growth (rehash + re-run), export / import
// ------------------------------------------------------------------------------------------------
static int launch_scan_raw(kta_handle *h, ScanParams prm, int64_t key_readable, int64_t key_bytes);
static int ring_flush(kta_handle *h);
static int hk_finalize(kta_handle *h);

static int alive_create(kta_handle *h) {
    // open-addressed last-writer table keyed by the 32-bit hash, sized by the number of DISTINCT hashes and grown
    // on demand (alive_settle): 256 MiB = 2^25 slots holds the 1e7 keys of BASELINE configs[2] at load 0.3 (at 0.6
    // every third first-seen key finds its home pair taken and probes on; the table does not fit L2 at either size)
    const int64_t kib = h->cfg.alive_table_kib;
    if (kib < 0 || kib > ALIVE_MAX_KIB) return fail(KTA_ERR_INVALID, "alive_table_kib %d out of range [0, %d]", (int)kib, ALIVE_MAX_KIB);
    AliveKeys &a = h->alive;
    a.pairs = (uint32_t)std::max<int64_t>((kib ? kib : ALIVE_DEFAULT_KIB) * 64, 16);   // 16 bytes per pair
    int rc;
    if ((rc = a.d_table.alloc((int64_t)a.pairs * 2)) || (rc = a.d_status.alloc(3)) || (rc = a.d_count.alloc(3)) ||
        (rc = a.d_cache.alloc((int64_t)1 << ALIVE_CACHE_SET_BITS)) || (rc = a.h_status.alloc(2 * (NCHUNK + 1))))
        return rc;
    return KTA_OK;
}

static int alive_reset(kta_handle *h) {
    AliveKeys &a = h->alive;
    if (!a.d_table) return KTA_OK;
    // the table is a few hundred MB at most for the topics it is meant for: wiping it is one short memset
    CU(cudaMemsetAsync(a.d_table, 0xff, (size_t)a.pairs * 16, h->stream));
    CU(cudaMemsetAsync(a.d_status, 0, 12, h->stream));
    a.now = a.occupied = a.origin = 0;
    a.rebased = false;
    a.window_errors = 0;
    a.pending.clear();
    return KTA_OK;
}

static int alive_grow(kta_handle *h, uint32_t new_pairs) {
    AliveKeys &a = h->alive;
    cudaStream_t s = h->stream;
    DevBuf<unsigned long long> nt;
    int rc;
    if ((rc = nt.alloc((int64_t)new_pairs * 2))) return rc;
    CU(cudaMemsetAsync(nt, 0xff, (size_t)new_pairs * 16, s));
    alive_rehash_kernel<<<h->sm_count * 8, THREADS, 0, s>>>(a.d_table, (size_t)a.pairs * 2, nt, new_pairs, a.d_status);
    h->launches++;
    CU(cudaGetLastError());
    CU(cudaStreamSynchronize(s));
    a.d_table = std::move(nt);   // nt frees the old table
    a.pairs = new_pairs;
    a.grows++;
    return KTA_OK;
}

// applies a pending entry's stamps (again) to the table as it is now: an import as it was, a scan stamps-only
static int alive_apply(kta_handle *h, const AlivePending &p) {
    AliveKeys &a = h->alive;
    if (p.count) {
        const int grid = (int)std::min<int64_t>((p.count + THREADS - 1) / THREADS, (int64_t)h->sm_count * 8);
        alive_import_kernel<<<grid, THREADS, 0, h->stream>>>(AliveTable{a.d_table, a.pairs, a.d_status, 0}, a.origin, p.hash,
                                                             reinterpret_cast<const unsigned long long *>(p.stamp), p.count);
        h->launches++;
        CU(cudaGetLastError());
        return KTA_OK;
    }
    ScanParams prm = p.prm;
    prm.alive_only = 1;
    prm.alive_table = a.d_table;   // the table may have grown since
    prm.alive_pairs = a.pairs;
    a.reruns++;                    // re-stamped batches (kta.h): imports are not counted
    return launch_scan_raw(h, prm, p.key_readable, p.key_bytes);
}

// Confirms every pending entry: waits for the stream, reads the status words, and while stamps were dropped applies
// the pending entries again (idempotent: atomicMax).  Afterwards nothing is pending.
//   * If the table would stay at most 60 % full even were every dropped stamp a new key, the drops are a probe-limit
//     artefact: keys whose mixed hashes lie close together share a home pair at every table size, and a crafted run of
//     a few hundred of them would otherwise double the table up to its 32 GiB cap.  The re-run keeps the table and lets
//     the probe run over all of it (status[2]); a linear probe in a table at most 60 % full always reaches an empty slot.
//   * Otherwise the table is grown first.  It is also grown ahead of need once it is more than 60 % full.
static int alive_settle(kta_handle *h) {
    AliveKeys &a = h->alive;
    if (!a.d_table) return KTA_OK;
    cudaStream_t s = h->stream;
    for (int round = 0;; round++) {
        unsigned long long counts[3] = {0, 0, 0};   // alive, (export cursor), occupied
        CU(cudaMemsetAsync(a.d_count, 0, 24, s));
        alive_count_kernel<<<h->sm_count * 8, THREADS, 0, s>>>(a.d_table, (size_t)a.pairs * 2, a.d_count);
        h->launches++;
        CU(cudaGetLastError());
        CU(cudaMemcpyAsync(a.h_status, a.d_status, 8, cudaMemcpyDeviceToHost, s));
        CU(cudaMemcpyAsync(counts, a.d_count, 24, cudaMemcpyDeviceToHost, s));
        CU(cudaStreamSynchronize(s));
        const unsigned long long occupied = counts[2];
        a.now = counts[0];
        a.occupied = occupied;
        const uint32_t dropped = a.h_status[0];
        a.window_errors += a.h_status[1];
        if (dropped || a.h_status[1]) CU(cudaMemsetAsync(a.d_status, 0, 8, s));
        const uint64_t slots = (uint64_t)a.pairs * 2;
        const bool crowded = occupied * 10 > slots * 6;
        if (!dropped && !crowded) break;
        const bool wide = dropped && (occupied + dropped) * 10 <= slots * 6;
        int rc;
        if (!wide) {
            if (a.pairs >= (uint32_t)ALIVE_MAX_KIB * 64u) {
                if (dropped) return fail(KTA_ERR_NOMEM, "alive-key table is at its maximum (32 GiB) and still too full");
                break;
            }
            // at least double; enough for every known entry plus every dropped stamp at load <= 0.5
            uint64_t want = slots * 2;
            while (want < (occupied + dropped) * 2) want *= 2;
            want = std::min<uint64_t>(want, (uint64_t)ALIVE_MAX_KIB * 128ull);
            if ((rc = alive_grow(h, (uint32_t)(want / 2)))) return rc;
            if (!dropped) break;   // grown ahead of need: every pending stamp had landed
        }
        if (round > 40) return fail(KTA_ERR_INVALID, "alive-key table growth did not converge");
        if (wide) CU(cudaMemsetAsync(a.d_status + 2, 0xff, 4, s));
        for (const AlivePending &p : a.pending)
            if ((rc = alive_apply(h, p))) return rc;
        if (wide) CU(cudaMemsetAsync(a.d_status + 2, 0, 4, s));
    }
    a.pending.clear();
    return KTA_OK;
}

// settles only when something is pending (no count of the table otherwise)
static int alive_settle_if_any(kta_handle *h) { return h->alive.pending.empty() ? KTA_OK : alive_settle(h); }

// Fills in the alive-table fields (zero so far) of a MODE_EXACT scan's params; the stamps must fit the table's 31-bit window
// [origin, origin + ALIVE_FIELD_MAX).  `seq_ends`: host copy of seq[0], seq[n-1] when the seq column came from the host.
static int alive_prepare(kta_handle *h, ScanParams &prm, const uint64_t *seq_ends) {
    AliveKeys &a = h->alive;
    int rc;
    if ((uint64_t)prm.n > (uint64_t)ALIVE_FIELD_MAX - 1)
        return fail(KTA_ERR_INVALID, "batch of %lld records with count_alive_keys: split it (< 2^31 per scan)", (long long)prm.n);
    if (prm.seq_base < a.origin)
        return fail(KTA_ERR_INVALID, "seq_base %llu lies before the alive-key table's window origin %llu (batches must not "
                    "go back past a rebase)", (unsigned long long)prm.seq_base, (unsigned long long)a.origin);
    // explicit seq columns are checked record by record in the kernel; the implicit range is checked here
    if (!prm.seq && prm.seq_base - a.origin + (uint64_t)prm.n > (uint64_t)ALIVE_FIELD_MAX) {
        // rebase: everything already in the table is older than this batch; forget by how much.  A re-run launches
        // the params of its first launch, origin and waves included, so nothing may stay pending across a rebase.
        if ((rc = alive_settle(h))) return rc;
        if (!a.pending.empty()) return fail(KTA_ERR_INVALID, "internal: alive-key stamps pending across a rebase");
        alive_rebase_kernel<<<h->sm_count * 8, THREADS, 0, h->stream>>>(a.d_table, (size_t)a.pairs * 2);
        h->launches++;
        CU(cudaGetLastError());
        a.origin = prm.seq_base;
        a.rebased = true;
    }
    prm.alive_table = a.d_table;
    prm.alive_pairs = a.pairs;
    prm.alive_origin = a.origin;
    prm.alive_fbase = prm.seq_base - a.origin + 1ull;
    prm.alive_status = a.d_status;
    if (prm.n >= ALIVE_CACHE_MIN_RECORDS) {
        // the seen cache pays for its clearing (a 32 MiB memset) on batches of a million records and more.
        // Waves cut the batch's seq range [lo, hi] into <= 127 equal slices (any monotone function of seq will do).
        uint64_t lo = prm.seq_base, hi = prm.seq_base + (uint64_t)prm.n - 1;
        bool ok = true;
        if (prm.seq) {
            // explicit sequence numbers: the range is read off the column's ends (records of a batch are in seq order; a
            // record outside the range just lands in the first or last wave)
            uint64_t ends[2];
            if (seq_ends) { ends[0] = seq_ends[0]; ends[1] = seq_ends[1]; }
            else {
                CU(cudaMemcpyAsync(&ends[0], prm.seq, 8, cudaMemcpyDeviceToHost, h->stream));
                CU(cudaMemcpyAsync(&ends[1], prm.seq + (prm.n - 1), 8, cudaMemcpyDeviceToHost, h->stream));
                CU(cudaStreamSynchronize(h->stream));
            }
            lo = std::min(ends[0], ends[1]);
            hi = std::max(ends[0], ends[1]);
            ok = lo >= a.origin && hi - a.origin < (uint64_t)ALIVE_FIELD_MAX;
        }
        if (ok) {
            prm.alive_cache = a.d_cache;
            int sh = 0;
            while (((hi - lo) >> sh) + 1 > (uint64_t)ALIVE_CACHE_WAVES) sh++;
            prm.alive_wave_shift = sh;
            prm.alive_wave_base = (uint32_t)(lo - a.origin + 1ull);   // the stamp field of seq lo
        }
    }
    return KTA_OK;
}

// a MODE_EXACT scan was launched: its stamps are pending; a ring chunk's scan is followed by a status snapshot
static int alive_scanned(kta_handle *h, const ScanParams &prm, int64_t key_readable, int64_t key_bytes, int chunk) {
    AliveKeys &a = h->alive;
    if (chunk >= 0) CU(cudaMemcpyAsync(a.h_status + 2 * (chunk + 1), a.d_status, 8, cudaMemcpyDeviceToHost, h->stream));
    a.pending.push_back(AlivePending{prm, key_readable, key_bytes, chunk, nullptr, nullptr, 0});
    return KTA_OK;
}

// a ring chunk is about to be overwritten: its scan must be confirmed first (the chunk's event has been waited for,
// so its status snapshot is valid)
static int alive_release_chunk(kta_handle *h, int ci) {
    AliveKeys &a = h->alive;
    size_t keep = a.pending.size();   // one past the newest entry of this chunk
    while (keep > 0 && a.pending[keep - 1].chunk != ci) keep--;
    if (keep == 0) return KTA_OK;
    const uint32_t *snap = a.h_status + 2 * (ci + 1);
    if (snap[0] | snap[1]) return alive_settle(h);   // something was dropped up to this scan: settle everything
    // nothing dropped up to and including this chunk's scan: it — and every older pending entry — is confirmed
    a.pending.erase(a.pending.begin(), a.pending.begin() + (long)keep);
    return KTA_OK;
}

static int alive_export(kta_handle *h, int mode, uint32_t *dh, uint64_t *ds, int64_t cap, int64_t *count) {
    if (!h || !count) return fail(KTA_ERR_INVALID, "bad argument");
    AliveKeys &a = h->alive;
    if (!a.d_table) return fail(KTA_ERR_NOT_ENABLED, "count_alive_keys was not enabled");
    int rc;
    if ((rc = set_device(h))) return rc;
    if ((rc = ring_flush(h))) return rc;
    if ((rc = alive_settle(h))) return rc;
    if (a.rebased)
        return fail(KTA_ERR_INVALID, "the alive-key table was rebased (more than 2^31 sequence numbers since kta_reset): its "
                    "entries no longer carry absolute sequence numbers and cannot be merged across GPUs");
    CU(cudaMemsetAsync(a.d_count + 1, 0, 8, h->stream));
    alive_export_kernel<<<h->sm_count * 8, THREADS, 0, h->stream>>>(
        a.d_table, (size_t)a.pairs * 2, a.origin, mode, a.d_count + 1, dh,
        reinterpret_cast<unsigned long long *>(ds), (unsigned long long)cap);
    h->launches++;
    CU(cudaGetLastError());
    unsigned long long c = 0;
    CU(cudaMemcpyAsync(&c, a.d_count + 1, 8, cudaMemcpyDeviceToHost, h->stream));
    CU(cudaStreamSynchronize(h->stream));
    *count = (int64_t)c;
    if (mode == 1 && (int64_t)c > cap) return fail(KTA_ERR_INVALID, "export buffer too small: %llu > %lld", c, (long long)cap);
    return KTA_OK;
}

extern "C" int kta_alive_export_count(kta_handle *h, int64_t *count) { return alive_export(h, 0, nullptr, nullptr, 0, count); }

extern "C" int kta_alive_export_device(kta_handle *h, uint32_t *dev_hash, uint64_t *dev_stamp, int64_t cap, int64_t *count) {
    if (!dev_hash || !dev_stamp) return fail(KTA_ERR_INVALID, "bad argument");
    return alive_export(h, 1, dev_hash, dev_stamp, cap, count);
}

// an imported list is pending work like a scan: applied, then settled
extern "C" int kta_alive_import_device(kta_handle *h, const uint32_t *dev_hash, const uint64_t *dev_stamp, int64_t count) {
    if (!h || count < 0 || (count && (!dev_hash || !dev_stamp))) return fail(KTA_ERR_INVALID, "bad argument");
    AliveKeys &a = h->alive;
    if (!a.d_table) return fail(KTA_ERR_NOT_ENABLED, "count_alive_keys was not enabled");
    if (count == 0) return KTA_OK;
    int rc;
    if ((rc = set_device(h))) return rc;
    if ((rc = alive_settle(h))) return rc;
    const AlivePending p{ScanParams{}, 0, 0, -1, dev_hash, dev_stamp, count};
    if ((rc = alive_apply(h, p))) return rc;
    a.pending.push_back(p);
    if ((rc = alive_settle(h))) return rc;
    h->finalized = false;
    return KTA_OK;
}

static int state_reset_device(kta_handle *h) {
    state_init_kernel<<<64, 256, 0, h->stream>>>(h->d_sums, h->nsums, h->d_minmax, h->d_hll, h->nhll, h->d_hll_floor);
    h->launches++;
    CU(cudaGetLastError());
    return alive_reset(h);
}

// the handle's buffers free themselves; its streams and events are released here
extern "C" int kta_destroy(kta_handle *h) {
    if (!h) return KTA_OK;
    cudaSetDevice(h->device);
    if (h->stream) cudaStreamSynchronize(h->stream);
    for (auto &c : h->chunks)
        if (c.free_ev) cudaEventDestroy(c.free_ev);
    for (auto &e : h->ev_pool) { cudaEventDestroy(e.first); cudaEventDestroy(e.second); }
    cudaStream_t own = h->own_stream ? h->stream : nullptr;
    delete h;
    if (own) cudaStreamDestroy(own);
    cudaGetLastError();
    return KTA_OK;
}

static int create_impl(const kta_config *cfg, kta_handle *h) {
    h->cfg = *cfg;
    if (cfg->num_partitions < 1 || cfg->num_partitions > (1 << 20))
        return fail(KTA_ERR_INVALID, "num_partitions %d out of range [1, 2^20]", cfg->num_partitions);
    if (cfg->hll_precision != 0 && (cfg->hll_precision < 4 || cfg->hll_precision > 18))
        return fail(KTA_ERR_INVALID, "hll_precision %d not 0 or 4..18", cfg->hll_precision);
    if (cfg->isolation_level != KTA_READ_UNCOMMITTED && cfg->isolation_level != KTA_READ_COMMITTED)
        return fail(KTA_ERR_INVALID, "isolation_level %d is neither KTA_READ_UNCOMMITTED (0) nor KTA_READ_COMMITTED (1)", cfg->isolation_level);
    int ndev = 0;
    CU(cudaGetDeviceCount(&ndev));
    if (ndev < 1) return fail(KTA_ERR_CUDA, "no CUDA device (this library has no CPU fallback)");
    if (cfg->device >= 0) h->device = cfg->device;
    else CU(cudaGetDevice(&h->device));
    if (h->device >= ndev) return fail(KTA_ERR_INVALID, "device %d >= device count %d", h->device, ndev);
    CU(cudaSetDevice(h->device));
    cudaDeviceProp prop;
    CU(cudaGetDeviceProperties(&prop, h->device));
    if (prop.major != 9 || prop.minor != 0) return fail(KTA_ERR_CUDA, "device %s is sm_%d%d; this library is built for sm_90a only",
                                     prop.name, prop.major, prop.minor);
    h->sm_count = prop.multiProcessorCount;
    CU(cudaStreamCreateWithFlags(&h->stream, cudaStreamNonBlocking));
    h->need_hash = cfg->count_alive_keys == 1 || cfg->hll_precision != 0;
    h->pc.hash = keys_travel(h);   // kta_push reads it before its first (slow-path) call has bound the ring
    if (cfg->now_s == INT64_MIN) {
        const auto now = std::chrono::system_clock::now().time_since_epoch();
        const int64_t ns = std::chrono::duration_cast<std::chrono::nanoseconds>(now).count();
        h->cfg.now_s = ns / 1000000000ll;
        h->cfg.now_ns = (int32_t)(ns % 1000000000ll);
    }
    h->ring_records = cfg->ring_records > 0 ? cfg->ring_records : DEFAULT_RING_RECORDS;
    h->ring_records = (h->ring_records + TILE - 1) / TILE * TILE;
    h->ring_key_bytes = cfg->ring_key_bytes > 0 ? cfg->ring_key_bytes : h->ring_records * 24;

    const int P = cfg->num_partitions;
    h->nsums = sums_words(P);
    h->nhll = cfg->hll_precision ? ((size_t)1 << cfg->hll_precision) : 0;
    int rc;
    if ((rc = h->d_sums.alloc((int64_t)h->nsums)) || (rc = h->d_minmax.alloc(4)) || (rc = h->d_hll_floor.alloc(HLL_SLICES + 2)))
        return rc;
    if (h->nhll && (rc = h->d_hll.alloc((int64_t)h->nhll))) return rc;
    if (cfg->count_alive_keys == 1 && (rc = alive_create(h))) return rc;
    h->smem_optin = prop.sharedMemPerBlockOptin;
    if (cfg->shard_world > 1) {
        if (cfg->shard_rank < 0 || cfg->shard_rank >= cfg->shard_world || cfg->shard_world > P)
            return fail(KTA_ERR_INVALID, "shard_rank %d / shard_world %d invalid for %d partitions", cfg->shard_rank, cfg->shard_world, P);
        // the scan finds a partition's column p / G as mulhi(p, m), m = ceil(2^32 / G) (ScanParams::shard_magic).  With
        // e = m G - 2^32 that is exact whenever p e < 2^32, so the shape is taken only if the largest id, P - 1, meets it:
        // every P <= 65536 and every G <= 4096 does (e < G)
        const uint64_t G = (uint64_t)cfg->shard_world, e = (((uint64_t)1 << 32) + G - 1) / G * G - ((uint64_t)1 << 32);
        if ((uint64_t)(P - 1) * e >= (uint64_t)1 << 32)
            return fail(KTA_ERR_INVALID, "shard_world %d with %d partitions: the scan's partition division is exact only when "
                        "(P - 1) * (ceil(2^32 / G) * G - 2^32) < 2^32 (every P <= 65536 and every G <= 4096 qualify)",
                        cfg->shard_world, P);
        h->shard_world = cfg->shard_world;
        h->shard_rank = cfg->shard_rank;
    }
    h->columns = (P - h->shard_rank + h->shard_world - 1) / h->shard_world;   // partitions p < P with p % world == rank
    // counters in shared memory as long as at least 8 warps of 2 smallest key-only stages still fit beside them
    h->smem_counters = smem_counter_bytes(h->columns) + 8 * warp_smem_bytes(true, KEYBUF_MIN, 2, false) <= h->smem_optin;
    for (const auto &by_mode : SCAN_KERNELS[h->smem_counters])
        for (const auto &by_capture : by_mode)
            for (const ScanFn f : by_capture)
                if (f) CU(cudaFuncSetAttribute(f, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)h->smem_optin));
    if ((rc = log_scan_create(h->log, cfg->isolation_level == KTA_READ_COMMITTED, h->smem_optin))) return rc;
    if ((rc = state_reset_device(h))) return rc;
    CU(cudaStreamSynchronize(h->stream));
    return KTA_OK;
}

extern "C" int kta_create(const kta_config *cfg, kta_handle **out) {
    if (!cfg || !out) return fail(KTA_ERR_INVALID, "null argument");
    if (cfg->struct_size != (int32_t)sizeof(kta_config))
        return fail(KTA_ERR_INVALID, "kta_config.struct_size %d != %zu (ABI version %d)", cfg->struct_size, sizeof(kta_config), KTA_ABI_VERSION);
    kta_handle *h = new (std::nothrow) kta_handle();
    if (!h) return fail(KTA_ERR_NOMEM, "out of host memory");
    const int rc = create_impl(cfg, h);
    if (rc) {
        char keep[sizeof(g_err)];
        memcpy(keep, g_err, sizeof(keep));
        kta_destroy(h);
        memcpy(g_err, keep, sizeof(keep));
        *out = nullptr;
        return rc;
    }
    *out = h;
    return KTA_OK;
}

extern "C" void *kta_stream(kta_handle *h) { return h ? (void *)h->stream : nullptr; }

extern "C" int kta_set_stream(kta_handle *h, void *stream) {
    if (!h) return fail(KTA_ERR_INVALID, "null handle");
    int rc;
    if ((rc = set_device(h))) return rc;
    CU(cudaStreamSynchronize(h->stream));
    if (h->own_stream) CU(cudaStreamDestroy(h->stream));
    h->stream = (cudaStream_t)stream;
    h->own_stream = false;
    return KTA_OK;
}

// ------------------------------------------------------------------------------------------------
// scan launch
// ------------------------------------------------------------------------------------------------
// one launch of the fused scan; prm is complete apart from the state pointers filled in here
static int launch_scan_raw(kta_handle *h, ScanParams prm, int64_t key_readable, int64_t key_bytes) {
    const int P = h->cfg.num_partitions;
    const bool exact = h->cfg.count_alive_keys == 1;
    const bool capture = h->d_hash_out != nullptr && !prm.alive_only;
    // with -c the sketch is built from the resolved set at finalize, not in-stream.  A capture-only
    // handle (no -c, no HLL) runs the HLL-mode kernel against a null sketch of precision 0.
    const int mode = exact ? MODE_EXACT : (h->cfg.hll_precision || capture) ? MODE_HLL : MODE_COUNTERS;
    if (mode == MODE_HLL && !h->cfg.hll_precision)
        return fail(KTA_ERR_INVALID, "hash capture needs count_alive_keys or hll_precision");
    prm.shard_world = h->shard_world;
    prm.shard_rank = h->shard_rank;
    prm.Pc = h->columns;
    prm.shard_magic = h->shard_world > 1 ? (uint32_t)((((uint64_t)1 << 32) + (uint64_t)h->shard_world - 1) / (uint64_t)h->shard_world) : 0u;
    prm.ntiles = (prm.n + TILE - 1) / TILE;
    if (prm.ntiles >= (int64_t)1 << 30) return fail(KTA_ERR_INVALID, "batch of %lld records: split it (one scan takes < 2^37 records)", (long long)prm.n);
    prm.P = P;
    prm.hll_p = h->cfg.hll_precision;
    prm.sums = h->d_sums;
    prm.minmax = h->d_minmax;
    prm.hll = h->d_hll;
    prm.hll_floor = h->d_hll_floor;
    prm.hash_out = capture ? h->d_hash_out : nullptr;
    if (mode != MODE_COUNTERS) {
        if (!prm.key_tile_base) return fail(KTA_ERR_INVALID, "internal: key_tile_base missing");
        if (!prm.key_bytes && key_readable > 0) return fail(KTA_ERR_INVALID, "key_bytes is NULL but keys are required");
        prm.stage_limit = (((uintptr_t)prm.key_bytes & 15u) == 0) ? ((uint64_t)key_readable & ~15ull) : 0;
    }
    if (capture && h->shard_world > 1) return fail(KTA_ERR_INVALID, "hash capture is not available on a partition-sharded handle");
    int threads = 0, keybuf = 0, stages = 0;
    bool hdr = false;
    size_t sm = 0;
    const uintptr_t cols = (uintptr_t)prm.partition | (uintptr_t)prm.ts_ms | (uintptr_t)prm.key_len | (uintptr_t)prm.value_len;
    scan_shape(h, mode != MODE_COUNTERS, (cols & 15u) == 0, prm.n, key_bytes, threads, keybuf, stages, hdr, sm);
    prm.hdr_stage = hdr;
    if (sm > h->smem_optin) return fail(KTA_ERR_INVALID, "scan kernel does not fit: %zu B shared memory", sm);
    prm.keybuf = keybuf;
    prm.stages = stages;
    const int grid = (int)std::min<int64_t>((prm.ntiles + threads / 32 - 1) / (threads / 32), h->sm_count);
    if (prm.alive_cache) CU(cudaMemsetAsync(prm.alive_cache, 0, (size_t)4 << ALIVE_CACHE_SET_BITS, h->stream));
    cudaEvent_t e0 = nullptr, e1 = nullptr;
    if (h->timing) {
        if (h->ev_used == h->ev_pool.size()) {
            cudaEvent_t a, b;
            CU(cudaEventCreate(&a));
            CU(cudaEventCreate(&b));
            h->ev_pool.emplace_back(a, b);
        }
        e0 = h->ev_pool[h->ev_used].first;
        e1 = h->ev_pool[h->ev_used].second;
        h->ev_used++;
        CU(cudaEventRecord(e0, h->stream));
    }
    SCAN_KERNELS[h->smem_counters][h->shard_world > 1][mode][capture]<<<grid, threads, sm, h->stream>>>(prm);
    CU(cudaGetLastError());
    h->launches++;
    if (h->timing) CU(cudaEventRecord(e1, h->stream));
    return KTA_OK;
}

// Launch shape of the timeline pass over n records: one CTA of TL_THREADS per resident slot (at most one warp per tile),
// and enough CTAs that none takes more than TL_MAX_CTA_TILES tiles
static void timeline_shape(const kta_handle *h, int64_t n, int &grid, int &threads, size_t &smem) {
    const Timeline &t = h->tl;
    const int64_t ntiles = (n + TILE - 1) / TILE;
    threads = TL_THREADS;
    smem = t.smem ? (size_t)h->cfg.num_partitions * (size_t)(t.buckets + 2) * 16 : 0;
    const int64_t warps = TL_THREADS / 32;
    int64_t g = std::min<int64_t>((ntiles + warps - 1) / warps, (int64_t)h->sm_count * t.blocks_per_sm);
    g = std::max<int64_t>(g, (ntiles + TL_MAX_CTA_TILES - 1) / TL_MAX_CTA_TILES);
    grid = (int)std::max<int64_t>(g, 1);
}

// the timeline pass over the columns a counted scan has just read (same stream, so a ring chunk's free_ev, recorded
// after launch_scan, covers it)
static int launch_timeline(kta_handle *h, const ScanParams &prm) {
    const Timeline &t = h->tl;
    TimelineParams tp{};
    tp.n = prm.n;
    tp.ntiles = (prm.n + TILE - 1) / TILE;
    tp.partition = prm.partition;
    tp.ts_ms = prm.ts_ms;
    tp.key_len = prm.key_len;
    tp.value_len = prm.value_len;
    tp.P = h->cfg.num_partitions;
    tp.shard_world = h->shard_world;
    tp.shard_rank = h->shard_rank;
    tp.B = t.buckets;
    tp.origin = t.origin;
    tp.width = (uint64_t)t.width;
    tp.span = (uint64_t)t.buckets * (uint64_t)t.width;
    tp.inv_width = 1.0 / (double)t.width;
    tp.out = t.d_bins;
    int grid = 0, threads = 0;
    size_t smem = 0;
    timeline_shape(h, prm.n, grid, threads, smem);
    if (t.smem) timeline_kernel<true><<<grid, threads, smem, h->stream>>>(tp);
    else timeline_kernel<false><<<grid, threads, 0, h->stream>>>(tp);
    CU(cudaGetLastError());
    h->launches++;
    return KTA_OK;
}

// Launch shape of the partitioner pass over n records with key_bytes key bytes: PC_THREADS per CTA, a stage per warp
// sized from the mean key span of a tile (12.5 % headroom, as the scan sizes its key stage) within what the shared memory
// leaves beside the table and the counters, as many CTAs as are resident (at most one warp per tile), and enough that none
// takes more than PC_MAX_CTA_TILES tiles
// a warp's key stage for a pass over n records with key_bytes key bytes: the mean key span of a tile with 12.5 % headroom,
// within [PC_STAGE_MIN, PC_STAGE_MAX] and the `room` bytes a warp has
static int pass_stage_bytes(int64_t n, int64_t key_bytes, int64_t room) {
    const int64_t per_tile = n > 0 ? (std::max<int64_t>(key_bytes, 0) * TILE + n - 1) / n : 0;
    int64_t want = (per_tile + per_tile / 8 + 64 + 15) / 16 * 16;
    want = std::min<int64_t>(std::max<int64_t>(want, PC_STAGE_MIN), PC_STAGE_MAX);
    return (int)std::min<int64_t>(want, room / 16 * 16);
}

static int partitioner_shape(const kta_handle *h, int64_t n, int64_t key_bytes, int &grid, int &stage, size_t &smem) {
    const Partitioner &t = h->pt;
    const int64_t ntiles = (n + TILE - 1) / TILE;
    const size_t fixed = (size_t)PC_TABLE_WORDS * 4 + (t.smem ? ((size_t)(2 * t.ncounts + 1) * h->cfg.num_partitions + 3) / 4 * 16 : 0);
    const int64_t room = ((int64_t)h->smem_optin - (int64_t)fixed) / PC_WARPS - PC_STAGE_PAD;
    stage = pass_stage_bytes(n, key_bytes, room);
    smem = fixed + (size_t)PC_WARPS * (size_t)(stage + PC_STAGE_PAD);
    int per_sm = 0;
    if (t.smem) CU(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, partitioner_kernel<true>, PC_THREADS, smem));
    else CU(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, partitioner_kernel<false>, PC_THREADS, smem));
    if (per_sm < 1) return fail(KTA_ERR_CUDA, "partitioner kernel does not fit an SM (%zu B shared memory)", smem);
    int64_t g = std::min<int64_t>((ntiles + PC_WARPS - 1) / PC_WARPS, (int64_t)h->sm_count * per_sm);
    if (t.max_grid) g = std::min<int64_t>(g, t.max_grid);
    g = std::max<int64_t>(g, (ntiles + PC_MAX_CTA_TILES - 1) / PC_MAX_CTA_TILES);
    grid = (int)std::max<int64_t>(g, 1);
    return KTA_OK;
}

// the partitioner pass over the columns and key bytes a counted scan has just read (same stream, so a ring chunk's
// free_ev, recorded after launch_scan, covers it)
static int launch_partitioner(kta_handle *h, const ScanParams &prm, int64_t key_bytes) {
    const Partitioner &t = h->pt;
    PartitionerParams pp{};
    pp.n = prm.n;
    pp.ntiles = (prm.n + TILE - 1) / TILE;
    pp.partition = prm.partition;
    pp.key_len = prm.key_len;
    pp.key_bytes = prm.key_bytes;
    pp.key_tile_base = prm.key_tile_base;
    pp.P = h->cfg.num_partitions;
    pp.shard_world = h->shard_world;
    pp.shard_rank = h->shard_rank;
    pp.C = t.ncounts;
    for (int j = 0; j < t.ncounts; j++) {
        pp.count[j] = (uint32_t)t.counts[j];
        pp.recip[j] = ~0ull / (uint64_t)t.counts[j] + 1ull;   // ceil(2^64 / N) mod 2^64
    }
    pp.tables = h->d_crc32_tables;
    pp.out = t.d_counts;
    int grid = 0, rc;
    size_t smem = 0;
    if ((rc = partitioner_shape(h, prm.n, key_bytes, grid, pp.stage, smem))) return rc;
    if (t.smem) partitioner_kernel<true><<<grid, PC_THREADS, smem, h->stream>>>(pp);
    else partitioner_kernel<false><<<grid, PC_THREADS, smem, h->stream>>>(pp);
    CU(cudaGetLastError());
    h->launches++;
    return KTA_OK;
}

// ------------------------------------------------------------------------------------------------
// hot-key table: growth by rehash, the pass in slices that cannot overfill the table, export / import, finalize
// ------------------------------------------------------------------------------------------------
static constexpr uint64_t HK_DEFAULT_SLOTS = 1ull << 20, HK_MIN_SLOTS = 16, HK_MAX_SLOTS = 1ull << 31;

// the table cannot grow: it stops counting until kta_reset, and the entry point that scanned reports it (hk_reported)
static int hk_nomem(kta_handle *h, uint64_t want, const char *why) {
    HotKeys &k = h->hk;
    cudaGetLastError();   // a failed cudaMalloc must not be reported by the next launch check
    snprintf(k.nomem_msg, sizeof k.nomem_msg, "hot-key table: cannot grow from %llu to %llu slots (%s); it has stopped counting "
             "until kta_reset", (unsigned long long)k.slots, (unsigned long long)want, why);
    k.nomem = k.unreported = true;
    return fail(KTA_ERR_NOMEM, "%s", k.nomem_msg);
}

// KTA_ERR_NOMEM once for a table that ran out of memory during this call (every other metric has counted the batch)
static int hk_reported(kta_handle *h) {
    if (!h->hk.unreported) return KTA_OK;
    h->hk.unreported = false;
    return fail(KTA_ERR_NOMEM, "%s", h->hk.nomem_msg);
}

// the exact occupancy (one copy to the host and a stream synchronisation); a probe that found no slot is reported here
static int hk_occupancy(kta_handle *h, uint64_t &occ) {
    unsigned long long w[2] = {0, 0};
    CU(cudaMemcpyAsync(w, h->hk.d_word, 16, cudaMemcpyDeviceToHost, h->stream));
    CU(cudaStreamSynchronize(h->stream));
    if ((uint32_t)w[1]) return fail(KTA_ERR_INVALID, "internal: a hot-key probe ran over the whole table");
    occ = w[0];
    return KTA_OK;
}

static int hk_grid(const kta_handle *h, int64_t items) {
    return (int)std::max<int64_t>(std::min<int64_t>((items + 255) / 256, (int64_t)h->sm_count * 8), 1);
}

// doubles the table until it has at least `want` slots, by rehash; KTA_ERR_NOMEM (hk_nomem) when it cannot
static int hk_grow(kta_handle *h, uint64_t want) {
    HotKeys &k = h->hk;
    uint64_t slots = k.slots;
    while (slots < want) slots *= 2;
    if (slots > HK_MAX_SLOTS) return hk_nomem(h, slots, "more than 2^31 slots");
    if (k.max_slots && slots > k.max_slots) return hk_nomem(h, slots, "kta_hot_keys_limit_slots");
    DevBuf<HkSlot> nt;
    if (nt.alloc((int64_t)slots + 1)) return hk_nomem(h, slots, "cudaMalloc");
    cudaStream_t s = h->stream;
    CU(cudaMemsetAsync(nt, 0, (size_t)(slots + 1) * sizeof(HkSlot), s));
    // the rehash counts its claims again, in word [2]: the table's occupancy word is replaced only once it has run
    CU(cudaMemsetAsync(k.d_word + 2, 0, 8, s));
    const HkTable to{nt, slots, k.d_word + 2, reinterpret_cast<unsigned int *>(k.d_word.get() + 1)};
    hot_keys_rehash_kernel<<<hk_grid(h, (int64_t)k.slots + 1), 256, 0, s>>>(k.d_table, k.slots, to);
    h->launches++;
    CU(cudaGetLastError());
    CU(cudaMemcpyAsync(k.d_word, k.d_word + 2, 8, cudaMemcpyDeviceToDevice, s));
    CU(cudaStreamSynchronize(s));
    k.d_table = std::move(nt);   // nt frees the old table
    k.slots = slots;
    k.grows++;
    return KTA_OK;
}

// the hot-key pass over tiles [t0, t1) of a counted scan's columns
static int launch_hot_keys_tiles(kta_handle *h, const ScanParams &prm, int64_t key_bytes, int64_t t0, int64_t t1) {
    HotKeysParams hp{};
    hp.n = prm.n;
    hp.tile_lo = t0;
    hp.tile_hi = t1;
    hp.partition = prm.partition;
    hp.key_len = prm.key_len;
    hp.value_len = prm.value_len;
    hp.ts_ms = prm.ts_ms;
    hp.key_bytes = prm.key_bytes;
    hp.key_tile_base = prm.key_tile_base;
    hp.P = h->cfg.num_partitions;
    hp.shard_world = h->shard_world;
    hp.shard_rank = h->shard_rank;
    hp.tables = h->d_crc32_tables;
    hp.table = h->hk.table();
    const int64_t room = ((int64_t)h->smem_optin - (int64_t)PC_TABLE_WORDS * 4) / HK_WARPS - PC_STAGE_PAD;
    hp.stage = pass_stage_bytes(prm.n, key_bytes, room);
    const size_t smem = (size_t)PC_TABLE_WORDS * 4 + (size_t)HK_WARPS * (size_t)(hp.stage + PC_STAGE_PAD);
    int per_sm = 0;
    CU(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, hot_keys_kernel, HK_THREADS, smem));
    if (per_sm < 1) return fail(KTA_ERR_CUDA, "hot-key kernel does not fit an SM (%zu B shared memory)", smem);
    const int grid = (int)std::max<int64_t>(std::min<int64_t>((t1 - t0 + HK_WARPS - 1) / HK_WARPS, (int64_t)h->sm_count * per_sm), 1);
    hot_keys_kernel<<<grid, HK_THREADS, smem, h->stream>>>(hp);
    CU(cudaGetLastError());
    h->launches++;
    return KTA_OK;
}

// The hot-key pass over a counted scan's columns (same stream, so a ring chunk's free_ev, recorded after launch_scan, covers
// it).  Counting is not idempotent, so no insert may fail: the table is kept at most half full.  U (bound) is an upper bound
// on the occupancy, raised by every launch's records; a launch goes ahead without a read-back while U + n <= slots / 2.
// Otherwise the exact occupancy is read back, the table grows while it is more than a quarter full or has less than a tile
// of room, and the batch is cut into tile-aligned slices of at most slots / 2 - U records, reading back between slices.
// A table that cannot grow stops counting (hk_nomem): the scan goes on, so every other metric counts the batch.
static int launch_hot_keys(kta_handle *h, const ScanParams &prm, int64_t key_bytes) {
    HotKeys &k = h->hk;
    if (k.nomem) return KTA_OK;
    const int64_t ntiles = (prm.n + TILE - 1) / TILE;
    int rc;
    for (int64_t t = 0; t < ntiles;) {
        int64_t t1 = ntiles;
        if (k.bound + (uint64_t)(prm.n - t * TILE) > k.slots / 2) {
            uint64_t occ = 0;
            if ((rc = hk_occupancy(h, occ))) return rc;
            k.bound = occ;
            while (k.bound * 4 > k.slots || k.slots / 2 - k.bound < (uint64_t)TILE)
                if ((rc = hk_grow(h, k.slots * 2))) return k.nomem ? KTA_OK : rc;   // (hk_nomem has recorded an out-of-memory)
            t1 = std::min<int64_t>(ntiles, t + (int64_t)((k.slots / 2 - k.bound) / TILE));
        }
        if (t1 - t < ntiles) k.slices++;
        if ((rc = launch_hot_keys_tiles(h, prm, key_bytes, t, t1))) return rc;
        k.bound += (uint64_t)(std::min<int64_t>(prm.n, t1 * TILE) - t * TILE);
        t = t1;
    }
    return KTA_OK;
}

// one scan of a batch whose columns lie in ring chunk `chunk` (-1: elsewhere); `seq_ends`: see alive_prepare
static int launch_scan(kta_handle *h, ScanParams prm, int64_t key_readable, int64_t key_bytes, int chunk = -1,
                       const uint64_t *seq_ends = nullptr) {
    if (prm.n <= 0) return KTA_OK;
    const bool exact = h->alive.d_table != nullptr;
    int rc;
    if (h->pt.ncounts) {   // (checked before anything is launched: a refused batch leaves the handle as it was)
        if (!prm.key_tile_base) return fail(KTA_ERR_INVALID, "internal: key_tile_base missing");
        if (!prm.key_bytes && key_readable > 0) return fail(KTA_ERR_INVALID, "key_bytes is NULL but the partitioner check needs the keys");
    }
    if (h->hk.top_k) {
        if (!prm.key_tile_base) return fail(KTA_ERR_INVALID, "internal: key_tile_base missing");
        if (!prm.key_bytes && key_readable > 0) return fail(KTA_ERR_INVALID, "key_bytes is NULL but the hot-key table needs the keys");
    }
    if (exact && (rc = alive_prepare(h, prm, seq_ends))) return rc;
    if ((rc = launch_scan_raw(h, prm, key_readable, key_bytes))) return rc;
    if (h->tl.buckets && (rc = launch_timeline(h, prm))) return rc;
    if (h->pt.ncounts && (rc = launch_partitioner(h, prm, key_bytes))) return rc;
    if (h->hk.top_k && (rc = launch_hot_keys(h, prm, key_bytes))) return rc;
    if (exact && (rc = alive_scanned(h, prm, key_readable, key_bytes, chunk))) return rc;
    h->records += (uint64_t)prm.n;
    h->finalized = false;
    return KTA_OK;
}

static int collect_timing(kta_handle *h) {
    for (size_t i = 0; i < h->ev_used; i++) {
        float ms = 0;
        CU(cudaEventElapsedTime(&ms, h->ev_pool[i].first, h->ev_pool[i].second));
        h->scan_ms += ms;
        h->scan_launches_timed++;
    }
    h->ev_used = 0;
    return KTA_OK;
}

// what the log path's steps (kta_logscan.cuh) need of the handle
static LogEnv log_env(kta_handle *h) {
    return LogEnv{h->stream, h->sm_count, h->smem_optin, h->cfg.num_partitions, h->d_tb_scratch, h->launches};
}

// the key_tile_base column of n records' key lengths, into h->d_tb_scratch ([ntiles] = the key bytes in all)
static int derive_tile_base(kta_handle *h, const int32_t *d_klen, int64_t n) { return log_tile_base(log_env(h), d_klen, n); }

// a scan's params over the columns of n records from seq_base on (ScanParams' leading fields, in their order; the rest zero)
static ScanParams scan_params(int64_t n, uint64_t seq_base, const int32_t *partition, const int64_t *ts_ms, const int32_t *key_len,
                              const int32_t *value_len, const uint8_t *key_bytes, const uint64_t *key_tile_base, const uint64_t *seq) {
    return ScanParams{n, seq_base, partition, ts_ms, key_len, value_len, key_bytes, key_tile_base, seq};
}

// the checks a batch passes at both batch entry points (an empty batch passes: there is nothing to scan)
static int check_batch(const kta_handle *h, const kta_batch *b) {
    if (!h || !b) return fail(KTA_ERR_INVALID, "null argument");
    if (b->n < 0) return fail(KTA_ERR_INVALID, "negative n");
    if (b->n > 0 && (!b->partition || !b->ts_ms || !b->key_len || !b->value_len))
        return fail(KTA_ERR_INVALID, "partition/ts_ms/key_len/value_len columns are required");
    return KTA_OK;
}

// seq of a batch's record 0.  KTA_SEQ_AUTO continues the handle's running count (what kta_push and the log-segment
// entry points do).  With -c and no explicit seq column, last-writer-wins is decided by seq_base + i alone, so a batch
// that re-uses sequence numbers the handle has already handed out would silently let OLDER records win: refused.
static int resolve_seq_base(kta_handle *h, const kta_batch *b, uint64_t *out) {
    if (b->seq_base == KTA_SEQ_AUTO) {
        *out = h->next_seq;
        return KTA_OK;
    }
    if (h->cfg.count_alive_keys == 1 && !b->seq && b->seq_base < h->next_seq)
        return fail(KTA_ERR_INVALID, "seq_base %llu < %llu, the next sequence number of this handle: batches without a seq "
                    "column must be pushed in stream order (use KTA_SEQ_AUTO to continue the running count)",
                    (unsigned long long)b->seq_base, (unsigned long long)h->next_seq);
    *out = b->seq_base;
    return KTA_OK;
}

// scans a checked, non-empty batch of device columns behind the records the handle has already scanned
static int scan_device_batch(kta_handle *h, const kta_batch *b) {
    uint64_t seq_base = 0;
    int rc;
    if ((rc = resolve_seq_base(h, b, &seq_base))) return rc;
    ScanParams prm = scan_params(b->n, seq_base, b->partition, b->ts_ms, b->key_len, b->value_len, b->key_bytes, b->key_tile_base, b->seq);
    if (keys_travel(h) && !prm.key_tile_base) {
        if ((rc = derive_tile_base(h, b->key_len, b->n))) return rc;
        prm.key_tile_base = h->d_tb_scratch;
    }
    if ((h->pt.ncounts || h->hk.top_k) && !b->key_bytes) {
        // The partitioner check and the hot-key table hash every key: without key bytes the batch may only have null and empty keys.  A
        // declared byte count is refused at once; otherwise the tile base's total is read back, one host round trip.  Only a
        // caller's batch without key bytes pays it: the log path hands over its gather buffer, which is never NULL.
        if (b->key_bytes_len > 0) return fail(KTA_ERR_INVALID, "key_bytes is NULL but key_bytes_len is %lld", (long long)b->key_bytes_len);
        uint64_t total = 0;
        CU(cudaMemcpyAsync(&total, prm.key_tile_base + (b->n + TILE - 1) / TILE, 8, cudaMemcpyDeviceToHost, h->stream));
        CU(cudaStreamSynchronize(h->stream));
        if (total) return fail(KTA_ERR_INVALID, "key_bytes is NULL but the batch has %llu key bytes (the partitioner check or the "
                               "hot-key table hashes them)", (unsigned long long)total);
    }
    if ((rc = launch_scan(h, prm, b->key_bytes_len, b->key_bytes_len))) return rc;
    h->next_seq = std::max<uint64_t>(h->next_seq, seq_base + (uint64_t)b->n);
    return KTA_OK;
}

extern "C" int kta_scan_batch_device(kta_handle *h, const kta_batch *b) {
    int rc;
    if ((rc = check_batch(h, b)) || b->n == 0) return rc;
    if ((rc = set_device(h))) return rc;
    if ((rc = ring_flush(h)) || (rc = scan_device_batch(h, b))) return rc;   // records pushed earlier come first in seq order
    return hk_reported(h);
}

// ------------------------------------------------------------------------------------------------
// Kafka RecordBatch v2 segments → SoA → scan (SURVEY.md §8 f2; kernels in kta_logdecode.cuh)
// ------------------------------------------------------------------------------------------------

static int scan_log_batches(kta_handle *h, int32_t partition, const int32_t *dev_batch_partition, const uint8_t *dev_bytes,
                            int64_t len, int64_t readable /* bytes of dev_bytes that may be READ (>= len when the buffer has slack) */,
                            const uint64_t *dev_batch_off, int64_t nbatches, int64_t *records_out) {
    if (!h || len < 0 || nbatches < 0 || (nbatches && (!dev_bytes || !dev_batch_off))) return fail(KTA_ERR_INVALID, "bad argument");
    if (records_out) *records_out = 0;
    if (nbatches == 0) return KTA_OK;
    int rc;
    if ((rc = set_device(h))) return rc;
    if ((rc = ring_flush(h))) return rc;   // keep seq order with records pushed earlier
    if ((rc = alive_settle_if_any(h))) return rc;   // the decode scratch of an earlier call is about to be reused
    LogScan &L = h->log;
    const LogEnv e = log_env(h);
    LogHeaders hd;
    if ((rc = log_headers(L, e, partition, dev_batch_partition, dev_bytes, len, dev_batch_off, nbatches, hd))) return rc;
    const int64_t ncut = hd.word.cut;
    uint64_t nrec = hd.nrec, dropped = 0;
    if (hd.nrec > 0) {
        const uint32_t codecs = hd.word.flags & LOGB_CODECS;
        if (codecs) {
            uint64_t unc_total = 0;
            uint32_t bad = 0;
            if ((rc = log_unc_size(L, e, dev_bytes, nbatches, codecs, &unc_total, &bad))) return rc;
            if (bad) return fail(KTA_ERR_INVALID, "malformed compressed record batch in partition %d", partition);
            if ((rc = log_unc_copy(L, e, dev_bytes, nbatches, codecs, unc_total))) return rc;
        }
        if (ncut && (rc = log_cut_count(L, e, dev_bytes, nbatches, ncut, &nrec, &dropped))) return rc;
        // (cut batches that keep no record are still decoded, so damage in them refuses the call as elsewhere)
        const bool keys = nrec > 0 && keys_travel(h);
        kta_batch b;
        if ((rc = log_decode(L, e, dev_bytes, readable, nbatches, nrec, hd.word.longest, keys, ncut, b))) return rc;
        if ((rc = log_gather_keys(L, e, partition, dev_bytes, keys, b))) return rc;
        if (nrec > 0 && (rc = scan_device_batch(h, &b))) return rc;
    }
    // the call succeeded: its transaction counters, CRC results and what its windows left out join the handle's totals
    for (int i = 0; i < 3; i++) L.txn.totals[i] += hd.txn_stats[i];
    const uint32_t not_served = hd.word.not_served;
    OffsetState &o = L.offsets;
    o.totals[0] += not_served;
    o.totals[1] += hd.word.not_served_records + dropped;
    CrcState &c = L.crc;
    if (c.on) {
        c.totals[0] += (uint64_t)nbatches - not_served;
        c.totals[1] += hd.word.crc_failed;
        c.totals[2] += hd.word.crc_failed_bytes;
        c.kept.insert(c.kept.end(), hd.crc_fails.begin(), hd.crc_fails.end());
    }
    if (records_out) *records_out = (int64_t)nrec;
    return KTA_OK;
}

extern "C" int kta_scan_log_segment_device(kta_handle *h, int32_t partition, const uint8_t *dev_bytes, int64_t len,
                                           const uint64_t *dev_batch_off, int64_t nbatches, int64_t *records_out) {
    const int rc = scan_log_batches(h, partition, nullptr, dev_bytes, len, len, dev_batch_off, nbatches, records_out);
    return rc ? rc : hk_reported(h);
}

extern "C" int kta_scan_log_batches_device(kta_handle *h, const uint8_t *dev_bytes, int64_t len, const uint64_t *dev_batch_off,
                                           const int32_t *dev_batch_partition, int64_t nbatches, int64_t *records_out) {
    if (nbatches && !dev_batch_partition) return fail(KTA_ERR_INVALID, "dev_batch_partition is NULL");
    const int rc = scan_log_batches(h, 0, dev_batch_partition, dev_bytes, len, len, dev_batch_off, nbatches, records_out);
    return rc ? rc : hk_reported(h);
}

extern "C" int kta_push_log_segments_host(kta_handle *h, int32_t nsegs, const int32_t *partitions, const uint8_t *const *bytes,
                                          const int64_t *lens, int64_t *records_out) {
    if (!h || nsegs < 0 || (nsegs && (!partitions || !bytes || !lens))) return fail(KTA_ERR_INVALID, "bad argument");
    if (records_out) *records_out = 0;
    // the batches of each segment, found on the host (log_walk_batches: a truncated tail is ignored).  All segments go to
    // ONE staging buffer and are decoded and scanned together (one decode, one scan, two host round trips in total).
    std::vector<uint64_t> offs;
    std::vector<int32_t> parts;
    std::vector<int64_t> used((size_t)nsegs, 0), base((size_t)nsegs, 0);
    int64_t total = 0;
    for (int32_t sgi = 0; sgi < nsegs; sgi++) {
        if (lens[sgi] < 0 || (lens[sgi] && !bytes[sgi])) return fail(KTA_ERR_INVALID, "bad segment %d", sgi);
        base[(size_t)sgi] = total;
        const int64_t pos = log_walk_batches(bytes[sgi], lens[sgi], total, offs);
        parts.resize(offs.size(), partitions[sgi]);
        used[(size_t)sgi] = pos;
        total += (pos + 15) & ~(int64_t)15;
    }
    if (offs.empty()) return KTA_OK;
    int rc;
    if ((rc = set_device(h))) return rc;
    cudaStream_t s = h->stream;
    LogScan &L = h->log;
    const int64_t nb = (int64_t)offs.size();
    if ((rc = L.bytes.grow(s, total + 64)) || (rc = L.off.grow(s, nb)) || (rc = L.part.grow(s, nb))) return rc;
    for (int32_t sgi = 0; sgi < nsegs; sgi++)
        if (used[(size_t)sgi])
            CU(cudaMemcpyAsync(L.bytes + base[(size_t)sgi], bytes[sgi], (size_t)used[(size_t)sgi], cudaMemcpyHostToDevice, s));
    CU(cudaMemcpyAsync(L.off, offs.data(), offs.size() * 8, cudaMemcpyHostToDevice, s));
    CU(cudaMemcpyAsync(L.part, parts.data(), parts.size() * 4, cudaMemcpyHostToDevice, s));
    // the staging buffer has 64 bytes of slack behind `total`: 16-byte-granular bulk copies may run into it
    if ((rc = scan_log_batches(h, 0, L.part, L.bytes, total, total + 48, L.off, nb, records_out))) return rc;
    CU(cudaStreamSynchronize(s));   // the caller may reuse its buffers, and the scratch may be reused by the next call
    if ((rc = collect_timing(h))) return rc;
    return hk_reported(h);
}

extern "C" int kta_push_log_segment_host(kta_handle *h, int32_t partition, const uint8_t *bytes, int64_t len,
                                         int64_t *records_out) {
    return kta_push_log_segments_host(h, 1, &partition, &bytes, &len, records_out);
}

// A .txnindex image: 34-byte big-endian entries version i16 (= 0) | producerId i64 | firstOffset i64 | lastOffset i64 |
// lastStableOffset i64.  All of it is checked before any range is added.
extern "C" int kta_log_add_txn_index_host(kta_handle *h, int32_t partition, const uint8_t *bytes, int64_t len) {
    if (!h || len < 0 || (len && !bytes)) return fail(KTA_ERR_INVALID, "bad argument");
    if (!h->log.read_committed) return fail(KTA_ERR_INVALID, "transaction index on a read_uncommitted handle");
    if (partition < 0 || partition >= h->cfg.num_partitions)
        return fail(KTA_ERR_INVALID, "partition %d outside [0, %d)", partition, h->cfg.num_partitions);
    constexpr int64_t ENTRY = 34;
    if (len % ENTRY) return fail(KTA_ERR_INVALID, "transaction index of %lld bytes: not a multiple of %lld", (long long)len, (long long)ENTRY);
    auto be = [](const uint8_t *p, int n) { uint64_t v = 0; for (int i = 0; i < n; i++) v = (v << 8) | p[i]; return v; };
    std::vector<TxnRange> add;
    for (int64_t at = 0; at < len; at += ENTRY) {
        const uint8_t *e = bytes + at;
        const TxnRange r{partition, 0u, be(e + 2, 8), (int64_t)be(e + 10, 8), (int64_t)be(e + 18, 8)};
        if (be(e, 2) != 0) return fail(KTA_ERR_INVALID, "transaction index entry %lld: version %d", (long long)(at / ENTRY), (int)be(e, 2));
        if (r.first > r.last)
            return fail(KTA_ERR_INVALID, "transaction index entry %lld: firstOffset %lld > lastOffset %lld", (long long)(at / ENTRY),
                        (long long)r.first, (long long)r.last);
        add.push_back(r);
    }
    if (add.empty()) return KTA_OK;
    int rc;
    if ((rc = set_device(h))) return rc;
    return log_add_txn_ranges(h->log, log_env(h), add);
}

extern "C" int kta_log_txn_stats(kta_handle *h, uint64_t *aborted_batches, uint64_t *aborted_records, uint64_t *undecided_records) {
    if (!h) return fail(KTA_ERR_INVALID, "null handle");
    if (!h->log.read_committed) return fail(KTA_ERR_NOT_ENABLED, "the handle is read_uncommitted");
    if (aborted_batches) *aborted_batches = h->log.txn.totals[0];
    if (aborted_records) *aborted_records = h->log.txn.totals[1];
    if (undecided_records) *undecided_records = h->log.txn.totals[2];
    return KTA_OK;
}

extern "C" int kta_log_set_check_crcs(kta_handle *h, int enabled) {
    if (!h) return fail(KTA_ERR_INVALID, "null handle");
    if (enabled != 0 && enabled != 1) return fail(KTA_ERR_INVALID, "check_crcs %d is neither 0 nor 1", enabled);
    h->log.crc.on = enabled == 1;
    return KTA_OK;
}

extern "C" int kta_log_crc_stats(kta_handle *h, uint64_t *checked_batches, uint64_t *failed_batches, uint64_t *failed_bytes) {
    if (!h) return fail(KTA_ERR_INVALID, "null handle");
    if (checked_batches) *checked_batches = h->log.crc.totals[0];
    if (failed_batches) *failed_batches = h->log.crc.totals[1];
    if (failed_bytes) *failed_bytes = h->log.crc.totals[2];
    return KTA_OK;
}

extern "C" int kta_log_set_offsets(kta_handle *h, int32_t partition, int64_t log_start_offset, int64_t high_watermark) {
    if (!h) return fail(KTA_ERR_INVALID, "null handle");
    if (partition < 0 || partition >= h->cfg.num_partitions)
        return fail(KTA_ERR_INVALID, "partition %d outside [0, %d)", partition, h->cfg.num_partitions);
    if (log_start_offset < -1 || high_watermark < -1)
        return fail(KTA_ERR_INVALID, "log start offset %lld / high watermark %lld below -1", (long long)log_start_offset,
                    (long long)high_watermark);
    if (log_start_offset >= 0 && high_watermark >= 0 && log_start_offset > high_watermark)
        return fail(KTA_ERR_INVALID, "log start offset %lld above the high watermark %lld", (long long)log_start_offset,
                    (long long)high_watermark);
    log_set_window(h->log, h->cfg.num_partitions, partition, log_start_offset, high_watermark);
    return KTA_OK;
}

extern "C" int kta_log_offset_stats(kta_handle *h, uint64_t *batches_not_served, uint64_t *records_left_out) {
    if (!h) return fail(KTA_ERR_INVALID, "null handle");
    if (batches_not_served) *batches_not_served = h->log.offsets.totals[0];
    if (records_left_out) *records_left_out = h->log.offsets.totals[1];
    return KTA_OK;
}

extern "C" int kta_log_crc_failures(kta_handle *h, kta_log_crc_failure *out, int64_t cap, int64_t *count) {
    if (!h || cap < 0 || (cap && !out)) return fail(KTA_ERR_INVALID, "bad argument");
    const std::vector<kta_log_crc_failure> &kept = h->log.crc.kept;
    const size_t n = std::min<size_t>((size_t)cap, kept.size());
    if (n) memcpy(out, kept.data(), n * sizeof(kta_log_crc_failure));
    if (count) *count = (int64_t)kept.size();
    return KTA_OK;
}

// ------------------------------------------------------------------------------------------------
// landing ring: host records → pinned chunk → cudaMemcpyAsync → HBM chunk → scan
// ------------------------------------------------------------------------------------------------
static int ring_dev_init(kta_handle *h) {
    if (h->ring_dev_ready) return KTA_OK;
    const int64_t R = h->ring_records, KB = h->ring_key_bytes;
    int rc;
    for (auto &c : h->chunks) {
        if ((rc = c.d_partition.alloc(R)) || (rc = c.d_klen.alloc(R)) || (rc = c.d_vlen.alloc(R)) || (rc = c.d_ts.alloc(R)) ||
            (rc = c.d_seq.alloc(R)) || (rc = c.d_keys.alloc(KB + 64)) || (rc = c.d_tile_base.alloc(R / TILE + 2)))
            return rc;
        if (!c.free_ev) CU(cudaEventCreateWithFlags(&c.free_ev, cudaEventDisableTiming));
    }
    h->ring_dev_ready = true;
    return KTA_OK;
}

static int ring_host_init(kta_handle *h) {
    if (h->ring_host_ready) return KTA_OK;
    int rc;
    if ((rc = ring_dev_init(h))) return rc;
    const int64_t R = h->ring_records, KB = h->ring_key_bytes;
    for (auto &c : h->chunks)
        if ((rc = c.h_partition.alloc(R)) || (rc = c.h_klen.alloc(R)) || (rc = c.h_vlen.alloc(R)) || (rc = c.h_ts.alloc(R)) ||
            (rc = c.h_keys.alloc(KB + 64)) || (rc = c.h_tile_base.alloc(R / TILE + 2)))
            return rc;
    h->ring_host_ready = true;
    return KTA_OK;
}

static void push_cursor_bind(kta_handle *h) {
    Chunk &c = h->chunks[h->cur];
    auto &pc = h->pc;
    pc.part = c.h_partition; pc.klen = c.h_klen; pc.vlen = c.h_vlen; pc.ts = c.h_ts; pc.keys = c.h_keys; pc.tile_base = c.h_tile_base;
    pc.n = 0; pc.kb = 0;
    pc.cap = h->ring_host_ready ? h->ring_records : 0;
    pc.kcap = h->ring_key_bytes;
    pc.hash = keys_travel(h);
}

// scan the columns staged in ring chunk `cur` and move on to the next chunk
static int ring_scan_chunk(kta_handle *h, const ScanParams &prm, int64_t key_readable, int64_t key_bytes,
                           const uint64_t *seq_ends = nullptr) {
    int rc;
    if ((rc = launch_scan(h, prm, key_readable, key_bytes, h->cur, seq_ends))) return rc;
    CU(cudaEventRecord(h->chunks[h->cur].free_ev, h->stream));
    h->cur = (h->cur + 1) % NCHUNK;
    return KTA_OK;
}

// ring chunk ci is about to be overwritten: wait for the scan that read it and confirm that scan's stamps
static int ring_reuse_chunk(kta_handle *h, int ci) {
    CU(cudaEventSynchronize(h->chunks[ci].free_ev));
    return alive_release_chunk(h, ci);
}

// stage one pinned chunk and scan it
static int ring_flush(kta_handle *h) {
    if (h->pc.n == 0) return KTA_OK;
    Chunk &c = h->chunks[h->cur];
    const int64_t n = h->pc.n, kb = h->pc.kb;
    const int64_t ntiles = (n + TILE - 1) / TILE;
    c.h_tile_base[ntiles] = (uint64_t)kb;
    cudaStream_t s = h->stream;
    CU(cudaMemcpyAsync(c.d_partition, c.h_partition, n * 4, cudaMemcpyHostToDevice, s));
    CU(cudaMemcpyAsync(c.d_ts, c.h_ts, n * 8, cudaMemcpyHostToDevice, s));
    CU(cudaMemcpyAsync(c.d_klen, c.h_klen, n * 4, cudaMemcpyHostToDevice, s));
    CU(cudaMemcpyAsync(c.d_vlen, c.h_vlen, n * 4, cudaMemcpyHostToDevice, s));
    if (keys_travel(h)) {
        if (kb) CU(cudaMemcpyAsync(c.d_keys, c.h_keys, kb, cudaMemcpyHostToDevice, s));
        CU(cudaMemcpyAsync(c.d_tile_base, c.h_tile_base, (ntiles + 1) * 8, cudaMemcpyHostToDevice, s));
    }
    const ScanParams prm = scan_params(n, h->next_seq, c.d_partition, c.d_ts, c.d_klen, c.d_vlen, c.d_keys, c.d_tile_base, nullptr);
    int rc;
    if ((rc = ring_scan_chunk(h, prm, (kb + 15) & ~(int64_t)15, kb))) return rc;
    h->next_seq += (uint64_t)n;
    push_cursor_bind(h);
    // the next chunk may still be in flight from NCHUNK flushes ago
    return ring_reuse_chunk(h, h->cur);
}

// kta_push off the fast path: first call (ring not yet allocated), chunk full, or an oversized key
static int __attribute__((noinline)) push_slow(kta_handle *h, int64_t kl) {
    int rc;
    if ((rc = set_device(h))) return rc;
    if (!h->ring_host_ready) {
        if ((rc = ring_host_init(h))) return rc;
        push_cursor_bind(h);
    }
    if (kl > h->ring_key_bytes) return fail(KTA_ERR_INVALID, "key of %lld bytes exceeds ring_key_bytes", (long long)kl);
    if (h->pc.n == h->pc.cap || h->pc.kb + kl > h->pc.kcap) return ring_flush(h);
    return KTA_OK;
}

extern "C" int kta_push(kta_handle *h, int32_t partition, int64_t offset, int64_t ts_ms, const uint8_t *key,
                        int32_t key_len, int32_t value_len) {
    (void)offset;  // never read by a metric (SURVEY.md D7); termination logic stays with the caller
    if (__builtin_expect(!h, 0)) return fail(KTA_ERR_INVALID, "null handle");
    auto &pc = h->pc;
    const int64_t kl = (pc.hash && key_len > 0) ? key_len : 0;  // key bytes only travel when they are hashed
    int late = KTA_OK;   // a hot-key table that ran out of memory in the flush (the record still lands)
    if (__builtin_expect(pc.n == pc.cap || pc.kb + kl > pc.kcap, 0)) {
        const int rc = push_slow(h, kl);
        if (rc) return rc;
        late = hk_reported(h);
    }
    const int64_t i = pc.n;
    if ((i & (TILE - 1)) == 0) pc.tile_base[i / TILE] = (uint64_t)pc.kb;
    pc.part[i] = partition;
    pc.ts[i] = ts_ms;
    pc.klen[i] = key_len < 0 ? -1 : key_len;
    pc.vlen[i] = value_len < 0 ? -1 : value_len;
    if (kl) {
        if (__builtin_expect(!key, 0)) return fail(KTA_ERR_INVALID, "key is NULL with key_len %d", key_len);
        uint8_t *dst = pc.keys + pc.kb;
        if (kl == 16) {            // ids, hashes, UUIDs: two register moves instead of a call
            uint64_t a, b;
            memcpy(&a, key, 8); memcpy(&b, key + 8, 8);
            memcpy(dst, &a, 8); memcpy(dst + 8, &b, 8);
        } else if (kl <= 8) {      // short keys: byte-exact, no call (the landing area has slack only at its end)
            for (int64_t j = 0; j < kl; j++) dst[j] = key[j];
        } else {
            memcpy(dst, key, (size_t)kl);
        }
        pc.kb += kl;
    }
    pc.n = i + 1;
    h->finalized = false;
    return late;
}

extern "C" int kta_push_batch_host(kta_handle *h, const kta_batch *b) {
    int rc;
    if ((rc = check_batch(h, b)) || b->n == 0) return rc;
    const bool hash = keys_travel(h);
    if (hash && !b->key_bytes && b->key_bytes_len > 0) return fail(KTA_ERR_INVALID, "key_bytes is NULL");
    if ((h->pt.ncounts || h->hk.top_k) && !b->key_bytes)
        for (int64_t i = 0; i < b->n; i++)
            if (b->key_len[i] > 0) return fail(KTA_ERR_INVALID, "key_bytes is NULL but record %lld has a %d-byte key (the partitioner "
                                               "check or the hot-key table hashes it)", (long long)i, b->key_len[i]);
    if ((rc = set_device(h))) return rc;
    if ((rc = ring_flush(h))) return rc;  // keep seq order with earlier kta_push records
    if ((rc = ring_dev_init(h))) return rc;
    uint64_t seq_base = 0;
    if ((rc = resolve_seq_base(h, b, &seq_base))) return rc;
    cudaStream_t s = h->stream;
    const bool use_seq = b->seq && h->cfg.count_alive_keys == 1;
    std::vector<uint64_t> tb_host;  // only when the caller gave no tile bases
    uint64_t koff = 0;              // absolute key byte offset of the next chunk's first key
    int64_t r0 = 0;
    while (r0 < b->n) {
        int64_t cn = std::min<int64_t>(h->ring_records, b->n - r0);
        const int ci = h->cur;
        Chunk &c = h->chunks[ci];
        uint64_t k0 = 0, k1 = 0;
        const uint64_t *tb_src = nullptr;
        if (hash) {
            // the chunk ends at a tile boundary chosen so that its keys fit the staging buffer; only a SINGLE tile
            // whose keys exceed ring_key_bytes cannot be staged
            const int64_t tiles_max = (cn + TILE - 1) / TILE;
            int64_t tiles = 0;
            if (b->key_tile_base) {
                const uint64_t *tb = b->key_tile_base + r0 / TILE;
                k0 = tb[0];
                // largest t with tb[t] - k0 <= ring_key_bytes (tile bases are non-decreasing)
                tiles = std::upper_bound(tb, tb + tiles_max + 1, k0 + (uint64_t)h->ring_key_bytes) - tb - 1;
                tiles = std::min<int64_t>(tiles, tiles_max);
                if (tiles >= 1) k1 = tb[tiles];
                tb_src = tb;
            } else {
                tb_host.resize((size_t)tiles_max + 1);
                uint64_t acc = koff;
                tb_host[0] = acc;
                for (; tiles < tiles_max; tiles++) {
                    const int64_t lo = r0 + tiles * TILE, hi = std::min<int64_t>(lo + TILE, r0 + cn);
                    uint64_t tile_bytes = 0;
                    for (int64_t i = lo; i < hi; i++) tile_bytes += b->key_len[i] > 0 ? (uint64_t)b->key_len[i] : 0;
                    if (acc + tile_bytes - koff > (uint64_t)h->ring_key_bytes) break;
                    acc += tile_bytes;
                    tb_host[(size_t)tiles + 1] = acc;
                }
                k0 = koff;
                k1 = acc;
                tb_src = tb_host.data();
            }
            if (tiles < 1)
                return fail(KTA_ERR_INVALID, "the keys of one %d-record tile (records %lld..) exceed ring_key_bytes %lld; "
                            "%lld earlier record(s) of this batch were scanned", TILE, (long long)r0, (long long)h->ring_key_bytes,
                            (long long)r0);
            cn = std::min<int64_t>(cn, tiles * TILE);
        }
        if ((rc = ring_reuse_chunk(h, ci))) return rc;
        const int64_t ntiles = (cn + TILE - 1) / TILE;
        CU(cudaMemcpyAsync(c.d_partition, b->partition + r0, cn * 4, cudaMemcpyHostToDevice, s));
        CU(cudaMemcpyAsync(c.d_ts, b->ts_ms + r0, cn * 8, cudaMemcpyHostToDevice, s));
        CU(cudaMemcpyAsync(c.d_klen, b->key_len + r0, cn * 4, cudaMemcpyHostToDevice, s));
        CU(cudaMemcpyAsync(c.d_vlen, b->value_len + r0, cn * 4, cudaMemcpyHostToDevice, s));
        if (use_seq) CU(cudaMemcpyAsync(c.d_seq, b->seq + r0, cn * 8, cudaMemcpyHostToDevice, s));
        // keep absolute offsets: place the keys so that (virtual base + k0) is where they land and the
        // virtual base stays 16-byte aligned
        const uint64_t shift = k0 & 15ull;
        if (hash) {
            if (k1 > k0) CU(cudaMemcpyAsync(c.d_keys + shift, b->key_bytes + k0, k1 - k0, cudaMemcpyHostToDevice, s));
            CU(cudaMemcpyAsync(c.d_tile_base, tb_src, (ntiles + 1) * 8, cudaMemcpyHostToDevice, s));
        }
        const ScanParams prm = scan_params(cn, seq_base + (uint64_t)r0, c.d_partition, c.d_ts, c.d_klen, c.d_vlen,
                                           hash ? c.d_keys + shift - k0 : nullptr, hash ? c.d_tile_base.get() : nullptr,
                                           use_seq ? c.d_seq.get() : nullptr);
        const uint64_t seq_ends[2] = {use_seq ? b->seq[r0] : 0, use_seq ? b->seq[r0 + cn - 1] : 0};
        if ((rc = ring_scan_chunk(h, prm, (int64_t)((k1 + 15) & ~15ull), (int64_t)(k1 - k0), use_seq ? seq_ends : nullptr))) return rc;
        koff = k1;
        r0 += cn;
    }
    // the caller may reuse its buffers when we return: all host→device copies must have been consumed
    CU(cudaStreamSynchronize(s));
    if ((rc = collect_timing(h))) return rc;
    h->next_seq = std::max<uint64_t>(h->next_seq, seq_base + (uint64_t)b->n);
    return hk_reported(h);
}

extern "C" int kta_sync(kta_handle *h) {
    if (!h) return fail(KTA_ERR_INVALID, "null handle");
    int rc;
    if ((rc = set_device(h))) return rc;
    if ((rc = ring_flush(h))) return rc;
    CU(cudaStreamSynchronize(h->stream));
    if ((rc = alive_settle(h)) || (rc = collect_timing(h))) return rc;
    return hk_reported(h);
}

extern "C" int kta_reset(kta_handle *h) {
    if (!h) return fail(KTA_ERR_INVALID, "null handle");
    int rc;
    if ((rc = set_device(h))) return rc;
    h->pc.n = 0;
    h->pc.kb = 0;
    h->next_seq = 0;
    h->finalized = false;
    h->launches = 0;
    h->records = 0;
    h->log.txn.ranges.clear();
    for (uint64_t &v : h->log.txn.totals) v = 0;
    for (uint64_t &v : h->log.crc.totals) v = 0;   // (the check.crcs switch itself stays as it is)
    h->log.crc.kept.clear();
    OffsetState &o = h->log.offsets;   // windows and their totals
    std::fill(o.win.begin(), o.win.end(), make_longlong2(-1, -1));
    o.set = 0;
    o.dirty = !o.win.empty();
    for (uint64_t &v : o.totals) v = 0;
    if (h->tl.buckets) CU(cudaMemsetAsync(h->tl.d_bins, 0, h->tl.words() * 8, h->stream));   // (its configuration stays)
    if (h->pt.ncounts) CU(cudaMemsetAsync(h->pt.d_counts, 0, h->pt.words() * 8, h->stream));   // (so does the check's)
    if (h->hk.top_k) {   // (the hot-key table keeps its configuration and its allocation)
        HotKeys &k = h->hk;
        CU(cudaMemsetAsync(k.d_table, 0, (size_t)(k.slots + 1) * sizeof(HkSlot), h->stream));
        CU(cudaMemsetAsync(k.d_word, 0, 5 * 8, h->stream));
        k.bound = 0;
        k.nomem = k.unreported = false;
        k.h_top.clear();
        k.h_distinct = k.h_keyed = 0;
    }
    return state_reset_device(h);
}

extern "C" int kta_finalize(kta_handle *h) {
    if (!h) return fail(KTA_ERR_INVALID, "null handle");
    int rc;
    if ((rc = set_device(h))) return rc;
    if ((rc = ring_flush(h))) return rc;
    cudaStream_t s = h->stream;
    if ((rc = alive_settle(h))) return rc;   // every stamp has landed (grows the table and re-runs batches if it was too small)
    if (h->alive.d_table && h->nhll) {
        // EXTENSION: with -c the sketch describes the resolved alive set, so it is rebuilt from the table
        CU(cudaMemsetAsync(h->d_hll, 0, h->nhll * 4, s));
        alive_hll_kernel<<<h->sm_count * 8, THREADS, 0, s>>>(h->alive.d_table, (size_t)h->alive.pairs * 2, h->d_hll,
                                                             h->cfg.hll_precision);
        CU(cudaGetLastError());
        h->launches++;
    }
    h->h_sums.resize(h->nsums);
    h->h_hll.resize(h->nhll);
    CU(cudaMemcpyAsync(h->h_sums.data(), h->d_sums, h->nsums * 8, cudaMemcpyDeviceToHost, s));
    CU(cudaMemcpyAsync(h->h_minmax, h->d_minmax, 32, cudaMemcpyDeviceToHost, s));
    if (h->nhll) CU(cudaMemcpyAsync(h->h_hll.data(), h->d_hll, h->nhll * 4, cudaMemcpyDeviceToHost, s));
    if (h->tl.buckets) {
        h->tl.h_bins.resize(h->tl.words());
        CU(cudaMemcpyAsync(h->tl.h_bins.data(), h->tl.d_bins, h->tl.words() * 8, cudaMemcpyDeviceToHost, s));
    }
    if (h->pt.ncounts) {
        h->pt.h_counts.resize(h->pt.words());
        CU(cudaMemcpyAsync(h->pt.h_counts.data(), h->pt.d_counts, h->pt.words() * 8, cudaMemcpyDeviceToHost, s));
    }
    if (h->hk.top_k && !h->hk.nomem && (rc = hk_finalize(h))) return rc;
    CU(cudaStreamSynchronize(s));
    if ((rc = collect_timing(h))) return rc;
    h->h_alive = h->alive.now;   // counted over the table by alive_settle above (sum_all_alive, src/metric.rs:282-284)
    h->finalized = true;
    if (h->alive.window_errors)
        return fail(KTA_ERR_INVALID, "%llu record(s) carried a sequence number outside the alive-key table's window "
                    "[origin, origin + 2^31 - 2): with an explicit seq column the span between kta_reset calls is limited",
                    (unsigned long long)h->alive.window_errors);
    // Records with a partition outside [0, P) took part in nothing (no counter, no extremum, no alive key): the getters
    // are valid and describe the in-range records; the status tells the caller that some were left out.
    const uint64_t bad = h->h_sums[h->nsums - 1];
    if (bad)
        return fail(KTA_ERR_PARTITION, "%llu record(s) had a partition outside [0, %d) and were left out of every metric",
                    (unsigned long long)bad, h->cfg.num_partitions);
    return hk_reported(h);   // (after the statuses above: the hot-key getters keep returning KTA_ERR_NOMEM either way)
}

// ------------------------------------------------------------------------------------------------
// getters (host arithmetic on the finalized state)
// ------------------------------------------------------------------------------------------------
static int check_read(const kta_handle *h, int32_t p, bool per_partition) {
    if (!h) return fail(KTA_ERR_INVALID, "null handle");
    if (!h->finalized) return fail(KTA_ERR_NOT_FINALIZED, "call kta_finalize first");
    if (per_partition && (p < 0 || p >= h->cfg.num_partitions)) return -1;  // unseen partition: reads as 0
    return KTA_OK;
}

static uint64_t raw_counter(const kta_handle *h, int which, int32_t p) {
    const int P = h->cfg.num_partitions;
    const uint64_t *s = h->h_sums.data();
    uint64_t knn = 0, alive = 0;
    for (int b = 0; b < NB; b++) {
        knn += s[(size_t)p * NB + b];
        alive += s[(size_t)(P + p) * NB + b];
    }
    const uint64_t knull = s[(size_t)P * (2 * NB + 2) + p];
    const uint64_t total = knn + knull;
    switch (which) {
        case KTA_TOTAL: return total;
        case KTA_TOMBSTONES: return total - alive;
        case KTA_ALIVE: return alive;
        case KTA_KEY_NULL: return knull;
        case KTA_KEY_NON_NULL: return knn;
        case KTA_KEY_SIZE_SUM: return s[(size_t)P * (2 * NB) + p];
        case KTA_VALUE_SIZE_SUM: return s[(size_t)P * (2 * NB + 1) + p];
    }
    return 0;
}

extern "C" int kta_counter(const kta_handle *h, int which, int32_t partition, uint64_t *out) {
    if (!out || which < 0 || which > KTA_VALUE_SIZE_SUM) return fail(KTA_ERR_INVALID, "bad argument");
    const int rc = check_read(h, partition, true);
    if (rc > 0) return rc;
    *out = rc < 0 ? 0 : raw_counter(h, which, partition);  // src/metric.rs:198-203: None => 0
    return KTA_OK;
}

extern "C" int kta_avg(const kta_handle *h, int which, int32_t partition, uint64_t *out) {
    if (!out || which < 0 || which > KTA_MESSAGE_SIZE_AVG) return fail(KTA_ERR_INVALID, "bad argument");
    const int rc = check_read(h, partition, true);
    if (rc > 0) return rc;
    if (rc < 0) { *out = 0; return KTA_OK; }
    const uint64_t ks = raw_counter(h, KTA_KEY_SIZE_SUM, partition), vs = raw_counter(h, KTA_VALUE_SIZE_SUM, partition);
    const uint64_t alive = raw_counter(h, KTA_ALIVE, partition);
    // src/metric.rs:132-157: every average divides by alive(p), guarded only by `sum > 0`
    const uint64_t sum = which == KTA_KEY_SIZE_AVG ? ks : which == KTA_VALUE_SIZE_AVG ? vs : ks + vs;
    if (sum > 0) {
        if (alive == 0)
            return fail(KTA_ERR_DIV_BY_ZERO, "partition %d: sum %llu > 0 with alive == 0 (the reference panics here)",
                        partition, (unsigned long long)sum);
        *out = sum / alive;
    } else {
        *out = 0;
    }
    return KTA_OK;
}

extern "C" int kta_dirty_ratio(const kta_handle *h, int32_t partition, float *out) {
    if (!out) return fail(KTA_ERR_INVALID, "bad argument");
    const int rc = check_read(h, partition, true);
    if (rc > 0) return rc;
    *out = 0.0f;
    if (rc < 0) return KTA_OK;
    const uint64_t total = raw_counter(h, KTA_TOTAL, partition), tomb = raw_counter(h, KTA_TOMBSTONES, partition);
    if (total > 0 && tomb > 0) {  // src/metric.rs:159-167, f32 throughout, same operation order
        const volatile float t = (float)tomb;
        const volatile float d = (float)total / 100.0f;
        *out = t / d;
    }
    return KTA_OK;
}

extern "C" int kta_global(const kta_handle *h, int which, uint64_t *out) {
    if (!out) return fail(KTA_ERR_INVALID, "bad argument");
    const int rc = check_read(h, 0, false);
    if (rc) return rc;
    const int P = h->cfg.num_partitions;
    const unsigned long long *mm = reinterpret_cast<const unsigned long long *>(h->h_minmax);
    switch (which) {
        case KTA_SMALLEST_MESSAGE: *out = mm[2] == ~0ull ? 0 : mm[2]; return KTA_OK;  // metric.rs:177-183
        case KTA_LARGEST_MESSAGE: *out = mm[3]; return KTA_OK;
        case KTA_OVERALL_SIZE: {
            uint64_t s = 0;
            for (int p = 0; p < P; p++) s += raw_counter(h, KTA_KEY_SIZE_SUM, p) + raw_counter(h, KTA_VALUE_SIZE_SUM, p);
            *out = s;  // metric.rs:224,238
            return KTA_OK;
        }
        case KTA_OVERALL_COUNT: {
            uint64_t s = 0;
            for (int p = 0; p < P; p++) s += raw_counter(h, KTA_TOTAL, p);
            *out = s;  // metric.rs:215
            return KTA_OK;
        }
    }
    return fail(KTA_ERR_INVALID, "bad global id %d", which);
}

extern "C" int kta_timestamps(const kta_handle *h, int64_t *earliest_s, int32_t *earliest_ns, int64_t *latest_s) {
    const int rc = check_read(h, 0, false);
    if (rc) return rc;
    // src/metric.rs:39-40,65-72,209-211: seconds = ms / 1000 truncating; earliest starts at Utc::now(),
    // latest at the epoch.  Truncating division is monotone, so min/max commute with it.
    // The device tracks the extrema of the RAW ts_ms column; "not available" (-1) maps to 0 (metric.rs:209).
    // That map only moves -1 to 0, so: raw min == -1 ⇒ every other value is >= 0 ⇒ mapped min is 0, otherwise
    // the mapped min is the raw min; raw max == -1 ⇒ every other value is < -1 ⇒ mapped max is 0, otherwise
    // the mapped max is the raw max.
    int64_t es = h->cfg.now_s, ls = 0;
    int32_t ens = h->cfg.now_ns;
    if (h->h_minmax[0] != INT64_MAX) {
        const int64_t raw_mn = h->h_minmax[0] == -1 ? 0 : h->h_minmax[0];
        const int64_t raw_mx = h->h_minmax[1] == -1 ? 0 : h->h_minmax[1];
        const int64_t mn = raw_mn / 1000, mx = raw_mx / 1000;
        if (es > mn || (es == mn && ens > 0)) { es = mn; ens = 0; }
        if (ls < mx) ls = mx;
    }
    if (earliest_s) *earliest_s = es;
    if (earliest_ns) *earliest_ns = ens;
    if (latest_s) *latest_s = ls;
    return KTA_OK;
}

extern "C" int kta_alive_keys(const kta_handle *h, uint64_t *out) {
    if (!out) return fail(KTA_ERR_INVALID, "bad argument");
    const int rc = check_read(h, 0, false);
    if (rc) return rc;
    if (h->cfg.count_alive_keys != 1) return fail(KTA_ERR_NOT_ENABLED, "count_alive_keys was not enabled");
    *out = h->h_alive;
    return KTA_OK;
}

extern "C" int kta_bad_partition_records(const kta_handle *h, uint64_t *out) {
    if (!out) return fail(KTA_ERR_INVALID, "bad argument");
    const int rc = check_read(h, 0, false);
    if (rc) return rc;
    *out = h->h_sums[h->nsums - 1];
    return KTA_OK;
}

extern "C" int kta_hist(const kta_handle *h, int which, int32_t partition, uint64_t out[KTA_HIST_BUCKETS]) {
    if (!out || which < 0 || which > 1) return fail(KTA_ERR_INVALID, "bad argument");
    const int rc = check_read(h, partition, true);
    if (rc > 0) return rc;
    const int P = h->cfg.num_partitions;
    for (int b = 0; b < NB; b++)
        out[b] = rc < 0 ? 0 : h->h_sums[(size_t)((which ? P : 0) + partition) * NB + b];
    return KTA_OK;
}

extern "C" int kta_set_timeline(kta_handle *h, int64_t origin_s, int64_t width_s, int32_t buckets) {
    if (!h) return fail(KTA_ERR_INVALID, "null handle");
    if (h->records || h->pc.n)
        return fail(KTA_ERR_INVALID, "the timeline is configured before the first record: records were pushed or scanned "
                    "since create or the last kta_reset");
    if (width_s < 1) return fail(KTA_ERR_INVALID, "timeline width %lld s: must be at least 1", (long long)width_s);
    if (buckets < 0 || buckets > TL_MAX_BUCKETS)
        return fail(KTA_ERR_INVALID, "timeline buckets %d outside [0, %d]", buckets, TL_MAX_BUCKETS);
    __int128 end = (__int128)origin_s + (__int128)buckets * (__int128)width_s;
    if (end > (__int128)INT64_MAX)
        return fail(KTA_ERR_INVALID, "timeline origin %lld + %d buckets x %lld s overflows int64", (long long)origin_s, buckets,
                    (long long)width_s);
    const int64_t P = h->cfg.num_partitions;
    const int64_t bins = P * ((int64_t)buckets + 2);
    if (buckets && bins > TL_MAX_BINS)
        return fail(KTA_ERR_INVALID, "timeline of %lld partitions x %d indices exceeds 2^24 bins", (long long)P, buckets + 2);
    int rc;
    if ((rc = set_device(h))) return rc;
    // the new configuration is built aside and swapped in only when complete: a failure keeps the old one
    Timeline t;
    if (buckets) {
        if ((rc = t.d_bins.alloc(3 * bins))) return rc;
        t.buckets = buckets;
        t.origin = origin_s;
        t.width = width_s;
        t.smem = (size_t)bins * 16 <= h->smem_optin;
        if (t.smem) {
            CU(cudaFuncSetAttribute(timeline_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)h->smem_optin));
            CU(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&t.blocks_per_sm, timeline_kernel<true>, TL_THREADS, (size_t)bins * 16));
        } else {
            CU(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&t.blocks_per_sm, timeline_kernel<false>, TL_THREADS, 0));
        }
        if (t.blocks_per_sm < 1) return fail(KTA_ERR_CUDA, "timeline kernel does not fit an SM");
        CU(cudaMemsetAsync(t.d_bins, 0, (size_t)t.d_bins.cap * 8, h->stream));
        t.h_bins.assign((size_t)t.d_bins.cap, 0);   // nothing scanned yet: a finalized handle reads zeros
    }
    CU(cudaStreamSynchronize(h->stream));   // the zeroing has landed, and no queued pass still uses the old arrays
    h->tl = std::move(t);
    return KTA_OK;
}

extern "C" int kta_timeline(const kta_handle *h, int which, int32_t partition, uint64_t *out, int64_t cap) {
    if (!h || which < KTA_TIMELINE_RECORDS || which > KTA_TIMELINE_BYTES || cap < 0 || (cap && !out))
        return fail(KTA_ERR_INVALID, "bad argument");
    if (!h->tl.buckets) return fail(KTA_ERR_NOT_ENABLED, "the timeline is off (kta_set_timeline)");
    const int rc = check_read(h, partition, true);
    if (rc > 0) return rc;
    const int64_t row = (int64_t)h->tl.buckets + 2, n = std::min<int64_t>(cap, row);
    if (rc < 0) {
        std::fill(out, out + n, (uint64_t)0);
        return KTA_OK;
    }
    const size_t at = ((size_t)which * (size_t)h->cfg.num_partitions + (size_t)partition) * (size_t)row;
    std::copy(h->tl.h_bins.begin() + (long)at, h->tl.h_bins.begin() + (long)(at + (size_t)n), out);
    return KTA_OK;
}

// test hook: the timeline pass's launch shape for a scan of n records (grid, threads, 1 = bins in shared memory)
extern "C" int kta_timeline_shape(const kta_handle *h, int64_t n, int32_t *grid, int32_t *threads, int32_t *smem_bins) {
    if (!h || n < 0 || !grid || !threads || !smem_bins) return fail(KTA_ERR_INVALID, "bad argument");
    if (!h->tl.buckets) return fail(KTA_ERR_NOT_ENABLED, "the timeline is off (kta_set_timeline)");
    int g = 0, th = 0;
    size_t sm = 0;
    timeline_shape(h, n, g, th, sm);
    *grid = g;
    *threads = th;
    *smem_bins = h->tl.smem ? 1 : 0;
    return KTA_OK;
}

// the zlib CRC-32 slicing tables of the partitioner check and the hot-key table, made on first use
static int crc32_tables(kta_handle *h) {
    if (h->d_crc32_tables) return KTA_OK;
    uint32_t tables[4][256];
    crc_slicing_tables_host(tables, ZLIB_CRC32_POLY);
    DevBuf<uint32_t> d;
    int rc;
    if ((rc = d.alloc(PC_TABLE_WORDS))) return rc;
    CU(cudaMemcpy(d, &tables[0][0], sizeof tables, cudaMemcpyHostToDevice));
    h->d_crc32_tables = std::move(d);
    return KTA_OK;
}

extern "C" int kta_set_partitioner_check(kta_handle *h, const int32_t *counts, int32_t ncounts) {
    if (!h) return fail(KTA_ERR_INVALID, "null handle");
    if (h->records || h->pc.n)
        return fail(KTA_ERR_INVALID, "the partitioner check is configured before the first record: records were pushed or "
                    "scanned since create or the last kta_reset");
    if (ncounts < 0 || ncounts > KTA_PARTITIONER_MAX_COUNTS)
        return fail(KTA_ERR_INVALID, "partitioner check of %d counts: outside [0, %d]", ncounts, KTA_PARTITIONER_MAX_COUNTS);
    if (ncounts && !counts) return fail(KTA_ERR_INVALID, "counts is NULL");
    for (int j = 0; j < ncounts; j++) {
        if (counts[j] < 1) return fail(KTA_ERR_INVALID, "partition count %d: outside [1, 2^31 - 1]", counts[j]);
        for (int i = 0; i < j; i++)
            if (counts[i] == counts[j]) return fail(KTA_ERR_INVALID, "partition count %d given twice", counts[j]);
    }
    int rc;
    if ((rc = set_device(h))) return rc;
    if (ncounts && (rc = crc32_tables(h))) return rc;
    // the new configuration is built aside and swapped in only when complete: a failure keeps the old one
    Partitioner t;
    if (ncounts) {
        const int64_t words = (int64_t)(2 * ncounts + 1) * h->cfg.num_partitions;
        if ((rc = t.d_counts.alloc(words))) return rc;
        t.ncounts = ncounts;
        std::copy(counts, counts + ncounts, t.counts);
        // counters in shared memory when they fit beside the table and a smallest stage per warp
        t.smem = (size_t)PC_TABLE_WORDS * 4 + (size_t)(words + 3) / 4 * 16 + (size_t)PC_WARPS * (PC_STAGE_MIN + PC_STAGE_PAD) <= h->smem_optin;
        CU(cudaFuncSetAttribute(partitioner_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)h->smem_optin));
        CU(cudaFuncSetAttribute(partitioner_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)h->smem_optin));
        CU(cudaMemsetAsync(t.d_counts, 0, (size_t)words * 8, h->stream));
        t.h_counts.assign((size_t)words, 0);   // nothing scanned yet: a finalized handle reads zeros
    }
    CU(cudaStreamSynchronize(h->stream));   // the zeroing has landed, and no queued pass still uses the old counters
    h->pt = std::move(t);
    h->pc.hash = keys_travel(h);   // from now on kta_push copies the keys (nothing is in the landing ring)
    return KTA_OK;
}

extern "C" int kta_partitioner_check(const kta_handle *h, int32_t partition, uint64_t *out, int64_t cap) {
    if (!h || cap < 0 || (cap && !out)) return fail(KTA_ERR_INVALID, "bad argument");
    if (!h->pt.ncounts) return fail(KTA_ERR_NOT_ENABLED, "the partitioner check is off (kta_set_partitioner_check)");
    const int rc = check_read(h, partition, true);
    if (rc > 0) return rc;
    const int64_t nv = 2 * (int64_t)h->pt.ncounts + 1, n = std::min<int64_t>(cap, nv);
    for (int64_t b = 0; b < n; b++)
        out[b] = rc < 0 ? 0 : h->pt.h_counts[(size_t)b * (size_t)h->cfg.num_partitions + (size_t)partition];
    return KTA_OK;
}

// test hook: the partitioner pass's launch shape for a scan of n records with key_bytes key bytes (grid, stage bytes per
// warp, 1 = counters in shared memory)
extern "C" int kta_partitioner_shape(const kta_handle *h, int64_t n, int64_t key_bytes, int32_t *grid, int32_t *stage,
                                     int32_t *smem_counters) {
    if (!h || n < 0 || !grid || !stage || !smem_counters) return fail(KTA_ERR_INVALID, "bad argument");
    if (!h->pt.ncounts) return fail(KTA_ERR_NOT_ENABLED, "the partitioner check is off (kta_set_partitioner_check)");
    int rc;
    if ((rc = set_device(h))) return rc;
    int g = 0, st = 0;
    size_t sm = 0;
    if ((rc = partitioner_shape(h, n, key_bytes, g, st, sm))) return rc;
    *grid = g;
    *stage = st;
    *smem_counters = h->pt.smem ? 1 : 0;
    return KTA_OK;
}

// test hook: at most max_ctas CTAs per partitioner pass (0: as many as are resident), so that one CTA can be given its full
// PC_MAX_CTA_TILES tiles; the tile cap still raises the grid above the limit
extern "C" int kta_partitioner_limit_grid(kta_handle *h, int32_t max_ctas) {
    if (!h || max_ctas < 0) return fail(KTA_ERR_INVALID, "bad argument");
    if (!h->pt.ncounts) return fail(KTA_ERR_NOT_ENABLED, "the partitioner check is off (kta_set_partitioner_check)");
    h->pt.max_grid = max_ctas;
    return KTA_OK;
}

extern "C" int kta_set_hot_keys(kta_handle *h, int32_t top_k, int64_t table_slots) {
    if (!h) return fail(KTA_ERR_INVALID, "null handle");
    if (h->records || h->pc.n)
        return fail(KTA_ERR_INVALID, "the hot-key table is configured before the first record: records were pushed or scanned "
                    "since create or the last kta_reset");
    if (top_k < 0 || top_k > KTA_HOT_KEYS_MAX) return fail(KTA_ERR_INVALID, "top_k %d outside [0, %d]", top_k, KTA_HOT_KEYS_MAX);
    if (table_slots != 0 && (table_slots < (int64_t)HK_MIN_SLOTS || table_slots > (int64_t)HK_MAX_SLOTS || (table_slots & (table_slots - 1))))
        return fail(KTA_ERR_INVALID, "table_slots %lld: 0 or a power of two in [16, 2^31]", (long long)table_slots);
    int rc;
    if ((rc = set_device(h))) return rc;
    // the new configuration is built aside and swapped in only when complete: a failure keeps the old one
    HotKeys k;
    if (top_k) {
        if ((rc = crc32_tables(h))) return rc;
        k.slots = table_slots ? (uint64_t)table_slots : HK_DEFAULT_SLOTS;
        if ((rc = k.d_table.alloc((int64_t)k.slots + 1)) || (rc = k.d_word.alloc(5))) return rc;
        CU(cudaFuncSetAttribute(hot_keys_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)h->smem_optin));
        CU(cudaMemsetAsync(k.d_table, 0, (size_t)(k.slots + 1) * sizeof(HkSlot), h->stream));
        CU(cudaMemsetAsync(k.d_word, 0, 5 * 8, h->stream));
        k.top_k = top_k;
    }
    CU(cudaStreamSynchronize(h->stream));   // the zeroing has landed, and no queued pass still uses the old table
    h->hk = std::move(k);
    h->pc.hash = keys_travel(h);   // from now on kta_push copies the keys (nothing is in the landing ring)
    return KTA_OK;
}

static int hk_check(const kta_handle *h) {
    if (!h) return fail(KTA_ERR_INVALID, "null handle");
    if (!h->hk.top_k) return fail(KTA_ERR_NOT_ENABLED, "the hot-key table is off (kta_set_hot_keys)");
    if (h->hk.nomem) return fail(KTA_ERR_NOMEM, "%s", h->hk.nomem_msg);
    return KTA_OK;
}

extern "C" int kta_hot_keys(const kta_handle *h, kta_hot_key *out, int64_t cap, int64_t *count) {
    if (!h || cap < 0 || (cap && !out)) return fail(KTA_ERR_INVALID, "bad argument");
    int rc;
    if ((rc = hk_check(h)) || (rc = check_read(h, 0, false))) return rc;
    const std::vector<kta_hot_key> &top = h->hk.h_top;
    const size_t n = std::min<size_t>((size_t)cap, top.size());
    if (n) memcpy(out, top.data(), n * sizeof(kta_hot_key));
    if (count) *count = (int64_t)top.size();
    return KTA_OK;
}

extern "C" int kta_hot_key_stats(const kta_handle *h, uint64_t *distinct_keys, uint64_t *keyed_records, uint64_t *slots,
                                 uint64_t *grows, uint64_t *slices) {
    int rc;
    if ((rc = hk_check(h)) || (rc = check_read(h, 0, false))) return rc;
    const HotKeys &k = h->hk;
    if (distinct_keys) *distinct_keys = k.h_distinct;
    if (keyed_records) *keyed_records = k.h_keyed;
    if (slots) *slots = k.slots;
    if (grows) *grows = k.grows;
    if (slices) *slices = k.slices;
    return KTA_OK;
}

// every entry into out[0, cap) (cap 0: none); `records` (may be NULL) gets their records' sum; count = the occupancy
static int hk_export(kta_handle *h, kta_hot_key *out, int64_t cap, unsigned long long *records, uint64_t &count) {
    HotKeys &k = h->hk;
    int rc;
    if ((rc = hk_occupancy(h, count))) return rc;
    cudaStream_t s = h->stream;
    CU(cudaMemsetAsync(k.d_word + 2, 0, 16, s));
    hot_keys_export_kernel<<<hk_grid(h, (int64_t)k.slots + 1), 256, 0, s>>>(k.d_table, k.slots, k.d_word + 2, k.d_word + 3, out,
                                                                            (unsigned long long)cap);
    h->launches++;
    CU(cudaGetLastError());
    if (records) CU(cudaMemcpyAsync(records, k.d_word + 3, 8, cudaMemcpyDeviceToHost, s));
    return KTA_OK;
}

// finalize: the occupied slots compacted, sorted by (records descending, id ascending), the first top_k to the host
static int hk_finalize(kta_handle *h) {
    HotKeys &k = h->hk;
    cudaStream_t s = h->stream;
    uint64_t n = 0;
    unsigned long long keyed = 0;
    int rc;
    if ((rc = hk_occupancy(h, n)) || (rc = k.d_entries.grow(s, (int64_t)std::max<uint64_t>(n, 1))) ||
        (rc = hk_export(h, k.d_entries, k.d_entries.cap, &keyed, n)))
        return rc;
    k.bound = n;
    const int64_t top = (int64_t)std::min<uint64_t>(n, (uint64_t)k.top_k);
    k.h_top.resize((size_t)top);
    if (n) {
        size_t tmp = 0;
        CU(hot_keys_sort(nullptr, tmp, nullptr, nullptr, nullptr, nullptr, (int64_t)n, s));
        if ((rc = k.d_keys.grow(s, 2 * (int64_t)n)) || (rc = k.d_idx.grow(s, 2 * (int64_t)n)) || (rc = k.d_sort_tmp.grow(s, (int64_t)tmp)) ||
            (rc = k.d_top.grow(s, top)))
            return rc;
        tmp = (size_t)k.d_sort_tmp.cap;
        hot_keys_sort_keys_kernel<<<hk_grid(h, (int64_t)n), 256, 0, s>>>(k.d_entries, (int64_t)n, k.d_keys, k.d_idx);
        CU(hot_keys_sort(k.d_sort_tmp, tmp, k.d_keys, k.d_keys + n, k.d_idx, k.d_idx + n, (int64_t)n, s));
        hot_keys_gather_kernel<<<hk_grid(h, top), 256, 0, s>>>(k.d_entries, k.d_idx + n, top, k.d_top);
        h->launches += 3;
        CU(cudaGetLastError());
        CU(cudaMemcpyAsync(k.h_top.data(), k.d_top, (size_t)top * sizeof(kta_hot_key), cudaMemcpyDeviceToHost, s));
    }
    CU(cudaStreamSynchronize(s));
    k.h_distinct = n;
    k.h_keyed = keyed;
    return KTA_OK;
}

extern "C" int kta_hot_keys_export_count(kta_handle *h, int64_t *count) {
    if (!count) return fail(KTA_ERR_INVALID, "bad argument");
    int rc;
    if ((rc = hk_check(h)) || (rc = set_device(h)) || (rc = ring_flush(h))) return rc;
    if (h->hk.nomem) return hk_check(h);   // (the flush may have run the table out of memory)
    uint64_t n = 0;
    if ((rc = hk_occupancy(h, n))) return rc;
    *count = (int64_t)n;
    return KTA_OK;
}

extern "C" int kta_hot_keys_export_device(kta_handle *h, kta_hot_key *dev_out, int64_t cap, int64_t *count) {
    if (!count || cap < 0 || (cap && !dev_out)) return fail(KTA_ERR_INVALID, "bad argument");
    int rc;
    if ((rc = hk_check(h)) || (rc = set_device(h)) || (rc = ring_flush(h))) return rc;
    if (h->hk.nomem) return hk_check(h);
    uint64_t n = 0;
    if ((rc = hk_export(h, dev_out, cap, nullptr, n))) return rc;
    CU(cudaStreamSynchronize(h->stream));
    *count = (int64_t)n;
    if ((int64_t)n > cap) return fail(KTA_ERR_INVALID, "export buffer too small: %llu > %lld", (unsigned long long)n, (long long)cap);
    return KTA_OK;
}

// the list is checked on the device (one read-back) before anything is applied; the table grows first, so that every entry
// finds a slot and the table stays at most half full
extern "C" int kta_hot_keys_import_device(kta_handle *h, const kta_hot_key *dev_in, int64_t count) {
    if (count < 0 || (count && !dev_in)) return fail(KTA_ERR_INVALID, "bad argument");
    int rc;
    if ((rc = hk_check(h))) return rc;
    if (count == 0) return KTA_OK;
    if ((rc = set_device(h))) return rc;
    HotKeys &k = h->hk;
    cudaStream_t s = h->stream;
    unsigned int bad = 0;
    CU(cudaMemsetAsync(k.d_word + 4, 0, 8, s));
    hot_keys_validate_kernel<<<hk_grid(h, count), 256, 0, s>>>(dev_in, count, h->cfg.num_partitions,
                                                               reinterpret_cast<unsigned int *>(k.d_word.get() + 4));
    h->launches++;
    CU(cudaGetLastError());
    CU(cudaMemcpyAsync(&bad, k.d_word + 4, 4, cudaMemcpyDeviceToHost, s));
    CU(cudaStreamSynchronize(s));
    if (bad)
        return fail(KTA_ERR_INVALID, "hot-key import refused: an entry has records == 0, tombstones > records, key_len < 0, a "
                    "nonzero reserved word, or a partition range outside [0, %d)", h->cfg.num_partitions);
    uint64_t occ = 0;
    if ((rc = hk_occupancy(h, occ))) return rc;
    k.bound = occ + (uint64_t)count;
    if (k.bound > k.slots / 2 && (rc = hk_grow(h, k.bound * 2))) return k.nomem ? hk_reported(h) : rc;
    hot_keys_import_kernel<<<hk_grid(h, count), 256, 0, s>>>(dev_in, count, k.table());
    h->launches++;
    CU(cudaGetLastError());
    h->finalized = false;
    return hk_occupancy(h, occ);   // (the caller may free its list when this returns)
}

extern "C" int kta_hot_keys_limit_slots(kta_handle *h, int64_t max_slots) {
    if (!h || max_slots < 0) return fail(KTA_ERR_INVALID, "bad argument");
    if (!h->hk.top_k) return fail(KTA_ERR_NOT_ENABLED, "the hot-key table is off (kta_set_hot_keys)");
    h->hk.max_slots = (uint64_t)max_slots;
    return KTA_OK;
}

// Ertl 2017, "New cardinality estimation algorithms for HyperLogLog sketches": improved raw estimator
static double hll_sigma(double x) {
    if (x == 1.0) return INFINITY;
    double y = 1.0, z = x, zo;
    do { x *= x; zo = z; z += x * y; y += y; } while (zo != z);
    return z;
}
static double hll_tau(double x) {
    if (x == 0.0 || x == 1.0) return 0.0;
    double y = 1.0, z = 1.0 - x, zo;
    do { x = std::sqrt(x); zo = z; y *= 0.5; z -= (1.0 - x) * (1.0 - x) * y; } while (zo != z);
    return z / 3.0;
}

extern "C" int kta_alive_keys_hll(const kta_handle *h, double *out) {
    if (!out) return fail(KTA_ERR_INVALID, "bad argument");
    const int rc = check_read(h, 0, false);
    if (rc) return rc;
    if (!h->nhll) return fail(KTA_ERR_NOT_ENABLED, "hll_precision was 0");
    const int p = h->cfg.hll_precision, q = 32 - p;
    const double m = (double)h->nhll;
    std::vector<double> C((size_t)q + 2, 0.0);
    for (uint32_t r : h->h_hll) C[std::min<uint32_t>(r, (uint32_t)q + 1)] += 1.0;
    double z = m * hll_tau(1.0 - C[(size_t)q + 1] / m);
    for (int k = q; k >= 1; k--) z = 0.5 * (z + C[(size_t)k]);
    z += m * hll_sigma(C[0] / m);
    *out = 0.72134752044448170368 * m * m / z;
    return KTA_OK;
}

extern "C" int kta_hll_registers(const kta_handle *h, uint8_t *out, size_t cap) {
    if (!out) return fail(KTA_ERR_INVALID, "bad argument");
    const int rc = check_read(h, 0, false);
    if (rc) return rc;
    if (!h->nhll) return fail(KTA_ERR_NOT_ENABLED, "hll_precision was 0");
    if (cap < h->nhll) return fail(KTA_ERR_INVALID, "buffer too small: %zu < %zu", cap, h->nhll);
    for (size_t i = 0; i < h->nhll; i++) out[i] = (uint8_t)h->h_hll[i];
    return KTA_OK;
}

extern "C" int kta_fnv32_host(kta_handle *h, int64_t n, const int32_t *key_len, const uint8_t *key_bytes,
                              int64_t key_bytes_len, uint32_t *out) {
    if (!h || n < 0 || (n && (!key_len || !out))) return fail(KTA_ERR_INVALID, "bad argument");
    if (n == 0) return KTA_OK;
    int rc;
    if ((rc = set_device(h))) return rc;
    std::vector<uint64_t> off((size_t)n);
    uint64_t acc = 0;
    for (int64_t i = 0; i < n; i++) {
        off[(size_t)i] = acc;
        acc += key_len[i] > 0 ? (uint64_t)key_len[i] : 0;
    }
    if ((int64_t)acc > key_bytes_len) return fail(KTA_ERR_INVALID, "key_bytes_len %lld < sum of key_len %llu",
                                                  (long long)key_bytes_len, (unsigned long long)acc);
    DevBuf<int32_t> d_len;
    DevBuf<uint64_t> d_off;
    DevBuf<uint8_t> d_keys;
    DevBuf<uint32_t> d_out;
    cudaStream_t s = h->stream;
    if ((rc = d_len.alloc(n)) || (rc = d_off.alloc(n)) || (rc = d_keys.alloc((int64_t)acc + 16)) || (rc = d_out.alloc(n))) return rc;
    CU(cudaMemcpyAsync(d_len, key_len, n * 4, cudaMemcpyHostToDevice, s));
    CU(cudaMemcpyAsync(d_off, off.data(), n * 8, cudaMemcpyHostToDevice, s));
    if (acc) CU(cudaMemcpyAsync(d_keys, key_bytes, acc, cudaMemcpyHostToDevice, s));
    fnv32_kernel<<<(int)std::min<int64_t>((n + 255) / 256, 1024), 256, 0, s>>>(n, d_len, d_off, d_keys, d_out);
    h->launches++;
    CU(cudaGetLastError());
    CU(cudaMemcpyAsync(out, d_out, n * 4, cudaMemcpyDeviceToHost, s));
    CU(cudaStreamSynchronize(s));
    return KTA_OK;
}

extern "C" int kta_partitioner_hash_host(kta_handle *h, int64_t n, const int32_t *key_len, const uint8_t *key_bytes,
                                         int64_t key_bytes_len, uint32_t *murmur2, uint32_t *crc32) {
    if (!h || n < 0 || (n && (!key_len || !murmur2 || !crc32))) return fail(KTA_ERR_INVALID, "bad argument");
    if (n == 0) return KTA_OK;
    int rc;
    if ((rc = set_device(h))) return rc;
    std::vector<uint64_t> off((size_t)n);
    uint64_t acc = 0;
    for (int64_t i = 0; i < n; i++) {
        off[(size_t)i] = acc;
        acc += key_len[i] > 0 ? (uint64_t)key_len[i] : 0;
    }
    if ((int64_t)acc > key_bytes_len) return fail(KTA_ERR_INVALID, "key_bytes_len %lld < sum of key_len %llu",
                                                  (long long)key_bytes_len, (unsigned long long)acc);
    if (acc && !key_bytes) return fail(KTA_ERR_INVALID, "key_bytes is NULL");
    uint32_t tables[4][256];
    crc_slicing_tables_host(tables, ZLIB_CRC32_POLY);
    DevBuf<int32_t> d_len;
    DevBuf<uint64_t> d_off;
    DevBuf<uint8_t> d_keys;
    DevBuf<uint32_t> d_out, d_tables;
    cudaStream_t s = h->stream;
    if ((rc = d_len.alloc(n)) || (rc = d_off.alloc(n)) || (rc = d_keys.alloc((int64_t)acc + 16)) || (rc = d_out.alloc(2 * n)) ||
        (rc = d_tables.alloc(PC_TABLE_WORDS)))
        return rc;
    CU(cudaMemcpyAsync(d_len, key_len, n * 4, cudaMemcpyHostToDevice, s));
    CU(cudaMemcpyAsync(d_off, off.data(), n * 8, cudaMemcpyHostToDevice, s));
    CU(cudaMemcpyAsync(d_tables, &tables[0][0], sizeof tables, cudaMemcpyHostToDevice, s));
    if (acc) CU(cudaMemcpyAsync(d_keys, key_bytes, acc, cudaMemcpyHostToDevice, s));
    partitioner_hash_kernel<<<(int)std::min<int64_t>((n + 255) / 256, 1024), 256, 0, s>>>(n, d_len, d_off, d_keys, d_tables, d_out,
                                                                                         d_out + n);
    h->launches++;
    CU(cudaGetLastError());
    CU(cudaMemcpyAsync(murmur2, d_out, n * 4, cudaMemcpyDeviceToHost, s));
    CU(cudaMemcpyAsync(crc32, d_out + n, n * 4, cudaMemcpyDeviceToHost, s));
    CU(cudaStreamSynchronize(s));
    return KTA_OK;
}

// test hook: capture the per-record hash computed inside the fused scan (device buffer of n u32, or NULL)
extern "C" int kta_set_hash_capture(kta_handle *h, uint32_t *dev_out) {
    if (!h) return fail(KTA_ERR_INVALID, "null handle");
    int rc;
    if ((rc = set_device(h))) return rc;
    if ((rc = ring_flush(h))) return rc;   // records already landed were taken with the old setting
    h->d_hash_out = dev_out;
    h->pc.hash = keys_travel(h);
    return KTA_OK;
}

// ------------------------------------------------------------------------------------------------
// multi-GPU merge
// ------------------------------------------------------------------------------------------------
// words of the merge buffer in front of the timeline segment (the partitioner check's segment follows the timeline's)
static size_t merge_base_words(const kta_handle *h, int32_t world) { return h->nsums + (size_t)world * 4 + (size_t)world * (h->nhll / 8); }

extern "C" int64_t kta_merge_words(const kta_handle *h, int32_t world) {
    if (!h || world < 1) return -1;
    return (int64_t)(merge_base_words(h, world) + h->tl.words() + h->pt.words());
}

extern "C" int kta_merge_export_device(kta_handle *h, int32_t rank, int32_t world, uint64_t *dev_buf) {
    if (!h || !dev_buf || world < 1 || rank < 0 || rank >= world) return fail(KTA_ERR_INVALID, "bad argument");
    int rc;
    if ((rc = set_device(h))) return rc;
    if ((rc = ring_flush(h))) return rc;
    if ((rc = alive_settle_if_any(h))) return rc;
    merge_export_kernel<<<h->sm_count, 256, 0, h->stream>>>(h->d_sums, h->nsums, h->d_minmax, h->d_hll, h->nhll, rank,
                                                           world, reinterpret_cast<unsigned long long *>(dev_buf));
    h->launches++;
    CU(cudaGetLastError());
    // the timeline arrays go at the end as they are: the SUM all-reduce adds every rank's rows (foreign rows are zero)
    if (h->tl.buckets)
        CU(cudaMemcpyAsync(dev_buf + merge_base_words(h, world), h->tl.d_bins, h->tl.words() * 8, cudaMemcpyDeviceToDevice, h->stream));
    // so do the partitioner check's counters, behind the timeline's
    if (h->pt.ncounts)
        CU(cudaMemcpyAsync(dev_buf + merge_base_words(h, world) + h->tl.words(), h->pt.d_counts, h->pt.words() * 8,
                           cudaMemcpyDeviceToDevice, h->stream));
    // With its own stream the handle must finish before the caller's collective may read the buffer.  On an
    // adopted stream (kta_set_stream) the caller's collective is ordered behind this kernel by the stream itself.
    if (h->own_stream) {
        CU(cudaStreamSynchronize(h->stream));
        return collect_timing(h);
    }
    return KTA_OK;
}

extern "C" int kta_merge_import_device(kta_handle *h, int32_t world, const uint64_t *dev_buf) {
    if (!h || !dev_buf || world < 1) return fail(KTA_ERR_INVALID, "bad argument");
    int rc;
    if ((rc = set_device(h))) return rc;
    merge_import_kernel<<<h->sm_count, 256, 0, h->stream>>>(h->d_sums, h->nsums, h->d_minmax, h->d_hll, h->nhll,
                                                           h->d_hll_floor, world,
                                                           reinterpret_cast<const unsigned long long *>(dev_buf));
    h->launches++;
    CU(cudaGetLastError());
    if (h->tl.buckets)
        CU(cudaMemcpyAsync(h->tl.d_bins, dev_buf + merge_base_words(h, world), h->tl.words() * 8, cudaMemcpyDeviceToDevice, h->stream));
    if (h->pt.ncounts)
        CU(cudaMemcpyAsync(h->pt.d_counts, dev_buf + merge_base_words(h, world) + h->tl.words(), h->pt.words() * 8,
                           cudaMemcpyDeviceToDevice, h->stream));
    h->finalized = false;
    if (h->own_stream) CU(cudaStreamSynchronize(h->stream));
    return KTA_OK;
}

// ------------------------------------------------------------------------------------------------
// introspection
// ------------------------------------------------------------------------------------------------
extern "C" int kta_stats(const kta_handle *h, uint64_t *kernel_launches, uint64_t *records_scanned) {
    if (!h) return fail(KTA_ERR_INVALID, "null handle");
    if (kernel_launches) *kernel_launches = h->launches;
    if (records_scanned) *records_scanned = h->records;
    return KTA_OK;
}

extern "C" int kta_alive_table_stats(kta_handle *h, uint64_t *slots, uint64_t *occupied, uint64_t *grows, uint64_t *reruns) {
    if (!h) return fail(KTA_ERR_INVALID, "null handle");
    if (!h->alive.d_table) return fail(KTA_ERR_NOT_ENABLED, "count_alive_keys was not enabled");
    int rc;
    if ((rc = set_device(h))) return rc;
    if ((rc = ring_flush(h))) return rc;
    if ((rc = alive_settle(h))) return rc;   // confirms every stamp and counts the table
    if (slots) *slots = (uint64_t)h->alive.pairs * 2;
    if (occupied) *occupied = h->alive.occupied;
    if (grows) *grows = h->alive.grows;
    if (reruns) *reruns = h->alive.reruns;
    return KTA_OK;
}

extern "C" int kta_set_timing(kta_handle *h, int enabled) {
    if (!h) return fail(KTA_ERR_INVALID, "null handle");
    h->timing = enabled != 0;
    h->scan_ms = 0;
    h->scan_launches_timed = 0;
    return KTA_OK;
}

extern "C" int kta_scan_time_ms(kta_handle *h, double *total_ms, uint64_t *launches) {
    if (!h) return fail(KTA_ERR_INVALID, "null handle");
    int rc;
    if ((rc = set_device(h))) return rc;
    CU(cudaStreamSynchronize(h->stream));
    if ((rc = collect_timing(h))) return rc;
    if (total_ms) *total_ms = h->scan_ms;
    if (launches) *launches = h->scan_launches_timed;
    return KTA_OK;
}
