// kta_logcrc.cuh — check.crcs for the RecordBatch v2 decoder (kta_logdecode.cuh): every batch's CRC-32C is computed on the
// GPU and a batch whose stored CRC does not match is skipped, as librdkafka with check.crcs=true hands it to the
// application as a consumer error instead of its records.
//
// Kafka's batch CRC is CRC-32C (Castagnoli, reflected polynomial 0x82F63B78, init and xorout 0xFFFFFFFF) over the batch from
// `attributes` (byte 21) to its end (byte 12 + batchLength), as stored (compressed bytes for a compressed batch); the stored
// value is the big-endian u32 at bytes 17-20.  baseOffset, batchLength, partitionLeaderEpoch and magic lie outside it: they
// frame the batch, and the header pass keeps refusing a call for them.
//
// The passes, run before the header pass checks any CRC-covered field (only while the switch is on; the kernels and their
// launches are in kta_logoffsets.cuh, next to the window switch's):
//   count   (log_crc_count_kernel, thread per batch)  framed batches: the number of LOG_CRC_SPAN-byte spans of the CRC
//                                     region; acc[b] = 0
//   scan    (tile_base_scan_kernel)  span counts → the first span of every batch
//   spans   (warp per run of spans)  each lane one span: its CRC from shared-memory tables, moved to the end of its batch
//                                     by a multiplication mod P, xor-combined per batch into acc[b]
//   header  (log_header_kernel<true, W>)  the header pass, which compares acc[b] ^ 0xFFFFFFFF with the stored CRC first: a
//                                     batch that fails is LOGB_SKIP_CRC with records = 0, raises no error bit, and is listed
// Spans are aligned to the region's END, so every span but a batch's first is exactly LOG_CRC_SPAN bytes long and span i of
// n is moved by x^(8 * LOG_CRC_SPAN * (n - 1 - i)): the register is linear, R(init, A | B) = R(init, A) * x^(8|B|) ^
// R(0, B), so the first span starts from the init value, the others from 0, and the batch's register is the xor of all.
// The work is balanced by bytes, not by batches: a 16 MiB batch is spread over 16 Ki lanes like 16 Ki small batches.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "kta_codec.cuh"
#include "kta_logdecode.cuh"

namespace kta {

constexpr uint32_t CRC32C_POLY = 0x82F63B78u;   // reflected: bit 31 is x^0
constexpr uint32_t CRC32C_ONE = 0x80000000u;    // the polynomial 1
constexpr uint32_t LOG_CRC_FROM = 21;            // the CRC region starts at `attributes`
constexpr uint32_t LOG_CRC_SPAN = 1024;          // bytes per span (S)
constexpr int LOG_CRC_POW_LO = 4096;             // x^(8 S k) for k < 4096 ...
constexpr int LOG_CRC_POW_HI = 512;              // ... times x^(8 S 4096 j): k < 2^21 spans = a 2 GiB region
constexpr int LOG_CRC_THREADS = 1024;
constexpr size_t LOG_CRC_SMEM = 4 * 256 * 32 * sizeof(uint32_t);   // the 4 slicing tables, one replica per lane (128 KiB)

// The constant tables, built on the host (log_crc_tables_host) and read by the span pass
struct LogCrcTables {
    uint32_t t[4][256];                  // slicing-by-4: t[0] the byte table, t[k][i] = t[0] applied to t[k-1][i] once more
    uint32_t pow_lo[LOG_CRC_POW_LO];     // x^(8 S k) mod P
    uint32_t pow_hi[LOG_CRC_POW_HI];     // x^(8 S 4096 j) mod P
};

// A batch that failed its check, in the order the header pass met it (the host sorts by batch)
struct LogCrcFail {
    uint32_t batch;
    uint32_t batch_bytes;                // 12 + batchLength
    int64_t base_offset;
    int32_t partition;
    uint32_t stored, computed;
    uint32_t pad;
};

// a * b mod P, both residues in the reflected representation (zlib's multmodp)
__host__ __device__ __forceinline__ uint32_t crc32c_mulmod(uint32_t a, uint32_t b) {
    uint32_t p = 0;
#pragma unroll
    for (int i = 0; i < 32; i++) {
        p ^= (0u - ((a >> (31 - i)) & 1u)) & b;
        b = (b >> 1) ^ ((0u - (b & 1u)) & CRC32C_POLY);
    }
    return p;
}

// the four slicing-by-4 tables of a reflected CRC-32 with polynomial `poly` (0x82F63B78 CRC-32C, 0xEDB88320 zlib's CRC-32):
// t[0] the byte table, t[k][i] = t[0] applied to t[k-1][i] once more
inline void crc_slicing_tables_host(uint32_t (&t)[4][256], uint32_t poly) {
    for (uint32_t i = 0; i < 256; i++) {
        uint32_t c = i;
        for (int k = 0; k < 8; k++) c = (c >> 1) ^ ((0u - (c & 1u)) & poly);
        t[0][i] = c;
    }
    for (int k = 1; k < 4; k++)
        for (int i = 0; i < 256; i++) t[k][i] = (t[k - 1][i] >> 8) ^ t[0][t[k - 1][i] & 0xffu];
}

inline void log_crc_tables_host(LogCrcTables &t) {
    crc_slicing_tables_host(t.t, CRC32C_POLY);
    uint32_t xs = CRC32C_ONE;   // x^(8 S)
    for (uint32_t i = 0; i < 8 * LOG_CRC_SPAN; i++) xs = (xs >> 1) ^ ((0u - (xs & 1u)) & CRC32C_POLY);
    t.pow_lo[0] = CRC32C_ONE;
    for (int k = 1; k < LOG_CRC_POW_LO; k++) t.pow_lo[k] = crc32c_mulmod(t.pow_lo[k - 1], xs);
    const uint32_t xhi = crc32c_mulmod(t.pow_lo[LOG_CRC_POW_LO - 1], xs);
    t.pow_hi[0] = CRC32C_ONE;
    for (int j = 1; j < LOG_CRC_POW_HI; j++) t.pow_hi[j] = crc32c_mulmod(t.pow_hi[j - 1], xhi);
}

// the batch at `off` is framed: its header and its batchLength bytes lie in the buffer, batchLength >= 49, magic 2 (the
// fields outside the CRC; *len = 12 + batchLength)
__device__ __forceinline__ bool log_framed(const uint8_t *bytes, int64_t nbytes, uint64_t off, uint32_t *len) {
    if (off + LOG_HEADER_BYTES > (uint64_t)nbytes) return false;
    const int32_t batch_len = (int32_t)be_u32(bytes + off + 8);
    if ((int8_t)__ldg(bytes + off + 16) != 2 || batch_len < LOG_HEADER_BYTES - 12 || off + 12 + (uint64_t)batch_len > (uint64_t)nbytes)
        return false;
    *len = 12u + (uint32_t)batch_len;
    return true;
}

// thread per batch: spans[b + 1] = spans of batch b's CRC region (0 when it is not framed: the header pass refuses the
// call; with a Window, also 0 when the batch is not served, kta_logoffsets.cuh), acc[b] = 0
template <typename Window>
__device__ __forceinline__ void log_crc_count_pass(const uint8_t *bytes, int64_t nbytes, const uint64_t *batch_off, int64_t nbatches,
                                                   uint64_t *spans, uint32_t *acc, int32_t partition, const int32_t *batch_partition,
                                                   const Window &window) {
    for (int64_t b = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; b < nbatches; b += (int64_t)gridDim.x * blockDim.x) {
        uint32_t len = 0;
        bool framed = log_framed(bytes, nbytes, batch_off[b], &len);
        if constexpr (Window::on)
            framed = framed && window.test(bytes + batch_off[b], batch_partition ? batch_partition[b] : partition) != LOG_WIN_SKIP;
        spans[b + 1] = framed ? (len - LOG_CRC_FROM + LOG_CRC_SPAN - 1) / LOG_CRC_SPAN : 0;
        acc[b] = 0;
    }
    if (blockIdx.x == 0 && threadIdx.x == 0) spans[0] = 0;
}

// The slicing steps of any reflected CRC-32: the polynomial lives in the tables (crc_slicing_tables_host).  Table k, entry
// i, sits at word (k * 256 + i) * R of the table base tl.  R = 32: one replica per lane (tl = table base + lane), so the
// word lies in the lane's own bank; R = 1: one shared copy.
#define LOG_CRC_T(k, i) tl[((k) * 256 + (i)) * R]

template <int R = 32>
__device__ __forceinline__ uint32_t crc_byte(uint32_t crc, uint32_t byte, const uint32_t *tl) {
    return LOG_CRC_T(0, (crc ^ byte) & 0xffu) ^ (crc >> 8);
}
template <int R = 32>
__device__ __forceinline__ uint32_t crc_word(uint32_t crc, uint32_t w, const uint32_t *tl) {
    crc ^= w;
    return LOG_CRC_T(3, crc & 0xffu) ^ LOG_CRC_T(2, (crc >> 8) & 0xffu) ^ LOG_CRC_T(1, (crc >> 16) & 0xffu) ^ LOG_CRC_T(0, crc >> 24);
}

// the register after [a, e) from `crc`: bytes up to 16-byte alignment, 64 then 16 bytes per step, the rest byte by byte
__device__ __forceinline__ uint32_t crc_span(const uint8_t *a, const uint8_t *e, uint32_t crc, const uint32_t *tl) {
    for (; a < e && (reinterpret_cast<uintptr_t>(a) & 15u); a++) crc = crc_byte(crc, __ldg(a), tl);
    for (; e - a >= 64; a += 64) {
        uint4 q[4];
#pragma unroll
        for (int j = 0; j < 4; j++) q[j] = __ldg(reinterpret_cast<const uint4 *>(a) + j);
#pragma unroll
        for (int j = 0; j < 4; j++) {
            crc = crc_word(crc, q[j].x, tl);
            crc = crc_word(crc, q[j].y, tl);
            crc = crc_word(crc, q[j].z, tl);
            crc = crc_word(crc, q[j].w, tl);
        }
    }
    for (; e - a >= 16; a += 16) {
        const uint4 q = __ldg(reinterpret_cast<const uint4 *>(a));
        crc = crc_word(crc, q.x, tl);
        crc = crc_word(crc, q.y, tl);
        crc = crc_word(crc, q.z, tl);
        crc = crc_word(crc, q.w, tl);
    }
    for (; a < e; a++) crc = crc_byte(crc, __ldg(a), tl);
    return crc;
}
#undef LOG_CRC_T

// Each warp takes one contiguous run of the call's spans (spans[nbatches] in all, so the grid needs no host round trip),
// 32 at a time, lane j span g0 + j.  The batch of a span is looked for among the 32 batch ends behind the warp's current
// batch b0 (the batch of the previous round's last span, or of `start`): when every batch has a span, the 32 spans of a
// round lie in batches b0 .. b0 + 32.  Under offset windows a batch that is not served has no span, so a round can reach
// further; a lane whose span lies past batch b0 + 32 finds its batch by a binary search of the rest of the scan.  Lanes of
// one batch xor their shares together before one of them adds the result to acc[b].
__global__ void __launch_bounds__(LOG_CRC_THREADS) log_crc_span_kernel(const uint8_t *bytes, const uint64_t *batch_off, int64_t nbatches,
                                                                       const uint64_t *spans, const LogCrcTables *tables, uint32_t *acc) {
    extern __shared__ uint32_t crc_smem[];
    const uint32_t *flat = &tables->t[0][0];
    for (int w = threadIdx.x; w < 4 * 256 * 32; w += blockDim.x) crc_smem[w] = __ldg(flat + (w >> 5));
    __syncthreads();
    const int lane = threadIdx.x & 31;
    const uint32_t *tl = crc_smem + lane;
    const uint64_t total = spans[nbatches];
    const uint64_t nwarps = ((uint64_t)gridDim.x * blockDim.x) >> 5, warp = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const uint64_t per = (total + nwarps - 1) / nwarps;
    const uint64_t start = warp * per, end = min(total, start + per);
    if (start >= end) return;
    // b0: the batch of span `start` (the last batch whose first span is <= start)
    int64_t lo = 0, hi = nbatches - 1;
    while (lo < hi) {
        const int64_t mid = (lo + hi + 1) >> 1;
        if (spans[mid] <= start) lo = mid;
        else hi = mid - 1;
    }
    int64_t b0 = lo;
    for (uint64_t g0 = start; g0 < end; g0 += 32) {
        const uint64_t g = g0 + lane, gc = min(g, end - 1);
        const bool active = g < end;
        const int64_t nb = b0 + 1 + lane;
        const uint64_t bound = nb <= nbatches ? spans[nb] : ~0ull;   // the end of batch b0 + lane
        // c = the number of those ends at or before gc (they increase with the lane)
        int c = 0;
#pragma unroll
        for (int step = 16; step >= 1; step >>= 1)
            if (__shfl_sync(0xffffffffu, bound, c + step - 1) <= gc) c += step;
        // (every lane takes part in the shuffle: a full-mask shuffle that only some lanes reach is undefined)
        const uint64_t bound31 = __shfl_sync(0xffffffffu, bound, 31);
        if (c == 31 && bound31 <= gc) c = 32;
        int64_t b = b0 + c;
        // past the lookahead: batch b0 + 32 ends at or before gc, so batches without spans lie behind b0 and gc's batch is
        // the last one in [b0 + 33, nbatches - 1] whose first span is <= gc (spans[b0 + 33] <= gc < total, so b0 + 33 <
        // nbatches); without batches that lack spans this is never taken
        if (c == 32 && spans[b + 1] <= gc) {
            int64_t hi_b = nbatches - 1;
            for (b = b + 1; b < hi_b;) {
                const int64_t mid = (b + hi_b + 1) >> 1;
                if (spans[mid] <= gc) b = mid;
                else hi_b = mid - 1;
            }
        }
        uint32_t share = 0;
        if (active) {
            const uint64_t first = spans[b], n = spans[b + 1] - first, i = g - first;
            if (g >= first && i < n) {
                const uint64_t off = batch_off[b];
                const uint32_t len = 12u + be_u32(bytes + off + 8);
                const uint8_t *region = bytes + off + LOG_CRC_FROM;
                const uint8_t *e = region + (len - LOG_CRC_FROM) - (n - 1 - i) * LOG_CRC_SPAN;
                const uint8_t *a = i == 0 ? region : e - LOG_CRC_SPAN;
                share = crc_span(a, e, i == 0 ? 0xffffffffu : 0u, tl);
                const uint64_t k = n - 1 - i;   // spans behind this one
                if (k) {
                    uint32_t pw = __ldg(tables->pow_lo + (k & (LOG_CRC_POW_LO - 1)));
                    if (k >= (uint64_t)LOG_CRC_POW_LO) pw = crc32c_mulmod(pw, __ldg(tables->pow_hi + (k / LOG_CRC_POW_LO)));
                    share = crc32c_mulmod(share, pw);
                }
            }
        }
        // xor the shares of each batch's lanes (consecutive: b grows with the lane) into its last lane
        const int64_t key = active ? b : INT64_MAX;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
            const uint32_t t = __shfl_up_sync(0xffffffffu, share, d);
            const int64_t tk = __shfl_up_sync(0xffffffffu, key, d);
            if (lane >= d && tk == key) share ^= t;
        }
        const int64_t next_key = __shfl_down_sync(0xffffffffu, key, 1);
        if (active && (lane == 31 || next_key != key) && share) atomicXor(acc + b, share);
        b0 = __shfl_sync(0xffffffffu, b, 31);
    }
}

// The header pass's question for a framed batch: does the CRC that the span pass computed differ from the stored one?  A
// failure is listed in fails[] (capacity: the call's batches) and counted in the header word's crc_failed and
// crc_failed_bytes.
struct CrcAccCheck {
    const uint32_t *acc;
    LogCrcFail *fails;
    LogHeaderWord *word;
    __device__ __forceinline__ bool operator()(const uint8_t *p, uint32_t len, int64_t b, int32_t partition) const {
        const uint32_t stored = be_u32(p + 17), computed = acc[b] ^ 0xffffffffu;
        if (stored == computed) return false;
        const uint32_t slot = atomicAdd(&word->crc_failed, 1u);
        fails[slot] = LogCrcFail{(uint32_t)b, len, (int64_t)be_u64(p), partition, stored, computed, 0u};
        atomicAdd(&word->crc_failed_bytes, (unsigned long long)len);
        return true;
    }
};

}  // namespace kta
