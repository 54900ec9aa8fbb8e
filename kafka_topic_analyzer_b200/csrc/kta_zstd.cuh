// kta_zstd.cuh — Zstandard frames (RFC 8878): the records section of a Kafka record batch whose attributes name codec 4
// (zstd), which librdkafka decompresses inside poll before the handlers see a message (src/kafka.rs:93).  Used by
// log_zstd_size_kernel and log_decompress_kernel<true> (kta_logdecode.cuh), one warp per batch.
//
// Accepted: any number of frames, with or without Frame_Content_Size (one-shot compressors write it, streaming ones such as
// the Java client's do not), skippable frames among them, Raw / RLE / Compressed blocks, every literals and sequences mode.
// The Content_Checksum (XXH64) is skipped, not verified, like gzip's CRC32 (the batch CRC is, with check.crcs on).  Dictionaries
// (a non-zero Dictionary_ID) are rejected: Kafka does not use them.
//
// Shape (like kta_inflate.cuh): every lane of the warp reads the same headers and bitstreams (lane-uniform control flow,
// shared-memory tables read as broadcasts).  Of the FSE decode tables, lane t builds table t (LL, OF, ML); the Huffman table is
// filled by all lanes; the four streams of Huffman literals are decoded by lanes 0-3, one each, into the literal buffer at
// the block's output offset (a block's literals are at most its output, so they always fit); all lanes copy literals and
// matches.  The tables live in a per-warp ZstdWork that persists over the blocks of a frame (Repeat mode, Treeless
// literals) and is reset at each frame.
// The code is __host__ __device__ so that tests/test_zstd_host.py (through tests/native/codec_harness.cu, compiled by nvcc as
// a plain host program, one "lane") runs the same statements against pyarrow's zstd; the product only ever calls it on the
// device.
#pragma once
#include <stdint.h>

#include "kta_codec.cuh"

namespace kta {

constexpr uint32_t ZSTD_BLOCK_MAX = 128u * 1024u;

struct ZstdWork {            // per warp, in shared memory on the device
    uint32_t ll[512], ml[512], of[256];   // FSE decode tables: symbol | nbBits << 8 | baseline << 16
    uint32_t hwt[64];                     // FSE decode table of the Huffman weights
    uint16_t huf[2048];                   // Huffman decode table (<= 11 bits): symbol | nbBits << 8
    int16_t norm[3][64];                  // normalized counts of the tables being built
    uint16_t next[3][64];                 // per-symbol state counters while building
    uint8_t hw[256];                      // Huffman weights
    uint16_t rank[12][KTA_LANES];         // per lane: next Huffman table cell of each weight
};

__host__ __device__ __forceinline__ int zstd_hibit(uint32_t v) {   // v > 0
#ifdef __CUDA_ARCH__
    return 31 - __clz(v);
#else
    return 31 - __builtin_clz(v);
#endif
}

__host__ __device__ __forceinline__ uint32_t zstd_le(const uint8_t *p, int nb) {
    uint32_t v = 0;
    for (int i = 0; i < nb; i++) v |= (uint32_t)p[i] << (8 * i);
    return v;
}

// Backward bitstream (RFC 8878 4.1 / 4.2): the bits of the little-endian byte string p[0, n) below its last byte's highest set
// bit (the padding marker) are read from the top down.  pos = bits not yet read; bits below the start read as zeros and
// drive pos negative, which the callers check.
struct ZstdBits {
    const uint8_t *p;
    uint32_t n;
    int32_t pos;
};
__host__ __device__ inline bool zstd_bits_init(ZstdBits &s, const uint8_t *p, uint32_t n) {
    if (n == 0 || p[n - 1] == 0) return false;
    s.p = p;
    s.n = n;
    s.pos = (int32_t)(8u * (n - 1u)) + zstd_hibit(p[n - 1]);
    return true;
}
__host__ __device__ inline uint32_t zstd_bits_peek(const ZstdBits &s, int k) {   // k <= 32
    if (k == 0 || s.pos <= 0) return 0;
    const int32_t lo = s.pos - k;
    uint64_t v = 0;
    if (lo >= 0) {
        const uint32_t b0 = (uint32_t)lo >> 3, nb = s.n - b0 < 5u ? s.n - b0 : 5u;   // (lo & 7) + k <= 39 bits
        for (uint32_t j = 0; j < nb; j++) v |= (uint64_t)s.p[b0 + j] << (8 * j);
        return (uint32_t)((v >> (lo & 7)) & ((1ull << k) - 1ull));
    }
    for (int32_t j = 0; j < (s.pos + 7) >> 3; j++) v |= (uint64_t)s.p[j] << (8 * j);
    return (uint32_t)((v & ((1ull << s.pos) - 1ull)) << (-lo));
}
__host__ __device__ __forceinline__ uint32_t zstd_bits_read(ZstdBits &s, int k) {
    const uint32_t v = zstd_bits_peek(s, k);
    s.pos -= k;
    return v;
}

// FSE table description (RFC 8878 4.1.1), a forward little-endian bitstream in b[0, n): the normalized counts of symbols
// 0..nsym-1 (lane 0 writes them to norm) and the accuracy log.  used = bytes the description takes.
__host__ __device__ inline uint32_t zstd_fwd_peek(const uint8_t *b, uint32_t n, uint32_t bit, int k) {   // k <= 16, zeros past n
    uint32_t v = 0;
    for (uint32_t j = 0; j < 4u && (bit >> 3) + j < n; j++) v |= (uint32_t)b[(bit >> 3) + j] << (8 * j);
    return (v >> (bit & 7)) & ((1u << k) - 1u);
}
__host__ __device__ inline bool zstd_fse_norm(const uint8_t *b, uint32_t n, int max_al, int max_sym, int16_t *norm, int &al, int &nsym,
                                              uint32_t &used, int lane) {
    uint32_t bit = 0;
    al = (int)zstd_fwd_peek(b, n, 0, 4) + 5;
    bit = 4;
    if (al > max_al) return false;
    int remaining = 1 << al, sym = 0;
    while (remaining > 0) {
        if (sym > max_sym) return false;
        const int bits = zstd_hibit((uint32_t)remaining + 1u) + 1;
        uint32_t val = zstd_fwd_peek(b, n, bit, bits);
        const uint32_t lower = (1u << (bits - 1)) - 1u, threshold = (1u << bits) - 1u - (uint32_t)(remaining + 1);
        if ((val & lower) < threshold) {        // small values take one bit less
            val &= lower;
            bit += (uint32_t)bits - 1u;
        } else {
            if (val > lower) val -= threshold;
            bit += (uint32_t)bits;
        }
        const int proba = (int)val - 1;         // -1: "less than 1", one cell
        remaining -= proba < 0 ? -proba : proba;
        if (remaining < 0) return false;
        if (lane == 0) norm[sym] = (int16_t)proba;
        sym++;
        if (proba == 0) {                       // 2-bit repeat flags: more zero counts follow
            uint32_t rep;
            do {
                rep = zstd_fwd_peek(b, n, bit, 2);
                bit += 2;
                if (sym + (int)rep > max_sym + 1 || bit > 8u * n) return false;
                for (uint32_t r = 0; r < rep; r++) {
                    if (lane == 0) norm[sym] = 0;
                    sym++;
                }
            } while (rep == 3);
        }
        if (bit > 8u * n) return false;
    }
    nsym = sym;
    used = (bit + 7u) >> 3;
    return true;
}

// Decode table from normalized counts (RFC 8878 4.1.1, "FSE decoding table"), by ONE lane.  Cannot fail: zstd_fse_norm
// guarantees the counts fill the table exactly.
__host__ __device__ inline void zstd_fse_build(uint32_t *dt, const int16_t *norm, int nsym, int al, uint16_t *next) {
    const uint32_t size = 1u << al, mask = size - 1u, step = (size >> 1) + (size >> 3) + 3u;
    uint32_t high = size;
    for (int s = 0; s < nsym; s++)
        if (norm[s] == -1) {                    // "less than 1" symbols: one cell each, from the end of the table
            dt[--high] = (uint32_t)s;
            next[s] = 1;
        }
    uint32_t pos = 0;
    for (int s = 0; s < nsym; s++) {
        if (norm[s] <= 0) continue;
        next[s] = (uint16_t)norm[s];
        for (int i = 0; i < norm[s]; i++) {
            dt[pos] = (uint32_t)s;
            do pos = (pos + step) & mask;
            while (pos >= high);
        }
    }
    for (uint32_t i = 0; i < size; i++) {
        const uint32_t s = dt[i] & 0xffu, d = next[s]++;
        const uint32_t nb = (uint32_t)al - (uint32_t)zstd_hibit(d);
        dt[i] = s | (nb << 8) | (((d << nb) - size) << 16);
    }
}

// The predefined distributions (RFC 8878 3.1.1.3.2.2), as characters 'a' + count + 1
__host__ __device__ __forceinline__ const char *zstd_predefined(int t) {
    return t == 0 ? "fedddddddddddcccdddddddddedcccccaaaa"                     // literal lengths, accuracy 6
         : t == 1 ? "ccccccdddcccccccccccccccaaaaa"                            // offsets, accuracy 5 (29 codes)
                  : "cfeddddddcccccccccccccccccccccccccccccccccccccaaaaaaa";    // match lengths, accuracy 6
}

// Literal length and match length codes (RFC 8878 3.1.1.3.2.1.1): extra bits and baseline, in closed form
__host__ __device__ __forceinline__ int zstd_ll_bits(uint32_t c) {
    return c < 16 ? 0 : c < 20 ? 1 : c < 22 ? 2 : c < 24 ? 3 : c == 24 ? 4 : c == 25 ? 6 : (int)c - 19;
}
__host__ __device__ __forceinline__ uint32_t zstd_ll_base(uint32_t c) {
    return c < 16 ? c : c < 20 ? 16u + 2u * (c - 16u) : c < 22 ? 24u + 4u * (c - 20u) : c < 24 ? 32u + 8u * (c - 22u) : c == 24 ? 48u : c == 25 ? 64u
                                                                                                                                        : 1u << (c - 19u);
}
__host__ __device__ __forceinline__ int zstd_ml_bits(uint32_t c) {
    return c < 32 ? 0 : c < 36 ? 1 : c < 38 ? 2 : c < 40 ? 3 : c < 42 ? 4 : c == 42 ? 5 : (int)c - 36;
}
__host__ __device__ __forceinline__ uint32_t zstd_ml_base(uint32_t c) {
    return c < 32 ? c + 3u : c < 36 ? 35u + 2u * (c - 32u) : c < 38 ? 43u + 4u * (c - 36u) : c < 40 ? 51u + 8u * (c - 38u) : c < 42 ? 67u + 16u * (c - 40u)
         : c == 42                                                                                                          ? 99u
                                                                                                                             : (1u << (c - 36u)) + 3u;
}

// What persists over the blocks of one frame besides the tables (every lane holds the same copy)
struct ZstdFrame {
    uint64_t op;             // output position (bytes written by all frames so far)
    uint64_t start;          // op at the start of this frame: matches may not reach before it
    uint32_t bmax;           // Block_Maximum_Size = min(Window_Size, 128 KiB)
    uint32_t rep0, rep1, rep2;
    int al[3];               // accuracy logs of the LL, OF, ML tables
    int kind[3];             // 0 none yet, 1 predefined, 2 from this frame's data
    int huf_bits;            // Huffman table log, 0 = no table yet
};

// Huffman tree description (RFC 8878 4.2.1) at b[0, cs) → w.huf; q = bytes it takes.
__host__ __device__ inline bool zstd_huf_table(const uint8_t *b, uint32_t cs, uint32_t &q, ZstdWork &w, ZstdFrame &f, int lane) {
    if (cs < 1) return false;
    const uint32_t hb = b[0];
    uint32_t nw = 0;
    KTA_LANE_SYNC();   // every lane is done with the previous table and weights
    if (hb >= 128) {  // direct: 4 bits per weight
        nw = hb - 127u;
        const uint32_t nb = (nw + 1u) >> 1;
        if (nb > cs - 1u) return false;
        if (lane == 0)
            for (uint32_t i = 0; i < nw; i++) w.hw[i] = (i & 1u) ? (b[1 + i / 2] & 15u) : (b[1 + i / 2] >> 4);
        q = 1u + nb;
    } else {          // FSE-compressed weights: hb bytes, two interleaved states
        if (hb > cs - 1u) return false;
        int al, nsym;
        uint32_t used;
        if (!zstd_fse_norm(b + 1, hb, 6, 12, w.norm[0], al, nsym, used, lane)) return false;
        KTA_LANE_SYNC();
        if (lane == 0) zstd_fse_build(w.hwt, w.norm[0], nsym, al, w.next[0]);
        KTA_LANE_SYNC();
        ZstdBits s;
        if (used > hb || !zstd_bits_init(s, b + 1 + used, hb - used)) return false;
        uint32_t s1 = zstd_bits_read(s, al), s2 = zstd_bits_read(s, al);
        if (s.pos < 0) return false;
        // decoding ends when a state update reads past the start: then the other state yields its last symbol
        for (;;) {
            if (nw >= 255u) return false;
            uint32_t e = w.hwt[s1];
            if (lane == 0) w.hw[nw] = (uint8_t)e;
            nw++;
            s1 = (e >> 16) + zstd_bits_read(s, (int)((e >> 8) & 0xffu));
            if (s.pos < 0) {
                if (nw >= 255u) return false;
                if (lane == 0) w.hw[nw] = (uint8_t)w.hwt[s2];
                nw++;
                break;
            }
            if (nw >= 255u) return false;
            e = w.hwt[s2];
            if (lane == 0) w.hw[nw] = (uint8_t)e;
            nw++;
            s2 = (e >> 16) + zstd_bits_read(s, (int)((e >> 8) & 0xffu));
            if (s.pos < 0) {
                if (nw >= 255u) return false;
                if (lane == 0) w.hw[nw] = (uint8_t)w.hwt[s1];
                nw++;
                break;
            }
        }
        q = 1u + hb;
    }
    KTA_LANE_SYNC();
    // the last weight is implied: the weights' powers of two must add up to the next power of two
    uint32_t total = 0;
    for (uint32_t i = 0; i < nw; i++) {
        const uint32_t x = w.hw[i];
        if (x > 11u) return false;
        if (x) total += 1u << (x - 1u);
    }
    if (total == 0) return false;
    const int bits = zstd_hibit(total) + 1;
    if (bits > 11) return false;
    const uint32_t rest = (1u << bits) - total;
    if (rest & (rest - 1u)) return false;
    if (lane == 0) w.hw[nw] = (uint8_t)(zstd_hibit(rest) + 1);
    KTA_LANE_SYNC();
    // table: the symbols of weight x fill 2^(x-1) cells each, weight 1 first, symbols in order within a weight
    uint16_t *start = &w.rank[0][lane];   // start[x * KTA_LANES]: this lane's copy, no bank conflicts
    for (int x = 0; x < 12; x++) start[x * KTA_LANES] = 0;
    for (uint32_t i = 0; i <= nw; i++) start[w.hw[i] * KTA_LANES]++;
    uint32_t at = 0;
    for (int x = 1; x <= bits; x++) {
        const uint32_t c = (uint32_t)start[x * KTA_LANES] << (x - 1);
        start[x * KTA_LANES] = (uint16_t)at;
        at += c;
    }
    for (uint32_t i = 0; i <= nw; i++) {
        const uint32_t x = w.hw[i];
        if (!x) continue;
        const uint32_t a = start[x * KTA_LANES], len = 1u << (x - 1u);
        start[x * KTA_LANES] = (uint16_t)(a + len);
        const uint16_t e = (uint16_t)(i | ((uint32_t)(bits + 1 - (int)x) << 8));
        for (uint32_t j = a + (((uint32_t)lane - a) & (KTA_LANES - 1u)); j < a + len; j += KTA_LANES) w.huf[j] = e;
    }
    f.huf_bits = bits;
    KTA_LANE_SYNC();
    return true;
}

// one Huffman-coded stream of cnt literals → dst (one lane)
__host__ __device__ inline bool zstd_huf_stream(const uint8_t *src, uint32_t len, uint8_t *dst, uint32_t cnt, const uint16_t *tab, int bits) {
    ZstdBits s;
    if (!zstd_bits_init(s, src, len)) return false;
    for (uint32_t i = 0; i < cnt; i++) {
        const uint32_t e = tab[zstd_bits_peek(s, bits)];
        s.pos -= (int32_t)(e >> 8);
        if (s.pos < 0) return false;
        dst[i] = (uint8_t)e;
    }
    return s.pos == 0;
}

// One Compressed_Block (RFC 8878 3.1.1.3) in b[0, bs).  COPY: literals to lit + f.op, output to out + f.op (cap bytes in both);
// otherwise only f.op advances (the literals are not decoded).
template <bool COPY>
__host__ __device__ inline bool zstd_block(const uint8_t *b, uint32_t bs, uint8_t *out, uint8_t *lit, uint64_t cap, ZstdWork &w, ZstdFrame &f,
                                           int lane) {
    // --- literals section
    if (bs < 1) return false;
    const uint32_t lt = b[0] & 3u, sf = (b[0] >> 2) & 3u;
    uint32_t hl, rs, cs = 0, nstreams = 1;
    if (lt < 2) {                           // Raw / RLE
        hl = (sf & 1u) == 0 ? 1u : sf == 1 ? 2u : 3u;
        if (bs < hl) return false;
        rs = hl == 1 ? (uint32_t)b[0] >> 3 : zstd_le(b, (int)hl) >> 4;
    } else {                                // Huffman-compressed / Treeless
        hl = sf < 2 ? 3u : sf + 2u;
        if (bs < hl) return false;
        const int fb = sf < 2 ? 10 : sf == 2 ? 14 : 18;
        const uint64_t h = (uint64_t)zstd_le(b, hl < 4 ? (int)hl : 4) | (hl == 5 ? (uint64_t)b[4] << 32 : 0ull);
        rs = (uint32_t)(h >> 4) & ((1u << fb) - 1u);
        cs = (uint32_t)(h >> (4 + fb)) & ((1u << fb) - 1u);
        nstreams = sf == 0 ? 1u : 4u;
    }
    if (rs > f.bmax || (COPY && rs > cap - f.op)) return false;
    uint32_t q = hl;
    const uint8_t *lits = COPY ? lit + f.op : nullptr;
    if (lt == 0) {
        if (rs > bs - q) return false;
        lits = b + q;
        q += rs;
    } else if (lt == 1) {
        if (q >= bs) return false;
        if (COPY)
            for (uint32_t i = lane; i < rs; i += KTA_LANES) lit[f.op + i] = b[q];
        q += 1;
    } else {
        if (cs > bs - q) return false;
        if (COPY) {
            uint32_t t = 0;
            if (lt == 2 && !zstd_huf_table(b + q, cs, t, w, f, lane)) return false;
            if (f.huf_bits == 0) return false;   // Treeless without an earlier table in this frame
            const uint8_t *src = b + q + t;
            const uint32_t avail = cs - t;
            bool ok;
            if (nstreams == 1) {
                ok = true;
                if (lane == 0) ok = zstd_huf_stream(src, avail, lit + f.op, rs, w.huf, f.huf_bits);
            } else {
                const uint32_t seg = (rs + 3u) >> 2;
                if (avail < 6u || rs < 3u * seg) return false;
                const uint32_t l0 = zstd_le(src, 2), l1 = zstd_le(src + 2, 2), l2 = zstd_le(src + 4, 2);
                if ((uint64_t)l0 + l1 + l2 > avail - 6u) return false;
                const uint32_t l3 = avail - 6u - l0 - l1 - l2;
                ok = true;
#pragma unroll
                for (int k = 0; k < 4; k++) {
                    if (KTA_LANES > 1 && lane != k) continue;
                    const uint32_t off = 6u + (k > 0 ? l0 : 0u) + (k > 1 ? l1 : 0u) + (k > 2 ? l2 : 0u);
                    const uint32_t len = k == 0 ? l0 : k == 1 ? l1 : k == 2 ? l2 : l3;
                    ok = zstd_huf_stream(src + off, len, lit + f.op + (uint64_t)k * seg, k < 3 ? seg : rs - 3u * seg, w.huf, f.huf_bits) && ok;
                }
            }
            if (!lanes_all(ok)) return false;
        } else if (lt == 2) f.huf_bits = 1;     // (the size pass only notes that a table exists)
        else if (f.huf_bits == 0) return false;
        q += cs;
    }
    KTA_LANE_SYNC();   // the literals are in the buffer
    // --- sequences section
    if (q >= bs) return false;
    uint32_t nseq = b[q++];
    if (nseq >= 128u) {
        if (nseq < 255u) {
            if (q >= bs) return false;
            nseq = ((nseq - 128u) << 8) + b[q++];
        } else {
            if (bs - q < 2u) return false;
            nseq = zstd_le(b + q, 2) + 0x7f00u;
            q += 2;
        }
    }
    const uint64_t bstart = f.op;
    uint32_t lit_pos = 0;
    if (nseq > 0) {
        if (q >= bs) return false;
        const uint32_t modes = b[q++];
        if (modes & 3u) return false;
        KTA_LANE_SYNC();   // every lane is done with the previous block's tables
        uint32_t build = 0;
        int nsym[3] = {0, 0, 0};
#pragma unroll
        for (int t = 0; t < 3; t++) {       // LL, OF, ML
            const uint32_t mode = (modes >> (6 - 2 * t)) & 3u;
            const int max_sym = t == 0 ? 35 : t == 1 ? 31 : 52, max_al = t == 1 ? 8 : 9;
            if (mode == 0) {                // Predefined (kept while the next blocks keep it)
                if (f.kind[t] != 1) {
                    const char *d = zstd_predefined(t);
                    nsym[t] = t == 0 ? 36 : t == 1 ? 29 : 53;
                    if (lane == 0)
                        for (int i = 0; i < nsym[t]; i++) w.norm[t][i] = (int16_t)(d[i] - 'a' - 1);
                    f.al[t] = t == 1 ? 5 : 6;
                    f.kind[t] = 1;
                    build |= 1u << t;
                }
            } else if (mode == 1) {         // RLE: one symbol, no state bits
                if (q >= bs || b[q] > (uint32_t)max_sym) return false;
                if (lane == 0) w.norm[t][0] = (int16_t)b[q];
                q++;
                nsym[t] = 0;
                f.al[t] = 0;
                f.kind[t] = 2;
                build |= 1u << t;
            } else if (mode == 2) {         // FSE_Compressed
                uint32_t used;
                if (!zstd_fse_norm(b + q, bs - q, max_al, max_sym, w.norm[t], f.al[t], nsym[t], used, lane)) return false;
                q += used;
                f.kind[t] = 2;
                build |= 1u << t;
            } else if (f.kind[t] == 0) return false;   // Repeat, but nothing to repeat
        }
        KTA_LANE_SYNC();
#pragma unroll
        for (int t = 0; t < 3; t++) {       // lane t builds table t
            if (!((build >> t) & 1u) || (KTA_LANES > 1 && lane != t)) continue;
            uint32_t *dt = t == 0 ? w.ll : t == 1 ? w.of : w.ml;
            if (nsym[t] == 0) dt[0] = (uint32_t)w.norm[t][0];   // RLE
            else zstd_fse_build(dt, w.norm[t], nsym[t], f.al[t], w.next[t]);
        }
        KTA_LANE_SYNC();
        // the interleaved bitstream: initial states LL, OF, ML; per sequence the OF, ML, LL extra bits, then the LL, ML, OF
        // state updates (none after the last sequence)
        ZstdBits s;
        if (!zstd_bits_init(s, b + q, bs - q)) return false;
        uint32_t sll = zstd_bits_read(s, f.al[0]), sof = zstd_bits_read(s, f.al[1]), sml = zstd_bits_read(s, f.al[2]);
        for (uint32_t i = 0; i < nseq; i++) {
            const uint32_t ell = w.ll[sll], eof = w.of[sof], eml = w.ml[sml];
            const uint32_t ofc = eof & 0xffu, mlc = eml & 0xffu, llc = ell & 0xffu;
            const uint32_t ov = (1u << ofc) + zstd_bits_read(s, (int)ofc);
            const uint32_t ml = zstd_ml_base(mlc) + zstd_bits_read(s, zstd_ml_bits(mlc));
            const uint32_t ll = zstd_ll_base(llc) + zstd_bits_read(s, zstd_ll_bits(llc));
            if (i + 1 < nseq) {
                sll = (ell >> 16) + zstd_bits_read(s, (int)((ell >> 8) & 0xffu));
                sml = (eml >> 16) + zstd_bits_read(s, (int)((eml >> 8) & 0xffu));
                sof = (eof >> 16) + zstd_bits_read(s, (int)((eof >> 8) & 0xffu));
            }
            if (s.pos < 0) return false;
            // repeat offsets (RFC 8878 3.1.1.5): values 1-3 name rep0..2, shifted by one when the literal length is 0
            uint32_t offset;
            if (ov > 3u) {
                offset = ov - 3u;
                f.rep2 = f.rep1;
                f.rep1 = f.rep0;
                f.rep0 = offset;
            } else {
                const uint32_t idx = ov - 1u + (ll == 0 ? 1u : 0u);
                if (idx == 0) offset = f.rep0;
                else {
                    offset = idx == 1 ? f.rep1 : idx == 2 ? f.rep2 : f.rep0 - 1u;
                    if (idx != 1) f.rep2 = f.rep1;
                    f.rep1 = f.rep0;
                    f.rep0 = offset;
                }
            }
            if (ll > rs - lit_pos || (uint64_t)ll + ml > (uint64_t)f.bmax - (f.op - bstart)) return false;
            if (COPY && (uint64_t)ll + ml > cap - f.op) return false;
            lz_emit_literals<COPY>(out, f.op, lits + lit_pos, ll, lane);
            f.op += ll;
            lit_pos += ll;
            if (offset == 0 || offset > f.op - f.start) return false;
            lz_emit_match<COPY>(out, f.op, offset, ml, lane);
            f.op += ml;
        }
        if (s.pos != 0) return false;         // the bitstream must be consumed exactly
    } else if (q != bs) return false;
    const uint32_t left = rs - lit_pos;
    if ((uint64_t)left > (uint64_t)f.bmax - (f.op - bstart) || (COPY && left > cap - f.op)) return false;
    lz_emit_literals<COPY>(out, f.op, lits + lit_pos, left, lane);
    f.op += left;
    KTA_LANE_SYNC();   // the block's output is complete before the next block reads it
    return true;
}

// The records section in[0, n): one or more zstd frames, skippable frames among them.  COPY: the whole warp calls this
// (lane-uniform control flow) and writes out[0, out_cap) and lit[0, out_cap).  Without COPY it computes the size: a frame's
// Frame_Content_Size when it has one (bounded by what its block headers allow: a forged field must not size the scratch
// buffer), otherwise by decoding the frame's sequences (lengths only, nothing is copied).
template <bool COPY>
__host__ __device__ LzWalk zstd_walk(const uint8_t *in, uint32_t n, uint8_t *out, uint8_t *lit, uint64_t out_cap, ZstdWork &w, int lane) {
    LzWalk r{0, false};
    if (n == 0) return r;
    uint32_t p = 0;
    while (p < n) {
        if (n - p < 4u) return r;
        const uint32_t magic = zstd_le(in + p, 4);
        if ((magic & 0xfffffff0u) == 0x184d2a50u) {   // skippable frame
            if (n - p < 8u) return r;
            const uint32_t sz = zstd_le(in + p + 4, 4);
            p += 8;
            if (sz > n - p) return r;
            p += sz;
            continue;
        }
        if (magic != 0xfd2fb528u) return r;
        p += 4;
        if (p >= n) return r;
        const uint32_t fhd = in[p++];
        if (fhd & 8u) return r;                        // reserved bit
        const bool single = (fhd >> 5) & 1u, checksum = (fhd >> 2) & 1u;
        uint64_t window = 0;
        if (!single) {
            if (p >= n) return r;
            const uint32_t wd = in[p++];
            const uint64_t base = 1ull << (10u + (wd >> 3));
            window = base + (base >> 3) * (wd & 7u);
        }
        const uint32_t did_bytes = (fhd & 3u) == 3u ? 4u : fhd & 3u;
        if (n - p < did_bytes) return r;
        if (zstd_le(in + p, (int)did_bytes) != 0) return r;   // dictionaries are not used by Kafka
        p += did_bytes;
        const uint32_t fcs_code = fhd >> 6, fcs_bytes = fcs_code == 0 ? (single ? 1u : 0u) : 1u << fcs_code;
        if (n - p < fcs_bytes) return r;
        uint64_t fcs = 0;
        for (uint32_t i = 0; i < fcs_bytes; i++) fcs |= (uint64_t)in[p + i] << (8 * i);
        if (fcs_bytes == 2) fcs += 256;
        p += fcs_bytes;
        if (single) window = fcs;
        ZstdFrame f{};
        f.op = f.start = r.out_len;
        f.bmax = (uint32_t)(window < ZSTD_BLOCK_MAX ? window : ZSTD_BLOCK_MAX);
        f.rep0 = 1;
        f.rep1 = 4;
        f.rep2 = 8;
        const bool sized = !COPY && fcs_bytes > 0;    // size pass: the field, checked against the block headers
        uint64_t bound = 0;
        for (;;) {
            if (n - p < 3u) return r;
            const uint32_t bh = zstd_le(in + p, 3), bt = (bh >> 1) & 3u, bsz = bh >> 3;
            p += 3;
            if (bt == 3u || bsz > f.bmax) return r;   // reserved type; a block larger than the window or 128 KiB
            if (bt == 1u) {                           // RLE: one byte repeated bsz times
                if (p >= n) return r;
                if (COPY) {
                    if (bsz > out_cap - f.op) return r;
                    for (uint32_t i = lane; i < bsz; i += KTA_LANES) out[f.op + i] = in[p];
                }
                f.op += bsz;
                bound += bsz;
                p += 1;
            } else {
                if (bsz > n - p) return r;
                if (bt == 0u) {                       // Raw
                    if (COPY && bsz > out_cap - f.op) return r;
                    lz_emit_literals<COPY>(out, f.op, in + p, bsz, lane);
                    f.op += bsz;
                    bound += bsz;
                } else if (sized) bound += f.bmax;
                else if (!zstd_block<COPY>(in + p, bsz, out, lit, out_cap, w, f, lane)) return r;
                p += bsz;
            }
            if (bh & 1u) break;                       // Last_Block
        }
        if (checksum) {                               // Content_Checksum: skipped, not verified
            if (n - p < 4u) return r;
            p += 4;
        }
        if (sized) {
            if (fcs > bound) return r;
            r.out_len += fcs;
        } else {
            if (fcs_bytes > 0 && f.op - f.start != fcs) return r;
            r.out_len = f.op;
        }
        KTA_LANE_SYNC();
    }
    r.ok = true;
    return r;
}

}  // namespace kta
