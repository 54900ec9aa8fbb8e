// kta_inflate.cuh — DEFLATE (RFC 1951) inside a gzip member (RFC 1952): the records section of a Kafka record batch whose
// attributes name codec 1 (gzip), which librdkafka inflates inside poll before the handlers see a message
// (src/kafka.rs:93).  Used by log_unc_size_kernel (gzip_size) and log_decompress_kernel (gzip_walk) in kta_logdecode.cuh,
// one warp per batch for the copy.
//
// Shape: every lane of the warp walks the same bit stream (lane-uniform control flow, shared-memory tables read as
// broadcasts); lane 0 alone writes tables and literals, all 32 lanes copy the bytes of a match.  Huffman codes are decoded
// canonically, one bit at a time against the per-length code counts (the tables are 16 counts + the symbols in code order:
// no lookup tables to build per block) — a batch is a few thousand symbols, and thousands of batches decode side by side.
// The code is __host__ __device__ so that tests/test_inflate_host.py and tests/test_lzwalk_host.py (through
// tests/native/codec_harness.cu, compiled by nvcc as a plain host program, one lane) run the same statements against zlib's
// output; the product only ever calls it on the device.
#pragma once
#include <stdint.h>

#include "kta_codec.cuh"

namespace kta {

struct InfBits {
    const uint8_t *p;
    uint32_t n, pos;
    uint64_t buf;
    int cnt;
    bool bad;   // ran past the end of the input
};

__host__ __device__ inline uint32_t inf_bits(InfBits &s, int need) {   // need <= 16; bits come LSB first (RFC 1951 3.1.1)
    while (s.cnt < need) {
        if (s.pos >= s.n) {
            s.bad = true;
            return 0;
        }
        s.buf |= (uint64_t)s.p[s.pos++] << s.cnt;
        s.cnt += 8;
    }
    const uint32_t v = (uint32_t)s.buf & ((1u << need) - 1u);
    s.buf >>= need;
    s.cnt -= need;
    return v;
}

// canonical Huffman code: count[l] = codes of length l, symbol[] = the symbols ordered by (length, value);
// fast[] = direct lookup by the next INF_FAST_BITS bits of the stream for the codes that short: symbol | length << 12,
// 0 = a longer code (or none): decode bit by bit
constexpr int INF_FAST_BITS = 9;
struct InfHuff {
    uint16_t *count;    // [16]
    uint16_t *symbol;
    uint16_t *fast;     // [1 << INF_FAST_BITS], or nullptr (the code-length code: 19 symbols, used a few dozen times)
};

struct InfWork {        // per warp, in shared memory on the device
    uint16_t lencnt[16], lensym[288], distcnt[16], distsym[32], lengths[320], offs[16];
    uint16_t lenfast[1 << INF_FAST_BITS], distfast[1 << INF_FAST_BITS];
};

// Huffman codes are packed MSB first (RFC 1951 3.1.1): extend the code bit by bit until it falls into the range of codes
// of its length.  Returns the symbol, or -1 (no such code / out of input).
__host__ __device__ inline int inf_decode(InfBits &s, const InfHuff &h) {
    // look at up to 15 bits at once (the buffer is topped up a byte at a time; near the end of the input fewer are there)
    while (s.cnt <= 48 && s.pos < s.n) {
        s.buf |= (uint64_t)s.p[s.pos++] << s.cnt;
        s.cnt += 8;
    }
    if (h.fast) {
        const uint32_t e = h.fast[(uint32_t)s.buf & ((1u << INF_FAST_BITS) - 1u)];
        const int len = (int)(e >> 12);
        if (e != 0 && len <= s.cnt) {
            s.buf >>= len;
            s.cnt -= len;
            return (int)(e & 0xfffu);
        }
    }
    uint32_t bits = (uint32_t)s.buf;
    int code = 0, first = 0, index = 0;
    for (int len = 1; len <= 15; len++) {
        code |= (int)(bits & 1u);
        bits >>= 1;
        const int count = h.count[len];
        if (code - count < first) {
            if (len > s.cnt) break;   // the code runs past the end of the input
            s.buf >>= len;
            s.cnt -= len;
            return h.symbol[index + (code - first)];
        }
        index += count;
        first += count;
        first <<= 1;
        code <<= 1;
    }
    s.bad = s.bad || s.cnt < 15;
    return -1;
}

// Build the decoding tables from n code lengths (0 = symbol unused).  Returns 0 for a complete code, > 0 for an
// incomplete one (codes left over), < 0 for an over-subscribed one.  count / symbol are written by lane 0, the lookup
// table by all lanes.
__host__ __device__ inline int inf_construct(InfHuff &h, const uint16_t *length, int n, uint16_t *offs, int lane) {
    if (lane == 0) {
        for (int l = 0; l <= 15; l++) h.count[l] = 0;
        for (int i = 0; i < n; i++) h.count[length[i]]++;
    }
    KTA_LANE_SYNC();
    if (h.fast) {   // no entry of an earlier block's code may survive
        for (int i = lane; i < (1 << INF_FAST_BITS); i += KTA_LANES) h.fast[i] = 0;
        KTA_LANE_SYNC();
    }
    if (h.count[0] == n) return 0;   // no codes at all: complete, but decoding anything will fail
    int left = 1;
    for (int l = 1; l <= 15; l++) {
        left <<= 1;
        left -= h.count[l];
        if (left < 0) return left;
    }
    if (lane == 0) {
        offs[1] = 0;
        for (int l = 1; l < 15; l++) offs[l + 1] = offs[l] + h.count[l];
        for (int i = 0; i < n; i++)
            if (length[i] != 0) h.symbol[offs[length[i]]++] = (uint16_t)i;
    }
    KTA_LANE_SYNC();
    if (h.fast) {
        // the lookup table: the code of the j-th symbol of length l is first_l + j (canonical order), sent MSB first, so
        // it occupies the LOW l bits of the look-ahead in reversed order; every setting of the bits above it maps to it
        int first = 0, index = 0;
        for (int l = 1; l <= INF_FAST_BITS; l++) {
            const int count = h.count[l];
            for (int j = lane; j < count; j += KTA_LANES) {
                uint32_t code = (uint32_t)(first + j), rev = 0;
                for (int b = 0; b < l; b++) {
                    rev = (rev << 1) | (code & 1u);
                    code >>= 1;
                }
                const uint16_t e = (uint16_t)(h.symbol[index + j] | (l << 12));
                for (uint32_t k = rev; k < (1u << INF_FAST_BITS); k += 1u << l) h.fast[k] = e;
            }
            index += count;
            first = (first + count) << 1;
        }
        KTA_LANE_SYNC();
    }
    return left;
}

// Output policy Out (InfOut below):  bool lit(uint8_t)  |  bool match(uint32_t dist, uint32_t len)  |  bool stored(const uint8_t *,
// uint32_t), each returning false when the output would overflow or a distance reaches before the start.

// length / distance symbols, RFC 1951 3.2.5, in closed form (no tables in local memory): a length symbol s = 0..28 (code
// 257 + s) carries e = (s - 4) / 4 extra bits from s = 8 on and starts at 3 + ((4 + s % 4) << e); a distance symbol s = 0..29
// carries e = (s - 2) / 2 extra bits from s = 4 on and starts at 1 + ((2 + s % 2) << e).
__host__ __device__ inline int inf_len_extra(int s) { return s < 8 || s == 28 ? 0 : (s - 4) >> 2; }
__host__ __device__ inline uint32_t inf_len_base(int s) {
    return s < 8 ? 3u + (uint32_t)s : s == 28 ? 258u : 3u + ((4u + ((uint32_t)s & 3u)) << inf_len_extra(s));
}
__host__ __device__ inline int inf_dist_extra(int s) { return s < 4 ? 0 : (s - 2) >> 1; }
__host__ __device__ inline uint32_t inf_dist_base(int s) {
    return s < 4 ? 1u + (uint32_t)s : 1u + ((2u + ((uint32_t)s & 1u)) << inf_dist_extra(s));
}

template <class Out>
__host__ __device__ inline bool inf_codes(InfBits &s, Out &out, const InfHuff &lencode, const InfHuff &distcode) {
    for (;;) {
        int sym = inf_decode(s, lencode);
        if (sym < 0) return false;
        if (sym < 256) {
            if (!out.lit((uint8_t)sym)) return false;
        } else if (sym == 256) {
            return true;   // end of block
        } else {
            sym -= 257;
            if (sym >= 29) return false;
            const uint32_t len = inf_len_base(sym) + inf_bits(s, inf_len_extra(sym));
            const int ds = inf_decode(s, distcode);
            if (ds < 0 || ds >= 30) return false;
            const uint32_t dist = inf_dist_base(ds) + inf_bits(s, inf_dist_extra(ds));
            if (s.bad || !out.match(dist, len)) return false;
        }
    }
}

// The deflate stream at s (positioned on its first block header) up to and including the final block.
template <class Out>
__host__ __device__ inline bool inf_stream(InfBits &s, Out &out, InfWork &w, int lane) {
    InfHuff lencode{w.lencnt, w.lensym, w.lenfast}, distcode{w.distcnt, w.distsym, w.distfast};
    InfHuff clcode{w.lencnt, w.lensym, nullptr};   // the code-length code borrows the literal code's arrays
    for (;;) {
        const uint32_t last = inf_bits(s, 1), type = inf_bits(s, 2);
        if (s.bad) return false;
        if (type == 0) {
            // stored: skip to the byte boundary (whole bytes the decoder looked ahead at go back), LEN, ~LEN, bytes
            s.pos -= (uint32_t)(s.cnt >> 3);
            s.buf = 0;
            s.cnt = 0;
            if (s.pos + 4 > s.n) return false;
            const uint32_t len = (uint32_t)s.p[s.pos] | ((uint32_t)s.p[s.pos + 1] << 8);
            const uint32_t nlen = (uint32_t)s.p[s.pos + 2] | ((uint32_t)s.p[s.pos + 3] << 8);
            s.pos += 4;
            if ((len ^ nlen) != 0xffffu || len > s.n - s.pos) return false;
            if (!out.stored(s.p + s.pos, len)) return false;
            s.pos += len;
        } else if (type == 1 || type == 2) {
            KTA_LANE_SYNC();   // every lane is done with the previous block's tables
            if (type == 1) {
                // fixed codes (RFC 1951 3.2.6)
                if (lane == 0) {
                    for (int i = 0; i < 144; i++) w.lengths[i] = 8;
                    for (int i = 144; i < 256; i++) w.lengths[i] = 9;
                    for (int i = 256; i < 280; i++) w.lengths[i] = 7;
                    for (int i = 280; i < 288; i++) w.lengths[i] = 8;
                }
                KTA_LANE_SYNC();
                inf_construct(lencode, w.lengths, 288, w.offs, lane);
                KTA_LANE_SYNC();
                if (lane == 0)
                    for (int i = 0; i < 30; i++) w.lengths[i] = 5;
                KTA_LANE_SYNC();
                inf_construct(distcode, w.lengths, 30, w.offs, lane);
            } else {
                // dynamic codes (RFC 1951 3.2.7): the code lengths are themselves Huffman coded
                const int nlen = (int)inf_bits(s, 5) + 257, ndist = (int)inf_bits(s, 5) + 1, ncode = (int)inf_bits(s, 4) + 4;
                if (s.bad || nlen > 286 || ndist > 30) return false;
                const uint8_t order[19] = {16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15};
                {
                    uint16_t cl[19];   // every lane reads the same bits; lane 0 stores them
                    for (int i = 0; i < 19; i++) cl[i] = 0;
                    for (int i = 0; i < ncode; i++) cl[order[i]] = (uint16_t)inf_bits(s, 3);
                    if (s.bad) return false;
                    if (lane == 0)
                        for (int i = 0; i < 19; i++) w.lengths[i] = cl[i];
                }
                KTA_LANE_SYNC();
                if (inf_construct(clcode, w.lengths, 19, w.offs, lane) != 0) return false;   // the code-length code must be complete
                KTA_LANE_SYNC();
                // the nlen + ndist lengths; they go to a second array (the code-length code's own lengths are still in use
                // through lencode's tables only, so w.lengths may be overwritten now)
                int index = 0;
                uint32_t prev = 0;
                while (index < nlen + ndist) {
                    const int sym = inf_decode(s, clcode);
                    if (sym < 0) return false;
                    uint32_t val = 0;
                    int rep = 1;
                    if (sym < 16) {
                        val = (uint32_t)sym;
                    } else if (sym == 16) {
                        if (index == 0) return false;
                        val = prev;
                        rep = 3 + (int)inf_bits(s, 2);
                    } else if (sym == 17) {
                        rep = 3 + (int)inf_bits(s, 3);
                    } else {
                        rep = 11 + (int)inf_bits(s, 7);
                    }
                    if (s.bad || index + rep > nlen + ndist) return false;
                    if (lane == 0)
                        for (int r = 0; r < rep; r++) w.lengths[index + r] = (uint16_t)val;
                    index += rep;
                    prev = val;
                }
                KTA_LANE_SYNC();
                if (w.lengths[256] == 0) return false;   // no end-of-block code
                // an incomplete code is allowed only when it is a single code of length 1 (RFC 1951 as zlib reads it)
                int err = inf_construct(lencode, w.lengths, nlen, w.offs, lane);
                if (err < 0 || (err > 0 && nlen != lencode.count[0] + lencode.count[1])) return false;
                KTA_LANE_SYNC();
                err = inf_construct(distcode, w.lengths + nlen, ndist, w.offs, lane);
                if (err < 0 || (err > 0 && ndist != distcode.count[0] + distcode.count[1])) return false;
            }
            KTA_LANE_SYNC();
            if (!inf_codes(s, out, lencode, distcode)) return false;
        } else {
            return false;
        }
        if (last) return true;
    }
}

// gzip member header (RFC 1952 2.3): returns the offset of the deflate stream, or 0 if this is not a gzip member
__host__ __device__ inline uint32_t gzip_header_len(const uint8_t *in, uint32_t n) {
    if (n < 18 || in[0] != 0x1f || in[1] != 0x8b || in[2] != 8) return 0;
    const uint32_t flg = in[3];
    if (flg & 0xe0u) return 0;          // reserved bits
    uint32_t p = 10;
    if (flg & 4u) {                     // FEXTRA
        if (p + 2 > n) return 0;
        p += 2u + ((uint32_t)in[p] | ((uint32_t)in[p + 1] << 8));
    }
    for (int f = 0; f < 2; f++)         // FNAME, FCOMMENT: zero-terminated
        if (flg & (f ? 16u : 8u)) {
            while (p < n && in[p] != 0) p++;
            p++;
        }
    if (flg & 2u) p += 2;               // FHCRC
    return p + 8 <= n ? p : 0;          // room for the trailer (CRC32, ISIZE)
}
// ISIZE: the uncompressed length mod 2^32, the last four bytes of the member
__host__ __device__ inline uint32_t gzip_isize(const uint8_t *in, uint32_t n) {
    return (uint32_t)in[n - 4] | ((uint32_t)in[n - 3] << 8) | ((uint32_t)in[n - 2] << 16) | ((uint32_t)in[n - 1] << 24);
}

// gzip: one member (what producers write: the records section is one gzip stream).  The size pass trusts ISIZE, but not
// beyond what DEFLATE can expand n bytes to (a forged trailer must not size the scratch buffer); the copy pass is bounded by
// it and must produce exactly that many bytes.  The CRC32 of the trailer is not verified (the batch CRC is, with check.crcs on).
__host__ __device__ inline LzWalk gzip_size(const uint8_t *in, uint32_t n) {
    if (gzip_header_len(in, n) && (uint64_t)gzip_isize(in, n) <= (uint64_t)n * 1032u + 64u) return LzWalk{gzip_isize(in, n), true};
    return LzWalk{0, false};
}

// The output policy of the copy: lane 0 writes the literals, all lanes copy matches and stored blocks (on the host, lane 0 is
// the only lane).
struct InfOut {
    uint8_t *out;
    uint64_t op, cap;
    int lane;
    __host__ __device__ bool lit(uint8_t b) {
        if (op >= cap) return false;
        if (lane == 0) out[op] = b;
        op++;
        return true;
    }
    __host__ __device__ bool match(uint32_t dist, uint32_t len) {
        if (dist > op || op + len > cap) return false;
        lz_emit_match<true>(out, op, dist, len, lane);   // syncs the warp first: lane 0's literals are visible
        op += len;
        return true;
    }
    __host__ __device__ bool stored(const uint8_t *src, uint32_t len) {
        if (op + len > cap) return false;
        lz_emit_literals<true>(out, op, src, len, lane);
        op += len;
        return true;
    }
};

// The copy of the member at in[0, n) into out[0, out_cap), the whole warp (out_cap: what gzip_size gave)
__host__ __device__ inline LzWalk gzip_walk(const uint8_t *in, uint32_t n, uint8_t *out, uint64_t out_cap, InfWork &work, int lane) {
    LzWalk w{0, false};
    const uint32_t hl = gzip_header_len(in, n);
    if (!hl) return w;
    InfBits s{in + hl, n - hl - 8u, 0u, 0ull, 0, false};
    InfOut o{out, 0, out_cap, lane};
    const bool ok = inf_stream(s, o, work, lane);
    w.out_len = o.op;
    w.ok = ok && o.op == (uint64_t)gzip_isize(in, n);
    return w;
}

}  // namespace kta
