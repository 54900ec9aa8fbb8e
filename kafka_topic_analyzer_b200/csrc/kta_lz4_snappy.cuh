// kta_lz4_snappy.cuh — the records section of a Kafka record batch whose attributes name codec 3 (LZ4) or 2 (Snappy), which
// librdkafka decompresses inside poll before the handlers see a message (src/kafka.rs:93).  Used by log_unc_size_kernel and
// log_decompress_kernel (kta_logdecode.cuh), one thread per batch for the size, one warp per batch for the copy.
//   LZ4: the frame format (magic 0x184D2204 | FLG | BD | [content size] | [dict id] | HC | blocks… | EndMark | [checksum]);
//        a block is a u32 LE size (top bit = stored uncompressed) + data [+ block checksum]; block data = sequences of
//        token | literal length… | literals | offset u16 | match length… ; matches may reach back into earlier blocks.
//   Snappy: raw (uvarint uncompressed length, then elements: literal / copy with 1-, 2-, 4-byte offset) or the xerial
//        framing Java clients write ("\x82SNAPPY\0", two version words, then chunks of u32 BE length + raw snappy).
// One lane parses, all lanes of the warp copy (kta_codec.cuh).  The walks are __host__ __device__ so that
// tests/test_lzwalk_host.py (through tests/native/codec_harness.cu, one lane) runs them against pyarrow's compressors.
#pragma once
#include <stdint.h>

#include "kta_codec.cuh"

namespace kta {

// LZ4 frame at in[0, n).  COPY: the whole warp calls this (lane-uniform control flow: every lane parses the same bytes).
template <bool COPY>
__host__ __device__ LzWalk lz4_frame_walk(const uint8_t *in, uint32_t n, uint8_t *out, uint64_t out_cap, int lane) {
    LzWalk w{0, false};
    if (n < 7 || in[0] != 0x04 || in[1] != 0x22 || in[2] != 0x4D || in[3] != 0x18) return w;
    const uint32_t flg = in[4];
    if ((flg >> 6) != 1) return w;
    uint32_t ip = 6 + ((flg & 0x08) ? 8u : 0u) + ((flg & 0x01) ? 4u : 0u) + 1u;   // FLG, BD, [content size], [dict id], HC
    const bool block_checksum = (flg & 0x10) != 0;
    for (;;) {
        if (ip + 4 > n) return w;
        const uint32_t bs = (uint32_t)in[ip] | ((uint32_t)in[ip + 1] << 8) | ((uint32_t)in[ip + 2] << 16) | ((uint32_t)in[ip + 3] << 24);
        ip += 4;
        if (bs == 0) break;                                  // EndMark
        const uint32_t blen = bs & 0x7fffffffu;
        if (blen > n - ip) return w;
        if (bs & 0x80000000u) {                              // stored block
            if (COPY && w.out_len + blen > out_cap) return w;
            lz_emit_literals<COPY>(out, w.out_len, in + ip, blen, lane);
            w.out_len += blen;
        } else {
            uint32_t p = ip;
            const uint32_t bend = ip + blen;
            while (p < bend) {
                const uint32_t token = in[p++];
                uint32_t lit = token >> 4;
                if (lit == 15) {
                    uint32_t b;
                    do { if (p >= bend) return w; b = in[p++]; lit += b; } while (b == 255);
                }
                if (lit > bend - p) return w;
                if (COPY && w.out_len + lit > out_cap) return w;
                lz_emit_literals<COPY>(out, w.out_len, in + p, lit, lane);
                w.out_len += lit;
                p += lit;
                if (p >= bend) break;                        // the last sequence of a block has no match
                if (p + 2 > bend) return w;
                const uint32_t offset = (uint32_t)in[p] | ((uint32_t)in[p + 1] << 8);
                p += 2;
                uint32_t ml = (token & 15u) + 4u;
                if ((token & 15u) == 15u) {
                    uint32_t b;
                    do { if (p >= bend) return w; b = in[p++]; ml += b; } while (b == 255);
                }
                if (offset == 0 || offset > w.out_len) return w;
                if (COPY && w.out_len + ml > out_cap) return w;
                lz_emit_match<COPY>(out, w.out_len, offset, ml, lane);
                w.out_len += ml;
            }
        }
        ip += blen + (block_checksum ? 4u : 0u);
    }
    w.ok = true;
    return w;
}

// one raw Snappy block at in[0, n)
template <bool COPY>
__host__ __device__ bool snappy_raw_walk(const uint8_t *in, uint32_t n, uint8_t *out, uint64_t out_cap, uint64_t &op, int lane) {
    uint64_t want;
    const int hn = uvarint_g(in, in + n, want);
    if (hn <= 0) return false;
    const uint64_t start = op;
    uint32_t p = (uint32_t)hn;
    while (p < n) {
        const uint32_t tag = in[p++];
        if ((tag & 3u) == 0) {                               // literal
            uint32_t len = (tag >> 2) + 1u;
            if (len > 60) {
                const uint32_t nb = len - 60;                // 1..4 length bytes follow
                if (p + nb > n) return false;
                len = 0;
                for (uint32_t i = 0; i < nb; i++) len |= (uint32_t)in[p + i] << (8 * i);
                len += 1u;
                p += nb;
            }
            if (len > n - p) return false;
            if (COPY && op + len > out_cap) return false;
            lz_emit_literals<COPY>(out, op, in + p, len, lane);
            op += len;
            p += len;
        } else {
            uint32_t len, offset;
            if ((tag & 3u) == 1) {
                if (p + 1 > n) return false;
                len = ((tag >> 2) & 7u) + 4u;
                offset = ((tag >> 5) << 8) | in[p];
                p += 1;
            } else if ((tag & 3u) == 2) {
                if (p + 2 > n) return false;
                len = (tag >> 2) + 1u;
                offset = (uint32_t)in[p] | ((uint32_t)in[p + 1] << 8);
                p += 2;
            } else {
                if (p + 4 > n) return false;
                len = (tag >> 2) + 1u;
                offset = (uint32_t)in[p] | ((uint32_t)in[p + 1] << 8) | ((uint32_t)in[p + 2] << 16) | ((uint32_t)in[p + 3] << 24);
                p += 4;
            }
            if (offset == 0 || offset > op - start) return false;
            if (COPY && op + len > out_cap) return false;
            lz_emit_match<COPY>(out, op, offset, len, lane);
            op += len;
        }
    }
    return op - start == want;
}

template <bool COPY>
__host__ __device__ LzWalk snappy_walk(const uint8_t *in, uint32_t n, uint8_t *out, uint64_t out_cap, int lane) {
    LzWalk w{0, false};
    const bool xerial = n >= 16 && in[0] == 0x82 && in[1] == 'S' && in[2] == 'N' && in[3] == 'A' && in[4] == 'P' && in[5] == 'P' &&
                        in[6] == 'Y' && in[7] == 0;
    if (!xerial) {
        w.ok = snappy_raw_walk<COPY>(in, n, out, out_cap, w.out_len, lane);
        return w;
    }
    uint32_t p = 16;                                         // magic (8) + version (4) + compatible version (4)
    while (p < n) {
        if (p + 4 > n) return w;
        const uint32_t cl = ((uint32_t)in[p] << 24) | ((uint32_t)in[p + 1] << 16) | ((uint32_t)in[p + 2] << 8) | in[p + 3];
        p += 4;
        if (cl > n - p) return w;
        if (!snappy_raw_walk<COPY>(in + p, cl, out, out_cap, w.out_len, lane)) return w;
        p += cl;
    }
    w.ok = true;
    return w;
}

}  // namespace kta
