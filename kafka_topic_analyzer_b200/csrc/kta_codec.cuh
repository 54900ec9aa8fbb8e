// kta_codec.cuh — what the decompressors of the RecordBatch decoder share (kta_inflate.cuh, kta_lz4_snappy.cuh, kta_zstd.cuh):
// the lane primitives, the result of a walk and its two copies, and the varint reader the record parsers use.
//
// A codec walk runs one warp per batch on the device and one "lane" on the host, where tests/native/codec_harness.cu runs the
// same statements as a plain host program: KTA_LANES lanes share the strided copies, KTA_LANE_SYNC() orders them, lanes_all()
// is the warp's vote.
#pragma once
#include <stdint.h>

#ifdef __CUDA_ARCH__
#define KTA_LANE_SYNC() __syncwarp()
#define KTA_LANES 32        // copies and table fills are spread over the warp
#else
#define KTA_LANE_SYNC() ((void)0)
#define KTA_LANES 1
#endif

namespace kta {

__host__ __device__ __forceinline__ bool lanes_all(bool v) {   // the warp agrees (on the host the "warp" is one lane)
#ifdef __CUDA_ARCH__
    return __all_sync(0xffffffffu, v);
#else
    return v;
#endif
}

// unsigned LEB128 at p (bounded by end); returns bytes consumed, 0 on malformed input.  Generic byte loads: the batch may
// sit in shared memory or in global memory.
__host__ __device__ __forceinline__ int uvarint_g(const uint8_t *p, const uint8_t *end, uint64_t &out) {
    uint64_t v = 0;
    int shift = 0, n = 0;
    while (p + n < end && n < 10) {
        const uint8_t b = p[n];
        n++;
        v |= (uint64_t)(b & 0x7f) << shift;
        if (!(b & 0x80)) {
            out = v;
            return n;
        }
        shift += 7;
    }
    return 0;
}

// A walk goes through a compressed section once; with COPY = false (out == nullptr) it only adds up the output size.
struct LzWalk {
    uint64_t out_len;   // bytes produced
    bool ok;
};

// The copies, all lanes: literals from the input, and a match that refers back into the output.  A match that overlaps itself
// repeats with period `offset`, so every byte's source is known up front: out[op + i] = out[op - offset + i % offset].
template <bool COPY>
__host__ __device__ __forceinline__ void lz_emit_literals(uint8_t *out, uint64_t op, const uint8_t *in, uint32_t n, int lane) {
    if (COPY) for (uint32_t i = lane; i < n; i += KTA_LANES) out[op + i] = in[i];
}
template <bool COPY>
__host__ __device__ __forceinline__ void lz_emit_match(uint8_t *out, uint64_t op, uint32_t offset, uint32_t n, int lane) {
    if (COPY) {
        KTA_LANE_SYNC();   // the bytes the match refers to have been written
        for (uint32_t i = lane; i < n; i += KTA_LANES) out[op + i] = out[op - offset + (i % offset)];
        KTA_LANE_SYNC();
    }
}

}  // namespace kta
