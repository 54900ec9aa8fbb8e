// TEST INFRASTRUCTURE: the zstd walk of the RecordBatch decoder (csrc/kta_zstd.cuh: the __host__ __device__ statements
// log_zstd_size_kernel and log_decompress_kernel run on the GPU) on the host, one "lane".
// stdin: cases of u32 length + bytes; stdout per case: u8 ok, u32 size-pass length, u32 length, bytes.  The output and literal
// buffers are allocated at exactly the size pass's length, so that an overrun of the copy pass is a heap overflow an
// address-sanitizer build reports.
#include <cstdio>
#include <cstdint>
#include <cstdlib>

#include "../../kafka_topic_analyzer_b200/csrc/kta_logdecode.cuh"

int main() {
    uint32_t n;
    kta::ZstdWork *w = (kta::ZstdWork *)malloc(sizeof(kta::ZstdWork));
    while (fread(&n, 4, 1, stdin) == 1) {
        // exact-size heap copies: reads past the input are heap overflows too
        uint8_t *in = (uint8_t *)malloc(n ? n : 1);
        if (n && fread(in, 1, n, stdin) != n) return 2;
        const kta::LzWalk size = kta::zstd_walk<false>(in, n, nullptr, nullptr, 0, *w, 0);
        kta::LzWalk copy{0, false};
        const bool fits = size.ok && size.out_len <= (64u << 20);
        uint8_t *out = (uint8_t *)malloc(fits && size.out_len ? size.out_len : 1);
        uint8_t *lit = (uint8_t *)malloc(fits && size.out_len ? size.out_len : 1);
        if (fits) copy = kta::zstd_walk<true>(in, n, out, lit, size.out_len, *w, 0);
        const uint8_t okb = size.ok && copy.ok && copy.out_len == size.out_len ? 1 : 0;
        const uint32_t sl = (uint32_t)size.out_len, len = okb ? (uint32_t)copy.out_len : 0;
        fwrite(&okb, 1, 1, stdout);
        fwrite(&sl, 4, 1, stdout);
        fwrite(&len, 4, 1, stdout);
        if (len) fwrite(out, 1, len, stdout);
        free(lit);
        free(out);
        free(in);
    }
    free(w);
    return 0;
}
