// TEST INFRASTRUCTURE: the codec walks of the RecordBatch decoder on the host, one "lane": the size pass and the copy pass of
// csrc/kta_logdecode.cuh (section_size / section_copy for gzip, LZ4 and Snappy, zstd_walk for zstd), the statements
// log_unc_size_kernel, log_zstd_size_kernel and log_decompress_kernel run on the GPU.
// stdin: cases of u8 Kafka codec id (1 gzip, 2 Snappy, 3 LZ4, 4 zstd) + u32 length + bytes; stdout per case: u8 ok, u32 size-pass
// length, u32 length, bytes.  Input, output and zstd literal buffers are heap blocks of exactly their size, so that a read or
// write outside them is a heap overflow an address-sanitizer build reports.
#include <cstdint>
#include <cstdio>
#include <cstdlib>

#include "../../kafka_topic_analyzer_b200/csrc/kta_logdecode.cuh"

int main() {
    kta::InfWork *iw = (kta::InfWork *)malloc(sizeof(kta::InfWork));
    kta::ZstdWork *zw = (kta::ZstdWork *)malloc(sizeof(kta::ZstdWork));
    uint8_t codec;
    uint32_t n;
    while (fread(&codec, 1, 1, stdin) == 1 && fread(&n, 4, 1, stdin) == 1) {
        if (codec < 1 || codec > 4) return 2;
        const uint32_t flag = kta::log_codec_flag(codec);
        const bool zstd = flag == kta::LOGB_ZSTD;
        uint8_t *in = (uint8_t *)malloc(n ? n : 1);
        if (n && fread(in, 1, n, stdin) != n) return 2;
        const kta::LzWalk size = zstd ? kta::zstd_walk<false>(in, n, nullptr, nullptr, 0, *zw, 0) : kta::section_size(flag, in, n);
        const bool fits = size.ok && size.out_len <= (64u << 20);
        const size_t cap = fits && size.out_len ? size.out_len : 1;
        uint8_t *out = (uint8_t *)malloc(cap), *lit = zstd ? (uint8_t *)malloc(cap) : nullptr;
        kta::LzWalk copy{0, false};
        if (fits) copy = zstd ? kta::zstd_walk<true>(in, n, out, lit, size.out_len, *zw, 0) : kta::section_copy(flag, in, n, out, 0, size.out_len, *iw, 0);
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
    free(zw);
    free(iw);
    return 0;
}
