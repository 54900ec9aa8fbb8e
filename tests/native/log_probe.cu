// TEST INFRASTRUCTURE: the log entry points' steps (csrc/kta_logscan.cuh) on the GPU, with everything they produce made
// visible.  Per case it applies the windows, aborted ranges and switches through the functions the handle's setters call,
// then calls the steps in the order scan_log_batches (csrc/kta_api.cu) calls them — the header step (CRC spans, header pass,
// read_committed's passes, the record-count scan), the size and copy steps of compressed batches, the cut count, the
// record decode and the key gather — and stops where the library stops.  The one exception is `decompress`: with it the
// size and copy steps run whenever the header step accepted the call and saw compressed batches, even when the library
// would stop first (a call without records, a size-step refusal), so that one launch can carry many damaged batches.
// The scan of the decoded records is the handle's and is not run.  tests/log_probe.py drives it.
//
// stdin, per case (little-endian): u64 nbytes, the bytes; u32 slack (bytes behind nbytes that may be read; the caller's
// buffer is exactly nbytes + slack long); i64 nbatches, then u64 batch offsets (-1: none, the batches are found by
// log_walk_batches as kta_push_log_segments_host finds them); u32 with_partitions, then i32 per batch partitions (0: every
// batch is partition 0); u32 nwin, then nwin x (i64 S, i64 H), the window table of partitions [0, nwin) (-1: that side
// unbounded); u32 read_committed, u32 nranges, then nranges TxnRange images; u32 check_crcs; u32 span_grid (the span
// pass's blocks, 0: the library's rule); u32 decompress.
// stdout: a block for the device, then one per case.  A block is a list of named arrays, each u32 name length, the name, u32
// dtype length, the dtype (u1 i4 u4 i8 u8, or LogBatchInfo, LogCrcFail, TxnKey), u64 count, u64 bytes, the bytes; a name of
// length 0 ends the block, followed by i32 the return code of the step that stopped the case (0: none), u32 length and
// the kta_last_error text.  Before a step runs, the LogScan buffers it writes are grown and filled with 0xA5 (so the step's
// own grow allocates nothing and an entry the step does not write shows up); buffers are reused from case to case.
//
// `log_probe crc32c` is a plain reference instead, which touches no CUDA: stdin, per region, u64 n and n bytes; stdout the
// u32 CRC-32C of each, one byte at a time with a table of its own.
#include <cstring>

#include "../../kafka_topic_analyzer_b200/csrc/kta_logscan.cuh"

#define CK(call)                                                                                           \
    do {                                                                                                   \
        cudaError_t e_ = (call);                                                                           \
        if (e_ != cudaSuccess) {                                                                           \
            fprintf(stderr, "%s: %s (%s:%d)\n", #call, cudaGetErrorString(e_), __FILE__, __LINE__);        \
            exit(3);                                                                                       \
        }                                                                                                  \
    } while (0)

// an allocation the probe itself makes (not a step's): failing ends the program
static void need(int rc) {
    if (rc) {
        fprintf(stderr, "allocation failed: %s\n", g_err);
        exit(3);
    }
}

static void put(const void *p, size_t n) {
    if (n && fwrite(p, 1, n, stdout) != n) exit(4);
}

static void get(void *p, size_t n) {
    if (n && fread(p, 1, n, stdin) != n) exit(2);
}

template <typename T> static T get1() {
    T v;
    get(&v, sizeof v);
    return v;
}

static void put_str(const char *s) {
    const uint32_t n = (uint32_t)strlen(s);
    put(&n, 4);
    put(s, n);
}

template <typename T> static void put_host(const char *name, const char *dtype, const T *p, size_t count) {
    put_str(name);
    put_str(dtype);
    const uint64_t head[2] = {count, count * sizeof(T)};
    put(head, 16);
    put(p, count * sizeof(T));
}

template <typename T> static std::vector<T> from_dev(const T *d, size_t count, cudaStream_t s) {
    std::vector<T> h(count);
    CK(cudaStreamSynchronize(s));
    if (count) CK(cudaMemcpy(h.data(), d, count * sizeof(T), cudaMemcpyDeviceToHost));
    return h;
}

template <typename T> static void put_dev(const char *name, const char *dtype, const T *d, size_t count, cudaStream_t s) {
    put_host(name, dtype, from_dev(d, count, s).data(), count);
}

static void end_block(int rc) {
    const uint32_t zero = 0;
    put(&zero, 4);
    put(&rc, 4);
    put_str(rc ? g_err : "");
}

// the LogScan buffer a step is about to write: grown to n elements and filled with 0xA5
template <typename T> static void sentinel(DevBuf<T> &b, int64_t n, cudaStream_t s) {
    need(b.grow(s, n));
    if (n) CK(cudaMemsetAsync(b.get(), 0xA5, (size_t)n * sizeof(T), s));
}

// CRC-32C (reflected 0x82F63B78, init and xorout 0xFFFFFFFF), one byte at a time
static int crc32c_mode() {
    uint32_t t[256];
    for (uint32_t i = 0; i < 256; i++) {
        uint32_t c = i;
        for (int k = 0; k < 8; k++) c = (c & 1u) ? (c >> 1) ^ 0x82F63B78u : c >> 1;
        t[i] = c;
    }
    std::vector<uint8_t> buf;
    uint64_t n;
    while (fread(&n, 8, 1, stdin) == 1) {
        buf.resize(n);
        get(buf.data(), n);
        uint32_t crc = 0xFFFFFFFFu;
        for (uint64_t i = 0; i < n; i++) crc = t[(crc ^ buf[i]) & 0xFFu] ^ (crc >> 8);
        crc ^= 0xFFFFFFFFu;
        put(&crc, 4);
    }
    fflush(stdout);
    return 0;
}

// One case, from the header step to where the library stops.  Returns the return code of the step that stopped it.
static int run_case(LogScan &L, const LogEnv &e, const uint8_t *bytes, int64_t n, int64_t readable, const uint64_t *offs,
                    const int32_t *parts, int64_t nb, bool decompress) {
    cudaStream_t s = e.stream;
    int rc;
    // the header step
    sentinel(L.info, nb + 1, s);
    sentinel(L.cnt, nb + 1, s);
    if (L.offsets.set > 0) sentinel(L.offsets.d_cut, nb, s);
    if (L.crc.on) sentinel(L.crc.d_spans, nb + 1, s), sentinel(L.crc.d_acc, nb, s), sentinel(L.crc.d_fails, nb, s);
    if (L.read_committed) {
        sentinel(L.txn.d_keys, nb, s), sentinel(L.txn.d_sorted, nb, s), sentinel(L.txn.d_kind, nb, s), sentinel(L.txn.d_res, nb, s);
        sentinel(L.txn.d_tile, 2 * log_txn_tiles(nb), s);
    }
    LogHeaders hd;
    const int hrc = log_headers(L, e, 0, parts, bytes, n, offs, nb, hd);
    uint64_t nrec = hd.nrec;
    // per batch only the flags and records of the header step's LogBatchInfo (a case may have millions of batches)
    const std::vector<LogBatchInfo> info = from_dev(L.info.get(), (size_t)nb, s);
    std::vector<uint32_t> flags((size_t)nb);
    std::vector<int32_t> records((size_t)nb);
    for (size_t b = 0; b < (size_t)nb; b++) flags[b] = info[b].flags, records[b] = info[b].records;
    const LogHeaderWord word = from_dev(L.err.get(), 1, s)[0];
    put_host("word", "u4", reinterpret_cast<const uint32_t *>(&word), sizeof word / 4);
    put_dev("cnt", "u8", L.cnt.get(), (size_t)nb + 1, s);
    put_host("nrec", "u8", &hd.nrec, 1);   // (as read back by the header step; 0 when it stopped before)
    put_host("flags", "u4", flags.data(), flags.size());
    put_host("records", "i4", records.data(), records.size());
    // the shape log_decode launches for these batches: staged, stage, grid
    const LogDecodeShape shape = log_decode_shape(word.longest, nb, e.sm_count, e.smem_optin);
    const uint32_t shape3[3] = {shape.staged ? 1u : 0u, shape.stage, (uint32_t)shape.grid};
    put_host("shape", "u4", shape3, 3);
    if (L.crc.on) {
        const uint32_t grid = (uint32_t)log_crc_grid(L.crc, n, nb, e.sm_count);
        put_host("crc_grid", "u4", &grid, 1);
        put_dev("spans", "u8", L.crc.d_spans.get(), (size_t)nb + 1, s);
        put_dev("acc", "u4", L.crc.d_acc.get(), (size_t)nb, s);
        put_dev("crc_fails", "LogCrcFail", L.crc.d_fails.get(), std::min<size_t>(word.crc_failed, (size_t)nb), s);
    }
    if (L.read_committed) {
        const std::vector<uint32_t> w = from_dev(L.txn.d_word.get(), 2, s);
        const uint32_t ran = hd.txn_ran;
        put_host("txn_word", "u4", w.data(), 2);
        put_host("txn_ran", "u4", &ran, 1);
        put_host("txn_stats", "u8", hd.txn_stats, 3);
        put_dev("kind", "u1", L.txn.d_kind.get(), (size_t)nb, s);
        if (ran) {
            put_dev("sorted", "TxnKey", L.txn.d_sorted.get(), w[0], s);
            put_dev("res", "u1", L.txn.d_res.get(), w[0], s);
            put_dev("tile", "u1", L.txn.d_tile.get(), (size_t)(2 * log_txn_tiles(w[0])), s);
        }
    }
    if (hrc) return hrc;
    const uint32_t codecs = hd.word.flags & LOGB_CODECS;
    uint64_t unc_total = 0;
    if (codecs && (hd.nrec > 0 || decompress)) {
        // the size step, then the copy step
        uint32_t bad = 0;
        sentinel(L.unc_slot, nb + 2, s);
        if ((rc = log_unc_size(L, e, bytes, nb, codecs, &unc_total, &bad))) return rc;
        put_host("size_flags", "u4", &bad, 1);
        put_dev("slot", "u8", L.unc_slot.get(), (size_t)nb + 1, s);
        if (bad && !decompress) return fail(KTA_ERR_INVALID, "malformed compressed record batch in partition %d", 0);
        sentinel(L.unc, (int64_t)unc_total + 64, s);
        if (codecs & LOGB_ZSTD) sentinel(L.unc_lit, (int64_t)unc_total + 64, s);
        if ((rc = log_unc_copy(L, e, bytes, nb, codecs, unc_total))) return rc;
        const int64_t unc_at = (int64_t)((uintptr_t)L.unc.get() - (uintptr_t)bytes);   // where info's offsets lead into unc
        put_dev("info", "LogBatchInfo", L.info.get(), (size_t)nb, s);
        put_dev("unc", "u1", L.unc.get(), (size_t)unc_total + 64, s);
        put_host("unc_at", "i8", &unc_at, 1);
        if (bad) return fail(KTA_ERR_INVALID, "malformed compressed record batch in partition %d", 0);
    }
    if (hd.nrec == 0) return KTA_OK;
    const int64_t ncut = hd.word.cut;
    if (ncut) {
        uint64_t dropped = 0;
        sentinel(L.offsets.d_drop, nb + 1, s);
        if ((rc = log_cut_count(L, e, bytes, nb, ncut, &nrec, &dropped))) return rc;
        put_dev("drop", "u8", L.offsets.d_drop.get(), (size_t)nb + 1, s);
    }
    // the record decode and the key gather, with keys as on a handle that hashes them
    const bool keys = nrec > 0;
    const uint32_t windowed = ncut ? 1u : 0u;
    put_host("windowed", "u4", &windowed, 1);
    for (DevBuf<int32_t> *c : {&L.dec_part, &L.dec_klen, &L.dec_vlen}) sentinel(*c, (int64_t)nrec, s);
    sentinel(L.dec_ts, (int64_t)nrec, s);
    sentinel(L.dec_ksrc, (int64_t)nrec, s);
    kta_batch b;
    if ((rc = log_decode(L, e, bytes, readable, nb, nrec, hd.word.longest, keys, ncut, b))) return rc;
    const int64_t ntiles = ((int64_t)nrec + TILE - 1) / TILE;
    if (keys) {
        sentinel(e.tile_base, ntiles + 1, s);
        sentinel(L.dec_keys, readable + (int64_t)unc_total + 64, s);   // (the keys cannot outnumber the records' bytes)
    }
    rc = log_gather_keys(L, e, 0, bytes, keys, b);
    put_dev("dec_flags", "u4", &L.err.get()->flags, 1, s);
    put_dev("part", "i4", L.dec_part.get(), nrec, s);
    put_dev("ts", "i8", L.dec_ts.get(), nrec, s);
    put_dev("klen", "i4", L.dec_klen.get(), nrec, s);
    put_dev("vlen", "i4", L.dec_vlen.get(), nrec, s);
    if (rc) return rc;
    if (keys) {
        put_dev("tile_base", "u8", e.tile_base.get(), (size_t)ntiles + 1, s);
        put_dev("keys", "u1", L.dec_keys.get(), (size_t)b.key_bytes_len + 64, s);
    }
    return KTA_OK;
}

int main(int argc, char **argv) {
    if (argc > 1 && !strcmp(argv[1], "crc32c")) return crc32c_mode();
    int sm_count = 0, optin = 0;
    CK(cudaDeviceGetAttribute(&sm_count, cudaDevAttrMultiProcessorCount, 0));
    CK(cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, 0));
    put_host("sm_count", "u4", (const uint32_t *)&sm_count, 1);
    put_host("smem_optin", "u4", (const uint32_t *)&optin, 1);
    end_block(0);
    cudaStream_t s;
    CK(cudaStreamCreate(&s));
    LogScan L;
    DevBuf<uint64_t> tile_base;
    uint64_t launches = 0;
    need(log_scan_create(L, true, (size_t)optin));   // (read_committed's words exist; each case sets the switch itself)
    uint64_t n;
    while (fread(&n, 8, 1, stdin) == 1) {
        std::vector<uint8_t> seg(n);
        get(seg.data(), n);
        const uint32_t slack = get1<uint32_t>();
        int64_t nb = get1<int64_t>();
        const bool walked = nb < 0;
        std::vector<uint64_t> offs;
        if (!walked) {
            offs.resize((size_t)nb);
            get(offs.data(), offs.size() * 8);
        } else {
            log_walk_batches(seg.data(), (int64_t)n, 0, offs);
            nb = (int64_t)offs.size();
        }
        std::vector<int32_t> parts(get1<uint32_t>() ? (size_t)nb : 0);
        get(parts.data(), parts.size() * 4);
        std::vector<longlong2> win(get1<uint32_t>());
        get(win.data(), win.size() * sizeof(longlong2));
        const bool read_committed = get1<uint32_t>() != 0;
        std::vector<TxnRange> ranges(get1<uint32_t>());
        get(ranges.data(), ranges.size() * sizeof(TxnRange));
        const bool check_crcs = get1<uint32_t>() != 0;
        const int span_grid = (int)get1<uint32_t>();
        const bool decompress = get1<uint32_t>() != 0;

        // the caller's buffers
        DevBuf<uint8_t> d_bytes;
        DevBuf<uint64_t> d_off;
        DevBuf<int32_t> d_part;
        need(d_bytes.alloc((int64_t)n + slack));
        need(d_off.alloc(std::max<int64_t>(nb, 1)));
        if (!parts.empty()) need(d_part.alloc(nb));
        CK(cudaMemsetAsync(d_bytes.get(), 0, n + slack, s));
        CK(cudaMemcpyAsync(d_bytes.get(), seg.data(), n, cudaMemcpyHostToDevice, s));
        CK(cudaMemcpyAsync(d_off.get(), offs.data(), offs.size() * 8, cudaMemcpyHostToDevice, s));
        if (!parts.empty()) CK(cudaMemcpyAsync(d_part.get(), parts.data(), parts.size() * 4, cudaMemcpyHostToDevice, s));

        // the case's settings, through what the setters call, on a LogScan without windows or ranges
        const LogEnv e{s, sm_count, (size_t)optin, (int32_t)win.size(), tile_base, launches};
        L.offsets.win.clear();
        L.offsets.set = 0;
        L.offsets.d_win = DevBuf<longlong2>();   // (a handle's table has num_partitions entries; here each case has its own)
        for (size_t p = 0; p < win.size(); p++) log_set_window(L, (int32_t)win.size(), (int32_t)p, win[p].x, win[p].y);
        L.read_committed = read_committed;
        L.txn.ranges.clear();
        if (!ranges.empty()) need(log_add_txn_ranges(L, e, ranges));
        L.crc.on = check_crcs;
        L.crc.span_grid = span_grid;

        if (walked) put_host("offs", "u8", offs.data(), offs.size());
        const int rc = nb ? run_case(L, e, d_bytes, (int64_t)n, (int64_t)n + slack, d_off, parts.empty() ? nullptr : d_part.get(), nb,
                                     decompress)
                          : KTA_OK;
        CK(cudaStreamSynchronize(s));
        end_block(rc);
    }
    CK(cudaStreamDestroy(s));
    fflush(stdout);
    return 0;
}
