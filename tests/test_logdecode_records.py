"""The record stage of the RecordBatch decoder — log_header_kernel's recordsCount bound, log_decode_kernel (one warp per batch:
lane 0 hops 32 record-length varints, then 32 lanes parse), the key-length tile bases and log_gather_keys_kernel — checked
record by record.

tests/native/log_probe.cu runs scan_log_batches' steps up to the scan (kta_logscan.cuh) and returns every decoded column.
Every case compares partition, ts_ms, key_len and value_len of every record, the tile-base column (the running sum of
max(key_len, 0) per 128-record tile) and the packed key bytes with the records the case was built from, after the
consumer's rules (control and empty batches are not delivered; LogAppendTime stamps maxTimestamp; a timestamp is
baseTimestamp + timestampDelta).  The metrics behind the scan would hide most of these
errors (a timestamp that is not an extreme, value lengths shifted inside one partition)."""
import struct
from collections import namedtuple

import numpy as np
import pytest

import kafka_codec as kc
import log_probe

TS0 = 1_700_000_000_000
LOGB_BAD = 2
M64 = (1 << 64) - 1
FILL32, FILL64 = np.int32(-0x5A5A5A5B), np.int64(-0x5A5A5A5A5A5A5A5B)   # 0xA5 bytes: what the probe fills the columns with
# words, windowed, flags, drop: the window mode's outputs (cases with a window table, tests/test_logoffsets_records.py)
Result = namedtuple("Result", "hdr longest unc_err dec_err nrec staged stage grid ran part ts klen vlen tile_base keys "
                              "words windowed flags drop", defaults=(None,) * 4)


# ------------------------------------------------------------------------------------------------
# cases
# ------------------------------------------------------------------------------------------------
def i64(x):
    return (x + (1 << 63)) % (1 << 64) - (1 << 63)


def batch(records, base_ts=TS0, attributes=0, max_ts=None, compression=None, base_offset=0, pad=0):
    """records as for kafka_codec.encode_batch → (bytes, the records a consumer delivers: (ts, key|None, value_len)).  pad:
    bytes behind the last record, inside the batch (never read)"""
    b = kc.encode_batch(base_offset, base_ts, records, attributes, max_ts, compression)
    if pad:
        b = b[:8] + struct.pack(">i", len(b) - 12 + pad) + b[12:] + b"\xee" * pad
    mt = struct.unpack(">q", b[35:43])[0]
    want = []
    if not attributes & 0x20:
        for r in records:
            value = r[5] if len(r) > 5 else None
            vl = len(value) if value is not None else (-1 if r[3] is None else r[3])
            want.append((mt if attributes & 0x08 else i64(base_ts + r[1]), r[2], vl))
    return b, want


class Case:
    """batches laid out in one buffer: leads[i] filler bytes before batch i; parts: per-batch partitions or None (all 0);
    win: the window table [(S, H)] of partitions [0, len(win)), or None (no windows)"""
    win = None

    def __init__(self, name, batches, leads=None, parts=None, slack=0, check_reader=True):
        self.name, self.slack, self.parts = name, slack, parts
        leads = leads or [0] * len(batches)
        buf, offs, want, counts = bytearray(), [], [], []
        for i, ((b, w), lead) in enumerate(zip(batches, leads)):
            buf += bytes((0xEE + j) & 0xFF for j in range(lead))
            offs.append(len(buf))
            buf += b
            p = parts[i] if parts else 0
            want += [(p,) + r for r in w]
            counts.append(len(w))
        self.data, self.offs, self.counts = bytes(buf), offs, counts
        self.cols = columns(want)
        if check_reader:
            # the expected records are also what the codec's plain reader delivers
            got = [r for b, _ in batches for r in kc.delivered(b)]
            assert [(ts, key, -1 if vl is None else vl) for _, ts, key, vl in got] == [r[1:] for r in want], name


Cols = namedtuple("Cols", "part ts klen vlen keys")


def columns(recs):
    """(partition, ts, key|None, value_len) records → the decoded columns and the packed key bytes"""
    return Cols(np.array([r[0] for r in recs], np.int32), np.array([r[1] for r in recs], np.int64),
                np.array([-1 if r[2] is None else len(r[2]) for r in recs], np.int32), np.array([r[3] for r in recs], np.int32),
                b"".join(r[2] for r in recs if r[2]))


def tile_base(klen):
    t = np.add.reduceat(np.maximum(klen, 0).astype(np.uint64), np.arange(0, len(klen), 128)) if len(klen) else np.zeros(0, np.uint64)
    return np.concatenate([[0], np.cumsum(t)]).astype(np.uint64)


def decode(cases):
    """the cases through the library's steps (log_probe) → ((SM count, opt-in shared memory), a Result per case)"""
    res = []
    for c, r in zip(cases, log_probe.run([log_probe.inputs(c.data, c.offs, c.parts or None, c.slack, () if c.win is None else c.win) for c in cases])):
        w, nb = r.word, len(c.offs)
        ran = r.get("part") is not None
        nrec = len(r.part) if ran else int(r.cnt[-1])
        keys = r.get("keys")
        extra = ()
        if c.win is not None and len(c.win):
            drop = r.get("drop")
            extra = ((int(w[6]), int(w[7]), int(w[8]) | int(w[9]) << 32), int(r.get("windowed", [0])[0]), r.flags,
                     np.zeros(nb + 1, np.uint64) if drop is None else drop)
        res.append(Result(int(w[0]), int(w[1]), int(r.get("size_flags", [0])[0]), int(r.get("dec_flags", [0])[0]), nrec,
                          *(int(x) for x in r.shape), int(ran), r.get("part"), r.get("ts"), r.get("klen"), r.get("vlen"),
                          r.get("tile_base"), None if keys is None else keys.tobytes(), *extra))
    return log_probe.device(), res


def decode_shape(longest, nbatches, sm_count, optin):
    """log_decode_shape (kta_logdecode_launch.cuh): (staged, stage, blocks per SM, grid)"""
    stage = (longest + 16 + 1023) // 1024 * 1024
    staged = stage <= 48 * 1024
    smem = 4 * (192 + (stage if staged else 0))
    per_sm = max(1, min(16, optin // smem))
    return staged, stage if staged else 0, per_sm, min((nbatches + 3) // 4, sm_count * per_sm)


def check(case, r, cols=None, counts=None):
    """every column of every record, the tile bases and the key bytes; the first bad record is named with its batch, lane and
    warp"""
    cols = cols or case.cols
    counts = case.counts if counts is None else counts
    assert r.hdr & LOGB_BAD == 0 and r.unc_err == 0 and r.dec_err == 0, (case.name, r.hdr, r.unc_err, r.dec_err)
    assert r.nrec == len(cols.part), (case.name, r.nrec, len(cols.part))
    if r.nrec == 0:
        return
    assert r.ran
    bad = np.zeros(r.nrec, bool)
    for name in ("part", "ts", "klen", "vlen"):
        bad |= getattr(r, name) != getattr(cols, name)
    if bad.any():
        i = int(np.argmax(bad))
        starts = np.concatenate([[0], np.cumsum(counts)])
        b = int(np.searchsorted(starts, i, "right") - 1)
        j = i - int(starts[b])
        # rows the decoder never wrote still hold the 0xA5 fill in every column
        unwritten = np.flatnonzero((r.part == FILL32) & (r.ts == FILL64) & (r.klen == FILL32) & (r.vlen == FILL32))
        pytest.fail("%s: record %d (batch %d, record %d of it, lane %d, warp %d of %d; %d bad records, %d rows unwritten%s): "
                    "got (%d, %d, %d, %d), want (%d, %d, %d, %d)"
                    % (case.name, i, b, j, j % 32, b % (4 * r.grid), 4 * r.grid, int(bad.sum()), len(unwritten),
                       ", the first row %d" % unwritten[0] if len(unwritten) else "", r.part[i], r.ts[i], r.klen[i], r.vlen[i],
                       cols.part[i], cols.ts[i], cols.klen[i], cols.vlen[i]))
    want_tb = tile_base(cols.klen)
    assert np.array_equal(r.tile_base, want_tb), (case.name, "tile base", int(np.argmax(r.tile_base != want_tb)))
    n = len(cols.keys)
    if r.keys[:n] != cols.keys:
        k = next(i for i in range(n) if r.keys[i] != cols.keys[i])
        rec = int(np.searchsorted(np.cumsum(np.maximum(cols.klen, 0)), k, "right"))
        pytest.fail("%s: key byte %d (record %d) differs" % (case.name, k, rec))
    assert r.keys[n:] == b"\xa5" * 64, (case.name, "the gather wrote past the packed keys")


def key(i, n):
    return bytes((i * 7 + j * 13 + 1) & 0xFF for j in range(n))


# ---- lane rounds ---------------------------------------------------------------------------------------------------------
def rounds_batches(counts):
    out = []
    for c in counts:
        recs = [(j, j * 3 - 50, None if j % 9 == 4 else key(j, j % 11), None if j % 7 == 3 else (j * 5) % 30) for j in range(c)]
        out.append(batch(recs, base_ts=TS0 + c))
    return out


def lane_round_cases():
    counts = [1, 31, 32, 33, 63, 64, 65, 1000]
    return [Case("rounds", rounds_batches(counts)),
            Case("rounds-4097", rounds_batches([4097, 32, 64])),
            # a batch that runs out of records at a round boundary, followed by one whose records end mid-round
            Case("rounds-boundary", rounds_batches([64, 96, 33, 128, 1]))]


# ---- varints --------------------------------------------------------------------------------------------------------------
def varint_cases():
    rng = np.random.default_rng(61)
    recs = []
    for n in (0, 1, 20, 60, 62, 63, 64, 100, 4000, 8100, 8200, 9000):          # record lengths of 1, 2 and 3 bytes
        recs.append((len(recs), len(recs), b"k", n))
    for w in range(1, 11):                                                    # padded varints, every field
        for field in ("len", "ts", "key", "value"):
            recs.append((len(recs), -w, key(w, w), w * 3, (), None, {field: w}))
        recs.append((len(recs), w, None, None, (), None, {"len": w, "ts": w, "key": w, "value": w}))
    for kl in (0, 1, 63, 64, 8191):
        recs.append((len(recs), 0, key(kl, kl), 1))
    for d in (0, 1, -1, 2 ** 31, -2 ** 31, 2 ** 62, -2 ** 62, 2 ** 31 - 1, -2 ** 31 + 1):
        recs.append((len(recs), d, b"ts", 2))
    recs.append((len(recs), -1 - TS0, b"minus-one", 3))                       # a sum of exactly -1: "not available"
    recs.append((len(recs), -2 - TS0, b"minus-two", 4))
    for j in range(40):                                                       # offset deltas: garbage, but well formed
        recs.append((int(rng.integers(-2 ** 62, 2 ** 62)), j, key(j, 3), j))
    hrecs = []
    for nh in (0, 1, 2, 17, 200):                                             # headers with multi-byte lengths
        hdrs = tuple((key(h, 64 + h % 64), None if h % 3 == 0 else key(h, h % 20)) for h in range(nh))
        hrecs.append((len(hrecs), nh, key(nh, 5), nh, hdrs))
    small, headers = batch(recs), batch(hrecs, base_ts=TS0 - 3)
    big = batch([(0, 5, key(1, 8192), 3), (1, -5, key(2, 70_000), 8192), (2, 9, None, 70_000)])
    base_m1 = batch([(0, 0, b"a", 1), (1, 1, b"b", 2), (2, -1, b"c", 3), (3, 1234, None, 4), (4, -2 ** 62, b"d", 5)], base_ts=-1)
    return [Case("varints", [small, headers, base_m1]), Case("varints-in-place", [big, base_m1, headers, small])]


# ---- batch kinds ----------------------------------------------------------------------------------------------------------
def kind_batches():
    recs = [(j, j * 11 - 7, key(j, j % 5 + 1), j) for j in range(40)]
    return [batch(recs[:7]),
            batch(recs, attributes=0x08, max_ts=TS0 + 999_999),               # LogAppendTime with nonzero deltas
            batch([(0, 0, kc.marker_record_key(True), None)], attributes=0x30),   # a control batch
            batch([]),                                                        # a batch without records
            batch(recs[:33], base_ts=TS0 - 5),
            batch([(0, 0, kc.marker_record_key(False), None)], attributes=0x20),
            batch([]),
            batch(recs[5:], attributes=0x08, max_ts=-1),                      # LogAppendTime without a maxTimestamp
            batch(recs[:1])]


def kind_cases():
    b = kind_batches()
    return [Case("kinds", b), Case("kinds-partitions", b, parts=[7, 3, 3, 0, 2 ** 31 - 1, 5, 6, 1, 4])]


# ---- staging edges ----------------------------------------------------------------------------------------------------------
def batch_of_length(n, i=0):
    """an uncompressed batch exactly n bytes long (12 + batchLength)"""
    recs = [(0, i, key(i, 16), None), (1, 2 * i, key(i + 1, 3), 0)]
    b, _ = batch(recs)
    pad = n - len(b)
    assert pad >= 0
    return batch(recs, pad=pad)


def staging_cases():
    rng = np.random.default_rng(67)
    out = []
    small = [batch([(j, j, key(i + j, int(rng.integers(0, 40))), j) for j in range(int(rng.integers(1, 70)))], base_ts=TS0 + i)
             for i in range(16)]
    out.append(Case("alignment-mod-16", small, leads=[(i - len(b[0])) % 16 + (i * 16 if i % 3 else 0) for i, b in enumerate(small)]))
    # the longest batch fills a 48 KiB stage exactly (49136 + 16 bytes = 48 KiB): staged; one byte more: the launch is in place
    for n, name in ((49136, "stage-48k"), (49137, "stage-48k-plus-one")):
        long_b = batch_of_length(n, 3)
        out.append(Case(name, [small[0], long_b, small[1], batch_of_length(1000, 4), small[2]], leads=[0, 5, 0, 3, 0]))
    # the last batch ends exactly at the buffer's end, with and without readable slack behind it
    for slack in (0, 48):
        out.append(Case("end-slack-%d" % slack, small[:5], leads=[3, 0, 1, 0, 7], slack=slack))
    # compressed batches between staged ones: they decode from the scratch buffer, some from images longer than the stage
    zeros = [(j, j, key(j, 30), None, (), bytes(25_000)) for j in range(4)]
    mixed = []
    for i, codec in enumerate(["gzip", "lz4", "snappy", "snappy-xerial", "zstd", "zstd-stream"]):
        mixed += [small[i], batch(zeros[:1 + i % 4], compression=codec, base_ts=TS0 - i),
                  batch([(j, j, key(j, 9), j) for j in range(40)], compression=codec)]
    mixed.append(small[15])
    out.append(Case("compressed-between-staged", mixed, leads=[i % 5 for i in range(len(mixed))]))
    return out


# ---- gather -----------------------------------------------------------------------------------------------------------------
def gather_case(slack):
    """keys of 1-9, 15-17 and every multiple of 4 up to 4 KiB, at every source alignment mod 4 and both destination
    alignments (word-aligned: the funnel-shift path; not: the byte tail); the last key ends one byte before the buffer's end
    (the value-length varint behind it is the last byte read)"""
    lens = list(range(1, 10)) + [15, 16, 17] + list(range(4, 4097, 4))
    batches, leads, pos, dst = [], [], 0, 0
    for n in lens:
        for src in range(4):
            for dst_al in (0, 1 + n % 3):
                pad = (dst_al - dst) % 4
                recs = [(0, 0, key(pad, pad), None), (1, 1, key(n, n), None)]
                b = batch(recs)
                at = b[0].index(key(n, n), 61 + 2)            # the target key's offset inside the batch
                lead = (src - (pos + at)) % 4
                batches.append(b)
                leads.append(lead)
                pos += lead + len(b[0])
                dst = (dst + pad + n) % 4
    return Case("gather-slack-%d" % slack, batches, leads=leads, slack=slack, check_reader=False)


# ---- the cases, all in one probe run -----------------------------------------------------------------------------------------
def hand_built():
    return lane_round_cases() + varint_cases() + kind_cases() + staging_cases() + [gather_case(0), gather_case(48)]


@pytest.mark.gpu
def test_hand_built_cases_decode_record_by_record():
    cases = hand_built()
    (sm, optin), res = decode(cases)
    for c, r in zip(cases, res):
        staged, stage, _, grid = decode_shape(r.longest, len(c.offs), sm, optin)
        assert (r.staged, r.stage, r.grid) == (staged, stage, grid), c.name
        check(c, r)
    by = {c.name: r for c, r in zip(cases, res)}
    assert by["stage-48k"].staged and by["stage-48k"].stage == 48 * 1024
    assert not by["stage-48k-plus-one"].staged
    assert by["rounds"].staged and not by["rounds-4097"].staged
    assert by["varints"].staged and not by["varints-in-place"].staged and by["compressed-between-staged"].staged
    for name in ("part", "ts", "klen", "vlen", "keys"):
        assert np.array_equal(getattr(by["stage-48k"], name), getattr(by["stage-48k-plus-one"], name))


# ---- depth ------------------------------------------------------------------------------------------------------------------
def pool_batches(rng, big=None):
    """a pool of distinct small batches: mostly uncompressed (staged), some compressed (read in place from the scratch buffer),
    some control and empty ones (skipped), in a random order; `big`: one staged batch replaced by one of that length"""
    pool = []
    kinds = rng.permutation(["P"] * 9 + ["control"] * 4 + ["empty"] * 3 + ["S"] * 45)
    for i, kind in enumerate(kinds):
        nrec = int(rng.integers(1, 4))
        recs = [(j, int(rng.integers(-1000, 1000)), None if rng.integers(0, 8) == 0 else key(i * 3 + j, int(rng.integers(0, 24))),
                 int(rng.integers(-1, 100))) for j in range(nrec)]
        recs = [r if r[3] >= 0 else r[:3] + (None,) for r in recs]
        if kind == "P":
            pool.append(("P", batch(recs, compression=["gzip", "lz4", "snappy", "zstd"][i % 4], base_ts=TS0 + i)))
        elif kind == "control":
            pool.append(("-", batch(recs[:1], attributes=0x20)))
        elif kind == "empty":
            pool.append(("-", batch([])))
        else:
            pool.append(("S", batch(recs, base_ts=TS0 + i, attributes=0x08 if i % 11 == 3 else 0, max_ts=TS0 + 10 * i)))
    if big:
        pool[pool.index(next(p for p in pool if p[0] == "S"))] = ("S", batch_of_length(big, 5))
    return pool


def tiled(pool, nbatches, rng):
    """nbatches batches: pool[i % len(pool)] with baseOffset i * 100 and a random partition, packed back to back"""
    k = len(pool)
    reps = [pool[i % k][1] for i in range(nbatches)]
    data = bytearray(b"".join(b for b, _ in reps))
    lens = np.array([len(b) for b, _ in reps], np.int64)
    offs = np.concatenate([[0], np.cumsum(lens)[:-1]])
    arr = np.frombuffer(data, np.uint8)
    arr[(offs[:, None] + np.arange(8)).ravel()] = np.arange(nbatches, dtype=">i8").__mul__(100).view(np.uint8)
    parts = rng.integers(0, 1 << 20, nbatches).astype(np.int32)
    case = Case.__new__(Case)
    case.name, case.slack, case.parts, case.data, case.offs = "depth-%d" % nbatches, 48, parts.tolist(), bytes(data), offs.tolist()
    pc = [columns([(0,) + r for r in w]) for _, (_, w) in pool]
    idx = np.arange(nbatches) % k
    case.counts = [len(pc[i].part) for i in idx]
    case.cols = Cols(np.repeat(parts, case.counts), np.concatenate([pc[i].ts for i in idx]),
                     np.concatenate([pc[i].klen for i in idx]), np.concatenate([pc[i].vlen for i in idx]),
                     b"".join(pc[i].keys for i in idx))
    return case


@pytest.mark.gpu
@pytest.mark.parametrize("shape", ["small-batches", "stage-48k"])
def test_every_warp_decodes_many_batches(shape):
    """Every warp of the decode grid decodes >= 64 batches, so each one's mbarrier phase flips many times, stages are reused
    after __syncwarp, and staged and in-place batches alternate within one warp."""
    rng = np.random.default_rng(71 if shape == "small-batches" else 73)
    big = 49136 if shape == "stage-48k" else None
    pool = pool_batches(rng, big)
    sm, optin = log_probe.device()
    longest = max(len(b) for kind, (b, _) in pool if kind == "S")
    staged, stage, per_sm, grid = decode_shape(longest, 1 << 40, sm, optin)
    assert staged and per_sm == (16 if shape == "small-batches" else 1)
    warps = 4 * grid
    nb = 64 * warps + 17
    case = tiled(pool, nb, rng)
    # some warp decodes a staged batch, then one read in place, then a staged one again
    kinds = [pool[(w + j * warps) % len(pool)][0] for w in range(warps) for j in range(64)]
    seqs = ["".join(k for k in kinds[w * 64:(w + 1) * 64] if k != "-") for w in range(warps)]
    assert sum("SPS" in s for s in seqs) > warps // 4
    _, (r,) = decode([case])
    assert (r.staged, r.stage, r.grid) == (staged, stage, grid)
    print("%s: %d batches, %d records, %d warps, %.1f batches per warp" % (shape, nb, r.nrec, warps, nb / warps))
    check(case, r)


# ---- damaged record sections --------------------------------------------------------------------------------------------------
def contract(data, offs, n, with_offsets=False):
    """A plain restatement of what the header pass and the decoder accept (kta_logdecode.cuh), for uncompressed batches of
    partition 0: None when the call is refused, else the delivered records [(0, ts, key|None, value_len)], with_offsets: each
    with its offset baseOffset + offsetDelta (64-bit two's complement) behind.
    Framing: magic 2, batchLength >= 49 and inside the buffer, 7 * recordsCount + 49 <= batchLength.  Per record: a length
    varint of <= 10 bytes, >= 0 and inside the batch; the attributes byte; the timestamp, offset and key-length varints
    inside the record; key and value lengths in [-1, 2^31 - 1] with their bytes inside the record.  Headers, the bytes after
    the value and the bytes after the last of recordsCount records are not read.  This is more lenient than librdkafka, which
    parses every header and refuses a record whose fields do not end where its length says; bits beyond 64 in a 10-byte
    varint are dropped here, not refused."""
    def uvarint(p, end):
        v = 0
        for k in range(10):
            if p + k >= end:
                return 0, 0
            x = data[p + k]
            v |= (x & 0x7F) << (7 * k)
            if not x & 0x80:
                return k + 1, v & M64
        return 0, 0

    def unzz(u):
        return (u >> 1) ^ -(u & 1)

    out = []
    for off in offs:
        if off + 61 > n:
            return None
        base, bl = struct.unpack_from(">qi", data, off)
        magic, = struct.unpack_from(">b", data, off + 16)
        attrs, = struct.unpack_from(">H", data, off + 21)
        base_ts, max_ts = struct.unpack_from(">qq", data, off + 27)
        cnt, = struct.unpack_from(">i", data, off + 57)
        assert attrs & 7 == 0
        if not (magic == 2 and bl >= 49 and off + 12 + bl <= n and cnt >= 0 and cnt * 7 + 49 <= bl):
            return None
        if attrs & 0x20:
            continue
        end, pos = off + 12 + bl, off + 61
        for _ in range(cnt):
            k, u = uvarint(pos, end)
            if k == 0 or unzz(u) < 0 or pos + k + unzz(u) > end:
                return None
            q, rec_end = pos + k + 1, pos + k + unzz(u)
            pos = rec_end
            fields = []
            for _ in range(3):                                 # timestamp delta, offset delta, key length
                k, u = uvarint(q, rec_end)
                if not k:
                    return None
                fields.append(unzz(u))
                q += k
            ts_delta, off_delta, kl = fields
            if not (-1 <= kl <= 2 ** 31 - 1) or (kl > 0 and q + kl > rec_end):
                return None
            key = None if kl < 0 else bytes(data[q:q + kl])
            q += max(kl, 0)
            k, u = uvarint(q, rec_end)
            vl = unzz(u)
            if not k or not (-1 <= vl <= 2 ** 31 - 1) or (vl > 0 and q + k + vl > rec_end):
                return None
            rec = (0, max_ts if attrs & 0x08 else i64(base_ts + ts_delta), key, vl)
            out.append(rec + (i64(base + off_delta),) if with_offsets else rec)
    return out


def damaged_cases():
    """about 3000 single-byte mutations of uncompressed batches, each between two intact batches: in recordsCount, in the
    records section, and in the continuation bits of its varints"""
    rng = np.random.default_rng(79)
    bases = [batch([(j, j * 3, key(j, j % 9), j % 40) for j in range(40)])[0],
             batch([(j, -j, key(j, 70 + j), j, ((b"h", b"v"),) * (j % 3)) for j in range(20)])[0],
             batch([(j, j, key(j, 5), j, (), None, {"len": 1 + j % 10, "ts": 1 + j * 3 % 10, "key": 1 + j % 7})
                    for j in range(35)])[0],
             batch([(j, 2 ** 40 - j, None if j % 2 else b"", None) for j in range(33)], attributes=0x08, max_ts=TS0)[0]]
    before, after = batch([(0, 1, b"before", 1)])[0], batch([(0, 2, b"after", 2)])[0]
    cases = []
    for i in range(3000):
        b = bytearray(bases[i % len(bases)])
        kind = i % 3
        if kind == 0:                                          # recordsCount
            cnt = int.from_bytes(b[57:61], "big", signed=True)
            new = [0, 1, cnt - 1, cnt + 1, cnt - 32, cnt + 32, cnt * 2, 2 ** 31 - 1, -1, (len(b) - 61) // 7,
                   (len(b) - 61) // 7 + 1][(i // 3) % 11]
            b[57:61] = (new & 0xFFFFFFFF).to_bytes(4, "big")
            if (i // 33) % 2:                                  # and one byte of the records section too
                at = int(rng.integers(61, len(b)))
                b[at] = int(rng.integers(0, 256))
        elif kind == 1:                                        # any byte of the records section
            at = int(rng.integers(61, len(b)))
            b[at] = int(rng.integers(0, 256)) if i % 2 else b[at] ^ (1 << int(rng.integers(0, 8)))
        else:                                                  # a continuation bit
            at = int(rng.integers(61, len(b)))
            b[at] ^= 0x80
        data = before + bytes(b) + after
        offs = [0, len(before), len(before) + len(b)]
        c = Case.__new__(Case)
        c.name, c.slack, c.parts, c.data, c.offs = "damaged-%d" % i, 0, None, data, offs
        c.want = contract(data, offs, len(data))
        if c.want is not None:
            c.cols = columns(c.want)
            c.counts = [len(c.want)]
        cases.append(c)
    return cases


@pytest.mark.gpu
def test_damaged_record_sections_agree_with_the_contract():
    """Each mutated batch is refused exactly when the plain restatement of the decoder's contract refuses it, and otherwise
    decodes to that restatement's columns.  One probe run carries every case."""
    cases = damaged_cases()
    _, res = decode(cases)
    disagree = []
    for c, r in zip(cases, res):
        refused = bool(r.hdr & LOGB_BAD or r.unc_err or r.dec_err)
        if refused != (c.want is None):
            disagree.append((c.name, "refused" if refused else "accepted", r.hdr, r.dec_err))
        elif not refused:
            check(c, r)
    assert not disagree, "%d of %d cases: %s" % (len(disagree), len(cases), disagree[:20])
    assert 300 < sum(c.want is None for c in cases) < 2700    # both outcomes are exercised


# ---- the reference side, on the host ---------------------------------------------------------------------------------------
def test_restatement_and_reader_agree_on_the_hand_built_cases():
    """contract() (the decoder's rules) and kafka_codec.delivered (the consumer's) give the records every uncompressed
    hand-built case was built from"""
    for c in hand_built():
        if c.parts or any(c.data[o + 22] & 7 for o in c.offs):
            continue
        got = contract(c.data, c.offs, len(c.data))
        assert got is not None, c.name
        got = columns(got)
        assert all(np.array_equal(a, b) for a, b in zip(got[:4], c.cols[:4])) and got.keys == c.cols.keys, c.name


def test_timestamps_follow_the_consumer():
    """baseTimestamp + timestampDelta, -1 only when the sum is; LogAppendTime stamps maxTimestamp"""
    seg = kc.encode_batch(0, -1, [(0, 0, b"a", 1), (1, 5, b"b", 1)])
    seg += kc.encode_batch(2, TS0, [(0, -1 - TS0, b"c", 1), (1, -2 - TS0, b"d", 1)])
    seg += kc.encode_batch(4, TS0, [(0, 3, b"e", 1)], attributes=0x08, max_ts=TS0 + 77)
    seg += kc.encode_batch(5, TS0, [(0, 0, kc.marker_record_key(True), None)], attributes=0x30)
    seg += kc.encode_batch(6, TS0, [])
    assert [r[1] for r in kc.delivered(seg)] == [-1, 4, -1, -2, TS0 + 77]
    assert [r[1] for b in kc.read_segment(seg) for r in b.records] == [-1, 4, -1, -2, TS0 + 3, TS0]
    assert kc.varint(5, 10) == b"\x8a" + b"\x80" * 8 + b"\x00" and len(kc.varint(-1, 3)) == 3
