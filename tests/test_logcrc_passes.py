"""The check.crcs passes of the RecordBatch decoder (kta_logcrc.cuh) checked batch by batch: the span counts (windowed or not),
their scan, log_crc_span_kernel (each warp a contiguous run of the call's spans, 32 per round; a lane finds its span's batch
from the batch ends behind the warp's current batch, computes its span's register and moves it to the batch's end; the lanes
of one batch xor-combine their shares before one atomic) and the header pass's verdict.

tests/native/log_probe.cu runs scan_log_batches' steps (kta_logscan.cuh) for a handle with check.crcs on and returns
spans[0..nbatches], acc[b] for every batch, every batch's flags, the failure list and the header pass's error words.  Each case compares all of them with crc_contract(), a numpy restatement of the stage's contract: a framed batch
that is served has ceil((12 + batchLength - 21) / 1024) spans and acc = its plain CRC-32C ^ 0xFFFFFFFF, every other batch 0
spans and acc 0.  The plain CRC is kafka_codec's byte loop, run in lockstep over many regions with numpy, or the probe's host
mode for large regions; test_plain_crcs_agree pins them to each other.  The probe can also run the span pass on a grid of
one block (32 warps): the pass's body does not depend on its grid, so every warp then reaches many rounds with few spans.
A case built to reach an edge (a gap of unserved batches at lane j of round r of warp w) asserts from the spans that it does."""
import struct
from types import SimpleNamespace

import numpy as np
import pytest

import kafka_codec as kc
import log_probe

SPAN, FROM, THREADS = 1024, 21, 1024                          # LOG_CRC_SPAN, LOG_CRC_FROM, LOG_CRC_THREADS
LOGB_SKIP_CONTROL, LOGB_BAD, LOGB_COMPRESSED, LOGB_CODECS = 1, 2, 4, 8 | 16 | 32 | 64
LOGB_SKIP_CRC, LOGB_SKIP_OFFSET = 256, 512
CODEC_FLAG = np.array([0, 32, 16, 8, 64, 4, 4, 4], np.uint32)   # attributes & 7 → LOGB_*, 5..7: LOGB_COMPRESSED
FAIL = np.dtype([("batch", "<u4"), ("bytes", "<u4"), ("base", "<i8"), ("part", "<i4"), ("stored", "<u4"), ("computed", "<u4"),
                 ("pad", "<u4")])                              # LogCrcFail
HDR = struct.Struct(">qiibIhiqqqhii")                          # a batch header, recordsCount last
TS0 = 1_700_000_000_000
NEVER = 1 << 40                                                # a log start offset above every baseOffset here
KS = (1, 2, 3, 31, 32, 33, 64, 1000)                           # gap sizes (unserved batches in a row)
PERS = (1, 2, 31, 32, 33, 2048)                                # spans per warp with the one-block grid (2048: 64 rounds)
_T = np.array(kc._CRC32C, np.uint32)


# ------------------------------------------------------------------------------------------------
# the plain CRC
# ------------------------------------------------------------------------------------------------
def crc32c_lockstep(regions):
    """kafka_codec.crc32c of every region (uint8 arrays): the same byte loop, one step over all regions at a time"""
    n = len(regions)
    if n == 0:
        return np.zeros(0, np.uint32)
    lens = np.array([len(r) for r in regions], np.int64)
    order = np.argsort(-lens, kind="stable")
    m = np.zeros((int(lens.max()), n), np.uint8)               # column i: the i-th longest region
    for i, r in enumerate(order):
        m[:lens[r], i] = regions[r]
    sl, crc, live = lens[order], np.full(n, 0xFFFFFFFF, np.uint32), n
    for j in range(m.shape[0]):
        while live and sl[live - 1] <= j:
            live -= 1
        c = crc[:live]
        crc[:live] = _T[(c ^ m[j, :live]) & 0xFF] ^ (c >> 8)
    out = np.empty(n, np.uint32)
    out[order] = crc ^ 0xFFFFFFFF
    return out


def host_crcs(regions):
    """the probe's host mode (plain C++, no CUDA): the CRC-32C of every region"""
    return log_probe.crc32c(regions)


def plain_crcs(regions, large=1 << 16):
    """the plain CRC of every region: in lockstep up to `large` bytes, the host mode above it"""
    lens = np.array([len(r) for r in regions], np.int64)
    out = np.zeros(len(regions), np.uint32)
    small = np.flatnonzero(lens <= large)
    big = np.flatnonzero(lens > large)
    out[small] = crc32c_lockstep([regions[i] for i in small])
    if big.size:
        out[big] = host_crcs([regions[i] for i in big])
    return out


# ------------------------------------------------------------------------------------------------
# the restatement
# ------------------------------------------------------------------------------------------------
def _be(data, offs, at, width):
    """the big-endian unsigned field at offs + at of every batch (offsets past the buffer read its last byte)"""
    last = max(data.size - 1, 0)
    v = np.zeros(offs.size, np.uint64)
    for k in range(width):
        v = (v << np.uint64(8)) | data[np.minimum(offs + np.uint64(at + k), np.uint64(last))].astype(np.uint64)
    return v


def crc_contract(c):
    """what the passes give for case c: spans[0..nb], acc[nb], flags[nb], error words [0..9], the failure list.  c.crcs, when
    given, holds the plain CRC of the batches' regions (only read where a batch has spans)."""
    data, offs, n = c.data, c.offs, c.data.size
    nb = offs.size
    ok61 = offs + np.uint64(61) <= np.uint64(n)
    base = _be(data, offs, 0, 8).view(np.int64)
    bl = _be(data, offs, 8, 4).astype(np.uint32).view(np.int32).astype(np.int64)
    magic = _be(data, offs, 16, 1).astype(np.uint8).view(np.int8)
    stored = _be(data, offs, 17, 4).astype(np.uint32)
    attrs = _be(data, offs, 21, 2).astype(np.uint32)
    last_delta = _be(data, offs, 23, 4).astype(np.uint32).view(np.int32).astype(np.int64)
    count = _be(data, offs, 57, 4).astype(np.uint32).view(np.int32).astype(np.int64)
    framed = ok61 & (magic == 2) & (bl >= 49) & (offs.astype(np.int64) + 12 + bl <= n)
    part = c.parts if c.parts is not None else np.zeros(nb, np.int32)
    win = np.array(c.win, np.int64).reshape(-1, 2)
    has = (part >= 0) & (part < len(win))
    lo = np.where(has, win[np.clip(part, 0, max(len(win) - 1, 0))][:, 0] if len(win) else -1, -1)
    hi = np.where(has, win[np.clip(part, 0, max(len(win) - 1, 0))][:, 1] if len(win) else -1, -1)
    with np.errstate(over="ignore"):
        last = base + last_delta                              # 64-bit two's complement
    skip = framed & (((lo >= 0) & (last < lo)) | ((hi >= 0) & (last >= hi)))
    checked = framed & ~skip
    length = 12 + bl
    nspans = np.where(checked, (length - FROM + SPAN - 1) // SPAN, 0).astype(np.uint64)
    spans = np.concatenate([[0], np.cumsum(nspans)]).astype(np.uint64)
    if c.crcs is None:
        idx = np.flatnonzero(checked)
        crc = np.zeros(nb, np.uint32)
        crc[idx] = plain_crcs([data[int(offs[i]) + FROM:int(offs[i]) + int(length[i])] for i in idx])
    else:
        crc = c.crcs
    acc = np.where(checked, crc ^ np.uint32(0xFFFFFFFF), 0).astype(np.uint32)
    fail = checked & (stored != crc)
    codec, ctrl = attrs & 7, (attrs & 0x20) != 0
    read = framed & ~skip & ~fail & (count >= 0) & ((codec != 0) | (count * 7 + 49 <= bl))
    flags = np.full(nb, LOGB_BAD, np.uint32)
    flags[skip] = LOGB_SKIP_OFFSET
    flags[fail] = LOGB_SKIP_CRC
    flags[read & ctrl] = LOGB_SKIP_CONTROL
    flags[read & ~ctrl] = CODEC_FLAG[codec[read & ~ctrl]]
    err = np.zeros(10, np.uint32)
    err[0] = np.bitwise_or.reduce(flags & (LOGB_BAD | LOGB_COMPRESSED | LOGB_CODECS)) if nb else 0
    err[1] = length[flags == 0].max() if (flags == 0).any() else 0
    err[2] = fail.sum()
    fb = int(length[fail].sum())
    err[4], err[5] = fb & 0xFFFFFFFF, fb >> 32
    cut = read & ~ctrl & (codec <= 4) & (count > 0) & (lo >= 0) & (base < lo)
    left = int(count[skip & ~ctrl & (count > 0)].sum())
    err[6], err[7], err[8], err[9] = cut.sum(), skip.sum(), left & 0xFFFFFFFF, left >> 32
    fi = np.flatnonzero(fail)
    fails = np.zeros(fi.size, FAIL)
    fails["batch"], fails["bytes"], fails["base"], fails["part"] = fi, length[fi], base[fi], part[fi]
    fails["stored"], fails["computed"] = stored[fi], crc[fi]
    return SimpleNamespace(spans=spans, acc=acc, flags=flags, err=err, fails=fails, nspans=nspans, checked=checked, fail=fail,
                           skip=skip)


def span_grid(c, sm_count):
    """log_crc_span_grid, or the case's own grid"""
    if c.grid:
        return c.grid
    return int(max(1, min((c.data.size // SPAN + c.offs.size + THREADS - 1) // THREADS, sm_count)))


def place(g, total, nwarps):
    """where span g is met: (warp, round, lane, first span of the warp's run, last span of its run)"""
    per = -(-total // nwarps)
    w, o = divmod(g, per)
    return w, o // 32, o % 32, o == 0, o == per - 1 or g == total - 1


def gaps(want, nwarps):
    """every run of batches without spans: (its length, where the first span behind it is met, or None at the call's end,
    whether it opens the call)"""
    z = np.concatenate([[False], want.nspans == 0, [False]])
    d = np.diff(z.astype(np.int8))
    starts, ends = np.flatnonzero(d == 1), np.flatnonzero(d == -1)
    total = int(want.spans[-1])
    out = []
    for a, e in zip(starts, ends):
        g = int(want.spans[e])
        out.append((int(e - a), place(g, total, nwarps) if g < total else None, a == 0))
    return out


# ------------------------------------------------------------------------------------------------
# batches
# ------------------------------------------------------------------------------------------------
class Pool:
    """batch templates with their stored CRC set and their plain CRC known; a case places them at baseOffsets of its own
    (baseOffset lies outside the CRC region)"""

    def __init__(self):
        self.raw, self.crc = [], np.zeros(0, np.uint32)

    def add(self, raws):
        raws = [bytearray(r) for r in raws]
        crcs = plain_crcs([np.frombuffer(bytes(r[FROM:]), np.uint8) for r in raws])
        for r, v in zip(raws, crcs):
            r[17:21] = int(v).to_bytes(4, "big")
        first = len(self.raw)
        self.raw += [np.frombuffer(bytes(r), np.uint8) for r in raws]
        self.crc = np.concatenate([self.crc, crcs])
        return np.arange(first, len(self.raw))

    def blank(self, regions, rng):
        """batches without records whose CRC region is `region` bytes: the 40-byte header tail, then unread random bytes"""
        return self.add([HDR.pack(0, r + 9, 0, 2, 0, 0, 0, TS0, TS0, -1, -1, -1, 0) + rng.bytes(r - 40) for r in regions])


def case(name, pool, tidx, bases=None, parts=None, win=(), grid=0, bad=None, pad=None):
    """the templates tidx back to back (pad[i] filler bytes before batch i), batch i at baseOffset bases[i] in partition
    parts[i]; bad: batches whose stored CRC is one bit off"""
    tidx = np.asarray(tidx, np.int64)
    nb = tidx.size
    lens = np.array([pool.raw[t].size for t in tidx], np.int64)
    pad = np.zeros(nb, np.int64) if pad is None else np.asarray(pad, np.int64)
    offs = (np.cumsum(lens + pad) - lens).astype(np.uint64)
    pieces = []
    for t, p in zip(tidx, pad):
        if p:
            pieces.append(np.full(p, 0xEE, np.uint8))
        pieces.append(pool.raw[t])
    data = np.concatenate(pieces) if pieces else np.zeros(0, np.uint8)
    if bases is not None:
        be = np.asarray(bases, np.int64).astype(">i8").view(np.uint8).reshape(nb, 8)
        data[offs[:, None].astype(np.int64) + np.arange(8)] = be
    if bad is not None:
        data[offs[np.asarray(bad)].astype(np.int64) + 20] ^= 1
    return SimpleNamespace(name=name, data=data, offs=offs, parts=None if parts is None else np.asarray(parts, np.int32),
                           slack=0, win=list(win), grid=grid, crcs=pool.crc[tidx].copy())


def regrid(c, grid):
    return SimpleNamespace(**{**vars(c), "grid": grid, "name": "%s/grid=%s" % (c.name, grid or "library")})


# ------------------------------------------------------------------------------------------------
# the probe
# ------------------------------------------------------------------------------------------------
def spans(cases):
    """the cases through the library's steps with check.crcs on (log_probe) → per case the passes' arrays"""
    sm_count = log_probe.device()[0]
    ins = [log_probe.inputs(c.data, c.offs, c.parts, c.slack, c.win, check_crcs=True, span_grid=c.grid) for c in cases]
    return [SimpleNamespace(sm_count=sm_count, grid=int(r.crc_grid[0]), spans=r.spans, acc=r.acc, flags=r.flags, err=r.word,
                            fails=np.sort(r.crc_fails, order="batch").astype(FAIL)) for r in log_probe.run(ins)]


def check(c, g, want=None):
    """every array the probe gave equals the contract's; returns the contract"""
    w = crc_contract(c) if want is None else want
    assert g.grid == span_grid(c, g.sm_count), c.name
    assert np.array_equal(g.spans, w.spans), "%s: spans differ first at batch %d" % (c.name, np.flatnonzero(g.spans != w.spans)[0] - 1)
    total, nwarps = int(w.spans[-1]), 32 * g.grid
    bad = np.flatnonzero(g.acc != w.acc)
    if bad.size:
        b = int(bad[0])
        first = int(w.spans[b])
        where = "span %d: warp %d, round %d, lane %d" % ((first,) + place(first, total, nwarps)[:3]) if w.nspans[b] else "no spans"
        raise AssertionError("%s: acc differs at %d batches, first batch %d (%d spans, first %s): 0x%08x, want 0x%08x"
                             % (c.name, bad.size, b, int(w.nspans[b]), where, g.acc[b], w.acc[b]))
    bad = np.flatnonzero(g.flags != w.flags)
    assert not bad.size, "%s: flags differ at batch %d: %d, want %d" % (c.name, bad[0], g.flags[bad[0]], w.flags[bad[0]])
    assert np.array_equal(g.err, w.err), "%s: error words %s, want %s" % (c.name, g.err.tolist(), w.err.tolist())
    assert np.array_equal(g.fails, w.fails), c.name
    return w


def probe_all(cases):
    out = []
    for c, g in zip(cases, spans(cases)):
        out.append((c, g, check(c, g)))
    return out


# ------------------------------------------------------------------------------------------------
# cases
# ------------------------------------------------------------------------------------------------
_pools = {}


def one_span_pool():
    """1000 batches of one span each (CRC regions of 40 to 600 bytes)"""
    if "one" not in _pools:
        rng = np.random.default_rng(1)
        p = Pool()
        p.blank(rng.integers(40, 601, 1000).tolist(), rng)
        _pools["one"] = p
    return _pools["one"]


def gap_offsets(P, mode):
    """per warp of a one-block grid with P spans per warp, where in its run the gap goes: "lanes": warp w at lane w % 32
    (of a round spread over the run), "ends": the first span of the run (even warps) or its last (odd warps)"""
    rounds, out = -(-P // 32), []
    for w in range(32):
        if mode == "lanes" and w == 0 and P > 32:
            out.append(32)                                     # lane 0 of round 1: a round boundary
        elif mode == "lanes":
            j = w % min(32, P)
            r = min(rounds - 1, w * rounds // 32)
            while 32 * r + j >= P:
                r -= 1
            out.append(32 * r + j)
        else:
            out.append(0 if w % 2 == 0 else P - 1)
    return out


def served_layout(name, total, gap_at, seed, pool=None):
    """total served one-span batches (partitions 0 and 2 alternating), with gap_at[g] unserved batches (partition 1, wholly
    below its log start offset) before the served batch of span g; gap_at[total]: unserved batches at the call's end"""
    pool = pool or one_span_pool()
    rng = np.random.default_rng(seed)
    k = np.zeros(total + 1, np.int64)
    for g, n in gap_at.items():
        k[g] += n
    served = np.arange(total)
    # batch sequence: before served span g, k[g] unserved
    pos_served = served + np.cumsum(k)[:total]
    nb = total + int(k.sum())
    is_served = np.zeros(nb, bool)
    is_served[pos_served] = True
    parts = np.where(is_served, 0, 1).astype(np.int32)
    parts[pos_served[1::2]] = 2
    tidx = rng.integers(0, len(pool.raw), nb)
    bad = np.flatnonzero(~is_served & (rng.random(nb) < 0.5))   # (a failed batch that is not served is not reported)
    return case(name, pool, tidx, bases=np.arange(nb), parts=parts, win=[(-1, -1), (NEVER, -1), (0, -1)], grid=1, bad=bad)


def gap_cases(P, k):
    total = 32 * P
    out = []
    for mode in ("lanes", "ends"):
        at = {w * P + o: k for w, o in enumerate(gap_offsets(P, mode))}
        if mode == "ends":
            at[total] = k                                      # the call's last batches (and at[0]: its first)
        out.append(served_layout("gaps k=%d per=%d %s" % (k, P, mode), total, at, seed=1000 * P + k))
    return out


def seam_case():
    """partition 0: 100 one-span batches; partition 1: 40 batches below its log start offset, then 100 served ones"""
    pool = one_span_pool()
    rng = np.random.default_rng(7)
    parts = [0] * 100 + [1] * 140
    bases = list(range(100)) + list(range(140))
    return case("partition seam", pool, rng.integers(0, len(pool.raw), 240), bases=bases, parts=parts, win=[(-1, -1), (40, -1)])


def saturated_case(sm_count=132):
    """enough one-span batches that the library's grid is capped at the SM count (40 spans per warp), with gaps of two
    unserved batches at 3000 random places"""
    total = sm_count * 32 * 40
    rng = np.random.default_rng(8)
    at = {int(g): 2 for g in rng.choice(total, 3000, replace=False)}
    c = served_layout("saturated grid, gaps of 2", total, at, seed=9)
    c.grid = 0
    return c


def multi_span_case():
    """one-block grid, 33 spans per warp: a two-span batch from lane 31 of round 0 into lane 0 of round 1; batches of 33,
    64 and 300 spans, the last across nine warps' runs (several warps add to one acc); gaps of 2 and 40 in front of two"""
    rng = np.random.default_rng(10)
    pool = Pool()
    spans = [1] * 31 + [2] + [1] * 67 + [300] + [1] * 5 + [33] + [1] * 20 + [64]
    P = 33
    total = 32 * P
    spans += [1] * (total - sum(spans))
    regions = [s * SPAN - int(rng.integers(0, SPAN)) if s > 1 else int(rng.integers(40, SPAN + 1)) for s in spans]
    served = pool.blank(regions, rng)
    unserved = pool.blank(rng.integers(40, 3000, 42).tolist(), rng)
    tidx, parts = [], []
    for i, t in enumerate(served):
        if spans[i] in (300, 64):
            some = unserved[40:42] if spans[i] == 300 else unserved[:40]
            tidx += some.tolist()
            parts += [1] * some.size
        tidx.append(t)
        parts.append(0)
    return case("several warps per batch", pool, tidx, bases=np.arange(len(tidx)), parts=parts, win=[(-1, -1), (NEVER, -1)], grid=1)


def all_unserved_case():
    pool = one_span_pool()
    return case("every batch unserved", pool, np.arange(300), bases=np.arange(300), parts=[1] * 300, win=[(-1, -1), (NEVER, -1)],
                bad=np.arange(0, 300, 3))


# ------------------------------------------------------------------------------------------------
# CPU
# ------------------------------------------------------------------------------------------------
def test_plain_crcs_agree():
    """kafka_codec.crc32c, the lockstep loop and the probe's host mode: the RFC 3720 answers, and each other on random regions
    of 0 to 3000 bytes"""
    known = [(b"123456789", 0xE3069283), (bytes(32), 0x8A9136AA), (b"\xff" * 32, 0x62A8AB43), (bytes(range(32)), 0x46DD794E),
             (bytes(range(31, -1, -1)), 0x113FDB5C)]
    regions = [np.frombuffer(d, np.uint8) for d, _ in known]
    want = np.array([v for _, v in known], np.uint32)
    assert np.array_equal(crc32c_lockstep(regions), want)
    assert np.array_equal(host_crcs(regions), want)
    rng = np.random.default_rng(0)
    regions = [np.frombuffer(rng.bytes(int(n)), np.uint8) for n in list(range(0, 70)) + rng.integers(0, 3000, 200).tolist()]
    py = np.array([kc.crc32c(r.tobytes()) for r in regions], np.uint32)
    assert np.array_equal(crc32c_lockstep(regions), py)
    assert np.array_equal(host_crcs(regions), py)
    assert np.array_equal(plain_crcs(regions, large=1000), py)


def test_contract_reads_kafka_codec_batches():
    """on batches kafka_codec writes with their real CRCs: nothing fails, spans and flags as the header says"""
    rng = np.random.default_rng(2)
    raws = [kc.set_crcs(kc.encode_batch(10 * i, TS0, [(j, j, b"k%d" % j, int(rng.integers(0, 3000))) for j in range(5)],
                                        compression=codec))
            for i, codec in enumerate((None, "gzip", "snappy", "lz4", "zstd", None))]
    c = SimpleNamespace(data=np.frombuffer(b"".join(raws), np.uint8), offs=np.array(kc.batch_offsets(b"".join(raws)), np.uint64),
                        parts=None, win=[], crcs=None)
    w = crc_contract(c)
    assert not w.fail.any() and w.err[2] == 0
    assert w.nspans.tolist() == [-(-(len(r) - FROM) // SPAN) for r in raws]
    assert w.flags.tolist() == [0, 32, 16, 8, 64, 0]


def test_gap_layouts_reach_their_edges():
    """with the one-block grid: for every gap size and every run length, the gaps meet every lane a run reaches, the first
    and last span of runs, a round boundary past round 0, and the call's first and last batches"""
    for P in PERS:
        for k in KS:
            seen = set()
            opens = closes = False
            for c in gap_cases(P, k):
                w = crc_contract(c)
                assert int(w.spans[-1]) == 32 * P
                for n, where, first in gaps(w, 32):
                    assert n == k
                    opens |= bool(first)
                    if where is None:
                        closes = True
                    else:
                        seen.add(where)
            lanes = {x[2] for x in seen}
            assert lanes == set(range(min(32, P))), (P, k, sorted(lanes))
            assert any(x[3] for x in seen) and any(x[4] for x in seen) and opens and closes, (P, k)
            if P > 32:
                assert any(x[1] > 0 and x[2] == 0 for x in seen), (P, k)
            if P == 2048:
                assert max(x[1] for x in seen) >= 63


# ------------------------------------------------------------------------------------------------
# GPU
# ------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("P", PERS)
def test_gaps_at_lookahead_and_run_edges(P):
    """gaps of 1 to 1000 unserved batches at every lane, at the ends of every warp's run, and at the call's ends, with
    one-span batches (a round of one-span batches covers 32 batches, 33 with one empty batch in it), through the one-block
    grid and the library's grid"""
    cases = [c for k in KS for c in gap_cases(P, k)]
    for c, g, w in probe_all(cases + [regrid(c, 0) for c in cases]):
        assert int(g.err[7]) == int(w.skip.sum()) > 0


@pytest.mark.gpu
def test_gap_layouts_on_the_library_grid():
    """the partition seam (100 batches of partition 0, then 40 of partition 1 below its log start offset, then 100 served),
    the library's grid capped at the SM count with gaps of two, several warps per batch, every batch unserved"""
    cases = [seam_case(), saturated_case(), multi_span_case(), all_unserved_case()]
    cases.append(regrid(cases[2], 0))
    res = probe_all(cases)
    c, g, w = res[0]
    assert g.grid == 1 and -(-int(w.spans[-1]) // 32) == 7
    assert [where[1:3] for n, where, _ in gaps(w, 32) if where] == [(0, 2)]     # the seam at lane 2 of warp 14's round
    c, g, w = res[1]
    assert g.grid == g.sm_count and -(-int(w.spans[-1]) // (32 * g.grid)) > 32
    lanes = {where[2] for n, where, _ in gaps(w, 32 * g.grid) if where}
    assert lanes == set(range(32))
    c, g, w = res[2]
    per = -(-int(w.spans[-1]) // 32)
    first = int(w.spans[31])
    assert w.nspans[31] == 2 and place(first, int(w.spans[-1]), 32)[1:3] == (0, 31)
    for b in np.flatnonzero(w.nspans >= 300):                 # reaches over several seams between warps' runs
        assert (int(w.spans[b + 1]) - 1) // per - int(w.spans[b]) // per >= 8
    c, g, w = res[3]
    assert int(w.spans[-1]) == 0 and not g.acc.any() and int(g.err[2]) == 0


@pytest.mark.gpu
def test_region_lengths():
    """every CRC region of 40 to 2 * 1024 + 64 bytes; k * 1024 - 1, k * 1024 and k * 1024 + 1 bytes for k around 4096 (where a
    span's power of x starts to take a pow_hi factor) and around 8192 (pow_hi[2]); both grids"""
    rng = np.random.default_rng(11)
    pool = Pool()
    small = pool.blank(list(range(40, 2 * SPAN + 65)), rng)
    big = pool.blank([k * SPAN + d for k in (4095, 4096, 4097, 8191, 8192, 8193) for d in (-1, 0, 1)], rng)
    cases = [case("lengths 40..2112", pool, rng.permutation(small), bases=np.arange(small.size)),
             case("lengths around 4096 and 8192 spans", pool, np.concatenate([big, small[:50]]), bases=np.arange(big.size + 50))]
    cases += [regrid(c, 1) for c in cases]
    res = probe_all(cases)
    w = res[1][2]
    assert int(w.nspans.max()) == 8194 and {4095, 4096, 4097, 8192, 8193}.issubset(set(w.nspans.tolist()))


@pytest.mark.gpu
def test_largest_batch():
    """one batch with batchLength = 2^31 - 1 (2^21 spans: the last pow_hi entry), a batch without records followed by
    unread bytes, between two small ones.  The file's largest cost: on an H100 the test process peaked at 4.3 GiB of host
    memory and the device at 2.5 GiB."""
    rng = np.random.default_rng(12)
    pool = Pool()
    small = pool.blank([100, 5000], rng)
    region = (1 << 31) - 1 - 9
    hdr = HDR.pack(0, (1 << 31) - 1, 0, 2, 0, 0, 0, TS0, TS0, -1, -1, -1, 0)
    raw = np.empty(61 + region - 40, np.uint8)
    raw[:61] = np.frombuffer(hdr, np.uint8)
    raw[61:] = rng.integers(0, 256, raw.size - 61, dtype=np.uint8)
    crc = host_crcs([raw[FROM:]])[0]
    raw[17:21] = np.frombuffer(int(crc).to_bytes(4, "big"), np.uint8)
    pool.raw.append(raw)
    pool.crc = np.concatenate([pool.crc, [crc]]).astype(np.uint32)
    c = case("batchLength 2^31 - 1", pool, [small[0], len(pool.raw) - 1, small[1]], bases=[0, 1, 2])
    del raw
    (c2, g, w), = probe_all([c])
    assert int(w.nspans[1]) == 1 << 21 and int(g.err[2]) == 0


@pytest.mark.gpu
def test_alignment():
    """batch offsets at every residue mod 16 times CRC regions at every residue mod 64, of one span and of three: every
    head, 64-byte, 16-byte and tail path of crc_span, for the first span of a batch and the later ones; both grids"""
    rng = np.random.default_rng(13)
    pool = Pool()
    regions = [base + r for base in (960, 2048) for _ in range(16) for r in range(64)]
    tidx = pool.blank(regions, rng)
    lens = np.array([pool.raw[t].size for t in tidx], np.int64)
    # pad so that the 64 regions of repetition j start at residue j mod 16
    want = np.arange(tidx.size) // 64 % 16
    pad = np.zeros(tidx.size, np.int64)
    at = 0
    for i in range(tidx.size):
        pad[i] = (want[i] - at) % 16
        at += pad[i] + lens[i]
    c = case("alignment", pool, tidx, bases=np.arange(tidx.size), pad=pad)
    for one in (True, False):
        sel = (lens - FROM <= SPAN) == one
        assert len(set(zip((c.offs[sel] % 16).tolist(), ((lens[sel] - FROM) % 64).tolist()))) == 16 * 64
    probe_all([c, regrid(c, 1)])


@pytest.mark.gpu
def test_verdicts():
    """stored CRC equal and one bit off; a failed batch that is not served (not reported); a cut batch (checked whole);
    compressed batches of every codec (checked over their stored bytes); control batches"""
    rng = np.random.default_rng(14)
    pool = Pool()
    raws = []
    for codec in (None, "gzip", "snappy", "snappy-xerial", "lz4", "zstd", "zstd-stream"):
        recs = [(j, j, b"k%d" % j, int(rng.integers(0, 2500))) for j in range(int(rng.integers(2, 12)))]
        raws.append(kc.encode_batch(0, TS0, recs, compression=codec))
    raws.append(kc.marker(0, 5, 0, True, TS0))
    t = pool.add(raws)
    # each template four times: served, served and failing, cut (baseOffset below S, last at or above), not served and failing
    tidx, bases, parts, bad, win = [], [], [], [], []
    for x in t:
        for kind in range(4):
            parts.append(len(win))
            win.append(((15, -1), (-1, -1), (15, -1), (NEVER, -1))[kind])
            bases.append(14 if kind == 2 else 20)             # kind 2: baseOffset below S, its last record at or above
            if kind in (1, 3):
                bad.append(len(tidx))
            tidx.append(x)
    c = case("verdicts", pool, tidx, bases=bases, parts=parts, win=win, bad=bad)
    (c, g, w), = probe_all([c])
    n = len(t)
    assert w.fail.tolist() == [k == 1 for _ in t for k in range(4)]
    assert int(g.err[6]) == n - 1 and int(g.err[7]) == n + 1  # every data batch cut once; the marker's last is below S


@pytest.mark.gpu
def test_single_bit_damage():
    """3000 single-bit flips, each in its own batch, at random positions of the CRC region or the stored CRC field: exactly
    the damaged batches fail, each with the plain CRC of its damaged bytes as computed"""
    rng = np.random.default_rng(15)
    pool = Pool()
    tidx = pool.blank(rng.integers(40, 4000, 6000).tolist(), rng)
    c = case("damage", pool, tidx, bases=np.arange(tidx.size))
    hit = np.sort(rng.choice(tidx.size, 3000, replace=False))
    lens = np.array([pool.raw[t].size for t in tidx], np.int64)
    pos = c.offs[hit].astype(np.int64) + 17 + (rng.random(hit.size) * (lens[hit] - 17)).astype(np.int64)
    c.data[pos] ^= (1 << rng.integers(0, 8, hit.size)).astype(np.uint8)
    c.crcs = None                                              # the contract computes the CRC of the damaged bytes
    (c, g, w), = probe_all([c])
    assert np.array_equal(np.flatnonzero(w.fail), hit)


@pytest.mark.gpu
def test_at_depth():
    """the library's grid at its cap with every warp at least 64 rounds of 32 spans: ~9 million one-span batches (about
    0.5 GB, tiled from 64 templates), in partitions of 1000 to 3000 batches whose log start offsets leave out their first 1
    to 40 batches, so gaps sit at every partition seam"""
    rng = np.random.default_rng(16)
    pool = Pool()
    tmpl = pool.blank(rng.integers(40, 64, 64).tolist(), rng)
    block = rng.integers(0, 64, 1 << 16)
    blk = np.concatenate([pool.raw[t] for t in tmpl[block]])
    blen = np.array([pool.raw[t].size for t in tmpl[block]], np.int64)
    need = 132 * 32 * 64 * 32
    reps = -(-(need + 4 * need // 100) // block.size)
    nb = reps * block.size
    data = np.tile(blk, reps)
    offs = (np.cumsum(np.tile(blen, reps)) - np.tile(blen, reps)).astype(np.uint64)
    plen = rng.integers(1000, 3001, nb // 1000 + 1)
    pstart = np.concatenate([[0], np.cumsum(plen)])
    npart = int(np.searchsorted(pstart, nb, side="right"))
    parts = (np.searchsorted(pstart, np.arange(nb), side="right") - 1).astype(np.int32)
    bases = np.arange(nb, dtype=np.int64) - pstart[parts]
    skipped = rng.integers(1, 41, npart)
    at = offs.astype(np.int64)
    be = bases.astype(">i8").view(np.uint8).reshape(nb, 8)
    for k in range(8):
        data[at + k] = be[:, k]
    del be
    unserved = bases < skipped[parts]
    data[at[unserved] + 20] ^= 0x40                            # (and their stored CRCs are wrong)
    c = SimpleNamespace(name="depth", data=data, offs=offs, parts=parts, slack=0, win=[(int(s), -1) for s in skipped], grid=0,
                        crcs=np.tile(pool.crc[tmpl[block]], reps))
    (c, g, w), = probe_all([c])
    per = -(-int(w.spans[-1]) // (32 * g.grid))
    assert g.grid == g.sm_count and per >= 64 * 32, (g.grid, per)
    assert int(g.err[7]) == int(unserved.sum()) and int(g.err[2]) == 0
