"""The read_committed passes of the RecordBatch decoder (kta_logtxn.cuh) checked key by key: txn_classify_kernel, the radix sort,
txn_resolve_kernel (a warp-shuffle scan from the right, then across the warps of a 256-key tile), txn_carry_kernel (one block
over chunks of 1024 tiles, from the last chunk down) and txn_apply_kernel with its binary search of the aborted ranges.

tests/native/logtxn_probe.cu launches what log_headers launches for a read_committed handle, through the same launch functions,
and returns every array the passes produce: the error word, the sorted keys, kind per batch, res per key, tile_head and carry
per tile, every batch's flags, records and row count, and the three counters.  Each case compares them with txn_contract(), a
plain restatement of the rule of include/kta.h over (partition, producerId, baseOffset, kind) per batch; it knows nothing of
warps, and of tiles only where res is cut at a tile's end.  A case that is built to reach an edge (a chain behind six all-PASS
warps, a group that ends on the last key of a carry chunk) asserts from the sorted keys that it does.  The scan's metrics
behind these passes say that some verdict was wrong; these arrays say which key, in which pass."""
import struct
import subprocess
from types import SimpleNamespace

import numpy as np
import pytest

import kafka_codec as kc
import native_build
from feed import LOG_ENTRIES, scan_log
from kafka_topic_analyzer_b200 import KtaEngine
from parity import assert_parity, oracle_in_order
from test_log_txn import NOW, TS0, gen_topic, librdkafka_walk, rule_model

UNDECIDED, ABORT, COMMIT, DATA, PASS, NONE = 0, 1, 2, 3, 4, 0xA5   # TxnKind; NONE: the 0xA5 the probe fills kind with
ERR_MARKER, ERR_ORDER = 1, 2
LOGB_SKIP_CONTROL, LOGB_SKIP_ABORTED = 1, 128
TILE, CHUNK = 256, 1024 * 256                                      # keys per resolve tile / per chunk of the carry pass
NOPID = (1 << 64) - 1                                              # producerId -1
# what the builder writes (the first four as TxnKind): N a data batch without the transactional bit, X a control batch of
# another control type, B a control batch whose marker is version 1
D, A, C, N, X, B = DATA, ABORT, COMMIT, 10, 11, 12
RANGE = np.dtype([("part", "<i4"), ("pad", "<u4"), ("pid", "<u8"), ("first", "<i8"), ("last", "<i8")])   # TxnRange
KEY = np.dtype([("pid", "<u8"), ("part", "<u4"), ("batch", "<u4")])                                        # TxnKey


@pytest.fixture(scope="module")
def probe():
    return native_build.build("logtxn_probe")


# ------------------------------------------------------------------------------------------------
# the restatement
# ------------------------------------------------------------------------------------------------
def no_ranges():
    return np.zeros(0, RANGE)


def range_table(part, pid, first, last):
    """the ranges as the handle keeps them: sorted by (partition signed, producerId unsigned, first)"""
    t = np.zeros(len(part), RANGE)
    t["part"], t["pid"], t["first"], t["last"] = part, pid, first, last
    return t[np.lexsort((t["first"], t["pid"], t["part"]))]


def covered(part, pid, off, ranges):
    """per batch: some range of its (partition, producerId) holds its baseOffset.  Every (partition, producerId) gets a
    number; then the first range of every pair is tried, the second, and so on"""
    out = np.zeros(len(off), bool)
    if not len(ranges):
        return out
    nr = len(ranges)
    P = np.concatenate([ranges["part"], part]).astype(np.int64)
    Q = np.concatenate([ranges["pid"], pid])
    o = np.lexsort((Q, P))
    new = np.ones(len(o), bool)
    new[1:] = (P[o][1:] != P[o][:-1]) | (Q[o][1:] != Q[o][:-1])
    pair = np.empty(len(o), np.int64)
    pair[o] = np.cumsum(new) - 1
    rg, bg = pair[:nr], pair[nr:]
    by = np.argsort(rg, kind="stable")
    rg, rf, rl = rg[by], ranges["first"][by], ranges["last"][by]
    rank = np.arange(nr) - np.searchsorted(rg, rg)
    for j in range(int(rank.max()) + 1):
        first, last = np.ones(int(pair.max()) + 1, np.int64), np.zeros(int(pair.max()) + 1, np.int64)   # empty
        first[rg[rank == j]], last[rg[rank == j]] = rf[rank == j], rl[rank == j]
        out |= (first[bg] <= off) & (off <= last[bg])
    return out


def txn_contract(part, pid, off, kind, records, ranges=None):
    """The rule of include/kta.h over one call's batches, in call order: partition (i32), producerId (u64), baseOffset (i64),
    kind (DATA, ABORT, COMMIT, or NONE for a batch that takes part in nothing) and the rows the header pass gives the batch.
    The batches of a (partition bit pattern, producerId) form a group; within it, in call order, a data batch is decided by
    the nearest marker behind it: aborted if that is an ABORT marker or a range of its (partition, producerId) holds its
    baseOffset, undecided if there is no marker and no range.  The call is refused when a group's baseOffsets do not
    increase strictly.  From that, what the passes must produce (all arrays; keys in sorted order)."""
    ranges = no_ranges() if ranges is None else ranges
    part, pid, off = np.asarray(part, np.int32), np.asarray(pid, np.uint64), np.asarray(off, np.int64)
    kind, records = np.asarray(kind, np.uint8), np.asarray(records, np.int32)
    idx = np.flatnonzero(kind != NONE)
    pu = part.view(np.uint32)
    batch = idx[np.lexsort((idx, pid[idx], pu[idx]))]         # the batch of every key, sorted by (partition, id, call order)
    m = len(batch)
    w = SimpleNamespace(m=m, batch=batch, err=0, aborted=np.zeros(len(kind), bool), records=records.copy(), stats=(0, 0, 0))
    if m == 0:
        return w
    sp, sq, sk, so = pu[batch], pid[batch], kind[batch], off[batch]
    new = np.ones(m, bool)
    new[1:] = (sp[1:] != sp[:-1]) | (sq[1:] != sq[:-1])
    starts = np.flatnonzero(new)
    w.group = np.cumsum(new) - 1
    gend = np.append(starts[1:], m)[w.group]                 # one past the last key of the key's group
    i = np.arange(m)
    # the nearest marker at or behind every key (every group walked from its last batch to its first)
    w.nxt = np.minimum.accumulate(np.where(sk != DATA, i, m)[::-1])[::-1]
    found = w.nxt < gend
    w.decider = np.where(found, w.nxt, gend - 1)             # the key that decides: that marker, else the group's last key
    w.verdict = np.where(found, sk[np.minimum(w.nxt, m - 1)], UNDECIDED).astype(np.uint8)
    tend = (i // TILE + 1) * TILE                            # the one line that knows of tiles: res stops at the tile's end
    w.res = np.where(found & (w.nxt < tend), w.verdict, np.where(gend <= tend, UNDECIDED, PASS)).astype(np.uint8)
    w.tile_head = w.res[::TILE]
    w.carry = np.append(w.verdict[TILE::TILE], PASS).astype(np.uint8)   # behind tile t: what the first key of t + 1 finds
    if np.any(~new[1:] & (so[1:] <= so[:-1])):
        w.err = ERR_ORDER
        return w
    is_data = sk == DATA
    ab = is_data & ((w.verdict == ABORT) | covered(part[batch], sq, so, ranges))
    und = is_data & ~ab & (w.verdict == UNDECIDED)
    w.aborted[batch[ab]] = True
    w.stats = (int(ab.sum()), int(records[batch[ab]].sum()), int(records[batch[und]].sum()))
    w.records[w.aborted] = 0
    return w


# ------------------------------------------------------------------------------------------------
# the builder: a call of single-record batches, written column by column
# ------------------------------------------------------------------------------------------------
_DATA = np.frombuffer(kc.txn_batch(0, TS0, [(0, 0, b"K" * 8, 2)], pid=0), np.uint8)
_MARK = np.frombuffer(kc.marker(0, 0, 0, True, TS0), np.uint8)
BL = len(_DATA)
assert len(_MARK) == BL                                      # so a call is a (batches, BL) array
KPOS_D = _DATA.tobytes().index(b"K" * 8, 61)
KPOS_M = _MARK.tobytes().index(kc.marker_record_key(True), 61)


def be64(a, dt):
    return np.ascontiguousarray(a, dt).astype(dt.replace("<", ">").replace("=", ">")).view(np.uint8).reshape(-1, 8)


def build_batches(code, pid, off, keyid):
    """one batch per entry, templates of kafka_codec tiled and patched: baseOffset, the transactional and control bits,
    producerId, the marker's type (or version) and the data record's 8 key bytes.  CRCs stay 0."""
    code = np.asarray(code, np.uint8)
    ctrl = np.isin(code, (A, C, X, B))
    buf = np.where(ctrl[:, None], _MARK, _DATA)
    buf[:, 0:8] = be64(off, "<i8")
    buf[:, 22] = np.where(ctrl, 0x30, np.where(code == N, 0x00, 0x10))
    buf[:, 43:51] = be64(pid, "<u8")
    buf[ctrl, KPOS_M + 3] = np.select([code[ctrl] == A, code[ctrl] == C], [0, 1], 2)
    buf[code == B, KPOS_M + 1] = 1
    buf[~ctrl, KPOS_D:KPOS_D + 8] = be64(np.asarray(keyid)[~ctrl], "<u8")
    return buf


def txn_codes(L, fate):
    """transactions one after the other: L[t] data batches, then the marker fate[t] (A or C; 0: none) → (codes, the
    transaction of every batch)"""
    L, fate = np.asarray(L, np.int64), np.asarray(fate, np.uint8)
    size = L + (fate != 0)
    end = np.cumsum(size)
    codes = np.full(int(end[-1]), D, np.uint8)
    codes[end[fate != 0] - 1] = fate[fate != 0]
    return codes, np.repeat(np.arange(len(L)), size)


class Layout:
    """A call laid out by its sorted order: groups are added in the order the sort must give them (ascending producer ids
    in one partition unless told otherwise), add() returns the sorted position of the group's first key, and case()
    interleaves the groups batch by batch at random, every group in its own order, with the call position as baseOffset
    unless a group brings its own."""

    def __init__(self, seed=1, part=0):
        self.rng, self.part, self.pid, self.nkeys = np.random.default_rng(seed), part, 1000, 0
        self.cols = []                      # per added block: codes, partitions, producer ids, baseOffsets (-1: call position)
        self.marks = {}                     # name -> sorted position a test asserts

    def block(self, codes, part, pid, offs=None):
        codes = np.asarray(codes, np.uint8)
        n = len(codes)
        pid = np.broadcast_to(np.asarray(pid, np.uint64), n)
        start = self.nkeys
        self.cols.append((codes, np.broadcast_to(np.int32(part), n), pid,
                          np.full(n, -1, np.int64) if offs is None else np.asarray(offs, np.int64)))
        self.nkeys += int((np.isin(codes, (D, A, C)) & (pid != NOPID)).sum())
        return start

    def add(self, codes, part=None, pid=None, offs=None):
        """one group; the next producer id when none is given"""
        if pid is None:
            pid, self.pid = self.pid, self.pid + 1
        return self.block(codes, self.part if part is None else part, pid, offs)

    def fill(self, n, L=3):
        """n keys of committed transactions of L data batches, a group each (the last one shorter)"""
        if n <= 0:
            assert n == 0
            return
        sizes = np.full(-(-n // (L + 1)), L + 1)
        sizes[-1] = n - (len(sizes) - 1) * (L + 1)
        codes, t = txn_codes(sizes - 1, np.full(len(sizes), C))
        self.block(codes, self.part, self.pid + t.astype(np.uint64))
        self.pid += len(sizes)

    def fill_to(self, pos):
        self.fill(pos - self.nkeys)

    def case(self, name, ranges=None, shuffle=True):
        code, part, pid, offs = (np.concatenate(c) for c in zip(*self.cols))
        n = len(code)
        run = np.ones(n, bool)
        run[1:] = (part[1:] != part[:-1]) | (pid[1:] != pid[:-1])
        gid = np.cumsum(run)
        r = self.rng.random(n) if shuffle else np.arange(n, dtype=float)
        r = r[np.lexsort((r, gid))]                          # ascending within every group
        pos = np.empty(n, np.int64)
        pos[np.argsort(r, kind="stable")] = np.arange(n)     # the call position of every batch
        c = SimpleNamespace(name=name, marks=self.marks, ranges=no_ranges() if ranges is None else ranges)
        c.code, c.part, c.pid, c.off = (np.empty(n, a.dtype) for a in (code, part, pid, offs))
        c.code[pos], c.part[pos], c.pid[pos], c.off[pos] = code, part, pid, np.where(offs < 0, pos, offs)
        return finish(c)


def finish(c):
    """the contract's view of what the builder writes, and the expected arrays"""
    n = len(c.code)
    c.kind = np.where(np.isin(c.code, (D, A, C)) & (c.pid != NOPID), c.code, NONE).astype(np.uint8)
    c.ctrl = np.isin(c.code, (A, C, X, B))
    c.records0 = np.where(c.ctrl, 0, 1).astype(np.int32)
    c.bad_marker = bool((c.code == B).any())
    c.want = txn_contract(c.part, c.pid, c.off, c.kind, c.records0, c.ranges)
    c.keyid = np.arange(n, dtype=np.uint64)
    return c


def blob(c):
    buf = build_batches(c.code, c.pid, c.off, c.keyid)
    n = len(c.code)
    return b"".join([struct.pack("<I", buf.size), buf.tobytes(), struct.pack("<I", n), (np.arange(n, dtype="<u8") * BL).tobytes(),
                     c.part.astype("<i4").tobytes(), struct.pack("<I", len(c.ranges)), c.ranges.tobytes()])


def run_probe(exe, cases):
    r = subprocess.run([exe], input=b"".join(blob(c) for c in cases), capture_output=True)
    assert r.returncode == 0, r.stderr.decode("utf-8", "replace")[-3000:]
    out, at, res = r.stdout, 4, []

    def take(dt, n):
        nonlocal at
        a = np.frombuffer(out, dt, n, at)
        at += a.nbytes
        return a
    for c in cases:
        nb = len(c.code)
        g = SimpleNamespace()
        g.hdr, g.keys, g.err, g.ran = (int(x) for x in take("<u4", 4))
        g.stats, g.nrec = tuple(int(x) for x in take("<u8", 3)), int(take("<u8", 1)[0])
        g.kind, g.flags, g.records, g.cnt = take("u1", nb), take("<u4", nb), take("<i4", nb), take("<u8", nb + 1)
        if g.ran:
            nt = -(-g.keys // TILE)
            g.sorted, g.res, g.tile_head, g.carry = take(KEY, g.keys), take("u1", g.keys), take("u1", nt), take("u1", nt)
        res.append(g)
    assert at == len(out)
    return res


def where(c, i):
    """sorted key i of case c, for a failure message"""
    w = c.want
    b = int(w.batch[i])
    return ("key %d (tile %d, warp %d, lane %d; carry chunk %d) = batch %d (partition %d, producerId %d, baseOffset %d, kind %d), "
            "group %d, decided by key %d" % (i, i // TILE, i % TILE // 32, i % 32, i // CHUNK, b, c.part[b], c.pid[b], c.off[b],
                                             c.kind[b], w.group[i], w.decider[i]))


def first_bad(c, name, got, want, per_key):
    if np.array_equal(got, want):
        return
    assert len(got) == len(want), (c.name, name, len(got), len(want))
    bad = np.flatnonzero(got != want)
    j = int(bad[0])
    at = where(c, j) if per_key else "tile %d: first %s" % (j, where(c, j * TILE)) if per_key is None else "batch %d" % j
    pytest.fail("%s: %s differs in %d places, first at %s: got %s, want %s" % (c.name, name, len(bad), at, got[j], want[j]))


def check(c, g):
    """every array the probe returns against the restatement"""
    w = c.want
    flags0 = np.where(c.ctrl, LOGB_SKIP_CONTROL, 0).astype(np.uint32)
    assert g.hdr & 6 == 0, (c.name, g.hdr)
    assert g.keys == w.m, (c.name, "keys classified", g.keys, w.m)
    first_bad(c, "kind", g.kind, c.kind, False)
    if c.bad_marker or w.m == 0:
        assert (g.err, g.ran) == (ERR_MARKER if c.bad_marker else 0, 0), (c.name, g.err, g.ran)
    else:
        assert g.ran == 1, c.name
        got_keys = np.stack([g.sorted["part"].astype(np.uint64), g.sorted["pid"], g.sorted["batch"].astype(np.uint64)])
        want_keys = np.stack([c.part.view(np.uint32)[w.batch].astype(np.uint64), c.pid[w.batch], w.batch.astype(np.uint64)])
        bad = np.flatnonzero((got_keys != want_keys).any(0))
        assert not len(bad), "%s: the sort differs at %d keys, first at %s: got %s" % (c.name, len(bad), where(c, bad[0]), g.sorted[bad[0]])
        first_bad(c, "res", g.res, w.res, True)
        first_bad(c, "tile_head", g.tile_head, w.tile_head, None)
        first_bad(c, "carry", g.carry, w.carry, None)
        assert g.err == w.err, (c.name, "error word", g.err, w.err)
    refused = c.bad_marker or w.err
    first_bad(c, "flags", g.flags, np.where(w.aborted & (not refused), LOGB_SKIP_ABORTED, flags0), False)
    first_bad(c, "records", g.records, c.records0 if refused else w.records, False)
    first_bad(c, "rec_count", g.cnt, np.append(0, c.records0 if refused else w.records).astype(np.uint64), False)
    assert g.stats == ((0, 0, 0) if refused else w.stats), (c.name, g.stats, w.stats)
    assert g.nrec == int((c.records0 if refused else w.records).sum()), c.name


# ------------------------------------------------------------------------------------------------
# where a chain finds its answer, from the restatement alone
# ------------------------------------------------------------------------------------------------
def depth(w):
    """over the data keys: the all-PASS warps between a key and the key that decides it inside its tile, the all-PASS tiles
    between them when they lie in different tiles, and how many chains cross a carry chunk's end"""
    i = np.arange(w.m)
    dt = w.decider // TILE - i // TILE
    dw = (w.decider // 32 - i // 32)[dt == 0]
    return SimpleNamespace(warps=set((dw[dw > 0] - 1).tolist()) | ({-1} if (dw == 0).any() else set()),   # -1: the same warp
                           tiles=set((dt[dt > 0] - 1).tolist()),
                           cross_warp=int((w.decider // 32 != i // 32).sum()), cross_tile=int((dt > 0).sum()),
                           cross_chunk=int((w.decider // CHUNK != i // CHUNK).sum()))


# ------------------------------------------------------------------------------------------------
# cases
# ------------------------------------------------------------------------------------------------
LONG = (255, 256, 257, 511, 512, 513, 1000, 5000)


def chain_case():
    """a. one transaction of L data batches ending in ABORT, COMMIT or nothing, its first key at every lane (L up to 70) and
    at tile positions 0, 1, 31, 32, 254 and 255 (every L)"""
    lay = Layout(seed=11)
    starts = []
    for L in list(range(1, 71)) + [100, 130, 165, 200, 230] + list(LONG):
        for mod, at in ((32, range(32) if L <= 70 else ()), (TILE, (0, 1, 31, 32, 254, 255))):
            for pos in at:
                for end in (A, C, 0):
                    lay.fill((pos - lay.nkeys) % mod)
                    starts.append((lay.add([D] * L + ([end] if end else [])), L, end, mod, pos))
    lay.marks["chains"] = starts
    return lay.case("chains")


def edge_cases():
    """b. groups whose last key, a data batch with no marker behind it, sits on lane 31, thread 255, the last key of a carry
    chunk and the last key of all; each followed by a group that begins with an ABORT marker.  Groups of markers only, and two
    markers back to back.  Once with m a multiple of 256, once with m = 1 mod 256."""
    out = []
    for name, tail in (("edges-m%256=0", 0), ("edges-m%256=1", 1)):
        lay = Layout(seed=12)
        ends = []
        for end in (31, 255, 256 + 31, 3 * TILE - 1, CHUNK - 1):
            lay.fill_to(end + 1 - 3)
            ends.append(lay.add([D, D, D]) + 2)
            lay.add([A, D, C])
        lay.add([A, C, A])                                      # markers only
        lay.add([D, C, A, D, A])                                # an empty transaction: COMMIT, then ABORT back to back
        lay.add([C, C])
        lay.fill_to(CHUNK + 2 * TILE - 5 + tail)
        ends.append(lay.add([D, D, D, D, D]) + 4)               # the last key of all
        lay.marks["ends"], lay.marks["m"] = ends, CHUNK + 2 * TILE + tail
        out.append(lay.case(name))
    return out


def mixed(lay, upto, rng):
    """transactions of 1 to 700 batches, a group each, 1 in 8 aborted and 1 in 10 open, up to sorted position `upto`"""
    while lay.nkeys < upto:
        L = rng.choice([1, 2, 3, 5, 40, 300, 700], 200)
        fate = rng.choice([C, A, 0], 200, p=[0.775, 0.125, 0.1]).astype(np.uint8)
        keep = np.cumsum(L + (fate != 0)) <= upto - lay.nkeys
        if not keep.any():
            break
        codes, t = txn_codes(L[keep], fate[keep])
        lay.block(codes, lay.part, lay.pid + t.astype(np.uint64))
        lay.pid += int(keep.sum())
    lay.fill_to(upto)


def carry_cases():
    """c. 1, 2, 1023, 1024, 1025, 2047, 2048, 2049 and 3100 tiles; with more than one chunk, a chain from tile 1023 into tile
    1024, and one that covers all of tile 1024 (the chunk's first tile is PASS); with 2049 tiles, a chain from tile 2047 to an
    ABORT marker that is the first key of tile 2048 (the chunk's first tile is not PASS); with 3100 tiles, one transaction
    from chunk 0 to chunk 2 that makes chunk 1 all PASS"""
    out = []
    for nt in (1, 2, 1023, 1024, 1025, 2047, 2048, 2049, 3100):
        rng = np.random.default_rng(nt)
        lay = Layout(seed=nt)
        m = nt * TILE - 100
        if nt == 3100:
            mixed(lay, 1000 * TILE + 17, rng)
            lay.marks["through"] = lay.add([D] * (CHUNK + 40 * TILE) + [A])
        elif nt == 1025:
            mixed(lay, 1023 * TILE + 200, rng)
            lay.marks["into"] = lay.add([D] * 100 + [A])          # tile 1023 -> tile 1024, whose first key finds the marker
        elif nt > 1024:
            mixed(lay, 1024 * TILE - 7, rng)
            lay.marks["over"] = lay.add([D] * 300 + [A])          # tile 1023 -> tile 1025, all of tile 1024 PASS
            if nt == 2049:                                        # tile 2047 -> an ABORT marker that is the first key of tile 2048
                mixed(lay, 2048 * TILE - 50, rng)
                lay.marks["h0"] = lay.add([D] * 50 + [A])
        mixed(lay, m, rng)
        lay.marks["ntiles"] = nt
        out.append(lay.case("carry-%d-tiles" % nt))
    return out


def id_case():
    """d. producer ids 0, 1, 2^63 - 1, 2^63, 2^64 - 2 in partitions 0, 6, 2^31 - 1 and -1 with an outcome of their own in each;
    non-transactional batches and other control types of the same id in between; producerId -1 with and without the
    transactional bit, data and markers"""
    lay = Layout(seed=13)
    ids = (0, 1, (1 << 63) - 1, 1 << 63, (1 << 64) - 2)
    rp, rq, rf, rl = [], [], [], []
    for gi, p in enumerate((0, 6, (1 << 31) - 1, -1)):
        lay.add([D, A, N, C, X], part=p, pid=NOPID)              # takes part in nothing
        for qi, q in enumerate(ids):
            k = (gi * 5 + qi) % 4
            codes = [[D, N, D, X, D, A, D, N, C], [N, D, D, X, C, D, X, N], [D, D, N, N, A, X, D, D], [X, D, C, D, N, D]][k]
            offs = np.arange(len(codes)) * 10 + 100
            lay.add(codes, part=p, pid=q, offs=offs)
            if (gi + qi) % 3 == 0:                               # a range over the group's last data batches
                rp.append(p), rq.append(q), rf.append(int(offs[-3])), rl.append(int(offs[-1]))
    return lay.case("ids", range_table(rp, rq, rf, rl))


def range_case(pairs=40_000, seed=14, top=(1 << 63) - 1):
    """e. ~130 000 ranges over `pairs` (partition, producerId) pairs, half the ids with the top bit set, offsets up to
    2^63 - 1, every other gap between two ranges closed (a.last + 1 == b.first); per pair, batches at first - 1, first, last
    and last + 1 of its ranges, some pairs with a COMMIT marker behind them; and ids the table does not have"""
    rng = np.random.default_rng(seed)
    lay = Layout(seed=seed)
    pid = np.unique(rng.integers(0, 1 << 64, pairs, dtype=np.uint64, endpoint=False))
    part = rng.integers(0, 8, len(pid)).astype(np.int32)
    rp, rq, rf, rl = [], [], [], []
    for j in range(len(pid)):
        hi = j % 50 == 0                                          # the last range ends at the largest offset
        cuts = np.unique(rng.integers(1, 1 << 40, 2 * int(rng.integers(1, 7)))) + (top - (1 << 40) if hi else 0)
        k = len(cuts) // 2
        first, last = cuts[0:2 * k:2].copy(), cuts[1:2 * k:2].copy()
        last[:-1:2] = first[1::2][:len(last[:-1:2])] - 1          # every other gap closed
        if hi:
            last[-1] = top
        probes = np.unique(np.concatenate([first - 1, first, last, last[last < top] + 1]))
        codes = [D] * len(probes)
        offs = probes.tolist()
        if j % 3 == 0 and offs[-1] < top:
            codes.append(C)
            offs.append(offs[-1] + 1)
        lay.add(codes, part=int(part[j]), pid=int(pid[j]), offs=offs)
        if j % 7 == 0:                                            # an id next to it that the table does not have
            lay.add([D, D], part=int(part[j]), pid=int(pid[j]) ^ 1, offs=[int(first[0]), int(last[0])])
        rp += [part[j]] * k
        rq += [pid[j]] * k
        rf += first.tolist()
        rl += last.tolist()
    lay.add([D, D], part=-1, pid=5, offs=[3, 4])                  # below and above every pair of the table
    lay.add([D, D], part=9, pid=5, offs=[3, 4])
    return lay.case("ranges", range_table(rp, rq, rf, rl))


def refusal_cases():
    """f. a group whose baseOffsets are equal or decrease at one pair of sorted neighbours: inside a warp, across lanes 31 | 0,
    across threads 255 | 0 of two tiles, between a marker and the data batch behind it; one unreadable marker among 300 000
    good keys"""
    out = []
    for name, pos, codes, bump in (("order-in-warp", 5, [D, D, C], 0), ("order-lanes-31|0", 31, [D, D, C], -1),
                                   ("order-tiles-255|0", 255, [D, D, C], 0), ("order-marker-data", 600, [D, A, D, C], -1)):
        lay = Layout(seed=len(out))
        lay.fill_to(pos - (1 if len(codes) == 4 else 0))
        offs = 10 + np.arange(len(codes)) * 4
        offs[-2] = offs[-3] + bump                              # the pair (pos, pos + 1): equal or decreasing
        lay.marks["pair"] = lay.add(codes, offs=offs) + len(codes) - 3
        mixed(lay, 700, np.random.default_rng(3))
        out.append(lay.case(name))
    lay = Layout(seed=9)
    mixed(lay, 200_000, np.random.default_rng(4))
    lay.add([D, D, B])
    mixed(lay, 300_000, np.random.default_rng(5))
    out.append(lay.case("unreadable-marker"))
    return out


def depth_case(target=2_400_000, groups=3000, seed=15):
    """g. ~2.4 million keys in one call: transactions of 1 to 20 000 batches from a heavy-tailed law spread over `groups`
    (partition, producerId) groups of 16 partitions, 10 % aborted, 5 % left open, ranges for half of the aborted and the
    open ones, every group interleaved with every other batch by batch"""
    rng = np.random.default_rng(seed)
    L = np.minimum(20_000, (1.0 / rng.random(target // 8) ** 1.1).astype(np.int64))
    L = L[np.cumsum(L + 1) <= target]
    fate = rng.choice([C, A, 0], len(L), p=[0.85, 0.10, 0.05]).astype(np.uint8)
    g = np.sort(rng.integers(0, groups, len(L)))
    gpid = rng.integers(0, 1 << 64, groups, dtype=np.uint64, endpoint=False)
    gpart = rng.permutation(16)[rng.integers(0, 16, groups)].astype(np.int32)
    o = np.lexsort((gpid[g], gpart.view(np.uint32)[g]))          # groups in sorted order, transactions in theirs
    L, fate, g = L[o], fate[o], g[o]
    codes, t = txn_codes(L, fate)
    lay = Layout(seed=seed)
    lay.cols.append((codes, gpart[g][t], gpid[g][t], np.full(len(codes), -1, np.int64)))
    c = lay.case("depth")
    # ranges from the offsets the layout gave: [first data batch, last batch] of some aborted and open transactions
    w = c.want
    end = np.cumsum(L + (fate != 0))
    pick = np.flatnonzero((fate != C) & (rng.random(len(L)) < 0.5))
    first, last = w.batch[end[pick] - (L + (fate != 0))[pick]], w.batch[end[pick] - 1]
    c.ranges = range_table(gpart[g][pick], gpid[g][pick], c.off[first], c.off[last])
    return finish(c)


SMALL = [chain_case, edge_cases, id_case, refusal_cases]


def flat(makers):
    return [c for mk in makers for c in (lambda r: r if isinstance(r, list) else [r])(mk())]


# ---- CPU tests --------------------------------------------------------------------------------------------------------
def contract_of_topic(calls, ranges):
    """txn_contract over calls of test_log_txn's batches → (delivered [(p, record)], summed stats)"""
    table = [(p, q & NOPID, f, l) for p, rs in ranges.items() for q, f, l in rs]
    table = range_table(*zip(*table)) if table else no_ranges()
    out, stats = [], np.zeros(3, np.int64)
    for call in calls:
        kind = [NONE if (b.pid == -1 or (b.txn is None and not b.is_marker)) else (COMMIT if b.commit else ABORT) if b.is_marker else DATA
                for b in call]
        w = txn_contract([b.p for b in call], [b.pid & NOPID for b in call], [b.off for b in call], kind,
                         [0 if b.is_marker else len(b.recs) for b in call], table)
        assert w.err == 0
        out += [(b.p, r) for b, ab in zip(call, w.aborted) if not ab and not b.is_marker for r in b.recs]
        stats += w.stats
    return out, tuple(int(x) for x in stats)


@pytest.mark.parametrize("seed", [1, 2, 3, 4])
def test_restatement_agrees_with_the_rule_model_and_the_librdkafka_walk(seed):
    t = gen_topic(seed)
    whole = [b for p in t.batches for b in t.batches[p]]
    assert contract_of_topic([whole], {}) == rule_model([whole], {})
    for p in t.batches:
        got = [r for _, r in contract_of_topic([t.batches[p]], {})[0]]
        assert got == librdkafka_walk(t.segment(p), [(q, f) for q, f, _ in t.aborted[p]])
    # cut in two calls, with and without the index ranges
    cut = {p: len(t.batches[p]) // 2 for p in t.batches}
    calls = [[b for p in t.batches for b in t.batches[p][:cut[p]]], [b for p in t.batches for b in t.batches[p][cut[p]:]]]
    for ranges in ({}, t.aborted):
        assert contract_of_topic(calls, ranges) == rule_model(calls, ranges)
    # with the index the two calls deliver what the generator decided
    assert sorted(map(repr, contract_of_topic(calls, t.aborted)[0])) == sorted(repr((p, r)) for p in t.batches for r in t.truth(p))


def test_builder_reads_back():
    rng = np.random.default_rng(2)
    n = 5000
    code = rng.choice([D, A, C, N, X], n).astype(np.uint8)
    pid = rng.integers(0, 1 << 64, n, dtype=np.uint64, endpoint=False)
    pid[::17] = NOPID
    off = np.sort(rng.integers(0, 1 << 63, n))
    buf = build_batches(code, pid, off, np.arange(n, dtype=np.uint64) * 0x0101010101010101)
    got = kc.read_segment(buf.tobytes())
    assert len(got) == n
    for i, b in enumerate(got):
        ctrl = code[i] in (A, C, X)
        assert (b.base_offset, b.producer_id & NOPID, b.count) == (off[i], pid[i], 1)
        assert b.attributes == (0x30 if ctrl else 0 if code[i] == N else 0x10)
        key = b.records[0][2]
        assert key == (struct.pack(">hh", 0, {A: 0, C: 1, X: 2}[code[i]]) if ctrl else struct.pack(">Q", i * 0x0101010101010101 & NOPID))
        assert b.records[0][0] == off[i] and b.records[0][3] == (6 if ctrl else 2)
    bad = kc.read_segment(build_batches([B], [7], [1], [0]).tobytes())[0]
    assert bad.records[0][2] == struct.pack(">hh", 1, 2) and bad.attributes == 0x30


def placed(c, got_batch=None):
    """the case reaches the edges it names; from the restatement's sorted order, or from the probe's"""
    w, mk = c.want, c.marks
    batch = w.batch if got_batch is None else got_batch
    assert np.array_equal(batch, w.batch), c.name
    k = c.kind[batch]
    if "chains" in mk:
        for start, L, end, mod, pos in mk["chains"]:
            assert start % mod == pos, (start, L, mod, pos)
            assert (k[start:start + L] == DATA).all() and (w.group[start:start + L] == w.group[start]).all()
            assert (start == 0 or w.group[start - 1] != w.group[start]) and w.decider[start] == start + L - (0 if end else 1)
            assert w.verdict[start] == end
        d = depth(w)
        assert d.warps >= {-1, 0, 1, 2, 3, 4, 5, 6} and d.tiles >= {0, 1, 2, 19}, (d.warps, d.tiles)
        lanes = {(L, e, s % 32) for s, L, e, _, _ in mk["chains"]}
        assert all((L, e, lane) in lanes for L in range(1, 71) for e in (A, C, 0) for lane in range(32))
        at = {(L, e, s % TILE) for s, L, e, _, _ in mk["chains"]}
        assert all((L, e, p) in at for L in list(range(1, 71)) + list(LONG) for e in (A, C, 0) for p in (0, 1, 31, 32, 254, 255))
    if "ends" in mk:
        assert w.m == mk["m"] and [e % CHUNK for e in mk["ends"]] == [31, 255, 256 + 31, 3 * TILE - 1, CHUNK - 1, (w.m - 1) % CHUNK]
        assert mk["ends"][-1] == w.m - 1
        for e in mk["ends"]:
            assert k[e] == DATA and w.verdict[e] == UNDECIDED and w.res[e] == UNDECIDED
            assert e == w.m - 1 or (k[e + 1] == ABORT and w.group[e + 1] != w.group[e])
    if "ntiles" in mk:
        assert len(w.tile_head) == mk["ntiles"]
    if "into" in mk:
        s = mk["into"]
        assert (s // TILE, w.decider[s] // TILE) == (1023, 1024) and w.carry[1023] == ABORT and w.tile_head[1024] == ABORT
    if "over" in mk:
        s = mk["over"]
        assert (s // TILE, w.decider[s] // TILE) == (1023, 1025) and w.tile_head[1024] == PASS and (w.res[1024 * TILE:1025 * TILE] == PASS).all()
    if "through" in mk:
        s = mk["through"]
        assert (s // CHUNK, w.decider[s] // CHUNK) == (0, 2) and (w.tile_head[1024:2049] == PASS).all()
        assert depth(w).cross_chunk > CHUNK
    if "h0" in mk:
        s = mk["h0"]
        assert (s // TILE, w.decider[s]) == (2047, 2048 * TILE) and w.tile_head[2048] == ABORT and w.carry[2047] == ABORT
    if "pair" in mk:
        i = mk["pair"]
        assert w.err == ERR_ORDER and w.group[i] == w.group[i + 1] and c.off[batch[i + 1]] <= c.off[batch[i]]
        assert i % TILE == {"order-in-warp": 5, "order-lanes-31|0": 31, "order-tiles-255|0": 255, "order-marker-data": 600 % TILE}[c.name]
        # and it is the only such pair
        so, same = c.off[batch], w.group[1:] == w.group[:-1]
        assert np.flatnonzero(same & (so[1:] <= so[:-1])).tolist() == [i]


def test_hand_built_cases_reach_the_edges_they_name():
    cases = flat(SMALL + [carry_cases])
    for c in cases:
        placed(c)
    by = {c.name: c for c in cases}
    assert by["unreadable-marker"].bad_marker and by["unreadable-marker"].want.m >= 300_000
    w = by["ids"].want
    assert w.stats[0] > 0 and w.stats[2] > 0 and (by["ids"].kind[by["ids"].pid == NOPID] == NONE).all()
    # the cases small enough for the quadratic model agree with it
    for c in (by["ids"], by["order-in-warp"]):
        if c.want.err:
            continue
        calls, ranges = as_model(c)
        assert contract_of_topic(calls, ranges)[1] == rule_model(calls, ranges)[1] == c.want.stats


def as_model(c):
    """a case as test_log_txn's batches and ranges, for rule_model"""
    from test_log_txn import Bt
    sgn = lambda q: int(q) - (1 << 64) if int(q) >> 63 else int(q)
    call = [Bt(int(c.part[i]), int(c.off[i]), sgn(c.pid[i]), 0, 1 if c.code[i] == D else None, [] if c.ctrl[i] else [(TS0, b"k", 2)],
               (c.code[i] == C) if c.code[i] in (A, C) else None) for i in range(len(c.code)) if c.code[i] != X]
    ranges = {}
    for r in c.ranges:
        ranges.setdefault(int(r["part"]), []).append((sgn(r["pid"]), int(r["first"]), int(r["last"])))
    return [call], ranges


def test_range_case_covers_its_edges():
    c = range_case(pairs=2000)
    r, w = c.ranges, c.want
    assert (r["pid"] >> np.uint64(63)).any() and (r["last"] == (1 << 63) - 1).any()
    same = (r["part"][1:] == r["part"][:-1]) & (r["pid"][1:] == r["pid"][:-1])
    assert (same & (r["last"][:-1] + 1 == r["first"][1:])).any() and not (same & (r["last"][:-1] >= r["first"][1:])).any()
    d = c.kind == DATA
    assert 0 < w.aborted.sum() < d.sum()
    assert (w.aborted[w.batch] & (w.verdict == COMMIT)).any()     # a COMMIT marker and a covering range: aborted
    # against a dictionary of the ranges, batch by batch
    table = {}
    for x in r:
        table.setdefault((int(x["part"]), int(x["pid"])), []).append((int(x["first"]), int(x["last"])))
    for b in np.flatnonzero(d):
        hit = any(f <= c.off[b] <= l for f, l in table.get((int(c.part[b]), int(c.pid[b])), ()))
        assert hit == w.aborted[b], b


# ---- GPU tests --------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_chains_edges_ids_and_refusals(probe):
    """a, b, d, f"""
    cases = flat(SMALL)
    for c, g in zip(cases, run_probe(probe, cases)):
        if g.ran:
            placed(c, g.sorted["batch"].astype(np.int64))
        check(c, g)


@pytest.mark.gpu
def test_carry_chunks(probe):
    """c"""
    cases = carry_cases()
    for c, g in zip(cases, run_probe(probe, cases)):
        placed(c, g.sorted["batch"].astype(np.int64))
        check(c, g)


@pytest.mark.gpu
def test_range_search(probe):
    """e, the device's search: a table deep enough for 17 steps"""
    c = range_case()
    assert len(c.ranges) > 1 << 16
    g, = run_probe(probe, [c])
    check(c, g)
    assert c.want.stats[0] > 100_000


@pytest.mark.gpu
def test_at_depth(probe):
    """g"""
    c = depth_case()
    d = depth(c.want)
    assert c.want.m > 8 * CHUNK and len(c.ranges) > 1000
    assert d.cross_warp > 500_000 and d.cross_tile > 100_000 and d.cross_chunk > 1000, (d.cross_warp, d.cross_tile, d.cross_chunk)
    g, = run_probe(probe, [c])
    check(c, g)
    assert c.want.stats[0] > 0 and c.want.stats[2] > 0


@pytest.mark.gpu
def test_registered_ranges_through_the_public_abi():
    """e, the host's sort and merge: the table registered over several calls in shuffled order, with duplicates and ranges
    cut into overlapping pieces; every probed offset a single-record batch with a key and value length of its own"""
    rng = np.random.default_rng(21)
    P = 4
    c = range_case(pairs=300, seed=22, top=1 << 62)
    c.part %= P
    c.ranges["part"] %= P
    keep = c.part >= 0
    pieces = []
    for r in c.ranges:
        p, q, f, l = int(r["part"]), int(r["pid"]), int(r["first"]), int(r["last"])
        mid = f + (l - f) // 2
        pieces += [(p, q, f, l)] if l - f < 2 else [(p, q, f, min(l, mid + 1)), (p, q, mid, l), (p, q, f, mid)]
    pieces += [pieces[i] for i in rng.integers(0, len(pieces), 200)]
    sgn = lambda q: q - (1 << 64) if q >> 63 else q
    with KtaEngine(P, count_alive_keys=True, now=NOW, isolation_level="read_committed") as e:
        for chunk in np.array_split(rng.permutation(len(pieces)), 9):
            for p in range(P):
                e.push_txn_index(p, kc.txn_index([(sgn(pieces[i][1]), pieces[i][2], pieces[i][3]) for i in chunk if pieces[i][0] == p]))
        segs, recs = {p: [] for p in range(P)}, {p: [] for p in range(P)}
        for b in np.flatnonzero(keep):
            p, rec = int(c.part[b]), (TS0 + int(b), b"key-%d" % (b % 700), int(b) % 53)
            if c.ctrl[b]:
                segs[p].append(kc.marker(int(c.off[b]), sgn(int(c.pid[b])), 0, c.code[b] == C, TS0))
            else:
                segs[p].append(kc.txn_batch(int(c.off[b]), rec[0], [(0, 0, rec[1], rec[2])], pid=sgn(int(c.pid[b]))))
                recs[p].append((b, rec))
        want = txn_contract(c.part[keep], c.pid[keep], c.off[keep], c.kind[keep], c.records0[keep], c.ranges)
        ab = np.zeros(len(c.code), bool)
        ab[np.flatnonzero(keep)] = want.aborted
        assert want.err == 0 and 0 < want.stats[0] < int((c.kind[keep] == DATA).sum())
        delivered = [(p, *rec) for p in range(P) for b, rec in recs[p] if not ab[b]]
        assert e.push_log_segments([(p, b"".join(segs[p])) for p in range(P)]) == len(delivered)
        e.finalize()
        assert e.log_txn_stats() == want.stats
        assert_parity(e, oracle_in_order(delivered), P, check_alive=True)


@pytest.mark.gpu
@pytest.mark.parametrize("entry", LOG_ENTRIES)
def test_long_transactions_through_the_entry_points(entry):
    """h. three partitions with transactions of 300, 600 and 70 000 batches among short ones, aborted and committed, -c on"""
    P = 3
    rng = np.random.default_rng(31)
    L = rng.choice([1, 2, 4, 9], 400)
    L[[20, 170, 333]], L[[90, 250]] = (300, 600, 70_000), (600, 300)
    fate = rng.choice([C, A, 0], len(L), p=[0.7, 0.25, 0.05]).astype(np.uint8)
    fate[[20, 170, 333, 90, 250]] = (A, C, A, A, C)
    grp = np.sort(rng.integers(0, 12, len(L)))                    # 12 (partition, producerId) groups, their transactions in a row
    codes, t = txn_codes(L, fate)
    lay = Layout(seed=31)
    lay.cols.append((codes, (grp[t] % P).astype(np.int32), (grp[t] // P + 40).astype(np.uint64), np.full(len(codes), -1, np.int64)))
    c = lay.case("long")
    c.keyid = np.arange(len(c.code), dtype=np.uint64) % 5000
    buf = build_batches(c.code, c.pid, c.off, c.keyid)
    parts = {p: [SimpleNamespace(p=p, raw=buf[b].tobytes(), i=int(b)) for b in np.flatnonzero(c.part == p)] for p in range(P)}
    d = depth(c.want)
    assert max(d.tiles) > 250 and d.tiles >= {0, 1} and c.want.stats[0] > 70_000    # chains behind up to ~270 all-PASS tiles
    with KtaEngine(P, count_alive_keys=True, now=NOW, isolation_level="read_committed") as e:
        total, order = scan_log(e, entry, parts)
        e.finalize()
        # one call of all partitions, or one per partition: the rule looks at a batch's own partition only
        want = [(b.p, TS0, struct.pack(">Q", int(c.keyid[b.i])), 2) for b in order if not c.ctrl[b.i] and not c.want.aborted[b.i]]
        assert total == len(want)
        assert e.log_txn_stats() == c.want.stats
        assert_parity(e, oracle_in_order(want), P, check_alive=True)
