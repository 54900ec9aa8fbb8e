"""The fused scan at depth: every scan_kernel instance, bit-exact against the torch restatement of its outputs (scan_ref.py).

"At depth" means a batch long enough that every warp works through at least 64 tiles of its own (tile t belongs to warp
t mod warps), with a tail tile and a number of tiles the warps do not divide.  Only then does a warp reuse each stage and
flip each mbarrier phase many times, turn its ring of key bounds over (every 32nd tile), refresh and re-read the HLL floor
(every 4th and 16th tile), re-probe for run-structured input (every 16th) and drain its split sums (every 8th).  The depth is
computed from the device's SM count with the most warps a launch can have (32 in counters mode, 16 in the hashing modes),
so it holds whatever shape the launch picks.  The reference runs on the device next to the kernel; keys of 4 KiB or more
are hashed by oracle/ instead (a byte loop over a 1 MiB key is a million steps in torch).

Case ids name the instance they launch: mode, counters in shared or global memory, sharded, capture."""
import gc
import os
import re

import numpy as np
import pytest
import torch

import scan_ref as R
from kafka_topic_analyzer_b200 import KtaEngine, synth
from kafka_topic_analyzer_b200 import _native as N
from feed import Topic, alive_import, capture_hashes, device, push_host, rekey, scan, settle, take
from oracle_lib import COUNTERS, fnv32 as oracle_fnv32

NOW = (4102444800, 123456789)
T = N.KTA_KEY_TILE
DEPTH = 64                                              # tiles per warp, at the most warps a launch can have
MAX_WARPS = {"counters": 32, "hll": 16, "exact": 16}
HLL_P = 12
GIB = 1 << 30
PEAK_GIB = 16                                           # the torch side of every case stays under this


# ------------------------------------------------------------------------------------------------
# launch facts restated from the host code (scan_shape, create_impl)
# ------------------------------------------------------------------------------------------------
def sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def smem_counters(columns):
    """create_impl: counters in shared memory iff their rows and 8 warps of two smallest key-only stages fit the opt-in"""
    optin = getattr(torch.cuda.get_device_properties(0), "shared_memory_per_block_optin", 227 * 1024)
    rows = (columns * 70 * 4 + 127) // 128 * 128 + 128
    return rows + 8 * (128 + 2 * (T * 18 + 32)) <= optin


def columns(P, world, rank):
    return (P - rank + world - 1) // world


def inst(mode, smem, shard=False, capture=False):
    return "%s-%s%s%s" % (mode, "smem" if smem else "global", "-shard" if shard else "", "-capture" if capture else "")


def depth_n(mode, tail=77):
    """records: 64 tiles for each of the most warps the launch can have, one tile more, the last one `tail` records long"""
    return DEPTH * MAX_WARPS[mode] * sms() * T + tail


def assert_depth(n, mode, tail=True):
    warps = MAX_WARPS[mode] * sms()
    ntiles = -(-n // T)
    assert ntiles // warps >= DEPTH, (n, ntiles, warps)
    assert ntiles % warps, (ntiles, warps)                   # the last round of the key-bound ring is partial
    if tail:
        assert n % T, n                                      # a tail tile
    return ntiles / warps


def need(gib):
    free, _ = torch.cuda.mem_get_info()
    if free < gib * GIB:
        pytest.skip("needs %.0f GiB of free device memory, %.1f GiB free" % (gib, free / GIB))


@pytest.fixture(autouse=True)
def _budget(request):
    if request.node.get_closest_marker("gpu") is None:
        yield
        return
    torch.cuda.reset_peak_memory_stats()
    yield
    peak = torch.cuda.max_memory_allocated()
    gc.collect()
    torch.cuda.empty_cache()
    print("peak %.2f GiB" % (peak / GIB))
    assert peak < PEAK_GIB * GIB, peak


# ------------------------------------------------------------------------------------------------
# topics in HBM
# ------------------------------------------------------------------------------------------------
def generate(n, P, run_len=1, **kw):
    """the first n records of a synthetic topic, generated in HBM"""
    unit = P * run_len
    spec = synth.make_spec(-(-n // unit) * unit, P, run_len=run_len, **kw)
    d = synth.DeviceTopic(spec, count=n)
    return Topic(d.partition, d.ts_ms, d.key_len, d.value_len, d.key_bytes, d.key_bytes_len)


def long_fn(kb):
    """keys of LONG_KEY bytes or more, hashed by the C restatement in oracle/"""
    def f(off, kl):
        out = [oracle_fnv32(kb[o: o + n].cpu().numpy().tobytes()) for o, n in zip(off.tolist(), kl.tolist())]
        return torch.tensor(out, dtype=torch.int64)
    return f


# ------------------------------------------------------------------------------------------------
# engine side
# ------------------------------------------------------------------------------------------------
def engine(mode, P, shard=None, hll_p=HLL_P, **kw):
    if mode == "counters":
        return KtaEngine(P, now=NOW, shard=shard, **kw)
    return KtaEngine(P, count_alive_keys=mode == "exact", hll_precision=hll_p, now=NOW, shard=shard, **kw)


def first_mismatch(got, want):
    bad = np.nonzero(np.asarray(got) != np.asarray(want))[0]
    return None if bad.size == 0 else (int(bad[0]), np.asarray(got)[bad[0]], np.asarray(want)[bad[0]], int(bad.size))


def check(e, mm, P, regs=None, alive=None):
    """every counter and histogram row of every partition, the globals, the HLL registers, the alive count and occupancy"""
    for i, name in enumerate(COUNTERS):
        got = [e.counter(i, p) for p in range(P)]
        assert got == mm[name].tolist(), (name, first_mismatch(got, mm[name].cpu().numpy()))
    for which, name in ((0, "khist"), (1, "vhist")):
        got = np.stack([e.hist(which, p) for p in range(P)]).astype(np.int64)
        want = mm[name].cpu().numpy()
        assert np.array_equal(got, want), (name, first_mismatch(got.reshape(-1), want.reshape(-1)))
    m = e.message_metrics
    assert (m.smallest_message(), m.largest_message(), m.overall_size(), m.overall_count()) == \
        (mm["smallest"], mm["largest"], mm["overall_size"], mm["overall_count"])
    assert m.earliest_message() == R.earliest(mm, NOW) and m.latest_message() == R.latest(mm)
    assert e.bad_partition_records() == mm["bad"]
    if regs is not None:
        got = e.hll_registers().astype(np.int64)
        want = regs.cpu().numpy()
        assert np.array_equal(got, want), ("hll", first_mismatch(got, want))
    if alive is not None:
        assert e.alive_keys() == alive[0]
        assert e.alive_table_stats()[1] == alive[1]


def reference(mode, t, P, hll_p=HLL_P, mask=None, seq=None):
    """(metrics, registers, (alive, distinct), hashes) of the records of t where mask holds (all when None)"""
    cols = [t.partition, t.ts_ms, t.key_len, t.value_len]
    if mask is not None:
        cols = [c[mask] for c in cols]
    mm = R.message_metrics(P, *cols)
    if mode == "counters":
        return mm, None, None, None
    h = R.fnv32(t.key_len, t.keys, long_fn(t.keys))
    part, kl, vl = t.partition, t.key_len, t.value_len
    sel = torch.ones_like(kl, dtype=torch.bool) if mask is None else mask
    inrange = (part >= 0) & (part < P) & sel
    if mode == "hll":
        return mm, R.hll_regs(h, R.stream_mask(part, kl, vl, P) & sel, hll_p), None, h
    ah, distinct = R.alive_hashes(h, kl, vl, seq=seq, mask=inrange)
    return mm, R.hll_regs(ah, None, hll_p), (int(ah.numel()), distinct), h


def run(mode, t, P, hll_p=HLL_P, capture=False, host=False, cols=None, key_bytes=None, **kw):
    """one unsharded scan of t, checked against the reference; with capture, every record's hash as well"""
    assert smem_counters(P) == kw.pop("smem")
    mm, regs, alive, h = reference(mode, t, P, hll_p)
    with engine(mode, P, hll_p=hll_p, **kw) as e:
        out = None
        if capture:
            out = torch.full((t.n,), -1, dtype=torch.int32, device="cuda")
            capture_hashes(e, out)
        if host:
            push_host(e, t)
        else:
            scan(e, t, cols=cols, key_bytes=key_bytes)
        e.finalize()
        if capture:
            capture_hashes(e, None)
            got = out.to(torch.int64) & R.M32
            bad = torch.nonzero(got != h).flatten()
            if bad.numel():
                r = int(bad[0])
                pytest.fail("captured hash of %d records differs, first record %d (tile %d): %#x, want %#x"
                            % (bad.numel(), r, r // T, int(got[r]), int(h[r])))
        check(e, mm, P, regs, alive)
    return h


# ------------------------------------------------------------------------------------------------
# 1. the instance matrix: every SCAN_KERNELS entry at depth
# ------------------------------------------------------------------------------------------------
# (P, world): counters in shared memory (64 columns, 32 per shard), in global memory (800, 100 000 columns, 50 000 per
# shard), and 2101 partitions over 3 shards: 701 / 700 / 700 columns, all in global memory
LAYOUTS = [(64, 1, True), (64, 2, True), (800, 1, False), (100_000, 1, False), (100_000, 2, False), (2101, 3, False)]
MATRIX = [(mode, P, world, smem) for mode in ("counters", "hll", "exact") for P, world, smem in LAYOUTS]
CAPTURE = [(mode, P, smem) for mode in ("hll", "exact") for P, smem in ((64, True), (800, False))]


@pytest.mark.gpu
@pytest.mark.parametrize("mode,P,world,smem", MATRIX,
                         ids=["%s/P%d-w%d" % (inst(m, s, w > 1), P, w) for m, P, w, s in MATRIX])
def test_instance_at_depth(mode, P, world, smem):
    if world == 1:
        need(8)
        n = depth_n(mode)
        assert_depth(n, mode)
        t = generate(n, P, key_mode=2, tombstone_per_10k=2000, null_key_per_10k=150, ts_missing_per_10k=20)
        run(mode, t, P, smem=smem)
        return
    need(14)
    # shard r: the first m_r of the records of partitions p = r (mod world); m_r differ, none a multiple of 128
    m = [depth_n(mode) + 13 * r for r in range(world)]
    # shard r holds columns(P, world, r) of every P consecutive records
    # (counters mode reads no key: 16-byte keys keep the generator's key buffer small)
    t = generate(max(-(-(m[r] + 2 * P) * P // columns(P, world, r)) for r in range(world)), P,
                 key_mode=0 if mode == "counters" else 2, tombstone_per_10k=2000, null_key_per_10k=150, ts_missing_per_10k=20)
    keep = torch.zeros(t.n, dtype=torch.bool, device="cuda")
    idx = []
    for r in range(world):
        i = torch.nonzero(t.partition % world == r).flatten()
        assert i.numel() >= m[r]
        idx.append(i[: m[r]])
        keep[idx[-1]] = True
        assert smem_counters(columns(P, world, r)) == smem
    mm, regs, alive, _ = reference(mode, t, P, mask=keep)
    engines = [engine(mode, P, shard=(r, world)) for r in range(world)]
    try:
        words = engines[0].merge_words(world)
        total = torch.zeros(words, dtype=torch.int64, device="cuda")
        lists = []
        for r, e in enumerate(engines):
            s = take(t, idx[r]) if mode != "counters" else \
                Topic(*(c[idx[r]] for c in (t.partition, t.ts_ms, t.key_len, t.value_len)), t.key_bytes, 0)
            assert_depth(s.n, mode)
            scan(e, s, seq=s.seq if mode == "exact" else None)
            if mode != "exact":
                e.finalize()
            buf = torch.zeros(words, dtype=torch.int64, device="cuda")
            settle()
            e.merge_export(r, world, buf)               # returns once the engine's stream has written buf
            total += buf
            if mode == "exact":
                cnt = e.alive_export_count()
                h = torch.zeros(cnt, dtype=torch.int32, device="cuda")
                st = torch.zeros(cnt, dtype=torch.int64, device="cuda")
                settle()
                assert e.alive_export(h, st, cnt) == cnt
                e.sync()
                lists.append((h, st, cnt))
            del s
        e0 = engines[0]
        settle()
        e0.merge_import(world, total)
        for h, st, cnt in lists[1:]:
            alive_import(e0, h, st, cnt)
        e0.finalize()
        check(e0, mm, P, regs, alive)
    finally:
        for e in engines:
            e.close()


@pytest.mark.gpu
@pytest.mark.parametrize("mode,P,smem", CAPTURE, ids=["%s/P%d" % (inst(m, s, capture=True), P) for m, P, s in CAPTURE])
def test_capture_instance_at_depth(mode, P, smem):
    """every captured hash equals the reference's, record by record over the whole batch (in exact mode the tiles are
    walked newest first, so the tail tile is the first one scanned)"""
    need(8)
    n = depth_n(mode)
    assert_depth(n, mode)
    t = generate(n, P, key_mode=2, tombstone_per_10k=2000, null_key_per_10k=150)
    run(mode, t, P, capture=True, smem=smem)


# ------------------------------------------------------------------------------------------------
# 2. stage bookkeeping: staged and unstaged keys and headers, and keys that do not fit their stage
# ------------------------------------------------------------------------------------------------
ALIGN = [(hdr, key) for hdr in (0, 1) for key in (0, 1)]
STAGING = {(0, 0): "keys+headers", (1, 0): "keys-only", (0, 1): "headers-only", (1, 1): "neither"}


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["hll", "exact"], ids=[inst("hll", True), inst("exact", True)])
@pytest.mark.parametrize("hdr_shift,key_shift", ALIGN, ids=[STAGING[a] for a in ALIGN])
def test_stage_bookkeeping_at_depth(mode, hdr_shift, key_shift):
    """16-byte keys at 64 partitions from aligned and misaligned columns and key buffers: a misaligned column leaves the
    headers to global loads; a misaligned key buffer (stage_limit 0) leaves the keys to global loads, and with the headers
    staged the stage's wait happens in load_headers"""
    need(8)
    n = depth_n(mode)
    assert_depth(n, mode)
    t = generate(n, 64, key_mode=0, distinct_keys=1_000_000, tombstone_per_10k=1500)
    cols = [device(c, hdr_shift) for c in (t.partition, t.ts_ms, t.key_len, t.value_len)]
    kb = device(t.key_bytes, key_shift)
    run(mode, t, 64, cols=cols, key_bytes=kb, smem=True)


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["hll", "exact"], ids=[inst("hll", True), inst("exact", True)])
def test_stages_arrive_irregularly_at_depth(mode):
    """about every 40th tile holds one ~30 KB key that fits no stage: that tile is read from global memory, so a warp's
    stages are filled irregularly and each stage's phase bit must follow its own count"""
    need(8)
    n = depth_n(mode)
    assert_depth(n, mode)
    t = generate(n, 64, key_mode=0, distinct_keys=1_000_000, tombstone_per_10k=1500)
    ntiles = -(-n // T)
    rng = np.random.default_rng(40)
    tiles = np.nonzero(rng.random(ntiles) < 1 / 40)[0]
    rows = np.minimum(tiles * T + rng.integers(0, T, size=tiles.size), n - 1)
    kl = t.key_len.clone()
    kl[torch.from_numpy(rows).cuda()] = torch.from_numpy(30_000 + rng.integers(0, 500, size=rows.size)).to(torch.int32).cuda()
    t = rekey(t, kl)
    assert int((t.key_len >= 16384).sum()) == rows.size >= ntiles // 50
    run(mode, t, 64, smem=True)


# ------------------------------------------------------------------------------------------------
# 3. key shapes, every hash captured
# ------------------------------------------------------------------------------------------------
SHAPES = ["ascii", "ragged", "fixed17", "fixed16"]


@pytest.mark.gpu
@pytest.mark.parametrize("shape", SHAPES, ids=["%s/%s" % (inst("hll", True, capture=True), s) for s in SHAPES])
def test_key_shapes_at_depth(shape):
    """ASCII keys (5-12 B) and 0-40 B ragged keys with nulls reach the packed short-key offsets and the FNV of staged keys
    with a lead, in a key stage sized from the mean; 17-byte keys the fixed-length path with per-key reads; 16-byte keys
    the LDS.128 path, from tiles without nulls (multiply offsets) and with nulls (ballot offsets)"""
    need(8)
    n = depth_n("hll")
    assert_depth(n, "hll")
    km = {"ascii": 1, "ragged": 2, "fixed17": 2, "fixed16": 0}[shape]
    t = generate(n, 64, key_mode=km, distinct_keys=2_000_000, null_key_per_10k=100)
    if shape == "fixed17":
        t = rekey(t, torch.where(t.key_len >= 0, 17, -1).to(torch.int32))
    if shape == "fixed16":
        nt = -(-n // T)
        nulls = torch.cat([(t.key_len < 0), torch.zeros(nt * T - n, dtype=torch.bool, device="cuda")]).view(nt, T).any(1)
        assert 0.1 < float(nulls.float().mean()) < 0.9        # both kinds of tiles, many of each
    run("hll", t, 64, capture=True, smem=True)


# ------------------------------------------------------------------------------------------------
# 4. run-structured counters
# ------------------------------------------------------------------------------------------------
RUNS = [(mode, run_len) for mode in ("counters", "hll") for run_len in (3000, 100)]


@pytest.mark.gpu
@pytest.mark.parametrize("mode,run_len", RUNS, ids=["%s/run%d" % (inst(m, True), r) for m, r in RUNS])
def test_run_structured_counters_at_depth(mode, run_len):
    """runs of 3000 records (whole tiles in one partition) and of 100 (rows across a run boundary: two groups).  Values of
    2^24 and 2^26 and more sprinkled through the runs make the whole-tile and per-row reductions fall back mid-run; tiles
    of such values only switch the run probe off until it is re-probed"""
    need(8)
    n = depth_n(mode)
    assert_depth(n, mode)
    t = generate(n, 64, run_len=run_len, key_mode=0, distinct_keys=1_000_000, tombstone_per_10k=800)
    g = torch.Generator(device="cuda").manual_seed(run_len)
    u = torch.rand(n, device="cuda", generator=g)
    vl = t.value_len
    vl[u < 0.002] = (1 << 24) + 5
    vl[(u >= 0.002) & (u < 0.003)] = (1 << 26) + 11
    nt = -(-n // T)
    big_tiles = torch.nonzero(torch.rand(nt, device="cuda", generator=g) < 0.02).flatten()
    rows = (big_tiles[:, None] * T + torch.arange(T, device="cuda")).flatten()
    vl[rows[rows < n]] = (1 << 27) + 3
    assert ((vl >= (1 << 24)) & (vl < (1 << 26))).any() and (vl >= (1 << 26)).any()
    run(mode, t, 64, smem=True)


# ------------------------------------------------------------------------------------------------
# 5. the HLL floor
# ------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("p", [4, 6, 10, 16], ids=["%s/p%d" % (inst("hll", True), p) for p in (4, 6, 10, 16)])
def test_hll_floor_at_depth(p):
    """in-stream sketches of over a million distinct keys: small sketches fill up early, so the floor filters most of the
    scan, and a skip rule off by one bit shows in the registers"""
    need(8)
    n = depth_n("hll")
    assert_depth(n, "hll")
    t = generate(n, 64, key_mode=0, distinct_keys=1_500_000, tombstone_per_10k=1000)
    h = run("hll", t, 64, hll_p=p, smem=True)
    mask = R.stream_mask(t.partition, t.key_len, t.value_len, 64)
    assert torch.unique(h[mask]).numel() >= 1_000_000
    if p <= 6:
        assert int(R.hll_regs(h, mask, p).min()) >= 8


# ------------------------------------------------------------------------------------------------
# 6. the alive-key table
# ------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("shape", ["c1", "zipf"], ids=["%s/%s" % (inst("exact", True), s) for s in ("c1", "zipf")])
def test_exact_at_depth(shape):
    """C1's shape with -c (1e6 distinct keys, 25 % tombstones) and Zipf keys: alive count, occupancy = distinct reference
    hashes, and the alive set's registers"""
    need(8)
    n = depth_n("exact")
    assert_depth(n, "exact")
    t = generate(n, 64, key_mode=0, distinct_keys=1_000_000, tombstone_per_10k=2500, null_key_per_10k=0,
                 zipf_keys=shape == "zipf")
    run("exact", t, 64, smem=True)


@pytest.mark.gpu
def test_exact_three_batches_at_depth():
    """exact-smem: three device batches into one handle, cut at a tile boundary and inside a tile, the later ones
    continuing the handle's seq; each batch at depth"""
    need(10)
    a = (DEPTH * MAX_WARPS["exact"] * sms() + 1) * T                # tile-aligned cut
    b = a + depth_n("exact")                                        # a cut inside a tile
    n = b + depth_n("exact", tail=51)
    t = generate(n, 64, key_mode=2, distinct_keys=1_000_000, tombstone_per_10k=2500, null_key_per_10k=100)
    mm, regs, alive, _ = reference("exact", t, 64)
    off = R.key_offsets(t.key_len)
    with engine("exact", 64) as e:
        for i, (lo, hi) in enumerate(((0, a), (a, b), (b, n))):
            assert_depth(hi - lo, "exact", tail=i > 0)
            k0 = int(off[lo]) if lo < n else t.kbl
            part = Topic(t.partition[lo:hi], t.ts_ms[lo:hi], t.key_len[lo:hi], t.value_len[lo:hi], t.key_bytes[k0:],
                         (int(off[hi]) if hi < n else t.kbl) - k0)
            scan(e, part, seq_base=0 if i == 0 else None)
        e.finalize()
        check(e, mm, 64, regs, alive)


# ------------------------------------------------------------------------------------------------
# 7. keys of 1 MiB and more
# ------------------------------------------------------------------------------------------------
MIB = 1 << 20
WIDE_WARPS = 64


def wide_topic(mode):
    """Ragged keys with wide tiles at the first tile of 64 warps (the first tiles scanned: the newest in exact mode), each
    warp scanning at least 2 x 4 ordinary tiles after it, so the stage a wide tile used as scratch is refilled by later
    bulk copies.  Warp w's wide tile, by w mod 4: one key of 2^20 + 1 B among ragged ones; two such keys; a longest key of
    2^20 - 1 B (still the 32-bit path); a longest key of 2^20 B.  Warp 64's first tile: 32 keys of 2^20 B, the rest null
    (one length, too long for the fixed-length path)."""
    warps = MAX_WARPS[mode] * sms()
    n = 9 * warps * T + 77
    t = generate(n, 64, key_mode=2, distinct_keys=200_000, tombstone_per_10k=1500, null_key_per_10k=100)
    ntiles = -(-n // T)
    phys = (lambda w: ntiles - 1 - w) if mode == "exact" else (lambda w: w)
    kl = t.key_len.cpu().numpy().copy()
    for w in range(WIDE_WARPS):
        r0 = phys(w) * T
        rows = min(T, n - r0)
        lead = (w * 37) % rows
        kind = w % 4
        if kind == 0:
            kl[r0 + lead] = MIB + 1
        elif kind == 1:
            kl[r0 + lead] = kl[r0 + (lead + 61) % rows] = MIB + 1
        else:
            kl[r0 + lead] = MIB - 1 if kind == 2 else MIB
    r0 = phys(WIDE_WARPS) * T
    kl[r0: r0 + T] = -1
    kl[r0: r0 + 32] = MIB
    t = rekey(t, torch.from_numpy(kl).cuda())
    assert int((t.key_len >= MIB).sum()) == 16 + 32 + 16 + 32
    return t


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["counters", "hll", "exact"])
@pytest.mark.parametrize("entry", ["device", "host"])
def test_wide_keys(mode, entry):
    """tiles whose longest key is 1 MiB or more are hashed by the 64-bit wide path into the warp's scratch in a stage;
    every later tile of those warps must still hash, count and stamp exactly"""
    need(6)
    t = wide_topic(mode)
    assert t.kbl > 100 * MIB and -(-t.n // T) // (MAX_WARPS[mode] * sms()) >= 2 * 4 + 1
    run(mode, t, 64, host=entry == "host", ring_key_bytes=64 * MIB, smem=True)


# ------------------------------------------------------------------------------------------------
# every instance the library launches is named by a case above
# ------------------------------------------------------------------------------------------------
def _case_ids():
    ids = ["%s/P%d-w%d" % (inst(m, s, w > 1), P, w) for m, P, w, s in MATRIX]
    ids += ["%s/P%d" % (inst(m, s, capture=True), P) for m, P, s in CAPTURE]
    return ids


def test_every_scan_kernel_instance_has_a_depth_case():
    src = open(os.path.join(N.CSRC, "kta_api.cu")).read()
    table = src[src.index("SCAN_KERNELS[2][2][3][2] = {"):]
    table = table[: table.index("};")]
    found = re.findall(r"scan_kernel<MODE_(\w+), (true|false), (true|false), (true|false)>", table)
    assert len(found) == 16
    ids = _case_ids()
    for mode, smem, capture, shard in found:
        name = inst(mode.lower(), smem == "true", shard == "true", capture == "true")
        assert any(i.startswith(name + "/") for i in ids), name
