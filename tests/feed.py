"""Topics and how they reach an engine (TEST INFRASTRUCTURE): host builders, device topics, and one feeder per entry point.

The engine works on its own stream, which nothing orders behind torch's.  So every feeder here that hands the engine
device memory torch has written (columns, key bytes, tile bases, seq columns, import lists, segment buffers, capture
buffers) first waits for torch's stream: settle().  Only torch's stream is waited for, so work already queued on the
engine's stream stays queued."""
import ctypes as C

import numpy as np
import torch

import kafka_codec as kc
import native_build
import np_oracle
import scan_ref as R
from kafka_topic_analyzer_b200 import KtaEngine, lib
from kafka_topic_analyzer_b200 import _native as N
from kafka_topic_analyzer_b200.synth import HostTopic, tile_base_from_key_len
from parity import last_writer

NOW = (4102444800, 123456789)   # 2100-01-01: later than every synthetic record
T = N.KTA_KEY_TILE
MASK32 = 0xFFFFFFFF
FNV = 0x811C9DC5                # basis and multiplier of the reference hash (src/fnv32.rs)
FNV_INV = pow(FNV, -1, 1 << 32)


def settle():
    """torch's writes so far have landed"""
    torch.cuda.current_stream().synchronize()


# ------------------------------------------------------------------------------------------------
# host topics
# ------------------------------------------------------------------------------------------------
def random_topic(rng, n, P, max_key=40, big=False):
    """Adversarial random SoA batch: nulls, empties, ragged key lengths, missing/negative timestamps."""
    part = rng.integers(0, P, size=n).astype(np.int32)
    kl = rng.integers(-1, max_key + 1, size=n).astype(np.int32)
    vl = rng.choice(np.array([-1, -1, 0, 1, 2, 3, 127, 128, 255, 256, 1000, 65535, 65536, (1 << 31) - 1 if big else 99999],
                             dtype=np.int64), size=n).astype(np.int32)
    ts = (1_500_000_000_000 + rng.integers(-10**9, 10**9, size=n)).astype(np.int64)
    ts[rng.random(n) < 0.02] = -1
    ts[rng.random(n) < 0.01] = rng.integers(-5000, 5000)
    nkeys = max(4, n // 8)
    pool = [bytes(rng.integers(0, 256, size=int(l), dtype=np.uint8)) for l in rng.integers(0, max_key + 1, size=nkeys)]
    blob = []
    for i in range(n):
        if kl[i] < 0:
            continue
        k = pool[int(rng.integers(0, nkeys))]
        kl[i] = len(k)
        blob.append(k)
    kb = np.frombuffer(b"".join(blob) or b"", dtype=np.uint8).copy()
    seq = np.arange(n, dtype=np.uint64)
    return HostTopic(part, np.zeros(n, dtype=np.int64), ts, kl, vl, seq, kb, tile_base_from_key_len(kl))


def fixed_width_topic(rng, n, P, L, null_frac, pool):
    """n records of L-byte keys drawn from `pool` random keys, a null_frac share of them null, over P partitions"""
    kl = np.where(rng.random(n) < null_frac, -1, L).astype(np.int32)
    keys = rng.integers(0, 256, size=(pool, L), dtype=np.uint8)
    kb = keys[rng.integers(0, pool, size=int((kl >= 0).sum()))].reshape(-1)
    return HostTopic(rng.integers(0, P, size=n).astype(np.int32), np.zeros(n, dtype=np.int64),
                     (1_600_000_000_000 + np.arange(n)).astype(np.int64), kl, rng.integers(-1, 300, size=n).astype(np.int32),
                     np.arange(n, dtype=np.uint64), kb, tile_base_from_key_len(kl))


def gather(blob, off, lens):
    """Concatenation of blob[off[i] : off[i] + lens[i]] (lens >= 0)."""
    lens = lens.astype(np.int64)
    total = int(lens.sum())
    if total == 0:
        return np.zeros(0, dtype=np.uint8)
    starts = np.repeat(off.astype(np.int64) - (np.cumsum(lens) - lens), lens)
    return blob[starts + np.arange(total, dtype=np.int64)]


def partition_lists(t):
    """per-partition record lists (ts, key, value_len) in offset order, from a HostTopic"""
    kl = t.key_len
    koff = np.concatenate([[0], np.cumsum(np.maximum(kl, 0))])
    per = {}
    for i in range(t.n):
        key = None if kl[i] < 0 else t.key_bytes[koff[i]:koff[i] + kl[i]].tobytes()
        vl = None if t.value_len[i] < 0 else int(t.value_len[i])
        per.setdefault(int(t.partition[i]), []).append((int(t.ts_ms[i]), key, vl))
    return per


# ------------------------------------------------------------------------------------------------
# topics in HBM
# ------------------------------------------------------------------------------------------------
def device(a, shift=0):
    """a (numpy, uint64 viewed as int64; or a torch tensor) on the device; with shift, the column starts `shift`
    elements past a 16-byte-aligned base"""
    if not isinstance(a, torch.Tensor):
        a = np.ascontiguousarray(a)
        a = torch.from_numpy(a.view(np.int64) if a.dtype == np.uint64 else a)
    if shift:
        buf = torch.zeros(a.numel() + 16, dtype=a.dtype, device="cuda")
        assert buf.data_ptr() % 16 == 0
        col = buf[shift: shift + a.numel()]
        col.copy_(a)
    else:
        col = a.cuda()
    assert (col.data_ptr() % 16 == 0) == (shift == 0)
    return col


class Topic:
    """SoA columns on the device, keys packed in record order with 64 bytes of slack, key_tile_base from key_len."""

    def __init__(self, partition, ts_ms, key_len, value_len, key_bytes, key_bytes_len, seq=None, key_tile_base=None):
        self.partition, self.ts_ms, self.key_len, self.value_len = partition, ts_ms, key_len, value_len
        self.key_bytes, self.kbl, self.seq = key_bytes, int(key_bytes_len), seq
        self.n = int(partition.numel())
        self.key_tile_base = tile_base(key_len) if key_tile_base is None else key_tile_base

    @property
    def keys(self):
        return self.key_bytes[: self.kbl]


def tile_base(key_len):
    kl = key_len.to(torch.int64).clamp(min=0)
    nt = -(-kl.numel() // T)
    sums = torch.cat([kl, kl.new_zeros(nt * T - kl.numel())]).view(nt, T).sum(1)
    return torch.cat([kl.new_zeros(1), torch.cumsum(sums, 0)])


def to_device(h):
    """a HostTopic copied to the device, its key_tile_base column included"""
    kb = torch.zeros(h.key_bytes.size + 64, dtype=torch.uint8, device="cuda")
    if h.key_bytes.size:
        kb[: h.key_bytes.size] = device(h.key_bytes)
    return Topic(*(device(c) for c in (h.partition, h.ts_ms, h.key_len, h.value_len)), kb, h.key_bytes.size,
                 seq=device(h.seq), key_tile_base=device(h.key_tile_base))


def made_byte(r, pos):
    return ((r * 2654435761 + pos * 40503 + (pos >> 8) * 97) >> 5) & 0xFF


def pack_keys(kb_src, src_off, lens, made=None, chunk=1 << 21):
    """Packed key bytes (+ 64 B of slack): record i's key is lens[i] bytes from kb_src[src_off[i]:], or where made[i],
    bytes made from i and the position.  Chunked over records, so no index tensor spans the whole key buffer."""
    lens = lens.to(torch.int64).clamp(min=0)
    dst = torch.cumsum(lens, 0) - lens
    total = int(lens.sum())
    out = torch.zeros(total + 64, dtype=torch.uint8, device=lens.device)
    for a in range(0, lens.numel(), chunk):
        b = min(lens.numel(), a + chunk)
        cnt = int(lens[a:b].sum())
        if not cnt:
            continue
        r = torch.repeat_interleave(torch.arange(a, b, device=lens.device), lens[a:b])
        pos = torch.arange(cnt, device=lens.device) - (dst[r] - dst[a])
        if made is None:
            val = kb_src[src_off[r] + pos]
        else:
            m = made[r]
            val = kb_src[torch.where(m, 0, src_off[r] + pos)].to(torch.int64)
            val = torch.where(m, made_byte(r, pos), val).to(torch.uint8)
        out[dst[a]: dst[a] + cnt] = val
        del r, pos, val
    return out, total


def rekey(t, new_kl):
    """t with key lengths new_kl: a record whose length is unchanged keeps its key, any other gets made bytes"""
    kb, total = pack_keys(t.keys, R.key_offsets(t.key_len), new_kl, made=new_kl != t.key_len)
    return Topic(t.partition, t.ts_ms, new_kl.to(torch.int32), t.value_len, kb, total, t.seq)


def take(t, idx):
    """the records idx of t, in that order, with their keys.  A host topic's records keep their seq; a device topic's
    get seq = idx (their place in t)."""
    if isinstance(t, Topic):
        kb, total = pack_keys(t.keys, R.key_offsets(t.key_len)[idx], t.key_len[idx])
        return Topic(t.partition[idx], t.ts_ms[idx], t.key_len[idx], t.value_len[idx], kb, total, seq=idx.to(torch.int64))
    kl0 = np.maximum(t.key_len.astype(np.int64), 0)
    kl = t.key_len[idx]
    return HostTopic(t.partition[idx], t.offset[idx], t.ts_ms[idx], kl, t.value_len[idx], t.seq[idx],
                     gather(t.key_bytes, (np.cumsum(kl0) - kl0)[idx], kl0[idx]).copy(), tile_base_from_key_len(kl))


# ------------------------------------------------------------------------------------------------
# alive-key hashes
# ------------------------------------------------------------------------------------------------
def fmix32(h):
    h ^= h >> 16
    h = (h * 0x85EBCA6B) & MASK32
    h ^= h >> 13
    h = (h * 0xC2B2AE35) & MASK32
    return h ^ (h >> 16)


def unmix32(x):
    """fmix32^-1 (the constants of hll_unmix, csrc/kta_kernels.cuh)."""
    x ^= x >> 16
    x = (x * 0x7ED1B41D) & MASK32
    x ^= (x >> 13) ^ (x >> 26)
    x = (x * 0xA5CB9243) & MASK32
    return x ^ (x >> 16)


_forward = None


def _fnv_forward3():
    """The 2^24 FNV states after three bytes, sorted, with the prefix that reaches each (built once per process)."""
    global _forward
    if _forward is None:
        h = np.full(1, FNV, dtype=np.uint32)
        for _ in range(3):
            h = ((h[:, None] ^ np.arange(256, dtype=np.uint32)[None, :]) * np.uint32(FNV)).reshape(-1)
        order = np.argsort(h, kind="stable").astype(np.uint32)
        _forward = (h[order], order)   # prefix index = b0 << 16 | b1 << 8 | b2
    return _forward


def keys_for_mixed(xs):
    """One 5-byte key per target: fmix32(fnv32(key)) == x.  Meet in the middle: two backward FNV steps from the target
    (2^16 candidates) looked up among the forward states after three bytes (2^24): about 256 hits per target."""
    states, prefix = _fnv_forward3()
    b = np.arange(1 << 16, dtype=np.uint32)
    b3, b4 = b >> 8, b & 0xFF
    keys = []
    for x in xs:
        h4 = np.uint32((unmix32(int(x)) * FNV_INV) & MASK32) ^ b4     # undo the last step for every last byte
        h3 = (h4 * np.uint32(FNV_INV)) ^ b3
        pos = np.searchsorted(states, h3)
        pos = np.minimum(pos, states.size - 1)
        hit = np.nonzero(states[pos] == h3)[0]
        assert hit.size, "no 5-byte preimage for x = %#x" % int(x)
        j = int(hit[0])
        pre = int(prefix[pos[j]])
        keys.append(bytes([pre >> 16, (pre >> 8) & 0xFF, pre & 0xFF, int(b3[j]), int(b4[j])]))
    return keys


def last_writer_map(t, seq, keep=None, parts=8):
    """Independent statement of the alive-key table: for every hash of a keyed record of a partition in [0, parts) that
    is kept, the largest (seq + 1) << 1 | alive.  Sorted (hash u32, stamp u64) arrays."""
    h = np_oracle.fnv32_many(t.key_len, t.key_bytes)
    m = (t.key_len >= 0) & (t.partition >= 0) & (t.partition < parts)
    if keep is not None:
        m &= keep
    return last_writer(h[m], np.asarray(seq, dtype=np.uint64)[m], t.value_len[m] >= 0)


def engine(P=8, **kw):
    """an engine counting alive keys exactly (-c), with 2^12 HLL registers"""
    return KtaEngine(P, count_alive_keys=True, hll_precision=12, now=NOW, **kw)


# ------------------------------------------------------------------------------------------------
# entry points
# ------------------------------------------------------------------------------------------------
def scan(e, t, *, tile_base=True, seq=None, seq_base=None, cols=None, key_bytes=None):
    """kta_scan_batch_device over t (a HostTopic is copied to the device first); seq a column, numpy or on the device"""
    if not isinstance(t, Topic):
        t = to_device(t)
    if seq is not None and not isinstance(seq, torch.Tensor):
        seq = device(np.asarray(seq, dtype=np.uint64))
    settle()
    e.scan_batch_device(*(cols or (t.partition, t.ts_ms, t.key_len, t.value_len)),
                        key_bytes=t.key_bytes if key_bytes is None else key_bytes, key_bytes_len=t.kbl,
                        key_tile_base=t.key_tile_base if tile_base else None, seq=seq, seq_base=seq_base)


def push_host(e, t, *, tile_base=True, seq=None, seq_base=None):
    """kta_push_batch_host over t (a device Topic is copied to the host first)"""
    if isinstance(t, Topic):
        h = lambda a: a.cpu().numpy()
        cols, kb, tb = [h(c) for c in (t.partition, t.ts_ms, t.key_len, t.value_len)], h(t.keys), h(t.key_tile_base).view(np.uint64)
    else:
        cols, kb, tb = [t.partition, t.ts_ms, t.key_len, t.value_len], t.key_bytes, t.key_tile_base
    e.push_batch_host(*cols, kb, tb if tile_base else None,
                      seq=None if seq is None else np.ascontiguousarray(seq, dtype=np.uint64), seq_base=seq_base)


_push_loop = None


def push_loop():
    """tests/native/push_loop.cu, loaded once"""
    global _push_loop
    if _push_loop is None:
        f = C.CDLL(native_build.build("push_loop")).push_loop
        f.restype = C.c_int
        f.argtypes = [C.c_void_p] * 2 + [C.c_int64] + [C.c_void_p] * 8
        _push_loop = f
    return _push_loop


def push_records(e, t, count=None, start=0):
    """records [start, start + count) of a HostTopic (to its end when count is None), one kta_push each, called from C.
    A refused record raises KtaError, with the records before it taken."""
    kl = np.ascontiguousarray(t.key_len, dtype=np.int32)
    off = np.cumsum(np.maximum(kl, 0), dtype=np.int64) - np.maximum(kl, 0)
    stop = t.n if count is None else start + count
    cols = [np.ascontiguousarray(c[start:stop], dtype=d) for c, d in ((t.partition, np.int32), (t.offset, np.int64),
                                                                       (t.ts_ms, np.int64), (kl, np.int32),
                                                                       (t.value_len, np.int32), (off, np.int64))]
    keys = np.ascontiguousarray(t.key_bytes, dtype=np.uint8) if t.key_bytes.size else np.zeros(1, dtype=np.uint8)
    failed = C.c_int64(-1)
    rc = push_loop()(C.cast(lib().kta_push, C.c_void_p), e.handle, stop - start, *(c.ctypes.data for c in cols[:5]),
                     keys.ctypes.data, cols[5].ctypes.data, C.addressof(failed))
    N.check(rc)


def feed(e, t, entry):
    """t through the entry point a parametrized test names"""
    if entry == "device":
        scan(e, t)
    elif entry == "device_no_tile_base":
        scan(e, t, tile_base=False)
    elif entry in ("host", "host_batch"):
        push_host(e, t)
    elif entry == "push":
        push_records(e, t)
    else:
        raise ValueError(entry)


def capture_hashes(e, out):
    """kta_set_hash_capture: every scanned record's hash into the device int32 column out; None stops capturing"""
    settle()
    assert lib().kta_set_hash_capture(e.handle, None if out is None else out.data_ptr()) == 0


def alive_import(e, h, stamp, count=None):
    """kta_alive_import_device of (hash, stamp) lists, numpy or on the device"""
    h, stamp = (a if isinstance(a, torch.Tensor) else device(a) for a in (h, stamp))
    settle()
    e.alive_import(h, stamp, h.numel() if count is None else count)


def stage_batches(segments):
    """(partition, RecordBatch bytes) segments in one device buffer, byte for byte with no slack behind the last batch:
    (buffer, length, batch offsets, batch partitions, batch count), the arguments of scan_log_batches_device"""
    offs, parts, at = [], [], 0
    for p, s in segments:
        o = kc.batch_offsets(s)
        offs += [at + x for x in o]
        parts += [p] * len(o)
        at += len(s)
    buf = device(np.frombuffer(b"".join(bytes(s) for _, s in segments), dtype=np.uint8).copy())
    return buf, at, device(np.array(offs, dtype=np.int64)), device(np.array(parts, dtype=np.int32)), len(offs)


def scan_log_batches(e, staged):
    """kta_scan_log_batches_device over stage_batches(...); returns the records delivered"""
    settle()
    return e.scan_log_batches_device(*staged)


def scan_log_segment(e, p, seg):
    """kta_scan_log_segment_device: partition p's batches from a device buffer; returns the records delivered"""
    buf, length, offs, _, nb = stage_batches([(p, seg)])
    n = C.c_int64()
    settle()
    N.check(lib().kta_scan_log_segment_device(e.handle, p, buf.data_ptr(), length, offs.data_ptr(), nb, C.byref(n)))
    e.sync()
    return n.value


def interleaved(parts):
    """the batches of {partition: [batch]}, round-robin over the partitions, each partition's in its order"""
    lists = [list(parts[p]) for p in sorted(parts)]
    out = []
    while any(lists):
        for l in lists:
            if l:
                out.append(l.pop(0))
    return out


LOG_ENTRIES = ("segment_host", "segments_host", "segment_device", "batches_device")


def scan_log(e, entry, parts):
    """{partition: [batch]} (anything with .p and .raw bytes) through one log entry point: segment_host and
    segment_device take each partition's batches as one segment, one call per partition; segments_host takes every
    partition's segment in one call; batches_device takes every batch, interleaved, in one device buffer.  Returns
    (records delivered, the batches in the order they were scanned)."""
    order = [b for p in sorted(parts) for b in parts[p]]
    segs = [(p, b"".join(b.raw for b in parts[p])) for p in sorted(parts)]
    if entry == "segment_host":
        n = sum(e.push_log_segment(p, s) for p, s in segs)
    elif entry == "segments_host":
        n = e.push_log_segments(segs)
    elif entry == "segment_device":
        n = sum(scan_log_segment(e, p, s) for p, s in segs)
    elif entry == "batches_device":
        order = interleaved(parts)
        n = scan_log_batches(e, stage_batches([(b.p, b.raw) for b in order]))
    else:
        raise ValueError(entry)
    return n, order
