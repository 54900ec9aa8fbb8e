"""Restatements of the timeline extension (include/kta.h, kta_set_timeline) (TEST INFRASTRUCTURE).

record_index states it one record at a time in Python integers, as the semantics read; timeline_np states it over
numpy columns, timeline_torch over torch tensors (for depth-sized batches on the device).  The CPU tests pin
timeline_np to record_counts and timeline_torch to timeline_np on CPU tensors; the GPU tests compare the engine with
them."""
import numpy as np

RECORDS, TOMBSTONES, BYTES = 0, 1, 2
U64 = (1 << 64) - 1


def second(ts_ms: int) -> int:
    """t = (ts_ms == -1 ? 0 : ts_ms) / 1000, truncating toward zero"""
    t = 0 if ts_ms == -1 else ts_ms
    q = abs(t) // 1000
    return q if t >= 0 else -q


def record_index(ts_ms: int, origin: int, width: int, buckets: int) -> int:
    t = second(ts_ms)
    if t < origin:
        return 0
    if t >= origin + buckets * width:
        return buckets + 1
    return 1 + (t - origin) // width


def record_counts(P, origin, width, buckets, records, shard=None):
    """[3][P][B + 2] Python-int counts over (partition, ts_ms, key_len, value_len) records, one at a time"""
    out = np.zeros((3, P, buckets + 2), dtype=np.uint64)
    for p, ts, kl, vl in records:
        if not 0 <= p < P or (shard is not None and p % shard[1] != shard[0]):
            continue
        i = record_index(ts, origin, width, buckets)
        out[RECORDS, p, i] += np.uint64(1)
        out[TOMBSTONES, p, i] += np.uint64(vl < 0)
        out[BYTES, p, i] += np.uint64(max(kl, 0) + max(vl, 0))
    return out


SMAX = 9_223_372_036_854_775   # |second(ts_ms)| of every int64 ts_ms: the reachable seconds are [-SMAX, SMAX]


def kernel_quotient(d: int, width: int, buckets: int) -> int:
    """timeline_index's quotient before its correction step: (uint64)((double)d * inv_width) clamped to B - 1, with
    inv_width = 1.0 / (double)W as the host computes it.  Python floats are IEEE doubles: float() of an int rounds to
    nearest like the kernel's u64 → f64 conversion, the product rounds to nearest like DMUL, and int() truncates
    toward zero like cvt.rzi."""
    return min(int(float(d) * (1.0 / float(width))), buckets - 1)


def kernel_index(ts_ms: int, origin: int, width: int, buckets: int):
    """timeline_index (csrc/kta_timeline.cuh) restated statement by statement.  Returns (index, step): step is -1 where
    the correction ran q--, +1 where it ran q++, 0 where the quotient stood"""
    s = second(ts_ms)
    if s < origin:
        return 0, 0
    d = s - origin                        # (uint64)s - (uint64)O: in [0, 2^64) since s >= O
    if d >= buckets * width:              # span = B W < 2^64
        return buckets + 1, 0
    q = kernel_quotient(d, width, buckets)
    lo = q * width                        # <= (B - 1) W: no wrap
    if lo > d:
        return q, -1                      # 1 + (q - 1)
    if d - lo >= width:
        return q + 2, 1                   # 1 + (q + 1)
    return q + 1, 0


def boundary_ms(origin: int, width: int, buckets: int, ends: int = 1024, sample: int = 4096, seed: int = 0):
    """int64 timestamps at q W - 1, q W and q W + 1 seconds past O for q = 0 .. B, each at millisecond 0 and 999 of its
    second (truncating toward zero: second -5 at 999 ms is -5999 ms), clipped to int64 (which keeps the second);
    seconds outside [-SMAX, SMAX] cannot occur and are left out.  When B + 1 > 2 ends + sample: the q within `ends` of
    either end and a seeded sample of `sample` between them."""
    if buckets + 1 <= 2 * ends + sample:
        qs = list(range(buckets + 1))
    else:
        mid = np.random.default_rng(seed).choice(np.arange(ends, buckets + 1 - ends), sample, replace=False)
        qs = list(range(ends)) + sorted(mid.tolist()) + list(range(buckets + 1 - ends, buckets + 1))
    out = []
    for q in qs:
        for s in (origin + q * width - 1, origin + q * width, origin + q * width + 1):
            if -SMAX <= s <= SMAX:
                out += [min(max(s * 1000 + (ms if s >= 0 else -ms), -(1 << 63)), (1 << 63) - 1) for ms in (0, 999)]
    return np.array(out, dtype=np.int64)


def shard_accepted(P: int, G: int) -> bool:
    """kta_create's rule for a sharded handle (G = shard_world > 1, G <= P): the scan's column p / G is
    mulhi(p, m) with m = ceil(2^32 / G), exact when p e < 2^32 for e = m G - 2^32; the shape is accepted when the
    largest partition id, P - 1, meets that"""
    m = -(-(1 << 32) // G)
    return (P - 1) * (m * G - (1 << 32)) < 1 << 32


def shard_column_mulhi(p, G: int):
    """the scan's column of partition ids p (numpy, < 2^32): __umulhi(p, ceil(2^32 / G))"""
    m = np.uint64(-(-(1 << 32) // G))
    return (np.asarray(p, dtype=np.uint64) * m) >> np.uint64(32)


def seconds_np(ts_ms):
    t = np.where(ts_ms == -1, 0, ts_ms).astype(np.int64)
    q = t // 1000
    return q + ((t % 1000 != 0) & (t < 0))   # floor → truncation toward zero


def index_np(ts_ms, origin, width, buckets):
    t = seconds_np(np.asarray(ts_ms, dtype=np.int64))
    d = t.view(np.uint64) - np.uint64(origin & U64)    # t - O as an unsigned difference (wraps below O: masked)
    inside = 1 + d // np.uint64(width)
    idx = np.where(d >= np.uint64(buckets * width), buckets + 1, inside.astype(np.int64) if buckets else 0)
    return np.where(t < origin, 0, idx).astype(np.int64)


def timeline_np(P, origin, width, buckets, partition, ts_ms, key_len, value_len, shard=None):
    """[3][P][B + 2] u64 over SoA columns"""
    p = np.asarray(partition, dtype=np.int64)
    kl = np.asarray(key_len, dtype=np.int64)
    vl = np.asarray(value_len, dtype=np.int64)
    ok = (p >= 0) & (p < P)
    if shard is not None:
        ok &= p % shard[1] == shard[0]
    row = buckets + 2
    key = (p * row + index_np(ts_ms, origin, width, buckets))[ok]
    nb = P * row
    out = np.zeros((3, nb), dtype=np.uint64)
    out[RECORDS] = np.bincount(key, minlength=nb).astype(np.uint64)
    out[TOMBSTONES] = np.bincount(key, weights=(vl[ok] < 0).astype(np.float64), minlength=nb).astype(np.uint64)
    b = (np.maximum(kl, 0) + np.maximum(vl, 0))[ok]
    lo = np.bincount(key, weights=(b & 0xFFFF).astype(np.float64), minlength=nb)   # < 2^16 per record: exact in float64
    hi = np.bincount(key, weights=(b >> 16).astype(np.float64), minlength=nb)
    out[BYTES] = lo.astype(np.uint64) + (hi.astype(np.uint64) << np.uint64(16))
    return out.reshape(3, P, row)


def timeline_torch(P, origin, width, buckets, partition, ts_ms, key_len, value_len, shard=None):
    """[3][P][B + 2] int64 tensor (on the columns' device) over SoA tensors.  Counts stay below 2^63 at these sizes."""
    import torch
    p = partition.to(torch.int64)
    ts = ts_ms.to(torch.int64)
    t = torch.where(ts == -1, torch.zeros_like(ts), ts)
    sec = torch.div(t, 1000, rounding_mode="trunc")
    ok = (p >= 0) & (p < P)
    if shard is not None:
        ok &= p % shard[1] == shard[0]
    # sec < O → 0; sec >= O + B W → B + 1; else 1 + (sec - O) // W, where 0 <= sec - O < B W < 2^63: exact in int64
    # (the subtraction may wrap in between, its result does not)
    assert buckets * width < 1 << 63, "timeline_torch takes ranges of B W < 2^63 seconds"
    end = origin + buckets * width
    before = sec < origin
    after = sec >= end
    d = torch.where(before | after, torch.zeros_like(sec), sec - origin)
    idx = torch.where(before, torch.zeros_like(sec), torch.where(after, torch.full_like(sec, buckets + 1),
                                                                  1 + torch.div(d, width, rounding_mode="floor")))
    row = buckets + 2
    key = (p * row + idx)[ok]
    nb = P * row
    kl = key_len.to(torch.int64).clamp(min=0)
    vl = value_len.to(torch.int64)
    out = torch.zeros(3, nb, dtype=torch.int64, device=partition.device)
    out[RECORDS].index_add_(0, key, torch.ones_like(key))
    out[TOMBSTONES].index_add_(0, key, (vl[ok] < 0).to(torch.int64))
    out[BYTES].index_add_(0, key, (kl + vl.clamp(min=0))[ok])
    return out.view(3, P, row)
