"""Plain restatement of the fused scan's outputs in torch — TEST INFRASTRUCTURE.

Device-agnostic: the same functions run on CPU tensors in the CPU suite (where they are pinned to oracle/ and np_oracle)
and on CUDA tensors next to the kernel.  Vectorised over records, written from the reference (src/fnv32.rs:92-101,
src/metric.rs:206-253, :288-305) and nothing else: no tiles, no warps, no shortcuts taken from the kernel.  Every
integer stays int64 and below 2^63; no float enters any count, sum or register."""
import torch

FNV_BASIS = 0x811C9DC5
FNV_MULT = 0x811C9DC5     # src/fnv32.rs:97 multiplies by the basis, not by the FNV prime
M32 = 0xFFFFFFFF
NB = 32                   # log2 buckets of the key and value histograms
LONG_KEY = 1 << 12        # fnv32: keys this long go to `long_fn` when one is given


def _mul32(a, c):
    """(a * c) mod 2^32 for an int64 tensor a in [0, 2^32) and a constant c < 2^32: c in 16-bit halves, so that no
    product reaches 2^49 (int64 wrap-around is never relied on)."""
    lo, hi = c & 0xFFFF, c >> 16
    return (a * lo + (((a * hi) & 0xFFFF) << 16)) & M32


def key_offsets(key_len):
    """byte offset of every record's key in the packed key bytes (null keys take no bytes)"""
    kl = key_len.to(torch.int64).clamp(min=0)
    return torch.cumsum(kl, 0) - kl


def fnv32(key_len, key_bytes, long_fn=None):
    """The reference hash of every packed key as int64 in [0, 2^32); null keys hash to 0.  One byte position at a time
    over the keys still running.  long_fn(offsets, lengths) -> hashes, when given, takes the keys of LONG_KEY bytes or
    more (a byte loop over a 1 MiB key is a million steps here)."""
    kl = key_len.to(torch.int64)
    off = key_offsets(key_len)
    h = torch.full_like(kl, FNV_BASIS)
    long = (kl >= LONG_KEY) if long_fn is not None else torch.zeros_like(kl, dtype=torch.bool)
    live = torch.nonzero((kl > 0) & ~long).flatten()
    j = 0
    while live.numel():
        b = key_bytes[off[live] + j].to(torch.int64)
        h[live] = _mul32(h[live] ^ b, FNV_MULT)
        j += 1
        live = live[kl[live] > j]
    if long_fn is not None and bool(long.any()):
        idx = torch.nonzero(long).flatten()
        h[idx] = long_fn(off[idx], kl[idx]).to(h.device, torch.int64)
    h[kl < 0] = 0
    return h


def bucket(lens):
    """log2 bucket of each length >= 0: 0 for 0, else floor(log2 len) + 1 — counted by comparisons, not log2"""
    lens = lens.to(torch.int64)
    out = torch.zeros_like(lens)
    for j in range(NB - 1):
        out += (lens >= (1 << j)).to(torch.int64)
    return out


def message_metrics(P, partition, ts_ms, key_len, value_len):
    """The same dict as np_oracle.message_metrics (int64 tensors per partition, ints for the globals), plus "bad": the
    records whose partition lies outside [0, P); they take part in nothing else."""
    p = partition.to(torch.int64)
    ok = (p >= 0) & (p < P)
    bad = int((~ok).sum())
    p, ts = p[ok], ts_ms.to(torch.int64)[ok]
    kl, vl = key_len.to(torch.int64)[ok], value_len.to(torch.int64)[ok]
    keyed, valued = kl >= 0, vl >= 0
    z = lambda m=1: torch.zeros(P * m, dtype=torch.int64, device=p.device)

    def add(mask, w=None, idx=None, m=1):
        i = (p if idx is None else idx)[mask]
        return z(m).scatter_add_(0, i, torch.ones_like(i) if w is None else w[mask])

    every = torch.ones_like(keyed)
    out = {
        "total": add(every), "tombstones": add(~valued), "alive": add(valued),
        "key_null": add(~keyed), "key_non_null": add(keyed),
        "key_size_sum": add(keyed, kl), "value_size_sum": add(valued, vl),
    }
    ts0 = torch.where(ts == -1, torch.zeros_like(ts), ts)                              # metric.rs:209
    ts_s = torch.where(ts0 >= 0, torch.div(ts0, 1000, rounding_mode="trunc"), -torch.div(-ts0, 1000, rounding_mode="trunc"))
    out["min_ts_s"] = int(ts_s.min()) if ts_s.numel() else None
    out["max_ts_s"] = int(ts_s.max()) if ts_s.numel() else None
    size = torch.where(keyed, kl, torch.zeros_like(kl)) + vl
    out["largest"] = int(size[valued].max()) if bool(valued.any()) else 0              # metric.rs:249-251
    out["smallest"] = int(size[valued].min()) if bool(valued.any()) else 0             # metric.rs:177-183
    out["overall_size"] = int(out["key_size_sum"].sum() + out["value_size_sum"].sum())
    out["overall_count"] = int(p.numel())
    out["khist"] = add(keyed, idx=p * NB + bucket(kl), m=NB).view(P, NB)
    out["vhist"] = add(valued, idx=p * NB + bucket(vl), m=NB).view(P, NB)
    out["bad"] = bad
    return out


def earliest(mm, now):
    """MessageMetrics.earliest_message: starts at Utc::now() and only moves to an earlier whole second (metric.rs:39, 65-72)"""
    s = mm["min_ts_s"]
    return (s, 0) if s is not None and (s < now[0] or (s == now[0] and now[1] > 0)) else tuple(now)


def latest(mm):
    """MessageMetrics.latest_message: starts at the epoch (metric.rs:40)"""
    return max(0, mm["max_ts_s"]) if mm["max_ts_s"] is not None else 0


def fmix32(h):
    h = h.to(torch.int64) & M32
    h = h ^ (h >> 16)
    h = _mul32(h, 0x85EBCA6B)
    h = h ^ (h >> 13)
    h = _mul32(h, 0xC2B2AE35)
    return h ^ (h >> 16)


def clz32(v):
    """leading zeros of each 32-bit value: sum over j of [v < 2^j] (32 for 0)"""
    out = torch.zeros_like(v)
    for j in range(32):
        out += (v < (1 << j)).to(torch.int64)
    return out


def hll_regs(hashes, mask, p):
    """HLL registers of precision p over the hashes where mask holds: index x >> (32 - p), rho = clz(x << p) + 1 capped
    at 33 - p, x = fmix32(hash).  Returns int64 registers."""
    x = fmix32(hashes[mask] if mask is not None else hashes)
    idx = x >> (32 - p)
    rho = torch.clamp(clz32((x << p) & M32) + 1, max=33 - p)
    regs = torch.zeros(1 << p, dtype=torch.int64, device=x.device)
    return regs.scatter_reduce_(0, idx, rho, reduce="amax", include_self=True)


def alive_hashes(hashes, key_len, value_len, seq=None, mask=None):
    """metric.rs:288-305 replayed: the hashes whose last writer (by seq) had a value, and the distinct hashes written.
    Sorted by (hash, seq); the last element of every hash run is that hash's last writer."""
    keep = key_len >= 0
    if mask is not None:
        keep = keep & mask
    h = hashes.to(torch.int64)[keep]
    s = (torch.arange(key_len.numel(), device=h.device) if seq is None else seq.to(torch.int64))[keep]
    alive = (value_len >= 0)[keep]
    assert s.numel() == 0 or int(s.max()) < (1 << 31)
    _, order = torch.sort(h * (1 << 31) + s)
    h, alive = h[order], alive[order]
    last = torch.ones_like(alive)
    last[:-1] = h[1:] != h[:-1]
    return h[last & alive], int(last.sum())


def alive(hashes, key_len, value_len, seq=None, mask=None):
    """(alive keys, distinct hashes written): LogCompactionInMemoryMetrics.sum_all_alive and the table's occupancy"""
    a, distinct = alive_hashes(hashes, key_len, value_len, seq, mask)
    return int(a.numel()), distinct


def stream_mask(partition, key_len, value_len, P):
    """the records the in-stream sketch takes: in range, with a key and a value"""
    return (partition >= 0) & (partition < P) & (key_len >= 0) & (value_len >= 0)
