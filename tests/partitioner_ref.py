"""Restatements of the partitioner check (include/kta.h, kta_set_partitioner_check) (TEST INFRASTRUCTURE).

murmur2 / crc32 / record_counts state it one record at a time in Python integers (CRC-32 is zlib.crc32); murmur2_np /
crc32_np / counts_np over numpy columns of packed keys; counts_torch over torch tensors of per-record hashes, for
depth-sized batches on the device.  The CPU tests pin them to each other; the GPU tests compare the engine with them."""
import zlib

import numpy as np

SEED, M = 0x9747B28C, 0x5BD1E995
MASK = 0xFFFFFFFF


def murmur2(key: bytes) -> int:
    """Kafka's Utils.murmur2 as an unsigned 32-bit value: seed 0x9747b28c, m 0x5bd1e995, r 24, little-endian 4-byte
    words, the tail bytes folded high to low (Java's switch falls through) before one multiply"""
    n = len(key)
    h = (SEED ^ n) & MASK
    for i in range(n // 4):
        k = int.from_bytes(key[4 * i:4 * i + 4], "little")
        k = (k * M) & MASK
        k ^= k >> 24
        k = (k * M) & MASK
        h = (h * M) & MASK
        h ^= k
    t, r = n & ~3, n % 4
    if r >= 3:
        h ^= key[t + 2] << 16
    if r >= 2:
        h ^= key[t + 1] << 8
    if r >= 1:
        h ^= key[t]
        h = (h * M) & MASK
    h ^= h >> 13
    h = (h * M) & MASK
    h ^= h >> 15
    return h


def signed(h: int) -> int:
    return h - (1 << 32) if h & 0x80000000 else h


def crc32(key: bytes) -> int:
    return zlib.crc32(key) & MASK


def verdict(key, p, counts):
    """the 2C + 1 booleans of one record: murmur2 at each count, CRC-32 at each count, neither"""
    m, c = murmur2(key) & 0x7FFFFFFF, crc32(key)
    bits = [m % n == p for n in counts] + [c % n == p for n in counts]
    return bits + [not any(bits)]


def record_counts(P, counts, records, shard=None):
    """[2C + 1][P] counts over (partition, key bytes or None) records, one at a time"""
    out = np.zeros((2 * len(counts) + 1, P), dtype=np.uint64)
    for p, key in records:
        if key is None or not 0 <= p < P or (shard is not None and p % shard[1] != shard[0]):
            continue
        for b, hit in enumerate(verdict(key, p, counts)):
            out[b, p] += np.uint64(hit)
    return out


# ---- numpy ----------------------------------------------------------------------------------------------------------
def _offsets(key_len):
    kl = np.maximum(np.asarray(key_len, dtype=np.int64), 0)
    off = np.zeros(kl.size, dtype=np.int64)
    np.cumsum(kl[:-1], out=off[1:])
    return off, kl


def murmur2_np(key_len, key_bytes):
    """u32 murmur2 of every packed key (0 for null keys), vectorised over records word by word"""
    off, kl = _offsets(key_len)
    kb = np.concatenate([np.asarray(key_bytes, dtype=np.uint8), np.zeros(4, np.uint8)]).astype(np.uint64)
    m = np.uint64(M)
    h = (np.uint64(SEED) ^ kl.astype(np.uint64)) & np.uint64(MASK)
    nw = kl // 4
    for i in range(int(nw.max()) if kl.size else 0):
        sel = nw > i
        a = off[sel] + 4 * i
        k = kb[a] | (kb[a + 1] << np.uint64(8)) | (kb[a + 2] << np.uint64(16)) | (kb[a + 3] << np.uint64(24))
        k = (k * m) & np.uint64(MASK)
        k ^= k >> np.uint64(24)
        k = (k * m) & np.uint64(MASK)
        h[sel] = ((h[sel] * m) & np.uint64(MASK)) ^ k
    r, t = kl % 4, off + (kl & ~3)
    for b in (2, 1, 0):
        sel = r > b
        h[sel] ^= kb[t[sel] + b] << np.uint64(8 * b)
    sel = r > 0
    h[sel] = (h[sel] * m) & np.uint64(MASK)
    h ^= h >> np.uint64(13)
    h = (h * m) & np.uint64(MASK)
    h ^= h >> np.uint64(15)
    h[np.asarray(key_len) < 0] = 0
    return h.astype(np.uint32)


_CRC_T = np.zeros(256, dtype=np.uint32)
for _i in range(256):
    _c = _i
    for _ in range(8):
        _c = (_c >> 1) ^ (0xEDB88320 if _c & 1 else 0)
    _CRC_T[_i] = _c


def crc32_np(key_len, key_bytes):
    """u32 zlib CRC-32 of every packed key (0 for null keys), vectorised over records byte by byte"""
    off, kl = _offsets(key_len)
    kb = np.asarray(key_bytes, dtype=np.uint8)
    c = np.full(kl.size, MASK, dtype=np.uint32)
    for i in range(int(kl.max()) if kl.size else 0):
        sel = kl > i
        c[sel] = _CRC_T[(c[sel] ^ kb[off[sel] + i]) & 0xFF] ^ (c[sel] >> np.uint32(8))
    c ^= np.uint32(MASK)
    c[np.asarray(key_len) < 0] = 0
    return c


def counts_from_hashes_np(P, counts, partition, key_len, mm, cc, shard=None):
    part = np.asarray(partition, dtype=np.int64)
    ok = (np.asarray(key_len) >= 0) & (part >= 0) & (part < P)
    if shard is not None:
        ok &= part % shard[1] == shard[0]
    part, m, c = part[ok], (np.asarray(mm, np.uint64)[ok] & np.uint64(0x7FFFFFFF)), np.asarray(cc, np.uint64)[ok]
    hits = [(m % np.uint64(n)).astype(np.int64) == part for n in counts] + \
           [(c % np.uint64(n)).astype(np.int64) == part for n in counts]
    hits.append(~np.any(np.stack(hits), axis=0) if hits else np.ones(part.size, bool))
    return np.stack([np.bincount(part[h], minlength=P).astype(np.uint64) for h in hits])


def counts_np(P, counts, partition, key_len, key_bytes, shard=None):
    """[2C + 1][P] over numpy columns (partition, key_len) and the packed key bytes"""
    return counts_from_hashes_np(P, counts, partition, key_len, murmur2_np(key_len, key_bytes), crc32_np(key_len, key_bytes),
                                 shard=shard)


# ---- torch ----------------------------------------------------------------------------------------------------------
def counts_torch(P, counts, partition, key_len, mm, cc):
    """[2C + 1][P] (int64 tensor) from torch columns and per-record u32 hashes held in int64 tensors, on their device"""
    import torch
    ok = (key_len >= 0) & (partition >= 0) & (partition < P)
    part = partition[ok].long()
    m, c = mm[ok] & 0x7FFFFFFF, cc[ok]
    hits = [torch.remainder(m, n) == part for n in counts] + [torch.remainder(c, n) == part for n in counts]
    hits.append(~torch.stack(hits).any(0))
    return torch.stack([torch.bincount(part[h], minlength=P) for h in hits])


def place(keys, N, fn):
    """the partition fn ('murmur2' or 'crc32') puts each key at under N partitions"""
    if fn == "murmur2":
        return [(murmur2(k) & 0x7FFFFFFF) % N for k in keys]
    return [crc32(k) % N for k in keys]


def hashes_torch(keys):
    """(murmur2, crc32) of n keys of one length L, given as an [n, L] uint8 tensor, as int64 tensors on its device"""
    import torch
    n, L = keys.shape
    k64 = keys.long()
    h = torch.full((n,), (SEED ^ L) & MASK, dtype=torch.int64, device=keys.device)
    for i in range(L // 4):
        k = k64[:, 4 * i] | (k64[:, 4 * i + 1] << 8) | (k64[:, 4 * i + 2] << 16) | (k64[:, 4 * i + 3] << 24)
        k = (k * M) & MASK
        k ^= k >> 24
        k = (k * M) & MASK
        h = ((h * M) & MASK) ^ k
    t, r = L & ~3, L % 4
    for b in range(r - 1, -1, -1):
        h ^= k64[:, t + b] << (8 * b)
    if r:
        h = (h * M) & MASK
    h ^= h >> 13
    h = (h * M) & MASK
    h ^= h >> 15
    table = torch.from_numpy(_CRC_T.astype(np.int64)).to(keys.device)
    c = torch.full((n,), MASK, dtype=torch.int64, device=keys.device)
    for i in range(L):
        c = table[(c ^ k64[:, i]) & 0xFF] ^ (c >> 8)
    return h, c ^ MASK
