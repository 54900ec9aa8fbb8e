"""Plain restatements of the hot-key table (include/kta.h, kta_set_hot_keys; csrc/kta_hotkeys.cuh), independent of the
library: per key id, (uint64)crc32(key) << 32 | murmur2(key), its records, tombstones (value_len < 0), bytes
(key_len + max(value_len, 0)), latest second ((ts_ms == -1 ? 0 : ts_ms) / 1000, truncating), partition range, key_len and
prefix, over the records the counters count with key_len >= 0.

Three of them, pinned to each other by tests/test_hot_keys.py:
  * record_table: a dict, record at a time;
  * table_np: numpy (np.unique, np.add.at, minimum.at / maximum.at);
  * table_torch: torch on the columns' device, from partitioner_ref.hashes_torch and torch.unique (for depth).
Each returns the whole table as a numpy array of HOT_KEY_DTYPE sorted by id; top() orders it as kta_hot_keys does.  When
two keys share an id the library keeps the prefix of whichever claimed the slot; the restatements keep the first
record's, so tests compare prefixes only where ids are unique (always, for the keys they use)."""
import zlib

import numpy as np

import partitioner_ref as R
from kafka_topic_analyzer_b200._native import HOT_KEY_DTYPE, HOT_KEY_PREFIX


def key_id(key: bytes) -> int:
    return zlib.crc32(key) << 32 | R.murmur2(key)


def second(ts_ms: int) -> int:
    t = 0 if ts_ms == -1 else int(ts_ms)
    return -((-t) // 1000) if t < 0 else t // 1000   # truncating toward zero


def _counted(P, partition, key_len, shard):
    part = np.asarray(partition, dtype=np.int64)
    ok = (np.asarray(key_len) >= 0) & (part >= 0) & (part < P)
    if shard is not None:
        ok &= part % shard[1] == shard[0]
    return ok


def _prefix(key: bytes) -> np.ndarray:
    out = np.zeros(HOT_KEY_PREFIX, np.uint8)
    out[:min(len(key), HOT_KEY_PREFIX)] = np.frombuffer(key[:HOT_KEY_PREFIX], np.uint8)
    return out


# ---- record at a time -----------------------------------------------------------------------------------------------
def record_table(P, records, shard=None):
    """records: iterable of (partition, key or None, value_len or None-for-tombstone-as -1, ts_ms)"""
    d = {}
    for p, key, vl, ts in records:
        if key is None or not 0 <= p < P or (shard is not None and p % shard[1] != shard[0]):
            continue
        i = key_id(key)
        e = d.get(i)
        if e is None:
            e = d[i] = dict(records=0, tombstones=0, bytes=0, latest_s=-(1 << 63), min_partition=p, max_partition=p,
                            key_len=len(key), key_prefix=_prefix(key))
        e["records"] += 1
        e["tombstones"] += int(vl < 0)
        e["bytes"] += len(key) + max(vl, 0)
        e["latest_s"] = max(e["latest_s"], second(ts))
        e["min_partition"] = min(e["min_partition"], p)
        e["max_partition"] = max(e["max_partition"], p)
    out = np.zeros(len(d), HOT_KEY_DTYPE)
    for j, i in enumerate(sorted(d)):
        out[j]["id"] = i
        for f, v in d[i].items():
            out[j][f] = v
    return out


# ---- numpy ------------------------------------------------------------------------------------------------------------
def table_from_ids_np(P, partition, key_len, value_len, ts_ms, ids, key_bytes=None, shard=None):
    ok = _counted(P, partition, key_len, shard)
    ids = np.asarray(ids, np.uint64)[ok]
    part = np.asarray(partition, np.int64)[ok]
    kl = np.asarray(key_len, np.int64)
    off = np.zeros(kl.size, np.int64)
    np.cumsum(np.maximum(kl, 0)[:-1], out=off[1:])
    off, kl = off[ok], kl[ok]
    vl = np.asarray(value_len, np.int64)[ok]
    ts = np.asarray(ts_ms, np.int64)[ok]
    ts = np.where(ts == -1, 0, ts)
    sec = np.sign(ts) * (np.abs(ts) // 1000)
    u, first, inv = np.unique(ids, return_index=True, return_inverse=True)
    out = np.zeros(u.size, HOT_KEY_DTYPE)
    out["id"] = u
    rec = np.zeros(u.size, np.uint64)
    np.add.at(rec, inv, np.uint64(1))
    out["records"] = rec
    tomb = np.zeros(u.size, np.uint64)
    np.add.at(tomb, inv, (vl < 0).astype(np.uint64))
    out["tombstones"] = tomb
    byt = np.zeros(u.size, np.uint64)
    np.add.at(byt, inv, (kl + np.maximum(vl, 0)).astype(np.uint64))
    out["bytes"] = byt
    lat = np.full(u.size, np.iinfo(np.int64).min, np.int64)
    np.maximum.at(lat, inv, sec)
    out["latest_s"] = lat
    lo = np.full(u.size, P, np.int64)
    np.minimum.at(lo, inv, part)
    hi = np.full(u.size, -1, np.int64)
    np.maximum.at(hi, inv, part)
    out["min_partition"], out["max_partition"] = lo, hi
    out["key_len"] = kl[first]
    if key_bytes is not None:
        kb = np.concatenate([np.asarray(key_bytes, np.uint8), np.zeros(HOT_KEY_PREFIX, np.uint8)])
        for j in range(HOT_KEY_PREFIX):
            out["key_prefix"][:, j] = np.where(j < kl[first], kb[off[first] + j], 0)
    return out


def ids_np(key_len, key_bytes):
    return (R.crc32_np(key_len, key_bytes).astype(np.uint64) << np.uint64(32)) | R.murmur2_np(key_len, key_bytes).astype(np.uint64)


def table_np(P, partition, key_len, value_len, ts_ms, key_bytes, shard=None):
    return table_from_ids_np(P, partition, key_len, value_len, ts_ms, ids_np(key_len, key_bytes), key_bytes, shard)


# ---- torch ------------------------------------------------------------------------------------------------------------
def ids_torch(key_len, keys_by_len):
    """int64 ids (the u64 bit pattern) of n records: key_len a torch int tensor, keys_by_len {L: (rows, [m, L] uint8)}"""
    import torch
    ids = torch.zeros(key_len.numel(), dtype=torch.int64, device=key_len.device)
    for L, (rows, keys) in keys_by_len.items():
        mm, cc = R.hashes_torch(keys)
        ids[rows] = (cc << 32) | mm
    return ids


def table_torch(P, partition, key_len, value_len, ts_ms, ids):
    """(ids, records, tombstones, bytes, latest_s, min_partition, max_partition) tensors sorted by id as u64 (id tensors
    hold the u64 bit pattern in int64), from torch columns on their device"""
    import torch
    ok = (key_len >= 0) & (partition >= 0) & (partition < P)
    ids, part = ids[ok], partition[ok].long()
    kl, vl, ts = key_len[ok].long(), value_len[ok].long(), ts_ms[ok].long()
    ts = torch.where(ts == -1, torch.zeros_like(ts), ts)
    sec = torch.div(ts, 1000, rounding_mode="trunc")
    flip = ids ^ (-(1 << 63))   # signed order of the flipped pattern = unsigned order of the id
    u, inv = torch.unique(flip, return_inverse=True)
    n = u.numel()
    z = lambda: torch.zeros(n, dtype=torch.int64, device=ids.device)
    rec = z().index_add_(0, inv, torch.ones_like(inv))
    tomb = z().index_add_(0, inv, (vl < 0).long())
    byt = z().index_add_(0, inv, kl + vl.clamp(min=0))
    lat = torch.full((n,), -(1 << 63), dtype=torch.int64, device=ids.device).scatter_reduce_(0, inv, sec, "amax")
    lo = torch.full((n,), P, dtype=torch.int64, device=ids.device).scatter_reduce_(0, inv, part, "amin")
    hi = torch.full((n,), -1, dtype=torch.int64, device=ids.device).scatter_reduce_(0, inv, part, "amax")
    return u ^ (-(1 << 63)), rec, tomb, byt, lat, lo, hi


# ---- order ------------------------------------------------------------------------------------------------------------
def top(table, k):
    """kta_hot_keys' order: records descending, then id ascending; the first k"""
    order = np.lexsort((table["id"], np.iinfo(np.uint64).max - table["records"]))
    return table[order][:k]


def by_id(table):
    return table[np.argsort(table["id"], kind="stable")]
