"""A plain restatement of the synthetic topic (include/kta.h, synthetic-topic section; csrc/kta_synth.h), in vectorised
numpy uint64 with wrap-around arithmetic.  It loads neither library: the host and the device generators both evaluate
kta_synth.h, so a mistake in that header passes a host-vs-device comparison and only an independent restatement sees it.

fill(spec, rank, world, start, count) returns the same synth.HostTopic that synth.fill_host does: every column, the
packed key bytes and key_tile_base."""
from __future__ import annotations

import numpy as np

from kafka_topic_analyzer_b200 import synth

U = np.uint64
M64 = (1 << 64) - 1
GOLDEN = 0x9E3779B97F4A7C15            # 2^64 / phi: splitmix64's increment, also the second word of a 16-byte key
STREAM = 0xD1B54A32D192ED03
INT32_MAX = (1 << 31) - 1
TS_BASE = 1_500_000_000_000
MAX_KEY = 40
CHUNK = 1 << 20                        # records per key-byte chunk (bounds the (n, 40) byte matrices)
POW10 = np.array([10 ** d for d in range(20)], dtype=U)


def _splitmix64(x):
    x = x + U(GOLDEN)
    x = (x ^ (x >> U(30))) * U(0xBF58476D1CE4E5B9)
    x = (x ^ (x >> U(27))) * U(0x94D049BB133111EB)
    return x ^ (x >> U(31))


def splitmix64(x: int) -> int:
    with np.errstate(over="ignore"):
        return int(_splitmix64(np.array([x & M64], dtype=U))[0])


def mix(seed: int, i, stream: int) -> np.ndarray:
    """Stream `stream` of the counter-based generator at counters `i` (uint64 array)."""
    h = splitmix64(seed ^ ((stream * STREAM) & M64))
    with np.errstate(over="ignore"):
        return _splitmix64(U(h) + np.asarray(i, dtype=U) * U(GOLDEN))


def valid(spec, rank: int = 0, world: int = 1) -> bool:
    """The specs kta.h accepts."""
    P, R, n = spec.num_partitions, spec.run_len, spec.n_total
    if P < 1 or R < 1 or n < 0 or world < 1 or not 0 <= rank < world:
        return False
    km = spec.key_mode
    if km < 0 or km & 0xFF > 2 or km & ~0x3FF or not 0 <= spec.value_mean <= synth.MAX_VALUE_MEAN:
        return False
    return n % (P * R) == 0 and (world == 1 or P % world == 0)


def local_to_global(spec, rank: int, world: int, j) -> np.ndarray:
    """Global index of local record j of shard `rank` (partitions p % world == rank), in global order.  Cycle c deals
    its P runs to slots 0..P-1 and slot s goes to partition (s + shift_c) % P, so the shard owns the slots with
    (s + shift_c) % world == rank: every world-th slot from (rank - shift_c) mod world, P / world of them per cycle."""
    j = np.asarray(j, dtype=U)
    if world <= 1:
        return j.copy()
    P, R, G = spec.num_partitions, spec.run_len, world
    lrun, within = j // U(R), j % U(R)
    cycle, m = lrun // U(P // G), lrun % U(P // G)
    shift = (mix(spec.seed, cycle, 0) % U(P)).astype(np.int64)
    first = (rank - shift) % G                       # numpy's % of a negative int64 is the mathematical modulus
    slot = first.astype(U) + m * U(G)
    return (cycle * U(P) + slot) * U(R) + within


def local_index_of(spec, rank, world, g):
    """The first local index of shard `rank` whose global index is at least g (a shard's order is global order)."""
    lo, hi = 0, spec.n_total // world
    while lo < hi:
        mid = (lo + hi) // 2
        if int(local_to_global(spec, rank, world, [mid])[0]) < g:
            lo = mid + 1
        else:
            hi = mid
    return lo


def key_len_of(spec, key_id) -> np.ndarray:
    key_id = np.asarray(key_id, dtype=U)
    fmt = spec.key_mode & 0xFF
    if fmt == 0:
        return np.full(key_id.shape, 16, dtype=np.int32)
    if fmt == 1:
        digits = np.ones(key_id.shape, dtype=np.int32)
        for d in range(1, 20):
            digits += key_id >= U(10 ** d)
        return 4 + digits
    return (mix(spec.seed, key_id, 7) % U(MAX_KEY + 1)).astype(np.int32)


def record_at(spec, i) -> dict:
    """Every column of the global records i (uint64 array), as kta.h defines them; key_id is the key's id (valid where
    key_len >= 0)."""
    i = np.asarray(i, dtype=U)
    seed, P, R = spec.seed, spec.num_partitions, spec.run_len
    with np.errstate(over="ignore"):
        run, within = i // U(R), i % U(R)
        cycle, slot = run // U(P), run % U(P)
        p = (slot + mix(seed, cycle, 0) % U(P)) % U(P)
        offset = (cycle * U(R) + within).astype(np.int64)

        null_key = mix(seed, i, 1) % U(10000) < U(spec.null_key_per_10k)
        K = max(spec.distinct_keys // P, 1)            # keys per partition
        kidx = mix(seed, i, 2)
        if spec.key_mode & synth.KEYS_LOGUNIFORM:
            # a bit length b uniform in [0, floor(log2 K)], then an index uniform among those of that length
            nbits = min(K.bit_length() - 1, 63)
            b = (kidx >> U(40)) % U(nbits + 1)
            low = (U(1) << b) - U(1)
            kidx = low + (kidx & low)
        key_id = (kidx % U(K)) * U(P) + p
        key_len = np.where(null_key, np.int32(-1), key_len_of(spec, key_id)).astype(np.int32)

        rv = mix(seed, i, 3)
        tomb = rv % U(10000) < U(spec.tombstone_per_10k)
        empty = (rv >> U(20)) % U(10000) < U(spec.empty_value_per_10k)
        m = spec.value_mean                            # < 2^31, so v < 2^32 and v * 2^6 < 2^38: no wrap below
        v = U(m // 2) + mix(seed, i, 4) % U(m + 1)
        if spec.key_mode & synth.VALUES_GEOMETRIC:
            # times 2^k, P(k) = 2^-(k+1) for k < 6: k = the trailing zero bits of stream 6, capped at 6
            g = mix(seed, i, 6)
            k = np.zeros(i.shape, dtype=U)
            zeros_so_far = np.ones(i.shape, dtype=bool)
            for t in range(6):
                zeros_so_far &= ((g >> U(t)) & U(1)) == U(0)
                k += zeros_so_far
            v = np.minimum(v << k, U(INT32_MAX))
        v = v.astype(np.int64)
        assert v.size == 0 or v.max() <= INT32_MAX     # the spec's bound on value_mean keeps the uniform lengths in int32
        value_len = np.where(tomb, -1, np.where(empty, 0, v)).astype(np.int32)

        rt = mix(seed, i, 5)
        ts_missing = rt % U(10000) < U(spec.ts_missing_per_10k)
        ts = (U(TS_BASE) + i * U(7) + (rt >> U(32)) % U(1000)).astype(np.int64)
        ts_ms = np.where(ts_missing, np.int64(-1), ts)
    return dict(seq=i.copy(), partition=p.astype(np.int32), offset=offset, ts_ms=ts_ms, key_len=key_len,
                value_len=value_len, key_id=key_id)


def key_matrix(spec, key_id) -> np.ndarray:
    """(n, 40) uint8: row r holds the bytes of key key_id[r] in its first key_len_of(key_id[r]) columns."""
    key_id = np.asarray(key_id, dtype=U)
    n = key_id.shape[0]
    fmt = spec.key_mode & 0xFF
    out = np.zeros((n, MAX_KEY), dtype=np.uint8)
    with np.errstate(over="ignore"):
        if fmt == 0:                                   # (id, id * phi64), both little-endian
            words = np.stack([key_id, key_id * U(GOLDEN)], axis=1).astype("<u8")
            out[:, :16] = words.view(np.uint8).reshape(n, 16)
        elif fmt == 1:                                 # "key-" then the decimal digits, most significant first
            out[:, :4] = np.frombuffer(b"key-", dtype=np.uint8)
            nd = key_len_of(spec, key_id) - 4
            for t in range(20):                        # column 4 + t holds the digit of 10^(nd - 1 - t)
                e = nd - 1 - t
                digit = (key_id // POW10[np.maximum(e, 0)]) % U(10)
                out[:, 4 + t] = np.where(e >= 0, U(48) + digit, U(0)).astype(np.uint8)
        else:                                          # byte j: byte j % 8 of stream 8 + j / 8
            words = np.stack([mix(spec.seed, key_id, 8 + w) for w in range(MAX_KEY // 8)], axis=1).astype("<u8")
            out[:] = words.view(np.uint8).reshape(n, MAX_KEY)
    return out


def key_bytes_of(spec, key_id, key_len) -> np.ndarray:
    """The packed key buffer: the bytes of every non-null key, in record order, nothing for null or empty keys."""
    parts = []
    for a in range(0, len(key_len), CHUNK):
        kl = np.asarray(key_len[a:a + CHUNK])
        mat = key_matrix(spec, key_id[a:a + CHUNK])
        parts.append(mat[np.arange(MAX_KEY)[None, :] < kl[:, None]])
    return np.concatenate(parts) if parts else np.zeros(0, dtype=np.uint8)


def fill(spec, rank: int = 0, world: int = 1, start: int = 0, count: int | None = None) -> synth.HostTopic:
    """Local records [start, start + count) of shard `rank` of `world`, as synth.fill_host returns them."""
    if not valid(spec, rank, world):
        raise ValueError("invalid synthetic topic spec")
    shard = spec.n_total // world
    if count is None:
        count = shard - start
    if start < 0 or count < 0 or start + count > shard:
        raise ValueError("slice outside the shard")
    j = U(start) + np.arange(count, dtype=U)
    r = record_at(spec, local_to_global(spec, rank, world, j))
    kb = key_bytes_of(spec, r["key_id"], r["key_len"])
    return synth.HostTopic(r["partition"], r["offset"], r["ts_ms"], r["key_len"], r["value_len"], r["seq"], kb,
                           synth.tile_base_from_key_len(r["key_len"]))


COLUMNS = ("partition", "offset", "ts_ms", "key_len", "value_len", "seq", "key_bytes", "key_tile_base")


def first_difference(got: synth.HostTopic, want: synth.HostTopic, columns=COLUMNS):
    """None, or (column, first differing index, got, want) over `columns`; a length or type mismatch reports itself."""
    for name in columns:
        a, b = np.asarray(getattr(got, name)), np.asarray(getattr(want, name))
        if a.shape != b.shape or a.dtype != b.dtype:
            return name, min(a.size, b.size), (a.dtype.name, a.size), (b.dtype.name, b.size)
        bad = np.flatnonzero(a != b)
        if bad.size:
            k = int(bad[0])
            return name, k, a[k].item(), b[k].item()
    return None
