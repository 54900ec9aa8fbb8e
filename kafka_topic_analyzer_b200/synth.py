"""Synthetic in-memory topic (BASELINE.json configs; SURVEY.md §8 d) — Python face of
csrc/kta_synth.{h,cu}.  The generator itself is C++ shared by host and device."""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass
from typing import Optional

import numpy as np

from . import _native as N
from ._native import SynthSpec, KtaError, lib, synth_lib

DEFAULT_SEED = 0x4B544131  # "KTA1"
KEYS_LOGUNIFORM = 0x100     # include/kta.h KTA_SYNTH_KEYS_LOGUNIFORM
VALUES_GEOMETRIC = 0x200    # include/kta.h KTA_SYNTH_VALUES_GEOMETRIC
MAX_VALUE_MEAN = 1431655765  # include/kta.h KTA_SYNTH_MAX_VALUE_MEAN: floor(mean/2) + mean == INT32_MAX


@dataclass
class HostTopic:
    partition: np.ndarray
    offset: np.ndarray
    ts_ms: np.ndarray
    key_len: np.ndarray
    value_len: np.ndarray
    seq: np.ndarray
    key_bytes: np.ndarray
    key_tile_base: np.ndarray

    @property
    def n(self) -> int:
        return int(self.partition.shape[0])


def make_spec(n_total: int, num_partitions: int, *, seed: int = DEFAULT_SEED, run_len: int = 1,
              distinct_keys: Optional[int] = None, key_mode: int = 0, value_mean: int = 256,
              null_key_per_10k: int = 100, tombstone_per_10k: int = 500, ts_missing_per_10k: int = 0,
              empty_value_per_10k: int = 0, zipf_keys: bool = False, geometric_values: bool = False) -> SynthSpec:
    """`zipf_keys`: log-uniform key ids (a Zipf s = 1 staircase: few hot keys, long cold tail);
    `geometric_values`: value length x 2^g with P(g = k) = 2^-(k+1), g <= 6 (SURVEY.md §8 d stress cases)."""
    s = SynthSpec()
    s.seed = seed
    s.n_total = n_total
    s.num_partitions = num_partitions
    s.run_len = run_len
    s.distinct_keys = distinct_keys if distinct_keys is not None else max(num_partitions, n_total // 10)
    s.key_mode = key_mode | (KEYS_LOGUNIFORM if zipf_keys else 0) | (VALUES_GEOMETRIC if geometric_values else 0)
    s.value_mean = value_mean
    s.null_key_per_10k = null_key_per_10k
    s.tombstone_per_10k = tombstone_per_10k
    s.ts_missing_per_10k = ts_missing_per_10k
    s.empty_value_per_10k = empty_value_per_10k
    return s


def shard_records(spec: SynthSpec, rank: int = 0, world: int = 1) -> int:
    n = synth_lib().kta_synth_shard_records(C.byref(spec), rank, world)
    if n < 0:
        raise KtaError(N.ERR_INVALID, "invalid synthetic topic spec (n_total must be a multiple of "
                       "num_partitions*run_len; num_partitions a multiple of world; value_mean at most "
                       "%d)" % MAX_VALUE_MEAN)
    return n


def tile_base_from_key_len(key_len: np.ndarray) -> np.ndarray:
    """key_tile_base column for a host batch (a feeder-side prefix sum, not a metric)."""
    kl = np.maximum(key_len.astype(np.int64), 0)
    n = kl.shape[0]
    ntiles = (n + N.KTA_KEY_TILE - 1) // N.KTA_KEY_TILE
    pad = ntiles * N.KTA_KEY_TILE - n
    sums = np.concatenate([kl, np.zeros(pad, dtype=np.int64)]).reshape(ntiles, N.KTA_KEY_TILE).sum(axis=1)
    out = np.zeros(ntiles + 1, dtype=np.uint64)
    out[1:] = np.cumsum(sums).astype(np.uint64)
    return out


def fill_host(spec: SynthSpec, rank: int = 0, world: int = 1, start: int = 0, count: Optional[int] = None) -> HostTopic:
    if count is None:
        count = shard_records(spec, rank, world) - start
    part = np.zeros(count, dtype=np.int32)
    off = np.zeros(count, dtype=np.int64)
    ts = np.zeros(count, dtype=np.int64)
    kl = np.zeros(count, dtype=np.int32)
    vl = np.zeros(count, dtype=np.int32)
    seq = np.zeros(count, dtype=np.uint64)
    cap = count * 40 + 16
    kb = np.zeros(cap, dtype=np.uint8)
    kbl = C.c_int64()
    rc = synth_lib().kta_synth_fill_host(C.byref(spec), rank, world, start, count, part.ctypes.data, off.ctypes.data,
                                   ts.ctypes.data, kl.ctypes.data, vl.ctypes.data, seq.ctypes.data, kb.ctypes.data,
                                   cap, C.byref(kbl))
    if rc != 0:
        raise KtaError(rc, "kta_synth_fill_host failed")
    kb = kb[: kbl.value].copy()
    return HostTopic(part, off, ts, kl, vl, seq, kb, tile_base_from_key_len(kl))


def encode_segment(spec: SynthSpec, partition: int, start: int = 0, count: Optional[int] = None, batch_records: int = 500) -> np.ndarray:
    """One partition of the synthetic topic as an uncompressed RecordBatch v2 log segment (host bytes)."""
    if count is None:
        count = spec.n_total // spec.num_partitions - start
    n = C.c_int64()
    rc = synth_lib().kta_synth_encode_segment_host(C.byref(spec), partition, start, count, batch_records, None, 0, C.byref(n))
    if rc != 0:
        raise KtaError(rc, "kta_synth_encode_segment_host failed")
    out = np.empty(n.value, dtype=np.uint8)
    rc = synth_lib().kta_synth_encode_segment_host(C.byref(spec), partition, start, count, batch_records, out.ctypes.data, out.size, C.byref(n))
    if rc != 0:
        raise KtaError(rc, "kta_synth_encode_segment_host failed")
    return out


class DeviceTopic:
    """SoA columns of one shard of the synthetic topic, generated directly in HBM (torch owns the memory)."""

    def __init__(self, spec: SynthSpec, rank: int = 0, world: int = 1, start: int = 0, count: Optional[int] = None,
                 device: int = 0, with_seq: bool = False, with_offset: bool = False, max_key: int = 40):
        import torch

        if count is None:
            count = shard_records(spec, rank, world) - start
        dev = torch.device("cuda", device)
        self.n = count
        self.partition = torch.empty(count, dtype=torch.int32, device=dev)
        self.ts_ms = torch.empty(count, dtype=torch.int64, device=dev)
        self.key_len = torch.empty(count, dtype=torch.int32, device=dev)
        self.value_len = torch.empty(count, dtype=torch.int32, device=dev)
        self.seq = torch.empty(count, dtype=torch.int64, device=dev) if with_seq else None
        self.offset = torch.empty(count, dtype=torch.int64, device=dev) if with_offset else None
        fmt = spec.key_mode & 0xFF
        per_key = 16 if fmt == 0 else (24 if fmt == 1 else max_key)
        cap = count * per_key + 64
        self.key_bytes = torch.empty(cap, dtype=torch.uint8, device=dev)
        ntiles = (count + N.KTA_KEY_TILE - 1) // N.KTA_KEY_TILE
        self.key_tile_base = torch.empty(ntiles + 1, dtype=torch.int64, device=dev)
        kbl = C.c_int64()
        torch.cuda.synchronize(dev)
        rc = lib().kta_synth_fill_device(
            C.byref(spec), device, rank, world, start, count, self.partition.data_ptr(),
            self.offset.data_ptr() if with_offset else None, self.ts_ms.data_ptr(), self.key_len.data_ptr(),
            self.value_len.data_ptr(), self.seq.data_ptr() if with_seq else None, self.key_bytes.data_ptr(), cap,
            self.key_tile_base.data_ptr(), C.byref(kbl))
        if rc != 0:
            raise KtaError(rc, "kta_synth_fill_device failed")
        self.key_bytes_len = kbl.value

    def to_host(self) -> HostTopic:
        z = np.zeros(0, dtype=np.int64)
        return HostTopic(
            self.partition.cpu().numpy(), self.offset.cpu().numpy() if self.offset is not None else z,
            self.ts_ms.cpu().numpy(), self.key_len.cpu().numpy(), self.value_len.cpu().numpy(),
            self.seq.cpu().numpy().view(np.uint64) if self.seq is not None else z.view(np.uint64),
            self.key_bytes[: self.key_bytes_len].cpu().numpy(), self.key_tile_base.cpu().numpy().view(np.uint64))
