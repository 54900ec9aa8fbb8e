"""ctypes binding of libkta_gpu.so (include/kta.h) + the in-tree nvcc build recipe.

The library is the product; this module only loads it.  There is no Python/CPU implementation of
the scan anywhere in this package: if the shared object is missing or CUDA is unusable, calls fail
loudly (KtaError / OSError) instead of falling back.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess
import sys

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(_HERE, "csrc")
LIB_PATH = os.path.join(_HERE, "libkta_gpu.so")
SYNTH_LIB_PATH = os.path.join(_HERE, "libkta_synth.so")   # host-only synthetic topic generator (no CUDA)
INCLUDE = os.path.normpath(os.path.join(_HERE, "..", "include"))

KTA_KEY_TILE = 128
KTA_HIST_BUCKETS = 32
INT64_MIN = -(1 << 63)
SEQ_AUTO = (1 << 64) - 1   # include/kta.h KTA_SEQ_AUTO
READ_UNCOMMITTED, READ_COMMITTED = 0, 1   # include/kta.h KTA_READ_UNCOMMITTED / KTA_READ_COMMITTED
TIMELINE_RECORDS, TIMELINE_TOMBSTONES, TIMELINE_BYTES = 0, 1, 2   # include/kta.h KTA_TIMELINE_*
TIMELINE_MAX_BUCKETS = 65536
PARTITIONER_MAX_COUNTS = 8   # include/kta.h KTA_PARTITIONER_MAX_COUNTS
HOT_KEYS_MAX, HOT_KEY_PREFIX = 65536, 32   # include/kta.h KTA_HOT_KEYS_MAX / KTA_HOT_KEY_PREFIX

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17",
    "-Xcompiler", "-fPIC", "-shared", "--cudart", "static",
]


def _sources():
    return [os.path.join(CSRC, f) for f in sorted(os.listdir(CSRC)) if os.path.isfile(os.path.join(CSRC, f))] + \
           [os.path.join(INCLUDE, "kta.h")]


def build_synth(force: bool = False) -> str:
    """libkta_synth.so: the host half of the synthetic topic generator, plain g++, no CUDA anywhere."""
    srcs = [os.path.join(CSRC, "kta_synth_host.cpp"), os.path.join(CSRC, "kta_synth.h"), os.path.join(INCLUDE, "kta.h")]
    if not force and os.path.exists(SYNTH_LIB_PATH) and os.path.getmtime(SYNTH_LIB_PATH) >= max(os.path.getmtime(p) for p in srcs):
        return SYNTH_LIB_PATH
    cmd = [os.environ.get("CXX") or "g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-Wall", "-o", SYNTH_LIB_PATH, srcs[0]]
    res = subprocess.run(cmd, capture_output=True, text=True)
    if res.returncode != 0:
        raise RuntimeError("g++ failed:\n" + res.stdout + res.stderr)
    return SYNTH_LIB_PATH


def build(force: bool = False, verbose: bool = False) -> str:
    """Compile libkta_gpu.so for sm_90a (H100) with nvcc (cross-compiles without a GPU)."""
    out = LIB_PATH
    if not force and os.path.exists(out):
        newest = max(os.path.getmtime(p) for p in _sources())
        if os.path.getmtime(out) >= newest:
            return out
    nvcc = os.environ.get("NVCC") or "/usr/local/cuda/bin/nvcc"
    cmd = [nvcc, *NVCC_FLAGS, "-o", out, os.path.join(CSRC, "kta_lib.cu")]
    if verbose:
        cmd.insert(1, "-Xptxas=-v")
    res = subprocess.run(cmd, capture_output=True, text=True)
    if verbose:
        sys.stderr.write(res.stdout + res.stderr)
    if res.returncode != 0:
        raise RuntimeError("nvcc failed:\n" + res.stdout + res.stderr)
    return out


class KtaError(RuntimeError):
    def __init__(self, code: int, msg: str):
        super().__init__(f"kta error {code}: {msg}")
        self.code = code


OK, ERR_INVALID, ERR_CUDA, ERR_NOMEM, ERR_PARTITION, ERR_DIV_BY_ZERO, ERR_NOT_ENABLED, ERR_NOT_FINALIZED = range(8)


class Config(C.Structure):
    _fields_ = [
        ("struct_size", C.c_int32), ("device", C.c_int32), ("num_partitions", C.c_int32),
        ("count_alive_keys", C.c_int32), ("hll_precision", C.c_int32), ("alive_table_kib", C.c_int32),
        ("ring_records", C.c_int64), ("ring_key_bytes", C.c_int64), ("now_s", C.c_int64),
        ("now_ns", C.c_int32), ("isolation_level", C.c_int32), ("shard_world", C.c_int32), ("shard_rank", C.c_int32),
    ]


class Batch(C.Structure):
    _fields_ = [
        ("n", C.c_int64), ("seq_base", C.c_uint64), ("partition", C.c_void_p), ("offset", C.c_void_p),
        ("ts_ms", C.c_void_p), ("key_len", C.c_void_p), ("value_len", C.c_void_p), ("key_bytes", C.c_void_p),
        ("key_bytes_len", C.c_int64), ("key_tile_base", C.c_void_p), ("seq", C.c_void_p),
    ]


class SynthSpec(C.Structure):
    _fields_ = [
        ("seed", C.c_uint64), ("n_total", C.c_int64), ("num_partitions", C.c_int32), ("run_len", C.c_int32),
        ("distinct_keys", C.c_uint64), ("key_mode", C.c_int32), ("value_mean", C.c_int32),
        ("null_key_per_10k", C.c_int32), ("tombstone_per_10k", C.c_int32), ("ts_missing_per_10k", C.c_int32),
        ("empty_value_per_10k", C.c_int32),
    ]


class CrcFailure(C.Structure):
    _fields_ = [
        ("partition", C.c_int32), ("batch_bytes", C.c_uint32), ("base_offset", C.c_int64),
        ("stored_crc", C.c_uint32), ("computed_crc", C.c_uint32),
    ]


LOG_CRC_KEEP = 4096   # include/kta.h KTA_LOG_CRC_KEEP


class HotKey(C.Structure):
    _fields_ = [
        ("id", C.c_uint64), ("records", C.c_uint64), ("tombstones", C.c_uint64), ("bytes", C.c_uint64),
        ("latest_s", C.c_int64), ("min_partition", C.c_int32), ("max_partition", C.c_int32), ("key_len", C.c_int32),
        ("reserved", C.c_uint32), ("key_prefix", C.c_uint8 * HOT_KEY_PREFIX),
    ]


# include/kta.h kta_hot_key as a numpy record (88 bytes, the same offsets)
HOT_KEY_DTYPE = np.dtype([
    ("id", "<u8"), ("records", "<u8"), ("tombstones", "<u8"), ("bytes", "<u8"), ("latest_s", "<i8"),
    ("min_partition", "<i4"), ("max_partition", "<i4"), ("key_len", "<i4"), ("reserved", "<u4"),
    ("key_prefix", "u1", (HOT_KEY_PREFIX,))])


# every symbol include/kta.h declares: name -> (restype, argtypes)
_P = C.c_void_p
SYMBOLS = {
    "kta_last_error": (C.c_char_p, []),
    "kta_abi_version": (C.c_int, []),
    "kta_device_count": (C.c_int, []),
    "kta_create": (C.c_int, [C.POINTER(Config), C.POINTER(_P)]),
    "kta_destroy": (C.c_int, [_P]),
    "kta_reset": (C.c_int, [_P]),
    "kta_push": (C.c_int, [_P, C.c_int32, C.c_int64, C.c_int64, _P, C.c_int32, C.c_int32]),
    "kta_push_batch_host": (C.c_int, [_P, C.POINTER(Batch)]),
    "kta_scan_batch_device": (C.c_int, [_P, C.POINTER(Batch)]),
    "kta_sync": (C.c_int, [_P]),
    "kta_finalize": (C.c_int, [_P]),
    "kta_counter": (C.c_int, [_P, C.c_int, C.c_int32, C.POINTER(C.c_uint64)]),
    "kta_avg": (C.c_int, [_P, C.c_int, C.c_int32, C.POINTER(C.c_uint64)]),
    "kta_dirty_ratio": (C.c_int, [_P, C.c_int32, C.POINTER(C.c_float)]),
    "kta_global": (C.c_int, [_P, C.c_int, C.POINTER(C.c_uint64)]),
    "kta_timestamps": (C.c_int, [_P, C.POINTER(C.c_int64), C.POINTER(C.c_int32), C.POINTER(C.c_int64)]),
    "kta_alive_keys": (C.c_int, [_P, C.POINTER(C.c_uint64)]),
    "kta_bad_partition_records": (C.c_int, [_P, C.POINTER(C.c_uint64)]),
    "kta_alive_table_stats": (C.c_int, [_P, C.POINTER(C.c_uint64), C.POINTER(C.c_uint64), C.POINTER(C.c_uint64),
                                        C.POINTER(C.c_uint64)]),
    "kta_hist": (C.c_int, [_P, C.c_int, C.c_int32, C.POINTER(C.c_uint64)]),
    "kta_alive_keys_hll": (C.c_int, [_P, C.POINTER(C.c_double)]),
    "kta_hll_registers": (C.c_int, [_P, _P, C.c_size_t]),
    "kta_fnv32_host": (C.c_int, [_P, C.c_int64, _P, _P, C.c_int64, _P]),
    "kta_set_timeline": (C.c_int, [_P, C.c_int64, C.c_int64, C.c_int32]),
    "kta_timeline": (C.c_int, [_P, C.c_int, C.c_int32, C.POINTER(C.c_uint64), C.c_int64]),
    "kta_set_partitioner_check": (C.c_int, [_P, C.POINTER(C.c_int32), C.c_int32]),
    "kta_partitioner_check": (C.c_int, [_P, C.c_int32, C.POINTER(C.c_uint64), C.c_int64]),
    "kta_partitioner_hash_host": (C.c_int, [_P, C.c_int64, _P, _P, C.c_int64, _P, _P]),
    "kta_set_hot_keys": (C.c_int, [_P, C.c_int32, C.c_int64]),
    "kta_hot_keys": (C.c_int, [_P, _P, C.c_int64, C.POINTER(C.c_int64)]),
    "kta_hot_key_stats": (C.c_int, [_P, C.POINTER(C.c_uint64), C.POINTER(C.c_uint64), C.POINTER(C.c_uint64),
                                    C.POINTER(C.c_uint64), C.POINTER(C.c_uint64)]),
    "kta_hot_keys_export_count": (C.c_int, [_P, C.POINTER(C.c_int64)]),
    "kta_hot_keys_export_device": (C.c_int, [_P, _P, C.c_int64, C.POINTER(C.c_int64)]),
    "kta_hot_keys_import_device": (C.c_int, [_P, _P, C.c_int64]),
    "kta_hot_keys_limit_slots": (C.c_int, [_P, C.c_int64]),
    "kta_merge_words": (C.c_int64, [_P, C.c_int32]),
    "kta_merge_export_device": (C.c_int, [_P, C.c_int32, C.c_int32, _P]),
    "kta_merge_import_device": (C.c_int, [_P, C.c_int32, _P]),
    "kta_alive_export_count": (C.c_int, [_P, C.POINTER(C.c_int64)]),
    "kta_alive_export_device": (C.c_int, [_P, _P, _P, C.c_int64, C.POINTER(C.c_int64)]),
    "kta_alive_import_device": (C.c_int, [_P, _P, _P, C.c_int64]),
    "kta_scan_log_segment_device": (C.c_int, [_P, C.c_int32, _P, C.c_int64, _P, C.c_int64, C.POINTER(C.c_int64)]),
    "kta_scan_log_batches_device": (C.c_int, [_P, _P, C.c_int64, _P, _P, C.c_int64, C.POINTER(C.c_int64)]),
    "kta_push_log_segment_host": (C.c_int, [_P, C.c_int32, _P, C.c_int64, C.POINTER(C.c_int64)]),
    "kta_push_log_segments_host": (C.c_int, [_P, C.c_int32, _P, _P, _P, C.POINTER(C.c_int64)]),
    "kta_log_add_txn_index_host": (C.c_int, [_P, C.c_int32, _P, C.c_int64]),
    "kta_log_txn_stats": (C.c_int, [_P, C.POINTER(C.c_uint64), C.POINTER(C.c_uint64), C.POINTER(C.c_uint64)]),
    "kta_log_set_check_crcs": (C.c_int, [_P, C.c_int]),
    "kta_log_crc_stats": (C.c_int, [_P, C.POINTER(C.c_uint64), C.POINTER(C.c_uint64), C.POINTER(C.c_uint64)]),
    "kta_log_crc_failures": (C.c_int, [_P, C.POINTER(CrcFailure), C.c_int64, C.POINTER(C.c_int64)]),
    "kta_log_set_offsets": (C.c_int, [_P, C.c_int32, C.c_int64, C.c_int64]),
    "kta_log_offset_stats": (C.c_int, [_P, C.POINTER(C.c_uint64), C.POINTER(C.c_uint64)]),
    "kta_stats": (C.c_int, [_P, C.POINTER(C.c_uint64), C.POINTER(C.c_uint64)]),
    "kta_set_timing": (C.c_int, [_P, C.c_int]),
    "kta_scan_time_ms": (C.c_int, [_P, C.POINTER(C.c_double), C.POINTER(C.c_uint64)]),
    "kta_stream": (_P, [_P]),
    "kta_set_stream": (C.c_int, [_P, _P]),
    "kta_synth_shard_records": (C.c_int64, [C.POINTER(SynthSpec), C.c_int32, C.c_int32]),
    "kta_synth_fill_host": (C.c_int, [C.POINTER(SynthSpec), C.c_int32, C.c_int32, C.c_int64, C.c_int64,
                                      _P, _P, _P, _P, _P, _P, _P, C.c_int64, C.POINTER(C.c_int64)]),
    "kta_synth_fill_device": (C.c_int, [C.POINTER(SynthSpec), C.c_int32, C.c_int32, C.c_int32, C.c_int64, C.c_int64,
                                        _P, _P, _P, _P, _P, _P, _P, C.c_int64, _P, C.POINTER(C.c_int64)]),
    "kta_synth_encode_segment_host": (C.c_int, [C.POINTER(SynthSpec), C.c_int32, C.c_int64, C.c_int64, C.c_int32, _P, C.c_int64,
                                                C.POINTER(C.c_int64)]),
    # test hook, not part of kta.h's stable surface
    "kta_set_hash_capture": (C.c_int, [_P, _P]),
    "kta_timeline_shape": (C.c_int, [_P, C.c_int64, C.POINTER(C.c_int32), C.POINTER(C.c_int32), C.POINTER(C.c_int32)]),
    "kta_partitioner_limit_grid": (C.c_int, [_P, C.c_int32]),
    "kta_partitioner_shape": (C.c_int, [_P, C.c_int64, C.c_int64, C.POINTER(C.c_int32), C.POINTER(C.c_int32),
                                        C.POINTER(C.c_int32)]),
}

_lib = None
_synth = None
SYNTH_HOST_SYMBOLS = ("kta_synth_shard_records", "kta_synth_fill_host", "kta_synth_encode_segment_host")


def synth_lib() -> C.CDLL:
    """The host-only generator library (never touches CUDA; safe for the CPU reference arm)."""
    global _synth
    if _synth is None:
        if not (os.environ.get("KTA_NO_BUILD") == "1" and os.path.exists(SYNTH_LIB_PATH)):
            build_synth()
        _synth = C.CDLL(SYNTH_LIB_PATH)
        for name in SYNTH_HOST_SYMBOLS:
            fn = getattr(_synth, name)
            fn.restype, fn.argtypes = SYMBOLS[name]
    return _synth


def lib() -> C.CDLL:
    """Load libkta_gpu.so (building it first if the sources are newer / it is missing)."""
    global _lib
    if _lib is None:
        path = os.environ.get("KTA_LIB")   # KTA_LIB: an experimental build of the same sources, used as it is
        if not path:
            # (re)build when the library is missing or older than any source; a failed nvcc run surfaces as an error
            # instead of silently testing a stale binary.  KTA_NO_BUILD=1: use the shipped .so as it is (no nvcc needed).
            path = LIB_PATH
            if not (os.environ.get("KTA_NO_BUILD") == "1" and os.path.exists(path)):
                build()
        _lib = C.CDLL(path)
        for name, (res, args) in SYMBOLS.items():
            fn = getattr(_lib, name)  # AttributeError if the export is missing: loud by design
            fn.restype = res
            fn.argtypes = args
    return _lib


def check(rc: int) -> None:
    if rc != 0:
        raise KtaError(rc, (lib().kta_last_error() or b"").decode("utf-8", "replace"))
