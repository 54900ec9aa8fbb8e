"""The synthetic topic generated in HBM, record by record against tests/synth_ref.py (itself pinned to the host
generator by tests/test_synth_ref.py).

kta_synth_fill_device runs synth_columns_kernel (the six columns), then derives key_tile_base with the library's own
tile_key_bytes_kernel (one warp per 128-record tile) and tile_base_scan_kernel (one CTA, 1024 tiles per pass, a carry
between passes), then synth_keys_kernel (one warp per tile, a lane owning 4 consecutive records) writes the key bytes.
Every column, seq, the packed key bytes and key_tile_base are compared whole, at the tile and lane edges of the key
kernel, the pass edges of the scan, shards of power-of-two and other worlds, global indices past 2^31 and 2^32, and the
topics bench.py scans.  A mismatch names its column and first differing index."""
import ctypes as C
import sys

import numpy as np
import pytest
import torch

import synth_ref as R
from kafka_topic_analyzer_b200 import synth
from kafka_topic_analyzer_b200 import _native as N

T = N.KTA_KEY_TILE
SCAN_PASS = 1024                         # tiles per pass of tile_base_scan_kernel
C3_SPEC = dict(num_partitions=256, distinct_keys=80_000_000, value_mean=1024, tombstone_per_10k=500,
               null_key_per_10k=100)     # bench.py's C3 topic (n_total 4e9: 8 ranks of 5e8)


def on_device(spec, rank, world, start, count):
    t = synth.DeviceTopic(spec, rank=rank, world=world, start=start, count=count, with_seq=True, with_offset=True)
    h = t.to_host()
    assert h.key_tile_base.size == (count + T - 1) // T + 1
    return h


def assert_device_matches(spec, rank, world, start, count, want=None, what="restatement"):
    got = on_device(spec, rank, world, start, count)
    want = R.fill(spec, rank, world, start, count) if want is None else want
    diff = R.first_difference(got, want)
    assert diff is None, "rank %d/%d slice [%d, +%d): %s differs at %d: device %r, %s %r" % (
        (rank, world, start, count) + diff[:3] + (what, diff[3]))
    return got


# ------------------------------------------------------------------------------------------------
# synth_keys_kernel: a warp per 128-record tile, 4 consecutive records per lane
# ------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("world", [1, 3])
@pytest.mark.parametrize("key_mode", [0, 1, 2])
def test_tile_and_lane_edges(key_mode, world):
    spec = synth.make_spec(12 * 3 * 3000, 12, run_len=3, key_mode=key_mode, distinct_keys=5000, null_key_per_10k=1500,
                           tombstone_per_10k=1000, empty_value_per_10k=500, ts_missing_per_10k=300)
    rank = world - 1
    shard = synth.shard_records(spec, rank, world)
    kinds = set()
    for count in (1, 31, 32, 33, 127, 128, 129, 4095):
        for start in (0, 1, 127, 129, shard - count):
            t = assert_device_matches(spec, rank, world, start, count)
            kinds |= set(np.sign(t.key_len).tolist())
    assert {-1, 1} <= kinds and (key_mode != 2 or 0 in kinds)   # null keys present; key_mode 2 also has 0-byte keys


# ------------------------------------------------------------------------------------------------
# tile_base_scan_kernel: 1024 tiles per pass, the carry from the second pass on
# ------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("ntiles", [1023, 1024, 1025, 2048, 2049])
def test_tile_base_scan_pass_edges(ntiles):
    spec = synth.make_spec(16 * 2 ** 20, 16, key_mode=2, distinct_keys=10 ** 6, null_key_per_10k=500)
    count = (ntiles - 1) * T + 77                                    # the last tile is a partial one
    t = assert_device_matches(spec, 0, 1, 1000, count)
    assert t.key_tile_base.size == ntiles + 1 and int(t.key_tile_base[-1]) == t.key_bytes.size


@pytest.mark.gpu
def test_tile_base_scan_at_129_passes():
    """2^24 + 77 records = 131 073 tiles: 128 full passes of the scan and one of a single tile, at the end of C3's rank 5
    with ragged keys.  The host generator is the reference at this size (the restatement is pinned to it)."""
    spec = synth.make_spec(4_000_000_000, **dict(C3_SPEC, null_key_per_10k=300), key_mode=2, ts_missing_per_10k=50)
    count = 2 ** 24 + 77
    start = synth.shard_records(spec, 5, 8) - count
    assert (count + T - 1) // T == 128 * SCAN_PASS + 1
    assert_device_matches(spec, 5, 8, start, count, want=synth.fill_host(spec, 5, 8, start, count), what="host")


# ------------------------------------------------------------------------------------------------
# shards and runs: every rank, slices starting mid-run and mid-cycle, and each shard's last records
# ------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("run_len", [1, 3, 500])
@pytest.mark.parametrize("P,world", [(16, 2), (16, 4), (16, 8), (16, 16), (256, 8), (30, 3), (30, 5), (30, 6)])
def test_shards_and_runs(P, world, run_len):
    # non-power-of-two worlds: a wrapped uint64 subtraction taken % world is only harmless when world divides 2^64
    cycles = 2 ** 20
    spec = synth.make_spec(P * run_len * cycles, P, run_len=run_len, distinct_keys=P * 1000 + 7, ts_missing_per_10k=100,
                           empty_value_per_10k=100)
    runs = P // world                                               # runs of one shard per cycle
    start = (777_777 * runs + runs // 2) * run_len + run_len // 2
    for rank in range(world):
        spec.key_mode = rank % 3
        shard = synth.shard_records(spec, rank, world)
        t = assert_device_matches(spec, rank, world, start, 3000)
        assert np.all(t.partition % world == rank)
        assert_device_matches(spec, rank, world, shard - 700, 700)


# ------------------------------------------------------------------------------------------------
# global indices past 2^31 and 2^32 (only the slice is generated)
# ------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("key_mode", [0, 1, 2])
def test_past_2_32(key_mode):
    # C3's 4e9 records end below 2^32: its rank 5 crosses 2^31, and the same sharding at 2^33 records crosses 2^32
    for n_total, edge in ((4_000_000_000, 2 ** 31), (2 ** 33, 2 ** 32)):
        spec = synth.make_spec(n_total, **C3_SPEC, key_mode=key_mode, ts_missing_per_10k=100)
        j = R.local_index_of(spec, 5, 8, edge)
        t = assert_device_matches(spec, 5, 8, j - 2 ** 15, 2 ** 16)
        assert int(t.seq[2 ** 15 - 1]) < edge <= int(t.seq[2 ** 15])
        for rank in (5, 7):
            assert_device_matches(spec, rank, 8, spec.n_total // 8 - 2 ** 16, 2 ** 16)
    one = synth.make_spec(2 ** 33, 64, key_mode=key_mode, distinct_keys=2 ** 64 - 1, zipf_keys=True, geometric_values=True)
    t = assert_device_matches(one, 0, 1, 2 ** 32 - 2 ** 15, 2 ** 16)
    assert int(t.seq[2 ** 15]) == 2 ** 32


# ------------------------------------------------------------------------------------------------
# the topics bench.py scans, built the way bench.py builds them
# ------------------------------------------------------------------------------------------------
def bench_args(monkeypatch, argv):
    import bench
    monkeypatch.setattr(sys, "argv", ["bench.py", "--gpus", "1"] + argv)
    return bench, bench.parse()


@pytest.mark.gpu
@pytest.mark.parametrize("argv", [["--config", "C1"], ["--config", "C2"], ["--config", "C3"], ["--config", "C4"],
                                  ["--config", "C4", "--value-mean", "65536"],
                                  ["--config", "C1", "--key-mode", "1"], ["--config", "C1", "--key-mode", "2"],
                                  ["--config", "C1", "--zipf-keys"], ["--config", "C1", "--geometric-values"]],
                         ids=lambda a: "-".join(x.strip("-") for x in a))
def test_bench_topics(monkeypatch, argv):
    bench, a = bench_args(monkeypatch, argv)
    spec, world = bench.make_spec(a, 1), bench.virtual_world(a, 1)
    assert world == (8 if a.config == "C3" else 1)
    n = 2 ** 20
    for rank in sorted({0, world - 1}):
        shard = synth.shard_records(spec, rank, world)
        assert shard == a.n
        for start in (0, (shard - n) // 2, shard - n):
            assert_device_matches(spec, rank, world, start, n)


# ------------------------------------------------------------------------------------------------
# the key buffer's cap, the refusal without tile bases, the value_mean bound
# ------------------------------------------------------------------------------------------------
class Raw:
    """The columns of one direct kta_synth_fill_device call, prefilled with sentinels."""
    SENTINEL = -7

    def __init__(self, count, key_cap):
        dev = torch.device("cuda", 0)
        self.count = count
        self.partition = torch.full((count,), self.SENTINEL, dtype=torch.int32, device=dev)
        self.ts_ms = torch.full((count,), self.SENTINEL, dtype=torch.int64, device=dev)
        self.key_len = torch.full((count,), self.SENTINEL, dtype=torch.int32, device=dev)
        self.value_len = torch.full((count,), self.SENTINEL, dtype=torch.int32, device=dev)
        self.key_bytes = torch.full((key_cap,), 0xA5, dtype=torch.uint8, device=dev)
        self.key_tile_base = torch.full(((count + T - 1) // T + 1,), self.SENTINEL, dtype=torch.int64, device=dev)
        self.kbl = C.c_int64(self.SENTINEL)

    def fill(self, spec, start, cap, key_bytes=True, key_tile_base=True, key_bytes_len=True):
        torch.cuda.synchronize()
        return N.lib().kta_synth_fill_device(
            C.byref(spec), 0, 0, 1, start, self.count, self.partition.data_ptr(), None, self.ts_ms.data_ptr(),
            self.key_len.data_ptr(), self.value_len.data_ptr(), None, self.key_bytes.data_ptr() if key_bytes else None,
            cap, self.key_tile_base.data_ptr() if key_tile_base else None, C.byref(self.kbl) if key_bytes_len else None)

    def untouched(self):
        cols = (self.partition, self.ts_ms, self.key_len, self.value_len, self.key_tile_base)
        return all(bool((c == self.SENTINEL).all()) for c in cols) and bool((self.key_bytes == 0xA5).all()) \
            and self.kbl.value == self.SENTINEL


@pytest.mark.gpu
@pytest.mark.parametrize("key_mode", [0, 1, 2])
def test_key_buffer_cap(key_mode):
    spec = synth.make_spec(8 * 5000, 8, key_mode=key_mode, distinct_keys=4000, null_key_per_10k=800)
    want = R.fill(spec, 0, 1, 333, 5000)
    total = want.key_bytes.size
    raw = Raw(5000, total + 64)
    assert raw.fill(spec, 333, total) == N.OK and raw.kbl.value == total
    kb = raw.key_bytes.cpu().numpy()
    assert np.array_equal(kb[:total], want.key_bytes) and np.all(kb[total:] == 0xA5)
    assert np.array_equal(raw.key_tile_base.cpu().numpy().view(np.uint64), want.key_tile_base)
    raw = Raw(5000, total + 64)
    assert raw.fill(spec, 333, total - 1) == N.ERR_NOMEM
    assert bool((raw.key_bytes == 0xA5).all())                  # not one key byte, the one just past the cap included


@pytest.mark.gpu
@pytest.mark.parametrize("key_mode,longest", [(0, 16), (1, 24), (2, 40)])
def test_per_mode_cap_holds_for_the_largest_key_ids(key_mode, longest):
    """DeviceTopic sizes its key buffer at 16 / 24 / 40 bytes a record; key ids reach D - 1 = 2^64 - 2 here, so ASCII keys
    reach "key-" + 20 digits."""
    spec = synth.make_spec(8 * 8192, 8, key_mode=key_mode, distinct_keys=2 ** 64 - 1, null_key_per_10k=0)
    t = assert_device_matches(spec, 0, 1, 0, 8 * 8192)
    assert t.key_len.max() == longest and t.key_bytes.size <= longest * t.n


@pytest.mark.gpu
def test_key_bytes_without_tile_bases_are_refused():
    """The key bytes are placed by the tile bases; a call that asks for key bytes or their length without them is
    refused before anything is written."""
    spec = synth.make_spec(8 * 1000, 8, key_mode=2)
    for kb, kbl in ((True, True), (True, False), (False, True)):
        raw = Raw(1000, 1000 * 40)
        assert raw.fill(spec, 0, 1000 * 40, key_bytes=kb, key_tile_base=False, key_bytes_len=kbl) == N.ERR_INVALID, (kb, kbl)
        assert raw.untouched(), (kb, kbl)
    raw = Raw(1000, 1000 * 40)                                  # columns only, no key bytes: still a valid call
    assert raw.fill(spec, 0, 0, key_bytes=False, key_tile_base=False, key_bytes_len=False) == N.OK
    want = R.fill(spec, 0, 1, 0, 1000)
    assert np.array_equal(raw.key_len.cpu().numpy(), want.key_len)
    assert np.array_equal(raw.value_len.cpu().numpy(), want.value_len)


@pytest.mark.gpu
@pytest.mark.parametrize("geometric", [False, True])
def test_value_mean_bound_on_device(geometric):
    top = synth.MAX_VALUE_MEAN
    spec = synth.make_spec(4 * 10_000, 4, value_mean=top, tombstone_per_10k=0, geometric_values=geometric)
    host = synth.fill_host(spec)
    t = assert_device_matches(spec, 0, 1, 0, spec.n_total, want=host, what="host")
    assert t.value_len.min() >= top // 2
    assert R.first_difference(t, R.fill(spec)) is None
    spec.value_mean = top + 1
    raw = Raw(1000, 1000 * 16)
    assert raw.fill(spec, 0, 1000 * 16) == N.ERR_INVALID and raw.untouched()
