"""The synthetic topic record by record: tests/synth_ref.py, a plain numpy restatement of include/kta.h's definitions,
against the host generator (kta_synth_fill_host) over every column, seq, the packed key bytes and their length.  The
host and device generators share csrc/kta_synth.h, so these tests are the ones that can see a mistake in that header;
tests/test_synth_device.py then holds the device generator to the same restatement."""
import numpy as np
import pytest
from hypothesis import example, given, settings, strategies as st

from kafka_topic_analyzer_b200 import synth
from kafka_topic_analyzer_b200._native import ERR_INVALID, KtaError
import synth_ref as R

C3_SPEC = dict(n_total=4_000_000_000, num_partitions=256, distinct_keys=80_000_000, value_mean=1024,
               tombstone_per_10k=500, null_key_per_10k=100)   # bench.py's C3 topic: 8 ranks of 5e8 records


def assert_same(spec, rank, world, start, count):
    want = R.fill(spec, rank, world, start, count)
    got = synth.fill_host(spec, rank, world, start, count)
    diff = R.first_difference(got, want)
    assert diff is None, "rank %d/%d slice [%d, +%d): %s differs at %d: host %r, restatement %r" % (
        (rank, world, start, count) + diff)
    return want


@st.composite
def specs_and_slices(draw):
    P = draw(st.integers(1, 300))
    run_len = draw(st.sampled_from([1, 3, 500]))
    cycles = draw(st.one_of(st.integers(1, 8), st.integers(1, (2 ** 63 - 1) // (P * run_len))))
    distinct = draw(st.one_of(st.integers(0, P - 1), st.integers(P + 1, 10 ** 9).map(lambda d: d + (d % P == 0 and P > 1)),
                              st.just(2 ** 63), st.just(2 ** 64 - 1)))
    rate = st.one_of(st.sampled_from([0, 10000]), st.integers(0, 10000))
    value_mean = draw(st.one_of(st.sampled_from([0, 1, synth.MAX_VALUE_MEAN]), st.integers(0, synth.MAX_VALUE_MEAN)))
    spec = synth.make_spec(P * run_len * cycles, P, seed=draw(st.integers(0, 2 ** 64 - 1)), run_len=run_len,
                           distinct_keys=distinct, key_mode=draw(st.sampled_from([0, 1, 2])), value_mean=value_mean,
                           null_key_per_10k=draw(rate), tombstone_per_10k=draw(rate), ts_missing_per_10k=draw(rate),
                           empty_value_per_10k=draw(rate), zipf_keys=draw(st.booleans()),
                           geometric_values=draw(st.booleans()))
    world = draw(st.sampled_from([g for g in range(1, P + 1) if P % g == 0]))
    rank = draw(st.integers(0, world - 1))
    shard = spec.n_total // world
    start = draw(st.one_of(st.integers(0, shard), st.just(max(shard - 1, 0))))
    count = draw(st.one_of(st.sampled_from([0, 1]), st.integers(0, 700))) if start < shard else 0
    return spec, rank, world, start, min(count, shard - start)


@settings(max_examples=300, deadline=None)
@given(specs_and_slices())
@example((synth.make_spec(30 * 500 * 1000, 30, run_len=500, key_mode=1, value_mean=synth.MAX_VALUE_MEAN,
                          geometric_values=True), 2, 3, 3_777_777, 500))
def test_restatement_matches_host_generator(case):
    spec, rank, world, start, count = case
    assert synth.shard_records(spec, rank, world) == spec.n_total // world
    assert_same(spec, rank, world, start, count)


@pytest.mark.parametrize("run_len", [1, 3, 500])
@pytest.mark.parametrize("P,world", [(16, 16), (256, 8), (30, 3), (30, 5), (30, 6)])
def test_every_rank_mid_run_and_mid_cycle(P, world, run_len):
    # non-power-of-two worlds: a wrapped uint64 subtraction taken % world is only harmless when world divides 2^64
    spec = synth.make_spec(P * run_len * 2 ** 20, P, run_len=run_len, distinct_keys=P * 1000 + 7, ts_missing_per_10k=100)
    runs = P // world                                               # runs of one shard per cycle
    start = (777_777 * runs + runs // 2) * run_len + run_len // 2
    for rank in range(world):
        spec.key_mode = rank % 3
        t = assert_same(spec, rank, world, start, 1500)
        assert np.all(t.partition % world == rank)


@pytest.mark.parametrize("key_mode", [0, 1, 2])
@pytest.mark.parametrize("world,rank,where", [
    (1, 0, 2 ** 32 - 300), (1, 0, 2 ** 33 - 600),           # across global index 2^32, and the topic's end
])
def test_world_one_past_2_32(key_mode, world, rank, where):
    spec = synth.make_spec(2 ** 33, 64, key_mode=key_mode, distinct_keys=2 ** 64 - 1, ts_missing_per_10k=100,
                           empty_value_per_10k=100, zipf_keys=key_mode == 1, geometric_values=key_mode == 2)
    t = assert_same(spec, rank, world, where, 600)
    assert int(t.seq[0]) == where and int(t.seq[-1]) == where + 599


# C3's 4e9 records end below 2^32: rank 5 of 8 crosses 2^31 there, and the same topic at 2^33 records crosses 2^32
@pytest.mark.parametrize("n_total,edge", [(4_000_000_000, 2 ** 31), (2 ** 33, 2 ** 32)])
@pytest.mark.parametrize("key_mode", [0, 1, 2])
def test_rank_5_of_8_crossing(n_total, edge, key_mode):
    spec = synth.make_spec(**dict(C3_SPEC, n_total=n_total), key_mode=key_mode)
    j = R.local_index_of(spec, 5, 8, edge)
    t = assert_same(spec, 5, 8, j - 300, 600)
    assert int(t.seq[299]) < edge <= int(t.seq[300])
    assert np.all(t.partition % 8 == 5)


@pytest.mark.parametrize("rank", [0, 5, 7])
def test_last_records_of_the_4e9_topic(rank):
    spec = synth.make_spec(**C3_SPEC, key_mode=2, ts_missing_per_10k=100)
    shard = spec.n_total // 8
    t = assert_same(spec, rank, 8, shard - 1, 1)
    assert_same(spec, rank, 8, shard - 500, 500)
    if rank == 7:                                            # the same topic unsharded: its very last record
        last = assert_same(spec, 0, 1, spec.n_total - 1, 1)
        assert int(last.seq[0]) == 4_000_000_000 - 1 and int(t.seq[0]) <= int(last.seq[0])


def test_value_mean_bound():
    """kta.h: value_len is uniform in [mean/2, 3*mean/2]; the largest mean whose top length fits int32 is accepted, the
    next one refused by every host entry point."""
    top = synth.MAX_VALUE_MEAN
    assert top // 2 + top == 2 ** 31 - 1
    spec = synth.make_spec(4 * 10_000, 4, value_mean=top, tombstone_per_10k=0, empty_value_per_10k=0)
    t = assert_same(spec, 0, 1, 0, 40_000)
    assert t.value_len.min() >= top // 2 and t.value_len.max() <= 2 ** 31 - 1
    geo = synth.make_spec(4 * 10_000, 4, value_mean=top, tombstone_per_10k=0, geometric_values=True)
    g = assert_same(geo, 0, 1, 0, 40_000)
    assert g.value_len.min() >= top // 2 and (g.value_len == 2 ** 31 - 1).mean() > 0.4   # the clamp is reached
    over = synth.make_spec(4 * 10_000, 4, value_mean=top + 1)
    assert synth.synth_lib().kta_synth_shard_records(over, 0, 1) == -1
    assert not R.valid(over)
    with pytest.raises(KtaError) as e:
        synth.fill_host(over, count=10)
    assert e.value.code == ERR_INVALID


@settings(max_examples=300, deadline=None)
@given(P=st.integers(-2, 20), run_len=st.integers(-1, 4), cycles=st.integers(-1, 5), extra=st.sampled_from([0, 0, 1]),
       world=st.integers(-1, 8), rank=st.integers(-1, 8), key_mode=st.sampled_from([0, 1, 2, 3, 0x100, 0x302, 0x400, -1]),
       value_mean=st.sampled_from([-1, 0, synth.MAX_VALUE_MEAN, synth.MAX_VALUE_MEAN + 1, 2 ** 31 - 1]))
def test_spec_checks_match_kta_h(P, run_len, cycles, extra, world, rank, key_mode, value_mean):
    spec = synth.make_spec(P * run_len * cycles + extra, P, run_len=run_len, distinct_keys=7, value_mean=value_mean)
    spec.key_mode = key_mode
    n = synth.synth_lib().kta_synth_shard_records(spec, rank, world)
    assert n == (spec.n_total // world if R.valid(spec, rank, world) else -1)


def test_key_formats_at_the_extremes():
    """The largest key id a spec can produce is D - 1 < 2^64: ASCII "key-" + 20 digits is 24 bytes, the per-record
    bound DeviceTopic sizes its key buffer by; 16-byte keys are (id, id * phi64) little-endian."""
    ids = np.array([0, 9, 10, 99, 10 ** 19 - 1, 10 ** 19, 2 ** 64 - 1], dtype=np.uint64)
    ascii_spec = synth.make_spec(4, 1, key_mode=1)
    assert R.key_len_of(ascii_spec, ids).tolist() == [5, 5, 6, 6, 23, 24, 24]
    m = R.key_matrix(ascii_spec, ids)
    assert bytes(m[6, :24]) == b"key-18446744073709551615" and bytes(m[2, :6]) == b"key-10"
    m0 = R.key_matrix(synth.make_spec(4, 1, key_mode=0), ids[-1:])
    assert bytes(m0[0, :16]) == (2 ** 64 - 1).to_bytes(8, "little") + \
        (((2 ** 64 - 1) * 0x9E3779B97F4A7C15) % 2 ** 64).to_bytes(8, "little")
    assert R.splitmix64(0) == 0xE220A8397B1DCDAF          # splitmix64's published first output for state 0
    # a topic whose key ids reach 20 digits: the host generator agrees and no key is longer than 24 bytes
    spec = synth.make_spec(8 * 4096, 8, key_mode=1, distinct_keys=2 ** 64 - 1, null_key_per_10k=0)
    t = assert_same(spec, 0, 1, 0, 8 * 4096)
    assert t.key_len.max() == 24 and t.key_bytes.size <= 24 * t.n
