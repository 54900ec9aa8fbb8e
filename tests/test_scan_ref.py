"""The torch restatement of the scan's outputs (scan_ref.py), pinned to the CPU oracle and to np_oracle on CPU tensors, so
that the GPU depth tests that rely on it (test_scan_depth.py) compare the kernel with something already checked."""
import numpy as np
import pytest
import torch

import np_oracle
import scan_ref as R
from kafka_topic_analyzer_b200 import synth
from feed import random_topic, take
from oracle_lib import COUNTERS
from parity import oracle_for

NOW = (4102444800, 123456789)
N = 1 << 16


def _topics():
    rng = np.random.default_rng(4)
    t = random_topic(rng, N, 7, big=True)
    neg = rng.random(N) < 0.01                      # timestamps before the epoch: truncating division
    t.ts_ms[neg] = rng.choice(np.array([-2, -999, -1000, -1001, -1_500_000_000_000], dtype=np.int64), size=int(neg.sum()))
    yield "random_big", t, 7
    for km in (0, 1, 2):
        spec = synth.make_spec(N, 64, key_mode=km, distinct_keys=3000, tombstone_per_10k=2000, null_key_per_10k=300,
                               ts_missing_per_10k=50, empty_value_per_10k=100)
        yield "synth_keys%d" % km, synth.fill_host(spec), 64
    t = random_topic(np.random.default_rng(5), N, 5)
    bad = np.random.default_rng(6).random(N) < 0.05
    t.partition[bad] = np.random.default_rng(7).choice(np.array([-1, -7, 5, 6, 1 << 30], dtype=np.int32), size=int(bad.sum()))
    yield "out_of_range", t, 5


TOPICS = list(_topics())


@pytest.mark.parametrize("name,t,P", TOPICS, ids=[n for n, _, _ in TOPICS])
def test_reference_equals_the_oracle(name, t, P):
    cols = {k: torch.from_numpy(np.ascontiguousarray(getattr(t, k))) for k in ("partition", "ts_ms", "key_len", "value_len")}
    kb = torch.from_numpy(t.key_bytes)
    h = R.fnv32(cols["key_len"], kb)
    assert np.array_equal(h.numpy().astype(np.uint32), np_oracle.fnv32_many(t.key_len, t.key_bytes))
    if name == "random_big":
        assert (t.value_len == (1 << 31) - 1).any() and (t.ts_ms == -1).any() and (t.ts_ms < -1).any()
        assert (t.key_len == 0).any() and (t.key_len < 0).any() and (t.value_len == 0).any() and (t.value_len < 0).any()
    # the oracle sees the in-range records only, in order (out-of-range records take part in nothing)
    good = (t.partition >= 0) & (t.partition < P)
    o = oracle_for(take(t, np.nonzero(good)[0]), count_alive_keys=True, track_stream=True, now=NOW)

    mm = R.message_metrics(P, cols["partition"], cols["ts_ms"], cols["key_len"], cols["value_len"])
    assert mm["bad"] == int((~good).sum())
    for name_ in COUNTERS:
        assert mm[name_].tolist() == [o.counter(name_, p) for p in range(P)], name_
    for p in range(P):
        assert mm["khist"][p].tolist() == o.hist(0, p).tolist() and mm["vhist"][p].tolist() == o.hist(1, p).tolist(), p
    for k in ("smallest", "largest", "overall_size", "overall_count"):
        assert mm[k] == o.scalar(k + "_message" if k in ("smallest", "largest") else k), k
    assert R.earliest(mm, NOW) == o.earliest() and R.latest(mm) == o.latest()

    stream = R.stream_mask(cols["partition"], cols["key_len"], cols["value_len"], P)
    good_t = torch.from_numpy(good)
    alive_h, distinct = R.alive_hashes(h, cols["key_len"], cols["value_len"], mask=good_t)
    assert alive_h.numel() == o.scalar("sum_all_alive")
    assert R.alive(h, cols["key_len"], cols["value_len"], mask=good_t) == (alive_h.numel(), distinct)
    assert distinct == len(set(h[good_t & (cols["key_len"] >= 0)].tolist()))
    for p in (4, 10, 18):
        assert np.array_equal(R.hll_regs(h, stream, p).numpy(), o.hll_stream_regs(p)), ("stream", p)
        assert np.array_equal(R.hll_regs(alive_h, None, p).numpy(), o.hll_alive_regs(p)), ("alive", p)


def test_mul32_and_clz_at_their_edges():
    """the 16-bit split product and the comparison clz, at the values where a wrap or a float log2 would go wrong"""
    a = torch.tensor([0, 1, 0xFFFF, 0x10000, 0x7FFFFFFF, 0x80000000, 0xFFFFFFFF, 0xDEADBEEF], dtype=torch.int64)
    for c in (R.FNV_MULT, 0x85EBCA6B, 0xC2B2AE35, 0xFFFFFFFF, 1):
        assert R._mul32(a, c).tolist() == [(int(x) * c) % (1 << 32) for x in a.tolist()]
    v = torch.tensor([0, 1, 2, 3, (1 << 31) - 1, 1 << 31, 0xFFFFFFFF, 1 << 20, (1 << 20) - 1], dtype=torch.int64)
    assert R.clz32(v).tolist() == [32 - int(x).bit_length() for x in v.tolist()]
    lens = torch.tensor([0, 1, 2, 3, 4, 255, 256, (1 << 24) - 1, 1 << 24, (1 << 31) - 1], dtype=torch.int64)
    assert R.bucket(lens).tolist() == [int(x).bit_length() for x in lens.tolist()]
