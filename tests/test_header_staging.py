"""Header columns whose base is not 16-byte aligned cannot be staged by bulk copies: the scan then loads them from global
memory, like the tail tile of any batch.  The same seeded batch, scanned from aligned and from misaligned column
pointers in each mode, must match the CPU oracle both times."""
import numpy as np
import pytest

from feed import device, fixed_width_topic, scan, to_device
from kafka_topic_analyzer_b200 import KtaEngine, synth
from parity import assert_parity, expected

pytestmark = pytest.mark.gpu
NOW = (4102444800, 123456789)
P = 16


def scan_from(e, t, shift):
    """t's header columns from `shift` elements past a 16-byte-aligned base, its keys and tile bases as they are"""
    d = to_device(t)
    scan(e, d, cols=[device(c, shift) for c in (t.partition, t.ts_ms, t.key_len, t.value_len)])
    e.finalize()


@pytest.fixture(scope="module")
def topic():
    # a tail tile of 16 records, null keys, tombstones and missing timestamps
    spec = synth.make_spec(P * 4001, P, key_mode=2, distinct_keys=5000, tombstone_per_10k=1500,
                           null_key_per_10k=300, ts_missing_per_10k=20)
    return synth.fill_host(spec)


@pytest.mark.parametrize("shift", [0, 1])
@pytest.mark.parametrize("mode", ["counters", "hll", "alive"])
def test_scan_from_aligned_and_misaligned_columns(topic, mode, shift):
    o, kw = expected({"alive": "exact"}.get(mode, mode), topic, 12)
    with KtaEngine(P, count_alive_keys=mode == "alive", hll_precision=0 if mode == "counters" else 12, now=NOW) as e:
        scan_from(e, topic, shift)
        assert_parity(e, o, P, **kw)


@pytest.mark.parametrize("P,L", [(512, 16), (700, 16), (256, 36), (64, 64)])
def test_launch_shapes_for_many_partitions_and_long_keys(P, L):
    """Shapes away from the 12 warps x 3 stages of 16-byte keys on 64 partitions: the counter rows of 512 partitions leave
    room for key-only stages only, 700 partitions keep their counters in global memory, 36- and 64-byte keys need larger
    key stages (2 stages with headers, or keys only).  Both hashing modes, vs the oracle."""
    t = fixed_width_topic(np.random.default_rng(P * 100 + L), 40_000 + 37, P, L, 0.02, 3000)
    for mode in ("hll", "exact"):
        o, kw = expected(mode, t, 12)
        with KtaEngine(P, count_alive_keys=mode == "exact", hll_precision=12, now=NOW) as e:
            scan_from(e, t, 0)
            assert_parity(e, o, P, **kw)
