"""Exact alive keys (-c): kta_alive_import_device, the all-gather step of distributed.py, on its own.

Each case imports a (reference hash, (seq + 1) << 1 | alive) list with duplicate hashes and compares the exported table,
entry by entry, with the list's last-writer map: the import goes through the same growth, wide re-run and seq-window
handling as a scan."""
import numpy as np
import pytest

from feed import alive_import, engine, unmix32
from kafka_topic_analyzer_b200 import KtaError
from parity import assert_same_map, exported, last_writer


def stamped(rng, hashes, copies):
    """Every hash `copies` times on average (at least once), in random order, with distinct seqs and random alive bits."""
    h = np.concatenate([hashes, rng.choice(hashes, size=(copies - 1) * hashes.size)]).astype(np.uint32)
    h = h[rng.permutation(h.size)]
    seq = rng.permutation(h.size).astype(np.uint64) + np.uint64(100)
    return h, seq


def import_list(e, h, seq, alive):
    stamp = ((seq + np.uint64(1)) << np.uint64(1)) | alive.astype(np.uint64)
    alive_import(e, h.view(np.int32), stamp)


@pytest.mark.gpu
def test_import_grows_a_small_table():
    """About 6000 distinct hashes into a 128-slot table: the table grows and the list is applied again (no batch is
    re-stamped, so reruns stays 0)."""
    rng = np.random.default_rng(71)
    hashes = np.unique(rng.integers(0, 1 << 32, size=6100, dtype=np.uint64))[:6000]
    h, seq = stamped(rng, hashes, 3)
    alive = rng.random(h.size) < 0.6
    want = last_writer(h, seq, alive)
    with engine(alive_table_kib=1) as e:
        assert e.alive_table_stats()[0] == 128
        import_list(e, h, seq, alive)
        e.finalize()
        assert_same_map(exported(e), want)
        slots, occupied, grows, reruns = e.alive_table_stats()
        assert grows >= 1 and reruns == 0
        assert occupied == hashes.size and occupied * 10 <= slots * 6
        assert e.alive_keys() == int((want[1] & np.uint64(1)).sum())


@pytest.mark.gpu
@pytest.mark.parametrize("cluster", [200, 400])
def test_import_of_clustered_home_pairs_keeps_the_table(cluster):
    """`cluster` hashes with consecutive mixed values share a home pair and outlast the 96-pair probe limit: the import
    is applied again with the probe allowed over the whole table, which keeps its size."""
    rng = np.random.default_rng(cluster)
    x0 = int(rng.integers(0, (1 << 32) - 4096)) & ~0xFFF
    hashes = np.array([unmix32(x0 + i) for i in range(cluster)], dtype=np.uint32)
    h, seq = stamped(rng, hashes, 3)
    alive = rng.random(h.size) < 0.5
    want = last_writer(h, seq, alive)
    with engine(alive_table_kib=64) as e:
        slots0 = e.alive_table_stats()[0]
        import_list(e, h, seq, alive)
        e.finalize()
        assert_same_map(exported(e), want)
        slots, occupied, grows, reruns = e.alive_table_stats()
        assert (slots, grows, reruns) == (slots0, 0, 0)
        assert occupied == cluster


@pytest.mark.gpu
def test_import_outside_the_window():
    """Stamps whose seq lies past the table's 31-bit window are left out and reported by finalize; the in-window
    entries are imported exactly."""
    rng = np.random.default_rng(73)
    hashes = np.unique(rng.integers(0, 1 << 32, size=3100, dtype=np.uint64))[:3000]
    h, seq = stamped(rng, hashes, 3)
    out = np.zeros(h.size, dtype=bool)
    out[rng.choice(h.size, size=500, replace=False)] = True
    seq[out] = np.uint64((1 << 31) + 5) + np.arange(int(out.sum()), dtype=np.uint64)
    alive = rng.random(h.size) < 0.6
    want = last_writer(h[~out], seq[~out], alive[~out])
    with engine() as e:
        import_list(e, h, seq, alive)
        with pytest.raises(KtaError) as ei:
            e.finalize()
        assert ei.value.code == 1 and "window" in str(ei.value)
        assert_same_map(exported(e), want)
        assert e.alive_keys() == int((want[1] & np.uint64(1)).sum())
