"""What the engine must report, and the comparisons that check it (TEST INFRASTRUCTURE)."""
import numpy as np

from kafka_topic_analyzer_b200 import metrics as M
from oracle_lib import COUNTERS, Oracle

NOW = (4102444800, 123456789)


def oracle_for(topic, count_alive_keys=False, track_stream=False, now=NOW, order=None):
    """Runs the CPU oracle over a HostTopic record by record, in seq order (src/kafka.rs:99)."""
    o = Oracle(count_alive_keys=count_alive_keys, track_stream=track_stream, now=now)
    o.handle_batch(topic.partition, topic.ts_ms, topic.key_len, topic.value_len, topic.key_bytes)
    return o


def oracle_over(per, count_alive_keys=False, track_stream=False, now=NOW):
    """The CPU oracle over partition lists (feed.partition_lists), partition by partition, as the log entry points
    deliver them; a timestamp of -1 is "not available"."""
    o = Oracle(count_alive_keys=count_alive_keys, track_stream=track_stream, now=now)
    for p in sorted(per):
        for ts, key, vl in per[p]:
            o.handle_message(p, None if ts == -1 else ts, key, vl)
    return o


def oracle_in_order(records, count_alive_keys=True, now=NOW):
    """The CPU oracle over (partition, ts, key, value_len) records in the order given, which must be the order the
    engine delivered them: the exact alive-key count of a hash that several partitions write depends on it."""
    o = Oracle(count_alive_keys=count_alive_keys, now=now)
    for p, ts, key, vl in records:
        o.handle_message(p, ts, key, vl)
    return o


def expected(mode, t, hll_p):
    """(oracle, assert_parity keywords) for a scan of t in mode counters, hll (the in-stream sketch) or exact (-c); t is
    a HostTopic or partition lists"""
    flags = {"counters": {}, "hll": dict(track_stream=True), "exact": dict(count_alive_keys=True)}[mode]
    o = oracle_over(t, **flags) if isinstance(t, dict) else oracle_for(t, **flags)
    if mode == "counters":
        return o, {}
    if mode == "hll":
        return o, dict(hll_regs=o.hll_stream_regs(hll_p))
    return o, dict(check_alive=True, hll_regs=o.hll_alive_regs(hll_p))


def assert_parity(engine, o, P, check_alive=False, hll_regs=None, extra_partitions=(-1,)):
    """Bit-exact comparison of everything the reference's report reads (src/main.rs:130-170)."""
    mm = engine.message_metrics
    for p in list(range(P)) + [P + 3] + list(extra_partitions):
        for i, name in enumerate(COUNTERS):
            assert engine.counter(i, p) == o.counter(name, p), (name, p)
        for name, which in (("key_size_avg", M.KEY_SIZE_AVG), ("value_size_avg", M.VALUE_SIZE_AVG),
                            ("message_size_avg", M.MESSAGE_SIZE_AVG)):
            try:
                want = o.avg(name, p)
            except ZeroDivisionError:
                want = "panic"
            try:
                got = engine.avg(which, p)
            except ZeroDivisionError:
                got = "panic"
            assert got == want, (name, p, got, want)
        assert mm.dirty_ratio(p) == o.dirty_ratio(p), ("dirty_ratio", p)   # f32, bit-exact
        if 0 <= p < P:
            assert engine.hist(0, p).tolist() == o.hist(0, p).tolist(), ("khist", p)
            assert engine.hist(1, p).tolist() == o.hist(1, p).tolist(), ("vhist", p)
    assert mm.smallest_message() == o.scalar("smallest_message")
    assert mm.largest_message() == o.scalar("largest_message")
    assert mm.overall_size() == o.scalar("overall_size")
    assert mm.overall_count() == o.scalar("overall_count")
    assert mm.earliest_message() == o.earliest()
    assert mm.latest_message() == o.latest()
    if check_alive:
        assert engine.alive_keys() == o.scalar("sum_all_alive")
    if hll_regs is not None:
        assert engine.hll_registers().tolist() == hll_regs.tolist()


# ------------------------------------------------------------------------------------------------
# the alive-key table, entry by entry
# ------------------------------------------------------------------------------------------------
def last_writer(h, seq, alive):
    """Sorted (hash u32, stamp u64) arrays: for every hash the largest stamp (seq + 1) << 1 | alive of its records."""
    stamp = ((seq + np.uint64(1)) << np.uint64(1)) | alive.astype(np.uint64)
    order = np.lexsort((stamp, h))
    h, stamp = h[order], stamp[order]
    last = np.ones(h.size, dtype=bool)
    last[:-1] = h[1:] != h[:-1]
    return h[last], stamp[last]


def exported(e):
    """the engine's table (kta_alive_export_device) as sorted (hash, stamp) arrays"""
    import torch
    from feed import settle
    n = e.alive_export_count()
    dh = torch.zeros(max(n, 1), dtype=torch.int32, device="cuda")
    ds = torch.zeros(max(n, 1), dtype=torch.int64, device="cuda")
    settle()
    assert e.alive_export(dh, ds, n) == n
    h = dh[:n].cpu().numpy().view(np.uint32)
    s = ds[:n].cpu().numpy().view(np.uint64)
    order = np.argsort(h, kind="stable")
    return h[order], s[order]


def assert_same_map(got, want):
    gh, gs = got
    wh, ws = want
    if np.array_equal(gh, wh) and np.array_equal(gs, ws):
        return
    only_got = np.setdiff1d(gh, wh)
    only_want = np.setdiff1d(wh, gh)
    common, gi, wi = np.intersect1d(gh, wh, return_indices=True)
    bad = np.nonzero(gs[gi] != ws[wi])[0]
    detail = [(hex(int(common[i])), int(gs[gi[i]]), int(ws[wi[i]])) for i in bad[:5]]
    raise AssertionError("alive table != last-writer map: %d entries exported, %d expected; %d only exported, %d missing, "
                         "%d with a different stamp, e.g. (hash, got, want) %s"
                         % (gh.size, wh.size, only_got.size, only_want.size, bad.size, detail))


# ------------------------------------------------------------------------------------------------
# the reference's one real output
# ------------------------------------------------------------------------------------------------
def replay_demo_row(row, demo, handler):
    """Re-creates one partition of the demo topic as records: 9-byte keys (K-Bytes / Total == 9 exactly),
    values spread so that V-Bytes matches, one smallest (139) and one largest (750) message."""
    n, vsum = row["total"], row["v_bytes"]
    vl = np.full(n, 0, dtype=np.int64)
    vl[0], vl[1] = demo["smallest_message"] - 9, demo["largest_message"] - 9
    rest = vsum - int(vl[0]) - int(vl[1])
    base, extra = divmod(rest, n - 2)
    vl[2:] = base
    vl[2:2 + extra] += 1
    assert int(vl.sum()) == vsum and vl.min() >= 130 and vl.max() <= 741
    ts = np.full(n, demo["earliest_message_s"] * 1000 + 500, dtype=np.int64)
    ts[n // 2] = demo["earliest_message_s"] * 1000 + 999      # still the same second (truncation)
    ts[-1] = demo["latest_message_s"] * 1000 + 1
    kl = np.full(n, 9, dtype=np.int32)
    part = np.full(n, row["P"], dtype=np.int32)
    handler(part, ts, kl, vl.astype(np.int32))
