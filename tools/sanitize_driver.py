"""Small end-to-end runs of every scan-kernel mode for compute-sanitizer (tools/sanitize.sh): counters, in-stream HLL,
exact alive keys (table starting far too small, so growth + stamps-only re-runs happen too), ragged keys, a tail tile,
the host ring path, the log-segment decoder, its read_committed passes and its offset windows.  Each run is checked against the oracle so a 'clean' sanitizer log is the
log of a run that also computed the right answer."""
import itertools, os, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))
import kafka_codec as kc
import offsets_codec as oc
import kafka_topic_analyzer_b200 as kta
from kafka_topic_analyzer_b200 import synth
from parity import assert_parity, oracle_for

NOW = (4102444800, 1)
which = sys.argv[1:] or ["counters", "hll", "exact", "ragged", "ring", "log", "logz", "logzstd", "logtxn", "logcrc", "logoffsets"]


def rotate(seg, codecs, first):
    """every batch of an uncompressed segment with its records section compressed by codecs[(first + i) % len(codecs)]
    for its index i (None: left uncompressed)"""
    pick = itertools.islice(itertools.cycle(codecs), first, None)
    return kc.recompress(seg, lambda: next(pick))


P = 8
n = P * 4096 + 0
for name in which:
    if name == "logtxn":   # read_committed: markers, aborted compressed batches, registered ranges, two calls
        import test_log_txn as lt
        t = lt.gen_topic(3, P=P, steps=200)
        cut = {p: len(t.batches[p]) // 2 for p in range(P)}
        calls = [[b for p in range(P) for b in t.batches[p][:cut[p]]], [b for p in range(P) for b in t.batches[p][cut[p]:]]]
        want, stats = lt.rule_model(calls, t.aborted)
        with kta.KtaEngine(P, count_alive_keys=True, device=0, now=NOW, alive_table_kib=1, isolation_level="read_committed") as e:
            for p in range(P):
                e.push_txn_index(p, kc.txn_index(t.aborted[p]))
            e.push_log_segments([(p, t.segment(p, 0, cut[p])) for p in range(P)])
            e.push_log_segments([(p, t.segment(p, cut[p])) for p in range(P)])
            e.finalize()
            assert e.log_txn_stats() == stats and e.message_metrics.overall_count() == len(want)
        print(name, "ok", stats)
        continue
    if name == "logcrc":   # check.crcs: batches of one to many spans at odd offsets, every third one damaged
        segs, bad, nb = [], 0, 0
        for p in range(P):
            s = bytearray(kc.set_crcs(rotate(synth.encode_segment(synth.make_spec(n, P), p, 0, n // P, batch_records=7 + 60 * p),
                                             ("gzip", "lz4", "snappy"), p)))
            for i, o in enumerate(kc.batch_offsets(s)):
                nb += 1
                if i % 3 == 0:
                    s[o + 40] ^= 1
                    bad += 1
            segs.append((p, bytes(s) + b"\x00" * (p % 3)))
        with kta.KtaEngine(P, count_alive_keys=True, device=0, now=NOW, check_crcs=True) as e:
            e.push_log_segments(segs)
            e.finalize()
            assert e.log_crc_stats()[:2] == (nb, bad), (e.log_crc_stats(), nb, bad)
        print(name, "ok", nb, bad)
        continue
    if name == "logoffsets":   # windows: cut compressed and plain batches, batches not served, check.crcs on, two calls
        segs, want, nb_out = [], 0, 0
        for p in range(P):
            s = kc.set_crcs(rotate(synth.encode_segment(synth.make_spec(n, P), p, 0, n // P, batch_records=7 + 60 * p),
                                   ("gzip", "zstd", None, "lz4"), p))
            lo, hi = 13 * p + 5, n // P - 40 * p - 3
            segs.append((p, s, lo, hi))
            want += len(oc.fetched(s, lo, hi))
            nb_out += oc.fetch_stats(s, lo, hi)[0]
        with kta.KtaEngine(P, count_alive_keys=True, device=0, now=NOW, check_crcs=True) as e:
            for p, _, lo, hi in segs:
                e.set_log_offsets(p, lo, hi)
            got = e.push_log_segments([(p, s) for p, s, _, _ in segs[:P // 2]])
            got += e.push_log_segments([(p, s) for p, s, _, _ in segs[P // 2:]])
            e.finalize()
            assert got == want == e.message_metrics.overall_count() and e.log_offset_stats()[0] == nb_out, (got, want)
        print(name, "ok", got, nb_out)
        continue
    key_mode = 2 if name in ("ragged", "ring") else 0
    spec = synth.make_spec(n, P, key_mode=key_mode, distinct_keys=3000, tombstone_per_10k=2500, ts_missing_per_10k=20,
                           run_len=64 if name == "counters" else 1)
    if name in ("log", "logz", "logzstd"):
        host = synth.fill_host(spec)
        o = oracle_for(host, count_alive_keys=True, now=NOW)
        with kta.KtaEngine(P, count_alive_keys=True, hll_precision=10, device=0, now=NOW, alive_table_kib=1) as e:
            per = n // P
            segs = [(p, synth.encode_segment(spec, p, 0, per, batch_records=100)) for p in range(P)]
            if name == "logz":   # gzip / LZ4 / Snappy batches: the decompressors run first
                segs = [(p, rotate(s, ("gzip", "lz4", "snappy"), p)) for p, s in segs]
            if name == "logzstd":   # zstd one-shot / streaming batches and uncompressed ones
                segs = [(p, rotate(s, ("zstd", "zstd-stream", None), p)) for p, s in segs]
            e.push_log_segments(segs)
            e.finalize()
            got = (e.message_metrics.overall_count(), e.alive_keys())
            assert e.alive_keys() == o.scalar("sum_all_alive")
        print(name, "ok", got)
        assert got[0] == n
        continue
    topic = synth.DeviceTopic(spec, device=0, count=n - 37)     # a ragged tail tile
    host = topic.to_host()
    exact = name in ("exact", "ragged", "ring")
    with kta.KtaEngine(P, count_alive_keys=exact, hll_precision=0 if name == "counters" else 10, device=0, now=NOW,
                       ring_records=4096, alive_table_kib=1 if exact else 0) as e:
        if name == "ring":
            e.push_batch_host(host.partition, host.ts_ms, host.key_len, host.value_len, host.key_bytes, None)
        else:
            e.scan_batch_device(topic.partition, topic.ts_ms, topic.key_len, topic.value_len, key_bytes=topic.key_bytes,
                                key_bytes_len=topic.key_bytes_len, key_tile_base=topic.key_tile_base)
        e.finalize()
        o = oracle_for(host, count_alive_keys=exact, track_stream=not exact, now=NOW)
        regs = None if name == "counters" else (o.hll_alive_regs(10) if exact else o.hll_stream_regs(10))
        assert_parity(e, o, P, check_alive=exact, hll_regs=regs)
        print(name, "ok", e.stats(), e.alive_table_stats() if exact else "")
