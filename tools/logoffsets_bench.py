"""Cost of offset windows (kta_log_set_offsets, kta_logoffsets.cuh) on the GPU RecordBatch v2 decoder.

Workloads: the synthetic topic stored broker-style (16 partitions, 8e6 records), staged to HBM once and decoded + scanned
(counters) + finalized from device memory with kta_scan_log_batches_device:
  16k:   ~16 KB batches (56 records each);
  240k:  ~240 KB batches (840 records each).
Arms, per workload:
  none:      no window (what every handle without one runs);
  boundary:  every partition a window whose start and watermark fall on batch boundaries (no batch is cut);
  cut:       every partition's start one record into a batch (one cut batch per partition: the count pass, its host round
             trip and the windowed decode);
  half:      windows that leave out half of each partition's batches (a quarter below the start, a quarter at and above
             the watermark).
Method: the arms alternate inside every repetition; the median and range over the repetitions are printed, with the
records each arm delivers checked against the batch headers.  The card's name and power limit are printed first.
usage: python tools/logoffsets_bench.py [reps]"""
import os
import struct
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import numpy as np
import torch

import kafka_codec as kc
import kafka_topic_analyzer_b200 as kta
from feed import stage_batches
from kafka_topic_analyzer_b200 import synth

P, N, VM = 16, 8_000_000, 256
REPS = int(sys.argv[1]) if len(sys.argv) > 1 else 9
ARMS = ("none", "boundary", "cut", "half")


def headers(seg):
    """(baseOffset, last, recordsCount) of every batch"""
    out = []
    for o in kc.batch_offsets(seg):
        base, = struct.unpack(">q", seg[o:o + 8])
        delta, = struct.unpack(">i", seg[o + 23:o + 27])
        count, = struct.unpack(">i", seg[o + 57:o + 61])
        out.append((base, base + delta, count))
    return out


def window(arm, hdr):
    nb = len(hdr)
    if arm == "boundary":
        return hdr[1][0], hdr[nb - 1][0]                 # the first and the last batch left out whole
    if arm == "cut":
        return hdr[nb // 2][0] + 1, None                 # one record into the middle batch
    if arm == "half":
        return hdr[nb // 4][0], hdr[nb - nb // 4][0]
    return None


def expected(win, hdr):
    """records served under win, from the headers (the synthetic batches have consecutive offsets)"""
    if win is None:
        return sum(c for _, _, c in hdr)
    lo, hi = win
    n = 0
    for base, last, count in hdr:
        if last < lo or (hi is not None and last >= hi):
            continue
        n += count - max(0, lo - base)
    return n


def main():
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()
    print("card:", card, flush=True)
    spec = synth.make_spec(N, P, value_mean=VM, distinct_keys=1_000_000)
    work, hdrs = {}, {}
    for w, per in (("16k", 56), ("240k", 840)):
        segs = [(p, bytes(synth.encode_segment(spec, p, batch_records=per))) for p in range(P)]
        work[w] = stage_batches(segs)
        hdrs[w] = {p: headers(s) for p, s in segs}
        s = work[w]
        print("workload %-5s %d records, %d batches, %.3f GB, %.1f KB per batch" % (w, N, s[4], s[1] / 1e9, s[1] / s[4] / 1e3), flush=True)
    modes = [(w, a) for w in work for a in ARMS]
    engines, want = {}, {}
    for m in modes:
        e = kta.KtaEngine(P)
        wins = {p: window(m[1], hdrs[m[0]][p]) for p in range(P)}
        for p, wn in wins.items():
            if wn is not None:
                e.set_log_offsets(p, *wn)
        engines[m] = e
        want[m] = sum(expected(wins[p], hdrs[m[0]][p]) for p in range(P))
    times = {m: [] for m in modes}
    for rep in range(REPS + 1):
        for m in modes:
            e = engines[m]
            e.sync()
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            n = e.scan_log_batches_device(*work[m[0]])
            e.finalize()
            dt = time.perf_counter() - t0
            assert n == want[m] and e.message_metrics.overall_count() == want[m] * (rep + 1), (m, n, want[m])
            if rep:                                      # rep 0 warms every shape up
                times[m].append(dt * 1e3)
    for m in modes:
        t = np.array(times[m])
        print("%-5s %-8s %8d records  decode+scan+finalize  median %.3f ms  min %.3f  max %.3f  (%d reps)" %
              (m[0], m[1], want[m], np.median(t), t.min(), t.max(), len(t)), flush=True)
    for w in work:
        a = np.median(times[(w, "none")])
        for arm in ARMS[1:]:
            b = np.median(times[(w, arm)])
            print("%-5s %-8s - none: %+.3f ms (%+.1f %%)" % (w, arm, b - a, 100 * (b - a) / a))
    for e in engines.values():
        e.close()


if __name__ == "__main__":
    main()
