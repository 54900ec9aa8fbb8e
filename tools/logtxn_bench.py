"""Cost of read_committed isolation (kta_logtxn.cuh) on the GPU RecordBatch v2 decoder.

Workloads: the synthetic topic of tools/logdecode_bench.py stored broker-style (16 partitions, ~16 KB batches, 8e6
records), staged to HBM once and decoded + scanned from device memory with kta_scan_log_batches_device.
  plain: the batches as they are (no transactional batch): read_committed adds only the classify pass.
  txn:   every batch rewritten as transactional: 32 producers per partition take the batches in turn, 4 batches per
         transaction, then a COMMIT or ABORT marker (1 transaction in 10 aborted, chosen by a seeded generator).
Method: the modes alternate inside every repetition (so drift of the shared host hits them alike); the median and the
range over the repetitions are printed.  A separate torch.profiler pass gives the device time of the transaction passes
(classify, the CUB sort, resolve, carry, apply) next to the whole decode + scan.  The card's name and power limit are
printed first.
usage: python tools/logtxn_bench.py [reps] [out_dir]"""
import os
import struct
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]
import numpy as np
import torch

import kafka_codec as kc
import kafka_topic_analyzer_b200 as kta
from feed import stage_batches
from kafka_topic_analyzer_b200 import synth

P, N, VM, BR = 16, 8_000_000, 256, 56
PRODUCERS, TXN_BATCHES, ABORT = 32, 4, 0.1
REPS = int(sys.argv[1]) if len(sys.argv) > 1 else 9
OUT = sys.argv[2] if len(sys.argv) > 2 else None


# The marker and the producer patch of transactional() write other bytes than the test encoders (kafka_codec.marker,
# with_producer): the marker has baseTimestamp 0, baseSequence -1 and coordinatorEpoch 0, and the patch sets producerId
# only, leaving producerEpoch and baseSequence as the synthetic encoder wrote them.
def marker(offset, pid, commit):
    body = bytes([0]) + bytes([0, 0]) + bytes([8]) + struct.pack(">hh", 0, 1 if commit else 0) + bytes([12]) + struct.pack(">hi", 0, 0) + bytes([0])
    rec = bytes([len(body) * 2]) + body
    after = struct.pack(">iBIhiqqqhii", 0, 2, 0, 0x30, 0, 0, 0, pid, 0, -1, 1) + rec
    return struct.pack(">qi", offset, len(after)) + after


def transactional(batches, p, rng):
    """producer j = batch index mod PRODUCERS; its 4th batch of a transaction is followed by the marker"""
    out, seen, aborted = [], [0] * PRODUCERS, 0
    fate, in_txn = {}, [0] * PRODUCERS    # records of the producer's open transaction
    for i, b in enumerate(batches):
        j = i % PRODUCERS
        pid = 1000 * (p + 1) + j
        if seen[j] % TXN_BATCHES == 0:
            fate[j] = rng.random() >= ABORT
            in_txn[j] = 0
        in_txn[j] += int.from_bytes(b[57:61], "big")
        x = bytearray(b)
        x[21:23] = struct.pack(">h", struct.unpack(">h", b[21:23])[0] | 0x10)
        x[43:51] = struct.pack(">q", pid)
        out.append(bytes(x))
        seen[j] += 1
        if seen[j] % TXN_BATCHES == 0:
            base = int.from_bytes(b[:8], "big")
            out.append(marker(base + 1, pid, fate[j]))      # inside the batch's offset span: before the producer's next batch
            if not fate[j]:
                aborted += in_txn[j]
    return out, aborted


def main():
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()
    print("card:", card, flush=True)
    spec = synth.make_spec(N, P, value_mean=VM, distinct_keys=1_000_000)
    rng = np.random.default_rng(17)
    plain, txn, n_aborted = [], [], 0
    for p in range(P):
        bs = kc.split_batches(synth.encode_segment(spec, p, batch_records=BR))
        plain.append(bs)
        t, a = transactional(bs, p, rng)
        txn.append(t)
        n_aborted += a
    work = {w: stage_batches([(p, b"".join(bs)) for p, bs in enumerate(v)]) for w, v in (("plain", plain), ("txn", txn))}
    print("workloads: %d records, plain %d batches (%.2f GB), txn %d batches, %d records aborted" %
          (N, work["plain"][4], work["plain"][1] / 1e9, work["txn"][4], n_aborted), flush=True)
    modes = [(w, lvl, exact) for exact in (False, True) for w in ("plain", "txn") for lvl in ("read_uncommitted", "read_committed")]
    engines = {m: kta.KtaEngine(P, count_alive_keys=m[2], isolation_level=m[1]) for m in modes}
    times = {m: [] for m in modes}
    for rep in range(REPS + 1):
        for m in modes:
            e = engines[m]
            e.reset()
            e.sync()
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            n = e.scan_log_batches_device(*work[m[0]])
            e.finalize()
            dt = time.perf_counter() - t0
            want = N - (n_aborted if (m[0] == "txn" and m[1] == "read_committed") else 0)
            assert n == want and e.message_metrics.overall_count() == want, (m, n, want)
            if rep:                                      # rep 0 warms every shape up
                times[m].append(dt * 1e3)
    for m in modes:
        t = np.array(times[m])
        print("%-5s %-16s %-8s decode+scan  median %.3f ms  min %.3f  max %.3f  (%d reps)" %
              (m[0], m[1], "-c" if m[2] else "counters", np.median(t), t.min(), t.max(), len(t)), flush=True)
    for exact in (False, True):
        for w in ("plain", "txn"):
            a = np.median(times[(w, "read_uncommitted", exact)])
            b = np.median(times[(w, "read_committed", exact)])
            print("%-5s %-8s read_committed - read_uncommitted: %+.3f ms (%+.1f %%)" % (w, "-c" if exact else "counters", b - a, 100 * (b - a) / a))
    # device time per kernel (profiled run of its own)
    from torch.profiler import ProfilerActivity, profile
    for w in ("plain", "txn"):
        e = engines[(w, "read_committed", False)]
        e.reset()
        e.sync()
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(3):
                e.scan_log_batches_device(*work[w])
                e.sync()
            torch.cuda.synchronize()
        tot, passes = {}, {}
        for ev in prof.events():
            if ev.device_type != torch.autograd.DeviceType.CUDA:
                continue
            name = ev.name
            us = ev.device_time if hasattr(ev, "device_time") else ev.cuda_time
            tot[name] = tot.get(name, 0.0) + us
            if "txn_" in name or "RadixSort" in name or "Onesweep" in name:
                passes[name] = passes.get(name, 0.0) + us
        all_us = sum(v for k, v in tot.items() if "Memcpy" not in k and "Memset" not in k)
        print("%s, read_committed, counters: device time per call: all kernels %.1f us, transaction passes %.1f us" %
              (w, all_us / 3, sum(passes.values()) / 3))
        for k, v in sorted(passes.items(), key=lambda kv: -kv[1]):
            print("    %8.1f us  %s" % (v / 3, k[:110]))
        if OUT:
            os.makedirs(OUT, exist_ok=True)
            prof.export_chrome_trace(os.path.join(OUT, "logtxn_%s.trace.json" % w))
    for e in engines.values():
        e.close()


if __name__ == "__main__":
    main()
