"""Cost of check.crcs (kta_logcrc.cuh) on the GPU RecordBatch v2 decoder.

Workloads: the synthetic topic stored broker-style with real CRCs (16 partitions, 8e6 records), staged to HBM once and
decoded + scanned from device memory with kta_scan_log_batches_device:
  16k:      ~16 KB batches (56 records each);
  240k:     ~240 KB batches (840 records each);
  16k-zstd: the 16 KB batches with their records sections recompressed with zstd (CRCs rewritten over the stored bytes).
Method: the switch off and on alternate inside every repetition (so drift of the shared host hits both alike); the median
and the range over the repetitions are printed.  A separate torch.profiler pass gives the device time of the CRC passes
(count, span, the CRC header pass) next to log_decode_kernel, which also reads every byte, and the CRC span pass's bytes/s
over the call's bytes as a share of the H100's 3.35 TB/s.  The card's name and power limit are printed first.
usage: python tools/logcrc_bench.py [reps]"""
import os
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
HBM = 3.35e12
REPS = int(sys.argv[1]) if len(sys.argv) > 1 else 9


def main():
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()
    print("card:", card, flush=True)
    spec = synth.make_spec(N, P, value_mean=VM, distinct_keys=1_000_000)
    work = {}
    small = [(p, synth.encode_segment(spec, p, batch_records=56)) for p in range(P)]
    work["16k"] = stage_batches(small)
    work["240k"] = stage_batches([(p, synth.encode_segment(spec, p, batch_records=840)) for p in range(P)])
    work["16k-zstd"] = stage_batches([(p, kc.set_crcs(kc.recompress(s, lambda: "zstd"))) for p, s in small])
    for w, s in work.items():
        print("workload %-8s %d records, %d batches, %.3f GB, %.1f KB per batch" % (w, N, s[4], s[1] / 1e9, s[1] / s[4] / 1e3), flush=True)
    modes = [(w, crc) for w in work for crc in (False, True)]
    engines = {m: kta.KtaEngine(P, check_crcs=m[1]) for m in modes}
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
            assert n == N and e.message_metrics.overall_count() == N, (m, n)
            if m[1]:
                assert e.log_crc_stats() == (work[m[0]][4], 0, 0), e.log_crc_stats()
            if rep:                                      # rep 0 warms every shape up
                times[m].append(dt * 1e3)
    for m in modes:
        t = np.array(times[m])
        print("%-8s check.crcs=%-5s decode+scan  median %.3f ms  min %.3f  max %.3f  (%d reps)" %
              (m[0], str(m[1]).lower(), np.median(t), t.min(), t.max(), len(t)), flush=True)
    for w in work:
        a, b = np.median(times[(w, False)]), np.median(times[(w, True)])
        print("%-8s on - off: %+.3f ms (%+.1f %%)" % (w, b - a, 100 * (b - a) / a))
    # device time per kernel (profiled run of its own)
    from torch.profiler import ProfilerActivity, profile
    for w in work:
        e = engines[(w, True)]
        e.reset()
        e.sync()
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(3):
                e.scan_log_batches_device(*work[w])
                e.sync()
            torch.cuda.synchronize()
        tot = {}
        for ev in prof.events():
            if ev.device_type != torch.autograd.DeviceType.CUDA:
                continue
            us = ev.device_time if hasattr(ev, "device_time") else ev.cuda_time
            tot[ev.name] = tot.get(ev.name, 0.0) + us / 3
        span = sum(v for k, v in tot.items() if "log_crc_span" in k)
        crc = sum(v for k, v in tot.items() if "log_crc_" in k or "log_header_kernel<true" in k)
        dec = sum(v for k, v in tot.items() if "log_decode_kernel" in k)
        all_us = sum(v for k, v in tot.items() if "Memcpy" not in k and "Memset" not in k)
        nbytes = work[w][1]
        print("%-8s device time per call: all kernels %.1f us, CRC passes %.1f us (span pass %.1f us: %.2f TB/s over the "
              "call's %.3f GB = %.0f %% of 3.35 TB/s), log_decode_kernel %.1f us" %
              (w, all_us, crc, span, nbytes / (span * 1e-6) / 1e12, nbytes / 1e9, 100 * nbytes / (span * 1e-6) / HBM, dec))
        for k, v in sorted(tot.items(), key=lambda kv: -kv[1])[:8]:
            print("    %8.1f us  %s" % (v, k[:110]))
    for e in engines.values():
        e.close()


if __name__ == "__main__":
    main()
