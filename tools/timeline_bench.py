"""Cost of the timeline pass (include/kta.h, kta_set_timeline) on the GPU.

Per shape, one synthetic batch is generated in HBM and scanned by kta_scan_batch_device on a counters-only handle,
alternating a handle without the timeline and one with it, `--reps` times each.  torch.profiler (CUDA activities) gives
each launch's kernel time: the pass is `timeline_kernel`, the scan `scan_kernel`.  Reported per shape: the medians, the
pass's rate as 20 B per record (partition, ts_ms, key_len, value_len) over its kernel time against the data sheet's
3.35 TB/s, the ratio to the scan's time on the same batch, and the end-to-end call time (CUDA events around the call) with
and without the pass.  The card's name and power limit are read in the same run.

    python tools/timeline_bench.py [--n 100000000] [--reps 9] [--out profiles/h100_timeline.log]
"""
import argparse
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402
from torch.profiler import ProfilerActivity, profile  # noqa: E402

from kafka_topic_analyzer_b200 import KtaEngine, synth  # noqa: E402

HBM = 3.35e12
T0 = 1_500_000_000   # the synthetic topic's first timestamp, in seconds (ts = 1.5e12 ms + 7 i + jitter)


def card():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as ex:   # the number is reported without it, and says so
        q = "unknown (%s)" % ex
    return name, q


def shapes(n):
    # (name, partitions, run_len, timeline (origin, width, buckets))
    span_h = n * 7 // 3_600_000 + 2
    return [
        ("C1 1-hour buckets (shared-memory bins)", 64, 1, (T0 - T0 % 3600, 3600, span_h)),
        ("C1 run_len=512, 1-hour buckets (fetch-shaped)", 64, 512, (T0 - T0 % 3600, 3600, span_h)),
        ("C1 1-minute buckets (global bins)", 64, 1, (T0 - T0 % 60, 60, n * 7 // 60_000 + 2)),
        ("C1 run_len=512, 1-minute buckets (global bins)", 64, 512, (T0 - T0 % 60, 60, n * 7 // 60_000 + 2)),
    ]


def run(n_req, reps):
    rows = []
    for name, P, run_len, (O, W, B) in shapes(n_req):
        n = n_req // (P * run_len) * (P * run_len)   # the generator deals whole runs to every partition
        spec = synth.make_spec(n, P, run_len=run_len, distinct_keys=10_000_000, value_mean=256, null_key_per_10k=100,
                               tombstone_per_10k=0)
        topic = synth.DeviceTopic(spec, device=0)
        cols = (topic.partition, topic.ts_ms, topic.key_len, topic.value_len)
        off, on = KtaEngine(P, device=0), KtaEngine(P, device=0)
        on.set_timeline(O, W, B)
        smem = on.timeline_shape(n)[2]

        def call(e):
            e.reset()
            e.scan_batch_device(*cols)
            e.sync()

        for e in (off, on, off, on):   # warm-up: module load, first launches
            call(e)
        wall = {"off": [], "on": []}
        for _ in range(reps):
            for tag, e in (("off", off), ("on", on)):
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                torch.cuda.synchronize()
                a.record()
                call(e)
                b.record()
                b.synchronize()
                wall[tag].append(a.elapsed_time(b))
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(reps):
                call(off)
                call(on)
        tl, sc = [], []
        for ev in prof.events():
            if ev.device_type.name != "CUDA":
                continue
            t = ev.device_time / 1000.0   # ms
            if "timeline_kernel" in ev.name:
                tl.append(t)
            elif "scan_kernel" in ev.name:
                sc.append(t)
        tl_ms, sc_ms = statistics.median(tl), statistics.median(sc)
        rows.append(dict(shape=name, n=n, partitions=P, run_len=run_len, origin=O, width=W, buckets=B, smem_bins=smem,
                         timeline_ms=tl_ms, scan_ms=sc_ms, ratio=tl_ms / sc_ms,
                         timeline_tb_s=20 * n / (tl_ms * 1e-3) / 1e12, share_of_hbm=20 * n / (tl_ms * 1e-3) / HBM,
                         call_off_ms=statistics.median(wall["off"]), call_on_ms=statistics.median(wall["on"]),
                         samples=(len(tl), len(sc))))
        # the pass counts every record, and its rows sum to the counters
        on.finalize()
        assert sum(int(on.timeline(0, p).sum()) for p in range(P)) == n
        off.close(); on.close()
        del topic
        torch.cuda.empty_cache()
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=100_000_000)
    ap.add_argument("--reps", type=int, default=9)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("timeline_bench needs a CUDA device")
    name, power = card()
    lines = ["card: %s; power.limit, clocks.max.sm: %s" % (name, power),
             "n = %d records per batch, medians of %d runs, timeline off and on alternated" % (a.n, a.reps)]
    for r in run(a.n, a.reps):
        lines.append("%-48s n=%d B=%-6d %s  pass %.3f ms  scan %.3f ms  pass/scan %.2f  pass %.2f TB/s = %.0f %% of 3.35 TB/s  "
                     "call off %.3f ms  on %.3f ms" % (r["shape"], r["n"], r["buckets"], "smem  " if r["smem_bins"] else "global",
                                                       r["timeline_ms"], r["scan_ms"], r["ratio"], r["timeline_tb_s"],
                                                       100 * r["share_of_hbm"], r["call_off_ms"], r["call_on_ms"]))
    text = "\n".join(lines) + "\n"
    sys.stdout.write(text)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(text)


if __name__ == "__main__":
    main()
