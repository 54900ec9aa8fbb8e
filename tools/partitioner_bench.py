"""Cost of the partitioner check's pass (include/kta.h, kta_set_partitioner_check) on the GPU.

Per shape, one synthetic batch is generated in HBM and scanned by kta_scan_batch_device on a counters-only handle,
alternating a handle without the check and one with it, `--reps` times each.  torch.profiler (CUDA activities) gives each
launch's kernel time: the pass is `partitioner_kernel`, the scan `scan_kernel`.  Reported per shape: the medians, the
pass's bytes (8 B per record for partition and key_len, plus the mean key length K) over its kernel time against the data
sheet's 3.35 TB/s, the ratio to the scan's time on the same batch, and the end-to-end call time (CUDA events around the
call) with and without the pass.  The card's name and power limit are read in the same run.

    python tools/partitioner_bench.py [--n 100000000] [--reps 9] [--out profiles/h100_partitioner.log]
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


def card():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as ex:   # the number is reported without it, and says so
        q = "unknown (%s)" % ex
    return name, q


def shapes():
    # (name, partitions, key_mode, counts): key modes as bench.py's --key-mode (0 = 16 B, 1 = ASCII key-<id>, 2 = 0..40 B)
    eight = [64, 32, 16, 12, 24, 48, 96, 128]
    return [
        ("C1 C=1 (16 B keys)", 64, 0, [64]),
        ("C1 C=8 (16 B keys)", 64, 0, eight),
        ("C1 C=1 ASCII keys", 64, 1, [64]),
        ("C1 C=1 ragged 0..40 B keys", 64, 2, [64]),
        ("C1 C=8 ragged 0..40 B keys", 64, 2, eight),
        ("6000 partitions C=8 (global counters)", 6000, 0, [6000] + eight[1:]),
    ]


def run(n_req, reps):
    rows = []
    for name, P, key_mode, counts in shapes():
        n = n_req // P * P
        spec = synth.make_spec(n, P, distinct_keys=10_000_000, value_mean=256, null_key_per_10k=100, tombstone_per_10k=0,
                               key_mode=key_mode)
        topic = synth.DeviceTopic(spec, device=0)
        kw = dict(key_bytes=topic.key_bytes, key_bytes_len=topic.key_bytes_len, key_tile_base=topic.key_tile_base)
        cols = (topic.partition, topic.ts_ms, topic.key_len, topic.value_len)
        off, on = KtaEngine(P, device=0), KtaEngine(P, device=0)
        on.set_partitioner_check(counts)
        grid, stage, smem = on.partitioner_shape(n, topic.key_bytes_len)

        def call(e):
            e.reset()
            e.scan_batch_device(*cols, **kw)
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
        pc, sc = [], []
        for ev in prof.events():
            if ev.device_type.name != "CUDA":
                continue
            t = ev.device_time / 1000.0   # ms
            if "partitioner_kernel" in ev.name:
                pc.append(t)
            elif "scan_kernel" in ev.name:
                sc.append(t)
        pc_ms, sc_ms = statistics.median(pc), statistics.median(sc)
        nbytes = 8 * n + topic.key_bytes_len
        rows.append(dict(shape=name, n=n, P=P, C=len(counts), kbar=topic.key_bytes_len / n, grid=grid, stage=stage, smem=smem,
                         pass_ms=pc_ms, scan_ms=sc_ms, ratio=pc_ms / sc_ms, tb_s=nbytes / (pc_ms * 1e-3) / 1e12,
                         share=nbytes / (pc_ms * 1e-3) / HBM, call_off_ms=statistics.median(wall["off"]),
                         call_on_ms=statistics.median(wall["on"]), samples=(len(pc), len(sc))))
        # every keyed record has a verdict: each partition's counters cover its keyed records
        on.finalize()
        keyed = sum(on.counter(4, p) for p in range(P))
        assert keyed > 0 and all(int(on.partitioner_check(p).max()) <= on.counter(4, p) for p in range(P))
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
        raise SystemExit("partitioner_bench needs a CUDA device")
    name, power = card()
    lines = ["card: %s; power.limit, clocks.max.sm: %s" % (name, power),
             "n = %d records per batch, medians of %d runs, check off and on alternated; library: %s" %
             (a.n, a.reps, os.environ.get("KTA_LIB") or "in-tree build")]
    for r in run(a.n, a.reps):
        lines.append("%-40s P=%-5d C=%d K=%.1f B  grid %d stage %d %s  pass %.3f ms  scan %.3f ms  pass/scan %.2f  "
                     "pass %.2f TB/s = %.0f %% of 3.35 TB/s  call off %.3f ms  on %.3f ms" %
                     (r["shape"], r["P"], r["C"], r["kbar"], r["grid"], r["stage"], "smem  " if r["smem"] else "global",
                      r["pass_ms"], r["scan_ms"], r["ratio"], r["tb_s"], 100 * r["share"], r["call_off_ms"], r["call_on_ms"]))
    text = "\n".join(lines) + "\n"
    sys.stdout.write(text)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(text)


if __name__ == "__main__":
    main()
