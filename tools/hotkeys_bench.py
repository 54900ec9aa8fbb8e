"""Cost of the hot-key pass (csrc/kta_hotkeys.cuh) on one GPU: prints the lines of profiles/h100_hotkeys.log.

For each configuration (1e8 records, 64 partitions, 1e7 distinct keys, 1 % null keys): C1 with uniform 16-byte keys, C1
with log-uniform keys, run_len = 512, and ASCII keys ("key-<id>"), three handles scan the same batch generated in HBM:
  off  counters only, table off;
  on   counters with the table on (warmed by one scan, so the table has its final size);
  -c   the exact alive-key scan, table off (the other hashing scan, for scale).
A step is kta_scan_batch_device + kta_sync, timed by the host clock around a device synchronisation; the handles are
alternated, medians of 9.  Then, in a run of its own under torch.profiler, the kernel times of one `on` step: the
counters scan and the hot-key pass.  The first scan of a fresh handle from the default 2^20 slots gives the growth a 1e8
batch takes (grows, slices, final slots); finalize of the C1 table times the compaction and sort of its 1e7 entries.
"""
import argparse
import statistics
import subprocess
import sys
import time
import os

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from kafka_topic_analyzer_b200 import KtaEngine, synth   # noqa: E402

HBM = 3.35e12
CONFIGS = [("C1 uniform 16 B", dict(key_mode=0)), ("C1 log-uniform 16 B", dict(key_mode=0, zipf_keys=True)),
           ("run_len 512", dict(key_mode=0, run_len=512)), ("ASCII key-<id>", dict(key_mode=1))]


def step(e, t):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    e.scan_batch_device(t.partition, t.ts_ms, t.key_len, t.value_len, key_bytes=t.key_bytes, key_bytes_len=t.key_bytes_len,
                        key_tile_base=t.key_tile_base)
    e.sync()
    return (time.perf_counter() - t0) * 1e3


def kernel_ms(e, t):
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        step(e, t)
    out = {}
    for ev in prof.key_averages():
        us = getattr(ev, "device_time_total", None)
        if us is None:
            us = getattr(ev, "cuda_time_total", 0)
        for tag in ("hot_keys_kernel", "scan_kernel", "DeviceRadixSort"):
            if tag in ev.key:
                out[tag] = out.get(tag, 0.0) + us / 1e3
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=100_000_000)
    ap.add_argument("--keys", type=int, default=10_000_000)
    ap.add_argument("--reps", type=int, default=9)
    ap.add_argument("--only", default=None, help="comma-separated indices of CONFIGS to run")
    a = ap.parse_args()
    print(subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip())
    P = 64
    for i, (name, kw) in enumerate(CONFIGS):
        if a.only is not None and str(i) not in a.only.split(","):
            continue
        group = P * kw.get("run_len", 1)
        n = a.n // group * group   # (a whole number of runs per partition)
        spec = synth.make_spec(n, P, distinct_keys=a.keys, **kw)
        t = synth.DeviceTopic(spec, device=0)
        kbar = t.key_bytes_len / n
        fresh = KtaEngine(P, now=(4102444800, 0))
        fresh.set_hot_keys(100)
        first = step(fresh, t)
        fresh.finalize()
        distinct, keyed, slots, grows, slices = fresh.hot_key_stats()
        print("%s (%d records): K=%.1f B/record, %d distinct ids; first scan from 2^20 slots: %.1f ms, %d grows, %d slices, %d slots (%.2f GB)"
              % (name, n, kbar, distinct, first, grows, slices, slots, slots * 96 / 1e9))
        if name.startswith("C1 uniform"):
            ms = []
            for _ in range(3):
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                fresh.finalize()
                ms.append((time.perf_counter() - t0) * 1e3)
            k = kernel_ms_finalize(fresh)
            print("  finalize of %d entries (export, sort, top 100 to the host): %s ms, median %.2f; radix sort kernels %.2f ms"
                  % (distinct, " ".join("%.2f" % m for m in ms), statistics.median(ms), k))
        on, off, exact = fresh, KtaEngine(P, now=(4102444800, 0)), KtaEngine(P, count_alive_keys=True, now=(4102444800, 0))
        for e in (off, exact):
            step(e, t)
        before = on.hot_key_stats()[3:]
        times = {"off": [], "on": [], "-c": []}
        for _ in range(a.reps):
            for tag, e in (("off", off), ("on", on), ("-c", exact)):
                times[tag].append(step(e, t))
        on.finalize()
        after = on.hot_key_stats()[3:]
        med = {k: statistics.median(v) for k, v in times.items()}
        print("  step ms, medians of %d alternated: off %.3f, on %.3f (pass +%.3f), -c %.3f; %d slices per step in steady state"
              % (a.reps, med["off"], med["on"], med["on"] - med["off"], med["-c"], (after[1] - before[1]) // a.reps))
        k = kernel_ms(on, t)
        hk, sc = k.get("hot_keys_kernel", 0.0), k.get("scan_kernel", 0.0)
        byts = n * (20 + kbar)
        print("  kernels of one step: counters scan %.3f ms, hot-key pass %.3f ms (%.0f%% of %.2f TB/s at 20 + K bytes per record;"
              " that bound is %.3f ms)" % (sc, hk, 100 * byts / (hk / 1e3) / HBM if hk else 0, HBM / 1e12, byts / HBM * 1e3))
        for e in (on, off, exact):
            e.close()
        del t
        torch.cuda.empty_cache()


def kernel_ms_finalize(e):
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        e.finalize()
    total = 0.0
    for ev in prof.key_averages():
        if "DeviceRadixSort" in ev.key:
            us = getattr(ev, "device_time_total", None)
            total += (us if us is not None else getattr(ev, "cuda_time_total", 0)) / 1e3
    return total


if __name__ == "__main__":
    main()
