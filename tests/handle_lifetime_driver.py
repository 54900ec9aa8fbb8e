"""Takes handles through every path that allocates device or pinned memory, destroys them, and does all of it twice.
tests/test_handle_lifetime.py runs it under compute-sanitizer's leak check.  It uses ctypes and numpy only (no torch), so
every device allocation in the process is either the library's or one made here through libcudart and freed here."""
import ctypes as C
import glob
import itertools
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]
import numpy as np  # noqa: E402

from kafka_topic_analyzer_b200 import KtaEngine, KtaError, synth  # noqa: E402
import kafka_codec as kc  # noqa: E402
import test_log_txn as lt  # noqa: E402

NOW = (4102444800, 1)
P = 8


def _cudart():
    home = os.environ.get("CUDA_HOME", "/usr/local/cuda")
    names = [os.path.join(home, "lib64", "libcudart.so.12"), "libcudart.so.12", "libcudart.so"]
    names += sorted(glob.glob(os.path.join(os.path.dirname(np.__file__), "..", "nvidia", "cuda_runtime", "lib", "libcudart.so*")))
    for name in names:
        try:
            return C.CDLL(name)
        except OSError:
            pass
    raise OSError("libcudart not found")


rt = _cudart()
rt.cudaMalloc.argtypes = [C.POINTER(C.c_void_p), C.c_size_t]
rt.cudaMemcpy.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_int]
rt.cudaFree.argtypes = [C.c_void_p]


class Dev:
    """device buffers of this driver (cudaMemcpyHostToDevice = 1, DeviceToHost = 2), freed on exit from the block"""

    def __init__(self):
        self.ptrs = []

    def alloc(self, nbytes):
        p = C.c_void_p()
        assert rt.cudaMalloc(C.byref(p), max(int(nbytes), 1)) == 0
        self.ptrs.append(p.value)
        return p.value

    def put(self, a):
        p = self.alloc(a.nbytes)
        assert rt.cudaMemcpy(p, a.ctypes.data, a.nbytes, 1) == 0
        return p

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        for p in self.ptrs:
            assert rt.cudaFree(p) == 0


def refused(fn, *args):
    try:
        fn(*args)
    except KtaError:
        return
    raise AssertionError("the call was not refused")


def one_round():
    spec = synth.make_spec(P * 2048, P, key_mode=2, distinct_keys=1500, tombstone_per_10k=2000)
    host = synth.fill_host(spec)
    n = host.n
    codec = itertools.cycle(["gzip", "zstd", None])
    segs = [(p, kc.recompress(synth.encode_segment(spec, p, 0, 256, batch_records=50).tobytes(), lambda: next(codec)))
            for p in range(P)]
    with Dev() as dev, KtaEngine(P, count_alive_keys=True, hll_precision=10, device=0, now=NOW, ring_records=1024,
                                 alive_table_kib=1) as e:   # a 1 KiB alive-key table: it grows
        kb = 0
        for i in range(3000):   # kta_push across ring chunks
            kl = int(host.key_len[i])
            key = None if kl < 0 else host.key_bytes[kb:kb + kl].tobytes()
            kb += max(kl, 0)
            e.push(int(host.partition[i]), i, int(host.ts_ms[i]), key, int(host.value_len[i]))
        e.push_batch_host(host.partition, host.ts_ms, host.key_len, host.value_len, host.key_bytes)
        e.scan_batch_device(dev.put(host.partition), dev.put(host.ts_ms), dev.put(host.key_len), dev.put(host.value_len),
                            key_bytes=dev.put(host.key_bytes), key_bytes_len=int(host.key_bytes.size), n=n)   # tile bases derived
        assert e.push_log_segments(segs) == P * 256   # compressed batches, gzip and zstd
        bad = bytearray(segs[0][1])
        bad[16] = 1   # magic 1: a refused call, after the header pass has run
        refused(e.push_log_segment, 0, bytes(bad))
        assert len(e.fnv32([b"a", None, b"hello"])) == 3
        e.finalize()
        assert e.message_metrics.overall_count() == 3000 + 2 * n + P * 256
        cnt = e.alive_export_count()
        dh, ds = dev.alloc(4 * cnt), dev.alloc(8 * cnt)
        assert e.alive_export(dh, ds, cnt) == cnt
        with KtaEngine(P, count_alive_keys=True, device=0, now=NOW, alive_table_kib=1) as e2:
            e2.alive_import(dh, ds, cnt)
            e2.finalize()
            assert e2.alive_keys() == e.alive_keys()
        assert e.alive_table_stats()[2] > 0   # grown
    t = lt.gen_topic(3, P=P, steps=80)
    with KtaEngine(P, count_alive_keys=True, device=0, now=NOW, alive_table_kib=1, isolation_level="read_committed") as e:
        for p in range(P):
            e.push_txn_index(p, kc.txn_index(t.aborted[p]))
        e.push_log_segments([(p, t.segment(p)) for p in range(P)])
        e.finalize()
        assert e.log_txn_stats() == lt.rule_model([[b for p in range(P) for b in t.batches[p]]], t.aborted)[1]
    # shard_rank 5 of 2 is refused after the state buffers exist
    refused(lambda: KtaEngine(P, count_alive_keys=True, hll_precision=10, device=0, shard=(5, 2), isolation_level="read_committed"))


for r in range(2):
    one_round()
    print("round", r, "ok")
assert rt.cudaDeviceReset() == 0   # the leak check reports what is still allocated when the context goes
