"""TEST INFRASTRUCTURE: runs tests/native/log_probe.cu, the log entry points' steps (kta_logscan.cuh) in the library's order with
everything they produce made visible.

  inputs(data, ...)  one case: the bytes and what the probe applies before the steps (see `inputs`)
  run(cases)         one probe run over the cases → per case a Result: `rc` and `msg` (the step that stopped the case, 0 and
                     "" when none did) and every array the probe wrote, by name (kta_logscan.cuh / log_probe.cu say which
                     step writes which); an array of a step that did not run is absent (Result.get gives None)
  device()           (SM count, opt-in shared memory per block) of the GPU the probe runs on
  crc32c(regions)    the probe's plain host CRC-32C of every region (no GPU)

stdin is fed from a thread: a case may carry gigabytes."""
import struct
import subprocess
import threading
from types import SimpleNamespace

import numpy as np

import native_build

KTA_ERR_INVALID = 1
LOGB_OK = 0
# the structs the probe writes, as the library lays them out
DTYPES = {
    "LogBatchInfo": np.dtype([("off", "<u8"), ("len", "<u4"), ("flags", "<u4"), ("partition", "<i4"), ("records", "<i4"),
                              ("base_offset", "<i8"), ("base_ts", "<i8"), ("max_ts", "<i8"), ("log_append_time", "<u4"),
                              ("pad", "<u4")]),
    "LogCrcFail": np.dtype([("batch", "<u4"), ("bytes", "<u4"), ("base", "<i8"), ("part", "<i4"), ("stored", "<u4"),
                            ("computed", "<u4"), ("pad", "<u4")]),
    "TxnKey": np.dtype([("pid", "<u8"), ("part", "<u4"), ("batch", "<u4")]),
    "TxnRange": np.dtype([("part", "<i4"), ("pad", "<u4"), ("pid", "<u8"), ("first", "<i8"), ("last", "<i8")]),
}


class Result(SimpleNamespace):
    def get(self, name, default=None):
        return getattr(self, name, default)


def inputs(data, offs=None, parts=None, slack=0, win=(), read_committed=False, ranges=None, check_crcs=False, span_grid=0,
           decompress=False):
    """data: the bytes (bytes or uint8 array), in a buffer of exactly len(data) + slack bytes; offs: the batch offsets, or None
    for the host walk of kta_push_log_segments_host; parts: per-batch partitions, or None (all 0); win: [(S, H)] of partitions
    [0, len(win)); ranges: aborted ranges (a TxnRange array, in any order: the probe registers them as the handle does);
    span_grid: the span pass's blocks (0: the library's rule); decompress: run the size and copy steps even where the
    library stops before or between them"""
    return SimpleNamespace(data=data, offs=offs, parts=parts, slack=slack, win=win, read_committed=read_committed, ranges=ranges,
                           check_crcs=check_crcs, span_grid=span_grid, decompress=decompress)


def _pieces(c):
    data = np.frombuffer(c.data, np.uint8) if isinstance(c.data, (bytes, bytearray)) else np.ascontiguousarray(c.data, np.uint8)
    yield struct.pack("<Q", data.size)
    yield data
    yield struct.pack("<I", c.slack)
    if c.offs is None:
        yield struct.pack("<q", -1)
    else:
        offs = np.ascontiguousarray(c.offs, "<u8")
        yield struct.pack("<q", offs.size)
        yield offs
    if c.parts is None:
        yield struct.pack("<I", 0)
    else:
        yield struct.pack("<I", 1)
        yield np.ascontiguousarray(c.parts, "<i4")
    win = np.ascontiguousarray(np.asarray(c.win, "<i8").reshape(-1, 2))
    yield struct.pack("<I", len(win))
    yield win
    ranges = np.zeros(0, DTYPES["TxnRange"]) if c.ranges is None else np.ascontiguousarray(c.ranges, DTYPES["TxnRange"])
    yield struct.pack("<II", int(c.read_committed), ranges.size)
    yield ranges
    yield struct.pack("<III", int(c.check_crcs), c.span_grid, int(c.decompress))


def _blocks(out):
    at = 0

    def take(fmt):
        nonlocal at
        v = struct.unpack_from(fmt, out, at)
        at += struct.calcsize(fmt)
        return v

    def text(n):
        nonlocal at
        s = out[at:at + n].decode()
        at += n
        return s
    while at < len(out):
        r = Result()
        while True:
            name = text(take("<I")[0])
            if not name:
                break
            dname = text(take("<I")[0])
            dtype = DTYPES.get(dname) or np.dtype("<" + dname)
            count, nbytes = take("<QQ")
            assert count * dtype.itemsize == nbytes, (name, dtype, count, nbytes)
            setattr(r, name, np.frombuffer(out, dtype, count, at))
            at += nbytes
        r.rc, = take("<i")
        r.msg = text(take("<I")[0])
        yield r


def run(cases):
    """one probe run over the cases → [Result per case]"""
    p = subprocess.Popen([native_build.build("log_probe")], stdin=subprocess.PIPE, stdout=subprocess.PIPE, stderr=subprocess.PIPE)

    def feed():
        try:
            for c in cases:
                for x in _pieces(c):
                    p.stdin.write(memoryview(x) if isinstance(x, np.ndarray) else x)
            p.stdin.close()
        except BrokenPipeError:
            pass
    t = threading.Thread(target=feed)
    t.start()
    out = p.stdout.read()
    t.join()
    err = p.stderr.read()
    assert p.wait() == 0, err.decode("utf-8", "replace")[-3000:]
    res = list(_blocks(out))
    assert len(res) == len(cases) + 1
    return res[1:]


_device = []


def device():
    """(SM count, opt-in shared memory per block)"""
    if not _device:
        out = subprocess.run([native_build.build("log_probe")], input=b"", capture_output=True, check=True).stdout
        d = next(_blocks(out))
        _device.append((int(d.sm_count[0]), int(d.smem_optin[0])))
    return _device[0]


def crc32c(regions):
    """the probe's plain host CRC-32C (no CUDA) of every region (uint8 arrays)"""
    p = subprocess.Popen([native_build.build("log_probe"), "crc32c"], stdin=subprocess.PIPE, stdout=subprocess.PIPE)

    def feed():
        for r in regions:
            p.stdin.write(struct.pack("<Q", len(r)))
            p.stdin.write(memoryview(np.ascontiguousarray(r, np.uint8)))
        p.stdin.close()
    t = threading.Thread(target=feed)
    t.start()
    out = p.stdout.read()
    t.join()
    assert p.wait() == 0
    return np.frombuffer(out, "<u4").astype(np.uint32)
