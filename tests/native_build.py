"""Build recipe of the native test programs — TEST INFRASTRUCTURE.

  logdecomp_probe  tests/native/logdecomp_probe.cu: the product's decompression stage on the GPU, output made visible
                   (sm_90a, the library's nvcc flags without -shared / -fPIC)
  logdecode_probe  tests/native/logdecode_probe.cu: the product's record stage (decode, tile bases, key gather) on the GPU,
                   every decoded column made visible (built like logdecomp_probe)
  logtxn_probe     tests/native/logtxn_probe.cu: the product's read_committed passes (classify, sort, resolve, carry, apply) on
                   the GPU, every array they produce made visible (built like logdecomp_probe)
  logcrc_probe     tests/native/logcrc_probe.cu: the product's check.crcs passes (span counts, span pass, header verdict) on
                   the GPU, every array they produce made visible, and a plain host CRC-32C that needs no GPU (built like
                   logdecomp_probe)
  codec_harness    tests/native/codec_harness.cu: the same codec walks as plain host code, one "lane" (codec_harness.py runs it)
  push_loop        tests/native/push_loop.cu: a shared library (host code only) that calls kta_push record by record over
                   numpy columns (feed.push_records)

build() makes the plain programs in tests/native/build/ (git-ignored).  __graft_entry__.build() builds them, because the machine
that runs the GPU tests may have no nvcc; build() rebuilds one when it is older than the sources, and fails when it is missing
and cannot be built.  build_sanitized() makes the host tests' address-sanitizer build of the harness."""
import os
import shutil
import subprocess

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
CSRC = os.path.join(ROOT, "kafka_topic_analyzer_b200", "csrc")
NATIVE = os.path.join(HERE, "native")
OUT = os.path.join(NATIVE, "build")
PROGRAMS = ("logdecomp_probe", "logdecode_probe", "logtxn_probe", "logcrc_probe", "codec_harness", "push_loop")
LIBRARIES = ("push_loop",)
GPU_PROGRAMS = ("logdecomp_probe", "logdecode_probe", "logtxn_probe", "logcrc_probe")
SANITIZE = ["-g", "-Xcompiler", "-fsanitize=address,-fno-omit-frame-pointer"]


def nvcc():
    path = os.environ.get("NVCC") or "/usr/local/cuda/bin/nvcc"
    return path if os.path.exists(path) else shutil.which("nvcc")


def _command(nvcc, name, exe, flags=()):
    src = os.path.join(NATIVE, name + ".cu")
    if name in GPU_PROGRAMS:
        from kafka_topic_analyzer_b200 import _native
        lib_flags = " ".join(_native.NVCC_FLAGS).replace("-Xcompiler -fPIC", "").replace("-shared", "").split()
        return [nvcc, *lib_flags, "-o", exe, src]
    if name in LIBRARIES:
        return [nvcc, "-O2", "-std=c++17", "-shared", "-Xcompiler", "-fPIC", *flags, "-o", exe, src]
    return [nvcc, "-O1", "-std=c++17", *flags, "-o", exe, src]


def _stale(name, exe):
    if not os.path.exists(exe):
        return True
    srcs = [os.path.join(NATIVE, name + ".cu"), os.path.join(NATIVE, "probe.h")] + [os.path.join(CSRC, f) for f in os.listdir(CSRC) if os.path.isfile(os.path.join(CSRC, f))]
    return os.path.getmtime(exe) < max(os.path.getmtime(p) for p in srcs)


def build(name, force=False):
    exe = os.path.join(OUT, name)
    if not force and not _stale(name, exe):
        return exe
    cc = nvcc()
    if not cc:
        if os.path.exists(exe):
            return exe                   # older than the sources, but nothing here can rebuild it: used as it is
        raise RuntimeError("%s is missing and there is no nvcc to build it (run __graft_entry__.build())" % exe)
    os.makedirs(OUT, exist_ok=True)
    r = subprocess.run(_command(cc, name, exe), capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError("nvcc failed for %s:\n%s%s" % (name, r.stdout, r.stderr))
    return exe


def build_all(force=False):
    return [build(n, force) for n in PROGRAMS]


_sanitized = {}


def build_sanitized(name, out_dir):
    """`name` built into out_dir with the address sanitizer, so that a read or write outside a buffer ends the program with a
    report; plainly when this toolchain has no sanitizer runtime.  Built once per out_dir.  Returns (exe, which build it is)."""
    key = (name, out_dir)
    if key not in _sanitized:
        cc = nvcc()
        exe = os.path.join(out_dir, name + "_asan")
        r = subprocess.run(_command(cc, name, exe, SANITIZE), capture_output=True, text=True)
        how = "%s: address-sanitizer build" % name
        if r.returncode != 0:
            exe = os.path.join(out_dir, name)
            subprocess.run(_command(cc, name, exe), check=True, capture_output=True)
            how = "%s: plain build, no address sanitizer (%s)" % (name, (r.stderr.strip().splitlines() or ["nvcc failed"])[-1])
        _sanitized[key] = (exe, how)
    return _sanitized[key]
