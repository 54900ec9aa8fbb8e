"""Build recipe of the native test programs the GPU tests run — TEST INFRASTRUCTURE.

  logdecomp_probe  tests/native/logdecomp_probe.cu: the product's decompression stage on the GPU, output made visible
                   (sm_90a, the library's nvcc flags without -shared / -fPIC)
  zstd_harness     tests/native/zstd_harness.cu and lzwalk_harness.cu: the same walks as plain host code, one "lane"
  lzwalk_harness   (the host tests build their own address-sanitizer copies; these are the plain builds the GPU tests compare with)

The programs go to tests/native/build/ (git-ignored).  __graft_entry__.build() builds them, because the machine that runs the
GPU tests may have no nvcc; ensure() rebuilds one when it is older than the sources, and fails when it is missing and cannot be
built."""
import os
import shutil
import subprocess

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
CSRC = os.path.join(ROOT, "kafka_topic_analyzer_b200", "csrc")
NATIVE = os.path.join(HERE, "native")
OUT = os.path.join(NATIVE, "build")
PROGRAMS = ("logdecomp_probe", "zstd_harness", "lzwalk_harness")


def _nvcc():
    nvcc = os.environ.get("NVCC") or "/usr/local/cuda/bin/nvcc"
    return nvcc if os.path.exists(nvcc) else shutil.which("nvcc")


def _command(nvcc, name, exe):
    src = os.path.join(NATIVE, name + ".cu")
    if name == "logdecomp_probe":
        from kafka_topic_analyzer_b200 import _native
        flags = " ".join(_native.NVCC_FLAGS).replace("-Xcompiler -fPIC", "").replace("-shared", "").split()
        return [nvcc, *flags, "-o", exe, src]
    return [nvcc, "-O2", "-std=c++17", "-o", exe, src]


def _stale(name, exe):
    if not os.path.exists(exe):
        return True
    srcs = [os.path.join(NATIVE, name + ".cu")] + [os.path.join(CSRC, f) for f in os.listdir(CSRC) if os.path.isfile(os.path.join(CSRC, f))]
    return os.path.getmtime(exe) < max(os.path.getmtime(p) for p in srcs)


def build(name, force=False):
    exe = os.path.join(OUT, name)
    if not force and not _stale(name, exe):
        return exe
    nvcc = _nvcc()
    if not nvcc:
        if os.path.exists(exe):
            return exe                   # older than the sources, but nothing here can rebuild it: used as it is
        raise RuntimeError("%s is missing and there is no nvcc to build it (run __graft_entry__.build())" % exe)
    os.makedirs(OUT, exist_ok=True)
    r = subprocess.run(_command(nvcc, name, exe), capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError("nvcc failed for %s:\n%s%s" % (name, r.stdout, r.stderr))
    return exe


def build_all(force=False):
    return [build(n, force) for n in PROGRAMS]
