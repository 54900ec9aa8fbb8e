"""Handle lifetime: kta_destroy releases every buffer a handle allocated, also when kta_create fails part way; and one
process can drive handles on two devices (the decoder's kernel attributes are set per device)."""
import os
import shutil
import subprocess
import sys

import numpy as np
import pytest

import kafka_codec as kc
from feed import NOW, partition_lists
from kafka_topic_analyzer_b200 import KtaEngine, lib, synth
from parity import assert_parity, oracle_over

HERE = os.path.dirname(os.path.abspath(__file__))


def _sanitizer():
    path = shutil.which("compute-sanitizer") or os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin", "compute-sanitizer")
    return path if os.path.exists(path) else None


@pytest.mark.gpu
def test_destroy_releases_everything_the_handle_allocated():
    driver = [sys.executable, os.path.join(HERE, "handle_lifetime_driver.py")]
    env = dict(os.environ, KTA_NO_BUILD="1")
    plain = subprocess.run(driver, capture_output=True, text=True, env=env, timeout=600)
    assert plain.returncode == 0, plain.stdout + plain.stderr
    san = _sanitizer()
    if san is None:
        pytest.skip("compute-sanitizer not found")
    memcheck = [san, "--tool", "memcheck", "--leak-check", "full", "--error-exitcode", "77"]
    probe = subprocess.run([*memcheck, sys.executable, "-c", "from kafka_topic_analyzer_b200 import KtaEngine; KtaEngine(1, device=0).close()"],
                           capture_output=True, text=True, env=dict(env, PYTHONPATH=os.path.dirname(HERE)), timeout=300)
    if probe.returncode != 0:   # the sanitizer cannot run CUDA work on this machine (the plain run above has passed)
        pytest.skip("compute-sanitizer cannot create a handle here: " + (probe.stdout + probe.stderr)[-300:])
    r = subprocess.run([*memcheck, *driver], capture_output=True, text=True, env=env, timeout=1800)
    out = r.stdout + r.stderr
    assert r.returncode == 0, out[-4000:]
    assert "round 1 ok" in out and "Leaked" not in out, out[-4000:]


def _longest_batch(seg):
    return int(np.diff(kc.batch_offsets(seg) + [seg.size]).max())


@pytest.mark.gpu
def test_log_decode_on_two_devices_in_one_process():
    if lib().kta_device_count() < 2:
        pytest.skip("needs two CUDA devices")
    P = 4
    spec = synth.make_spec(P * 1000, P, key_mode=2, distinct_keys=500, tombstone_per_10k=1000, value_mean=150)
    segs = [(p, synth.encode_segment(spec, p, batch_records=100)) for p in range(P)]
    # batches of about 16 KB are staged, and 4 warps' stages of >= 12 KiB need the opt-in shared memory
    assert 12 * 1024 <= max(_longest_batch(s) for _, s in segs) <= 40 * 1024
    o = oracle_over(partition_lists(synth.fill_host(spec)), count_alive_keys=True)
    for device in (0, 1):
        with KtaEngine(P, count_alive_keys=True, hll_precision=10, device=device, now=NOW) as e:
            assert e.push_log_segments(segs) == spec.n_total
            e.finalize()
            assert_parity(e, o, P, check_alive=True, hll_regs=o.hll_alive_regs(10))
