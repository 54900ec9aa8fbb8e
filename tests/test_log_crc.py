"""check.crcs for the log entry points (include/kta.h, kta_logcrc.cuh): every record batch's CRC-32C is computed on the
GPU, and a batch whose stored CRC does not match is skipped unread and listed, as librdkafka with check.crcs=true reports
it as a consumer error and goes on with the next batch.

Each GPU case compares the engine with the oracle fed exactly the records of the batches that passed."""
import os
import re
import struct
import subprocess
from dataclasses import dataclass, field

import numpy as np
import pytest

import kafka_codec as kc
from feed import LOG_ENTRIES, interleaved, scan_log, scan_log_batches, scan_log_segment, stage_batches
from kafka_topic_analyzer_b200 import KtaEngine, KtaError, _native, lib, synth
from parity import assert_parity, oracle_in_order

NOW = (4102444800, 123456789)
TS0 = 1_700_000_000_000
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
# the span size of the device pass (every span but a batch's first is this long): the region lengths below straddle it
SPAN = int(re.search(r"LOG_CRC_SPAN = (\d+)", open(os.path.join(ROOT, "kafka_topic_analyzer_b200", "csrc", "kta_logcrc.cuh")).read()).group(1))
CODECS = (None, "gzip", "snappy", "snappy-xerial", "lz4", "zstd", "zstd-stream")


# ---- batches whose delivered records are known ------------------------------------------------------------------------
@dataclass
class B:
    p: int
    raw: bytes
    recs: list = field(default_factory=list)   # (ts, key, value_len) as delivered
    bad: bool = False                          # its CRC fails

    @property
    def crc(self):
        return struct.unpack(">I", self.raw[17:21])[0]

    @property
    def base_offset(self):
        return struct.unpack(">q", self.raw[:8])[0]


def batch(p, off, recs, codec=None, values=None):
    """recs [(ts, key, value_len)] as one batch at baseOffset `off` with its real CRC; values: explicit value bytes"""
    base = recs[0][0] if recs else TS0 + off
    rows = [(j, ts - base, k, vl, (), None if values is None else values[j]) for j, (ts, k, vl) in enumerate(recs)]
    return B(p, kc.set_crcs(kc.encode_batch(off, base, rows, compression=codec)), list(recs))


def random_recs(rng, n, off, keys=30):
    out = []
    for j in range(n):
        k = None if rng.random() < 0.05 else b"key-%d" % int(rng.integers(0, keys))
        vl = None if rng.random() < 0.15 else int(rng.integers(0, 200))
        out.append((TS0 + 10 * (off + j) + int(rng.integers(0, 7)), k, vl))
    return out


def gen(seed, P=4, nb=60, codecs=CODECS):
    """P partitions of nb batches each, every batch with its own codec"""
    rng = np.random.default_rng(seed)
    parts = {}
    for p in range(P):
        out, off = [], 0
        for _ in range(nb):
            n = int(rng.integers(1, 30))
            out.append(batch(p, off, random_recs(rng, n, off), codecs[int(rng.integers(0, len(codecs)))]))
            off += n
        parts[p] = out
    return parts


def damage(b: B, at=17, bit=0):
    """flip one bit of the batch (by default in its stored CRC); bytes 17 and up are all covered by the check"""
    raw = bytearray(b.raw)
    raw[at] ^= 1 << bit
    b.raw, b.bad = bytes(raw), True
    return b


def flip_crc(b: B):
    raw = bytearray(b.raw)
    raw[17:21] = bytes(x ^ 0xFF for x in raw[17:21])
    b.raw, b.bad = bytes(raw), True
    return b


def seg(batches):
    return b"".join(b.raw for b in batches)


def passed(batches):
    """the (partition, ts, key, value_len) records of the batches that pass, in order"""
    return [(b.p, *r) for b in batches if not b.bad for r in b.recs]


def failure(b: B, computed):
    return (b.p, len(b.raw), b.base_offset, b.crc, computed)


def engine(P, **kw):
    return KtaEngine(P, count_alive_keys=True, hll_precision=10, now=NOW, check_crcs=True, **kw)


# ---- CPU ------------------------------------------------------------------------------------------------------------
def test_crc32c_known_answers():
    assert kc.crc32c(b"123456789") == 0xE3069283
    assert kc.crc32c(bytes(32)) == 0x8A9136AA                        # RFC 3720 B.4
    assert kc.crc32c(b"\xff" * 32) == 0x62A8AB43
    assert kc.crc32c(bytes(range(32))) == 0x46DD794E
    assert kc.crc32c(bytes(range(31, -1, -1))) == 0x113FDB5C


@pytest.mark.parametrize("key_mode,batch_records", [(0, 100), (1, 333), (2, 1000)])
def test_synth_encoder_writes_real_crcs(key_mode, batch_records):
    spec = synth.make_spec(8000, 4, key_mode=key_mode, value_mean=64)
    for p in (0, 3):
        s = bytes(synth.encode_segment(spec, p, batch_records=batch_records))
        offs = kc.batch_offsets(s)
        assert len(offs) == -(-2000 // batch_records)
        for o in offs:
            assert struct.unpack(">I", s[o + 17:o + 21])[0] == kc.batch_crc(s, o)
        assert kc.set_crcs(s) == s


def test_set_crcs_round_trip():
    rng = np.random.default_rng(3)
    recs = [(TS0 + i, b"k%d" % (i % 7), int(rng.integers(0, 90))) for i in range(300)]
    s = kc.encode_partition(recs, rng, max_batch=40)                  # CRC fields 0
    offs = kc.batch_offsets(s)
    assert all(s[o + 17:o + 21] == bytes(4) for o in offs)
    t = kc.set_crcs(s)
    assert len(t) == len(s) and kc.batch_offsets(t) == offs
    for o in offs:
        assert t[o:o + 17] == s[o:o + 17] and t[o + 21:o + 61] == s[o + 21:o + 61]
        assert struct.unpack(">I", t[o + 17:o + 21])[0] == kc.crc32c(t[o + 21:o + 12 + struct.unpack(">i", t[o + 8:o + 12])[0]])
    assert kc.set_crcs(t) == t
    u = bytearray(t)
    u[offs[1] + 17:offs[1] + 21] = b"\xde\xad\xbe\xef"
    assert kc.set_crcs(bytes(u)) == t


def test_cli_rejects_a_bad_check_crcs_value(tmp_path):
    from test_report import CLI_DIR, _build
    _build()
    cli = os.path.join(CLI_DIR, "kafka-topic-analyzer")
    r = subprocess.run([cli, "-t", "orders", "-b", "x", "--log-dir", str(tmp_path), "--librdkafka", "check.crcs=maybe"],
                       capture_output=True, text=True)
    assert r.returncode == 2 and "check.crcs" in r.stderr


# ---- GPU ------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("entry", LOG_ENTRIES)
def test_valid_crcs_deliver_everything(entry):
    parts = gen(11)
    nb = sum(len(v) for v in parts.values())
    with engine(4) as e:
        n, order = scan_log(e, entry, parts)
        e.finalize()
        o = oracle_in_order(passed(order))
        assert n == len(passed(order))
        assert_parity(e, o, 4, check_alive=True, hll_regs=o.hll_alive_regs(10))
        assert e.log_crc_stats() == (nb, 0, 0) and e.log_crc_failures() == []


@pytest.mark.gpu
@pytest.mark.parametrize("entry", ["segments_host", "batches_device"])
def test_every_crc_flipped_delivers_nothing(entry):
    parts = gen(12, nb=40)
    ref = {id(b): b.crc for v in parts.values() for b in v}
    for v in parts.values():
        for b in v:
            flip_crc(b)
    with engine(4) as e:
        n, order = scan_log(e, entry, parts)
        e.finalize()
        assert n == 0 and e.message_metrics.overall_count() == 0
        assert e.log_crc_failures() == [failure(b, ref[id(b)]) for b in order]
        assert e.log_crc_stats() == (len(order), len(order), sum(len(b.raw) for b in order))


def sized_batch(p, off, region, rng):
    """a batch whose CRC region (attributes to the end) is `region` bytes long: below one record (47 bytes), a batch
    without records followed by unread bytes; else one record whose value fills the rest"""
    if region < 47:
        raw = bytearray(kc.encode_batch(off, TS0 + off, [])) + rng.bytes(region - 40)
        raw[8:12] = struct.pack(">i", len(raw) - 12)
        return B(p, kc.set_crcs(bytes(raw)))
    v = max(0, region - 49)
    for _ in range(4):
        b = batch(p, off, [(TS0 + off, None, v)], values=[rng.bytes(v)])
        d = region - (len(b.raw) - 21)
        if d == 0:
            return b
        v += d
    raise AssertionError(region)


@pytest.mark.gpu
def test_crc_region_lengths():
    """regions of 40 bytes, S - 1 / S / S + 1, several spans, ~1 MiB and 16 MiB (more spans than the first power table
    holds) among small batches: exact whether they pass (nothing fails) or all fail (computed = the reference CRC)"""
    rng = np.random.default_rng(5)
    S = SPAN
    regions = [40, 41, 47, 100, S - 1, S, S + 1, 2 * S - 1, 2 * S, 2 * S + 1, 7 * S + 13, (1 << 20) + 5, 16 << 20]
    out, off = [], 0
    for r in regions:
        for _ in range(2):                                            # small ones around every sized one
            recs = random_recs(rng, 3, off)
            out.append(batch(0, off, recs))
            off += 3
        out.append(sized_batch(0, off, r, rng))
        assert len(out[-1].raw) - 21 == r
        off += max(1, len(out[-1].recs))
    ref = [b.crc for b in out]
    for flipped in (False, True):
        if flipped:
            for b in out:
                flip_crc(b)
        with engine(1) as e:
            n = scan_log_batches(e, stage_batches([(0, seg(out))]))
            e.finalize()
            assert n == len(passed(out))
            assert_parity(e, oracle_in_order(passed(out)), 1, check_alive=True)
            want = [failure(b, c) for b, c in zip(out, ref)] if flipped else []
            assert e.log_crc_failures() == want


@pytest.mark.gpu
def test_batches_at_odd_byte_offsets():
    """segments staged back to back behind 3 bytes of junk: batch headers at odd offsets of one device buffer"""
    parts = gen(13, P=3, nb=30)
    for v in parts.values():
        for b in v[::5]:
            damage(b, at=len(b.raw) - 1 - (len(b.raw) % 13), bit=3)
    order = interleaved(parts)
    staged = stage_batches([(0, b"\x01\x02\x03")] + [(b.p, b.raw) for b in order])
    assert any(int(o) % 2 for o in staged[2].cpu().numpy())
    with engine(3) as e:
        n = scan_log_batches(e, staged)
        e.finalize()
        assert n == len(passed(order))
        assert_parity(e, oracle_in_order(passed(order)), 3, check_alive=True)
        bad = [b for b in order if b.bad]
        assert [f[:4] for f in e.log_crc_failures()] == [failure(b, 0)[:4] for b in bad]
        assert [f[4] for f in e.log_crc_failures()] == [kc.batch_crc(b.raw, 0) for b in bad]


@pytest.mark.gpu
def test_failed_bytes_carry_past_2_32():
    """260 copies of one 16 MiB batch whose stored CRC is wrong, repeated on the device into one call of
    kta_scan_log_batches_device (4.4 GB on the device, nothing that size on the host): the failed bytes sum past 2^32, so the
    header pass's u64 carries into its high word.  baseOffset lies outside the CRC, so one reference serves every copy."""
    import torch
    from test_logcrc_passes import host_crcs
    rng = np.random.default_rng(30)
    b = flip_crc(sized_batch(0, 0, 16 << 20, rng))
    copies, size = 260, len(b.raw)
    assert copies * size > 1 << 32
    computed = int(host_crcs([np.frombuffer(b.raw, np.uint8)[21:]])[0])
    buf = torch.from_numpy(np.frombuffer(b.raw, np.uint8).copy()).cuda().repeat(copies)
    offs = torch.arange(copies, dtype=torch.int64, device="cuda") * size
    parts = torch.zeros(copies, dtype=torch.int32, device="cuda")
    with engine(1) as e:
        assert scan_log_batches(e, (buf, buf.numel(), offs, parts, copies)) == 0
        assert e.log_crc_stats() == (copies, copies, copies * size)
        assert e.log_crc_failures() == [failure(b, computed)] * copies


def _damaged(kind, rng):
    """a call of good batches with one batch damaged by a single bit inside its CRC region, and the refusal that damage
    causes without the check"""
    good = [batch(0, 10 * i, random_recs(rng, 5, 10 * i), codec) for i, codec in enumerate((None, "gzip", "lz4", None, "zstd"))]
    recs = [(TS0 + 100 + j, b"key-%d" % j, 40) for j in range(20)]
    if kind == "section":                                             # deflate block type: reserved or stored
        b, at, bit, msg = batch(0, 100, recs, "gzip"), 61 + 10, 2, "malformed (compressed )?record"
    elif kind == "records_count":                                     # recordsCount + 2^30
        b, at, bit, msg = batch(0, 100, recs), 57, 6, "malformed record batch header"
    else:                                                             # gzip (1) → 5, an unassigned codec
        b, at, bit, msg = batch(0, 100, recs, "gzip"), 22, 2, "unknown compression codec"
    return good[:2] + [damage(b, at, bit)] + good[2:], msg


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["section", "records_count", "codec_bits"])
def test_single_bit_damage(kind):
    batches, msg = _damaged(kind, np.random.default_rng(21))
    with engine(1) as e:
        assert e.push_log_segment(0, seg(batches)) == len(passed(batches))
        e.finalize()
        assert_parity(e, oracle_in_order(passed(batches)), 1, check_alive=True)
        assert e.log_crc_stats() == (len(batches), 1, len(batches[2].raw))
    with KtaEngine(1, count_alive_keys=True, now=NOW) as e:
        with pytest.raises(KtaError, match=msg):
            e.push_log_segment(0, seg(batches))


# ---- read_committed ---------------------------------------------------------------------------------------------------
def txn(p, off, recs, pid):
    rows = [(j, ts - recs[0][0], k, vl) for j, (ts, k, vl) in enumerate(recs)]
    return B(p, kc.set_crcs(kc.txn_batch(off, recs[0][0], rows, pid)), list(recs))


def abort_marker(p, off, pid):
    return B(p, kc.set_crcs(kc.marker(off, pid, 0, False, TS0)))


@pytest.mark.gpu
def test_read_committed_corrupted_abort_marker():
    """a marker that fails its CRC is not seen: its transaction is undecided, or aborted by the registered range"""
    recs = [(TS0 + i, b"k%d" % i, 10) for i in range(4)]
    plain = batch(0, 6, [(TS0 + 6, b"z", 1)])
    for with_index in (False, True):
        bs = [txn(0, 0, recs, 5), damage(abort_marker(0, 4, 5), at=70), plain]
        with engine(1, isolation_level="read_committed") as e:
            if with_index:
                e.push_txn_index(0, kc.txn_index([(5, 0, 4)]))
            n = e.push_log_segment(0, seg(bs))
            e.finalize()
            if with_index:
                bs[0].bad = True                                      # (left out as aborted)
                assert n == 1 and e.log_txn_stats() == (1, 4, 0)
            else:
                assert n == 5 and e.log_txn_stats() == (0, 0, 4)
            assert_parity(e, oracle_in_order(passed(bs)), 1, check_alive=True)
            assert e.log_crc_stats()[1] == 1 and e.log_crc_failures()[0][2] == 4


@pytest.mark.gpu
def test_read_committed_corrupted_aborted_batch_counts_as_crc_failure():
    recs = [(TS0 + i, b"k%d" % i, 10) for i in range(4)]
    bs = [damage(txn(0, 0, recs, 5), at=61 + 3), abort_marker(0, 4, 5), batch(0, 5, [(TS0 + 5, b"z", 1)])]
    with engine(1, isolation_level="read_committed") as e:
        assert e.push_log_segment(0, seg(bs)) == 1
        e.finalize()
        assert e.log_txn_stats() == (0, 0, 0)
        assert e.log_crc_stats() == (3, 1, len(bs[0].raw))
        assert_parity(e, oracle_in_order(passed(bs)), 1, check_alive=True)


@pytest.mark.gpu
def test_alive_keys_skipped_batch_held_the_last_write():
    """-c: the batch with a key's last write (a tombstone) fails its CRC: the previous writer wins"""
    bs = [batch(0, 0, [(TS0, b"k1", 5), (TS0 + 1, b"k2", 3)]), batch(0, 2, [(TS0 + 2, b"k1", None), (TS0 + 3, b"k3", 7)])]
    damage(bs[1], at=61 + 2)
    with engine(1) as e:
        assert e.push_log_segment(0, seg(bs)) == 2
        e.finalize()
        assert e.alive_keys() == 2
        o = oracle_in_order(passed(bs))
        assert_parity(e, o, 1, check_alive=True, hll_regs=o.hll_alive_regs(10))
    with KtaEngine(1, count_alive_keys=True, now=NOW) as e:
        assert e.push_log_segment(0, seg(bs)) == 4
        e.finalize()
        assert e.alive_keys() == 2                                    # k2, k3


# ---- the handle's state -----------------------------------------------------------------------------------------------
def tiny(p, n, off0=0):
    return [flip_crc(batch(p, off0 + i, [(TS0 + i, b"k%d" % (i % 50), i % 9)])) for i in range(n)]


@pytest.mark.gpu
def test_handle_state():
    bs = tiny(0, 10)
    s = seg(bs)
    with KtaEngine(2, now=NOW) as e:
        assert lib().kta_log_set_check_crcs(e.handle, 2) == _native.ERR_INVALID
        assert e.push_log_segment(0, s) == 10                          # off by default
        assert e.log_crc_stats() == (0, 0, 0) and e.log_crc_failures() == []
        e.set_check_crcs(True)
        assert e.push_log_segment(0, s) == 0
        e.set_check_crcs(False)
        assert e.push_log_segment(0, s) == 10
        e.set_check_crcs(True)
        assert e.log_crc_stats() == (10, 10, len(s))
        # a refused call (a batch with magic 3) counts nothing
        broken = bytearray(batch(0, 99, [(TS0, b"x", 1)]).raw)
        broken[16] = 3
        with pytest.raises(KtaError):
            e.push_log_segment(0, s + bytes(broken))
        assert e.log_crc_stats() == (10, 10, len(s)) and len(e.log_crc_failures()) == 10
        # the first KTA_LOG_CRC_KEEP failures, in call order, in batch order within a call
        e.reset()
        assert e.log_crc_stats() == (0, 0, 0) and e.log_crc_failures() == []
        a, b = tiny(0, 3000), tiny(1, 3000, off0=10_000)
        assert scan_log_segment(e, 0, seg(a)) == 0                     # (the switch survived the reset)
        assert e.push_log_segments([(1, seg(b))]) == 0
        got = e.log_crc_failures()
        assert len(got) == _native.LOG_CRC_KEEP
        assert got == [failure(x, kc.batch_crc(x.raw, 0)) for x in (a + b)[:_native.LOG_CRC_KEEP]]
        assert e.log_crc_stats()[:2] == (6000, 6000)


@pytest.mark.gpu
def test_default_off_accepts_zero_crcs():
    """segments of the encoders that write CRC 0 are accepted as before with the switch off, and all fail with it on"""
    rng = np.random.default_rng(4)
    recs = [(TS0 + i, b"k%d" % (i % 11), int(rng.integers(0, 50))) for i in range(400)]
    s = kc.encode_partition(recs, rng, max_batch=30, compression=["gzip", "lz4", None])
    nb = len(kc.batch_offsets(s))
    with KtaEngine(1, count_alive_keys=True, now=NOW) as e:
        assert e.push_log_segment(0, s) == 400
        e.finalize()
        assert_parity(e, oracle_in_order((0, *r) for r in recs), 1, check_alive=True)
        e.set_check_crcs(True)
        assert e.push_log_segment(0, s) == 0
        assert e.log_crc_stats()[:2] == (nb, nb)


# ---- CLI --------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_cli_check_crcs(tmp_path):
    from test_report import CLI_DIR, _build
    _build()
    P = 2
    parts = gen(14, P=P, nb=25, codecs=(None, "gzip"))
    old = parts[1][7]                                                 # replaced by an uncompressed batch ending in a
    victim = batch(1, old.base_offset, old.recs[:-1] + [old.recs[-1][:2] + (40,)])   # 40-byte value
    parts[1][7] = victim
    stored = victim.crc
    raw = bytearray(victim.raw)
    raw[-5] ^= 0x10                                                   # a byte of that value: it still decodes
    victim.raw = bytes(raw)
    for p in range(P):
        d = tmp_path / ("orders-%d" % p)
        d.mkdir()
        (d / "00000000000000000000.log").write_bytes(seg(parts[p]))
    cli = os.path.join(CLI_DIR, "kafka-topic-analyzer")
    base = [cli, "-t", "orders", "-b", "unused:9092", "-c", "--log-dir", str(tmp_path)]
    for check in (False, True):                       # without the option: every batch, as before, and no warning
        victim.bad = check
        r = subprocess.run(base + (["--librdkafka", "check.crcs=true"] if check else []), capture_output=True, text=True)
        assert r.returncode == 0, r.stderr
        o = oracle_in_order(passed([b for p in range(P) for b in parts[p]]))
        lines = r.stdout.splitlines()
        assert "Alive keys: %d" % o.scalar("sum_all_alive") in lines
        assert "Topic Size: %d bytes" % o.scalar("overall_size") in lines
        rows = [l for l in lines if l.startswith("| ") and l[2].isdigit()]
        assert len(rows) == P
        for l in rows:
            c = [x.strip() for x in l.strip("|").split("|")]
            p = int(c[0])
            assert [int(c[3]), int(c[4]), int(c[5])] == [o.counter("total", p), o.counter("alive", p), o.counter("tombstones", p)]
            assert [int(c[10]), int(c[11])] == [o.counter("key_size_sum", p), o.counter("value_size_sum", p)]
        warn = [l for l in r.stderr.splitlines() if "CRC32C" in l]
        if check:
            assert warn == ["warning: Kafka error: MessageSet at offset %d (%d bytes) of partition 1 failed CRC32C check "
                            "(original 0x%08x != calculated 0x%08x)" % (victim.base_offset, len(victim.raw), stored,
                                                                       kc.batch_crc(victim.raw, 0))]
        else:
            assert warn == []
