"""Streaming sessions over several time-aligned captures (btle_b200_streams_*, BtleRx.streams, btle_rx_b200 with several
-i / --iq-dir): the records equal one rx_batch call over the captures cut to the shortest one, whatever the segment size
and however the bytes arrive; the program reads files and live FIFOs through them."""
import ctypes
import json
import os
import signal
import subprocess
import sys
import time

import numpy as np
import pytest

import orc
from btle_b200 import BtleError, BtleRx, REC_DTYPE, make_cfgs, synth

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CLI = os.path.join(ROOT, "btle_b200", "btle_rx_b200")
CHUNK = 16384
EINVAL = -1


@pytest.fixture(scope="module")
def rx():
    import __graft_entry__ as ge
    ge.build()
    r = BtleRx(0)
    yield r
    r.close()


def _same(a, b):
    assert len(a) == len(b), (len(a), len(b))
    if a.tobytes() != b.tobytes():
        for i, (x, y) in enumerate(zip(a, b)):
            assert x.tobytes() == y.tobytes(), (i, x, y)


def _default_seg(n):
    return max(16, (4096 // n + 15) // 16 * 16)


def _captures(n, chunks, seed):
    """n captures of different lengths (none a multiple of 16384) with mixed channels, access addresses, CRC inits, flags
    0..3, a sparse mask on two advertising captures (rejected hits with -v) and one capture in raw mode."""
    rng = np.random.default_rng(seed)
    cfgs = synth.channel_plan(40)[rng.permutation(40)[:n]] if n > 1 else synth.channel_plan(38)[37:38]
    if n >= 3:
        cfgs[:3] = synth.channel_plan(40)[[37, 9, 38]]
    lens = [chunks * CHUNK + int(rng.integers(1, 3 * CHUNK)) for _ in range(n)]
    while any(l_ % CHUNK == 0 for l_ in lens):
        lens = [l_ + 1 for l_ in lens]
    iq, _ = synth.synth_streams_device(cfgs, max(lens), seed, slot_samples=3300, corrupt_every=5, straddle_every=3, want_truth=False)
    iq = iq.cpu().numpy()
    cfgs["rssi"] = np.arange(n) % 4
    adv = np.flatnonzero(cfgs["channel"] >= 37)
    cfgs["access_mask"][adv[:2]] = 0x0F000000
    cfgs["rssi"][adv[:2]] |= 2
    if n > 1:
        cfgs["raw"][1] = 1
    return [iq[i, :lens[i]].copy() for i in range(n)], cfgs


def _batch(rx, caps, cfgs):
    """rx_batch over the captures cut to the shortest one: what a session must return."""
    m = min(c.size for c in caps)
    return rx.rx_batch(np.stack([c[:m] for c in caps]), cfgs)


def _feed(s_, caps, rng, sizes):
    """Random push sizes, interleaved across the captures in random order; returns the list of returned arrays."""
    pos, parts = [0] * len(caps), []
    while True:
        live = [i for i in range(len(caps)) if pos[i] < caps[i].size]
        if not live:
            break
        i = int(rng.choice(live))
        k = int(rng.choice(sizes))
        parts.append(s_.push(i, caps[i][pos[i]:pos[i] + k]))
        pos[i] += k
    parts.append(s_.finish())
    return parts


def _check_set_order(got, seg):
    """Within each segment set records are in (stream, chunk) order and sets follow each other; `chunk` is stream-wide."""
    key = np.stack([got["chunk"] // seg, got["stream"], got["chunk"]], axis=1).astype(np.int64)
    for a, b in zip(key[:-1], key[1:]):
        assert tuple(a) <= tuple(b), (a, b)


_CACHE = {}


def _case(rx, n):
    if n not in _CACHE:
        caps, cfgs = _captures(n, {1: 150, 3: 60, 40: 12}[n], seed=500 + n)
        _CACHE[n] = (caps, cfgs, _batch(rx, caps, cfgs))
    return _CACHE[n]


@pytest.mark.parametrize("n", [1, 3, 40])
@pytest.mark.parametrize("seg", [1, 5, 16, 64, 0])
def test_session_equals_batch(rx, n, seg):
    caps, cfgs, exp = _case(rx, n)
    assert len(exp) > 30 * n and ((exp["flags"] & 4) != 0).any()
    rng = np.random.default_rng(seg * 100 + n)
    eff = seg or _default_seg(n)
    sizes = [1, 7, 100, 4096, CHUNK, 50000, eff * CHUNK + 4096, 3 * eff * CHUNK]
    with rx.streams(cfgs, segment_chunks=seg) as s_:
        parts = _feed(s_, caps, rng, sizes)
    got = np.concatenate(parts)
    for p in parts:
        _check_set_order(p, eff)
    _check_set_order(got, eff)
    # (stream, chunk) order of the batch call; inside a chunk, the reference's order
    order = np.lexsort((got["chunk"], got["stream"]))
    _same(got[order], exp)


def test_session_slice_equals_oracle(rx):
    """The batch call the sessions are compared with is itself the oracle's answer: spot check of the 3-capture case."""
    caps, cfgs, exp = _case(rx, 3)
    m = min(c.size for c in caps)
    for i in range(3):
        c = cfgs[i]
        want = orc.rx_flags(caps[i][:m], int(c["rssi"]), channel=int(c["channel"]), access_addr=int(c["access_addr"]),
                            access_mask=int(c["access_mask"]), crc_init=int(c["crc_init"]), raw=int(c["raw"]), stream=i)
        _same(exp[exp["stream"] == i], want)


def test_short_tail_cut_into_more_units_than_a_full_segment(rx):
    """A tail of 512 chunks behind the default 4096-chunk segment is spread over the grid in one-chunk units: more units
    than a full segment has.  The single-capture session and a one-capture btle_b200_streams both decode it."""
    iq, _ = synth.make_adv_stream(512 * CHUNK + 999, seed=5, channel=37, slot_samples=4096, device="cuda")
    iq = iq.cpu().numpy()
    exp = rx.rx(iq, channel=37, rssi=1)
    assert len(exp) > 1000
    with rx.stream(channel=37, rssi=1) as s_:
        _same(np.concatenate([s_.push(iq), s_.finish()]), exp)
    with rx.streams(make_cfgs(1, channel=37, rssi=1)) as s_:
        _same(np.concatenate([s_.push(0, iq), s_.finish()]), exp)


def test_set_cfg_mid_session(rx):
    """Capture 1 changes its CRC init and capture 2 its access address after segment set k: chunks before the switch
    equal rx_batch with the old cfg, chunks after it rx_batch with the new one; capture 0 is unaffected."""
    caps, cfgs = _captures(3, 40, seed=77)
    caps[2] = caps[0][: caps[2].size].copy()                       # capture 2: capture 0's ADV bursts, then a wrong AA
    cfgs[2] = cfgs[0]
    cfgs["rssi"], cfgs["raw"], cfgs["access_mask"] = 1, 0, 0xFFFFFFFF
    new = cfgs.copy()
    new[1]["crc_init"] ^= 0x000101
    new[2]["access_addr"] = 0x12345678
    seg, k = 4, 2
    cut = (k + 1) * seg * CHUNK + 4096                             # every capture's part of set k (look-ahead included) is complete
    with rx.streams(cfgs, segment_chunks=seg) as s_:
        parts = [s_.push(i, caps[i][:cut]) for i in range(3)]
        s_.set_cfg(1, crc_init=int(new[1]["crc_init"]))
        s_.set_cfg(2, access_addr=0x12345678)
        parts += [s_.push(i, caps[i][cut:]) for i in range(3)] + [s_.finish()]
    got = np.concatenate(parts)
    got = got[np.lexsort((got["chunk"], got["stream"]))]
    old_b, new_b = _batch(rx, caps, cfgs), _batch(rx, caps, new)
    K = (k + 1) * seg
    exp = np.concatenate([np.concatenate([old_b[(old_b["stream"] == i) & (old_b["chunk"] < K)],
                                          new_b[(new_b["stream"] == i) & (new_b["chunk"] >= K)]]) for i in range(3)])
    assert (new_b[new_b["stream"] == 1]["crc_bad"] == 1).all() and (new_b["stream"] == 2).sum() == 0
    assert ((exp["stream"] == 1) & (exp["chunk"] >= K)).sum() > 10 and ((exp["stream"] == 2) & (exp["chunk"] < K)).sum() > 10
    _same(got, exp)


def _raw_session(rx, cfgs, seg):
    L = rx._L
    h = ctypes.c_void_p()
    rc = L.btle_b200_streams_open(rx._h, cfgs.ctypes.data, len(cfgs), seg, ctypes.byref(h))
    return rc, h


def _raw_push(L, h, stream, data, out, cap):
    """acquire / commit until `data` is in or the capture's part is full; returns (records, bytes taken)"""
    got, done = [], 0
    while done < data.size:
        buf, space = ctypes.c_void_p(), ctypes.c_size_t(0)
        assert L.btle_b200_streams_acquire(h, stream, ctypes.byref(buf), ctypes.byref(space)) == 0
        k = min(space.value, data.size - done)
        if k == 0:
            return got, done
        ctypes.memmove(buf.value, data[done:].ctypes.data, k)
        n = ctypes.c_size_t(0)
        assert L.btle_b200_streams_commit(h, stream, k, out.ctypes.data, cap, ctypes.byref(n)) == 0
        got.append(out[:n.value].copy())
        done += k
    return got, done


@pytest.mark.parametrize("flags", [2, 3])
def test_worst_case_density_with_a_small_cap(rx, flags):
    """Mask 0 and -v on three all-zero captures on channel 38: 123 rejected records per chunk.  With `cap` far below a
    set's count every record still arrives, over repeated commit / finish calls (BTLE_EOVERFLOW until drained)."""
    L = rx._L
    z = np.zeros(9 * CHUNK + 5000, dtype=np.int8)
    cfgs = make_cfgs(3, channel=38, access_addr=0, access_mask=0, rssi=flags)
    exp = rx.rx_batch(np.stack([z, z, z]), cfgs)
    assert len(exp) == 3 * 9 * 123
    cap = 50
    out = np.zeros(cap, dtype=REC_DTYPE)
    rc, h = _raw_session(rx, cfgs, 2)
    assert rc == 0
    try:
        parts, pos = [], [0, 0, 0]
        while any(p < z.size for p in pos):
            for i in range(3):
                g, k = _raw_push(L, h, i, z[pos[i]:pos[i] + 30000], out, cap)
                parts += g
                pos[i] += k
            n = ctypes.c_size_t(0)                                   # drain with zero-byte commits
            while True:
                assert L.btle_b200_streams_commit(h, 0, 0, out.ctypes.data, cap, ctypes.byref(n)) == 0
                parts.append(out[:n.value].copy())
                if n.value < cap:
                    break
        calls = 0
        while True:
            n = ctypes.c_size_t(0)
            rc = L.btle_b200_streams_finish(h, out.ctypes.data, cap, ctypes.byref(n))
            parts.append(out[:n.value].copy())
            calls += 1
            if rc != -5:
                assert rc == 0
                break
            assert n.value == cap
        assert calls > 1
    finally:
        L.btle_b200_streams_close(h)
    got = np.concatenate(parts)
    _same(got[np.lexsort((got["chunk"], got["stream"]))], exp)


def test_validation_errors_leave_the_session_usable(rx):
    L = rx._L
    caps, cfgs = _captures(3, 8, seed=9)
    exp = _batch(rx, caps, cfgs)
    with pytest.raises(BtleError) as e:
        rx.streams(make_cfgs(0))
    assert e.value.code == EINVAL
    bad = cfgs.copy()
    bad[2]["channel"] = 40
    with pytest.raises(BtleError) as e:
        rx.streams(bad)
    assert e.value.code == EINVAL
    with rx.streams(cfgs, segment_chunks=3) as s_:
        parts = [s_.push(0, caps[0][:70000])]
        with pytest.raises(BtleError) as e:
            s_.push(3, caps[0][:10])
        assert e.value.code == EINVAL and "out of range" in str(e.value)
        with pytest.raises(BtleError) as e:
            s_.set_cfg(1, channel=41)
        assert e.value.code == EINVAL
        with pytest.raises(BtleError) as e:
            s_.set_cfg(5, channel=1)
        assert e.value.code == EINVAL
        buf, space = ctypes.c_void_p(), ctypes.c_size_t(0)
        assert L.btle_b200_streams_acquire(s_._h, 1, ctypes.byref(buf), ctypes.byref(space)) == 0
        n = ctypes.c_size_t(0)
        assert L.btle_b200_streams_commit(s_._h, 1, space.value + 1, None, 0, ctypes.byref(n)) == EINVAL
        assert b"more bytes than acquired" in L.btle_b200_last_error(rx._h)
        assert L.btle_b200_streams_acquire(s_._h, 3, ctypes.byref(buf), ctypes.byref(space)) == EINVAL
        parts += [s_.push(0, caps[0][70000:]), s_.push(1, caps[1]), s_.push(2, caps[2]), s_.finish()]
    got = np.concatenate(parts)
    _same(got[np.lexsort((got["chunk"], got["stream"]))], exp)


# ---- the program ----------------------------------------------------------------------------------------------------
def _run(args, **kw):
    return subprocess.run([CLI] + args, capture_output=True, text=True, **kw)


def _pk(s_):
    return [l for l in s_.splitlines() if '"t":"pkt"' in l]


@pytest.fixture(scope="module")
def cli_caps(tmp_path_factory, rx):
    d = tmp_path_factory.mktemp("caps")
    a, _ = synth.make_adv_stream(40 * CHUNK + 3333, seed=21, channel=37, slot_samples=2600, straddle_every=4)
    b, _ = synth.make_adv_stream(41 * CHUNK + 777, seed=22, channel=9, slot_samples=3100, access_addr=0x60850A24, crc_init=0xA77B2B,
                                 data_channel_pdu=True, corrupt_every=6)
    c, _ = synth.make_adv_stream(40 * CHUNK + 9000, seed=23, channel=38, slot_samples=2900, straddle_every=5)
    raw = {"a": a.numpy(), "b": b.numpy(), "c": c.numpy()}
    for k, v in raw.items():
        v.tofile(d / f"{k}.bin")
    return d, raw


def _multi_args(d, a="a.bin", b="b.bin", c="c.bin"):
    return ["-i", f"{d}/{a}:37", "-i", f"{d}/{b}:9:60850a24:a77b2b", "-i", f"{d}/{c}:38"]


def test_cli_multi_capture_streams_like_the_batch(cli_caps, tmp_path):
    """Several -i: the same text, NDJSON and pcap for every segment size; the packets are those of the single-capture runs
    on the captures cut to the shortest one, merged in time order (what the whole-file batch printed); --iq-dir (without -o)
    prints the same."""
    d, raw = cli_caps
    m = min(v.size for v in raw.values())
    outs, pcaps = [], []
    for seg in (["--segment-chunks", "1"], ["--segment-chunks", "3"], []):
        wd = tmp_path / f"run{len(outs)}"                          # same pcap name in every run: the banner prints it
        wd.mkdir()
        p = _run(_multi_args(d) + ["-j", "-s", "out.pcap"] + seg, cwd=wd)
        assert p.returncode == 0, p.stdout + p.stderr
        outs.append(p.stdout)
        pcaps.append((wd / "out.pcap").read_bytes())
    assert outs[0] == outs[1] == outs[2] and pcaps[0] == pcaps[1] == pcaps[2]
    got = [json.loads(l) for l in _pk(outs[0])]
    singles = []
    for k, ch, extra in (("a", 37, []), ("b", 9, ["-a", "60850a24", "-k", "a77b2b"]), ("c", 38, [])):
        f = tmp_path / f"{k}.cut"
        raw[k][:m].tofile(f)
        r = _run(["-i", str(f), "-c", str(ch), "-j", "-Q"] + extra)
        assert r.returncode == 0
        singles += [json.loads(l) for l in _pk(r.stdout)]
    assert len(got) == len(singles) > 60
    assert [e["ts"] for e in got] == sorted(e["ts"] for e in got)
    strip = lambda e: {k: v for k, v in e.items() if k != "pkt"}
    assert sorted(map(json.dumps, map(strip, got))) == sorted(map(json.dumps, map(strip, singles)))
    stop = json.loads([l for l in outs[0].splitlines() if '"t":"status"' in l][-1])
    assert stop["event"] == "stop" and stop["ts"] == pytest.approx((m // 2) / 4e6, abs=1e-6)
    # --iq-dir: the same captures as ch09 / ch37 / ch38
    dd = tmp_path / "dir"
    dd.mkdir()
    for k, ch in (("a", 37), ("b", 9), ("c", 38)):
        os.symlink(d / f"{k}.bin", dd / f"ch{ch:02d}.bin")
    q = _run(["--iq-dir", str(dd), "-a", "60850a24", "-k", "a77b2b", "-j"])
    assert q.returncode == 0, q.stdout + q.stderr
    assert _pk(q.stdout) == _pk(outs[0])


_WRITER = r"""
import os, random, sys, time
src, dst, seed, pace = sys.argv[1], sys.argv[2], int(sys.argv[3]), float(sys.argv[4])
data = open(src, "rb").read()
rnd = random.Random(seed)
try:
    with open(dst, "wb", buffering=0) as f:
        pos = 0
        while pos < len(data):
            k = rnd.choice([1, 333, 4096, 20000, 65536, 150000])
            f.write(data[pos:pos + k])
            pos += k
            time.sleep(pace * rnd.random())
except BrokenPipeError:
    pass
"""


def _writers(d, fifo_dir, paces):
    procs = []
    for k, seed, pace in zip("abc", (1, 2, 3), paces):
        os.mkfifo(fifo_dir / f"{k}.fifo")
        procs.append(subprocess.Popen([sys.executable, "-c", _WRITER, str(d / f"{k}.bin"), str(fifo_dir / f"{k}.fifo"), str(seed),
                                       str(pace)], stderr=subprocess.DEVNULL))
    return procs


def _reap(procs):
    for p in procs:
        try:
            p.wait(timeout=60)
        except subprocess.TimeoutExpired:
            p.kill()
            p.wait()


def test_cli_live_fifos(cli_caps, tmp_path):
    """Three writer processes feed three FIFOs in random pieces at different paces: the same output as the files.  A second
    run is stopped with SIGINT mid-stream: exit code 0, NDJSON ends with 'stop', and the packets printed are the first
    packets of the full run, in time order."""
    d, raw = cli_caps
    full = _run(_multi_args(d) + ["-j", "-Q", "--segment-chunks", "2"])
    assert full.returncode == 0
    f1 = tmp_path / "run1"
    f1.mkdir()
    procs = _writers(d, f1, (0.0, 0.002, 0.01))
    try:
        live = _run(_multi_args(f1, "a.fifo", "b.fifo", "c.fifo") + ["-j", "-Q", "--segment-chunks", "2"], timeout=300)
    finally:
        _reap(procs)
    assert live.returncode == 0, live.stdout + live.stderr
    assert _pk(live.stdout) == _pk(full.stdout) and len(_pk(full.stdout)) > 60
    # SIGINT mid-stream
    f2 = tmp_path / "run2"
    f2.mkdir()
    procs = _writers(d, f2, (0.2, 0.3, 0.4))
    try:
        p = subprocess.Popen([CLI] + _multi_args(f2, "a.fifo", "b.fifo", "c.fifo") + ["-j", "-Q", "--segment-chunks", "2"],
                             stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True)
        lines, t0 = [], time.time()
        while time.time() - t0 < 120:
            line = p.stdout.readline()
            if not line:
                break
            lines.append(line.rstrip("\n"))
            if sum('"t":"pkt"' in l for l in lines) >= 5:
                break
        p.send_signal(signal.SIGINT)
        rest = p.stdout.read()
        assert p.wait(timeout=60) == 0
    finally:
        if p.poll() is None:
            p.kill()
            p.wait()
        _reap(procs)
    out = lines + rest.splitlines()
    ev = [json.loads(l) for l in out if l.startswith("{")]
    assert ev[-1]["t"] == "status" and ev[-1]["event"] == "stop"
    got, want = _pk("\n".join(out)), _pk(full.stdout)
    assert 5 <= len(got) < len(want)
    assert got == want[:len(got)]
