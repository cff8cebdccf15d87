"""Connections on a streaming session (btle_b200_streams_add_cfg / remove_cfg / resident / set_discover / take_cands,
RxStreams, hop.ConnectionMonitor): every cfg's records equal rx_batch on its capture kept for [from_chunk, until_chunk),
backfilled over the sets still on the device; discovery per set equals the whole-capture scan; the live monitor finds
what decode_connections() finds on the recorded captures."""
import os

import numpy as np
import pytest
import torch

from btle_b200 import BtleError, BtleRx, make_cfgs, synth
from btle_b200.hop import ConnectionMonitor, decode_connections
from btle_b200._native import BTLE_EINVAL
from test_rx_multi import _traffic, connections_capture
from test_stream_sessions_gpu import CHUNK, _feed, _same

pytestmark = pytest.mark.gpu

AAS = [0x8E89BED6, 0x60850A1B, 0x50850A1C, 0x12345679, 0x3A5C96E1]


@pytest.fixture(scope="module")
def rx():
    import __graft_entry__ as ge
    ge.build()
    r = BtleRx(0)
    yield r
    r.close()


@pytest.fixture(scope="module")
def traffic():
    """Four captures (channels 37, 5, 38, 22) with bursts of five access addresses, ragged lengths."""
    iq = _traffic(40 * CHUNK + 5000, [37, 5, 38, 22], AAS, seed=3)
    return [iq[0].copy(), iq[1, :-3000].copy(), iq[2, :-77].copy(), iq[3].copy()]


def _expect(rx, caps, entries):
    """entries: {index: (capture, cfg[1], from, until)} -> rx_batch of each on its capture (cut to the shortest), kept for
    [from, until), stream = index, in (index, chunk, n0) order."""
    m = min(c.size for c in caps)
    out = []
    for j in sorted(entries):
        cap, cfg, lo, hi = entries[j]
        r = rx.rx_batch(caps[cap][:m], cfg).copy()
        r = r[(r["chunk"] >= lo) & (r["chunk"] < hi)]
        r["stream"] = j
        out.append(r)
    return np.concatenate(out)


def _by_cfg(got):
    return got[np.lexsort((got["chunk"], got["stream"]))]


def _extra_cfgs(K, capture_channel, seed):
    rng = np.random.default_rng(seed)
    masks = [0xFFFFFFFF, 0xFFFFFFFF, 0xFFFF00FF, 0x0000FFFF, 0xFFFFFFF0, 0, 0xFFFFFFFF, 0x7FFFFFFE]
    out = []
    for k in range(K):
        aa = AAS[k % 5] if k < 10 else int(rng.integers(0, 1 << 32))
        crc = 0x555555 if capture_channel >= 37 else 0x227BA7 ^ (aa & 0xFFFF)
        out.append(dict(channel=capture_channel, access_addr=aa, access_mask=masks[k % 8], crc_init=crc, raw=int(k == 3), rssi=k % 4))
    return out


@pytest.mark.parametrize("seg", [16, 17, 1])
@pytest.mark.parametrize("K,remove_base", [(1, False), (8, False), (9, True), (20, False), (20, True)])
def test_fixed_lists_equal_rx_batch(rx, traffic, seg, K, remove_base):
    caps = traffic
    base = make_cfgs(4, channel=[37, 5, 38, 22], crc_init=[0x555555, 0x227BA7, 0x555555, 0x227BA7], rssi=1)
    entries = {} if remove_base else {i: (i, base[i:i + 1], 0, 1 << 40) for i in range(4)}
    rng = np.random.default_rng(seg * 100 + K)
    with rx.streams(base, segment_chunks=seg) as s_:
        if remove_base:
            assert [s_.remove_cfg(i) for i in range(4)] == [0] * 4
        for f in _extra_cfgs(K, 5, seed=K):
            j, frm = s_.add_cfg(1, **f)
            assert frm == 0
            entries[j] = (1, make_cfgs(1, **f), 0, 1 << 40)
        sizes = [1, 7, 4096, CHUNK, 50000, seg * CHUNK + 4096, 3 * seg * CHUNK]
        parts = _feed(s_, caps, rng, sizes)
        launches = rx.last_launches
    got = np.concatenate(parts)
    for p in parts:                                            # inside a set: (cfg, chunk) order
        key = np.stack([p["chunk"] // seg, p["stream"], p["chunk"]], axis=1)
        assert all(tuple(a) <= tuple(b) for a, b in zip(key[:-1], key[1:]))
    exp = _expect(rx, caps, entries)
    assert len(exp) > 50
    _same(_by_cfg(got), exp)
    # the tail set: one rx_multi round per 8 cfgs of the busiest capture
    assert launches == -(-(K + (0 if remove_base else 1)) // 8)


def test_no_added_cfg_keeps_the_single_launch(rx, traffic):
    base = make_cfgs(4, channel=[37, 5, 38, 22], rssi=1)
    with rx.streams(base, segment_chunks=4) as s_:
        parts = [s_.push(i, traffic[i][:5 * 4 * CHUNK]) for i in range(4)]
        assert rx.last_launches == 1 and s_.resident == 2 * 4   # sets 0..3 submitted: 2 and 3 still on the device
        parts += [s_.push(i, traffic[i][5 * 4 * CHUNK:]) for i in range(4)] + [s_.finish()]
    got = np.concatenate(parts)
    m = min(c.size for c in traffic)
    _same(_by_cfg(got), rx.rx_batch(np.stack([c[:m] for c in traffic]), base))


@pytest.mark.parametrize("seg", [1, 4, 17])
def test_replaced_cfg_keeps_the_single_launch(rx, traffic, seg):
    """Capture 1's cfg removed, then another access address added on capture 1 from chunk 0: one cfg per capture in
    capture order again, but under index 4.  Every set is one launch, and the records are rx_batch with the replaced
    cfg, stream = 4 for capture 1."""
    base = make_cfgs(4, channel=[37, 5, 38, 22], crc_init=[0x555555, 0x227BA7, 0x555555, 0x227BA7], rssi=1)
    f = dict(access_addr=AAS[1], crc_init=0x227BA7 ^ (AAS[1] & 0xFFFF))
    new = base[1:2].copy()
    for k, v in f.items():
        new[k] = v
    entries = {i: (i, base[i:i + 1], 0, 1 << 40) for i in (0, 2, 3)}
    entries[4] = (1, new, 0, 1 << 40)
    step = seg * CHUNK
    with rx.streams(base, segment_chunks=seg) as s_:
        assert s_.remove_cfg(1) == 0
        assert s_.add_cfg(1, 0, **f) == (4, 0)
        parts = []
        for pos in range(0, max(c.size for c in traffic), step):
            parts += [s_.push(i, traffic[i][pos:pos + step]) for i in range(4)]
            if pos:                                            # sets 0.. are submitted from the second round on
                assert rx.last_launches == 1, pos
        parts.append(s_.finish())
        assert rx.last_launches == 1                           # the tail set
    for p in parts:                                            # inside a set: (cfg, chunk) order
        key = np.stack([p["chunk"] // seg, p["stream"], p["chunk"]], axis=1)
        assert all(tuple(a) <= tuple(b) for a, b in zip(key[:-1], key[1:]))
    got = np.concatenate(parts)
    exp = _expect(rx, traffic, entries)
    assert (exp["stream"] == 4).sum() > 5 and len(exp) > 50
    _same(_by_cfg(got), exp)


def test_mid_stream_add_remove_and_backfill(rx, traffic):
    caps = traffic
    base = make_cfgs(4, channel=[37, 5, 38, 22], crc_init=[0x555555, 0x227BA7, 0x555555, 0x227BA7])
    seg, k = 3, 4
    entries = {i: (i, base[i:i + 1], 0, 1 << 40) for i in range(4)}
    extra = _extra_cfgs(6, 5, seed=1) + _extra_cfgs(2, 22, seed=2)
    cut = (k + 1) * seg * CHUNK + 4096                         # sets 0..k complete: k in flight, k-1 handed out
    rng = np.random.default_rng(5)
    with rx.streams(base, segment_chunks=seg) as s_:
        parts = [s_.push(i, caps[i][:cut]) for i in range(4)]
        res = s_.resident
        assert res == (k - 1) * seg                            # the handed-out set and the one in flight
        with pytest.raises(BtleError) as e:
            s_.add_cfg(1, res - 1, **extra[0])
        assert e.value.code == BTLE_EINVAL and "resident" in str(e.value)
        for f, frm in zip(extra[:3], (res, res + 1, res + seg + 1)):   # at resident, one after, inside the in-flight set
            j, got_frm = s_.add_cfg(1, frm, **f)
            assert got_frm == frm
            entries[j] = (1, make_cfgs(1, **f), frm, 1 << 40)
        j, _ = s_.add_cfg(3, None, **extra[6])
        entries[j] = (3, make_cfgs(1, **extra[6]), res, 1 << 40)
        until = s_.remove_cfg(3)                               # at the boundary of the next set
        assert until == (k + 1) * seg
        entries[3] = (3, base[3:4], 0, until)
        with pytest.raises(BtleError):
            s_.remove_cfg(3)
        # the rest in random pieces, one more add at a later set boundary
        pos = [cut] * 4
        while any(p < c.size for p, c in zip(pos, caps)):
            i = int(rng.integers(4))
            n = int(rng.choice([100, 5000, CHUNK, 3 * CHUNK]))
            parts.append(s_.push(i, caps[i][pos[i]:pos[i] + n]))
            pos[i] += n
            if len(entries) == 8 and s_.resident >= 20:
                f = extra[3]
                j, frm = s_.add_cfg(1, None, **f)
                entries[j] = (1, make_cfgs(1, **f), frm, 1 << 40)
        parts.append(s_.finish())
        # an add after the last hand-out: its backfill comes from the next finish
        res = s_.resident
        f = dict(channel=22, access_addr=0x12345679, access_mask=0, crc_init=0x227BA7 ^ 0x5679, raw=0, rssi=1)   # hits everywhere
        j, frm = s_.add_cfg(3, None, **f)
        assert frm == res
        entries[j] = (3, make_cfgs(1, **f), frm, 1 << 40)
        late = s_.finish()
        assert len(late) and (late["stream"] == j).all()
        parts.append(late)
        assert len(s_.finish()) == 0
    assert len(entries) == 10
    got = np.concatenate(parts)
    exp = _expect(rx, caps, entries)
    for j in entries:
        assert (exp["stream"] == j).sum() > 0, j
    _same(_by_cfg(got), exp)


# ---- discovery per set ------------------------------------------------------------------------------------------------
def _empty_pdu(ch, aa=0x5A3C96E1, crc=0x13579B):
    return synth.air_bytes(synth.ll_data_pdu(1, 0, 0, 0, b""), ch, aa, crc)


def _place_clip(cap, ch, p, air, amp=70):
    """air at sample p of capture ch, cut at the capture's end"""
    wav = synth.modulate(air).astype(np.int32) * amp // 127
    a = 2 * p
    k = min(wav.size, cap.shape[1] - a)
    cap[ch, a:a + k] = np.clip(cap[ch, a:a + k].astype(np.int32) + wav[:k], -128, 127).astype(np.int8)


def _boundary_capture(seg, n_chunks=110):
    """37 data captures with empty PDUs at n0 0..40 samples after a set start and 280..290 before a set end (one offset
    per capture and set), at the first and last valid window, and a dense run (an empty PDU every 400 samples on every
    capture) through set 5 that overflows the set's first candidate buffer."""
    n = n_chunks * CHUNK + 1234
    gen = torch.Generator(); gen.manual_seed(seg)
    cap = synth.noise_floor(40 * n, gen).numpy().reshape(40, n).copy()
    per_set = seg * 8192
    for c in range(37):
        S1, S2 = per_set * (1 + c % 3), per_set * (2 + c % 3)
        _place_clip(cap, c, S1 + c * 41 // 37 - 34, _empty_pdu(c))
        _place_clip(cap, c, S2 - 280 - c % 11 - 34, _empty_pdu(c))
    _place_clip(cap, 5, 0, _empty_pdu(5))                      # n0 ~ 33: the first valid window
    for c, back in ((6, 319), (7, 320), (8, 321), (9, 300), (10, 360)):   # around the last valid window of the capture
        _place_clip(cap, c, n // 2 - back, _empty_pdu(c))
    for c in range(37):
        for p in range(5 * per_set + 1000, 6 * per_set - 1000, 400):
            _place_clip(cap, c, p, _empty_pdu(c, 0x71764129, 0x0BADC0))
    return cap


def _random_capture():
    rng = np.random.default_rng(3)
    return rng.integers(-128, 128, (40, 30 * CHUNK + 999), dtype=np.int8)


@pytest.mark.parametrize("seg", [16, 17])
@pytest.mark.parametrize("kind", ["connections", "boundaries", "random"])
def test_discovery_per_set_equals_whole_capture(rx, seg, kind):
    cap = {"connections": lambda: connections_capture()[0], "boundaries": lambda: _boundary_capture(seg), "random": _random_capture}[kind]()
    caps = [cap[c].copy() for c in range(40)]
    if kind == "random":
        caps = [c[:c.size - 7 * i] for i, c in enumerate(caps)]   # ragged: cut to the shortest
    m = min(c.size for c in caps)
    exp = rx.discover(np.stack([c[:m] for c in caps[:37]]), np.arange(37, dtype=np.int32))
    assert len(exp) > 10
    with rx.streams(make_cfgs(40, channel=list(range(40))), segment_chunks=seg) as s_:
        s_.set_discover(list(range(37)) + [-1] * 3)
        rng = np.random.default_rng(seg)
        got = []
        pos = [0] * 40
        while any(p < c.size for p, c in zip(pos, caps)):
            i = int(rng.integers(40))
            n = int(rng.choice([333, 20000, CHUNK, 5 * CHUNK]))
            s_.push(i, caps[i][pos[i]:pos[i] + n])
            pos[i] += n
            got.append(s_.candidates())
        s_.finish()
        got.append(s_.candidates())
    got = np.concatenate(got)
    got = got[np.lexsort((got["sample"], got["stream"]))]
    assert got.tobytes() == exp.tobytes(), (len(got), len(exp))


def test_discover_argument_errors(rx):
    with rx.streams(make_cfgs(3, channel=[1, 2, 37])) as s_:
        with pytest.raises(BtleError) as e:
            s_.set_discover([1, 37, -1])
        assert e.value.code == BTLE_EINVAL
        with pytest.raises(BtleError):
            s_.add_cfg(3)
        with pytest.raises(BtleError):
            s_.remove_cfg(7)


# ---- the monitor --------------------------------------------------------------------------------------------------------
KEYS = ("access_addr", "crc_init", "tracked", "interval", "hop", "t_first", "first_channel", "n_events")


@pytest.mark.parametrize("seg", [4, 9])
def test_monitor_equals_decode_connections(rx, seg):
    cap, _ = connections_capture()
    adv, offline = decode_connections(rx, cap)
    rng = np.random.default_rng(seg)
    with rx.streams(make_cfgs(40, channel=list(range(40))), segment_chunks=seg) as s_:
        mon = ConnectionMonitor(s_)
        pos = [0] * 40
        while any(p < cap.shape[1] for p in pos):
            i = int(rng.integers(40))
            n = int(rng.choice([777, 20000, CHUNK, 3 * CHUNK]))
            mon.push(i, cap[i, pos[i]:pos[i] + n])
            pos[i] += n
        mon.finish()
        live = mon.connections()
    got_adv = mon.adv
    assert got_adv[np.argsort(got_adv["stream"], kind="stable")].tobytes() == adv.tobytes()
    assert len(live) == len(offline) == 3
    for a, b in zip(live, offline):
        assert {k: a.get(k) for k in KEYS} == {k: b.get(k) for k in KEYS}
        want = b["traffic"][b["traffic"]["chunk"] >= a["from_chunk"]]
        _same(a["traffic"], want)
        if not b.get("discovered"):
            assert a["from_chunk"] == 0
            _same(a["traffic"], b["traffic"])
        assert len(want) > 5


# ---- the program: btle_rx_b200 --iq-dir DIR --connections --------------------------------------------------------------
def _pkt_key(e):
    return (e["ts"], e["ch"], e["aa"], e["crc_ok"])


def test_cli_connections_over_files_and_fifos(rx, tmp_path):
    """The program runs the monitor's policy over its poll() loop: its packet lines are the monitor's records in time order
    (every CRC-ok one; those the sinks drop, such as unparsable noise hits, excepted), its track_start lines those
    hop_events() forms for the monitor's connections, and files and paced FIFOs print the same.  -o is refused."""
    import json
    import subprocess
    from btle_b200.hop import hop_events
    from test_stream_sessions_gpu import CLI, _WRITER, _reap
    import sys
    cap, _ = connections_capture()
    seg = 8
    with rx.streams(make_cfgs(40, channel=list(range(40))), segment_chunks=seg) as s_:
        mon = ConnectionMonitor(s_)
        step = seg * CHUNK
        for pos in range(0, cap.shape[1], step):
            for i in range(40):
                mon.push(i, cap[i, pos:pos + step])
        mon.finish()
        conns = mon.connections()
    recs = np.concatenate([mon.adv] + [c["traffic"] for c in conns])
    t = (recs["chunk"].astype(np.int64) * 8192 + recs["n0"]) / 4e6
    want = {("%.6f" % x, int(r["channel"]), "%08x" % int(r["access_addr"]), not r["crc_bad"]) for x, r in zip(t, recs)}
    want_ok = {k for k in want if k[3]}
    norm = lambda e: json.dumps(dict(e, ts="%.6f" % e["ts"]), sort_keys=True)     # the program prints ts with %.6f
    starts = sorted(norm(e) for e in hop_events(conns) if e["event"] == "track_start")
    assert len(starts) >= 1
    d = tmp_path / "files"
    d.mkdir()
    for c in range(40):
        cap[c].tofile(d / f"ch{c:02d}.bin")
    args = ["--connections", "-j", "-Q", "--segment-chunks", str(seg)]
    outs = []
    p = subprocess.run([CLI, "--iq-dir", str(d)] + args, capture_output=True, text=True, timeout=300)
    assert p.returncode == 0, p.stdout + p.stderr
    outs.append(p.stdout)
    f = tmp_path / "fifos"
    f.mkdir()
    procs = []
    for c in range(40):
        os.mkfifo(f / f"ch{c:02d}.bin")
        procs.append(subprocess.Popen([sys.executable, "-c", _WRITER, str(d / f"ch{c:02d}.bin"), str(f / f"ch{c:02d}.bin"), str(c),
                                       str(0.002 * (c % 3))], stderr=subprocess.DEVNULL))
    try:
        q = subprocess.run([CLI, "--iq-dir", str(f)] + args, capture_output=True, text=True, timeout=300)
    finally:
        _reap(procs)
    assert q.returncode == 0, q.stdout + q.stderr
    outs.append(q.stdout)
    for out in outs:
        ev = [json.loads(l) for l in out.splitlines() if l.startswith("{")]
        pk = [e for e in ev if e["t"] == "pkt"]
        got = [("%.6f" % e["ts"], e["ch"], e["aa"], e["crc_ok"]) for e in pk]
        assert [e["ts"] for e in pk] == sorted(e["ts"] for e in pk)
        assert len(set(got)) == len(got) and set(got) <= want and want_ok <= set(got) and len(want_ok) > 30
        hop = [e for e in ev if e["t"] == "hop"]
        assert [e["event"] for e in hop] == ["track_start"] * len(hop)
        assert sorted(norm(e) for e in hop) == starts
    assert outs[0] == outs[1]
    # the text line per connection, and -o refused
    r = subprocess.run([CLI, "--iq-dir", str(d), "--connections", "--segment-chunks", str(seg)], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0 and sum(" Connection AA:" in l for l in r.stdout.splitlines()) == len(conns)
    r = subprocess.run([CLI, "--iq-dir", str(d), "--connections", "-o"], capture_output=True, text=True, timeout=60)
    assert r.returncode != 0 and "cannot be combined with -o" in r.stdout
