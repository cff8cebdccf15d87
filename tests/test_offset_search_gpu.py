"""BTLE_CFG_OFFSET_SEARCH (include/btle_b200.h) on the GPU.  The oracle is the definition: seven calls of the existing
*_offset path at f_c + delta_h, merged by the restatement (offset_search_ref.py).  Every entry point with the flag equals it
byte for byte, record order and directory counts included; a noiseless capture with packets on every grid offset comes
back CRC-ok; the refused combinations are BTLE_EINVAL; a short cap reports a count that, used as cap, returns everything."""
import json
import os
import subprocess

import numpy as np
import pytest
import torch

import mode_ref
import offset_search_ref as osr
import rx_ber_ref as R
from btle_b200 import BtleRx, ber, make_cfgs
from btle_b200._native import (BTLE_EINVAL, BTLE_EOVERFLOW, CFG_CENTRE_HITS, CFG_CORRECT, CFG_LOWPASS, CFG_OFFSET_SEARCH, CFG_RECOVER,
                               CFG_REPORT_REJECTED, CFG_RSSI, CFG_SYMBOL_SPACED, DIR_DTYPE, REC_DTYPE, REC_OFFSET_SEARCH, BtleError)

pytestmark = pytest.mark.gpu

CHUNK = 16384
OS = CFG_OFFSET_SEARCH
MODES = {"quarter": 0, "symbol": CFG_SYMBOL_SPACED | CFG_CENTRE_HITS | CFG_RECOVER,
         "lowpass": CFG_SYMBOL_SPACED | CFG_LOWPASS | CFG_CENTRE_HITS | CFG_RECOVER | CFG_CORRECT}


@pytest.fixture(scope="module")
def rx():
    import __graft_entry__ as ge
    ge.build()
    r = BtleRx(0)
    yield r
    r.close()


def _same(a, b):
    assert a.size == b.size and a.tobytes() == b.tobytes(), (a.size, b.size)


def _capture(snr, cfo_hz, n=24, seed=1, channel=37):
    cfg = ber.rx_ber_cfg(snr, 0.0, cfo_hz, amplitude=64, slot_samples=2048, channel=channel, seed=seed)[0]
    iq, _, _ = R.capture(cfg, 0, n)
    return np.asarray(iq, dtype=np.int8)


def _mixed(n_per=12, seed=3, snr=14.0):
    """captures at five offsets, slot by slot interleaved into one capture (same seed: the same packets, moved)"""
    parts = [_capture(snr, hz, n_per, seed) for hz in (-120e3, -60e3, 0.0, 60e3, 120e3)]
    slot = 2 * 2048
    n = min(p.size for p in parts) // slot
    out = np.empty(n * slot, dtype=np.int8)
    for k in range(n):
        out[k * slot:(k + 1) * slot] = parts[k % 5][k * slot:(k + 1) * slot]
    return out


def _caps(snr):
    """four captures: mixed offsets, a 90-kHz one, a noisier -140-kHz one, an unimpaired one; cut to one length (ragged)"""
    c = [_mixed(snr=snr), _capture(snr - 2, 90e3, 30, 5), _capture(snr - 5, -140e3, 30, 6), _capture(snr - 1, 0.0, 30, 7)]
    n = min(x.size for x in c) - 1234
    return np.ascontiguousarray(np.stack([x[:n] for x in c]))


@pytest.fixture(scope="module")
def caps():
    """SNRs where the symbol-spaced modes lose the off-offset packets without the bank"""
    return _caps(14.0)


@pytest.fixture(scope="module")
def caps_hi():
    """SNRs where the default (quarter-symbol) mode receives packets"""
    return _caps(30.0)


def _oracle_batch(rx, iq2d, cfgs, f_c):
    f = np.broadcast_to(np.asarray(f_c, dtype=np.float32), (iq2d.shape[0],))
    plain = cfgs.copy()
    plain["rssi"] &= ~OS
    per = [rx.rx_batch(iq2d, plain, offset_hz=hz) for hz in osr.hyp_offsets(f)]
    return osr.merge(per, cfgs.size), per


def _oracle_multi(rx, iq2d, cfgs, capture, f_c):
    f = np.broadcast_to(np.asarray(f_c, dtype=np.float32), (iq2d.shape[0],))
    plain = cfgs.copy()
    plain["rssi"] &= ~OS
    per = [rx.rx_multi(iq2d, plain, capture, offset_hz=hz) for hz in osr.hyp_offsets(f)]
    return osr.merge(per, cfgs.size)


@pytest.mark.parametrize("mode", list(MODES))
def test_rx_batch_and_rx(rx, caps, caps_hi, mode):
    caps = caps_hi if mode == "quarter" else caps
    cfgs = make_cfgs(4, channel=37, rssi=CFG_RSSI | CFG_REPORT_REJECTED | MODES[mode] | OS)
    for f_c in (None, [0.0, 30e3, -20e3, 5e3]):
        want, per = _oracle_batch(rx, caps, cfgs, 0.0 if f_c is None else f_c)
        got = rx.rx_batch(caps, cfgs, offset_hz=f_c)
        _same(got, want)
        # hypothesis 0 is the call without the flag; the bank adds CRC-ok packets on the off-offset captures
        ok = lambda r: int(((r["crc_bad"] == 0) & ((r["flags"] & 5) == 0)).sum())
        assert ok(got) >= ok(per[0]) > 0
        if mode != "quarter":
            assert ok(got) > ok(per[0]) and ((got["flags"] & REC_OFFSET_SEARCH) != 0).sum() > 0
    one = rx.rx(caps[1], channel=37, rssi=MODES[mode] | OS)
    _same(one, _oracle_batch(rx, caps[1:2], make_cfgs(1, channel=37, rssi=MODES[mode] | OS), 0.0)[0])


@pytest.mark.parametrize("mode", ["quarter", "lowpass"])
def test_rx_multi(rx, caps, caps_hi, mode):
    """several cfgs per capture (one with another access address, one without RSSI), a capture no cfg names"""
    capture = np.array([0, 0, 0, 2, 3, 3], dtype=np.int32)
    cfgs = make_cfgs(6, channel=37, access_addr=[0x8E89BED6, 0x12345678, 0x8E89BED6, 0x8E89BED6, 0x8E89BED6, 0x8E89BED6],
                     rssi=[CFG_RSSI, 0, CFG_REPORT_REJECTED, CFG_RSSI, 0, CFG_RSSI | CFG_REPORT_REJECTED])
    cfgs["rssi"] |= MODES[mode] | OS
    caps = caps_hi if mode == "quarter" else caps
    for f_c in (None, [10e3, 0.0, -30e3, 45e3]):
        want = _oracle_multi(rx, caps, cfgs, capture, 0.0 if f_c is None else f_c)
        _same(rx.rx_multi(caps, cfgs, capture, offset_hz=f_c), want)


def _device(rx, caps, cfgs, capture, f_c, with_count, cap=None):
    dev = torch.device("cuda", 0)
    n = caps.shape[1]
    pad = np.zeros((caps.shape[0], (n + 15) // 16 * 16), dtype=np.int8)
    pad[:, :n] = caps
    d_iq = torch.from_numpy(pad).to(dev)[:, :n]
    units = rx.units(caps.shape[0], n) if capture is None else rx.multi_units(caps.shape[0], capture, n)
    cap = cfgs.size * (n // CHUNK) * 123 * 7 if cap is None else cap
    d_out = torch.zeros(max(cap, 1) * 64, dtype=torch.uint8, device=dev)
    d_dir = torch.zeros(max(units, 1) * 8, dtype=torch.uint8, device=dev)
    d_count = torch.zeros(1, dtype=torch.int32, device=dev) if with_count else None
    st = torch.cuda.Stream(dev)
    if capture is None:
        rx.rx_device_dir(d_iq, cfgs, d_out[:cap * 64], d_count, d_dir, st.cuda_stream, offset_hz=f_c)
    else:
        rx.rx_multi_device_dir(d_iq, cfgs, capture, d_out[:cap * 64], d_count, d_dir, st.cuda_stream, offset_hz=f_c)
    st.synchronize()
    recs = d_out.cpu().numpy().view(REC_DTYPE)
    d = d_dir.cpu().numpy().view(DIR_DTYPE)[:units]
    cnt = int(d_count.item()) if with_count else int(d["count"].sum())
    return recs, d, cnt, units


@pytest.mark.parametrize("mode", ["quarter", "symbol"])
def test_device_dir(rx, caps, caps_hi, mode):
    """rx_device_dir and rx_multi_device_dir, with and without d_count: the directory has the unflagged call's entries,
    walks in (cfg, chunk, n0) order, and its counts sum to the count"""
    cfgs = make_cfgs(4, channel=37, rssi=CFG_RSSI | CFG_REPORT_REJECTED | MODES[mode] | OS)
    caps = caps_hi if mode == "quarter" else caps
    f_c = [0.0, 30e3, -20e3, 5e3]
    want, _ = _oracle_batch(rx, caps, cfgs, f_c)
    for with_count in (True, False):
        recs, d, cnt, units = _device(rx, caps, cfgs, None, np.asarray(f_c, dtype=np.float32), with_count)
        assert cnt == want.size == int(d["count"].sum())
        _same(rx.gather_ordered(recs, d), want)
        per = units // cfgs.size
        for u, (b, c) in enumerate(d):
            blk = recs[b:b + c]
            assert (blk["stream"] == u // per).all()
            assert (np.diff(blk["chunk"].astype(np.int64) * 8192 + blk["n0"]) > 0).all()
    capture = np.array([0, 0, 1, 3], dtype=np.int32)
    mc = cfgs.copy()
    mc["access_addr"][1] = 0x12345678
    want = _oracle_multi(rx, caps, mc, capture, 0.0)
    for with_count in (True, False):
        recs, d, cnt, units = _device(rx, caps, mc, capture, None, with_count)
        assert cnt == want.size == int(d["count"].sum()) and units == rx.multi_units(4, capture, caps.shape[1])
        _same(rx.gather_ordered(recs, d), want)


def test_grid_offsets_noiseless(rx):
    """a noiseless capture with packets on every grid offset from -150 to +150 kHz: every packet CRC-ok with the flag"""
    from btle_b200 import synth
    offs = osr.HYP_HZ
    part = 8 * CHUNK
    segs, n_pkts = [], 0
    for k, hz in enumerate(offs):
        iq, truth = synth.make_adv_stream(part, seed=40 + k, channel=37, slot_samples=3000, corrupt_every=0)
        segs.append(mode_ref.rotate(np.asarray(iq.cpu() if hasattr(iq, "cpu") else iq, dtype=np.int8), hz))
    iq = np.concatenate(segs)
    for mode in ("quarter", "lowpass"):
        plain = rx.rx(iq, channel=37, rssi=MODES[mode] & (CFG_SYMBOL_SPACED | CFG_LOWPASS))
        got = rx.rx(iq, channel=37, rssi=(MODES[mode] & (CFG_SYMBOL_SPACED | CFG_LOWPASS)) | OS)
        ok = got[got["crc_bad"] == 0]
        # every packet found by hypothesis 0 (the 0-kHz segment) and by the bank on the others, none failing
        assert (got["crc_bad"] == 0).all(), mode
        per_seg = np.bincount((ok["chunk"] // 8).astype(np.int64), minlength=len(offs))
        assert (per_seg >= per_seg[0] - 1).all() and per_seg[0] > 10, (mode, per_seg)
        assert ok.size >= (plain["crc_bad"] == 0).sum()


def test_refused(rx, caps):
    def einval(f, *a, **k):
        with pytest.raises(BtleError) as e:
            f(*a, **k)
        assert e.value.code == BTLE_EINVAL
    mixed = make_cfgs(4, channel=37, offset_search=[1, 0, 1, 1])
    einval(rx.rx_batch, caps, mixed)
    einval(rx.rx, caps[0], channel=37, raw=1, offset_search=1)
    einval(rx.rx, caps[0], channel=37, offset_search=1, offset_hz=350001.0)
    assert rx.rx(caps[0], channel=37, offset_search=1, offset_hz=350000.0).dtype == REC_DTYPE
    with rx.streams(make_cfgs(2, channel=37, offset_search=1)) as s:
        einval(s.set_cfg, 0, offset_search=0)
        einval(s.add_cfg, 1, access_addr=0x12345678, offset_search=0)
        einval(s.set_offset, 0, -360e3)
        s.set_offset(0, -300e3)
    with rx.streams(make_cfgs(2, channel=37)) as s:
        einval(s.set_cfg, 0, offset_search=1)
        einval(s.add_cfg, 1, offset_search=1)


def test_overflow_second_call(rx, caps):
    cfgs = make_cfgs(4, channel=37, rssi=CFG_REPORT_REJECTED | OS)
    want, _ = _oracle_batch(rx, caps, cfgs, 0.0)
    import ctypes
    for cap in (1, want.size // 2, want.size):
        out = np.zeros(max(cap, 1), dtype=REC_DTYPE)
        n = ctypes.c_size_t(0)
        rc = rx._L.btle_b200_rx_batch(rx._h, caps.ctypes.data, 4, caps.shape[1], caps.shape[1], cfgs.ctypes.data, out.ctypes.data, cap,
                                      ctypes.byref(n))
        if rc == BTLE_EOVERFLOW:
            assert n.value > cap
            _same(rx.rx_batch(caps, cfgs, cap=n.value), want)
        else:
            assert rc == 0 and n.value == want.size
            _same(out[:n.value], want)
    _same(rx.rx_batch(caps, cfgs), want)                   # the default capacity, grown once


def test_dense_chunk_within_bound(rx):
    """many CRC-ok packets at different offsets in every chunk (short slots, each slot at its own grid offset, -v with a
    mask that matches everywhere): within BTLE_MAX_MERGED_RECS_PER_CHUNK and equal to the oracle"""
    from btle_b200 import synth
    iq, _ = synth.make_adv_stream(6 * CHUNK, seed=77, channel=37, slot_samples=420, corrupt_every=0)
    iq = np.asarray(iq.cpu() if hasattr(iq, "cpu") else iq, dtype=np.int8)
    slot = 2 * 420
    parts = [mode_ref.rotate(iq, hz) for hz in osr.HYP_HZ]
    x = np.concatenate([parts[k % 7][k * slot:(k + 1) * slot] for k in range(iq.size // slot)])
    x = x[:x.size // CHUNK * CHUNK]
    for mask in (0xFFFFFFFF, 0x0000FFFF):
        cfgs = make_cfgs(1, channel=37, access_mask=mask, rssi=CFG_REPORT_REJECTED | OS)
        want, _ = _oracle_batch(rx, x[None, :], cfgs, 0.0)
        got = rx.rx_batch(x[None, :], cfgs)
        _same(got, want)
        assert np.bincount(got["chunk"]).max() <= osr.MAX_MERGED_RECS_PER_CHUNK
        assert ((got["flags"] & REC_OFFSET_SEARCH) != 0).sum() > 0


def test_streams_session(rx, caps):
    """a session with the flag, set_offset and a backfilled add_cfg equals rx_batch_offset / rx_multi_offset with the flag"""
    cfgs = make_cfgs(4, channel=37, rssi=CFG_RSSI | CFG_REPORT_REJECTED | OS | CFG_SYMBOL_SPACED)
    f_c = np.array([0.0, 25e3, -40e3, 0.0], dtype=np.float32)
    n = caps.shape[1] // CHUNK * CHUNK
    with rx.streams(cfgs, segment_chunks=16) as s:
        for i in range(4):
            s.set_offset(i, float(f_c[i]))
        out = []
        step = 5 * CHUNK + 77
        for o in range(0, n, step):
            for i in range(4):
                out.append(s.push(i, caps[i, o:min(o + step, n)]))
            if o == 0:
                j, _ = s.add_cfg(2, access_addr=0x12345678)
        out.append(s.finish())
    got = np.concatenate(out)
    want = _oracle_batch(rx, caps[:, :n], cfgs, f_c)[0]
    _same(np.sort(got[got["stream"] < 4], order=["stream", "chunk", "n0"]), want)
    mc = make_cfgs(1, channel=37, access_addr=0x12345678, rssi=int(cfgs["rssi"][0]))
    extra = _oracle_multi(rx, caps[:, :n], mc, np.array([2], np.int32), f_c)
    e = got[got["stream"] == j].copy()
    e["stream"] = 0
    _same(e, extra)


def test_rx_ber(rx):
    """rx_ber_run with the flag at 100 kHz: the bank receives what the unflagged receiver loses, and the merged directory
    scores no extra or wrong records"""
    kw = dict(cfo_hz=100e3, symbol_spaced=True, centre_hits=True, recover=True, lowpass=True)
    plain = ber.rx_ber_point(rx, 12.0, 2000, **kw)
    bank = ber.rx_ber_point(rx, 12.0, 2000, offset_search=True, **kw)
    assert bank["per"] < 0.5 * plain["per"] and bank["per"] < 0.2, (plain["per"], bank["per"])
    assert bank["crc_ok_wrong"] == 0
    corr = ber.rx_ber_point(rx, 12.0, 2000, offset_hz=20e3, offset_search=True, **kw)   # the *_offset path, centred at 20 kHz
    assert corr["per"] < 0.2 and corr["crc_ok_wrong"] == 0, corr["per"]


def test_decode_connections_flag(rx, caps):
    from btle_b200 import hop
    c = np.zeros((40, caps.shape[1]), dtype=np.int8)
    c[37] = caps[0]
    adv, _ = hop.decode_connections(rx, c, discover=False, offset_search=True)
    want, _ = _oracle_batch(rx, c[37:40], make_cfgs(3, channel=[37, 38, 39], offset_search=1), 0.0)
    want["stream"] += 37
    _same(adv, want)


def test_cli_offset_search(tmp_path, rx, caps):
    """--offset-search text and NDJSON equal the library's records; --offset HZ sets the centre; -r and --iq-bin16 refused"""
    cli = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "btle_b200", "btle_rx_b200")
    f = tmp_path / "cap.bin"
    caps[0].tofile(f)
    for off in (None, 20000.0):
        want = rx.rx(caps[0], channel=37, rssi=1, offset_search=1, offset_hz=off)
        extra = [] if off is None else ["--offset", str(int(off))]
        p = subprocess.run([cli, "-i", str(f), "-c", "37", "-j", "-Q", "-R", "--offset-search", *extra], capture_output=True, text=True,
                           check=True)
        lines = [json.loads(s) for s in p.stdout.splitlines() if '"t":"pkt"' in s]
        assert len(lines) == want.size and want.size > 0
        for r, l in zip(want, lines):
            assert l["crc_ok"] == (r["crc_bad"] == 0)
            assert bytes.fromhex(l["payload_hex"]) == bytes(r["bytes"][2:2 + l["plen"]])
            assert l.get("offset_search", False) == bool(r["flags"] & REC_OFFSET_SEARCH)
        txt = subprocess.run([cli, "-i", str(f), "-c", "37", "--offset-search", *extra], capture_output=True, text=True, check=True).stdout
        assert txt.count("CRC0") == int((want["crc_bad"] == 0).sum())
    auto = subprocess.run([cli, "-i", str(f), "-c", "37", "--offset-search", "--offset", "auto", "-j", "-Q"], capture_output=True, text=True,
                          check=True)
    assert sum('"t":"pkt"' in s for s in auto.stdout.splitlines()) > 0
    for args in (["-i", str(f), "-r", "--offset-search"], ["--iq-bin16", str(f), "--offset-search"]):
        bad = subprocess.run([cli, *args], capture_output=True, text=True)
        assert bad.returncode != 0 and "--offset-search cannot be combined" in bad.stdout
