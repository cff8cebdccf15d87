"""BTLE_CFG_LOWPASS (include/btle_b200.h) on the GPU: every receive path in the low-pass mode returns what the restatement
(tests/lowpass_ref.py) returns — goldens, fuzz, a 40-capture batch, rx_multi with 8 cfgs per capture, rotated launches,
BTLE_CFG_RECOVER / CENTRE_HITS / CORRECT, -v with mask 0, raw mode and RSSI, a streamed capture and the CLI; rx_ber_run's
batches count what one long capture counts; the refused combinations are BTLE_EINVAL."""
import os
import subprocess

import numpy as np
import pytest
import torch

import golden_util
import lowpass_ref
import mode_ref
import multi_fuzz
import rx_ber_ref as R
from btle_b200 import BtleRx, ber, make_cfgs
from btle_b200._native import (BTLE_EINVAL, CFG_CENTRE_HITS, CFG_CORRECT, CFG_LOWPASS, CFG_RECOVER, CFG_RSSI, CFG_SYMBOL_SPACED,
                               DIR_DTYPE, REC_DTYPE, RX_BER_RESULT_DTYPE, BtleError)

pytestmark = pytest.mark.gpu

CHUNK = 16384
DATA = dict(channel=9, access_addr=0x60850A27, crc_init=0xA77B2E)
ADV = dict(channel=37, access_addr=0x8E89BED6, crc_init=0x555555)
CLI = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "btle_b200", "btle_rx_b200")
LP = CFG_SYMBOL_SPACED | CFG_LOWPASS
REPAIR = CFG_RECOVER | CFG_CENTRE_HITS | CFG_CORRECT


@pytest.fixture(scope="module")
def rx():
    import __graft_entry__ as ge
    ge.build()
    r = BtleRx(0)
    yield r
    r.close()


def _capture(snr, channel, n=24, seed=1, cfo_hz=0.0):
    base = ADV if channel >= 37 else DATA
    cfg = ber.rx_ber_cfg(snr, 0.0, cfo_hz, amplitude=64, slot_samples=2048, channel=channel, seed=seed, crc_init=base["crc_init"],
                         access_addr=base["access_addr"])[0]
    iq, _, _ = R.capture(cfg, 0, n)
    return iq, dict(base, channel=channel)


def _same(a, b):
    assert a.size == b.size and a.tobytes() == b.tobytes(), (a.size, b.size)


def _expected(iq, cfg, rssi=0, raw=0, stream=0, hz=0.0, access_mask=0xFFFFFFFF):
    return lowpass_ref.rx_stream(iq, hz, rssi=rssi, raw=raw, stream=stream, access_mask=access_mask, **cfg)


def test_goldens(rx):
    """every golden capture, with RSSI and with the repair flags"""
    for name in golden_util.cases():
        z, cfg = golden_util.load(name)
        kw = golden_util.rx_cfg(cfg)
        iq = np.asarray(z["iq"], dtype=np.int8)
        for extra in (CFG_RSSI, CFG_RSSI | REPAIR):
            rssi = kw.get("rssi", 0) | extra
            c = {k: v for k, v in kw.items() if k != "rssi"}
            _same(rx.rx(iq, rssi=rssi, symbol_spaced=1, lowpass=1, **c), lowpass_ref.rx_stream(iq, 0.0, rssi=rssi, **c))


@pytest.mark.parametrize("snr", [7.0, 10.0, 16.0])
def test_rx_flags(rx, snr):
    """noisy captures with every repair flag combination, RSSI and -v"""
    for ch in (37, 9):
        iq, cfg = _capture(snr, ch, n=40, seed=int(snr) + ch)
        for extra in (0, 1 | 2, CFG_RECOVER, CFG_CENTRE_HITS | CFG_CORRECT, REPAIR | 1 | 2):
            _same(rx.rx(iq, rssi=extra, symbol_spaced=1, lowpass=1, **cfg), _expected(iq, cfg, rssi=extra))


@pytest.fixture(scope="module")
def caps40():
    caps = [_capture(7 + k % 9, 37 if k % 2 == 0 else 9, n=16, seed=900 + k) for k in range(40)]
    n = min(c[0].size for c in caps) - 1234                                    # ragged
    return np.stack([c[0][:n] for c in caps]), [c[1] for c in caps]


def test_batch_40_multi_and_device(rx, caps40):
    """rx_batch over 40 captures, rx_multi with 8 cfgs per capture, and the device form"""
    iq, cc = caps40
    flags = [(k % 4) | (REPAIR if k % 3 == 0 else 0) for k in range(40)]
    cfgs = np.concatenate([make_cfgs(1, rssi=flags[k], symbol_spaced=1, lowpass=1, **c) for k, c in enumerate(cc)])
    got = rx.rx_batch(iq, cfgs)
    assert got.size > 100
    _same(got, np.concatenate([_expected(iq[k], cc[k], rssi=flags[k], stream=k) for k in range(40)]))
    cap = np.repeat(np.arange(3), 8).astype(np.int32)
    mi = iq[0:3]
    mc = np.concatenate([make_cfgs(8, symbol_spaced=1, lowpass=1, **cc[c]) for c in range(3)])
    mc["raw"][3::8] = 1
    mc["rssi"][2::8] |= 2 | CFG_RECOVER
    mc["rssi"][4::8] |= 1 | CFG_CENTRE_HITS
    mc["access_mask"][5::8] = 0xFFFFFF00
    mc["access_mask"][6::8] = 0
    mc["rssi"][6::8] |= 2
    mc["rssi"][7::8] |= REPAIR
    _same(rx.rx_multi(mi, mc, cap), lowpass_ref.rx_multi(mi, mc, cap))
    iq = np.ascontiguousarray(iq[:, :iq.shape[1] // 16 * 16])
    d_iq = torch.from_numpy(iq).cuda()
    want = rx.rx_batch(iq, cfgs)
    d_out = torch.empty(want.size * 64 + 64 * 64, dtype=torch.uint8, device="cuda")
    d_dir = torch.empty(rx.units(40, iq.shape[1]) * 8, dtype=torch.uint8, device="cuda")
    rx.rx_device_dir(d_iq, cfgs, d_out, None, d_dir, torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    _same(rx.gather_ordered(d_out.cpu().numpy().view(REC_DTYPE), d_dir.cpu().numpy().view(DIR_DTYPE)), want)


@pytest.mark.parametrize("rot", [0, 1])
def test_multi_fuzz(rx, rot):
    """multi_fuzz launches (ragged ends, degenerate masks, several cfgs per capture), unrotated and rotated"""
    rng = np.random.default_rng(131 + rot)
    for _ in range(3):
        iq, cfgs, capture, offsets = multi_fuzz.draw_mode(rng, (rot, 1), max_captures=6, max_chunks=10)
        cfgs["rssi"] |= CFG_LOWPASS
        cfgs["rssi"][::3] |= CFG_RECOVER
        cfgs["rssi"][::4] |= CFG_CORRECT | CFG_CENTRE_HITS
        _same(rx.rx_multi(iq, cfgs, capture, offset_hz=offsets), lowpass_ref.rx_multi(iq, cfgs, capture, offsets))


@pytest.mark.parametrize("hz", [0.0, 100e3, -150e3, 300e3])
def test_offset_entry_points(rx, hz):
    """rx_batch_offset and rx_device_dir with offset_hz, with the repair flags (whose bits are rotated too)"""
    caps = [_capture(9.0, ch, n=20, seed=int(abs(hz)) % 89 + ch, cfo_hz=hz) for ch in (37, 9)]
    n = min(c[0].size for c in caps) // 16 * 16
    iq = np.stack([c[0][:n] for c in caps])
    cc = [c[1] for c in caps]
    for rssi in (0, 1 | 2, REPAIR):
        cfgs = np.concatenate([make_cfgs(1, rssi=rssi, symbol_spaced=1, lowpass=1, **c) for c in cc])
        want = np.concatenate([_expected(iq[k], cc[k], rssi=rssi, stream=k, hz=hz) for k in range(2)])
        _same(rx.rx_batch(iq, cfgs, offset_hz=hz), want)
        d_iq = torch.from_numpy(iq).cuda()
        d_out = torch.empty(want.size * 64 + 64 * 64, dtype=torch.uint8, device="cuda")
        d_dir = torch.empty(rx.units(2, n) * 8, dtype=torch.uint8, device="cuda")
        rx.rx_device_dir(d_iq, cfgs, d_out, None, d_dir, torch.cuda.current_stream().cuda_stream, offset_hz=hz)
        torch.cuda.synchronize()
        _same(rx.gather_ordered(d_out.cpu().numpy().view(REC_DTYPE), d_dir.cpu().numpy().view(DIR_DTYPE)), want)


def test_report_rejected_mask0_raw(rx):
    """mask 0 with -v on channel 38 over a capture whose chunks start with zeros (more hits than a chunk's hit row: the late
    rows), with recovery; raw mode with RSSI"""
    iq, cfg = _capture(10.0, 38, n=24, seed=9)
    s = iq.reshape(-1, 2).copy()
    for c in range(s.shape[0] // 8192):
        s[8192 * c: 8192 * c + 4600] = 0
    iq = s.reshape(-1)
    for extra in (0, CFG_RECOVER | CFG_CORRECT):
        exp = _expected(iq, cfg, rssi=2 | 1 | extra, access_mask=0)
        assert max(np.bincount(exp["chunk"])) > 68
        _same(rx.rx(iq, rssi=2 | 1 | extra, access_mask=0, symbol_spaced=1, lowpass=1, **cfg), exp)
    _same(rx.rx(iq, raw=1, rssi=1, symbol_spaced=1, lowpass=1, **cfg), _expected(iq, cfg, rssi=1, raw=1))


def test_stream_segments(rx):
    """a capture streamed in odd pieces through segment sets (each set decoded behind the previous set's lead) equals the
    whole capture and the restatement, with recovery reading filtered samples across set boundaries"""
    a, ca = _capture(9.0, 37, n=60, seed=71)
    for seg in (1, 3):
        parts = []
        with rx.stream(segment_chunks=seg, rssi=1 | CFG_RECOVER, symbol_spaced=1, lowpass=1, **ca) as s_:
            pos, rng = 0, np.random.default_rng(5 + seg)
            while pos < a.size:
                k = int(rng.choice([1, 777, 5000, CHUNK + 3, 3 * CHUNK + 1]))
                parts.append(s_.push(a[pos:pos + k]))
                pos += k
            parts.append(s_.finish())
        _same(np.concatenate(parts), _expected(a, ca, rssi=1 | CFG_RECOVER))


def test_refused(rx, caps40):
    """mixed cfgs in one launch, the flag without BTLE_CFG_SYMBOL_SPACED, a session set_cfg / add_cfg with the other value
    and rx_ber_run with the flag alone are BTLE_EINVAL; the context stays usable"""
    iq, cc = caps40
    mixed = np.concatenate([make_cfgs(1, symbol_spaced=1, lowpass=k % 2, **c) for k, c in enumerate(cc[:4])])
    alone = np.concatenate([make_cfgs(1, lowpass=1, **c) for c in cc[:4]])
    for cfgs in (mixed, alone):
        for call in (lambda: rx.rx_batch(iq[:4], cfgs), lambda: rx.rx_multi(iq[:2], cfgs[:2], np.array([0, 0], np.int32)),
                     lambda: rx.rx_batch(iq[:4], cfgs, offset_hz=0.0)):
            with pytest.raises(BtleError) as e:
                call()
            assert e.value.code == BTLE_EINVAL
            assert b"LOWPASS" in rx._L.btle_b200_last_error(rx._h)
        d_iq = torch.from_numpy(np.ascontiguousarray(iq[:4])).cuda()
        d_out = torch.empty(64 * 4096, dtype=torch.uint8, device="cuda")
        d_dir = torch.empty(rx.units(4, iq.shape[1]) * 8, dtype=torch.uint8, device="cuda")
        with pytest.raises(BtleError) as e:
            rx.rx_device_dir(d_iq, cfgs, d_out, None, d_dir, torch.cuda.current_stream().cuda_stream)
        assert e.value.code == BTLE_EINVAL
    for opened, other in ((mixed[1:2], {"lowpass": 0}), (mixed[0:1], {"lowpass": 1})):
        with rx.streams(opened, segment_chunks=2) as s_:
            for call in (lambda: s_.set_cfg(0, **other), lambda: s_.add_cfg(0, None, **other)):
                with pytest.raises(BtleError) as e:
                    call()
                assert e.value.code == BTLE_EINVAL
            s_.set_cfg(0, rssi=int(opened["rssi"][0]) | 1)                       # the session's own mode is still accepted
    with pytest.raises(BtleError):
        rx.streams(mixed[:2], segment_chunks=2)
    with pytest.raises(BtleError):
        rx.streams(alone[:1], segment_chunks=2)
    for bad in (CFG_LOWPASS, CFG_LOWPASS | CFG_RECOVER, CFG_LOWPASS | 8, LP | 32):
        run = ber.rx_ber_cfg(20.0, seed=1)
        run["flags"] = bad
        assert rx._L.btle_b200_rx_ber_run(rx._h, run.ctypes.data, 16, np.zeros(1, dtype=RX_BER_RESULT_DTYPE).ctypes.data) == BTLE_EINVAL
    ok = np.concatenate([make_cfgs(1, symbol_spaced=1, lowpass=1, **c) for c in cc[:4]])
    _same(rx.rx_batch(iq[:4], ok), np.concatenate([_expected(iq[k], cc[k], stream=k) for k in range(4)]))


def test_rx_ber_run_batches_and_synth_device(rx):
    """btle_b200_rx_ber_run over 40000 packets (two batches or more) counts what one long capture, synthesised, decoded and
    scored in one piece, counts; the receiver's records on an rx_ber_synth_device capture fetched to the host are the
    restatement's; the filter removes packet errors at 8 dB"""
    n = 40000
    for flags in (LP | CFG_CENTRE_HITS, LP | REPAIR):
        run = ber.rx_ber_cfg(8.0, slot_samples=2048, seed=8)
        run["flags"] = flags
        res = np.zeros(1, dtype=RX_BER_RESULT_DTYPE)
        rx._check(rx._L.btle_b200_rx_ber_run(rx._h, run.ctypes.data, n, res.ctypes.data))
        assert rx.last_launches >= 6                                           # two batches or more (synth, receive, score each)
        ni = ((n * 2048 + 8191) // 8192) * CHUNK
        d_iq = torch.empty(ni, dtype=torch.int8, device="cuda")
        d_t = torch.empty(n * 64, dtype=torch.uint8, device="cuda")
        rx._check(rx._L.btle_b200_rx_ber_synth_device(rx._h, run.ctypes.data, 0, n, d_iq.data_ptr(), d_t.data_ptr(), None))
        scfg = make_cfgs(1, rssi=2 | flags, **ADV)
        units = rx.units(1, ni)
        d_out = torch.empty(ni // CHUNK * 123 * 64, dtype=torch.uint8, device="cuda")
        d_dir = torch.empty(units * 8, dtype=torch.uint8, device="cuda")
        rx.rx_device_dir(d_iq.view(1, -1), scfg, d_out, None, d_dir, 0)
        d_res = torch.zeros(RX_BER_RESULT_DTYPE.itemsize, dtype=torch.uint8, device="cuda")
        rx._check(rx._L.btle_b200_rx_ber_score_device(rx._h, d_t.data_ptr(), n, d_out.data_ptr(), ni // CHUNK * 123, d_dir.data_ptr(),
                                                      units, d_res.data_ptr(), None))
        torch.cuda.synchronize()
        one = d_res.cpu().numpy().view(RX_BER_RESULT_DTYPE)
        for k in ("packets", "pkt_err", "bit_err", "aa_miss", "len_reject", "crc_ok_wrong", "extra_recs", "extra_crc_ok"):
            assert int(res[0][k]) == int(one[0][k]), (flags, k)
        sym = ber.rx_ber_cfg(8.0, slot_samples=2048, seed=8)
        sym["flags"] = flags & ~CFG_LOWPASS
        res_s = np.zeros(1, dtype=RX_BER_RESULT_DTYPE)
        rx._check(rx._L.btle_b200_rx_ber_run(rx._h, sym.ctypes.data, n, res_s.ctypes.data))
        assert int(res[0]["pkt_err"]) < int(res_s[0]["pkt_err"]), (flags, int(res[0]["pkt_err"]), int(res_s[0]["pkt_err"]))
    m = 400
    mi = ((m * 2048 + 8191) // 8192) * CHUNK
    d_iq = torch.empty(mi, dtype=torch.int8, device="cuda")
    d_t = torch.empty(m * 64, dtype=torch.uint8, device="cuda")
    run = ber.rx_ber_cfg(8.0, slot_samples=2048, seed=4)
    rx._check(rx._L.btle_b200_rx_ber_synth_device(rx._h, run.ctypes.data, 0, m, d_iq.data_ptr(), d_t.data_ptr(), None))
    torch.cuda.synchronize()
    iq = d_iq.cpu().numpy()
    for rssi in (2 | CFG_CENTRE_HITS, 2 | REPAIR):
        _same(rx.rx(iq, rssi=rssi, symbol_spaced=1, lowpass=1, **ADV), _expected(iq, ADV, rssi=rssi))


def test_decode_connections(rx):
    """hop.decode_connections(symbol_spaced=True, lowpass=True): the advertising records are the restatement's"""
    from btle_b200 import hop
    caps = np.zeros((40, 24 * 2048 * 2 // CHUNK * CHUNK + CHUNK), dtype=np.int8)
    for ch in (37, 38, 39):
        iq, _ = _capture(9.0, ch, n=24, seed=ch)
        caps[ch, :min(iq.size, caps.shape[1])] = iq[:caps.shape[1]]
    adv, _ = hop.decode_connections(rx, caps, discover=False, symbol_spaced=True, lowpass=True)
    want = np.concatenate([_expected(caps[ch], dict(ADV, channel=ch), stream=ch - 37) for ch in (37, 38, 39)])
    want["stream"] += 37
    _same(adv, want)


def test_cli_lowpass(tmp_path, rx):
    iq, cfg = _capture(9.0, 37, n=200, seed=13)
    f = tmp_path / "cap.bin"
    iq.tofile(f)
    want = rx.rx(iq, rssi=1, symbol_spaced=1, lowpass=1, **cfg)
    _same(want, _expected(iq, cfg, rssi=1))
    import json
    p = subprocess.run([CLI, "-i", str(f), "-c", "37", "-j", "-Q", "-R", "--symbol-spaced", "--lowpass"], capture_output=True, text=True,
                       check=True)
    lines = [json.loads(s) for s in p.stdout.splitlines() if '"t":"pkt"' in s]
    assert len(lines) == want.size
    for r, l in zip(want, lines):
        assert l["crc_ok"] == (r["crc_bad"] == 0)
        assert bytes.fromhex(l["payload_hex"]) == bytes(r["bytes"][2:2 + l["plen"]])
    txt = subprocess.run([CLI, "-i", str(f), "-c", "37", "--symbol-spaced", "--lowpass"], capture_output=True, text=True, check=True).stdout
    sym = subprocess.run([CLI, "-i", str(f), "-c", "37", "--symbol-spaced"], capture_output=True, text=True, check=True).stdout
    assert txt.count("CRC0") == int((want["crc_bad"] == 0).sum()) > sym.count("CRC0")
    auto = subprocess.run([CLI, "-i", str(f), "-c", "37", "--symbol-spaced", "--lowpass", "--offset", "auto", "-j", "-Q"], capture_output=True,
                          text=True, check=True)
    assert sum('"t":"pkt"' in s for s in auto.stdout.splitlines()) > 0
    for args in (["-i", str(f), "--lowpass"], ["--iq-bin16", str(f), "--lowpass"]):
        bad = subprocess.run([CLI, *args], capture_output=True, text=True)
        assert bad.returncode != 0 and "--lowpass needs --symbol-spaced" in bad.stdout
