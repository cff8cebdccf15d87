"""BTLE_CFG_CORRECT (include/btle_b200.h) on the GPU: every receive path with the flag returns what the restatement
(tests/correct_ref.py) returns, in every (ROT, SYM) mode, with the flag mixed per cfg and combined with BTLE_CFG_RECOVER
and BTLE_CFG_CENTRE_HITS; streamed and batched forms equal the whole capture; the CLI's --correct; hop.decode_connections;
and btle_b200_rx_ber_run with the flag."""
import json
import os
import subprocess

import numpy as np
import pytest
import torch

import correct_ref
import mode_ref
import multi_fuzz
import rx_ber_ref as R
from btle_b200 import BtleRx, ber, make_cfgs
from btle_b200._native import (BTLE_EINVAL, CFG_CENTRE_HITS, CFG_CORRECT, CFG_RECOVER, CFG_SYMBOL_SPACED, DIR_DTYPE, REC_CORRECTED,
                               REC_DTYPE, RX_BER_RESULT_DTYPE)

pytestmark = pytest.mark.gpu

CHUNK = 16384
DATA = dict(channel=9, access_addr=0x60850A27, crc_init=0xA77B2E)
ADV = dict(channel=37, access_addr=0x8E89BED6, crc_init=0x555555)
CLI = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "btle_b200", "btle_rx_b200")
CORRECT, CENTRE = CFG_CORRECT, CFG_CENTRE_HITS


@pytest.fixture(scope="module")
def rx():
    import __graft_entry__ as ge
    ge.build()
    r = BtleRx(0)
    yield r
    r.close()


def _capture(snr, channel, n=24, seed=1, cfo_hz=0.0, ppm=0.0):
    base = ADV if channel >= 37 else DATA
    cfg = ber.rx_ber_cfg(snr, ppm, cfo_hz, amplitude=64, slot_samples=2048, channel=channel, seed=seed, crc_init=base["crc_init"],
                         access_addr=base["access_addr"])[0]
    iq, truth, _ = R.capture(cfg, 0, n)
    return iq, dict(base, channel=channel)


def _same(a, b):
    assert a.size == b.size and a.tobytes() == b.tobytes(), (a.size, b.size)


def _expected(iq, cfg, rssi=0, raw=0, stream=0, hz=0.0, sym=False, access_mask=0xFFFFFFFF):
    return correct_ref.rx_stream(iq, hz, sym, rssi=rssi, raw=raw, stream=stream, access_mask=access_mask, **cfg)


def _by_cfg(iq2d, cfgs, capture, offsets=None):
    out = []
    for j, c in enumerate(np.asarray(capture).reshape(-1)):
        f = cfgs[j]
        out.append(correct_ref.rx_stream(iq2d[c], 0.0 if offsets is None else float(np.float32(offsets[c])),
                                         bool(f["rssi"] & CFG_SYMBOL_SPACED), *mode_ref._fields(f, j)[:-1], stream=j))
    return np.concatenate(out) if out else np.zeros(0, dtype=REC_DTYPE)


def _corrected(recs):
    return int(((recs["flags"] & REC_CORRECTED) != 0).sum())


@pytest.mark.parametrize("sym", [0, 1])
def test_rx(rx, sym):
    """rx with the flag, alone and with RSSI, recovery and centre hits, at SNRs where CRC failures are common"""
    n_corr = 0
    for snr, ch in ((11.0, 37), (13.0, 9), (20.0, 37)) if sym else ((18.0, 37), (20.0, 9), (24.0, 37)):
        iq, cfg = _capture(snr, ch, n=40, seed=int(snr) + ch)
        for extra in (0, 1, CFG_RECOVER, CENTRE, CFG_RECOVER | CENTRE | 2):
            got = rx.rx(iq, rssi=extra | CORRECT, symbol_spaced=sym, **cfg)
            _same(got, _expected(iq, cfg, rssi=extra | CORRECT, sym=bool(sym)))
            n_corr += _corrected(got)
    assert n_corr > 10


@pytest.fixture(scope="module")
def caps40():
    caps = [_capture(12 + k % 9, 37 if k % 2 == 0 else 9, n=16, seed=700 + k) for k in range(40)]
    n = min(c[0].size for c in caps) - 1234                                    # ragged
    return np.stack([c[0][:n] for c in caps]), [c[1] for c in caps]


@pytest.mark.parametrize("sym", [0, 1])
def test_batch_40_mixed_multi_and_device(rx, caps40, sym):
    """rx_batch over 40 captures with the flag on most captures and RSSI, -v, recovery and centre hits in every
    combination; rx_multi (the 8-cfg kernel) with the flag on and off for cfgs of one capture; the device form"""
    iq, cc = caps40
    flags = [(k % 8) | (CENTRE if k % 5 == 0 else 0) | (CORRECT if (k // 8) % 2 == 0 or k % 3 == 0 else 0) for k in range(40)]
    assert {f & 7 for f in flags if f & CORRECT} == set(range(8))
    cfgs = np.concatenate([make_cfgs(1, rssi=flags[k], symbol_spaced=sym, **c) for k, c in enumerate(cc)])
    got = rx.rx_batch(iq, cfgs)
    assert got.size > 100 and _corrected(got) > 0
    _same(got, np.concatenate([_expected(iq[k], cc[k], rssi=flags[k], stream=k, sym=bool(sym)) for k in range(40)]))
    cap = np.repeat(np.arange(3), 8).astype(np.int32)
    first = 6 if sym == 0 else 0                                              # 18-20 dB / 12-14 dB: CRC failures in either mode
    mi = iq[first:first + 3]
    mc = np.concatenate([make_cfgs(8, symbol_spaced=sym, **cc[c]) for c in range(first, first + 3)])
    mc["rssi"][0::2] |= CORRECT                                               # cfgs 0 and 1 of a capture: the same cfg, on / off
    mc["raw"][3::8] = 1
    mc["rssi"][2::8] |= 2 | CFG_RECOVER
    mc["rssi"][4::8] |= 1 | CENTRE
    mc["access_mask"][5::8] = 0xFFFFFF00
    mc["access_mask"][6::8] = 0
    mc["rssi"][6::8] |= 2
    mc["rssi"][7::8] |= CORRECT | CFG_RECOVER | CENTRE
    multi = rx.rx_multi(mi, mc, cap)
    _same(multi, _by_cfg(mi, mc, cap))
    assert _corrected(multi) > 0
    iq = np.ascontiguousarray(iq[:, :iq.shape[1] // 16 * 16])
    d_iq = torch.from_numpy(iq).cuda()
    want = rx.rx_batch(iq, cfgs)
    d_out = torch.empty(want.size * 64 + 64 * 64, dtype=torch.uint8, device="cuda")
    d_dir = torch.empty(rx.units(40, iq.shape[1]) * 8, dtype=torch.uint8, device="cuda")
    rx.rx_device_dir(d_iq, cfgs, d_out, None, d_dir, torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    _same(rx.gather_ordered(d_out.cpu().numpy().view(REC_DTYPE), d_dir.cpu().numpy().view(DIR_DTYPE)), want)


@pytest.mark.parametrize("mode", mode_ref.MODES, ids=mode_ref.mode_id)
def test_multi_fuzz_every_mode(rx, mode):
    """multi_fuzz launches in every (ROT, SYM) mode, the flag on every other cfg"""
    rng = np.random.default_rng(91 + 2 * mode[0] + mode[1])
    for _ in range(2):
        iq, cfgs, capture, offsets = multi_fuzz.draw_mode(rng, mode, max_captures=6, max_chunks=10)
        cfgs["rssi"][::2] |= CORRECT
        cfgs["rssi"][::3] |= CFG_RECOVER
        cfgs["rssi"][::5] |= CENTRE
        _same(rx.rx_multi(iq, cfgs, capture, offset_hz=offsets), correct_ref.rx_multi(iq, cfgs, capture, offsets))


@pytest.mark.parametrize("hz", [0.0, 100e3, -150e3, 300e3])
@pytest.mark.parametrize("sym", [0, 1])
def test_offset_entry_points(rx, hz, sym):
    """rx_batch_offset and rx_device_dir with offset_hz, both discriminators, with recovery (whose bits are rotated)"""
    caps = [_capture(12.0 if sym else 19.0, ch, n=20, seed=int(abs(hz)) % 89 + ch, cfo_hz=hz) for ch in (37, 9)]
    n = min(c[0].size for c in caps) // 16 * 16
    iq = np.stack([c[0][:n] for c in caps])
    cc = [c[1] for c in caps]
    for rssi in (CORRECT, CORRECT | 1 | 2, CORRECT | CFG_RECOVER | CENTRE):
        cfgs = np.concatenate([make_cfgs(1, rssi=rssi, symbol_spaced=sym, **c) for c in cc])
        want = np.concatenate([_expected(iq[k], cc[k], rssi=rssi, stream=k, hz=hz, sym=bool(sym)) for k in range(2)])
        _same(rx.rx_batch(iq, cfgs, offset_hz=hz), want)
        d_iq = torch.from_numpy(iq).cuda()
        d_out = torch.empty(want.size * 64 + 64 * 64, dtype=torch.uint8, device="cuda")
        d_dir = torch.empty(rx.units(2, n) * 8, dtype=torch.uint8, device="cuda")
        rx.rx_device_dir(d_iq, cfgs, d_out, None, d_dir, torch.cuda.current_stream().cuda_stream, offset_hz=hz)
        torch.cuda.synchronize()
        _same(rx.gather_ordered(d_out.cpu().numpy().view(REC_DTYPE), d_dir.cpu().numpy().view(DIR_DTYPE)), want)


@pytest.mark.parametrize("sym", [0, 1])
def test_report_rejected_mask0_step4(rx, sym):
    """mask 0 with -v on channel 38 over a capture whose chunks start with zeros: more hits than a chunk's hit row, so the
    late rows (step 4) decode and repair them; raw mode is never touched"""
    iq, cfg = _capture(14.0 if sym else 19.0, 38, n=24, seed=9)
    s = iq.reshape(-1, 2).copy()
    for c in range(s.shape[0] // 8192):
        s[8192 * c: 8192 * c + 4600] = 0
    iq = s.reshape(-1)
    for extra in (0, CFG_RECOVER):
        got = rx.rx(iq, rssi=2 | 1 | CORRECT | extra, access_mask=0, symbol_spaced=sym, **cfg)
        exp = _expected(iq, cfg, rssi=2 | 1 | CORRECT | extra, access_mask=0, sym=bool(sym))
        assert max(np.bincount(exp["chunk"])) > 68
        _same(got, exp)
    _same(rx.rx(iq, raw=1, rssi=1 | CORRECT, symbol_spaced=sym, **cfg), _expected(iq, cfg, rssi=1, raw=1, sym=bool(sym)))


@pytest.mark.parametrize("sym", [0, 1])
def test_stream_odd_segments_and_backfill(rx, sym):
    (a, ca), (b, cb) = _capture(13.0 if sym else 19.0, 37, n=60, seed=71), _capture(13.0 if sym else 19.0, 9, n=60, seed=72)
    parts = []
    with rx.stream(segment_chunks=3, rssi=1 | CORRECT, symbol_spaced=sym, **ca) as s_:
        pos, rng = 0, np.random.default_rng(5)
        while pos < a.size:
            k = int(rng.choice([1, 777, 5000, CHUNK + 3, 3 * CHUNK + 1]))
            parts.append(s_.push(a[pos:pos + k]))
            pos += k
        parts.append(s_.finish())
    whole_a = rx.rx(a, rssi=1 | CORRECT, symbol_spaced=sym, **ca)
    _same(np.concatenate(parts), whole_a)
    _same(whole_a, _expected(a, ca, rssi=1 | CORRECT, sym=bool(sym)))
    assert _corrected(whole_a) > 0
    m = min(a.size, b.size)
    base = make_cfgs(2, channel=[ca["channel"], cb["channel"]], access_addr=[ca["access_addr"], cb["access_addr"]],
                     crc_init=[ca["crc_init"], cb["crc_init"]], symbol_spaced=sym, correct=[1, 0])
    with rx.streams(base, segment_chunks=2) as s_:
        parts = [s_.push(0, a[:4 * CHUNK]), s_.push(1, b[:4 * CHUNK])]
        frm = s_.resident
        j, _ = s_.add_cfg(1, frm, recover=1, correct=1, **cb)
        pos = 4 * CHUNK
        while pos < m:
            parts += [s_.push(0, a[pos:pos + 5000]), s_.push(1, b[pos:pos + 5000])]
            pos += 5000
        parts.append(s_.finish())
    got = np.concatenate(parts)
    got = got[np.lexsort((got["n0"], got["chunk"], got["stream"]))]
    whole = rx.rx_batch(np.stack([a[:m], b[:m]]), base)
    e2 = _expected(b[:m], cb, rssi=CFG_RECOVER | CORRECT, stream=j, sym=bool(sym))
    exp = np.concatenate([whole, e2[e2["chunk"] >= frm]])
    _same(got, exp[np.lexsort((exp["n0"], exp["chunk"], exp["stream"]))])


def test_decode_connections(rx):
    """hop.decode_connections(correct=True): the advertising records are the restatement's with the flag"""
    from btle_b200 import hop
    caps = np.zeros((40, 24 * 2048 * 2 // CHUNK * CHUNK + CHUNK), dtype=np.int8)
    for ch in (37, 38, 39):
        iq, _ = _capture(19.0, ch, n=24, seed=ch)
        caps[ch, :min(iq.size, caps.shape[1])] = iq[:caps.shape[1]]
    adv, _ = hop.decode_connections(rx, caps, discover=False, correct=True)
    want = np.concatenate([_expected(caps[ch], dict(ADV, channel=ch), rssi=CORRECT, stream=ch - 37) for ch in (37, 38, 39)])
    want["stream"] += 37
    _same(adv, want)
    assert _corrected(adv) > 0


def _ber_run(rx, flags, snr, n, seed=3, symbol=False):
    run = ber.rx_ber_cfg(snr, slot_samples=2048, seed=seed)
    run["flags"] = flags | (CFG_SYMBOL_SPACED if symbol else 0)
    res = np.zeros(1, dtype=RX_BER_RESULT_DTYPE)
    rx._check(rx._L.btle_b200_rx_ber_run(rx._h, run.ctypes.data, n, res.ctypes.data))
    return res[0]


def test_rx_ber_run(rx):
    """on one seed the flag never adds a packet error and leaves the chain's counters alone; it removes errors at
    symbol-spaced 11 dB and default 20 dB; the flags it is accepted with; two batches count what one capture counts"""
    for snr, sym, base in ((11.0, True, CENTRE), (20.0, False, CENTRE), (20.0, False, 0), (11.0, True, CENTRE | CFG_RECOVER)):
        off = _ber_run(rx, base, snr, 4000, symbol=sym)
        on = _ber_run(rx, base | CORRECT, snr, 4000, symbol=sym)
        assert int(on["pkt_err"]) <= int(off["pkt_err"]), (snr, sym, base)
        for k in ("packets", "aa_miss", "len_reject", "extra_recs"):
            assert int(on[k]) == int(off[k]), (snr, sym, base, k)
        if base != CENTRE | CFG_RECOVER:
            assert int(on["pkt_err"]) < int(off["pkt_err"]), (snr, sym, base)
    for extra in range(8):
        flags = CORRECT | (CFG_RECOVER if extra & 1 else 0) | (CFG_SYMBOL_SPACED if extra & 2 else 0) | (CENTRE if extra & 4 else 0)
        run = ber.rx_ber_cfg(30.0, slot_samples=2048, seed=2)
        run["flags"] = flags
        res = np.zeros(1, dtype=RX_BER_RESULT_DTYPE)
        rx._check(rx._L.btle_b200_rx_ber_run(rx._h, run.ctypes.data, 64, res.ctypes.data))
        assert int(res[0]["packets"]) == 64
    for bad in (8, 32, 128, CORRECT | 8, CORRECT | 32, CORRECT | 128):
        run = ber.rx_ber_cfg(20.0, seed=1)
        run["flags"] = bad
        assert rx._L.btle_b200_rx_ber_run(rx._h, run.ctypes.data, 16, np.zeros(1, dtype=RX_BER_RESULT_DTYPE).ctypes.data) == BTLE_EINVAL
    n = 40000
    for flags in (CORRECT | CENTRE, CORRECT | CENTRE | CFG_SYMBOL_SPACED | CFG_RECOVER):
        run = ber.rx_ber_cfg(19.0 if not flags & CFG_SYMBOL_SPACED else 11.0, slot_samples=2048, seed=8)
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


def test_cli_correct(tmp_path, rx):
    iq, cfg = _capture(19.0, 37, n=200, seed=13)
    f = tmp_path / "cap.bin"
    iq.tofile(f)
    want = rx.rx(iq, rssi=1 | CORRECT, **cfg)
    _same(want, _expected(iq, cfg, rssi=1 | CORRECT))
    assert _corrected(want) > 0
    p = subprocess.run([CLI, "-i", str(f), "-c", "37", "-j", "-Q", "-R", "--correct"], capture_output=True, text=True, check=True)
    lines = [json.loads(s) for s in p.stdout.splitlines() if '"t":"pkt"' in s]
    assert len(lines) == want.size
    for r, l in zip(want, lines):
        assert l["crc_ok"] == (r["crc_bad"] == 0)
        assert l.get("corrected", False) == bool(r["flags"] & REC_CORRECTED)
        assert bytes.fromhex(l["payload_hex"]) == bytes(r["bytes"][2:2 + l["plen"]])
    txt = subprocess.run([CLI, "-i", str(f), "-c", "37", "--correct"], capture_output=True, text=True, check=True).stdout
    plain = subprocess.run([CLI, "-i", str(f), "-c", "37"], capture_output=True, text=True, check=True).stdout
    assert txt.count("CRC0") == int((want["crc_bad"] == 0).sum()) > plain.count("CRC0")
    both = subprocess.run([CLI, "-i", str(f), "-c", "37", "--correct", "--recover", "--centre-hits", "-j", "-Q"], capture_output=True,
                          text=True, check=True)
    want2 = rx.rx(iq, rssi=CORRECT | CFG_RECOVER | CENTRE, **cfg)
    assert sum('"t":"pkt"' in s for s in both.stdout.splitlines()) == want2.size
    for args in (["--iq-bin16", str(f), "--correct"], ["-i", str(f), "-o", "--correct"]):
        bad = subprocess.run([CLI, *args], capture_output=True, text=True)
        assert bad.returncode != 0 and "--correct cannot be combined with -o or --iq-bin16" in bad.stdout
