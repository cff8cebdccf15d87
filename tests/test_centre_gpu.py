"""BTLE_CFG_CENTRE_HITS (include/btle_b200.h) on the GPU: every receive path with the flag returns what the restatement
(tests/centre_ref.py) returns, in every (ROT, SYM) mode, with the flag mixed per cfg; streamed and batched forms equal the
whole capture; the CLI's --centre-hits; and btle_b200_rx_ber_run with the flag."""
import json
import os
import subprocess

import numpy as np
import pytest
import torch

import centre_ref
import golden_util
import mode_ref
import multi_fuzz
import rx_ber_ref as R
from btle_b200 import BtleRx, ber, make_cfgs
from btle_b200._native import (BTLE_EINVAL, CFG_CENTRE_HITS, CFG_RECOVER, CFG_SYMBOL_SPACED, DIR_DTYPE, REC_DTYPE,
                               RX_BER_RESULT_DTYPE)

pytestmark = pytest.mark.gpu

CHUNK = 16384
DATA = dict(channel=9, access_addr=0x60850A27, crc_init=0xA77B2E)
ADV = dict(channel=37, access_addr=0x8E89BED6, crc_init=0x555555)
CLI = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "btle_b200", "btle_rx_b200")
CENTRE = CFG_CENTRE_HITS


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
    return centre_ref.rx_stream(iq, hz, sym, rssi=rssi, raw=raw, stream=stream, access_mask=access_mask, **cfg)


def _by_cfg(iq2d, cfgs, capture, offsets=None):
    """the restatement per cfg (stream = cfg index), in cfg order"""
    out = []
    for j, c in enumerate(np.asarray(capture).reshape(-1)):
        f = cfgs[j]
        out.append(centre_ref.rx_stream(iq2d[c], 0.0 if offsets is None else float(np.float32(offsets[c])), bool(f["rssi"] & CFG_SYMBOL_SPACED),
                                        *mode_ref._fields(f, j)[:-1], stream=j))
    return np.concatenate(out) if out else np.zeros(0, dtype=REC_DTYPE)


@pytest.mark.parametrize("sym", [0, 1])
def test_rx_goldens(rx, sym):
    """rx on every golden with the flag, with RSSI, -v and recovery; at least one record moves"""
    moved = 0
    for name in golden_util.cases():
        z, cfg = golden_util.load(name)
        kw = golden_util.rx_cfg(cfg)
        for extra in (0, 1, 4):
            rssi = kw.get("rssi", 0) | extra | CENTRE
            k = {a: b for a, b in kw.items() if a != "rssi"}
            got = rx.rx(z["iq"], rssi=rssi, symbol_spaced=sym, **k)
            _same(got, centre_ref.rx_stream(z["iq"], 0.0, bool(sym), rssi=rssi, **k))
            off = rx.rx(z["iq"], rssi=rssi & ~CENTRE, symbol_spaced=sym, **k)
            moved += int(got.size != off.size or (got["n0"] != off["n0"]).any())
    assert moved > 0


@pytest.fixture(scope="module")
def caps40():
    caps = [_capture(15 + k % 7, 37 if k % 2 == 0 else 9, n=16, seed=500 + k) for k in range(40)]
    n = min(c[0].size for c in caps) - 1234                                    # ragged
    return np.stack([c[0][:n] for c in caps]), [c[1] for c in caps]


@pytest.mark.parametrize("sym", [0, 1])
def test_batch_40_mixed_and_multi(rx, caps40, sym):
    """rx_batch over 40 captures with the flag on every other capture and RSSI, -v and recovery in every combination;
    rx_multi with 8 cfgs per capture, the flag mixed; the device form"""
    iq, cc = caps40
    flags = [(k % 8) | (CENTRE if (k // 8) % 2 == 0 or k % 3 == 0 else 0) for k in range(40)]
    assert {f & 7 for f in flags if f & CENTRE} == set(range(8))
    cfgs = np.concatenate([make_cfgs(1, rssi=flags[k], symbol_spaced=sym, **c) for k, c in enumerate(cc)])
    got = rx.rx_batch(iq, cfgs)
    assert got.size > 100
    _same(got, np.concatenate([_expected(iq[k], cc[k], rssi=flags[k], stream=k, sym=bool(sym)) for k in range(40)]))
    cap = np.repeat(np.arange(3), 8).astype(np.int32)
    mc = np.concatenate([make_cfgs(8, symbol_spaced=sym, **cc[c]) for c in range(3)])
    mc["rssi"][0::2] |= CENTRE
    mc["raw"][1::8] = 1
    mc["rssi"][2::8] |= 2 | 4
    mc["rssi"][3::8] |= 1
    mc["access_mask"][4::8] = 0xFFFFFF00
    mc["access_addr"][5::8] = 0x12345678
    mc["access_mask"][6::8] = 0
    mc["rssi"][6::8] |= 2
    mc["rssi"][7::8] |= CENTRE | 4
    _same(rx.rx_multi(iq[:3], mc, cap), _by_cfg(iq[:3], mc, cap))
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
    rng = np.random.default_rng(61 + 2 * mode[0] + mode[1])
    for _ in range(2):
        iq, cfgs, capture, offsets = multi_fuzz.draw_mode(rng, mode, max_captures=6, max_chunks=10)
        cfgs["rssi"][::2] |= CENTRE
        cfgs["rssi"][::5] |= CFG_RECOVER
        _same(rx.rx_multi(iq, cfgs, capture, offset_hz=offsets), centre_ref.rx_multi(iq, cfgs, capture, offsets))


@pytest.mark.parametrize("hz", [0.0, 100e3, -150e3, 300e3, -500e3])
@pytest.mark.parametrize("sym", [0, 1])
def test_offset_entry_points(rx, hz, sym):
    """rx_batch_offset and rx_device_dir with offset_hz, at several offsets, both discriminators"""
    caps = [_capture(22.0, ch, n=20, seed=int(abs(hz)) % 89 + ch, cfo_hz=hz) for ch in (37, 9)]
    n = min(c[0].size for c in caps) // 16 * 16
    iq = np.stack([c[0][:n] for c in caps])
    cc = [c[1] for c in caps]
    for rssi in (CENTRE, CENTRE | 1 | 2, CENTRE | 4):
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
    late rows re-run the chain"""
    iq, cfg = _capture(21.0, 38, n=24, seed=9)
    s = iq.reshape(-1, 2).copy()
    for c in range(s.shape[0] // 8192):
        s[8192 * c: 8192 * c + 4600] = 0
    iq = s.reshape(-1)
    got = rx.rx(iq, rssi=2 | 1 | CENTRE, access_mask=0, symbol_spaced=sym, **cfg)
    exp = _expected(iq, cfg, rssi=2 | 1 | CENTRE, access_mask=0, sym=bool(sym))
    assert max(np.bincount(exp["chunk"])) > 68
    _same(got, exp)
    for mask in (0xFFFF0000, 0x000000F0):
        _same(rx.rx(iq, rssi=2 | CENTRE, access_mask=mask, symbol_spaced=sym, **cfg),
              _expected(iq, cfg, rssi=2 | CENTRE, access_mask=mask, sym=bool(sym)))
    _same(rx.rx(iq, raw=1, rssi=1 | CENTRE, symbol_spaced=sym, **cfg), _expected(iq, cfg, rssi=1 | CENTRE, raw=1, sym=bool(sym)))


@pytest.mark.parametrize("sym", [0, 1])
def test_stream_odd_segments_and_backfill(rx, sym):
    (a, ca), (b, cb) = _capture(18.0, 37, n=60, seed=71), _capture(18.0, 9, n=60, seed=72)
    parts = []
    with rx.stream(segment_chunks=3, rssi=1 | CENTRE, symbol_spaced=sym, **ca) as s_:
        pos, rng = 0, np.random.default_rng(5)
        while pos < a.size:
            k = int(rng.choice([1, 777, 5000, CHUNK + 3, 3 * CHUNK + 1]))
            parts.append(s_.push(a[pos:pos + k]))
            pos += k
        parts.append(s_.finish())
    whole_a = rx.rx(a, rssi=1 | CENTRE, symbol_spaced=sym, **ca)
    _same(np.concatenate(parts), whole_a)
    _same(whole_a, _expected(a, ca, rssi=1 | CENTRE, sym=bool(sym)))
    m = min(a.size, b.size)
    base = make_cfgs(2, channel=[ca["channel"], cb["channel"]], access_addr=[ca["access_addr"], cb["access_addr"]],
                     crc_init=[ca["crc_init"], cb["crc_init"]], symbol_spaced=sym, centre_hits=[1, 0])
    with rx.streams(base, segment_chunks=2) as s_:
        parts = [s_.push(0, a[:4 * CHUNK]), s_.push(1, b[:4 * CHUNK])]
        frm = s_.resident
        j, _ = s_.add_cfg(1, frm, recover=1, centre_hits=1, **cb)
        pos = 4 * CHUNK
        while pos < m:
            parts += [s_.push(0, a[pos:pos + 5000]), s_.push(1, b[pos:pos + 5000])]
            pos += 5000
        parts.append(s_.finish())
    got = np.concatenate(parts)
    got = got[np.lexsort((got["n0"], got["chunk"], got["stream"]))]
    whole = rx.rx_batch(np.stack([a[:m], b[:m]]), base)
    e2 = _expected(b[:m], cb, rssi=CFG_RECOVER | CENTRE, stream=j, sym=bool(sym))
    exp = np.concatenate([whole, e2[e2["chunk"] >= frm]])
    _same(got, exp[np.lexsort((exp["n0"], exp["chunk"], exp["stream"]))])


def test_rx_ber_run(rx):
    """the flag is accepted alone and with the other two; two batches count what one capture counts; the noiseless run
    has no packet error and no extra record"""
    for flags in (CENTRE, CENTRE | CFG_RECOVER, CENTRE | CFG_SYMBOL_SPACED, CENTRE | CFG_RECOVER | CFG_SYMBOL_SPACED):
        run = ber.rx_ber_cfg(30.0, slot_samples=2048, seed=2)
        run["flags"] = flags
        res = np.zeros(1, dtype=RX_BER_RESULT_DTYPE)
        rx._check(rx._L.btle_b200_rx_ber_run(rx._h, run.ctypes.data, 64, res.ctypes.data))
        assert int(res[0]["packets"]) == 64
    for bad in (8, 32, 128, CENTRE | 8):
        run = ber.rx_ber_cfg(20.0, seed=1)
        run["flags"] = bad
        assert rx._L.btle_b200_rx_ber_run(rx._h, run.ctypes.data, 16, np.zeros(1, dtype=RX_BER_RESULT_DTYPE).ctypes.data) == BTLE_EINVAL
    n = 40000
    for flags in (CENTRE, CENTRE | CFG_SYMBOL_SPACED | CFG_RECOVER):
        run = ber.rx_ber_cfg(17.0, slot_samples=2048, seed=8)
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
    for sym in (False, True):
        for channel in (37, 0):
            aa = 0x8E89BED6 if channel >= 37 else 0x50654A3C
            r = ber.rx_ber_point(rx, 200.0, 2000, channel=channel, access_addr=aa, slot_samples=2048, symbol_spaced=sym, centre_hits=True)
            assert r["packets"] == 2000 and r["pkt_err"] == 0 and r["extra_recs"] == 0 and r["aa_miss"] == 0, r


def test_cli_centre_hits(tmp_path, rx):
    iq, cfg = _capture(20.0, 37, n=200, seed=13)
    f = tmp_path / "cap.bin"
    iq.tofile(f)
    want = rx.rx(iq, rssi=1 | CENTRE, **cfg)
    _same(want, _expected(iq, cfg, rssi=1 | CENTRE))
    p = subprocess.run([CLI, "-i", str(f), "-c", "37", "-j", "-Q", "-R", "--centre-hits"], capture_output=True, text=True, check=True)
    lines = [json.loads(s) for s in p.stdout.splitlines() if '"t":"pkt"' in s]
    assert len(lines) == want.size
    for r, l in zip(want, lines):
        assert l["crc_ok"] == (r["crc_bad"] == 0)
        assert bytes.fromhex(l["payload_hex"]) == bytes(r["bytes"][2:2 + l["plen"]])
    txt = subprocess.run([CLI, "-i", str(f), "-c", "37", "--centre-hits"], capture_output=True, text=True, check=True).stdout
    plain = subprocess.run([CLI, "-i", str(f), "-c", "37"], capture_output=True, text=True, check=True).stdout
    assert txt.count("CRC0") == int((want["crc_bad"] == 0).sum()) > plain.count("CRC0")
    both = subprocess.run([CLI, "-i", str(f), "-c", "37", "--centre-hits", "--symbol-spaced", "--recover", "--offset", "auto", "-j", "-Q"],
                          capture_output=True, text=True, check=True)
    assert "offset estimate" in both.stderr
    bad = subprocess.run([CLI, "--iq-bin16", str(f), "--centre-hits"], capture_output=True, text=True)
    assert bad.returncode != 0 and "--centre-hits cannot be combined with --iq-bin16" in bad.stdout
