"""The symbol-spaced discriminator (BTLE_CFG_SYMBOL_SPACED, include/btle_b200.h) on the GPU: every receive path in that mode
returns what the numpy restatement over the oracle chain returns (tests/symbol_ref.py); streamed and
batched forms equal rx_batch on the whole capture; one mode per launch; and the new mode's error rates against the
default's."""
import json
import os
import subprocess

import numpy as np
import pytest
import torch

import golden_util
import multi_fuzz
import symbol_ref
import rx_ber_ref as R
from btle_b200 import BtleRx, ber, make_cfgs
from btle_b200._native import BTLE_EINVAL, CFG_SYMBOL_SPACED, DIR_DTYPE, REC_DTYPE, RX_BER_RESULT_DTYPE, BtleError

pytestmark = pytest.mark.gpu

CHUNK = 16384
DATA = dict(channel=9, access_addr=0x60850A27, crc_init=0xA77B2E)
ADV = dict(channel=37, access_addr=0x8E89BED6, crc_init=0x555555)
CLI = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "btle_b200", "btle_rx_b200")


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
    iq, truth, _ = R.capture(cfg, 0, n)
    return iq, dict(base, channel=channel)


def _same(a, b):
    assert a.size == b.size and a.tobytes() == b.tobytes()


def _expected(iq, cfg, rssi=0, raw=0, stream=0, hz=0.0, access_mask=0xFFFFFFFF):
    return symbol_ref.rx_stream(iq, hz, rssi=rssi, raw=raw, stream=stream, access_mask=access_mask, sym=True, **cfg)


def test_goldens_and_fuzz(rx):
    n = 0
    for name in golden_util.cases():
        z, cfg = golden_util.load(name)
        kw = golden_util.rx_cfg(cfg)
        for extra in (0, 1, 4):
            rssi = kw.get("rssi", 0) | extra
            k = {a: b for a, b in kw.items() if a != "rssi"}
            got = rx.rx(z["iq"], rssi=rssi, symbol_spaced=1, **k)
            want = symbol_ref.rx_stream(z["iq"], 0.0, rssi=rssi, sym=True, **k)
            _same(got, want)
            n += got.size
    assert n > 0
    rng = np.random.default_rng(31)
    for _ in range(3):
        iq, cfgs, capture = multi_fuzz.draw(rng, max_captures=8, max_chunks=24)
        cfgs = cfgs.copy()
        cfgs["rssi"] |= CFG_SYMBOL_SPACED
        got = rx.rx_multi(iq, cfgs, capture)
        want = np.concatenate([symbol_ref.rx_stream(iq[capture[j]], 0.0, stream=j, sym=True, **{
            k: int(cfgs[j][k]) for k in ("channel", "access_addr", "access_mask", "crc_init", "raw")}, rssi=int(cfgs[j]["rssi"]) & 7)
            for j in range(cfgs.size)])
        _same(got, want)


@pytest.fixture(scope="module")
def caps40():
    caps = [_capture(15 + k % 7, 37 if k % 2 == 0 else 9, n=16, seed=400 + k) for k in range(40)]
    n = min(c[0].size for c in caps) - 1234                                    # ragged
    return np.stack([c[0][:n] for c in caps]), [c[1] for c in caps]


def test_batch_40_captures_and_multi(rx, caps40):
    iq, cc = caps40
    flags = [(k % 8) for k in range(40)]                                       # RSSI, -v, recover in every combination
    cfgs = np.concatenate([make_cfgs(1, rssi=flags[k], symbol_spaced=1, **c) for k, c in enumerate(cc)])
    got = rx.rx_batch(iq, cfgs)
    assert got.size > 100
    want = np.concatenate([_expected(iq[k], cc[k], rssi=flags[k], stream=k) for k in range(40)])
    _same(got, want)
    # 8 cfgs per capture: the capture's own cfg with raw / -v / recover / masks and other access addresses
    cap = np.repeat(np.arange(3), 8).astype(np.int32)
    mc = np.concatenate([make_cfgs(8, symbol_spaced=1, **cc[c]) for c in range(3)])
    mc["raw"][1::8] = 1
    mc["rssi"][2::8] |= 2 | 4
    mc["rssi"][3::8] |= 1
    mc["access_mask"][4::8] = 0xFFFFFF00
    mc["access_addr"][5::8] = 0x12345678
    mc["access_mask"][6::8] = 0
    mc["rssi"][6::8] |= 2
    got = rx.rx_multi(iq[:3], mc, cap)
    for j, c in enumerate(cap):
        f = mc[j]
        w = symbol_ref.rx_stream(iq[c], 0.0, channel=int(f["channel"]), access_addr=int(f["access_addr"]), access_mask=int(f["access_mask"]),
                                 crc_init=int(f["crc_init"]), raw=int(f["raw"]), rssi=int(f["rssi"]) & 7, stream=j, sym=True)
        _same(got[got["stream"] == j], w)
    # device form equals the host form (rows of a multiple of 16 bytes)
    iq = np.ascontiguousarray(iq[:, :iq.shape[1] // 16 * 16])
    d_iq = torch.from_numpy(iq).cuda()
    want = rx.rx_batch(iq, cfgs)
    d_out = torch.empty(want.size * 64 + 64 * 64, dtype=torch.uint8, device="cuda")
    d_dir = torch.empty(rx.units(40, iq.shape[1]) * 8, dtype=torch.uint8, device="cuda")
    rx.rx_device_dir(d_iq, cfgs, d_out, None, d_dir, torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    _same(rx.gather_ordered(d_out.cpu().numpy().view(REC_DTYPE), d_dir.cpu().numpy().view(DIR_DTYPE)), want)


@pytest.mark.parametrize("hz", [0.0, 100e3, -150e3, 300e3, -500e3])
def test_rotated(rx, hz):
    for channel in (37, 9):
        iq, cfg = _capture(22.0, channel, n=20, seed=int(abs(hz)) % 89 + channel, cfo_hz=hz)
        iq = iq[:iq.size - 2 * 777]
        for rssi in (0, 1 | 2, 4):
            got = rx.rx(iq, offset_hz=hz, rssi=rssi, symbol_spaced=1, **cfg)
            _same(got, _expected(iq, cfg, rssi=rssi, hz=hz))


def test_report_rejected_mask0_step4(rx):
    """mask 0 with -v on channel 38 over a capture whose chunks start with zeros: more hits than a chunk's hit row"""
    iq, cfg = _capture(21.0, 38, n=24, seed=9)
    s = iq.reshape(-1, 2).copy()
    for c in range(s.shape[0] // 8192):
        s[8192 * c: 8192 * c + 4600] = 0
    iq = s.reshape(-1)
    got = rx.rx(iq, rssi=2 | 1, access_mask=0, symbol_spaced=1, **cfg)
    exp = _expected(iq, cfg, rssi=2 | 1, access_mask=0)
    assert max(np.bincount(exp["chunk"])) > 68
    _same(got, exp)
    _same(rx.rx(iq, raw=1, rssi=1, symbol_spaced=1, **cfg), _expected(iq, cfg, rssi=1, raw=1))


def test_stream_odd_segments_and_backfill(rx):
    (a, ca), (b, cb) = _capture(18.0, 37, n=60, seed=71), _capture(18.0, 9, n=60, seed=72)
    parts = []
    with rx.stream(segment_chunks=3, rssi=1, symbol_spaced=1, **ca) as s_:
        pos, rng = 0, np.random.default_rng(5)
        while pos < a.size:
            k = int(rng.choice([1, 777, 5000, CHUNK + 3, 3 * CHUNK + 1]))
            parts.append(s_.push(a[pos:pos + k]))
            pos += k
        parts.append(s_.finish())
    _same(np.concatenate(parts), rx.rx(a, rssi=1, symbol_spaced=1, **ca))
    m = min(a.size, b.size)
    base = make_cfgs(2, channel=[ca["channel"], cb["channel"]], access_addr=[ca["access_addr"], cb["access_addr"]],
                     crc_init=[ca["crc_init"], cb["crc_init"]], symbol_spaced=1)
    with rx.streams(base, segment_chunks=2) as s_:
        parts = [s_.push(0, a[:4 * CHUNK]), s_.push(1, b[:4 * CHUNK])]
        frm = s_.resident
        j, _ = s_.add_cfg(1, frm, recover=1, **cb)
        with pytest.raises(BtleError) as e:                                  # the other mode: refused, the session goes on
            s_.add_cfg(0, frm, symbol_spaced=0)
        assert e.value.code == BTLE_EINVAL
        pos = 4 * CHUNK
        while pos < m:
            parts += [s_.push(0, a[pos:pos + 5000]), s_.push(1, b[pos:pos + 5000])]
            pos += 5000
        parts.append(s_.finish())
    got = np.concatenate(parts)
    got = got[np.lexsort((got["n0"], got["chunk"], got["stream"]))]
    whole = rx.rx_batch(np.stack([a[:m], b[:m]]), base)
    e2 = rx.rx(b[:m], recover=1, symbol_spaced=1, **cb)
    e2["stream"] = j
    exp = np.concatenate([whole, e2[e2["chunk"] >= frm]])
    _same(got, exp[np.lexsort((exp["n0"], exp["chunk"], exp["stream"]))])


def test_one_mode_per_launch(rx, caps40):
    iq, cc = caps40
    cfgs = np.concatenate([make_cfgs(1, symbol_spaced=k % 2, **c) for k, c in enumerate(cc[:4])])
    for call in (lambda: rx.rx_batch(iq[:4], cfgs), lambda: rx.rx_multi(iq[:2], cfgs[:2], np.array([0, 0], np.int32)),
                 lambda: rx.rx_batch(iq[:4], cfgs, offset_hz=0.0)):
        with pytest.raises(BtleError) as e:
            call()
        assert e.value.code == BTLE_EINVAL
        assert b"SYMBOL_SPACED" in rx._L.btle_b200_last_error(rx._h)
    d_iq = torch.from_numpy(np.ascontiguousarray(iq[:4])).cuda()
    d_out = torch.empty(64 * 4096, dtype=torch.uint8, device="cuda")
    d_dir = torch.empty(rx.units(4, iq.shape[1]) * 8, dtype=torch.uint8, device="cuda")
    with pytest.raises(BtleError) as e:
        rx.rx_device_dir(d_iq, cfgs, d_out, None, d_dir, torch.cuda.current_stream().cuda_stream)
    assert e.value.code == BTLE_EINVAL
    with rx.streams(cfgs[:1], segment_chunks=2) as s_:
        for call in (lambda: s_.set_cfg(0, symbol_spaced=1), lambda: s_.add_cfg(0, None, symbol_spaced=1)):
            with pytest.raises(BtleError) as e:
                call()
            assert e.value.code == BTLE_EINVAL
        s_.set_cfg(0, rssi=1)                                                   # the session's own mode is still accepted
    with pytest.raises(BtleError):
        rx.streams(cfgs[:2], segment_chunks=2)
    cfgs["rssi"] |= CFG_SYMBOL_SPACED                                           # a correct call afterwards
    _same(rx.rx_batch(iq[:4], cfgs), np.concatenate([_expected(iq[k], cc[k], stream=k) for k in range(4)]))


def test_rx_ber_run_batches_equal_the_long_capture(rx):
    """Records of a capture cut into two parts on a chunk boundary equal the whole capture's: the first part decoded with
    its look-ahead and 2 samples more, the second streamed behind a lead.  And btle_b200_rx_ber_run over 40000 packets (two
    batches at 2048-sample slots) counts what one long capture, synthesised, decoded and scored in one piece, counts."""
    cfg = ber.rx_ber_cfg(16.0, slot_samples=2048, seed=5)[0]
    iq, _, _ = R.capture(cfg, 0, 64)
    c = dict(ADV)
    whole = rx.rx(iq, rssi=2, symbol_spaced=1, **c)
    _same(whole, _expected(iq, c, rssi=2))
    half = R.capture_int8(32, 2048)
    a = rx.rx(iq[:half + 3008 + 4], rssi=2, symbol_spaced=1, **c)
    _same(np.concatenate([a[a["chunk"] < half // CHUNK], whole[whole["chunk"] >= half // CHUNK]]), whole)
    n = 40000
    for flags in (CFG_SYMBOL_SPACED, CFG_SYMBOL_SPACED | 4):
        run = ber.rx_ber_cfg(17.0, slot_samples=2048, seed=8)
        run["flags"] = flags
        res = np.zeros(1, dtype=RX_BER_RESULT_DTYPE)
        rx._check(rx._L.btle_b200_rx_ber_run(rx._h, run.ctypes.data, n, res.ctypes.data))
        assert rx.last_launches >= 7                                           # more than one batch
        ni = ((n * 2048 + 8191) // 8192) * CHUNK
        d_iq = torch.empty(ni, dtype=torch.int8, device="cuda")
        d_t = torch.empty(n * 64, dtype=torch.uint8, device="cuda")
        rx._check(rx._L.btle_b200_rx_ber_synth_device(rx._h, run.ctypes.data, 0, n, d_iq.data_ptr(), d_t.data_ptr(), None))
        scfg = make_cfgs(1, rssi=2 | flags, **c)
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
            assert int(res[0][k]) == int(one[0][k]), k


def test_rx_ber_noiseless_all_delays(rx):
    for channel in (37, 0):
        aa = 0x8E89BED6 if channel >= 37 else 0x50654A3C
        r = ber.rx_ber_point(rx, 200.0, 2000, channel=channel, access_addr=aa, slot_samples=2048, symbol_spaced=True)
        assert r["packets"] == 2000 and r["pkt_err"] == 0 and r["extra_recs"] == 0 and r["aa_miss"] == 0, r


def _bound(p0, n):
    return 3 * np.sqrt(max(p0 * (1 - p0), 1.0 / n) / n)


def test_per_below_default(rx):
    n = 20000
    for snr in (16.0, 20.0, 30.0):
        off = ber.rx_ber_point(rx, snr, n, seed=3)
        on = ber.rx_ber_point(rx, snr, n, seed=3, symbol_spaced=True)
        print(f"\n{snr} dB: PER default {off['per']:.4f} (aa_miss {off['aa_miss']}), symbol-spaced {on['per']:.4f} (aa_miss {on['aa_miss']})")
        assert on["per"] + _bound(off["per"], n) < off["per"]


def test_rec_offset_on_symbol_records(rx):
    cfg = ber.rx_ber_cfg(200.0, 0.0, 0.0, amplitude=100, slot_samples=2048)
    ni = ((400 * 2048 + 8191) // 8192) * 16384
    d_iq = torch.empty(ni, dtype=torch.int8, device="cuda")
    d_t = torch.empty(400 * 64, dtype=torch.uint8, device="cuda")
    rx._check(rx._L.btle_b200_rx_ber_synth_device(rx._h, cfg.ctypes.data, 0, 400, d_iq.data_ptr(), d_t.data_ptr(), None))
    torch.cuda.synchronize()
    iq = d_iq.cpu().numpy()
    recs = rx.rx(iq, symbol_spaced=1)
    ok = recs[recs["crc_bad"] == 0]
    assert ok.size >= 390
    est = rx.rec_offsets(iq, ok)
    print(f"\nnoiseless symbol-spaced records: median rec_offset {float(np.median(est)):+.1f} Hz")
    assert abs(float(np.median(est))) <= 1000.0


def test_rx_ber_flags(rx):
    """flags may hold BTLE_CFG_RECOVER and BTLE_CFG_SYMBOL_SPACED; any other bit is BTLE_EINVAL and the context stays usable"""
    for bad in (1, 2, 8, 32, 0x80000000, 5, 16 | 8):
        cfg = ber.rx_ber_cfg(20.0, seed=1)
        cfg["flags"] = bad
        res = np.zeros(1, dtype=RX_BER_RESULT_DTYPE)
        assert rx._L.btle_b200_rx_ber_run(rx._h, cfg.ctypes.data, 16, res.ctypes.data) == BTLE_EINVAL
        assert b"flags" in rx._L.btle_b200_last_error(rx._h)
    assert ber.rx_ber_point(rx, 30.0, 64, recover=True)["packets"] == 64
    assert ber.rx_ber_point(rx, 30.0, 64, recover=True, symbol_spaced=True)["packets"] == 64
    with pytest.raises(BtleError):
        bad = ber.rx_ber_cfg(20.0)
        bad["flags"] = 6
        rx._check(rx._L.btle_b200_rx_ber_run(rx._h, bad.ctypes.data, 16, np.zeros(1, dtype=RX_BER_RESULT_DTYPE).ctypes.data))


def test_cli_symbol_spaced(tmp_path, rx):
    iq, cfg = _capture(15.0, 37, n=200, seed=13)
    f = tmp_path / "cap.bin"
    iq.tofile(f)
    want = rx.rx(iq, rssi=1, symbol_spaced=1, **cfg)
    pcap = tmp_path / "o.pcap"
    p = subprocess.run([CLI, "-i", str(f), "-c", "37", "-j", "-Q", "-R", "--symbol-spaced", "-s", str(pcap)], capture_output=True,
                       text=True, check=True)
    lines = [json.loads(s) for s in p.stdout.splitlines() if '"t":"pkt"' in s]
    assert len(lines) == want.size
    for r, l in zip(want, lines):
        assert l["crc_ok"] == (r["crc_bad"] == 0)
        assert bytes.fromhex(l["payload_hex"]) == bytes(r["bytes"][2:2 + l["plen"]])
    data, pk, at = pcap.read_bytes(), [], 24                                  # big-endian records: 16-byte header, 10-byte PHDR, AA
    while at < len(data):
        n = int.from_bytes(data[at + 8:at + 12], "big")
        pk.append(data[at + 16 + 14:at + 16 + n])
        at += 16 + n
    ok = [bytes(r["bytes"][:int(r["n_bytes"]) - 3]) for r in want if r["crc_bad"] == 0]
    assert len(ok) > 0 and pk in (ok, [bytes(r["bytes"][:int(r["n_bytes"]) - 3]) for r in want])
    txt = subprocess.run([CLI, "-i", str(f), "-c", "37", "--symbol-spaced"], capture_output=True, text=True, check=True).stdout
    plain = subprocess.run([CLI, "-i", str(f), "-c", "37"], capture_output=True, text=True, check=True).stdout
    assert txt.count("CRC0") == int((want["crc_bad"] == 0).sum()) > plain.count("CRC0")
    both = subprocess.run([CLI, "-i", str(f), "-c", "37", "--symbol-spaced", "--recover", "--offset", "auto", "-j", "-Q"],
                          capture_output=True, text=True, check=True)
    assert "offset estimate" in both.stderr
    bad = subprocess.run([CLI, "--iq-bin16", str(f), "--symbol-spaced"], capture_output=True, text=True)
    assert bad.returncode != 0 and "--symbol-spaced cannot be combined with --iq-bin16" in bad.stdout
