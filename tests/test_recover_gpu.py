"""BTLE_CFG_RECOVER on the GPU: every receive path with the flag returns the numpy restatement's records
(tests/recover_ref.py over the oracle's), cfgs without the flag stay the reference's, and btle_b200_rx_ber_run with the flag
loses no more packets than without it."""
import numpy as np
import pytest
import torch

import orc
import recover_ref as RR
import rx_ber_ref as R
from btle_b200 import BtleRx, ber, make_cfgs
from btle_b200._native import BTLE_EINVAL, DIR_DTYPE, BtleError, RX_BER_RESULT_DTYPE
from test_stream_sessions_gpu import CHUNK, _feed, _same

pytestmark = pytest.mark.gpu

DATA = dict(channel=9, access_addr=0x60850A27, crc_init=0xA77B2E)


@pytest.fixture(scope="module")
def rx():
    import __graft_entry__ as ge
    ge.build()
    r = BtleRx(0)
    yield r
    r.close()


def _capture(snr, channel, n=48, seed=1, ppm=0.0):
    adv = channel >= 37
    cfg = ber.rx_ber_cfg(snr, ppm, amplitude=64, slot_samples=2048, channel=channel, seed=seed,
                         crc_init=0x555555 if adv else DATA["crc_init"], access_addr=0x8E89BED6 if adv else DATA["access_addr"])[0]
    iq, _, _ = R.capture(cfg, 0, n)
    return iq, dict(channel=channel, access_addr=int(cfg["access_addr"]), crc_init=int(cfg["crc_init"]))


def _expected(iq, cfg, flags=0, stream=0):
    rec = orc.rx_flags(iq, flags, **cfg)
    rec["stream"] = stream
    return RR.apply(rec, iq, crc_init=cfg["crc_init"])


@pytest.fixture(scope="module")
def caps():
    """40 impaired captures around the PER-0.5 point, channels 37 and 9, ragged lengths"""
    out = []
    for k in range(40):
        ch = 37 if k % 2 == 0 else 9
        iq, cfg = _capture(17 + (k % 5), ch, n=24, seed=100 + k)
        out.append((iq[:iq.size - 2 * (k % 3) * 700], cfg))
    return out


def test_rx_and_flag_off_records_unchanged(rx, caps):
    n_rec = 0
    for iq, cfg in caps[:6]:
        off = rx.rx(iq, **cfg)
        on = rx.rx(iq, recover=1, **cfg)
        _same(on, _expected(iq, cfg))
        _same(off, orc.rx_flags(iq, 0, **cfg))
        # same (stream, chunk, n0) sequence; every record that was not recovered is the flag-off record, byte for byte
        assert (on[["stream", "chunk", "n0"]] == off[["stream", "chunk", "n0"]]).all()
        keep = (on["flags"] & RR.REC_RECOVERED) == 0
        _same(on[keep], off[keep])
        n_rec += int((~keep).sum())
    assert n_rec > 0


def test_rx_batch_40_captures_with_and_without_the_flag(rx, caps):
    n = min(iq.size for iq, _ in caps)
    iq2 = np.stack([iq[:n] for iq, _ in caps])
    cfgs = make_cfgs(40, channel=[c["channel"] for _, c in caps], access_addr=[c["access_addr"] for _, c in caps],
                     crc_init=[c["crc_init"] for _, c in caps], rssi=[k % 4 for k in range(40)], recover=[k % 3 != 0 for k in range(40)])
    got = rx.rx_batch(iq2, cfgs)
    exp = []
    for k, (_, c) in enumerate(caps):
        e = _expected(iq2[k], c, flags=k % 4, stream=k)
        exp.append(e if k % 3 != 0 else orc.rx_flags(iq2[k], k % 4, stream=k, **c))
    _same(got, np.concatenate(exp))
    assert ((got["flags"] & RR.REC_RECOVERED) != 0).sum() > 10


def test_rx_device_dir(rx, caps):
    n = min(iq.size for iq, _ in caps[:8])
    iq2 = np.stack([iq[:n] for iq, _ in caps[:8]])
    cfgs = make_cfgs(8, channel=[c["channel"] for _, c in caps[:8]], access_addr=[c["access_addr"] for _, c in caps[:8]],
                     crc_init=[c["crc_init"] for _, c in caps[:8]], rssi=1, recover=1)
    d_iq = torch.from_numpy(iq2).cuda()
    units = rx.units(8, n)
    d_out = torch.zeros(8 * (n // CHUNK) * 51 * 64, dtype=torch.uint8, device="cuda")
    d_dir = torch.zeros(units * 8, dtype=torch.uint8, device="cuda")
    rx.rx_device_dir(d_iq, cfgs, d_out, None, d_dir)
    torch.cuda.synchronize()
    got = rx.gather_ordered(d_out.cpu().numpy().view(orc.REC_DTYPE), d_dir.cpu().numpy().view(DIR_DTYPE))
    _same(got, np.concatenate([_expected(iq2[k], c, flags=1, stream=k) for k, (_, c) in enumerate(caps[:8])]))


def test_rx_multi_same_capture_with_and_without_the_flag(rx, caps):
    iq, cfg = caps[0]
    iq9, cfg9 = caps[1]
    n = min(iq.size, iq9.size)
    iq2 = np.stack([iq[:n], iq9[:n]])
    cfgs = np.concatenate([make_cfgs(1, **cfg), make_cfgs(1, recover=1, **cfg), make_cfgs(1, rssi=3, recover=1, **cfg),
                           make_cfgs(1, recover=1, **cfg9), make_cfgs(1, **cfg9)])
    got = rx.rx_multi(iq2, cfgs, [0, 0, 0, 1, 1])
    exp = [orc.rx_flags(iq2[0], 0, stream=0, **cfg), _expected(iq2[0], cfg, 0, 1), _expected(iq2[0], cfg, 3, 2),
           _expected(iq2[1], cfg9, 0, 3), orc.rx_flags(iq2[1], 0, stream=4, **cfg9)]
    _same(got, np.concatenate(exp))


def test_stream_with_odd_segments(rx, caps):
    iq, cfg = caps[2]
    parts = []
    with rx.stream(segment_chunks=3, recover=1, rssi=1, **cfg) as s_:
        pos, rng = 0, np.random.default_rng(5)
        while pos < iq.size:
            k = int(rng.choice([1, 777, 5000, CHUNK + 3, 3 * CHUNK + 1]))
            parts.append(s_.push(iq[pos:pos + k]))
            pos += k
        parts.append(s_.finish())
    _same(np.concatenate(parts), _expected(iq, cfg, flags=1))


def test_streams_add_cfg_backfill(rx, caps):
    (a, ca), (b, cb) = caps[4], caps[5]
    base = make_cfgs(2, channel=[ca["channel"], cb["channel"]], access_addr=[ca["access_addr"], cb["access_addr"]],
                     crc_init=[ca["crc_init"], cb["crc_init"]], recover=[1, 0])
    rng = np.random.default_rng(7)
    with rx.streams(base, segment_chunks=2) as s_:
        parts = [s_.push(0, a[:4 * CHUNK]), s_.push(1, b[:4 * CHUNK])]
        frm = s_.resident
        j, got_frm = s_.add_cfg(1, frm, recover=1, **cb)
        assert got_frm == frm
        parts += _feed(s_, [a[4 * CHUNK:], b[4 * CHUNK:]], rng, [1, 5000, CHUNK, 3 * CHUNK])
    got = np.concatenate(parts)
    got = got[np.lexsort((got["n0"], got["chunk"], got["stream"]))]
    m = min(a.size, b.size)
    e2 = _expected(b[:m], cb, stream=j)
    exp = np.concatenate([_expected(a[:m], ca, stream=0), orc.rx_flags(b[:m], 0, stream=1, **cb), e2[e2["chunk"] >= frm]])
    _same(got, exp[np.lexsort((exp["n0"], exp["chunk"], exp["stream"]))])


def test_report_rejected_degenerate_mask_step4(rx):
    """mask 0 with -v on channel 38: the zero first half of every chunk gives ~66 rejected hits (the whitening's header
    length is outside 6..37), so the counted packets of the second half lie behind the chunk's 68-hit row and are stored
    by the chunk's own lane (resolver step 4).  Mask 0 counts noise windows, so none of those passes an alternative here;
    the records must still be the restatement's"""
    packets, cfg = _capture(21, 38, n=24, seed=9)
    s = packets.reshape(-1, 2).copy()
    for c in range(s.shape[0] // 8192):
        s[8192 * c: 8192 * c + 4600] = 0
    iq = s.reshape(-1)
    c = dict(cfg, access_mask=0)
    got = rx.rx(iq, rssi=2, recover=1, **c)
    exp = _expected(iq, c, flags=2)
    late = np.concatenate([np.arange(n) for n in np.bincount(exp["chunk"])]) >= 68
    counted = (exp["flags"] & 4) == 0
    assert (late & counted & (exp["crc_bad"] == 1)).sum() >= 10            # step 4 tries the rule on each of them
    _same(got, exp)


def test_rx_ber_run_with_the_flag(rx):
    for snr, ppm in ((30, 0), (20, 0), (24, 50)):
        off = ber.rx_ber_point(rx, snr, 4096, ppm=ppm, seed=11)
        on = ber.rx_ber_point(rx, snr, 4096, ppm=ppm, seed=11, recover=True)
        assert on["pkt_err"] <= off["pkt_err"]
        for k in ("packets", "aa_miss", "len_reject", "extra_recs", "clipped"):
            assert on[k] == off[k], k
        if snr == 30:
            assert on["pkt_err"] < off["pkt_err"]
    # the recovery window is the chunk's own (data behind it reads 0): a capture cut into two batches on a chunk
    # boundary, the first with its 3008-int8 look-ahead, gives the records of the long capture
    cfg = ber.rx_ber_cfg(20.0, slot_samples=2048, seed=5)[0]
    iq, _, _ = R.capture(cfg, 0, 64)
    c = dict(channel=37, access_addr=0x8E89BED6, crc_init=0x555555)
    recs = rx.rx(iq, rssi=2, recover=1, **c)
    _same(recs, _expected(iq, c, flags=2))
    half = R.capture_int8(32, 2048)
    a = rx.rx(iq[:half + 3008], rssi=2, recover=1, **c)
    b = rx.rx(iq[half:], rssi=2, recover=1, **c)
    b["chunk"] += half // CHUNK
    _same(np.concatenate([a, b]), recs)
    assert (recs["flags"] & RR.REC_RECOVERED).any()


def test_rx_ber_unknown_flags_are_einval(rx):
    for bad in (1, 2, 8, 0x80000000, 5):
        cfg = ber.rx_ber_cfg(20.0, seed=1)
        cfg["flags"] = bad
        res = np.zeros(1, dtype=RX_BER_RESULT_DTYPE)
        assert rx._L.btle_b200_rx_ber_run(rx._h, cfg.ctypes.data, 16, res.ctypes.data) == BTLE_EINVAL
        assert b"flags" in rx._L.btle_b200_last_error(rx._h)
    assert ber.rx_ber_point(rx, 30.0, 64, recover=True)["packets"] == 64
    with pytest.raises(BtleError):
        bad = ber.rx_ber_cfg(20.0)
        bad["flags"] = 6
        rx._check(rx._L.btle_b200_rx_ber_run(rx._h, bad.ctypes.data, 16, np.zeros(1, dtype=RX_BER_RESULT_DTYPE).ctypes.data))


def test_cli_recover(tmp_path):
    import json
    import os
    import subprocess
    from test_recover import ADV, damaged_packet
    cli = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "btle_b200", "btle_rx_b200")
    iq, _, truth = damaged_packet(ADV)
    f = tmp_path / "cap.bin"
    iq.tofile(f)
    q = int(RR.apply(orc.rx_flags(iq, 0, **ADV), iq)[0]["flags"]) >> 4 & 3
    plain = subprocess.run([cli, "-i", str(f), "-c", "37"], capture_output=True, text=True, check=True).stdout
    rec = subprocess.run([cli, "-i", str(f), "-c", "37", "--recover"], capture_output=True, text=True, check=True).stdout
    assert "CRC1" in plain and "CRC0" not in plain
    assert "CRC0" in rec and "CRC1" not in rec
    lines = [json.loads(s) for s in subprocess.run([cli, "-i", str(f), "-c", "37", "--recover", "-j", "-Q"], capture_output=True,
                                                     text=True, check=True).stdout.splitlines() if '"t":"pkt"' in s]
    assert len(lines) == 1 and lines[0]["crc_ok"] and lines[0]["recovered"] == q
    assert bytes.fromhex(lines[0]["payload_hex"]) == bytes(truth[2:2 + lines[0]["plen"]])
    plain_j = [s for s in subprocess.run([cli, "-i", str(f), "-c", "37", "-j", "-Q"], capture_output=True, text=True,
                                         check=True).stdout.splitlines() if '"t":"pkt"' in s]
    assert len(plain_j) == 1 and "recovered" not in plain_j[0]
    bad = subprocess.run([cli, "-i", str(f), "--recover", "-o"], capture_output=True, text=True)
    assert bad.returncode != 0 and "--recover cannot be combined with -o" in bad.stdout
