"""LE Coded PHY receiver (btle_b200_rx_coded*, include/btle_b200.h "LE Coded PHY") on the GPU, pinned to the restatement
coded_ref.py field for field: noiseless and noisy captures, CRC-failed and CI-reserved records, corrected carrier offsets,
several streams with a padded stride, the window edges and truncated packets, two CUDA streams at once, capacity, no
false records on 1M captures, and the sensitivity against the best 1M chain on the same PDUs and noise."""
import ctypes

import numpy as np
import pytest
import torch

import coded_ref as cr
import test_coded as tc
from btle_b200 import BtleRx, make_cfgs, synth
from btle_b200._native import BTLE_EINVAL, BTLE_EOVERFLOW, CFG_CENTRE_HITS, CFG_CORRECT, CFG_LOWPASS, CFG_RECOVER, CFG_RSSI, \
    CFG_SYMBOL_SPACED, CODED_REC_DTYPE, BtleError

pytestmark = pytest.mark.gpu

AA = 0x8E89BED6


@pytest.fixture(scope="module")
def rx():
    import __graft_entry__ as ge
    ge.build()
    r = BtleRx(0)
    yield r
    r.close()


def _cfgs(n, channel=37, aa=AA, crc_init=0x555555, rssi=CFG_RSSI):
    return make_cfgs(n, channel=channel, access_addr=aa, crc_init=crc_init, rssi=rssi)


def _same(got, exp):
    assert got.size == exp.size, (got["sample"], exp["sample"])
    for name in CODED_REC_DTYPE.names:
        assert np.array_equal(got[name], exp[name]), name
    assert got.tobytes() == exp.tobytes()


def _bursts(specs, rng, channel=37, crc_init=0x555555, aa=AA):
    """[(n0, wav)] for specs [(n0, L, s, ci)] and the PDUs sent"""
    out, pdus = [], []
    for n0, L, s, ci in specs:
        pdu = bytes([0x07, L]) + rng.integers(0, 256, L, dtype=np.uint8).tobytes()
        out.append((n0, synth.coded_air(pdu, channel, aa, crc_init, s=s, ci=ci)))
        pdus.append(pdu)
    return out, pdus


def _packet_samples(L, s):
    return 4 * (80 + 296 + (16 + 8 * L + 27) * s)


def _grid_capture(channel, rng):
    """every L of the grid at S = 2 and 8, at all four sample phases"""
    specs, n0 = [], 1000
    for L in (0, 1, 37, 38, 200, 255):
        for s in (2, 8):
            specs.append((n0 + len(specs) % 4, L, s, None))
            n0 += _packet_samples(L, s) + 1600
    bursts, pdus = _bursts(specs, rng, channel, 0x123456)
    return cr.place(n0 + 2000, bursts), specs, pdus


def test_noiseless_grid(rx):
    rng = np.random.default_rng(1)
    for channel in (37, 39, 0, 36):
        iq, specs, pdus = _grid_capture(channel, rng)
        cfg = _cfgs(1, channel, crc_init=0x123456)
        got = rx.rx_coded(iq, cfg)
        exp = cr.rx_coded(iq, cfg)
        _same(got, exp)
        for (n0, L, s, _), pdu in zip(specs, pdus):
            r = got[got["sample"] == n0]
            assert len(r) == 1 and r[0]["crc_bad"] == 0 and bytes(r[0]["bytes"][:L + 2]) == pdu and r[0]["s"] == s


@pytest.mark.parametrize("snr", [-4.0, -1.0, 4.0])
def test_noisy_bit_exact(rx, snr):
    rng = np.random.default_rng(int(snr * 10) + 100)
    specs, n0 = [], 800
    for k in range(24):
        L, s, ci = int(rng.integers(0, 60)), (2, 8)[k % 2], (None, None, None, 2, None, 3)[k % 6]
        specs.append((n0 + k % 4, L, s, ci))
        n0 += _packet_samples(L, s) + 2000
    bursts, _ = _bursts(specs, rng)
    iq = cr.place(n0 + 3000, bursts, 100, cr.sigma_of(snr, 100), rng)
    cfg = _cfgs(1)
    got = rx.rx_coded(iq, cfg)
    exp = cr.rx_coded(iq, cfg)
    _same(got, exp)
    assert (got["flags"] & cr.CI_RESERVED).any()
    if snr < 0:
        assert (got["crc_bad"][(got["flags"] & cr.CI_RESERVED) == 0] == 1).any()


@pytest.mark.parametrize("hz", [-100e3, 100e3])
def test_corrected_offset(rx, hz):
    rng = np.random.default_rng(7)
    specs, n0 = [], 900
    for k in range(6):
        specs.append((n0 + k % 4, 20 + k, (2, 8)[k % 2], None))
        n0 += _packet_samples(20 + k, (2, 8)[k % 2]) + 1000
    bursts, pdus = _bursts(specs, rng)
    iq = cr.place(n0 + 2000, bursts, 100, cr.sigma_of(8.0, 100), rng, offset_hz=hz)
    cfg = _cfgs(1)
    got = rx.rx_coded(iq, cfg, offset_hz=hz)
    _same(got, cr.rx_coded(iq, cfg, offset_hz=hz))
    assert int((got["crc_bad"] == 0).sum()) >= 5


def test_streams_padded_stride_and_two_cuda_streams(rx):
    rng = np.random.default_rng(3)
    n = 2 * 120000
    caps, cfgs = [], _cfgs(3, channel=[37, 5, 39], aa=[AA, 0x12345678, 0x50654E3A], crc_init=[0x555555, 0xABCDEF, 0x13579B])
    for s in range(3):
        specs, n0 = [], 700
        for k in range(8):
            specs.append((n0 + (k + s) % 4, 10 * k, (2, 8)[(k + s) % 2], None))
            n0 += _packet_samples(10 * k, (2, 8)[(k + s) % 2]) + 1000
        assert n0 < n // 2
        bursts, _ = _bursts(specs, rng, int(cfgs[s]["channel"]), int(cfgs[s]["crc_init"]), int(cfgs[s]["access_addr"]))
        caps.append(cr.place(n // 2, bursts, 90, cr.sigma_of(2.0, 90), rng))
    iq = np.stack(caps)
    exp = cr.rx_coded(iq, cfgs)
    _same(rx.rx_coded(iq, cfgs), exp)
    stride = n + 48
    d_iq = torch.zeros((3, stride), dtype=torch.int8, device="cuda")
    d_iq[:, :n] = torch.from_numpy(iq).cuda()
    view = d_iq[:, :n]
    outs = []
    streams = [torch.cuda.Stream(), torch.cuda.Stream()]
    for st in streams:
        d_out = torch.zeros(4096 * 304, dtype=torch.uint8, device="cuda")
        d_count = torch.zeros(1, dtype=torch.int32, device="cuda")
        rx.rx_coded_device(view, cfgs, d_out, d_count, stream_ptr=st.cuda_stream)
        outs.append((d_out, d_count))
    torch.cuda.synchronize()
    for d_out, d_count in outs:
        c = int(d_count.item())
        recs = d_out.cpu().numpy()[:c * 304].view(CODED_REC_DTYPE)
        _same(np.sort(recs, order=["stream", "sample"]), exp)


def test_edges_and_truncation(rx):
    rng = np.random.default_rng(4)
    n = 6000
    (b,), _ = _bursts([(0, 30, 8, None)], rng)
    for n0 in (322, 323, n - 1024, n - 1023):
        iq = cr.place(n, [(n0, b[1])])
        got = rx.rx_coded(iq, _cfgs(1))
        _same(got, cr.rx_coded(iq, _cfgs(1)))
        assert (n0 in got["sample"]) == (323 <= n0 <= n - 1024)
        if n0 in got["sample"]:
            assert got[got["sample"] == n0][0]["flags"] & cr.TRUNCATED
    # first and last legal n0 of a capture long enough to hold the packet, and a capture cut one sample short
    syms, _ = synth.coded_symbols(bytes([7, 30]) + bytes(30), 37, AA, s=8)
    end = 323 + 4 * (syms.size - 80 - 1) + 3
    for n, trunc in [(end + 1, 0), (end, cr.TRUNCATED)]:
        iq = cr.place(n, [(323, b[1])])
        got = rx.rx_coded(iq, _cfgs(1))
        _same(got, cr.rx_coded(iq, _cfgs(1)))
        assert got[got["sample"] == 323][0]["flags"] == trunc


def test_capacity(rx):
    rng = np.random.default_rng(5)
    specs = [(600 + 2600 * k + k % 4, 4, 2, None) for k in range(40)]
    bursts, _ = _bursts(specs, rng)
    iq = cr.place(600 + 2600 * 40 + 2000, bursts)
    exp = cr.rx_coded(iq, _cfgs(1))
    assert exp.size >= 40
    out = np.zeros(5, CODED_REC_DTYPE)
    n_out = ctypes.c_size_t(0)
    cfg = _cfgs(1)
    rc = rx._L.btle_b200_rx_coded(rx._h, iq.ctypes.data, 1, iq.size, iq.size, cfg.ctypes.data, None, out.ctypes.data, 5, ctypes.byref(n_out))
    assert rc == BTLE_EOVERFLOW and n_out.value == exp.size
    _same(rx.rx_coded(iq, _cfgs(1), cap=exp.size), exp)
    _same(rx.rx_coded(iq, _cfgs(1)), exp)
    # the device count is exact whatever cap is
    d_iq = torch.from_numpy(iq).cuda()[None, :]
    d_out = torch.zeros(3 * 304, dtype=torch.uint8, device="cuda")
    d_count = torch.zeros(1, dtype=torch.int32, device="cuda")
    rx.rx_coded_device(d_iq, _cfgs(1), d_out, d_count)
    torch.cuda.synchronize()
    assert int(d_count.item()) == exp.size


def test_refused_arguments(rx):
    iq = np.zeros(8192, np.int8)
    bad = [dict(channel=40), dict(raw=1), dict(access_mask=0xFFFFFFFE)]
    for kw in bad:
        c = _cfgs(1)
        for k, v in kw.items():
            c[k] = v
        with pytest.raises(BtleError) as e:
            rx.rx_coded(iq, c)
        assert e.value.code == BTLE_EINVAL
    for flag in (2, CFG_RECOVER, CFG_SYMBOL_SPACED, CFG_CENTRE_HITS, CFG_CORRECT, CFG_LOWPASS, 1024):
        with pytest.raises(BtleError) as e:
            rx.rx_coded(iq, _cfgs(1, rssi=CFG_RSSI | flag))
        assert e.value.code == BTLE_EINVAL
    for hz in (float("nan"), 600e3):
        with pytest.raises(BtleError) as e:
            rx.rx_coded(iq, _cfgs(1), offset_hz=hz)
        assert e.value.code == BTLE_EINVAL


def test_no_false_records(rx):
    iq, _ = synth.make_adv_stream(64 * 16384, seed=11, channel=37, corrupt_every=6, slot_samples=3000)
    assert rx.rx_coded(iq.numpy(), _cfgs(1)).size == 0
    hot = np.random.default_rng(12).integers(-128, 128, 4 << 20).astype(np.int8)
    assert rx.rx_coded(hot, _cfgs(1)).size == 0


def test_sensitivity_against_1m_chain(rx):
    """At tc.PER_SNR_DB, S=8 loses fewer packets than tc.PER_S8_BOUND, and strictly fewer than the same PDUs sent as 1M
    packets through symbol + low-pass + centre + RECOVER + CORRECT with the same noise."""
    rng = np.random.default_rng(21)
    n_pkts, amp = 60, 100
    sigma = cr.sigma_of(tc.PER_SNR_DB, amp)
    pdus = [bytes([0x07, L]) + rng.integers(0, 256, L, dtype=np.uint8).tobytes() for L in rng.integers(6, 38, n_pkts)]
    coded_bad = one_m_bad = 0
    for k, pdu in enumerate(pdus):
        n0 = 700 + k % 4
        wav = synth.coded_air(pdu, 37, AA, s=8)
        seed = int(rng.integers(1 << 30))
        iq = cr.place(n0 + wav.size // 2 + 1200, [(n0, wav)], amp, sigma, np.random.default_rng(seed))
        r = rx.rx_coded(iq, _cfgs(1, rssi=0))
        coded_bad += not any(x["crc_bad"] == 0 and abs(int(x["sample"]) - n0) <= 3 and bytes(x["bytes"][:len(pdu)]) == pdu for x in r)
        w1 = synth.modulate(synth.air_bytes(pdu, 37)).astype(np.float64).reshape(-1, 2) * amp / 127
        x = np.zeros((16384 * 2, 2))
        x[700:700 + w1.shape[0]] = w1
        x += np.random.default_rng(seed).normal(0.0, sigma, x.shape)
        iq1 = np.clip(np.round(x), -128, 127).astype(np.int8).reshape(-1)
        recs = rx.rx(iq1, channel=37, rssi=CFG_SYMBOL_SPACED | CFG_LOWPASS | CFG_CENTRE_HITS | CFG_RECOVER | CFG_CORRECT)
        one_m_bad += not any(x["crc_bad"] == 0 and bytes(x["bytes"][:len(pdu)]) == pdu for x in recs)
    assert coded_bad / n_pkts < tc.PER_S8_BOUND, coded_bad
    assert coded_bad < one_m_bad, (coded_bad, one_m_bad)
