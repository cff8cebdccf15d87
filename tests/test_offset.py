"""Carrier-offset correction on the CPU: the dense warps' rotated arithmetic (emulated with the PTX semantics of prmt /
dp2a) against the definition in include/btle_b200.h, the numpy restatement over the oracle chain against the oracle at
offset 0, the rotated recovery step against its restatement, and the per-packet estimate on hand-built tones."""
import numpy as np
import pytest

import golden_util
import offset_ref
import orc
import rx_ber_ref
from btle_b200 import _native, rx as rxmod

EDGE = np.array([-128, -127, -64, -1, 0, 1, 63, 126, 127], dtype=np.int8)
OFFSETS = [0.0, 1.0, -1.0, 25e3, -25e3, 100e3, -100e3, 150e3, -150e3, 122.5e3, 300e3, -300e3, 499_999.0, 500e3, -500e3]


def _check_dense(iq, c, s):
    ng = (iq.size - 4) // 256
    got = offset_ref.emul_dbits(iq, c, s)
    want = offset_ref.dbits(iq, 128 * ng, c, s)
    bad = np.flatnonzero(got != want)
    assert bad.size == 0, (c, s, bad[:8], iq[2 * bad[0]:2 * bad[0] + 4])


def test_rotation_words():
    assert offset_ref.rot(0.0) == (16384, 0) and offset_ref.rot(0.0, 4) == (16384, 0)
    c, s = offset_ref.rot(100e3)
    assert abs(c - 16384 * np.cos(np.pi / 20)) <= 0.5 and abs(s - 16384 * np.sin(np.pi / 20)) <= 0.5
    # the sign of btle_rx_ber_cfg.cfo_hz: a carrier at +f turns every sample by +phi, and C Im z + ... with S > 0 undoes it
    assert s > 0


@pytest.mark.parametrize("hz", OFFSETS)
def test_dense_edges(hz):
    """every pair of int8 edge values, as (sample n, sample n+1) at both word halves and across words"""
    a, b, c_, d = np.meshgrid(EDGE, EDGE, EDGE, EDGE, indexing="ij")
    pairs = np.stack([a.ravel(), b.ravel(), c_.ravel(), d.ravel()], axis=1).reshape(-1)      # I0 Q0 I1 Q1 ...
    for shift in (0, 2):                                                                     # pair at an even / odd sample
        iq = np.concatenate([np.zeros(shift, np.int8), pairs])
        iq = np.concatenate([iq, np.zeros(-(iq.size - 4) % 256 + 4, np.int8)])
        _check_dense(iq, *offset_ref.rot(hz))


def test_dense_random():
    rng = np.random.default_rng(7)
    iq = rng.integers(-128, 128, size=2 * (1 << 20) + 4, dtype=np.int16).astype(np.int8)  # 2^20 sample pairs
    for hz in OFFSETS:
        _check_dense(iq, *offset_ref.rot(hz))
    _check_dense(iq, 16384, 0)
    _check_dense(iq, -16384, 16384)                                                          # the largest |u| the int32 form meets


def test_zero_offset_is_the_reference():
    """at offset 0 the restatement on the oracle's own functions returns the oracle's records, every golden capture"""
    for name in golden_util.cases():
        z, cfg = golden_util.load(name)
        iq = z["iq"]
        flags = 2 if cfg.get("report_rejected") else 0
        kw = {k: v for k, v in cfg.items() if k != "report_rejected"}
        for rssi in (flags, flags | 1):
            want = orc.rx_flags(iq, rssi, **kw)
            got = offset_ref.rx_stream(iq, 0.0, rssi=rssi, **kw)
            assert got.tobytes() == want.tobytes(), name


def _impaired(cfo_hz, snr_db, channel, n=24, ppm=0.0, seed=3):
    cfg = np.zeros(1, dtype=_native.RX_BER_CFG_DTYPE)[0]
    cfg["seed"], cfg["snr_db"], cfg["ppm"], cfg["cfo_hz"], cfg["amplitude"] = seed, snr_db, ppm, cfo_hz, 64
    cfg["slot_samples"], cfg["channel"], cfg["crc_init"], cfg["access_addr"] = 2048, channel, 0x555555, 0x8E89BED6 if channel >= 37 else 0x50654A3C
    return rx_ber_ref.capture(cfg, 0, n)[0], int(cfg["access_addr"])


@pytest.mark.parametrize("channel", [37, 9])
def test_correction_restores_packets(channel):
    """a 150 kHz capture decodes far worse uncorrected than corrected, and corrected about as the capture at 0"""
    iq, aa = _impaired(150e3, 40.0, channel)
    ok = lambda r: int(((r["crc_bad"] == 0) & ((r["flags"] & 4) == 0)).sum())
    plain = offset_ref.rx_stream(iq, 0.0, channel=channel, access_addr=aa)
    fixed = offset_ref.rx_stream(iq, 150e3, channel=channel, access_addr=aa)
    assert ok(fixed) > ok(plain) and ok(fixed) >= 18


@pytest.mark.parametrize("hz", [0.0, 100e3, -150e3])
def test_recover_rotated(hz):
    """the emulated recover_packet<true> equals the restatement's rotated recovery"""
    for channel, snr in ((37, 20.0), (9, 24.0)):
        iq, aa = _impaired(hz, snr, channel, n=32)
        cfgs = rxmod.make_cfgs(1, channel=channel, access_addr=aa, rssi=_native.CFG_RECOVER)
        plain = offset_ref.rx_stream(iq, hz, channel=channel, access_addr=aa)
        want = offset_ref.recover(plain, iq, hz)
        got = offset_ref.emul_recover(plain, iq, cfgs, hz)
        assert got.tobytes() == want.tobytes()
        if hz == 0.0:                                            # at 0, BTLE_CFG_RECOVER's own rule
            import recover_ref
            assert want.tobytes() == recover_ref.apply(plain, iq).tobytes()


def test_estimate_tones():
    aa = 0x8E89BED6
    ref_hz = offset_ref.ref_sum(aa) * 4e6 / (2 * np.pi * offset_ref.OFF_TURNS)
    n0 = 1000
    # the transmitter's own waveform, placed at n0, estimates 0 exactly
    t = offset_ref.tx_waveform(aa, 200)
    x = np.zeros((8192, 2), dtype=np.int64)
    x[n0 - offset_ref.AA_OFFSET:n0 - offset_ref.AA_OFFSET + 200] = t
    assert offset_ref.rec_offset(x.astype(np.int8).reshape(-1), 0, n0, aa) == pytest.approx(0.0, abs=1e-6)
    for f in (-150e3, -50e3, 0.0, 1e3, 50e3, 150e3, 400e3):
        n = np.arange(8192)
        tone = np.rint(120 * np.exp(2j * np.pi * f / 4e6 * n))
        iq = np.stack([tone.real, tone.imag], axis=1).astype(np.int8).reshape(-1)
        # a pure tone turns by exactly 2 pi f / 4 MHz per sample (to int8 rounding): the estimate is f minus the reference's
        assert offset_ref.rec_offset(iq, 0, n0, aa) + ref_hz == pytest.approx(f, abs=150.0)
        # the transmitter's waveform shifted by f estimates f (to int8 rounding of the rotated samples)
        rot = t[:, 0] + 1j * t[:, 1]
        rot = rot * np.exp(2j * np.pi * f / 4e6 * np.arange(200))
        y = np.zeros((8192, 2))
        y[n0 - offset_ref.AA_OFFSET:n0 - offset_ref.AA_OFFSET + 200] = np.stack([rot.real, rot.imag], axis=1)
        assert offset_ref.rec_offset(np.rint(y).astype(np.int8).reshape(-1), 0, n0, aa) == pytest.approx(f, abs=150.0)


def test_estimate_bias_follows_the_delay():
    """Why the noiseless estimate is not 0 on rx_ber_synth captures: the turns telescope to the phase turned between the
    window's two ends, and the synthesiser delays each packet by delta4 / 4 of a sample, which moves both ends.  Per delay
    the estimate is one value, about 0 at delta4 = 0 and about 200 Hz lower per quarter sample; the median over the four
    delays lands near -390 Hz.  So a bound of 1 kHz covers the worst delay (3/4 sample, about -600 Hz)."""
    cfg = np.zeros(1, dtype=_native.RX_BER_CFG_DTYPE)[0]
    cfg["seed"], cfg["snr_db"], cfg["amplitude"], cfg["slot_samples"], cfg["channel"] = 1, 200.0, 100, 2048, 37
    cfg["crc_init"], cfg["access_addr"] = 0x555555, 0x8E89BED6
    iq, truth, _ = rx_ber_ref.capture(cfg, 0, 80)
    recs = offset_ref.rx_stream(iq, 0.0)
    ok = recs[recs["crc_bad"] == 0]
    assert ok.size == 80
    by = {}
    for r in ok:
        p = int(r["chunk"]) * 8192 + int(r["n0"])
        k = int(np.argmin(np.abs(truth["aa_sample"] - p)))
        by.setdefault(int(truth["delta4"][k]), []).append(offset_ref.rec_offset(iq, int(r["chunk"]), int(r["n0"]), int(r["access_addr"])))
    assert sorted(by) == [0, 1, 2, 3]
    mean = {d: float(np.mean(v)) for d, v in by.items()}
    assert all(np.ptp(v) < 1.0 for v in by.values())
    assert abs(mean[0]) < 50.0
    for d in (1, 2, 3):
        assert mean[d] - mean[d - 1] == pytest.approx(-205.0, abs=40.0)
    assert max(abs(m) for m in mean.values()) < 1000.0
