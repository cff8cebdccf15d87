"""The error-rate flow of the 4-Msps receive chain restated in numpy (tests/rx_ber_ref.py: draws, float64 channel,
capture of slots, scoring), with the C oracle as the receiver, checked at its edges: noiseless packets at every
fractional delay, an access address 4 samples off, one flipped bit, a cut capture."""
import numpy as np
import pytest

import orc
import rx_ber_ref as R
from btle_b200 import ber


def oracle(iq, cfg):
    return orc.rx_stream(iq, channel=int(cfg["channel"]), access_addr=int(cfg["access_addr"]), crc_init=int(cfg["crc_init"]),
                         report_rejected=1)


# (at 50 ppm, 122.5 kHz of carrier error, the receiver loses packets without any noise: not an edge of the flow)
@pytest.mark.parametrize("channel,ppm,cfo", [(37, 0.0, 0.0), (39, 20.0, 0.0), (38, -20.0, 5000.0), (12, 0.0, 0.0), (3, 10.0, -8000.0)])
def test_noiseless_packets_decode_to_their_truth_at_every_delay(channel, ppm, cfo):
    cfg = ber.rx_ber_cfg(1000.0, ppm, cfo, amplitude=64, slot_samples=2048, channel=channel, seed=5 + channel,
                         access_addr=0x8E89BED6 if channel >= 37 else 0x50654A21, crc_init=0x555555 if channel >= 37 else 0x1A2B3C)
    n = 48
    iq, truth, real = R.capture(cfg[0], 0, n)
    assert set(truth["delta4"]) == {0, 1, 2, 3}
    assert np.abs(real).max() < 65                                     # no noise, no clipping (|IQ| of the table ~ 127)
    recs = oracle(iq, cfg[0])
    c = R.score(recs, truth)
    assert c["packets"] == n and c["pkt_err"] == 0 and c["crc_ok_wrong"] == 0 and c["extra_recs"] == 0 and c["clipped"] == 0, c
    # every record sits where the truth puts it: the receiver's n0 is the rounded position of tx sample 39
    pos = recs["chunk"].astype(np.int64) * R.CHUNK + recs["n0"]
    assert np.abs(pos - truth["aa_sample"]).max() <= 1


def test_truth_equals_the_model_flows_pdu_on_advertising_channels():
    """ADV PDUs are ber_run's: header 42 25 and the bytes of draw(seed, k, b >> 3, 9)"""
    p = R.pdu(77, 123, 37)
    assert p.size == 39 and p[0] == 0x42 and p[1] == 0x25
    d = R.pdu(77, 123, 5)
    assert d.size == 29 and d[0] == 0x02 and d[1] == 27 and np.array_equal(d[2:8], p[2:8])


def test_an_access_address_four_samples_off_is_not_matched():
    cfg = ber.rx_ber_cfg(1000.0, slot_samples=2048, seed=9)[0]
    iq, truth, _ = R.capture(cfg, 0, 8)
    recs = oracle(iq, cfg)
    assert len(recs) == 8
    at = int(recs["chunk"][2]) * R.CHUNK + int(recs["n0"][2])                   # where the receiver found packet 2
    for d in (-3, 3):
        t = truth.copy()
        t["aa_sample"][2] = at + d
        assert R.score(recs, t)["pkt_err"] == 0
    for d in (-4, 4):
        t = truth.copy()
        t["aa_sample"][2] = at + d
        c = R.score(recs, t)
        assert (c["aa_miss"], c["pkt_err"], c["bit_err"], c["extra_recs"], c["extra_crc_ok"]) == (1, 1, 8 * 39, 1, 1), c


@pytest.mark.parametrize("channel,bit", [(37, 16 + 5), (37, 8 * 38 + 7), (20, 8 * 10 + 2)])
def test_one_flipped_bit_is_one_bit_error(channel, bit):
    cfg = ber.rx_ber_cfg(1000.0, slot_samples=2048, channel=channel, seed=3)[0]
    iq, truth, _ = R.capture(cfg, 0, 6, corrupt={4: bit})
    c = R.score(oracle(iq, cfg), truth)
    assert (c["pkt_err"], c["bit_err"], c["aa_miss"], c["len_reject"], c["extra_recs"]) == (1, 1, 0, 0, 0), c


def test_a_cut_capture_misses_the_packets_behind_the_cut():
    cfg = ber.rx_ber_cfg(1000.0, slot_samples=2048, seed=4)[0]
    iq, truth, _ = R.capture(cfg, 0, 16)                  # 4 slots per chunk
    cut = 3 * 2 * R.CHUNK
    c = R.score(oracle(iq[:cut], cfg), truth)
    assert (c["aa_miss"], c["pkt_err"], c["bit_err"], c["extra_recs"]) == (4, 4, 4 * 8 * 39, 0), c


def test_noise_and_saturation_follow_the_definition():
    """sigma per rail, and the int8 saturation the truth counts: a hot amplitude at low SNR clips"""
    cfg = ber.rx_ber_cfg(-3.0, amplitude=120, slot_samples=1600, seed=8)[0]
    iq, truth, real = R.capture(cfg, 0, 40)
    r = np.rint(real[: 40 * 1600]).reshape(40, 1600, 2)
    assert np.array_equal(truth["clipped"], ((r < -128) | (r > 127)).any(axis=2).sum(axis=1))
    assert truth["clipped"].sum() > 100 and iq.min() == -128 and iq.max() == 127
    # noise only (no live packet): sigma = amplitude / 10^(snr / 20) / sqrt 2 per rail
    _, _, zr = R.capture(ber.rx_ber_cfg(10.0, amplitude=100, slot_samples=12000, seed=1)[0], 0, 1, n_live=0)
    assert abs(np.std(zr) - 100 / 10 ** 0.5 / 2 ** 0.5) < 0.3
