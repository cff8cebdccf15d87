"""BTLE_CFG_RECOVER on the CPU: the numpy restatement (tests/recover_ref.py, over the oracle's records) against the
kernel's shared per-lane function (recover_packet, tests/emul/btle_recover_emul.cpp) over the records of the test-only
emulator's whole-stream path and of its unit plan and resolver passes (tests/emul/)."""
import numpy as np
import pytest

import emul
import golden_util as G
import orc
import recover_ref as RR
import rx_ber_ref as R
from btle_b200 import ber, synth
from btle_b200.rx import make_cfgs

ADV = dict(channel=37, access_addr=0x8E89BED6, crc_init=0x555555)
DATA = dict(channel=9, access_addr=0x60850A27, crc_init=0xA77B2E)


def _same(a, b):
    assert len(a) == len(b), (len(a), len(b))
    for k, (x, y) in enumerate(zip(a, b)):
        assert x.tobytes() == y.tobytes(), (k, x, y)


def _emul_both(iq, cfg, flags=0):
    """emulator records with BTLE_CFG_RECOVER: the kernel's recovery step (recover_packet) over the records of the
    stream path and of the unit path (which must agree)"""
    iq2 = np.asarray(iq, dtype=np.int8).reshape(1, -1)
    cfgs = make_cfgs(1, **{k: v for k, v in cfg.items()}, rssi=flags, recover=1)
    a = emul.recover(emul.rx_stream(iq, span_chunks=4, rssi=flags | RR.CFG_RECOVER, **cfg), iq2, cfgs)
    b, d = emul.rx_batch_units(iq2, cfgs, grid=7)
    b = emul.recover(b, iq2, cfgs)
    _same(a, b)
    return a


def _expected(iq, cfg, flags=0):
    rec = orc.rx_flags(iq, flags, **cfg)
    return rec, RR.apply(rec, iq, crc_init=cfg["crc_init"], raw=cfg.get("raw", 0))


def damaged_packet(cfg, offset=3000, n_chunks=2):
    """one noiseless packet whose payload bit 43 has the reference's discriminator bit flipped by changing sample
    n0 + 4 * 43 + 1, which only alternative q = 3 reads.  -> (capture, record n0, truth bytes [n_bytes])"""
    ch = cfg["channel"]
    rng = np.random.default_rng(ch)
    if ch >= 37:
        pdu = synth.adv_pdu(0, 0, 0, rng.integers(0, 256, 20, dtype=np.uint8).tobytes())
    else:
        pdu = bytes([0x02, 27]) + rng.integers(0, 256, 27, dtype=np.uint8).tobytes()
    air = synth.air_bytes(pdu, ch, cfg["access_addr"], cfg["crc_init"])
    iq = np.zeros(2 * 8192 * n_chunks, dtype=np.int8)
    w = synth.modulate(air)
    iq[2 * offset: 2 * offset + w.size] = w
    clean = orc.rx_stream(iq, **cfg)
    assert len(clean) >= 1 and not clean["crc_bad"].any()
    n0 = int(clean[0]["n0"]) + 8192 * int(clean[0]["chunk"])
    truth = clean[0]["bytes"][:clean[0]["n_bytes"]].copy()
    s = iq.reshape(-1, 2).astype(np.int32)
    m = n0 + 4 * 43
    i0, q0 = s[m]
    d = i0 * s[m + 1, 1] - s[m + 1, 0] * q0 > 0
    s[m + 1] = (q0, -i0) if d else (-q0, i0)            # I0 Q1 - I1 Q0 = -(I0^2 + Q0^2) or +(I0^2 + Q0^2)
    return np.clip(s, -128, 127).astype(np.int8).reshape(-1), n0, truth


@pytest.mark.parametrize("cfg", [ADV, DATA], ids=["adv37", "data9"])
def test_damaged_packet_is_recovered_below_q3(cfg):
    iq, n0, truth = damaged_packet(cfg)
    ref, exp = _expected(iq, cfg)
    assert len(ref) == 1 and ref[0]["crc_bad"] == 1 and ref[0]["n0"] == n0
    got = _emul_both(iq, cfg)
    _same(got, exp)
    r = got[0]
    q = (int(r["flags"]) >> 4) & 3
    assert r["crc_bad"] == 0 and r["flags"] & RR.REC_RECOVERED and q < 3
    assert bytes(r["bytes"][:r["n_bytes"]]) == bytes(truth) and not r["bytes"][r["n_bytes"]:].any()
    assert (r["stream"], r["chunk"], r["n0"], r["access_addr"]) == (ref[0]["stream"], ref[0]["chunk"], ref[0]["n0"], ref[0]["access_addr"])


def test_damaged_packet_at_a_negative_n0():
    """the access address starts 2 samples in front of chunk 1: chunk 0 reports the packet at n0 = 8190 and chunk 1,
    through its zeroed history (bit 0 of the access address is 0), at n0 = -2"""
    iq, n0, truth = damaged_packet(ADV, offset=8192 - 2 - 39, n_chunks=3)
    ref, exp = _expected(iq, ADV)
    assert list(ref["chunk"]) == [0, 1] and ref["n0"][1] < 0 and ref["crc_bad"].all(), ref[["chunk", "n0", "crc_bad"]]
    got = _emul_both(iq, ADV)
    _same(got, exp)
    assert not got["crc_bad"].any()
    for r in got:
        assert bytes(r["bytes"][:r["n_bytes"]]) == bytes(truth)


def test_noiseless_captures_never_recover():
    for ch, kw in ((37, {}), (12, dict(access_addr=0x60850A27, crc_init=0xA77B2E, data_channel_pdu=True))):
        iq, _ = synth.make_adv_stream(12 * 16384, seed=5 + ch, channel=ch, corrupt_every=0, slot_samples=2500, **kw)
        iq = iq.numpy()
        cfg = dict(channel=ch, access_addr=kw.get("access_addr", 0x8E89BED6), crc_init=kw.get("crc_init", 0x555555))
        ref = orc.rx_flags(iq, 0, **cfg)
        assert len(ref) > 30 and not ref["crc_bad"].any()
        _same(_emul_both(iq, cfg), ref)


def _ber_capture(snr, ppm, channel, n=40, slot=2048, seed=3, cut=0):
    adv = channel >= 37
    cfg = ber.rx_ber_cfg(snr, ppm, amplitude=64, slot_samples=slot, channel=channel, seed=seed,
                         crc_init=0x555555 if adv else DATA["crc_init"], access_addr=0x8E89BED6 if adv else DATA["access_addr"])[0]
    iq, _, _ = R.capture(cfg, 0, n)
    if cut:
        iq = iq[:iq.size - cut]
    return iq, dict(channel=channel, access_addr=int(cfg["access_addr"]), crc_init=int(cfg["crc_init"]))


def test_emulator_equals_restatement_on_impaired_captures():
    """16 / 20 / 26 / 30 dB, ppm 0 and 50, channels 37 and 9, with and without -v: the emulator runs the shared function
    exactly as the restatement reads the rule, and some CRC failures are recovered while others are not"""
    stats = dict(recovered=0, failed=0)
    for snr in (16, 20, 26, 30):
        for ppm in (0, 50):
            for ch in (37, 9):
                iq, cfg = _ber_capture(snr, ppm, ch, seed=snr + ch + ppm)
                for flags in (0, 2):
                    ref, exp = _expected(iq, cfg, flags)
                    got = _emul_both(iq, cfg, flags)
                    _same(got, exp)
                    bad = (ref["crc_bad"] == 1) & (ref["flags"] & 4 == 0)
                    rec = (got["flags"] & RR.REC_RECOVERED) != 0
                    assert not (rec & ~bad).any()                       # only CRC-failed counted packets are touched
                    assert (got["flags"][ref["flags"] & 4 != 0] & RR.REC_RECOVERED == 0).all()
                    stats["recovered"] += int(rec.sum())
                    stats["failed"] += int((bad & ~rec).sum())
    assert stats["recovered"] > 20 and stats["failed"] > 0, stats


def test_skipped_alternatives_and_window_end():
    """channel 37 at low SNR: some alternatives' headers have a length outside 6..37 (skipped); captures cut inside the
    last chunk's window read zeros behind their end"""
    skipped = 0
    for seed in range(3):
        iq, cfg = _ber_capture(14, 0, 37, n=24, seed=40 + seed)
        ref = orc.rx_stream(iq, **cfg)
        for r in ref[ref["crc_bad"] == 1]:
            e = RR.sym_bits(RR.window(iq, int(r["chunk"])))
            for q in range(4):
                b = RR.to_bytes(RR.alternative(e, int(r["n0"]), q, 32 + 16)[32:]) ^ RR._WHITEN[37][:2]
                skipped += not 6 <= (int(b[1]) & 0x3F) <= 37
        for cut in (2 * 1000, 2 * 1473 + 8, 2 * 1700 + 6):
            iqc = iq[:iq.size - cut]
            ref, exp = _expected(iqc, cfg)
            _same(_emul_both(iqc, cfg), exp)
    assert skipped > 0


def test_raw_mode_and_rejected_hits_are_untouched():
    iq, cfg = _ber_capture(18, 0, 37, n=40, seed=77)
    raw = dict(cfg, raw=1)
    raw_cfgs = make_cfgs(1, **raw, recover=1)
    _same(emul.recover(emul.rx_stream(iq, span_chunks=4, rssi=RR.CFG_RECOVER, **raw), iq, raw_cfgs), orc.rx_flags(iq, 0, **raw))
    ref = orc.rx_flags(iq, 2, **cfg)
    got = _emul_both(iq, cfg, 2)
    rej = (ref["flags"] & 4) != 0
    assert rej.any()
    _same(got[rej], ref[rej])
    ok = ref["crc_bad"] == 0
    _same(got[ok], ref[ok])


@pytest.mark.parametrize("name", [n for n in G.cases() if n.startswith("fuzz_")])
def test_emulator_equals_restatement_on_fuzz_goldens(name):
    z, cfg = G.load(name)
    cfg = dict(cfg)
    cfg.pop("rssi", None)
    cfg.setdefault("crc_init", 0x555555)
    a = emul.recover(emul.rx_stream(z["iq"], span_chunks=3, rssi=RR.CFG_RECOVER, **cfg), z["iq"], make_cfgs(1, **cfg, recover=1))
    ref = orc.rx_flags(z["iq"], 0, **cfg)
    _same(a, RR.apply(ref, z["iq"], crc_init=cfg["crc_init"], raw=cfg.get("raw", 0)))
