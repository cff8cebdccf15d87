"""BTLE_CFG_CORRECT on the CPU: the shared syndrome table and lookup (btle_core.cuh, through the emulator library) against
the numpy restatement (tests/correct_ref.py), packets with planted one-bit, adjacent-pair and other errors, and the kernel
logic's CPU emulator against the restatement on impaired captures, fuzz goldens, raw mode, -v rejected hits and degenerate
masks, alone and with BTLE_CFG_RECOVER and BTLE_CFG_CENTRE_HITS."""
import numpy as np
import pytest

import correct_ref as CR
import correct_emul
import emul
import golden_util as G
import mode_ref
import orc
import recover_ref
import rx_ber_ref as R
from btle_b200 import _native, ber, synth
from btle_b200.rx import make_cfgs

CORRECT, RECOVER, CENTRE = _native.CFG_CORRECT, _native.CFG_RECOVER, _native.CFG_CENTRE_HITS
ADV = dict(channel=37, access_addr=0x8E89BED6, crc_init=0x555555)
DATA = dict(channel=9, access_addr=0x60850A27, crc_init=0xA77B2E)
UNROTATED = [(0, 0), (0, 1)]          # the modes the emulator's unit path runs (carrier-offset correction is checked on the GPU)


def _same(a, b):
    assert len(a) == len(b), (len(a), len(b))
    for k, (x, y) in enumerate(zip(a, b)):
        assert x.tobytes() == y.tobytes(), (k, x, y)


def emulated(iq, cfgs):
    """the emulated unit path (one cfg per capture), records in reference order, with the kernel's repair step"""
    iq2d = np.asarray(iq, dtype=np.int8).reshape(len(cfgs), -1)
    recs, d = emul.rx_batch_units(iq2d, cfgs, grid=7)
    recs = np.concatenate([recs[b:b + c] for b, c in d]) if len(d) else recs[:0]
    return correct_emul.repair(recs, iq2d, cfgs)


def restated(iq, cfg):
    return CR.rx_stream(iq, 0.0, bool(cfg["rssi"] & _native.CFG_SYMBOL_SPACED), *mode_ref._fields(cfg, 0)[:-1])


def check(iq, cfg):
    """the emulator equals the restatement for one cfg (CFG_DTYPE [1]); returns the records"""
    want = restated(iq, cfg[0])
    _same(emulated(iq, cfg), want)
    return want


# ---- the table ----------------------------------------------------------------------------------------------------------
def shared_table():
    n, tab = correct_emul.syndrome_table()
    return n, {int(e >> np.uint64(32)): (int(e & np.uint64(0xFFFFFFFF)) >> 1, (int(e) & 1) + 1) for e in tab if e}


def test_shared_table_holds_the_671_patterns():
    n, tab = shared_table()
    assert n == 671 and len(tab) == 671 and 0 not in tab
    assert tab == CR.table()
    kinds = {"single": 0, "body-body": 0, "crc-crc": 0, "straddle": 0}
    for u, w in tab.values():
        if w == 1:
            kinds["single"] += 1
        else:
            kinds["crc-crc" if u <= 23 else "straddle" if u == 24 else "body-body"] += 1
    assert kinds == {"single": 336, "body-body": 311, "crc-crc": 23, "straddle": 1}


def test_syndromes_depend_only_on_the_distance_from_the_end():
    """every body length 2..39: each pattern's syndrome is crc24(flipped) ^ crc24(original) (CRC bits: the bit itself)"""
    rng = np.random.default_rng(5)
    by_pattern = {p: s for s, p in CR.table().items()}
    for body_len in range(2, 40):
        body = rng.integers(0, 256, body_len, dtype=np.uint8)
        crc0 = synth.crc24(bytes(body), 0x123456)
        nbits = 8 * (body_len + 3)
        for i, w in CR.patterns(nbits):
            u = nbits - 1 - i
            if i + w <= 8 * body_len:
                s = synth.crc24(bytes(CR.flip(body, i, w)), 0x123456) ^ crc0
            else:
                crc_bits = sum(1 << (j - 8 * body_len) for j in range(i, i + w) if j >= 8 * body_len)
                s = crc_bits ^ (synth.crc24(bytes(CR.flip(body, i, 1)), 0x123456) ^ crc0 if i < 8 * body_len else 0)
            assert by_pattern[(u, w)] == s, (body_len, i, w)


def test_lookup_agrees_on_every_syndrome():
    """syndrome_lookup over all 2^24 syndromes, exhaustively"""
    code = correct_emul.syndrome_lookup(0, 1 << 24)
    want = np.full(1 << 24, -1, dtype=np.int16)
    for s, (u, w) in CR.table().items():
        want[s] = 2 * u + w - 1
    assert np.array_equal(code, want)


# ---- planted errors -----------------------------------------------------------------------------------------------------
SLOT = 2048


def planted(cfg, flips, body_len):
    """one noiseless packet per slot (from sample 1000 on), each with its own set of packet bits (dewhitened order, bit 0
    = the first header bit) inverted in the air; -> (capture, truth bytes)"""
    ch = cfg["channel"]
    rng = np.random.default_rng(ch + body_len)
    if ch >= 37:
        pdu = synth.adv_pdu(0, 0, 0, rng.integers(0, 256, body_len - 2, dtype=np.uint8).tobytes())
    else:
        pdu = bytes([0x02, body_len - 2]) + rng.integers(0, 256, body_len - 2, dtype=np.uint8).tobytes()
    air = np.frombuffer(synth.air_bytes(pdu, ch, cfg["access_addr"], cfg["crc_init"]), dtype=np.uint8)
    n_chunks = (1000 + SLOT * len(flips)) // 8192 + 2
    iq = np.zeros(2 * 8192 * n_chunks, dtype=np.int8)
    for k, bits in enumerate(flips):
        a = np.unpackbits(air, bitorder="little")
        for b in bits:
            a[40 + b] ^= 1                                # preamble (8) and access address (32) in front
        w = synth.modulate(np.packbits(a, bitorder="little").tobytes())
        at = 2 * (1000 + SLOT * k)
        iq[at:at + w.size] = w
    clean = np.zeros(2 * 8192 * 2, dtype=np.int8)
    w = synth.modulate(air.tobytes())
    clean[2000:2000 + w.size] = w
    return iq, orc.rx_stream(clean, **cfg)


def slot_of(r):
    return (int(r["chunk"]) * 8192 + int(r["n0"]) - 1000 + SLOT // 4) // SLOT


@pytest.mark.parametrize("cfg", [ADV, DATA], ids=["adv37", "data9"])
def test_planted_errors(cfg):
    body_len = 39 if cfg["channel"] >= 37 else 33
    nbits = 8 * (body_len + 3)
    lf = set(CR.length_field(cfg["channel"]))
    allowed = [tuple(range(i, i + w)) for i, w in CR.patterns(nbits) if not set(range(i, i + w)) & lf]
    touching = [tuple(range(i, i + w)) for i, w in CR.patterns(nbits) if set(range(i, i + w)) & lf]
    rng = np.random.default_rng(cfg["channel"])
    other = [tuple(sorted(rng.choice(nbits, 2, replace=False))) for _ in range(40)]
    other = [p for p in other if p[1] - p[0] > 1] + [tuple(int(x) for x in rng.choice(nbits, 3, replace=False)) for _ in range(40)]
    flips = allowed + touching + other
    iq, clean = planted(cfg, flips, body_len)
    assert len(clean) == 1 and not clean["crc_bad"].any()
    truth = clean[0]["bytes"][:clean[0]["n_bytes"]].tobytes()
    cfgs = make_cfgs(1, **cfg, correct=1)
    got = check(iq, cfgs)
    plain = orc.rx_flags(iq, 0, **cfg)
    counted = {}
    for r in got:
        counted.setdefault(slot_of(r), []).append(r)
    for k in range(len(allowed)):
        rs = counted[k]
        assert all(r["flags"] & _native.REC_CORRECTED and r["crc_bad"] == 0 and r["bytes"][:r["n_bytes"]].tobytes() == truth
                   for r in rs), (k, flips[k])
    n_corr = int(((got["flags"] & _native.REC_CORRECTED) != 0).sum())
    want_other = 0
    for r, p in zip(got, plain):                            # the chain and every record field but the repair are unchanged
        assert (r["chunk"], r["n0"], r["n_bytes"], r["mag_sum"]) == (p["chunk"], p["n0"], p["n_bytes"], p["mag_sum"])
        k = slot_of(r)
        if k >= len(allowed):
            want_other += bool(r["flags"] & _native.REC_CORRECTED)
            if not r["flags"] & _native.REC_CORRECTED:
                assert r.tobytes() == p.tobytes()
    assert len(got) == len(plain)
    assert n_corr >= len(allowed) and want_other < len(flips) - len(allowed)


# ---- the emulator against the restatement -------------------------------------------------------------------------------
def _ber_capture(snr, ppm, channel, n=40, slot=2048, seed=3):
    adv = channel >= 37
    cfg = ber.rx_ber_cfg(snr, ppm, amplitude=64, slot_samples=slot, channel=channel, seed=seed,
                         crc_init=0x555555 if adv else DATA["crc_init"], access_addr=0x8E89BED6 if adv else DATA["access_addr"])[0]
    iq, _, _ = R.capture(cfg, 0, n)
    return iq, dict(channel=channel, access_addr=int(cfg["access_addr"]), crc_init=int(cfg["crc_init"]))


@pytest.mark.parametrize("mode", UNROTATED, ids=mode_ref.mode_id)
def test_emulator_equals_restatement_on_impaired_captures(mode):
    """several SNRs, ppm 0 and 20, channels 37 and 9, with and without centre hits and recovery: some CRC failures are
    corrected (also after recovery), others are not"""
    stats = dict(corrected=0, recovered_corrected=0, failed=0)
    snrs = (9, 11, 13) if mode[1] else (16, 20, 24)
    for snr in snrs:
        for ppm in (0, 20):
            for ch in (37, 9):
                iq, cfg = _ber_capture(snr, ppm, ch, seed=snr + ch + ppm)
                for extra in (0, CENTRE, RECOVER, RECOVER | CENTRE, RECOVER | 2):
                    cfgs = mode_ref.with_mode(make_cfgs(1, **cfg, rssi=extra | CORRECT), mode)
                    got = check(iq, cfgs)
                    f = got["flags"]
                    stats["corrected"] += int(((f & _native.REC_CORRECTED) != 0).sum())
                    stats["recovered_corrected"] += int(((f & _native.REC_CORRECTED) != 0).__and__((f & 8) != 0).sum())
                    stats["failed"] += int(((got["crc_bad"] == 1) & (f & 4 == 0)).sum())
                    if not extra & RECOVER:
                        continue
                    # with both flags every record recovery alone makes CRC-ok is unchanged
                    alone = restated(iq, mode_ref.with_mode(make_cfgs(1, **cfg, rssi=extra), mode)[0])
                    rec = (alone["flags"] & 8) != 0
                    _same(got[rec], alone[rec])
    assert stats["corrected"] > 20 and stats["failed"] > 0, stats
    assert stats["recovered_corrected"] > 0 or not mode[1], stats         # the symbol-spaced captures reach step 4 of the order


@pytest.mark.parametrize("name", [n for n in G.cases() if n.startswith("fuzz_")])
def test_emulator_equals_restatement_on_fuzz_goldens(name):
    z, cfg = G.load(name)
    cfg = dict(cfg)
    cfg.pop("rssi", None)
    cfg.setdefault("crc_init", 0x555555)
    for extra in (0, RECOVER, 2):
        check(z["iq"], make_cfgs(1, **cfg, rssi=extra | CORRECT))


def test_raw_mode_rejected_hits_and_degenerate_masks():
    iq, cfg = _ber_capture(18, 0, 37, n=40, seed=77)
    raw = make_cfgs(1, **cfg, raw=1, correct=1, recover=1)
    _same(check(iq, raw), orc.rx_flags(iq, 0, **cfg, raw=1))
    ref = orc.rx_flags(iq, 2, **cfg)
    got = check(iq, make_cfgs(1, **cfg, rssi=2, correct=1))
    rej = (ref["flags"] & 4) != 0
    assert rej.any()
    _same(got[rej], ref[rej])
    ok = ref["crc_bad"] == 0
    _same(got[ok], ref[ok])
    for mask in (0, 0xFF, 0xFFFF0000):
        check(iq, make_cfgs(1, **cfg, access_mask=mask, rssi=2, correct=1))


def test_exact_alternative_wins_over_a_correctable_primary():
    """a packet whose primary decode has one wrong bit (correctable) and whose alternative q = 0 is exact: the record is
    the recovered one, as without BTLE_CFG_CORRECT"""
    iq, cfg = _ber_capture(30, 0, 37, n=8, seed=9)
    clean = orc.rx_stream(iq, **cfg)
    r = clean[2]
    n0 = int(r["chunk"]) * 8192 + int(r["n0"])
    s = iq.reshape(-1, 2).astype(np.int32).copy()
    m = n0 + 4 * 60                                       # packet bit 60: a body bit of the primary decode
    i0, q0 = s[m]
    d = i0 * s[m + 1, 1] - s[m + 1, 0] * q0 > 0
    s[m + 1] = (q0, -i0) if d else (-q0, i0)              # flips d[m] only (as tests/test_recover.py's damaged_packet)
    iq2 = np.clip(s, -128, 127).astype(np.int8).reshape(-1)
    both = check(iq2, make_cfgs(1, **cfg, correct=1, recover=1))
    only_c = check(iq2, make_cfgs(1, **cfg, correct=1))
    only_r = check(iq2, make_cfgs(1, **cfg, recover=1))
    k = int(np.flatnonzero((both["chunk"] == r["chunk"]) & (both["n0"] == r["n0"]))[0])
    assert only_c[k]["flags"] & _native.REC_CORRECTED and only_c[k]["crc_bad"] == 0
    assert only_r[k]["flags"] & 8 and not only_r[k]["flags"] & _native.REC_CORRECTED
    assert both[k].tobytes() == only_r[k].tobytes()
    assert recover_ref.REC_RECOVERED == 8


def test_decode_connections_and_session_cfgs_pass_the_flag():
    """hop.decode_connections gives every receive cfg it makes BTLE_CFG_CORRECT when asked, and no other cfg; set_cfg /
    add_cfg's correct= sets and clears the bit"""
    from btle_b200 import hop
    from btle_b200.rx import _with_fields

    class Recorder:
        def __init__(self):
            self.cfgs = []

        def rx_batch(self, iq, cfgs, **kw):
            self.cfgs.append(np.array(cfgs))
            return np.zeros(0, dtype=_native.REC_DTYPE)

    for on in (False, True):
        r = Recorder()
        hop.decode_connections(r, np.zeros((40, 16384), dtype=np.int8), discover=False, correct=on)
        assert len(r.cfgs) == 1 and all(bool(f & CORRECT) == on for f in r.cfgs[0]["rssi"])
    c = make_cfgs(1, recover=1)
    assert _with_fields(c, {"correct": True})["rssi"][0] == RECOVER | CORRECT
    assert _with_fields(make_cfgs(1, correct=1), {"correct": False})["rssi"][0] == 0
