"""LE Coded PHY (include/btle_b200.h, "LE Coded PHY") on the CPU: the transmitter (btle_b200.synth.coded_symbols) and the
receiver's restatement (coded_ref.py), which the GPU records are pinned to in test_coded_gpu.py.

No third-party coded-PHY test vector is available, so the transmitter is pinned by the impulse response its polynomials
imply and by a preamble and block-1 layout worked out by hand from the spec."""
import numpy as np
import pytest

import coded_ref as cr
from btle_b200 import synth
from btle_b200._native import CFG_DTYPE, CODED_REC_DTYPE

AA = 0x8E89BED6


def _cfg(channel=37, aa=AA, crc_init=0x555555, rssi=0):
    c = np.zeros(1, CFG_DTYPE)
    c["channel"], c["access_addr"], c["access_mask"], c["crc_init"], c["rssi"] = channel, aa, 0xFFFFFFFF, crc_init, rssi
    return c


def _pdu(L, seed=0):
    rng = np.random.default_rng(seed + L)
    return bytes([0x07, L]) + rng.integers(0, 256, L, dtype=np.uint8).tobytes()


def test_record_layout():
    assert cr.CODED_DTYPE == CODED_REC_DTYPE and CODED_REC_DTYPE.itemsize % 16 == 0


def test_encoder_impulse_response():
    coded, st = synth.conv_encode([1, 0, 0, 0])
    assert coded.reshape(4, 2).tolist() == [[1, 1], [1, 0], [1, 1], [1, 1]]
    assert st == 0


def test_encoder_terminates():
    rng = np.random.default_rng(1)
    for _ in range(50):
        bits = rng.integers(0, 2, int(rng.integers(1, 40)))
        _, st = synth.conv_encode(np.concatenate([bits, [0, 0, 0]]))
        assert st == 0


def test_preamble_and_block1_layout():
    syms, packed = synth.coded_symbols(_pdu(0), 37, AA, s=8)
    assert syms[:80].tolist() == [0, 0, 1, 1, 1, 1, 0, 0] * 10
    # AA 0x8E89BED6 LSB first starts 0, 1, 1: from state 0 bit 0 codes (0, 0) -> 0011 0011; bit 1 from state 0 codes
    # (1, 1) -> 1100 1100; bit 2 from state 1 codes (0, 1) -> 0011 1100
    assert syms[80:104].tolist() == [0, 0, 1, 1, 0, 0, 1, 1, 1, 1, 0, 0, 1, 1, 0, 0, 0, 0, 1, 1, 1, 1, 0, 0]
    assert np.array_equal(syms[:336], cr.pattern(AA))
    assert np.array_equal(np.unpackbits(np.frombuffer(packed, np.uint8), bitorder="little")[:syms.size], syms)


@pytest.mark.parametrize("s", [2, 8])
@pytest.mark.parametrize("L", [0, 1, 37, 255])
def test_block_lengths(s, L):
    syms, packed = synth.coded_symbols(_pdu(L), 12, AA, s=s)
    assert syms.size == 80 + 296 + (16 + 8 * L + 27) * 2 * (1 if s == 2 else 4)
    assert len(packed) == (syms.size + 7) // 8


def _one(L, s, channel, phase, extra=2000, **kw):
    pdu = _pdu(L)
    wav = synth.coded_air(pdu, channel, AA, 0x123456, s=s)
    n0 = 1000 + phase
    n = n0 + wav.size // 2 + extra
    iq = cr.place(n, [(n0, wav)])
    return pdu, n0, iq


@pytest.mark.parametrize("s", [2, 8])
@pytest.mark.parametrize("L", [0, 1, 37, 38, 200, 255])
def test_noiseless_round_trip(L, s):
    for k, (channel, phase) in enumerate(zip([37, 39, 0, 36], [0, 1, 2, 3])):
        pdu, n0, iq = _one(L, s, channel, phase)
        recs = cr.rx_coded(iq, _cfg(channel, crc_init=0x123456, rssi=1))
        assert n0 in recs["sample"], (L, s, channel, phase, recs["sample"])
        # the coded payload can resemble P somewhere inside the packet: such a hit is a record too, and fails the CRC
        others = recs[recs["sample"] != n0]
        assert np.all(others["sample"] > n0) and np.all(others["crc_bad"] == 1)
        r = recs[recs["sample"] == n0][0]
        assert r["sample"] == n0 and r["dist"] == 0 and r["s"] == s and r["ci"] == synth.CODED_CI[s]
        assert r["crc_bad"] == 0 and r["flags"] == 0 and r["n_bytes"] == L + 5
        assert bytes(r["bytes"][:L + 2]) == pdu and not r["bytes"][L + 5:].any()
        assert r["mag_sum"] > 0


def test_viterbi_corrects_single_and_pair_flips():
    # S=2 block 2 of an empty PDU: 43 info bits, 86 coded bits; d_free = 6, so any 2 wrong signs are corrected
    rng = np.random.default_rng(5)
    info = np.concatenate([rng.integers(0, 2, 40), [0, 0, 0]]).astype(np.uint8)
    coded, _ = synth.conv_encode(info)
    base = (2 * coded.astype(np.int64) - 1) * 50
    n = coded.size
    flips = [(i,) for i in range(n)] + [(i, j) for i in range(n) for j in range(i + 1, n)]
    for f in flips:
        Ls = base.copy()
        Ls[list(f)] *= -1
        _, dec = cr.viterbi(Ls, 43)
        assert np.array_equal(cr.traceback(dec, 43, 0), info), f


@pytest.mark.parametrize("ci", [0, 1, 2, 3])
def test_ci_values(ci):
    s = 2 if ci == 1 else 8
    pdu = _pdu(20)
    wav = synth.coded_air(pdu, 37, AA, s=s, ci=ci)
    iq = cr.place(8000 + wav.size // 2, [(1003, wav)])
    r = cr.rx_coded(iq, _cfg())
    assert len(r) == 1 and r[0]["ci"] == ci and r[0]["sample"] == 1003
    if ci >= 2:
        assert r[0]["flags"] == cr.CI_RESERVED and r[0]["s"] == 0 and r[0]["n_bytes"] == 0 and r[0]["crc_bad"] == 1
        assert not r[0]["bytes"].any() and r[0]["metric"] == 0
    else:
        assert r[0]["crc_bad"] == 0 and bytes(r[0]["bytes"][:22]) == pdu


def test_hit_rule_on_crafted_distances():
    D = np.full(80, 200, np.int64)
    D[:3] = -1
    D[10] = 50                                   # a lone minimum
    D[20], D[25] = 40, 40                        # equal values 5 apart: the first one wins (left strict, right not)
    D[35], D[44] = 30, 30                        # 9 apart: both
    D[62], D[64] = 97, 96                        # only <= 96
    assert cr.hits_from_distances(D).tolist() == [10, 20, 35, 44, 64]
    E = np.full(30, -1, np.int64)
    E[10:20] = 96
    assert cr.hits_from_distances(E).tolist() == [10]       # undefined neighbours do not count
    F = np.full(30, 10, np.int64)
    F[15] = 9
    assert cr.hits_from_distances(F).tolist() == [0, 15]    # a plateau's first sample; n0 = 0 has no left neighbour


def test_window_edges_and_truncation():
    syms, _ = synth.coded_symbols(_pdu(10), 37, AA, s=8)
    wav = synth.coded_air(_pdu(10), 37, AA, s=8)
    n = 4000
    for n0, want in [(322, 0), (323, 1), (n - 1024, 1), (n - 1023, 0)]:
        iq = cr.place(n, [(n0, wav)])
        r = cr.rx_coded(iq, _cfg())
        got = [int(x) for x in r["sample"]]
        assert (n0 in got) == bool(want), (n0, got)
        if want:
            rec = r[got.index(n0)]
            assert rec["flags"] & cr.TRUNCATED
    # a packet that ends exactly inside is not truncated, one sample less is
    end = 1000 + 4 * (syms.size - 80 - 1) + 3
    for n, trunc in [(end + 1, 0), (end, cr.TRUNCATED)]:
        r = cr.rx_coded(cr.place(n, [(1000, wav)]), _cfg())
        assert len(r) == 1 and r[0]["flags"] == trunc and (trunc or r[0]["crc_bad"] == 0)


def test_no_false_alarm_on_random_bits():
    h = np.random.default_rng(9).integers(0, 2, 1_000_000 + 1346).astype(np.uint8)
    D = cr.distances_bits(h, AA)
    assert D[D >= 0].size == 1_000_000
    assert D[D >= 0].min() > cr.MAX_DIST
    assert cr.hits_from_distances(D).size == 0


def _distances_loop(h, access_addr):
    """D(n0) as the header states it: one pass over the capture per known symbol j = -80..255"""
    P = cr.pattern(access_addr)
    D = np.full(h.size, -1, np.int64)
    lo, hi = 323, h.size - 1024
    if hi >= lo:
        n0 = np.arange(lo, hi + 1)
        D[lo:hi + 1] = sum((h[n0 + 4 * j] != P[j + 80]).astype(np.int64) for j in range(-80, 256))
    return D


def test_fast_distances_equal_the_loop():
    rng = np.random.default_rng(13)
    for n in (0, 1346, 1347, 1348, 1349, 1350, 1351, 4096, 50_001):
        for aa in (AA, 0x12345678, 0xFFFFFFFF, 0):
            h = rng.integers(0, 2, n).astype(np.uint8)
            assert np.array_equal(cr.distances_bits(h, aa), _distances_loop(h, aa)), (n, hex(aa))
    # captures holding bursts at every phase, noiseless and noisy, at a corrected carrier offset
    specs, n0 = [], 700
    for k in range(8):
        specs.append((n0 + k % 4, _pdu(3 * k, seed=k), 2 + 6 * (k % 2)))
        n0 += 4 * (376 + (43 + 24 * k) * specs[-1][2]) + 900
    bursts = [(n, synth.coded_air(p, 37, AA, s=s)) for n, p, s in specs]
    for snr, hz in ((None, 0.0), (0.0, 0.0), (-4.0, 60e3)):
        rng = np.random.default_rng(17)
        iq = cr.place(n0 + 1500, bursts, 100, 0.0 if snr is None else cr.sigma_of(snr, 100), rng, offset_hz=hz)
        cap = cr.Capture(iq, hz)
        D = cr.distances(cap, AA)
        assert np.array_equal(D, _distances_loop(cap.h, AA))
        assert (D[[n for n, _, _ in specs]] <= (0 if snr is None else 120)).all()


def test_path_metric_of_the_decoded_bytes_is_the_viterbi_metric():
    rng = np.random.default_rng(19)
    for L, s in ((0, 2), (9, 8), (40, 2)):
        pdu = _pdu(L, seed=s)
        wav = synth.coded_air(pdu, 12, AA, 0x123456, s=s)
        iq = cr.place(1001 + wav.size // 2 + 1500, [(1001, wav)], 100, cr.sigma_of(1.0, 100), rng)
        cap = cr.Capture(iq)
        r = cr.rx_coded(iq, _cfg(12, crc_init=0x123456))
        r = r[np.abs(r["sample"] - 1001) <= 3][0]
        n0 = int(r["sample"])
        assert r["s"] == s and r["n_bytes"] == L + 5
        assert cr.path_metric(cap, n0, s, bytes(r["bytes"][:L + 5]), 12) == r["metric"]
        crc = synth.crc24(pdu, 0x123456)
        sent = pdu + bytes([crc & 0xFF, (crc >> 8) & 0xFF, crc >> 16])
        assert cr.path_metric(cap, n0, s, sent, 12) <= r["metric"]


PER_SNR_DB = -3.0     # the GPU sensitivity point (test_coded_gpu.py): S=8 still decodes, the 1M chain does not
PER_S8_BOUND = 0.5     # its bound: twice what this run may measure


def per_run(s, snr_db, n_packets, seed, amplitude=100):
    rng = np.random.default_rng(seed)
    bad = 0
    for k in range(n_packets):
        pdu = _pdu(int(rng.integers(0, 38)), seed=int(rng.integers(1 << 30)))
        wav = synth.coded_air(pdu, 37, AA, s=s)
        n0 = 700 + k % 4
        iq = cr.place(n0 + wav.size // 2 + 1200, [(n0, wav)], amplitude, cr.sigma_of(snr_db, amplitude), rng)
        r = cr.rx_coded(iq, _cfg())
        ok = [x for x in r if x["sample"] == n0 or abs(int(x["sample"]) - n0) <= 3]
        bad += not any(x["crc_bad"] == 0 and bytes(x["bytes"][:len(pdu)]) == pdu for x in ok)
    return bad / n_packets


def test_small_per_run():
    per8 = per_run(8, PER_SNR_DB, 40, 1)
    assert per8 <= PER_S8_BOUND / 2, per8
    assert per_run(8, 15.0, 10, 2) == 0.0 and per_run(2, 15.0, 10, 3) == 0.0
