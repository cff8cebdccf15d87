"""LE Coded PHY connection discovery without a GPU: the restatement tests/coded_discover_ref.py of include/btle_b200.h
("Coded connection discovery") on noiseless and noisy coded bursts, at every data channel and sample phase, at the ladder
positions and the window edges, on packets that must give nothing and on noise; and hop.decode_connections(coded=True,
coded_discover=True) on a CPU backend.  tests/test_coded_discover_gpu.py checks the GPU against the same restatement."""
import numpy as np
import pytest

import coded_discover_ref as cd
import coded_ref as cr
from btle_b200 import CODED_CAND_DTYPE, synth
from btle_b200.hop import _group_candidates, decode_connections, discover_coded_connections
from discover_ref import crc_init_for
from test_coded_connections import CodedOracleRx, _place_coded, coded_connections_capture

GAP = 4 * (80 + 296 + 43 * 8) + 2500        # samples between two bursts of one capture


def empty_burst(rng, channel, s, aa=None, crc=None, header0=None):
    aa = int(rng.integers(0, 1 << 32)) if aa is None else aa
    crc = int(rng.integers(0, 1 << 24)) if crc is None else crc
    h0 = int(rng.choice([1, 5, 9, 13])) if header0 is None else header0      # LLID 1 with NESN / SN / MD bits
    return aa, crc, bytes([h0, 0]), synth.coded_air(bytes([h0, 0]), channel, aa, crc, s=s)


def check_cand(r, n0, aa, crc, hdr, s, channel, stream=0):
    assert (int(r["sample"]), int(r["stream"]), int(r["access_addr"]), int(r["crc_init"]), int(r["channel"])) == (n0, stream, aa, crc, channel)
    assert bytes(r["header"]) == hdr and int(r["s"]) == s and 0 <= int(r["dist"]) <= cd.T_Q


def test_dtype_is_the_library_one():
    assert cd.CODED_CAND_DTYPE == CODED_CAND_DTYPE
    assert CODED_CAND_DTYPE.fields["header"][1] == 21 and CODED_CAND_DTYPE.fields["s"][1] == 23


@pytest.mark.parametrize("channel", range(37))
def test_clean_empty_pdus_every_channel_phase_and_s(channel):
    rng = np.random.default_rng(channel)
    bursts, truth, n0 = [], [], 1000
    for k in range(8):                                   # phases 0..3 at S=8 and S=2
        s, n = (8, 2)[k // 4], n0 + k % 4
        aa, crc, hdr, wav = empty_burst(rng, channel, s)
        bursts.append((n, wav))
        truth.append((n, aa, crc, hdr, s))
        n0 += GAP
    iq = cr.place(n0 + 3000, bursts, 100)
    c = cd.discover_capture(iq, channel)
    assert len(c) == len(truth)
    for r, t in zip(c, truth):
        check_cand(r, t[0], t[1], t[2], t[3], t[4], channel)
        assert int(r["shift"]) == 0 or abs(int(r["shift"])) <= cd.SHIFTS


def test_the_ladder_is_realigned():
    """every position n0 + 32 k of the ladder of a clean packet decodes to n0 itself"""
    rng = np.random.default_rng(5)
    for s in (8, 2):
        aa, crc, hdr, wav = empty_burst(rng, 11, s)
        n0 = 2001
        iq = cr.place(n0 + GAP, [(n0, wav)], 100)
        cap = cr.Capture(iq)
        Dpre, Q = cd.statistics(cap.h)
        ladder = [n0 + 32 * k for k in range(-4, 5)]
        assert all(Q[n] >= Q[n0] for n in ladder) and max(Q[n] for n in ladder) > Q[n0]
        for k, n in zip(range(-4, 5), ladder):
            r = cd.decode_hit(cap, n, int(Q[n]), 0, 11)
            check_cand(r, n0, aa, crc, hdr, s, 11)
            assert int(r["shift"]) == -k


def test_packets_that_give_no_candidate():
    """non-empty PDUs, reserved CIs, a wrong LLID and 1M packets"""
    rng = np.random.default_rng(7)
    bursts, n0 = [], 1000
    for s in (8, 2):
        bursts.append((n0, synth.coded_air(bytes([2, 5]) + bytes(5), 9, 0x1234567, 0x55AA55, s=s))); n0 += GAP + 400
        bursts.append((n0, synth.coded_air(bytes([1, 3]) + bytes(3), 9, 0x7654321, 0x55AA55, s=s))); n0 += GAP + 400
        bursts.append((n0, synth.coded_air(bytes([2, 0]), 9, 0x7654321, 0x55AA55, s=s))); n0 += GAP   # LLID 2
    for ci in (2, 3):
        bursts.append((n0, synth.coded_air(bytes([1, 0]), 9, 0x2468ACE, 0x13579B, s=8, ci=ci))); n0 += GAP
    iq = cr.place(n0 + 3000, bursts, 100)
    assert len(cd.discover_capture(iq, 9)) == 0
    # 1M empty PDUs on the same channel
    cap = np.zeros(2 * 60000, np.int8)
    for k in range(6):
        air = synth.modulate(synth.air_bytes(synth.ll_data_pdu(1, k & 1, 0, 0, b""), 9, 0x50654321, 0x123456))
        p = 2 * (2000 + 9000 * k + k % 4)
        cap[p:p + air.size] = air
    assert len(cd.discover_capture(cap, 9)) == 0


@pytest.mark.parametrize("s", [8, 2])
def test_window_edges(s):
    rng = np.random.default_rng(s)
    aa, crc, hdr, wav = empty_burst(rng, 20, s)
    per = 4 if s == 8 else 1
    # the first sample at which a window may start
    iq = cr.place(3000, [(cd.LO, wav)], 100)
    c = cd.discover_capture(iq, 20)
    assert len(c) == 1
    check_cand(c[0], cd.LO, aa, crc, hdr, s, 20)
    # the capture's end: the last sample of block 2's 43 steps must be inside
    n0 = 1500
    n_need = n0 + 4 * (296 + 86 * per - 1) + 4
    full = cr.place(n_need + 2000, [(n0, wav)], 100)
    c = cd.discover_capture(full[:2 * n_need], 20)
    assert len(c) == 1
    check_cand(c[0], n0, aa, crc, hdr, s, 20)
    c = cd.discover_capture(full[:2 * n_need - 2], 20)
    assert all(int(r["sample"]) != n0 for r in c)
    # too short for any window
    assert len(cd.discover_capture(np.zeros(2 * (cd.LO + cd.SPAN - 1), np.int8), 20)) == 0
    assert cd.statistics(np.zeros(cd.LO + cd.SPAN, np.uint8))[1][cd.LO] >= 0


def test_crc_init_round_trip():
    rng = np.random.default_rng(9)
    for _ in range(200):
        hdr = bytes([int(rng.integers(0, 256)), int(rng.integers(0, 256))])
        crc_init = int(rng.integers(0, 1 << 24))
        assert crc_init_for(hdr, synth.crc24(hdr, crc_init)) == crc_init


def test_snr_plus_4_db_every_packet():
    """at +4 dB every empty PDU of a noisy capture gives its candidate (within 3 samples of its n0)"""
    rng = np.random.default_rng(13)
    for s in (8, 2):
        bursts, truth, n0 = [], [], 1500
        for k in range(12):
            aa, crc, hdr, wav = empty_burst(rng, 4, s)
            bursts.append((n0 + k % 4, wav))
            truth.append((n0 + k % 4, aa, crc))
            n0 += GAP
        iq = cr.place(n0 + 3000, bursts, 100, cr.sigma_of(4.0, 100), rng)
        c = cd.discover_capture(iq, 4)
        for n, aa, crc in truth:
            assert any(abs(int(r["sample"]) - n) <= 3 and int(r["access_addr"]) == aa and int(r["crc_init"]) == crc for r in c)


@pytest.mark.parametrize("sigma", [3.0, 40.0])
def test_noise_gives_nothing(sigma):
    rng = np.random.default_rng(int(sigma))
    iq = np.clip(np.round(rng.normal(0, sigma, 2 * 200000)), -128, 127).astype(np.int8)
    cap = cr.Capture(iq)
    Dpre, Q = cd.statistics(cap.h)
    q = Q[Q >= 0]
    assert 120 < q.mean() < 146 and q.min() > cd.T_Q
    assert len(cd.hits(Dpre, Q)) == 0
    assert len(cd.discover_capture(iq, 3, cap=cap)) == 0


def test_grouping_is_discover_connections_own():
    """_group_candidates() on coded candidates: the rule discover_connections() applies to 1M ones"""
    c = np.zeros(6, CODED_CAND_DTYPE)
    c["access_addr"], c["crc_init"] = 0x11223344, 0xABCDEF
    c["sample"] = [4000, 4400, 40000, 70000, 100000, 130000]
    c["channel"] = [3, 3, 10, 17, 24, 31]
    conns = _group_candidates(c, 4)
    assert len(conns) == 1 and conns[0]["n_events"] == 5 and conns[0]["n_candidates"] == 6
    assert _group_candidates(c[:4], 4) == []


# ---- decode_connections(coded=True, coded_discover=True) on a CPU backend --------------------------------------------------
CODED_ONLY = [(0x4D3C2B1A, 0x0F1E2D, 8, [1, 5, 9, 13, 20]), (0x5E6F7081, 0x3C4B5A, 2, [2, 6, 10, 14, 21])]


def coded_discover_capture():
    """coded_connections_capture() (CONNECT_REQ, discovered, AUX_CONNECT_REQ connections; 1M and coded traffic) plus two
    coded-only connections without AUX_CONNECT_REQ: empty coded PDUs (S=8 and S=2) on five events 3 ms apart on five
    channels, in the first 14 ms, where the data channels carry nothing else.  Returns (captures, truth) with
    truth["coded_only"] = [(aa, crc, [(channel, n0, s, pdu)])]."""
    cap, truth = coded_connections_capture()
    cap = cap.copy()
    truth["coded_only"] = []
    for q, (aa, crc, s, chans) in enumerate(CODED_ONLY):
        sent = []
        for e, ch in enumerate(chans):
            pdu = synth.ll_data_pdu(1, e & 1, (e + q) & 1, 0, b"")
            n0 = _place_coded(cap, ch, 0.001 + 0.0002 * q + 0.003 * e, synth.coded_air(pdu, ch, aa, crc, s=s))
            sent.append((ch, n0, s, pdu))
        truth["coded_only"].append((aa, crc, sent))
    return cap, truth


class CodedDiscoverOracleRx(CodedOracleRx):
    """CodedOracleRx plus discover_coded as the restatement, on the same kept captures"""

    def __init__(self):
        super().__init__()
        self.discover_coded_calls = 0

    def discover_coded(self, iq, channels, offset_hz=None):
        self.discover_coded_calls += 1
        iq = np.asarray(iq, dtype=np.int8)
        off = np.zeros(iq.shape[0], np.float32) if offset_hz is None else np.broadcast_to(np.asarray(offset_hz, np.float32), (iq.shape[0],))
        ch = np.broadcast_to(np.asarray(channels, np.int32), (iq.shape[0],))
        parts = [cd.discover_capture(iq[s], int(ch[s]), s, cap=self._capture(iq[s], float(off[s])).cap) for s in range(iq.shape[0])]
        return np.concatenate(parts)


def check_coded_discover_connections(rx):
    """decode_connections(coded=True, coded_discover=True) on coded_discover_capture(): returns (adv, conns)"""
    cap, truth = coded_discover_capture()
    adv, conns = decode_connections(rx, cap, coded=True, coded_discover=True)
    assert len(conns) == 13 and len({(c["access_addr"], c["crc_init"]) for c in conns}) == 13
    assert not any(c.get("coded") for c in conns[:11])
    found = conns[11:]
    assert [(c["access_addr"], c["crc_init"]) for c in found] == [(aa, crc) for aa, crc, _ in truth["coded_only"]]
    for c, (aa, crc, sent) in zip(found, truth["coded_only"]):
        assert c["discovered"] and c["coded"] and not c["tracked"] and c["n_events"] == 5 and c["hop"] is None
        assert len(c["traffic"]) == 0 or (c["traffic"]["crc_bad"] != 0).all()
        ct = c["coded_traffic"]
        ok = ct[ct["crc_bad"] == 0]
        assert len(ok) == len(sent)
        for (ch, n0, s, pdu), r in zip(sorted(sent, key=lambda x: x[1]), ok):
            assert int(r["channel"]) == ch and abs(int(r["sample"]) - n0) <= 3 and int(r["s"]) == s
            assert bytes(r["bytes"][:2]) == pdu
    return adv, conns


def test_decode_connections_coded_discover_cpu_backend():
    rx = CodedDiscoverOracleRx()
    adv, conns = check_coded_discover_connections(rx)
    assert rx.discover_coded_calls == 1
    # without coded_discover: the result and the coded calls of coded=True alone
    rx0 = CodedDiscoverOracleRx()
    adv0, conns0 = decode_connections(rx0, coded_discover_capture()[0], coded=True)
    assert rx0.discover_coded_calls == 0 and len(conns0) == 11
    rx1 = CodedDiscoverOracleRx()
    adv1, conns1 = decode_connections(rx1, coded_discover_capture()[0], coded=True, coded_discover=False)
    assert rx1.discover_coded_calls == 0 and rx1.coded_calls == rx0.coded_calls
    assert adv1.tobytes() == adv0.tobytes() and adv.tobytes() == adv0.tobytes()
    for a, b, c in zip(conns1, conns0, conns):
        assert set(a) == set(b) == set(c)
        for k in a:
            if isinstance(a[k], np.ndarray):
                assert a[k].tobytes() == b[k].tobytes() == c[k].tobytes(), k
            else:
                assert a[k] == b[k] == c[k], k


def test_discover_coded_connections_offsets_pass_through():
    class Rec:
        def __init__(self):
            self.kw = None

        def discover_coded(self, iq, channels, **kw):
            self.kw = kw
            assert iq.shape[0] == 37 and list(channels) == list(range(37))
            return np.zeros(0, CODED_CAND_DTYPE)

    r = Rec()
    cap = np.zeros((40, 64), np.int8)
    assert discover_coded_connections(r, cap) == [] and r.kw == {}
    discover_coded_connections(r, cap, offset_hz=np.arange(40) * 1000.0)
    assert np.array_equal(r.kw["offset_hz"], np.arange(37) * 1000.0)
