"""LE Coded PHY connections in hop.decode_connections(coded=True) without a GPU: the AUX_CONNECT_REQ parser on hand-built
PDUs, the rule that drops connections already known, the cfg layout of the several-cfgs-per-capture calls, and the whole
call on a CPU backend (the 1M oracle backends of test_rx_multi plus coded_ref.py run once per cfg) over a 40-channel
capture with 1M and coded connections.  tests/test_coded_connections_gpu.py runs the same capture on the GPU."""
import numpy as np
import torch

import coded_ref as cr
from btle_b200 import REC_DTYPE, synth
from btle_b200._native import MAX_CFGS_PER_CAPTURE
from btle_b200.hop import connection_cfgs, decode_connections, new_connections, parse_aux_connect_req, parse_connect_req
from test_hop import _place
from test_rx_multi import OracleMultiRx

ADV_AA, ADV_CRC = 0x8E89BED6, 0x555555


# ---- the restatement once per cfg, with the search done by FFT ----------------------------------------------------------
def _distances_fft(a_ph, spec, n_valid, access_addr):
    """D of one sample phase: a_ph = 2 h - 1 of that phase, spec its rfft (of length n_fft); the first n_valid windows"""
    p = 2 * cr.pattern(access_addr).astype(np.float64) - 1
    n_fft = 2 * (spec.size - 1)
    corr = np.fft.irfft(spec * np.conj(np.fft.rfft(p, n_fft)), n_fft)[:n_valid]
    return (p.size - np.rint(corr).astype(np.int64)) // 2


class _CapturePhases:
    """coded_ref.Capture plus the rfft of 2 h - 1 at each sample phase"""

    def __init__(self, iq, offset_hz):
        self.cap = cr.Capture(iq, offset_hz)
        a = 2 * self.cap.h.astype(np.float64) - 1
        self.a = [a[ph::4] for ph in range(4)]
        n_fft = 1 << int(np.ceil(np.log2(max(a.size // 4 + 1, 2) + 336)))
        self.spec = [np.fft.rfft(x, n_fft) for x in self.a]

    def distances(self, access_addr):
        """coded_ref.distances(), exactly"""
        N = self.cap.n
        D = np.full(N, -1, np.int64)
        lo, hi = 323, N - 1024
        if hi < lo:
            return D
        for ph in range(4):
            n0 = np.arange(lo + (ph - lo) % 4, hi + 1, 4)
            if n0.size == 0:
                continue
            m0, m1 = (n0[0] - ph) // 4, (n0[-1] - ph) // 4
            # window m reads a[ph::4][m - 80 .. m + 255]: the correlation from index m - 80
            d = _distances_fft(self.a[ph], self.spec[ph], m1 - 80 + 1, access_addr)
            D[n0] = d[m0 - 80:m1 - 80 + 1]
        return D


def _hits(D):
    """coded_ref.hits_from_distances(), evaluated only where D <= MAX_DIST"""
    N = D.size
    big = np.where(D < 0, 1 << 30, D)
    out = []
    for n in np.nonzero((D >= 0) & (D <= cr.MAX_DIST))[0]:
        d = big[n]
        if all((n - k < 0 or d < big[n - k]) and (n + k >= N or d <= big[n + k]) for k in range(1, 9)):
            out.append(int(n))
    return np.array(out, dtype=np.int64)


class CodedOracleRx(OracleMultiRx):
    """OracleMultiRx (rx_batch / discover / rx_multi on the oracles) plus rx_coded / rx_coded_multi as coded_ref.py run
    once per cfg: the definition of btle_b200_rx_coded_multi.  Captures are kept between calls by content."""

    def __init__(self):
        super().__init__()
        self.coded_calls = []
        self._caps = {}

    def _capture(self, iq, offset_hz):
        key = (iq.tobytes(), float(offset_hz))
        if key not in self._caps:
            self._caps[key] = _CapturePhases(iq, offset_hz)
        return self._caps[key]

    def rx_coded_multi(self, iq, cfgs, capture, offset_hz=None):
        iq = np.asarray(iq, dtype=np.int8)
        self.coded_calls.append((iq.shape[0], len(cfgs)))
        off = np.zeros(iq.shape[0], np.float32) if offset_hz is None else np.broadcast_to(np.asarray(offset_hz, np.float32), (iq.shape[0],))
        out = []
        for j, (cfg, c) in enumerate(zip(cfgs, capture)):
            cp = self._capture(iq[int(c)], float(off[int(c)]))
            D = cp.distances(int(cfg["access_addr"]))
            out += [cr.decode(cp.cap, int(n0), int(D[n0]), j, cfg) for n0 in _hits(D)]
        return np.array(out, dtype=cr.CODED_DTYPE) if out else np.zeros(0, cr.CODED_DTYPE)

    def rx_coded(self, iq, cfgs, offset_hz=None):
        return self.rx_coded_multi(iq, cfgs, np.arange(len(cfgs)), offset_hz)


def test_fft_search_equals_the_restatement():
    rng = np.random.default_rng(3)
    specs, n0 = [], 900
    for k in range(6):
        specs.append((n0 + k % 4, 5 + k, (2, 8)[k % 2]))
        n0 += 4 * (80 + 296 + (16 + 8 * (5 + k) + 27) * 8) + 700
    bursts = [(n, synth.coded_air(bytes([7, L]) + bytes(L), 5, 0x12345678, 0x222222, s=s)) for n, L, s in specs]
    iq = cr.place(n0 + 2000, bursts, 100, cr.sigma_of(2.0, 100), rng)
    cp = _CapturePhases(iq, 0.0)
    for aa in (0x12345678, ADV_AA, 0x71764129):
        D = cp.distances(aa)
        assert np.array_equal(D, cr.distances(cp.cap, aa))
        assert np.array_equal(_hits(D), cr.hits_from_distances(D))
    assert len(_hits(cp.distances(0x12345678))) >= 6


# ---- AUX_CONNECT_REQ ---------------------------------------------------------------------------------------------------
def _ll_data(aa, crc_init, interval=8, hop=9, init_a=bytes(range(6)), adv_a=bytes(range(6, 12)), chm=bytes.fromhex("ffffffff1f")):
    """InitA, AdvA and LLData of a CONNECT_IND / AUX_CONNECT_REQ (CRC init in the byte order parse_connect_req reads)"""
    return (init_a + adv_a + aa.to_bytes(4, "little") + crc_init.to_bytes(3, "big") + bytes([2]) + (3).to_bytes(2, "little") +
            interval.to_bytes(2, "little") + bytes(2) + (500).to_bytes(2, "little") + chm + bytes([hop | (2 << 5)]))


def _coded_rec(pdu, channel=17, sample=123456, crc_bad=0):
    r = np.zeros(1, cr.CODED_DTYPE)[0]
    r["sample"], r["channel"], r["crc_bad"], r["s"], r["n_bytes"] = sample, channel, crc_bad, 2, len(pdu) + 3
    r["bytes"][:len(pdu)] = np.frombuffer(pdu, np.uint8)
    return r


def test_aux_connect_req_parser():
    payload = _ll_data(0x50654E3A, 0x13579B, interval=24, hop=14)
    aux = synth.adv_pdu(5, 1, 1, payload)                      # TxAdd, RxAdd set: the type is the low nibble
    c = parse_aux_connect_req(_coded_rec(aux, channel=17, sample=400000))
    # the same fields as a CONNECT_IND with the same payload, t from the sample, the secondary channel, aux set
    r1 = np.zeros(1, dtype=REC_DTYPE)[0]
    r1["bytes"][:len(aux)] = np.frombuffer(aux, np.uint8)
    r1["channel"] = 38
    ref = parse_connect_req(r1)
    assert c["aux"] is True and c["t"] == 0.1 and c["adv_channel"] == 17
    assert {k: v for k, v in c.items() if k not in ("t", "adv_channel", "aux")} == {k: v for k, v in ref.items() if k not in ("t", "adv_channel")}
    assert c["access_addr"] == 0x50654E3A and c["crc_init"] == 0x13579B and c["interval"] == 24 and c["hop"] == 14 and c["sca"] == 2
    assert c["init_a"] == bytes(range(6))[::-1].hex() and c["chm"] == "1fffffffff" and c["win_offset"] == 3 and c["timeout"] == 500
    assert list(c)[:2] == ["t", "adv_channel"] and list(c)[2:-1] == list(ref)[2:]
    # refused: a failed CRC, another PDU type, another length (8-bit field: 34 + 64 is not 34), too short
    assert parse_aux_connect_req(_coded_rec(aux, crc_bad=1)) is None
    assert parse_aux_connect_req(_coded_rec(synth.adv_pdu(3, 0, 0, payload))) is None
    assert parse_aux_connect_req(_coded_rec(synth.adv_pdu(7, 0, 0, payload))) is None
    assert parse_aux_connect_req(_coded_rec(bytes([5, 34 + 64]) + payload)) is None
    assert parse_aux_connect_req(_coded_rec(synth.adv_pdu(5, 0, 0, payload[:33]))) is None


def test_known_connections_are_dropped_by_access_address_and_crc_init():
    known = [{"access_addr": 1, "crc_init": 10}, {"access_addr": 2, "crc_init": 20}]
    found = [{"access_addr": 1, "crc_init": 10, "n": 0},         # known: dropped
             {"access_addr": 1, "crc_init": 11, "n": 1},         # same access address, another CRC init: a new one
             {"access_addr": 3, "crc_init": 20, "n": 2},         # same CRC init, another access address: new
             {"access_addr": 3, "crc_init": 20, "n": 3},         # twice in found: the first one is kept
             {"access_addr": 2, "crc_init": 20, "n": 4}]
    assert [c["n"] for c in new_connections(known, found)] == [1, 2]
    assert new_connections([], []) == [] and [c["n"] for c in new_connections([], found)] == [0, 1, 2, 4]


def test_coded_batch_cfg_layout():
    for k in range(1, MAX_CFGS_PER_CAPTURE + 1):
        batch = [{"access_addr": 0x10000000 + i, "crc_init": 0x100 + i} for i in range(k)]
        cfgs, capture = connection_cfgs(batch)
        assert cfgs.size == capture.size == 37 * k and capture.dtype == np.int32
        j = np.arange(37 * k)
        assert np.array_equal(capture, j // k) and np.array_equal(cfgs["channel"], j // k)
        assert np.array_equal(cfgs["access_addr"], 0x10000000 + j % k) and np.array_equal(cfgs["crc_init"], 0x100 + j % k)
        assert (cfgs["rssi"] == 0).all() and (cfgs["raw"] == 0).all() and (cfgs["access_mask"] == 0xFFFFFFFF).all()
        assert (np.bincount(capture) == k).all() and (np.diff(capture) >= 0).all()
    # the 1M flags are passed to the 1M batches only
    cfgs, _ = connection_cfgs(batch, symbol_spaced=True, correct=True)
    assert (cfgs["rssi"] != 0).all()


# ---- the whole call -----------------------------------------------------------------------------------------------------
N_INT8 = 48 * 16384                 # 98 ms on every channel


class _Schedule:
    """Packets on the data channels that never overlap in time on one channel"""

    def __init__(self):
        self.busy = {ch: [] for ch in range(40)}

    def take(self, chans, t, dur):
        for ch in chans:
            if all(t + dur + 2e-4 < a or t - 2e-4 > b for a, b in self.busy[ch]):
                self.busy[ch].append((t, t + dur))
                return ch
        raise AssertionError("no free channel")


def _place_coded(cap, ch, t, wav, amp=100):
    """a coded_air() burst whose access address lands at sample round(t * 4 Msps) of capture row ch; returns that sample"""
    n0 = int(round(t * 4e6))
    w = wav.astype(np.int32) * amp // 127
    p = 2 * (n0 - synth.CODED_AA_SAMPLE)
    seg = cap[ch, p:p + w.size].astype(np.int32) + w[:cap.shape[1] - p]
    cap[ch, p:p + w.size] = np.clip(seg, -128, 127).astype(np.int8)
    return n0


def coded_connections_capture():
    """40 channels, 98 ms:
      A     a CONNECT_REQ connection that sends 1M packets, then coded ones (S=8 and S=2 alternating);
      B..G  six more CONNECT_REQ connections with 1M packets only;
      D'    a connection without CONNECT_REQ (empty PDUs on 5 events, CSA#1), then coded packets;
      H,I,J three AUX_CONNECT_REQs on coded secondary channels (S=8, S=2, S=8), then coded packets; I also sends 1M;
      dup   an AUX_CONNECT_REQ with A's access address and CRC init (a known connection: dropped).
    11 connections, so the 1M and the coded connection calls run in two batches each.  Returns (captures, truth):
    truth["coded"][aa] = [(channel, n0, s, pdu)] of every coded packet sent on a data channel, truth["m1"][aa] =
    [(channel, t)] of the 1M packets with a payload, truth["aux"] = [(aa, crc_init, channel)] of the AUX_CONNECT_REQs."""
    gen = torch.Generator(); gen.manual_seed(23)
    cap = synth.noise_floor(40 * N_INT8, gen).numpy().reshape(40, N_INT8).copy()
    rng = np.random.default_rng(29)
    sched = _Schedule()
    truth = {"coded": {}, "m1": {}, "aux": [], "creq": []}

    def m1(aa, crc, t, payload, chans):
        pdu = synth.ll_data_pdu(2, 0, 0, 0, payload)
        air = synth.air_bytes(pdu, 0, aa, crc)
        ch = sched.take(chans, t, (len(air) * 8 + 8) * 1e-6)
        _place(cap, ch, t, synth.air_bytes(pdu, ch, aa, crc), amp=62)
        truth["m1"].setdefault(aa, []).append((ch, t))

    def coded(aa, crc, t, s, chans):
        L = int(rng.integers(3, 24))
        pdu = synth.ll_data_pdu(2, 0, 0, 0, rng.integers(0, 256, L, dtype=np.uint8).tobytes())
        ch = sched.take(chans, t - 1e-4, (80 + 296 + (16 + 8 * L + 27) * s) * 1e-6 + 1e-4)
        n0 = _place_coded(cap, ch, t, synth.coded_air(pdu, ch, aa, crc, s=s))
        truth["coded"].setdefault(aa, []).append((ch, n0, s, pdu))

    def chans(seed):
        return [int(x) for x in np.random.default_rng(seed).permutation(37)]

    # CONNECT_REQ connections A..G on the primary channels
    for i in range(7):
        aa, crc = 0x50850A1B + 0x01030507 * i, 0x227BA7 ^ (i * 0x010203)
        creq = synth.adv_pdu(5, 0, 0, _ll_data(aa, crc, interval=8, hop=5 + i))
        adv_ch = 37 + i % 3
        _place(cap, adv_ch, 0.002 + 0.0035 * i, synth.air_bytes(creq, adv_ch))
        truth["creq"].append((aa, crc))
        for e in range(3):
            m1(aa, crc, 0.028 + 0.0023 * i + 0.008 * e, bytes([i, e]) * (1 + e), chans(100 * i + e))
        if i == 0:
            for e in range(4):
                coded(aa, crc, 0.054 + 0.01 * e, (8, 2)[e % 2], chans(7 + e))
    # a connection without CONNECT_REQ: empty PDUs of both sides on five CSA#1 events 7.5 ms apart, then coded packets
    aa_d, crc_d, ch = 0x3A5C96E1, 0x1F2E3D, 0
    for e in range(5):
        ch = (ch + 7) % 37
        t = 0.021 + 0.0075 * e
        for q, dt in enumerate((0.0, 0.0004)):
            pdu = synth.ll_data_pdu(1, (e + q) & 1, e & 1, 0, b"")
            sched.take([ch], t + dt, 1e-4)
            _place(cap, ch, t + dt, synth.air_bytes(pdu, ch, aa_d, crc_d), amp=62)
    for e in range(3):
        coded(aa_d, crc_d, 0.066 + 0.009 * e, (2, 8)[e % 2], chans(50 + e))
    # AUX_CONNECT_REQs on coded secondary channels (their LLData names the connection), and A's again
    aux = [(0x71764129, 0x0BADC0, 3, 8), (0x2A3B4C5D, 0x13579B, 17, 2), (0x6B7A8F91, 0x2468AC, 30, 8), (0x50850A1B, 0x227BA7, 25, 2)]
    for q, (aa, crc, sec, s) in enumerate(aux):
        pdu = synth.adv_pdu(5, 0, 1, _ll_data(aa, crc, interval=12, hop=0, init_a=bytes([q] * 6)))
        t = 0.004 + 0.005 * q
        sched.take([sec], t - 1e-4, (80 + 296 + (16 + 8 * 34 + 27) * s) * 1e-6 + 1e-4)
        _place_coded(cap, sec, t, synth.coded_air(pdu, sec, ADV_AA, ADV_CRC, s=s))
        truth["aux"].append((aa, crc, sec))
        if q == 3:
            continue
        for e in range(3):
            coded(aa, crc, 0.030 + 0.015 * e + 0.004 * q, (8, 2)[(e + q) % 2], chans(200 + 10 * q + e))
        if q == 1:
            for e in range(2):
                m1(aa, crc, 0.080 + 0.006 * e, bytes([0xA5, e]), chans(300 + e))
    return cap, truth


def check_coded_connections(rx):
    """decode_connections(coded=True) on coded_connections_capture(): returns (adv, conns)"""
    cap, truth = coded_connections_capture()
    adv, conns = decode_connections(rx, cap, coded=True)
    by_key = {(c["access_addr"], c["crc_init"]): c for c in conns}
    assert len(conns) == len(by_key) == 11
    assert sorted((c["access_addr"], c["crc_init"]) for c in conns[:7]) == sorted(truth["creq"])     # in advertising-record order
    assert conns[7].get("discovered") and conns[7]["access_addr"] == 0x3A5C96E1 and conns[7]["crc_init"] == 0x1F2E3D
    aux = conns[8:]
    assert [(c["access_addr"], c["crc_init"], c["adv_channel"]) for c in aux] == truth["aux"][:3]
    assert all(c["aux"] and not c["tracked"] and c["interval"] == 12 for c in aux)
    assert [c["init_a"] for c in aux] == [bytes([q] * 6).hex() for q in range(3)]
    assert not any(c.get("aux") for c in conns[:8])
    # AUX_CONNECT_REQ time: the sample of its access address / 4 Msps
    for c, t in zip(aux, (0.004, 0.009, 0.014)):
        assert abs(c["t"] - t) < 1e-6
    n_coded = 0
    for c in conns:
        ct = c["coded_traffic"]
        assert (ct["access_addr"] == c["access_addr"]).all() and (ct["stream"] == ct["channel"]).all() and (ct["channel"] <= 36).all()
        assert np.array_equal(np.lexsort((ct["channel"], ct["sample"])), np.arange(ct.size))
        sent = truth["coded"].get(c["access_addr"], [])
        for ch, n0, s, pdu in sent:
            r = ct[(ct["channel"] == ch) & (np.abs(ct["sample"] - n0) <= 3)]
            assert len(r) == 1 and r[0]["crc_bad"] == 0 and r[0]["s"] == s, (hex(c["access_addr"]), ch, n0)
            assert bytes(r[0]["bytes"][:len(pdu)]) == pdu
        # nothing CRC-ok but the packets this connection sent
        ok = ct[ct["crc_bad"] == 0]
        assert len(ok) == len(sent), (hex(c["access_addr"]), len(ok), len(sent))
        n_coded += len(sent)
        # the 1M traffic of every connection, AUX_CONNECT_REQ ones included
        tr = c["traffic"]
        t1 = tr["chunk"].astype(np.int64) * 8192 + tr["n0"]
        for ch, ts in truth["m1"].get(c["access_addr"], []):
            s0 = int(round(ts * 4e6))
            assert len(tr[(tr["channel"] == ch) & (t1 >= s0 + 30) & (t1 <= s0 + 50) & (tr["crc_bad"] == 0)]) == 1, (hex(c["access_addr"]), ch, ts)
    assert n_coded == sum(len(v) for v in truth["coded"].values()) >= 16
    assert len(by_key[(0x50850A1B, 0x227BA7)]["coded_traffic"]) >= 4 and len(by_key[(0x2A3B4C5D, 0x13579B)]["traffic"]) >= 2
    # coded=False: what the call returned without the argument
    adv0, conns0 = decode_connections(rx, cap)
    assert adv0.tobytes() == adv.tobytes() and len(conns0) == 8
    for a, b in zip(conns0, conns[:8]):
        assert set(b) - set(a) == {"coded_traffic"} and a["traffic"].tobytes() == b["traffic"].tobytes()
        assert {k: v for k, v in a.items() if k != "traffic"} == {k: v for k, v in b.items() if k not in ("traffic", "coded_traffic")}
    return adv, conns


def test_decode_connections_coded_with_cpu_backend():
    rx = CodedOracleRx()
    check_coded_connections(rx)
    # one rx_coded over the 37 data captures, then one rx_coded_multi per 8 connections (8 + 3), 8 and 3 cfgs per capture
    assert rx.coded_calls == [(37, 37), (37, 37 * 8), (37, 37 * 3)]
    assert rx.multi_calls == 2 + 1                            # two 1M batches with coded=True, one without
