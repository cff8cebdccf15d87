"""Several cfgs per capture (btle_b200_rx_multi) without a GPU: the kernel's multi-cfg unit path on the CPU emulator
(tests/emul/btle_emul.cpp) against the oracle run once per cfg, and hop.decode_connections() on an oracle backend."""
import time

import numpy as np
import pytest
import torch

import discover_ref as R
import emul
import orc
from btle_b200 import synth
from btle_b200._native import MAX_CFGS_PER_CAPTURE, REC_DTYPE
from btle_b200.hop import decode_connections, record_time
from btle_b200.rx import make_cfgs
from test_hop import _place


def oracle_multi(iq2d, cfgs, capture):
    """rx_batch() on iq2d[capture] with cfgs, through the oracle: the definition of rx_multi()."""
    out = [orc.rx_flags(iq2d[int(c)], int(cfg["rssi"]), channel=int(cfg["channel"]), access_addr=int(cfg["access_addr"]),
                        access_mask=int(cfg["access_mask"]), crc_init=int(cfg["crc_init"]), raw=int(cfg["raw"]), stream=j)
           for j, (cfg, c) in enumerate(zip(cfgs, capture))]
    return np.concatenate(out) if out else np.zeros(0, dtype=REC_DTYPE)


# ---- cases (shared with the GPU file) ---------------------------------------------------------------------------------
def _traffic(n_int8, channels, aas, seed, straddle=True):
    """Captures with bursts of several access addresses on each channel, over the reference capture's noise floor."""
    gen = torch.Generator(); gen.manual_seed(seed)
    iq = synth.noise_floor(len(channels) * n_int8, gen).numpy().reshape(len(channels), n_int8).copy()
    rng = np.random.default_rng(seed)
    for s, ch in enumerate(channels):
        t = 0.0002
        while 2 * int((t + 0.0006) * 4e6) < n_int8:
            aa = int(aas[rng.integers(len(aas))])
            crci = 0x555555 if ch >= 37 else 0x227BA7 ^ (aa & 0xFFFF)
            pdu = (synth.adv_pdu(0, 1, 0, rng.integers(0, 256, 6 + int(rng.integers(0, 20)), dtype=np.uint8).tobytes()) if ch >= 37
                   else synth.ll_data_pdu(1 + int(rng.integers(0, 2)), 0, 0, 0, rng.integers(0, 256, int(rng.integers(0, 27)), dtype=np.uint8).tobytes()))
            air = bytearray(synth.air_bytes(pdu, ch, aa, crci))
            if rng.random() < 0.15:
                air[-1] ^= 0x10                                  # CRC must fail
            _place(iq, s, t, bytes(air), amp=int(rng.integers(30, 90)))
            t += float(rng.uniform(0.0006, 0.0013))
    return iq


def multi_cases():
    """(name, iq2d, cfgs, capture): K = 1..8 random AAs and masks (mask 0 included), advertising and data channels, raw,
    RSSI and -v, one AA twice with different CRC inits, ragged and tiny captures, captures no cfg reads."""
    rng = np.random.default_rng(21)
    cases = []
    base_aas = [0x8E89BED6, 0x60850A1B, 0x50850A1C, 0x12345679, 0x3A5C96E1, 0x71764129, 0x23AF04C8, 0x5A5AC3C3]
    n = 20 * 16384 + 5000
    iq = _traffic(n, [37, 5, 38, 22], base_aas[:5], seed=3)
    for K in range(1, MAX_CFGS_PER_CAPTURE + 1):
        cfgs, cap = [], []
        for s, ch in enumerate([37, 5, 38, 22]):
            for k in range(K):
                aa = base_aas[k] if k < 5 or rng.random() < 0.5 else int(rng.integers(0, 1 << 32))
                mask = [0xFFFFFFFF, 0xFFFFFFFF, 0xFFFF00FF, 0x0000FFFF, 0xFFFFFFF0, 0, 0xFFFFFFFF, 0x7FFFFFFE][(k + s) % 8]
                cfgs.append((ch, aa, mask, 0x555555 if ch >= 37 else 0x227BA7 ^ (aa & 0xFFFF), int(k == 3), [0, 1, 2, 3][(k + K) % 4]))
                cap.append(s)
        c = make_cfgs(len(cfgs))
        for j, v in enumerate(cfgs):
            c[j] = v
        # K = 1: one more capture, which no cfg reads, keeps the list from mapping cfg j to capture j (the single-cfg kernel)
        cases.append((f"K{K}", iq if K > 1 else np.concatenate([iq, iq[:1]]), c, np.array(cap, dtype=np.int32)))
    # one AA twice with different CRC inits (a discovery noise group), different channels on one capture
    c = make_cfgs(4, channel=[5, 5, 6, 5], access_addr=[0x60850A1B, 0x60850A1B, 0x60850A1B, 0x50850A1C],
                  crc_init=[0x227BA7 ^ 0x0A1B, 0x123456, 0x227BA7 ^ 0x0A1B, 0x227BA7 ^ 0x0A1C], rssi=[1, 0, 1, 2])
    cases.append(("dup-aa", iq, c, np.array([1, 1, 1, 1], dtype=np.int32)))
    # captures no cfg reads, a capture read by cfgs on the far side of it
    c = make_cfgs(3, channel=[37, 22, 22], access_addr=[0x8E89BED6, 0x12345679, 0x3A5C96E1], crc_init=[0x555555, 0x227BA7 ^ 0x5679, 0x227BA7 ^ 0x96E1])
    cases.append(("skip", iq, c, np.array([0, 3, 3], dtype=np.int32)))
    # ragged and tiny captures (single chunks, pieces of spans), mask 0 with -v on advertising channels
    for name, m in (("tiny", 16384), ("two", 2 * 16384 + 77), ("ragged", 7 * 16384 + 300)):
        q = np.ascontiguousarray(iq[:, :m])
        c = make_cfgs(5, channel=[37, 37, 37, 5, 38], access_addr=[0x8E89BED6, 0x60850A1B, 0x8E89BED6, 0x12345679, 0x8E89BED6],
                      access_mask=[0xFFFFFFFF, 0xFFFFFFFF, 0, 0xFFFFFFFF, 0xFFFFFFFF], rssi=[1, 0, 2, 1, 3],
                      crc_init=[0x555555, 0x555555, 0x555555, 0x227BA7 ^ 0x5679, 0x555555])
        cases.append((name, q, c, np.array([0, 0, 0, 1, 2], dtype=np.int32)))
    return cases


@pytest.mark.parametrize("case", multi_cases(), ids=lambda c: c[0])
def test_multi_cfg_unit_path_equals_oracle_per_cfg(case):
    _, iq, cfgs, capture = case
    exp = oracle_multi(iq, cfgs, capture)
    for grid in (132, 7):                                      # whole spans, and pieces of them
        got = emul.rx_multi(iq, cfgs, capture, grid=grid)
        assert got.tobytes() == exp.tobytes(), (grid, len(got), len(exp))
    assert len(exp) > 0


def test_multi_cfg_unit_path_fuzz_equals_oracle_per_cfg():
    """Random launches of tests/multi_fuzz.py (the generator of tools/fuzz_multi_gpu.py, at most 12 captures of 16
    chunks) for about 15 s, each at grid 132 and at a random grid, against the oracle per cfg."""
    from multi_fuzz import draw
    rng = np.random.default_rng(20261016)
    t0, n, recs = time.time(), 0, 0
    while time.time() - t0 < 15 or n < 20:
        iq, cfgs, capture = draw(rng, max_captures=12, max_chunks=16)
        exp = oracle_multi(iq, cfgs, capture)
        for grid in (132, int(rng.integers(1, 300))):
            got = emul.rx_multi(iq, cfgs, capture, grid=grid)
            assert got.tobytes() == exp.tobytes(), (n, grid, iq.shape, cfgs.tolist(), capture.tolist(), len(got), len(exp))
        n, recs = n + 1, recs + len(exp)
    assert recs > 1000


def test_tapset_prefilter_equals_prefilter_any():
    rng = np.random.default_rng(4)
    words = rng.integers(0, 1 << 32, 4 * 4000, dtype=np.uint64).astype(np.uint32)
    sparse = words & rng.integers(0, 1 << 32, words.size, dtype=np.uint64).astype(np.uint32)
    for aa, mask in [(0x8E89BED6, 0xFFFFFFFF), (0x60850A1B, 0), (0x0000000F, 0xFFFFFFFF), (0xFFFFFFFF, 0x0000F00F), (0x12345679, 0x00000003)]:
        cfg = make_cfgs(1, access_addr=aa, access_mask=mask)
        for w in (words, sparse):
            assert emul.check_tapset(cfg, w) == 0, (hex(aa), hex(mask))


def test_bad_cfg_capture_is_refused():
    iq = np.zeros((2, 16384), dtype=np.int8)
    for cc in ([1, 0], [0, 2], [-1, 0], [0] * (MAX_CFGS_PER_CAPTURE + 1)):
        assert emul.rx_units(iq, make_cfgs(len(cc)), cc)[0] == -1


# ---- decode_connections ------------------------------------------------------------------------------------------------
class OracleMultiRx(R.OracleDiscoverRx):
    """rx_batch / discover on the oracle, rx_multi as the oracle run once per cfg."""

    def __init__(self):
        self.multi_calls = 0

    def rx_multi(self, iq, cfgs, capture):
        self.multi_calls += 1
        return oracle_multi(iq, cfgs, capture)


def connections_capture():
    """40 channels, 205 ms: (a) a CONNECT_REQ connection with a full map (CSA#1); (b) a connection on a partial map
    (CSA#1 remapped onto channels 0..19) and (c) one whose channels follow no CSA#1 sequence, both without CONNECT_REQ.
    Returns (captures, {aa: [(channel, t), ...] of every planted packet})."""
    n = 100 * 16384
    gen = torch.Generator(); gen.manual_seed(17)
    cap = synth.noise_floor(40 * n, gen).numpy().reshape(40, n).copy()
    planted = {}
    aa, crci, hop, interval = 0x60850A1B, 0x227BA7, 9, 16
    creq = synth.adv_pdu(5, 0, 0, bytes(range(12)) + aa.to_bytes(4, "little") + crci.to_bytes(3, "big") + bytes([2]) + (15).to_bytes(2, "little") +
                         interval.to_bytes(2, "little") + bytes(2) + (2000).to_bytes(2, "little") + bytes.fromhex("ffffffff1f") + bytes([hop | (5 << 5)]))
    _place(cap, 37, 0.002, synth.air_bytes(creq, 37))
    rng = np.random.default_rng(8)
    seqs = {}
    ch, seq = 0, []
    for _ in range(10):
        ch = (ch + hop) % 37
        seq.append(ch)
    seqs[(aa, crci, interval * 1.25e-3, 0.008)] = seq
    used, um, seq = list(range(20)), 0, []
    for _ in range(10):
        um = (um + 7) % 37
        seq.append(um if um in used else used[um % len(used)])
    seqs[(0x3A5C96E1, 0x1F2E3D, 0.025, 0.005)] = seq
    seqs[(0x71764129, 0x0BADC0, 0.0225, 0.011)] = [int(x) for x in rng.permutation(37)[:10]]
    for (a, k, iv, t0), seq in seqs.items():
        pk, t = [], t0
        for e, ch in enumerate(seq):
            if t > 0.195:
                break
            _place(cap, ch, t, synth.air_bytes(synth.ll_data_pdu(1, e & 1, e & 1, 0, bytes([e, 7] * (e % 4))), ch, a, k), amp=62)
            _place(cap, ch, t + 0.0004, synth.air_bytes(synth.ll_data_pdu(1, (e + 1) & 1, e & 1, 0, b""), ch, a, k), amp=62)
            pk += [(ch, t), (ch, t + 0.0004)]
            t += iv
        planted[a] = pk
    return cap, planted


def check_decode_connections(rx):
    cap, planted = connections_capture()
    adv, conns = decode_connections(rx, cap)
    assert len(adv) == 1
    by_aa = {c["access_addr"]: c for c in conns}
    assert len(conns) == 3 and set(by_aa) == set(planted)
    assert by_aa[0x60850A1B]["tracked"] and not by_aa[0x60850A1B].get("discovered")
    assert by_aa[0x3A5C96E1]["discovered"] and by_aa[0x71764129]["discovered"] and not by_aa[0x71764129]["tracked"]
    for a, pk in planted.items():
        tr = by_aa[a]["traffic"]
        assert (tr["access_addr"] == a).all() and (tr["channel"] <= 36).all() and (tr["stream"] == tr["channel"]).all()
        t = tr["chunk"].astype(np.int64) * 8192 + tr["n0"]
        assert (np.diff(t) >= 0).all()
        for ch, ts in pk:
            s = int(round(ts * 4e6))
            hit = tr[(tr["channel"] == ch) & (t >= s + 30) & (t <= s + 50) & (tr["crc_bad"] == 0)]
            assert len(hit) == 1, (hex(a), ch, ts)
        assert len(tr) >= len(pk) and all(record_time(r) > 0 for r in tr[:1])
    return adv, conns


def test_decode_connections_with_oracle_backend():
    rx = OracleMultiRx()
    check_decode_connections(rx)
    assert rx.multi_calls == 1                                 # three connections: one rx_multi call
