"""Connection discovery without a CONNECT_REQ: the empty-PDU candidate rule (numpy restatement, tests/discover_ref.py),
its BTLE_HD form through the CPU emulator, and the host logic of btle_b200/hop.py (discover_connections,
follow_connections(discover=True), hop_events) driven by an oracle-backed stand-in for BtleRx.  The checks named
check_* run again on the GPU with BtleRx (tests/test_discover_gpu.py)."""
import ctypes
import os
import subprocess

import numpy as np
import pytest
import torch

import discover_ref as R
from btle_b200 import CAND_DTYPE, synth
from btle_b200.hop import discover_connections, follow_connections, hop_events
from test_hop import _capture_with_many_connections, _place

AAS = (0x60850A1B, 0x50850A1C, 0x12345679, 0x8E89BED6)          # preamble 0x55 (bit 0 set) and 0xAA

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
EMUL_SRC = os.path.join(HERE, "emul", "btle_discover_emul.cpp")
EMUL_SO = os.path.join(HERE, "emul", "libbtle_discover_emul.so")      # built by __graft_entry__.build()
EMUL_DEPS = [EMUL_SRC, os.path.join(ROOT, "btle_b200", "csrc", "btle_core.cuh"), os.path.join(ROOT, "btle_b200", "csrc", "btle_params.h"),
             os.path.join(ROOT, "include", "btle_b200.h")]
_emul_lib = None


def _emul():
    """The CPU emulator of discover_kernel's per-lane logic (tests/emul/btle_discover_emul.cpp)."""
    global _emul_lib
    if _emul_lib is not None:
        return _emul_lib
    if (not os.path.exists(EMUL_SO)) or any(os.path.getmtime(EMUL_SO) < os.path.getmtime(d) for d in EMUL_DEPS):
        subprocess.run(["g++", "-O2", "-fPIC", "-shared", "-std=c++17", "-x", "c++", "-o", EMUL_SO, EMUL_SRC], check=True)
    L = _emul_lib = ctypes.CDLL(EMUL_SO)
    L.emul_discover.restype = ctypes.c_long
    L.emul_discover.argtypes = [ctypes.c_void_p, ctypes.c_long, ctypes.c_int, ctypes.c_int, ctypes.c_void_p, ctypes.c_long]
    L.emul_crc24_unwind.restype = ctypes.c_uint32
    L.emul_crc24_unwind.argtypes = [ctypes.c_uint32, ctypes.c_uint32, ctypes.c_int]
    return L


def emul_discover(iq, channel, stream=0):
    iq = np.ascontiguousarray(iq, dtype=np.int8)
    cap = iq.size // 8 + 64
    out = np.zeros(cap, dtype=CAND_DTYPE)
    n = _emul().emul_discover(iq.ctypes.data, iq.size, channel, stream, out.ctypes.data, cap)
    assert n <= cap
    out = out[:n]
    return out[np.argsort(out["sample"], kind="stable")]


def planted(channel, aa, crc_init=0x227BA7, at=3000, n_samples=8000, seed=1, header=(1, 0, 0, 0)):
    """Noise floor with one empty PDU (LLID, NESN, SN, MD = header) whose preamble starts at sample `at`."""
    gen = torch.Generator(); gen.manual_seed(seed)
    iq = synth.noise_floor(2 * n_samples, gen).numpy().copy()
    wav = synth.modulate(synth.air_bytes(synth.ll_data_pdu(*header, b""), channel, aa, crc_init)).astype(np.int32) * 64 // 127
    seg = iq[2 * at:2 * at + wav.size].astype(np.int32) + wav[:iq.size - 2 * at]
    iq[2 * at:2 * at + wav.size] = np.clip(seg, -128, 127).astype(np.int8)
    return iq


def edge_captures(channel=9, aa=0x60850A1B):
    """(tight, out_front, out_back): a capture cut so that the candidate at the burst's sample 40 reads d[0] as its first
    preamble bit and the last defined d[n] as its last CRC bit; and the same cut one sample further out at either end."""
    iq = planted(channel, aa, at=1000)
    n0 = 1040
    tight = iq[2 * (n0 - 32):2 * (n0 + 286)]
    return tight, iq[2 * (n0 - 31):2 * (n0 + 286)], iq[2 * (n0 - 32):2 * (n0 + 285)]


def many_connections(partial=False):
    """test_hop's six connections; partial=True adds a seventh whose channel map is partial (CSA#1 remapping onto
    channels 0..19), which discovery must report as untracked."""
    cap, truth = _capture_with_many_connections()
    if partial:
        aa, crci, hop, used = 0x3A5C96E1, 0x1F2E3D, 7, list(range(20))
        unmapped, t = 0, 0.004
        while t < 0.195:
            unmapped = (unmapped + hop) % 37
            ch = unmapped if unmapped in used else used[unmapped % len(used)]
            _place(cap, ch, t, synth.air_bytes(synth.ll_data_pdu(1, 0, 0, 0, b"\x01\x02"), ch, aa, crci), amp=62)
            _place(cap, ch, t + 0.0004, synth.air_bytes(synth.ll_data_pdu(1, 1, 0, 0, b""), ch, aa, crci), amp=62)
            t += 20 * 1.25e-3
        truth = truth + [dict(aa=aa, crci=crci, hop=None, interval=None)]
    return cap, truth


# ---- the rule --------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("aa", AAS)
def test_rule_finds_planted_empty_pdus_on_every_data_channel(aa):
    for ch in range(37):
        c = R.discover(planted(ch, aa, header=(1, ch & 1, (ch >> 1) & 1, (ch >> 2) & 1)), ch)
        hit = c[(c["sample"] >= 3030) & (c["sample"] <= 3050)]
        assert list(hit["sample"] - 3000) == [39, 40, 41], (ch, hit["sample"])
        assert (hit["access_addr"] == aa).all() and (hit["crc_init"] == 0x227BA7).all() and (hit["channel"] == ch).all()
        assert hit["header"][0, 0] & 3 == 1 and hit["header"][0, 1] == 0


def test_rule_edges():
    tight, front, back = edge_captures()
    c = R.discover(tight, 9)
    assert list(c["sample"]) == [32] and c["access_addr"][0] == 0x60850A1B and c["crc_init"][0] == 0x227BA7
    assert len(R.discover(front, 9)) == 0 and len(R.discover(back, 9)) == 0


def test_crc_init_recovery_round_trip():
    rng = np.random.default_rng(5)
    for _ in range(10000):
        header, init = rng.integers(0, 256, 2, dtype=np.uint8).tobytes(), int(rng.integers(0, 1 << 24))
        rx = synth.crc24(header, init)
        got = R.crc_init_for(header, rx)
        assert synth.crc24(header, got) == rx and got == init


def test_btle_hd_rule_equals_restatement():
    """The BTLE_HD functions the kernel runs (through the CPU emulator) == the numpy restatement."""
    L = _emul()
    rng = np.random.default_rng(2)
    for _ in range(2000):
        crc, bits = int(rng.integers(0, 1 << 24)), int(rng.integers(0, 1 << 16))
        assert L.emul_crc24_unwind(crc, bits, 16) == R.crc_unwind(crc, bits, 16)
    gen = torch.Generator(); gen.manual_seed(7)
    cases = [(synth.noise_floor(2 * 1000003, gen).numpy(), 5),
             (rng.integers(-128, 128, 2 * 4000000 + 3, dtype=np.int16).astype(np.int8), 17)]
    cases += [(planted(ch, aa, at=2000 + 37 * ch), ch) for ch in (0, 9, 36) for aa in AAS]
    cases += [(x, 9) for x in edge_captures()]
    for iq, ch in cases:
        a, b = R.discover(iq, ch), emul_discover(iq, ch)
        assert a.tobytes() == b.tobytes(), (ch, len(a), len(b))
    assert len(R.discover(cases[1][0], 17)) > 0                                 # full-scale noise does pass now and then


# ---- discovery and following (shared with the GPU file) --------------------------------------------------------------
def check_discover_connections(rx):
    cap, truth = many_connections(partial=True)
    cap[37:40] = 0
    found = discover_connections(rx, cap)
    tracked = [c for c in found if c["tracked"]]
    assert len(found) == 7 and len(tracked) == 6
    got = sorted((c["access_addr"], c["crc_init"], c["hop"], c["interval"]) for c in tracked)
    assert got == sorted((t["aa"], t["crci"], t["hop"], t["interval"]) for t in truth[:6])
    odd = next(c for c in found if not c["tracked"])
    assert (odd["access_addr"], odd["crc_init"], odd["hop"], odd["interval"]) == (truth[6]["aa"], truth[6]["crci"], None, None)
    for c in found:
        assert c["discovered"] and c["chm"] == "1fffffffff" and c["adv_channel"] is None and c["n_events"] >= 4
        assert c["n_candidates"] >= c["n_events"]
    # hop events: track_start at the first empty PDU's event on its channel, then one chan_change per event; none for
    # the untracked connection
    _, conns = follow_connections(rx, cap, discover=True)
    ev = hop_events(conns)
    assert {e["aa"] for e in ev} == {f"{t['aa']:08x}" for t in truth[:6]}
    for c in (c for c in conns if c["tracked"]):
        mine = [e for e in ev if e["aa"] == f"{c['access_addr']:08x}"]
        assert mine[0]["event"] == "track_start" and mine[0]["ts"] == c["t_first"] and mine[0]["ch"] == c["first_channel"]
        assert len(mine) == len(c["events"])


def _same_events(a, b, shift_s=0.0, first_t_hop=False):
    assert len(a) == len(b) and len(a) >= 4
    for k, (x, y) in enumerate(zip(a, b)):
        assert (x["channel"], x["anchored"], len(x["packets"])) == (y["channel"], y["anchored"], len(y["packets"])), k
        assert abs(x["t"] - y["t"] - shift_s) < 1e-9, k
        if k or first_t_hop:
            assert abs(x["t_hop"] - y["t_hop"] - shift_s) < 1e-9, k
        for p, q in zip(x["packets"], y["packets"]):
            assert p.tobytes()[8:] == q.tobytes()[8:]          # all but stream and chunk (compared through t)


def check_follow_discovered(rx):
    """Discovered walks == the CONNECT_REQ walks of the uncut capture: whole capture, and cut mid-connection."""
    cap, truth = many_connections()
    _, ref = follow_connections(rx, cap)
    ref = {c["access_addr"]: c for c in ref}
    zeroed = cap.copy()
    zeroed[37:40] = 0
    adv, conns = follow_connections(rx, zeroed, discover=True)
    assert len(adv) == 0 and len(conns) == 6
    for c in conns:
        _same_events(c["events"], ref[c["access_addr"]]["events"])
    # with the CONNECT_REQs present, those connections are followed once, from their CONNECT_REQ
    _, both = follow_connections(rx, cap, discover=True)
    _, plain = follow_connections(rx, cap)
    assert [c["events"] for c in both[:6]] == [c["events"] for c in plain]
    assert all("events" not in c for c in both[6:]) and len(both) == 12
    # cut at a chunk boundary between two events, mid-connection
    k = 24
    shift = k * 8192 / 4e6
    _, cut = follow_connections(rx, zeroed[:, k * 16384:].copy(), discover=True)
    assert len(cut) == 6
    for c in cut:
        full = ref[c["access_addr"]]["events"]
        j = next(i for i, e in enumerate(full) if e["anchored"] and e["t"] >= shift)
        _same_events(full[j:], c["events"], shift)


def check_noise_gives_nothing(rx):
    n = 40 * 16384
    gen = torch.Generator(); gen.manual_seed(9)
    floor = synth.noise_floor(40 * n, gen).numpy().reshape(40, n)
    uniform = np.random.default_rng(9).integers(-128, 128, (40, n), dtype=np.int16).astype(np.int8)
    for cap in (floor, uniform):
        assert discover_connections(rx, cap) == []
        assert discover_connections(rx, cap, min_events=1) != [] or cap is floor
        _, conns = follow_connections(rx, cap, discover=True)
        assert conns == []


def test_discover_connections_with_oracle_backend():
    check_discover_connections(R.OracleDiscoverRx())


def test_follow_discovered_connections_with_oracle_backend():
    check_follow_discovered(R.OracleDiscoverRx())


def test_noise_gives_no_connection_with_oracle_backend():
    check_noise_gives_nothing(R.OracleDiscoverRx())
