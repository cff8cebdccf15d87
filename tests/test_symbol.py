"""The symbol-spaced discriminator (BTLE_CFG_SYMBOL_SPACED) on the CPU: the dense warps' arithmetic in that mode (emulated
with the PTX semantics of prmt / dp2a, tests/emul/btle_symbol_emul.cpp) against the definition in include/btle_b200.h, and
the emulated unit path in that mode against the numpy restatement over the oracle chain (tests/symbol_ref.py)."""
import ctypes
import os

import numpy as np
import pytest

import golden_util
import mode_ref
import multi_fuzz
import offset_ref
import symbol_ref
import orc
import rx_ber_ref
from btle_b200 import _native, rx as rxmod
from emul import DEPS, HERE

EDGE = np.array([-128, -127, -64, -1, 0, 1, 63, 126, 127], dtype=np.int8)
OFFSETS = [0.0, 1.0, -1.0, 25e3, -25e3, 100e3, -100e3, 150e3, 300e3, -300e3, 499_999.0, 500e3, -500e3]
SO = os.path.join(HERE, "emul", "libbtle_symbol_emul.so")
SRC = os.path.join(HERE, "emul", "btle_symbol_emul.cpp")
_lib = None


def lib():
    global _lib
    if _lib is None:
        if (not os.path.exists(SO)) or any(os.path.getmtime(SO) < os.path.getmtime(d) for d in DEPS + [SRC]):
            import subprocess
            subprocess.run(["g++", "-O2", "-fPIC", "-shared", "-std=c++17", "-x", "c++", "-o", SO, SRC], check=True)
        _lib = ctypes.CDLL(SO)
        vp, lg = ctypes.c_void_p, ctypes.c_long
        _lib.emul_sym_phase_words.restype = None
        _lib.emul_sym_phase_words.argtypes = [vp, lg, lg, lg, lg, ctypes.c_int, ctypes.c_int, ctypes.c_int, vp]
        _lib.emul_rx_units_sym.restype = lg
        _lib.emul_rx_units_sym.argtypes = [vp, lg, lg, lg, vp, vp, lg, ctypes.c_int, ctypes.c_int, vp, lg, vp, lg, ctypes.POINTER(lg)]
    return _lib


def emul_bits(buf, at, n_int8, lead, g0, ng, hz=None):
    """d[128 g0 .. 128 (g0 + ng)) from the emulated dense pass; the capture is buf[at : at + n_int8], buf[at - lead : at]
    readable in front of it"""
    buf = np.ascontiguousarray(buf, dtype=np.int8)
    pd = np.zeros(4 * ng, dtype=np.uint32)
    c, s = (16384, 0) if hz is None else offset_ref.rot(hz, 4)
    lib().emul_sym_phase_words(buf.ctypes.data + at, n_int8, lead, g0, ng, int(hz is not None), c, s, pd.ctypes.data)
    bits = ((pd.reshape(ng, 4, 1) >> np.arange(32, dtype=np.uint32)) & 1).astype(np.uint8)
    return bits.transpose(0, 2, 1).reshape(-1)


def want_bits(buf, at, n_int8, lead, g0, ng, hz=None):
    """the definition: samples outside [-lead / 2, n_int8 / 2) of the capture read 0 (n_int8 even here)"""
    n = 128 * (g0 + ng) + 4
    x = np.zeros(2 * (n + 2), dtype=np.int64)               # x[2 (m + 2)] = I[m], m = -2 .. n + 1
    lo = -min(lead, 4) // 2
    for m in range(lo, min(n, n_int8 // 2)):
        x[2 * (m + 2)] = buf[at + 2 * m]
        x[2 * (m + 2) + 1] = buf[at + 2 * m + 1]
    c, s = (16384, 0) if hz is None else offset_ref.rot(hz, 4)
    return symbol_ref.dbits_sym(x, 128 * (g0 + ng), c, s)[128 * g0:]


def test_dense_random():
    """2^20 random sample pairs (n - 2, n + 2), unrotated and rotated"""
    rng = np.random.default_rng(11)
    ng = (1 << 20) // 128
    iq = rng.integers(-128, 128, size=256 * ng + 8, dtype=np.int16).astype(np.int8)
    x = np.concatenate([np.zeros(4, np.int8), iq])               # sample -2, -1 read 0 (no lead)
    for hz in [None] + OFFSETS:
        c, s = (16384, 0) if hz is None else offset_ref.rot(hz, 4)
        got = emul_bits(iq, 0, iq.size, 0, 0, ng, hz)
        want = symbol_ref.dbits_sym(x, 128 * ng, c, s)
        bad = np.flatnonzero(got != want)
        assert bad.size == 0, (hz, bad[:8])


@pytest.mark.parametrize("hz", [None, 0.0, 100e3, -250e3, 500e3, -500e3])
def test_dense_edges(hz):
    """every quadruple of int8 edge values (-128 included) as samples (n - 2, n + 2), at both word halves and at every
    sample phase; and every int8 pair against the edge values"""
    a, b, c_, d = np.meshgrid(EDGE, EDGE, EDGE, EDGE, indexing="ij")
    quads = np.stack([a.ravel(), b.ravel(), c_.ravel(), d.ravel()], axis=1)
    full = np.stack(np.meshgrid(np.arange(-128, 128), np.arange(-128, 128), indexing="ij"), -1).reshape(-1, 2).astype(np.int8)
    rng = np.random.default_rng(5)
    e2 = EDGE[rng.integers(0, EDGE.size, size=(full.shape[0], 2))]
    quads = np.concatenate([quads, np.concatenate([full, e2], axis=1)])
    for ph in range(4):                                          # sample n - 2 at phase ph of its symbol
        nq = quads.shape[0]
        samples = rng.integers(-128, 128, size=(8 * nq + 8, 2)).astype(np.int8)
        samples[8 * np.arange(nq) + ph] = quads[:, :2]
        samples[8 * np.arange(nq) + ph + 4] = quads[:, 2:]
        iq = samples.reshape(-1)
        iq = np.concatenate([iq, np.zeros(-iq.size % 256, np.int8)])
        ng = iq.size // 256
        got = emul_bits(iq, 0, iq.size, 0, 0, ng, hz)
        c, s = (16384, 0) if hz is None else offset_ref.rot(hz, 4)
        x = np.concatenate([np.zeros(4, np.int8), iq, np.zeros(8, np.int8)])
        want = symbol_ref.dbits_sym(x, 128 * ng, c, s)
        bad = np.flatnonzero(got != want)
        assert bad.size == 0, (hz, ph, bad[:8])


@pytest.mark.parametrize("lead", [0, 4, 256])
@pytest.mark.parametrize("hz", [None, 150e3])
def test_dense_capture_edges(lead, hz):
    """groups at the capture's start (with and without readable bytes in front), at the 32-group tile and 1024-group span
    edges, and at a ragged capture end (bytes behind n_int8 read 0)"""
    rng = np.random.default_rng(17)
    n_int8 = 256 * 1100 + 6                                      # ragged: 1100 groups and 3 samples
    buf = rng.integers(-128, 128, size=256 + n_int8 + 512, dtype=np.int16).astype(np.int8)
    at = 256
    for g0, ng in [(0, 3), (30, 4), (62, 4), (1022, 4), (1098, 3)]:
        got = emul_bits(buf, at, n_int8, lead, g0, ng, hz)
        want = want_bits(buf, at, n_int8, lead, g0, ng, hz)
        bad = np.flatnonzero(got != want)
        assert bad.size == 0, (g0, lead, bad[:8])


def emul_units_sym(iq2d, cfgs, capture=None, grid=132):
    iq2d = np.ascontiguousarray(iq2d, dtype=np.int8)
    ns, n = iq2d.shape
    cfgs = np.ascontiguousarray(cfgs).reshape(-1)
    cc = None if capture is None else np.ascontiguousarray(capture, dtype=np.int32)
    cap = cfgs.size * (n // 16384) * 123 + 8
    out = np.zeros(cap, dtype=orc.REC_DTYPE)
    dir_cap = cfgs.size * ((n // 16384 + 15) // 16 * 16 + 16)
    d = np.zeros((dir_cap, 2), dtype=np.uint32)
    nd = ctypes.c_long(0)
    cnt = lib().emul_rx_units_sym(iq2d.ctypes.data, ns, n, n, cfgs.ctypes.data, None if cc is None else cc.ctypes.data, cfgs.size, grid, 0,
                                  out.ctypes.data, cap, d.ctypes.data, dir_cap, ctypes.byref(nd))
    assert 0 <= cnt <= cap
    d = d[:nd.value]
    return np.concatenate([out[b:b + c] for b, c in d]) if len(d) else out[:0]


def restated(iq, cfg, stream=0):
    return symbol_ref.rx_stream(iq, 0.0, channel=int(cfg["channel"]), access_addr=int(cfg["access_addr"]),
                                access_mask=int(cfg["access_mask"]), crc_init=int(cfg["crc_init"]), raw=int(cfg["raw"]),
                                rssi=int(cfg["rssi"]) & ~_native.CFG_SYMBOL_SPACED, stream=stream, sym=True)


def test_restatement_with_reference_bits_is_the_oracle():
    """the restatement's bits argument leaves it the oracle: with sym=False every golden capture decodes as orc does"""
    for name in golden_util.cases():
        z, cfg = golden_util.load(name)
        flags = 2 if cfg.get("report_rejected") else 0
        kw = {k: v for k, v in cfg.items() if k != "report_rejected"}
        want = orc.rx_flags(z["iq"], flags | 1, **kw)
        assert symbol_ref.rx_stream(z["iq"], 0.0, rssi=flags | 1, sym=False, **kw).tobytes() == want.tobytes(), name


def test_unit_path_goldens():
    """the emulated unit path in the new mode equals the restatement on every golden capture, RSSI and -v included"""
    for name in golden_util.cases():
        z, cfg = golden_util.load(name)
        c = rxmod.make_cfgs(1, **golden_util.rx_cfg(cfg), symbol_spaced=1)
        c["rssi"] |= _native.CFG_RSSI
        iq = np.asarray(z["iq"], dtype=np.int8).reshape(1, -1)
        got = emul_units_sym(iq, c)
        want = restated(iq[0], c[0])
        assert got.tobytes() == want.tobytes(), name


def test_unit_path_fuzz_and_multi():
    """fuzz captures with several cfgs per capture (the <8> emulation) equal the restatement per cfg"""
    rng = np.random.default_rng(23)
    for _ in range(3):
        iq, cfgs, capture = multi_fuzz.draw(rng, max_captures=6, max_chunks=20)
        cfgs = cfgs.copy()
        cfgs["rssi"] |= _native.CFG_SYMBOL_SPACED
        got = emul_units_sym(iq, cfgs, capture)
        want = np.concatenate([restated(iq[capture[j]], cfgs[j], stream=j) for j in range(cfgs.size)] or [got[:0]])
        assert got.tobytes() == want.tobytes()


def test_unit_path_synthesised_and_gain():
    """a synthesised noisy capture: the unit path equals the restatement, and the new mode receives more packets"""
    cfg = np.zeros(1, dtype=_native.RX_BER_CFG_DTYPE)[0]
    cfg["seed"], cfg["snr_db"], cfg["amplitude"], cfg["slot_samples"], cfg["channel"] = 9, 14.0, 64, 2048, 37
    cfg["crc_init"], cfg["access_addr"] = 0x555555, 0x8E89BED6
    iq = rx_ber_ref.capture(cfg, 0, 160)[0]
    iq = np.asarray(iq, dtype=np.int8)[: iq.size // 16384 * 16384]
    c = rxmod.make_cfgs(1, channel=37, rssi=_native.CFG_REPORT_REJECTED, symbol_spaced=1)
    got = emul_units_sym(iq.reshape(1, -1), c)
    assert got.tobytes() == restated(iq, c[0]).tobytes()
    ok = lambda r: int(((r["crc_bad"] == 0) & ((r["flags"] & 4) == 0)).sum())
    plain = orc.rx_flags(iq, 2, channel=37)
    assert ok(got) > ok(plain), (ok(got), ok(plain))


def test_make_cfgs_flag():
    c = rxmod.make_cfgs(3, symbol_spaced=[0, 1, 1], recover=1)
    assert list(c["rssi"]) == [4, 20, 20]
    c = rxmod._with_fields(c, {"symbol_spaced": 0})
    assert list(c["rssi"]) == [4, 4, 4]
    assert _native.CFG_SYMBOL_SPACED == 16


@pytest.mark.parametrize("mode", mode_ref.MODES, ids=mode_ref.mode_id)
def test_mode_ref_rx_multi_equals_rx_stream_per_cfg(mode):
    """mode_ref.rx_multi (each capture's bits made once for all its cfgs; the oracle in the default mode) equals
    symbol_ref.rx_stream run once per cfg, on the goldens (with RSSI, -v and recovery) and on multi_fuzz draws"""
    rng = np.random.default_rng(41 + 2 * mode[0] + mode[1])
    n = 0
    for name in golden_util.cases():
        z, cfg = golden_util.load(name)
        kw = golden_util.rx_cfg(cfg)
        iq = np.asarray(z["iq"], dtype=np.int8).reshape(1, -1)
        cfgs = mode_ref.with_mode(rxmod.make_cfgs(3, **kw), mode)
        cfgs["rssi"] |= [1, 2 | 4, 4]
        offsets = mode_ref.draw_offsets(rng, 1, mode)
        iq = mode_ref.rotate_all(iq, offsets)
        got = mode_ref.rx_multi(iq, cfgs, np.zeros(3, dtype=np.int32), offsets)
        assert got.tobytes() == mode_ref.rx_multi_by_stream(iq, cfgs, np.zeros(3, dtype=np.int32), offsets).tobytes(), name
        n += got.size
    for _ in range(4):
        iq, cfgs, capture, offsets = multi_fuzz.draw_mode(rng, mode, max_captures=4, max_chunks=5)
        cfgs["rssi"][::3] |= rxmod._native.CFG_RECOVER
        got = mode_ref.rx_multi(iq, cfgs, capture, offsets)
        assert got.tobytes() == mode_ref.rx_multi_by_stream(iq, cfgs, capture, offsets).tobytes()
        n += got.size
    assert n > 100
