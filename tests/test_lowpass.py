"""The low-pass filter in front of the symbol-spaced discriminator (BTLE_CFG_LOWPASS) on the CPU: the filtered-word helper
and the dense walk over filtered words (btle_core.cuh, emulated in tests/emul/btle_lowpass_emul.cpp) against the definition
in include/btle_b200.h, and the emulated unit path in that mode against the numpy restatement (tests/lowpass_ref.py)."""
import numpy as np
import pytest

import golden_util
import lowpass_emul
import lowpass_ref
import mode_ref
import multi_fuzz
import offset_ref
import orc
import rx_ber_ref
from btle_b200 import _native, rx as rxmod

EDGE = np.array([-128, -127, -64, -2, -1, 0, 1, 2, 63, 126, 127], dtype=np.int8)
OFFSETS = [0.0, 25e3, -25e3, 150e3, -300e3, 499_999.0, 500e3, -500e3]
LP = _native.CFG_SYMBOL_SPACED | _native.CFG_LOWPASS


def want_words(p, c, n):
    """the definition on the two samples of c, with the last sample of p in front and the first of n behind"""
    x = np.stack([p, c, n], axis=1).astype("<u4").view(np.int8).reshape(-1, 6, 2).astype(np.int32)   # samples 2k - 2 .. 2k + 3
    f = np.stack([(x[:, 1] + 2 * x[:, 2] + x[:, 3]) >> 2, (x[:, 2] + 2 * x[:, 3] + x[:, 4]) >> 2], axis=1)
    return np.ascontiguousarray(f.astype(np.int8)).reshape(-1, 4).view("<u4").reshape(-1)


def test_lp_word_edges_and_random():
    """lp_word against the definition on words of int8 edge values and on 2^20 random words"""
    rng = np.random.default_rng(3)
    e = EDGE[rng.integers(0, EDGE.size, size=(1 << 18, 12))].view(np.uint8).reshape(-1, 3, 4)
    words = np.ascontiguousarray(e).view("<u4").reshape(-1, 3)
    r = rng.integers(0, 1 << 32, size=(1 << 20, 3), dtype=np.uint64).astype(np.uint32)
    for w in (words, r):
        got = lowpass_emul.lp_words(w[:, 0], w[:, 1], w[:, 2])
        assert np.array_equal(got, want_words(w[:, 0], w[:, 1], w[:, 2]))


def test_nested_avg_is_the_filter():
    """avg(avg(a, c), b) == (a + 2 b + c) >> 2 for every int8 triple, and the helper's offset-binary avg is floor((a + b) / 2)"""
    v = np.arange(-128, 128, dtype=np.int32)
    avg = lambda x, y: (x + y) >> 1
    a, c = np.meshgrid(v, v, indexing="ij")
    ac = avg(a, c)[..., None]
    b = v[None, None, :]
    assert np.array_equal(avg(ac, b), (a[..., None] + 2 * b + c[..., None]) >> 2)
    assert np.array_equal(lowpass_emul.avg_table().astype(np.int32), avg(a, c))


def want_dbits(buf, at, n_int8, lead, g0, ng, hz=None):
    """the definition: x outside [-lead / 2, n_int8 / 2) of the capture reads 0 (lead and n_int8 even), F filters x, d reads F"""
    n = 128 * (g0 + ng)
    x = np.zeros(2 * (n + 8), dtype=np.int8)                  # x[2 (m + 4)] = I[m], m = -4 .. n + 3
    lo = -min(lead, 8) // 2
    for m in range(lo, min(n + 4, n_int8 // 2)):
        x[2 * (m + 4):2 * (m + 4) + 2] = buf[at + 2 * m:at + 2 * m + 2]
    f = lowpass_ref.lowpass(x)
    c, s = (16384, 0) if hz is None else offset_ref.rot(hz, 4)
    return offset_ref.dbits_sym(f[4:], n, c, s)[128 * g0:]


def test_dense_random():
    """2^20 random samples, unrotated and rotated"""
    rng = np.random.default_rng(11)
    ng = (1 << 20) // 128
    iq = rng.integers(-128, 128, size=256 * ng, dtype=np.int16).astype(np.int8)
    for hz in [None] + OFFSETS:
        got = lowpass_emul.dbits(iq, 0, iq.size, 0, 0, ng, hz)
        bad = np.flatnonzero(got != want_dbits(iq, 0, iq.size, 0, 0, ng, hz))
        assert bad.size == 0, (hz, bad[:8])


@pytest.mark.parametrize("hz", [None, 0.0, 100e3, -250e3, 500e3, -500e3])
def test_dense_edge_values(hz):
    """captures of int8 edge values only, at every sample phase"""
    rng = np.random.default_rng(5)
    iq = EDGE[rng.integers(0, EDGE.size, size=256 * 64)]
    got = lowpass_emul.dbits(iq, 0, iq.size, 0, 0, 64, hz)
    bad = np.flatnonzero(got != want_dbits(iq, 0, iq.size, 0, 0, 64, hz))
    assert bad.size == 0, (hz, bad[:8])


@pytest.mark.parametrize("lead", [0, 2, 4, 6, 256])
@pytest.mark.parametrize("hz", [None, 150e3, -500e3])
def test_dense_capture_edges(lead, hz):
    """groups at the capture's start (with none to more than enough readable bytes in front), at the 32-group tile and
    1024-group span edges, and at a ragged capture end (bytes behind n_int8 read 0)"""
    rng = np.random.default_rng(17)
    n_int8 = 256 * 1100 + 6                                      # ragged: 1100 groups and 3 samples
    buf = rng.integers(-128, 128, size=256 + n_int8 + 512, dtype=np.int16).astype(np.int8)
    at = 256
    for g0, ng in [(0, 3), (30, 4), (62, 4), (1022, 4), (1098, 3)]:
        got = lowpass_emul.dbits(buf, at, n_int8, lead, g0, ng, hz)
        bad = np.flatnonzero(got != want_dbits(buf, at, n_int8, lead, g0, ng, hz))
        assert bad.size == 0, (g0, lead, bad[:8])


def restated(iq, cfg, stream=0, hz=0.0):
    return lowpass_ref.rx_stream(iq, hz, *mode_ref._fields(cfg, stream)[:6], stream=stream)


def test_restatement_filter_edges():
    """the restatement's filter: floors, the int8 range and zeros outside the array"""
    x = np.array([-128, 127, -128, 127, -1, 0, 1, -1], dtype=np.int8)
    f = lowpass_ref.lowpass(x)
    want = [(0 - 256 - 128) >> 2, (0 + 254 + 127) >> 2, (-128 - 256 - 1) >> 2, (127 + 254 + 0) >> 2, (-128 - 2 + 1) >> 2,
            (127 + 0 - 1) >> 2, (-1 + 2 + 0) >> 2, (0 - 2 + 0) >> 2]
    assert list(f) == want


@pytest.mark.parametrize("flags", [0, _native.CFG_RECOVER | _native.CFG_CENTRE_HITS, _native.CFG_CORRECT | _native.CFG_RECOVER])
def test_unit_path_goldens(flags):
    """the emulated unit path in the low-pass mode equals the restatement on every golden capture, RSSI and -v included"""
    n = 0
    for name in golden_util.cases():
        z, cfg = golden_util.load(name)
        c = rxmod.make_cfgs(1, **golden_util.rx_cfg(cfg), symbol_spaced=1, lowpass=1)
        c["rssi"] |= _native.CFG_RSSI | flags
        iq = np.asarray(z["iq"], dtype=np.int8)
        got = lowpass_emul.rx_stream(iq, c[0])
        assert got.tobytes() == restated(iq, c[0]).tobytes(), name
        n += got.size
    assert n > 0


def test_unit_path_fuzz_and_rotated():
    """fuzz captures, every cfg of a draw with its own flags, unrotated and rotated by the draw's offsets"""
    rng = np.random.default_rng(23)
    n = 0
    for k in range(6):
        iq, cfgs, capture, offsets = multi_fuzz.draw_mode(rng, (k % 2, 1), max_captures=3, max_chunks=6)
        for j in range(cfgs.size):
            c = cfgs[j].copy()
            c["rssi"] |= LP | int(rng.choice([0, _native.CFG_RECOVER, _native.CFG_CENTRE_HITS | _native.CFG_CORRECT]))
            hz = None if offsets is None else float(offsets[capture[j]])
            got = lowpass_emul.rx_stream(iq[capture[j]], c, j, hz)
            assert got.tobytes() == restated(iq[capture[j]], c, j, 0.0 if hz is None else hz).tobytes(), (k, j)
            n += got.size
    assert n > 50


def test_unit_path_synthesised_and_gain():
    """a synthesised capture at 8 dB: the unit path equals the restatement (with RECOVER), and the filter receives more
    packets than the symbol-spaced bits alone"""
    cfg = np.zeros(1, dtype=_native.RX_BER_CFG_DTYPE)[0]
    cfg["seed"], cfg["snr_db"], cfg["amplitude"], cfg["slot_samples"], cfg["channel"] = 9, 8.0, 64, 2048, 37
    cfg["crc_init"], cfg["access_addr"] = 0x555555, 0x8E89BED6
    iq = rx_ber_ref.capture(cfg, 0, 160)[0]
    iq = np.asarray(iq, dtype=np.int8)[: iq.size // 16384 * 16384]
    ok = lambda r: int(((r["crc_bad"] == 0) & ((r["flags"] & 4) == 0)).sum())
    for flags in (_native.CFG_CENTRE_HITS, _native.CFG_CENTRE_HITS | _native.CFG_RECOVER):
        c = rxmod.make_cfgs(1, channel=37, rssi=_native.CFG_REPORT_REJECTED | flags, symbol_spaced=1, lowpass=1)
        got = lowpass_emul.rx_stream(iq, c[0])
        assert got.tobytes() == restated(iq, c[0]).tobytes()
        plain = mode_ref.rx_stream(iq, 0.0, True, channel=37, rssi=_native.CFG_REPORT_REJECTED | flags)
        assert ok(got) > ok(plain), (flags, ok(got), ok(plain))


def test_make_cfgs_flag():
    c = rxmod.make_cfgs(3, symbol_spaced=1, lowpass=[0, 1, 1], recover=1)
    assert list(c["rssi"]) == [20, 532, 532]
    c = rxmod._with_fields(c, {"lowpass": 0})
    assert list(c["rssi"]) == [20, 20, 20]
    assert _native.CFG_LOWPASS == 512
    from btle_b200 import ber
    assert int(ber.rx_ber_cfg(10.0, symbol_spaced=True, lowpass=True)["flags"][0]) == LP
