"""The leaf entry points with the reference's signatures (btle_b200_search_unique_bits, _demod_byte, _scramble_byte,
_crc24_byte, _crc_init_reorder, _dbits) against the reference's own functions: oracle/_ref/libbtle_ref.so is the
reference's btle_rx.c compiled unmodified, and oracle/ref_wrap.c exports its search_unique_bits, demod_byte,
crc24_byte, scramble_table and crc_init_reorder (search_unique_bits itself is called too, for unique_bits bytes other
than 0/1).  Called through ctypes at the lengths, masks, inputs and init values
where a restatement goes wrong; btle_b200_rx_iq16 at every shift it accepts.  The CPU tests pin the C restatement the
rest of the suite trusts (oracle/btle_oracle.c) to the same reference functions on the same cases."""
import ctypes
import os

import numpy as np
import pytest

import orc
from btle_b200 import synth

REF_SO = os.path.join(orc.ORACLE_DIR, "_ref", "libbtle_ref.so")
pytestmark = pytest.mark.skipif(not os.path.exists(REF_SO), reason="oracle/_ref not built")

EINVAL = -1
SEARCH_EINVAL = EINVAL - 1000               # BTLE_SEARCH_ERR(BTLE_EINVAL)
SEARCH_LENS = list(range(1, 41)) + [63, 64, 65, 127, 128, 129, 2079, 4095, 4096]
MASKS = (0x0, 0x1, 0x80000000, 0x80000001, 0x3F, 0xFF00, 0xFFFFFFFE, 0xFFFFFFFF)
PLANT_AA = 0x8E89BED6
PAST_AA = 0x12345678                        # bit 31 clear: a window one symbol past the end would match on the zero behind
CRC_LENS = (0, 1, 2, 3, 39, 40, 255, 4095, 4096)

_ref = None


def ref():
    global _ref
    if _ref is None:
        L = ctypes.CDLL(REF_SO)
        vp, i32, u32 = ctypes.c_void_p, ctypes.c_int, ctypes.c_uint32
        L.ref_search_unique_bits.argtypes = [vp, i32, u32, u32]
        # the reference's own search_unique_bits (btle_rx.c:1510; a global function, as the Makefile passes -Dinline=),
        # for unique_bits / mask bytes other than the 0/1 that ref_search_unique_bits builds from a uint32
        L.search_unique_bits.argtypes = [vp, i32, vp, vp, i32]
        L.ref_demod_byte.argtypes = [vp, i32, vp]
        L.ref_demod_byte.restype = None
        L.ref_crc24_byte.argtypes = [vp, i32, u32]
        L.ref_crc24_byte.restype = u32
        L.ref_scramble_table.argtypes = [i32]
        L.ref_scramble_table.restype = vp
        L.ref_crc_init_reorder.argtypes = [u32]
        L.ref_crc_init_reorder.restype = u32
        _ref = L
    return _ref


def bits32(v):
    return np.array([(v >> p) & 1 for p in range(32)], dtype=np.uint8)


def iq_from_dbits(d, amp=100):
    """int8 IQ of len(d) + 1 samples whose discriminator bits are exactly d: quarter turns on a circle, counter-clockwise
    (cross product amp^2 > 0) for a 1, clockwise for a 0."""
    pts = np.array([[amp, 0], [0, amp], [-amp, 0], [0, -amp]], dtype=np.int8)
    k = np.concatenate([[0], np.cumsum(np.where(np.asarray(d) > 0, 1, -1))]) % 4
    return pts[k].reshape(-1)


def search_inputs(search_len):
    """(kind, iq, access address) for one search_len: 8 * search_len + 2 int8, the bytes the reference reads."""
    rng = np.random.default_rng(search_len)
    n8, ns = 8 * search_len + 2, 4 * search_len + 1
    yield "random", rng.integers(-128, 128, n8, dtype=np.int8), int(rng.integers(0, 2 ** 32))
    yield "ternary", rng.integers(-1, 2, n8, dtype=np.int8), int(rng.integers(0, 2 ** 32))
    yield "zero", np.zeros(n8, np.int8), int(rng.integers(0, 2 ** 32))
    yield "minus128", np.full(n8, -128, np.int8), 0                       # products of -128 cancel: every bit 0
    # the access address at the first window start with data only (n0 = 0), at the last one the search reports
    # (n0 = 4 search_len - 125) and one symbol past it (n0 = 4 search_len - 124, its bit 31 behind the data)
    for kind, n0, aa in (("plant_first", 0, PLANT_AA), ("plant_last", 4 * search_len - 125, PLANT_AA),
                         ("plant_past", 4 * search_len - 124, PAST_AA)):
        d = rng.integers(0, 2, ns - 1)
        for p in range(32):
            if 0 <= n0 + 4 * p < ns - 1:
                d[n0 + 4 * p] = (aa >> p) & 1
        yield kind, iq_from_dbits(d), aa


def search_cases():
    for sl in SEARCH_LENS:
        for kind, iq, aa in search_inputs(sl):
            for mask in MASKS:
                yield sl, kind, iq, aa, mask


def orc_search_unique_bits(iq, search_len, aa, mask):
    """The C restatement's search on the discriminator bits of iq, as the reference's return value."""
    d = np.concatenate([orc.dbits(np.concatenate([iq, np.zeros(2, np.int8)])), np.zeros(8, np.uint8)])
    n0 = ctypes.c_int(0)
    return 2 * n0.value if orc.lib().orc_search(d.ctypes.data, 0, search_len, aa, mask, ctypes.byref(n0)) else -1


def demod_inputs():
    rng = np.random.default_rng(11)
    for nb in range(1, 65):
        n8 = 64 * nb - 4                                                 # the reference reads rxp[0 .. 64 nb - 5]
        yield nb, "random", rng.integers(-128, 128, n8, dtype=np.int8)
        yield nb, "extreme", rng.choice(np.array([-128, 127], np.int8), n8)
        yield nb, "ternary", rng.integers(-1, 2, n8, dtype=np.int8)


def ref_demod(iq, nb):
    out = np.zeros(nb, np.uint8)
    ref().ref_demod_byte(iq.ctypes.data, nb, out.ctypes.data)
    return out


def crc_cases():
    rng = np.random.default_rng(12)
    inits = [0, 0xFFFFFF, 0x1000000, 0xFFFFFFFF] + [int(v) for v in rng.integers(0, 2 ** 32, 6, dtype=np.uint64)]
    for n in CRC_LENS:
        data = rng.integers(0, 256, n, dtype=np.uint8)
        for init in inits:
            yield data, init


def ref_crc(data, init):
    return ref().ref_crc24_byte(data.ctypes.data, data.size, init)


def scramble_table(ch):
    return np.frombuffer(ctypes.string_at(ref().ref_scramble_table(ch), 42), dtype=np.uint8)


# ---- CPU: the C restatement (oracle/btle_oracle.c) is the reference -------------------------------------------------------
def test_oracle_search_equals_reference():
    L = ref()
    seen = set()
    for sl, kind, iq, aa, mask in search_cases():
        exp = L.ref_search_unique_bits(iq.ctypes.data, sl, aa, mask)
        assert orc_search_unique_bits(iq, sl, aa, mask) == exp, (sl, kind, hex(mask))
        seen.add(exp)
    assert -248 in seen and -1 in seen


def test_oracle_demod_crc_reorder_equal_reference():
    L, O = ref(), orc.lib()
    for nb, kind, iq in demod_inputs():
        d = orc.dbits(np.concatenate([iq, np.zeros(4, np.int8)]))
        got = np.zeros(nb, np.uint8)
        O.orc_demod_bytes(d.ctypes.data, 0, nb, got.ctypes.data)
        assert (got == ref_demod(iq, nb)).all(), (nb, kind)
    for data, init in crc_cases():
        assert O.orc_crc24(data.ctypes.data, data.size, init) == ref_crc(data, init), (data.size, hex(init))
    rng = np.random.default_rng(13)
    for v in [0, 0xFFFFFFFF, 0x00FFFFFF, 0xFF000000] + [int(x) for x in rng.integers(0, 2 ** 32, 2000, dtype=np.uint64)]:
        assert O.orc_crc_init_reorder(v) == L.ref_crc_init_reorder(v), hex(v)


def test_crc_init_reorder_equals_reference():
    """btle_b200_crc_init_reorder is a host function of the library: no device involved."""
    from btle_b200 import _native
    lib = _native.load()
    rng = np.random.default_rng(14)
    for v in [0, 0xFFFFFFFF, 0x00FFFFFF, 0xFF000000, 0x555555] + [int(x) for x in rng.integers(0, 2 ** 32, 2000, dtype=np.uint64)]:
        assert lib.btle_b200_crc_init_reorder(v) == ref().ref_crc_init_reorder(v), hex(v)


# ---- GPU: the leaf entry points are the reference ------------------------------------------------------------------------
@pytest.fixture(scope="module")
def rx():
    import __graft_entry__ as ge
    ge.build()
    from btle_b200 import BtleRx
    r = BtleRx(0)
    yield r
    r.close()


@pytest.mark.gpu
def test_search_unique_bits_equals_reference(rx):
    """search_len 1..40 and across the 32-symbol groups up to 4096, eight masks, five input kinds and an access address
    at the first and last window start and one past the last.  Mask 0 matches the first window through the zeroed
    history: -248."""
    L = ref()
    seen = set()
    for sl, kind, iq, aa, mask in search_cases():
        exp = L.ref_search_unique_bits(iq.ctypes.data, sl, aa, mask)
        got = rx.search_unique_bits(iq, sl, bits32(aa), bits32(mask))
        assert got == exp, (sl, kind, hex(aa), hex(mask), got, exp)
        if mask == 0xFFFFFFFF and sl >= 32:
            planted = {"plant_first": 0, "plant_last": 8 * sl - 250, "plant_past": -1}
            assert exp == planted.get(kind, exp), (sl, kind, exp)
        seen.add(exp)
    assert -248 in seen and -1 in seen


@pytest.mark.gpu
def test_search_unique_bits_with_values_other_than_0_1(rx):
    """The reference compares demodulated 0/1 bits with unique_bits[p] where unique_bits_mask[p] is not 0: a masked 2 or
    255 never matches (-1), an unmasked one does not matter, any non-zero mask byte counts as set."""
    L = ref()
    sl = 64
    for kind, iq, aa in search_inputs(sl):
        if kind != "plant_last":
            continue
        ub, full = bits32(aa), np.ones(32, np.uint8)
        cases = []
        for p, v in ((0, 2), (5, 2), (31, 255), (17, 3)):
            b = ub.copy(); b[p] = v
            cases.append((b, full))                                       # masked: never matches
            m = full.copy(); m[p] = 0
            cases.append((b, m))                                          # unmasked: the planted address is found
            cases.append((b, np.zeros(32, np.uint8)))                     # mask 0: the first window
        cases.append((ub, np.full(32, 2, np.uint8)))                      # mask bytes of 2: all set
        cases.append((ub, np.where(np.arange(32) % 2, 7, 0).astype(np.uint8)))
        seen = set()
        for b, m in cases:
            exp = L.search_unique_bits(iq.ctypes.data, sl, b.ctypes.data, m.ctypes.data, 32)
            got = rx.search_unique_bits(iq, sl, b, m)
            assert got == exp, (b.tolist(), m.tolist(), got, exp)
            seen.add(exp)
        assert seen >= {-1, -248, 8 * sl - 250}


@pytest.mark.gpu
def test_demod_byte_equals_reference(rx):
    for nb, kind, iq in demod_inputs():
        assert (rx.demod_byte(iq, nb) == ref_demod(iq, nb)).all(), (nb, kind)


@pytest.mark.gpu
def test_crc24_byte_equals_reference(rx):
    """Any 32-bit init: the reference starts from all 32 bits and masks to 24 after each byte."""
    high = 0
    for data, init in crc_cases():
        exp = ref_crc(data, init)
        assert rx.crc24_byte(data, init) == exp, (data.size, hex(init), hex(exp))
        high += init >= 1 << 24 and data.size > 0
    assert high >= 40


@pytest.mark.gpu
def test_scramble_byte_equals_reference_table(rx):
    """All 40 channels: every offset with num_byte = 42 - offset, every num_byte at offset 0, and random pairs."""
    rng = np.random.default_rng(15)
    data = rng.integers(0, 256, 42, dtype=np.uint8)
    tables = [scramble_table(ch) for ch in range(40)]
    pairs = [(off, 42 - off) for off in range(43)] + [(0, nb) for nb in range(43)]
    for ch in range(40):
        for off, nb in pairs:
            got = rx.scramble_byte(data[:nb], ch, off)
            assert (got == data[:nb] ^ tables[ch][off:off + nb]).all(), (ch, off, nb)
    for _ in range(300):
        ch, off = int(rng.integers(0, 40)), int(rng.integers(0, 43))
        nb = int(rng.integers(0, 43 - off))
        d = rng.integers(0, 256, nb, dtype=np.uint8)
        assert (rx.scramble_byte(d, ch, off) == d ^ tables[ch][off:off + nb]).all(), (ch, off, nb)


@pytest.mark.gpu
def test_dbits_equals_oracle(rx):
    """The reference exports no dbits: the C restatement (pinned above through search and demod) is the yardstick."""
    rng = np.random.default_rng(16)
    for n in (1, 255, 256, 257, (1 << 24) + 1):
        for kind in ("minus128", "plus127", "mixed"):
            if kind == "mixed":
                iq = rng.choice(np.array([-128, -127, 127], np.int8), 2 * n + 2)
            else:
                iq = np.full(2 * n + 2, -128 if kind == "minus128" else 127, np.int8)
            got, exp = rx.dbits(iq), orc.dbits(iq)
            assert got.size == exp.size == n and (got == exp).all(), (n, kind)
            if kind == "mixed" and n > 1:
                assert 0 < int(exp.sum()) < n


@pytest.mark.gpu
def test_validation_edges(rx):
    """Each limit: the value at it is accepted, the one past it returns the documented code, and a valid call after it
    still gives the reference's answer."""
    L, R = rx._L, ref()
    h = rx._h
    rng = np.random.default_rng(17)
    aa, ub, um = PLANT_AA, bits32(PLANT_AA), np.ones(32, np.uint8)
    iq = rng.integers(-128, 128, 8 * 4097 + 2, dtype=np.int8)

    def check_search(sl):
        assert rx.search_unique_bits(iq, sl, ub, bits32(0xFF)) == R.ref_search_unique_bits(iq.ctypes.data, sl, aa, 0xFF)

    check_search(4096)
    assert L.btle_b200_search_unique_bits(h, iq.ctypes.data, 4097, ub.ctypes.data, um.ctypes.data, 32) == SEARCH_EINVAL
    check_search(4095)
    for nbits in (31, 33):
        assert L.btle_b200_search_unique_bits(h, iq.ctypes.data, 100, ub.ctypes.data, um.ctypes.data, nbits) == SEARCH_EINVAL
        check_search(100)

    out = np.zeros(65, np.uint8)
    assert (rx.demod_byte(iq, 64) == ref_demod(iq, 64)).all()
    assert L.btle_b200_demod_byte(h, iq.ctypes.data, 65, out.ctypes.data) == EINVAL
    assert (rx.demod_byte(iq, 7) == ref_demod(iq, 7)).all()

    data = rng.integers(0, 256, 4097, dtype=np.uint8)
    t39 = scramble_table(39)
    assert (rx.scramble_byte(data[:40], 39, 2) == data[:40] ^ t39[2:42]).all()
    assert L.btle_b200_scramble_byte(h, data.ctypes.data, 41, 39, 2, out.ctypes.data) == EINVAL         # 2 + 41 = 43
    assert L.btle_b200_scramble_byte(h, data.ctypes.data, 1, 39, 42, out.ctypes.data) == EINVAL
    assert L.btle_b200_scramble_byte(h, data.ctypes.data, 10, 40, 0, out.ctypes.data) == EINVAL
    assert (rx.scramble_byte(data[:10], 0, 32) == data[:10] ^ scramble_table(0)[32:42]).all()

    crc = ctypes.c_uint32(0)
    assert rx.crc24_byte(data[:4096], 0xFEDCBA98) == ref_crc(data[:4096], 0xFEDCBA98)
    assert L.btle_b200_crc24_byte(h, data.ctypes.data, 4097, 0x555555, ctypes.byref(crc)) == EINVAL
    assert rx.crc24_byte(data[:3], 0x89ABCDEF) == ref_crc(data[:3], 0x89ABCDEF)


@pytest.mark.gpu
@pytest.mark.parametrize("shift", range(9))
def test_rx_iq16_every_shift(rx, shift):
    """out = (x >> shift) & 0xFF for every shift 0..8, on an odd number of int16 whose bits outside the 8 kept are
    full-range junk: a packet stream in the kept bits, then pure junk with a sparse mask.  Shifts -1 and 9 are EINVAL."""
    from btle_b200 import REC_DTYPE, make_cfgs
    rng = np.random.default_rng(100 + shift)
    n = 5 * 16384 + 3001
    iq8, _ = synth.make_adv_stream(n, seed=40 + shift, channel=37, slot_samples=2600)
    field = iq8.numpy().view(np.uint8).astype(np.uint16) << shift
    keep = np.uint16((0xFF << shift) & 0xFFFF)
    junk = rng.integers(0, 1 << 16, n, dtype=np.uint16)
    iq16 = ((junk & ~keep) | field).view(np.int16)

    cfg = make_cfgs(1, channel=37)
    out = np.zeros(16, dtype=REC_DTYPE)
    n_out = ctypes.c_size_t(0)
    for bad in (-1, 9):
        assert rx._L.btle_b200_rx_iq16(rx._h, iq16.ctypes.data, n, bad, cfg.ctypes.data, out.ctypes.data, 16,
                                       ctypes.byref(n_out)) == EINVAL

    conv = ((iq16 >> shift) & 0xFF).astype(np.uint8).view(np.int8)
    assert (conv == iq8.numpy()).all()
    flags = 1 + shift % 3
    exp = orc.rx_flags(conv, flags, channel=37)
    assert len(exp) >= 10 and (exp["crc_bad"] == 0).sum() >= 10
    got = rx.rx_iq16(iq16, shift, channel=37, rssi=flags)
    assert got.tobytes() == exp.tobytes(), (len(got), len(exp))

    noise = rng.integers(-32768, 32768, 4 * 16384 + 1, dtype=np.int16)
    conv = ((noise >> shift) & 0xFF).astype(np.uint8).view(np.int8)
    exp = orc.rx_flags(conv, 3, channel=39, access_mask=0x0F000000)
    assert len(exp) > 0
    got = rx.rx_iq16(noise, shift, channel=39, access_mask=0x0F000000, rssi=3)
    assert got.tobytes() == exp.tobytes(), (len(got), len(exp))
