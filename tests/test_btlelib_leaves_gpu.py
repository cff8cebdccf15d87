"""The Python-model leaves of the btlelib-compatible shim (gfsk_demodulation_fixed_point, search_unique_bit_sequence,
crc24_core / crc24, scramble_core / scramble; GPU kernels behind btle_b200_gfsk_demod_i16, _search_bit_sequence,
_crc24_bits, _scramble_bits) against the reference's own python/btlelib.py at their edges: tests/golden/btlelib_leaves.npz
(oracle/gen_golden_btlelib.py --leaves) holds what the reference returned.  Inputs too large for that file are checked
against the short restatements below, which a CPU test pins to the same file."""
import os

import numpy as np
import pytest

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "btlelib_leaves.npz")


def seeded_bits(seed: int, n: int) -> np.ndarray:
    """n pseudo-random 0/1 int8 bits: the top bit of splitmix64(seed + k), the same on every numpy version."""
    with np.errstate(over="ignore"):
        z = (np.arange(n, dtype=np.uint64) + np.uint64(seed)) * np.uint64(0x9E3779B97F4A7C15)
        z = (z ^ (z >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
        z = (z ^ (z >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
        z ^= z >> np.uint64(31)
    return (z >> np.uint64(63)).astype(np.int8)


def big_search_input(meta):
    """The 2^20-bit search case of the fixture, rebuilt from (seed, n, m, planted position)."""
    seed, n, m, pos = (int(v) for v in meta[:4])
    bit = seeded_bits(seed, n)
    seq = seeded_bits(seed + n, m)
    bit[pos:pos + m] = seq
    return bit, seq


# ---- restatements of btlelib.py with the same formulas ---------------------------------------------------------------
def gfsk_demod_ref(i, q):
    """btlelib.py:395-400: int32 products of neighbouring samples; exact in int64 for int16 inputs."""
    i = np.asarray(i, dtype=np.int64)
    q = np.asarray(q, dtype=np.int64)
    sig = i[:-1] * q[1:] - i[1:] * q[:-1]
    return (sig > 0).astype(np.int8), sig.astype(np.int32)


def crc24_core_ref(bit_in, init_bits):
    """btlelib.py:191-219: stage k of the register is bit k; new bit = stage 23 + input, fed into stages 0, 1, 3, 4, 6,
    9 and 10; the result reads the register from stage 23 down to 0."""
    st = sum((int(b) & 1) << k for k, b in enumerate(init_bits))
    for b in np.asarray(bit_in, dtype=np.int64).tolist():
        fb = ((st >> 23) + b) & 1
        st = (st << 1) & 0xFFFFFF
        if fb:
            st ^= 0x00065B
    return np.array([(st >> (23 - k)) & 1 for k in range(24)], dtype=np.int8)


def scramble_core_ref(bit_in, channel):
    """btlelib.py:226-263: a 7-stage register seeded with 1 and channel bits 5..0; output = stage 6, which moves to stage
    0 and is added into stage 4.  Its output repeats every 127 bits."""
    reg = [1] + [(int(channel) >> (5 - k)) & 1 for k in range(6)]
    seq = []
    for _ in range(127):
        o = reg[6]
        seq.append(o)
        reg = [o, reg[0], reg[1], reg[2], reg[3] ^ o, reg[4], reg[5]]
    bit_in = np.asarray(bit_in, dtype=np.int8)
    return ((np.resize(np.array(seq, dtype=np.int8), bit_in.size) + bit_in) & 1).astype(np.int8)


# ---- fixture -----------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def z():
    return np.load(GOLD)


@pytest.fixture(scope="module")
def bl():
    import __graft_entry__ as ge
    ge.build()
    import btle_b200.btlelib_compat as bl
    return bl


def _same(got, exp, what):
    got = np.asarray(got)
    assert got.dtype == exp.dtype and got.shape == exp.shape, (what, got.dtype, got.shape, exp.dtype, exp.shape)
    if not np.array_equal(got, exp):
        k = int(np.flatnonzero(got != exp)[0])
        raise AssertionError(f"{what}: first difference at {k}: {got[k]} != {exp[k]}")


def test_fixture_covers_the_edges(z):
    """The fixture reaches the edges: every (i[k], q[k], i[k+1], q[k+1]) over the int16 extremes, products at both ends
    of the int32 range the formula reaches, scramble lengths past the 127-bit period, sequence lengths 0 (with n 0 too),
    n, n + 1, 4096 and 5000."""
    vals = np.array([-32768, -32767, -1, 0, 1, 32767])
    i, q = z["gfsk_db_i"].astype(np.int64), z["gfsk_db_q"].astype(np.int64)
    code = lambda a: np.searchsorted(vals, a)
    tup = ((code(i[:-1]) * 6 + code(q[:-1])) * 6 + code(i[1:])) * 6 + code(q[1:])
    assert np.isin(i, vals).all() and np.isin(q, vals).all() and np.unique(tup).size == 6 ** 4
    sig = z["gfsk_db_sig"]
    assert sig.max() == 2147450880 and sig.min() == -2147450880
    assert max(z["scr_len"]) > 2 * 127
    m = [z[f"seq{k}_seq"].size for k in range(int(z["seq_n"]))]
    n = [z[f"seq{k}_bit"].size for k in range(int(z["seq_n"]))]
    assert 0 in m and 5000 in m and 4096 in m and any(a == b for a, b in zip(m, n)) and any(a == b + 1 for a, b in zip(m, n))
    assert (0, 0) in zip(m, n)


# ---- CPU: the restatements are the reference's functions on the fixture --------------------------------------------
def test_restatements_equal_the_reference(z):
    for k in range(int(z["gfsk_n"])):
        b, s = gfsk_demod_ref(z[f"gfsk{k}_i"], z[f"gfsk{k}_q"])
        _same(b, z[f"gfsk{k}_bit"], f"gfsk {k} bit")
        _same(s, z[f"gfsk{k}_sig"], f"gfsk {k} sig")
    b, s = gfsk_demod_ref(z["gfsk_db_i"], z["gfsk_db_q"])
    _same(b, z["gfsk_db_bit"], "gfsk all tuples bit")
    _same(s, z["gfsk_db_sig"], "gfsk all tuples sig")
    for k in range(int(z["crc_n"])):
        _same(crc24_core_ref(z[f"crc{k}_bits"], z[f"crc{k}_init"]), z[f"crc{k}_core"], f"crc24_core {k}")
    bits = z["scr_bits"]
    for r, ch in enumerate(z["scr_ch"]):
        o = 0
        for n in z["scr_len"]:
            _same(scramble_core_ref(bits[:n], ch), z["scr_core"][r, o:o + n], f"scramble_core ch {ch} n {n}")
            o += n


def test_seeded_bits_are_stable(z):
    """The big search input is stored as a seed: its bits must be the ones the generator drew."""
    b = seeded_bits(int(z["seeded_probe"]), 4096)
    _same(b, z["seeded_probe_bits"], "seeded bits")
    assert 1800 < int(b.sum()) < 2300


# ---- GPU: the shim equals the reference's values, dtypes and lengths ----------------------------------------------------
@pytest.mark.gpu
def test_gfsk_demodulation_fixed_point(bl, z):
    for k in range(int(z["gfsk_n"])):
        b, s = bl.gfsk_demodulation_fixed_point(z[f"gfsk{k}_i"], z[f"gfsk{k}_q"])
        _same(b, z[f"gfsk{k}_bit"], f"gfsk {k} bit")
        _same(s, z[f"gfsk{k}_sig"], f"gfsk {k} sig")
    b, s = bl.gfsk_demodulation_fixed_point(z["gfsk_db_i"], z["gfsk_db_q"])
    _same(b, z["gfsk_db_bit"], "gfsk all tuples bit")
    _same(s, z["gfsk_db_sig"], "gfsk all tuples sig")


@pytest.mark.gpu
def test_crc24_core_and_crc24(bl, z):
    for k in range(int(z["crc_n"])):
        bits, init = z[f"crc{k}_bits"], z[f"crc{k}_init"]
        _same(bl.crc24_core(bits, init), z[f"crc{k}_core"], f"crc24_core {k} ({bits.size} bits)")
        _same(bl.crc24(bits, init), z[f"crc{k}_full"], f"crc24 {k} ({bits.size} bits)")


@pytest.mark.gpu
def test_scramble_core_and_scramble(bl, z):
    """Channels 0..63 on lengths across the 127-bit period, and integers outside 0..63 (the reference takes bits 5..0)."""
    bits = z["scr_bits"]
    for r, ch in enumerate(z["scr_ch"]):
        o = 0
        for n in z["scr_len"]:
            _same(bl.scramble_core(bits[:n], int(ch)), z["scr_core"][r, o:o + n], f"scramble_core ch {ch} n {n}")
            o += n
        _same(bl.scramble(bits, int(ch)), z["scr_full"][r], f"scramble ch {ch}")


@pytest.mark.gpu
def test_search_unique_bit_sequence(bl, z):
    """First match at 0 and at n - m, several matches, m == n, n + 1, 1 and 0 (with n == 0 too), m 4096 and 5000."""
    for k in range(int(z["seq_n"])):
        got = bl.search_unique_bit_sequence(z[f"seq{k}_bit"], z[f"seq{k}_seq"])
        assert type(got) is int and got == int(z["seq_idx"][k]), (k, z[f"seq{k}_bit"].size, z[f"seq{k}_seq"].size, got,
                                                                 int(z["seq_idx"][k]))
    bit, seq = big_search_input(z["seq_big"])
    assert bl.search_unique_bit_sequence(bit, seq) == int(z["seq_big"][4]) == bit.size - seq.size


# ---- GPU: sizes beyond the fixture, against the restatements ----------------------------------------------------------
@pytest.mark.gpu
def test_gfsk_demod_2pow24_plus_3(bl):
    rng = np.random.default_rng(7)
    n = (1 << 24) + 3
    i = rng.integers(-32768, 32768, n, dtype=np.int16)
    q = rng.integers(-32768, 32768, n, dtype=np.int16)
    i[:: 1001] = -32768
    q[1:: 1003] = -32768
    i[2:: 997] = 32767
    b, s = bl.gfsk_demodulation_fixed_point(i, q)
    eb, es = gfsk_demod_ref(i, q)
    _same(b, eb, "gfsk bit")
    _same(s, es, "gfsk sig")


@pytest.mark.gpu
def test_crc24_core_and_scramble_on_a_million_bits(bl):
    bits = seeded_bits(99, 1_000_000)
    for init in (np.zeros(24, np.int8), np.ones(24, np.int8), seeded_bits(5, 24)):
        _same(bl.crc24_core(bits, init), crc24_core_ref(bits, init), f"crc24_core init {init.tolist()}")
    for ch in (0, 37, 63, 64, -1):
        _same(bl.scramble_core(bits, ch), scramble_core_ref(bits, ch), f"scramble_core ch {ch}")
