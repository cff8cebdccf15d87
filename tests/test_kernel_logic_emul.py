"""The per-lane kernel logic (btle_core.cuh / btle_params.h), executed on the CPU by the
test-only emulator, against the oracle and the reference-generated golden vectors.  This is the
no-GPU safety net for the CUDA path; the GPU parity tests proper are in test_gpu_parity.py."""
import numpy as np
import pytest

import emul
import golden_util as G
import orc
from btle_b200 import synth


def _same(a, b):
    assert len(a) == len(b), (len(a), len(b))
    assert a.tobytes() == b.tobytes()


@pytest.mark.parametrize("name", G.cases())
def test_emul_matches_reference_golden(name):
    z, cfg = G.load(name)
    for span in (1, 3, 16):
        rec = emul.rx_stream(z["iq"], span_chunks=span, **cfg)
        G.assert_matches_golden(rec, z)


def test_emul_tables_equal_reference_tables():
    t = G.tables()
    w, c = emul.tables()
    assert (w == np.array(t["scramble_table"], dtype=np.uint8)).all()
    assert (c == np.array(t["crc_table"], dtype=np.uint32)).all()


@pytest.mark.parametrize("seed", range(8))
def test_emul_equals_oracle_on_adversarial_fuzz(seed):
    rng = np.random.default_rng(1000 + seed)
    iq = rng.integers(-128, 128, 6 * 16384 + int(rng.integers(0, 16384)), dtype=np.int8)
    masks = [0x0000000F, 0x000000FF, 0x80000001, 0x00000000, 0xF0000000, 0x00010100, 0x0000FFFF, 0xFFFF0000]
    aas = [0x8E89BED6, 0x00000000, 0xFFFFFFFF, 0x55555555, 0x80000000, 0x12345678, 0x0000BED6, 0x8E890000]
    for ch in (37, 5):
        for raw in (0, 1):
            cfg = dict(channel=ch, access_addr=aas[seed], access_mask=masks[seed], raw=raw, crc_init=0x123456)
            _same(emul.rx_stream(iq, span_chunks=4, **cfg), orc.rx_stream(iq, **cfg))


def test_emul_equals_oracle_on_synth_streams():
    for ch, kw in ((37, {}), (12, dict(access_addr=0x60850A27, crc_init=0xA77B2E, data_channel_pdu=True))):
        iq, _ = synth.make_adv_stream(40 * 16384, seed=77 + ch, channel=ch, corrupt_every=9, slot_samples=2500, **kw)
        cfg = dict(channel=ch, access_addr=kw.get("access_addr", 0x8E89BED6), crc_init=kw.get("crc_init", 0x555555))
        a = emul.rx_stream(iq.numpy(), span_chunks=16, **cfg)
        b = orc.rx_stream(iq.numpy(), **cfg)
        assert len(b) > 100
        _same(a, b)


def test_emul_small_values_and_ragged():
    rng = np.random.default_rng(5)
    for n in (0, 1000, 16384, 16385, 3 * 16384 + 3007):
        iq = rng.integers(-1, 2, n, dtype=np.int8)
        cfg = dict(channel=38, access_addr=0x2AA, access_mask=0x3FF)
        _same(emul.rx_stream(iq, span_chunks=2, **cfg), orc.rx_stream(iq, **cfg))


def test_sliced_crc_equals_bytewise_crc():
    L = emul.lib()
    rng = np.random.default_rng(8)
    O = orc.lib()
    for n in range(0, 40):
        for _ in range(20):
            data = rng.integers(0, 256, max(n, 1), dtype=np.uint8)
            init = int(rng.integers(0, 2**24))
            assert L.emul_crc24_words(data.ctypes.data, n, init) == O.orc_crc24(data.ctypes.data, n, init)


def _walk(rec, d):
    """btle_b200_gather_ordered's walk of the unit directory."""
    parts = [rec[int(b):int(b) + int(c)] for b, c in d]
    return np.concatenate(parts) if parts else rec[:0]


@pytest.mark.parametrize("grid", [1, 3, 7, 132, 148])
def test_unit_plan_and_resolver_passes_equal_oracle(grid):
    """Plan / unit_info (last wave cut into pieces), chain pass -> prefix -> decode pass, block per unit +
    directory: walking the directory gives the oracle's records in the oracle's order, for any unit finishing order."""
    from btle_b200._native import CFG_DTYPE
    rng = np.random.default_rng(40 + grid)
    for nchunks, ns in ((1, 1), (5, 3), (37, 2), (16, 1), (67, 1)):
        n = nchunks * 16384 + int(rng.choice([0, 7, 3008, 9000]))
        iq = np.zeros((ns, n), dtype=np.int8)
        cfgs = np.zeros(ns, dtype=CFG_DTYPE)
        exp = []
        for s_ in range(ns):
            ch = [37, 9, 39][s_ % 3]
            aa = 0x8E89BED6 if ch >= 37 else 0x60850A1B + ch
            ci = 0x555555 if ch >= 37 else 0xA77B22 ^ ch
            t, _ = synth.make_adv_stream(n, seed=900 + 10 * nchunks + s_, channel=ch, access_addr=aa, crc_init=ci, corrupt_every=7,
                                         slot_samples=2100, data_channel_pdu=ch < 37, straddle_every=3)
            iq[s_] = t.numpy()
            cfgs[s_] = (ch, aa, 0xFFFFFFFF, ci, 0, 1)
            exp.append(orc.rx_stream(iq[s_], channel=ch, access_addr=aa, crc_init=ci, stream=s_))
        exp = np.concatenate(exp)
        for rev in (False, True):
            rec, d = emul.rx_batch_units(iq, cfgs, grid=grid, reverse_units=rev)
            assert int(d[:, 1].sum()) == len(rec) == len(exp)
            got = _walk(rec, d)
            assert got.tobytes() == exp.tobytes(), (grid, nchunks, ns, rev)


def test_unit_plan_tiles_every_chunk_once():
    import ctypes
    L = emul.lib()
    from btle_b200._native import CFG_DTYPE
    # degenerate masks: up to 51 packets per chunk go through the hit rows
    rng = np.random.default_rng(3)
    iq = rng.integers(-128, 128, (2, 9 * 16384 + 100), dtype=np.int8)
    cfgs = np.zeros(2, dtype=CFG_DTYPE)
    iq[0] = 0
    cfgs[0] = (1, 0, 0, 0x555555, 0, 1)
    cfgs[1] = (4, 0x12345678, 0x0000000F, 0x123456, 1, 1)
    rec, d = emul.rx_batch_units(iq, cfgs, grid=5)
    exp = np.concatenate([orc.rx_stream(iq[0], channel=1, access_addr=0, access_mask=0, stream=0),
                          orc.rx_stream(iq[1], channel=4, access_addr=0x12345678, access_mask=0xF, crc_init=0x123456, raw=1, stream=1)])
    assert np.bincount(exp['chunk'][exp['stream'] == 0]).max() == 51
    assert _walk(rec, d).tobytes() == exp.tobytes()


@pytest.mark.parametrize("seed", range(6))
def test_exact_hit_lists_equal_candidate_walk_on_fuzz(seed):
    """The resolver's list-driven chain (exact hits enumerated per flag word, cursor walk) against the candidate walk of
    search_from() and against the oracle, on the adversarial inputs of the fuzz tools: sparse masks (lists overflow ->
    fall-back), zero-history hits, dense bursts, periodic patterns."""
    from btle_b200._native import CFG_DTYPE
    rng = np.random.default_rng(7000 + seed)
    for _ in range(6):
        ns = int(rng.choice([1, 3]))
        n = int(rng.integers(1, 20)) * 16384 + int(rng.choice([0, 255, 3008, 9000]))
        iq = np.empty((ns, n), dtype=np.int8)
        cfgs = np.zeros(ns, dtype=CFG_DTYPE)
        for s_ in range(ns):
            kind = int(rng.integers(0, 4))
            ch = int(rng.integers(0, 40))
            aa = int(rng.integers(0, 1 << 32))
            pop = int(rng.choice([0, 2, 6, 10, 16, 32]))
            mask = 0
            for p_ in rng.permutation(32)[:pop]:
                mask |= 1 << int(p_)
            if kind == 0:
                iq[s_] = rng.integers(-128, 128, n, dtype=np.int8)
            elif kind == 1:
                iq[s_] = rng.integers(-1, 2, n, dtype=np.int8)
            elif kind == 2:
                t, _ = synth.make_adv_stream(n, seed=int(rng.integers(0, 1 << 30)), channel=ch, access_addr=aa, crc_init=0x123456, corrupt_every=3,
                                             slot_samples=int(rng.choice([1500, 2048, 3300])), data_channel_pdu=ch < 37, straddle_every=int(rng.choice([0, 2])))
                iq[s_] = t.numpy()
                mask = 0xFFFFFFFF if rng.integers(0, 2) else (mask | 0xFF)
            else:
                iq[s_] = np.resize(rng.integers(-100, 101, int(rng.choice([2, 4, 8, 64])), dtype=np.int8), n)
            cfgs[s_] = (ch, aa, mask, 0x123456, int(rng.integers(0, 4) == 0), 1)
        a, da = emul.rx_batch_units(iq, cfgs, grid=int(rng.choice([1, 5, 132])))
        b, db = emul.rx_batch_units(iq, cfgs, grid=132, force_walk=True)
        exp = np.concatenate([orc.rx_stream(iq[s_], channel=int(c["channel"]), access_addr=int(c["access_addr"]), access_mask=int(c["access_mask"]),
                                            crc_init=int(c["crc_init"]), raw=int(c["raw"]), stream=s_) for s_, c in enumerate(cfgs)])
        assert _walk(a, da).tobytes() == exp.tobytes() and _walk(b, db).tobytes() == exp.tobytes()


def test_unit_plan_covers_every_chunk_exactly_once_in_order():
    """make_plan / unit_info for random launch shapes and grid sizes: the units tile all (stream, chunk) pairs exactly once,
    in (stream, chunk) order (== reference order of the unit directory), no unit holds more than 16 chunks, and small inputs
    are cut into enough pieces to occupy the grid."""
    rng = np.random.default_rng(12)
    shapes = [(1, 65536, 132), (40, 16384, 132), (4096, 1024, 132), (1, 1, 132), (1, 17, 132), (3, 100, 132), (1, 128, 132), (7, 33, 5)]
    shapes += [(int(rng.integers(1, 60)), int(rng.integers(1, 3000)), int(rng.choice([1, 4, 132, 264]))) for _ in range(40)]
    for ns, nch, grid in shapes:
        u = emul.plan(ns, nch, grid)
        n = len(u)
        assert n > 0, (ns, nch, grid)
        assert (u[:, 2] >= 0).all() and (u[:, 2] <= 16).all()
        live = u[u[:, 2] > 0]
        exp_s, exp_c = 0, 0
        for s_, c0, k in live:                       # contiguous, ordered, complete
            assert (s_, c0) == (exp_s, exp_c), (ns, nch, grid)
            exp_c += k
            if exp_c == nch:
                exp_s, exp_c = exp_s + 1, 0
        assert (exp_s, exp_c) == (ns, 0)
        spans = ns * ((nch + 15) // 16)
        if spans < grid:
            assert n >= min(grid, 4 * spans) or n == ns * nch          # pieces: at least 4 per span (or one per chunk)


def test_dense_loop_discriminator_is_exact_for_every_int8_input():
    """btle_core.cuh dbits8_dense: t = dp2a([Q0 << 8 | (~I0) << 8 | 0xFF], [I1, Q1], 127) = 256 v + 127 - Q1 has the sign of
    v = Q0*I1 - I0*Q1 (btle_rx.c:1533) for all 2^32 inputs, |t| < 2^24, and both sign-bit gathers add exactly the two bits —
    checked on the PTX ISA's semantics of prmt / dp2a / dp4a (the instructions themselves are checked by the GPU parity tests;
    the emulator's unit path runs the same arithmetic against the oracle in the tests above)."""
    assert emul.check_discriminator() == 0


# ---- -v: rejected hits (flags 2 and 3) ---------------------------------------------------------------------------------
def _rejected_cases(rng):
    """(iq, cfg) pairs with many rejected hits: the zero capture with mask 0 (123 per chunk on channels 38 / 39, more than
    a hit row holds), full-scale noise with sparse masks, planted bad-length headers, and configs where -v changes nothing."""
    z = np.zeros(3 * 16384 + 3008, dtype=np.int8)
    out = [(z, dict(channel=ch, access_addr=0, access_mask=0)) for ch in (37, 38, 39)]
    noise = np.random.default_rng(0).integers(-128, 128, 8 * 16384 + 3008, dtype=np.int8)
    for mask in (0x00000000, 0x0000000F, 0x80000001, 0x0F000000, 0x000000FF):
        out.append((noise, dict(channel=int(rng.choice([37, 38, 39])), access_mask=mask)))
    out.append((noise, dict(channel=7, access_mask=0x0F000000)))
    out.append((noise, dict(channel=38, access_mask=0x000000FF, raw=1)))
    pdus = [synth.adv_pdu(0, 1, 0, bytes(range(6 + k))) for k in range(6)]
    pdus.insert(1, synth.adv_pdu(0, 1, 0, b"\x01\x02\x03"))
    pdus.insert(4, bytes([0x02, 45]) + bytes(range(20)))
    out.append((synth.make_pdu_stream(pdus, 39, seed=9, corrupt={2}), dict(channel=39)))
    return out


@pytest.mark.parametrize("flags", [2, 3])
def test_emul_rejected_hits_equal_oracle_per_chunk(flags):
    for iq, cfg in _rejected_cases(np.random.default_rng(flags)):
        for span in (1, 5, 16):
            _same(emul.rx_stream(iq, rssi=flags, span_chunks=span, **cfg), orc.rx_flags(iq, flags, **cfg))


@pytest.mark.parametrize("flags", [2, 3])
@pytest.mark.parametrize("grid", [1, 5, 132])
def test_emul_resolver_passes_report_every_rejected_hit(flags, grid):
    """The kernel's chain pass keeps 68 hits per chunk; with -v a chunk may have up to 123 (BTLE_MAX_RECS_PER_CHUNK).  Through the
    exact-hit lists and the candidate walk (force_walk), every unit finishing order: all of them, equal to the oracle."""
    from btle_b200._native import CFG_DTYPE
    cases = _rejected_cases(np.random.default_rng(10 * grid + flags))
    n = max(iq.size for iq, _ in cases)
    iq2d = np.zeros((len(cases), n), dtype=np.int8)
    cfgs = np.zeros(len(cases), dtype=CFG_DTYPE)
    exp = []
    for s_, (iq, cfg) in enumerate(cases):
        iq2d[s_, :iq.size] = iq
        full = dict(channel=37, access_addr=0x8E89BED6, access_mask=0xFFFFFFFF, crc_init=0x555555, raw=0)
        full.update(cfg)
        cfgs[s_] = (full["channel"], full["access_addr"], full["access_mask"], full["crc_init"], full["raw"], flags)
        exp.append(orc.rx_flags(iq2d[s_], flags, stream=s_, **full))
    exp = np.concatenate(exp)
    assert int(np.bincount(exp["chunk"][exp["stream"] == 1]).max()) == 123
    for kw in (dict(), dict(reverse_units=True), dict(force_walk=True)):
        rec, d = emul.rx_batch_units(iq2d, cfgs, grid=grid, **kw)
        assert int(d[:, 1].sum()) == len(rec) == len(exp)
        _same(_walk(rec, d), exp)
