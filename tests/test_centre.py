"""BTLE_CFG_CENTRE_HITS on the CPU: the restatement (tests/centre_ref.py) against mode_ref's chain without the flag, and the
kernel logic's CPU emulator (unit path, candidate walk, stream path) against the restatement with it, on goldens, fuzz,
impaired captures, degenerate masks and captures whose discriminator bits are laid out sample by sample to put a run of
matching phases at each edge of the chain."""
import numpy as np
import pytest

import centre_ref
import emul
import golden_util
import mode_ref
import multi_fuzz
import orc
import rx_ber_ref
from btle_b200 import _native, ber, synth
from btle_b200.rx import _with_fields, make_cfgs

CENTRE = _native.CFG_CENTRE_HITS
UNROTATED = [(0, 0), (0, 1)]          # the modes the emulator's unit path runs (carrier-offset correction is checked on the GPU)


def restated(iq, cfg, stream=0, sym=None, offset_hz=0.0):
    """centre_ref's records of one cfg (CFG_DTYPE) over one capture, in the cfg's own discriminator mode unless sym is given"""
    sym = bool(cfg["rssi"] & _native.CFG_SYMBOL_SPACED) if sym is None else sym
    return centre_ref.rx_stream(iq, offset_hz, sym, *mode_ref._fields(cfg, stream)[:-1], stream=stream)


def emulated(iq2d, cfgs, force_walk=False):
    """the emulated unit path with one cfg per capture, records gathered in reference order, recovery applied as the kernel
    applies it"""
    recs, d = emul.rx_batch_units(iq2d, cfgs, grid=7, force_walk=force_walk)
    recs = np.concatenate([recs[b:b + c] for b, c in d]) if len(d) else recs[:0]
    return emul.recover(recs, iq2d, cfgs)


def check_units(iq2d, cfgs):
    """both chain paths of the emulated unit path equal the restatement; returns the records"""
    want = np.concatenate([restated(iq2d[j], cfgs[j], j) for j in range(cfgs.size)] or [np.zeros(0, orc.REC_DTYPE)])
    for walk in (False, True):
        got = emulated(iq2d, cfgs, walk)
        assert got.tobytes() == want.tobytes(), (walk, len(got), len(want))
    return want


# ---- captures laid out bit by bit ---------------------------------------------------------------------------------------
def iq_from_bits(d):
    """int8 capture whose default-mode discriminator bits are d: the phase steps by +pi/4 where d is 1 and by -pi/4 where
    it is 0 (|cross product| ~ 7071 at amplitude 100, far from the rounding of the samples)"""
    th = np.concatenate([[0.0], np.cumsum(np.where(d != 0, 1.0, -1.0) * np.pi / 4)])
    z = 100 * np.exp(1j * th)
    iq = np.empty(2 * z.size, dtype=np.int8)
    iq[0::2], iq[1::2] = np.rint(z.real), np.rint(z.imag)
    return iq


def packet_bits(body_len=20, channel=37, aa=0x8E89BED6, seed=0):
    body = np.random.default_rng(seed).integers(0, 256, body_len, dtype=np.uint8).tobytes()
    air = synth.air_bytes(synth.adv_pdu(0, 1, 0, bytes(6) + body), channel, aa)[1:]          # access address onwards
    return np.unpackbits(np.frombuffer(air, dtype=np.uint8), bitorder="little")


def plant(d, n, bits, run):
    """packet bit j held on samples n + 4j .. n + 4j + run - 1 and inverted on the rest of its symbol: the windows
    n .. n + run - 1 match the access address, n + run does not"""
    for j, b in enumerate(bits):
        d[n + 4 * j:n + 4 * j + run] = b
        d[n + 4 * j + run:n + 4 * j + 4] = 1 - b


def laid_out(plants, n_chunks=2, seed=1):
    """capture of n_chunks chunks of random bits with packets planted at (n, run, body_len)"""
    rng = np.random.default_rng(seed)
    d = rng.integers(0, 2, n_chunks * 8192 + 1600, dtype=np.uint8)
    for k, (n, run, body) in enumerate(plants):
        plant(d, n, packet_bits(body, seed=k), run)
    return iq_from_bits(d)[:n_chunks * 16384]


def edge_records(plants, flags=0, n_chunks=2):
    """records of a laid-out capture with the flag: the emulator (both chain paths, both discriminators) against the
    restatement; returns the default-mode records"""
    iq = laid_out(plants, n_chunks)
    out = None
    for mode in UNROTATED:
        cfgs = mode_ref.with_mode(make_cfgs(1, rssi=flags | CENTRE), mode)
        recs = check_units(iq[None], cfgs)
        out = recs if out is None else out
    return out


def test_run_at_the_chunks_last_window_starts():
    """n + q = 8191 is a window start of the chunk, 8192 is not (the limit is also n0_lim of the first search); the same
    packet in the next chunk is a hit through the zeroed history and stays where the search put it"""
    for n, run, want0, want1 in [(8188, 4, 8189, -4), (8189, 4, 8190, -3), (8190, 4, 8190, -2), (8189, 3, 8190, -3)]:
        r = edge_records([(n, run, 20)])
        assert [(int(x["chunk"]), int(x["n0"])) for x in r] == [(0, want0), (1, want1)], (n, run, r[["chunk", "n0"]])
        assert not r["crc_bad"].any()


def test_run_cut_by_the_search_limit():
    """a first packet centred to n0' = 4001 leaves n0_lim = 8189 for the next search: the run 8187.. stops at 8188"""
    r = edge_records([(4000, 3, 20), (8187, 4, 6)])
    assert [int(x["n0"]) for x in r if x["chunk"] == 0] == [4001, 8187], r[["chunk", "n0"]]


def test_run_across_the_two_flag_words():
    """the exact-hit lists of a chunk are split at sample 4096: a run from one list into the other"""
    for n, run, want in [(4094, 4, 4095), (4095, 3, 4096), (4093, 4, 4094), (4095, 2, 4095)]:
        r = edge_records([(n, run, 20)])
        assert [int(x["n0"]) for x in r if x["chunk"] == 0] == [want], (n, run)


def test_chunk_whose_lists_overflow():
    """five packets of four matching phases in the first flag word: 20 exact hits > kExactCap, so the chunk takes the
    candidate walk; every packet moves by one"""
    starts = [200, 900, 1600, 2300, 3000]
    r = edge_records([(n, 4, 0) for n in starts])
    assert [int(x["n0"]) for x in r if x["chunk"] == 0] == [n + 1 for n in starts]
    assert not r["crc_bad"].any()


@pytest.mark.parametrize("run", [1, 2, 3, 4])
def test_run_lengths(run):
    """L = 1, 2 keep the hit, L = 3, 4 move it by one; with and without -v, RSSI and recovery the emulator agrees"""
    for flags in (0, 1 | 2, _native.CFG_RECOVER):
        r = edge_records([(3000, run, 20)], flags)
        assert int(r["n0"][0]) == 3000 + (run - 1) // 2


# ---- the restatement without the flag ------------------------------------------------------------------------------------
@pytest.mark.parametrize("mode", mode_ref.MODES, ids=mode_ref.mode_id)
def test_flag_off_is_mode_ref(mode):
    """without the flag the restatement is mode_ref's chain, record for record, with RSSI, -v and recovery"""
    rng = np.random.default_rng(3 + 2 * mode[0] + mode[1])
    for name in golden_util.cases():
        z, cfg = golden_util.load(name)
        kw = golden_util.rx_cfg(cfg)
        hz = float(mode_ref.draw_offsets(rng, 1, mode)[0]) if mode[0] else 0.0
        iq = mode_ref.rotate(z["iq"], hz)
        for flags in (1, 2, 4):
            kw2 = dict(kw, rssi=kw.get("rssi", 0) | flags)
            a = centre_ref.rx_stream(iq, hz, bool(mode[1]), **kw2)
            assert a.tobytes() == mode_ref.rx_stream(iq, hz, bool(mode[1]), **kw2).tobytes(), (name, flags)
    for _ in range(3):
        iq, cfgs, capture, offsets = multi_fuzz.draw_mode(rng, mode, max_captures=3, max_chunks=4)
        cfgs["rssi"][::2] |= _native.CFG_RECOVER
        assert centre_ref.rx_multi(iq, cfgs, capture, offsets).tobytes() == mode_ref.rx_multi(iq, cfgs, capture, offsets).tobytes()


# ---- the emulator against the restatement with the flag ------------------------------------------------------------------
@pytest.mark.parametrize("mode", UNROTATED, ids=mode_ref.mode_id)
def test_emulator_goldens(mode):
    """every golden and fuzz golden, with RSSI, -v and recovery on top"""
    moved = 0
    for name in golden_util.cases():
        z, cfg = golden_util.load(name)
        iq = np.asarray(z["iq"], dtype=np.int8)
        iq = iq[: iq.size // 16384 * 16384].reshape(1, -1)
        for flags in (1, 1 | 2, 2 | _native.CFG_RECOVER):
            cfgs = mode_ref.with_mode(make_cfgs(1, **golden_util.rx_cfg(cfg)), mode)
            cfgs["rssi"] |= flags | CENTRE
            got = check_units(iq, cfgs)
            off = restated(iq[0], _with_fields(cfgs.copy(), {"centre_hits": 0})[0])
            moved += int(len(got) != len(off) or (got["n0"] != off["n0"]).any())
    assert moved > 0


def test_emulator_stream_path():
    """the emulator's span-by-span stream path (default discriminator) equals the restatement"""
    for name in golden_util.cases():
        z, cfg = golden_util.load(name)
        kw = golden_util.rx_cfg(cfg)
        for flags in (1, 1 | 2):
            kw2 = dict(kw, rssi=kw.get("rssi", 0) | flags | CENTRE)
            got = emul.rx_stream(z["iq"], span_chunks=3, **kw2)
            assert got.tobytes() == centre_ref.rx_stream(z["iq"], **kw2).tobytes(), name


@pytest.mark.parametrize("mode", UNROTATED, ids=mode_ref.mode_id)
def test_emulator_fuzz_with_the_flag_mixed(mode):
    """multi_fuzz launches (several cfgs per capture, the <8> path) with the flag on every other cfg"""
    rng = np.random.default_rng(71 + mode[1])
    for _ in range(3):
        iq, cfgs, capture, _ = multi_fuzz.draw_mode(rng, mode, max_captures=5, max_chunks=6)
        cfgs["rssi"][::2] |= CENTRE
        got = emul.rx_multi(iq, cfgs, capture)
        assert got.tobytes() == centre_ref.rx_multi(iq, cfgs, capture).tobytes()


def impaired(snr, ppm, channel, n=40, seed=5):
    cfg = ber.rx_ber_cfg(snr, ppm, slot_samples=2048, channel=channel, seed=seed, access_addr=0x8E89BED6 if channel >= 37 else 0x50654A21,
                         crc_init=0x555555 if channel >= 37 else 0x1A2B3C)[0]
    iq, truth, _ = rx_ber_ref.capture(cfg, 0, n)
    return iq, truth, cfg


@pytest.mark.parametrize("mode", UNROTATED, ids=mode_ref.mode_id)
@pytest.mark.parametrize("channel", [37, 9])
def test_emulator_impaired_captures(mode, channel):
    """the BER flow's captures at 16, 20 and 30 dB, 0 and 50 ppm, with -v and recovery, raw mode too"""
    for snr in (16.0, 20.0, 30.0):
        for ppm in (0.0, 50.0):
            iq, truth, c = impaired(snr, ppm, channel)
            iq = iq.reshape(1, -1)
            kw = dict(channel=channel, access_addr=int(c["access_addr"]), crc_init=int(c["crc_init"]))
            cfgs = mode_ref.with_mode(np.concatenate([make_cfgs(1, rssi=f | CENTRE, **kw) for f in (2, 1 | 2 | _native.CFG_RECOVER)]
                                                     + [make_cfgs(1, raw=1, rssi=CENTRE, **kw)]), mode)
            check_units(np.repeat(iq, 3, axis=0), cfgs)


@pytest.mark.parametrize("mode", UNROTATED, ids=mode_ref.mode_id)
def test_degenerate_and_sparse_masks(mode):
    """mask 0 (every hit comes through the zeroed history, so none moves: the records are those without the flag, -v
    reaching the late rows) and sparse masks, whose hits at a restart come through the zeroed history and must stay"""
    rng = np.random.default_rng(9)
    z = np.zeros(4 * 16384, dtype=np.int8)
    noise = rng.integers(-3, 4, 4 * 16384, dtype=np.int8)
    iq, _, _ = impaired(20.0, 0.0, 37, n=30)
    iq = iq[:4 * 16384]
    for cap in (z, noise, iq):
        for ch in (37, 38, 12):
            cfgs = mode_ref.with_mode(make_cfgs(1, channel=ch, access_mask=0, rssi=2 | CENTRE), mode)
            got = check_units(cap[None], cfgs)
            assert got.tobytes() == restated(cap, _with_fields(cfgs.copy(), {"centre_hits": 0})[0]).tobytes()
        for mask in (0xFFFF0000, 0xF0F00000, 0x80000000, 0x00000100, 0xFFFFFF00):
            cfgs = mode_ref.with_mode(make_cfgs(1, channel=37, access_mask=mask, rssi=1 | 2 | CENTRE), mode)
            check_units(cap[None], cfgs)


@pytest.mark.parametrize("mode", UNROTATED, ids=mode_ref.mode_id)
@pytest.mark.parametrize("channel", [37, 0])
def test_noiseless_packets_are_found_near_their_truth(mode, channel):
    """at every quarter-sample delay every packet is found with a good CRC, once, within 3 samples of the truth"""
    cfg = ber.rx_ber_cfg(1000.0, slot_samples=2048, channel=channel, seed=11 + channel, access_addr=0x8E89BED6 if channel >= 37 else 0x50654A21,
                         crc_init=0x555555 if channel >= 37 else 0x1A2B3C)[0]
    iq, truth, _ = rx_ber_ref.capture(cfg, 0, 48)
    assert set(truth["delta4"]) == {0, 1, 2, 3}
    cfgs = mode_ref.with_mode(make_cfgs(1, channel=channel, access_addr=int(cfg["access_addr"]), crc_init=int(cfg["crc_init"]),
                                        rssi=2 | CENTRE), mode)
    recs = check_units(iq.reshape(1, -1), cfgs)
    c = rx_ber_ref.score(recs, truth)
    assert c["pkt_err"] == 0 and c["extra_recs"] == 0 and c["crc_ok_wrong"] == 0, c
    pos = recs["chunk"].astype(np.int64) * 8192 + recs["n0"]
    assert np.abs(pos - truth["aa_sample"]).max() <= 3


def test_flag_bits():
    assert _native.CFG_CENTRE_HITS == 64
    c = make_cfgs(3, centre_hits=[0, 1, 1], symbol_spaced=1)
    assert list(c["rssi"]) == [16, 80, 80]
    assert list(_with_fields(c, {"centre_hits": 0})["rssi"]) == [16, 16, 16]
    assert int(ber.rx_ber_cfg(10.0, centre_hits=True, recover=True)["flags"][0]) == 64 | 4


def test_decode_connections_passes_the_flag():
    """hop.decode_connections gives every receive cfg it makes BTLE_CFG_CENTRE_HITS when asked, and no other cfg"""
    from btle_b200 import hop

    class Recorder:
        def __init__(self):
            self.cfgs = []

        def rx_batch(self, iq, cfgs, **kw):
            self.cfgs.append(np.array(cfgs))
            return np.zeros(0, dtype=_native.REC_DTYPE)

    for on in (False, True):
        r = Recorder()
        hop.decode_connections(r, np.zeros((40, 16384), dtype=np.int8), discover=False, centre_hits=on, symbol_spaced=True)
        assert len(r.cfgs) == 1 and all(bool(f & CENTRE) == on and f & _native.CFG_SYMBOL_SPACED for f in r.cfgs[0]["rssi"])
