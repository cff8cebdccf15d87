"""Random launches of the multi-cfg receive path (btle_b200_rx_multi), shared by tools/fuzz_multi_gpu.py (the CUDA kernel)
and tests/test_rx_multi.py (the CPU emulator of its unit path); both compare with the oracle run once per cfg
(test_rx_multi.oracle_multi).

A draw: 1..max_captures captures of k x 16384 + {0, 1, 2, 255, 256, 3007, 3008, 3009, random} bytes, 0..8 cfgs per capture
(some captures no cfg names), each cfg with its own channel 0..39, access address, mask of popcount 0..32, 24-bit CRC
init, raw about a quarter of the time and flags 0..3.  Captures are uniform noise, +-1 values, all zeros (with mask 0
and -v the worst case of 123 records per chunk), a short periodic pattern, or bursts of the capture's own cfgs' access
addresses over a low noise floor: across chunk boundaries, cut by both ends of the capture, some with a corrupted CRC.
draw_mode() puts a draw in a mode (ROT, SYM) of tests/mode_ref.py: every cfg symbol-spaced or not and, with ROT, every
capture at an offset of its own, rotated onto it."""
import numpy as np

import mode_ref
from btle_b200 import synth
from btle_b200._native import MAX_CFGS_PER_CAPTURE
from btle_b200.rx import make_cfgs
from test_ingest_edges_gpu import _plant

CHUNK = 16384
TAILS = (0, 1, 2, 255, 256, 3007, 3008, 3009)
KINDS = ("noise", "pm1", "zeros", "periodic", "bursts")


def _mask(rng):
    m = 0
    for p in rng.permutation(32)[:int(rng.integers(0, 33))]:
        m |= 1 << int(p)
    return m


def _bursts(rng, iq, cfgs):
    """Bursts of the cfgs' access addresses (each with its cfg's channel and CRC init) written over iq."""
    n_samples = iq.size // 2
    for _ in range(int(rng.integers(2, 4 + n_samples // 20000))):
        c = cfgs[int(rng.integers(len(cfgs)))]
        ch, aa = int(c["channel"]), int(c["access_addr"])
        body = rng.integers(0, 256, int(rng.integers(0, 28)), dtype=np.uint8).tobytes()
        pdu = synth.adv_pdu(0, 1, 0, bytes(6) + body) if ch >= 37 else synth.ll_data_pdu(1 + int(rng.integers(0, 2)), 0, 0, 0, body[:27])
        air = bytearray(synth.air_bytes(pdu, ch, aa, int(c["crc_init"])))
        if rng.random() < 0.2:
            air[-1 - int(rng.integers(0, 3))] ^= 1 << int(rng.integers(0, 8))     # CRC must fail
        if rng.random() < 0.5:                                # access address near a chunk boundary (a straddle)
            at = int(rng.integers(0, n_samples // 8192 + 1)) * 8192 + int(rng.integers(-500, 200))
        else:                                                 # anywhere, cut by the capture's front or end
            at = int(rng.integers(-200, n_samples + 40))
        _plant(iq, at, bytes(air), amp=int(rng.integers(20, 110)))


def draw(rng, max_captures=40, max_chunks=24):
    """(iq int8 [n_captures, n_int8], cfgs, capture): one random rx_multi launch."""
    ns = int(rng.integers(1, max_captures + 1))
    tail = int(rng.choice(TAILS)) if rng.random() < 0.85 else int(rng.integers(0, CHUNK))
    n = int(rng.integers(1, max_chunks + 1)) * CHUNK + tail
    counts = rng.integers(0, MAX_CFGS_PER_CAPTURE + 1, ns)
    counts[rng.random(ns) < 0.2] = 0
    if counts.sum() == 0:
        counts[int(rng.integers(0, ns))] = int(rng.integers(1, MAX_CFGS_PER_CAPTURE + 1))
    capture = np.repeat(np.arange(ns, dtype=np.int32), counts)
    cfgs = make_cfgs(len(capture))
    iq = np.zeros((ns, n), dtype=np.int8)
    for s in range(ns):
        kind = KINDS[int(rng.integers(0, len(KINDS)))]
        mine = np.flatnonzero(capture == s)
        for j in mine:
            cfgs[j] = (int(rng.integers(0, 40)), int(rng.integers(0, 1 << 32)), _mask(rng), int(rng.integers(0, 1 << 24)),
                       int(rng.integers(0, 4) == 0), int(rng.integers(0, 4)))
            if kind == "bursts" and rng.random() < 0.75:      # masks that let the planted bursts through
                cfgs[j]["access_mask"] = 0xFFFFFFFF if rng.random() < 0.5 else cfgs[j]["access_mask"] | 0xFF
            if kind == "zeros" and rng.random() < 0.5:        # every position a hit: 51 packets or 123 records per chunk
                cfgs[j]["access_mask"] = 0
        if kind == "noise":
            iq[s] = rng.integers(-128, 128, n, dtype=np.int8)
        elif kind == "pm1":
            iq[s] = rng.integers(-1, 2, n, dtype=np.int8)
        elif kind == "periodic":
            iq[s] = np.resize(rng.integers(-100, 101, int(rng.choice([2, 4, 6, 8, 16, 64])), dtype=np.int8), n)
        elif kind == "bursts":
            iq[s] = rng.integers(-6, 7, n, dtype=np.int8)
            if mine.size:
                _bursts(rng, iq[s], cfgs[mine])
    return iq, cfgs, capture


def draw_mode(rng, mode, **kw):
    """(iq, cfgs, capture, offsets): a draw() in `mode`; offsets (Hz per capture) are None unless the mode has ROT."""
    iq, cfgs, capture = draw(rng, **kw)
    offsets = mode_ref.draw_offsets(rng, iq.shape[0], mode)
    return mode_ref.rotate_all(iq, offsets), mode_ref.with_mode(cfgs, mode), capture, offsets
