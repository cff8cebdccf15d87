"""numpy restatement of BTLE_CFG_RECOVER (definition in include/btle_b200.h): the records of a cfg with the flag from the
records without it (the oracle's, tests/orc.py, or tests/mode_ref.py's in the other modes) and the capture, with the
symbol-spaced bits rotated by (C4, S4) under carrier-offset correction.  Used by tests/test_recover.py and
tests/test_offset.py against the CPU emulator, by tests/mode_ref.py, and by tests/test_recover_gpu.py against every GPU
path."""
from __future__ import annotations

import numpy as np

import offset_ref
from btle_b200 import synth

CHUNK = 8192
WIN = 9696                       # receiver()'s demod_buf_len in samples (19392 int8)
REC_RECOVERED = 8                # BTLE_REC_RECOVERED
CFG_RECOVER = 4                  # BTLE_CFG_RECOVER
_WHITEN = synth.whitening_table()


def window(iq: np.ndarray, chunk: int) -> np.ndarray:
    """int32 [WIN, 2]: the chunk's window of the capture, zero behind the capture's end"""
    iq = np.asarray(iq, dtype=np.int8).reshape(-1)
    w = np.zeros((WIN, 2), dtype=np.int32)
    part = iq[2 * CHUNK * chunk: 2 * (CHUNK * chunk + WIN)]
    n = part.size // 2
    w[:n] = part[:2 * n].reshape(-1, 2)
    return w


def sym_bits(w: np.ndarray, c4: int = 16384, s4: int = 0) -> np.ndarray:
    """e[s] = the discriminator of samples s and s + 4 rotated by (c4, s4) (offset_ref.disc) for s in [0, WIN), samples
    behind the window read as 0; (16384, 0) is the unrotated (I[s] Q[s+4] - I[s+4] Q[s]) > 0"""
    nxt = np.zeros_like(w)
    nxt[:-4] = w[4:]
    return offset_ref.disc(w[:, 0], w[:, 1], nxt[:, 0], nxt[:, 1], c4, s4)


def alternative(e: np.ndarray, n0: int, q: int, nbits: int) -> np.ndarray:
    """packet bits j = 0 .. nbits-1 of alternative q: e[n0 + 4j + q - 2] (0 outside the window)"""
    s = n0 + 4 * np.arange(nbits) + q - 2
    ok = (s >= 0) & (s < WIN)
    out = np.zeros(nbits, dtype=np.uint8)
    out[ok] = e[s[ok]]
    return out


def to_bytes(bits: np.ndarray) -> np.ndarray:
    return np.packbits(bits.reshape(-1, 8), axis=1, bitorder="little").reshape(-1)


def recover_one(e: np.ndarray, n0: int, channel: int, crc_init: int):
    """(q, bytes [n_bytes]) of the first alternative whose CRC is good, or None"""
    adv = channel >= 37
    for q in range(4):
        bits = alternative(e, n0, q, 32 + 8 * 42)[32:]
        b = to_bytes(bits) ^ _WHITEN[channel]
        length = int(b[1]) & (0x3F if adv else 0x1F)
        if adv and not 6 <= length <= 37:
            continue
        nb = length + 5
        rx_crc = int(b[nb - 3]) | (int(b[nb - 2]) << 8) | (int(b[nb - 1]) << 16)
        if synth.crc24(bytes(b[:nb - 3]), crc_init) == rx_crc:
            return q, b[:nb]
    return None


def apply(recs: np.ndarray, iq: np.ndarray, crc_init: int = 0x555555, raw: int = 0, offset_hz: float = 0.0) -> np.ndarray:
    """recs: one cfg's records (REC_DTYPE) over capture iq without the flag -> the records with it; offset_hz: the
    capture's carrier-offset correction (0: none; rot(0, 4) is the unrotated bit)"""
    out = recs.copy()
    if raw:
        return out
    c4, s4 = offset_ref.rot(offset_hz, 4)
    cache = {}
    for k, r in enumerate(out):
        if not r["crc_bad"] or r["flags"] & 4:
            continue
        c = int(r["chunk"])
        if c not in cache:
            cache[c] = sym_bits(window(iq, c), c4, s4)
        got = recover_one(cache[c], int(r["n0"]), int(r["channel"]), crc_init)
        if got is None:
            continue
        q, b = got
        r["bytes"][:] = 0
        r["bytes"][:b.size] = b
        r["n_bytes"], r["crc_bad"] = b.size, 0
        r["flags"] = int(r["flags"]) | REC_RECOVERED | (q << 4)
        out[k] = r
    return out
