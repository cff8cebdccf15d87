"""numpy restatement of BTLE_CFG_CORRECT (definition in include/btle_b200.h): the patterns, their syndromes derived from
synth.crc24 by flipping bits, the correction of one packet, and the order with BTLE_CFG_RECOVER's alternatives
(tests/recover_ref.py).  The records of a cfg with the flag follow from the records without it (centre_ref's chain, which
is mode_ref's without BTLE_CFG_CENTRE_HITS) and the capture.  Used by tests/test_correct.py against the CPU emulator and by
tests/test_correct_gpu.py against every GPU path."""
from __future__ import annotations

import functools

import numpy as np

import centre_ref
import mode_ref
import offset_ref
import orc
import recover_ref
from btle_b200 import synth
from btle_b200._native import CFG_CORRECT, CFG_RECOVER, CFG_SYMBOL_SPACED, REC_CORRECTED, REC_RECOVERED

MAX_BODY = 39                    # bytes: the longest body (advertising length 37 + the 2 header bytes)
_WHITEN = recover_ref._WHITEN


def patterns(nbits: int) -> list:
    """(i, w) of every single bit (w = 1) and adjacent pair (i, i + 1; w = 2) of a packet of nbits bits (body and CRC)"""
    return [(i, 1) for i in range(nbits)] + [(i, 2) for i in range(nbits - 1)]


def _crc_field(b: np.ndarray, nb: int) -> int:
    return int(b[nb - 3]) | (int(b[nb - 2]) << 8) | (int(b[nb - 1]) << 16)


def syndrome(b: np.ndarray, crc_init: int) -> int:
    """crc24(body) XOR the received CRC of packet bytes b (body, then 3 CRC bytes)"""
    b = np.asarray(b, dtype=np.uint8)
    return synth.crc24(bytes(b[:-3]), crc_init) ^ _crc_field(b, b.size)


def flip(b: np.ndarray, i: int, w: int) -> np.ndarray:
    """b with packet bits i .. i + w - 1 (LSB first) inverted"""
    bits = np.unpackbits(np.asarray(b, dtype=np.uint8), bitorder="little")
    bits[i:i + w] ^= 1
    return np.packbits(bits, bitorder="little")


@functools.lru_cache(maxsize=None)
def table() -> dict:
    """{syndrome: (u, w)} of the patterns of the longest body, u = the pattern's first bit counted from the packet's end
    (u = 0: the last CRC bit): each syndrome found by flipping the pattern in a packet with a good CRC"""
    rng = np.random.default_rng(0)
    body = rng.integers(0, 256, MAX_BODY, dtype=np.uint8)
    crc = synth.crc24(bytes(body), 0x555555)
    good = np.concatenate([body, np.array([crc & 0xFF, (crc >> 8) & 0xFF, crc >> 16], dtype=np.uint8)])
    n = 8 * good.size
    out = {}
    for i, w in patterns(n):
        s = syndrome(flip(good, i, w), 0x555555)
        assert s != 0 and s not in out, (i, w)
        out[s] = (n - 1 - i, w)
    return out


def length_field(channel: int) -> range:
    """header bits of the length field: 8..13 on channels 37..39, 8..12 on 0..36"""
    return range(8, 14) if channel >= 37 else range(8, 13)


def correct(b: np.ndarray, channel: int, crc_init: int):
    """packet bytes b (body and CRC, dewhitened) with a failed CRC -> the corrected bytes, or None"""
    b = np.asarray(b, dtype=np.uint8)
    hit = table().get(syndrome(b, crc_init))
    if hit is None:
        return None
    u, w = hit
    i = 8 * b.size - 1 - u
    if i < 0 or set(range(i, i + w)) & set(length_field(channel)):
        return None
    return flip(b, i, w)


def _alternative(e: np.ndarray, n0: int, q: int, channel: int):
    """alternative q's bytes [n_bytes] (recover_ref's bits and length rule), None when its advertising length is skipped"""
    b = recover_ref.to_bytes(recover_ref.alternative(e, n0, q, 32 + 8 * 42)[32:]) ^ _WHITEN[channel]
    length = int(b[1]) & (0x3F if channel >= 37 else 0x1F)
    if channel >= 37 and not 6 <= length <= 37:
        return None
    return b[:length + 5]


def repair(r, iq: np.ndarray, crc_init: int, recover: bool, corr: bool, c4: int, s4: int, cache: dict):
    """(flags, bytes) of one counted CRC-failed record in the rule's order, None when nothing applies"""
    channel, n0, nb = int(r["channel"]), int(r["n0"]), int(r["n_bytes"])
    e = None
    if recover:
        c = int(r["chunk"])
        if c not in cache:
            cache[c] = recover_ref.sym_bits(recover_ref.window(iq, c), c4, s4)
        e = cache[c]
        got = recover_ref.recover_one(e, n0, channel, crc_init)
        if got is not None:
            return REC_RECOVERED | (got[0] << 4), got[1]
    if not corr:
        return None
    fixed = correct(r["bytes"][:nb], channel, crc_init)
    if fixed is not None:
        return REC_CORRECTED, fixed
    if recover:
        for q in range(4):
            b = _alternative(e, n0, q, channel)
            fixed = None if b is None else correct(b, channel, crc_init)
            if fixed is not None:
                return REC_RECOVERED | (q << 4) | REC_CORRECTED, fixed
    return None


def apply(recs: np.ndarray, iq: np.ndarray, crc_init: int = 0x555555, raw: int = 0, offset_hz: float = 0.0, recover: bool = False,
          corr: bool = True) -> np.ndarray:
    """recs: one cfg's records (REC_DTYPE) over capture iq without BTLE_CFG_RECOVER and BTLE_CFG_CORRECT -> the records
    with the given flags; offset_hz: the capture's carrier-offset correction (the alternatives' rotation)"""
    out = recs.copy()
    if raw:
        return out
    c4, s4 = offset_ref.rot(offset_hz, 4)
    cache = {}
    for k, r in enumerate(out):
        if not r["crc_bad"] or r["flags"] & 4:
            continue
        got = repair(r, iq, crc_init, recover, corr, c4, s4, cache)
        if got is None:
            continue
        flags, b = got
        r["bytes"][:] = 0
        r["bytes"][:b.size] = b
        r["n_bytes"], r["crc_bad"] = b.size, 0
        r["flags"] = int(r["flags"]) | flags
        out[k] = r
    return out


def _decode(iq: np.ndarray, offset_hz: float, sym: bool, cfgs: list) -> list:
    """centre_ref._decode with both repair flags taken off the cfgs and applied here"""
    plain = [f[:5] + (f[5] & ~(CFG_RECOVER | CFG_CORRECT),) + f[6:] for f in cfgs]
    recs = centre_ref._decode(iq, offset_hz, sym, plain)
    return [apply(r, iq, f[3], f[4], offset_hz, bool(f[5] & CFG_RECOVER), bool(f[5] & CFG_CORRECT)) for r, f in zip(recs, cfgs)]


def rx_stream(iq: np.ndarray, offset_hz: float = 0.0, sym: bool = False, channel=37, access_addr=0x8E89BED6, access_mask=0xFFFFFFFF,
              crc_init=0x555555, raw=0, rssi=0, stream=0) -> np.ndarray:
    """records of one capture decoded with one cfg (centre_ref.rx_stream's arguments; rssi's BTLE_CFG_CORRECT,
    BTLE_CFG_RECOVER and BTLE_CFG_CENTRE_HITS are read, its BTLE_CFG_SYMBOL_SPACED is not: sym chooses the bits)"""
    return _decode(iq, offset_hz, sym, [(channel, access_addr, access_mask, crc_init, raw, rssi, stream)])[0]


def rx_multi(iq2d: np.ndarray, cfgs: np.ndarray, capture, offsets=None) -> np.ndarray:
    """What btle_b200_rx_multi(_offset) returns for iq2d, cfgs (CFG_DTYPE, the flags set per cfg), capture and offsets
    (None: no correction, else Hz per capture): records with stream = cfg index, in (cfg, chunk, n0) order"""
    iq2d = np.ascontiguousarray(iq2d, dtype=np.int8)
    if iq2d.ndim == 1:
        iq2d = iq2d[None, :]
    capture = np.asarray(capture).reshape(-1)
    sym = bool(cfgs["rssi"][0] & CFG_SYMBOL_SPACED) if len(cfgs) else False
    assert all(bool(r & CFG_SYMBOL_SPACED) == sym for r in cfgs["rssi"])
    hz = np.zeros(iq2d.shape[0], dtype=np.float32) if offsets is None else np.asarray(offsets, dtype=np.float32)
    per = [None] * len(cfgs)
    for c in np.unique(capture):
        mine = np.flatnonzero(capture == c)
        for j, r in zip(mine, _decode(iq2d[c], float(hz[c]), sym, [mode_ref._fields(cfgs[j], int(j)) for j in mine])):
            per[j] = r
    out = [p for p in per if len(p)]
    return np.concatenate(out) if out else np.zeros(0, dtype=orc.REC_DTYPE)
