"""numpy restatement of the symbol-spaced discriminator (BTLE_CFG_SYMBOL_SPACED, definition in include/btle_b200.h) over the
pinned oracle chain: the bits go through orc_search / orc_demod_bytes as orc_receiver_chunk_ex uses them
(oracle/btle_oracle.c), so with the reference's bits (sym=False) this is the oracle itself, as offset_ref's chain is.
Used by tests/test_symbol.py (CPU) and tests/test_symbol_gpu.py."""
from __future__ import annotations

import ctypes

import numpy as np

import offset_ref
import orc
import recover_ref

CHUNK_INT8, WIN_INT8, SEARCH_INT8 = offset_ref.CHUNK_INT8, offset_ref.WIN_INT8, offset_ref.SEARCH_INT8
WIN_SAMPLES = WIN_INT8 // 2
_WHITEN = offset_ref._WHITEN


def dbits_sym(x: np.ndarray, n: int, c: int = 16384, s: int = 0) -> np.ndarray:
    """symbol-spaced d[0..n): the (rotated) discriminator of samples m - 2 and m + 2; x = int8 interleaved samples from
    sample -2 on (at least 2 (n + 4) values).  (16384, 0) is the unrotated bit, (C4, S4) the rotated one."""
    x = np.asarray(x, dtype=np.int64)
    return offset_ref.disc(x[0:2 * n:2], x[1:2 * n:2], x[8:2 * n + 8:2], x[9:2 * n + 8:2], c, s).astype(np.uint8)


def receiver_chunk(win: np.ndarray, d_win: np.ndarray, channel: int, access_addr: int, access_mask: int, crc_init: int, raw: int,
                   rssi: int, stream: int, chunk: int) -> list:
    """orc_receiver_chunk_ex on the given bits d_win[0 .. WIN_SAMPLES); win = 256 int8 in front of the chunk, its 19392-int8
    window, 8 behind (for mag_sum)"""
    L = orc.lib()
    d = np.zeros(WIN_SAMPLES + 4, dtype=np.uint8)
    d[:WIN_SAMPLES] = d_win
    adv = 37 <= channel <= 39
    crc_r = L.orc_crc_init_reorder(crc_init)
    E, left, out = 0, SEARCH_INT8 // 8, []
    n0 = ctypes.c_int(0)
    b = np.zeros(48, dtype=np.uint8)
    report_rejected = bool(rssi & 2)

    def rec(n0v, nbytes, crc_bad, rejected):
        r = np.zeros(1, dtype=orc.REC_DTYPE)[0]
        r["stream"], r["chunk"], r["n0"], r["channel"], r["n_bytes"], r["crc_bad"] = stream, chunk, n0v, channel, nbytes, crc_bad
        r["flags"] = (1 if raw else 0) | (2 if adv else 0) | (4 if rejected else 0)
        r["access_addr"] = access_addr
        r["mag_sum"] = offset_ref._mag(win, n0v) if rssi & 1 else 0
        r["bytes"][:nbytes] = b[:nbytes]
        return r

    while True:
        if not L.orc_search(d.ctypes.data, E // 2, left, access_addr, access_mask, ctypes.byref(n0)):
            break
        E = 2 * n0.value + 256
        hdr = E // 2
        nb = 42 if raw else 2
        E += 64 * nb
        if E > WIN_INT8:
            break
        b[:] = 0
        L.orc_demod_bytes(d.ctypes.data, hdr, nb, b.ctypes.data)
        if not raw:
            b[:2] ^= _WHITEN[channel][:2]
        left = int((SEARCH_INT8 - E) / 8)          # C division (truncates towards 0)
        nbytes, crc_bad = 42, 0
        if not raw:
            plen = int(b[1]) & (0x3F if adv else 0x1F)
            if adv and not 6 <= plen <= 37:
                if report_rejected:
                    out.append(rec(n0.value, 2, 0, True))
                continue
            E += 64 * (plen + 3)
            if E > WIN_INT8:
                break
            L.orc_demod_bytes(d.ctypes.data, hdr + 64, plen + 3, b[2:].ctypes.data)
            b[2:plen + 5] ^= _WHITEN[channel][2:plen + 5]
            left = int((SEARCH_INT8 - E) / 8)
            calc = L.orc_crc24(b.ctypes.data, plen + 2, crc_r)
            rx = int(b[plen + 2]) | (int(b[plen + 3]) << 8) | (int(b[plen + 4]) << 16)
            crc_bad, nbytes = int(calc != rx), plen + 5
        out.append(rec(n0.value, nbytes, crc_bad, False))
    return out


def rx_stream(iq: np.ndarray, offset_hz: float = 0.0, channel=37, access_addr=0x8E89BED6, access_mask=0xFFFFFFFF, crc_init=0x555555,
              raw=0, rssi=0, stream=0, sym=True) -> np.ndarray:
    """records of one capture (orc_rx_stream_ex's chunking; samples in front of and behind the capture read 0).  sym: the
    symbol-spaced bits rotated by (C4, S4) of offset_hz; else the reference's bits rotated by (C, S), i.e. offset_ref's
    chain.  BTLE_CFG_RECOVER in rssi is applied with the 4-sample rotation (offset_ref.recover)."""
    iq = np.asarray(iq, dtype=np.int8).reshape(-1)
    c, s = offset_ref.rot(offset_hz, 4 if sym else 1)
    recs = []
    for k in range(iq.size // CHUNK_INT8):
        base = k * CHUNK_INT8
        win = np.zeros(256 + WIN_INT8 + 8, dtype=np.int8)
        lo, hi = max(base - 256, 0), min(base + WIN_INT8 + 8, iq.size)
        win[lo - base + 256:hi - base + 256] = iq[lo:hi]
        d = dbits_sym(win[252:], WIN_SAMPLES, c, s) if sym else offset_ref.dbits(win[256:], WIN_SAMPLES, c, s)
        recs += receiver_chunk(win, d, channel, access_addr, access_mask, crc_init, raw, rssi, stream, k)
    out = np.array(recs, dtype=orc.REC_DTYPE) if recs else np.zeros(0, dtype=orc.REC_DTYPE)
    if rssi & recover_ref.CFG_RECOVER and not raw:
        out = offset_ref.recover(out, iq, offset_hz, crc_init)
    return out
