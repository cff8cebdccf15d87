"""numpy restatement of BTLE_CFG_CENTRE_HITS (definition in include/btle_b200.h): tests/mode_ref.py's chain on the bits of
any mode, with each full-window hit moved to the centre of its run of matching sample phases.  Without the flag it is
mode_ref's chain, record for record; BTLE_CFG_RECOVER is applied on the moved n0 (recover_ref.apply).  Used by
tests/test_centre.py against the CPU emulator and by tests/test_centre_gpu.py against every GPU path."""
from __future__ import annotations

import ctypes

import numpy as np

import mode_ref
import offset_ref
import orc
import recover_ref
from btle_b200._native import CFG_CENTRE_HITS, CFG_SYMBOL_SPACED

CHUNK_SAMPLES = 8192
WIN_INT8, SEARCH_INT8, WIN_SAMPLES = mode_ref.WIN_INT8, mode_ref.SEARCH_INT8, mode_ref.WIN_SAMPLES
_WHITEN = mode_ref._WHITEN


def matches(d: np.ndarray, n: int, aa: int, mask: int) -> bool:
    """the 32 bits d[n + 4j] (j = 0..31) equal the access address under the mask (all inside d)"""
    w = int(np.packbits(d[n + 4 * np.arange(32)], bitorder="little").view("<u4")[0])
    return ((w ^ aa) & mask) == 0


def run_length(d: np.ndarray, n: int, n0_lim: int, aa: int, mask: int) -> int:
    """L = 1 + the number of consecutive q = 1, 2, 3 whose window n + q lies below n0_lim and below the chunk's 8192 window
    starts and matches"""
    L = 1
    for q in (1, 2, 3):
        c = n + q
        if c >= n0_lim or c >= CHUNK_SAMPLES or not matches(d, c, aa, mask):
            break
        L += 1
    return L


def centred(d: np.ndarray, n: int, R: int, n0_lim: int, aa: int, mask: int) -> int:
    """the hit the chain goes on with: n + (L - 1) // 2 for a full-window hit (n >= R), n for a part-A hit"""
    if n < R:
        return n
    return n + (run_length(d, n, n0_lim, aa, mask) - 1) // 2


def receiver_chunk(win: np.ndarray, d_win: np.ndarray, channel: int, access_addr: int, access_mask: int, crc_init: int, raw: int,
                   rssi: int, stream: int, chunk: int) -> list:
    """mode_ref.receiver_chunk, with every hit centred when rssi has BTLE_CFG_CENTRE_HITS"""
    L = orc.lib()
    d = np.zeros(WIN_SAMPLES + 4, dtype=np.uint8)
    d[:WIN_SAMPLES] = d_win
    adv = 37 <= channel <= 39
    crc_r = L.orc_crc_init_reorder(crc_init)
    E, left, out = 0, SEARCH_INT8 // 8, []
    hit = ctypes.c_int(0)
    b = np.zeros(48, dtype=np.uint8)
    report_rejected, centre = bool(rssi & 2), bool(rssi & CFG_CENTRE_HITS)

    def rec(n0v, nbytes, crc_bad, rejected):
        r = np.zeros(1, dtype=orc.REC_DTYPE)[0]
        r["stream"], r["chunk"], r["n0"], r["channel"], r["n_bytes"], r["crc_bad"] = stream, chunk, n0v, channel, nbytes, crc_bad
        r["flags"] = (1 if raw else 0) | (2 if adv else 0) | (4 if rejected else 0)
        r["access_addr"] = access_addr
        r["mag_sum"] = mode_ref._mag(win, n0v) if rssi & 1 else 0
        r["bytes"][:nbytes] = b[:nbytes]
        return r

    while True:
        R = E // 2
        if left <= 0 or not L.orc_search(d.ctypes.data, R, left, access_addr, access_mask, ctypes.byref(hit)):
            break
        n0 = hit.value
        if centre:
            n0 = centred(d, n0, R, R + 4 * left - 124, access_addr, access_mask)
        E = 2 * n0 + 256
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
                    out.append(rec(n0, 2, 0, True))
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
        out.append(rec(n0, nbytes, crc_bad, False))
    return out


def _decode(iq: np.ndarray, offset_hz: float, sym: bool, cfgs: list) -> list:
    """mode_ref._decode through this module's chain: records of one capture for each of cfgs = [(channel, access_addr,
    access_mask, crc_init, raw, rssi, stream)], each chunk's bits made once for all of them"""
    iq = np.asarray(iq, dtype=np.int8).reshape(-1)
    c, s = offset_ref.rot(offset_hz, 4 if sym else 1)
    per = [[] for _ in cfgs]
    for k in range(iq.size // mode_ref.CHUNK_INT8):
        base = k * mode_ref.CHUNK_INT8
        win = np.zeros(256 + WIN_INT8 + 8, dtype=np.int8)
        lo, hi = max(base - 256, 0), min(base + WIN_INT8 + 8, iq.size)
        win[lo - base + 256:hi - base + 256] = iq[lo:hi]
        d = offset_ref.dbits_sym(win[252:], WIN_SAMPLES, c, s) if sym else offset_ref.dbits(win[256:], WIN_SAMPLES, c, s)
        for p, f in zip(per, cfgs):
            p += receiver_chunk(win, d, *f, k)
    out = []
    for p, (channel, access_addr, access_mask, crc_init, raw, rssi, stream) in zip(per, cfgs):
        r = np.array(p, dtype=orc.REC_DTYPE) if p else np.zeros(0, dtype=orc.REC_DTYPE)
        if rssi & recover_ref.CFG_RECOVER:
            r = recover_ref.apply(r, iq, crc_init, raw, offset_hz)
        out.append(r)
    return out


def rx_stream(iq: np.ndarray, offset_hz: float = 0.0, sym: bool = False, channel=37, access_addr=0x8E89BED6, access_mask=0xFFFFFFFF,
              crc_init=0x555555, raw=0, rssi=0, stream=0) -> np.ndarray:
    """records of one capture decoded with one cfg (mode_ref.rx_stream's arguments; rssi's BTLE_CFG_CENTRE_HITS is read,
    its BTLE_CFG_SYMBOL_SPACED is not: sym chooses the bits)"""
    return _decode(iq, offset_hz, sym, [(channel, access_addr, access_mask, crc_init, raw, rssi, stream)])[0]


def rx_multi(iq2d: np.ndarray, cfgs: np.ndarray, capture, offsets=None) -> np.ndarray:
    """What btle_b200_rx_multi(_offset) returns for iq2d, cfgs (CFG_DTYPE, the flag set per cfg), capture and offsets (None:
    no correction, else Hz per capture): records with stream = cfg index, in (cfg, chunk, n0) order.  All cfgs share the
    SYM bit, as a launch requires."""
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
