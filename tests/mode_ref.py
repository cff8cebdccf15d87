"""Expected records of the receive path in each of its four modes: (ROT, SYM) = carrier-offset correction on / off
(BTLE_CFG_* and offset_hz, include/btle_b200.h) x symbol-spaced discriminator on / off.  rx_stream() is the pinned oracle
chain restated on the bits of any mode (tests/offset_ref.py): they go through orc_search / orc_demod_bytes as
orc_receiver_chunk_ex uses them (oracle/btle_oracle.c), so with the reference's bits at offset 0 it is the oracle itself,
and BTLE_CFG_RECOVER is applied with the 4-sample rotation (recover_ref.apply).  rx_multi() is the oracle
(test_rx_multi.oracle_multi) in the default mode and the same chain in every other, each capture's bits made once for all
cfgs that read it; tests/test_symbol.py shows that equals rx_stream per cfg.  Also the mode axis the GPU edge tests
share: the modes, the per-capture offsets they draw, and captures rotated onto those offsets."""
from __future__ import annotations

import ctypes

import numpy as np

import offset_ref
import orc
import recover_ref
from btle_b200 import synth
from btle_b200._native import CFG_SYMBOL_SPACED

CHUNK_INT8, WIN_INT8, SEARCH_INT8 = 16384, 19392, 16632
WIN_SAMPLES = WIN_INT8 // 2
_WHITEN = synth.whitening_table()

MODES = [(0, 0), (1, 0), (0, 1), (1, 1)]           # (ROT, SYM)
NEW_MODES = MODES[1:]                              # the instantiations the default kernels' edge tests do not reach
OFFSETS = (0.0, 25e3, -25e3, 137e3, -137e3, 310e3, -310e3, 500e3, -500e3)


def mode_id(mode) -> str:
    return "rot%d-sym%d" % tuple(mode)


def with_mode(cfgs: np.ndarray, mode) -> np.ndarray:
    """cfgs with BTLE_CFG_SYMBOL_SPACED set (SYM) or cleared"""
    c = cfgs.copy()
    c["rssi"] = (c["rssi"] & ~CFG_SYMBOL_SPACED) | (CFG_SYMBOL_SPACED if mode[1] else 0)
    return c


def draw_offsets(rng, n_captures: int, mode):
    """None (no correction) without ROT; else one offset per capture from OFFSETS, consecutive captures distinct"""
    if not mode[0]:
        return None
    out = [float(rng.choice(OFFSETS))]
    while len(out) < n_captures:
        h = float(rng.choice(OFFSETS))
        if h != out[-1]:
            out.append(h)
    return np.array(out, dtype=np.float32)


def rotate(iq: np.ndarray, hz: float) -> np.ndarray:
    """int8 interleaved iq moved hz off its carrier (received = sent x exp(+j 2 pi hz t)), rounded and clipped to int8, so
    the receiver corrected by hz finds its packets"""
    x = np.asarray(iq, dtype=np.int8).reshape(-1)
    if hz == 0.0 or x.size < 2:
        return x.copy()
    m = x.size // 2
    z = (x[0:2 * m:2].astype(np.float64) + 1j * x[1:2 * m:2]) * np.exp(2j * np.pi * float(np.float32(hz)) / 4e6 * np.arange(x.size // 2))
    out = x.copy()
    out[0:2 * z.size:2] = np.clip(np.rint(z.real), -128, 127)
    out[1:2 * z.size:2] = np.clip(np.rint(z.imag), -128, 127)
    return out


def rotate_all(iq2d: np.ndarray, offsets) -> np.ndarray:
    if offsets is None:
        return np.ascontiguousarray(iq2d, dtype=np.int8)
    return np.stack([rotate(row, h) for row, h in zip(iq2d, offsets)])


def _mag(win: np.ndarray, n0: int) -> int:
    a = 2 * n0 + np.arange(256)
    v = np.where((a >= -256) & (a < win.size - 256), win[np.clip(a + 256, 0, win.size - 1)].astype(np.int64), 0)
    return int(np.abs(v).sum()) & 0xFFFF


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
        r["mag_sum"] = _mag(win, n0v) if rssi & 1 else 0
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


def _decode(iq: np.ndarray, offset_hz: float, sym: bool, cfgs: list) -> list:
    """records of one capture for each of cfgs = [(channel, access_addr, access_mask, crc_init, raw, rssi, stream)]
    (orc_rx_stream_ex's chunking; samples in front of and behind the capture read 0), each chunk's bits made once for all
    of them.  sym: the symbol-spaced bits rotated by (C4, S4) of offset_hz; else the reference's bits rotated by (C, S)."""
    iq = np.asarray(iq, dtype=np.int8).reshape(-1)
    c, s = offset_ref.rot(offset_hz, 4 if sym else 1)
    per = [[] for _ in cfgs]
    for k in range(iq.size // CHUNK_INT8):
        base = k * CHUNK_INT8
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
    """records of one capture decoded with one cfg, corrected by offset_hz (0: the uncorrected bits), symbol-spaced or
    not (sym; rssi's own BTLE_CFG_SYMBOL_SPACED bit is not read)"""
    return _decode(iq, offset_hz, sym, [(channel, access_addr, access_mask, crc_init, raw, rssi, stream)])[0]


def _fields(f, stream: int) -> tuple:
    return (int(f["channel"]), int(f["access_addr"]), int(f["access_mask"]), int(f["crc_init"]), int(f["raw"]), int(f["rssi"]),
            stream)


def rx_multi(iq2d: np.ndarray, cfgs: np.ndarray, capture, offsets=None) -> np.ndarray:
    """What btle_b200_rx_multi(_offset) returns for iq2d, cfgs, capture and offsets (None: no correction, else one Hz
    value per capture): records with stream = cfg index, in (cfg, chunk, n0) order.  All cfgs share the SYM bit, as a
    launch requires."""
    from test_rx_multi import oracle_multi
    iq2d = np.ascontiguousarray(iq2d, dtype=np.int8)
    if iq2d.ndim == 1:
        iq2d = iq2d[None, :]
    capture = np.asarray(capture).reshape(-1)
    sym = bool(cfgs["rssi"][0] & CFG_SYMBOL_SPACED) if len(cfgs) else False
    assert all(bool(r & CFG_SYMBOL_SPACED) == sym for r in cfgs["rssi"])
    if offsets is None and not sym:
        return oracle_multi(iq2d, cfgs, capture)
    hz = np.zeros(iq2d.shape[0], dtype=np.float32) if offsets is None else np.asarray(offsets, dtype=np.float32)
    per = [None] * len(cfgs)
    for c in np.unique(capture):
        mine = np.flatnonzero(capture == c)
        for j, r in zip(mine, _decode(iq2d[c], float(hz[c]), sym, [_fields(cfgs[j], int(j)) for j in mine])):
            per[j] = r
    out = [p for p in per if len(p)]
    return np.concatenate(out) if out else np.zeros(0, dtype=orc.REC_DTYPE)


def rx_multi_by_stream(iq2d, cfgs, capture, offsets=None) -> np.ndarray:
    """rx_multi through rx_stream once per cfg: the definition rx_multi() is checked against"""
    iq2d = np.ascontiguousarray(iq2d, dtype=np.int8)
    if iq2d.ndim == 1:
        iq2d = iq2d[None, :]
    out = []
    for j, (f, c) in enumerate(zip(cfgs, np.asarray(capture).reshape(-1))):
        out.append(rx_stream(iq2d[c], 0.0 if offsets is None else float(np.float32(offsets[c])), bool(f["rssi"] & CFG_SYMBOL_SPACED),
                             *_fields(f, j)))
    return np.concatenate(out) if out else np.zeros(0, dtype=orc.REC_DTYPE)
