"""Expected records of the multi-cfg receive path in each of its four modes: (ROT, SYM) = carrier-offset correction on /
off (BTLE_CFG_* and offset_hz, include/btle_b200.h) x symbol-spaced discriminator on / off.  The default mode is the
oracle (test_rx_multi.oracle_multi); every other mode is symbol_ref.rx_stream, the oracle chain on the rotated or
symbol-spaced bits with recovery through offset_ref.recover.  rx_multi() computes each capture's bits once for all cfgs
that read it; tests/test_symbol.py shows that equals rx_stream per cfg.  Also the mode axis the GPU edge tests share:
the modes, the per-capture offsets they draw, and captures rotated onto those offsets."""
from __future__ import annotations

import numpy as np

import offset_ref
import orc
import recover_ref
import symbol_ref
from btle_b200._native import CFG_SYMBOL_SPACED

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


def _windows(iq: np.ndarray, hz: float, sym: bool):
    """(chunk, window, bits) of every chunk of one capture, as symbol_ref.rx_stream makes them"""
    c, s = offset_ref.rot(hz, 4 if sym else 1)
    C, W = symbol_ref.CHUNK_INT8, symbol_ref.WIN_INT8
    for k in range(iq.size // C):
        base = k * C
        win = np.zeros(256 + W + 8, dtype=np.int8)
        lo, hi = max(base - 256, 0), min(base + W + 8, iq.size)
        win[lo - base + 256:hi - base + 256] = iq[lo:hi]
        d = symbol_ref.dbits_sym(win[252:], symbol_ref.WIN_SAMPLES, c, s) if sym else offset_ref.dbits(win[256:], symbol_ref.WIN_SAMPLES, c, s)
        yield k, win, d


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
    per = [[] for _ in range(len(cfgs))]
    for c in np.unique(capture):
        mine = np.flatnonzero(capture == c)
        for k, win, d in _windows(iq2d[c], float(hz[c]), sym):
            for j in mine:
                f = cfgs[j]
                per[j] += symbol_ref.receiver_chunk(win, d, int(f["channel"]), int(f["access_addr"]), int(f["access_mask"]), int(f["crc_init"]),
                                                    int(f["raw"]), int(f["rssi"]), int(j), k)
        for j in mine:
            f = cfgs[j]
            r = np.array(per[j], dtype=orc.REC_DTYPE) if per[j] else np.zeros(0, dtype=orc.REC_DTYPE)
            if f["rssi"] & recover_ref.CFG_RECOVER and not f["raw"]:
                r = offset_ref.recover(r, iq2d[c], float(hz[c]), int(f["crc_init"]))
            per[j] = r
    out = [p for p in per if len(p)]
    return np.concatenate(out) if out else np.zeros(0, dtype=orc.REC_DTYPE)


def rx_multi_by_stream(iq2d, cfgs, capture, offsets=None) -> np.ndarray:
    """rx_multi through symbol_ref.rx_stream once per cfg: the definition rx_multi() is checked against"""
    iq2d = np.ascontiguousarray(iq2d, dtype=np.int8)
    if iq2d.ndim == 1:
        iq2d = iq2d[None, :]
    out = []
    for j, (f, c) in enumerate(zip(cfgs, np.asarray(capture).reshape(-1))):
        out.append(symbol_ref.rx_stream(iq2d[c], 0.0 if offsets is None else float(np.float32(offsets[c])), channel=int(f["channel"]),
                                        access_addr=int(f["access_addr"]), access_mask=int(f["access_mask"]), crc_init=int(f["crc_init"]),
                                        raw=int(f["raw"]), rssi=int(f["rssi"]), stream=j, sym=bool(f["rssi"] & CFG_SYMBOL_SPACED)))
    return np.concatenate(out) if out else np.zeros(0, dtype=orc.REC_DTYPE)
