"""numpy restatement of BTLE_CFG_LOWPASS (definition in include/btle_b200.h): the [1, 2, 1] filter, then tests/centre_ref.py's
chain on the symbol-spaced bits of the filtered samples, and BTLE_CFG_RECOVER / BTLE_CFG_CORRECT (tests/correct_ref.py) on
the filtered capture.  mag_sum comes from the raw samples.  Used by tests/test_lowpass.py against the CPU emulator and by
tests/test_lowpass_gpu.py against every GPU path."""
from __future__ import annotations

import numpy as np

import centre_ref
import correct_ref
import mode_ref
import offset_ref
import orc
from btle_b200._native import CFG_CORRECT, CFG_LOWPASS, CFG_RECOVER

WIN_INT8, WIN_SAMPLES = mode_ref.WIN_INT8, mode_ref.WIN_SAMPLES


def lowpass(iq: np.ndarray) -> np.ndarray:
    """F[n] = (x[n-1] + 2 x[n] + x[n+1]) >> 2 per rail of int8 interleaved samples (x outside the array reads 0), int8, the
    array's length"""
    x = np.asarray(iq, dtype=np.int8).reshape(-1)
    s = np.zeros((x.size // 2 + 2, 2), dtype=np.int32)
    s[1:-1] = x[:x.size // 2 * 2].reshape(-1, 2)
    out = x.copy()
    out[:x.size // 2 * 2] = ((s[:-2] + 2 * s[1:-1] + s[2:]) >> 2).astype(np.int8).reshape(-1)
    return out


def _decode(iq: np.ndarray, offset_hz: float, cfgs: list) -> list:
    """records of one capture for each of cfgs = [(channel, access_addr, access_mask, crc_init, raw, rssi, stream)]"""
    iq = np.asarray(iq, dtype=np.int8).reshape(-1)
    c, s = offset_ref.rot(offset_hz, 4)
    plain = [f[:5] + (f[5] & ~(CFG_RECOVER | CFG_CORRECT),) + f[6:] for f in cfgs]
    per = [[] for _ in cfgs]
    for k in range(iq.size // mode_ref.CHUNK_INT8):
        base = k * mode_ref.CHUNK_INT8
        win = np.zeros(256 + WIN_INT8 + 8, dtype=np.int8)        # 128 samples in front of the chunk, 4 behind its window
        lo, hi = max(base - 256, 0), min(base + WIN_INT8 + 8, iq.size)
        win[lo - base + 256:hi - base + 256] = iq[lo:hi]
        d = offset_ref.dbits_sym(lowpass(win)[252:], WIN_SAMPLES, c, s)
        for p, f in zip(per, plain):
            p += centre_ref.receiver_chunk(win, d, *f, k)
    f_iq = lowpass(iq)
    out = []
    for p, (channel, access_addr, access_mask, crc_init, raw, rssi, stream) in zip(per, cfgs):
        r = np.array(p, dtype=orc.REC_DTYPE) if p else np.zeros(0, dtype=orc.REC_DTYPE)
        if rssi & (CFG_RECOVER | CFG_CORRECT):
            r = correct_ref.apply(r, f_iq, crc_init, raw, offset_hz, bool(rssi & CFG_RECOVER), bool(rssi & CFG_CORRECT))
        out.append(r)
    return out


def rx_stream(iq: np.ndarray, offset_hz: float = 0.0, channel=37, access_addr=0x8E89BED6, access_mask=0xFFFFFFFF, crc_init=0x555555,
              raw=0, rssi=0, stream=0) -> np.ndarray:
    """records of one capture decoded with one cfg in the low-pass mode (rssi's BTLE_CFG_CENTRE_HITS, BTLE_CFG_RECOVER and
    BTLE_CFG_CORRECT are read; the mode bits are not)"""
    return _decode(iq, offset_hz, [(channel, access_addr, access_mask, crc_init, raw, rssi, stream)])[0]


def rx_multi(iq2d: np.ndarray, cfgs: np.ndarray, capture, offsets=None) -> np.ndarray:
    """What btle_b200_rx_multi(_offset) returns for iq2d and cfgs that all carry BTLE_CFG_LOWPASS: records with stream = cfg
    index, in (cfg, chunk, n0) order"""
    iq2d = np.ascontiguousarray(iq2d, dtype=np.int8)
    if iq2d.ndim == 1:
        iq2d = iq2d[None, :]
    capture = np.asarray(capture).reshape(-1)
    assert all(r & CFG_LOWPASS for r in cfgs["rssi"])
    hz = np.zeros(iq2d.shape[0], dtype=np.float32) if offsets is None else np.asarray(offsets, dtype=np.float32)
    per = [None] * len(cfgs)
    for c in np.unique(capture):
        mine = np.flatnonzero(capture == c)
        for j, r in zip(mine, _decode(iq2d[c], float(hz[c]), [mode_ref._fields(cfgs[j], int(j)) for j in mine])):
            per[j] = r
    out = [p for p in per if len(p)]
    return np.concatenate(out) if out else np.zeros(0, dtype=orc.REC_DTYPE)
