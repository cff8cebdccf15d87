"""Wrappers of the CPU emulator's BTLE_CFG_LOWPASS functions (tests/emul/btle_lowpass_emul.cpp, one of the sources of the
emulator library that tests/emul.py loads): the filtered-word helper, the dense walk over filtered words and the unit path
of one capture in the low-pass mode."""
import ctypes

import numpy as np

import emul
import offset_ref
from orc import REC_DTYPE

_vp, _lg, _int = ctypes.c_void_p, ctypes.c_long, ctypes.c_int
_SIGNATURES = {
    "emul_lp_words": (None, [_vp, _vp, _vp, _lg, _vp]),
    "emul_lp_avg_table": (None, [_vp]),
    "emul_lp_phase_words": (None, [_vp, _lg, _lg, _lg, _lg, _int, _int, _int, _vp]),
    "emul_lp_rx_stream": (_lg, [_vp, _lg, ctypes.POINTER(emul.StreamCfg), _int, _int, _int, _int, _vp, _lg]),
}


def lib():
    L = emul.lib()
    for name, (res, args) in _SIGNATURES.items():
        getattr(L, name).restype = res
        getattr(L, name).argtypes = args
    return L


def lp_words(prev, cur, nxt):
    """lp_word of each (prev, cur, next) triple of uint32 IQ words"""
    prev, cur, nxt = (np.ascontiguousarray(a, dtype=np.uint32) for a in (prev, cur, nxt))
    out = np.zeros(cur.size, dtype=np.uint32)
    lib().emul_lp_words(prev.ctypes.data, cur.ctypes.data, nxt.ctypes.data, cur.size, out.ctypes.data)
    return out


def avg_table():
    """int8 [256, 256]: the helper's per-byte avg of (a, b), a and b from -128"""
    out = np.zeros(256 * 256, dtype=np.int8)
    lib().emul_lp_avg_table(out.ctypes.data)
    return out.reshape(256, 256)


def dbits(buf, at, n_int8, lead, g0, ng, hz=None):
    """low-pass d[128 g0 .. 128 (g0 + ng)) from the emulated dense walk, rotated by (C4, S4) of hz (None: unrotated); the
    capture is buf[at : at + n_int8], buf[at - lead : at] readable in front of it"""
    buf = np.ascontiguousarray(buf, dtype=np.int8)
    pd = np.zeros(4 * ng, dtype=np.uint32)
    c, s = (16384, 0) if hz is None else offset_ref.rot(hz, 4)
    lib().emul_lp_phase_words(buf.ctypes.data + at, n_int8, lead, g0, ng, int(hz is not None), c, s, pd.ctypes.data)
    return emul._bits(pd, ng)


def rx_stream(iq, cfg, stream=0, hz=None):
    """records of one capture (nothing readable in front of it) with one cfg (CFG_DTYPE row) in the low-pass mode, repair
    flags applied; hz: the walk and recovery rotated by (C4, S4) of hz (None: unrotated)"""
    iq = np.ascontiguousarray(iq, dtype=np.int8).reshape(-1)
    c = emul.StreamCfg(int(cfg["channel"]), int(cfg["access_addr"]), int(cfg["access_mask"]), int(cfg["crc_init"]), int(cfg["raw"]),
                       int(cfg["rssi"]))
    c4, s4 = (16384, 0) if hz is None else offset_ref.rot(hz, 4)
    cap = (iq.size // 16384) * 123 + 8     # BTLE_MAX_RECS_PER_CHUNK
    out = np.zeros(cap, dtype=REC_DTYPE)
    n = lib().emul_lp_rx_stream(iq.ctypes.data, iq.size, ctypes.byref(c), stream, int(hz is not None), c4, s4, out.ctypes.data, cap)
    assert 0 <= n <= cap
    return out[:n]
