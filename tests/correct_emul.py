"""Wrappers of the CPU emulator's BTLE_CFG_CORRECT functions (tests/emul/btle_correct_emul.cpp, one of the sources of the
emulator library that tests/emul.py loads): the kernel's repair step over emulated records, the shared syndrome table and
its lookup."""
import ctypes

import numpy as np

import emul
import offset_ref
from orc import REC_DTYPE

_vp, _lg = ctypes.c_void_p, ctypes.c_long
_SIGNATURES = {
    "emul_repair_records": (_lg, [_vp, _lg, _lg, _vp, _vp, _vp, _lg]),
    "emul_syndrome_table": (_lg, [_vp]),
    "emul_syndrome_lookup": (None, [ctypes.c_uint32, _lg, _vp]),
}


def lib():
    L = emul.lib()
    for name, (res, args) in _SIGNATURES.items():
        getattr(L, name).restype = res
        getattr(L, name).argtypes = args
    return L


def repair(recs, iq2d, cfgs, offsets=None):
    """records (REC_DTYPE, stream = row of iq2d / index of cfgs) after the kernel's repair step (BTLE_CFG_RECOVER and
    BTLE_CFG_CORRECT); iq2d int8 [n_streams, n_int8], cfgs CFG_DTYPE [n_streams]; offsets: None (no correction) or Hz per
    stream (one value for all)"""
    out = np.ascontiguousarray(recs, dtype=REC_DTYPE).copy()
    iq2d = np.ascontiguousarray(iq2d, dtype=np.int8)
    if iq2d.ndim == 1:
        iq2d = iq2d[None, :]
    cfgs = np.ascontiguousarray(cfgs)
    r4 = None if offsets is None else np.ascontiguousarray(
        [offset_ref.rot(h, 4) for h in np.broadcast_to(offsets, (iq2d.shape[0],))], dtype=np.int32)
    n = lib().emul_repair_records(iq2d.ctypes.data, iq2d.shape[1], iq2d.shape[1], cfgs.ctypes.data, None if r4 is None else r4.ctypes.data,
                                  out.ctypes.data, out.size)
    assert n >= 0
    return out


def syndrome_table():
    """(number of patterns, the table's 4096 uint64 entries: syndrome << 32 | code, 0 = empty)"""
    tab = np.zeros(4096, dtype=np.uint64)
    n = lib().emul_syndrome_table(tab.ctypes.data)
    return n, tab


def syndrome_lookup(s0, n):
    """int16 [n]: syndrome_lookup's code of s0 .. s0 + n - 1 (-1: none)"""
    code = np.empty(n, dtype=np.int16)
    lib().emul_syndrome_lookup(s0, n, code.ctypes.data)
    return code
