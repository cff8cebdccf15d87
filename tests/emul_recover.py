"""Loader for the test-only CPU emulator of BTLE_CFG_RECOVER (tests/emul/btle_recover_emul.cpp): the kernel's
recover_packet over the records of the emulated receive passes (tests/emul.py)."""
import ctypes
import os
import subprocess

import numpy as np

from emul import DEPS, HERE
from orc import REC_DTYPE

SRC = os.path.join(HERE, "emul", "btle_recover_emul.cpp")
SO = os.path.join(HERE, "emul", "libbtle_recover_emul.so")

_lib = None


def lib():
    global _lib
    if _lib is None:
        if (not os.path.exists(SO)) or any(os.path.getmtime(SO) < os.path.getmtime(d) for d in DEPS[1:] + [SRC]):
            subprocess.run(["g++", "-O2", "-fPIC", "-shared", "-std=c++17", "-x", "c++", "-o", SO, SRC], check=True)
        _lib = ctypes.CDLL(SO)
        _lib.emul_recover_records.restype = ctypes.c_long
        _lib.emul_recover_records.argtypes = [ctypes.c_void_p, ctypes.c_long, ctypes.c_long, ctypes.c_void_p, ctypes.c_void_p,
                                              ctypes.c_long]
    return _lib


def recover(recs, iq2d, cfgs):
    """records (REC_DTYPE, stream = row of iq2d / index of cfgs) after the kernel's recovery step; iq2d int8
    [n_streams, n_int8], cfgs CFG_DTYPE [n_streams]"""
    out = np.ascontiguousarray(recs, dtype=REC_DTYPE).copy()
    iq2d = np.ascontiguousarray(iq2d, dtype=np.int8)
    if iq2d.ndim == 1:
        iq2d = iq2d[None, :]
    cfgs = np.ascontiguousarray(cfgs)
    lib().emul_recover_records(iq2d.ctypes.data, iq2d.shape[1], iq2d.shape[1], cfgs.ctypes.data, out.ctypes.data, out.size)
    return out
