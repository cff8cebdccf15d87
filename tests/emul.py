"""Loader for the test-only CPU emulator of the kernel logic (tests/emul/btle_emul.cpp)."""
import ctypes
import os
import subprocess

import numpy as np

from orc import REC_DTYPE

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
SRC = os.path.join(HERE, "emul", "btle_emul.cpp")
SO = os.path.join(HERE, "emul", "libbtle_emul.so")
DEPS = [SRC, os.path.join(ROOT, "btle_b200", "csrc", "btle_core.cuh"), os.path.join(ROOT, "btle_b200", "csrc", "btle_params.h"),
        os.path.join(ROOT, "include", "btle_b200.h")]


class StreamCfg(ctypes.Structure):
    _fields_ = [("channel", ctypes.c_int32), ("access_addr", ctypes.c_uint32), ("access_mask", ctypes.c_uint32),
                ("crc_init", ctypes.c_uint32), ("raw", ctypes.c_int32), ("rssi", ctypes.c_int32)]


_lib = None


def lib():
    global _lib
    if _lib is None:
        if (not os.path.exists(SO)) or any(os.path.getmtime(SO) < os.path.getmtime(d) for d in DEPS):
            subprocess.run(["g++", "-O2", "-fPIC", "-shared", "-std=c++17", "-x", "c++", "-o", SO, SRC], check=True)
        _lib = ctypes.CDLL(SO)
        _lib.emul_rx_stream.restype = ctypes.c_long
        _lib.emul_rx_stream.argtypes = [ctypes.c_void_p, ctypes.c_long, ctypes.POINTER(StreamCfg), ctypes.c_int,
                                        ctypes.c_int, ctypes.c_void_p, ctypes.c_long]
        vp, lg = ctypes.c_void_p, ctypes.c_long
        _lib.emul_rx_units.restype = lg
        _lib.emul_rx_units.argtypes = [vp, lg, lg, lg, vp, vp, lg, ctypes.c_int, ctypes.c_int, vp, lg, vp, lg, ctypes.POINTER(lg)]
        _lib.emul_check_tapset.restype = lg
        _lib.emul_check_tapset.argtypes = [vp, vp, lg]
    return _lib


def rx_stream(iq, channel=37, access_addr=0x8E89BED6, access_mask=0xFFFFFFFF, crc_init=0x555555, raw=0, rssi=1,
              stream=0, span_chunks=16, report_rejected=0):
    """rssi: btle_stream_cfg flags (bit 0 RSSI, bit 1 report rejected hits); report_rejected=1 sets bit 1 as well."""
    iq = np.ascontiguousarray(iq, dtype=np.int8)
    cfg = StreamCfg(channel, access_addr, access_mask, crc_init, raw, rssi | (2 if report_rejected else 0))
    cap = (iq.size // 16384) * 123 + 8     # BTLE_MAX_RECS_PER_CHUNK
    out = np.zeros(cap, dtype=REC_DTYPE)
    n = lib().emul_rx_stream(iq.ctypes.data, iq.size, ctypes.byref(cfg), stream, span_chunks, out.ctypes.data, cap)
    assert n <= cap
    return out[:n]


def rx_units(iq2d, cfgs, capture=None, grid=132, reverse_units=False, force_walk=False):
    """The kernel's unit plan + resolver passes on the CPU (emul_rx_units), the kernel chosen as launch_rx chooses it.
    iq2d: int8 [n_captures, n_int8]; cfgs: CFG_DTYPE array; capture[j]: the capture cfg j decodes (None: cfg j on capture j).
    Returns (count, records as stored (block per (cfg, unit)), dir uint32 [n_entries, 2]); count is -1 for a refused launch."""
    iq2d = np.ascontiguousarray(iq2d, dtype=np.int8)
    ns, n = iq2d.shape
    cfgs = np.ascontiguousarray(cfgs).reshape(-1)
    cc = None if capture is None else np.ascontiguousarray(capture, dtype=np.int32)
    cap = cfgs.size * (n // 16384) * 123 + 8      # BTLE_MAX_RECS_PER_CHUNK
    out = np.zeros(cap, dtype=REC_DTYPE)
    dir_cap = cfgs.size * ((n // 16384 + 15) // 16 * 16 + 16)
    d = np.zeros((dir_cap, 2), dtype=np.uint32)
    nd = ctypes.c_long(0)
    cnt = lib().emul_rx_units(iq2d.ctypes.data, ns, n, n, cfgs.ctypes.data, None if cc is None else cc.ctypes.data, cfgs.size, grid,
                              int(reverse_units) | (2 if force_walk else 0), out.ctypes.data, cap, d.ctypes.data, dir_cap, ctypes.byref(nd))
    assert cnt <= cap
    return cnt, out[:max(cnt, 0)], d[:nd.value]


def rx_batch_units(iq2d, cfgs, grid=132, reverse_units=False, force_walk=False):
    """rx_units with one cfg per capture: (records as stored (block per unit), dir uint32 [n_units, 2])."""
    cnt, out, d = rx_units(iq2d, cfgs, None, grid, reverse_units, force_walk)
    assert cnt >= 0
    return out, d


def rx_multi(iq2d, cfgs, capture, grid=132, reverse_units=False, force_walk=False):
    """rx_units with a cfg list, records gathered through the unit directory (reference order)."""
    cnt, out, d = rx_units(iq2d, cfgs, capture, grid, reverse_units, force_walk)
    assert cnt >= 0
    return np.concatenate([out[b:b + c] for b, c in d]) if len(d) else out[:0]


def check_tapset(cfg, words):
    """prefilter_union of one cfg against prefilter_any, over consecutive (lo, hi) word pairs; returns the mismatches."""
    return int(lib().emul_check_tapset(cfg.ctypes.data, words.ctypes.data, words.size))


def tables():
    w = np.zeros((40, 42), dtype=np.uint8)
    c = np.zeros(256, dtype=np.uint32)
    lib().emul_tables(w.ctypes.data, c.ctypes.data)
    return w, c


def check_discriminator():
    """Exhaustive check (2^32 int8 quadruples) of the dense loop's one-dp2a discriminator and of its two sign-bit gathers on
    the modelled prmt / dp2a / dp4a semantics; returns the number of violations."""
    L = lib()
    L.emul_check_discriminator.restype = ctypes.c_long
    L.emul_check_discriminator.argtypes = []
    return int(L.emul_check_discriminator())
