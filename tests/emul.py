"""Loader for the test-only CPU emulator of the kernel logic (tests/emul/, one library; its sources are listed in
__graft_entry__.EMUL_SRCS), and the thin wrappers the tests call it through."""
import ctypes
import os
import subprocess

import numpy as np

import offset_ref
from __graft_entry__ import EMUL_SO as SO, EMUL_SRCS as SRCS
from btle_b200 import CAND_DTYPE
from btle_b200._native import CFG_SYMBOL_SPACED
from orc import REC_DTYPE

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DEPS = SRCS + [os.path.join(ROOT, "btle_b200", "csrc", "btle_core.cuh"), os.path.join(ROOT, "btle_b200", "csrc", "btle_params.h"),
               os.path.join(ROOT, "include", "btle_b200.h")]


class StreamCfg(ctypes.Structure):
    _fields_ = [("channel", ctypes.c_int32), ("access_addr", ctypes.c_uint32), ("access_mask", ctypes.c_uint32),
                ("crc_init", ctypes.c_uint32), ("raw", ctypes.c_int32), ("rssi", ctypes.c_int32)]


_vp, _lg, _int, _u32 = ctypes.c_void_p, ctypes.c_long, ctypes.c_int, ctypes.c_uint32
_SIGNATURES = {                                   # name: (restype, argtypes)
    "emul_rx_stream": (_lg, [_vp, _lg, ctypes.POINTER(StreamCfg), _int, _int, _vp, _lg]),
    "emul_rx_units": (_lg, [_vp, _lg, _lg, _lg, _vp, _vp, _lg, _int, _int, _int, _vp, _lg, _vp, _lg, ctypes.POINTER(_lg)]),
    "emul_check_tapset": (_lg, [_vp, _vp, _lg]),
    "emul_crc24_words": (_u32, [_vp, _int, _u32]),
    "emul_tables": (None, [_vp, _vp]),
    "emul_plan": (_lg, [_lg, _lg, _int, _vp, _lg]),
    "emul_rot_phase_words": (None, [_vp, _lg, _int, _int, _vp]),
    "emul_sym_phase_words": (None, [_vp, _lg, _lg, _lg, _lg, _int, _int, _int, _vp]),
    "emul_check_discriminator": (_lg, []),
    "emul_recover_records": (_lg, [_vp, _lg, _lg, _vp, _vp, _vp, _lg]),
    "emul_discover": (_lg, [_vp, _lg, _int, _int, _vp, _lg]),
    "emul_crc24_unwind": (_u32, [_u32, _u32, _int]),
}
_lib = None


def lib():
    global _lib
    if _lib is None:
        if (not os.path.exists(SO)) or any(os.path.getmtime(SO) < os.path.getmtime(d) for d in DEPS):
            subprocess.run(["g++", "-O2", "-fPIC", "-shared", "-std=c++17", "-o", SO, *SRCS], check=True)
        L = ctypes.CDLL(SO)
        for name, (res, args) in _SIGNATURES.items():
            getattr(L, name).restype = res
            getattr(L, name).argtypes = args
        _lib = L
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
    """The kernel's unit plan + resolver passes on the CPU (emul_rx_units), the kernel chosen as launch_rx chooses it (the
    symbol-spaced dense pass when the cfgs have BTLE_CFG_SYMBOL_SPACED).  iq2d: int8 [n_captures, n_int8]; cfgs: CFG_DTYPE
    array; capture[j]: the capture cfg j decodes (None: cfg j on capture j).  Returns (count, records as stored (block per
    (cfg, unit)), dir uint32 [n_entries, 2]); count is -1 for a refused launch."""
    iq2d = np.ascontiguousarray(iq2d, dtype=np.int8)
    ns, n = iq2d.shape
    cfgs = np.ascontiguousarray(cfgs).reshape(-1)
    cc = None if capture is None else np.ascontiguousarray(capture, dtype=np.int32)
    sym = int(cfgs.size > 0 and bool(cfgs["rssi"][0] & CFG_SYMBOL_SPACED))
    cap = cfgs.size * (n // 16384) * 123 + 8      # BTLE_MAX_RECS_PER_CHUNK
    out = np.zeros(cap, dtype=REC_DTYPE)
    dir_cap = cfgs.size * ((n // 16384 + 15) // 16 * 16 + 16)
    d = np.zeros((dir_cap, 2), dtype=np.uint32)
    nd = ctypes.c_long(0)
    cnt = lib().emul_rx_units(iq2d.ctypes.data, ns, n, n, cfgs.ctypes.data, None if cc is None else cc.ctypes.data, cfgs.size, grid,
                              int(reverse_units) | (2 if force_walk else 0), sym, out.ctypes.data, cap, d.ctypes.data, dir_cap,
                              ctypes.byref(nd))
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


def recover(recs, iq2d, cfgs, offsets=None):
    """records (REC_DTYPE, stream = row of iq2d / index of cfgs) after the kernel's recovery step; iq2d int8
    [n_streams, n_int8], cfgs CFG_DTYPE [n_streams]; offsets: None (no correction) or Hz per stream (one value for all)"""
    out = np.ascontiguousarray(recs, dtype=REC_DTYPE).copy()
    iq2d = np.ascontiguousarray(iq2d, dtype=np.int8)
    if iq2d.ndim == 1:
        iq2d = iq2d[None, :]
    cfgs = np.ascontiguousarray(cfgs)
    r4 = None if offsets is None else np.ascontiguousarray(
        [offset_ref.rot(h, 4) for h in np.broadcast_to(offsets, (iq2d.shape[0],))], dtype=np.int32)
    lib().emul_recover_records(iq2d.ctypes.data, iq2d.shape[1], iq2d.shape[1], cfgs.ctypes.data, None if r4 is None else r4.ctypes.data,
                               out.ctypes.data, out.size)
    return out


def _bits(pd, ng):
    """d[128 g + 4 i + ph] = bit i of phase word pd[4 g + ph]"""
    bits = ((pd.reshape(ng, 4, 1) >> np.arange(32, dtype=np.uint32)) & 1).astype(np.uint8)    # [g, ph, i]
    return bits.transpose(0, 2, 1).reshape(-1)


def rot_dbits(iq, c, s):
    """d[0 .. 128 ngroups) of the rotated discriminator with (c, s) from the emulated dense warps' phase words; iq int8 of
    256 ngroups + 4 values"""
    iq = np.ascontiguousarray(iq, dtype=np.int8)
    ng = (iq.size - 4) // 256
    words = iq[:256 * ng + 4].view(np.uint32)
    pd = np.zeros(4 * ng, dtype=np.uint32)
    lib().emul_rot_phase_words(words.ctypes.data, ng, c, s, pd.ctypes.data)
    return _bits(pd, ng)


def sym_dbits(buf, at, n_int8, lead, g0, ng, hz=None):
    """symbol-spaced d[128 g0 .. 128 (g0 + ng)) from the emulated dense pass, rotated by (C4, S4) of hz (None: unrotated);
    the capture is buf[at : at + n_int8], buf[at - lead : at] readable in front of it"""
    buf = np.ascontiguousarray(buf, dtype=np.int8)
    pd = np.zeros(4 * ng, dtype=np.uint32)
    c, s = (16384, 0) if hz is None else offset_ref.rot(hz, 4)
    lib().emul_sym_phase_words(buf.ctypes.data + at, n_int8, lead, g0, ng, int(hz is not None), c, s, pd.ctypes.data)
    return _bits(pd, ng)


def discover(iq, channel, stream=0):
    """emul_discover's candidates of one capture, in sample order"""
    iq = np.ascontiguousarray(iq, dtype=np.int8)
    cap = iq.size // 8 + 64
    out = np.zeros(cap, dtype=CAND_DTYPE)
    n = lib().emul_discover(iq.ctypes.data, iq.size, channel, stream, out.ctypes.data, cap)
    assert n <= cap
    out = out[:n]
    return out[np.argsort(out["sample"], kind="stable")]


def plan(n_streams, nchunks, grid):
    """int32 [n_units, 3]: (stream, chunk0, n_chunks) of every unit of a launch shape (make_plan / unit_info)"""
    cap = n_streams * ((nchunks + 15) // 16) * 16 + 16
    buf = np.zeros((cap, 3), dtype=np.int32)
    n = lib().emul_plan(n_streams, nchunks, grid, buf.ctypes.data, cap)
    assert 0 <= n <= cap, (n_streams, nchunks, grid, n)
    return buf[:n]


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
    return int(lib().emul_check_discriminator())
