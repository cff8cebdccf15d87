"""numpy restatement of the carrier-offset correction and of the per-packet offset estimate (definitions in
include/btle_b200.h), over the pinned oracle chain: the rotated discriminator bits go through orc_search /
orc_demod_bytes as orc_receiver_chunk_ex uses them (oracle/btle_oracle.c), so at offset 0 this is the oracle itself.
Also the loader of the test-only emulator tests/emul/btle_offset_emul.cpp.  Used by tests/test_offset.py (CPU) and
tests/test_offset_gpu.py."""
from __future__ import annotations

import ctypes
import os
import subprocess

import numpy as np

import orc
import recover_ref
from btle_b200 import synth
from emul import DEPS, HERE

CHUNK_INT8, WIN_INT8, SEARCH_INT8 = 16384, 19392, 16632
WIN_SAMPLES = WIN_INT8 // 2
MAX_RECS_PER_CHUNK = 123
AA_OFFSET = 39                     # BTLE_RX_BER_AA_OFFSET
OFF_LEAD, OFF_TURNS = 32, 156
_WHITEN = synth.whitening_table()


def rot(hz: float, k: int = 1):
    """(C, S) of offset hz over k samples: round(2^14 cos / sin (k phi)), phi = 2 pi hz / 4 MHz (hz as float32, as passed)"""
    ph = 2 * np.pi * float(np.float32(hz)) / 4e6 * k
    return int(np.rint(16384.0 * np.cos(ph))), int(np.rint(16384.0 * np.sin(ph)))


def disc(i0, q0, i1, q1, c: int, s: int) -> np.ndarray:
    """the rotated discriminator bit, int64 arithmetic: C (I0 Q1 - I1 Q0) - S (I0 I1 + Q0 Q1) > 0"""
    i0, q0, i1, q1 = (np.asarray(x, dtype=np.int64) for x in (i0, q0, i1, q1))
    return (c * (i0 * q1 - i1 * q0) - s * (i0 * i1 + q0 * q1)) > 0


def dbits(x: np.ndarray, n: int, c: int, s: int) -> np.ndarray:
    """d[0..n) of int8 interleaved samples x (at least 2 (n + 1) values)"""
    x = np.asarray(x, dtype=np.int64)
    return disc(x[0:2 * n:2], x[1:2 * n:2], x[2:2 * n + 2:2], x[3:2 * n + 2:2], c, s).astype(np.uint8)


def _mag(win: np.ndarray, n0: int) -> int:
    a = 2 * n0 + np.arange(256)
    v = np.where((a >= -256) & (a < win.size - 256), win[np.clip(a + 256, 0, win.size - 1)].astype(np.int64), 0)
    return int(np.abs(v).sum()) & 0xFFFF


def receiver_chunk(win: np.ndarray, c: int, s: int, channel: int, access_addr: int, access_mask: int, crc_init: int, raw: int,
                   rssi: int, stream: int, chunk: int) -> list:
    """orc_receiver_chunk_ex on the rotated bits; win = 256 int8 in front of the chunk, its 19392-int8 window, 8 behind"""
    L = orc.lib()
    d = np.zeros(WIN_SAMPLES + 4, dtype=np.uint8)
    d[:WIN_SAMPLES] = dbits(win[256:], WIN_SAMPLES, c, s)
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


def rx_stream(iq: np.ndarray, offset_hz: float, channel=37, access_addr=0x8E89BED6, access_mask=0xFFFFFFFF, crc_init=0x555555, raw=0,
              rssi=0, stream=0) -> np.ndarray:
    """records of one capture decoded with the correction (orc_rx_stream_ex's chunking; BTLE_CFG_RECOVER in rssi applied
    with the 4-sample rotation)"""
    iq = np.asarray(iq, dtype=np.int8).reshape(-1)
    c, s = rot(offset_hz)
    recs = []
    for k in range(iq.size // CHUNK_INT8):
        base = k * CHUNK_INT8
        win = np.zeros(256 + WIN_INT8 + 8, dtype=np.int8)
        lo, hi = max(base - 256, 0), min(base + WIN_INT8 + 8, iq.size)
        win[lo - base + 256:hi - base + 256] = iq[lo:hi]
        recs += receiver_chunk(win, c, s, channel, access_addr, access_mask, crc_init, raw, rssi, stream, k)
    out = np.array(recs, dtype=orc.REC_DTYPE) if recs else np.zeros(0, dtype=orc.REC_DTYPE)
    if rssi & recover_ref.CFG_RECOVER and not raw:
        out = recover(out, iq, offset_hz, crc_init)
    return out


def sym_bits(w: np.ndarray, c4: int, s4: int) -> np.ndarray:
    """recover_ref.sym_bits with the 4-sample rotation"""
    nxt = np.zeros_like(w)
    nxt[:-4] = w[4:]
    return disc(w[:, 0], w[:, 1], nxt[:, 0], nxt[:, 1], c4, s4)


def recover(recs: np.ndarray, iq: np.ndarray, offset_hz: float, crc_init: int = 0x555555) -> np.ndarray:
    """recover_ref.apply with the rotated symbol-spaced bits"""
    c4, s4 = rot(offset_hz, 4)
    out = recs.copy()
    cache = {}
    for k, r in enumerate(out):
        if not r["crc_bad"] or r["flags"] & 4:
            continue
        ch = int(r["chunk"])
        if ch not in cache:
            cache[ch] = sym_bits(recover_ref.window(iq, ch), c4, s4)
        got = recover_ref.recover_one(cache[ch], int(r["n0"]), int(r["channel"]), crc_init)
        if got is None:
            continue
        q, b = got
        r["bytes"][:] = 0
        r["bytes"][:b.size] = b
        r["n_bytes"], r["crc_bad"] = b.size, 0
        r["flags"] = int(r["flags"]) | recover_ref.REC_RECOVERED | (q << 4)
        out[k] = r
    return out


# ---- the per-packet estimate ------------------------------------------------------------------------------------------
_COS = np.rint(127 * np.cos(2 * np.pi * np.arange(1024) / 1024)).astype(np.int64)
_SIN = np.rint(127 * np.sin(2 * np.pi * np.arange(1024) / 1024)).astype(np.int64)
_GAUSS4 = np.array([2, 11, 32, 53, 60, 53, 32, 11, 2], dtype=np.int64)


def tx_waveform(access_addr: int, n_samples: int) -> np.ndarray:
    """int64 [n_samples, 2]: the btle_tx 4-sps waveform (table samples, phase before each frequency word) of the preamble
    and access address alone"""
    sb = [0x55 if access_addr & 1 else 0xAA] + [(access_addr >> (8 * i)) & 0xFF for i in range(4)]
    bits = np.array([(sb[k >> 3] >> (k & 7)) & 1 for k in range(40)]) * 2 - 1
    f = np.zeros(n_samples, dtype=np.int64)
    for m in range(n_samples):
        for j in range(3, 12):
            idx = m + j - 15
            if idx >= 0 and idx % 4 == 0 and idx // 4 < 40:
                f[m] += _GAUSS4[j - 3] * bits[idx // 4]
    ph = np.concatenate([[0], np.cumsum(f)[:-1]]) & 1023
    return np.stack([_COS[ph], _SIN[ph]], axis=1)


def turns(x: np.ndarray) -> np.ndarray:
    """arg(conj(x[n]) x[n+1]) of int [n, 2] samples, in float32 as the kernel's atan2f"""
    i0, q0, i1, q1 = x[:-1, 0], x[:-1, 1], x[1:, 0], x[1:, 1]
    return np.arctan2((i0 * q1 - q0 * i1).astype(np.float32), (i0 * i1 + q0 * q1).astype(np.float32))


def ref_sum(access_addr: int) -> float:
    t = tx_waveform(access_addr, AA_OFFSET - OFF_LEAD + OFF_TURNS + 1)
    return float(turns(t[AA_OFFSET - OFF_LEAD:]).astype(np.float64).sum())


def rec_offset(iq: np.ndarray, chunk: int, n0: int, access_addr: int) -> float:
    """the estimate of one record of capture iq (float64 sums; the kernel's float32 agrees to rounding)"""
    w = recover_ref.window(iq, chunk).astype(np.int64)
    n = n0 - OFF_LEAD + np.arange(OFF_TURNS + 1)
    x = np.where(((n >= 0) & (n < w.shape[0]))[:, None], w[np.clip(n, 0, w.shape[0] - 1)], 0)
    return 4e6 / (2 * np.pi * OFF_TURNS) * (float(turns(x).astype(np.float64).sum()) - ref_sum(access_addr))


# ---- emulator loader ---------------------------------------------------------------------------------------------------
SRC = os.path.join(HERE, "emul", "btle_offset_emul.cpp")
SO = os.path.join(HERE, "emul", "libbtle_offset_emul.so")
_lib = None


def emul():
    global _lib
    if _lib is None:
        if (not os.path.exists(SO)) or any(os.path.getmtime(SO) < os.path.getmtime(d) for d in DEPS[1:] + [SRC]):
            subprocess.run(["g++", "-O2", "-fPIC", "-shared", "-std=c++17", "-x", "c++", "-o", SO, SRC], check=True)
        _lib = ctypes.CDLL(SO)
        _lib.emul_rot_phase_words.restype = None
        _lib.emul_rot_phase_words.argtypes = [ctypes.c_void_p, ctypes.c_long, ctypes.c_int, ctypes.c_int, ctypes.c_void_p]
        _lib.emul_recover_records_rot.restype = ctypes.c_long
        _lib.emul_recover_records_rot.argtypes = [ctypes.c_void_p, ctypes.c_long, ctypes.c_long, ctypes.c_void_p, ctypes.c_void_p,
                                                  ctypes.c_void_p, ctypes.c_long]
    return _lib


def emul_dbits(iq: np.ndarray, c: int, s: int) -> np.ndarray:
    """d[0 .. 128 ngroups) from the emulated dense warps' phase words; iq int8 of 256 ngroups + 4 values"""
    iq = np.ascontiguousarray(iq, dtype=np.int8)
    ng = (iq.size - 4) // 256
    words = iq[:256 * ng + 4].view(np.uint32)
    pd = np.zeros(4 * ng, dtype=np.uint32)
    emul().emul_rot_phase_words(words.ctypes.data, ng, c, s, pd.ctypes.data)
    bits = ((pd.reshape(ng, 4, 1) >> np.arange(32, dtype=np.uint32)) & 1).astype(np.uint8)    # [g, ph, i]
    return bits.transpose(0, 2, 1).reshape(-1)                                                 # d[128 g + 4 i + ph]


def emul_recover(recs, iq2d, cfgs, offsets) -> np.ndarray:
    out = np.ascontiguousarray(recs, dtype=orc.REC_DTYPE).copy()
    iq2d = np.ascontiguousarray(iq2d, dtype=np.int8)
    if iq2d.ndim == 1:
        iq2d = iq2d[None, :]
    r4 = np.ascontiguousarray([rot(h, 4) for h in np.broadcast_to(offsets, (iq2d.shape[0],))], dtype=np.int32)
    cfgs = np.ascontiguousarray(cfgs)
    emul().emul_recover_records_rot(iq2d.ctypes.data, iq2d.shape[1], iq2d.shape[1], cfgs.ctypes.data, r4.ctypes.data, out.ctypes.data,
                                    out.size)
    return out
