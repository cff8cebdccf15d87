"""Test-side access to the oracle (oracle/libbtle_oracle.so = our C restatement,
oracle/_ref/btle_ref_driver = the unmodified reference receiver).  Only tests,
__graft_entry__.smoke() and bench.py's CPU-baseline legs may import this."""
from __future__ import annotations

import ctypes
import os
import subprocess
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ORACLE_DIR = os.path.join(ROOT, "oracle")
ORACLE_SO = os.path.join(ORACLE_DIR, "libbtle_oracle.so")
REF_DRIVER = os.path.join(ORACLE_DIR, "_ref", "btle_ref_driver")

# layout shared by orc_rec (oracle/btle_oracle.h) and btle_pkt_rec (include/btle_b200.h)
REC_DTYPE = np.dtype([
    ("stream", "<i4"), ("chunk", "<i4"), ("n0", "<i4"),
    ("channel", "u1"), ("n_bytes", "u1"), ("crc_bad", "u1"), ("flags", "u1"),
    ("access_addr", "<u4"), ("mag_sum", "<u2"), ("bytes", "u1", 42),
])
assert REC_DTYPE.itemsize == 64
REF_DTYPE = np.dtype([("chunk", "<i4"), ("n0", "<i4"), ("nbytes", "<i4"), ("crc_bad", "<i4"), ("bytes", "u1", 48)])


class OrcCfg(ctypes.Structure):
    _fields_ = [("channel", ctypes.c_int32), ("access_addr", ctypes.c_uint32), ("access_mask", ctypes.c_uint32),
                ("crc_init", ctypes.c_uint32), ("raw", ctypes.c_int32)]


def build_oracle():
    src = os.path.join(ORACLE_DIR, "btle_oracle.c")
    if (not os.path.exists(ORACLE_SO)) or os.path.getmtime(ORACLE_SO) < os.path.getmtime(src):
        subprocess.run(["make", "-C", ORACLE_DIR, "oracle"], check=True, capture_output=True)
    return ORACLE_SO


_lib = None


def lib():
    global _lib
    if _lib is None:
        _lib = ctypes.CDLL(build_oracle())
        _lib.orc_crc_init_reorder.restype = ctypes.c_uint32
        _lib.orc_crc_init_reorder.argtypes = [ctypes.c_uint32]
        _lib.orc_crc24.restype = ctypes.c_uint32
        _lib.orc_crc24.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_uint32]
        _lib.orc_whiten_byte.restype = ctypes.c_uint8
        _lib.orc_whiten_byte.argtypes = [ctypes.c_int, ctypes.c_int]
        _lib.orc_dbits.argtypes = [ctypes.c_void_p, ctypes.c_long, ctypes.c_void_p]
        _lib.orc_search.restype = ctypes.c_int
        _lib.orc_search.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_uint32, ctypes.c_uint32,
                                    ctypes.POINTER(ctypes.c_int)]
        _lib.orc_demod_bytes.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_void_p]
        _lib.orc_rx_stream.restype = ctypes.c_long
        _lib.orc_rx_stream.argtypes = [ctypes.c_void_p, ctypes.c_long, ctypes.POINTER(OrcCfg), ctypes.c_int32,
                                       ctypes.c_void_p, ctypes.c_long]
        _lib.orc_rx_stream_ex.restype = ctypes.c_long
        _lib.orc_rx_stream_ex.argtypes = [ctypes.c_void_p, ctypes.c_long, ctypes.POINTER(OrcCfg), ctypes.c_int, ctypes.c_int32,
                                          ctypes.c_void_p, ctypes.c_long]
    return _lib


MAX_RECS_PER_CHUNK = 123                   # BTLE_MAX_RECS_PER_CHUNK (include/btle_b200.h)


def rx_stream(iq: np.ndarray, channel=37, access_addr=0x8E89BED6, access_mask=0xFFFFFFFF, crc_init=0x555555,
              raw=0, stream=0, report_rejected=0) -> np.ndarray:
    """Our C restatement over one capture -> REC_DTYPE array in reference order.  report_rejected (-v): the ADV hits
    the reference prints as PktBAD come back too, as header-only records with flags bit 2 set."""
    iq = np.ascontiguousarray(iq, dtype=np.int8)
    cfg = OrcCfg(channel, access_addr, access_mask, crc_init, raw)
    cap = (iq.size // 16384) * MAX_RECS_PER_CHUNK + 8
    out = np.zeros(cap, dtype=REC_DTYPE)
    n = lib().orc_rx_stream_ex(iq.ctypes.data, iq.size, ctypes.byref(cfg), int(bool(report_rejected)), stream, out.ctypes.data, cap)
    assert n <= cap
    return out[:n]


def rx_flags(iq: np.ndarray, flags: int, **cfg) -> np.ndarray:
    """The oracle's records as the GPU returns them for btle_stream_cfg.rssi == flags: bit 0 (BTLE_CFG_RSSI) keeps
    mag_sum (else 0), bit 1 (BTLE_CFG_REPORT_REJECTED) adds the rejected hits."""
    rec = rx_stream(iq, report_rejected=(flags >> 1) & 1, **cfg)
    if not flags & 1:
        rec["mag_sum"] = 0
    return rec


def dbits(iq: np.ndarray) -> np.ndarray:
    """d[n] for n in [0, len/2 - 1)."""
    iq = np.ascontiguousarray(iq, dtype=np.int8)
    n = iq.size // 2 - 1
    d = np.zeros(n, dtype=np.uint8)
    lib().orc_dbits(iq.ctypes.data, n, d.ctypes.data)
    return d


def ref_available() -> bool:
    return os.path.exists(REF_DRIVER)


def ref_rx_stream(iq: np.ndarray, channel=37, access_addr=0x8E89BED6, access_mask=0xFFFFFFFF, crc_init=0x555555,
                  raw=0, report_rejected=0) -> np.ndarray:
    """The unmodified reference receiver() over one capture -> REF_DTYPE array.  report_rejected: also the hits it
    rejects for their ADV header length (what -v prints as PktBAD), as records with nbytes 2 and the two header bytes."""
    iq = np.ascontiguousarray(iq, dtype=np.int8)
    with tempfile.TemporaryDirectory() as td:
        fi, fo = os.path.join(td, "iq.bin"), os.path.join(td, "out.rec")
        iq.tofile(fi)
        subprocess.run([REF_DRIVER, "run", fi, str(channel), f"{access_addr:x}", f"{crc_init:x}", f"{access_mask:x}",
                        str(int(raw)), fo] + (["rejected"] if report_rejected else []), check=True, capture_output=True)
        return np.fromfile(fo, dtype=REF_DTYPE)


def ref_time(iq_path: str, channel=37, access_addr=0x8E89BED6, access_mask=0xFFFFFFFF, crc_init=0x555555, raw=0,
             procs=1, reps=1) -> dict:
    import json
    p = subprocess.run([REF_DRIVER, "time", iq_path, str(channel), f"{access_addr:x}", f"{crc_init:x}",
                        f"{access_mask:x}", str(int(raw)), str(procs), str(reps)], check=True, capture_output=True)
    return json.loads(p.stdout.decode().strip().splitlines()[-1])


def assert_same_as_ref(rec: np.ndarray, ref: np.ndarray):
    """REC_DTYPE records (oracle or GPU) vs REF_DTYPE records (reference)."""
    assert len(rec) == len(ref), f"packet count {len(rec)} != reference {len(ref)}"
    for a, b in zip(rec, ref):
        assert a["chunk"] == b["chunk"] and a["n0"] == b["n0"], (a["chunk"], a["n0"], b["chunk"], b["n0"])
        assert a["n_bytes"] == b["nbytes"] and a["crc_bad"] == b["crc_bad"]
        assert bool(a["flags"] & 4) == (b["nbytes"] == 2), (a["chunk"], a["n0"])    # rejected hit <=> header only
        nb = int(b["nbytes"])
        assert bytes(a["bytes"][:nb]) == bytes(b["bytes"][:nb])
