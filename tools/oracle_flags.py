"""The oracle's records as the GPU returns them for a given btle_stream_cfg.rssi flag word, for the fuzz tools:
bit 0 (BTLE_CFG_RSSI) keeps mag_sum (else 0), bit 1 (BTLE_CFG_REPORT_REJECTED) adds the rejected hits
(orc_rx_stream_ex, oracle/btle_oracle.h).  Uses only the loader and record layout of tests/orc.py."""
import ctypes

import numpy as np

import orc


def expect(iq, flags, channel=37, access_addr=0x8E89BED6, access_mask=0xFFFFFFFF, crc_init=0x555555, raw=0, stream=0):
    iq = np.ascontiguousarray(iq, dtype=np.int8)
    L = orc.lib()
    L.orc_rx_stream_ex.restype = ctypes.c_long
    L.orc_rx_stream_ex.argtypes = [ctypes.c_void_p, ctypes.c_long, ctypes.POINTER(orc.OrcCfg), ctypes.c_int, ctypes.c_int32,
                                   ctypes.c_void_p, ctypes.c_long]
    cfg = orc.OrcCfg(channel, access_addr, access_mask, crc_init, raw)
    cap = (iq.size // 16384) * 123 + 8          # BTLE_MAX_RECS_PER_CHUNK
    out = np.zeros(cap, dtype=orc.REC_DTYPE)
    n = L.orc_rx_stream_ex(iq.ctypes.data, iq.size, ctypes.byref(cfg), (flags >> 1) & 1, stream, out.ctypes.data, cap)
    assert n <= cap
    rec = out[:n]
    if not flags & 1:
        rec["mag_sum"] = 0
    return rec
