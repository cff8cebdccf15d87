"""numpy restatement of the receive kernel's discriminator bits in every mode and of the per-packet offset estimate
(definitions in include/btle_b200.h): the carrier-offset rotation, the reference's and the symbol-spaced bits, and
btle_b200_rec_offset.  The oracle chain over these bits is tests/mode_ref.py."""
from __future__ import annotations

import numpy as np

import recover_ref

AA_OFFSET = 39                     # BTLE_RX_BER_AA_OFFSET
OFF_LEAD, OFF_TURNS = 32, 156


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


def dbits_sym(x: np.ndarray, n: int, c: int = 16384, s: int = 0) -> np.ndarray:
    """symbol-spaced d[0..n): the (rotated) discriminator of samples m - 2 and m + 2; x = int8 interleaved samples from
    sample -2 on (at least 2 (n + 4) values).  (16384, 0) is the unrotated bit, (C4, S4) the rotated one."""
    x = np.asarray(x, dtype=np.int64)
    return disc(x[0:2 * n:2], x[1:2 * n:2], x[8:2 * n + 8:2], x[9:2 * n + 8:2], c, s).astype(np.uint8)


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
