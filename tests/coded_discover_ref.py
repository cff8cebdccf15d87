"""Restatement of LE Coded PHY connection discovery (include/btle_b200.h, "Coded connection discovery") in numpy and
plain Python.

It is written from the rules in the header and uses the coded receiver's restatement (coded_ref.py) for the
discriminator, the soft values and the trellis.  The GPU candidates of btle_b200_discover_coded* are checked against it
byte for byte (tests/test_coded_discover_gpu.py)."""
from __future__ import annotations

import numpy as np

import coded_ref as cr
from discover_ref import crc_init_for
from btle_b200 import synth

T_PRE, T_Q, WIDE, SHIFTS = 24, 80, 256, 4     # BTLE_CODED_DISC_T_PRE, _T_Q, _W, _K
LO, SPAN = 323, 1184                          # Q(n0) is defined for LO <= n0 and n0 + SPAN <= n_samples
PRE_WORD = 0x3C3C3C3C

# btle_coded_cand, 32 bytes
CODED_CAND_DTYPE = np.dtype([("sample", "<i8"), ("stream", "<i4"), ("access_addr", "<u4"), ("crc_init", "<u4"), ("channel", "u1"),
                             ("header", "u1", 2), ("s", "u1"), ("dist", "<i2"), ("shift", "i1"), ("reserved", "u1"), ("metric", "<i4")])
assert CODED_CAND_DTYPE.itemsize == 32


def statistics(h: np.ndarray):
    """(Dpre, Q) for every n0 of a capture of hard bits h (h.size samples), -1 where Q is not defined.

    Dpre(n0) = #{j = -80..-1 : h[n0 + 4j] != preamble[j]}; C(n0) = sum over the 74 groups k of block 1 (symbols 4k..4k+3)
    of the Hamming distance to the nearer of 0,0,1,1 and 1,1,0,0; Q = Dpre + C."""
    h = np.asarray(h, dtype=np.int64)
    N = h.size
    Dpre = np.full(N, -1, np.int64)
    Q = np.full(N, -1, np.int64)
    hi = N - SPAN
    if hi < LO:
        return Dpre, Q
    n0 = np.arange(LO, hi + 1)
    dp = np.zeros(n0.size, np.int64)
    for j in range(-80, 0):
        dp += h[n0 + 4 * j] != synth.CODED_PREAMBLE[j + 80]
    # per-sample group term: g[n] = distance of (h[n], h[n+4], h[n+8], h[n+12])
    m = N - 12
    s0, s1, s2, s3 = h[0:m], h[4:m + 4], h[8:m + 8], h[12:m + 12]
    g = (s0 != s1).astype(np.int64) + (s2 != s3) + 2 * ((s0 == s1) & (s1 == s2) & (s2 == s3))
    c = np.zeros(n0.size, np.int64)
    for k in range(74):
        c += g[n0 + 16 * k]
    Dpre[n0], Q[n0] = dp, dp + c
    return Dpre, Q


def hits(Dpre: np.ndarray, Q: np.ndarray) -> np.ndarray:
    """n0 with Dpre <= T_PRE, Q <= T_Q, Q strictly below every defined Q in [n0 - WIDE, n0 - 1] and no higher than every
    defined one in [n0 + 1, n0 + WIDE]"""
    big = np.where(Q < 0, 1 << 30, Q)
    out = []
    for n in np.nonzero((Q >= 0) & (Q <= T_Q) & (Dpre <= T_PRE))[0]:
        q = big[n]
        left, right = big[max(n - WIDE, 0):n], big[n + 1:n + 1 + WIDE]
        if np.all(q < left) and np.all(q <= right):
            out.append(int(n))
    return np.array(out, dtype=np.int64)


def _pre_sign() -> np.ndarray:
    return 2 * synth.CODED_PREAMBLE.astype(np.int64) - 1


def alignment(cap: cr.Capture, m: int):
    """(score, block-1 decisions) of alignment m: the preamble's soft correlation plus the block-1 path metric ending in
    state 0 (37 steps of the coded trellis from state 0, S=8 soft values of symbols 0..295)"""
    y = cap.y_at(m + 4 * np.arange(-80, 296))
    pre = int((_pre_sign() * y[:80]).sum())
    yb = y[80:].reshape(74, 4)
    L = yb[:, 0] + yb[:, 1] - yb[:, 2] - yb[:, 3]
    hist, dec = cr.viterbi(L, 37)
    return pre + hist[-1][0], dec


def decode_hit(cap: cr.Capture, n0: int, q: int, stream: int, channel: int):
    """The candidate of the hit at n0 (a CODED_CAND_DTYPE row), or None"""
    N = cap.n
    best = None
    for k in range(-SHIFTS, SHIFTS + 1):
        m = n0 + 32 * k
        if m < LO or m + SPAN > N:
            continue
        score, dec = alignment(cap, m)
        if best is None or score > best[0]:
            best = (score, k, m, dec)
    _, k, m, dec = best
    bits = cr.traceback(dec, 37, 0)
    aa = int(np.packbits(bits[:32], bitorder="little").view("<u4")[0])
    ci = int(bits[32]) | int(bits[33]) << 1
    if ci >= 2:
        return None
    s = 8 if ci == 0 else 2
    per = 4 if s == 8 else 1
    if m + 4 * (296 + 86 * per - 1) + 3 >= N:           # block 2's 43 steps must lie inside the capture
        return None
    Ls = cr.coded_soft(cap, m, s, 86)
    hist, dec2 = cr.viterbi(Ls, 43)
    b2 = cr.traceback(dec2, 43, 0)[:40] ^ synth.whitening_bits(channel, 40)
    body = np.packbits(b2, bitorder="little")
    if (body[0] & 3) != 1 or body[1] != 0:
        return None
    crc_rx = int(body[2]) | int(body[3]) << 8 | int(body[4]) << 16
    r = np.zeros(1, CODED_CAND_DTYPE)[0]
    r["sample"], r["stream"], r["access_addr"], r["channel"] = m, stream, aa, channel
    r["crc_init"] = crc_init_for(bytes(body[:2]), crc_rx)
    r["header"][0], r["header"][1] = body[0], body[1]
    r["s"], r["dist"], r["shift"], r["metric"] = s, q, k, hist[-1][0]
    return r


def discover_capture(iq: np.ndarray, channel: int, stream: int = 0, offset_hz: float = 0.0, cap: cr.Capture | None = None) -> np.ndarray:
    """Candidates of one capture in sample order"""
    cap = cr.Capture(iq, offset_hz) if cap is None else cap
    Dpre, Q = statistics(cap.h)
    out = [decode_hit(cap, int(n), int(Q[n]), stream, channel) for n in hits(Dpre, Q)]
    out = [r for r in out if r is not None]
    return np.array(out, dtype=CODED_CAND_DTYPE) if out else np.zeros(0, CODED_CAND_DTYPE)


def discover_coded(iq: np.ndarray, channels, offset_hz=None) -> np.ndarray:
    """BtleRx.discover_coded() restated: captures [n_streams, n_int8] (or [n_int8]), sorted by (stream, sample)"""
    iq = np.asarray(iq, dtype=np.int8)
    if iq.ndim == 1:
        iq = iq[None, :]
    ns = iq.shape[0]
    ch = np.broadcast_to(np.asarray(channels, np.int32), (ns,))
    off = np.zeros(ns, np.float32) if offset_hz is None else np.broadcast_to(np.asarray(offset_hz, np.float32), (ns,))
    parts = [discover_capture(iq[s], int(ch[s]), s, float(off[s])) for s in range(ns)]
    return np.concatenate(parts) if parts else np.zeros(0, CODED_CAND_DTYPE)
