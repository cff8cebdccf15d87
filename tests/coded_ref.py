"""Restatement of the LE Coded PHY receiver of include/btle_b200.h ("LE Coded PHY") in numpy and plain Python.

It is written from the rules in the header, not from the kernels, and the GPU records of btle_b200_rx_coded* are
checked against it field for field (tests/test_coded_gpu.py).  The transmitter is btle_b200.synth.coded_symbols."""
from __future__ import annotations

import math

import numpy as np

from btle_b200 import synth

MAX_DIST = 96                    # BTLE_CODED_MAX_DIST
CI_RESERVED, TRUNCATED = 1, 2    # btle_coded_rec.flags
MAX_BYTES = 260
NEG = -(1 << 29)                 # metric of a state not yet reachable
CFG_RSSI = 1

# btle_coded_rec, 304 bytes
CODED_DTYPE = np.dtype([("sample", "<i8"), ("stream", "<i4"), ("access_addr", "<u4"), ("channel", "u1"), ("s", "u1"), ("ci", "u1"),
                        ("crc_bad", "u1"), ("flags", "u1"), ("reserved0", "u1"), ("n_bytes", "<u2"), ("dist", "<i4"), ("metric", "<i4"),
                        ("mag_sum", "<u4"), ("bytes", "u1", MAX_BYTES), ("reserved", "u1", 8)])
assert CODED_DTYPE.itemsize == 304


def rot4(offset_hz: float):
    """(C4, S4) of a carrier offset: round(2^14 (cos, sin) 4 phi), phi = 2 pi hz / 4 MHz, nearest with ties to even"""
    ph = 2 * math.pi * float(np.float32(offset_hz)) / 4e6
    return int(round(16384.0 * math.cos(4 * ph))), int(round(16384.0 * math.sin(4 * ph)))


def pattern(access_addr: int) -> np.ndarray:
    """P: the 336 known symbols j = -80..255 (preamble + block-1 coding of the access address)"""
    coded, _ = synth.conv_encode(synth._lsb_bits(access_addr, 32))
    return np.concatenate([synth.CODED_PREAMBLE, synth.pattern_map(coded, 8)])


class Capture:
    """One capture: v[n] of the rotated low-pass symbol-spaced discriminator at any n (x outside the capture reads 0)."""

    def __init__(self, iq: np.ndarray, offset_hz: float = 0.0):
        x = np.asarray(iq, dtype=np.int8).astype(np.int64).reshape(-1, 2)
        self.n = x.shape[0]
        self.x = x
        self.c4, self.s4 = rot4(offset_hz)
        pad = np.zeros((3, 2), np.int64)
        xp = np.concatenate([pad, x, pad])                 # xp[k] = x[k - 3]
        F = (xp[:-2] + 2 * xp[1:-1] + xp[2:]) >> 2           # F[k] = F at n = k - 2, n = -2 .. n + 1
        self._F = F
        nn = np.arange(self.n)
        self.v = self.v_at(nn)
        self.h = (self.v > 0).astype(np.uint8)

    def F_at(self, n):
        n = np.asarray(n, dtype=np.int64)
        out = np.zeros(n.shape + (2,), np.int64)
        k = n + 2
        ok = (k >= 0) & (k < self._F.shape[0])
        out[ok] = self._F[k[ok]]
        # outside the range kept F reads x = 0 everywhere around it
        return out

    def v_at(self, n):
        n = np.asarray(n, dtype=np.int64)
        a, b = self.F_at(n - 2), self.F_at(n + 2)
        v = self.c4 * (a[..., 0] * b[..., 1] - b[..., 0] * a[..., 1]) - self.s4 * (a[..., 0] * b[..., 0] + a[..., 1] * b[..., 1])
        assert np.all(np.abs(v) < 2 ** 31)
        return v

    def y_at(self, n):
        return np.clip(self.v_at(n) >> 22, -127, 127)


def distances(cap: Capture, access_addr: int) -> np.ndarray:
    """D(n0) for every n0 of the capture, -1 where it is not defined"""
    return distances_bits(cap.h, access_addr)


def distances_bits(h: np.ndarray, access_addr: int) -> np.ndarray:
    """D(n0) over hard bits h[n] (0/1) of a capture of h.size samples, -1 where it is not defined.

    D(n0) = sum_j [h[n0 + 4 j] != P[j + 80]], j = -80..255.  With a = 2 h - 1 and p = 2 P - 1 (+-1), a mismatch is
    (1 - a p) / 2, so D = (336 - sum_j a[n0 + 4 j] p[j + 80]) / 2: one integer correlation per sample phase n0 % 4."""
    p = 2 * pattern(access_addr).astype(np.int64) - 1
    N = h.size
    D = np.full(N, -1, np.int64)
    lo, hi = 323, N - 1024                    # defined for lo <= n0 <= hi
    if hi < lo:
        return D
    a = 2 * np.asarray(h, dtype=np.int64) - 1
    for ph in range(4):
        n0 = np.arange(lo + (ph - lo) % 4, hi + 1, 4)
        if n0.size == 0:
            continue
        m0, m1 = (n0[0] - ph) // 4, (n0[-1] - ph) // 4   # n0 = 4 m + ph reads a[ph + 4 (m + j)], m + j = m - 80 .. m + 255
        D[n0] = (p.size - np.correlate(a[ph::4][m0 - 80:m1 + 256], p, "valid")) // 2
    return D


def hits_from_distances(D: np.ndarray) -> np.ndarray:
    """the local-minimum rule on D (-1 = not defined)"""
    N = D.size
    big = np.where(D < 0, 1 << 30, D)
    ok = (D >= 0) & (D <= MAX_DIST)
    for k in range(1, 9):
        left = np.full(N, 1 << 30, np.int64)
        left[k:] = big[:-k]
        right = np.full(N, 1 << 30, np.int64)
        right[:-k] = big[k:]
        ok &= (big < left) & (big <= right)
    return np.nonzero(ok)[0]


def _bm(state: int, b: int, L0: int, L1: int) -> int:
    s0, s1, s2 = state & 1, (state >> 1) & 1, (state >> 2) & 1
    a0, a1 = b ^ s0 ^ s1 ^ s2, b ^ s1 ^ s2
    return (2 * a0 - 1) * L0 + (2 * a1 - 1) * L1


def viterbi(Ls: np.ndarray, n_steps: int):
    """ACS over n_steps info bits from state 0; Ls int [2 n_steps].  Returns (metrics after each step [n+1][8],
    decisions [n][8]: 1 if the predecessor with bit 2 set won)."""
    m = [0] + [NEG] * 7
    hist, dec = [m], []
    for t in range(n_steps):
        L0, L1 = int(Ls[2 * t]), int(Ls[2 * t + 1])
        new, d = [0] * 8, [0] * 8
        for ns in range(8):
            b, p0 = ns & 1, ns >> 1
            p1 = p0 | 4
            c0, c1 = m[p0] + _bm(p0, b, L0, L1), m[p1] + _bm(p1, b, L0, L1)
            new[ns], d[ns] = (c1, 1) if c1 > c0 else (c0, 0)
        m = new
        hist.append(m)
        dec.append(d)
    return hist, dec


def traceback(dec, n_steps: int, state: int) -> np.ndarray:
    bits = np.zeros(n_steps, np.uint8)
    for t in range(n_steps - 1, -1, -1):
        bits[t] = state & 1
        state = (state >> 1) | (dec[t][state] << 2)
    return bits


def coded_soft(cap: Capture, n0: int, s: int, n_coded: int) -> np.ndarray:
    """L of coded bits 0 .. n_coded - 1 of block 2"""
    per = 1 if s == 2 else 4                # symbols per coded bit
    j = 296 + np.arange(n_coded * per)
    y = cap.y_at(n0 + 4 * j).reshape(n_coded, per)
    if s == 2:
        return y.reshape(-1)
    return y[:, 0] + y[:, 1] - y[:, 2] - y[:, 3]


def path_metric(cap: Capture, n0: int, s: int, body: bytes, channel: int) -> int:
    """Correlation of block 2 as sent for `body` (the L + 5 bytes of PDU and CRC, before whitening) with the soft values
    of the hit at n0: the whitened bits and TERM2, coded from state 0, as +-1 against coded_soft.  For the decoded bytes
    it is the metric of the Viterbi path they lie on, computed without the trellis."""
    bits = np.unpackbits(np.frombuffer(bytes(body), np.uint8), bitorder="little")
    bits = np.concatenate([bits ^ synth.whitening_bits(channel, bits.size), np.zeros(3, np.uint8)])
    coded, st = synth.conv_encode(bits)
    assert st == 0
    return int(((2 * coded.astype(np.int64) - 1) * coded_soft(cap, n0, s, coded.size)).sum())


def decode(cap: Capture, n0: int, dist: int, stream: int, cfg) -> np.ndarray:
    """The record of the hit at n0 (cfg: CFG_DTYPE row)"""
    aa, channel, crc_init = int(cfg["access_addr"]), int(cfg["channel"]), int(cfg["crc_init"])
    r = np.zeros(1, CODED_DTYPE)[0]
    r["sample"], r["stream"], r["access_addr"], r["channel"], r["dist"] = n0, stream, aa, channel, dist
    if int(cfg["rssi"]) & CFG_RSSI:
        r["mag_sum"] = int(np.abs(cap.x[n0:n0 + 1024]).sum())
    # CI
    st = ((aa >> 31) & 1) | (((aa >> 30) & 1) << 1) | (((aa >> 29) & 1) << 2)
    y = cap.y_at(n0 + 4 * np.arange(256, 296))
    M = []
    for c in range(4):
        coded, _ = synth.conv_encode([c & 1, c >> 1, 0, 0, 0], st)
        sym = synth.pattern_map(coded, 8).astype(np.int64)
        M.append(int(((2 * sym - 1) * y).sum()))
    ci = int(np.argmax(M))                  # first maximum: the lower c on a tie
    r["ci"] = ci
    if ci >= 2:
        r["flags"] = CI_RESERVED | (TRUNCATED if n0 + 4 * 295 + 3 >= cap.n else 0)
        r["crc_bad"] = 1
        return r
    s = 8 if ci == 0 else 2
    r["s"] = s
    Lh = coded_soft(cap, n0, s, 80)
    hist40, dec40 = viterbi(Lh, 40)
    best = int(np.argmax(hist40[-1]))      # lowest index on a tie
    hb = traceback(dec40, 40, best)[:16] ^ synth.whitening_bits(channel, 16)
    L = int(np.packbits(hb[8:16], bitorder="little")[0])
    n_steps = 16 + 8 * L + 27
    Ls = coded_soft(cap, n0, s, 2 * n_steps)
    hist, dec = viterbi(Ls, n_steps)
    bits = traceback(dec, n_steps, 0)[:n_steps - 3] ^ synth.whitening_bits(channel, n_steps - 3)
    body = np.packbits(bits, bitorder="little")
    nb = L + 5
    r["n_bytes"] = nb
    r["bytes"][:nb] = body
    crc_rx = int(body[L + 2]) | int(body[L + 3]) << 8 | int(body[L + 4]) << 16
    r["crc_bad"] = int(synth.crc24(body[:L + 2].tobytes(), crc_init) != crc_rx)
    r["metric"] = hist[-1][0]
    j_last = 296 + s * n_steps - 1         # block 2 is n_steps * S symbols
    r["flags"] = TRUNCATED if n0 + 4 * j_last + 3 >= cap.n else 0
    return r


def rx_coded(iq: np.ndarray, cfgs: np.ndarray, offset_hz=None) -> np.ndarray:
    """Records of every capture (iq [n_streams, n_int8] or [n_int8]), sorted by (stream, sample)."""
    iq = np.asarray(iq, dtype=np.int8)
    if iq.ndim == 1:
        iq = iq[None, :]
    cfgs = np.atleast_1d(cfgs)
    off = np.zeros(iq.shape[0], np.float32) if offset_hz is None else np.broadcast_to(np.asarray(offset_hz, np.float32), (iq.shape[0],))
    out = []
    for s in range(iq.shape[0]):
        cap = Capture(iq[s], float(off[s]))
        D = distances(cap, int(cfgs[s]["access_addr"]))
        for n0 in hits_from_distances(D):
            out.append(decode(cap, int(n0), int(D[n0]), s, cfgs[s]))
    return np.array(out, dtype=CODED_DTYPE) if out else np.zeros(0, CODED_DTYPE)


def place(n_samples: int, bursts, amplitude: int = 100, noise_sigma: float = 0.0, rng=None, offset_hz: float = 0.0) -> np.ndarray:
    """int8 capture of n_samples samples holding coded bursts [(n0, iq)] (iq from synth.coded_air; the burst's access
    address lands at sample n0), scaled to `amplitude`, turned by a carrier offset, with Gaussian noise of noise_sigma
    per rail (rounded, saturated)."""
    x = np.zeros((n_samples, 2), np.float64)
    for n0, wav in bursts:
        w = wav.astype(np.float64).reshape(-1, 2) * amplitude / 127.0
        start = n0 - synth.CODED_AA_SAMPLE
        lo, hi = max(start, 0), min(start + w.shape[0], n_samples)
        if hi > lo:
            x[lo:hi] += w[lo - start:hi - start]
    if offset_hz:
        ph = 2 * np.pi * offset_hz / 4e6 * np.arange(n_samples)
        z = (x[:, 0] + 1j * x[:, 1]) * np.exp(1j * ph)
        x = np.stack([z.real, z.imag], axis=1)
    if noise_sigma:
        x = x + rng.normal(0.0, noise_sigma, x.shape)
    return np.clip(np.round(x), -128, 127).astype(np.int8).reshape(-1)


def sigma_of(snr_db: float, amplitude: int) -> float:
    """noise per rail of rx_ber_run: amplitude / 10^(snr/20) / sqrt 2"""
    return amplitude / 10 ** (snr_db / 20) / math.sqrt(2)
