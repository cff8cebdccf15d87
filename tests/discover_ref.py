"""Numpy restatement of the connection-discovery candidate rule (include/btle_b200.h, btle_conn_cand) — test
infrastructure: what btle_b200_discover must return, written straight from the definition, sample by sample."""
from __future__ import annotations

import numpy as np

from btle_b200 import CAND_DTYPE, REC_DTYPE, synth
from btle_b200.synth import crc_init_reorder

WHITEN = synth.whitening_table()


def dbits(iq: np.ndarray) -> np.ndarray:
    """d[n] = (I[n] Q[n+1] - I[n+1] Q[n]) > 0 for n + 1 < n_samples."""
    iq = np.asarray(iq, dtype=np.int8)
    n = iq.size // 2
    i = iq[0:2 * n:2].astype(np.int32)
    q = iq[1:2 * n:2].astype(np.int32)
    return (i[:-1] * q[1:] - i[1:] * q[:-1]) > 0


def whiten_bits(channel: int, first: int, count: int) -> np.ndarray:
    """Whitening bits first .. first+count-1 of `channel` (bit k of the sequence = bit k%8 of byte k//8)."""
    k = np.arange(first, first + count)
    return ((WHITEN[channel][k // 8] >> (k % 8)) & 1).astype(bool)


def crc_unwind(crc: int, bits: int, nbits: int) -> int:
    """The CRC-24 register from which `nbits` message bits (LSB first) lead to `crc` (the LFSR run backwards)."""
    for j in range(nbits - 1, -1, -1):
        f = (crc >> 23) & 1
        crc = (((crc ^ (0xDA6000 if f else 0)) << 1) | (f ^ ((bits >> j) & 1))) & 0xFFFFFF
    return crc


def crc_init_for(header: bytes, crc_rx: int) -> int:
    """The -k value for which synth.crc24(header, value) == crc_rx."""
    bits = int.from_bytes(bytes(header), "little")
    return crc_init_reorder(crc_unwind(crc_rx, bits, 8 * len(header)))


def _pack(bits: np.ndarray) -> np.ndarray:
    """rows of bits (LSB first) -> integers"""
    return (bits.astype(np.uint64) << np.arange(bits.shape[1], dtype=np.uint64)).sum(axis=1)


def discover(iq: np.ndarray, channel: int, stream: int = 0) -> np.ndarray:
    """Candidates of one capture in sample order (CAND_DTYPE)."""
    d = dbits(iq)
    n_samples = np.asarray(iq).size // 2
    lo, hi = 32, n_samples - 286                       # n0 - 32 >= 0, n0 + 285 < n_samples
    if hi < lo:
        return np.zeros(0, dtype=CAND_DTYPE)
    n0 = np.arange(lo, hi + 1)
    sym = lambda k: d[n0 + 4 * k]                      # bit k of the window (k < 0: preamble)
    ok = np.ones(n0.size, dtype=bool)
    for j in range(8):                                 # preamble d[n0-32+4j], j = 0..7, then d[n0]: alternating
        ok &= sym(j - 8) != sym(j - 7)
    wh = whiten_bits(channel, 0, 16)
    ok &= (sym(32) ^ wh[0]) & ~(sym(33) ^ wh[1])      # LLID = 1
    for j in range(8, 16):                             # byte 1 = 0
        ok &= ~(sym(32 + j) ^ wh[j])
    n0 = n0[ok]
    out = np.zeros(n0.size, dtype=CAND_DTYPE)
    if not n0.size:
        return out
    take = lambda first, count: np.stack([d[n0 + 4 * (first + k)] for k in range(count)], axis=1)
    aa = _pack(take(0, 32))
    hdr = _pack(take(32, 16) ^ whiten_bits(channel, 0, 16))
    crc = _pack(take(48, 24) ^ whiten_bits(channel, 16, 24))
    out["sample"], out["stream"], out["access_addr"], out["channel"] = n0, stream, aa, channel
    out["header"][:, 0], out["header"][:, 1] = hdr & 0xFF, hdr >> 8
    out["crc_init"] = [crc_init_for(int(h).to_bytes(2, "little"), int(c)) for h, c in zip(hdr, crc)]
    return out


def discover_batch(iq2d: np.ndarray, channels) -> np.ndarray:
    """BtleRx.discover() restated: captures [n_streams, n_int8], sorted by (stream, sample)."""
    iq2d = np.asarray(iq2d, dtype=np.int8)
    if iq2d.ndim == 1:
        iq2d = iq2d[None, :]
    channels = np.broadcast_to(np.asarray(channels), (iq2d.shape[0],))
    parts = [discover(iq2d[s], int(channels[s]), s) for s in range(iq2d.shape[0])]
    return np.concatenate(parts) if parts else np.zeros(0, dtype=CAND_DTYPE)


class OracleDiscoverRx:
    """rx_batch() with the oracle and discover() with the restatement — lets the discovery logic run without a GPU."""

    def rx_batch(self, iq, cfgs):
        import orc
        out = [orc.rx_stream(iq[s], channel=int(c["channel"]), access_addr=int(c["access_addr"]),
                             access_mask=int(c["access_mask"]), crc_init=int(c["crc_init"]), stream=s)
               for s, c in enumerate(cfgs)]
        return np.concatenate(out) if out else np.zeros(0, dtype=REC_DTYPE)

    def discover(self, iq, channels):
        return discover_batch(iq, channels)
