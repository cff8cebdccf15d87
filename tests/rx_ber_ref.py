"""numpy restatement of the 4-Msps error-rate flow (btle_b200_rx_ber_*; definition in include/btle_b200.h): the packet
source from the kernels' counter-based draws, the channel in float64, the capture of slots, and the scoring of receive
records against the truth.  Used by tests/test_rx_ber.py (with the C oracle as the receiver) and the GPU tests."""
from __future__ import annotations

import numpy as np

from btle_b200 import synth
from btle_b200._native import RX_BER_COUNTERS, RX_BER_TRUTH_DTYPE

M64 = np.uint64(0xFFFFFFFFFFFFFFFF)
CHUNK = 8192
AA_OFFSET, MATCH = 39, 3                 # BTLE_RX_BER_AA_OFFSET, BTLE_RX_BER_MATCH


def mix64(x):
    x = (x + np.uint64(0x9E3779B97F4A7C15)) & M64
    x = ((x ^ (x >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)) & M64
    x = ((x ^ (x >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)) & M64
    return x ^ (x >> np.uint64(31))


def draw(seed, stream, a, k):
    """the kernels' counter-based generator: splitmix64 finaliser of (seed, stream, position, kind), uint64"""
    with np.errstate(over="ignore"):
        stream, a = np.asarray(stream, dtype=np.uint64), np.asarray(a, dtype=np.uint64)
        s = mix64(np.uint64(seed) ^ (stream * np.uint64(0xD1B54A32D192ED03)))
        return mix64(s ^ (a * np.uint64(0x9E3779B97F4A7C15)) ^ (np.uint64(k) << np.uint64(56)))


def pdu_bytes(channel):
    return 39 if channel >= 37 else 29


def packet_len(channel):
    """L: samples of one packet out of the btle_tx PHY (32 per air byte + 16)"""
    return 32 * (1 + 4 + pdu_bytes(channel) + 3) + 16


def capture_int8(n_packets, slot):
    return -(-n_packets * slot // CHUNK) * 2 * CHUNK


def pdu(seed, k, channel):
    nb = pdu_bytes(channel)
    b = np.arange(nb)
    r = draw(seed, k, b >> 3, 9)
    out = ((r >> (np.uint64(8) * (b & 7).astype(np.uint64))) & np.uint64(0xFF)).astype(np.uint8)
    out[:2] = (0x42, 0x25) if channel >= 37 else (0x02, nb - 2)
    return out


def placement(seed, k, slot, channel):
    """(offset of the packet in its slot, 4 delta)"""
    r = int(draw(seed, k, 0, 12))
    return r % (slot - packet_len(channel) + 1), (r >> 32) & 3


def sigma(amplitude, snr_db):
    """the kernel's float32 sigma (exp10f as a float64 power rounded to float32)"""
    with np.errstate(over="ignore"):                    # exp10f overflows to inf for a huge SNR: no noise at all
        return float(np.float32(amplitude) / np.float32(10.0 ** float(np.float32(snr_db) / np.float32(20))) * np.float32(0.70710678))


def gauss(seed, k, idx):
    """Box-Muller on the kernel's float32 uniforms, in float64: (g_i, g_q)"""
    r = draw(seed, k, idx, 11)
    f = np.float32(2.3283064365386963e-10)
    u1 = ((r & np.uint64(0xFFFFFFFF)).astype(np.float32) + np.float32(0.5)) * f
    u2 = (r >> np.uint64(32)).astype(np.float32) * f
    rad = np.sqrt(-2.0 * np.log(u1.astype(np.float64)))
    ang = 2 * np.pi * u2.astype(np.float64)
    return rad * np.cos(ang), rad * np.sin(ang)


def packet_wave(cfg, k, corrupt_bit=None):
    """the scaled transmit waveform of packet k (float32 values as float64, [L] I and Q) and its PDU"""
    ch = int(cfg["channel"])
    p = pdu(int(cfg["seed"]), k, ch)
    air = synth.air_bytes(bytes(p), ch, int(cfg["access_addr"]), int(cfg["crc_init"]), corrupt_bit=corrupt_bit)
    w = synth.modulate(air).reshape(-1, 2).astype(np.float32)
    scale = np.float32(int(cfg["amplitude"])) / np.float32(127)
    w = (w * scale).astype(np.float64)
    return w[:, 0], w[:, 1], p


def channel(cfg, wi, wq, delta):
    """steps 1 and 2 in float64: np.interp at (m - delta)(1 + e), then the rotation"""
    L = wi.size
    m = np.arange(L, dtype=np.float64)
    e = float(np.float32(cfg["ppm"])) * 1e-6
    x = (m - delta) * (1.0 + e)
    vi, vq = np.interp(x, m, wi), np.interp(x, m, wq)
    rate = e * 2450e6 * (0.25e-6 * (1.0 + e)) + float(np.float32(cfg["cfo_hz"])) / 4e6
    if rate != 0:
        turns = rate * m
        ang = 2 * np.pi * (turns - np.floor(turns))
        vi, vq = vi * np.cos(ang) - vq * np.sin(ang), vi * np.sin(ang) + vq * np.cos(ang)
    return vi, vq


def capture(cfg, first, n, n_live=None, corrupt=None):
    """(int8 capture, truth rows, real values before rounding [n_samples, 2]) of packets first .. first+n-1, as
    btle_b200_rx_ber_synth_device writes them.  corrupt = {k: bit}: packet k is sent with that bit of PDU + CRC flipped
    (the truth keeps the PDU as drawn)."""
    seed, S, ch = int(cfg["seed"]), int(cfg["slot_samples"]), int(cfg["channel"])
    n_live = first + n if n_live is None else n_live
    ns = capture_int8(n, S) // 2
    real = np.zeros((ns, 2))
    truth = np.zeros(n, dtype=RX_BER_TRUTH_DTYPE)
    sg = sigma(int(cfg["amplitude"]), float(cfg["snr_db"]))
    e = float(np.float32(cfg["ppm"])) * 1e-6
    for s in range(-(-ns // S)):
        k = first + s
        lo, hi = s * S, min(ns, (s + 1) * S)
        gi, gq = gauss(seed, k, np.arange(hi - lo))
        real[lo:hi, 0], real[lo:hi, 1] = sg * gi, sg * gq
        if k < n_live:
            off, d4 = placement(seed, k, S, ch)
            wi, wq, p = packet_wave(cfg, k, (corrupt or {}).get(k))
            vi, vq = channel(cfg, wi, wq, 0.25 * d4)
            a, b = lo + off, min(hi, lo + off + wi.size)
            real[a:b, 0] += vi[:b - a]
            real[a:b, 1] += vq[:b - a]
            if s < n:
                t = truth[s]
                t["aa_sample"] = lo + off + int(np.floor(AA_OFFSET / (1.0 + e) + 0.25 * d4 + 0.5))
                t["offset"], t["n_bytes"], t["delta4"] = off, p.size, d4
                t["pdu"][:p.size] = p
                r = np.rint(real[lo:hi])
                t["clipped"] = int(((r < -128) | (r > 127)).any(axis=1).sum())
    iq = np.clip(np.rint(real), -128, 127).astype(np.int8).reshape(-1)
    return iq, truth, real


def score_fields(chunk, n0, n_bytes, crc_bad, rejected, rec_bytes, truth) -> dict:
    """the counters of btle_rx_ber_result from records in reference order (vectorised: packet k's record is the record of
    lowest order among those within +-MATCH samples of its access address)"""
    pos = np.asarray(chunk, dtype=np.int64) * CHUNK + np.asarray(n0, dtype=np.int64)
    n_bytes, crc_bad, rejected = np.asarray(n_bytes, dtype=np.int64), np.asarray(crc_bad, dtype=bool), np.asarray(rejected, dtype=bool)
    rec_bytes = np.asarray(rec_bytes, dtype=np.uint8).reshape(pos.size, -1)[:, :39] if pos.size else np.zeros((0, 39), np.uint8)
    a = truth["aa_sample"].astype(np.int64)
    nb = truth["n_bytes"].astype(np.int64)
    order = np.argsort(pos, kind="stable")
    sp = pos[order]
    lo, hi = np.searchsorted(sp, a - MATCH, "left"), np.searchsorted(sp, a + MATCH, "right")
    none = np.iinfo(np.int64).max
    best = np.full(a.size, none, dtype=np.int64)
    for j in range(int((hi - lo).max(initial=0))):
        idx = lo + j
        cand = order[np.minimum(idx, max(pos.size - 1, 0))] if pos.size else np.zeros(a.size, dtype=np.int64)
        take = (idx < hi) & (cand < best)
        best = np.where(take, cand, best)
    m = best != none
    b = np.where(m, best, 0)
    rej = m & rejected[b] if pos.size else m
    ok = m & ~rej & ~crc_bad[b] if pos.size else m
    got = rec_bytes[b] if pos.size else np.zeros((a.size, 39), dtype=np.uint8)
    ref = truth["pdu"][:, :39]
    byte_ix = np.arange(39)[None, :]
    wrong = ok & (((n_bytes[b] - 3) != nb if pos.size else False) | ((got != ref) & (byte_ix < nb[:, None])).any(axis=1))
    common = np.clip(np.where(rej, 2, (n_bytes[b] if pos.size else 0) - 3), 0, nb)
    diff = np.unpackbits(got ^ ref, axis=1).reshape(a.size, 39, 8).sum(axis=2)
    bits = np.where(byte_ix < common[:, None], diff, 0).sum(axis=1)
    bad = ~ok
    c = dict.fromkeys(RX_BER_COUNTERS, 0)
    c["packets"], c["bit_total"], c["clipped"] = int(a.size), int(8 * nb.sum()), int(truth["clipped"].sum())
    c["pkt_err"], c["aa_miss"], c["len_reject"], c["crc_ok_wrong"] = int(bad.sum()), int((~m).sum()), int(rej.sum()), int(wrong.sum())
    c["bit_err"] = int(np.where(~m, 8 * nb, np.where(bad, bits, 0)).sum())
    c["extra_recs"] = int(pos.size - m.sum())
    c["extra_crc_ok"] = int((~rejected & ~crc_bad).sum() - ok.sum())
    return c


def score(recs, truth) -> dict:
    """REC_DTYPE records (GPU or oracle, reference order)"""
    return score_fields(recs["chunk"], recs["n0"], recs["n_bytes"], recs["crc_bad"], (recs["flags"] & 4) != 0, recs["bytes"], truth)


def score_ref(ref, truth) -> dict:
    """the reference receiver's records (orc.REF_DTYPE): a rejected hit is a header-only record"""
    return score_fields(ref["chunk"], ref["n0"], ref["nbytes"], ref["crc_bad"] != 0, ref["nbytes"] == 2, ref["bytes"], truth)


def add(a: dict, b: dict) -> dict:
    return {k: a[k] + b[k] for k in RX_BER_COUNTERS}
