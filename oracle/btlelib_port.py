"""CPU restatement of the reference's bit-true Python receiver and of its streaming form.  TEST INFRASTRUCTURE ONLY:
only tests/ may import this; nothing under btle_b200/ does.

* rx_window(): btlelib.btle_rx on one window (the reference's python/btlelib.py:414-541: symbol-spaced differential demod on each
  of the 8 sample phases :395-400,:461-467; first exact access-address match :402-412; dewhitening from bit 40 on :265-268;
  payload length from 6 / 5 bits :477-483; CRC position clamp :488-490; crc24_core :191-219; first CRC-ok phase wins
  :517), vectorised with numpy instead of the reference's per-bit Python loops.  Pinned to the reference's btlelib on
  random packets at all SNRs with arbitrary alignment (tests/test_oracle_btlelib_port.py against the reference's recorded
  verdicts, tests/golden/btlelib_rx_random.npz) and to the committed golden vectors (tests/golden/btlelib_rx.npz).
* rx_stream(): the streaming rules of include/btle_b200.h (btle_b200_rx_sps8): access-address hits on the 8 absolute sample
  phases -> clusters -> aligned windows -> rx_window() -> greedy skip."""
from __future__ import annotations

import numpy as np

WINDOW = 3072                 # BTLE_SPS8_WINDOW
MARGIN_SYMBOLS = 2            # BTLE_SPS8_MARGIN_SYMBOLS
MIN_PACKET_SYMBOLS = 72       # BTLE_SPS8_MIN_PACKET_SYMBOLS
SPS = 8


def bits_lsb_first(value: int, nbytes: int) -> np.ndarray:
    """hex_string_to_bit of the value's bytes in transmission order: every byte LSB first (btlelib.py:270-293)."""
    return np.array([(value >> (8 * b + k)) & 1 for b in range(nbytes) for k in range(8)], dtype=np.int8)


def whitening(channel: int, n: int) -> np.ndarray:
    """scramble_core's sequence (btlelib.py:226-263)."""
    reg = [1] + [(channel >> (5 - i)) & 1 for i in range(6)]
    out = np.zeros(n, dtype=np.int8)
    for t in range(n):
        o = reg[6]
        out[t] = o
        reg = [o, reg[0], reg[1], reg[2], reg[3] ^ o, reg[4], reg[5]]
    return out


def crc24_core(bits: np.ndarray, init_bits: np.ndarray) -> np.ndarray:
    """btlelib.py:191-219: 24-stage LFSR, feedback = stage 23 ^ input, taps into stages 0,1,3,4,6,9,10; result = stages 23..0."""
    st = 0
    for k in range(24):
        st |= (int(init_bits[k]) & 1) << k
    for b in bits:
        fb = ((st >> 23) ^ int(b)) & 1
        st = (st << 1) & 0xFFFFFF
        if fb:
            st ^= 0x00065B
    return np.array([(st >> (23 - k)) & 1 for k in range(24)], dtype=np.int8)


def crc_init_bits(crc_init: int) -> np.ndarray:
    """crc_state_init_bit for a CRC init given as btle_rx's -k value (0x555555, 0xA77B22 = bytes A7 7B 22 on air, LSB first each)."""
    return bits_lsb_first(int.from_bytes(crc_init.to_bytes(3, "big"), "little"), 3)


def demod_phase(i: np.ndarray, q: np.ndarray) -> np.ndarray:
    a, b = i.astype(np.int32), q.astype(np.int32)
    with np.errstate(over="ignore"):
        s = a[:-1] * b[1:] - a[1:] * b[:-1]
    return (s > 0).astype(np.int8)


def rx_window(i, q, channel=37, crc_init=0x555555, access_addr=0x8E89BED6, sps=SPS):
    """-> dict(pdu_bit, crc_ok, plen, phase, start, found) with btle_rx's meaning at `sps` samples per symbol (the
    reference's SAMPLE_PER_SYMBOL); `found` = 1 + last phase the access address was found on (0: never); `start` = its
    symbol index on the reported phase.  Where the access address ends so close to the window's end that the length field
    is not complete (start + 40 + 6 / 5 > num_bit), the reference raises IndexError; here, as in model_rx_batch_kernel,
    the missing header bits read as 0 before dewhitening."""
    i = np.asarray(i).astype(np.int16)
    q = np.asarray(q).astype(np.int16)
    n = len(i)
    num_bit = round(n / sps) - 1
    aa = bits_lsb_first(access_addr, 4)
    init = crc_init_bits(crc_init)
    adv = channel in (37, 38, 39)
    res = dict(pdu_bit=np.zeros(0, dtype=np.int8), crc_ok=False, plen=0, phase=sps - 1, start=-1, found=0)
    wh_cache = None
    for ph in range(sps):
        b = demod_phase(i[ph::sps], q[ph::sps])
        bits = np.zeros(num_bit, dtype=np.int8)
        m = min(len(b), num_bit)
        bits[:m] = b[:m]
        if m < num_bit:
            bits[-1] = b[-1]
        if num_bit < 32:
            continue
        win = np.lib.stride_tricks.sliding_window_view(bits, 32)
        hit = np.nonzero((win == aa).all(axis=1))[0]
        if len(hit) == 0:
            continue
        start = int(hit[0])
        phy = np.concatenate((np.zeros(8, dtype=np.int8), bits[start:]))
        if wh_cache is None or len(wh_cache) < len(phy) + 16:
            wh_cache = whitening(channel, max(len(phy) + 16, 400))
        info = phy.copy()
        info[40:] ^= wh_cache[: len(phy) - 40]
        nb = 6 if adv else 5
        hdr = np.concatenate((phy, np.zeros(16, dtype=np.int8)))[40:56] ^ wh_cache[:16]
        plen = int(sum(int(hdr[8 + k]) << k for k in range(nb)))
        crc_start = 56 + 8 * plen
        if crc_start + 24 > len(info):
            crc_start = len(info) - 24
        pdu = info[40:crc_start] if crc_start > 40 else np.zeros(0, dtype=np.int8)
        rx_crc = info[crc_start:crc_start + 24]
        ok = bool(len(rx_crc) == 24 and np.array_equal(crc24_core(pdu, init), rx_crc))
        res.update(pdu_bit=pdu, crc_ok=ok, plen=plen, start=start, found=ph + 1)
        if ok:
            res["phase"] = ph
            break
    return res


def find_hits(iq16: np.ndarray, access_addr: int) -> np.ndarray:
    """All sample indices n where the 32 symbol-spaced differential bits starting at n (phase n mod 8) equal the access address."""
    iq = np.asarray(iq16, dtype=np.int16).reshape(-1, 2)
    n = len(iq)
    aa = bits_lsb_first(access_addr, 4)
    hits = []
    for ph in range(SPS):
        b = demod_phase(iq[ph::SPS, 0], iq[ph::SPS, 1])
        if len(b) < 32:
            continue
        win = np.lib.stride_tricks.sliding_window_view(b, 32)
        s = np.nonzero((win == aa).all(axis=1))[0]
        pos = 8 * s + ph
        hits.append(pos[pos + 8 * 32 < n])
    return np.sort(np.concatenate(hits)) if hits else np.zeros(0, dtype=np.int64)


def rx_stream(iq16: np.ndarray, channel=37, crc_init=0x555555, access_addr=0x8E89BED6):
    """-> list of dicts(sample, window, + rx_window's fields), the packets btle_b200_rx_sps8 must report."""
    iq = np.asarray(iq16, dtype=np.int16).reshape(-1, 2)
    n = len(iq)
    out = []
    if n < WINDOW:
        return out
    last, cursor = -(1 << 60), -1
    for h in find_hits(iq, access_addr):
        h = int(h)
        if h < last + 8 * MIN_PACKET_SYMBOLS:
            continue
        last = h
        w0 = max(0, 8 * (h // 8 - MARGIN_SYMBOLS))
        if w0 + WINDOW > n:
            continue
        if h < cursor:
            continue
        r = rx_window(iq[w0:w0 + WINDOW, 0], iq[w0:w0 + WINDOW, 1], channel, crc_init, access_addr)
        at = h
        if r["found"]:
            at = w0 + 8 * r["start"] + (r["phase"] if r["crc_ok"] else r["found"] - 1)
        cursor = at + 8 * (32 + 16 + 8 * (r["plen"] if r["found"] else 0) + 24)
        out.append(dict(r, sample=at, window=w0))
    return out


def phase_bits_to_iq(bits: np.ndarray, n: int | None = None, amp: int = 1000, sps: int = SPS) -> np.ndarray:
    """int16 [n, 2] (I, Q) whose symbol-spaced differential bits on phase p are exactly bits[p] (bits [sps, m]): sample
    a + sps is sample a turned by +90 degrees for a 1 and by -90 degrees for a 0, every sample one of (amp, 0), (0, amp),
    (-amp, 0), (0, -amp), so bit k of phase p (samples p + sps k and p + sps (k + 1)) decides on +-amp^2.  n defaults to
    sps (m + 1); samples beyond sps (m + 1) are not allowed."""
    bits = np.asarray(bits, dtype=np.int64)
    m = bits.shape[1]
    n = sps * (m + 1) if n is None else n
    assert bits.shape[0] == sps and n <= sps * (m + 1)
    turn = np.where(bits > 0, 1, -1)
    quadrant = np.concatenate((np.arange(sps)[:, None] % 4, np.cumsum(turn, axis=1) + np.arange(sps)[:, None] % 4), axis=1) % 4
    pts = np.array([[amp, 0], [0, amp], [-amp, 0], [0, -amp]], dtype=np.int64)
    iq = pts[quadrant.T.reshape(-1)][:n]                       # sample p + sps k = quadrant[p, k]
    return iq.astype(np.int16)


def tx_bits(pdu: bytes, channel=37, crc_init=0x555555, access_addr=0x8E89BED6) -> np.ndarray:
    """preamble + access address + whitened(PDU + CRC) as PHY bits (btlelib.btle_tx's bit path, btlelib.py:344-393)."""
    pdu_bits = np.array([(v >> k) & 1 for v in pdu for k in range(8)], dtype=np.int8)
    crc = crc24_core(pdu_bits, crc_init_bits(crc_init))
    body = np.concatenate((pdu_bits, crc)) ^ whitening(channel, len(pdu_bits) + 24)
    pre = bits_lsb_first(0x55 if access_addr & 1 else 0xAA, 1)
    return np.concatenate((pre, bits_lsb_first(access_addr, 4), body)).astype(np.int8)
