#!/usr/bin/env python
"""Golden vectors for the btlelib-compatible shim, produced by importing the REFERENCE's own
python/btlelib.py here (from a writable copy: it writes table files next to itself on first TX
call, btlelib.py:90-91,155).  Writes tests/golden/btlelib_rx.npz (committed); with --random, instead
tests/golden/btlelib_rx_random.npz: the reference receiver's verdicts on the 60 random-packet windows of
tests/test_oracle_btlelib_port.py, whose inputs the test rebuilds itself (checked here against btle_tx / add_noise); with
--sps, tests/golden/btlelib_rx_sps.npz: the reference receiver at SAMPLE_PER_SYMBOL 1, 2, 4, 8 and 16 on crafted windows
(sps_windows), inputs stored with the verdicts."""
import os
import shutil
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = os.environ.get("BTLE_REFERENCE", "/root/reference")


def random_cases(bl):
    sys.path.insert(0, ROOT)
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    from test_oracle_btlelib_port import random_windows
    n = 60
    cols = {c: [] for c in ("ch", "n", "crc_ok", "plen", "phase", "pdu_len")}
    pdu_bits = []
    for w in random_windows(n):
        k, ch, crc_hex, aa_hex, snr, ri, rq = w["k"], w["ch"], w["crc_hex"], w["aa_hex"], w["snr"], w["i"], w["q"]
        args = [ch] + ([bl.hex_string_to_bit(crc_hex), aa_hex] if crc_hex else [])
        ti, tq, _, _ = bl.btle_tx(bl.hex_string_to_bit(w["pdu"].hex()), *args)
        np.random.seed(100 + k)
        ni, nq = bl.add_noise(ti, tq, snr)
        # the window the test rebuilds is the reference's: same waveform, same noise (the padding is drawn after it, by the
        # same code, from the same generator state)
        assert np.array_equal(np.double(ti), w["tx"][0]) and np.array_equal(np.double(tq), w["tx"][1]), k
        assert np.array_equal(ni, w["noisy"][0]) and np.array_equal(nq, w["noisy"][1]), k
        r = bl.btle_rx(ri, rq, *args)
        pdu = np.asarray(r[0], dtype=np.uint8)
        for c, v in zip(cols, (ch, len(ri), int(bool(r[1])), int(r[2]), int(r[6]), len(pdu))):
            cols[c].append(v)
        pdu_bits.append(pdu)
        print(k, "ch", ch, "snr", snr, "crc_ok", r[1], "plen", r[2], "phase", r[6])
    out = {c: np.array(v, dtype=np.int32) for c, v in cols.items()}
    out["pdu_bits"] = np.packbits(np.concatenate(pdu_bits))                  # per window pdu_len bits, back to back
    np.savez_compressed(os.path.join(ROOT, "tests", "golden", "btlelib_rx_random.npz"), **out)


SPS_SET = (1, 2, 4, 8, 16)
ADV = (37, 0x555555, 0x8E89BED6)
DATA = (11, 0xA77B22, 0x60850A1B)        # btle_rx -k / -a style values


def sps_windows():
    """Crafted windows for the model receiver at every sample rate: per-phase bit sequences (btlelib_port.phase_bits_to_iq)
    with packets planted at exact symbol indices.  Yields (name, sps, (channel, crc_init, access_addr), i, q)."""
    sys.path.insert(0, os.path.join(ROOT, "oracle"))
    import btlelib_port as P
    rng = np.random.default_rng(1234)

    def pdu_for(cfg, plen, rfu=0):
        if cfg[0] >= 37:
            return bytes([0x40, plen]) + rng.integers(0, 256, plen, dtype=np.uint8).tobytes()
        return bytes([0x01, plen | rfu]) + rng.integers(0, 256, plen, dtype=np.uint8).tobytes()

    def window(sps, nsym, cfg, plants, amp=1000):
        """plants: {phase: (symbol index of the access address, air bits from the access address on)}; other bits random"""
        bits = rng.integers(0, 2, (sps, nsym - 1)).astype(np.int8)
        for ph, (s, b) in plants.items():
            b = b[: nsym - 1 - s]
            bits[ph, s:s + len(b)] = b
        iq = P.phase_bits_to_iq(bits, amp=amp, sps=sps)
        return iq[:, 0].copy(), iq[:, 1].copy()

    def air(cfg, pdu, flip_crc=False):
        b = P.tx_bits(pdu, *cfg)[8:].copy()              # from the access address on
        if flip_crc:
            b[-3] ^= 1
        return b

    for sps in SPS_SET:
        nsym = 400 if sps >= 8 else 2048
        for cfg in (ADV, DATA):
            tag = "adv" if cfg is ADV else "data"
            # 37 = 0b100101 and a set RFU bit above the 5-bit data length: a length read with the other channel's mask differs
            pdu = pdu_for(cfg, 37 if cfg is ADV else 27, rfu=0x20)
            good, bad = air(cfg, pdu), air(cfg, pdu, flip_crc=True)
            yield f"{tag}_clean", sps, cfg, *window(sps, nsym, cfg, {p: (20, good) for p in range(sps)})
            if sps > 1:
                later = {p: (20, bad) for p in range(sps // 2)}
                later.update({p: (20, good) for p in range(sps // 2, sps)})
                yield f"{tag}_ok_on_later_phase", sps, cfg, *window(sps, nsym, cfg, later)
            yield f"{tag}_never_ok", sps, cfg, *window(sps, nsym, cfg, {p: (30, bad) for p in range(max(1, sps - 1))})
            num_bit = nsym - 1
            long_pdu = pdu_for(cfg, 31 if cfg is DATA else 37)
            # CRC position clamped, crc_start >= 40: the header's length runs past the window
            yield f"{tag}_clamp_ge40", sps, cfg, *window(sps, nsym, cfg, {0: (num_bit + 8 - 150, air(cfg, long_pdu))})
            # crc_start < 40: the access address ends 13..23 bits before the window's end (len(info) 53/54 .. 63)
            for li in ((54, 63) if cfg is ADV else (53, 60)):
                yield f"{tag}_clamp_lt40_{li}", sps, cfg, *window(sps, nsym, cfg, {sps - 1: (num_bit + 8 - li, air(cfg, long_pdu))})
            # the access address at the last index: the reference raises (no complete header)
            yield f"{tag}_aa_last", sps, cfg, *window(sps, nsym, cfg, {0: (num_bit - 32, air(cfg, pdu))})
        yield "never_found", sps, ADV, *window(sps, nsym, ADV, {})
        yield "n34_noise", sps, ADV, *window(sps, 34, ADV, {})
        for s in (0, 1):
            yield f"n34_aa_at_{s}", sps, ADV, *window(sps, 34, ADV, {0: (s, air(ADV, pdu_for(ADV, 6)))})
        if sps <= 4:
            # the CRC's last bit is the window's last bit: the clamp's boundary (crc_start + 24 == len(info)) on its other side
            yield "n2048_data_at_end", sps, DATA, *window(sps, 2048, DATA, {p: (2047 - (32 + 16 + 8 * 27 + 24), air(DATA, pdu_for(DATA, 27)))
                                                                           for p in range(sps)})
        # int16 extremes: a clean packet at full scale (-32767 -> -32768), and full-scale random samples
        i, q = window(sps, 300, ADV, {p: (10, air(ADV, pdu_for(ADV, 20))) for p in range(sps)}, amp=32767)
        i[i == -32767] = -32768
        q[q == -32767] = -32768
        yield "extreme_packet", sps, ADV, i, q
        r = rng.choice(np.array([-32768, 32767], dtype=np.int16), (2, 300 * sps))
        yield "extreme_random", sps, ADV, r[0].copy(), r[1].copy()


def sps_cases(bl):
    """tests/golden/btlelib_rx_sps.npz: the reference's btle_rx with SAMPLE_PER_SYMBOL 1, 2, 4, 8, 16 on sps_windows()."""
    out, names = {}, []
    for k, (name, sps, (ch, crc, aa), i, q) in enumerate(sps_windows()):
        bl.SAMPLE_PER_SYMBOL = sps
        args = [ch, bl.hex_string_to_bit(f"{crc:06X}"), aa.to_bytes(4, "little").hex().upper()]
        raises = 0
        try:
            pdu_bit, crc_ok, plen, phy_bit, bit_all, _, phase = bl.btle_rx(i, q, *args)
        except IndexError:
            raises = 1
        names.append(name)
        out[f"w{k}_i"], out[f"w{k}_q"] = np.int16(i), np.int16(q)
        meta = [sps, ch, crc, aa, raises]
        if not raises:
            aa_bits = bl.hex_string_to_bit(args[2])
            found = [p for p in range(phase + 1) if bl.search_unique_bit_sequence(bit_all[p], aa_bits) >= 0]
            start = (bit_all.shape[1] - (len(phy_bit) - 8)) if found else -1
            meta += [int(bool(crc_ok)), int(plen), int(phase), 1 + found[-1] if found else 0, start]
            out[f"w{k}_pdu_bit"] = np.asarray(pdu_bit, dtype=np.int8)
        else:
            meta += [0, 0, 0, 0, 0]
            out[f"w{k}_pdu_bit"] = np.zeros(0, dtype=np.int8)
        out[f"w{k}_meta"] = np.array(meta, dtype=np.int64)
        print(k, name, "sps", sps, "ch", ch, "raises" if raises else meta[5:])
    out["names"] = np.array(names)
    bl.SAMPLE_PER_SYMBOL = 8
    np.savez_compressed(os.path.join(ROOT, "tests", "golden", "btlelib_rx_sps.npz"), **out)


def main():
    td = tempfile.mkdtemp()
    shutil.copytree(os.path.join(REF, "python"), os.path.join(td, "python"))
    os.makedirs(os.path.join(td, "verilog"))
    os.chdir(os.path.join(td, "python"))
    sys.path.insert(0, os.getcwd())
    import btlelib as bl
    if "--random" in sys.argv:
        random_cases(bl)
        return
    if "--sps" in sys.argv:
        sps_cases(bl)
        return
    out = {}
    cases = [
        (37, "", "", "4225" + "0289674523" + "01" * 32, 20.0, 1),
        (37, "", "", "4225" + "0289674523" + "01" * 32, 7.0, 2),          # noisy: CRC may fail on early phases
        (9, "A77B22", "1B0A8560", "030c00020f0e50040706d007ffee", 15.0, 3),
        (10, "123456", "1B0A8511", "0100", 12.0, 4),
        (38, "", "", "40" + "10" + "a1b2c3d4e5f6" + "00112233445566778899", -3.0, 5),   # hopeless SNR
    ]
    for n, (ch, crc_hex, aa_hex, pdu_hex, snr, seed) in enumerate(cases):
        pdu_bit = bl.hex_string_to_bit(pdu_hex)
        crc_bits = bl.hex_string_to_bit(crc_hex) if crc_hex else []
        args_tx = [ch] + ([crc_bits, aa_hex] if crc_hex else [])
        tx_i, tx_q, _, _ = bl.btle_tx(pdu_bit, *args_tx)
        np.random.seed(seed)
        rx_i, rx_q = bl.add_noise(tx_i, tx_q, snr)
        args_rx = [ch] + ([crc_bits, aa_hex] if crc_hex else [])
        r = bl.btle_rx(rx_i, rx_q, *args_rx)
        out[f"c{n}_i"] = np.int16(rx_i); out[f"c{n}_q"] = np.int16(rx_q)
        out[f"c{n}_ch"] = ch; out[f"c{n}_crc_hex"] = crc_hex; out[f"c{n}_aa_hex"] = aa_hex
        out[f"c{n}_pdu_bit"] = np.asarray(r[0], dtype=np.int8); out[f"c{n}_crc_ok"] = bool(r[1])
        out[f"c{n}_plen"] = int(r[2]); out[f"c{n}_phy_bit"] = np.asarray(r[3], dtype=np.int8)
        out[f"c{n}_bit_all"] = r[4]; out[f"c{n}_sig_all"] = r[5]; out[f"c{n}_phase"] = int(r[6])
        print(n, "ch", ch, "snr", snr, "crc_ok", r[1], "plen", r[2], "phase", r[6])
    out["n_cases"] = len(cases)
    # TX waveforms (for the batched 8-sps synthesiser used by the BER harness)
    for n, (ch, crc_hex, aa_hex, pdu_hex) in enumerate([(37, "", "", "422506050403020119095344522f426c7565746f6f74682f4c6f772f456e657267791234567890"),
                                                       (11, "A77B22", "1B0A8560", "0103112233")]):
        pdu_bit = bl.hex_string_to_bit(pdu_hex)
        args_tx = [ch] + ([bl.hex_string_to_bit(crc_hex), aa_hex] if crc_hex else [])
        ti, tq, phy_bit, _ = bl.btle_tx(pdu_bit, *args_tx)
        out[f"tx{n}_i"], out[f"tx{n}_q"], out[f"tx{n}_phy_bit"], out[f"tx{n}_pdu_bit"] = np.int8(ti), np.int8(tq), np.int8(phy_bit), pdu_bit
        out[f"tx{n}_ch"], out[f"tx{n}_crc_hex"], out[f"tx{n}_aa_hex"] = ch, crc_hex, aa_hex
    out["gauss_fir_int8"] = np.int8(bl.gfsk_modulation_fixed_point.gauss_fir)
    out["cos_table"] = np.int8(bl.vco_fixed_point.cos_table)
    # leaf vectors
    rng = np.random.default_rng(3)
    bits = rng.integers(0, 2, 400).astype(np.int8)
    init = bl.hex_string_to_bit("A77B22")
    out["leaf_bits"] = bits
    out["leaf_crc_init"] = init
    out["leaf_crc24_core"] = bl.crc24_core(bits, init)
    for ch in (0, 17, 37):
        out[f"leaf_scramble_{ch}"] = bl.scramble_core(bits, ch)
    seq = bits[123:155].copy()
    out["leaf_seq"] = seq
    out["leaf_seq_idx"] = bl.search_unique_bit_sequence(bits, seq)
    out["leaf_seq_miss"] = bl.search_unique_bit_sequence(bits, 1 - np.zeros(64, dtype=np.int8))
    i16 = rng.integers(-300, 300, 777).astype(np.int16); q16 = rng.integers(-300, 300, 777).astype(np.int16)
    b, s = bl.gfsk_demodulation_fixed_point(i16, q16)
    out["leaf_i16"], out["leaf_q16"], out["leaf_gfsk_bit"], out["leaf_gfsk_sig"] = i16, q16, b, s
    out["hex_bits"] = bl.hex_string_to_bit("D6BE898E")
    np.savez_compressed(os.path.join(ROOT, "tests", "golden", "btlelib_rx.npz"), **out)


if __name__ == "__main__":
    main()
