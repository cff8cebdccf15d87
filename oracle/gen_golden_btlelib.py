#!/usr/bin/env python
"""Golden vectors for the btlelib-compatible shim, produced by importing the REFERENCE's own
python/btlelib.py here (from a writable copy: it writes table files next to itself on first TX
call, btlelib.py:90-91,155).  Writes tests/golden/btlelib_rx.npz (committed); with --random, instead
tests/golden/btlelib_rx_random.npz: the reference receiver's verdicts on the 60 random-packet windows of
tests/test_oracle_btlelib_port.py, whose inputs the test rebuilds itself (checked here against btle_tx / add_noise); with
--sps, tests/golden/btlelib_rx_sps.npz: the reference receiver at SAMPLE_PER_SYMBOL 1, 2, 4, 8 and 16 on crafted windows
(sps_windows), inputs stored with the verdicts; with --leaves, tests/golden/btlelib_leaves.npz: the reference's leaf
functions (gfsk_demodulation_fixed_point, crc24_core / crc24, scramble_core / scramble, search_unique_bit_sequence) at
their edges (leaves_cases), written with fixed time stamps so that a rerun gives the same bytes."""
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


def save_npz_stable(path, arrays):
    """np.savez_compressed, but with fixed member time stamps, so that the same arrays give the same file bytes."""
    import io
    import zipfile
    with zipfile.ZipFile(path, "w", compression=zipfile.ZIP_DEFLATED) as zf:
        for key, val in arrays.items():
            buf = io.BytesIO()
            np.lib.format.write_array(buf, np.asanyarray(val), allow_pickle=False)
            info = zipfile.ZipInfo(key + ".npy", date_time=(1980, 1, 1, 0, 0, 0))
            info.compress_type = zipfile.ZIP_DEFLATED
            zf.writestr(info, buf.getvalue())


def de_bruijn_pairs(k):
    """A cyclic de Bruijn sequence of order 2 over 0..k-1 (every ordered pair once, cyclically), as a list."""
    a, seq = [0] * (2 * k), []

    def db(t, p):
        if t > 2:
            if 2 % p == 0:
                seq.extend(a[1:p + 1])
            return
        a[t] = a[t - p]
        db(t + 1, p)
        for j in range(a[t - p] + 1, k):
            a[t] = j
            db(t + 1, t)
    db(1, 1)
    return seq


def leaves_cases(bl):
    """tests/golden/btlelib_leaves.npz: the reference's gfsk_demodulation_fixed_point, crc24_core / crc24, scramble_core /
    scramble and search_unique_bit_sequence at their edges (tests/test_btlelib_leaves_gpu.py)."""
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    from test_btlelib_leaves_gpu import big_search_input, seeded_bits
    rng = np.random.default_rng(2024)
    out = {}
    # gfsk_demodulation_fixed_point: short lengths on full-range samples, then every (i[k], q[k], i[k+1], q[k+1]) over
    # the int16 extremes: a de Bruijn sequence of the 36 (i, q) pairs, closed by its first pair
    lens = (0, 1, 2, 3, 256, 257, 513)
    for k, n in enumerate(lens):
        i = rng.integers(-32768, 32768, n, dtype=np.int16)
        q = rng.integers(-32768, 32768, n, dtype=np.int16)
        i[::7], q[3::11] = -32768, 32767
        b, s = bl.gfsk_demodulation_fixed_point(i, q)
        out[f"gfsk{k}_i"], out[f"gfsk{k}_q"], out[f"gfsk{k}_bit"], out[f"gfsk{k}_sig"] = i, q, b, s
    out["gfsk_n"] = len(lens)
    vals = np.array([-32768, -32767, -1, 0, 1, 32767], dtype=np.int16)
    sym = de_bruijn_pairs(36)
    sym = np.array(sym + sym[:1])
    i, q = vals[sym // 6], vals[sym % 6]
    b, s = bl.gfsk_demodulation_fixed_point(i, q)
    assert s.max() == 2147450880 and s.min() == -2147450880
    out["gfsk_db_i"], out["gfsk_db_q"], out["gfsk_db_bit"], out["gfsk_db_sig"] = i, q, b, s
    # crc24_core / crc24: bit counts around one register length and past the 40 bits crc24 skips
    inits = [np.zeros(24, np.int8), np.ones(24, np.int8), np.array([1, 0] * 12, np.int8), rng.integers(0, 2, 24).astype(np.int8)]
    k = 0
    for n in (0, 1, 23, 24, 25, 400, 2000):
        bits = rng.integers(0, 2, n).astype(np.int8)
        for init in inits:
            out[f"crc{k}_bits"], out[f"crc{k}_init"] = bits, init
            out[f"crc{k}_core"] = bl.crc24_core(bits, init.copy())
            out[f"crc{k}_full"] = bl.crc24(bits, init.copy())
            k += 1
    out["crc_n"] = k
    # scramble_core / scramble: every 6-bit channel and integers outside 0..63, lengths across the 127-bit period
    bits = rng.integers(0, 2, 1000).astype(np.int8)
    chans = list(range(64)) + [64, 100, -1, -64]
    scr_len = (1, 7, 127, 128, 254, 1000)
    out["scr_bits"], out["scr_ch"], out["scr_len"] = bits, np.array(chans, np.int32), np.array(scr_len, np.int32)
    out["scr_core"] = np.array([np.concatenate([bl.scramble_core(bits[:n], ch) for n in scr_len]) for ch in chans], np.int8)
    out["scr_full"] = np.array([bl.scramble(bits, ch) for ch in chans], np.int8)
    # search_unique_bit_sequence
    seqs = []
    base = rng.integers(0, 2, 300).astype(np.int8)
    seqs.append((base, base[:32].copy()))                            # match at 0
    b = base.copy(); s = rng.integers(0, 2, 40).astype(np.int8); b[-40:] = s
    seqs.append((b, s))                                              # match at n - m
    b = base.copy(); s = rng.integers(0, 2, 24).astype(np.int8)
    for p in (50, 120, 200):
        b[p:p + 24] = s
    seqs.append((b, s))                                              # several matches: the first wins
    seqs.append((base, base.copy()))                                 # m == n
    s = base.copy(); s[-1] ^= 1
    seqs.append((base, s))                                           # m == n, last bit differs
    seqs.append((base, np.concatenate([base, [0]]).astype(np.int8)))  # m == n + 1
    b = np.zeros(300, np.int8); b[173] = 1
    seqs.append((b, np.ones(1, np.int8)))                            # m == 1
    seqs.append((np.ones(300, np.int8), np.zeros(1, np.int8)))       # m == 1, never
    seqs.append((base, np.zeros(0, np.int8)))                        # m == 0
    seqs.append((np.zeros(0, np.int8), np.zeros(0, np.int8)))        # m == n == 0
    seqs.append((np.zeros(0, np.int8), np.ones(1, np.int8)))         # n == 0, m == 1
    long_bits = rng.integers(0, 2, 6000).astype(np.int8)
    seqs.append((long_bits, long_bits[1904:].copy()))                # m 4096 at n - m
    seqs.append((long_bits, long_bits[1000:].copy()))                # m 5000 at n - m
    s = long_bits[700:5700].copy(); s[4321] ^= 1
    seqs.append((long_bits, s))                                      # m 5000, one bit off
    seqs.append((long_bits[:4999], long_bits[:5000].copy()))         # m 5000 > n
    for k, (b, s) in enumerate(seqs):
        out[f"seq{k}_bit"], out[f"seq{k}_seq"] = b, s
    out["seq_idx"] = np.array([bl.search_unique_bit_sequence(b, s) for b, s in seqs], np.int64)
    out["seq_n"] = len(seqs)
    # a match in the last position of a 2^20-bit input, kept as (seed, n, m, position, result)
    meta = np.array([777, 1 << 20, 48, (1 << 20) - 48, 0], np.int64)
    b, s = big_search_input(meta)
    meta[4] = bl.search_unique_bit_sequence(b, s)
    out["seq_big"] = meta
    out["seeded_probe"] = 4242
    out["seeded_probe_bits"] = seeded_bits(4242, 4096)
    print({k: v for k, v in zip(range(len(seqs)), out["seq_idx"].tolist())}, "big", meta.tolist())
    save_npz_stable(os.path.join(ROOT, "tests", "golden", "btlelib_leaves.npz"), out)


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
    if "--leaves" in sys.argv:
        leaves_cases(bl)
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
