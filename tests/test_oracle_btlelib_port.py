"""oracle/btlelib_port.py (numpy restatement of the reference's bit-true Python receiver) pinned to the reference: against
the committed golden vectors and against the reference btlelib's recorded verdicts on 60 random packets (both written by
oracle/gen_golden_btlelib.py)."""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "oracle"))
import btlelib_port as P  # noqa: E402

GOLD = os.path.join(ROOT, "tests", "golden", "btlelib_rx.npz")
GOLD_RANDOM = os.path.join(ROOT, "tests", "golden", "btlelib_rx_random.npz")


def _hex_le(h):            # 'A77B22' as btlelib passes it -> the -k style integer
    return int(h, 16)


def test_port_equals_reference_golden_vectors():
    z = np.load(GOLD)
    for n in range(int(z["n_cases"])):
        ch, crc_hex, aa_hex = int(z[f"c{n}_ch"]), str(z[f"c{n}_crc_hex"]), str(z[f"c{n}_aa_hex"])
        crc = int(crc_hex, 16) if crc_hex else 0x555555
        aa = int.from_bytes(bytes.fromhex(aa_hex), "little") if aa_hex else 0x8E89BED6
        r = P.rx_window(z[f"c{n}_i"], z[f"c{n}_q"], ch, crc, aa)
        assert r["crc_ok"] == bool(z[f"c{n}_crc_ok"]) and r["plen"] == int(z[f"c{n}_plen"]) and r["phase"] == int(z[f"c{n}_phase"]), n
        assert np.array_equal(r["pdu_bit"], z[f"c{n}_pdu_bit"]), n


def random_windows(n=60):
    """The 60 noisy random-packet windows the reference's btlelib.btle_rx was run on, rebuilt in-repo: the port's PHY bits
    through the 8-sps modulator (sample for sample btlelib.btle_tx, checked by the generator), then btlelib.add_noise's rule
    (normal noise on each rail, sigma = 127 / 10^(snr/20) / sqrt(2), drawn right after np.random.seed(100 + k)), random
    alignment padding and truncation to whole symbols.  Yields one dict per window: k, ch, crc_hex, aa_hex, pdu, snr, the
    transmitted waveform tx = (i, q), the noisy waveform before padding noisy = (i, q) and the window i, q (float)."""
    import torch
    from btle_b200 import synth
    rng = np.random.default_rng(5)
    for k in range(n):
        ch = int(rng.choice([37, 38, 39, 3, 20]))
        adv = ch >= 37
        plen = int(rng.integers(6, 38)) if adv else int(rng.integers(0, 28))
        pdu = bytes([int(rng.integers(0, 16)), plen]) + rng.integers(0, 256, plen, dtype=np.uint8).tobytes()
        crc_hex, aa_hex = ("", "") if adv else ("A77B22", "1B0A8560")
        bits = P.tx_bits(pdu, ch, int(crc_hex, 16) if crc_hex else 0x555555,
                         int.from_bytes(bytes.fromhex(aa_hex), "little") if aa_hex else 0x8E89BED6)
        ti, tq = synth.modulate_batch_8sps(torch.from_numpy(bits[None, :]))
        ti, tq = ti[0].numpy().astype(np.float64), tq[0].numpy().astype(np.float64)
        np.random.seed(100 + k)
        snr = float(rng.choice([4.0, 7.0, 9.0, 12.0, 20.0]))
        sigma = 127 / np.power(10, snr / 20) / np.sqrt(2)
        ni = ti + np.random.normal(0, sigma, len(ti))
        nq = tq + np.random.normal(0, sigma, len(tq))
        pad = int(rng.integers(0, 5)) * 8 + int(rng.integers(0, 8))          # arbitrary alignment, like a window cut from a stream
        ri = np.concatenate((np.random.normal(0, 3, pad), ni, np.random.normal(0, 3, 64)))
        rq = np.concatenate((np.random.normal(0, 3, pad), nq, np.random.normal(0, 3, 64)))
        ri, rq = ri[: len(ri) // 8 * 8], rq[: len(rq) // 8 * 8]
        yield dict(k=k, ch=ch, crc_hex=crc_hex, aa_hex=aa_hex, pdu=pdu, snr=snr, tx=(ti, tq), noisy=(ni, nq), i=ri, q=rq)


def test_port_equals_imported_reference_on_random_packets():
    """The port on 60 random packets at SNR 4..20 dB with arbitrary alignment against what the reference's own btlelib.btle_rx
    returned on the same windows (tests/golden/btlelib_rx_random.npz)."""
    z = np.load(GOLD_RANDOM)
    assert len(z["ch"]) == 60
    ends = np.cumsum(z["pdu_len"])
    ref_bits = np.unpackbits(z["pdu_bits"])[:ends[-1]].astype(np.int8)
    n_ok = n_bad = 0
    for w in random_windows(len(z["ch"])):
        k, ch, crc_hex, aa_hex, snr, ri, rq = w["k"], w["ch"], w["crc_hex"], w["aa_hex"], w["snr"], w["i"], w["q"]
        assert z["ch"][k] == ch and z["n"][k] == len(ri), k                     # same window as the reference saw
        got = P.rx_window(np.int16(ri), np.int16(rq), ch, int(crc_hex, 16) if crc_hex else 0x555555,
                          int.from_bytes(bytes.fromhex(aa_hex), "little") if aa_hex else 0x8E89BED6)
        ref_ok = bool(z["crc_ok"][k])
        assert got["crc_ok"] == ref_ok and got["plen"] == z["plen"][k] and got["phase"] == z["phase"][k], (k, snr)
        assert np.array_equal(got["pdu_bit"], ref_bits[ends[k] - z["pdu_len"][k]:ends[k]]), (k, snr)
        n_ok += ref_ok; n_bad += not ref_ok
    assert n_ok > 20 and n_bad > 5


GOLD_SPS = os.path.join(ROOT, "tests", "golden", "btlelib_rx_sps.npz")


def sps_windows():
    """The crafted windows of tests/golden/btlelib_rx_sps.npz with the reference's verdicts (oracle/gen_golden_btlelib.py
    --sps: btlelib.btle_rx with SAMPLE_PER_SYMBOL 1, 2, 4, 8, 16)."""
    z = np.load(GOLD_SPS)
    for k, name in enumerate(z["names"]):
        sps, ch, crc, aa, raises, crc_ok, plen, phase, found, start = (int(v) for v in z[f"w{k}_meta"])
        yield dict(name=str(name), sps=sps, ch=ch, crc=crc, aa=aa, raises=bool(raises), crc_ok=bool(crc_ok), plen=plen, phase=phase,
                   found=found, start=start, pdu_bit=z[f"w{k}_pdu_bit"], i=z[f"w{k}_i"], q=z[f"w{k}_q"])


def test_port_equals_reference_at_every_sps():
    """rx_window(sps=...) against the reference's btle_rx at 1, 2, 4, 8 and 16 samples per symbol: 34 and 2048 symbols, the
    access address at the last index, both arms of the CRC-position clamp (crc_start < 40 too), 6- and 5-bit lengths, never
    found, found but never CRC-ok, CRC-ok on a later phase than the first hit, int16 extremes."""
    seen = set()
    for w in sps_windows():
        got = P.rx_window(w["i"], w["q"], w["ch"], w["crc"], w["aa"], sps=w["sps"])
        seen.add((w["name"], w["sps"]))
        if w["raises"]:
            # the reference indexes past its header here; the port (like the kernel) reads the missing bits as 0
            assert got["found"] and got["start"] + 40 + (6 if w["ch"] >= 37 else 5) > len(w["i"]) // w["sps"] - 1, w["name"]
            continue
        key = (w["name"], w["sps"])
        assert (got["crc_ok"], got["plen"], got["phase"], got["found"], got["start"]) == \
            (w["crc_ok"], w["plen"], w["phase"], w["found"], w["start"]), key
        assert np.array_equal(got["pdu_bit"], w["pdu_bit"]), key
    for sps in (1, 2, 4, 8, 16):
        for name in ("adv_clean", "data_never_ok", "adv_clamp_lt40_54", "data_clamp_lt40_53", "adv_aa_last", "n34_noise", "n34_aa_at_1",
                     "extreme_packet"):
            assert (name, sps) in seen, (name, sps)
    assert ("n2048_data_at_end", 1) in seen and ("adv_ok_on_later_phase", 16) in seen


def test_port_stream_finds_what_it_sent():
    """The streaming rules on a synthetic 8-Msps capture built with the port's own transmitter bits and the 8-sps modulator:
    every packet comes back once, with its bytes, in order."""
    import torch
    from btle_b200 import synth
    rng = np.random.default_rng(9)
    pdus = [bytes([0x40, 6 + k % 20]) + rng.integers(0, 256, 6 + k % 20, dtype=np.uint8).tobytes() for k in range(12)]
    n = 12 * 6000 + 4096
    cap = rng.normal(0, 2.0, (n, 2))
    pos = []
    for k, pdu in enumerate(pdus):
        bits = P.tx_bits(pdu, 37)
        ti, tq = synth.modulate_batch_8sps(torch.from_numpy(bits[None, :]))
        p0 = 6000 * k + 500 + int(rng.integers(0, 1000))
        cap[p0:p0 + ti.shape[1], 0] += ti[0].numpy()
        cap[p0:p0 + ti.shape[1], 1] += tq[0].numpy()
        pos.append(p0)
    iq16 = cap.astype(np.int16)
    got = P.rx_stream(iq16, 37)
    assert len(got) == len(pdus)
    for g, pdu, p0 in zip(got, pdus, pos):
        assert g["crc_ok"] and bytes(np.packbits(g["pdu_bit"], bitorder="little")) == pdu
        assert 0 <= g["sample"] - p0 - 8 * 8 < 24                 # preamble (8 symbols) + modulator delay
