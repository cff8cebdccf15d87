#!/usr/bin/env python
"""Packet error rate of the LE Coded PHY receiver (btle_b200_rx_coded) against SNR, for S=2 and S=8, and of the same PDUs
sent as 1M packets through the best 1M chain (symbol-spaced + low-pass + centred hits + RECOVER + CORRECT), same noise
definition and the same packets per point.
  Noise as rx_ber_run: sigma = amplitude / 10^(snr/20) / sqrt 2 per rail, rounded and saturated to int8.  Each point is
  one capture holding --packets bursts (ADV PDUs with 6..37 payload bytes on channel 37) 1000 samples apart, at integer
  positions that cover all four sample phases.  A packet counts as received when a CRC-ok record within 3 samples of its
  access address carries its PDU.  Prints one JSON line per point with the card's name and power limit.
  python tools/coded_ber_report.py [--packets 500] [--snr -6 -5 ... 8]"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np

from btle_b200 import BtleRx, make_cfgs, synth
from btle_b200._native import CFG_CENTRE_HITS, CFG_CORRECT, CFG_LOWPASS, CFG_RECOVER, CFG_SYMBOL_SPACED

BEST_1M = CFG_SYMBOL_SPACED | CFG_LOWPASS | CFG_CENTRE_HITS | CFG_RECOVER | CFG_CORRECT


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True)
    return q.stdout.strip()


def capture(waves, aa_offset, snr_db, amplitude, rng):
    """one capture of the bursts back to back; returns (int8 iq, access-address sample of each burst)"""
    starts, pos = [], 500
    for k, w in enumerate(waves):
        starts.append(pos + k % 4)
        pos += w.size // 2 + 1000 + 4
    x = np.zeros((pos + 2000, 2))
    for s, w in zip(starts, waves):
        x[s:s + w.size // 2] += w.astype(np.float64).reshape(-1, 2) * amplitude / 127
    x += rng.normal(0.0, amplitude / 10 ** (snr_db / 20) / np.sqrt(2), x.shape)
    return np.clip(np.round(x), -128, 127).astype(np.int8).reshape(-1), np.array(starts) + aa_offset


def lost(recs, sample_key, n0s, pdus):
    ok = recs[recs["crc_bad"] == 0]
    bad = 0
    for n0, pdu in zip(n0s, pdus):
        near = ok[np.abs(sample_key(ok) - n0) <= 3]
        bad += not any(bytes(r["bytes"][:len(pdu)]) == pdu for r in near)
    return bad


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--packets", type=int, default=500)
    ap.add_argument("--snr", type=float, nargs="+", default=[-6, -5, -4, -3, -2, -1, 0, 1, 2, 4, 6, 8])
    ap.add_argument("--amplitude", type=int, default=100)
    ap.add_argument("--seed", type=int, default=1)
    a = ap.parse_args()
    rx = BtleRx(0)
    name = card()
    rng = np.random.default_rng(a.seed)
    pdus = [synth.adv_pdu(2, 1, 0, rng.integers(0, 256, int(L), dtype=np.uint8).tobytes()) for L in rng.integers(6, 38, a.packets)]
    waves = {s: [synth.coded_air(p, 37, s=s) for p in pdus] for s in (2, 8)}
    waves["1m"] = [synth.modulate(synth.air_bytes(p, 37)) for p in pdus]
    for snr in a.snr:
        row = {"what": "per", "snr_db": snr, "packets": a.packets, "card": name}
        for way in (8, 2, "1m"):
            seed = int(rng.integers(1 << 30))
            if way == "1m":
                iq, n0s = capture(waves[way], 39, snr, a.amplitude, np.random.default_rng(seed))
                recs = rx.rx(iq, channel=37, rssi=BEST_1M)
                bad = lost(recs, lambda r: r["chunk"].astype(np.int64) * 8192 + r["n0"], n0s, pdus)
            else:
                iq, n0s = capture(waves[way], synth.CODED_AA_SAMPLE, snr, a.amplitude, np.random.default_rng(seed))
                recs = rx.rx_coded(iq, make_cfgs(1, channel=37))
                bad = lost(recs, lambda r: r["sample"], n0s, pdus)
            row[f"per_{way if way == '1m' else 's%d' % way}"] = round(bad / a.packets, 4)
        print(json.dumps(row), flush=True)


if __name__ == "__main__":
    main()
