#!/usr/bin/env python
"""Cost and effect of the carrier-offset correction.
  time   receive-kernel time of one 1 GiB c2-like capture (channel 37, 1 % corrupted bursts, straddling packets) three
         ways, calls alternating, CUDA events around each call, median of --calls each: the default kernel
         (btle_b200_rx_device_dir), the rotated kernel at offset 0 and at 100 kHz (btle_b200_rx_device_dir_offset); time
         per GiB and the share of 3.35 TB/s (H100 SXM HBM3) the capture's bytes would need at that time.
  per    rx_ber_point PER at --snr dB, --packets per point: carrier offsets 0 / 50 / 100 / 150 kHz and 50 ppm, each
         uncorrected and corrected by the offset the synthesiser applies, recover off and on.
Prints JSON lines with the card's name and power limit read in the same run.
  python tools/bench_offset.py [--calls 12] [--snr 24] [--packets 20000]"""
import argparse
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

from btle_b200 import BtleRx, ber, make_cfgs, synth

N_INT8 = 1 << 30


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True)
    return q.stdout.strip()


def timing(rx, iq, calls):
    cap = 2_000_000
    out = torch.empty(cap * 64, dtype=torch.uint8, device="cuda")
    d_dir = torch.empty(rx.units(1, N_INT8) * 8, dtype=torch.uint8, device="cuda")
    cfgs = make_cfgs(1, channel=37)
    ways = {"default": None, "rot0": 0.0, "rot100k": 100e3}
    times = {k: [] for k in ways}
    st = torch.cuda.current_stream().cuda_stream
    for i in range(3 * (calls + 2)):
        k = list(ways)[i % 3]
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        rx.rx_device_dir(iq.view(1, -1), cfgs, out, None, d_dir, st, offset_hz=ways[k])
        b.record()
        torch.cuda.synchronize()
        if i >= 6:
            times[k].append(a.elapsed_time(b))
    res = {}
    for k, v in times.items():
        ms = float(np.median(v))
        res[k] = {"ms_per_gib": round(ms, 4), "hbm_share": round(N_INT8 / (ms * 1e-3) / 3.35e12, 4)}
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=12)
    ap.add_argument("--snr", type=float, default=24.0)
    ap.add_argument("--packets", type=int, default=20000)
    a = ap.parse_args()
    rx = BtleRx(0)
    name = card()
    iq, _ = synth.make_adv_stream(N_INT8, seed=0x37E15163, channel=37, corrupt_every=100, device=torch.device("cuda", 0),
                                  use_cuda_modulator=False, straddle_every=100)
    print(json.dumps({"what": "time", "card": name, "calls": a.calls, **timing(rx, iq, a.calls)}), flush=True)
    del iq
    ppm_hz = 50e-6 * 2450e6 * (1 + 50e-6)
    for rec in (False, True):
        for cfo, ppm in ((0.0, 0.0), (50e3, 0.0), (100e3, 0.0), (150e3, 0.0), (0.0, 50.0)):
            applied = cfo + (ppm_hz if ppm else 0.0)
            p = ber.rx_ber_point(rx, a.snr, a.packets, ppm=ppm, cfo_hz=cfo, recover=rec)
            q = ber.rx_ber_point(rx, a.snr, a.packets, ppm=ppm, cfo_hz=cfo, recover=rec, offset_hz=applied)
            print(json.dumps({"what": "per", "card": name, "snr_db": a.snr, "cfo_hz": cfo, "ppm": ppm, "recover": rec,
                              "per": round(p["per"], 4), "aa_miss": p["aa_miss"], "per_corrected": round(q["per"], 4),
                              "aa_miss_corrected": q["aa_miss"], "packets": p["packets"]}), flush=True)


if __name__ == "__main__":
    main()
