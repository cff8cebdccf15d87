#!/usr/bin/env python
"""Cost of BTLE_CFG_RECOVER: receive-kernel time of btle_b200_rx_device on one 1 GiB capture with the flag off and on
(CUDA events around each call, calls alternating, median of --calls per side), on two inputs:
  c2   the benchmark's c2-like capture (channel 37, 1 % corrupted bursts, straddling packets);
  ber  1 GiB from btle_b200_rx_ber_synth_device at --snr dB (channel 37, slot 2048), where many packets fail the CRC.
Prints one JSON line per input with the card's name and power limit read in the same run.
  python tools/bench_recover.py [--calls 24] [--snr 20]"""
import argparse
import ctypes
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

from btle_b200 import BtleRx, ber, make_cfgs, synth
from btle_b200._native import RX_BER_TRUTH_DTYPE

N_INT8 = 1 << 30


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True)
    return q.stdout.strip()


def measure(rx, iq, calls):
    cap = 2_000_000
    out = torch.empty(cap * 64, dtype=torch.uint8, device="cuda")
    cnt = torch.zeros(1, dtype=torch.int32, device="cuda")
    cfgs = {f: make_cfgs(1, channel=37, recover=f) for f in (0, 1)}
    times, found = {0: [], 1: []}, {}
    for i in range(4 + 2 * calls):
        f = i & 1
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        rx.rx_device(iq.view(1, -1), cfgs[f], out, cnt)
        b.record()
        torch.cuda.synchronize()
        if i >= 4:
            times[f].append(a.elapsed_time(b))
        n = int(cnt.item())
        recs = out[:min(n, cap) * 64].cpu().numpy().view([("x", "u1", 15), ("flags", "u1"), ("y", "u1", 48)])
        found[f] = (n, int(((recs["flags"] & 8) != 0).sum()))
    med = {f: float(np.median(times[f])) for f in (0, 1)}
    return {"off_ms": round(med[0], 4), "on_ms": round(med[1], 4), "cost_pct": round(100 * (med[1] / med[0] - 1), 2),
            "records": found[0][0], "recovered": found[1][1], "calls_per_side": calls}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=24)
    ap.add_argument("--snr", type=float, default=20.0)
    a = ap.parse_args()
    rx = BtleRx(0)
    name = card()
    iq, _ = synth.make_adv_stream(N_INT8, seed=0x37E15163, channel=37, corrupt_every=100, device=torch.device("cuda", 0),
                                  use_cuda_modulator=False, straddle_every=100)
    print(json.dumps({"input": "c2", "card": name, **measure(rx, iq, a.calls)}), flush=True)
    del iq
    cfg = ber.rx_ber_cfg(a.snr, slot_samples=2048, seed=1)
    n_packets = N_INT8 // 2 // 2048
    d_iq = torch.empty(N_INT8, dtype=torch.int8, device="cuda")
    d_truth = torch.empty(n_packets * RX_BER_TRUTH_DTYPE.itemsize, dtype=torch.uint8, device="cuda")
    rx._check(rx._L.btle_b200_rx_ber_synth_device(rx._h, cfg.ctypes.data, 0, n_packets, d_iq.data_ptr(), d_truth.data_ptr(),
                                                  ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)))
    torch.cuda.synchronize()
    print(json.dumps({"input": f"ber{a.snr:g}dB", "card": name, **measure(rx, d_iq, a.calls)}), flush=True)


if __name__ == "__main__":
    main()
