#!/usr/bin/env python
"""Cost of the low-pass filter in front of the symbol-spaced discriminator (BTLE_CFG_LOWPASS).
  receive-kernel time of one 1 GiB c2-like capture (channel 37, 1 % corrupted bursts, straddling packets) and of 1 GiB of
  full-scale random IQ (bench.py's hot input) four ways each, calls alternating, CUDA events around each call, median of
  --calls each: symbol-spaced, symbol-spaced + low-pass, and the rotated form of each at 100 kHz (btle_b200_rx_device_dir /
  _offset).  Prints the time per GiB, the share of 3.35 TB/s (H100 SXM HBM3) the capture's bytes would need at that time,
  and the record count of each way, which must not change from call to call.  One JSON line per input with the card's name
  and power limit read in the same run.
  python tools/bench_lowpass.py [--calls 12]"""
import argparse
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

from btle_b200 import BtleRx, make_cfgs, synth

N_INT8 = 1 << 30


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True)
    return q.stdout.strip()


def run(rx, iq, calls):
    cap = 2_000_000
    out = torch.empty(cap * 64, dtype=torch.uint8, device="cuda")
    count = torch.zeros(1, dtype=torch.int32, device="cuda")
    d_dir = torch.empty(rx.units(1, N_INT8) * 8, dtype=torch.uint8, device="cuda")
    sym, lp = make_cfgs(1, channel=37, symbol_spaced=1), make_cfgs(1, channel=37, symbol_spaced=1, lowpass=1)
    ways = {"symbol": (sym, None), "lowpass": (lp, None), "symbol_rot100k": (sym, 100e3), "lowpass_rot100k": (lp, 100e3)}
    times = {k: [] for k in ways}
    counts = {k: set() for k in ways}
    st = torch.cuda.current_stream().cuda_stream
    names = list(ways)
    for i in range(len(names) * (calls + 2)):
        k = names[i % len(names)]
        cfgs, hz = ways[k]
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        rx.rx_device_dir(iq.view(1, -1), cfgs, out, count, d_dir, st, offset_hz=hz)
        e1.record()
        torch.cuda.synchronize()
        counts[k].add(int(count.item()))
        if i >= 2 * len(names):
            times[k].append(e0.elapsed_time(e1))
    res = {}
    for k, v in times.items():
        assert len(counts[k]) == 1, (k, counts[k])
        ms = float(np.median(v))
        res[k] = {"ms_per_gib": round(ms, 4), "hbm_share": round(N_INT8 / (ms * 1e-3) / 3.35e12, 4), "records": counts[k].pop()}
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=12)
    a = ap.parse_args()
    rx = BtleRx(0)
    name = card()
    dev = torch.device("cuda", 0)
    iq, _ = synth.make_adv_stream(N_INT8, seed=0x37E15163, channel=37, corrupt_every=100, device=dev, use_cuda_modulator=False,
                                  straddle_every=100)
    print(json.dumps({"what": "time", "input": "c2", "card": name, "calls": a.calls, **run(rx, iq, a.calls)}), flush=True)
    del iq
    g = torch.Generator(device=dev)
    g.manual_seed(5)
    hot = torch.randint(-128, 128, (N_INT8,), generator=g, device=dev, dtype=torch.int8)
    print(json.dumps({"what": "time", "input": "hot", "card": name, "calls": a.calls, **run(rx, hot, a.calls)}), flush=True)


if __name__ == "__main__":
    main()
