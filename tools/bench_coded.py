#!/usr/bin/env python
"""Cost of the LE Coded PHY receiver (btle_b200_rx_coded_device) against the 1M receive launch (btle_b200_rx_device).
  Three 1 GiB inputs: a c2-like 1M capture (channel 37, 1 % corrupted bursts, straddling packets), full-scale random IQ
  (bench.py's hot input), and a capture dense with coded bursts (S=2 and S=8, 0..255-byte PDUs, back to back at 10 dB).
  Calls alternate, CUDA events around each call, median of --calls each.  Prints the time per GiB and the record count of
  each way, which must not change from call to call.  One JSON line per input with the card's name and power limit read in
  the same run.
  python tools/bench_coded.py [--calls 12]"""
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


def coded_capture(dev):
    """1 GiB of noise with coded bursts back to back: a pool of 64 modulated bursts placed again and again"""
    rng = np.random.default_rng(17)
    pool = []
    for k in range(64):
        L = int(rng.integers(0, 256))
        pdu = bytes([0x07, L]) + rng.integers(0, 256, L, dtype=np.uint8).tobytes()
        pool.append(torch.from_numpy(synth.coded_air(pdu, 37, s=(2, 8)[k % 2]).astype(np.int16) * 100 // 127))
    g = torch.Generator(device=dev)
    g.manual_seed(3)
    iq = (torch.randn(N_INT8, generator=g, device=dev) * (100 / 10 ** 0.5 / 2 ** 0.5)).round().to(torch.int16)
    pos, k, n = 0, 0, 0
    while True:
        w = pool[k % 64].to(dev)
        if pos + w.numel() + 2000 > N_INT8:
            break
        iq[pos:pos + w.numel()] += w
        pos += w.numel() + 2 * int(rng.integers(200, 2000))
        k += 1
        n += 1
    return iq.clamp_(-128, 127).to(torch.int8), n


def run(rx, iq, calls):
    cap1, capc = 2_000_000, 400_000
    out1 = torch.empty(cap1 * 64, dtype=torch.uint8, device="cuda")
    outc = torch.empty(capc * 304, dtype=torch.uint8, device="cuda")
    count = torch.zeros(1, dtype=torch.int32, device="cuda")
    cfg1, cfgc = make_cfgs(1, channel=37), make_cfgs(1, channel=37)
    st = torch.cuda.current_stream().cuda_stream
    ways = {"rx_device": lambda: rx.rx_device(iq.view(1, -1), cfg1, out1, count, st),
            "rx_coded_device": lambda: rx.rx_coded_device(iq.view(1, -1), cfgc, outc, count, st)}
    times = {k: [] for k in ways}
    counts = {k: set() for k in ways}
    names = list(ways)
    for i in range(len(names) * (calls + 2)):
        k = names[i % len(names)]
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        ways[k]()
        e1.record()
        torch.cuda.synchronize()
        counts[k].add(int(count.item()))
        if i >= 2 * len(names):
            times[k].append(e0.elapsed_time(e1))
    res = {}
    for k, v in times.items():
        assert len(counts[k]) == 1, (k, counts[k])
        res[k] = {"ms_per_gib": round(float(np.median(v)), 4), "spread_ms": round(float(np.max(v) - np.min(v)), 4), "records": counts[k].pop()}
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
    del hot
    dense, n = coded_capture(dev)
    print(json.dumps({"what": "time", "input": "coded_dense", "bursts": n, "card": name, "calls": a.calls, **run(rx, dense, a.calls)}),
          flush=True)


if __name__ == "__main__":
    main()
