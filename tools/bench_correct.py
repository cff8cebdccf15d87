#!/usr/bin/env python
"""Cost of the CRC-24 syndrome correction (BTLE_CFG_CORRECT).
  receive-kernel time with the flag off and on, calls alternating, CUDA events around each call, median of --calls each,
  on three captures: one 1 GiB c2-like capture (channel 37, 1 % corrupted bursts, straddling packets) and two captures of
  the BER flow (btle_b200_rx_ber_synth_device, 2048-sample slots, 1 GiB): 20 dB in the default mode and 11 dB with the
  symbol-spaced discriminator, where many packets fail the CRC, both with BTLE_CFG_REPORT_REJECTED as
  btle_b200_rx_ber_run decodes them (btle_b200_rx_device_dir).  Prints ms per call, the on / off ratio and the record
  count of each way, which must not change from call to call.  One JSON line per capture with the card's name and power
  limit read in the same run.
  python tools/bench_correct.py [--calls 12]"""
import argparse
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

from btle_b200 import BtleRx, ber, make_cfgs, synth
from btle_b200._native import CFG_REPORT_REJECTED

N_INT8 = 1 << 30


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True)
    return q.stdout.strip()


def time_ways(rx, d_iq, ways, calls):
    n_int8 = d_iq.numel()
    cap = n_int8 // 16384 * 123
    out = torch.empty(cap * 64, dtype=torch.uint8, device="cuda")
    count = torch.zeros(1, dtype=torch.int32, device="cuda")
    d_dir = torch.empty(rx.units(1, n_int8) * 8, dtype=torch.uint8, device="cuda")
    st = torch.cuda.current_stream().cuda_stream
    names = list(ways)
    times, counts = {k: [] for k in names}, {k: set() for k in names}
    for i in range(len(names) * (calls + 2)):
        k = names[i % len(names)]
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        rx.rx_device_dir(d_iq.view(1, -1), ways[k], out, count, d_dir, st)
        e1.record()
        torch.cuda.synchronize()
        counts[k].add(int(count.item()))
        if i >= 2 * len(names):
            times[k].append(e0.elapsed_time(e1))
    res = {}
    for k in names:
        assert len(counts[k]) == 1, (k, counts[k])
        res[k] = {"ms": round(float(np.median(times[k])), 4), "records": counts[k].pop()}
    res["on_over_off"] = round(res["on"]["ms"] / res["off"]["ms"], 4)
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=12)
    a = ap.parse_args()
    rx = BtleRx(0)
    name = card()
    iq, _ = synth.make_adv_stream(N_INT8, seed=0x37E15163, channel=37, corrupt_every=100, device=torch.device("cuda", 0),
                                  use_cuda_modulator=False, straddle_every=100)
    ways = {"off": make_cfgs(1, channel=37), "on": make_cfgs(1, channel=37, correct=1)}
    print(json.dumps({"what": "c2-like 1 GiB", "card": name, "calls": a.calls, **time_ways(rx, iq, ways, a.calls)}), flush=True)
    del iq
    n = N_INT8 // 2 // 2048
    d_iq = torch.empty(N_INT8, dtype=torch.int8, device="cuda")
    d_truth = torch.empty(n * 64, dtype=torch.uint8, device="cuda")
    for snr, sym in ((20.0, 0), (11.0, 1)):
        cfg = ber.rx_ber_cfg(snr, slot_samples=2048, seed=7)
        rx._check(rx._L.btle_b200_rx_ber_synth_device(rx._h, cfg.ctypes.data, 0, n, d_iq.data_ptr(), d_truth.data_ptr(), None))
        torch.cuda.synchronize()
        ways = {"off": make_cfgs(1, channel=37, rssi=CFG_REPORT_REJECTED, symbol_spaced=sym),
                "on": make_cfgs(1, channel=37, rssi=CFG_REPORT_REJECTED, symbol_spaced=sym, correct=1)}
        what = f"rx_ber {snr:g} dB {'symbol-spaced' if sym else 'default'} 1 GiB"
        print(json.dumps({"what": what, "card": name, "calls": a.calls, **time_ways(rx, d_iq, ways, a.calls)}), flush=True)


if __name__ == "__main__":
    main()
