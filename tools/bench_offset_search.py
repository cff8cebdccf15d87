#!/usr/bin/env python
"""Cost of the bank of seven carrier-offset hypotheses (BTLE_CFG_OFFSET_SEARCH).
  Receive time of one 1 GiB c2-like capture (channel 37, 1 % corrupted bursts, straddling packets) and of 1 GiB of
  full-scale random IQ (bench.py's hot input) in the default, symbol-spaced and symbol-spaced + low-pass modes, each with
  the flag off and on: btle_b200_rx_device_dir, calls alternating, CUDA events around each call, median of --calls.  Then
  one flagged call per mode under torch.profiler, for the merge kernel's own time.  Prints the time per GiB, the flagged
  call's ratio to the unflagged one, and the record counts, which must not change from call to call.  One JSON line per
  input with the card's name and power limit read in the same run.
  python tools/bench_offset_search.py [--calls 8]"""
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
MODES = {"default": {}, "symbol": {"symbol_spaced": 1}, "symbol_lowpass": {"symbol_spaced": 1, "lowpass": 1}}


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True)
    return q.stdout.strip()


def run(rx, iq, calls):
    cap = 4_000_000
    out = torch.empty(cap * 64, dtype=torch.uint8, device="cuda")
    count = torch.zeros(1, dtype=torch.int32, device="cuda")
    d_dir = torch.empty(rx.units(1, N_INT8) * 8, dtype=torch.uint8, device="cuda")
    ways = {}
    for m, kw in MODES.items():
        ways[m] = make_cfgs(1, channel=37, **kw)
        ways[m + "_bank"] = make_cfgs(1, channel=37, offset_search=1, **kw)
    times = {k: [] for k in ways}
    counts = {k: set() for k in ways}
    st = torch.cuda.current_stream().cuda_stream
    names = list(ways)
    for i in range(len(names) * (calls + 2)):
        k = names[i % len(names)]
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        rx.rx_device_dir(iq.view(1, -1), ways[k], out, count, d_dir, st)
        e1.record()
        torch.cuda.synchronize()
        counts[k].add(int(count.item()))
        if i >= 2 * len(names):
            times[k].append(e0.elapsed_time(e1))
    merge = {}
    from torch.profiler import ProfilerActivity, profile
    for m in MODES:
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            rx.rx_device_dir(iq.view(1, -1), ways[m + "_bank"], out, count, d_dir, st)
            torch.cuda.synchronize()
        us = [e.device_time for e in prof.events() if "btle_offset_merge_kernel" in e.name]
        merge[m] = round(sum(us) / 1e3, 4) if us else None
    res = {}
    for k, v in times.items():
        assert len(counts[k]) == 1, (k, counts[k])
        res[k] = {"ms_per_gib": round(float(np.median(v)), 4), "records": counts[k].pop()}
    for m in MODES:
        res[m + "_bank"]["ratio"] = round(res[m + "_bank"]["ms_per_gib"] / res[m]["ms_per_gib"], 3)
        res[m + "_bank"]["merge_ms"] = merge[m]
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=8)
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
