#!/usr/bin/env python
"""Cost of LE Coded PHY connection discovery (btle_b200_discover_coded_device) next to the coded receiver
(btle_b200_rx_coded_device) on the same 1 GiB captures: c2-like 1M input, full-scale random IQ (bench.py's hot input) and
a capture dense with coded bursts (tools/bench_coded.py's three inputs).  Calls alternate, CUDA events around each
call, median of --calls each; the candidate and record counts must not change from call to call.  One JSON line per
input with the card's name and power limit read in the same run.
  python tools/bench_coded_discover.py [--calls 12]"""
import argparse
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import torch

from bench_coded import N_INT8, alternate, card, coded_capture
from btle_b200 import BtleRx, make_cfgs, synth


def run(rx, iq, calls):
    capd, capc = 400_000, 400_000
    outd = torch.empty(capd * 32, dtype=torch.uint8, device="cuda")
    outc = torch.empty(capc * 304, dtype=torch.uint8, device="cuda")
    cd, cc = torch.zeros(1, dtype=torch.int32, device="cuda"), torch.zeros(1, dtype=torch.int32, device="cuda")
    cfgc = make_cfgs(1, channel=37)
    st = torch.cuda.current_stream().cuda_stream
    ways = {"discover_coded_device": (lambda: rx.discover_coded_device(iq.view(1, -1), [5], outd, cd, st), cd),
            "rx_coded_device": (lambda: rx.rx_coded_device(iq.view(1, -1), cfgc, outc, cc, st), cc)}
    res = alternate(ways, calls)
    for v in res.values():
        v["ms_per_gib"] = v.pop("ms")
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
    print(json.dumps({"input": "c2", "card": name, "calls": a.calls, **run(rx, iq, a.calls)}), flush=True)
    del iq
    g = torch.Generator(device=dev)
    g.manual_seed(5)
    hot = torch.randint(-128, 128, (N_INT8,), generator=g, device=dev, dtype=torch.int8)
    print(json.dumps({"input": "hot", "card": name, "calls": a.calls, **run(rx, hot, a.calls)}), flush=True)
    del hot
    dense, n = coded_capture(dev)
    print(json.dumps({"input": "coded_dense", "bursts": n, "card": name, "calls": a.calls, **run(rx, dense, a.calls)}), flush=True)


if __name__ == "__main__":
    main()
