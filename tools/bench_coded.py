#!/usr/bin/env python
"""Cost of the LE Coded PHY receiver (btle_b200_rx_coded_device) against the 1M receive launch (btle_b200_rx_device).
  Three 1 GiB inputs: a c2-like 1M capture (channel 37, 1 % corrupted bursts, straddling packets), full-scale random IQ
  (bench.py's hot input), and a capture dense with coded bursts (S=2 and S=8, 0..255-byte PDUs, back to back at 10 dB).
  Calls alternate, CUDA events around each call, median of --calls each.  Prints the time per GiB and the record count of
  each way, which must not change from call to call.  One JSON line per input with the card's name and power limit read in
  the same run.  --ab-lib PATH adds that build's rx_coded_device to the same alternation ("rx_coded_device_ab").
  Several cfgs per capture ("what": "multi"): on the c2 and coded_dense captures, one rx_coded_multi_device call with k =
  1, 2, 4, 8 cfgs on the capture against k rx_coded_device calls on it, one cfg each, alternating; the marginal cost of a
  cfg is (t(k) - t(1)) / (k - 1) of the multi call.  "conn" is the decode_connections shape: 37 captures of 64 MiB
  (coded_dense rows) with 8 cfgs each in one call, against 8 rx_coded_device calls over the 37 captures.
  python tools/bench_coded.py [--calls 12] [--ab-lib other/libbtle_b200.so]"""
import argparse
import ctypes
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


class OtherBuild:
    """btle_b200_rx_coded_device of another build of the library, loaded beside this one"""

    def __init__(self, path):
        self.L = ctypes.CDLL(os.path.abspath(path))
        vp, sz = ctypes.c_void_p, ctypes.c_size_t
        self.L.btle_b200_create.argtypes = [ctypes.POINTER(vp), ctypes.c_int]
        self.L.btle_b200_rx_coded_device.argtypes = [vp, vp, sz, sz, sz, vp, vp, vp, sz, vp, vp]
        self.h = vp()
        assert self.L.btle_b200_create(ctypes.byref(self.h), 0) == 0

    def rx_coded_device(self, d_iq, cfgs, d_out, d_count, st):
        ns, n = d_iq.shape
        cap = d_out.numel() // 304
        assert self.L.btle_b200_rx_coded_device(self.h, d_iq.data_ptr(), ns, d_iq.stride(0), n, cfgs.ctypes.data, None, d_out.data_ptr(), cap,
                                                d_count.data_ptr(), ctypes.c_void_p(st)) == 0


def alternate(ways, calls):
    """ways: name -> (call, count tensor); each call once per round, CUDA events around it; medians in ms"""
    times = {k: [] for k in ways}
    counts = {k: set() for k in ways}
    names = list(ways)
    for i in range(len(names) * (calls + 2)):
        k = names[i % len(names)]
        call, count = ways[k]
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        call()
        e1.record()
        torch.cuda.synchronize()
        counts[k].add(int(count.sum().item()))
        if i >= 2 * len(names):
            times[k].append(e0.elapsed_time(e1))
    res = {}
    for k, v in times.items():
        assert len(counts[k]) == 1, (k, counts[k])
        res[k] = {"ms": round(float(np.median(v)), 4), "spread_ms": round(float(np.max(v) - np.min(v)), 4), "records": counts[k].pop()}
    return res


def run(rx, iq, calls, other=None):
    cap1, capc = 2_000_000, 400_000
    out1 = torch.empty(cap1 * 64, dtype=torch.uint8, device="cuda")
    outc = torch.empty(capc * 304, dtype=torch.uint8, device="cuda")
    count = torch.zeros(1, dtype=torch.int32, device="cuda")
    cfg1, cfgc = make_cfgs(1, channel=37), make_cfgs(1, channel=37)
    st = torch.cuda.current_stream().cuda_stream
    ways = {"rx_device": (lambda: rx.rx_device(iq.view(1, -1), cfg1, out1, count, st), count),
            "rx_coded_device": (lambda: rx.rx_coded_device(iq.view(1, -1), cfgc, outc, count, st), count)}
    if other is not None:
        ways["rx_coded_device_ab"] = (lambda: other.rx_coded_device(iq.view(1, -1), cfgc, outc, count, st), count)
    res = alternate(ways, calls)
    for v in res.values():
        v["ms_per_gib"] = v.pop("ms")
    return res


def cfg_list(k):
    """k cfgs on channel 37: the advertising access address (the coded_dense bursts'), then others"""
    rng = np.random.default_rng(k)
    return make_cfgs(k, channel=37, access_addr=[0x8E89BED6] + [int(a) for a in rng.integers(0, 1 << 32, k - 1)])


def run_multi(rx, iq, calls):
    """one rx_coded_multi_device call with k cfgs on the capture against k rx_coded_device calls, k = 1, 2, 4, 8"""
    capc = 400_000
    d_iq = iq.view(1, -1)
    st = torch.cuda.current_stream().cuda_stream
    out = torch.empty(capc * 304, dtype=torch.uint8, device="cuda")
    res = {}
    for k in (1, 2, 4, 8):
        cfgs = cfg_list(k)
        cnt_m = torch.zeros(1, dtype=torch.int32, device="cuda")
        cnt_s = torch.zeros(k, dtype=torch.int32, device="cuda")
        outs = [torch.empty(capc * 304 // k // 16 * 16, dtype=torch.uint8, device="cuda") for _ in range(k)]

        def separate():
            for j in range(k):
                rx.rx_coded_device(d_iq, cfgs[j:j + 1], outs[j], cnt_s[j:j + 1], st)
        r = alternate({"multi": (lambda: rx.rx_coded_multi_device(d_iq, cfgs, np.zeros(k, np.int32), out, cnt_m, st), cnt_m),
                       "separate": (separate, cnt_s)}, calls)
        assert r["multi"]["records"] == r["separate"]["records"], r
        res[k] = r
    t1 = res[1]["multi"]["ms"]
    return {"k": {k: {"multi_ms": v["multi"]["ms"], "multi_spread_ms": v["multi"]["spread_ms"], "separate_ms": v["separate"]["ms"],
                      "separate_spread_ms": v["separate"]["spread_ms"], "records": v["multi"]["records"],
                      "marginal_ms_per_cfg": round((v["multi"]["ms"] - t1) / (k - 1), 4) if k > 1 else None}
                  for k, v in res.items()}}


def run_conn(rx, dense, calls):
    """37 captures x 64 MiB x 8 cfgs in one call against 8 single-cfg calls over the 37 captures"""
    rows = dense[:16 << 26].view(16, 1 << 26)
    caps = torch.cat([rows, rows, rows[:5]])
    st = torch.cuda.current_stream().cuda_stream
    k, capc = 8, 1_000_000
    cfgs = make_cfgs(37 * k, channel=np.repeat(np.arange(37), k), access_addr=[int(c["access_addr"]) for c in cfg_list(k)] * 37)
    capture = np.repeat(np.arange(37, dtype=np.int32), k)
    out = torch.empty(capc * 304, dtype=torch.uint8, device="cuda")
    outs = [torch.empty(capc // k * 304, dtype=torch.uint8, device="cuda") for _ in range(k)]
    cnt_m = torch.zeros(1, dtype=torch.int32, device="cuda")
    cnt_s = torch.zeros(k, dtype=torch.int32, device="cuda")

    def separate():
        for i in range(k):
            rx.rx_coded_device(caps, cfgs[i::k], outs[i], cnt_s[i:i + 1], st)
    r = alternate({"multi": (lambda: rx.rx_coded_multi_device(caps, cfgs, capture, out, cnt_m, st), cnt_m),
                   "separate": (separate, cnt_s)}, calls)
    assert r["multi"]["records"] == r["separate"]["records"], r
    return r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=12)
    ap.add_argument("--ab-lib", default=None)
    a = ap.parse_args()
    rx = BtleRx(0)
    other = OtherBuild(a.ab_lib) if a.ab_lib else None
    name = card()
    dev = torch.device("cuda", 0)
    iq, _ = synth.make_adv_stream(N_INT8, seed=0x37E15163, channel=37, corrupt_every=100, device=dev, use_cuda_modulator=False,
                                  straddle_every=100)
    print(json.dumps({"what": "time", "input": "c2", "card": name, "calls": a.calls, **run(rx, iq, a.calls, other)}), flush=True)
    print(json.dumps({"what": "multi", "input": "c2", "card": name, "calls": a.calls, **run_multi(rx, iq, a.calls)}), flush=True)
    del iq
    g = torch.Generator(device=dev)
    g.manual_seed(5)
    hot = torch.randint(-128, 128, (N_INT8,), generator=g, device=dev, dtype=torch.int8)
    print(json.dumps({"what": "time", "input": "hot", "card": name, "calls": a.calls, **run(rx, hot, a.calls, other)}), flush=True)
    del hot
    dense, n = coded_capture(dev)
    print(json.dumps({"what": "time", "input": "coded_dense", "bursts": n, "card": name, "calls": a.calls, **run(rx, dense, a.calls, other)}),
          flush=True)
    print(json.dumps({"what": "multi", "input": "coded_dense", "bursts": n, "card": name, "calls": a.calls, **run_multi(rx, dense, a.calls)}),
          flush=True)
    print(json.dumps({"what": "conn", "input": "37 x 64 MiB coded_dense rows, 8 cfgs each", "card": name, "calls": a.calls,
                      **run_conn(rx, dense, a.calls)}), flush=True)


if __name__ == "__main__":
    main()
