#!/usr/bin/env python
"""Where does the receive kernel's feed lose HBM bandwidth?  Runs the probe kernels of tools/probe_feed.cu (the receive
kernel's launch shape, tile walk and tensor-map geometry over the c2 capture, with the dense arithmetic or a cheap XOR as
the consumer) next to the receive kernel itself (btle_rx_persistent_kernel of every library given with --rx-lib, e.g. an
A/B build with -DBTLE_CTAS_PER_SM=2) and discover_kernel on the same 1 GiB, in alternation: every round runs every entry
once, each entry is timed with CUDA events around --launches back-to-back launches on one stream.  Prints one line per
entry (median ms per launch over --rounds, HBM bytes / time against the H100 SXM data sheet's 3.35 TB/s) and the card,
its power limit and the SM clock read in the same run.

    python tools/probe_feed.py [--lib libprobe_feed.so] [--rx-lib NAME=PATH ...] [--out FILE]

Without --lib the probe is compiled with nvcc into a temporary directory."""
import argparse
import ctypes
import json
import os
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

HBM_BPS = 3.35e12          # H100 SXM data sheet, HBM3
VARIANTS = ["A", "B", "B2", "C3w12", "C4w8", "C3w16", "Cpf", "D"]
SPAN_BYTES = 16 * 16384    # one unit of the c2 capture
LOOKAHEAD_BYTES = 12 * 256


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return (q.stdout.strip().splitlines() or ["?"])[0]


def build_probe(out_dir):
    lib = os.path.join(out_dir, "libprobe_feed.so")
    subprocess.run([os.environ.get("NVCC", "nvcc"), "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17",
                    "-Xcompiler", "-fPIC", "-shared", "-o", lib, os.path.join(ROOT, "tools", "probe_feed.cu")], check=True)
    return lib


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--lib", default=None, help="prebuilt libprobe_feed.so")
    ap.add_argument("--rx-lib", action="append", default=[], help="NAME=PATH of a libbtle_b200.so to time the receive kernel of")
    ap.add_argument("--rounds", type=int, default=10)
    ap.add_argument("--launches", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()

    import numpy as np
    import torch
    assert torch.cuda.is_available(), "probe_feed needs a CUDA device"
    from btle_b200 import BtleRx, synth
    from btle_b200._native import CFG_DTYPE

    tmp = tempfile.mkdtemp(prefix="probe_feed_")
    P = ctypes.CDLL(args.lib or build_probe(tmp))
    P.probe_feed_launch.argtypes = [ctypes.c_char_p, ctypes.c_int, ctypes.c_void_p, ctypes.c_longlong, ctypes.c_void_p, ctypes.c_int,
                                    ctypes.c_void_p]
    dev = torch.device("cuda", 0)
    sms = torch.cuda.get_device_properties(dev).multi_processor_count
    n_int8 = 1 << 30
    iq, _ = synth.make_adv_stream(n_int8, seed=0x37E15163, channel=37, corrupt_every=100, device=dev)
    iq = iq.view(1, -1)
    sink = torch.empty(sms * 1024, dtype=torch.int32, device=dev)
    st = torch.cuda.current_stream(dev)

    entries = {}
    units = n_int8 // SPAN_BYTES
    for v in VARIANTS:
        for dense in (0, 1):
            def go(v=v, dense=dense):
                rc = P.probe_feed_launch(v.encode(), dense, iq.data_ptr(), n_int8, sink.data_ptr(), sms, ctypes.c_void_p(st.cuda_stream))
                assert rc == 0, (v, rc)
            fetched = units * (SPAN_BYTES + (0 if v == "D" else LOOKAHEAD_BYTES))
            entries[f"probe {v} {'dense' if dense else 'xor'}"] = (go, fetched)
    cfg = np.zeros(1, dtype=CFG_DTYPE)
    cfg[0] = (37, 0x8E89BED6, 0xFFFFFFFF, 0x555555, 0, 0)
    cap = 400000
    outs = torch.empty(cap * 64, dtype=torch.uint8, device=dev)
    cnt = torch.zeros(1, dtype=torch.int32, device=dev)
    vp, sz = ctypes.c_void_p, ctypes.c_size_t
    rx_libs = [("rx", os.path.join(ROOT, "btle_b200", "libbtle_b200.so"))] + [tuple(s.split("=", 1)) for s in args.rx_lib]
    for name, path in rx_libs:
        L = ctypes.CDLL(os.path.abspath(path))
        L.btle_b200_create.argtypes = [ctypes.POINTER(vp), ctypes.c_int]
        L.btle_b200_rx_device.argtypes = [vp, vp, sz, sz, sz, vp, vp, sz, vp, vp]
        h = vp()
        assert L.btle_b200_create(ctypes.byref(h), 0) == 0

        def go(L=L, h=h):
            rc = L.btle_b200_rx_device(h, iq.data_ptr(), 1, n_int8, n_int8, cfg.ctypes.data, outs.data_ptr(), cap, cnt.data_ptr(),
                                       ctypes.c_void_p(st.cuda_stream))
            assert rc == 0, rc
        entries[f"btle_rx_persistent_kernel ({name})"] = (go, units * (SPAN_BYTES + LOOKAHEAD_BYTES))
    rx = BtleRx(0)
    d_cand = torch.empty((n_int8 // 16384 + 1) * 8 * 32 + 8192, dtype=torch.uint8, device=dev)
    d_n = torch.zeros(1, dtype=torch.int32, device=dev)
    entries["discover_kernel"] = (lambda: rx.discover_device(iq, [0], d_cand, d_n, st.cuda_stream), n_int8)

    clocks_before = gpu_info()
    for go, _ in entries.values():
        go()
    torch.cuda.synchronize()
    times = {k: [] for k in entries}
    for _ in range(args.rounds):
        for k, (go, _) in entries.items():
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record(st)
            for _ in range(args.launches):
                go()
            b.record(st)
            b.synchronize()
            times[k].append(a.elapsed_time(b) / args.launches)
    clocks_after = gpu_info()
    rows = []
    print(f"gpu (name, power.limit, clocks.sm, clocks.max.sm): before {clocks_before} | after {clocks_after}")
    print(f"{'entry':40s} {'ms':>7s} {'min':>7s} {'1GiB/ms share':>13s} {'fetched/ms share':>16s}")
    for k, ts in times.items():
        ms = float(np.median(ts))
        fetched = entries[k][1]
        row = {"entry": k, "ms": round(ms, 4), "ms_min": round(float(np.min(ts)), 4),
               "share_algorithmic": round(n_int8 / (ms * 1e-3) / HBM_BPS, 3), "share_fetched": round(fetched / (ms * 1e-3) / HBM_BPS, 3)}
        rows.append(row)
        print(f"{k:40s} {row['ms']:7.4f} {row['ms_min']:7.4f} {row['share_algorithmic']:13.3f} {row['share_fetched']:16.3f}")
    if args.out:
        with open(args.out, "w") as f:
            json.dump({"gpu_before": clocks_before, "gpu_after": clocks_after, "rows": rows}, f, indent=1)


if __name__ == "__main__":
    main()
