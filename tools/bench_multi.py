"""Several access addresses per capture: one btle_b200_rx_multi launch against K single-cfg launches.

    python tools/bench_multi.py [--mib 256] [--iters 20] [--warmup 3] [--ks 1,2,4,8] [--out FILE]

Input: 37 data-channel captures x `--mib` MiB from synth_streams_device with the c3 channel plan (bench.py), capture c
carrying bursts of its own access address.  For every K, capture c is decoded with K cfgs: its own access address plus
K - 1 others (those of captures c + 1 .. c + K - 1).  Timed with CUDA events, in one process, alternating per iteration:
  (a) multi   one rx_multi_device_dir call over the 37 captures with 37 K cfgs;
  (b) single  K rx_device_dir calls, call k with cfg k of every capture;
  (c) plain   (K = 1 only) the plain rx_device_dir call, i.e. what bench.py's c3 row runs on 37 captures.
Medians of `--iters` calls after `--warmup`.  The records of (a) and (b) are compared after gather_ordered, with (b)'s
`stream` mapped to the cfg index.  The GPU name, power limit and SM clock are recorded before and after.  Prints one JSON
line (and writes it to --out)."""
import argparse
import json
import os
import statistics
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from btle_b200 import BtleRx, synth  # noqa: E402
from btle_b200._native import DIR_DTYPE, REC_DTYPE  # noqa: E402


def gpu_state():
    q = "name,power.limit,clocks.sm,clocks.max.sm,temperature.gpu"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True,
                             timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        out = ""
    return dict(zip(q.split(","), [x.strip() for x in out.split(",")])) if out else {"name": torch.cuda.get_device_name(0)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--mib", type=int, default=256)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--ks", default="1,2,4,8")
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    ks = [int(k) for k in a.ks.split(",")]
    before = gpu_state()
    rx = BtleRx(0)
    n = a.mib << 20
    plan = synth.channel_plan(40)[:37]
    d_iq, _ = synth.synth_streams_device(plan, n, seed=1000, want_truth=False)
    torch.cuda.synchronize()
    st = torch.cuda.current_stream().cuda_stream
    cap = 37 * (n // 16384) * 4 + 4096
    d_out_a = torch.empty(cap * 64, dtype=torch.uint8, device="cuda")
    d_outs_b = [torch.empty(cap * 64, dtype=torch.uint8, device="cuda") for _ in range(max(ks))]
    rows = []

    def timed(fn):
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        fn()
        e.record()
        e.synchronize()
        return s.elapsed_time(e)

    for K in ks:
        capture = np.repeat(np.arange(37, dtype=np.int32), K)
        cfgs = np.concatenate([plan[[(c + k) % 37 for k in range(K)]] for c in range(37)])
        cfgs["channel"] = np.repeat(plan["channel"], K)
        sets = [cfgs[np.arange(37) * K + k] for k in range(K)]
        d_dir_a = torch.empty(max(rx.multi_units(37, capture, n), 1) * 8, dtype=torch.uint8, device="cuda")
        units = rx.units(37, n)
        d_dirs_b = [torch.empty(units * 8, dtype=torch.uint8, device="cuda") for _ in range(K)]
        run_a = lambda: rx.rx_multi_device_dir(d_iq, cfgs, capture, d_out_a, None, d_dir_a, st)

        def run_b():
            for k in range(K):
                rx.rx_device_dir(d_iq, sets[k], d_outs_b[k], None, d_dirs_b[k], st)

        ta, tb, tc = [], [], []
        for i in range(a.warmup + a.iters):
            x, y = timed(run_a), timed(run_b)
            z = timed(lambda: rx.rx_device_dir(d_iq, sets[0], d_outs_b[0], None, d_dirs_b[0], st)) if K == 1 else None
            if i >= a.warmup:
                ta.append(x); tb.append(y)
                if z is not None:
                    tc.append(z)
        # outputs: (a) == (b) with stream -> cfg index
        run_a(); run_b(); torch.cuda.synchronize()
        got = rx.gather_ordered(d_out_a.cpu().numpy().view(REC_DTYPE), d_dir_a.cpu().numpy().view(DIR_DTYPE))
        parts = []
        for k in range(K):
            r = rx.gather_ordered(d_outs_b[k].cpu().numpy().view(REC_DTYPE), d_dirs_b[k].cpu().numpy().view(DIR_DTYPE)).copy()
            r["stream"] = r["stream"] * K + k
            parts.append(r)
        exp = np.concatenate(parts)
        exp = exp[np.argsort(exp["stream"], kind="stable")]
        gib = 37 * n / 2**30
        row = {"K": K, "multi_ms": round(statistics.median(ta), 3), "single_x_k_ms": round(statistics.median(tb), 3),
               "multi_gib_s": round(gib / (statistics.median(ta) / 1e3), 1), "records": int(len(got)), "equal": bool(got.tobytes() == exp.tobytes())}
        if tc:
            row["plain_ms"] = round(statistics.median(tc), 3)
        rows.append(row)
        print(json.dumps(row), file=sys.stderr, flush=True)
    res = {"tool": "bench_multi", "captures": 37, "mib_per_capture": a.mib, "iters": a.iters, "rows": rows,
           "gpu_before": before, "gpu_after": gpu_state()}
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")
    if not all(r["equal"] for r in rows):
        sys.exit(1)


if __name__ == "__main__":
    main()
