#!/usr/bin/env python
"""Throughput of the multi-capture streaming session (btle_b200_streams_*) against one btle_b200_rx_batch() call.

For N in --streams (default 1, 3, 40) captures of --mib MiB each (c3-style: stream k on BLE channel k mod 40, bursts from
synth_streams_device, copied into page-locked host memory), times with a host clock around work that ends in a
synchronise, after a warm-up:
  (a) the captures pushed through BtleRx.streams() with the default segment, one segment part per capture in turn (the
      session is opened before the clock starts; push() copies every byte once into its page-locked buffers);
  (b) the same with segment_chunks=16 (the low-latency setting);
  (c) one rx_batch() call on the same page-locked data.
Checks that (a), (b) and (c) return identical records and prints one JSON line per N with G samples/s and records/s,
the host's single-thread copy rate between page-locked buffers (host_copy_gbs, what (a) and (b) pay on top of (c)),
plus the GPU name and power limit.  --out FILE also writes the lines there."""
import argparse
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import numpy as np
import torch

CHUNK = 16384


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    name, power = (q.stdout.strip().splitlines() or ["?, ?"])[0].split(", ")[:2]
    return name, power


def push_all(s_, host, n_int8, step):
    """Every capture's bytes through an open session, one segment part per capture in turn; returns the records in
    (stream, chunk) order."""
    parts = []
    for pos in range(0, n_int8, step):
        for i in range(host.shape[0]):
            parts.append(s_.push(i, host[i, pos:pos + step]))
    parts.append(s_.finish())
    got = np.concatenate(parts)
    return got[np.lexsort((got["chunk"], got["stream"]))]


def session_run(rx, cfgs, host, n_int8, seg):
    """(records, seconds): the session is opened (page-locked buffers allocated) before the clock starts."""
    ns = host.shape[0]
    eff = seg or max(16, (4096 // ns + 15) // 16 * 16)
    with rx.streams(cfgs, segment_chunks=seg) as s_:
        return timed(lambda: push_all(s_, host, n_int8, eff * CHUNK))


def timed(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    r = fn()
    torch.cuda.synchronize()
    return r, time.perf_counter() - t0


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--streams", type=int, nargs="+", default=[1, 3, 40])
    ap.add_argument("--mib", type=int, default=256, help="MiB per capture")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_streams needs a CUDA device"
    from btle_b200 import BtleRx, synth
    from btle_b200._native import bind_host_numa
    name, power = gpu_info()
    node = bind_host_numa(0)                                      # page-locked buffers and this thread next to the GPU (as bench.py's e2e)
    rx = BtleRx(0)
    n_int8 = args.mib << 20
    lines = []
    for ns in args.streams:
        cfgs = synth.channel_plan(ns)
        d_iq, _ = synth.synth_streams_device(cfgs, n_int8, seed=7, want_truth=False)      # c3 parameters: 4096-sample slots, 1 % corrupt / straddling
        host = torch.empty((ns, n_int8), dtype=torch.int8, pin_memory=True)
        host.copy_(d_iq)
        del d_iq
        torch.cuda.synchronize()
        torch.cuda.empty_cache()
        h = host.numpy()
        warm = 64 * CHUNK + 5000                                  # warm-up: every entry point on a short prefix
        session_run(rx, cfgs, h[:, :warm], warm, 0)
        session_run(rx, cfgs, h[:, :warm], warm, 16)
        rx.rx_batch(h[:, :warm], cfgs)
        c, t_c = timed(lambda: rx.rx_batch(h, cfgs))
        a, t_a = session_run(rx, cfgs, h, n_int8, 0)
        b, t_b = session_run(rx, cfgs, h, n_int8, 16)
        same = a.tobytes() == c.tobytes() and b.tobytes() == c.tobytes()
        # what a producer pays to put the bytes into the session's page-locked buffers: one host copy of every byte
        dst = torch.empty(n_int8, dtype=torch.int8, pin_memory=True).numpy()
        _, t_m = timed(lambda: [np.copyto(dst, h[i]) for i in range(ns)])
        del dst
        samples = ns * n_int8 / 2
        row = {"n_streams": ns, "mib_per_stream": args.mib, "records": int(len(c)), "identical": bool(same),
               "gpu": name, "power_limit": power, "numa_node": node, "host_copy_gbs": round(ns * n_int8 / t_m / 1e9, 2)}
        for key, t in (("streams_default", t_a), ("streams_seg16", t_b), ("rx_batch", t_c)):
            row[key] = {"seconds": round(t, 4), "gsamples_per_s": round(samples / t / 1e9, 3), "records_per_s": round(len(c) / t, 1)}
        lines.append(json.dumps(row))
        print(lines[-1], flush=True)
        del host, h
        assert same, "session records differ from rx_batch"
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
