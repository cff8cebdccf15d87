#!/usr/bin/env python
"""Live connection decoding (hop.ConnectionMonitor over btle_b200_streams_*) against the plain session and the offline
hop.decode_connections() on the same 40 captures.

40 captures of --mib MiB (row c = BLE channel c, bursts from synth_streams_device with the c3 channel plan, plus the
connections of tests' connections_capture() over the first 100 chunks: a CONNECT_REQ connection and two found by
discovery; the data captures' own bursts may add discovered connections), in page-locked host memory.  Host clock around work that ends in a synchronise, after a warm-up:
  (a) plain session: the 40 base cfgs, no discovery (BtleRx.streams, --seg chunks per set);
  (b) the monitor on the same session layout: advertising cfgs, discovery on 0..36, 37 cfgs per connection, backfill;
  (c) offline decode_connections() on the whole captures.
Reports G samples/s of each, and for (b) the GPU kernel time per set (torch.profiler, CUDA activities, in a run of its
own) against the set's air time (seg * 8192 samples at 4 Msps), plus whether the records are identical: (a) equals
rx_batch, (b)'s connection list equals (c)'s and each connection's traffic equals (c)'s from its from_chunk on.  One
JSON line with the GPU name and power limit; --out FILE also writes it there."""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np
import torch

CHUNK = 16384
KEYS = ("access_addr", "crc_init", "tracked", "interval", "hop", "t_first", "first_channel", "n_events")


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    name, power = (q.stdout.strip().splitlines() or ["?, ?"])[0].split(", ")[:2]
    return name, power


def timed(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    r = fn()
    torch.cuda.synchronize()
    return r, time.perf_counter() - t0


def feed(target, host, step):
    """Every capture's bytes, one set part per capture in turn; returns the records handed out."""
    parts = []
    for pos in range(0, host.shape[1], step):
        for i in range(host.shape[0]):
            parts.append(target.push(i, host[i, pos:pos + step]))
    parts.append(target.finish())
    return np.concatenate(parts)


def captures(n_int8, seed):
    from btle_b200 import synth
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    from test_rx_multi import connections_capture
    d_iq, _ = synth.synth_streams_device(synth.channel_plan(40), n_int8, seed=seed, amplitude=40, want_truth=False)
    host = torch.empty((40, n_int8), dtype=torch.int8, pin_memory=True)
    host.copy_(d_iq)
    del d_iq
    torch.cuda.synchronize()
    h = host.numpy()
    conn, _ = connections_capture()                            # 100 chunks with three connections, added on top of the bursts
    m = min(conn.shape[1], n_int8)
    np.copyto(h[:, :m], np.clip(h[:, :m].astype(np.int16) + conn[:, :m], -128, 127).astype(np.int8))
    return host, h


def kernel_ms(fn):
    """Summed device time of the project's kernels while fn() runs (torch.profiler, CUDA activities)."""
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    tot = 0.0
    for e in prof.key_averages():
        if "kernel" in e.key and ("btle" in e.key or "discover" in e.key):
            tot += getattr(e, "device_time_total", getattr(e, "cuda_time_total", 0.0))
    return tot / 1e3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--mib", type=int, default=64, help="MiB per capture")
    ap.add_argument("--seg", type=int, default=16, help="chunks per segment set")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_conn_stream needs a CUDA device"
    from btle_b200 import BtleRx, make_cfgs
    from btle_b200._native import bind_host_numa
    from btle_b200.hop import ConnectionMonitor, decode_connections
    name, power = gpu_info()
    bind_host_numa(0)
    rx = BtleRx(0)
    n_int8 = max(args.mib, 5) << 20
    host, h = captures(n_int8, seed=7)
    cfgs = make_cfgs(40, channel=list(range(40)))
    step = args.seg * CHUNK

    def plain(x):
        with rx.streams(cfgs, segment_chunks=args.seg) as s_:
            return timed(lambda: feed(s_, x, step))

    def monitor(x):
        with rx.streams(cfgs, segment_chunks=args.seg) as s_:
            mon = ConnectionMonitor(s_)
            _, t = timed(lambda: feed(mon, x, step))
            return mon, t

    warm = 300 * CHUNK
    plain(h[:, :warm]); monitor(h[:, :warm]); decode_connections(rx, h[:, :warm])
    a, t_a = plain(h)
    a = a[np.lexsort((a["chunk"], a["stream"]))]
    same_a = a.tobytes() == rx.rx_batch(h, cfgs).tobytes()
    mon, t_b = monitor(h)
    (adv, offline), t_c = timed(lambda: decode_connections(rx, h))
    live = mon.connections()
    same_b = len(live) == len(offline) and all(
        {k: x.get(k) for k in KEYS} == {k: y.get(k) for k in KEYS}
        and x["traffic"].tobytes() == y["traffic"][y["traffic"]["chunk"] >= x["from_chunk"]].tobytes() for x, y in zip(live, offline))
    ms = kernel_ms(lambda: monitor(h))
    n_sets = -(-(n_int8 // CHUNK) // args.seg)
    samples = 40 * n_int8 / 2
    row = {"gpu": name, "power_limit": power, "captures": 40, "mib_per_capture": round(n_int8 / 2**20, 1), "segment_chunks": args.seg,
           "connections": len(live), "cfgs": len(mon._owner) + 3, "plain_identical_to_rx_batch": bool(same_a),
           "monitor_identical_to_offline": bool(same_b),
           "monitor_gpu_ms_per_set": round(ms / n_sets, 3), "set_air_ms": round(args.seg * 8192 / 4e3, 3)}
    for key, t in (("plain_session", t_a), ("monitor", t_b), ("offline_decode_connections", t_c)):
        row[key] = {"seconds": round(t, 4), "gsamples_per_s": round(samples / t / 1e9, 3)}
    line = json.dumps(row)
    print(line, flush=True)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")
    assert same_a and same_b, "records differ"


if __name__ == "__main__":
    main()
