#!/usr/bin/env python
"""GPU fuzz: the CUDA path through the C-ABI vs the oracle on random access addresses / masks / channels /
CRC inits / raw mode / flags (RSSI, rejected hits) and a mix of input kinds, several captures per batch.  FUZZ_SECONDS (default 120)."""
import os, sys, time
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))
import numpy as np
from oracle_flags import expect
from btle_b200 import BtleRx, CFG_DTYPE, synth

rx = BtleRx(0)
rng = np.random.default_rng(int(sys.argv[1]) if len(sys.argv) > 1 else 0)
t0, n_case, n_pkt = time.time(), 0, 0
while time.time() - t0 < float(os.environ.get("FUZZ_SECONDS", "120")):
    ns = int(rng.choice([1, 2, 5, 33]))
    nchunks = int(rng.integers(1, 40))
    n = nchunks * 16384 + int(rng.choice([0, 1, 2, 255, 256, 3007, 3008, 3009, int(rng.integers(0, 16384))]))
    iq = np.empty((ns, n), dtype=np.int8)
    cfgs = np.zeros(ns, dtype=CFG_DTYPE)
    for s in range(ns):
        kind = int(rng.integers(0, 5))
        ch = int(rng.integers(0, 40))
        aa = int(rng.integers(0, 1 << 32))
        crc_init = int(rng.integers(0, 1 << 24))
        pop = int(rng.choice([0, 1, 2, 4, 8, 12, 16, 24, 32]))
        mask = 0
        for p in rng.permutation(32)[:pop]:
            mask |= 1 << int(p)
        if kind == 0:
            iq[s] = rng.integers(-128, 128, n, dtype=np.int8)
        elif kind == 1:
            iq[s] = rng.integers(-1, 2, n, dtype=np.int8)
        elif kind in (2, 3):
            t, _ = synth.make_adv_stream(n, seed=int(rng.integers(0, 1 << 30)), channel=ch, access_addr=aa, crc_init=crc_init,
                                         corrupt_every=int(rng.choice([0, 3, 50])), slot_samples=int(rng.choice([1500, 2048, 3000, 4096])),
                                         data_channel_pdu=ch < 37, straddle_every=int(rng.choice([0, 2, 5])))
            iq[s] = t.numpy()
            mask = 0xFFFFFFFF if rng.integers(0, 2) else (mask | 0xFF)
            if kind == 3:
                for _ in range(8):
                    a = int(rng.integers(0, max(1, n - 4000)))
                    iq[s, a:a + 4000] = rng.integers(-128, 128, min(4000, n - a), dtype=np.int8)
        else:
            period = int(rng.choice([2, 4, 6, 8, 16, 64]))
            iq[s] = np.resize(rng.integers(-100, 101, period, dtype=np.int8), n)
        cfgs[s] = (ch, aa, mask, crc_init, int(rng.integers(0, 4) == 0), int(rng.integers(0, 4)))   # flags: RSSI, -v rejected hits
    exp = np.concatenate([expect(iq[s], int(cfgs[s]["rssi"]), channel=int(cfgs[s]["channel"]), access_addr=int(cfgs[s]["access_addr"]),
                                       access_mask=int(cfgs[s]["access_mask"]), crc_init=int(cfgs[s]["crc_init"]),
                                       raw=int(cfgs[s]["raw"]), stream=s) for s in range(ns)])
    got = rx.rx_batch(iq, cfgs)
    assert got.tobytes() == exp.tobytes(), ("GPU != oracle", ns, n, cfgs.tolist(), len(got), len(exp))
    n_case += 1; n_pkt += len(exp)
print(f"gpu fuzz ok: {n_case} batches, {n_pkt} packets compared bit for bit")
