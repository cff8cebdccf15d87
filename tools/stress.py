#!/usr/bin/env python
"""Soak test on the GPU: many random batch shapes against the oracle, and repeated runs of one large
input for run-to-run determinism (any race in the producer/consumer ring would show up here)."""
import os, sys, time
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests"))
import numpy as np, torch
from oracle_flags import expect
from btle_b200 import BtleRx, make_cfgs, synth, REC_DTYPE

rx = BtleRx(0)
rng = np.random.default_rng(int(sys.argv[1]) if len(sys.argv) > 1 else 0)
t0 = time.time()
ncase = 0
while time.time() - t0 < float(os.environ.get("STRESS_SECONDS", "120")):
    n_streams = int(rng.choice([1, 2, 3, 7, 40, 149, 300]))
    nchunks = int(rng.integers(1, max(2, 600 // n_streams)))
    n = nchunks * 16384 + int(rng.integers(0, 16384))
    base, _ = synth.make_adv_stream(n, seed=int(rng.integers(0, 1 << 30)), channel=37, slot_samples=int(rng.choice([1600, 2400, 4096])))
    base = base.numpy()
    iq = np.stack([np.roll(base, 2 * int(rng.integers(0, 3000))) for _ in range(n_streams)])
    flags = int(rng.integers(0, 4))                       # RSSI, -v rejected hits (more of them with the sparse mask)
    mask = int(rng.choice([0xFFFFFFFF, 0x0F000000]))
    cfgs = make_cfgs(n_streams, access_mask=mask, rssi=flags)
    exp = np.concatenate([expect(iq[s], flags, access_mask=mask, stream=s) for s in range(n_streams)])
    got = rx.rx_batch(iq, cfgs)
    assert got.tobytes() == exp.tobytes(), (n_streams, nchunks, len(got), len(exp))
    ncase += 1
print("random shapes ok:", ncase)
iq, _ = synth.make_adv_stream(1 << 28, seed=5, channel=37, device="cuda")
cfgs = make_cfgs(1)
cap = (1 << 28) // 16384 * 3
d_out = torch.empty(cap * 64, dtype=torch.uint8, device="cuda"); d_cnt = torch.zeros(1, dtype=torch.int32, device="cuda")
ref = None
for it in range(300):
    rx.rx_device(iq.view(1, -1), cfgs, d_out, d_cnt, torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    n = int(d_cnt.item())
    r = rx.sort_records(d_out[: n * 64].cpu().numpy().view(REC_DTYPE))
    b = r.tobytes()
    if ref is None: ref = b
    assert b == ref, f"run {it} differs"
print("300 repeated runs identical, packets:", n)
