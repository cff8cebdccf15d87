#!/usr/bin/env python
"""GPU fuzz of the multi-cfg receive path against the oracle run once per cfg: random launches of tests/multi_fuzz.py
(1..40 captures, 0..8 cfgs each, random channels / access addresses / masks / CRC inits / raw / flags, five input kinds)
through btle_b200_rx_multi (host), or btle_b200_rx_multi_device_dir with a counter or with the context's counter ring,
gathered through the unit directory.  FUZZ_SECONDS (default 120), seed argv[1].  --mode ROT,SYM (default 0,0): 1,0
corrects a random carrier offset per capture (the captures rotated onto it), 0,1 decodes symbol-spaced, 1,1 both; the
records are then compared with tests/mode_ref.py's restatement instead of the oracle."""
import argparse, os, sys, time
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))
import numpy as np
from btle_b200 import BtleRx
from multi_fuzz import draw
from test_rx_multi import oracle_multi
from test_rx_multi_gpu import device_multi, gathered, to_device

ap = argparse.ArgumentParser()
ap.add_argument("seed", nargs="?", type=int, default=0)
ap.add_argument("--mode", default="0,0", choices=["0,0", "1,0", "0,1", "1,1"])
args = ap.parse_args()
mode = tuple(int(v) for v in args.mode.split(","))
if mode != (0, 0):
    import mode_ref
    from multi_fuzz import draw_mode
rx = BtleRx(0)
rng = np.random.default_rng(args.seed)
t0, n_launch, n_rec, paths = time.time(), 0, 0, {"host": 0, "count": 0, "ring": 0}
while time.time() - t0 < float(os.environ.get("FUZZ_SECONDS", "120")):
    if mode == (0, 0):
        iq, cfgs, capture = draw(rng)
        offsets, exp = None, oracle_multi(iq, cfgs, capture)
    else:
        iq, cfgs, capture, offsets = draw_mode(rng, mode)
        exp = mode_ref.rx_multi(iq, cfgs, capture, offsets)
    corr = {} if offsets is None else {"offset_hz": offsets}
    path = ("host", "count", "ring")[int(rng.integers(0, 3))]
    if path == "host":
        got = rx.rx_multi(iq, cfgs, capture, **corr)
    else:
        d_out, d_dir, d_count = device_multi(rx, to_device(iq), cfgs, capture, with_count=path == "count", **corr)
        got = gathered(rx, d_out, d_dir)
        if d_count is not None:
            assert int(d_count.item()) == len(exp), ("counter != oracle", int(d_count.item()), len(exp))
    assert got.tobytes() == exp.tobytes(), ("GPU != oracle", path, iq.shape, cfgs.tolist(), capture.tolist(), len(got), len(exp))
    n_launch += 1; n_rec += len(exp); paths[path] += 1
print(f"gpu multi fuzz (mode {args.mode}) ok: {n_launch} launches ({paths}), {n_rec} records compared bit for bit")
