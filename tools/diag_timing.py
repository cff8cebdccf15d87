import ctypes, os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np, torch
from btle_b200 import BtleRx, make_cfgs, synth, _native
dev = torch.device("cuda", 0)
iq, _ = synth.make_adv_stream(1 << 30, seed=7, channel=37, corrupt_every=100, device=dev)
rx = BtleRx(0)
L = _native.load()
L.btle_b200_debug_timing.argtypes = [ctypes.c_void_p, ctypes.c_int]
cfgs = make_cfgs(1)
d_out = torch.empty(400000 * 64, dtype=torch.uint8, device=dev); d_cnt = torch.zeros(1, dtype=torch.int32, device=dev)
st = torch.cuda.current_stream()
FULL = (1 << 30) / (16 * 16384 * 132)      # spans per CTA of a 1 GiB capture: 4096 spans over 132 CTAs
DENSE, RESOLVE = 16, 3                     # dense and resolver warps per CTA (the default launch shape)
for spans in (4, FULL):
    n_int8 = int(round(spans * 132)) * 16 * 16384
    v = iq[:n_int8].view(1, -1)
    for _ in range(3): rx.rx_device(v, cfgs, d_out, d_cnt, st.cuda_stream)
    torch.cuda.synchronize()
    L.btle_b200_debug_timing(None, 1)
    rx.rx_device(v, cfgs, d_out, d_cnt, st.cuda_stream)
    torch.cuda.synchronize()
    t = np.zeros(132 * 16, dtype=np.uint64)
    L.btle_b200_debug_timing(t.ctypes.data, 0)
    t = t.reshape(132, 16).astype(np.int64)
    t0 = t[:, 0].min()
    rel = (t - t0) / 1000.0
    names = ["start", "init_done", "first_tile", "dense_done", "resolver_last_begin", "resolver_end", "last_fixup_done", "last_chain_done",
             "last_reserve_issued", "last_decode_done", "first_tma_issued", "params_built"]
    print(f"spans/CTA {spans}: (us, median over CTAs / max)")
    for i, nm in enumerate(names):
        print(f"   {nm:22s} {np.median(rel[:, i]):8.1f} {rel[:, i].max():8.1f}")
    # cumulative wait cycles (slots 12..15), per warp, as a share of a dense warp's cycles from start-up to its last unit
    dense_total = t[:, 15].sum() / DENSE
    print(f"   dense warp: TMA mbar_wait {t[:, 12].sum() / DENSE / dense_total:6.1%}, empty-slot wait "
          f"{t[:, 13].sum() / DENSE / dense_total:6.1%};  resolver warp: idle on full {t[:, 14].sum() / RESOLVE / dense_total:6.1%}"
          f"  (of {dense_total / 132:.0f} cycles per dense warp)")
