"""PER / BER of the reference's 4-Msps int8 receiver (btle_b200_rx_ber_run) next to the Python model's 8-sps receiver
(btle_b200_ber_run) at the same SNR and ppm, plus the 4-Msps receiver under extra carrier offsets, and where the time of
rx_ber_run goes (CUDA events around its three kernels on one batch).

    python tools/rx_ber_report.py [--packets N] [--json out.json] [--recover] [--symbol-spaced] [--centre-hits] [--correct]
                                  [--lowpass] [--offset-search] [--mixed-cfo] [--snrs 8:31] [--no-cfo]

--recover adds the 4-sps PER / BER with BTLE_CFG_RECOVER (CRC-failed packets demodulated again) next to the plain ones.
--symbol-spaced adds them with BTLE_CFG_SYMBOL_SPACED (the symbol-spaced discriminator), and with --recover also with both.
--centre-hits adds, next to each of those, the same receiver with BTLE_CFG_CENTRE_HITS (each hit centred on its run of
matching sample phases), and prints the SNR at PER 0.5 and the error breakdown of every 4-sps variant per ppm.
--correct adds, next to the plain receiver and each of those, the same receiver with BTLE_CFG_CORRECT (one-bit and
adjacent-pair errors of CRC-failed packets corrected from the syndrome), and prints the same breakdown.
--lowpass adds, next to each symbol-spaced variant, the same receiver with BTLE_CFG_LOWPASS (the symbol-spaced bits read
[1, 2, 1]-filtered samples), and prints the same breakdown.
--offset-search adds, next to the plain receiver and each of those, the same receiver with BTLE_CFG_OFFSET_SEARCH (seven
carrier-offset hypotheses, merged per packet), and prints the same breakdown.
--mixed-cfo adds rows of one capture whose slots alternate between five carrier offsets (-120, -60, 0, +60, +120 kHz):
rx_ber_synth_device runs at each offset with one seed (so every run has the same truth rows), interleaved slot by slot and
scored with rx_ber_score_device, for every variant uncorrected, with a single estimate_offset correction, and with the bank.
--snrs LO:HI sweeps SNR LO .. HI-1 dB (default -5:31); --no-cfo leaves out the extra-carrier-offset rows.

Prints a markdown table (one row per point) and the throughput of both flows."""
import argparse
import ctypes
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from btle_b200 import BtleRx, ber  # noqa: E402
from btle_b200._native import DIR_DTYPE, RX_BER_RESULT_DTYPE  # noqa: E402,F401
from btle_b200.rx import make_cfgs  # noqa: E402


def kernel_times(rx, n_packets=32768, slot=2048, reps=5):
    """ms per batch of synth, receive and score (median of reps), on one batch of n_packets packets"""
    import torch
    cfg = ber.rx_ber_cfg(6.0, slot_samples=slot, seed=3)
    n_int8 = -(-n_packets * slot // 8192) * 16384
    d_iq = torch.empty(n_int8, dtype=torch.int8, device="cuda")
    d_truth = torch.empty((n_packets, 64), dtype=torch.uint8, device="cuda")
    cap = (n_int8 // 16384) * 123
    d_out = torch.empty(cap * 64, dtype=torch.uint8, device="cuda")
    units = rx.units(1, n_int8)
    d_dir = torch.empty(units * 8, dtype=torch.uint8, device="cuda")
    d_res = torch.zeros(RX_BER_RESULT_DTYPE.itemsize, dtype=torch.uint8, device="cuda")
    cfgs = make_cfgs(1, channel=37, rssi=2)
    st = torch.cuda.current_stream()
    sp = ctypes.c_void_p(st.cuda_stream)
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(4)]
    out = {"synth": [], "receive": [], "score": []}
    for _ in range(reps + 1):
        ev[0].record()
        rx._check(rx._L.btle_b200_rx_ber_synth_device(rx._h, cfg.ctypes.data, 0, n_packets, d_iq.data_ptr(), d_truth.data_ptr(), sp))
        ev[1].record()
        rx.rx_device_dir(d_iq.view(1, -1), cfgs, d_out, None, d_dir, stream_ptr=st.cuda_stream)
        ev[2].record()
        rx._check(rx._L.btle_b200_rx_ber_score_device(rx._h, d_truth.data_ptr(), n_packets, d_out.data_ptr(), cap, d_dir.data_ptr(), units,
                                                      d_res.data_ptr(), sp))
        ev[3].record()
        torch.cuda.synchronize()
        for k, name in enumerate(out):
            out[name].append(ev[k].elapsed_time(ev[k + 1]))
    return {k: float(np.median(v[1:])) for k, v in out.items()} | {"packets": n_packets, "slot_samples": slot}


def snr_at_half(points):
    """SNR where PER falls through 0.5 (linear between the two points around it), None if the sweep does not cross it"""
    pts = sorted((p["snr_db"], p["per"]) for p in points)
    for (s0, p0), (s1, p1) in zip(pts, pts[1:]):
        if p0 >= 0.5 > p1:
            return s0 + (p0 - 0.5) / (p0 - p1) * (s1 - s0)
    return None


def breakdown(rows, keys, label):
    """per ppm (no extra carrier offset) and variant: SNR at PER 0.5, and the error counters summed over the sweep"""
    print("\n| ppm | receiver | SNR dB at PER 0.5 | pkt_err | aa_miss | len_reject | crc_ok_wrong | extra_recs |")
    print("|---:|---|---:|---:|---:|---:|---:|---:|")
    for ppm in sorted({r["ppm"] for r in rows if r["cfo_hz"] == 0.0}):
        mine = [r for r in rows if r["ppm"] == ppm and r["cfo_hz"] == 0.0]
        for k in keys:
            pts = [r[k] for r in mine]
            s = snr_at_half(pts)
            tot = {c: sum(p[c] for p in pts) for c in ("pkt_err", "aa_miss", "len_reject", "crc_ok_wrong", "extra_recs")}
            print(f"| {ppm:g} | {label[k]} | {'-' if s is None else f'{s:.2f}'} | {tot['pkt_err']} | {tot['aa_miss']} | {tot['len_reject']} | "
                  f"{tot['crc_ok_wrong']} | {tot['extra_recs']} |")
        s = snr_at_half([r["model8"] for r in mine])
        print(f"| {ppm:g} | 8-sps model | {'-' if s is None else f'{s:.2f}'} | | | | | |")


MIXED_HZ = (-120e3, -60e3, 0.0, 60e3, 120e3)


def mixed_cfo(rx, snrs, n_packets, ways, label):
    """--mixed-cfo: per SNR and variant (without its bank suffix), PER uncorrected, with one estimate_offset correction of
    the whole capture, and with the bank; the capture's slot k comes from the rx_ber_synth_device run at MIXED_HZ[k % 5]"""
    import torch
    dev = torch.device("cuda", rx.device)
    st = torch.cuda.current_stream(dev)
    base = [("rx4", False, False, False, False, False)] + [w for w in ways if not w[0].endswith("_bank")]
    rows = []
    for snr in snrs:
        cfg0 = ber.rx_ber_cfg(snr, slot_samples=2048, seed=11)
        n = min(n_packets, 8192 * 8192 // 2048)
        chunks = (n * 2048 + 8191) // 8192
        caps = []
        d_truth = torch.empty(n * 64, dtype=torch.uint8, device=dev)
        for hz in MIXED_HZ:
            c = cfg0.copy()
            c["cfo_hz"] = hz
            d_iq = torch.zeros(chunks * 16384, dtype=torch.int8, device=dev)
            rx._check(rx._L.btle_b200_rx_ber_synth_device(rx._h, c.ctypes.data, 0, n, d_iq.data_ptr(), d_truth.data_ptr(), st.cuda_stream))
            caps.append(d_iq)
        slot = 2 * 2048
        x = torch.stack(caps).view(len(MIXED_HZ), -1)[:, :n * slot].reshape(len(MIXED_HZ), n, slot)
        iq = x[torch.arange(n, device=dev) % len(MIXED_HZ), torch.arange(n, device=dev)].reshape(1, -1)
        iq = torch.nn.functional.pad(iq, (0, chunks * 16384 - iq.shape[1])).contiguous()
        units = rx.units(1, iq.shape[1])
        row = {"snr_db": snr}
        for k, rc, sy, ce, co, lp in base:
            kw = dict(recover=rc, symbol_spaced=sy, centre_hits=ce, correct=co, lowpass=lp)
            est = rx.estimate_offset(iq.cpu().numpy().reshape(-1), channel=37, symbol_spaced=sy, lowpass=lp, centre_hits=ce)
            for how, os_, off in (("plain", 0, None), ("estimate", 0, est or 0.0), ("bank", 1, None)):
                cfgs = make_cfgs(1, channel=37, rssi=2, offset_search=os_, **kw)
                cap = chunks * 123 * 7
                d_out = torch.empty(cap * 64, dtype=torch.uint8, device=dev)
                d_dir = torch.empty(max(units, 1) * 8, dtype=torch.uint8, device=dev)
                d_res = torch.zeros(RX_BER_RESULT_DTYPE.itemsize, dtype=torch.uint8, device=dev)
                rx.rx_device_dir(iq, cfgs, d_out, None, d_dir, st.cuda_stream, offset_hz=off)
                rx._check(rx._L.btle_b200_rx_ber_score_device(rx._h, d_truth.data_ptr(), n, d_out.data_ptr(), cap, d_dir.data_ptr(), units,
                                                              d_res.data_ptr(), st.cuda_stream))
                st.synchronize()
                r = d_res.cpu().numpy().view(RX_BER_RESULT_DTYPE)[0]
                row[f"{label[k]} {how}"] = {"per": int(r["pkt_err"]) / max(int(r["packets"]), 1), "crc_ok_wrong": int(r["crc_ok_wrong"]),
                                            "extra_recs": int(r["extra_recs"]), "estimate_hz": est}
        rows.append(row)
    keys = [k for k in rows[0] if k != "snr_db"] if rows else []
    print("| mixed cfo SNR dB |" + "".join(f" PER {k} |" for k in keys))
    print("|---:|" + "---:|" * len(keys))
    for r in rows:
        print(f"| {r['snr_db']:g} |" + "".join(f" {r[k]['per']:.4f} |" for k in keys))
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--packets", type=int, default=20000)
    ap.add_argument("--json", default=None)
    ap.add_argument("--recover", action="store_true", help="also measure the receiver with BTLE_CFG_RECOVER")
    ap.add_argument("--symbol-spaced", action="store_true", help="also measure the receiver with BTLE_CFG_SYMBOL_SPACED")
    ap.add_argument("--centre-hits", action="store_true", help="also measure every 4-sps variant with BTLE_CFG_CENTRE_HITS")
    ap.add_argument("--correct", action="store_true", help="also measure every 4-sps variant with BTLE_CFG_CORRECT")
    ap.add_argument("--lowpass", action="store_true", help="also measure every symbol-spaced variant with BTLE_CFG_LOWPASS")
    ap.add_argument("--offset-search", action="store_true", help="also measure every 4-sps variant with BTLE_CFG_OFFSET_SEARCH")
    ap.add_argument("--mixed-cfo", action="store_true", help="add the rows of a capture that alternates between five offsets")
    ap.add_argument("--snrs", default="-5:31", help="LO:HI, SNR points LO .. HI-1 dB")
    ap.add_argument("--no-cfo", action="store_true", help="leave out the extra-carrier-offset rows")
    args = ap.parse_args()
    rx = BtleRx(0)
    lo, hi = (int(v) for v in args.snrs.split(":"))
    snrs = list(range(lo, hi))             # the 4-sps receiver's curve falls between 15 and 30 dB
    # the 4-sps variants: (key, recover, symbol_spaced, centre_hits, correct, lowpass)
    ways = [("rx4_recover", True, False, False, False, False)] if args.recover else []
    if args.symbol_spaced:
        ways += [("rx4_symbol", False, True, False, False, False)] + ([("rx4_symbol_recover", True, True, False, False, False)] if args.recover else [])
    if args.centre_hits:
        ways += [("rx4_centre", False, False, True, False, False)] + [(k + "_centre", rc, sy, True, False, False) for k, rc, sy, _, _, _ in ways]
    if args.correct:
        ways += [("rx4_correct", False, False, False, True, False)] + [(k + "_correct", rc, sy, ce, True, False) for k, rc, sy, ce, _, _ in ways]
    if args.lowpass:
        ways += [(k + "_lowpass", rc, sy, ce, co, True) for k, rc, sy, ce, co, _ in ways if sy]
    if args.offset_search:                 # the bank's variants are keyed "..._bank"
        ways += [("rx4_bank", False, False, False, False, False)] + [(k + "_bank", *f) for k, *f in ways]
    rows = []
    for ppm in (0.0, 20.0, 50.0):
        r4 = ber.rx_ber_sweep(snrs, args.packets, ppm=ppm, rx=rx)
        r8 = ber.ber_sweep(snrs, args.packets, ppm=ppm, rx=rx)
        rw = {k: ber.rx_ber_sweep(snrs, args.packets, ppm=ppm, rx=rx, recover=rc, symbol_spaced=sy, centre_hits=ce, correct=co, lowpass=lp,
                                  offset_search=k.endswith("_bank"))
              for k, rc, sy, ce, co, lp in ways}
        for i, (a, b) in enumerate(zip(r4, r8)):
            rows.append({"ppm": ppm, "cfo_hz": 0.0, "rx4": a, "model8": b, **{k: v[i] for k, v in rw.items()}})
    cfos = (25e3, 50e3, 100e3, 150e3) if not args.offset_search else (-150e3, -125e3, -100e3, -75e3, -50e3, -25e3, 25e3, 50e3, 75e3, 100e3,
                                                                      125e3, 150e3)
    for cfo in () if args.no_cfo else cfos:
        r4 = ber.rx_ber_sweep(snrs, args.packets, cfo_hz=cfo, rx=rx)
        rw = {k: ber.rx_ber_sweep(snrs, args.packets, cfo_hz=cfo, rx=rx, recover=rc, symbol_spaced=sy, centre_hits=ce, correct=co, lowpass=lp,
                                  offset_search=k.endswith("_bank"))
              for k, rc, sy, ce, co, lp in ways}
        for i, a in enumerate(r4):
            rows.append({"ppm": 0.0, "cfo_hz": cfo, "rx4": a, "model8": None, **{k: v[i] for k, v in rw.items()}})
    label = {"rx4_recover": "recover", "rx4_symbol": "symbol", "rx4_symbol_recover": "symbol+recover"}
    label.update({"rx4_centre": "centre"} | {k + "_centre": v + "+centre" for k, v in label.items()})
    label.update({"rx4_correct": "correct"} | {k + "_correct": v + "+correct" for k, v in label.items()})
    label.update({k + "_lowpass": v + "+lowpass" for k, v in label.items()})
    label.update({"rx4_bank": "bank"} | {k + "_bank": v + "+bank" for k, v in label.items()})
    extra_h = "".join(f" 4-sps PER {label[k]} | 4-sps BER {label[k]} | aa_miss {label[k]} |" for k, *_ in ways)
    print(f"| ppm | cfo kHz | SNR dB | 4-sps PER | 4-sps BER |{extra_h} aa_miss | len_reject | extra | 8-sps model PER | 8-sps model BER |")
    print("|---:|---:|---:|---:|---:|" + "---:|---:|---:|" * len(ways) + "---:|---:|---:|---:|---:|")
    for r in rows:
        a, b = r["rx4"], r["model8"]
        m = f"{b['per']:.4f} | {b['ber']:.2e}" if b else "- | -"
        rc = "".join(f" {r[k]['per']:.4f} | {r[k]['ber']:.2e} | {r[k]['aa_miss']} |" for k, *_ in ways)
        print(f"| {r['ppm']:g} | {r['cfo_hz'] / 1e3:g} | {a['snr_db']:g} | {a['per']:.4f} | {a['ber']:.2e} |{rc} {a['aa_miss']} | {a['len_reject']} | "
              f"{a['extra_recs']} | {m} |")
    if args.centre_hits or args.correct or args.lowpass or args.offset_search:
        breakdown(rows, ["rx4"] + [k for k, *_ in ways], {"rx4": "default", **label})
    mixed = mixed_cfo(rx, snrs, args.packets, ways, {"rx4": "default", **label}) if args.mixed_cfo else []
    r4 = [r["rx4"] for r in rows]
    r8 = [r["model8"] for r in rows if r["model8"]]
    thr = {"rx4_packets_per_s": float(np.median([a["packets_per_s"] for a in r4])),
           "rx4_generated_iq_gbytes_per_s": float(np.median([a["generated_iq_gbytes_per_s"] for a in r4])),
           "model8_packets_per_s": float(np.median([b["packets_per_s"] for b in r8])),
           "model8_generated_iq_gbytes_per_s": float(np.median([b["generated_iq_gbytes_per_s"] for b in r8]))}
    kt = kernel_times(rx)
    print(json.dumps({"throughput": thr, "kernel_ms_per_batch": kt}))
    if args.json:
        with open(args.json, "w") as f:
            json.dump({"rows": rows, "mixed_cfo": mixed, "throughput": thr, "kernel_ms_per_batch": kt}, f, indent=1)


if __name__ == "__main__":
    main()
