"""BER sweep on the GPU (BASELINE.json configs[3]; the reference flow is python/test_btle_ber.py): random 37-byte ADV
payloads -> CRC-24 + whitening -> the Python model's 8-samples-per-symbol integer GFSK modulator -> clock / carrier error
(ppm) -> AWGN at the requested SNR -> int16 truncation -> the Python model's receiver (8 phases, first CRC-ok phase wins)
-> bit-error accounting exactly as test_btle_ber.py:62-72 (bit errors are counted only in packets whose CRC failed).

Everything runs in three hand-written kernels behind ONE C-ABI call per point (btle_b200_ber_run: ber_synth_kernel,
model_rx_batch_kernel, ber_score_kernel); this module only loops over the points.

rx_ber_point / rx_ber_sweep measure the other receiver, the reference's 4-Msps int8 receive chain: impaired captures
(clock and carrier error, extra carrier offset, AWGN, int8 rounding and saturation) through btle_rx_persistent_kernel,
scored on the device (btle_b200_rx_ber_run: rx_ber_synth_kernel, the receive kernel, rx_ber_score_kernel)."""
from __future__ import annotations

import numpy as np

from . import _native
from .rx import BtleRx

PDU_HEX = "422506050403020119095344522f426c7565746f6f74682f4c6f772f456e657267791234567890"   # test_btle_ber.py:27
IQ_BYTES_PER_PACKET = 3024 * 2 * 2        # int16 I and Q, 8 samples per symbol, 376 PHY bits + 16 samples


def ber_point(rx: BtleRx, snr_db: float, n_packets: int, ppm: float = 0.0, channel: int = 37, crc_init: int = 0x555555,
              access_addr: int = 0x8E89BED6, seed: int = 1) -> dict:
    cfg = np.zeros(1, dtype=_native.BER_CFG_DTYPE)
    cfg["seed"], cfg["snr_db"], cfg["ppm"], cfg["channel"], cfg["crc_init"], cfg["access_addr"] = seed, snr_db, ppm, channel, crc_init, access_addr
    res = np.zeros(1, dtype=_native.BER_RESULT_DTYPE)
    rx._check(rx._L.btle_b200_ber_run(rx._h, cfg.ctypes.data, int(n_packets), res.ctypes.data))
    r = res[0]
    sec = float(r["seconds"])
    return {"snr_db": float(snr_db), "ppm": float(ppm), "packets": int(r["packets"]), "ber": int(r["bit_err"]) / max(int(r["bit_total"]), 1),
            "per": int(r["pkt_err"]) / max(int(r["packets"]), 1), "bit_err": int(r["bit_err"]), "bit_total": int(r["bit_total"]),
            "pkt_err": int(r["pkt_err"]), "aa_miss": int(r["aa_miss"]), "seconds": sec,
            "packets_per_s": int(r["packets"]) / sec if sec > 0 else 0.0,
            "generated_iq_gbytes_per_s": int(r["packets"]) * IQ_BYTES_PER_PACKET / sec / 1e9 if sec > 0 else 0.0}


def ber_sweep(snr_db, n_packets: int, channel: int = 37, crc_init: int = 0x555555, access_addr: int = 0x8E89BED6, seed: int = 1,
              device: int = 0, rx: BtleRx | None = None, ppm: float = 0.0):
    """One dict per SNR point: ber, per, counts, packets/s, generated IQ GB/s."""
    rx = rx or BtleRx(device)
    return [ber_point(rx, s, n_packets, ppm, channel, crc_init, access_addr, seed + 7919 * k) for k, s in enumerate(snr_db)]


# ---- the 4-Msps receive chain (btle_b200_rx_ber_run; definition in include/btle_b200.h) --------------------------------
def rx_ber_cfg(snr_db: float, ppm: float = 0.0, cfo_hz: float = 0.0, amplitude: int = 64, slot_samples: int = 2048, channel: int = 37,
               crc_init: int = 0x555555, access_addr: int = 0x8E89BED6, seed: int = 1, recover: bool = False,
               symbol_spaced: bool = False, centre_hits: bool = False, correct: bool = False, lowpass: bool = False,
               offset_search: bool = False) -> np.ndarray:
    """recover: the receiver runs with BTLE_CFG_RECOVER (CRC-failed packets demodulated again); symbol_spaced: with
    BTLE_CFG_SYMBOL_SPACED (the symbol-spaced discriminator); centre_hits: with BTLE_CFG_CENTRE_HITS (each hit moved to the
    centre of its run of matching sample phases); correct: with BTLE_CFG_CORRECT (one-bit and adjacent-pair errors of
    CRC-failed packets corrected from the syndrome); lowpass: with BTLE_CFG_LOWPASS (the symbol-spaced bits read [1, 2, 1]
    filtered samples; only with symbol_spaced); offset_search: with BTLE_CFG_OFFSET_SEARCH (seven carrier-offset hypotheses,
    merged per packet)"""
    cfg = np.zeros(1, dtype=_native.RX_BER_CFG_DTYPE)
    cfg["seed"], cfg["snr_db"], cfg["ppm"], cfg["cfo_hz"], cfg["amplitude"] = seed, snr_db, ppm, cfo_hz, amplitude
    cfg["slot_samples"], cfg["channel"], cfg["crc_init"], cfg["access_addr"] = slot_samples, channel, crc_init, access_addr
    cfg["flags"] = ((_native.CFG_RECOVER if recover else 0) | (_native.CFG_SYMBOL_SPACED if symbol_spaced else 0) |
                    (_native.CFG_CENTRE_HITS if centre_hits else 0) | (_native.CFG_CORRECT if correct else 0) |
                    (_native.CFG_LOWPASS if lowpass else 0) | (_native.CFG_OFFSET_SEARCH if offset_search else 0))
    return cfg


def _rx_ber_corrected(rx: BtleRx, cfg: np.ndarray, n_packets: int, offset_hz: float) -> np.ndarray:
    """btle_b200_rx_ber_run's counters with the receiver corrected by offset_hz: rx_ber_synth_device -> the rotated receive
    kernel (rx_device_dir with offset_hz) -> rx_ber_score_device.  Batches of whole slots, each a capture of its own (its
    last chunk's look-ahead is noise, not the next batch's slots); one batch up to 8192 chunks, as btle_b200_rx_ber_run."""
    import torch
    from .rx import make_cfgs
    dev = torch.device("cuda", rx.device)
    st = torch.cuda.current_stream(dev)
    S = int(cfg["slot_samples"][0])
    per_batch = max(1, 8192 * 8192 // S)
    scfg = make_cfgs(1, channel=int(cfg["channel"][0]), access_addr=int(cfg["access_addr"][0]), crc_init=int(cfg["crc_init"][0]),
                     rssi=_native.CFG_REPORT_REJECTED | int(cfg["flags"][0]))
    d_res = torch.zeros(_native.RX_BER_RESULT_DTYPE.itemsize, dtype=torch.uint8, device=dev)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(st)
    for done in range(0, n_packets, per_batch):
        n = min(per_batch, n_packets - done)
        chunks = (n * S + 8191) // 8192
        d_iq = torch.empty((1, chunks * 16384), dtype=torch.int8, device=dev)
        d_truth = torch.empty(n * _native.RX_BER_TRUTH_DTYPE.itemsize, dtype=torch.uint8, device=dev)
        rx._check(rx._L.btle_b200_rx_ber_synth_device(rx._h, cfg.ctypes.data, done, n, d_iq.data_ptr(), d_truth.data_ptr(), st.cuda_stream))
        # BTLE_MAX_RECS_PER_CHUNK per chunk, or with BTLE_CFG_OFFSET_SEARCH per hypothesis (the merge never overflows then)
        cap = chunks * 123 * (7 if int(cfg["flags"][0]) & _native.CFG_OFFSET_SEARCH else 1)
        units = rx.units(1, chunks * 16384)
        d_out = torch.empty(cap * 64, dtype=torch.uint8, device=dev)
        d_dir = torch.empty(max(units, 1) * 8, dtype=torch.uint8, device=dev)
        rx.rx_device_dir(d_iq, scfg, d_out, None, d_dir, st.cuda_stream, offset_hz=offset_hz)
        rx._check(rx._L.btle_b200_rx_ber_score_device(rx._h, d_truth.data_ptr(), n, d_out.data_ptr(), cap, d_dir.data_ptr(), units,
                                                      d_res.data_ptr(), st.cuda_stream))
    e1.record(st)
    st.synchronize()
    res = d_res.cpu().numpy().view(_native.RX_BER_RESULT_DTYPE).copy()
    res["seconds"] = e0.elapsed_time(e1) * 1e-3
    return res


def rx_ber_point(rx: BtleRx, snr_db: float, n_packets: int, ppm: float = 0.0, cfo_hz: float = 0.0, amplitude: int = 64,
                 slot_samples: int = 2048, channel: int = 37, crc_init: int = 0x555555, access_addr: int = 0x8E89BED6, seed: int = 1,
                 recover: bool = False, offset_hz: float | None = None, symbol_spaced: bool = False, centre_hits: bool = False,
                 correct: bool = False, lowpass: bool = False, offset_search: bool = False) -> dict:
    """PER / BER of the reference's 4-Msps int8 receiver (btle_rx_persistent_kernel) at one channel point: ber_point()'s dict
    plus cfo_hz, amplitude and the counters len_reject, crc_ok_wrong, extra_recs, extra_crc_ok and clipped.
    generated_iq_gbytes_per_s counts the int8 capture the run synthesised and decoded (2 bytes per sample).
    offset_hz: the receiver corrects that carrier offset (the *_offset entry points; the sign of cfo_hz, so offset_hz =
    cfo_hz undoes the impairment); None: btle_b200_rx_ber_run, uncorrected.  symbol_spaced: the receiver uses the
    symbol-spaced discriminator (BTLE_CFG_SYMBOL_SPACED).  centre_hits: the chain centres each hit on its run of matching
    sample phases (BTLE_CFG_CENTRE_HITS).  correct: CRC-failed packets are corrected from their syndrome (BTLE_CFG_CORRECT).
    lowpass: the symbol-spaced bits read [1, 2, 1]-filtered samples (BTLE_CFG_LOWPASS).  offset_search: the receiver decodes at
    seven carrier offsets around offset_hz (or 0) and merges the packets (BTLE_CFG_OFFSET_SEARCH)."""
    cfg = rx_ber_cfg(snr_db, ppm, cfo_hz, amplitude, slot_samples, channel, crc_init, access_addr, seed, recover, symbol_spaced,
                     centre_hits, correct, lowpass, offset_search)
    if offset_hz is None:
        res = np.zeros(1, dtype=_native.RX_BER_RESULT_DTYPE)
        rx._check(rx._L.btle_b200_rx_ber_run(rx._h, cfg.ctypes.data, int(n_packets), res.ctypes.data))
    else:
        res = _rx_ber_corrected(rx, cfg, int(n_packets), float(offset_hz))
    r = res[0]
    c = {k: int(r[k]) for k in _native.RX_BER_COUNTERS}
    sec = float(r["seconds"])
    return {"snr_db": float(snr_db), "ppm": float(ppm), "cfo_hz": float(cfo_hz), "amplitude": int(amplitude), "recover": bool(recover),
            "symbol_spaced": bool(symbol_spaced), "centre_hits": bool(centre_hits), "correct": bool(correct), "lowpass": bool(lowpass),
            "offset_search": bool(offset_search),
            "offset_hz": offset_hz, **c,
            "ber": c["bit_err"] / max(c["bit_total"], 1), "per": c["pkt_err"] / max(c["packets"], 1), "seconds": sec,
            "packets_per_s": c["packets"] / sec if sec > 0 else 0.0,
            "generated_iq_gbytes_per_s": c["packets"] * slot_samples * 2 / sec / 1e9 if sec > 0 else 0.0}


def rx_ber_sweep(snr_db, n_packets: int, ppm: float = 0.0, cfo_hz: float = 0.0, amplitude: int = 64, slot_samples: int = 2048,
                 channel: int = 37, crc_init: int = 0x555555, access_addr: int = 0x8E89BED6, seed: int = 1, device: int = 0,
                 rx: BtleRx | None = None, recover: bool = False, offset_hz: float | None = None, symbol_spaced: bool = False,
                 centre_hits: bool = False, correct: bool = False, lowpass: bool = False, offset_search: bool = False):
    """One rx_ber_point dict per SNR point (seeds as ber_sweep)."""
    rx = rx or BtleRx(device)
    return [rx_ber_point(rx, s, n_packets, ppm, cfo_hz, amplitude, slot_samples, channel, crc_init, access_addr, seed + 7919 * k, recover,
                         offset_hz, symbol_spaced, centre_hits, correct, lowpass, offset_search) for k, s in enumerate(snr_db)]
