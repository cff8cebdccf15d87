"""The GPU path built on the reference's Python model (btlelib.py) against exact references at its edges:
sps8_hits_kernel (btle_b200_sps8_hits_device) against btlelib_port.find_hits, the streaming windows of btle_b200_rx_sps8
against btlelib_port.rx_stream, model_rx_batch_kernel at 1..16 samples per symbol against the reference's btle_rx
(tests/golden/btlelib_rx_sps.npz) and the port, ber_synth_kernel / ber_score_kernel against a float64 numpy restatement,
and the --iq-bin16 mode of btle_rx_b200.

Captures are built from per-phase bit sequences (btlelib_port.phase_bits_to_iq): on phase p, sample a + 8 is sample a
turned by +-90 degrees, so the symbol-spaced differential bit of every phase is exactly the planted bit and an access
address can be put at any sample index."""
import ctypes
import json
import os
import subprocess
import sys

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "oracle"))
import btlelib_port as P  # noqa: E402
from test_oracle_btlelib_port import sps_windows  # noqa: E402

ADV_AA, ADV_CRC = 0x8E89BED6, 0x555555
AA_MSB0 = 0x60850A1B                     # bit 31 (the last one on air) is 0, like a zero-filled sample's bit
TILE = 32 * 256                          # sps8_hits_kernel: 32 groups of 256 samples per CTA
EINVAL, EOVERFLOW = -1, -5


@pytest.fixture(scope="module")
def rx():
    import __graft_entry__ as ge
    ge.build()
    from btle_b200 import BtleRx
    return BtleRx(0)


def aa_bits(aa):
    return P.bits_lsb_first(aa, 4)


def capture(n, plants=(), rng=None, amp=1000, bits=None):
    """int16 [n, 2]: random per-phase bits (or `bits` [8, m]) with plants = [(sample index, bit array)] written from that
    sample on its phase (index mod 8); bits that would need samples at or behind n are simply not there."""
    m = max(1, -(-n // 8))
    if bits is None:
        bits = (rng or np.random.default_rng(n)).integers(0, 2, (8, m)).astype(np.int8)
    for h, b in plants:
        k = h // 8
        b = b[: m - k]
        bits[h % 8, k:k + len(b)] = b
    return P.phase_bits_to_iq(bits, n=n, amp=amp, sps=8)


# ---- a. sps8_hits_device against find_hits ------------------------------------------------------------------------
def hits_device(rx, iq, aa, cap=None, offset=0, stream=None):
    """(rc, count, sorted hits written) of btle_b200_sps8_hits_device on a copy of iq placed `offset` bytes into a larger
    device buffer."""
    import torch
    n = len(iq)
    raw = torch.zeros(offset + 4 * n + 64, dtype=torch.uint8, device="cuda")
    if n:
        raw[offset:offset + 4 * n] = torch.from_numpy(np.ascontiguousarray(iq).view(np.uint8).reshape(-1)).cuda()
    cap = n // 8 + 64 if cap is None else cap
    d_hits = torch.full((max(cap, 1),), -1, dtype=torch.int64, device="cuda")
    d_cnt = torch.full((1,), 12345, dtype=torch.int32, device="cuda")
    st = stream or torch.cuda.current_stream()
    torch.cuda.synchronize()
    rc = rx._L.btle_b200_sps8_hits_device(rx._h, raw.data_ptr() + offset, n, aa, d_hits.data_ptr(), cap, d_cnt.data_ptr(),
                                          ctypes.c_void_p(st.cuda_stream))
    st.synchronize()
    cnt = int(d_cnt.cpu()[0]) & 0xFFFFFFFF
    got = d_hits.cpu().numpy()[: min(cnt, cap)] if rc == 0 else np.zeros(0, np.int64)
    return rc, cnt, np.sort(got)


def edge_lengths():
    ls = [0, 1, 7, 8, 255, 256, 257, 263, 264, 265, 8191, 8192, 8193, TILE + 263, TILE + 264, TILE + 265, 3 * TILE + 2, 12345, 30001]
    for k in (2, 3, 5):
        ls += [k * TILE + s * d for d in (1, 4, 263, 264) for s in (-1, 1)]
    return ls


def hit_plants(n, aa, first_inadmissible):
    """an access address on every phase at the last admissible start (n + 256 < n_samples) or at the first inadmissible
    one; at sample 0; and straddling every tile boundary (on phases that do not collide with the ones at the end)"""
    a = aa_bits(aa)
    plants, end = [], n - 257 + (1 if first_inadmissible else 0)
    for p in range(8):
        h = end + ((p - end) % 8) if first_inadmissible else end - ((end - p) % 8)
        if h >= 0:
            plants.append((h, a))
    if n > 600:
        plants.append((0, a))
    for t in range(1, n // TILE + 1):
        for j, d in enumerate((1, 16, 31)):                # the boundary after bit d - 1 of the access address
            h = t * TILE - 8 * d + ((t + j) % 8)
            if 300 < h < n - 800:
                plants.append((h, a))
    return plants


@pytest.mark.parametrize("aa", [ADV_AA, AA_MSB0])
def test_sps8_hits_equal_find_hits_at_every_edge(rx, aa):
    import torch
    st = torch.cuda.Stream()
    n_checked = n_hits = 0
    for n in edge_lengths():
        for kind in ("bits", "full_scale", "noise"):
            for first_inadmissible in (False, True):
                rng = np.random.default_rng([n, aa & 0xFFFF, int(first_inadmissible), len(kind)])
                if kind == "noise":
                    if first_inadmissible:
                        continue
                    iq = rng.integers(-32768, 32768, (n, 2)).astype(np.int16)
                    for h, b in hit_plants(n, aa, False):   # planted with noise-level amplitudes around them
                        seg = capture(n, [(h, b)], rng, amp=int(rng.integers(1, 32767)))
                        k = np.arange(h, min(n, h + 264))
                        iq[k] = seg[k]
                else:
                    iq = capture(n, hit_plants(n, aa, first_inadmissible), rng, amp=32767 if kind == "full_scale" else 1000)
                    if kind == "full_scale":
                        iq[iq == -32767] = -32768
                exp = P.find_hits(iq, aa)
                off = [0, 16, 48, 4096 + 16][n_checked % 4]
                rc, cnt, got = hits_device(rx, iq, aa, offset=off, stream=st if n_checked % 2 else None)
                assert rc == 0 and cnt == len(exp), (n, kind, first_inadmissible, cnt, len(exp))
                assert np.array_equal(got, exp), (n, kind, first_inadmissible)
                if kind != "noise" and not first_inadmissible and n >= 257 + 7:
                    assert len(exp) >= 8, n                 # every phase's last admissible start is a hit
                n_checked += 1
                n_hits += len(exp)
    assert n_hits > 1000


def test_sps8_hits_dense_capture_and_small_cap(rx):
    """A capture that hits every 32 symbols on every phase; a `cap` below the count still counts exactly and writes a
    subset of the true hits, each once."""
    n = 3 * TILE + 100
    reps = -(-n // 8) // 32 + 1
    bits = np.tile(np.tile(aa_bits(ADV_AA), reps)[: -(-n // 8)], (8, 1)).astype(np.int8)
    iq = capture(n, bits=bits)
    exp = P.find_hits(iq, ADV_AA)
    assert len(exp) > 700
    rc, cnt, got = hits_device(rx, iq, ADV_AA)
    assert rc == 0 and cnt == len(exp) and np.array_equal(got, exp)
    for cap in (0, 1, 100, len(exp) - 1):
        rc, cnt, got = hits_device(rx, iq, ADV_AA, cap=cap)
        assert rc == 0 and cnt == len(exp) and len(got) == cap
        assert len(np.unique(got)) == cap and np.isin(got, exp).all()


def test_sps8_hits_rejects_a_capture_that_is_not_16_byte_aligned(rx):
    iq = capture(TILE + 300, hit_plants(TILE + 300, ADV_AA, False))
    exp = P.find_hits(iq, ADV_AA)
    for off in (4, 8, 12, 16 + 4):
        rc, _, _ = hits_device(rx, iq, ADV_AA, offset=off)
        assert rc == EINVAL, off
        assert b"16-byte" in rx._L.btle_b200_last_error(rx._h), off
        rc, cnt, got = hits_device(rx, iq, ADV_AA, offset=off - off % 16)   # the context stays usable
        assert rc == 0 and cnt == len(exp) and np.array_equal(got, exp)


# ---- b. rx_sps8 against rx_stream at the capture edges --------------------------------------------------------------
def assert_sps8_equal(got, exp):
    assert len(got) == len(exp), (len(got), len(exp))
    for g, e in zip(got, exp):
        r = g["rx"]
        assert int(g["sample"]) == e["sample"] and int(g["window"]) == e["window"]
        assert bool(r["crc_ok"]) == e["crc_ok"] and int(r["payload_len"]) == e["plen"] and int(r["phase"]) == e["phase"]
        assert int(r["found"]) == e["found"] and int(r["start"]) == e["start"] and int(r["n_pdu_bits"]) == len(e["pdu_bit"])
        assert np.array_equal(np.unpackbits(r["pdu"], bitorder="little")[: len(e["pdu_bit"])], e["pdu_bit"])


def adv_packet(rng, plen, flip_crc=False):
    pdu = bytes([0x40, plen]) + rng.integers(0, 256, plen, dtype=np.uint8).tobytes()
    b = P.tx_bits(pdu, 37)[8:].copy()                  # from the access address on
    if flip_crc:
        b[-1] ^= 1
    return pdu, b


def stream_case(rx, n, plants, rng):
    iq = capture(n, plants, rng)
    got, exp = rx.rx_sps8(iq.reshape(-1), 37), P.rx_stream(iq, 37)
    assert_sps8_equal(got, exp)
    return exp


def test_rx_sps8_equals_rx_stream_at_the_capture_edges(rx):
    rng = np.random.default_rng(77)
    W = P.WINDOW
    _, pk = adv_packet(rng, 20)
    every = lambda k, b: [(8 * k + p, b) for p in range(8)]            # one packet on all 8 phases from symbol k
    # first hit within the first 16 symbols: window clamped to 0
    for k in (0, 1, 2, 15):
        e = stream_case(rx, 2 * W, every(k, pk), rng)
        assert len(e) == 1 and e[0]["window"] == max(0, 8 * (k - 2)) and e[0]["crc_ok"]
    # the window ends exactly at the capture's end, or 8 samples behind it (dropped)
    k = 300
    w0 = 8 * (k - 2)
    e = stream_case(rx, w0 + W, every(k, pk), rng)
    assert len(e) == 1 and e[0]["window"] == w0
    assert stream_case(rx, w0 + W - 8, every(k, pk), rng) == []
    # capture lengths around one window
    for n in (W - 1, W, W + 1):
        e = stream_case(rx, n, every(1, pk), rng)
        assert len(e) == (n >= W)
    # two packets exactly 576 samples (72 symbols, the shortest packet) apart on phase 0: two clusters, both reported;
    # 575 apart (phase 7 one symbol earlier): one cluster
    _, p0 = adv_packet(rng, 0)
    e = stream_case(rx, 4 * W, [(8 * 100, p0), (8 * 100 + 576, p0)], rng)
    assert [x["sample"] for x in e] == [800, 800 + 576] and all(x["crc_ok"] for x in e)
    e = stream_case(rx, 4 * W, [(8 * 100, p0), (8 * 100 + 575, p0)], rng)
    assert len(e) == 1
    # hits on neighbouring phases closer than 72 symbols, not all of the same packet: one cluster
    e = stream_case(rx, 4 * W, [(8 * 100 + 3, pk), (8 * 100 + 3 + 8 * 71 + 2, pk)], rng)
    assert len(e) == 1
    # a window that starts inside the packet accepted before it (greedy skip): an access address on phase 5, 100 symbols
    # into a long packet carried by phases 0..4
    _, plong = adv_packet(rng, 37)
    e = stream_case(rx, 4 * W, [(8 * 100 + p, plong) for p in range(5)] + [(8 * 200 + 5, aa_bits(ADV_AA))], rng)
    assert len(e) == 1 and e[0]["crc_ok"] and e[0]["plen"] == 37
    # the same access address outside the packet is a packet of its own
    e = stream_case(rx, 4 * W, [(8 * 100 + p, plong) for p in range(5)] + [(8 * 100 + 8 * 368 + 5, aa_bits(ADV_AA))], rng)
    assert len(e) == 2
    # found but never CRC-ok, and CRC-ok on a later phase only
    _, bad = adv_packet(rng, 12, flip_crc=True)
    e = stream_case(rx, 2 * W, [(8 * 40 + p, bad) for p in range(8)], rng)
    assert len(e) == 1 and not e[0]["crc_ok"] and e[0]["found"] == 8 and e[0]["phase"] == 7
    e = stream_case(rx, 2 * W, [(8 * 40 + p, bad) for p in range(3)] + [(8 * 40 + p, pk) for p in range(3, 8)], rng)
    assert len(e) == 1 and e[0]["crc_ok"] and e[0]["phase"] == 3 and e[0]["sample"] == 8 * 40 + 3


def test_rx_sps8_too_small_cap_reports_the_exact_count(rx):
    from btle_b200._native import SPS8_REC_DTYPE
    rng = np.random.default_rng(5)
    _, pk = adv_packet(rng, 10)
    iq = capture(20 * 1600 + P.WINDOW, [(8 * (200 * j + 10) + j % 8, pk) for j in range(20)], rng)
    exp = P.rx_stream(iq, 37)
    assert len(exp) >= 15          # (a window opened by a phase-7 hit reports the phase-0 packet behind it: 18 of 20)
    for cap in (0, 7, len(exp) - 1):
        out = np.zeros(max(cap, 1), dtype=SPS8_REC_DTYPE)
        n_out = ctypes.c_size_t(0)
        rc = rx._L.btle_b200_rx_sps8(rx._h, iq.ctypes.data, len(iq), 37, ADV_CRC, ADV_AA, out.ctypes.data, cap, ctypes.byref(n_out))
        assert rc == EOVERFLOW and n_out.value == len(exp), cap
        assert_sps8_equal(out[:cap], exp[:cap])


# ---- c. the model receiver at every sps --------------------------------------------------------------------------------
def test_model_rx_equals_reference_and_port_at_every_sps(rx):
    """btle_b200_model_rx_batch and _device (planar windows, a non-default stream) against the reference's btle_rx at 1, 2,
    4, 8, 16 samples per symbol (tests/golden/btlelib_rx_sps.npz) and against rx_window(sps=...), record for record."""
    import torch
    from btle_b200 import btlelib_compat as bl
    from btle_b200._native import MODEL_REC_DTYPE
    st = torch.cuda.Stream()
    n = 0
    for w in sps_windows():
        sps, key = w["sps"], (w["name"], w["sps"])
        r = bl.btle_rx_batch(w["i"][None, :], w["q"][None, :], w["ch"], w["crc"], w["aa"], sps=sps)[0]
        di, dq = torch.from_numpy(w["i"][None, :].copy()).cuda(), torch.from_numpy(w["q"][None, :].copy()).cuda()
        d_out = torch.zeros(MODEL_REC_DTYPE.itemsize, dtype=torch.uint8, device="cuda")
        torch.cuda.synchronize()
        rx._check(rx._L.btle_b200_model_rx_batch_device(rx._h, di.data_ptr(), dq.data_ptr(), 1, len(w["i"]), sps, w["ch"], w["crc"], w["aa"],
                                                        d_out.data_ptr(), ctypes.c_void_p(st.cuda_stream)))
        st.synchronize()
        assert d_out.cpu().numpy().tobytes() == r.tobytes(), key
        p = P.rx_window(w["i"], w["q"], w["ch"], w["crc"], w["aa"], sps=sps)
        refs = [p] if w["raises"] else [p, dict(w)]
        for e in refs:
            assert (bool(r["crc_ok"]), int(r["payload_len"]), int(r["phase"]), int(r["found"]), int(r["start"])) == \
                (e["crc_ok"], e["plen"], e["phase"], e["found"], e["start"]), key
            nb = len(e["pdu_bit"])
            assert int(r["n_pdu_bits"]) == nb and np.array_equal(np.unpackbits(r["pdu"], bitorder="little")[:nb], e["pdu_bit"]), key
            assert not np.unpackbits(r["pdu"], bitorder="little")[nb:].any(), key
        n += 1
    assert n >= 90


# ---- d. the BER flow, exact --------------------------------------------------------------------------------------------
BER_SAMPLES = 3024
M64 = np.uint64(0xFFFFFFFFFFFFFFFF)


def mix64(x):
    x = (x + np.uint64(0x9E3779B97F4A7C15)) & M64
    x = ((x ^ (x >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)) & M64
    x = ((x ^ (x >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)) & M64
    return x ^ (x >> np.uint64(31))


def draw(seed, stream, a, k):
    """the kernels' counter-based generator (splitmix64 finaliser of seed, stream, position, kind) in uint64"""
    with np.errstate(over="ignore"):
        stream, a = np.asarray(stream, dtype=np.uint64), np.asarray(a, dtype=np.uint64)
        s = mix64(np.uint64(seed) ^ (stream * np.uint64(0xD1B54A32D192ED03)))
        return mix64(s ^ (a * np.uint64(0x9E3779B97F4A7C15)) ^ (np.uint64(k) << np.uint64(56)))


def ber_truth(seed, packets):
    """the 39 PDU bytes of each packet: header 42 25 + 37 random bytes, byte b from draw(seed, packet, b >> 3, 9)"""
    packets = np.asarray(packets, dtype=np.uint64)
    r = draw(seed, packets[:, None], np.arange(5)[None, :], 9)                # [n, 5] words
    b = np.arange(39)
    out = ((r[:, b >> 3] >> (np.uint64(8) * (b & 7).astype(np.uint64))) & np.uint64(0xFF)).astype(np.uint8)
    out[:, 0], out[:, 1] = 0x42, 0x25
    return out


def ber_cfg(seed, snr_db, ppm, channel=37, crc=ADV_CRC, aa=ADV_AA):
    from btle_b200._native import BER_CFG_DTYPE
    c = np.zeros(1, dtype=BER_CFG_DTYPE)
    c["seed"], c["snr_db"], c["ppm"], c["channel"], c["crc_init"], c["access_addr"] = seed, snr_db, ppm, channel, crc, aa
    return c


def ber_synth(rx, cfg, first, n, stream=None):
    import torch
    di = torch.empty((n, BER_SAMPLES), dtype=torch.int16, device="cuda")
    dq = torch.empty_like(di)
    dt = torch.zeros((n, 40), dtype=torch.uint8, device="cuda")
    st = stream or torch.cuda.current_stream()
    rx._check(rx._L.btle_b200_ber_synth_device(rx._h, cfg.ctypes.data, first, n, di.data_ptr(), dq.data_ptr(), dt.data_ptr(),
                                               ctypes.c_void_p(st.cuda_stream)))
    st.synchronize()
    return di, dq, dt


def modulate_air(air):
    """tx_modulate_kernel (sps 8) on air bytes [n, 47]: the model's modulator, int8 -> float64"""
    import torch
    from btle_b200 import synth
    a = torch.from_numpy(np.ascontiguousarray(air)).cuda()
    oi, oq = synth.modulate_batch_cuda(a, torch.full((len(air),), air.shape[1], dtype=torch.int32), sps=8)
    torch.cuda.synchronize()
    return oi.cpu().numpy().astype(np.float64), oq.cpu().numpy().astype(np.float64)


def air_bytes(truth, channel=37, crc=ADV_CRC, aa=ADV_AA):
    return np.stack([np.packbits(P.tx_bits(bytes(t[:39]), channel, crc, aa), bitorder="little") for t in truth])


def channel_reference(txi, txq, seed, packets, snr_db, ppm):
    """float64 restatement of ber_synth_kernel's channel: np.interp at m (1 + e) (clamped to the last sample), the carrier
    rotation by e * 2450 MHz at the resampled time, Box-Muller on the kernel's float32 uniforms, truncation toward zero
    left to the caller (returns the real values)."""
    m = np.arange(BER_SAMPLES, dtype=np.float64)
    vi, vq = txi, txq
    if ppm != 0:
        e = float(np.float32(ppm)) * 1e-6
        x = m * (1.0 + e)
        vi = np.stack([np.interp(x, m, t) for t in txi])
        vq = np.stack([np.interp(x, m, t) for t in txq])
        turns = e * 2450e6 * (0.125e-6 * (1.0 + e)) * m
        ang = 2 * np.pi * (turns - np.floor(turns))
        vi, vq = vi * np.cos(ang) - vq * np.sin(ang), vi * np.sin(ang) + vq * np.cos(ang)
    r = draw(seed, np.asarray(packets, dtype=np.uint64)[:, None], np.arange(BER_SAMPLES)[None, :], 10)
    f = np.float32(2.3283064365386963e-10)
    u1 = ((r & np.uint64(0xFFFFFFFF)).astype(np.float32) + np.float32(0.5)) * f
    u2 = (r >> np.uint64(32)).astype(np.float32) * f
    rad = np.sqrt(-2.0 * np.log(u1.astype(np.float64)))
    g = np.float32(127.0) / np.float32(10.0 ** (np.float32(snr_db) / np.float32(20.0))) * np.float32(0.70710678)
    sigma = float(g)
    return vi + sigma * rad * np.cos(2 * np.pi * u2.astype(np.float64)), vq + sigma * rad * np.sin(2 * np.pi * u2.astype(np.float64))


def test_ber_synth_noiseless_equals_the_modulator_and_truth_equals_draw(rx):
    seed, first, n = 0x5EED, 70000, 64
    cfg = ber_cfg(seed, 1000.0, 0.0)                   # 127 / exp10f(50) == 0 in float32: no noise at all
    di, dq, dt = ber_synth(rx, cfg, first, n)
    truth = ber_truth(seed, np.arange(first, first + n))
    assert np.array_equal(dt.cpu().numpy()[:, :39], truth)
    assert len({bytes(t[2:]) for t in truth}) == n
    mi, mq = modulate_air(air_bytes(truth))
    assert mi.shape == (n, BER_SAMPLES)
    assert np.array_equal(di.cpu().numpy(), mi) and np.array_equal(dq.cpu().numpy(), mq)
    # the same packets from another first_packet / batch split are the same samples
    di2, _, dt2 = ber_synth(rx, cfg, first + 7, 9)
    assert np.array_equal(di2.cpu().numpy(), di.cpu().numpy()[7:16]) and np.array_equal(dt2.cpu().numpy(), dt.cpu().numpy()[7:16])


@pytest.mark.parametrize("ppm", [-50.0, -12.5, 20.0, 50.0, 0.0])
def test_ber_synth_channel_equals_float64_restatement(rx, ppm):
    seed, first, n, snr = 31, 40000, 96, 8.0
    cfg = ber_cfg(seed, snr, ppm)
    di, dq, dt = ber_synth(rx, cfg, first, n)
    truth = dt.cpu().numpy()[:, :39]
    txi, txq = modulate_air(air_bytes(truth))
    ri, rq = channel_reference(txi, txq, seed, np.arange(first, first + n), snr, ppm)
    ref = np.concatenate((np.trunc(ri), np.trunc(rq)))
    got = np.concatenate((di.cpu().numpy(), dq.cpu().numpy())).astype(np.float64)
    assert np.abs(got - ref).max() <= 1
    # a sample can differ only where the kernel's float32 error moves the value across an integer.  Per sample, with
    # V = max |value| and eps = float32 epsilon, the error terms are: the float32 sum vi + sigma * g and the product
    # sigma * g (<= V eps / 2 each, the dominant terms, V ~ 127 + 5 sigma); sigma itself (exp10f, ~2 ulp: <= 2 V eps);
    # the interpolation weight and vi (<= 254 eps + 127 eps); the turns cast to float and sincospif (~127 (2 pi + 1) eps);
    # __logf (2^-21.4 absolute on ln u1, i.e. sigma |g| eps-sized except for the rare u1 ~ 1).  Their sum is below
    # delta = 8 V eps, and a value within delta of an integer has probability <= 2 delta
    real = np.concatenate((ri, rq))
    delta = 8 * np.finfo(np.float32).eps * (np.abs(real).max() + 1)
    bound = 2 * delta
    frac = np.mean(got != ref)
    near = np.mean(np.abs(real - np.round(real)) < delta)
    assert frac <= bound and 1e-4 < bound < 2e-3, (frac, bound, near)



def test_ber_entries_reject_a_ppm_that_would_index_before_the_packet(rx):
    """m (1 + ppm 1e-6) must stay a sample index >= 0: ppm <= -1e6 or not finite is BTLE_EINVAL in both BER entries, before
    any launch, and the context stays usable."""
    import torch
    from btle_b200._native import BER_RESULT_DTYPE
    d = torch.zeros(BER_SAMPLES, dtype=torch.int16, device="cuda")
    dt = torch.zeros(40, dtype=torch.uint8, device="cuda")
    res = np.zeros(1, dtype=BER_RESULT_DTYPE)
    for ppm in (-1e6, -2e6, 1e6, float("nan"), float("inf"), float("-inf")):
        cfg = ber_cfg(1, 10.0, ppm)
        assert rx._L.btle_b200_ber_synth_device(rx._h, cfg.ctypes.data, 0, 1, d.data_ptr(), d.data_ptr(), dt.data_ptr(), None) == EINVAL
        assert rx._L.btle_b200_ber_run(rx._h, cfg.ctypes.data, 1, res.ctypes.data) == EINVAL
        assert b"ppm" in rx._L.btle_b200_last_error(rx._h)
    cfg = ber_cfg(1, float("nan"), 0.0)
    assert rx._L.btle_b200_ber_run(rx._h, cfg.ctypes.data, 1, res.ctypes.data) == EINVAL
    rx._check(rx._L.btle_b200_ber_run(rx._h, ber_cfg(1, 30.0, -50.0).ctypes.data, 64, res.ctypes.data))
    assert int(res["packets"][0]) == 64 and int(res["pkt_err"][0]) == 0

def score(recs, truth):
    """test_btle_ber.py:62-72 on model records: bit errors only in CRC-failed packets, an empty pdu counts all 312 bits"""
    bad = recs["crc_ok"] == 0
    nb = recs["n_pdu_bits"].astype(np.int64)
    common = np.minimum(nb, 312)
    a = np.unpackbits(recs["pdu"][:, :39], axis=1, bitorder="little")
    b = np.unpackbits(truth[:, :39], axis=1, bitorder="little")
    diff = ((a != b) & (np.arange(312)[None, :] < common[:, None])).sum(axis=1)
    err = np.where(nb == 0, 312, diff)
    return int(bad.sum()), int(err[bad].sum()), int((bad & (recs["found"] == 0)).sum())


# 0xF7CFF7CF is the whitened header 42 25 of channel 37 twice: one bit error in the first half of the access address and
# the receiver finds it 16 symbols late, in the header, so the CRC position is clamped and n_pdu_bits (321 - start) is
# below 312 and not a whole number of bytes -- the scorer's partial-byte mask is then used
AA_IN_HEADER = 0xF7CFF7CF


@pytest.mark.parametrize("ppm,snr,aa", [(0.0, 7.5, ADV_AA), (37.5, 13.5, ADV_AA), (0.0, 7.5, AA_IN_HEADER)])
def test_ber_run_equals_synth_model_rx_and_numpy_scoring(rx, ppm, snr, aa):
    """ber_synth_device -> model_rx_batch_device -> numpy scoring == btle_b200_ber_run's counters, exactly, for 32768 + 300
    packets (ber_run's batch boundary crossed; the synth here in other batches, with non-zero first packets), at SNRs where
    a large share of the packets fails (tests/golden/btlelib_ber.json: PER 0.69 at 8 dB, ppm 0)."""
    import torch
    from btle_b200._native import BER_RESULT_DTYPE, MODEL_REC_DTYPE
    seed, N = 4242, 32768 + 300
    cfg = ber_cfg(seed, snr, ppm, aa=aa)
    st = torch.cuda.Stream()
    recs, truths, win = [], [], None
    for first, n in ((0, 12000), (12000, 20768), (32768, 300)):
        with torch.cuda.stream(st):
            di, dq, dt = ber_synth(rx, cfg, first, n, stream=st)
            d_rec = torch.zeros((n, MODEL_REC_DTYPE.itemsize), dtype=torch.uint8, device="cuda")
        rx._check(rx._L.btle_b200_model_rx_batch_device(rx._h, di.data_ptr(), dq.data_ptr(), n, BER_SAMPLES, 8, 37, ADV_CRC, aa,
                                                        d_rec.data_ptr(), ctypes.c_void_p(st.cuda_stream)))
        st.synchronize()
        recs.append(d_rec.cpu().numpy().view(MODEL_REC_DTYPE).reshape(-1))
        truths.append(dt.cpu().numpy())
        if first == 32768:
            win = (di.cpu().numpy(), dq.cpu().numpy())
    recs, truth = np.concatenate(recs), np.concatenate(truths)
    pkt_err, bit_err, aa_miss = score(recs, truth)
    res = np.zeros(1, dtype=BER_RESULT_DTYPE)
    rx._check(rx._L.btle_b200_ber_run(rx._h, cfg.ctypes.data, N, res.ctypes.data))
    assert int(res["packets"][0]) == N
    assert (int(res["pkt_err"][0]), int(res["bit_err"][0]), int(res["aa_miss"][0])) == (pkt_err, bit_err, aa_miss)
    # the SNR gives failures in numbers: CRC failed with a PDU decoded (bit errors counted over it), and at ppm 0 also
    # access addresses lost (all 312 bits counted)
    bad = recs["crc_ok"] == 0
    partial = bad & (recs["found"] > 0)
    assert partial.sum() > 300 and pkt_err < 0.995 * N and (aa_miss > 100 or ppm != 0 or aa != ADV_AA), (aa_miss, partial.sum(), pkt_err)
    if aa == AA_IN_HEADER:
        nb = recs["n_pdu_bits"]
        odd = bad & (nb % 8 != 0) & (nb < 312)
        assert odd.sum() > 100, odd.sum()
    # >= 300 of the windows (the last batch, first packet 32768) against the port, record for record
    for k in range(300):
        e = P.rx_window(win[0][k], win[1][k], 37, ADV_CRC, aa)
        r = recs[32768 + k]
        assert (bool(r["crc_ok"]), int(r["payload_len"]), int(r["phase"]), int(r["found"]), int(r["start"])) == \
            (e["crc_ok"], e["plen"], e["phase"], e["found"], e["start"]), k
        nb = len(e["pdu_bit"])
        assert int(r["n_pdu_bits"]) == nb and np.array_equal(np.unpackbits(r["pdu"], bitorder="little")[:nb], e["pdu_bit"]), k


# ---- e. btle_rx_b200 --iq-bin16 ----------------------------------------------------------------------------------------
def test_cli_iq_bin16_prints_one_json_line_per_decoded_sps8_record(rx, tmp_path):
    rng = np.random.default_rng(21)
    plants, k = [], 40
    for j, (plen, flip) in enumerate([(6, False), (20, False), (37, False), (12, True), (31, False), (63, False), (9, True)]):
        if plen == 63:                                   # a length the window cannot hold: the CRC position is clamped
            pdu = bytes([0x40, 63]) + rng.integers(0, 256, 63, dtype=np.uint8).tobytes()
            b = P.tx_bits(pdu, 37)[8:]
        else:
            _, b = adv_packet(rng, plen, flip)
        plants += [(8 * k + p, b) for p in range(8)]
        k += 700
    iq = capture(8 * k + P.WINDOW, plants, rng)
    f = tmp_path / "cap.bin"
    iq.reshape(-1).tofile(f)
    recs = rx.rx_sps8(iq.reshape(-1), 37)
    exp = []
    for g in recs:
        r = g["rx"]
        if not r["found"] or r["n_pdu_bits"] < 16:
            continue
        have = int(r["n_pdu_bits"]) // 8
        b = np.zeros(42, np.uint8)
        b[:min(have, 39)] = r["pdu"][:min(have, 39)]
        plen = min(have - 2, int(b[1]) & 0x3F)
        exp.append(dict(ts=float(g["sample"]) / 8e6, crc_ok=bool(r["crc_ok"]), plen=plen, payload_hex=bytes(b[2:2 + plen]).hex()))
    assert len(exp) == 7 and sum(e["crc_ok"] for e in exp) == 4 and any(e["plen"] < 63 and e["plen"] > 37 for e in exp)
    p = subprocess.run([os.path.join(ROOT, "btle_b200", "btle_rx_b200"), "-c", "37", "-j", "-Q", "--iq-bin16", str(f)],
                       capture_output=True, text=True, timeout=300)
    assert p.returncode == 0, p.stdout + p.stderr
    pk = [json.loads(line) for line in p.stdout.splitlines() if line.startswith("{") and '"t":"pkt"' in line]
    assert len(pk) == len(exp)
    for got, e in zip(pk, exp):
        assert got["ts"] == pytest.approx(e["ts"], abs=1e-6) and got["crc_ok"] == e["crc_ok"], (got, e)
        assert got["plen"] == e["plen"] and got["payload_hex"] == e["payload_hex"], (got, e)
