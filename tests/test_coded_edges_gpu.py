"""The LE Coded PHY receiver (btle_b200_rx_coded*) at its kernel edges, pinned to coded_ref.py byte for byte: warps of
coded_decode_kernel that decode a second hit, hits on and around the seams of coded_search_kernel's tiles, a carrier
offset and a channel per capture in one call, poisoned device views and odd lengths, saturated IQ, capacity cuts, the
cfg cache under several CUDA streams, minimum and empty shapes, sample and byte offsets past 2^31, and captures of the
PER report's size.  Every CRC-ok and CRC-failed record of a packet that was sent is also checked without the restated
trellis: the survivor path its bytes code for has the record's metric, and the codeword sent has no higher one."""
import ctypes

import numpy as np
import pytest
import torch

import coded_ref as cr
from btle_b200 import make_cfgs, synth
from btle_b200._native import BTLE_EOVERFLOW, CFG_DTYPE, CFG_RSSI, CODED_REC_DTYPE
from test_coded_gpu import AA, _bursts, _packet_samples, _same, rx  # noqa: F401  (rx: the module's fixture)
from test_ingest_edges_gpu import _device_view, _walk

pytestmark = pytest.mark.gpu

TILE = 115 * 128                 # window starts of one coded_search_kernel CTA (kCodedGroups groups of 128 samples)
METRIC_BOUND = 2.2e6             # |metric| of the longest S=8 block 2 with every soft value saturated: 4166 * 508 < 2.2e6
REC = CODED_REC_DTYPE.itemsize


def _sort(recs):
    return np.sort(recs, order=["stream", "sample"])


def _sent_body(pdu, crc_init):
    crc = synth.crc24(pdu, crc_init)
    return pdu + bytes([crc & 0xFF, (crc >> 8) & 0xFF, crc >> 16])


def _expect(iqs, cfgs, offsets, sent=None):
    """coded_ref records of captures iqs [n, n_int8] (rows with equal content, cfg and offset are restated once), and
    the independent Viterbi checks of every record of a packet in sent[row] = [(n0, s, pdu)]"""
    memo, out = {}, []
    for k in range(len(iqs)):
        key = (iqs[k].tobytes(), cfgs[k].tobytes(), float(offsets[k]))
        if key not in memo:
            r = cr.rx_coded(iqs[k], cfgs[k:k + 1], offsets[k])
            if sent is not None:
                _check_paths(cr.Capture(iqs[k], float(offsets[k])), r, sent[k], cfgs[k])
            memo[key] = r
        r = memo[key].copy()
        r["stream"] = k
        out.append(r)
    return np.concatenate(out) if out else np.zeros(0, CODED_REC_DTYPE)


def _check_paths(cap, recs, sent, cfg):
    """For each record of a sent packet that went through the trellis (CRC ok or not): the decoded bytes, whitened and
    coded with TERM2, correlate with the soft values to exactly its metric (traceback and survivors), and the codeword
    sent does not correlate higher (the search maximises the metric)."""
    n_checked = 0
    for n0, s, pdu in sent:
        for r in recs[(np.abs(recs["sample"] - n0) <= 3) & (recs["s"] == s) & ((recs["flags"] & cr.TRUNCATED) == 0)]:
            nb = int(r["n_bytes"])
            assert cr.path_metric(cap, int(r["sample"]), s, bytes(r["bytes"][:nb]), int(cfg["channel"])) == r["metric"], r["sample"]
            if nb == len(pdu) + 3:
                body = _sent_body(pdu, int(cfg["crc_init"]))
                assert cr.path_metric(cap, int(r["sample"]), s, body, int(cfg["channel"])) <= r["metric"], r["sample"]
            n_checked += 1
    return n_checked


def _to_device(iq):
    """captures iq [n, n_int8] as a CUDA view whose rows start 16-byte aligned (a stride of n_int8 rounded up)"""
    ns, n = iq.shape
    d = torch.zeros((ns, max(16, (n + 15) // 16 * 16)), dtype=torch.int8, device="cuda")
    d[:, :n] = torch.from_numpy(np.ascontiguousarray(iq)).cuda()
    return d[:, :n]


def _device_run(rx, iq, cfgs, offsets, cap):
    """btle_b200_rx_coded_device over host captures iq [n, n_int8]; returns (count, the records it wrote)"""
    d_iq = _to_device(iq)
    d_out = torch.zeros(max(cap, 1) * REC, dtype=torch.uint8, device="cuda")
    d_count = torch.zeros(1, dtype=torch.int32, device="cuda")
    rx.rx_coded_device(d_iq, cfgs, d_out, d_count, offset_hz=offsets)
    torch.cuda.synchronize()
    c = int(d_count.item())
    return c, d_out[:min(c, cap) * REC].cpu().numpy().view(CODED_REC_DTYPE)


# ---- coded_decode_kernel: every warp decodes more than one hit ---------------------------------------------------------
REUSE_CHANNELS = [37, 38, 39, 0, 5, 17, 36, 22]
REUSE_AAS = [AA, 0x12345678, 0x50654E3A, 0x71764129, 0x2A3B4C5D, 0x6B7A8F91, 0x1C2D3E4F, 0x4E5F6071]
REUSE_CRCS = [0x555555, 0xABCDEF, 0x13579B, 0x000001, 0xFFFFFF, 0x2468AC, 0x0F0F0F, 0x7E57ED]
REUSE_HZ = [0.0, 40e3, -75e3, 125e3, -125e3, 10e3, -3e3, 90e3]
# (L, S, CI sent): long and empty PDUs at S=2 and S=8, and the two reserved CIs
REUSE_KINDS = [(255, 8, None), (0, 2, None), (0, 8, None), (0, 2, 2), (255, 2, None), (0, 8, 3), (37, 2, None), (0, 2, None),
               (1, 8, None), (0, 2, 3), (255, 2, None), (0, 8, 2)]


def _reuse_capture(k, rng):
    specs, n0 = [], 700
    for q in range(45):
        L, s, ci = REUSE_KINDS[(q + k) % len(REUSE_KINDS)]
        specs.append((n0 + (q + k) % 4, L, s, ci))
        n0 += _packet_samples(L, s) + 600
    bursts, pdus = _bursts(specs, rng, REUSE_CHANNELS[k], REUSE_CRCS[k], REUSE_AAS[k])
    sigma = cr.sigma_of(4.0, 100) if k % 2 else 0.0
    return cr.place(n0 + 1500, bursts, 100, sigma, rng, offset_hz=REUSE_HZ[k]), \
        [(n, s, p) for (n, _, s, ci), p in zip(specs, pdus) if ci is None]


def test_decode_loop_reuse(rx):
    """More hits than coded_decode_kernel has warps (16 CTAs of 4 warps per SM), so warps decode a second and third hit on
    the shared state of the first: long after empty and empty after long PDUs, S=2 after S=8, reserved CIs, and other
    channels (whitening), access addresses, CRC inits and rotations, on the host and the device call."""
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    rng = np.random.default_rng(31)
    caps, sent = zip(*[_reuse_capture(k, rng) for k in range(8)])
    n = max(c.size for c in caps)
    base = np.stack([np.pad(c, (0, n - c.size)) for c in caps])
    cfgs8 = make_cfgs(8, channel=REUSE_CHANNELS, access_addr=REUSE_AAS, crc_init=REUSE_CRCS, rssi=[CFG_RSSI, 0] * 4)
    hz8 = np.asarray(REUSE_HZ, np.float32)
    exp8 = _expect(base, cfgs8, hz8, sent)
    reps = -(-int(2.2 * 64 * sms) // exp8.size)                           # about 2.2 hits per warp
    iq = np.tile(base, (reps, 1))
    cfgs, hz = np.tile(cfgs8, reps), np.tile(hz8, reps)
    exp = np.concatenate([exp8] * reps)
    exp["stream"] = np.repeat(np.arange(reps) * 8, exp8.size) + exp["stream"]
    assert exp.size > 64 * sms, (exp.size, sms)
    assert (exp["s"] == 8).any() and (exp["s"] == 2).any() and (exp["flags"] & cr.CI_RESERVED).any()
    assert (exp["n_bytes"] == 260).any() and (exp["n_bytes"] == 5).any() and (exp["crc_bad"] == 1).any()
    _same(rx.rx_coded(iq, cfgs, offset_hz=hz, cap=exp.size + 100), exp)
    c, recs = _device_run(rx, iq, cfgs, hz, exp.size + 100)
    assert c == exp.size
    _same(_sort(recs), exp)


# ---- coded_search_kernel: tile seams, group boundaries, last tiles -----------------------------------------------------
def test_search_tile_seams(rx):
    """Bursts whose access address sits at TILE t + 128 g + delta, delta = -9..9 (every sample phase), for g = 0 (the tile
    seam), 1, 57 and 114 (the group in front of the next seam), noiseless (plateaus of equal D that cross the seam) and
    noisy; the hits near each seam are whatever the restatement finds there."""
    rng = np.random.default_rng(41)
    rows, sent, cfgs = [], [], []
    n = TILE * 21
    for g in (0, 1, 57, 114):
        for noisy in (False, True):
            specs = [(TILE * t + 128 * g + (t - 10), (3 * t) % 20, (2, 8)[t % 2], None) for t in range(1, 20)]
            bursts, pdus = _bursts(specs, rng)
            rows.append(cr.place(n, bursts, 100, cr.sigma_of(2.0, 100) if noisy else 0.0, rng))
            sent.append([(n0, s, p) for (n0, _, s, _), p in zip(specs, pdus)])
    iq = np.stack(rows)
    cfgs = make_cfgs(len(rows), channel=37, access_addr=AA, crc_init=0x555555, rssi=CFG_RSSI)
    hz = np.zeros(len(rows), np.float32)
    exp = _expect(iq, cfgs, hz, sent)
    near = exp[np.abs(exp["sample"] - TILE * np.round(exp["sample"] / TILE)) <= 8]
    assert sorted(set((near["sample"] % 4).tolist())) == [0, 1, 2, 3], near["sample"]
    _same(rx.rx_coded(iq, cfgs), exp)
    c, recs = _device_run(rx, iq, cfgs, None, exp.size)
    assert c == exp.size
    _same(_sort(recs), exp)


@pytest.mark.parametrize("groups_mod", [0, 1, 114])
def test_last_tile_shapes(rx, groups_mod):
    """Captures of 2 TILE + groups_mod groups of window starts (a full last tile, one group, all but one), with bursts on
    the last window starts and at the start of the last tile."""
    rng = np.random.default_rng(43 + groups_mod)
    groups = 2 * 115 + (groups_mod or 115)
    for extra in (0, 127):
        n = 1024 + 128 * (groups - 1) + extra
        last_tile = TILE * ((groups - 1) // 115)
        specs = [(last_tile + 5 - extra % 4, 12, 2, None), (n - 1024 - extra % 3, 40, 8, None)]
        if specs[1][0] - specs[0][0] < 9000:
            specs = specs[1:]
        specs = [(TILE - 3, 7, 8, None)] + specs
        bursts, _ = _bursts(specs, rng)
        iq = np.stack([cr.place(n, bursts), cr.place(n, bursts, 100, cr.sigma_of(0.0, 100), rng)])
        cfgs = make_cfgs(2, channel=37, access_addr=AA, crc_init=0x555555, rssi=CFG_RSSI)
        exp = cr.rx_coded(iq, cfgs)
        assert (n - 1024 - 128 < exp["sample"]).any()
        _same(rx.rx_coded(iq, cfgs), exp)
        c, recs = _device_run(rx, iq, cfgs, None, exp.size)
        assert c == exp.size
        _same(_sort(recs), exp)


# ---- rot[stream] and channel per capture ------------------------------------------------------------------------------
ROT_HZ = [0.0, 125e3, -125e3, 500e3, -500e3, 37e3]
ROT_CHANNELS = [37, 38, 39, 1, 2, 3]


def test_rotation_and_channel_per_capture(rx):
    """One call, a different carrier offset and channel on every capture (up to the largest offset accepted), the same
    PDUs at the same samples in each: taking one capture's rotation or channel for another changes the records."""
    rng = np.random.default_rng(51)
    specs, n0 = [], 800
    for k in range(8):
        specs.append((n0 + k % 4, 10 + 9 * k, (2, 8)[k % 2], None))
        n0 += _packet_samples(10 + 9 * k, (2, 8)[k % 2]) + 900
    pdus = [bytes([0x07, L]) + rng.integers(0, 256, L, dtype=np.uint8).tobytes() for _, L, _, _ in specs]
    rows, sent = [], []
    for ch, hz in zip(ROT_CHANNELS, ROT_HZ):
        bursts = [(n, synth.coded_air(p, ch, AA, 0x4A5B6C, s=s)) for (n, _, s, _), p in zip(specs, pdus)]
        rows.append(cr.place(n0 + 2000, bursts, 100, cr.sigma_of(6.0, 100), rng, offset_hz=hz))
        sent.append([(n, s, p) for (n, _, s, _), p in zip(specs, pdus)])
    iq = np.stack(rows)
    cfgs = make_cfgs(6, channel=ROT_CHANNELS, access_addr=AA, crc_init=0x4A5B6C, rssi=CFG_RSSI)
    hz = np.asarray(ROT_HZ, np.float32)
    exp = _expect(iq, cfgs, hz, sent)
    assert (exp["crc_bad"] == 0).sum() >= 6 * 7
    swapped_rot = cr.rx_coded(iq[1], cfgs[1:2], hz[0])
    swapped_ch = cr.rx_coded(iq[1], make_cfgs(1, channel=ROT_CHANNELS[0], access_addr=AA, crc_init=0x4A5B6C, rssi=CFG_RSSI), hz[1])
    mine = exp[exp["stream"] == 1].copy()
    mine["stream"] = 0
    assert swapped_rot.tobytes() != mine.tobytes() and swapped_ch.tobytes() != mine.tobytes()
    _same(rx.rx_coded(iq, cfgs, offset_hz=hz), exp)
    c, recs = _device_run(rx, iq, cfgs, hz, exp.size)
    assert c == exp.size
    _same(_sort(recs), exp)


# ---- bytes outside [0, n_int8) ------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n_int8", [2 * 1347 + 6, 2 * (TILE + 1700) + 10, 2 * (3 * TILE + 2300) + 2])
def test_poisoned_views(rx, n_int8):
    """Device views whose every byte outside [0, n_int8) is poison (0x7F or random), at 16-aligned offsets into their
    buffer with strides above n_int8, and n_int8 % 16 != 0: records == the restatement of the capture with zeros around
    it.  Bursts sit on the first window starts and on the last, truncated, so the decoder reads past the end."""
    rng = np.random.default_rng(n_int8)
    n = n_int8 // 2
    rows = []
    for s in range(3):
        specs = [(323 + s, 0, 2, None)] + ([(n - 1024 - s, 200, 2, None)] if n > 4000 else []) + \
            ([(n // 2 + s, 30, 8, None)] if n > 40000 else [])
        bursts, _ = _bursts(specs, rng)
        rows.append(cr.place(n, bursts, 100, cr.sigma_of(3.0, 100), rng))
    iqs = [np.concatenate([r, np.zeros(n_int8 - r.size, np.int8)]) for r in rows]   # n_int8 may be odd: no dangling byte
    cfgs = make_cfgs(3, channel=[37, 12, 39], access_addr=AA, crc_init=0x555555, rssi=CFG_RSSI)
    exp_all = cr.rx_coded(np.stack(rows), cfgs)
    assert (exp_all["flags"] & cr.TRUNCATED).any()
    for ns in (1, 2, 3):
        want = exp_all[exp_all["stream"] < ns]
        for front, extra, random in ((16, 16, True), (256, 48, False), (4096, 4096, True), (0, 4096, False)):
            stride = (n_int8 + 15) // 16 * 16 + extra
            buf, view = _device_view(iqs[:ns], stride, front, rng, random)
            d_out = torch.zeros(max(want.size, 1) * REC, dtype=torch.uint8, device="cuda")
            d_count = torch.zeros(1, dtype=torch.int32, device="cuda")
            rx.rx_coded_device(view, cfgs[:ns], d_out, d_count)
            torch.cuda.synchronize()
            assert int(d_count.item()) == want.size, (ns, front)
            _same(_sort(d_out[:want.size * REC].cpu().numpy().view(CODED_REC_DTYPE)), want)
            del buf, view


def test_odd_length_dangling_byte(rx):
    """A host capture of odd n_int8: the last byte is no sample, whatever it holds."""
    rng = np.random.default_rng(61)
    n = 40000
    (b,), _ = _bursts([(n - 1024, 60, 2, None)], rng)
    (a,), _ = _bursts([(5000, 20, 8, None)], rng)
    iq = cr.place(n, [a, b], 100, cr.sigma_of(5.0, 100), rng)
    exp = cr.rx_coded(iq, make_cfgs(1, rssi=CFG_RSSI))
    assert (exp["flags"] & cr.TRUNCATED).any()
    for last in (0x7F, -128, 0x55):
        odd = np.concatenate([iq, np.array([last], np.int8)])
        _same(rx.rx_coded(odd, make_cfgs(1, rssi=CFG_RSSI)), exp)
        buf, view = _device_view([odd], odd.size + 15 & ~15, 16, rng, True)
        d_out = torch.zeros(max(exp.size, 1) * REC, dtype=torch.uint8, device="cuda")
        d_count = torch.zeros(1, dtype=torch.int32, device="cuda")
        rx.rx_coded_device(view, make_cfgs(1, rssi=CFG_RSSI), d_out, d_count)
        torch.cuda.synchronize()
        assert int(d_count.item()) == exp.size
        _same(_sort(d_out[:exp.size * REC].cpu().numpy().view(CODED_REC_DTYPE)), exp)


# ---- saturated input: the discriminator's clamp and the metric's range ------------------------------------------------
CORNERS = np.array([(127, 127), (-128, 127), (-128, -128), (127, -128)], np.int64)   # counter-clockwise


def _corner_capture(n, n0, syms):
    """IQ that sits on a corner of the int8 square for 4 samples per symbol and turns a quarter counter-clockwise after
    a 1 and clockwise after a 0, where |v| = 16384 * 32640 or 32385, y = +-126 or +-127, and v >> 22 of the largest
    negative v is -128.  D is 0 on four sample phases; the hit rule takes the first, n0 - 1, whose F mixes two corners
    in the preamble and the access address.  So from block 2 on the corners sit one sample earlier, where the soft
    values read at n0 - 1 + 4 j see two whole corners: every one of them is saturated."""
    x = np.zeros((n, 2), np.int64)
    c = 0
    for j, b in enumerate(list(syms) + [0], start=-80):
        lo = n0 + 4 * j - 3 - (j >= 256)
        x[max(lo, 0):max(lo + 4, 0)] = CORNERS[c]
        c = (c + (1 if b else -1)) % 4
    return x.astype(np.int8).reshape(-1)


def test_saturated_input(rx):
    """Square-wave corner IQ (|v| up to 2^29, y at +127 and at the -127 clamp of -128) carrying an L=255 S=8 packet whose
    metric comes near the metric bound, decoded at 0 and +-125 kHz; the same turned by +-125 kHz; and full-scale GFSK
    bursts clipped at -128/127 by noise."""
    rng = np.random.default_rng(71)
    pdu = bytes([0x07, 255]) + rng.integers(0, 256, 255, dtype=np.uint8).tobytes()
    syms, _ = synth.coded_symbols(pdu, 37, AA, 0x555555, s=8)
    n0 = 1000
    n = n0 + 4 * (syms.size - 80) + 2000
    corner = _corner_capture(n, n0, syms)
    xs = corner.astype(np.float64).reshape(-1, 2)
    z = xs[:, 0] + 1j * xs[:, 1]

    def turn(hz):
        w = z * np.exp(2j * np.pi * hz / 4e6 * np.arange(n))
        return np.clip(np.round(np.stack([w.real, w.imag], axis=1)), -128, 127).astype(np.int8).reshape(-1)
    turned = [turn(125e3), turn(-125e3)]
    specs = [(1500 + 9000 * k + k % 4, 20 + k, (2, 8)[k % 2], None) for k in range(6)]
    bursts, pdus = _bursts(specs, rng)
    loud = [cr.place(n, bursts, 127, cr.sigma_of(8.0, 127), rng), cr.place(n, bursts, 190, cr.sigma_of(12.0, 190), rng)]
    iq = np.stack([corner, corner, corner] + turned + loud)
    hz = np.asarray([0.0, 125e3, -125e3, 125e3, -125e3, 0.0, 0.0], np.float32)
    cfgs = make_cfgs(iq.shape[0], channel=37, access_addr=AA, crc_init=0x555555, rssi=CFG_RSSI)
    body = [(n0, 8, pdu)]
    exp = _expect(iq, cfgs, hz, [body] * 5 + [[(a, s, p) for (a, _, s, _), p in zip(specs, pdus)]] * 2)
    cap = cr.Capture(corner)
    v = cap.v_at(n0 - 1 + 4 * np.arange(296, 296 + 2083 * 8))
    assert v.max() >> 22 == 127 and v.min() >> 22 == -128 and np.abs(v).max() >= 0.99 * 2 ** 29
    r = exp[(exp["stream"] == 0) & (exp["sample"] == n0 - 1)]
    assert r.size == 1 and r[0]["crc_bad"] == 0 and bytes(r[0]["bytes"][:257]) == pdu
    assert 0.9 * METRIC_BOUND < r[0]["metric"] < METRIC_BOUND
    assert np.abs(exp["metric"]).max() < METRIC_BOUND
    assert (exp[exp["stream"] >= 5]["crc_bad"] == 0).sum() >= 10
    assert (loud[0] == -128).any() and (loud[1] == 127).any()
    _same(rx.rx_coded(iq, cfgs, offset_hz=hz), exp)
    c, recs = _device_run(rx, iq, cfgs, hz, exp.size)
    assert c == exp.size
    _same(_sort(recs), exp)


# ---- capacity cuts ------------------------------------------------------------------------------------------------------
def test_capacity_cuts(rx):
    """cap below the count: the count is exact, the records written are whole records of distinct hits (each equal to
    the restatement's record at its sample), nothing past cap is written; the host call returns BTLE_EOVERFLOW with
    its cap records in (stream, sample) order."""
    rng = np.random.default_rng(81)
    rows = []
    for s in range(3):
        specs = [(700 + 3600 * k + (k + s) % 4, (5 * k) % 30, 2, (None, None, 2)[k % 3]) for k in range(14)]
        bursts, _ = _bursts(specs, rng)
        rows.append(cr.place(700 + 3600 * 14 + 2000, bursts, 100, cr.sigma_of(8.0, 100), rng))
    iq = np.stack(rows)
    cfgs = make_cfgs(3, channel=37, access_addr=AA, crc_init=0x555555, rssi=CFG_RSSI)
    exp = cr.rx_coded(iq, cfgs)
    count = exp.size
    assert count >= 40
    keyed = {(int(r["stream"]), int(r["sample"])): r for r in exp}
    d_iq = _to_device(iq)
    ns, n = iq.shape
    for cap in (1, count // 2, count - 1):
        d_buf = torch.full(((cap + 16) * REC,), 0xA5, dtype=torch.uint8, device="cuda")
        d_count = torch.zeros(1, dtype=torch.int32, device="cuda")
        rx.rx_coded_device(d_iq, cfgs, d_buf[:cap * REC], d_count)
        torch.cuda.synchronize()
        assert int(d_count.item()) == count
        host = d_buf.cpu().numpy()
        assert (host[cap * REC:] == 0xA5).all(), cap
        got = host[:cap * REC].view(CODED_REC_DTYPE)
        keys = [(int(r["stream"]), int(r["sample"])) for r in got]
        assert len(set(keys)) == cap
        for k, r in zip(keys, got):
            assert r.tobytes() == keyed[k].tobytes(), k
        out = np.frombuffer(np.full((cap + 16) * REC, 0xA5, np.uint8).tobytes(), CODED_REC_DTYPE).copy()
        n_out = ctypes.c_size_t(0)
        rc = rx._L.btle_b200_rx_coded(rx._h, iq.ctypes.data, ns, n, n, cfgs.ctypes.data, None, out.ctypes.data, cap, ctypes.byref(n_out))
        assert rc == BTLE_EOVERFLOW and n_out.value == count
        assert (out[cap:].view(np.uint8) == 0xA5).all()
        keys = [(int(r["stream"]), int(r["sample"])) for r in out[:cap]]
        assert keys == sorted(set(keys)) and len(keys) == cap
        for k, r in zip(keys, out[:cap]):
            assert r.tobytes() == keyed[k].tobytes(), k


# ---- the cfg cache under pressure ---------------------------------------------------------------------------------------
def test_cfg_cache_under_pressure(rx):
    """Six distinct cfg/offset arrays, coded launches on five CUDA streams back to back with no host sync, each followed
    by a 1M launch (btle_b200_rx_device_dir) of the same cfg bytes, which takes the unrotated cache key; one sync at the
    end, then every output is checked."""
    rng = np.random.default_rng(91)
    iq1m, _ = synth.make_adv_stream(16 * 16384, seed=13, channel=37, corrupt_every=5, slot_samples=3000)
    iq1m = iq1m.numpy()
    arrays = []
    for k in range(6):
        ns = 1 + k % 3
        cfgs = make_cfgs(ns, channel=[(37, 38, 39)[(k + s) % 3] for s in range(ns)], access_addr=synth.ADV_ACCESS_ADDR,
                         crc_init=[0x555555 ^ (k << 4) ^ s for s in range(ns)], rssi=CFG_RSSI if k % 2 else 0)
        hz = np.asarray([25e3 * (k + 1) * (-1) ** s for s in range(ns)], np.float32)
        rows = []
        for s in range(ns):
            specs = [(900 + 6400 * q + (q + k) % 4, (4 * q + k) % 12, (2, 8)[(q + s) % 2], None) for q in range(6)]
            bursts, _ = _bursts(specs, rng, int(cfgs[s]["channel"]), int(cfgs[s]["crc_init"]), synth.ADV_ACCESS_ADDR)
            rows.append(cr.place(900 + 6400 * 6 + 4000, bursts, 100, cr.sigma_of(6.0, 100), rng, offset_hz=float(hz[s])))
        iq = np.stack(rows)
        arrays.append((cfgs, hz, iq, cr.rx_coded(iq, cfgs, hz), rx.rx_batch(np.stack([iq1m] * ns), cfgs)))
    assert len({c.tobytes() + h.tobytes() for c, h, *_ in arrays}) == 6
    streams = [torch.cuda.Stream() for _ in range(5)]
    launches = []
    for rnd in range(2):
        for k, (cfgs, hz, iq, exp, exp1m) in enumerate(arrays):
            ns = cfgs.size
            d_iq = _to_device(iq)
            d_out = torch.zeros(max(exp.size, 1) * REC, dtype=torch.uint8, device="cuda")
            d_count = torch.zeros(1, dtype=torch.int32, device="cuda")
            d_iq1 = torch.from_numpy(np.stack([iq1m] * ns)).cuda()
            units = rx.units(ns, iq1m.size)
            d_out1 = torch.zeros(max(exp1m.size, 1) * 64, dtype=torch.uint8, device="cuda")
            d_dir = torch.zeros((units, 2), dtype=torch.int32, device="cuda")
            d_count1 = torch.zeros(1, dtype=torch.int32, device="cuda")
            launches.append((k, d_iq, d_out, d_count, d_iq1, d_out1, d_dir, d_count1, units))
    torch.cuda.synchronize()
    for i, (k, d_iq, d_out, d_count, d_iq1, d_out1, d_dir, d_count1, units) in enumerate(launches):
        cfgs, hz = arrays[k][:2]
        st = streams[i % 5].cuda_stream
        rx.rx_coded_device(d_iq, cfgs, d_out, d_count, stream_ptr=st, offset_hz=hz)
        rx.rx_device_dir(d_iq1, cfgs, d_out1, d_count1, d_dir, st)
    torch.cuda.synchronize()
    for k, d_iq, d_out, d_count, d_iq1, d_out1, d_dir, d_count1, units in launches:
        exp, exp1m = arrays[k][3:]
        assert int(d_count.item()) == exp.size
        _same(_sort(d_out[:exp.size * REC].cpu().numpy().view(CODED_REC_DTYPE)), exp)
        assert int(d_count1.item()) == exp1m.size
        got1m, _ = _walk(rx, d_out1, d_dir, units)
        assert got1m.tobytes() == exp1m.tobytes(), k


# ---- shapes -------------------------------------------------------------------------------------------------------------
def test_minimum_and_empty_shapes(rx):
    rng = np.random.default_rng(101)
    (b,), _ = _bursts([(0, 0, 2, None)], rng)
    cfg = make_cfgs(1, rssi=CFG_RSSI)
    for n, want in ((1346, 0), (1347, 1)):
        iq = cr.place(n, [(323, b[1])])
        exp = cr.rx_coded(iq, cfg)
        assert exp.size == want and (want == 0 or exp[0]["sample"] == 323)
        _same(rx.rx_coded(iq, cfg), exp)
        c, recs = _device_run(rx, iq[None, :], cfg, None, 4)
        assert c == want
        _same(_sort(recs), exp)
    none = np.zeros(0, CFG_DTYPE)
    assert rx.rx_coded(np.zeros((0, 4096), np.int8), none).size == 0
    assert rx.rx_coded(np.zeros((2, 0), np.int8), make_cfgs(2)).size == 0
    for ns, n in ((0, 4096), (2, 0), (3, 16)):
        d_out = torch.zeros(4 * REC, dtype=torch.uint8, device="cuda")
        d_count = torch.full((1,), 7, dtype=torch.int32, device="cuda")
        rx.rx_coded_device(_to_device(np.zeros((ns, n), np.int8)), make_cfgs(ns) if ns else none, d_out, d_count)
        torch.cuda.synchronize()
        assert int(d_count.item()) == 0 and not d_out.any()


def test_many_short_streams(rx):
    """300 captures of 2000 samples (window starts 323..976), one burst each at every phase, most of them truncated."""
    rng = np.random.default_rng(111)
    distinct, sent = [], []
    for k in range(30):
        n0 = 323 + (k * 23) % 654
        specs = [(n0, k % 3, (2, 8)[k % 2], None)]
        bursts, pdus = _bursts(specs, rng, 37, 0x555555)
        distinct.append(cr.place(2000, bursts, 100, cr.sigma_of(10.0, 100) if k % 3 == 2 else 0.0, rng))
    iq = np.stack(distinct * 10)
    cfgs = make_cfgs(300, channel=37, access_addr=AA, crc_init=0x555555, rssi=CFG_RSSI)
    exp = _expect(iq, cfgs, np.zeros(300, np.float32))
    assert exp.size >= 300 and set(np.unique(exp["stream"]).tolist()) == set(range(300))
    _same(rx.rx_coded(iq, cfgs), exp)
    c, recs = _device_run(rx, iq, cfgs, None, exp.size)
    assert c == exp.size
    _same(_sort(recs), exp)


# ---- sample indices and byte offsets past 2^31 ------------------------------------------------------------------------
def test_offsets_past_2_31(rx):
    """Two streams of 2^30 + 2^20 samples in one zero-filled device buffer (stream 1 starts past byte 2^31), bursts around
    sample 2^30 and on the last window starts.  Zero IQ gives D = 168 > 96, so the records are the restatement's on
    slices around the bursts, moved to their absolute samples."""
    n = (1 << 30) + (1 << 20)
    n_int8 = 2 * n
    stride = n_int8 + 4096
    assert stride > 1 << 31
    rng = np.random.default_rng(121)
    cfgs = make_cfgs(2, channel=[37, 9], access_addr=[AA, 0x12345678], crc_init=[0x555555, 0x0BCDEF], rssi=CFG_RSSI)
    buf = torch.zeros(2 * stride, dtype=torch.int8, device="cuda")
    view = buf.view(2, stride)[:, :n_int8]
    exp = []
    for s in range(2):
        c = cfgs[s]
        for n0, L, sp in (((1 << 30) - 3000 + s, 30, 8), ((1 << 30) + 40000 + 2 * s, 100, 2), (n - 1024 - s, 255, 2)):
            (b,), _ = _bursts([(n0, L, sp, None)], rng, int(c["channel"]), int(c["crc_init"]), int(c["access_addr"]))
            a = n0 - synth.CODED_AA_SAMPLE - 2000
            e = min(n, n0 + _packet_samples(L, sp) + 2000)
            piece = cr.place(e - a, [(n0 - a, b[1])], 100, cr.sigma_of(6.0, 100), rng)
            view[s, 2 * a:2 * e] = torch.from_numpy(piece).cuda()
            r = cr.rx_coded(piece, cfgs[s:s + 1])
            r["sample"] += a
            r["stream"] = s
            r["flags"] &= ~np.uint8(cr.TRUNCATED if e < n else 0)
            exp.append(r)
    exp = _sort(np.concatenate(exp))
    assert (exp["sample"] > 1 << 30).any() and exp["sample"].max() >= n - 1025
    d_out = torch.zeros(64 * REC, dtype=torch.uint8, device="cuda")
    d_count = torch.zeros(1, dtype=torch.int32, device="cuda")
    rx.rx_coded_device(view, cfgs, d_out, d_count)
    torch.cuda.synchronize()
    assert int(d_count.item()) == exp.size
    _same(_sort(d_out[:exp.size * REC].cpu().numpy().view(CODED_REC_DTYPE)), exp)
    del view, buf
    torch.cuda.empty_cache()


# ---- captures of the PER report's size ----------------------------------------------------------------------------------
def _report_capture(waves, snr_db, seed):
    """tools/coded_ber_report.py's layout: bursts 1000 samples apart at all four phases, noise as rx_ber_run"""
    starts, pos = [], 500
    for k, w in enumerate(waves):
        starts.append(pos + k % 4)
        pos += w.size // 2 + 1000 + 4
    x = np.zeros((pos + 2000, 2))
    for s, w in zip(starts, waves):
        x[s:s + w.size // 2] += w.astype(np.float64).reshape(-1, 2) * 100 / 127
    x += np.random.default_rng(seed).normal(0.0, cr.sigma_of(snr_db, 100), x.shape)
    return np.clip(np.round(x), -128, 127).astype(np.int8).reshape(-1), np.array(starts) + synth.CODED_AA_SAMPLE


def _report_pdus():
    """the report's PDUs and noise seeds for --seed 1 --packets 400 (one draw per SNR point and way: S=8, S=2, 1M)"""
    rng = np.random.default_rng(1)
    pdus = [synth.adv_pdu(2, 1, 0, rng.integers(0, 256, int(L), dtype=np.uint8).tobytes()) for L in rng.integers(6, 38, 400)]
    return pdus, [int(rng.integers(1 << 30)) for _ in range(36)]


@pytest.mark.parametrize("s,point", [(2, 11), (2, 3), (8, 11)])
def test_report_sized_captures(rx, s, point):
    """400 packets at 10 dB through rx_coded's default cap (below the count: the call overflows and is made again), equal
    to the restatement.  The S=2 capture of the 12th SNR point loses packet 205 in both: a noise burst flips a run of
    coded-bit signs, and the path decoded has a higher metric (14607) than the codeword sent (14599), so the decision is
    the maximum-likelihood one."""
    pdus, seeds = _report_pdus()
    waves = [synth.coded_air(p, 37, s=s) for p in pdus]
    iq, n0s = _report_capture(waves, 10.0, seeds[3 * point + (1 if s == 2 else 0)])
    cfg = make_cfgs(1, channel=37)
    exp = cr.rx_coded(iq, cfg)
    if s == 2:
        assert iq.size // 65536 * 4 + 68 < exp.size                        # the default cap overflows
    got = rx.rx_coded(iq, cfg)
    _same(got, exp)
    cap = cr.Capture(iq)
    assert _check_paths(cap, exp, [(int(a), s, p) for a, p in zip(n0s, pdus)], cfg[0]) >= 400
    ok = exp[exp["crc_bad"] == 0]
    lost = [k for k, (a, p) in enumerate(zip(n0s, pdus))
            if not any(bytes(r["bytes"][:len(p)]) == p for r in ok[np.abs(ok["sample"] - a) <= 3])]
    assert lost == ([205] if (s, point) == (2, 11) else []), lost
