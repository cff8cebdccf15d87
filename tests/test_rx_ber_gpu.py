"""Error rates of the 4-Msps receive chain on the device (btle_b200_rx_ber_run, _synth_device, _score_device) against the
numpy restatement (tests/rx_ber_ref.py), the transmit modulator, the unmodified reference receiver and the numpy scoring:
the capture byte for byte where it is exact, the channel within float32 rounding, the reference's records and counters
exactly, the composition of the entry points across batches, streams and split points, and the argument edges."""
import ctypes

import numpy as np
import pytest
import torch

import orc
import rx_ber_ref as R
from btle_b200 import ber, synth
from btle_b200._native import REC_DTYPE, DIR_DTYPE, RX_BER_COUNTERS, RX_BER_RESULT_DTYPE, RX_BER_TRUTH_DTYPE

pytestmark = pytest.mark.gpu
EINVAL = -1
DATA_AA, DATA_CRC = 0x50654A21, 0x1A2B3C


@pytest.fixture(scope="module")
def rx():
    import __graft_entry__ as ge
    ge.build()
    from btle_b200 import BtleRx
    return BtleRx(0)


def cfg_of(snr, ppm=0.0, cfo=0.0, amp=64, slot=2048, channel=37, seed=1):
    adv = channel >= 37
    return ber.rx_ber_cfg(snr, ppm, cfo, amp, slot, channel, 0x555555 if adv else DATA_CRC, 0x8E89BED6 if adv else DATA_AA, seed)


def synth_dev(rx, cfg, first, n, stream=None):
    st = stream or torch.cuda.current_stream()
    n_int8 = R.capture_int8(n, int(cfg["slot_samples"][0]))
    with torch.cuda.stream(st):
        d_iq = torch.full((max(n_int8, 16),), 99, dtype=torch.int8, device="cuda")
        d_truth = torch.zeros((max(n, 1), 64), dtype=torch.uint8, device="cuda")
    rx._check(rx._L.btle_b200_rx_ber_synth_device(rx._h, cfg.ctypes.data, first, n, d_iq.data_ptr(), d_truth.data_ptr(),
                                                  ctypes.c_void_p(st.cuda_stream)))
    st.synchronize()
    return d_iq[:n_int8], d_truth


def truth_of(d_truth, n):
    return d_truth[:n].cpu().numpy().reshape(-1).view(RX_BER_TRUTH_DTYPE)[:n]


def decode(rx, d_iq, cfg, stream=None):
    """rx_device_dir with BTLE_CFG_REPORT_REJECTED on the capture: (records in reference order, device records, device
    directory, units)"""
    st = stream or torch.cuda.current_stream()
    from btle_b200.rx import make_cfgs
    c = cfg[0]
    cfgs = make_cfgs(1, channel=int(c["channel"]), access_addr=int(c["access_addr"]), crc_init=int(c["crc_init"]), rssi=2)
    n = d_iq.numel()
    units = rx.units(1, n)
    cap = (n // 16384) * 123 + 1
    with torch.cuda.stream(st):
        d_out = torch.zeros(cap * 64, dtype=torch.uint8, device="cuda")
        d_dir = torch.zeros(max(units, 1) * 8, dtype=torch.uint8, device="cuda")
    rx.rx_device_dir(d_iq.view(1, -1), cfgs, d_out, None, d_dir, stream_ptr=st.cuda_stream)
    st.synchronize()
    recs = rx.gather_ordered(d_out.cpu().numpy().view(REC_DTYPE), d_dir.cpu().numpy().view(DIR_DTYPE)[:units])
    return recs, d_out, d_dir, units


def score_dev(rx, d_truth, n, d_out, d_dir, units, stream=None):
    st = stream or torch.cuda.current_stream()
    with torch.cuda.stream(st):
        d_res = torch.zeros(RX_BER_RESULT_DTYPE.itemsize, dtype=torch.uint8, device="cuda")
    rx._check(rx._L.btle_b200_rx_ber_score_device(rx._h, d_truth.data_ptr(), n, d_out.data_ptr(), d_out.numel() // 64, d_dir.data_ptr(), units,
                                                  d_res.data_ptr(), ctypes.c_void_p(st.cuda_stream)))
    st.synchronize()
    r = d_res.cpu().numpy().view(RX_BER_RESULT_DTYPE)[0]
    return {k: int(r[k]) for k in RX_BER_COUNTERS}


def run(rx, cfg, n):
    res = np.zeros(1, dtype=RX_BER_RESULT_DTYPE)
    rx._check(rx._L.btle_b200_rx_ber_run(rx._h, cfg.ctypes.data, n, res.ctypes.data))
    return {k: int(res[k][0]) for k in RX_BER_COUNTERS}


def assert_truth_equal(got, exp):
    for f in ("aa_sample", "offset", "n_bytes", "delta4", "pdu"):
        assert np.array_equal(got[f], exp[f]), f


# ---- 1. noiseless, ppm 0, delta 0: the modulator's samples, scaled, at the truth's offsets -----------------------------
@pytest.mark.parametrize("channel,amp", [(37, 64), (38, 127), (9, 23)])
def test_noiseless_capture_is_the_scaled_modulator_output(rx, channel, amp):
    cfg = cfg_of(1000.0, amp=amp, slot=1800, channel=channel, seed=11 + channel)
    first, n = 5000, 96
    d_iq, d_truth = synth_dev(rx, cfg, first, n)
    iq = d_iq.cpu().numpy().reshape(-1, 2)
    truth = truth_of(d_truth, n)
    _, exp, _ = R.capture(cfg[0], first, n)
    assert_truth_equal(truth, exp)
    assert int(truth["clipped"].sum()) == 0 and set(truth["delta4"]) == {0, 1, 2, 3}
    air = np.stack([np.frombuffer(synth.air_bytes(bytes(t["pdu"][:t["n_bytes"]]), channel, int(cfg["access_addr"][0]), int(cfg["crc_init"][0])),
                                  dtype=np.uint8) for t in truth])
    w = synth.modulate_batch_cuda(torch.from_numpy(air).cuda(), torch.full((n,), air.shape[1], dtype=torch.int32), sps=4)
    w = w.cpu().numpy().reshape(n, -1, 2)
    L = R.packet_len(channel)
    assert w.shape[1] == L
    scaled = np.rint(w.astype(np.float32) * (np.float32(amp) / np.float32(127))).astype(np.int8)
    S = 1800
    for k in np.nonzero(truth["delta4"] == 0)[0]:
        slot = iq[k * S:(k + 1) * S]
        o = int(truth["offset"][k])
        assert np.array_equal(slot[o:o + L], scaled[k]) and not slot[:o].any() and not slot[o + L:].any(), k
    assert not iq[n * S:].any()                                                      # the rounding-up tail: noise, here 0
    recs, d_out, d_dir, units = decode(rx, d_iq, cfg)
    c = R.score(recs, truth)
    assert (c["pkt_err"], c["crc_ok_wrong"], c["extra_recs"], c["aa_miss"]) == (0, 0, 0, 0), c
    assert score_dev(rx, d_truth, n, d_out, d_dir, units) == c


# ---- 2. the channel against the float64 restatement --------------------------------------------------------------------
@pytest.mark.parametrize("snr,ppm,cfo,amp,channel", [(8.0, 0.0, 0.0, 64, 37), (3.0, 20.0, 0.0, 100, 38), (12.0, -50.0, 30000.0, 64, 39),
                                                     (0.0, 35.0, -60000.0, 127, 7), (20.0, 0.0, 150000.0, 40, 22)])
def test_channel_equals_float64_restatement(rx, snr, ppm, cfo, amp, channel):
    """Every sample equals the restatement's rint + saturation, except where the kernel's float32 arithmetic moves a
    value across a rounding boundary (x.5).  Per sample, the float32 error terms (interpolation of the scaled table,
    rotation angle cast to float and sincospif, sigma from exp10f, sigma g and the final sum, __logf in Box-Muller) stay
    below tol = 64 eps (V + 1), V = the largest |value|, so every differing sample lies within tol of a boundary, differs
    by 1, and their share is at most about 2 tol (uniform fractions)."""
    cfg = cfg_of(snr, ppm, cfo, amp, slot=1700, channel=channel, seed=21)
    first, n = 123456, 64
    d_iq, d_truth = synth_dev(rx, cfg, first, n)
    got = d_iq.cpu().numpy().reshape(-1, 2).astype(np.int64)
    exp_iq, exp_truth, real = R.capture(cfg[0], first, n)
    truth = truth_of(d_truth, n)
    assert_truth_equal(truth, exp_truth)
    exp = exp_iq.reshape(-1, 2).astype(np.int64)
    tol = 64 * np.finfo(np.float32).eps * (np.abs(real).max() + 1)
    bad = got != exp
    assert np.abs(got - exp).max() <= 1
    near = np.abs(np.abs(real - np.floor(real)) - 0.5) < tol
    assert not (bad & ~near).any(), real[bad & ~near][:8]
    assert bad.mean() <= 2 * tol + 1e-4, (bad.mean(), tol)
    assert abs(int(truth["clipped"].sum()) - int(exp_truth["clipped"].sum())) <= int(bad.any(axis=1).sum())
    if amp == 127 and snr == 0.0:
        assert int(truth["clipped"].sum()) > 0


# ---- 3. the unmodified reference receiver on the same captures ---------------------------------------------------------
def failing_snrs(rx, cfg_fn, lo=10.0, hi=36.0):
    """about three SNRs where 10-70 % of the packets fail (found with rx_ber_run on 2000 packets)"""
    pts = []
    for s in np.arange(lo, hi, 1.0):
        c = run(rx, cfg_fn(float(s)), 2000)
        if 0.1 <= c["pkt_err"] / 2000 <= 0.7:
            pts.append(float(s))
    assert len(pts) >= 3, pts
    return [pts[0], pts[len(pts) // 2], pts[-1]]


@pytest.mark.skipif(not orc.ref_available(), reason="oracle/_ref not built")
@pytest.mark.parametrize("channel,ppm", [(37, 0.0), (39, 20.0), (17, 0.0)])
def test_reference_receiver_records_and_counts_equal_the_gpu_path(rx, channel, ppm):
    n = 600
    for snr in failing_snrs(rx, lambda s: cfg_of(s, ppm, channel=channel, seed=31)):
        cfg = cfg_of(snr, ppm, channel=channel, seed=31)
        d_iq, d_truth = synth_dev(rx, cfg, 0, n)
        truth = truth_of(d_truth, n)
        recs, d_out, d_dir, units = decode(rx, d_iq, cfg)
        ref = orc.ref_rx_stream(d_iq.cpu().numpy(), channel=channel, access_addr=int(cfg["access_addr"][0]), crc_init=int(cfg["crc_init"][0]),
                                report_rejected=1)
        orc.assert_same_as_ref(recs, ref)
        c = R.score_ref(ref, truth)
        assert 0.05 * n <= c["pkt_err"] <= 0.8 * n, (snr, c)
        assert run(rx, cfg, n) == c == score_dev(rx, d_truth, n, d_out, d_dir, units) == R.score(recs, truth)


# ---- 4. composition -----------------------------------------------------------------------------------------------------
def test_run_equals_synth_receive_and_numpy_scoring_across_a_batch(rx):
    """rx_ber_run over more packets than one of its batches holds (at most 8192 chunks: 32768 packets of 2048 samples)
    equals the one long capture from btle_b200_rx_ber_synth_device, decoded by rx_device_dir on a side stream and scored
    in numpy and by btle_b200_rx_ber_score_device; and runs split at arbitrary packets add up to it (a split moves the chunk
    boundaries, which changes records only through a 32-bit access-address match in noise or payload next to a boundary)."""
    N = 32768 + 700
    cfg = cfg_of(20.0, seed=41)
    side = torch.cuda.Stream()
    d_iq, d_truth = synth_dev(rx, cfg, 0, N, stream=side)
    truth = truth_of(d_truth, N)
    recs, d_out, d_dir, units = decode(rx, d_iq, cfg, stream=side)
    c = R.score(recs, truth)
    assert 0.01 * N < c["pkt_err"] < 0.99 * N, c
    assert run(rx, cfg, N) == c == score_dev(rx, d_truth, N, d_out, d_dir, units, stream=side)
    del d_iq, d_out
    total = dict.fromkeys(RX_BER_COUNTERS, 0)
    for first, n in ((0, 777), (777, 20000), (20777, N - 20777)):
        d_iq, d_truth = synth_dev(rx, cfg, first, n, stream=side)
        assert_truth_equal(truth_of(d_truth, n)[:50], R.capture(cfg[0], first, 50)[1])
        recs, d_out, d_dir, units = decode(rx, d_iq, cfg, stream=side)
        s = score_dev(rx, d_truth, n, d_out, d_dir, units, stream=side)
        assert s == R.score(recs, truth_of(d_truth, n))
        total = R.add(total, s)
    assert total == c


def test_run_is_reproducible_with_a_slot_that_does_not_divide_a_chunk(rx):
    """an odd slot: rx_ber_run's batches are 8192 slots (7996 chunks of 1999 samples) long, and its second batch still
    equals the long capture"""
    cfg = cfg_of(20.0, 10.0, 2000.0, slot=1999, seed=43)
    N = 32768 + 100
    a, b = run(rx, cfg, N), run(rx, cfg, N)
    assert a == b and a["packets"] == N
    d_iq, d_truth = synth_dev(rx, cfg, 0, N)
    recs, *_ = decode(rx, d_iq, cfg)
    assert R.score(recs, truth_of(d_truth, N)) == a


# ---- 5. edges -----------------------------------------------------------------------------------------------------------
def test_argument_errors_leave_the_context_usable(rx):
    d_iq = torch.zeros(1 << 16, dtype=torch.int8, device="cuda")
    d_truth = torch.zeros(64 * 4, dtype=torch.uint8, device="cuda")
    res = np.zeros(1, dtype=RX_BER_RESULT_DTYPE)
    bad = [dict(snr=float("nan")), dict(snr=float("inf")), dict(snr=float("-inf")), dict(ppm=float("nan")), dict(ppm=float("inf")),
           dict(ppm=1e6), dict(ppm=-1e6), dict(ppm=-2e6), dict(cfo=float("nan")), dict(cfo=float("-inf")), dict(amp=0), dict(amp=128),
           dict(amp=-5), dict(slot=1519), dict(slot=1199, channel=5), dict(slot=12001), dict(channel=40), dict(channel=-1)]
    for b in bad:
        kw = dict(snr=10.0, ppm=0.0, cfo=0.0, amp=64, slot=2048, channel=37)
        kw.update(b)
        cfg = cfg_of(kw["snr"], kw["ppm"], kw["cfo"], kw["amp"], kw["slot"], kw["channel"])
        assert rx._L.btle_b200_rx_ber_run(rx._h, cfg.ctypes.data, 10, res.ctypes.data) == EINVAL, b
        assert rx._L.btle_b200_last_error(rx._h).startswith(b"rx_ber"), b
        assert rx._L.btle_b200_rx_ber_synth_device(rx._h, cfg.ctypes.data, 0, 1, d_iq.data_ptr(), d_truth.data_ptr(), None) == EINVAL, b
        good = run(rx, cfg_of(1000.0), 8)
        assert good["packets"] == 8 and good["pkt_err"] == 0
    assert rx._L.btle_b200_rx_ber_synth_device(rx._h, cfg_of(30.0).ctypes.data, 0, 1, d_iq.data_ptr() + 1, d_truth.data_ptr(), None) == EINVAL
    assert rx._L.btle_b200_rx_ber_score_device(rx._h, d_truth.data_ptr(), 1, d_iq.data_ptr(), 10, d_iq.data_ptr(), 12273,
                                               d_truth.data_ptr(), None) == EINVAL
    assert run(rx, cfg_of(1000.0), 3)["pkt_err"] == 0


def test_zero_and_one_packet(rx):
    assert run(rx, cfg_of(10.0), 0) == dict.fromkeys(RX_BER_COUNTERS, 0)
    for snr, seed in ((40.0, 1), (-20.0, 2)):
        cfg = cfg_of(snr, seed=seed)
        c = run(rx, cfg, 1)
        d_iq, d_truth = synth_dev(rx, cfg, 0, 1)
        recs, *_ = decode(rx, d_iq, cfg)
        assert c == R.score(recs, truth_of(d_truth, 1)) and c["packets"] == 1 and c["bit_total"] == 8 * 39
        assert c["pkt_err"] == (0 if snr > 0 else 1)


@pytest.mark.parametrize("channel,slot", [(37, 1520), (12, 1200), (38, 1521), (20, 4096 + 7)])
def test_shortest_slots_and_packets_across_chunk_boundaries_at_every_delay(rx, channel, slot):
    cfg = cfg_of(40.0, slot=slot, channel=channel, seed=51)
    n = 4000
    c = run(rx, cfg, n)
    d_iq, d_truth = synth_dev(rx, cfg, 0, n)
    truth = truth_of(d_truth, n)
    recs, *_ = decode(rx, d_iq, cfg)
    assert c == R.score(recs, truth)
    assert (c["pkt_err"], c["crc_ok_wrong"]) == (0, 0), c
    # packets run into each other and across chunk boundaries: every record, extra ones included, is the oracle's
    exp = orc.rx_flags(d_iq.cpu().numpy(), 2, channel=channel, access_addr=int(cfg["access_addr"][0]), crc_init=int(cfg["crc_init"][0]))
    assert recs.tobytes() == exp.tobytes()
    L = R.packet_len(channel)
    start = np.arange(n) * slot + truth["offset"]
    across = start // R.CHUNK != (start + L - 1) // R.CHUNK
    assert across.sum() > 50 and set(truth["delta4"][across]) == {0, 1, 2, 3}
    for d in range(4):                                                      # each delta on its own
        assert R.score(recs, truth[truth["delta4"] == d])["pkt_err"] == 0


# ---- 6. sanity ----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("channel", [37, 12])
def test_per_at_the_ends_of_the_snr_range(rx, channel):
    """Noiseless: no packet error.  At 30 dB almost every access address is found, but the receiver keeps a floor of packet
    errors (10-20 % on an H100 run of this flow, see DESIGN.md), so only PER < 0.3 is asserted there.  At -10 dB
    practically every packet is lost."""
    assert run(rx, cfg_of(1000.0, channel=channel, seed=60), 20000)["pkt_err"] == 0
    hi = run(rx, cfg_of(30.0, channel=channel, seed=61), 20000)
    lo = run(rx, cfg_of(-10.0, channel=channel, seed=62), 20000)
    assert hi["aa_miss"] <= 20 and hi["pkt_err"] < 0.3 * 20000, hi
    assert lo["pkt_err"] > 0.99 * 20000, lo
    p = ber.rx_ber_point(rx, 1000.0, 1000, channel=channel)
    assert p["per"] == 0.0 and p["packets"] == 1000 and p["packets_per_s"] > 0
