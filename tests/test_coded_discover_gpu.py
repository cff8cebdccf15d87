"""LE Coded PHY connection discovery (btle_b200_discover_coded*, include/btle_b200.h "Coded connection discovery") on
the GPU, pinned to the restatement coded_discover_ref.py byte for byte: noise of two kinds, the connection scene, bursts
at tile seams and within W of them, per-capture carrier offsets, poisoned device views, more hits per CTA than decode
warps, capacity cuts, four CUDA streams sharing the cfg cache, argument errors; and decode_connections(coded=True,
coded_discover=True) against the CPU backend."""
import ctypes

import numpy as np
import pytest
import torch

import coded_discover_ref as cd
import coded_ref as cr
from btle_b200 import BtleRx, synth
from btle_b200._native import BTLE_EINVAL, BTLE_EOVERFLOW, CODED_CAND_DTYPE, BtleError
from btle_b200.hop import decode_connections
from test_coded_discover import CodedDiscoverOracleRx, check_coded_discover_connections, coded_discover_capture

pytestmark = pytest.mark.gpu

TILE = 111 * 128                    # window starts per CTA (kCdGroups groups of 128 samples)


@pytest.fixture(scope="module")
def rx():
    import __graft_entry__ as ge
    ge.build()
    r = BtleRx(0)
    yield r
    r.close()


def _same(got, exp):
    assert got.size == exp.size, (got["sample"], exp["sample"])
    for name in CODED_CAND_DTYPE.names:
        assert np.array_equal(got[name], exp[name]), name
    assert got.tobytes() == exp.tobytes()


def _device(rx, iq, channels, offset_hz=None, cap=None, stride_pad=0, offset=0, stream_ptr=0):
    """discover_coded_device on a copy of iq [ns, n] in rows of n + stride_pad bytes starting `offset` bytes into the
    buffer; returns (sorted candidates, count, raw output bytes)"""
    ns, n = iq.shape
    stride = (n + stride_pad + 15) // 16 * 16
    buf = torch.zeros(offset + ns * stride + 64, dtype=torch.int8, device="cuda")
    view = buf[offset:offset + ns * stride].view(ns, stride)[:, :n]
    view.copy_(torch.from_numpy(np.ascontiguousarray(iq)))
    cap = 4096 if cap is None else cap
    d_out = torch.full((cap * 32 + 64,), 0xA5, dtype=torch.uint8, device="cuda")
    d_count = torch.zeros(1, dtype=torch.int32, device="cuda")
    rx.discover_coded_device(view, channels, d_out[:cap * 32], d_count, stream_ptr, offset_hz=offset_hz)
    torch.cuda.synchronize()
    count = int(d_count.item())
    raw = d_out.cpu().numpy()
    got = raw[:min(count, cap) * 32].view(CODED_CAND_DTYPE)
    return np.sort(got, order=["stream", "sample"]), count, raw


def _check(rx, iq, channels, offset_hz=None, **kw):
    exp = cd.discover_coded(iq, channels, offset_hz)
    _same(rx.discover_coded(iq, channels, offset_hz=offset_hz), exp)
    got, count, _ = _device(rx, iq, channels, offset_hz, **kw)
    assert count == exp.size
    _same(got, exp)
    return exp


def _burst_capture(rng, n_samples, starts, channel, s_of=lambda k: (8, 2)[k % 2], amp=100, snr=None, offset_hz=0.0):
    bursts, truth = [], []
    for k, n0 in enumerate(starts):
        aa, crc = int(rng.integers(0, 1 << 32)), int(rng.integers(0, 1 << 24))
        hdr = bytes([int(rng.choice([1, 5, 9, 13])), 0])
        bursts.append((n0, synth.coded_air(hdr, channel, aa, crc, s=s_of(k))))
        truth.append((n0, aa, crc))
    sigma = cr.sigma_of(snr, amp) if snr is not None else 0.0
    return cr.place(n_samples, bursts, amp, sigma, rng, offset_hz), truth


@pytest.mark.parametrize("sigma", [3.0, 40.0])
def test_noise(rx, sigma):
    rng = np.random.default_rng(int(sigma))
    iq = np.clip(np.round(rng.normal(0, sigma, (3, 2 * 150000))), -128, 127).astype(np.int8)
    assert _check(rx, iq, [0, 17, 36]).size == 0


def test_seams_and_phases(rx):
    """bursts at tile seams, W either side of them and at every phase; several captures with odd lengths"""
    rng = np.random.default_rng(3)
    caps = []
    for c, delta in enumerate((-257, -256, -5, -1, 0, 3, 255, 256)):
        starts = [t * TILE + delta + (t + c) % 4 for t in range(1, 5)]
        caps.append(_burst_capture(rng, 5 * TILE + 4000, starts, 7 + c, snr=6.0 if c == 3 else None)[0])
    iq = np.stack(caps)
    exp = _check(rx, iq, list(range(7, 15)))
    assert exp.size >= 28
    # odd length with a dangling byte: the dangling byte is not a sample
    odd = np.concatenate([iq[1], np.array([77], np.int8)])[None, :]
    _same(rx.discover_coded(odd, 8), cd.discover_coded(odd[:, :-1], 8))


def test_offsets_per_capture(rx):
    rng = np.random.default_rng(5)
    hz = [125e3, -125e3, 60e3]
    caps = [_burst_capture(rng, 60000, [2000, 9000, 16000, 23000, 30000, 45000], 12, offset_hz=h, snr=8.0)[0] for h in hz]
    iq = np.stack(caps)
    exp = _check(rx, iq, 12, offset_hz=np.array(hz, np.float32))
    assert exp.size >= 15
    # without the correction the records differ
    assert cd.discover_coded(iq, 12).tobytes() != exp.tobytes()


def test_poisoned_views_and_many_hits(rx):
    """nonzero offsets, strides above n_int8, odd lengths; a dense capture with more hits per CTA than decode warps"""
    rng = np.random.default_rng(9)
    dense = list(range(1000, 3 * TILE, 2300))                # S=2 empty PDUs 2300 samples apart: 6 per tile
    iq, tr = _burst_capture(rng, 3 * TILE + 3000, dense, 30, s_of=lambda k: 2)
    other, _ = _burst_capture(rng, 3 * TILE + 3000, dense[::3], 31)
    both = np.stack([iq, other])
    exp = cd.discover_coded(both, [30, 31])
    assert np.bincount(exp[exp["stream"] == 0]["sample"] // TILE).max() > 4
    for stride_pad, offset in ((0, 0), (48, 16), (1000, 4096)):
        got, count, _ = _device(rx, both, [30, 31], stride_pad=stride_pad, offset=offset)
        assert count == exp.size
        _same(got, exp)
    cut = both[:, :2 * (2 * TILE) + 2]                       # n_int8 % 16 != 0
    got, count, _ = _device(rx, cut, [30, 31], stride_pad=32, offset=32)
    _same(got, cd.discover_coded(cut, [30, 31]))


def test_capacity_cuts(rx):
    rng = np.random.default_rng(11)
    iq, _ = _burst_capture(rng, 80000, list(range(1500, 75000, 6000)), 22)
    exp = cd.discover_coded(iq, 22)
    assert exp.size >= 10
    keys = {(int(r["stream"]), int(r["sample"])): r.tobytes() for r in exp}
    for cap in (0, 1, 3, exp.size - 1, exp.size):
        got, count, raw = _device(rx, iq[None, :], 22, cap=cap)
        assert count == exp.size
        assert len(got) == min(cap, exp.size)
        assert all(keys[(int(r["stream"]), int(r["sample"]))] == r.tobytes() for r in got)
        assert (raw[min(cap, exp.size) * 32:] == 0xA5).all()
    for cap in (1, exp.size - 1):
        with pytest.raises(BtleError) as e:
            rx.discover_coded(iq, 22, cap=cap)
        assert e.value.code == BTLE_EOVERFLOW
    out = np.zeros(2, CODED_CAND_DTYPE)
    n_out = ctypes.c_size_t(0)
    rc = rx._L.btle_b200_discover_coded(rx._h, iq.ctypes.data, 1, iq.size, iq.size, np.array([22], np.int32).ctypes.data, None,
                                        out.ctypes.data, 2, ctypes.byref(n_out))
    assert rc == BTLE_EOVERFLOW and n_out.value == exp.size
    assert all(keys[(int(r["stream"]), int(r["sample"]))] == r.tobytes() for r in out)
    _same(rx.discover_coded(iq, 22), exp)                     # grows once


def test_four_streams_share_the_cfg_cache(rx):
    rng = np.random.default_rng(13)
    caps = [_burst_capture(rng, 40000, [2000 + 97 * k, 14000, 27000], 3 + k)[0] for k in range(4)]
    iq = np.stack(caps)
    chans = [[3, 4, 5, 6], [6, 5, 4, 3]]
    hzs = [None, np.array([0, 50e3, -50e3, 125e3], np.float32)]
    exp = {(a, b): cd.discover_coded(iq, chans[a], hzs[b]) for a in range(2) for b in range(2)}
    streams = [torch.cuda.Stream() for _ in range(4)]
    d_iq = torch.from_numpy(iq).cuda()
    outs = [(torch.zeros(512 * 32, dtype=torch.uint8, device="cuda"), torch.zeros(1, dtype=torch.int32, device="cuda")) for _ in range(16)]
    torch.cuda.synchronize()
    for r in range(16):
        a, b = r % 2, (r // 2) % 2
        st = streams[r % 4]
        with torch.cuda.stream(st):
            rx.discover_coded_device(d_iq, chans[a], outs[r][0], outs[r][1], st.cuda_stream, offset_hz=hzs[b])
    torch.cuda.synchronize()
    for r in range(16):
        a, b = r % 2, (r // 2) % 2
        n = int(outs[r][1].item())
        got = np.sort(outs[r][0].cpu().numpy()[:n * 32].view(CODED_CAND_DTYPE), order=["stream", "sample"])
        _same(got, exp[(a, b)])


def test_argument_errors_leave_the_context_usable(rx):
    iq = np.zeros((2, 4000), np.int8)
    for kw in ({"channels": [0, 37]}, {"channels": [-1, 0]}, {"channels": [0, 1], "offset_hz": [0, 6e5]},
               {"channels": [0, 1], "offset_hz": [np.nan, 0]}):
        with pytest.raises(BtleError) as e:
            rx.discover_coded(iq, kw["channels"], offset_hz=kw.get("offset_hz"))
        assert e.value.code == BTLE_EINVAL
    d_iq = torch.zeros((2, 4000), dtype=torch.int8, device="cuda")
    d_out = torch.zeros(64 * 32 + 16, dtype=torch.uint8, device="cuda")
    d_count = torch.zeros(1, dtype=torch.int32, device="cuda")
    with pytest.raises(BtleError) as e:                         # misaligned output
        rx.discover_coded_device(d_iq, [0, 1], d_out[8:8 + 64 * 32], d_count)
    assert e.value.code == BTLE_EINVAL
    buf = torch.zeros(2 * 4008, dtype=torch.int8, device="cuda")
    with pytest.raises(BtleError) as e:                         # stride not a multiple of 16
        rx.discover_coded_device(buf.view(2, 4008)[:, :4000], [0, 1], d_out[:64 * 32], d_count)
    assert e.value.code == BTLE_EINVAL
    rng = np.random.default_rng(17)
    ok, _ = _burst_capture(rng, 20000, [2000, 9000], 5)
    _check(rx, np.stack([ok, ok]), [5, 5])


def test_decode_connections_coded_discover_equals_cpu_backend(rx):
    adv, conns = check_coded_discover_connections(rx)
    adv_c, conns_c = decode_connections(CodedDiscoverOracleRx(), coded_discover_capture()[0], coded=True, coded_discover=True)
    adv_c["mag_sum"] = 0                                       # the oracle's rx_batch always measures it; rssi is off here
    assert adv.tobytes() == adv_c.tobytes()
    assert len(conns) == len(conns_c)
    for x, y in zip(conns, conns_c):
        assert set(x) == set(y)
        for k in x:
            if isinstance(x[k], np.ndarray):
                assert x[k].dtype == y[k].dtype and x[k].tobytes() == y[k].tobytes(), k
            else:
                assert x[k] == y[k], k
    # the candidates themselves equal the restatement on the 37 data captures
    cap = coded_discover_capture()[0]
    _same(rx.discover_coded(cap[0:37], np.arange(37)), cd.discover_coded(cap[0:37], np.arange(37)))
