"""Connection discovery on the GPU (discover_kernel through btle_b200_discover / _device) against the numpy restatement
of the candidate rule (tests/discover_ref.py), and the discovery / following checks of tests/test_discover.py with BtleRx."""
import ctypes

import numpy as np
import pytest
import torch

import discover_ref as R
from btle_b200 import CAND_DTYPE, REC_DTYPE, synth
from btle_b200._native import BTLE_EINVAL, BTLE_EOVERFLOW, BtleError
from btle_b200.rx import make_cfgs
from test_discover import (AAS, check_discover_connections, check_follow_discovered, check_noise_gives_nothing, edge_captures,
                           many_connections, planted)

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def rx():
    import __graft_entry__ as ge
    ge.build()
    from btle_b200 import BtleRx
    return BtleRx(0)


def _noise(n_streams, n_int8, kind, seed):
    if kind == "floor":
        gen = torch.Generator(); gen.manual_seed(seed)
        return synth.noise_floor(n_streams * n_int8, gen).numpy().reshape(n_streams, n_int8).copy()
    return np.random.default_rng(seed).integers(-128, 128, (n_streams, n_int8), dtype=np.int16).astype(np.int8)


def _discover_strided(rx, iq2d, channels, stride):
    """btle_b200_discover with captures `stride` bytes apart (stride > n_int8)."""
    ns, n = iq2d.shape
    buf = np.zeros(ns * stride, dtype=np.int8)
    for s in range(ns):
        buf[s * stride:s * stride + n] = iq2d[s]
        buf[s * stride + n:(s + 1) * stride] = 77                      # padding that must not be read
    ch = np.ascontiguousarray(channels, dtype=np.int32)
    out = np.empty(ns * (n // 16384 + 1) * 8 + 256, dtype=CAND_DTYPE)
    got = ctypes.c_size_t(0)
    rx._check(rx._L.btle_b200_discover(rx._h, buf.ctypes.data, ns, stride, n, ch.ctypes.data, out.ctypes.data, out.size, ctypes.byref(got)))
    return out[:got.value]


@pytest.mark.parametrize("kind", ["floor", "uniform"])
@pytest.mark.parametrize("n_int8", [16 * 16384, 16 * 16384 + 4090, 1000003])
def test_discover_equals_restatement_on_noise(rx, kind, n_int8):
    iq = _noise(37, n_int8, kind, n_int8 % 1000)
    ch = np.arange(37, dtype=np.int32)
    exp = R.discover_batch(iq, ch)
    assert rx.discover(iq, ch).tobytes() == exp.tobytes()
    assert _discover_strided(rx, iq, ch, (n_int8 + 15) // 16 * 16 + 4096).tobytes() == exp.tobytes()
    one = rx.discover(iq[5], 5)
    assert one.tobytes() == R.discover(iq[5], 5).tobytes()
    assert _discover_strided(rx, iq[5:6], [5], n_int8 + 100).tobytes() == one.tobytes()


def test_discover_equals_restatement_on_connections_and_planted_packets(rx):
    cap, _ = many_connections(partial=True)
    ch = np.arange(37, dtype=np.int32)
    got = rx.discover(cap[:37], ch)
    assert len(got) > 150 and got.tobytes() == R.discover_batch(cap[:37], ch).tobytes()
    for aa in AAS:
        iqs = np.stack([planted(c, aa, at=2000 + 37 * c, n_samples=6001) for c in range(37)])
        got = rx.discover(iqs, ch)
        assert got.tobytes() == R.discover_batch(iqs, ch).tobytes()
        assert all(((got["stream"] == c) & (got["access_addr"] == aa) & (got["crc_init"] == 0x227BA7)).sum() == 3 for c in range(37))
    tight, front, back = edge_captures()
    for iq in (tight, front, back):
        assert rx.discover(iq, 9).tobytes() == R.discover(iq, 9).tobytes()
    assert list(rx.discover(tight, 9)["sample"]) == [32] and len(rx.discover(front, 9)) == 0 and len(rx.discover(back, 9)) == 0


def test_discover_device_and_overflow(rx):
    cap, _ = many_connections()
    ch = np.arange(37, dtype=np.int32)
    host = rx.discover(cap[:37], ch)
    d_iq = torch.from_numpy(cap[:37].copy()).cuda()
    d_out = torch.empty(len(host) * 32 + 4096, dtype=torch.uint8, device="cuda")
    d_count = torch.zeros(1, dtype=torch.int32, device="cuda")
    rx.discover_device(d_iq, ch, d_out, d_count, torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    n = int(d_count.item())
    dev = d_out[:n * 32].cpu().numpy().view(CAND_DTYPE)
    dev = dev[np.lexsort((dev["sample"], dev["stream"]))]
    assert n == len(host) and dev.tobytes() == host.tobytes()
    # a tiny cap: BTLE_EOVERFLOW with the exact count (device: the counter still counts everything)
    small = torch.empty(5 * 32, dtype=torch.uint8, device="cuda")
    rx.discover_device(d_iq, ch, small, d_count, torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    assert int(d_count.item()) == len(host)
    with pytest.raises(BtleError) as e:
        rx.discover(cap[:37], ch, cap=5)
    assert e.value.code == BTLE_EOVERFLOW
    out = np.empty(5, dtype=CAND_DTYPE)
    got = ctypes.c_size_t(0)
    c8 = np.ascontiguousarray(cap[:37])
    assert rx._L.btle_b200_discover(rx._h, c8.ctypes.data, 37, c8.shape[1], c8.shape[1], ch.ctypes.data, out.ctypes.data, 5,
                                    ctypes.byref(got)) == BTLE_EOVERFLOW
    assert got.value == len(host)


def test_every_crc_ok_empty_pdu_has_a_candidate(rx):
    """What rx_batch decodes with the true access address and CRC init: every CRC-ok empty PDU has its candidate at
    chunk * 8192 + n0 with that access address and CRC init."""
    cap, truth = many_connections()
    ch = np.arange(37, dtype=np.int32)
    cand = rx.discover(cap[:37], ch)
    keys = set(zip(cand["stream"].tolist(), cand["sample"].tolist(), cand["access_addr"].tolist(), cand["crc_init"].tolist()))
    seen = 0
    for t in truth:
        recs = rx.rx_batch(cap[:37], make_cfgs(37, channel=list(range(37)), access_addr=t["aa"], crc_init=t["crci"]))
        for r in recs:
            if r["crc_bad"] or r["bytes"][1] != 0 or (r["bytes"][0] & 3) != 1:
                continue
            seen += 1
            assert (int(r["stream"]), int(r["chunk"]) * 8192 + int(r["n0"]), t["aa"], t["crci"]) in keys
    assert seen > 40


def test_discovery_host_logic_with_gpu_backend(rx):
    check_discover_connections(rx)
    check_follow_discovered(rx)
    check_noise_gives_nothing(rx)


def test_validation_errors_leave_the_context_usable(rx):
    iq = _noise(2, 65536, "floor", 3)
    d_count = torch.zeros(1, dtype=torch.int32, device="cuda")
    d_out = torch.empty(4096, dtype=torch.uint8, device="cuda")
    d_iq = torch.from_numpy(iq).cuda()
    for bad in ([37, 0], [-1, 0]):
        with pytest.raises(BtleError) as e:
            rx.discover(iq, bad)
        assert e.value.code == BTLE_EINVAL and "0~36" in str(e.value)
        with pytest.raises(BtleError):
            rx.discover_device(d_iq, bad, d_out, d_count)
    flat = torch.zeros(2 * 65536 + 16, dtype=torch.int8, device="cuda")
    with pytest.raises(BtleError) as e:                                    # misaligned device pointer
        rx.discover_device(flat[1:1 + 2 * 65536].view(2, 65536), [1, 2], d_out, d_count)
    assert e.value.code == BTLE_EINVAL
    with pytest.raises(BtleError) as e:                                    # stride not a multiple of 16
        rx.discover_device(flat[:2 * 65000].view(2, 65000)[:, :64000], [1, 2], d_out, d_count)
    assert e.value.code == BTLE_EINVAL
    L = rx._L
    got = ctypes.c_size_t(7)
    assert L.btle_b200_discover(rx._h, None, 0, 0, 0, None, None, 0, ctypes.byref(got)) == 0 and got.value == 0
    assert L.btle_b200_discover(rx._h, iq.ctypes.data, 1, 600, 600, np.array([3], np.int32).ctypes.data, None, 0, ctypes.byref(got)) == 0
    assert got.value == 0                                                  # too short for one window
    assert L.btle_b200_discover_device(rx._h, d_iq.data_ptr(), 2, 65536, 65536, np.array([1, 2], np.int32).ctypes.data, d_out.data_ptr(),
                                       128, None, None) == BTLE_EINVAL
    assert rx.discover(iq, [1, 2]).tobytes() == R.discover_batch(iq, [1, 2]).tobytes()
    rec = rx.rx(synth.make_adv_stream(4 * 16384, seed=3)[0].numpy(), channel=37)
    assert rec.dtype == REC_DTYPE and len(rec) > 0
