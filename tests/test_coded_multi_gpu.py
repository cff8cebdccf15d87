"""Several LE Coded PHY cfgs per capture (btle_b200_rx_coded_multi*) on the GPU against btle_b200_rx_coded on a batch of
copies (stream j = capture cfg_capture[j] with cfgs[j] and that capture's offset), record bytes equal: seeded random
layouts of 1..8 cfgs per capture with captures no cfg names, repeated cfgs, one access address with other CRC inits and
channels, per-capture offsets and BTLE_CFG_RSSI on some cfgs, over S=2 and S=8 bursts of eight access addresses at the
search kernel's tile seams; more hits than decode warps; capacity cuts; argument errors; the cfg cache on several CUDA
streams against identity-map launches of the same cfg bytes.  tests/test_coded_gpu.py and test_coded_edges_gpu.py pin
btle_b200_rx_coded itself to coded_ref.py."""
import ctypes

import numpy as np
import pytest
import torch

import coded_ref as cr
from btle_b200 import make_cfgs, synth
from btle_b200._native import BTLE_EINVAL, BTLE_EOVERFLOW, CFG_RSSI, CFG_SYMBOL_SPACED, CODED_REC_DTYPE, BtleError
from test_coded_edges_gpu import TILE, _to_device
from test_coded_gpu import _packet_samples, _same, rx  # noqa: F401  (rx: the module's fixture)

pytestmark = pytest.mark.gpu

REC = CODED_REC_DTYPE.itemsize
AAS = [0x8E89BED6, 0x12345678, 0x50654E3A, 0x71764129, 0x2A3B4C5D, 0x6B7A8F91, 0x1C2D3E4F, 0x4E5F6071]
CRCS = [0x555555, 0xABCDEF, 0x13579B, 0x000001, 0xFFFFFF, 0x2468AC, 0x0F0F0F, 0x7E57ED]
CHANNELS = [37, 3, 17, 30, 0, 36, 22, 39]
HZ = [0.0, 40e3, -75e3, 125e3, -125e3, 10e3, -3e3, 90e3]


def _seam_captures(rng, n_caps=8):
    """capture c on channel CHANNELS[c] at offset HZ[c]: S=2 and S=8 bursts of the eight access addresses (with their
    CRC inits) whose access address sits within 9 samples of a tile seam of coded_search_kernel, every other one noisy"""
    caps = []
    for c in range(n_caps):
        bursts, t = [], 1
        while True:
            q = len(bursts)
            L, s = int(rng.integers(0, 40)), (2, 8)[(q + c) % 2]
            n0 = TILE * t + int(rng.integers(-9, 10))
            if n0 + _packet_samples(L, s) + 2000 > 16 * TILE:
                break
            k = (q * 3 + c) % 8
            pdu = bytes([0x07, L]) + rng.integers(0, 256, L, dtype=np.uint8).tobytes()
            bursts.append((n0, synth.coded_air(pdu, CHANNELS[c], AAS[k], CRCS[k], s=s)))
            t += -(-(_packet_samples(L, s) + 700) // TILE)
        sigma = cr.sigma_of(6.0, 100) if c % 2 else 0.0
        caps.append(cr.place(16 * TILE + 1500, bursts, 100, sigma, rng, offset_hz=HZ[c]))
    return np.stack(caps)


@pytest.fixture(scope="module")
def seams():
    return _seam_captures(np.random.default_rng(61))


def _copies(rx, iq, cfgs, capture, hz):
    """the definition: rx_coded on a batch whose stream j is capture[j], decoded with cfgs[j] and hz[capture[j]]"""
    capture = np.asarray(capture, dtype=np.int64)
    return rx.rx_coded(np.ascontiguousarray(iq[capture]), cfgs, offset_hz=None if hz is None else np.asarray(hz, np.float32)[capture])


def _multi_device(rx, iq, cfgs, capture, hz, cap, stream_ptr=0):
    d_iq = _to_device(iq)
    d_out = torch.zeros(max(cap, 1) * REC, dtype=torch.uint8, device="cuda")
    d_count = torch.zeros(1, dtype=torch.int32, device="cuda")
    rx.rx_coded_multi_device(d_iq, cfgs, capture, d_out, d_count, stream_ptr, offset_hz=hz)
    torch.cuda.synchronize()
    c = int(d_count.item())
    return c, d_out[:min(c, cap) * REC].cpu().numpy().view(CODED_REC_DTYPE)


def _layout(rng, n_caps):
    """a random cfg list: 0..8 cfgs per capture (0: the capture is not read), access addresses of the captures' bursts and
    others, the right or another CRC init and channel, a cfg repeated, BTLE_CFG_RSSI on some"""
    rows, capture = [], []
    for c in range(n_caps):
        k = int(rng.choice([0, 1, 2, 3, 5, 8]))
        for _ in range(k):
            a = int(rng.integers(0, 8))
            aa = AAS[a] if rng.random() < 0.85 else int(rng.integers(0, 1 << 32))
            crc = CRCS[a] if rng.random() < 0.7 else int(rng.integers(0, 1 << 24))
            ch = CHANNELS[c] if rng.random() < 0.8 else int(rng.integers(0, 40))
            rows.append((ch, aa, crc, CFG_RSSI if rng.random() < 0.4 else 0))
            capture.append(c)
        if k >= 2 and rng.random() < 0.5:
            rows[-1] = rows[-2]                                   # the same cfg twice
    cfgs = make_cfgs(len(rows), channel=[r[0] for r in rows], access_addr=[r[1] for r in rows], crc_init=[r[2] for r in rows],
                     rssi=[r[3] for r in rows])
    return cfgs, np.array(capture, dtype=np.int32)


def test_random_layouts_equal_copies(rx, seams):
    rng = np.random.default_rng(62)
    total, repeated, unread = 0, 0, 0
    for trial in range(8):
        cfgs, capture = _layout(rng, seams.shape[0])
        hz = None if trial == 0 else np.asarray(HZ, np.float32)[rng.permutation(8)]
        exp = _copies(rx, seams, cfgs, capture, hz)
        _same(rx.rx_coded_multi(seams, cfgs, capture, offset_hz=hz), exp)
        c, recs = _multi_device(rx, seams, cfgs, capture, hz, exp.size + 50)
        assert c == exp.size
        _same(np.sort(recs, order=["stream", "sample"]), exp)
        for j in range(1, cfgs.size):                             # a repeated cfg: identical records under both indices
            if capture[j] == capture[j - 1] and cfgs[j].tobytes() == cfgs[j - 1].tobytes():
                a, b = exp[exp["stream"] == j - 1].copy(), exp[exp["stream"] == j].copy()
                a["stream"] = b["stream"] = 0
                assert a.tobytes() == b.tobytes()
                repeated += 1
        total += exp.size
        unread += len(set(range(8)) - set(capture.tolist()))
    assert total > 300 and repeated >= 2 and unread >= 4


def test_one_access_address_other_crc_inits_and_channels(rx, seams):
    """cfgs of one access address on one capture: the CRC init decides crc_bad, the channel the dewhitened bytes"""
    c, k = 2, 1                                           # capture 2 carries bursts of AAS[1] on CHANNELS[2]
    ch = CHANNELS[c]
    cfgs = make_cfgs(8, channel=[ch, ch, 5, ch, 20, ch, ch, 5], access_addr=AAS[k],
                     crc_init=[CRCS[k], 0x123456, CRCS[k], CRCS[k], CRCS[k], 0x654321, CRCS[k], 0x123456],
                     rssi=[0, 0, 0, CFG_RSSI, 0, 0, 0, CFG_RSSI])
    hz = np.asarray(HZ, np.float32)
    for cc in (np.full(8, c, np.int32), np.arange(8, dtype=np.int32)):   # all eight on one capture, and one per capture
        _same(rx.rx_coded_multi(seams, cfgs, cc, offset_hz=hz), _copies(rx, seams, cfgs, cc, hz))
    on_c = _copies(rx, seams, cfgs, np.full(8, c, np.int32), hz)
    ok = {j: int((on_c[on_c["stream"] == j]["crc_bad"] == 0).sum()) for j in range(8)}
    assert ok[0] > 0 and ok[1] == 0 and ok[2] == 0 and ok[3] == ok[0] and ok[6] == ok[0], ok


def test_decode_loop_wraps_over_cfgs_and_captures(rx):
    """more hits than coded_decode_kernel has warps (16 CTAs of 4 warps per SM): 20 captures of back-to-back short bursts,
    eight cfgs on each (one access address, eight CRC init / channel pairs), so warps decode hits of other cfgs and
    captures after their first"""
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    rng = np.random.default_rng(63)
    caps = []
    for c in range(20):
        bursts, n0 = [], 800
        for q in range(72):
            s = (2, 8)[q % 5 == 0]
            L = int(rng.integers(0, 4))
            bursts.append((n0 + q % 4, synth.coded_air(bytes([0x07, L]) + bytes(L), CHANNELS[c % 8], AAS[c % 8], CRCS[c % 8], s=s)))
            n0 += _packet_samples(L, s) + 500
        caps.append(cr.place(n0 + 1500, bursts, 100, cr.sigma_of(8.0, 100) if c % 3 else 0.0, rng))
    n = max(x.size for x in caps)
    iq = np.stack([np.pad(x, (0, n - x.size)) for x in caps])
    capture = np.repeat(np.arange(20, dtype=np.int32), 8)
    cfgs = make_cfgs(160, channel=[CHANNELS[(c + (j % 3 == 1)) % 8] for c, j in zip(capture, range(160))],
                     access_addr=[AAS[c % 8] for c in capture], crc_init=[CRCS[c % 8] ^ (j % 8 // 2) for c, j in zip(capture, range(160))],
                     rssi=[CFG_RSSI * (j % 2) for j in range(160)])
    hz = np.zeros(20, np.float32)
    exp = _copies(rx, iq, cfgs, capture, hz)
    assert exp.size > 64 * sms, (exp.size, sms)
    assert (exp["crc_bad"] == 0).any() and (exp["crc_bad"] == 1).any()
    _same(rx.rx_coded_multi(iq, cfgs, capture, offset_hz=hz, cap=exp.size + 10), exp)
    c, recs = _multi_device(rx, iq, cfgs, capture, hz, exp.size + 10)
    assert c == exp.size
    _same(np.sort(recs, order=["stream", "sample"]), exp)


def test_capacity_cuts(rx, seams):
    rng = np.random.default_rng(64)
    cfgs, capture = _layout(rng, 8)
    while cfgs.size < 12:
        cfgs, capture = _layout(rng, 8)
    hz = np.asarray(HZ, np.float32)
    exp = _copies(rx, seams, cfgs, capture, hz)
    assert exp.size > 40
    keys = {(int(r["stream"]), int(r["sample"])): r.tobytes() for r in exp}
    L = rx._L
    iq = np.ascontiguousarray(seams)
    for cap in (0, 1, exp.size // 3, exp.size - 1, exp.size):
        # host: the exact count, BTLE_EOVERFLOW below it, whole records of distinct hits in (cfg, sample) order
        out = np.zeros(max(cap, 1), CODED_REC_DTYPE)
        n_out = ctypes.c_size_t(0)
        rc = L.btle_b200_rx_coded_multi(rx._h, iq.ctypes.data, 8, iq.shape[1], iq.shape[1], cfgs.ctypes.data, capture.ctypes.data, cfgs.size,
                                        hz.ctypes.data, out.ctypes.data, cap, ctypes.byref(n_out))
        assert n_out.value == exp.size and rc == (BTLE_EOVERFLOW if cap < exp.size else 0)
        got = out[:cap]
        assert np.array_equal(np.sort(got, order=["stream", "sample"]), got)
        assert all(keys[(int(r["stream"]), int(r["sample"]))] == r.tobytes() for r in got)
        # device: the exact count, a canary past cap
        d_iq = _to_device(seams)
        d_out = torch.full(((cap + 4) * REC,), 0xA5, dtype=torch.uint8, device="cuda")
        d_count = torch.zeros(1, dtype=torch.int32, device="cuda")
        rx.rx_coded_multi_device(d_iq, cfgs, capture, d_out[:cap * REC], d_count, offset_hz=hz)
        torch.cuda.synchronize()
        assert int(d_count.item()) == exp.size
        host = d_out.cpu().numpy()
        assert (host[cap * REC:] == 0xA5).all()
        recs = host[:cap * REC].view(CODED_REC_DTYPE)
        assert len({(int(r["stream"]), int(r["sample"])) for r in recs}) == cap
        assert all(keys[(int(r["stream"]), int(r["sample"]))] == r.tobytes() for r in recs)
    # the grown default capacity returns everything
    _same(rx.rx_coded_multi(seams, cfgs, capture, offset_hz=hz, cap=None), exp)


def test_argument_errors_leave_the_context_usable(rx, seams):
    ok_cfgs = make_cfgs(3, channel=CHANNELS[0], access_addr=AAS[0], crc_init=CRCS[0])
    exp = _copies(rx, seams, ok_cfgs, [0, 0, 1], None)
    bad = [
        (ok_cfgs, [1, 0, 1]),                                                  # decreasing
        (ok_cfgs, [0, 0, 8]),                                                  # out of range
        (ok_cfgs, [-1, 0, 0]),
        (make_cfgs(9), [2] * 9),                                               # nine on one capture
        (make_cfgs(3, rssi=[0, CFG_SYMBOL_SPACED, 0]), [0, 1, 2]),            # a 1M flag
        (make_cfgs(3, raw=[0, 0, 1]), [0, 1, 2]),                              # raw mode
        (make_cfgs(3, access_mask=[0xFFFFFFFF, 0xFFFF00FF, 0xFFFFFFFF]), [0, 1, 2]),   # a masked access address
    ]
    d_iq = _to_device(seams)
    d_out = torch.zeros(64 * REC, dtype=torch.uint8, device="cuda")
    d_count = torch.zeros(1, dtype=torch.int32, device="cuda")
    for cfgs, cc in bad:
        for call in (lambda: rx.rx_coded_multi(seams, cfgs, cc),
                     lambda: rx.rx_coded_multi_device(d_iq, cfgs, cc, d_out, d_count)):
            with pytest.raises(BtleError) as e:
                call()
            assert e.value.code == BTLE_EINVAL
            _same(rx.rx_coded_multi(seams, ok_cfgs, [0, 0, 1]), exp)
    assert rx.rx_coded_multi(seams, make_cfgs(0), []).size == 0


def test_cfg_cache_on_several_streams(rx, seams):
    """multi launches and identity-map rx_coded launches of the same cfg bytes, interleaved on four CUDA streams: the
    cache keys them apart (their capture groups differ), and every launch returns its own records"""
    rng = np.random.default_rng(65)
    hz = np.asarray(HZ, np.float32)
    cfgs = make_cfgs(8, channel=CHANNELS, access_addr=AAS, crc_init=CRCS, rssi=[CFG_RSSI, 0] * 4)
    multi_cc = [np.array([0, 0, 2, 2, 2, 5, 5, 7], np.int32), np.array([1, 1, 1, 1, 3, 3, 3, 3], np.int32), np.arange(8, dtype=np.int32)]
    d_iq = _to_device(seams)
    copies = {i: _to_device(np.ascontiguousarray(seams[cc])) for i, cc in enumerate(multi_cc)}
    exp = {i: _copies(rx, seams, cfgs, cc, hz) for i, cc in enumerate(multi_cc)}
    streams = [torch.cuda.Stream() for _ in range(4)]
    picks = [int(rng.integers(0, 3)) for _ in range(24)]
    bufs = [(torch.zeros((exp[i].size + 8) * REC, dtype=torch.uint8, device="cuda"), torch.zeros(1, dtype=torch.int32, device="cuda"))
            for i in picks]
    torch.cuda.synchronize()                               # the buffers exist before any stream writes them
    jobs = []
    for r, (i, (d_out, d_count)) in enumerate(zip(picks, bufs)):
        st = streams[r % 4]
        with torch.cuda.stream(st):
            if r % 2:
                rx.rx_coded_multi_device(d_iq, cfgs, multi_cc[i], d_out, d_count, st.cuda_stream, offset_hz=hz)
            else:                                              # the same cfg bytes on the copies, cfg j on capture j
                rx.rx_coded_device(copies[i], cfgs, d_out, d_count, st.cuda_stream, offset_hz=hz[multi_cc[i]])
        jobs.append((i, d_out, d_count))
    torch.cuda.synchronize()
    for i, d_out, d_count in jobs:
        c = int(d_count.item())
        assert c == exp[i].size
        _same(np.sort(d_out[:c * REC].cpu().numpy().view(CODED_REC_DTYPE), order=["stream", "sample"]), exp[i])
    assert exp[0].tobytes() != exp[1].tobytes()
