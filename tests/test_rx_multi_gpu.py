"""btle_b200_rx_multi on the GPU: equal to rx_batch() on replicated captures, record for record."""
import ctypes

import numpy as np
import pytest
import torch

import orc
from btle_b200 import BtleRx, synth
from btle_b200._native import BTLE_EINVAL, BTLE_EOVERFLOW, MAX_CFGS_PER_CAPTURE, BtleError, DIR_DTYPE, REC_DTYPE
from btle_b200.hop import decode_connections
from btle_b200.rx import make_cfgs
from test_rx_multi import OracleMultiRx, check_decode_connections, connections_capture, multi_cases, oracle_multi

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def rx():
    r = BtleRx(0)
    yield r
    r.close()


def replicated(rx, iq, cfgs, capture):
    return rx.rx_batch(np.ascontiguousarray(iq[capture]), cfgs)


def device_multi(rx, d_iq, cfgs, capture, stream_ptr=0, with_count=True, offset_hz=None):
    n_units = max(rx.multi_units(d_iq.shape[0], capture, d_iq.shape[1]), 1)
    cap = len(cfgs) * (d_iq.shape[1] // 16384) * 123 + 16
    d_out = torch.zeros(cap * 64, dtype=torch.uint8, device="cuda")
    d_dir = torch.zeros(n_units * 8, dtype=torch.uint8, device="cuda")
    d_count = torch.zeros(1, dtype=torch.int32, device="cuda") if with_count else None
    rx.rx_multi_device_dir(d_iq, cfgs, capture, d_out, d_count, d_dir, stream_ptr, offset_hz=offset_hz)
    return d_out, d_dir, d_count


def to_device(iq):
    """Captures in device memory, rows 16-byte aligned (the device entry points' stride rule)."""
    iq = np.ascontiguousarray(iq)
    pitch = (iq.shape[1] + 15) // 16 * 16
    d = torch.zeros((iq.shape[0], pitch), dtype=torch.int8, device="cuda")
    d[:, :iq.shape[1]] = torch.from_numpy(iq).cuda()
    return d[:, :iq.shape[1]]


def gathered(rx, d_out, d_dir):
    torch.cuda.synchronize()
    return rx.gather_ordered(d_out.cpu().numpy().view(REC_DTYPE), d_dir.cpu().numpy().view(DIR_DTYPE))


@pytest.mark.parametrize("case", multi_cases(), ids=lambda c: c[0])
def test_rx_multi_equals_rx_batch_on_replicated_captures(rx, case):
    _, iq, cfgs, capture = case
    exp = replicated(rx, iq, cfgs, capture)
    got = rx.rx_multi(iq, cfgs, capture)
    assert got.tobytes() == exp.tobytes() and len(exp) > 0
    d_iq = to_device(iq)
    d_out, d_dir, d_count = device_multi(rx, d_iq, cfgs, capture)
    dev = gathered(rx, d_out, d_dir)
    assert dev.tobytes() == exp.tobytes() and int(d_count.item()) == len(exp)
    # the seeded sample against the oracle itself
    assert got.tobytes() == oracle_multi(iq, cfgs, capture).tobytes()


def test_rx_multi_on_c3_like_data_captures(rx):
    """37 data-channel captures x 16 MiB, 4 cfgs each (its own access address and three others), from the GPU synthesiser."""
    n = 16 << 20
    cfg_s = make_cfgs(37, channel=list(range(37)), access_addr=[0x50850A1B + 0x01010101 * (c % 8) for c in range(37)],
                      crc_init=[0x227BA7 ^ c for c in range(37)], rssi=1)
    d_iq, _ = synth.synth_streams_device(cfg_s, n, seed=5, slot_samples=3300, amplitude=60, corrupt_every=7, straddle_every=5,
                                         want_truth=False)
    torch.cuda.synchronize()
    K = 4
    cfgs = make_cfgs(37 * K)
    capture = np.repeat(np.arange(37, dtype=np.int32), K)
    for c in range(37):
        for k in range(K):
            cfgs[c * K + k] = cfg_s[(c + 3 * k) % 37] if k else cfg_s[c]
            cfgs[c * K + k]["channel"] = c
    d_out, d_dir, _ = device_multi(rx, d_iq, cfgs, capture, with_count=False)
    got = gathered(rx, d_out, d_dir)
    # (b): K single-cfg launches, stream mapped to the cfg index
    parts = []
    for k in range(K):
        sel = np.arange(37) * K + k
        r = rx.rx_batch(d_iq.cpu().numpy(), cfgs[sel]).copy()
        r["stream"] = sel[r["stream"]]
        parts.append(r)
    exp = np.concatenate(parts)
    exp = exp[np.argsort(exp["stream"], kind="stable")]
    assert got.tobytes() == exp.tobytes() and len(got) > 37 * 1000


def test_overflow_reports_the_needed_count(rx):
    _, iq, cfgs, capture = multi_cases()[3]
    exp = replicated(rx, iq, cfgs, capture)
    out = np.zeros(5, dtype=REC_DTYPE)
    n_out = ctypes.c_size_t(0)
    iq = np.ascontiguousarray(iq)
    rc = rx._L.btle_b200_rx_multi(rx._h, iq.ctypes.data, iq.shape[0], iq.shape[1], iq.shape[1], cfgs.ctypes.data,
                                  np.ascontiguousarray(capture).ctypes.data, cfgs.size, out.ctypes.data, 5, ctypes.byref(n_out))
    n = n_out.value
    assert rc == BTLE_EOVERFLOW and n == len(exp)
    assert rx.rx_multi(iq, cfgs, capture, cap=len(exp)).tobytes() == exp.tobytes()   # the context stays usable


def test_argument_errors(rx):
    iq = np.zeros((3, 4 * 16384), dtype=np.int8)
    for cc in ([1, 0], [0, 3], [-1, 0], [0] * (MAX_CFGS_PER_CAPTURE + 1)):
        with pytest.raises(BtleError) as e:
            rx.rx_multi(iq, make_cfgs(len(cc)), cc)
        assert e.value.code == BTLE_EINVAL and "rx_multi" in str(e.value)
        assert rx.multi_units(3, cc, iq.shape[1]) == 0
    with pytest.raises(BtleError) as e:
        rx.rx_multi(iq, make_cfgs(2, channel=[5, 40]), [0, 1])
    assert e.value.code == BTLE_EINVAL
    d_iq = torch.zeros((3, 4 * 16384 + 16), dtype=torch.int8, device="cuda")
    with pytest.raises(BtleError) as e:                        # misaligned rows
        device_multi(rx, d_iq[:, 1:1 + 4 * 16384], make_cfgs(2), [0, 1])
    assert e.value.code == BTLE_EINVAL
    assert len(rx.rx_multi(iq, make_cfgs(2), [0, 2])) == 0     # still usable
    assert rx.multi_units(3, [0, 0, 2], iq.shape[1]) == 3 * rx.units(2, iq.shape[1]) // 2


def test_two_streams_and_counter_ring(rx):
    cases = multi_cases()
    s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()
    runs = []
    for i, (_, iq, cfgs, capture) in enumerate(cases[:6]):
        d_iq = to_device(iq)
        st = s1 if i % 2 else s2
        with torch.cuda.stream(st):
            runs.append((d_iq, device_multi(rx, d_iq, cfgs, capture, st.cuda_stream, with_count=i % 3 != 0), iq, cfgs, capture))
    torch.cuda.synchronize()
    for d_iq, (d_out, d_dir, _), iq, cfgs, capture in runs:
        assert gathered(rx, d_out, d_dir).tobytes() == replicated(rx, iq, cfgs, capture).tobytes()


def test_sample_against_reference(rx):
    if not orc.ref_available():
        pytest.skip("the reference build is not present")
    _, iq, cfgs, capture = multi_cases()[2]
    got = rx.rx_multi(iq, cfgs, capture)
    for j, (cfg, c) in enumerate(zip(cfgs, capture)):
        if cfg["raw"] or cfg["rssi"] & 2:
            continue
        mine = got[got["stream"] == j]
        ref = orc.ref_rx_stream(iq[c], channel=int(cfg["channel"]), access_addr=int(cfg["access_addr"]), access_mask=int(cfg["access_mask"]),
                                crc_init=int(cfg["crc_init"]))
        orc.assert_same_as_ref(mine, ref)


def test_decode_connections_equals_cpu_backend(rx):
    adv, conns = check_decode_connections(rx)
    adv_c, conns_c = decode_connections(OracleMultiRx(), connections_capture()[0])
    adv_c["mag_sum"] = 0                                       # the oracle's rx_batch always measures it; rssi is off here
    assert adv.tobytes() == adv_c.tobytes() and len(conns) == len(conns_c)
    for a, b in zip(conns, conns_c):
        assert a["access_addr"] == b["access_addr"] and a["traffic"].tobytes() == b["traffic"].tobytes()

