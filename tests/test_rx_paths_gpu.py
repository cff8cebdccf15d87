"""One receive path behind every rx entry point: a cfg list that maps cfg j to capture j for every capture decodes as the
single-cfg calls do (same records, same directory), btle_b200_rx_multi naming some captures once each equals the oracle,
and the device single-cfg calls refuse overlapping captures as the cfg-list and host calls do."""
import numpy as np
import pytest
import torch

from btle_b200 import BtleRx
from btle_b200._native import BTLE_EINVAL, DIR_DTYPE, REC_DTYPE, BtleError
from btle_b200.rx import make_cfgs
from test_rx_multi import _traffic, oracle_multi
from test_rx_multi_gpu import to_device

pytestmark = pytest.mark.gpu

CHANNELS = [37, 5, 38, 22]
AAS = [0x8E89BED6, 0x60850A1B, 0x8E89BED6, 0x60850A1B]              # cfg j's access address, bursts of both on every capture
OFFSETS = [0.0, 20e3, -15e3, 30e3]


@pytest.fixture(scope="module")
def rx():
    r = BtleRx(0)
    yield r
    r.close()


@pytest.fixture(scope="module")
def case():
    """Four captures of 61 chunks and a few hundred bytes, bursts of two access addresses on each; one cfg per capture."""
    iq = _traffic(61 * 16384 + 700, CHANNELS, AAS[:2], seed=11)
    cfgs = make_cfgs(4, channel=CHANNELS, access_addr=AAS, crc_init=[0x555555, 0x227BA7 ^ 0x0A1B, 0x555555, 0x227BA7 ^ 0x0A1B],
                     rssi=[1, 3, 0, 1])
    return iq, cfgs


def _device_run(rx, call, d_iq, n_units, with_count):
    """call(d_out, d_count, d_dir) on fresh buffers; (records in directory order, directory, count or None)."""
    n = d_iq.shape[1]
    d_out = torch.zeros(4 * (n // 16384) * 123 * 64 + 64, dtype=torch.uint8, device="cuda")
    d_dir = torch.zeros(max(n_units, 1) * 8, dtype=torch.uint8, device="cuda")
    d_count = torch.zeros(1, dtype=torch.int32, device="cuda") if with_count else None
    call(d_out, d_count, d_dir)
    torch.cuda.synchronize()
    ud = d_dir.cpu().numpy().view(DIR_DTYPE)[:n_units]
    recs = rx.gather_ordered(d_out.cpu().numpy().view(REC_DTYPE), ud)
    return recs, ud, None if d_count is None else int(d_count.item())


@pytest.mark.parametrize("offset", [False, True], ids=["plain", "offset"])
def test_identity_list_equals_single_cfg_calls(rx, case, offset):
    iq, cfgs = case
    ident = np.arange(4, dtype=np.int32)
    hz = OFFSETS if offset else None
    want = rx.rx_batch(iq, cfgs, offset_hz=hz)
    assert len(want) > (200 if hz is None else 50)                  # (a correction the captures do not need loses packets)
    got = rx.rx_multi(iq, cfgs, ident, offset_hz=hz)
    assert got.tobytes() == want.tobytes()

    d_iq = to_device(iq)
    st = torch.cuda.current_stream().cuda_stream
    n_units = rx.units(4, iq.shape[1])
    assert rx.multi_units(4, ident, iq.shape[1]) == n_units
    for with_count in (True, False):
        single = _device_run(rx, lambda o, c, d: rx.rx_device_dir(d_iq, cfgs, o, c, d, st, offset_hz=hz), d_iq, n_units, with_count)
        listed = _device_run(rx, lambda o, c, d: rx.rx_multi_device_dir(d_iq, cfgs, ident, o, c, d, st, offset_hz=hz), d_iq, n_units,
                             with_count)
        assert single[0].tobytes() == want.tobytes() and listed[0].tobytes() == want.tobytes()
        # the same entries: block bases follow the order units finish in, the counts are the launch's
        assert (single[1]["count"] == listed[1]["count"]).all() and int(single[1]["count"].sum()) == len(want)
        assert single[2] == listed[2] and (single[2] is None or single[2] == len(want))


def test_rx_multi_on_some_captures_once_each(rx, case):
    iq, cfgs = case
    capture = np.array([0, 2, 3], dtype=np.int32)                  # copied as runs [0] and [2, 3], then cfg j on capture j
    sub = cfgs[capture]
    exp = oracle_multi(iq, sub, capture)
    assert len(exp) > 150
    assert rx.rx_multi(iq, sub, capture).tobytes() == exp.tobytes()
    d_iq = to_device(iq)
    n_units = rx.multi_units(4, capture, iq.shape[1])
    st = torch.cuda.current_stream().cuda_stream
    dev = _device_run(rx, lambda o, c, d: rx.rx_multi_device_dir(d_iq, sub, capture, o, c, d, st), d_iq, n_units, True)
    assert dev[0].tobytes() == exp.tobytes() and dev[2] == len(exp)


def test_device_calls_refuse_overlapping_captures(rx, case):
    iq, cfgs = case
    n = iq.shape[1]
    base = torch.zeros(4 * n, dtype=torch.int8, device="cuda")
    view = base.as_strided((4, n), (n // 2 // 16 * 16, 1))         # rows 16-byte aligned, each overlapping the next
    st = torch.cuda.current_stream().cuda_stream
    n_units = rx.units(4, n)
    d_out = torch.zeros(1024 * 64, dtype=torch.uint8, device="cuda")
    d_dir = torch.zeros(n_units * 8, dtype=torch.uint8, device="cuda")
    d_count = torch.zeros(1, dtype=torch.int32, device="cuda")
    calls = [lambda: rx.rx_device_dir(view, cfgs, d_out, None, d_dir, st),
             lambda: rx.rx_device_dir(view, cfgs, d_out, d_count, d_dir, st, offset_hz=OFFSETS),
             lambda: rx.rx_device(view, cfgs, d_out, d_count, st)]
    for call in calls:
        with pytest.raises(BtleError) as e:
            call()
        assert e.value.code == BTLE_EINVAL and "stride" in str(e.value)
    # the context still decodes
    d_iq = to_device(iq)
    got = _device_run(rx, lambda o, c, d: rx.rx_device_dir(d_iq, cfgs, o, c, d, st), d_iq, n_units, True)
    want = rx.rx_batch(iq, cfgs)
    assert got[0].tobytes() == want.tobytes() and got[2] == len(want) > 200
