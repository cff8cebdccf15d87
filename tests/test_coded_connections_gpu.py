"""hop.decode_connections(coded=True) on the GPU: the capture of tests/test_coded_connections.py (CONNECT_REQ, discovered
and AUX_CONNECT_REQ connections, 1M and coded traffic, two batches of coded connection cfgs) gives every planted coded
packet to exactly its connection, and the whole result equals the CPU backend's (the oracles and coded_ref.py)."""
import numpy as np
import pytest

from btle_b200.hop import decode_connections
from test_coded_connections import CodedOracleRx, check_coded_connections, coded_connections_capture
from test_coded_gpu import rx  # noqa: F401  (the module's fixture)

pytestmark = pytest.mark.gpu


def _same_connections(a, b):
    assert len(a) == len(b)
    for x, y in zip(a, b):
        assert set(x) == set(y)
        for k in x:
            if isinstance(x[k], np.ndarray):
                assert x[k].dtype == y[k].dtype and x[k].tobytes() == y[k].tobytes(), k
            else:
                assert x[k] == y[k], k


def test_decode_connections_coded_equals_cpu_backend(rx):
    adv, conns = check_coded_connections(rx)
    adv_c, conns_c = decode_connections(CodedOracleRx(), coded_connections_capture()[0], coded=True)
    adv_c["mag_sum"] = 0                                       # the oracle's rx_batch always measures it; rssi is off here
    assert adv.tobytes() == adv_c.tobytes()
    _same_connections(conns, conns_c)
    assert sum(len(c["coded_traffic"]) for c in conns) >= 16


def test_decode_connections_coded_offsets(rx):
    """offset_hz reaches the coded calls: a zero offset per capture returns what no offset returns"""
    cap, _ = coded_connections_capture()
    a0, c0 = decode_connections(rx, cap, coded=True)
    a1, c1 = decode_connections(rx, cap, coded=True, offset_hz=np.zeros(40))
    assert a0.tobytes() == a1.tobytes()
    _same_connections(c0, c1)
