"""The receive kernel's rotated and symbol-spaced instantiations (btle_rx_persistent_kernel<1|8, ROT, SYM>) and the
per-packet offset estimate at the edges the existing edge tests do not fit, against the numpy restatements
(tests/mode_ref.py, offset_ref.rec_offset), byte for byte:

1. packets whose access addresses start on every edge of the dense loop (lane, tile, chunk and span boundaries, the last
   chunk's look-ahead, the capture's last samples), in all four modes, one and several cfgs per capture, host and device;
2. a symbol-spaced streaming session with a carrier offset per capture that changes mid-session and a backfilled cfg,
   which makes its rounds the multi-cfg rotated symbol-spaced kernel;
3. a bounded run of tools/fuzz_multi_gpu.py in each new mode;
4. btle_b200_rec_offset and _device on every record of several captures with padded, poisoned strides, on records the
   decoder never makes, and on records it must refuse."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import mode_ref
import offset_ref
from btle_b200 import REC_DTYPE, make_cfgs
from btle_b200._native import BTLE_EINVAL, CFG_RECOVER, BtleError
from test_ingest_edges_gpu import CHUNK, HostBuf, _air, _capture, _device_view, _plant, _poison, _same, _walk

pytestmark = pytest.mark.gpu

S_CHUNK = CHUNK // 2                                           # samples per chunk; a tile is 4096 samples, a lane 128


@pytest.fixture(scope="module")
def rx():
    import __graft_entry__ as ge
    ge.build()
    from btle_b200 import BtleRx
    r = BtleRx(0)
    yield r
    r.close()


# ---- 1. packets on every edge of the dense loop ------------------------------------------------------------------------
TAILS = (0, 1, 2, 3, 4, 5, 255, 256, 257, 3007, 3008, 3009)
N_CHUNKS = 18                                                  # one whole span and a second, short one
AIRS = [_air(s) for s in range(4)]


def _targets(n_samples, c):
    """Access-address samples of capture c, most wanted first: the span boundary, the capture's last samples and the last
    chunk's look-ahead, chunk boundaries (down to -124: hits a chunk reports in front of itself), the other tile
    boundaries, then lane boundaries -6..+6."""
    last = (n_samples // S_CHUNK) * S_CHUNK
    t = [16 * S_CHUNK + (-2, 0, 3)[c % 3], n_samples - 700, last - 300 - c]
    t += [k * S_CHUNK + (-124, -101, -64, -9, -3, 0, 2, 5)[(k + c) % 8] for k in range(1, n_samples // S_CHUNK + 1)]
    t += [k * 4096 + (-4, -1, 1, 4)[(k + c) % 4] for k in range(1, n_samples // 4096, 2)]
    t += [m * 128 + (m + c) % 13 - 6 for m in range(3, n_samples // 128, 3)]
    return t


def _edge_captures(tail, mode, n_captures=3):
    """(iq [n_captures, n_int8], offsets): a low noise floor with bursts at _targets, each taken when it lies 1700 samples
    from every burst already there (so the receiver's greedy chain sees each), every capture rotated onto its offset"""
    n = N_CHUNKS * CHUNK + tail
    rng = np.random.default_rng(1000 * tail + 10 * mode[0] + mode[1])
    iq = rng.integers(-5, 6, (n_captures, n), dtype=np.int8)
    for c in range(n_captures):
        at = []
        for a in _targets(n // 2, c):
            if all(abs(a - b) >= 1700 for b in at):
                _plant(iq[c], a, AIRS[(len(at) + c) % 4], amp=int(rng.integers(50, 100)))
                at.append(a)
    offsets = mode_ref.draw_offsets(rng, n_captures, mode)
    return mode_ref.rotate_all(iq, offsets), offsets


def _edges_hit(exp):
    """CRC-ok counted records within 4 samples of a lane, tile, chunk (n0 < 0) and span boundary"""
    ok = exp[(exp["crc_bad"] == 0) & ((exp["flags"] & 5) == 0)]
    pos = ok["chunk"].astype(np.int64) * S_CHUNK + ok["n0"]
    near = lambda p: np.abs((pos + p // 2) % p - p // 2) <= 4
    return {"lane": int(near(128).sum()), "tile": int(near(4096).sum()), "chunk": int((ok["n0"] < 0).sum()),
            "span": int((np.abs(pos - 16 * S_CHUNK) <= 4).sum())}


def _multi_cfgs(mode, n_captures):
    """Per capture: the exact address with RSSI, a masked one with -v, raw, and recovery (the <8> kernel)"""
    per = make_cfgs(4, access_mask=[0xFFFFFFFF, 0xFFFFFF00, 0xFFFFFFFF, 0xFFFFFFFF], raw=[0, 0, 1, 0], rssi=[1, 3, 0, 1 | CFG_RECOVER])
    return mode_ref.with_mode(np.tile(per, n_captures), mode), np.repeat(np.arange(n_captures, dtype=np.int32), 4)


def _device_rx_dir(rx, view, cfgs, offsets, want):
    units = rx.units(view.shape[0], view.shape[1])
    d_out = torch.zeros(len(want) * 64 + 64, dtype=torch.uint8, device="cuda")
    d_dir = torch.zeros((units, 2), dtype=torch.int32, device="cuda")
    rx.rx_device_dir(view, cfgs, d_out, None, d_dir, torch.cuda.current_stream().cuda_stream, offset_hz=offsets)
    torch.cuda.synchronize()
    return _walk(rx, d_out, d_dir, units)[0]


def _device_multi(rx, view, cfgs, capture, offsets, want):
    units = rx.multi_units(view.shape[0], capture, view.shape[1])
    d_out = torch.zeros(len(want) * 64 + 64, dtype=torch.uint8, device="cuda")
    d_dir = torch.zeros((units, 2), dtype=torch.int32, device="cuda")
    d_count = torch.zeros(1, dtype=torch.int32, device="cuda")
    rx.rx_multi_device_dir(view, cfgs, capture, d_out, d_count, d_dir, torch.cuda.current_stream().cuda_stream, offset_hz=offsets)
    torch.cuda.synchronize()
    assert int(d_count.item()) == len(want)
    return _walk(rx, d_out, d_dir, units)[0]


@pytest.mark.parametrize("mode", mode_ref.MODES, ids=mode_ref.mode_id)
@pytest.mark.parametrize("tail", TAILS)
def test_packets_on_every_dense_loop_edge(rx, tail, mode):
    """Bit for bit against mode_ref.rx_multi: one cfg per capture (<1>) through rx_batch and rx_device_dir, four cfgs per
    capture (<8>) through rx_multi and rx_multi_device_dir; device views in a poisoned buffer.  Tails of 0..5 bytes put
    the word behind (`tail`) and in front of (`head`) the last tiles across n_int8; 255..257 and 3007..3009 make the
    last tile ragged (a partial row filled by hand) or zeroed."""
    iq, offsets = _edge_captures(tail, mode)
    ns, n = iq.shape
    one = mode_ref.with_mode(make_cfgs(ns, rssi=[1, 3, 1]), mode)
    exp1 = mode_ref.rx_multi(iq, one, np.arange(ns), offsets)
    hit = _edges_hit(exp1)
    assert all(v > 0 for v in hit.values()), hit
    _same(rx.rx_batch(iq, one, offset_hz=offsets), exp1)
    cfgs, capture = _multi_cfgs(mode, ns)
    exp8 = mode_ref.rx_multi(iq, cfgs, capture, offsets)
    assert all(v > 0 for v in _edges_hit(exp8[exp8["stream"] % 4 == 0]).values())
    _same(rx.rx_multi(iq, cfgs, capture, offset_hz=offsets), exp8)
    rng = np.random.default_rng(tail)
    buf, view = _device_view(list(iq), (n + 15) // 16 * 16 + 32, 16, rng, random_poison=True)
    _same(_device_rx_dir(rx, view, one, offsets, exp1), exp1)
    _same(_device_multi(rx, view, cfgs, capture, offsets, exp8), exp8)
    del buf


# ---- 2. a symbol-spaced session with per-capture offsets and a backfill ----------------------------------------------
def test_symbol_spaced_session_offsets_and_backfill(rx):
    """Two captures, symbol-spaced, each with its own offset; odd push sizes; after the first segment sets a cfg is added
    on capture 0 for every resident chunk (two cfgs on one capture: the <8, ROT, SYM> rounds); capture 1's offset
    changes from segment set k + 1 on.  Each cfg's records equal mode_ref on its whole capture: capture 1 at the old
    offset before the switch's first chunk K, at the new one from K."""
    seg, k = 2, 2
    h0, h1, h1b = 137e3, -310e3, 25e3
    iq0, _ = _edge_captures(3009, (0, 0), n_captures=2)
    n = iq0.shape[1]
    K = (k + 1) * seg
    cut = K * CHUNK + 4096                                         # every capture's part of set k (look-ahead included) is in
    a = mode_ref.rotate(iq0[0], h0)
    b = np.concatenate([mode_ref.rotate(iq0[1], h1)[:K * CHUNK], mode_ref.rotate(iq0[1], h1b)[K * CHUNK:]])
    base = make_cfgs(2, rssi=[1, 3], symbol_spaced=1)
    added = dict(access_mask=0xFFFFFF00, rssi=1, recover=1, symbol_spaced=1)
    parts = []
    with rx.streams(base, segment_chunks=seg) as s_:
        s_.set_offset(0, h0)
        s_.set_offset(1, h1)
        first = 2 * seg * CHUNK + 12345
        for lo, hi in ((0, 777), (777, 70001), (70001, first)):
            parts += [s_.push(0, a[lo:hi]), s_.push(1, b[lo:hi])]
        idx, frm = s_.add_cfg(0, None, **added)                 # three cfgs on two captures: the cfg list is not the identity
        assert idx == 2
        parts += [s_.push(0, a[first:cut]), s_.push(1, b[first:cut])]
        s_.set_offset(1, h1b)
        for lo in range(cut, n, 99991):
            parts += [s_.push(0, a[lo:lo + 99991]), s_.push(1, b[lo:lo + 99991])]
        parts.append(s_.finish())
    got = np.concatenate(parts)
    got = got[np.lexsort((got["n0"], got["chunk"], got["stream"]))]
    cfgs = np.concatenate([base, make_cfgs(1, **added)])
    e0 = mode_ref.rx_multi(a, cfgs[[0, 2]], [0, 0], [h0])
    e0["stream"][e0["stream"] == 1] = 2
    e2 = e0[(e0["stream"] == 2) & (e0["chunk"] >= frm)]
    old = mode_ref.rx_multi(np.stack([b]), cfgs[1:2], [0], [h1])
    new = mode_ref.rx_multi(np.stack([b]), cfgs[1:2], [0], [h1b])
    e1 = np.concatenate([old[old["chunk"] < K], new[new["chunk"] >= K]])
    e1["stream"] = 1
    exp = np.concatenate([e0[e0["stream"] == 0], e1, e2])
    exp = exp[np.lexsort((exp["n0"], exp["chunk"], exp["stream"]))]
    assert ((e1["chunk"] >= K) & (e1["crc_bad"] == 0)).sum() > 5 and len(e2) > 5
    _same(got, exp)


# ---- 3. fuzz in each new mode ------------------------------------------------------------------------------------------
@pytest.mark.parametrize("mode", mode_ref.NEW_MODES, ids=mode_ref.mode_id)
def test_gpu_multi_fuzz_campaign_bounded_in_modes(mode):
    """tools/fuzz_multi_gpu.py --mode for 15 s of random launches (the restatement takes most of it)."""
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    p = subprocess.run([sys.executable, os.path.join(root, "tools", "fuzz_multi_gpu.py"), "20261017", "--mode", "%d,%d" % mode],
                       capture_output=True, text=True, timeout=600, env=dict(os.environ, FUZZ_SECONDS="15"))
    assert p.returncode == 0, p.stdout[-2000:] + p.stderr[-3000:]
    assert " ok" in p.stdout


# ---- 4. the per-packet offset estimate -----------------------------------------------------------------------------------
def _estimate_records(n):
    """(captures [3, n], records with stream = capture): every record of -v, raw, recovering and symbol-spaced cfgs on two
    burst captures and a noise capture, and records the decoder never makes: n0 of -124, 0, 31 in chunk 0, n0 near the
    end of the last chunk (its 157 samples run past the capture), a chunk past the capture."""
    iq = np.stack([_capture(n, 5, "burst", phase=1), _capture(n, 6, "noise"), _capture(n, 7, "burst", phase=2)])
    capture = np.array([0, 0, 0, 1, 2, 2], dtype=np.int32)
    recs = []
    for sym in (0, 1):
        cfgs = make_cfgs(6, access_mask=[0xFFFFFF00, 0xFFFFFFFF, 0xFFFFFFFF, 0, 0xFFFFFFFF, 0xFFFFFF00], raw=[0, 1, 0, 0, 0, 0],
                         rssi=[3, 1, 1 | CFG_RECOVER, 2, 1 | CFG_RECOVER, 3], symbol_spaced=sym)
        r = mode_ref.rx_multi(iq, cfgs, capture, [0.0, 0.0, 0.0] if sym == 0 else None)
        r["stream"] = capture[r["stream"]]
        recs.append(r)
    nplain = len(recs[0])
    recs = np.concatenate(recs)
    last = n // CHUNK - 1
    extra = np.zeros(9, dtype=REC_DTYPE)
    extra["stream"] = [0, 1, 2, 0, 2, 1, 0, 2, 1]
    extra["chunk"] = [0, 0, 0, last, last, last, last + 1, last + 3, 1 << 20]
    extra["n0"] = [-124, 0, 31, n // 2 - last * CHUNK // 2 - 120, n // 2 - last * CHUNK // 2 - 3, 8000, 5, -124, 100]
    extra["access_addr"] = 0x8E89BED6
    recs = np.concatenate([recs, extra])
    kinds = {"rejected": (recs["flags"] & 4) != 0, "raw": (recs["flags"] & 1) != 0, "symbol-spaced": np.arange(len(recs)) >= nplain,
             "n0<0": recs["n0"] < 0, "n0<32": (recs["n0"] >= 0) & (recs["n0"] < 32), "chunk0": recs["chunk"] == 0}
    assert all(v.any() for v in kinds.values()), {k: int(v.sum()) for k, v in kinds.items()}
    return iq, recs


def _rec_offset_host(rx, ptr, ns, stride, n, recs):
    hz = np.zeros(len(recs), dtype=np.float32)
    rx._check(rx._L.btle_b200_rec_offset(rx._h, ptr, ns, stride, n, recs.ctypes.data, len(recs), hz.ctypes.data))
    return hz


@pytest.mark.parametrize("tail", [0, 3007, 3009])
def test_rec_offset_every_record(rx, tail):
    """Host form from pageable memory with padded, poisoned strides and device form on views into a poisoned buffer, each
    record within 2 Hz of offset_ref.rec_offset (float32 atan2f sums against float64)."""
    n = 6 * CHUNK + tail
    iq, recs = _estimate_records(n)
    want = np.array([offset_ref.rec_offset(iq[int(r["stream"])], int(r["chunk"]), int(r["n0"]), int(r["access_addr"])) for r in recs])
    rng = np.random.default_rng(tail)
    for extra in (0, 7, 4096):
        buf = HostBuf("pageable", 3 * (n + extra))
        buf.a[:] = _poison(buf.a.size, rng, True)
        for s in range(3):
            buf.a[s * (n + extra):s * (n + extra) + n] = iq[s]
        got = _rec_offset_host(rx, buf.ptr, 3, n + extra, n, recs)
        assert np.abs(got - want).max() <= 2.0, (extra, np.abs(got - want).max())
    np.testing.assert_allclose(rx.rec_offsets(iq, recs), want, rtol=0, atol=2.0)
    for front, pad in ((16, 0), (4096, 4096)):
        dbuf, view = _device_view(list(iq), (n + 15) // 16 * 16 + pad, front, rng, random_poison=True)
        d_recs = torch.from_numpy(recs.view(np.uint8).copy()).cuda()
        d_hz = torch.full((len(recs),), float("nan"), dtype=torch.float32, device="cuda")
        rx.rec_offsets_device(view, d_recs, len(recs), d_hz, torch.cuda.current_stream().cuda_stream)
        torch.cuda.synchronize()
        np.testing.assert_allclose(d_hz.cpu().numpy(), want, rtol=0, atol=2.0)
        del dbuf


def test_rec_offset_refuses_bad_records(rx):
    """n = 0 is a no-op; a record whose stream is outside the captures or whose chunk is negative is BTLE_EINVAL with
    last_error set, and the context stays usable.  The device form reads no sample for a negative chunk: its estimate is
    that of an empty window, the same as for a chunk past the capture."""
    n = 4 * CHUNK + 5
    iq = np.stack([_capture(n, 9, "burst"), _capture(n, 10, "burst")])
    assert rx.rec_offsets(iq, np.zeros(0, dtype=REC_DTYPE)).size == 0
    good = np.zeros(2, dtype=REC_DTYPE)
    good["stream"], good["chunk"], good["n0"], good["access_addr"] = [0, 1], [1, 2], [40, -50], 0x8E89BED6
    want = rx.rec_offsets(iq, good)
    for field, value, msg in (("stream", 2, "stream"), ("stream", -1, "stream"), ("chunk", -1, "chunk"), ("chunk", -(1 << 31), "chunk")):
        bad = good.copy()
        bad[field][1] = value
        with pytest.raises(BtleError) as e:
            rx.rec_offsets(iq, bad)
        assert e.value.code == BTLE_EINVAL and msg in str(e.value)
        _same(rx.rec_offsets(iq, good), want)
    d_iq = torch.zeros((2, (n + 15) // 16 * 16), dtype=torch.int8, device="cuda")
    d_iq[:, :n] = torch.from_numpy(iq).cuda()
    probe = np.zeros(3, dtype=REC_DTYPE)
    probe["stream"], probe["chunk"], probe["n0"], probe["access_addr"] = [1, 0, 0], [-1, -(1 << 31), 99], [100, 100, 100], 0x8E89BED6
    d_hz = torch.zeros(3, dtype=torch.float32, device="cuda")
    rx.rec_offsets_device(d_iq[:, :n], torch.from_numpy(probe.view(np.uint8).copy()).cuda(), 3, d_hz, torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    empty = offset_ref.rec_offset(iq[0], 99, 100, 0x8E89BED6)
    np.testing.assert_allclose(d_hz.cpu().numpy(), [empty] * 3, rtol=0, atol=2.0)
