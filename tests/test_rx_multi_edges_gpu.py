"""The multi-cfg receive kernel (btle_rx_persistent_kernel<kMaxCfgsPerCapture>: btle_b200_rx_multi, _rx_multi_device_dir
and the cfg rounds of a streaming session) at its edges, against the oracle run once per cfg on the cfg's capture with
zeros around it (oracle_multi), byte for byte:

1. a bounded run of tools/fuzz_multi_gpu.py;
2. worst-case chunk densities: 123 records per chunk with -v and mask 0 (rows 68..122 stored by resolver step 4, once per
   cfg), 51 counted packets per chunk, and a degenerate cfg (the candidate walk) next to cfgs with exact hit lists;
3. every regime of the unit plan (1-chunk pieces, 4-chunk pieces, whole spans, and whole spans with more units per CTA
   than ring slots, where a slot's cfgs are reloaded between capture groups), with the directory checked entry by entry;
4. record capacities that cut between blocks, inside blocks and inside the late rows;
5. poisoned device views at every tile mode, and host captures copied from every kind of host memory, only the named
   ones, in runs.

2, 3, 4 and 5 also run in each mode the default kernels do not reach (tests/mode_ref.py): carrier-offset correction with
an offset of its own on every capture, the symbol-spaced discriminator, and both, against mode_ref.rx_multi, so that
every instantiation btle_rx_persistent_kernel<1|8, ROT, SYM> meets the spans and reuse regimes of the unit plan.

RSSI is on (flags 1 or 3) wherever bytes outside a capture could be read, so a stray read shows in mag_sum."""
import ctypes
import os
import subprocess
import sys
from functools import partial

import numpy as np
import pytest
import torch

from btle_b200 import CFG_DTYPE, DIR_DTYPE, REC_DTYPE, make_cfgs, synth
from btle_b200._native import BTLE_EOVERFLOW, CFG_RECOVER
import mode_ref
from test_ingest_edges_gpu import CHUNK, LENGTHS, SEG, SOURCES, HostBuf, _capture, _device_view, _plan, _poison, _same, _walk
from test_rx_multi import _traffic, oracle_multi

pytestmark = pytest.mark.gpu

CANARY = 0xA5
AAS = [0x8E89BED6, 0x60850A1B, 0x50850A1C, 0x12345679, 0x3A5C96E1, 0x71764129, 0x23AF04C8, 0x5A5AC3C3]
CRCS = [0x555555, 0x227BA7 ^ 0x0A1B, 0x227BA7 ^ 0x0A1C, 0x123456, 0x0BADC0, 0x1F2E3D, 0xA77B22, 0x000001]


@pytest.fixture(scope="module")
def rx():
    import __graft_entry__ as ge
    ge.build()
    from btle_b200 import BtleRx
    r = BtleRx(0)
    yield r
    r.close()


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _cfg_dict(c):
    return {k: int(c[k]) for k in CFG_DTYPE.names}


# ---- launches and their directory ----------------------------------------------------------------------------------------
def _group_of(capture):
    """Capture group (index among the distinct captures named) of every cfg."""
    cc = np.asarray(capture)
    return np.concatenate([[0], np.cumsum(cc[1:] != cc[:-1])]).astype(int)


def _multi_plan(rx, n_captures, capture, n_int8):
    """(plan rows (group, chunk0, n_chunks) of every unit, units per group); rx_multi_units == n_cfgs x units per group."""
    groups = int(_group_of(capture)[-1]) + 1
    plan = _plan(rx, groups, n_int8)
    per = len(plan) // groups
    assert per * groups == len(plan) and (plan[:, 0] == np.repeat(np.arange(groups), per)).all()
    assert rx.multi_units(n_captures, capture, n_int8) == len(capture) * per
    return plan, per


def _per_entry(exp, capture, plan, per):
    """Directory entry j * per + u: cfg j's oracle records in the chunks of unit u of its group."""
    g = _group_of(capture)
    out = []
    for j in range(len(capture)):
        e = exp[exp["stream"] == j]
        for u in range(per):
            _, c0, k = plan[g[j] * per + u]
            out.append(e[(e["chunk"] >= c0) & (e["chunk"] < c0 + k)])
    return out


def _launch(rx, d_iq, cfgs, capture, cap, room, with_count, offsets=None):
    """One btle_b200_rx_multi_device_dir(_offset) launch with record capacity `cap` into `room` records of CANARY bytes;
    the directory and counter start as -1.  Returns (record bytes [room, 64], directory, counter or None)."""
    ns, n = d_iq.shape
    cc = np.ascontiguousarray(capture, dtype=np.int32)
    off = None if offsets is None else np.ascontiguousarray(offsets, dtype=np.float32)
    units = rx.multi_units(ns, cc, n)
    d_out = torch.full((room, 64), CANARY, dtype=torch.uint8, device="cuda")
    d_dir = torch.full((units, 2), -1, dtype=torch.int32, device="cuda")
    d_count = torch.full((1,), -1, dtype=torch.int32, device="cuda") if with_count else None
    rx._check(rx._L.btle_b200_rx_multi_device_dir_offset(rx._h, d_iq.data_ptr(), ns, d_iq.stride(0), n, cfgs.ctypes.data, cc.ctypes.data,
                                                         cfgs.size, None if off is None else off.ctypes.data, d_out.data_ptr(), cap,
                                                         d_count.data_ptr() if with_count else None, d_dir.data_ptr(), units,
                                                         ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)))
    torch.cuda.synchronize()
    ud = np.ascontiguousarray(d_dir.cpu().numpy().view(np.uint32)).view(DIR_DTYPE).reshape(-1)
    return d_out.cpu().numpy(), ud, int(d_count.item()) if with_count else None


def _check_launch(rx, d_iq, cfgs, capture, exp, plan, per, cap, with_count, offsets=None):
    """A launch with capacity `cap` (<= the record count): nothing at or behind cap is written; the counter and the
    directory count every record; entry j * per + u holds cfg j's records of unit u (those below cap); blocks tile
    [0, total); gather_ordered returns the stored records in order, and BTLE_EOVERFLOW when some were cut."""
    total = len(exp)
    host, ud, count = _launch(rx, d_iq, cfgs, capture, cap, total + 64, with_count, offsets)
    assert (host[cap:] == CANARY).all(), f"cap {cap}: records stored at or behind cap"
    recs = host.reshape(-1).view(REC_DTYPE)
    if with_count:
        assert count == total
    want = _per_entry(exp, capture, plan, per)
    assert ud["count"].tolist() == [len(p) for p in want], cap
    live = np.flatnonzero(ud["count"])
    order = live[np.argsort(ud["base"][live])]
    assert ud["base"][order].tolist() == np.concatenate([[0], np.cumsum(ud["count"][order])[:-1]]).astype(int).tolist()
    avail = []
    for i, p in enumerate(want):
        b = int(ud["base"][i])
        m = max(0, min(len(p), cap - b))
        assert recs[b:b + m].tobytes() == p[:m].tobytes(), (cap, i)
        avail.append(p[:m])
    out = np.zeros(total, dtype=REC_DTYPE)
    got = ctypes.c_size_t(0)
    rc = rx._L.btle_b200_gather_ordered(recs.ctypes.data, cap, ud.ctypes.data, ud.size, out.ctypes.data, total, ctypes.byref(got))
    assert got.value == total and rc == (BTLE_EOVERFLOW if cap < total else 0)
    avail = np.concatenate(avail)
    _same(out[:len(avail)], avail)
    if cap == total:
        _same(out, exp)


def _device(iq):
    """Captures in device memory, rows 16 bytes apart (the device entry points' stride rule)."""
    pitch = (iq.shape[1] + 15) // 16 * 16
    d = torch.zeros((iq.shape[0], pitch), dtype=torch.int8, device="cuda")
    d[:, :iq.shape[1]] = torch.from_numpy(np.ascontiguousarray(iq)).cuda()
    return d[:, :iq.shape[1]]


# ---- 1. fuzz ---------------------------------------------------------------------------------------------------------------
def test_gpu_multi_fuzz_campaign_bounded():
    """tools/fuzz_multi_gpu.py for a bounded time: a fresh campaign of random rx_multi launches on every GPU run."""
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    p = subprocess.run([sys.executable, os.path.join(root, "tools", "fuzz_multi_gpu.py"), "20261016"], capture_output=True, text=True,
                       timeout=600, env=dict(os.environ, FUZZ_SECONDS="25"))
    assert p.returncode == 0, p.stdout[-2000:] + p.stderr[-3000:]
    assert " ok" in p.stdout


# ---- 2. worst-case chunk densities -----------------------------------------------------------------------------------------
N_WORST = 20 * CHUNK + 3008


def _rejected_cfgs():
    """Mask 0 with -v on the zero capture: 123 records in every chunk, rows 68..122 from step 4.  Eight access addresses
    and two channels, so a record stored under another cfg differs in its bytes."""
    return make_cfgs(8, channel=[38] * 5 + [39] + [38] * 2, access_addr=AAS, access_mask=0, crc_init=CRCS, rssi=[2, 3] * 4)


def _counted_cfgs():
    """Mask 0 on data channel 1 of the zero capture: 51 counted packets in every chunk."""
    return make_cfgs(8, channel=1, access_addr=AAS[::-1], access_mask=0, crc_init=CRCS, rssi=[0, 1, 2, 3] * 2)


def _mixed_cfgs():
    """One degenerate cfg (the candidate walk over the union candidates) next to four with exact hit lists."""
    return make_cfgs(5, channel=37, access_addr=AAS[:5], access_mask=[0xFFFFFFFF, 0, 0xFFFF00FF, 0xFFFFFFFF, 0xFFFFFFF0],
                     rssi=[1, 3, 3, 1, 3], raw=[0, 0, 0, 1, 0])


def _worst(mode):
    """Captures [zero, zero, traffic on channel 37], cfgs [8 rejected-hit cfgs, 8 counted-packet cfgs, the mixed five], in
    `mode`, where the -v cfgs also recover and the traffic capture sits at its own offset.  (iq, cfgs, capture, exp, offsets)."""
    iq = np.zeros((3, N_WORST), dtype=np.int8)
    iq[2] = _traffic(N_WORST, [37], AAS[:5], seed=29)[0]
    cfgs = np.concatenate([_rejected_cfgs(), _counted_cfgs(), _mixed_cfgs()])
    capture = np.repeat(np.arange(3, dtype=np.int32), [8, 8, 5])
    offsets = mode_ref.draw_offsets(np.random.default_rng(3 + mode[1]), 3, mode)
    if mode != (0, 0):
        cfgs = mode_ref.with_mode(cfgs, mode)
        cfgs["rssi"] |= np.where(cfgs["rssi"] & 2, CFG_RECOVER, 0).astype(np.int32)
        iq = mode_ref.rotate_all(iq, offsets)
    exp = mode_ref.rx_multi(iq, cfgs, capture, offsets)
    per_cfg = np.bincount(exp["stream"], minlength=len(cfgs))
    assert (per_cfg[:8] == 20 * 123).all() and (per_cfg[8:16] == 20 * 51).all()
    assert (exp["stream"] == 17).sum() > 20 * 5 and ((exp["stream"] >= 16) & (exp["crc_bad"] == 0) & (exp["stream"] != 17)).sum() > 10
    return iq, cfgs, capture, exp, offsets


@pytest.fixture(scope="module")
def worst():
    return _worst((0, 0))[:4]


def _densities(rx, iq, cfgs, capture, exp, offsets=None):
    assert len(exp) > len(cfgs) * 20 * 34 + 16
    _same(rx.rx_multi(iq, cfgs, capture, offset_hz=offsets), exp)
    d_iq = _device(iq)
    plan, per = _multi_plan(rx, 3, capture, N_WORST)
    for with_count in (True, False):
        _check_launch(rx, d_iq, cfgs, capture, exp, plan, per, len(exp), with_count, offsets)


def test_worst_case_densities_host_and_device(rx, worst):
    """rx_multi (its default capacity of 34 per chunk overflows: one retry at the exact count) and rx_multi_device_dir with a
    counter and with the counter ring, the directory checked entry by entry."""
    _densities(rx, *worst)


@pytest.mark.parametrize("seg", [1, 16])
def test_worst_case_densities_streaming_rounds(rx, worst, seg):
    """A one-capture session on the zero capture: the opening cfg removed, the 8 rejected-hit cfgs and 3 counted-packet
    cfgs added.  Every set takes two rx_multi rounds; the first finds exactly the records its capacity holds."""
    iq, _, _, _ = worst
    z = iq[0]
    added = [_cfg_dict(c) for c in _rejected_cfgs()] + [_cfg_dict(c) for c in _counted_cfgs()[:3]]
    with rx.streams(make_cfgs(1, channel=37, rssi=1), segment_chunks=seg) as s_:
        assert s_.remove_cfg(0) == 0
        idx = [s_.add_cfg(0, **f) for f in added]
        assert idx == [(j, 0) for j in range(1, 12)]
        parts = [s_.push(0, z)]
        assert rx.last_launches == 2
        parts.append(s_.finish())
        assert rx.last_launches == 2
    got = np.concatenate(parts)
    got = got[np.lexsort((got["chunk"], got["stream"]))]
    exp = oracle_multi(iq[:1], np.concatenate([make_cfgs(1, **f) for f in added]), np.zeros(len(added), dtype=np.int32))
    exp["stream"] += 1                                         # cfg j of the session is added cfg j - 1
    _same(got, exp)


# ---- 3. every unit plan, and slot refresh across capture groups ----------------------------------------------------------
COUNTS = [8, 1, 0, 5, 3, 8, 2, 7]                             # cfgs per capture, cycled: a slot's next group has another count


def _spliced(n_captures, n_int8, seed):
    """Bursts of all eight AAS on every capture: synth_streams_device captures, one per (address, capture) on the capture's
    channel, cut into eight segments and spliced so that segment i of capture c comes from address (c + i) % 8 (bursts
    cut short at the seams).  Returns (device view [n_captures, n_int8], channel of every capture)."""
    ch = (np.arange(n_captures) * 7 + 3) % 40
    src = make_cfgs(8 * n_captures, channel=np.tile(ch, 8), access_addr=np.repeat(AAS, n_captures), crc_init=np.repeat(CRCS, n_captures))
    d, _ = synth.synth_streams_device(src, n_int8, seed=seed, slot_samples=3300, amplitude=60, corrupt_every=6, straddle_every=4, want_truth=False)
    out = torch.zeros((n_captures, (n_int8 + 15) // 16 * 16), dtype=torch.int8, device="cuda")
    cuts = [i * (n_int8 // 8) for i in range(8)] + [n_int8]
    for i in range(8):
        rows = torch.tensor([((c + i) % 8) * n_captures + c for c in range(n_captures)], device="cuda")
        out[:, cuts[i]:cuts[i + 1]] = d[rows, cuts[i]:cuts[i + 1]]
    del d
    return out[:, :n_int8], ch


def _regime(G, name):
    """(named captures, n_int8) of a launch in each regime of make_plan; S = groups x spans per capture."""
    return {"pieces1": (max(1, G // 8 - 1), 17 * CHUNK + 3009),     # S = 2 x groups < G/4: 1-chunk pieces
            "pieces4": (G // 2 - 1, 17 * CHUNK + 255),              # G/4 <= S = G - 2 < G: 4-chunk pieces
            "spans": (3 * G // 10, 155 * CHUNK + 3008),             # G <= S <= 4G (10 spans): whole spans, <= 4 units per CTA
            "reuse": (G // 4 + 8, 249 * CHUNK + 3009)}[name]        # S > 4G (16 spans): ring slots reused across groups


@pytest.mark.parametrize("regime", ["pieces1", "pieces4", "spans", "reuse"])
def test_every_unit_plan(rx, regime):
    _every_unit_plan(rx, regime, (0, 0))


def _every_unit_plan(rx, regime, mode):
    G = _sms()
    groups, n = _regime(G, regime)
    counts = []
    while sum(k > 0 for k in counts) < groups:
        counts.append(COUNTS[len(counts) % len(COUNTS)])
    d_iq, ch = _spliced(len(counts), n, seed=len(counts) * 7 + n % 1000)
    iq = d_iq.cpu().numpy()
    rng = np.random.default_rng(n)
    offsets = mode_ref.draw_offsets(np.random.default_rng(n + 1), len(counts), mode)
    if offsets is not None:
        iq = mode_ref.rotate_all(iq, offsets)
        d_iq = _device(iq)
    cfgs, capture = [], []
    for c, k in enumerate(counts):
        for a in rng.permutation(8)[:k]:
            cfgs.append(make_cfgs(1, channel=int(ch[c]), access_addr=AAS[a], crc_init=CRCS[a], raw=int(rng.random() < 0.1),
                                  access_mask=int(rng.choice([0xFFFFFFFF, 0xFFFFFFFF, 0xFFFF00FF, 0xFFFFFFF0, 0x7FFFFFFE])),
                                  rssi=int(rng.choice([1, 3, 1, 3, 0, 2]))))
            capture.append(c)
    cfgs, capture = mode_ref.with_mode(np.concatenate(cfgs), mode), np.array(capture, dtype=np.int32)
    plan, per = _multi_plan(rx, len(counts), capture, n)
    spans = -(-(n // CHUNK) // 16)
    S = groups * spans
    assert plan[:, 2].max() == {"pieces1": 1, "pieces4": 4, "spans": 16, "reuse": 16}[regime]
    assert {"pieces1": S < G / 4, "pieces4": G / 4 <= S < G, "spans": G <= S <= 4 * G, "reuse": S > 4 * G}[regime]
    exp = mode_ref.rx_multi(iq, cfgs, capture, offsets)
    per_cfg = np.bincount(exp["stream"], minlength=len(cfgs))
    assert (per_cfg[cfgs["access_mask"] == 0xFFFFFFFF] > 0).all() and len(exp) > 4 * len(cfgs)
    for with_count in (True, False):
        _check_launch(rx, d_iq, cfgs, capture, exp, plan, per, len(exp), with_count, offsets)
    if mode == (0, 0):
        return
    # <1, ROT, SYM>: one cfg per capture (the first its list would hold, an exact mask), rx_batch and rx_device_dir
    ones = mode_ref.with_mode(make_cfgs(len(counts), channel=ch, access_addr=[AAS[c % 8] for c in range(len(counts))],
                                        crc_init=[CRCS[c % 8] for c in range(len(counts))], rssi=[1, 3] * (len(counts) // 2) + [1] * (len(counts) % 2)),
                              mode)
    exp1 = mode_ref.rx_multi(iq, ones, np.arange(len(counts)), offsets)
    assert (np.bincount(exp1["stream"], minlength=len(counts)) > 0).all()
    _same(rx.rx_batch(iq, ones, offset_hz=offsets), exp1)
    units = rx.units(len(counts), n)
    assert units == len(_plan(rx, len(counts), n))
    d_out = torch.zeros(len(exp1) * 64 + 64, dtype=torch.uint8, device="cuda")
    d_dir = torch.zeros((units, 2), dtype=torch.int32, device="cuda")
    rx.rx_device_dir(d_iq, ones, d_out, None, d_dir, torch.cuda.current_stream().cuda_stream, offset_hz=offsets)
    torch.cuda.synchronize()
    _same(_walk(rx, d_out, d_dir, units)[0], exp1)


@pytest.mark.parametrize("mode", mode_ref.NEW_MODES, ids=mode_ref.mode_id)
@pytest.mark.parametrize("regime", ["pieces1", "pieces4", "spans", "reuse"])
def test_every_unit_plan_in_modes(rx, regime, mode):
    """Every regime with the rotated and symbol-spaced kernels: the multi-cfg kernel <8, ROT, SYM> (the cfg list is not
    the identity) and the one-cfg kernel <1, ROT, SYM> through rx_batch and rx_device_dir on the same captures."""
    _every_unit_plan(rx, regime, mode)


# ---- 4. capacity cuts inside units -----------------------------------------------------------------------------------------
def test_capacity_cut_inside_units(rx, worst):
    """The zero capture with the 8 rejected-hit cfgs: 20 one-chunk units per cfg, 123 records each, so multiples of 123
    are block boundaries whatever the order the blocks are reserved in; cuts at 0 and 1, at a boundary, inside a block's
    hit row (+40, +67) and inside its late rows (+68, +100), at total - 1 and at total.  Then a mixed traffic batch with
    cuts inside blocks."""
    _capacity_cuts(rx, *worst)


@pytest.mark.parametrize("mode", mode_ref.NEW_MODES, ids=mode_ref.mode_id)
def test_worst_case_densities_and_capacity_cuts_in_modes(rx, mode):
    """The two tests above with the rotated and symbol-spaced kernels, recovery on the -v cfgs."""
    w = _worst(mode)
    _densities(rx, *w)
    _capacity_cuts(rx, *w, mode=mode)


def _capacity_cuts(rx, iq, cfgs, capture, exp, offsets=None, mode=(0, 0)):
    cfgs, capture, exp = cfgs[:8], capture[:8], exp[exp["stream"] < 8]
    off1 = None if offsets is None else offsets[:1]
    d_iq = _device(iq[:1])
    plan, per = _multi_plan(rx, 1, capture, N_WORST)
    assert (plan[:, 2] <= 1).all()
    total = len(exp)
    for with_count in (True, False):
        for cap in (0, 1, 5 * 123, 5 * 123 + 40, 5 * 123 + 67, 5 * 123 + 68, 5 * 123 + 100, total - 1, total):
            _check_launch(rx, d_iq, cfgs, capture, exp, plan, per, cap, with_count, off1)

    n = 40 * CHUNK + 777
    iq = _traffic(n, [37, 5, 38, 22], AAS[:5], seed=9)
    offsets = mode_ref.draw_offsets(np.random.default_rng(8), 4, mode)
    iq = mode_ref.rotate_all(iq, offsets)
    cfgs = make_cfgs(9, channel=[37, 37, 37, 5, 5, 38, 22, 22, 22],
                     access_addr=[AAS[0], AAS[4], AAS[1], AAS[1], AAS[3], AAS[2], AAS[4], AAS[3], AAS[0]],
                     access_mask=[0xFFFFFFFF, 0, 0xFFFFFFFF, 0xFFFFFFFF, 0xFFFF00FF, 0xFFFFFFFF, 0xFFFFFFFF, 0xFFFFFFFF, 0xFFFFFFF0],
                     crc_init=[0x555555, 0x555555, 0x555555, 0x227BA7 ^ 0x0A1B, 0x227BA7 ^ 0x5679, 0x555555, 0x227BA7 ^ 0x96E1,
                               0x227BA7 ^ 0x5679, 0x123456], rssi=[1, 3, 3, 1, 3, 1, 3, 1, 2])
    cfgs = mode_ref.with_mode(cfgs, mode)
    if mode != (0, 0):
        cfgs["rssi"] |= np.where(cfgs["rssi"] & 2, CFG_RECOVER, 0).astype(np.int32)
    capture = np.array([0, 0, 0, 1, 1, 2, 3, 3, 3], dtype=np.int32)
    exp = mode_ref.rx_multi(iq, cfgs, capture, offsets)
    assert len(exp) > 500 and (np.bincount(exp["stream"], minlength=9) > 0).all()
    d_iq = _device(iq)
    plan, per = _multi_plan(rx, 4, capture, n)
    for with_count in (True, False):
        for cap in (3, len(exp) // 3 + 1, len(exp) - 5, len(exp)):
            _check_launch(rx, d_iq, cfgs, capture, exp, plan, per, cap, with_count, offsets)


# ---- 5. poisoned device views and host ingest ------------------------------------------------------------------------------
def _view_cfgs():
    """Per capture of [burst, noise, burst]: the front-cut burst (mask 0xFFFFFF00), the hit at n0 = -124 in chunk 0 (mask 0
    with -v on noise), the burst cut at the capture's end, and cfgs that find nothing there."""
    cfgs = make_cfgs(9, channel=[37, 37, 38, 38, 37, 37, 37, 39, 37],
                     access_addr=[0x8E89BED6, 0x8E89BED6, 0x12345679, 0, 0x8E89BED6, 0x8E89BED6, 0x8E89BED6, 0x8E89BED6, 0x60850A1B],
                     access_mask=[0xFFFFFF00, 0xFFFFFFFF, 0xFFFFFFFF, 0, 0x0000000F, 0xFFFFFFFF, 0xFFFFFF00, 0xFFFF0000, 0xFFFFFFFF],
                     rssi=[3, 1, 1, 3, 3, 1, 3, 1, 3])
    return cfgs, np.array([0, 0, 0, 1, 1, 2, 2, 2, 2], dtype=np.int32)


@pytest.mark.parametrize("n_int8", LENGTHS)
def test_rx_multi_device_dir_poisoned_views(rx, n_int8):
    """Every byte outside [0, n_int8) of a view is poison; all three captures, and captures 0 and 2 alone (capture 1 is then
    read by no cfg)."""
    _poisoned_views(rx, n_int8, (0, 0))


@pytest.mark.parametrize("mode", mode_ref.NEW_MODES, ids=mode_ref.mode_id)
@pytest.mark.parametrize("n_int8", LENGTHS)
def test_rx_multi_device_dir_poisoned_views_in_modes(rx, n_int8, mode):
    """The same with the rotated and symbol-spaced kernels: the symbol-spaced dense loop reads the word in front of each
    tile (`head`), which for a capture's first tile lies in the poison and must read as 0."""
    _poisoned_views(rx, n_int8, mode)


def _poisoned_views(rx, n_int8, mode):
    rng = np.random.default_rng(n_int8 + 1)
    iq = np.stack([_capture(n_int8, n_int8 % 1013, "burst", phase=1), _capture(n_int8, n_int8 % 1013 + 1, "noise"),
                   _capture(n_int8, n_int8 % 1013 + 2, "burst", phase=3)])
    offsets = mode_ref.draw_offsets(np.random.default_rng(n_int8), 3, mode)
    iq = mode_ref.rotate_all(iq, offsets)
    cfgs, capture = _view_cfgs()
    cfgs = mode_ref.with_mode(cfgs, mode)
    exp = mode_ref.rx_multi(iq, cfgs, capture, offsets)
    assert ((exp["chunk"] == 0) & (exp["n0"] == -124)).any() and ((exp["chunk"] == 0) & (exp["n0"] < 0) & ((exp["flags"] & 4) == 0)).any()
    skip = capture != 1
    exp_skip = mode_ref.rx_multi(iq, cfgs[skip], capture[skip], offsets)
    for front, extra in ((16, 0), (256, 48), (4096, 4096)):
        stride = (n_int8 + 15) // 16 * 16 + extra
        buf, view = _device_view(list(iq), stride, front, rng, random_poison=front != 256)
        for sel, want in ((slice(None), exp), (skip, exp_skip)):
            n_units = rx.multi_units(3, capture[sel], n_int8)
            d_out = torch.zeros(len(want) + 16, 64, dtype=torch.uint8, device="cuda")
            d_dir = torch.zeros(n_units, 2, dtype=torch.int32, device="cuda")
            d_count = torch.zeros(1, dtype=torch.int32, device="cuda")
            rx.rx_multi_device_dir(view, cfgs[sel], capture[sel], d_out, d_count, d_dir, torch.cuda.current_stream().cuda_stream,
                                   offset_hz=offsets)
            torch.cuda.synchronize()
            assert int(d_count.item()) == len(want)
            ud = np.ascontiguousarray(d_dir.cpu().numpy().view(np.uint32)).view(DIR_DTYPE).reshape(-1)
            _same(rx.gather_ordered(d_out.cpu().numpy().view(REC_DTYPE).reshape(-1), ud), want)
        del buf


NAMED = [1, 2, 4, 7]                                           # of 8 captures: copy runs [1, 2], [4], [7]


def _host_case(n_int8, seed, device=None, mode=(0, 0)):
    """Captures NAMED of 8 (the others are never read), 2 or 3 cfgs each, in `mode`; (captures [8, n_int8], cfgs, capture,
    expected records, offsets)."""
    iq = np.zeros((8, n_int8), dtype=np.int8)
    offsets = mode_ref.draw_offsets(np.random.default_rng(seed), 8, mode)
    for k, c in enumerate(NAMED):
        iq[c] = _capture(n_int8, seed + c, "noise" if k == 2 else "burst", device, phase=k)
        if offsets is not None:
            iq[c] = mode_ref.rotate(iq[c], float(offsets[c]))
    per = [dict(channel=[37, 37, 38], access_mask=[0xFFFFFF00, 0xFFFFFFFF, 0], access_addr=[0x8E89BED6, 0x8E89BED6, 0x12345679], rssi=[3, 1, 3]),
           dict(channel=[37, 39], access_mask=[0xFFFFFFFF, 0xFFFFFF00], rssi=[1, 3]),
           dict(channel=[38, 37], access_addr=[0, 0x8E89BED6], access_mask=[0, 0x0000000F], rssi=[3, 3]),
           dict(channel=[37, 37, 22], access_mask=[0xFFFFFF00, 0xFFFFFFFF, 0xFFFFFFFF], access_addr=[0x8E89BED6, 0x8E89BED6, 0x3A5C96E1],
                crc_init=[0x555555, 0x555555, 0x227BA7 ^ 0x96E1], rssi=[1, 3, 1])]
    parts = [make_cfgs(len(p["channel"]), **p) for p in per]
    cfgs = mode_ref.with_mode(np.concatenate(parts), mode)
    capture = np.repeat(np.array(NAMED, dtype=np.int32), [len(p) for p in parts])
    return iq, cfgs, capture, mode_ref.rx_multi(iq, cfgs, capture, offsets), offsets


def _rx_multi_host(rx, ptr, stride, n_int8, cfgs, capture, offsets=None):
    cc = np.ascontiguousarray(capture, dtype=np.int32)
    off = None if offsets is None else np.ascontiguousarray(offsets, dtype=np.float32)
    return rx._grow_once(partial(rx._L.btle_b200_rx_multi_offset, rx._h, ptr, 8, stride, n_int8, cfgs.ctypes.data, cc.ctypes.data, cfgs.size,
                                 None if off is None else off.ctypes.data), REC_DTYPE, cfgs.size * (n_int8 // CHUNK) * 34 + 16)


def _lay_out_named(buf, iq, stride, rng, random_poison):
    """The named captures stride bytes apart in buf.a; poison in every other capture's place and in the padding."""
    buf.a[:] = _poison(buf.a.size, rng, random_poison)
    for c in NAMED:
        buf.a[c * stride:c * stride + iq.shape[1]] = iq[c]


@pytest.mark.parametrize("source", SOURCES)
def test_rx_multi_host_ingest_matrix(rx, source):
    """btle_b200_rx_multi from each kind of host memory with a stride: only the named captures are copied, one copy per
    run of consecutive ones; poisoned captures and padding must not change a record."""
    _host_ingest(rx, source, (0, 0))


@pytest.mark.parametrize("mode", mode_ref.NEW_MODES, ids=mode_ref.mode_id)
@pytest.mark.parametrize("source", SOURCES)
def test_rx_multi_host_ingest_matrix_in_modes(rx, source, mode):
    """The same through btle_b200_rx_multi_offset with the rotated and symbol-spaced kernels."""
    _host_ingest(rx, source, mode)


def _host_ingest(rx, source, mode):
    rng = np.random.default_rng(17)
    for n in (6 * CHUNK, 6 * CHUNK + 1005):
        iq, cfgs, capture, exp, offsets = _host_case(n, seed=n % 977, mode=mode)
        assert ((exp["chunk"] == 0) & (exp["n0"] < 0)).sum() >= 2 and (exp["flags"] & 4).any()
        for extra in (0, 7, 4096):
            buf = HostBuf(source, 8 * (n + extra))
            try:
                _lay_out_named(buf, iq, n + extra, rng, random_poison=extra != 7)
                _same(_rx_multi_host(rx, buf.ptr, n + extra, n, cfgs, capture, offsets), exp)
            finally:
                buf.close()


def test_rx_multi_host_captures_larger_than_a_staging_segment(rx):
    """Pageable captures of 32 MiB + 5 chunks + 3 bytes: every named capture is more than one staging segment."""
    n = SEG + 5 * CHUNK + 3
    iq, cfgs, capture, exp, _ = _host_case(n, seed=300, device="cuda")
    assert (np.bincount(exp["stream"], minlength=len(cfgs)) > 0).sum() >= 7
    buf = HostBuf("pageable", 8 * (n + 4099))
    _lay_out_named(buf, iq, n + 4099, np.random.default_rng(5), random_poison=True)
    _same(_rx_multi_host(rx, buf.ptr, n + 4099, n, cfgs, capture), exp)
