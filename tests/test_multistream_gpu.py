"""Launches of one context spread over several CUDA streams, against the oracle (tests/orc.py) and the discovery
restatement (tests/discover_ref.py).

The launches of a context share its cached parameter arrays (cfg slots) and, with d_count == NULL, its ring of
allocation counters.  Each scenario holds one stream behind a bounded spin kernel (torch.cuda._sleep) while other
streams enqueue work, so that a launch ordered only by the host's call order, and not on the device, reads stale
parameters or starts from a stale count.  Every scenario first checks that the hold was still running when the other
streams' work had been enqueued ("hold too short" otherwise), so it can not pass without having held anything.

What a kernel sees in these scenarios is always a valid parameter array of the right size, or a counter with a wrong
start value that the stores' bounds (`cap`) absorb: a stale read gives wrong records, never a fault."""
import ctypes
import itertools

import numpy as np
import pytest
import torch

import discover_ref as R
import orc
from btle_b200 import CAND_DTYPE, DIR_DTYPE, REC_DTYPE, BtleRx, make_cfgs, synth
from btle_b200._native import BTLE_EINVAL, SYNTH_CFG_DTYPE
from test_discover import AAS, planted

pytestmark = pytest.mark.gpu

HOLD_CYCLES = 2_000_000_000            # ~1 s of spinning at H100 clocks: far longer than enqueueing any scenario
N_INT8 = 20 * 16384 + 1000             # ~20 chunks per capture keeps the CPU oracle cheap
NS = 3


@pytest.fixture(scope="module")
def built():
    import __graft_entry__ as ge
    ge.build()


@pytest.fixture
def rx(built):
    """A context of its own per test: the cfg cache and the counter ring start empty."""
    r = BtleRx(0)
    yield r
    torch.cuda.synchronize()
    r.close()


def _same(a, b):
    assert len(a) == len(b), (len(a), len(b))
    if a.tobytes() != b.tobytes():
        for i, (x, y) in enumerate(zip(a, b)):
            assert x.tobytes() == y.tobytes(), (i, x, y)


class _Hold:
    """Holds `stream` behind a spin kernel; check() fails unless it is still spinning."""

    def __init__(self, stream):
        with torch.cuda.stream(stream):
            torch.cuda._sleep(HOLD_CYCLES)
        self.ev = torch.cuda.Event()
        self.ev.record(stream)

    def check(self):
        assert not self.ev.query(), "hold too short: the held stream finished before the other streams' work was enqueued"


# ---- captures, cfg sets and what the oracle says about them ----------------------------------------------------------
def _captures(ns=NS, n=N_INT8, seed=0):
    """ns advertising captures (channels 37, 38, 39 in turn): int8 host array [ns, n] and its 16-byte-pitched device copy."""
    iq = np.stack([synth.make_adv_stream(n, seed=seed + 17 * s, channel=37 + s % 3, corrupt_every=7, slot_samples=2500)[0].numpy()
                   for s in range(ns)])
    d = torch.zeros((ns, (n + 15) // 16 * 16), dtype=torch.int8, device="cuda")
    d[:, :n] = torch.from_numpy(iq).cuda()
    return iq, d[:, :n]


def _cfg_set(k, ns=NS):
    """Twelve distinct cfg sets of ns streams: each decodes the same captures differently (the advertising channels in
    one of their six orders, so the whitening differs; RSSI on or off), so a launch that reads another set's parameters
    returns other records.  Set 0 and set 6 decode _captures() on their own channels."""
    order = list(itertools.permutations((37, 38, 39)))[k % 6]
    return make_cfgs(ns, channel=[order[s % 3] for s in range(ns)], rssi=(k // 6) % 2)


def _expect(iq, cfgs):
    return np.concatenate([orc.rx_flags(iq[s], int(c["rssi"]), channel=int(c["channel"]), access_addr=int(c["access_addr"]),
                                        access_mask=int(c["access_mask"]), crc_init=int(c["crc_init"]), raw=int(c["raw"]), stream=s)
                           for s, c in enumerate(cfgs)])


def _distinct(exps):
    blobs = [e.tobytes() for e in exps]
    assert all(len(e) > 0 for e in exps) and len(set(blobs)) == len(blobs), "cfg sets must decode the captures differently"


class _Rx:
    """One rx_device_dir launch with buffers of its own: d_out holds exactly the expected records (cap = their count),
    d_count is the caller's counter or None (the context's ring)."""

    def __init__(self, rx, d_iq, cfgs, exp, ring):
        self.rx, self.d_iq, self.cfgs, self.exp, self.ring = rx, d_iq, cfgs, exp, ring
        self.cap = len(exp)
        self.units = rx.units(*d_iq.shape)
        self.d_out = torch.zeros(self.cap * 64, dtype=torch.uint8, device="cuda")
        self.d_dir = torch.full((self.units, 2), -1, dtype=torch.int32, device="cuda")
        self.d_count = None if ring else torch.zeros(1, dtype=torch.int32, device="cuda")

    def run(self, stream):
        self.rx.rx_device_dir(self.d_iq, self.cfgs, self.d_out, self.d_count, self.d_dir, stream.cuda_stream)

    def check(self, what=""):
        unit_dir = np.ascontiguousarray(self.d_dir.cpu().numpy().view(np.uint32)).view(DIR_DTYPE).reshape(-1)
        total = int(unit_dir["count"].sum())
        end = int((unit_dir["base"].astype(np.int64) + unit_dir["count"]).max())
        assert total == len(self.exp), f"{what}: {total} records in the directory, oracle {len(self.exp)}"
        assert end <= self.cap, f"{what}: blocks reach record {end} of cap {self.cap} (the counter did not start at 0)"
        if self.ring:
            assert total == end, (what, total, end)
        else:
            assert int(self.d_count.item()) == total, what
        _same(self.rx.gather_ordered(self.d_out.cpu().numpy().view(REC_DTYPE), unit_dir), self.exp)


def _prefill(rx, d_iq, sets, stream):
    """Fill every cfg slot with a set of the same stream count (a slot that has to grow is freed with cudaFree, which
    synchronises the device and would void a hold)."""
    keep = [(torch.zeros(64, dtype=torch.uint8, device="cuda"), torch.zeros(1, dtype=torch.int32, device="cuda"),
             torch.zeros((rx.units(*d_iq.shape), 2), dtype=torch.int32, device="cuda")) for _ in sets]
    torch.cuda.synchronize()
    for cfgs, (d_out, d_count, d_dir) in zip(sets, keep):
        rx.rx_device_dir(d_iq, cfgs, d_out, d_count, d_dir, stream.cuda_stream)
    torch.cuda.synchronize()


# ---- the cfg cache ---------------------------------------------------------------------------------------------------
def test_cache_hit_waits_for_an_upload_held_on_another_stream(rx):
    """A: held, then set X (a miss: X is copied into the least recently used slot on A).  B: X again (a hit).  B's kernel
    must read X, not what the slot held before A's copies ran."""
    iq, d_iq = _captures()
    sets = [_cfg_set(k) for k in range(5)]
    exps = [_expect(iq, c) for c in sets]
    _distinct(exps)
    s0, a, b = torch.cuda.Stream(), torch.cuda.Stream(), torch.cuda.Stream()
    _prefill(rx, d_iq, sets[:4], s0)
    ja, jb = _Rx(rx, d_iq, sets[4], exps[4], False), _Rx(rx, d_iq, sets[4], exps[4], False)
    torch.cuda.synchronize()
    hold = _Hold(a)
    ja.run(a)
    jb.run(b)
    hold.check()
    torch.cuda.synchronize()
    jb.check("hit on B")
    ja.check("miss on A")


def test_eviction_waits_for_every_stream_that_read_the_slot(rx):
    """X is uploaded.  A: held, then X.  B: X (the last launch that read X's slot is now B's).  C: four sets not in the
    cache; the fourth evicts X's slot.  A's kernel, which runs after all of that was enqueued, must still read X."""
    iq, d_iq = _captures(seed=40)
    sets = [_cfg_set(k) for k in range(9)]
    exps = [_expect(iq, c) for c in sets]
    _distinct(exps)
    pre, x, others = sets[:3], sets[3], sets[4:8]
    s0, a, b, c = (torch.cuda.Stream() for _ in range(4))
    _prefill(rx, d_iq, pre + [sets[8]], s0)
    _prefill(rx, d_iq, [x], s0)                                 # cache: pre + X, X the most recently used
    ja, jb = _Rx(rx, d_iq, x, exps[3], False), _Rx(rx, d_iq, x, exps[3], False)
    jc = [_Rx(rx, d_iq, o, e, False) for o, e in zip(others, exps[4:8])]
    torch.cuda.synchronize()
    hold = _Hold(a)
    ja.run(a)
    jb.run(b)
    for j in jc:
        j.run(c)
    hold.check()
    torch.cuda.synchronize()
    ja.check("held launch on A")
    jb.check("B")
    for i, j in enumerate(jc):
        j.check(f"C{i}")


# ---- the counter ring (d_count == NULL) ------------------------------------------------------------------------------
def _warm_ring(rx, d_iq, cfgs, exp, stream, n=64):
    """n ring launches on `stream`, so that every counter of the ring has been used (and holds a count) once."""
    j = _Rx(rx, d_iq, cfgs, exp, True)
    for _ in range(n):
        j.run(stream)
    torch.cuda.synchronize()
    j.check("warm-up")


def test_a_failed_launch_does_not_poison_the_ring(rx):
    """A launch rejected after its checks ("batch too large") must not take a ring position: the ring position it took
    would never be cleared, and the launch 32 later would start from the count of the launch 64 before it."""
    iq, d_iq = _captures(seed=80)
    cfgs = _cfg_set(0)
    exp = _expect(iq, cfgs)
    st = torch.cuda.Stream()
    _warm_ring(rx, d_iq, cfgs, exp, st)
    n_big = 1 << 46
    small = torch.zeros(4096, dtype=torch.uint8, device="cuda")
    units = rx.units(1, n_big)
    one = make_cfgs(1)
    rc = rx._L.btle_b200_rx_device_dir(rx._h, small.data_ptr(), 1, n_big, n_big, one.ctypes.data, small.data_ptr(), 64, None,
                                       small.data_ptr(), units, ctypes.c_void_p(st.cuda_stream))
    assert rc == BTLE_EINVAL and b"too large" in rx._L.btle_b200_last_error(rx._h)
    jobs = [_Rx(rx, d_iq, cfgs, exp, True) for _ in range(70)]
    for j in jobs:
        j.run(st)
    torch.cuda.synchronize()
    for i, j in enumerate(jobs):
        j.check(f"launch {i} after the failed one")


def test_ring_across_three_streams_with_one_held(rx):
    """After 64 ring launches: A held, then one launch; B and C 40 launches in turn.  The 32nd of them takes the counter
    A's launch clears, and clears the one A's launch counts on: it must wait for A."""
    iq, d_iq = _captures(seed=120)
    cfgs = _cfg_set(1)
    exp = _expect(iq, cfgs)
    s0, a, b, c = (torch.cuda.Stream() for _ in range(4))
    _warm_ring(rx, d_iq, cfgs, exp, s0)
    ja = _Rx(rx, d_iq, cfgs, exp, True)
    jobs = [_Rx(rx, d_iq, cfgs, exp, True) for _ in range(40)]
    torch.cuda.synchronize()
    hold = _Hold(a)
    ja.run(a)
    for i, j in enumerate(jobs):
        j.run((b, c)[i & 1])
    hold.check()
    torch.cuda.synchronize()
    for i, j in enumerate(jobs):
        j.check(f"launch {i} on {'BC'[i & 1]}")
    ja.check("held launch on A")


# ---- discovery and synthesis share the cfg cache ---------------------------------------------------------------------
def _plant(iq, channel, aa, at, crc_init=0x227BA7):
    wav = synth.modulate(synth.air_bytes(synth.ll_data_pdu(1, 0, 0, 0, b""), channel, aa, crc_init)).astype(np.int32) * 64 // 127
    seg = iq[2 * at:2 * at + wav.size].astype(np.int32) + wav
    iq[2 * at:2 * at + wav.size] = np.clip(seg, -128, 127).astype(np.int8)


def test_discovery_eviction_waits_for_every_stream(rx):
    """The eviction scenario with discover_device: channel sets travel through the same cfg cache."""
    chans = [3, 9, 17, 30]
    n_samples = N_INT8 // 2
    iq = np.stack([planted(ch, AAS[s], at=1500, n_samples=n_samples, seed=s + 1) for s, ch in enumerate(chans)])
    for s, ch in enumerate(chans):
        for at in range(12000, n_samples - 2000, 25000):
            _plant(iq[s], ch, AAS[s], at + 37 * s)
    d_iq = torch.zeros((len(chans), (N_INT8 + 15) // 16 * 16), dtype=torch.int8, device="cuda")
    d_iq[:, :N_INT8] = torch.from_numpy(iq).cuda()
    d_iq = d_iq[:, :N_INT8]
    sets = [np.array(chans, dtype=np.int32)] + [np.array([(ch + k + 1) % 37 for ch in chans], dtype=np.int32) for k in range(8)]
    exps = [R.discover_batch(iq, c) for c in sets]
    assert len(exps[0]) >= 4 * 6 and all(e.tobytes() != exps[0].tobytes() for e in exps[1:])

    class Job:
        def __init__(self, k):
            self.k = k
            self.d_out = torch.zeros(max(len(exps[k]), 1) * 32, dtype=torch.uint8, device="cuda")
            self.d_count = torch.zeros(1, dtype=torch.int32, device="cuda")

        def run(self, stream):
            rx.discover_device(d_iq, sets[self.k], self.d_out, self.d_count, stream.cuda_stream)

        def check(self, what):
            n = int(self.d_count.item())
            assert n == len(exps[self.k]), (what, n, len(exps[self.k]))
            got = self.d_out[:n * 32].cpu().numpy().view(CAND_DTYPE)
            got = got[np.lexsort((got["sample"], got["stream"]))]
            assert got.tobytes() == exps[self.k].tobytes(), what

    s0, a, b, c = (torch.cuda.Stream() for _ in range(4))
    pre = [Job(k) for k in (5, 6, 7, 0)]                        # cache: three other sets + X, X the most recently used
    torch.cuda.synchronize()
    for j in pre:
        j.run(s0)
    torch.cuda.synchronize()
    ja, jb, jc = Job(0), Job(0), [Job(k) for k in (1, 2, 3, 4)]
    torch.cuda.synchronize()
    hold = _Hold(a)
    ja.run(a)
    jb.run(b)
    for j in jc:
        j.run(c)
    hold.check()
    torch.cuda.synchronize()
    ja.check("held discovery on A")
    jb.check("B")
    for i, j in enumerate(jc):
        j.check(f"C{i}")


def _synth(rx, out, cfgs, stream):
    sc = np.zeros(1, dtype=SYNTH_CFG_DTYPE)
    sc["seed"], sc["slot_samples"], sc["amplitude"], sc["corrupt_every"], sc["straddle_every"] = 99, 3300, 64, 5, 3
    got = ctypes.c_size_t(0)
    rx._check(rx._L.btle_b200_synth_streams_device(rx._h, out.data_ptr(), out.shape[0], out.stride(0), N_INT8, cfgs.ctypes.data,
                                                   sc.ctypes.data, None, 0, ctypes.byref(got), ctypes.c_void_p(stream.cuda_stream)))


def test_synthesis_eviction_waits_for_every_stream(rx):
    """The eviction scenario with synth_streams_device: the held call on A must generate what the same call generates
    alone on one synchronised stream."""
    sets = [_cfg_set(k, 4) for k in range(9)]
    pitch = (N_INT8 + 15) // 16 * 16
    buf = lambda: torch.zeros((4, pitch), dtype=torch.int8, device="cuda")
    ref_ctx, st = BtleRx(0), torch.cuda.Stream()
    refs = []
    for cfgs in sets:                                           # each set alone, on a context of its own
        refs.append(buf())
        _synth(ref_ctx, refs[-1], cfgs, st)
        torch.cuda.synchronize()
    ref_ctx.close()
    assert all(not torch.equal(r, refs[3]) for i, r in enumerate(refs) if i != 3)
    s0, a, b, c = (torch.cuda.Stream() for _ in range(4))
    pre = [buf() for _ in range(5)]
    torch.cuda.synchronize()
    for out, k in zip(pre, (0, 1, 2, 8, 3)):                   # cache: three other sets + X (set 3), X the most recently used
        _synth(rx, out, sets[k], s0)
    outs = {"A": buf(), "B": buf(), "C": [buf() for _ in range(4)]}
    torch.cuda.synchronize()
    hold = _Hold(a)
    _synth(rx, outs["A"], sets[3], a)
    _synth(rx, outs["B"], sets[3], b)
    for i, k in enumerate((4, 5, 6, 7)):
        _synth(rx, outs["C"][i], sets[k], c)
    hold.check()
    torch.cuda.synchronize()
    assert torch.equal(outs["A"], refs[3]), "held synthesis on A"
    assert torch.equal(outs["B"], refs[3]), "B"
    for i, k in enumerate((4, 5, 6, 7)):
        assert torch.equal(outs["C"][i], refs[k]), f"C{i}"


# ---- the benchmark's pattern -----------------------------------------------------------------------------------------
def test_double_buffered_steady_state(rx):
    """200 d_count == NULL launches alternating over two streams (as bench.py runs them), with four (capture shape, cfg
    set) pairs in rotation: every launch equals the oracle."""
    shapes = [(NS, N_INT8, 0, 2), (NS, N_INT8, 0, 7), (2, 13 * 16384 + 500, 200, 4), (4, 8 * 16384, 300, 9)]
    combos = []
    for ns, n, seed, k in shapes:
        iq, d_iq = _captures(ns, n, seed)
        cfgs = _cfg_set(k, ns)
        combos.append((d_iq, cfgs, _expect(iq, cfgs)))
    pipe = [torch.cuda.current_stream(), torch.cuda.Stream()]
    jobs = [_Rx(rx, *combos[i % len(combos)], True) for i in range(200)]
    torch.cuda.synchronize()
    for i, j in enumerate(jobs):
        j.run(pipe[i & 1])
    torch.cuda.synchronize()
    for i, j in enumerate(jobs):
        j.check(f"launch {i}")
