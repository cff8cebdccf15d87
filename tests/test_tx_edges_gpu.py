"""The transmit modulator and the capture synthesiser at their edges, byte for byte against plain restatements.

- btle_b200_tx_modulate_device at every max_bytes up to 128, so packets end in the first, second and third pass of
  gfsk_block (2048 samples per pass at 4 sps, 4096 at 8 sps) and the phase is carried across passes; nbytes out of
  range is clamped to 0..max_bytes.  Reference: test_tx_reference_cpu.modulate4_ref / modulate8_ref.
- synth_noise_kernel's three floors on packed, strided and unaligned layouts, restated from the counter-based draw;
  no byte outside the captures is written.
- synth_bursts_kernel rebuilt from its truth on those layouts and at the minimum slot sizes, and where it places
  its bursts: order, gaps, slots, chunk boundaries, corrupt slots and PDU contents, over many seeds."""
import ctypes

import numpy as np
import pytest
import torch
from scipy.special import erfc

from btle_b200 import BtleRx, synth
from btle_b200._native import BTLE_EINVAL, SYNTH_CFG_DTYPE, SYNTH_TRUTH_DTYPE
from test_model_path_gpu import draw
from test_synth_bursts_exact_gpu import rebuild
from test_tx_reference_cpu import modulate4_ref, modulate8_ref, random_rows

pytestmark = pytest.mark.gpu

POISON = 0x5A
CHUNK = 8192                                 # kChunkSamples: the receive ring's chunk, which straddlers cross
INT32_MIN = -(1 << 31)


@pytest.fixture(scope="module")
def ctx():
    c = BtleRx(0)
    yield c
    c.close()


# ---- btle_b200_tx_modulate_device ------------------------------------------------------------------------------------
def tx_device(ctx, air, nb, sps, stream=None):
    """Modulate rows `air` [B, L] of lengths `nb` into buffers of B + 1 poisoned rows; the row behind the batch must
    keep its poison.  Returns int8 [B, 2 n_out] (sps 4) or ([B, n_out], [B, n_out]) (sps 8), n_out = 8 L sps + 16."""
    B, L = air.shape
    n_out = 8 * L * sps + 16
    d_air = torch.from_numpy(np.ascontiguousarray(air)).cuda()
    d_nb = torch.from_numpy(np.asarray(nb, dtype=np.int32)).cuda()
    outs = [torch.full((B + 1, 2 * n_out if sps == 4 else n_out), POISON, dtype=torch.int8, device="cuda") for _ in range(sps // 4)]
    torch.cuda.synchronize()
    st = stream if stream is not None else torch.cuda.current_stream()
    ctx._check(ctx._L.btle_b200_tx_modulate_device(ctx._h, d_air.data_ptr(), d_nb.data_ptr(), B, L, sps, outs[0].data_ptr(),
                                                   outs[-1].data_ptr() if sps == 8 else None, ctypes.c_void_p(st.cuda_stream)))
    st.synchronize()
    host = [o.cpu().numpy() for o in outs]
    for h in host:
        assert (h[B] == POISON).all(), "a row behind the batch was written"
    return host[0][:B] if sps == 4 else (host[0][:B], host[1][:B])


def tx_ref(air, nb, sps):
    nb = np.clip(np.asarray(nb, dtype=np.int64), 0, air.shape[1])
    return modulate4_ref(air, nb) if sps == 4 else modulate8_ref(air, nb)


def assert_tx_equal(got, ref, nb):
    for g, r in zip((got,) if isinstance(got, np.ndarray) else got, (ref,) if isinstance(ref, np.ndarray) else ref):
        bad = np.nonzero((g != r).any(axis=1))[0]
        assert bad.size == 0, f"rows {bad[:8].tolist()} (nbytes {np.asarray(nb)[bad[:8]].tolist()}) differ from the reference"


@pytest.mark.parametrize("max_bytes", [1, 2, 63, 64, 65, 100, 127, 128])
@pytest.mark.parametrize("sps", [4, 8])
def test_tx_modulate_every_length(ctx, sps, max_bytes):
    """Rows of 0, 1, max_bytes - 1 and max_bytes bytes, all-0x00 and all-0xFF rows (the phase runs furthest from zero),
    63 / 64 / 65 / 127 / 128 where they fit (the packet ends 16 samples before a pass edge, 16 and 48 samples after
    it, in the third pass), random lengths; bytes behind a row's length are random and must not matter."""
    rng = np.random.default_rng(100 * sps + max_bytes)
    lens = [max_bytes, max_bytes, 0, 1, max_bytes - 1] + [n for n in (63, 64, 65, 127, 128) if n <= max_bytes]
    lens += rng.integers(0, max_bytes + 1, 8).tolist()
    air, _ = random_rows(rng, len(lens), max_bytes)
    nb = np.array(lens)
    assert_tx_equal(tx_device(ctx, air, nb, sps), tx_ref(air, nb, sps), nb)


@pytest.mark.parametrize("sps", [4, 8])
def test_tx_modulate_batch_past_65535_rows(ctx, sps):
    rng = np.random.default_rng(7 + sps)
    air, nb = random_rows(rng, 70001, 3)
    assert_tx_equal(tx_device(ctx, air, nb, sps), tx_ref(air, nb, sps), nb)


def test_tx_modulate_on_a_side_stream(ctx):
    rng = np.random.default_rng(11)
    air, nb = random_rows(rng, 12, 128)
    side = torch.cuda.Stream()
    assert side.cuda_stream != torch.cuda.current_stream().cuda_stream
    assert_tx_equal(tx_device(ctx, air, nb, 8, stream=side), tx_ref(air, nb, 8), nb)


@pytest.mark.parametrize("max_bytes", [1, 64, 100])
@pytest.mark.parametrize("sps", [4, 8])
def test_tx_modulate_clamps_nbytes(ctx, sps, max_bytes):
    """nbytes above max_bytes is modulated as max_bytes, below 0 as 0.  Over-long rows stay at most 2 max_bytes (and 128)
    and are never the batch's last row, so an unclamped kernel reads only inside d_air and shows as a mismatch."""
    rng = np.random.default_rng(max_bytes)
    over = min(128, 2 * max_bytes)
    nb = np.array([over, max_bytes, -1, INT32_MIN, 0, max_bytes + 1, max_bytes])
    air, _ = random_rows(rng, len(nb), max_bytes, extremes=False)
    air[1] = air[0]
    got = tx_device(ctx, air, nb, sps)
    assert_tx_equal(got, tx_ref(air, nb, sps), nb)
    for g in (got,) if sps == 4 else got:
        assert np.array_equal(g[0], g[1]) and np.array_equal(g[2], g[4]) and np.array_equal(g[3], g[4])


# ---- btle_b200_synth_streams_device --------------------------------------------------------------------------------------
def noise_thresholds():
    """P(round(N(-0.3, 0.8)) <= v) * 2^32, floored, for v = -7 .. 5, in float64.  The library takes the same formula from
    glibc's erfc: a one-ulp difference between the two would change a byte only for a draw exactly on a threshold."""
    v = np.arange(-7, 6, dtype=np.float64)
    p = 0.5 * erfc(-((v + 0.5 + 0.3) / 0.8) / np.sqrt(2.0))
    return np.minimum(np.floor(p * 2.0 ** 32), 2.0 ** 32 - 1).astype(np.uint64)


def noise_ref(seed, n_streams, n_int8, kind):
    """synth_noise_kernel restated: the capture is 16-byte pieces p, a piece of kind 0 holds for q = 0..7 the floor values
    of the low and high halves of draw(seed, s, 8p + q, 1); kind 1 the bytes of draw(seed, s, 2p) and draw(seed, s, 2p + 1)
    little-endian; kind 2 zeros.  int8 [n_streams, n_int8]."""
    per = (n_int8 + 15) // 16
    out = np.zeros((n_streams, 16 * per), dtype=np.int8)
    if kind == 2:
        return out[:, :n_int8]
    for s in range(n_streams):
        if kind == 0:
            r = draw(seed, s, np.arange(8 * per, dtype=np.uint64), 1)
            halves = np.stack([r & np.uint64(0xFFFFFFFF), r >> np.uint64(32)], axis=1).reshape(-1)      # [16 per]
            v = np.full(halves.shape, -7, dtype=np.int64)
            for t in noise_thresholds():
                v += halves >= t
            out[s] = v.astype(np.int8)
        else:
            r = draw(seed, s, np.arange(2 * per, dtype=np.uint64), 1)
            out[s] = r.astype("<u8").view(np.int8)
    return out[:, :n_int8]


def synth_call(ctx, cfgs, n_int8, stride, offset, seed, truth=False, truth_short=0, **kw):
    """btle_b200_synth_streams_device into a poisoned buffer at `offset` bytes past a 256-byte-aligned base, with 64
    poisoned bytes behind the last capture.  Returns (rc, whole buffer int8, truth or None, *n_slots_out)."""
    ns = len(cfgs)
    buf = torch.full((offset + (ns - 1) * stride + n_int8 + 64,), POISON, dtype=torch.int8, device="cuda")
    assert buf.data_ptr() % 256 == 0
    sc = np.zeros(1, dtype=SYNTH_CFG_DTYPE)
    sc["seed"] = seed
    for k, v in dict(dict(slot_samples=3200, amplitude=0, corrupt_every=0, straddle_every=0, noise=0), **kw).items():
        sc[k] = v
    n_slots = (n_int8 // 2) // int(sc["slot_samples"][0])
    cap = ns * n_slots - truth_short
    d_truth = torch.zeros((max(1, cap), 64), dtype=torch.uint8, device="cuda") if truth else None
    got = ctypes.c_size_t(12345)
    cfgs = np.ascontiguousarray(cfgs)
    torch.cuda.synchronize()
    rc = ctx._L.btle_b200_synth_streams_device(ctx._h, buf.data_ptr() + offset, ns, stride, n_int8, cfgs.ctypes.data, sc.ctypes.data,
                                               d_truth.data_ptr() if truth else None, cap if truth else 0, ctypes.byref(got),
                                               ctypes.c_void_p(torch.cuda.current_stream().cuda_stream))
    torch.cuda.synchronize()
    t = d_truth[:cap].cpu().numpy().view(SYNTH_TRUTH_DTYPE).reshape(-1) if truth else None
    return rc, buf.cpu().numpy(), t, got.value


def captures(host, ns, stride, offset, n_int8):
    """the captures [ns, n_int8] out of the whole buffer, after checking that every byte between and around them is poison"""
    pad = np.ones(host.size, dtype=bool)
    for s in range(ns):
        pad[offset + s * stride:offset + s * stride + n_int8] = False
    assert (host[pad] == POISON).all(), f"{int((host[pad] != POISON).sum())} padding bytes written"
    return np.stack([host[offset + s * stride:offset + s * stride + n_int8] for s in range(ns)])


# capture stride from n_int8: packed (later captures are unaligned), odd padding, 16-byte pitch + 48
STRIDES = {"packed": lambda n: n, "odd": lambda n: n + 7, "pitched": lambda n: (n + 15) // 16 * 16 + 48}


def layouts(n_int8):
    """(stride, offset) of every stride with the base 0, 1 or 8 bytes off 256-byte alignment"""
    return [(st(n_int8), off) for st in STRIDES.values() for off in (0, 1, 8)]


@pytest.mark.parametrize("n_int8", [1, 15, 16, 17, 4109, (1 << 20) + 1])
def test_noise_floor_equals_its_restatement_on_every_layout(ctx, n_int8):
    cfgs = synth.channel_plan(5)
    for kind in (0, 1, 2):
        seed = 0x9E3779B97F4A7C15 + 1000 * kind + n_int8
        ref = noise_ref(seed, 5, n_int8, kind)
        for ns in (1, 5):
            for stride, off in layouts(n_int8):
                rc, host, _, _ = synth_call(ctx, cfgs[:ns], n_int8, stride, off, seed, noise=kind)
                assert rc == 0
                cap = captures(host, ns, stride, off, n_int8)
                assert np.array_equal(cap, ref[:ns]), (kind, ns, stride, off)


# bursts on every floor and layout: (slot_samples, straddle_every, noise, stride, offset, amplitude)
BURST_CASES = [
    (1600, 0, 0, "packed", 1, 127),
    (3200, 2, 0, "odd", 8, 64),
    (3200, 2, 1, "pitched", 0, 100),
    (1600, 0, 2, "odd", 1, 1),
]


@pytest.mark.parametrize("slot,straddle,noise,layout,offset,amplitude", BURST_CASES)
def test_bursts_equal_their_rebuilt_truth_on_every_layout(ctx, slot, straddle, noise, layout, offset, amplitude):
    cfgs = synth.channel_plan(40)[[0, 11, 24, 36, 37, 38, 39]]
    ns = len(cfgs)
    n_int8 = 2 * slot * 48 + 2 * 777 + 1                         # odd: the capture ends inside a slot
    stride = STRIDES[layout](n_int8)
    seed = 5000 + slot + noise
    rc, host, truth, n_slots = synth_call(ctx, cfgs, n_int8, stride, offset, seed, truth=True, slot_samples=slot, amplitude=amplitude,
                                          corrupt_every=3, straddle_every=straddle, noise=noise)
    assert rc == 0 and n_slots == 48 and len(truth) == ns * 48
    assert straddle == 0 or truth["straddle"].sum() >= 10
    assert (truth["corrupt"] == 1).any()
    got = captures(host, ns, stride, offset, n_int8)
    assert np.array_equal(got, rebuild(cfgs, truth, noise_ref(seed, ns, n_int8, noise), seed, amplitude))


def expected_pdus(seed, cfgs, truth):
    """every truth record's PDU (header + payload, zeros behind) from its definition"""
    s, k = truth["stream"].astype(np.uint64), truth["slot"].astype(np.uint64)
    adv = cfgs["channel"][truth["stream"]] >= 37
    r = draw(seed, s, k, 2)
    pdu_len = np.where(adv, 8 + (r % np.uint64(32)).astype(np.int64), 2 + (r % np.uint64(28)).astype(np.int64))
    words = np.stack([draw(seed, s, k, 3 + w) for w in range(5)], axis=1)             # payload bytes 0..39
    payload = words.astype("<u8").view(np.uint8).reshape(len(truth), 40)
    pdu = np.zeros((len(truth), 44), dtype=np.uint8)
    adva = truth["slot"].astype(np.uint64) | (s << np.uint64(32))
    llid = 1 + ((r >> np.uint64(8)) & np.uint64(1)).astype(np.int64)
    hdr = llid | ((truth["slot"] & 1) << 2) | (((truth["slot"] >> 1) & 1) << 3)
    for i in range(len(truth)):
        n = int(pdu_len[i])
        pdu[i, 1] = n - 2
        if adv[i]:
            pdu[i, 0] = 0x40
            pdu[i, 2:8] = np.frombuffer(int(adva[i]).to_bytes(6, "little"), dtype=np.uint8)
            pdu[i, 8:n] = payload[i, 6:n - 2]
        else:
            pdu[i, 0] = hdr[i]
            pdu[i, 2:n] = payload[i, :n - 2]
    return pdu_len, pdu


@pytest.mark.parametrize("slot,straddle", [(1600, 0), (3200, 2), (4096, 3)])
def test_burst_placement_and_pdus(ctx, slot, straddle):
    """Over 12 seeds on advertising and data channels: bursts in slot order, never overlapping, 32 samples clear of a
    straddling predecessor, inside their slot otherwise; straddlers cross a chunk boundary; corrupt exactly every
    corrupt_every-th slot; PDU header, length, AdvA and payload from the counter-based draw."""
    cfgs = synth.channel_plan(40)[[37, 38, 39, 0, 17, 36]]
    ns, n_slots = len(cfgs), 300
    n_int8 = 2 * slot * n_slots + 1001
    looked_back = 0
    for seed in range(12):
        ce = (0, 1, 2, 3, 7, 10)[seed % 6]
        rc, _, truth, got = synth_call(ctx, cfgs, n_int8, n_int8 + 7, 0, 77 * seed + slot, truth=True, slot_samples=slot, amplitude=1,
                                       corrupt_every=ce, straddle_every=straddle, noise=2)
        assert rc == 0 and got == n_slots
        sl = truth["slot"].astype(np.int64)
        assert np.array_equal(truth["stream"], np.repeat(np.arange(ns), n_slots)) and np.array_equal(sl, np.tile(np.arange(n_slots), ns))
        pdu_len, pdu = expected_pdus(77 * seed + slot, cfgs, truth)
        assert np.array_equal(truth["pdu_len"], pdu_len) and np.array_equal(truth["n_air_bytes"], pdu_len + 8)
        assert np.array_equal(truth["pdu"], pdu)
        assert np.array_equal(truth["corrupt"] == 1, (ce > 0) & (sl % max(ce, 1) == ce - 1))
        start = truth["start_sample"].reshape(ns, n_slots)
        end = start + 32 * truth["n_air_bytes"].reshape(ns, n_slots).astype(np.int64) + 16
        strad = truth["straddle"].reshape(ns, n_slots) == 1
        lo, hi = np.arange(n_slots) * slot, (np.arange(n_slots) + 1) * slot
        assert (start >= lo).all()
        assert (start[:, 1:] >= end[:, :-1]).all(), "bursts overlap or are out of slot order"
        follows = np.zeros_like(strad)
        follows[:, 1:] = strad[:, :-1]
        assert (start[follows] >= end[:, :-1][strad[:, :-1]] + 32).all(), "a burst starts within 32 samples of a straddler"
        assert (end[~strad & ~follows] <= np.broadcast_to(hi, strad.shape)[~strad & ~follows]).all()
        assert (start[strad] // CHUNK != (end[strad] - 1) // CHUNK).all(), "a straddler crosses no chunk boundary"
        assert straddle == 0 or not (strad & (np.arange(n_slots) % straddle != straddle - 1)).any()
        assert straddle == 0 or strad.sum() > 50
        looked_back += int((end[:, :-1][strad[:, :-1]] + 32 > hi[:-1][np.nonzero(strad[:, :-1])[1]]).sum())
    assert straddle == 0 or looked_back > 200                     # followers whose start the look-back moved


def test_synth_truth_cap_one_short(ctx):
    cfgs = synth.channel_plan(40)[[37, 5, 21]]
    n_int8 = 2 * 3200 * 10 + 99
    rc, host, truth, got = synth_call(ctx, cfgs, n_int8, n_int8, 0, 3, truth=True, truth_short=1, amplitude=50)
    assert rc == BTLE_EINVAL and got == 10
    assert (host == POISON).all() and not truth.view(np.uint8).any()
    rc, _, truth, got = synth_call(ctx, cfgs, n_int8, n_int8, 0, 3, truth=True, amplitude=50)
    assert rc == 0 and got == 10 and len(truth) == 30 and np.array_equal(truth["slot"], np.tile(np.arange(10), 3))
