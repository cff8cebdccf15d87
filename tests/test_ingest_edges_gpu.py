"""How IQ reaches the receive kernel and how records leave it, against the oracle (tests/orc.py) on the same bytes with
zeros around every capture.

- Host ingest of btle_b200_rx_batch / _rx_iq16 / _discover (h2d_rows): pageable memory through the two 32 MiB staging
  buffers, page-locked memory (torch pin_memory, an interior pointer of it, cudaHostRegister'ed numpy) by one 1-D or 2-D
  DMA; strides with padding behind every capture that holds bytes which must never be read.
- Device views for btle_b200_rx_device_dir inside a larger buffer, with poisoned bytes in front of them and between
  n_int8 and the stride, at every way the tile feed can end a capture: look-ahead tile entirely behind the capture
  (zeroed), partly in bounds (TMA zero fill), holding a partial 256-byte row (filled by hand), complete.
- A record capacity that cuts between units, inside a unit's block and inside a -v chunk's late records (hits 68..122):
  nothing is written at or behind `cap`, the counter and the unit directory still count every record, and
  btle_b200_gather_ordered returns BTLE_EOVERFLOW with the records that were stored, in reference order.

Every capture is decoded with RSSI on (flags 1 or 3), so a byte read from outside a capture shows in mag_sum even where it
does not change a decoded bit.  Random poison changes discriminator bits; 0x7F poison does not (I*Q' - I'*Q is 0 between
two 0x7F samples), but adds 127 to an RSSI sum for every byte read."""
import ctypes

import numpy as np
import pytest
import torch

import mode_ref
import orc
from btle_b200 import CAND_DTYPE, DIR_DTYPE, REC_DTYPE, make_cfgs, synth
from btle_b200._native import BTLE_EOVERFLOW

pytestmark = pytest.mark.gpu

SEG = 32 << 20                        # h2d_rows: pageable sources move through the staging buffers in segments of this size
CHUNK = 16384
SOURCES = ("pageable", "pinned", "pinned_interior", "registered")


@pytest.fixture(scope="module")
def rx():
    import __graft_entry__ as ge
    ge.build()
    from btle_b200 import BtleRx
    r = BtleRx(0)
    yield r
    r.close()


def _same(a, b):
    assert len(a) == len(b), (len(a), len(b))
    if a.tobytes() != b.tobytes():
        for i, (x, y) in enumerate(zip(a, b)):
            assert x.tobytes() == y.tobytes(), (i, x, y)


# ---- captures ------------------------------------------------------------------------------------------------------------
def _air(seed, channel=37):
    """Air bytes of an ADV_IND with the longest payload (37 bytes): its decode reads 42 bytes behind the access address."""
    payload = np.random.default_rng(seed).integers(0, 256, 37, dtype=np.uint8).tobytes()
    return synth.air_bytes(synth.adv_pdu(0, 1, 0, payload), channel)


def _plant(iq, aa_sample, air, amp=64):
    """Writes the burst `air` over iq so that its access address starts at sample `aa_sample` at the receiver (39 samples
    behind the burst's first); what falls before sample 0 or behind the end of iq is cut off."""
    wav = synth.modulate(air).astype(np.int32) * amp // 127
    a = 2 * (aa_sample - 39)
    lo, hi = max(a, 0), min(a + wav.size, iq.size)
    if lo < hi:
        iq[lo:hi] = wav[lo - a:hi - a].astype(np.int8)


def _capture(n_int8, seed, kind, device=None, phase=None):
    """'burst': synthesised ADV stream (bursts across chunk boundaries, corrupted CRCs) with one burst whose access address
    starts 20 samples before the capture (a chunk-0 hit at n0 < 0 under mask 0xFFFFFF00) and one whose payload runs into
    the capture's last samples (cut there) when the last chunk's search reaches that far.  With phase 1 and an odd
    n_int8 that burst samples d[n_int8 // 2 - 1], the last discriminator bit of the capture, which reads byte n_int8 as
    its Q[n + 1]; I = 100, Q = 0 in front of that byte make d exactly 0 with a zero there and non-zero with anything else.
    'noise': full-scale uniform noise."""
    if kind == "noise":
        return np.random.default_rng(seed).integers(-128, 128, n_int8, dtype=np.int8)
    iq, _ = synth.make_adv_stream(n_int8, seed=seed, slot_samples=3000, corrupt_every=5, straddle_every=3, device=device)
    iq = iq.cpu().numpy().copy()
    _plant(iq, -20, _air(seed))
    end, last = n_int8 // 2, (n_int8 // CHUNK) * (CHUNK // 2)       # samples: capture end, end of the last complete chunk
    _plant(iq, min(end - 700, last + 100) - (seed % 4 if phase is None else phase), _air(seed + 1))
    if n_int8 % 2:
        iq[-3:-1] = (100, 0)
    return iq


# stream s of a batch: (kind, cfg).  Mask 0xFFFFFF00 finds the burst cut at the front; mask 0 with -v on noise has a
# rejected hit at n0 = -124 in chunk 0 (its RSSI window starts 248 bytes before the capture) and ~123 records per chunk.
STREAM_KINDS = (
    ("burst", dict(channel=37, access_mask=0xFFFFFF00, rssi=3)),
    ("noise", dict(channel=38, access_addr=0, access_mask=0, rssi=3)),
    ("burst", dict(channel=37, rssi=1)),
    ("noise", dict(channel=37, access_mask=0x0000000F, rssi=3)),
)


def _batch(n_int8, n_streams, seed, device=None):
    """(captures, cfgs, expected records) for a batch of n_streams captures of STREAM_KINDS."""
    iqs, cfgs = [], make_cfgs(n_streams)
    for s in range(n_streams):
        kind, cfg = STREAM_KINDS[s % len(STREAM_KINDS)]
        iqs.append(_capture(n_int8, seed + 101 * s, kind, device, phase=1 + s % 4))
        for k, v in cfg.items():
            cfgs[s][k] = v
    return iqs, cfgs, _expected(iqs, cfgs)


def _expected(iqs, cfgs):
    return np.concatenate([orc.rx_flags(iq, int(c["rssi"]), channel=int(c["channel"]), access_addr=int(c["access_addr"]),
                                        access_mask=int(c["access_mask"]), crc_init=int(c["crc_init"]), raw=int(c["raw"]), stream=s)
                           for s, (iq, c) in enumerate(zip(iqs, cfgs))])


def _poison(n, rng, random):
    return rng.integers(-128, 128, n, dtype=np.int8) if random else np.full(n, 0x7F, dtype=np.int8)


# ---- host memory -----------------------------------------------------------------------------------------------------------
class HostBuf:
    """n bytes of host memory of one kind: `a` is the int8 numpy view, `ptr` the address handed to the library."""

    def __init__(self, kind, n):
        self.kind, self._reg = kind, None
        if kind == "pageable":
            self.a = np.empty(n, dtype=np.int8)
        elif kind in ("pinned", "pinned_interior"):
            off = 4096 + 1000 if kind == "pinned_interior" else 0          # not even 16-byte aligned inside the allocation
            self._t = torch.empty(n + off + 4096, dtype=torch.int8, pin_memory=True)
            self.a = self._t.numpy()[off:off + n]
        else:                                                             # numpy memory, page-locked in place
            self._raw = np.empty(n + 2 * 4096, dtype=np.int8)
            o = (-self._raw.ctypes.data) % 4096
            self.a = self._raw[o:o + n]
            self._reg = (self.a.ctypes.data, (n + 4095) // 4096 * 4096)
            cr = torch.cuda.cudart()
            assert cr.cudaHostRegister(self._reg[0], self._reg[1], 0) == cr.cudaError.success
        self.ptr = self.a.ctypes.data
        # the library picks the copy path from the pointer's attributes: check that it sees the kind intended here
        assert torch.from_numpy(self.a).is_pinned() == (kind != "pageable")

    def close(self):
        if self._reg:
            cr = torch.cuda.cudart()
            assert cr.cudaHostUnregister(self._reg[0]) == cr.cudaError.success
            self._reg = None


def _lay_out(buf, iqs, stride, rng, random_poison):
    """Captures stride bytes apart in buf.a, poison in front of nothing, between and behind every capture."""
    buf.a[:] = _poison(buf.a.size, rng, random_poison)
    for s, iq in enumerate(iqs):
        buf.a[s * stride:s * stride + iq.size] = iq


def _rx_batch(rx, ptr, n_streams, stride, n_int8, cfgs):
    cap = n_streams * (n_int8 // CHUNK) * orc.MAX_RECS_PER_CHUNK + 16
    out = np.zeros(cap, dtype=REC_DTYPE)
    got = ctypes.c_size_t(0)
    rx._check(rx._L.btle_b200_rx_batch(rx._h, ptr, n_streams, stride, n_int8, cfgs.ctypes.data, out.ctypes.data, cap, ctypes.byref(got)))
    return out[:got.value]


# ---- 1. btle_b200_rx_batch: every copy path --------------------------------------------------------------------------------
N16 = 6 * CHUNK                      # n_int8 % 16 == 0
NODD = 6 * CHUNK + 1005              # n_int8 % 16 == 13: the device pitch differs from the row length -> 2-D copy when page-locked
_SETS = {}


def _small_sets():
    if not _SETS:
        for n in (N16, NODD):
            _SETS[n] = _batch(n, 3, seed=n % 977)
    return _SETS


@pytest.mark.parametrize("source", SOURCES)
def test_rx_batch_host_ingest_matrix(rx, source):
    """Copy path by shape (page-locked sources): one capture -> 1-D copy; several with stride == n_int8 and n_int8 % 16 == 0 -> 1-D;
    several otherwise -> cudaMemcpy2DAsync.  Pageable sources are staged.  Padding between and behind the captures is 0x7F
    or random and must not change a record."""
    sets = _small_sets()
    rng = np.random.default_rng(7)
    for n, (iqs, cfgs, exp) in sets.items():
        assert ((exp["chunk"] == 0) & (exp["n0"] < 0)).sum() >= 2 and (exp["flags"] & 4).any()
        for ns in (1, 3):
            want = exp[exp["stream"] < ns]
            for extra in (0, 7, 4096):
                stride = n + extra
                buf = HostBuf(source, ns * stride)
                try:
                    _lay_out(buf, iqs[:ns], stride, rng, random_poison=extra != 7)
                    _same(_rx_batch(rx, buf.ptr, ns, stride, n, cfgs[:ns]), want)
                finally:
                    buf.close()


def _large_batch(n, seed):
    iqs, cfgs = [], make_cfgs(3)
    for s in range(3):
        kind, cfg = STREAM_KINDS[(0, 2, 1)[s]]
        iq = _capture(n, seed + s, kind, device="cuda")
        if kind == "burst" and n > SEG + CHUNK:
            _plant(iq, SEG // 2 - 300 - s, _air(50 + s))               # across the boundary: access address 300 samples before it
            _plant(iq, SEG // 2 + 1300 + s, _air(70 + s))              # and the next burst right behind that one
        iqs.append(iq)
        for k, v in cfg.items():
            cfgs[s][k] = v
    return iqs, cfgs, _expected(iqs, cfgs)


def test_rx_batch_rows_larger_than_a_staging_segment(rx):
    """Three captures of 33 MiB + 5 bytes: pageable (each row is two staging segments, 32 MiB and 1 MiB + 5, so the two
    staging buffers alternate across rows and a segment boundary falls in every row) and page-locked (2-D copy); bursts
    cross the 32 MiB boundary of every row.  Then three pageable captures of 32 MiB + 5: the 5-byte second segment is
    staged at once, so the next row's first segment is written into a staging buffer whose 32 MiB DMA has just started.
    A smaller batch decoded before and after each must not see the bytes the large one leaves in the context's device
    buffer behind its own rows."""
    small_iqs, small_cfgs, small_exp = _small_sets()[NODD]
    rng = np.random.default_rng(11)
    small = HostBuf("pageable", 3 * NODD)
    _lay_out(small, small_iqs, NODD, rng, random_poison=True)
    _same(_rx_batch(rx, small.ptr, 3, NODD, NODD, small_cfgs), small_exp)
    n = SEG + (1 << 20) + 5
    iqs, cfgs, exp = _large_batch(n, 900)
    at_seg = exp[(exp["chunk"] >= SEG // CHUNK - 1) & (exp["chunk"] <= SEG // CHUNK)]
    assert ((at_seg["stream"] != 2) & (at_seg["crc_bad"] == 0) & ((at_seg["flags"] & 4) == 0)).sum() >= 4
    cases = [(iqs, cfgs, exp, "pageable", n + 4096), (iqs, cfgs, exp, "pinned", n + 7)]
    n = SEG + 5
    iqs, cfgs, exp = _large_batch(n, 950)
    cases.append((iqs, cfgs, exp, "pageable", n))
    for iqs, cfgs, exp, source, stride in cases:
        buf = HostBuf(source, 3 * stride)
        _lay_out(buf, iqs, stride, rng, random_poison=True)
        _same(_rx_batch(rx, buf.ptr, 3, stride, iqs[0].size, cfgs), exp)
        del buf
        _same(_rx_batch(rx, small.ptr, 3, NODD, NODD, small_cfgs), small_exp)


# ---- 2. btle_b200_rx_iq16 larger than one staging segment --------------------------------------------------------------------
def test_rx_iq16_larger_than_a_staging_segment(rx):
    """17 Mi + 3 int16 (34 MiB: two staging segments when pageable, one 1-D copy when page-locked).  Every int16 carries
    random bits below and above the 8 that (x >> 4) & 0xFF keeps."""
    n = 17 * (1 << 20) + 3
    iq8 = _capture(n, 31, "burst", device="cuda")
    _plant(iq8, SEG // 4 - 500, _air(33))                              # across byte 32 Mi of the int16 buffer
    rng = np.random.default_rng(32)
    x = (iq8.view(np.uint8).astype(np.uint16) << 4) | rng.integers(0, 16, n, dtype=np.uint16) | (rng.integers(0, 16, n, dtype=np.uint16) << 12)
    x = x.view(np.int16)
    assert np.array_equal(((x >> 4) & 0xFF).astype(np.uint8).view(np.int8), iq8)
    cfg = make_cfgs(1, access_mask=0xFFFFFF00, rssi=3)
    exp = orc.rx_flags(iq8, 3, access_mask=0xFFFFFF00)
    assert len(exp) > 1000 and ((exp["chunk"] == SEG // 2 // CHUNK - 1) & (exp["crc_bad"] == 0)).any()
    pinned = torch.empty(n, dtype=torch.int16, pin_memory=True)
    pinned.numpy()[:] = x
    for src in (x, pinned.numpy()):
        cap = len(exp) + 64
        out = np.zeros(cap, dtype=REC_DTYPE)
        got = ctypes.c_size_t(0)
        rx._check(rx._L.btle_b200_rx_iq16(rx._h, src.ctypes.data, n, 4, cfg.ctypes.data, out.ctypes.data, cap, ctypes.byref(got)))
        _same(out[:got.value], exp)


# ---- 3. btle_b200_discover through the same copy paths ---------------------------------------------------------------------
def _empty_pdus(n_int8, channel, seed, at):
    """Noise floor with empty PDUs (one of test_discover's access addresses / CRC inits) whose preambles start at the
    samples `at` (cut by the capture's ends where they fall outside)."""
    gen = torch.Generator(); gen.manual_seed(seed)
    iq = synth.noise_floor(n_int8, gen).numpy().copy()
    for k, a in enumerate(at):
        aa = (0x60850A1B, 0x50850A1C, 0x12345679)[k % 3]
        _plant(iq, a + 39, synth.air_bytes(synth.ll_data_pdu(1, k & 1, 0, 0, b""), channel, aa, 0x227BA7 ^ k), amp=64)
    return iq


def _discover_device(rx, iqs, channels):
    """btle_b200_discover_device on a zero-padded device copy, sorted by (stream, sample)."""
    n = iqs[0].size
    d_iq = torch.zeros((len(iqs), (n + 15) // 16 * 16), dtype=torch.int8, device="cuda")
    d_iq[:, :n] = torch.from_numpy(np.stack(iqs)).cuda()
    cap = len(iqs) * (n // CHUNK + 1) * 8 + 256
    d_out = torch.zeros(cap * 32, dtype=torch.uint8, device="cuda")
    d_count = torch.zeros(1, dtype=torch.int32, device="cuda")
    rx.discover_device(d_iq[:, :n], channels, d_out, d_count, torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    k = int(d_count.item())
    assert k <= cap
    c = d_out[:k * 32].cpu().numpy().view(CAND_DTYPE)
    return c[np.lexsort((c["sample"], c["stream"]))]


def test_discover_host_copy_paths(rx):
    """Page-locked with a 2-D copy (three captures, n_int8 % 16 != 0, stride n_int8 + 7) and pageable with two captures
    of more than one staging segment each; empty PDUs at both ends of every capture and across the 32 MiB boundary;
    poisoned padding.  The host entry point == discover_device on a zero-padded device copy."""
    rng = np.random.default_rng(21)
    for source, n, stride, ns in (("pinned", 40 * CHUNK + 1003, 40 * CHUNK + 1010, 3), ("pageable", SEG + 5 * CHUNK + 3, SEG + 5 * CHUNK + 4099, 2)):
        half = n // 2
        at = [-40, 400, 2000, 5000, half // 2, half - 1200, half - 600, half - 250]      # bursts are 336 samples long
        if n > SEG:
            at += [SEG // 2 - 150 - 501 * k for k in range(4)]
        channels = np.array([3, 17, 36][:ns], dtype=np.int32)
        iqs = [_empty_pdus(n, int(channels[s]), 40 + s, [a + 3 * s for a in at]) for s in range(ns)]
        exp = _discover_device(rx, iqs, channels)
        assert len(exp) >= 8 * ns
        buf = HostBuf(source, ns * stride)
        _lay_out(buf, iqs, stride, rng, random_poison=True)
        out = np.zeros(len(exp) + 256, dtype=CAND_DTYPE)
        got = ctypes.c_size_t(0)
        rx._check(rx._L.btle_b200_discover(rx._h, buf.ptr, ns, stride, n, channels.ctypes.data, out.ctypes.data, out.size, ctypes.byref(got)))
        assert out[:got.value].tobytes() == exp.tobytes()


# ---- 4. poisoned device views for rx_device_dir ---------------------------------------------------------------------------
K = 5
LENGTHS = [K * CHUNK,                                # look-ahead tile entirely behind the capture: zeroed
           K * CHUNK + 256 * 5,                      # 12-row look-ahead tile partly in bounds: TMA zero fill
           *(K * CHUNK + r for r in (1, 4, 5, 128, 255)),   # partial row at the look-ahead's start: filled by hand
           K * CHUNK + 256 * 3 + 5,                  # partial row inside the look-ahead tile
           K * CHUNK + 3072 + 1,                     # look-ahead complete, capture ends one byte behind it
           K * CHUNK + 9001]                         # look-ahead complete


def _device_view(iqs, stride, front, rng, random_poison):
    """The captures at `front` + s * stride inside a poisoned CUDA buffer (4096 more poisoned bytes in front of `front`, so
    that no read a few hundred bytes too early leaves the allocation).  Returns (buffer, [n_streams, n_int8] view)."""
    ns, n = len(iqs), iqs[0].size
    lead = 4096 + front
    host = _poison(lead + ns * stride + 4096, rng, random_poison)
    for s, iq in enumerate(iqs):
        host[lead + s * stride:lead + s * stride + n] = iq
    d = torch.from_numpy(host).cuda()
    return d, d[lead:lead + ns * stride].view(ns, stride)[:, :n]


def _walk(rx, d_out, d_dir, units):
    unit_dir = np.ascontiguousarray(d_dir[:units].cpu().numpy().view(np.uint32)).view(DIR_DTYPE).reshape(-1)
    return rx.gather_ordered(d_out.cpu().numpy().view(REC_DTYPE), unit_dir), unit_dir


@pytest.mark.parametrize("n_int8", LENGTHS)
def test_rx_device_dir_poisoned_views(rx, n_int8):
    """Every byte outside [0, n_int8) of a view is poison; records == the oracle on the capture with zeros around it."""
    _poisoned_views(rx, n_int8, (0, 0))


@pytest.mark.parametrize("mode", mode_ref.NEW_MODES, ids=mode_ref.mode_id)
@pytest.mark.parametrize("n_int8", LENGTHS)
def test_rx_device_dir_poisoned_views_in_modes(rx, n_int8, mode):
    """The same with the rotated and symbol-spaced one-cfg kernels, each capture at its own offset, against
    tests/mode_ref.py: the symbol-spaced loop's word in front of a capture's first tile lies in the poison."""
    _poisoned_views(rx, n_int8, mode)


def _poisoned_views(rx, n_int8, mode):
    rng = np.random.default_rng(n_int8)
    iqs, cfgs, exp = _batch(n_int8, 4, seed=n_int8 % 1013)
    offsets = mode_ref.draw_offsets(np.random.default_rng(n_int8 + 5), 4, mode)
    if mode != (0, 0):
        iqs = list(mode_ref.rotate_all(np.stack(iqs), offsets))
        cfgs = mode_ref.with_mode(cfgs, mode)
        exp = mode_ref.rx_multi(np.stack(iqs), cfgs, np.arange(4), offsets)
    assert ((exp["chunk"] == 0) & (exp["n0"] == -124)).any() and ((exp["chunk"] == 0) & (exp["n0"] < 0) & ((exp["flags"] & 4) == 0)).any()
    st = torch.cuda.current_stream().cuda_stream
    for ns in (1, 4):
        want = exp[exp["stream"] < ns]
        units = rx.units(ns, n_int8)
        for front, extra in ((16, 0), (256, 48), (4096, 4096)):
            stride = (n_int8 + 15) // 16 * 16 + extra
            buf, view = _device_view(iqs[:ns], stride, front, rng, random_poison=front != 256)
            d_out = torch.zeros(max(len(want), 1) * 64, dtype=torch.uint8, device="cuda")
            d_dir = torch.zeros((units, 2), dtype=torch.int32, device="cuda")
            d_count = torch.zeros(1, dtype=torch.int32, device="cuda")
            rx.rx_device_dir(view, cfgs[:ns], d_out, d_count, d_dir, st, offset_hz=None if offsets is None else offsets[:ns])
            torch.cuda.synchronize()
            assert int(d_count.item()) == len(want)
            got, _ = _walk(rx, d_out, d_dir, units)
            _same(got, want)
            del buf


# ---- 5. capacity cut inside units ----------------------------------------------------------------------------------------
CANARY = 0xA5


def _plan(rx, n_streams, n_int8):
    """(stream, chunk0, n_chunks) of every unit of a launch: make_plan / unit_info through the emulator, at the device's
    grid (one persistent CTA per SM)."""
    import emul
    units = emul.plan(n_streams, n_int8 // CHUNK, torch.cuda.get_device_properties(0).multi_processor_count)
    assert len(units) == rx.units(n_streams, n_int8)
    return units


def _check_cut(rx, d_iq, cfgs, exp, plan, cap, with_count):
    """One launch with `cap` below the record count; d_out has room for every record, canary behind cap."""
    ns, n = d_iq.shape
    total, units = len(exp), len(plan)
    d_out = torch.full((total + 64, 64), CANARY, dtype=torch.uint8, device="cuda")
    d_dir = torch.full((units, 2), -1, dtype=torch.int32, device="cuda")
    d_count = torch.full((1,), -1, dtype=torch.int32, device="cuda") if with_count else None
    rx._check(rx._L.btle_b200_rx_device_dir(rx._h, d_iq.data_ptr(), ns, d_iq.stride(0), n, cfgs.ctypes.data, d_out.data_ptr(), cap,
                                            d_count.data_ptr() if with_count else None, d_dir.data_ptr(), units,
                                            ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)))
    torch.cuda.synchronize()
    host = d_out.cpu().numpy()
    assert (host[cap:] == CANARY).all(), f"cap {cap}: records stored at or behind cap"
    recs = host.reshape(-1).view(REC_DTYPE)
    ud = np.ascontiguousarray(d_dir.cpu().numpy().view(np.uint32)).view(DIR_DTYPE).reshape(-1)
    if with_count:
        assert int(d_count.item()) == total
    assert int(ud["count"].sum()) == total
    # per unit: the oracle's records of its chunks, in reference order
    per_unit = [exp[(exp["stream"] == s) & (exp["chunk"] >= c0) & (exp["chunk"] < c0 + k)] for s, c0, k in plan]
    assert [len(p) for p in per_unit] == ud["count"].tolist()
    live = np.flatnonzero(ud["count"])
    order = live[np.argsort(ud["base"][live])]                         # blocks tile [0, total) in the order units reserved them
    assert ud["base"][order].tolist() == np.concatenate([[0], np.cumsum(ud["count"][order])[:-1]]).tolist()
    avail = []                                                         # each unit's records that fit below cap
    for u in range(units):
        b = int(ud["base"][u])
        m = max(0, min(len(per_unit[u]), cap - b))
        assert recs[b:b + m].tobytes() == per_unit[u][:m].tobytes(), (cap, u)
        avail.append(per_unit[u][:m])
    out = np.zeros(total, dtype=REC_DTYPE)
    got = ctypes.c_size_t(0)
    rc = rx._L.btle_b200_gather_ordered(recs.ctypes.data, cap, ud.ctypes.data, units, out.ctypes.data, total, ctypes.byref(got))
    assert got.value == total and rc == (BTLE_EOVERFLOW if cap < total else 0)
    avail = np.concatenate(avail)
    _same(out[:len(avail)], avail)


def test_capacity_cut_inside_units(rx):
    """-v on the zero capture with mask 0 on channel 38: 123 rejected records in every chunk, 68..122 stored by the late
    path; the 20 chunks are single-chunk units, so multiples of 123 are block boundaries whatever the order the units
    reserve their blocks in.  Then three synthesised streams and a -v noise stream with caps inside the blocks."""
    n = 20 * CHUNK + 3008
    z = np.zeros((1, n), dtype=np.int8)
    cfgs = make_cfgs(1, channel=38, access_addr=0, access_mask=0, rssi=3)
    exp = orc.rx_flags(z[0], 3, channel=38, access_addr=0, access_mask=0)
    assert len(exp) == 20 * 123
    plan = _plan(rx, 1, n)
    assert (plan[:, 2] <= 1).all()
    d_iq = torch.zeros((1, (n + 15) // 16 * 16), dtype=torch.int8, device="cuda")[:, :n]
    for with_count in (True, False):
        for cap in (0, 1, 5 * 123, 5 * 123 + 40, 5 * 123 + 67, 5 * 123 + 68, 5 * 123 + 100, 20 * 123 - 1, 20 * 123):
            _check_cut(rx, d_iq, cfgs, exp, plan, cap, with_count)

    n = 40 * CHUNK + 777
    iqs, cfgs, exp = _batch(n, 4, seed=5)
    plan = _plan(rx, 4, n)
    assert len(plan) > 8 and len(exp) > 1000
    d_iq = torch.zeros((4, (n + 15) // 16 * 16), dtype=torch.int8, device="cuda")
    d_iq[:, :n] = torch.from_numpy(np.stack(iqs)).cuda()
    for with_count in (True, False):
        for cap in (3, len(exp) // 3 + 1, len(exp) - 5, len(exp)):
            _check_cut(rx, d_iq[:, :n], cfgs, exp, plan, cap, with_count)
