"""GPU parity tests proper: the CUDA path, called through the C-ABI (ctypes), against the oracle
on the same seeded inputs, against the committed reference-generated golden vectors, and —
at large sizes — through size-independent properties.  Bar: bit-exact records."""
import numpy as np
import pytest
import torch

import golden_util as G
import orc
from btle_b200 import BtleRx, make_cfgs, synth

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def rx():
    import __graft_entry__ as ge
    ge.build()
    r = BtleRx(0)
    yield r
    r.close()


def _same(a, b):
    assert len(a) == len(b), (len(a), len(b))
    if a.tobytes() != b.tobytes():
        for i, (x, y) in enumerate(zip(a, b)):
            assert x.tobytes() == y.tobytes(), (i, x, y)


@pytest.mark.parametrize("name", G.cases())
def test_gpu_matches_reference_golden(rx, name):
    z, cfg = G.load(name)
    rec = rx.rx(z["iq"], **G.rx_cfg(cfg))
    G.assert_matches_golden(rec, z)


@pytest.mark.parametrize("seed", range(8))
def test_gpu_equals_oracle_on_adversarial_fuzz(rx, seed):
    """Sparse masks on full-scale noise; flags (RSSI, -v rejected hits) rotate through 1, 2, 3 with the seed."""
    flags = (1, 2, 3)[seed % 3]
    rng = np.random.default_rng(1000 + seed)
    iq = rng.integers(-128, 128, 40 * 16384 + int(rng.integers(0, 16384)), dtype=np.int8)
    masks = [0x0000000F, 0x000000FF, 0x80000001, 0x00000000, 0xF0000000, 0x00010100, 0x0000FFFF, 0xFFFF0000]
    aas = [0x8E89BED6, 0x00000000, 0xFFFFFFFF, 0x55555555, 0x80000000, 0x12345678, 0x0000BED6, 0x8E890000]
    for ch in (37, 5):
        for raw in (0, 1):
            cfg = dict(channel=ch, access_addr=aas[seed], access_mask=masks[seed], raw=raw, crc_init=0x123456)
            _same(rx.rx(iq, rssi=flags, **cfg), orc.rx_flags(iq, flags, **cfg))


def test_gpu_equals_oracle_on_synth_streams(rx):
    for ch, kw in ((37, {}), (39, {}), (12, dict(access_addr=0x60850A27, crc_init=0xA77B2E, data_channel_pdu=True))):
        iq, _ = synth.make_adv_stream(100 * 16384 + 999, seed=77 + ch, channel=ch, corrupt_every=9, slot_samples=2500, **kw)
        cfg = dict(channel=ch, access_addr=kw.get("access_addr", 0x8E89BED6), crc_init=kw.get("crc_init", 0x555555))
        a = rx.rx(iq.numpy(), rssi=1, **cfg)
        b = orc.rx_stream(iq.numpy(), **cfg)
        assert len(b) > 250
        _same(a, b)


def test_gpu_ragged_empty_and_tiny(rx):
    rng = np.random.default_rng(5)
    for n in (0, 1, 1000, 16383, 16384, 16385, 16384 + 3007, 3 * 16384 + 3007, 17 * 16384 + 5):
        iq = rng.integers(-1, 2, n, dtype=np.int8)
        cfg = dict(channel=38, access_addr=0x2AA, access_mask=0x3FF)
        _same(rx.rx(iq, rssi=1, **cfg), orc.rx_stream(iq, **cfg))


def test_gpu_batch_of_40_channels(rx):
    """SURVEY §8d C3 in miniature: one stream per BLE channel, per-channel AA / CRCInit."""
    n = 20 * 16384
    iqs, cfgs, exp = [], make_cfgs(40), []
    for ch in range(40):
        adv = ch >= 37
        aa = 0x8E89BED6 if adv else 0x60850A1B + ch
        ci = 0x555555 if adv else 0xA77B22 ^ ch
        iq, _ = synth.make_adv_stream(n, seed=1000 + ch, channel=ch, access_addr=aa, crc_init=ci,
                                      data_channel_pdu=not adv, corrupt_every=10, slot_samples=3000)
        iqs.append(iq.numpy())
        cfgs[ch]["channel"], cfgs[ch]["access_addr"], cfgs[ch]["crc_init"], cfgs[ch]["rssi"] = ch, aa, ci, ch % 4
        if ch in (38, 39):                                                  # sparse mask: rejected hits with -v
            cfgs[ch]["access_mask"] = 0x0F000000
        exp.append(orc.rx_flags(iqs[-1], ch % 4, channel=ch, access_addr=aa, access_mask=int(cfgs[ch]["access_mask"]), crc_init=ci,
                                stream=ch))
    got = rx.rx_batch(np.stack(iqs), cfgs)
    exp = np.concatenate(exp)
    assert len(exp) > 40 * 40
    _same(got, exp)


def test_gpu_randomised_configs_with_planted_bursts(rx):
    """Random (channel, AA, mask, CRCInit, raw) per stream; bursts planted at adversarial places:
    straddling chunk boundaries, starting in the last samples of a chunk, back to back, inside the
    look-ahead of the last chunk, on top of full-scale random IQ."""
    rng = np.random.default_rng(77)
    n_streams, nchunks = 48, 6
    n = nchunks * 16384 + 2500
    iq = np.zeros((n_streams, n), dtype=np.int8)
    cfgs, exp = make_cfgs(n_streams), []
    for s in range(n_streams):
        ch = int(rng.integers(0, 40))
        flags = int(rng.integers(0, 4))
        aa = int(rng.integers(0, 2**32))
        mask = [0xFFFFFFFF, 0xFFFFFFFF, 0xFFFFFF00, 0x0FFFFFFF, 0xFFFF0000, 0x0F000000][s % 6]
        ci = int(rng.integers(0, 2**24))
        raw = int(s % 6 == 5)
        bg = rng.integers(-128, 128, n, dtype=np.int8) if s % 4 == 1 else rng.integers(-3, 4, n, dtype=np.int8)
        adv = ch >= 37
        pos = [8192 * 2 - 700, 8192 * 3 - 150, 8192 * 3 + 8000, 8192 * 4 - 40, 8192 * 5 + 100, 8192 * 6 - 900, 300, 1700]
        for k, p in enumerate(pos):
            plen = int(rng.integers(6, 38)) if adv else int(rng.integers(0, 28))
            body = rng.integers(0, 256, plen, dtype=np.uint8).tobytes()
            pdu = synth.adv_pdu(int(rng.integers(0, 7)), 1, 0, body) if adv else synth.ll_data_pdu(int(rng.integers(0, 4)), 0, 1, 0, body)
            wav = synth.modulate(synth.air_bytes(pdu, ch, aa, ci, 20 if k == 3 else None))
            p2 = 2 * (p + int(rng.integers(0, 4)))
            m = min(wav.size, n - p2)
            bg[p2:p2 + m] = wav[:m] // 2
        iq[s] = bg
        c = cfgs[s]
        c["channel"], c["access_addr"], c["access_mask"], c["crc_init"], c["raw"], c["rssi"] = ch, aa, mask, ci, raw, flags
        exp.append(orc.rx_flags(bg, flags, channel=ch, access_addr=aa, access_mask=mask, crc_init=ci, raw=raw, stream=s))
    exp = np.concatenate(exp)
    got = rx.rx_batch(iq, cfgs)
    assert len(exp) > 200
    _same(got, exp)


def test_gpu_many_short_streams(rx):
    """Hundreds of 1-3 chunk captures: spans with fewer tiles than dense warps, a parameter
    refresh at every span, more CTAs than spans and the opposite."""
    rng = np.random.default_rng(21)
    for n_streams, nchunks in ((5, 1), (300, 2), (700, 3)):
        n = nchunks * 16384 + 4000
        iq = np.zeros((n_streams, n), dtype=np.int8)
        cfgs, exp = make_cfgs(n_streams), []
        base, _ = synth.make_adv_stream(n, seed=9, channel=37, slot_samples=2600)
        base = base.numpy()
        for s in range(n_streams):
            ch = 37 + s % 3
            iq[s] = np.roll(base, 2 * int(rng.integers(0, 4000)))
            if s % 7 == 3:
                iq[s] = rng.integers(-128, 128, n, dtype=np.int8)
                cfgs[s]["access_mask"] = 0x0000FFFF if s % 2 else 0x80000001
            cfgs[s]["channel"], cfgs[s]["rssi"] = ch, s % 4
            exp.append(orc.rx_flags(iq[s], s % 4, channel=ch, access_mask=int(cfgs[s]["access_mask"]), stream=s))
        got = rx.rx_batch(iq, cfgs)
        _same(got, np.concatenate(exp))


def test_gpu_sc16q11_ingest(rx):
    """bladeRF samples: (x >> 4) & 0xFF as in the reference's stream_callback (btle_rx.c:307-308)."""
    iq8, _ = synth.make_adv_stream(12 * 16384 + 77, seed=31, channel=38, slot_samples=2700)
    rng = np.random.default_rng(2)
    iq16 = (iq8.numpy().astype(np.int16) << 4) | rng.integers(0, 16, iq8.numel(), dtype=np.int16)    # 12-bit samples
    iq16[::97] = rng.integers(-32768, 32767, iq16[::97].size, dtype=np.int16)                        # out-of-range junk wraps
    conv = ((iq16 >> 4) & 0xFF).astype(np.uint8).view(np.int8)
    for flags in (1, 2, 3):
        _same(rx.rx_iq16(iq16, 4, channel=38, rssi=flags), orc.rx_flags(conv, flags, channel=38))
    noise = rng.integers(-32768, 32767, 10 * 16384, dtype=np.int16)
    conv = ((noise >> 4) & 0xFF).astype(np.uint8).view(np.int8)
    for flags in (2, 3):
        exp = orc.rx_flags(conv, flags, channel=39, access_mask=0x0F000000)
        assert (exp["flags"] & 4).any()
        _same(rx.rx_iq16(noise, 4, channel=39, access_mask=0x0F000000, rssi=flags), exp)


def test_gpu_overflow_reports_needed_count(rx):
    from btle_b200 import BtleError
    iq, _ = synth.make_adv_stream(16 * 16384, seed=3, channel=37, slot_samples=3000)
    full = rx.rx(iq.numpy())
    with pytest.raises(BtleError) as e:
        rx.rx_batch(iq.numpy(), make_cfgs(1), cap=3)
    assert e.value.code == -5 and len(full) > 3


def test_gpu_bad_channel_is_einval(rx):
    from btle_b200 import BtleError
    with pytest.raises(BtleError) as e:
        rx.rx(np.zeros(16384, dtype=np.int8), channel=40)
    assert e.value.code == -1


# ---- leaf functions, reference signatures ---------------------------------------------------
def test_leaf_dbits(rx):
    rng = np.random.default_rng(1)
    for lo, hi in ((-128, 128), (-2, 3)):
        iq = rng.integers(lo, hi, 2 * 10001, dtype=np.int8)
        assert (rx.dbits(iq) == orc.dbits(iq)).all()


def test_leaf_search_unique_bits(rx):
    rng = np.random.default_rng(2)
    L = orc.lib()
    import ctypes
    for trial in range(24):
        search_len = int(rng.integers(1, 2080))
        iq = rng.integers(-128, 128, 8 * search_len + 2, dtype=np.int8)
        aa = int(rng.integers(0, 2**32))
        mask = [0xFFFFFFFF, 0x3F, 0xFF00, 0x80000001, 0, 0x7][trial % 6]
        bits = np.array([(aa >> p) & 1 for p in range(32)], dtype=np.uint8)
        mbits = np.array([(mask >> p) & 1 for p in range(32)], dtype=np.uint8)
        got = rx.search_unique_bits(iq, search_len, bits, mbits)
        d = np.concatenate([orc.dbits(np.concatenate([iq, np.zeros(2, np.int8)])), np.zeros(8, np.uint8)])
        n0 = ctypes.c_int(0)
        hit = L.orc_search(d.ctypes.data, 0, search_len, aa, mask, ctypes.byref(n0))
        assert got == (2 * n0.value if hit else -1), (trial, got, hit, n0.value)
    # planted access address: found at the planted place with the full mask
    air = synth.air_bytes(synth.adv_pdu(0, 1, 0, bytes(6)), 37)
    wav = synth.modulate(air)
    iq = np.zeros(8 * 1000 + 2, dtype=np.int8)
    iq[2 * 501:2 * 501 + wav.size] = wav
    aa = 0x8E89BED6
    bits = np.array([(aa >> p) & 1 for p in range(32)], dtype=np.uint8)
    got = rx.search_unique_bits(iq, 1000, bits, np.ones(32, np.uint8))
    assert got >= 0 and abs(got // 2 - (501 + 39)) <= 3


def test_leaf_demod_scramble_crc(rx):
    rng = np.random.default_rng(4)
    L = orc.lib()
    t = G.tables()
    for nb in (1, 2, 42, 64):
        iq = rng.integers(-128, 128, 64 * nb, dtype=np.int8)
        d = orc.dbits(np.concatenate([iq, np.zeros(4, np.int8)]))
        exp = np.zeros(nb, dtype=np.uint8)
        L.orc_demod_bytes(d.ctypes.data, 0, nb, exp.ctypes.data)
        assert (rx.demod_byte(iq, nb) == exp).all()
    st = np.array(t["scramble_table"], dtype=np.uint8)
    for ch in (0, 1, 17, 37, 39):
        data = rng.integers(0, 256, 40, dtype=np.uint8)
        assert (rx.scramble_byte(data, ch, 2) == (data ^ st[ch, 2:42])).all()
        assert (rx.scramble_byte(data[:2], ch, 0) == (data[:2] ^ st[ch, :2])).all()
    for n in (0, 1, 2, 39, 300):
        data = rng.integers(0, 256, n, dtype=np.uint8)
        for init in (int(rng.integers(0, 2**24)), int(rng.integers(0, 2**32, dtype=np.uint64))):   # bits 24..31 count too
            assert rx.crc24_byte(data, init) == L.orc_crc24(data.ctypes.data, n, init)
    assert rx.crc24_byte(np.frombuffer(bytes.fromhex("0100"), np.uint8), rx.crc_init_reorder(0x123456)) == 0x50899B


# ---- large sizes: size-independent properties -------------------------------------------------
def test_gpu_large_stream_properties(rx):
    """256 MiB stream generated on the device: every injected burst must come back exactly once
    with CRC ok unless it was corrupted, and a sample of chunks must equal the oracle."""
    n_int8 = 256 * 1024 * 1024
    iq, truth = synth.make_adv_stream(n_int8, seed=0xB7E15163 & 0x7FFFFFFF, channel=37, device="cuda", corrupt_every=100)
    cfgs = make_cfgs(1)
    cap = n_int8 // 16384 * 4
    d_out = torch.empty(cap * 64, dtype=torch.uint8, device="cuda")
    d_count = torch.zeros(1, dtype=torch.int32, device="cuda")
    rx.rx_device(iq.view(1, -1), cfgs, d_out, d_count, torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    n = int(d_count.item())
    from btle_b200 import REC_DTYPE
    rec = rx.sort_records(d_out[: n * 64].cpu().numpy().view(REC_DTYPE))
    pos = rec["chunk"].astype(np.int64) * 8192 + rec["n0"]
    exp_pos = truth["start_sample"] + 39          # preamble (32 samples) + modulator delay
    # match each truth burst to a record within +-3 samples
    idx = np.searchsorted(pos, exp_pos - 3)
    idx = np.clip(idx, 0, len(pos) - 1)
    hit = np.abs(pos[idx] - exp_pos) <= 3
    # bursts whose look-ahead crosses the end of the capture may be cut; all others must be found
    inside = truth["start_sample"] + 8 * truth["n_air_bytes"] * 4 + 64 < (n_int8 // 16384) * 8192
    assert hit[inside].all(), f"{(~hit[inside]).sum()} injected bursts not found"
    bad = rec["crc_bad"][idx].astype(bool)
    assert (bad[inside] == truth["corrupt"][inside]).all()
    # decoded bytes equal the transmitted PDU
    for s in range(0, len(exp_pos), 997):
        if inside[s] and not truth["corrupt"][s]:
            pdu = truth["pdus"][s]
            assert bytes(rec["bytes"][idx[s]][:len(pdu)]) == pdu
    # oracle on a sample of the stream (chunk-aligned slices keep chunk semantics)
    host = iq.cpu().numpy()
    for c0 in (0, 4097, 16000):
        sl = host[c0 * 16384:(c0 + 24) * 16384 + 4096]
        exp = orc.rx_stream(sl, channel=37)
        sel = rec[(rec["chunk"] >= c0) & (rec["chunk"] < c0 + 24)].copy()
        sel["chunk"] -= c0
        exp = exp[exp["chunk"] < 24]
        exp_nomag = exp.copy(); exp_nomag["mag_sum"] = 0
        _same(sel, exp_nomag)


def test_gpu_worst_case_packets_per_chunk_grows_capacity(rx):
    """51 packets per chunk (BTLE_MAX_PKTS_PER_CHUNK) exceed the wrapper's default capacity of 34 per chunk:
    the EOVERFLOW -> retry path must deliver all of them, equal to the oracle."""
    z = np.zeros(3 * 16384 + 3008, dtype=np.int8)
    got = rx.rx(z, channel=1, access_addr=0, access_mask=0, rssi=1)
    exp = orc.rx_stream(z, channel=1, access_addr=0, access_mask=0)
    assert int(np.bincount(got["chunk"]).max()) == 51
    assert got.tobytes() == exp.tobytes()


def test_gpu_unit_directory_walk_is_reference_order(rx):
    """rx_device_dir: one block per unit + directory; walking the directory equals the oracle's order, the sum of the
    directory counts equals the device counter, and every directory entry of the launch is written."""
    from btle_b200 import REC_DTYPE, DIR_DTYPE
    ns, n = 4, 70 * 16384 + 500
    iq = np.zeros((ns, n), dtype=np.int8)
    cfgs = make_cfgs(ns)
    exp = []
    for s_ in range(ns):
        ch = [37, 9, 39, 38][s_]
        aa = 0x8E89BED6 if ch >= 37 else 0x60850A1B + ch
        ci = 0x555555 if ch >= 37 else 0xA77B22 ^ ch
        t, _ = synth.make_adv_stream(n, seed=300 + s_, channel=ch, access_addr=aa, crc_init=ci, corrupt_every=7, slot_samples=2100,
                                     data_channel_pdu=ch < 37, straddle_every=3)
        iq[s_] = t.numpy()
        mask, flags = 0xFFFFFFFF, [1, 2, 3, 3][s_]
        if s_ == 3:                                       # -v with a sparse mask on noise: rejected records in the blocks
            iq[s_] = np.random.default_rng(5).integers(-128, 128, n, dtype=np.int8)
            mask = 0x0F000000
        cfgs[s_]["channel"], cfgs[s_]["access_addr"], cfgs[s_]["crc_init"], cfgs[s_]["access_mask"], cfgs[s_]["rssi"] = ch, aa, ci, mask, flags
        exp.append(orc.rx_flags(iq[s_], flags, channel=ch, access_addr=aa, access_mask=mask, crc_init=ci, stream=s_))
    exp = np.concatenate(exp)
    assert int(((exp["flags"] & 4) != 0).sum()) > 100
    d_iq = torch.zeros((ns, (n + 15) // 16 * 16), dtype=torch.int8, device="cuda")
    d_iq[:, :n] = torch.from_numpy(iq).cuda()
    units = rx.units(ns, n)
    assert units > ns * 5
    cap = len(exp) + 8
    d_out = torch.zeros(cap * 64, dtype=torch.uint8, device="cuda")
    d_dir = torch.full((units + 4, 2), -1, dtype=torch.int32, device="cuda")
    d_count = torch.zeros(1, dtype=torch.int32, device="cuda")
    rx.rx_device_dir(d_iq[:, :n], cfgs, d_out, d_count, d_dir, torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    hd = d_dir.cpu().numpy().view(np.uint32)
    assert (hd[units:] == 0xFFFFFFFF).all() and (hd[:units, 1] < 0xFFFF).all()
    unit_dir = np.ascontiguousarray(hd[:units]).view(DIR_DTYPE).reshape(-1)
    assert int(unit_dir["count"].sum()) == int(d_count.item()) == len(exp)
    got = rx.gather_ordered(d_out.cpu().numpy().view(REC_DTYPE), unit_dir)
    _same(got, exp)
    # d_count = None: reservations on the context's counter ring (no memset node), 100 launches back to back wrap the ring
    for it in range(100):
        d_dir.fill_(-1)
        rx.rx_device_dir(d_iq[:, :n], cfgs, d_out, None, d_dir, torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    hd = d_dir.cpu().numpy().view(np.uint32)
    unit_dir = np.ascontiguousarray(hd[:units]).view(DIR_DTYPE).reshape(-1)
    assert int(unit_dir["count"].sum()) == len(exp) and int((unit_dir["base"].astype(np.int64) + unit_dir["count"]).max()) == len(exp)
    _same(rx.gather_ordered(d_out.cpu().numpy().view(REC_DTYPE), unit_dir), exp)


def test_gpu_fuzz_campaign_bounded():
    """tools/fuzz_gpu.py (random access addresses / masks / channels / CRC inits / raw mode, five input kinds incl. bursts
    across chunk boundaries, 1..33 captures per batch, ragged lengths) for a bounded time inside the suite, so that every
    driver run of `-m gpu` carries a fresh fuzz campaign against the oracle — not only the builder's own long runs."""
    import os
    import subprocess
    import sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    for tool, env in (("fuzz_gpu.py", {"FUZZ_SECONDS": "25"}), ("stress.py", {"STRESS_SECONDS": "12"})):
        p = subprocess.run([sys.executable, os.path.join(root, "tools", tool), "20260923"], capture_output=True, text=True, timeout=600,
                           env=dict(os.environ, **env))
        assert p.returncode == 0, p.stdout[-2000:] + p.stderr[-3000:]
        assert " ok" in p.stdout


def test_gpu_stream_session_equals_whole_capture(rx):
    """btle_b200_stream_*: pieces of arbitrary size in, records of the whole-capture call out (reference order, stream-wide
    chunk numbers), for segment sizes around and below the capture length; records that exceed a call's buffer are handed
    out by the following calls."""
    iq, _ = synth.make_adv_stream(70 * 16384 + 1234, seed=61, channel=39, slot_samples=2200, straddle_every=3, corrupt_every=4)
    iq = iq.numpy()
    exp = orc.rx_stream(iq, channel=39)
    rng = np.random.default_rng(3)
    for seg in (1, 5, 32, 69, 70, 71, 0):
        with rx.stream(segment_chunks=seg, channel=39, rssi=1) as s_:
            parts, pos = [], 0
            while pos < iq.size:
                step = int(rng.choice([1, 100, 16384, 50000, 300000]))
                parts.append(s_.push(iq[pos:pos + step]))
                pos += step
            parts.append(s_.finish())
        got = np.concatenate(parts)
        _same(got, exp)
    # -v with a sparse mask on noise (rejected records in every segment), RSSI on and off
    iq = np.random.default_rng(8).integers(-128, 128, 12 * 16384 + 777, dtype=np.int8)
    for seg, flags in ((1, 3), (5, 2), (5, 3)):
        exp = orc.rx_flags(iq, flags, channel=39, access_mask=0x0F000000)
        assert int(((exp["flags"] & 4) != 0).sum()) > 50
        with rx.stream(segment_chunks=seg, channel=39, access_mask=0x0F000000, rssi=flags) as s_:
            got = np.concatenate([s_.push(iq[:70000]), s_.push(iq[70000:]), s_.finish()])
        _same(got, exp)


def test_gpu_worst_case_rejected_hits_per_chunk(rx):
    """-v on the zero capture with mask 0 on channel 38: every window matches, every header has an impossible ADV length,
    so each chunk returns BTLE_MAX_RECS_PER_CHUNK = 123 rejected records, more than the resolver's hit rows hold.  Through
    rx (default capacity of 34 per chunk -> BTLE_EOVERFLOW -> retry), rx_device_dir and a stream session."""
    from btle_b200 import REC_DTYPE, DIR_DTYPE
    nch = 20
    z = np.zeros(nch * 16384 + 3008, dtype=np.int8)
    cfg = dict(channel=38, access_addr=0, access_mask=0)
    for flags in (2, 3):
        exp = orc.rx_flags(z, flags, **cfg)
        assert len(exp) == nch * 123 and (exp["flags"] & 4).all()
        _same(rx.rx(z, rssi=flags, **cfg), exp)
        cfgs = make_cfgs(1, rssi=flags, **cfg)
        d_iq = torch.zeros((1, (z.size + 15) // 16 * 16), dtype=torch.int8, device="cuda")
        units = rx.units(1, z.size)
        d_out = torch.zeros(len(exp) * 64, dtype=torch.uint8, device="cuda")
        d_dir = torch.zeros((units, 2), dtype=torch.int32, device="cuda")
        d_count = torch.zeros(1, dtype=torch.int32, device="cuda")
        rx.rx_device_dir(d_iq[:, :z.size], cfgs, d_out, d_count, d_dir, torch.cuda.current_stream().cuda_stream)
        torch.cuda.synchronize()
        unit_dir = np.ascontiguousarray(d_dir.cpu().numpy().view(np.uint32)).view(DIR_DTYPE).reshape(-1)
        assert int(unit_dir["count"].sum()) == int(d_count.item()) == len(exp)
        _same(rx.gather_ordered(d_out.cpu().numpy().view(REC_DTYPE), unit_dir), exp)
        for seg in (1, 5):
            with rx.stream(segment_chunks=seg, rssi=flags, **cfg) as s_:
                got = np.concatenate([s_.push(z), s_.finish()])
            _same(got, exp)
