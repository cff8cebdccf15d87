"""Carrier-offset correction on the GPU (the *_offset entry points and btle_b200_rec_offset; definitions in
include/btle_b200.h): at offset 0 the rotated kernel returns the default kernel's records byte for byte; at other offsets
it returns what the numpy restatement over the oracle chain returns (tests/offset_ref.py); corrected error rates approach
the uncorrected ones at offset 0; the per-packet estimate finds the offset of noiseless and noisy captures."""
import numpy as np
import pytest
import torch

import golden_util
import offset_ref
import rx_ber_ref as R
from btle_b200 import BtleRx, ber, make_cfgs
from btle_b200._native import BTLE_EINVAL, DIR_DTYPE, REC_DTYPE, BtleError

pytestmark = pytest.mark.gpu

DATA = dict(channel=9, access_addr=0x60850A27, crc_init=0xA77B2E)
ADV = dict(channel=37, access_addr=0x8E89BED6, crc_init=0x555555)


@pytest.fixture(scope="module")
def rx():
    import __graft_entry__ as ge
    ge.build()
    r = BtleRx(0)
    yield r
    r.close()


def _capture(cfo_hz, snr, channel, n=24, seed=1, ppm=0.0, amplitude=64):
    base = ADV if channel >= 37 else DATA
    cfg = ber.rx_ber_cfg(snr, ppm, cfo_hz, amplitude=amplitude, slot_samples=2048, channel=channel, seed=seed, crc_init=base["crc_init"],
                         access_addr=base["access_addr"])[0]
    iq, truth, _ = R.capture(cfg, 0, n)
    return iq, dict(base, channel=channel)


def _same(a, b):
    assert a.size == b.size and a.tobytes() == b.tobytes()


def test_zero_offset_equals_default_goldens(rx):
    n = 0
    for name in golden_util.cases():
        z, cfg = golden_util.load(name)
        kw = golden_util.rx_cfg(cfg)
        for extra in (0, 1, 4):
            k = dict(kw, rssi=kw.get("rssi", 0) | extra)
            want = rx.rx(z["iq"], **k)
            _same(rx.rx(z["iq"], offset_hz=0.0, **k), want)
            n += want.size
    assert n > 0


def test_zero_offset_equals_default_batch_and_multi(rx):
    caps = []
    for k in range(40):
        iq, cfg = _capture(0.0, 17 + k % 5, 37 if k % 2 == 0 else 9, n=16, seed=200 + k)
        caps.append((iq, cfg))
    n = min(c[0].size for c in caps) - 1234
    iq = np.stack([c[0][:n] for c in caps])
    cfgs = np.concatenate([make_cfgs(1, rssi=(k % 8), **c[1]) for k, c in enumerate(caps)])
    want = rx.rx_batch(iq, cfgs)
    assert want.size > 100
    _same(rx.rx_batch(iq, cfgs, offset_hz=np.zeros(40)), want)
    # several cfgs per capture, -v / raw / recover among them
    cap = np.repeat(np.arange(4), 3)
    mc = np.concatenate([make_cfgs(1, **caps[c][1]) for c in cap])
    mc["raw"][1::3] = 1
    mc["rssi"][2::3] = 2 | 4
    _same(rx.rx_multi(iq[:4], mc, cap, offset_hz=0.0), rx.rx_multi(iq[:4], mc, cap))


def _expected(iq, cfg, hz, rssi=0, raw=0, stream=0):
    rec = offset_ref.rx_stream(iq, hz, rssi=rssi, raw=raw, **cfg)
    rec["stream"] = stream
    return rec


@pytest.mark.parametrize("hz", [25e3, -25e3, 100e3, -100e3, 150e3, -150e3, 300e3, -300e3])
def test_offsets_equal_the_cpu_reference(rx, hz):
    for channel in (37, 9):
        iq, cfg = _capture(hz, 22.0, channel, n=20, seed=int(abs(hz)) % 97 + channel)
        iq = iq[:iq.size - 2 * 777]                                    # ragged
        for rssi, raw in ((0, 0), (1 | 2, 0), (4, 0), (2 | 4, 0), (0, 1)):
            got = rx.rx(iq, offset_hz=hz, rssi=rssi, raw=raw, **cfg)
            want = _expected(iq, cfg, hz, rssi, raw)
            _same(got, want)
        plain = rx.rx(iq, **cfg)
        fixed = rx.rx(iq, offset_hz=hz, **cfg)
        if abs(hz) >= 150e3:
            assert (fixed["crc_bad"] == 0).sum() > (plain["crc_bad"] == 0).sum()


def test_mixed_batch_and_device_forms(rx):
    offs = [0.0, 100e3, -100e3]
    caps = [_capture(h, 24.0, 37 if k != 1 else 9, n=20, seed=50 + k) for k, h in enumerate(offs)]
    n = min(c[0].size for c in caps)
    iq = np.stack([c[0][:n] for c in caps])
    cfgs = np.concatenate([make_cfgs(1, rssi=4, **c[1]) for c in caps])
    got = rx.rx_batch(iq, cfgs, offset_hz=offs)
    parts = []
    for k in range(3):
        r = rx.rx_batch(iq[k:k + 1], cfgs[k:k + 1], offset_hz=offs[k])
        r["stream"] = k
        parts.append(r)
        _same(r[r["stream"] == k], _expected(iq[k], caps[k][1], offs[k], rssi=4, stream=k))
    _same(got, np.concatenate(parts))
    # device-resident forms
    d_iq = torch.from_numpy(iq).cuda()
    units = rx.units(3, n)
    d_out = torch.empty(got.size * 64 + 64 * 64, dtype=torch.uint8, device="cuda")
    d_dir = torch.empty(units * 8, dtype=torch.uint8, device="cuda")
    rx.rx_device_dir(d_iq, cfgs, d_out, None, d_dir, torch.cuda.current_stream().cuda_stream, offset_hz=offs)
    torch.cuda.synchronize()
    recs = d_out.cpu().numpy().view(REC_DTYPE)
    _same(rx.gather_ordered(recs, d_dir.cpu().numpy().view(DIR_DTYPE)), got)
    cap = np.array([0, 0, 1, 2, 2], dtype=np.int32)
    mc = cfgs[cap].copy()
    mc["raw"][1] = 1
    want = rx.rx_multi(iq, mc, cap, offset_hz=offs)
    for j, c in enumerate(cap):                                        # each cfg as its capture decoded alone
        r = rx.rx_batch(iq[c:c + 1], mc[j:j + 1], offset_hz=offs[c])
        r["stream"] = j
        _same(want[want["stream"] == j], r)
    mu = rx.multi_units(3, cap, n)
    d_dir = torch.empty(mu * 8, dtype=torch.uint8, device="cuda")
    rx.rx_multi_device_dir(d_iq, mc, cap, d_out, None, d_dir, torch.cuda.current_stream().cuda_stream, offset_hz=offs)
    torch.cuda.synchronize()
    _same(rx.gather_ordered(d_out.cpu().numpy().view(REC_DTYPE), d_dir.cpu().numpy().view(DIR_DTYPE)), want)


def test_bad_offsets_are_einval(rx):
    iq, cfg = _capture(0.0, 30.0, 37, n=8)
    for bad in (float("nan"), float("inf"), 500001.0, -6e5):
        with pytest.raises(BtleError) as e:
            rx.rx(iq, offset_hz=bad, **cfg)
        assert e.value.code == BTLE_EINVAL
    assert rx.rx(iq, offset_hz=500000.0, **cfg).size >= 0                  # the context stays usable, the limit is accepted


def _bound(p0, n):
    return 3 * np.sqrt(max(p0 * (1 - p0), 1.0 / n) / n)


def test_per_with_correction(rx):
    n = 20000
    base = ber.rx_ber_point(rx, 24.0, n)
    fixed = ber.rx_ber_point(rx, 24.0, n, cfo_hz=100e3, offset_hz=100e3)
    plain = ber.rx_ber_point(rx, 24.0, n, cfo_hz=100e3)
    ppm_hz = 50e-6 * 2450e6 * (1 + 50e-6)
    ppm_fixed = ber.rx_ber_point(rx, 24.0, n, ppm=50.0, offset_hz=ppm_hz)
    zero = ber.rx_ber_point(rx, 24.0, n, offset_hz=0.0)
    print(f"\nPER at 24 dB: cfo 0 {base['per']:.4f}, cfo 100k {plain['per']:.4f} -> corrected {fixed['per']:.4f}; "
          f"50 ppm corrected {ppm_fixed['per']:.4f}")
    assert {k: zero[k] for k in ("pkt_err", "bit_err", "aa_miss", "len_reject", "extra_recs")} == \
           {k: base[k] for k in ("pkt_err", "bit_err", "aa_miss", "len_reject", "extra_recs")}
    assert abs(fixed["per"] - base["per"]) <= _bound(base["per"], n)
    assert plain["per"] > fixed["per"]
    # 50 ppm is a carrier offset of ppm_hz and a sampling clock 50e-6 fast, which the correction leaves (out of scope).
    # The same carrier offset alone, corrected, is within the 3-sigma bound of the cfo-0 run: what is left at 50 ppm is
    # the clock's part.  Its bound is empirical: measured on an H100, corrected 50 ppm gives 0.191 against 0.215.
    cfo_only = ber.rx_ber_point(rx, 24.0, n, cfo_hz=ppm_hz, offset_hz=ppm_hz)
    print(f"carrier alone at {ppm_hz:.0f} Hz, corrected: {cfo_only['per']:.4f}")
    assert abs(cfo_only["per"] - base["per"]) <= _bound(base["per"], n)
    assert ppm_fixed["aa_miss"] == 0 and abs(ppm_fixed["per"] - base["per"]) <= 0.04


def _synth_device(rx, cfg, n):
    """the GPU synthesiser's capture (rx_ber_synth_device) on the host"""
    ni = ((n * int(cfg["slot_samples"][0]) + 8191) // 8192) * 16384
    d_iq = torch.empty(ni, dtype=torch.int8, device="cuda")
    d_t = torch.empty(n * 64, dtype=torch.uint8, device="cuda")
    rx._check(rx._L.btle_b200_rx_ber_synth_device(rx._h, cfg.ctypes.data, 0, n, d_iq.data_ptr(), d_t.data_ptr(), None))
    torch.cuda.synchronize()
    return d_iq.cpu().numpy()


def test_estimator(rx):
    meds = {}
    for hz in (-150e3, -50e3, 0.0, 50e3, 150e3):
        cfg = ber.rx_ber_cfg(200.0, 0.0, hz, amplitude=100, slot_samples=2048)        # noiseless
        iq = _synth_device(rx, cfg, 400)
        recs = rx.rx(iq, offset_hz=hz)
        ok = recs[recs["crc_bad"] == 0]
        assert ok.size >= 390
        est = rx.rec_offsets(iq, ok)
        # the kernel's float32 sums against the restatement's float64 ones
        for r, e in zip(ok[:20], est[:20]):
            assert e == pytest.approx(offset_ref.rec_offset(iq, int(r["chunk"]), int(r["n0"]), int(r["access_addr"])), abs=2.0)
        meds[hz] = float(np.median(est))
        print(f"\nnoiseless {hz / 1e3:+.0f} kHz: median {meds[hz]:+.1f} Hz, spread {np.percentile(est, 5):+.0f} .. {np.percentile(est, 95):+.0f}")
        # Measured on an H100: medians 400-450 Hz below the offset.  The sums telescope to the phase turned between the
        # window's two ends, and the synthesiser's quarter-sample delays move both ends; 1 kHz bounds that with room.
        assert abs(meds[hz] - hz) <= 1000.0
        est0 = rx.estimate_offset(iq)                                             # decoded uncorrected
        if abs(hz) <= 50e3:
            assert est0 is not None and abs(est0 - hz) <= 1000.0
        else:
            assert est0 is None or abs(est0 - hz) <= 1000.0
    cfg = ber.rx_ber_cfg(20.0, 0.0, 100e3, amplitude=64, slot_samples=2048)
    iq = _synth_device(rx, cfg, 2000)
    est = rx.estimate_offset(iq)
    recs = rx.rx(iq, offset_hz=100e3)
    ok = recs[recs["crc_bad"] == 0]
    spread = rx.rec_offsets(iq, ok)
    print(f"\n20 dB, 100 kHz: estimate {est}, per-packet spread (std) {np.std(spread):.0f} Hz over {ok.size} packets")
    assert est is not None and abs(est - 100e3) <= 5000.0
    n_est = int((rx.rx(iq, offset_hz=est)["crc_bad"] == 0).sum())
    assert n_est >= ok.size - max(3, ok.size // 100)
    assert rx.estimate_offset(np.zeros(16384 * 4, dtype=np.int8)) is None


def _streams_caps(n_caps=3, packets=40):
    caps = [_capture(0.0 if k != 1 else 100e3, 22.0, 37 if k != 2 else 9, n=packets, seed=300 + k) for k in range(n_caps)]
    cfgs = np.concatenate([make_cfgs(1, rssi=[1 | 4, 2, 0][k], **c[1]) for k, c in enumerate(caps)])
    return [c[0] for c in caps], cfgs


def _cut_batch(rx, caps, cfgs, offset_hz=None):
    n = min(c.size for c in caps)
    return rx.rx_batch(np.stack([c[:n] for c in caps]), cfgs, offset_hz=offset_hz)


def test_stream_sessions_at_zero_offset(rx):
    """set_offset(.., 0) takes the rotated kernel; the session still returns the default kernel's records"""
    caps, cfgs = _streams_caps()
    want = _cut_batch(rx, caps, cfgs)
    with rx.streams(cfgs, segment_chunks=2) as s_:
        for i in range(3):
            s_.set_offset(i, 0.0)
        got = np.concatenate([s_.push(i, c) for i, c in enumerate(caps)] + [s_.finish()])
    _same(got[np.lexsort((got["chunk"], got["stream"]))], want)
    with rx.stream(segment_chunks=2, rssi=4, **ADV) as s1:
        s1.set_offset(0.0)
        got1 = np.concatenate([s1.push(caps[0][:70001]), s1.push(caps[0][70001:]), s1.finish()])
    _same(got1, rx.rx(caps[0], rssi=4, **ADV))


def test_stream_set_offset_mid_session(rx):
    """Capture 1 (at +100 kHz) is corrected from segment set k on: chunks before the switch equal rx_batch without
    correction, chunks from it on rx_batch with capture 1 at 100 kHz (the set boundary included); the single-capture
    session does the same."""
    caps, cfgs = _streams_caps()
    seg, k = 2, 1
    cut = (k + 1) * seg * 16384 + 4096                             # every capture's part of set k (look-ahead included) is complete
    with rx.streams(cfgs, segment_chunks=seg) as s_:
        parts = [s_.push(i, caps[i][:cut]) for i in range(3)]
        s_.set_offset(1, 100e3)
        parts += [s_.push(i, caps[i][cut:]) for i in range(3)] + [s_.finish()]
    got = np.concatenate(parts)
    got = got[np.lexsort((got["chunk"], got["stream"]))]
    old_b, new_b = _cut_batch(rx, caps, cfgs), _cut_batch(rx, caps, cfgs, offset_hz=[0.0, 100e3, 0.0])
    K = (k + 1) * seg
    exp = np.concatenate([np.concatenate([old_b[(old_b["stream"] == i) & (old_b["chunk"] < K)],
                                          new_b[(new_b["stream"] == i) & (new_b["chunk"] >= K)]]) for i in range(3)])
    one = (exp["stream"] == 1)
    assert (one & (exp["chunk"] < K)).sum() > 0 and (one & (exp["chunk"] >= K) & (exp["crc_bad"] == 0)).sum() > 10
    _same(got, exp)
    with rx.stream(segment_chunks=seg, **ADV) as s1:
        p1 = [s1.push(caps[1][:cut])]
        s1.set_offset(100e3)
        p1 += [s1.push(caps[1][cut:]), s1.finish()]
    got1 = np.concatenate(p1)
    o1, n1 = rx.rx(caps[1], **ADV), rx.rx(caps[1], offset_hz=100e3, **ADV)
    _same(got1, np.concatenate([o1[o1["chunk"] < K], n1[n1["chunk"] >= K]]))


def test_cli_offset(tmp_path):
    import os
    import subprocess
    cli = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "btle_b200", "btle_rx_b200")
    iq, _ = _capture(100e3, 26.0, 37, n=400, seed=9)
    f = tmp_path / "cap.bin"
    iq.tofile(f)

    def ok_pkts(*args):
        p = subprocess.run([cli, "-i", str(f), "-c", "37", "-j", "-Q", *args], capture_output=True, text=True, check=True)
        return sum('"t":"pkt"' in s and '"crc_ok":true' in s for s in p.stdout.splitlines()), p.stderr

    plain, _ = ok_pkts()
    fixed, _ = ok_pkts("--offset", "100000")
    auto, err = ok_pkts("--offset", "auto")
    p = subprocess.run([cli, "-i", f"{f}:37:8e89bed6:555555:100000", "-j", "-Q"], capture_output=True, text=True, check=True)
    per_cap = sum('"t":"pkt"' in s and '"crc_ok":true' in s for s in p.stdout.splitlines())
    print(f"\nCLI CRC-ok packets at 100 kHz: plain {plain}, --offset 100000 {fixed}, auto {auto} ({err.strip()}), FILE:..:HZ {per_cap}")
    assert "offset estimate" in err and fixed > plain and per_cap == fixed
    assert auto >= fixed - max(1, fixed // 100)
    r = BtleRx(0)
    assert fixed == int((r.rx(iq, offset_hz=100e3)["crc_bad"] == 0).sum())
    r.close()
    bad = subprocess.run([cli, "--iq-bin16", str(f), "--offset", "1000"], capture_output=True, text=True)
    assert bad.returncode != 0 and "--offset cannot be combined with --iq-bin16" in bad.stdout
    bad = subprocess.run([cli, "-i", str(f), "--offset", "9e9"], capture_output=True, text=True)
    assert bad.returncode != 0 and "Invalid --offset" in bad.stdout


def test_decode_connections_passes_offsets(rx):
    """decode_connections hands offset_hz to its rx_batch and rx_multi calls: at 0 it returns what it returns without"""
    from btle_b200 import hop
    iq, _ = _capture(0.0, 30.0, 37, n=20, seed=5)
    caps = np.zeros((40, iq.size), dtype=np.int8)
    caps[37] = iq
    a0, c0 = hop.decode_connections(rx, caps, discover=False)
    a1, c1 = hop.decode_connections(rx, caps, discover=False, offset_hz=np.zeros(40))
    _same(a1, a0)
    assert len(c1) == len(c0)
