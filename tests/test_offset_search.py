"""BTLE_CFG_OFFSET_SEARCH on the CPU: the merge step the kernel runs (os_merge_step in btle_core.cuh, built into the emulator
library from tests/emul/btle_offset_search_emul.cpp) against the restatement (offset_search_ref.py) on generated record
lists, and end to end: the chain restatements at each hypothesis, merged by both."""
import ctypes

import numpy as np
import pytest

import emul
import golden_util
import lowpass_emul
import lowpass_ref
import mode_ref
import offset_search_ref as osr
from btle_b200 import _native, rx as rxmod
from orc import REC_DTYPE

REJ, RAW = 4, 1


def emul_merge(per_hyp):
    """the emulator's merge of one cfg's hypotheses (per_hyp[h]: records in (chunk, n0) order)"""
    L = emul.lib()
    f = L.emul_os_merge
    f.restype = ctypes.c_long
    f.argtypes = [ctypes.c_void_p] * 5 + [ctypes.c_long, ctypes.c_void_p]
    allr = np.concatenate(per_hyp) if per_hyp else np.zeros(0, dtype=REC_DTYPE)
    hyp = np.concatenate([np.full(len(p), h, dtype=np.int32) for h, p in enumerate(per_hyp)])
    chunk = np.ascontiguousarray(allr["chunk"], dtype=np.int32)
    n0 = np.ascontiguousarray(allr["n0"], dtype=np.int32)
    flags = np.ascontiguousarray(allr["flags"], dtype=np.uint8)
    bad = np.ascontiguousarray(allr["crc_bad"], dtype=np.uint8)
    out = np.zeros(allr.size + 1, dtype=np.int32)
    n = f(hyp.ctypes.data, chunk.ctypes.data, n0.ctypes.data, flags.ctypes.data, bad.ctypes.data, allr.size, out.ctypes.data)
    idx = out[:n].view(np.uint32)
    got = allr[(idx & 0x7FFFFFFF).astype(np.int64)].copy()
    got["flags"] |= np.where(idx >> 31, osr.REC_OFFSET_SEARCH, 0).astype(np.uint8)
    return got


def recs(rows, stream=0):
    """records from (chunk, n0, kind) rows, kind 'ok' / 'bad' (counted, CRC failed) / 'rej'; bytes tag the row"""
    r = np.zeros(len(rows), dtype=REC_DTYPE)
    for i, (k, n0, kind) in enumerate(rows):
        r[i]["stream"], r[i]["chunk"], r[i]["n0"], r[i]["channel"] = stream, k, n0, 37
        r[i]["crc_bad"] = kind == "bad"
        r[i]["flags"] = 2 | (REJ if kind == "rej" else 0)
        r[i]["n_bytes"] = 2 if kind == "rej" else 10
        r[i]["bytes"][0], r[i]["bytes"][1] = i & 255, len(rows) & 255
    return r[np.lexsort((r["n0"], r["chunk"]))] if len(rows) else r


def check(per_hyp):
    want = osr.merge(per_hyp, 1)
    got = emul_merge(per_hyp)
    assert got.tobytes() == want.tobytes()
    return want


def hyps(*lists):
    return [recs(x) for x in lists] + [recs([]) for _ in range(7 - len(lists))]


def test_window_edge_8_and_9():
    w = check(hyps([(0, 100, "bad"), (0, 500, "ok")], [(0, 108, "ok"), (0, 509, "ok")]))
    assert [(int(r["n0"]), int(r["flags"]) >> 7) for r in w] == [(108, 1), (500, 0), (509, 1)]
    w = check(hyps([(0, 100, "bad")], [(0, 109, "ok"), (0, 91, "ok")]))
    assert list(w["n0"]) == [91, 100, 109]          # 9 samples away: both inserted, the failed one stays
    w = check(hyps([(0, 100, "bad")], [(0, 92, "ok")]))
    assert list(w["n0"]) == [92]


def test_ok_failed_rejected():
    w = check(hyps([(0, 200, "ok"), (0, 400, "bad"), (0, 600, "rej")],
                   [(0, 203, "ok"), (0, 404, "ok"), (0, 597, "ok"), (0, 800, "bad"), (0, 900, "rej")]))
    assert [(int(r["n0"]), int(r["flags"]) & 128) for r in w] == [(200, 0), (404, 128), (597, 128)]


def test_one_insert_displaces_several():
    w = check(hyps([(0, 10, "rej"), (0, 14, "bad"), (0, 18, "rej"), (0, 30, "bad"), (0, 40, "ok")], [(0, 16, "ok"), (0, 33, "ok")]))
    assert list(w["n0"]) == [16, 30, 40]             # 10, 14, 18 go; 33 is within 8 of the CRC-ok record at 40


def test_hypothesis_order_at_equal_delta():
    w = check(hyps([], [(0, 300, "ok")], [(0, 302, "ok")]))       # -50 kHz (h = 1) before +50 kHz (h = 2)
    assert list(w["n0"]) == [300]
    w = check(hyps([], [], [(0, 302, "ok")], [(0, 299, "ok")]))   # +50 kHz (h = 2) before -100 kHz (h = 3)
    assert list(w["n0"]) == [302]


def test_chunk_independence():
    w = check(hyps([(0, 8190, "bad"), (1, 5, "ok")], [(0, 8191, "ok"), (1, -124, "ok"), (1, 6, "ok")]))
    assert [(int(r["chunk"]), int(r["n0"])) for r in w] == [(0, 8191), (1, -124), (1, 5)]


def test_density_bound():
    """hypothesis 0 with 123 records and six hypotheses with 51 CRC-ok packets each, all more than 8 samples apart: the
    merged chunk reaches the stated bound"""
    pos = iter(range(-124, 8192, 19))
    h0 = [(0, next(pos), "rej") for _ in range(123)]
    rest = [[(0, next(pos), "ok") for _ in range(51)] for _ in range(6)]
    w = check(hyps(h0, *rest))
    assert len(w) == osr.MAX_MERGED_RECS_PER_CHUNK == _native.MAX_MERGED_RECS_PER_CHUNK == 429


def test_generated_lists():
    rng = np.random.default_rng(5)
    for t in range(300):
        nch = int(rng.integers(1, 4))
        centres = rng.integers(-124, 8192, size=int(rng.integers(1, 12)))
        per = []
        for h in range(7):
            rows = []
            for k in range(nch):
                n = int(rng.integers(0, 8))
                n0 = np.clip(rng.choice(centres, n) + rng.integers(-10, 11, n), -124, 8191)
                kinds = rng.choice(["ok", "bad", "rej"], n, p=[0.5, 0.3, 0.2]) if h == 0 else rng.choice(["ok", "bad", "rej"], n)
                rows += sorted({(k, int(a)): str(b) for a, b in zip(n0, kinds)}.items())
            per.append(recs([(k, a, b) for (k, a), b in rows]))
        w = check(per)
        for k in range(nch):
            assert (w["chunk"] == k).sum() <= osr.MAX_MERGED_RECS_PER_CHUNK
        # invariants: every CRC-ok hypothesis-0 record stays unchanged; the others carry the flag and crc_bad 0
        ok0 = [r for r in per[0] if osr.ok(r)]
        assert all(any(r.tobytes() == x.tobytes() for x in w) for r in ok0)
        new = w[(w["flags"] & 128) != 0]
        assert (new["crc_bad"] == 0).all() and ((new["flags"] & REJ) == 0).all()


def restated_hyps(iq, f_c, fields, mode):
    """each hypothesis's records of one capture and cfg from the chain restatement in `mode` ('quarter', 'symbol', 'lowpass')"""
    out = []
    for hz in osr.hyp_offsets(f_c):
        if mode == "lowpass":
            out.append(lowpass_ref.rx_stream(iq, float(hz), **fields))
        else:
            out.append(mode_ref.rx_stream(iq, float(hz), mode == "symbol", **fields))
    return out


def several_offsets(n_chunks=16, seed=3):
    """a synthesised channel-37 capture, every four chunks moved to another carrier offset"""
    from btle_b200 import synth
    iq, _ = synth.make_adv_stream(n_chunks * 16384, seed=seed, channel=37, slot_samples=1500)
    iq = np.asarray(iq, dtype=np.int8).reshape(-1)
    offs = (-120e3, -40e3, 60e3, 140e3)
    part = n_chunks * 16384 // len(offs)
    return np.concatenate([mode_ref.rotate(iq[i * part:(i + 1) * part], hz) for i, hz in enumerate(offs)])


@pytest.mark.parametrize("mode", ["quarter", "symbol", "lowpass"])
def test_end_to_end_synthesised(mode):
    """packets at several offsets: the restated hypotheses merged by the emulator's step equal the restatement's merge, and
    the bank finds more CRC-ok packets than hypothesis 0"""
    iq = several_offsets()
    fields = dict(channel=37, rssi=_native.CFG_RSSI | _native.CFG_REPORT_REJECTED)
    per = restated_hyps(iq, 0.0, fields, mode)
    got = emul_merge(per)
    want = osr.merge(per, 1)
    assert got.tobytes() == want.tobytes()
    ok = lambda r: int(((r["crc_bad"] == 0) & ((r["flags"] & REJ) == 0)).sum())
    assert ok(want) > ok(per[0]), (ok(want), ok(per[0]))


def test_end_to_end_lowpass_unit_path():
    """the emulator's low-pass unit path at each hypothesis (rotated), merged by the shared step, equals the restatement"""
    iq = several_offsets(8, seed=4)
    c = rxmod.make_cfgs(1, channel=37, rssi=_native.CFG_REPORT_REJECTED | _native.CFG_CENTRE_HITS, symbol_spaced=1, lowpass=1)[0]
    per_emul = [lowpass_emul.rx_stream(iq, c, 0, float(hz)) for hz in osr.hyp_offsets(20e3)]
    per_ref = restated_hyps(iq, 20e3, dict(channel=37, rssi=int(c["rssi"])), "lowpass")
    for a, b in zip(per_emul, per_ref):
        assert a.tobytes() == b.tobytes()
    assert emul_merge(per_emul).tobytes() == osr.merge(per_ref, 1).tobytes()


def test_end_to_end_goldens():
    """every golden capture with its own cfg, -v and RSSI included"""
    n = 0
    for name in golden_util.cases():
        z, cfg = golden_util.load(name)
        fields = golden_util.rx_cfg(cfg)
        if fields.get("raw"):
            continue                                    # raw cfgs are refused with the flag
        fields["rssi"] = fields.get("rssi", 0) | _native.CFG_RSSI
        iq = np.asarray(z["iq"], dtype=np.int8)
        per = restated_hyps(iq, 0.0, fields, "quarter")
        got = emul_merge(per)
        assert got.tobytes() == osr.merge(per, 1).tobytes(), name
        n += got.size
    assert n > 0


def test_make_cfgs_flag():
    c = rxmod.make_cfgs(2, offset_search=1, symbol_spaced=1)
    assert list(c["rssi"]) == [1040, 1040]
    assert list(rxmod._with_fields(c, {"offset_search": 0})["rssi"]) == [16, 16]
    assert _native.CFG_OFFSET_SEARCH == 1024 and _native.REC_OFFSET_SEARCH == 128
    assert _native.OFFSET_SEARCH_HZ == osr.HYP_HZ
    from btle_b200 import ber
    assert int(ber.rx_ber_cfg(10.0, offset_search=True)["flags"][0]) == 1024
