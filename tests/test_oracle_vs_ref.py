"""Pins our C restatement (oracle/btle_oracle.c) to the reference itself
(oracle/_ref = the reference's btle_rx.c compiled unmodified).  Runs wherever
oracle/_ref exists (here, and on the GPU box where the built binaries travel)."""
import numpy as np
import pytest
import torch

import orc
from btle_b200 import synth

needs_ref = pytest.mark.skipif(not orc.ref_available(), reason="oracle/_ref not built")


def _cmp(iq, **cfg):
    rec = orc.rx_stream(iq, **cfg)
    ref = orc.ref_rx_stream(iq, **cfg)
    orc.assert_same_as_ref(rec, ref)
    return rec


@needs_ref
def test_synth_adv_stream_all_adv_channels():
    for ch in (37, 38, 39):
        iq, truth = synth.make_adv_stream(512 * 1024, seed=100 + ch, channel=ch, corrupt_every=7)
        rec = _cmp(iq.numpy(), channel=ch)
        assert len(rec) >= 60
        assert rec["crc_bad"].sum() >= 1


@needs_ref
def test_data_channels_custom_aa_crcinit():
    for ch in (0, 9, 10, 36):
        aa, ci = 0x60850A1B + ch, 0xA77B22 ^ ch
        iq, _ = synth.make_adv_stream(256 * 1024, seed=200 + ch, channel=ch, access_addr=aa, crc_init=ci,
                                      data_channel_pdu=True, corrupt_every=5, slot_samples=2048)
        rec = _cmp(iq.numpy(), channel=ch, access_addr=aa, crc_init=ci)
        assert len(rec) >= 50


@needs_ref
def test_raw_mode():
    iq, _ = synth.make_adv_stream(256 * 1024, seed=5, channel=37)
    rec = _cmp(iq.numpy(), channel=37, raw=1)
    assert len(rec) >= 30 and (rec["n_bytes"] == 42).all()


@needs_ref
@pytest.mark.parametrize("seed", range(6))
def test_fuzz_random_iq_loose_masks(seed):
    """Adversarial: full-scale random IQ with sparse masks -> very many hits, negative
    n0 through the zeroed history (App. A.2), hits in the look-ahead tail, length-guard
    breaks, bad ADV lengths."""
    rng = np.random.default_rng(seed)
    iq = rng.integers(-128, 128, 8 * 16384 + 5000, dtype=np.int8)
    masks = [0x0000000F, 0x000000FF, 0x80000001, 0x00000000, 0xF0000000, 0x00010100]
    aas = [0x8E89BED6, 0x00000000, 0xFFFFFFFF, 0x55555555, 0x80000000, 0x12345678]
    for ch in (37, 3):
        for raw in (0, 1):
            rec = _cmp(iq, channel=ch, access_addr=aas[seed], access_mask=masks[seed], raw=raw,
                       crc_init=0x123456)
            assert len(rec) > 8


@needs_ref
def test_fuzz_small_amplitude_zero_products():
    """d uses a strict > 0 (btle_rx.c:1533): zeros and tiny amplitudes must give bit 0."""
    rng = np.random.default_rng(99)
    iq = rng.integers(-1, 2, 6 * 16384, dtype=np.int8)
    _cmp(iq, channel=38, access_mask=0x000003FF, access_addr=0x2AA)
    _cmp(np.zeros(3 * 16384, dtype=np.int8), channel=37, access_addr=0, access_mask=0xFFFFFFFF)


@needs_ref
def test_short_and_ragged_lengths():
    rng = np.random.default_rng(3)
    for n in (0, 100, 16383, 16384, 16385, 16384 + 3007, 2 * 16384 + 1):
        iq = rng.integers(-128, 128, n, dtype=np.int8)
        _cmp(iq, channel=37, access_mask=0xFF)


@needs_ref
def test_worst_case_packets_per_chunk():
    """BTLE_MAX_PKTS_PER_CHUNK (include/btle_b200.h): with mask 0 every window matches, through the zeroed
    history up to 31 symbols before the restart point, so a zero-length data PDU advances the cursor by only
    328 int8 -> 51 packets in one chunk; with bit 0 of the mask set it is 576 int8 -> at most 34."""
    z = np.zeros(2 * 16384 + 3008, dtype=np.int8)
    best = 0
    for ch in range(37):
        rec = _cmp(z, channel=ch, access_addr=0, access_mask=0)
        best = max(best, int(np.bincount(rec["chunk"]).max()))
    assert best == 51
    # a 1 in bit 0 of the masked access address cannot be matched by the zeroed history
    rng = np.random.default_rng(0)
    for iq in (rng.integers(-128, 128, z.size, dtype=np.int8), rng.integers(-1, 2, z.size, dtype=np.int8)):
        for ch in (1, 9, 20):
            rec = _cmp(iq, channel=ch, access_addr=1, access_mask=1)
            assert len(rec) > 10 and int(np.bincount(rec["chunk"]).max()) <= 34


# ---- -v: hits the reference rejects for their ADV header length (PktBAD, btle_rx.c:2291-2298) -------------------------
def _cmp_rejected(iq, **cfg):
    """Oracle with report_rejected against the reference's counted packets and rejected hits, in the reference's order."""
    rec = orc.rx_stream(iq, report_rejected=1, **cfg)
    orc.assert_same_as_ref(rec, orc.ref_rx_stream(iq, report_rejected=1, **cfg))
    rej = rec[(rec["flags"] & 4) != 0]
    assert (rej["n_bytes"] == 2).all() and not rej["crc_bad"].any() and not rej["bytes"][:, 2:].any()
    assert rec[(rec["flags"] & 4) == 0].tobytes() == orc.rx_stream(iq, **cfg).tobytes()     # the flag only adds records
    mag = [int(np.abs(iq[16384 * r["chunk"] + 2 * r["n0"]:][:256].astype(np.int32)).sum()) & 0xFFFF
           for r in rej if 16384 * r["chunk"] + 2 * r["n0"] >= 0]
    assert mag == [int(r["mag_sum"]) for r in rej if 16384 * r["chunk"] + 2 * r["n0"] >= 0]   # summed before the length check
    return rec


@needs_ref
def test_rejected_hits_zero_capture_mask0_worst_case():
    """Mask 0 on zeros: every window matches through the zeroed history, every header is the channel's whitening
    sequence.  On channels 38 and 39 its length is outside 6..37: BTLE_MAX_RECS_PER_CHUNK = 123 rejected hits per chunk."""
    z = np.zeros(3 * 16384 + 3008, dtype=np.int8)
    for ch in (37, 38, 39):
        rec = _cmp_rejected(z, channel=ch, access_addr=0, access_mask=0)
        if ch != 37:
            assert len(rec) == 3 * 123 and (rec["flags"] & 4).all()
            assert list(np.bincount(rec["chunk"])) == [123] * 3


@needs_ref
@pytest.mark.parametrize("mask", [0x00000000, 0x0000000F, 0x80000001, 0x0F000000, 0x000000FF])
def test_rejected_hits_noise_sparse_masks(mask):
    rng = np.random.default_rng(mask & 0xFFFF)
    iq = rng.integers(-128, 128, 8 * 16384 + 3008, dtype=np.int8)
    n_rej = 0
    for ch in (37, 38, 39):
        rec = _cmp_rejected(iq, channel=ch, access_mask=mask)
        n_rej += int(((rec["flags"] & 4) != 0).sum())
    assert n_rej > 20


@needs_ref
def test_rejected_hits_planted_bad_lengths():
    """Bursts whose ADV header says PloadL 3, 45 and 5 between valid ones, on a quiet floor, with the full mask."""
    pdus = [synth.adv_pdu(0, 1, 0, bytes(range(6 + k))) for k in range(6)]
    pdus.insert(1, synth.adv_pdu(0, 1, 0, b"\x01\x02\x03"))
    pdus.insert(4, bytes([0x02, 45]) + bytes(range(20)))
    pdus.append(synth.adv_pdu(6, 0, 1, bytes(5)))
    for ch in (37, 39):
        iq = synth.make_pdu_stream(pdus, ch, seed=9, corrupt={2})
        rec = _cmp_rejected(iq, channel=ch)
        rej = rec[(rec["flags"] & 4) != 0]
        assert len(rej) == 3 and sorted(int(b[1]) & 0x3F for b in rej["bytes"]) == [3, 5, 45]
        assert len(rec) == len(pdus)


@needs_ref
def test_rejected_flag_changes_nothing_on_data_channels_and_raw():
    rng = np.random.default_rng(17)
    iq = rng.integers(-128, 128, 6 * 16384 + 3008, dtype=np.int8)
    for ch, raw in ((3, 0), (20, 0), (37, 1), (39, 1)):
        for mask in (0, 0x0F000000):
            rec = _cmp_rejected(iq, channel=ch, access_mask=mask, raw=raw)
            assert len(rec) > 5 and not (rec["flags"] & 4).any()
