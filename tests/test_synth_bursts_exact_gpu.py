"""synth_bursts_kernel byte for byte: every capture btle_b200_synth_streams_device writes is rebuilt from its own truth
records with the torch modulator (synth.air_bytes -> synth.modulate_batch -> floor(wave * amplitude / 127), added to the
floor with saturation) and must equal the device capture exactly."""
import numpy as np
import pytest
import torch

from btle_b200 import synth
from test_model_path_gpu import draw

pytestmark = pytest.mark.gpu

SLOT = 3300


def corrupt_bit(seed, stream, slot, pdu_len):
    """the bit synth_slot_geometry flips: truth only flags a corrupt burst, so restate it from the counter-based draw"""
    r = int(draw(seed, stream, slot, 2))
    return 16 + (r >> 16) % (8 * pdu_len - 16) if pdu_len > 2 else 8 * pdu_len + 3


def rebuild(cfgs, truth, floor, seed, amplitude):
    cap = floor.astype(np.int32)
    n_int8 = cap.shape[1]
    air = np.zeros((len(truth), 47), dtype=np.uint8)
    for k, t in enumerate(truth):
        c, n = cfgs[int(t["stream"])], int(t["pdu_len"])
        cb = corrupt_bit(seed, int(t["stream"]), int(t["slot"]), n) if t["corrupt"] else None
        a = synth.air_bytes(bytes(t["pdu"][:n]), int(c["channel"]), int(c["access_addr"]), int(c["crc_init"]), cb)
        assert len(a) == int(t["n_air_bytes"])
        air[k, :len(a)] = np.frombuffer(a, dtype=np.uint8)
    wav = synth.modulate_batch(torch.from_numpy(air), torch.from_numpy(truth["n_air_bytes"].astype(np.int64)))
    wav = ((wav.to(torch.int32) * amplitude) // 127).numpy()
    for k, t in enumerate(truth):
        a = 2 * int(t["start_sample"])
        m = min(2 * (32 * int(t["n_air_bytes"]) + 16), n_int8 - a)
        cap[int(t["stream"]), a:a + m] += wav[k, :m]
    return np.clip(cap, -128, 127).astype(np.int8)


@pytest.mark.parametrize("amplitude", [1, 64, 127])
@pytest.mark.parametrize("noise", [2, 1])
def test_device_captures_equal_their_rebuilt_truth(amplitude, noise):
    """Advertising and data-channel streams, straddling and corrupt bursts (2-byte PDUs too), a capture whose odd length
    ends inside a slot; on the zero floor (noise 2) and on full-scale noise (noise 1), where the sums saturate."""
    cfgs = synth.channel_plan(40)[[0, 11, 24, 36, 37, 38, 39]]
    n_int8 = 2 * SLOT * 160 + 2 * 1234 + 1
    seed = 1000 + amplitude
    kw = dict(slot_samples=SLOT, corrupt_every=3, straddle_every=4, noise=noise)
    iq, truth = synth.synth_streams_device(cfgs, n_int8, seed, amplitude=amplitude, **kw)
    floor, _ = synth.synth_streams_device(cfgs, n_int8, seed, amplitude=0, want_truth=False, **kw)
    floor = floor.cpu().numpy()
    assert noise == 1 or not floor.any()
    assert len(truth) == len(cfgs) * 160 and truth["straddle"].sum() > 20
    assert ((truth["pdu_len"] == 2) & (truth["corrupt"] == 1)).any() and ((truth["pdu_len"] > 2) & (truth["corrupt"] == 1)).any()
    assert np.array_equal(iq.cpu().numpy(), rebuild(cfgs, truth, floor, seed, amplitude))
