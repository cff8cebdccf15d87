"""Plain int64 restatements of the two transmit modulators, one sample at a time with the phase as an unbounded running
sum (no pass structure, no cumsum), pinned to the reference transmitters' own waveforms and to the torch modulators
(synth.modulate_batch / modulate_batch_8sps) up to the 128-byte rows btle_b200_tx_modulate_device accepts.
test_tx_edges_gpu.py compares the CUDA modulator with them."""
import numpy as np
import torch

import golden_util as G
from btle_b200 import synth

GAUSS4 = (2, 11, 32, 53, 60, 53, 32, 11, 2)                              # btle_tx.c gauss_coef_int8[4..12]
GAUSS8 = (0, 0, 0, 1, 4, 9, 15, 22, 24, 22, 15, 9, 4, 1, 0, 0, 0)        # btlelib.py:146-160


def phase_table(n):
    """round(127 cos / sin(2 pi k / n)) in float64, as int64"""
    k = np.arange(n, dtype=np.float64)
    return np.round(127.0 * np.cos(2 * np.pi * k / n)).astype(np.int64), np.round(127.0 * np.sin(2 * np.pi * k / n)).astype(np.int64)


def _symbols(air, nbytes):
    """+-1 per air bit (LSB first) for bits below 8 * nbytes, 0 behind: int64 [B, 8 L]"""
    air = np.asarray(air, dtype=np.uint8)
    nb = np.asarray(nbytes, dtype=np.int64)
    bits = np.unpackbits(air, axis=1, bitorder="little").astype(np.int64)
    return np.where(np.arange(bits.shape[1])[None, :] < 8 * nb[:, None], 2 * bits - 1, 0), nb


def modulate4_ref(air, nbytes, phases=None):
    """btle_tx.c:1022-1063 at 4 sps.  air uint8 [B, L], nbytes [B] in 0..L.  Returns int8 [B, 2 (32 L + 16)] interleaved
    I, Q; sample m < 32 nbytes + 16 is table[phase before word m mod 1024], the rest 0.  The impulse of symbol k sits at
    over-sampled index 15 + 4k, word m = sum_{j=3..11} g[j-3] os[m+j] for m < nsamp - 1.  `phases`, a list, receives
    the extreme unreduced phases reached."""
    sym, nb = _symbols(air, nbytes)
    B, nbit_max = sym.shape
    n_out = 4 * nbit_max + 16
    nsamp = 32 * nb + 16
    cos, sin = phase_table(1024)
    out = np.zeros((B, n_out, 2), dtype=np.int64)
    phase = np.zeros(B, dtype=np.int64)
    lo = hi = 0
    for m in range(n_out):
        on = m < nsamp
        out[on, m, 0] = cos[phase[on] % 1024]
        out[on, m, 1] = sin[phase[on] % 1024]
        word = np.zeros(B, dtype=np.int64)
        for j in range(3, 12):
            idx = m + j - 15                                  # over-sampled index m + j, less the 15-sample lead
            if idx >= 0 and idx % 4 == 0 and idx // 4 < nbit_max:
                word += GAUSS4[j - 3] * sym[:, idx // 4]
        phase += np.where(m < nsamp - 1, word, 0)
        lo, hi = min(lo, int(phase.min())), max(hi, int(phase.max()))
    if phases is not None:
        phases += [lo, hi]
    return out.reshape(B, 2 * n_out).astype(np.int8)


def modulate8_ref(air, nbytes, phases=None):
    """btlelib.py:146-189 at 8 sps.  air uint8 [B, L], nbytes [B] in 0..L.  Returns (i, q) int8 [B, 64 L + 16]; the input
    is 17 samples of -1, then the NRZ of the 8 nbytes bits at 8 samples each, then 0; word m = (sum_j g[j] x[17 - j + m])
    >> 1 for m < 64 nbytes + 16, and sample m is table[phase including word m mod 2048], 0 behind the packet."""
    sym, nb = _symbols(air, nbytes)
    B, nbit_max = sym.shape
    n_out = 8 * nbit_max + 16
    nsamp = 64 * nb + 16

    def x(t):
        if t < 17:
            return np.full(B, -1, dtype=np.int64)
        k = (t - 17) // 8
        return sym[:, k] if k < nbit_max else np.zeros(B, dtype=np.int64)

    cos, sin = phase_table(2048)
    oi = np.zeros((B, n_out), dtype=np.int64)
    oq = np.zeros((B, n_out), dtype=np.int64)
    phase = np.zeros(B, dtype=np.int64)
    lo = hi = 0
    for m in range(n_out):
        on = m < nsamp
        y = np.zeros(B, dtype=np.int64)
        for j in range(17):
            y += GAUSS8[j] * x(17 - j + m)
        phase += np.where(on, y >> 1, 0)
        oi[on, m] = cos[phase[on] % 2048]
        oq[on, m] = sin[phase[on] % 2048]
        lo, hi = min(lo, int(phase.min())), max(hi, int(phase.max()))
    if phases is not None:
        phases += [lo, hi]
    return oi.astype(np.int8), oq.astype(np.int8)


def random_rows(rng, B, L, extremes=True):
    """B rows of L air bytes with random lengths 0..L; the first rows are all-0x00 and all-0xFF at full length"""
    air = rng.integers(0, 256, (B, L), dtype=np.uint8)
    nb = rng.integers(0, L + 1, B)
    if extremes:
        air[0], air[1], nb[:2] = 0x00, 0xFF, L
    return air, nb


def test_references_equal_the_reference_transmitters_goldens():
    for i in range(4):
        z, cfg = G.load(f"tx_loopback_{i}.npz")
        air = synth.air_bytes(bytes.fromhex(str(z["pdu_hex"])), cfg["channel"], cfg.get("access_addr", synth.ADV_ACCESS_ADDR),
                              cfg.get("crc_init", synth.ADV_CRC_INIT))
        w = modulate4_ref(np.frombuffer(air, dtype=np.uint8)[None], [len(air)])[0]
        assert np.array_equal(w, z["tx_wave"]), i
    z = np.load(G.GOLD + "/btlelib_rx.npz")
    for n in (0, 1):
        air = np.packbits(z[f"tx{n}_phy_bit"].astype(np.uint8), bitorder="little")
        oi, oq = modulate8_ref(air[None], [air.size])
        assert np.array_equal(oi[0], z[f"tx{n}_i"]) and np.array_equal(oq[0], z[f"tx{n}_q"]), n


def test_4sps_reference_equals_torch_modulator_up_to_128_bytes():
    rng = np.random.default_rng(41)
    air, nb = random_rows(rng, 24, 128)
    nb[2:5] = 0, 1, 127
    phases = []
    ref = modulate4_ref(air, nb, phases)
    assert phases[0] < -2.5e5 and phases[1] > 2.5e5              # the all-0x00 / all-0xFF rows reach about -+2.6e5
    assert np.array_equal(ref, synth.modulate_batch(torch.from_numpy(air), torch.from_numpy(nb)).numpy())


def test_8sps_reference_equals_torch_modulator_up_to_128_bytes():
    rng = np.random.default_rng(42)
    air, nb = random_rows(rng, 10, 128)
    nb[2:4] = 1, 127
    phases = []
    oi, oq = modulate8_ref(air, nb, phases)
    assert phases[0] < -5e5 and phases[1] > 5e5                  # about -+5.2e5 on the all-0x00 / all-0xFF rows
    for b in range(len(nb)):
        bits = torch.from_numpy(np.unpackbits(air[b, :nb[b]], bitorder="little")).unsqueeze(0)
        ri, rq = synth.modulate_batch_8sps(bits)
        m = ri.shape[1]
        assert np.array_equal(oi[b, :m], ri[0].numpy()) and np.array_equal(oq[b, :m], rq[0].numpy()), b
        assert not oi[b, m:].any() and not oq[b, m:].any()
