// btle_params.h — host/device-neutral construction of the per-stream parameters and of the two
// protocol tables.  Shared by the CUDA library and by the test-only CPU emulator of the kernels.
#pragma once
#include "../../include/btle_b200.h"
#include "btle_core.cuh"

namespace btle {

// BLE data whitening, 7-bit LFSR x^7+x^4+1 whose register starts as 1 followed by the 6 channel
// bits, MSB first (matlab/scramble_gen.m:3-41).  Register bit k = stage k: stage 0 = the
// constant 1, stages 1..6 = channel bits 5..0.
BTLE_HD uint32_t whiten_seed(int channel) {
  uint32_t reg = 1u;
  for (int i = 0; i < 6; ++i) reg |= ((uint32_t)(channel >> (5 - i)) & 1u) << (1 + i);
  return reg;
}

// One LFSR step: returns the next whitening bit (stage 6) and advances the register.
BTLE_HD uint32_t whiten_step(uint32_t &reg) {
  const uint32_t o = (reg >> 6) & 1u;
  reg = ((reg << 1) & 0x7Fu) | o;     // stages move up, stage0 <- old stage6
  reg ^= o << 4;                      // stage4 <- old stage3 ^ old stage6
  return o;
}

// scramble_table[ch][i] (scramble_table.h:4): the whitening bytes of a channel, LSB first.
BTLE_HD void make_whiten_row(int channel, uint8_t out[48]) {
  uint32_t reg = whiten_seed(channel);
  for (int b = 0; b < 48; ++b) {
    uint32_t v = 0;
    for (int bit = 0; bit < 8; ++bit) v |= whiten_step(reg) << bit;
    out[b] = (b < 42) ? (uint8_t)v : 0;
  }
}

// crc_table[b] (btle_rx.c:971-1004): reflected CRC-24, polynomial 0xDA6000, one byte from 0.
BTLE_HD uint32_t make_crc_entry(uint32_t b) {
  uint32_t crc = b;
  for (int j = 0; j < 8; ++j) crc = (crc >> 1) ^ ((crc & 1u) ? 0xDA6000u : 0u);
  return crc;
}

// crc4[k*256 + b]: CRC register after byte b followed by k zero bytes (slicing-by-4 tables);
// crc4[0..255] is crc_table itself.
BTLE_HD void make_crc4(uint32_t *crc4 /*1024*/) {
  for (uint32_t b = 0; b < 256; ++b) crc4[b] = make_crc_entry(b);
  for (int k = 1; k < 4; ++k)
    for (uint32_t b = 0; b < 256; ++b) {
      const uint32_t x = crc4[(k - 1) * 256 + b];
      crc4[k * 256 + b] = crc4[x & 0xFFu] ^ (x >> 8);
    }
}

// crc_init_reorder (btle_rx.c:1969-1993): bit-reverse each of the three bytes.
BTLE_HD uint32_t crc_init_reorder(uint32_t k) {
  uint32_t r = 0;
  for (int byte = 0; byte < 3; ++byte)
    for (int i = 0; i < 8; ++i) r |= ((k >> (8 * byte + i)) & 1u) << (8 * byte + 7 - i);
  return r;
}

// The receive kernel's discriminator mode (its DISC parameter), one per launch: the reference's quarter-symbol bit,
// BTLE_CFG_SYMBOL_SPACED, or BTLE_CFG_SYMBOL_SPACED with BTLE_CFG_LOWPASS.
enum : int { kDiscQuarter = 0, kDiscSymbol = 1, kDiscLowpass = 2 };
BTLE_HD int disc_mode(const btle_stream_cfg &cfg) {
  if (!(cfg.rssi & BTLE_CFG_SYMBOL_SPACED)) return kDiscQuarter;
  return (cfg.rssi & BTLE_CFG_LOWPASS) ? kDiscLowpass : kDiscSymbol;
}

// whiten_words: 12 little-endian words of make_whiten_row(channel).
BTLE_HD void make_params(const btle_stream_cfg &cfg, const uint32_t *whiten_words, StreamParams &sp) {
  sp.aa = cfg.access_addr;
  sp.mask = cfg.access_mask;
  sp.crc_init = crc_init_reorder(cfg.crc_init);
  sp.channel = cfg.channel;
  sp.raw = cfg.raw ? 1 : 0;
  sp.adv = (cfg.channel == 37 || cfg.channel == 38 || cfg.channel == 39) ? 1 : 0;
  sp.rssi = (cfg.rssi & BTLE_CFG_RSSI) ? 1 : 0;
  sp.report_rejected = (cfg.rssi & BTLE_CFG_REPORT_REJECTED) ? 1 : 0;
  sp.centre_hits = (cfg.rssi & BTLE_CFG_CENTRE_HITS) ? 1 : 0;
  sp.recover = ((cfg.rssi & BTLE_CFG_RECOVER) && !cfg.raw) ? 1 : 0;
  sp.correct = ((cfg.rssi & BTLE_CFG_CORRECT) && !cfg.raw) ? 1 : 0;
  const uint32_t am = cfg.access_addr & cfg.access_mask;
  int tz = 0;
  while (tz < 31 && !((am >> tz) & 1u)) ++tz;
  sp.tz = tz;   // am == 0 -> 31 (a window may start at most 31 symbols before a restart)
  // Prefilter taps.  Which taps are chosen only affects speed, never results (every candidate is
  // re-checked exactly).  Off-packet IQ is a small-amplitude noise floor whose discriminator bits
  // are mostly 0 (products of 0/+-1 values rarely exceed 0), so taps that expect a 1 reject noise
  // far better than taps that expect a 0: take up to 2/3 of the taps from the 1-bits of the masked
  // access address and the rest from its 0-bits, each set spread evenly over the word.
  int ones[32], zeros[32], n1 = 0, n0 = 0;
  for (int p = 0; p < 32; ++p)
    if ((cfg.access_mask >> p) & 1u) {
      if ((cfg.access_addr >> p) & 1u) ones[n1++] = p; else zeros[n0++] = p;
    }
  int want1 = kTapsOne;
  if (want1 > n1) want1 = n1;
  int want0 = kMaxTaps - want1;
  if (want0 > n0) { want0 = n0; want1 = (kMaxTaps - want0 < n1) ? kMaxTaps - want0 : n1; }
  int nt = 0;
  for (int j = 0; j < want1; ++j) {
    const int p = ones[(j * n1) / want1];
    sp.tap_pos[nt] = (uint32_t)p; sp.tap_xor[nt] = 0u; ++nt;
  }
  for (int j = 0; j < want0; ++j) {
    const int p = zeros[(j * n0) / want0];
    sp.tap_pos[nt] = (uint32_t)p; sp.tap_xor[nt] = 0xFFFFFFFFu; ++nt;
  }
  sp.ntaps = nt;
  sp.typed = (want1 == kTapsOne && want0 == kMaxTaps - kTapsOne) ? 1 : 0;
  for (int t = nt; t < kMaxTaps; ++t) {
    sp.tap_pos[t] = nt ? sp.tap_pos[t % nt] : 0u;
    sp.tap_xor[t] = nt ? sp.tap_xor[t % nt] : 0u;
  }
  for (int j = 0; j < 12; ++j) sp.whiten[j] = whiten_words[j];
}

}  // namespace btle
