// Test-only CPU emulator of BTLE_CFG_LOWPASS: the filtered-word helper (lp_word), the dense walk over filtered words
// (dbits_group_lowpass) and recovery on filtered samples (repair_packet<.., true>), all from btle_b200/csrc/btle_core.cuh,
// run with the same chain and decode (resolve_chunk) the other emulated passes use.  Not part of the product.
#include <algorithm>
#include <cstring>
#include <vector>

#include "../../btle_b200/csrc/btle_params.h"

using namespace btle;

// out[k] = lp_word(prev[k], cur[k], next[k])
extern "C" void emul_lp_words(const uint32_t *prev, const uint32_t *cur, const uint32_t *next, long n, uint32_t *out) {
  for (long k = 0; k < n; ++k) out[k] = lp_word(prev[k], cur[k], next[k]);
}

// floor(avg) of every int8 pair through avg_u8x4 in offset binary: out[256 (a + 128) + (b + 128)]
extern "C" void emul_lp_avg_table(int8_t *out) {
  for (int a = -128; a < 128; ++a)
    for (int b = -128; b < 128; ++b) {
      const uint32_t x = (uint32_t)(uint8_t)a ^ 0x80u, y = (uint32_t)(uint8_t)b ^ 0x80u;
      out[256 * (a + 128) + (b + 128)] = (int8_t)(uint8_t)(avg_u8x4(x, y) ^ 0x80u);
    }
}

// Phase words of groups [g0, g0 + ngroups) of one capture of n_int8 bytes at `cap` in the low-pass mode: pd[4 (g - g0) + ph]
// bit i = d[128 g + 4 i + ph].  Bytes [-lead, n_int8) of the capture are readable, every other byte reads 0.  rot: rotated
// by (c, s).
extern "C" void emul_lp_phase_words(const int8_t *cap, long n_int8, long lead, long g0, long ngroups, int rot, int c, int s, uint32_t *pd) {
  for (long g = g0; g < g0 + ngroups; ++g) {
    auto word = [&](int k) -> uint32_t {
      uint32_t w = 0;
      for (int b = 0; b < 4; ++b) {
        const long a = 256L * g + 4L * k + b;
        if (a >= -lead && a < n_int8) w |= (uint32_t)(uint8_t)cap[a] << (8 * b);
      }
      return w;
    };
    uint32_t acc[4] = {0xDEADBEEFu, 0x12345678u, 0xFFFFFFFFu, 0x80000001u};   // the walk must shift all of it out
    if (rot) dbits_group_lowpass<true>(word, c, s, acc);
    else dbits_group_lowpass<false>(word, 0, 0, acc);
    for (int ph = 0; ph < 4; ++ph) pd[4 * (g - g0) + ph] = acc[ph];
  }
}

// Records of one capture (n_int8 bytes, nothing readable in front of it) decoded with one cfg in the low-pass mode, in the
// reference's order: the dense walk over each span's groups, the prefilter, resolve_chunk per chunk, then every CRC-failed
// counted record of a cfg with BTLE_CFG_RECOVER or BTLE_CFG_CORRECT repaired as the kernel's resolver repairs it.  rot: the
// walk and recovery rotated by (c4, s4).  Returns the number of records (-1: the syndrome table cannot be built).
extern "C" long emul_lp_rx_stream(const int8_t *iq, long n_int8, const btle_stream_cfg *cfg, int stream, int rot, int c4, int s4,
                                  btle_pkt_rec *out, long cap) {
  uint8_t wrow[48];
  make_whiten_row(cfg->channel, wrow);
  uint32_t ww[12];
  memcpy(ww, wrow, 48);
  StreamParams sp;
  make_params(*cfg, ww, sp);
  uint32_t crc4[1024];
  make_crc4(crc4);
  static uint64_t syn[kSyndromeSlots];
  if (make_syndrome_table(syn) != kCorrectPatterns) return -1;
  const long nchunks = n_int8 / kChunkInt8;
  long n = 0;
  auto word_at = [&](long byte_off) -> uint32_t {
    uint32_t w = 0;
    for (int b = 0; b < 4; ++b) { const long a = byte_off + b; if (a >= 0 && a < n_int8) w |= (uint32_t)(uint8_t)iq[a] << (8 * b); }
    return w;
  };
  for (long c0 = 0; c0 < nchunks; c0 += kSpanChunks) {
    const int nch = (int)std::min<long>(kSpanChunks, nchunks - c0);
    const int G = kGroupsPerChunk * nch + kHaloGroups;
    std::vector<uint32_t> pd(4 * (size_t)(G + 1), 0u), cand((size_t)G + 1, 0u), flagw(2 * (size_t)nch, 0u);
    const long base = c0 * kChunkInt8;
    for (int g = 0; g < G; ++g) {
      uint32_t acc[4] = {0xDEADBEEFu, 0x12345678u, 0xFFFFFFFFu, 0x80000001u};
      auto word = [&](int k) { return word_at(base + 256L * g + 4L * k); };
      if (rot) dbits_group_lowpass<true>(word, c4, s4, acc);
      else dbits_group_lowpass<false>(word, 0, 0, acc);
      for (int ph = 0; ph < 4; ++ph) pd[4 * g + ph] = acc[ph];
    }
    for (int g = 0; g < kGroupsPerChunk * nch; ++g) {
      const uint32_t a = prefilter_any(&pd[4 * (size_t)g], &pd[4 * (size_t)(g + 1)], sp);
      cand[g] = a;
      if (a) flagw[g >> 5] |= 1u << (g & 31);
    }
    for (int c = 0; c < nch; ++c) {
      const long chunk = c0 + c;
      auto emit = [&](int n0, int nbytes, int crc_bad, const uint32_t words[11], bool rejected) {
        const long slot = n++;
        if (slot >= cap) return;
        uint32_t w[11];
        memcpy(w, words, sizeof w);
        uint32_t extra = 0;
        if ((sp.recover || sp.correct) && crc_bad && !rejected) {
          const IqWindow win = iq_window(iq, n_int8, chunk);
          extra = rot ? repair_packet<true, true>(win, sp, crc4, syn, n0, w, nbytes, c4, s4)
                      : repair_packet<false, true>(win, sp, crc4, syn, n0, w, nbytes);
          if (extra) crc_bad = 0;
        }
        btle_pkt_rec &r = out[slot];
        memset(&r, 0, sizeof r);
        r.stream = stream; r.chunk = (int32_t)chunk; r.n0 = n0;
        r.channel = (uint8_t)sp.channel; r.n_bytes = (uint8_t)nbytes; r.crc_bad = (uint8_t)crc_bad;
        r.flags = (uint8_t)((sp.raw ? 1 : 0) | (sp.adv ? 2 : 0) | (rejected ? BTLE_REC_REJECTED : 0) | extra);
        r.access_addr = sp.aa;
        if (sp.rssi) {
          uint32_t mag = 0;
          for (int k = 0; k < 256; ++k) {
            const long a = chunk * kChunkInt8 + 2L * n0 + k;
            const int v = (a >= 0 && a < n_int8) ? iq[a] : 0;
            mag += (uint32_t)(v < 0 ? -v : v);
          }
          r.mag_sum = (uint16_t)mag;
        }
        memcpy(r.bytes, w, 42);
      };
      resolve_chunk(&pd[4 * (size_t)(kGroupsPerChunk * c)], &cand[(size_t)kGroupsPerChunk * c], &flagw[2 * (size_t)c], sp, crc4, emit);
    }
  }
  return n;
}
