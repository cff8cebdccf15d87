// Test-only CPU emulator of the multi-cfg receive path (btle_b200_rx_multi): the kernel's KC > 1 instantiation lane by
// lane, on the same btle_core.cuh / btle_params.h functions.  The plan runs over capture GROUPS (the captures some cfg
// names); per unit the phase words are built once, the candidate words are the union of the group's cfgs' prefilters
// (prefilter_union on make_tapset), and the resolver passes (exact hits, chain, prefix, decode, step 4) run once per cfg,
// each with its own block of the output and directory entry cfg * (units per group) + the unit's index in its group.
// Mirrors btle_rx_persistent_kernel<kMaxCfgsPerCapture>; keep in step with it.  Not part of the product.
#include <algorithm>
#include <cstring>
#include <vector>

#include "../../btle_b200/csrc/btle_params.h"

using namespace btle;

namespace {
void fill_rec(btle_pkt_rec &r, int stream, int chunk, int n0, int nbytes, int crc_bad, bool rej, const uint32_t words[11],
              const StreamParams &sp, const int8_t *iq, long n_int8) {
  memset(&r, 0, sizeof r);
  r.stream = stream; r.chunk = chunk; r.n0 = n0;
  r.channel = (uint8_t)sp.channel; r.n_bytes = (uint8_t)nbytes; r.crc_bad = (uint8_t)crc_bad;
  r.flags = (uint8_t)((sp.raw ? 1 : 0) | (sp.adv ? 2 : 0) | (rej ? 4 : 0));
  r.access_addr = sp.aa;
  if (sp.rssi) {
    uint32_t mag = 0;
    const long first = (long)chunk * kChunkInt8 + 2L * n0;
    for (int k = 0; k < 256; ++k) { const long a = first + k; const int v = (a >= 0 && a < n_int8) ? iq[a] : 0; mag += (uint32_t)(v < 0 ? -v : v); }
    r.mag_sum = (uint16_t)mag;
  }
  memcpy(r.bytes, words, 42);
}
}  // namespace

// Returns the number of records (stored in unit-completion order = unit order here, one block per (cfg, unit)), or -1 for an
// invalid cfg_capture / a directory that is too small.  dir: 2 words per entry; *n_dir_out = entries written.
extern "C" long emul_rx_multi_units(const int8_t *iq, long n_captures, long stride, long n_int8, const btle_stream_cfg *cfgs,
                                    const int32_t *cfg_capture, long n_cfgs, int grid, btle_pkt_rec *out, long cap, uint32_t *dir,
                                    long dir_cap, long *n_dir_out) {
  *n_dir_out = 0;
  std::vector<int> caps, cfg0, ncfg;
  for (long i = 0; i < n_cfgs; ++i) {
    if (cfg_capture[i] < 0 || cfg_capture[i] >= n_captures || (i && cfg_capture[i] < cfg_capture[i - 1])) return -1;
    if (!i || cfg_capture[i] != cfg_capture[i - 1]) { caps.push_back(cfg_capture[i]); cfg0.push_back((int)i); ncfg.push_back(0); }
    if (++ncfg.back() > kMaxCfgsPerCapture) return -1;
  }
  const long nchunks = n_int8 / kChunkInt8;
  if (nchunks == 0 || caps.empty()) return 0;
  const Plan pl = make_plan((long long)caps.size(), nchunks, grid);
  const int per_group = pl.big_units ? pl.spans_per_stream : pl.spans_per_stream << pl.piece_shift;
  if (pl.tail_units || (pl.big_units && pl.big_units != pl.total_units) || per_group * (long)caps.size() != pl.total_units) return -1;
  if ((long)per_group * n_cfgs > dir_cap) return -1;
  *n_dir_out = (long)per_group * n_cfgs;
  std::vector<StreamParams> sps(n_cfgs);
  for (long i = 0; i < n_cfgs; ++i) {
    uint8_t wrow[48];
    make_whiten_row(cfgs[i].channel, wrow);
    uint32_t ww[12];
    memcpy(ww, wrow, 48);
    make_params(cfgs[i], ww, sps[i]);
  }
  uint32_t crc4[1024];
  make_crc4(crc4);
  constexpr int kHitCap = BTLE_MAX_PKTS_PER_CHUNK + kRejectedInHitRow + 1;
  long count = 0;
  for (int u = 0; u < pl.total_units; ++u) {
    const UnitInfo ui = unit_info(u, pl);
    const int vs = ui.stream;
    const int8_t *cap_base = iq + (long)caps[vs] * stride;
    auto word_at = [&](long off) -> uint32_t {
      uint32_t w = 0;
      for (int b = 0; b < 4; ++b) { const long a = off + b; if (a >= 0 && a < n_int8) w |= (uint32_t)(uint8_t)cap_base[a] << (8 * b); }
      return w;
    };
    // dense pass, once per unit whatever the number of cfgs
    const int G = ui.groups;
    std::vector<uint32_t> pd(4 * (size_t)(G + 1) + 4, 0u), cand((size_t)G + 4, 0u), flagw(2 * (size_t)kSpanChunks + 2, 0u);
    const long base_off = (long)ui.chunk0 * kChunkInt8;
    for (int g = 0; g < G; ++g) {
      uint32_t acc[4] = {0xDEADBEEFu, 0x12345678u, 0xFFFFFFFFu, 0x80000001u};
      const long goff = base_off + 256L * g;
      auto word = [&](int k) -> uint32_t { return word_at(goff + 4L * k); };
      dbits_group_dense(word, acc);
      for (int ph = 0; ph < 4; ++ph) pd[4 * g + ph] = acc[ph];
    }
    TapSet taps[kMaxCfgsPerCapture];
    for (int j = 0; j < ncfg[vs]; ++j) taps[j] = make_tapset(sps[cfg0[vs] + j]);
    for (int g = 0; g < kGroupsPerChunk * ui.nch; ++g) {
      const uint32_t a = prefilter_union(&pd[4 * (size_t)g], &pd[4 * (size_t)(g + 1)], taps, ncfg[vs]);
      cand[g] = a;
      if (a) flagw[g >> 5] |= 1u << (g & 31);
    }
    // resolver passes, once per cfg
    for (int jc = 0; jc < ncfg[vs]; ++jc) {
      const int j = cfg0[vs] + jc;
      const StreamParams &sp = sps[j];
      uint16_t xh[2 * kSpanChunks][kExactCap + 1];
      for (int t = 0; t < 2 * ui.nch; ++t) xh[t][kExactCap] = (uint16_t)enumerate_exact_hits(pd.data(), cand.data(), flagw[t], t, sp, xh[t]);
      uint16_t hit[kSpanChunks][kHitCap];
      int mine[32] = {0};
      for (int lane = 0; lane < ui.nch; ++lane) {
        struct Note {
          uint16_t *row;
          void operator()(int i, int n0, bool rej) { if (i < kHitCap) row[i] = (uint16_t)((n0 + 124) | (rej ? 0x8000 : 0)); }
        } note{hit[lane]};
        const uint32_t *pdc = &pd[4 * (size_t)(kGroupsPerChunk * lane)];
        const int c0 = xh[2 * lane][kExactCap], c1 = xh[2 * lane + 1][kExactCap];
        if (c0 > kExactCap || c1 > kExactCap)
          mine[lane] = chain_chunk(pdc, &cand[(size_t)kGroupsPerChunk * lane], &flagw[2 * (size_t)lane], sp, note);
        else
          mine[lane] = chain_chunk_lists(pdc, xh[2 * lane], c0, xh[2 * lane + 1], c1, sp, note);
      }
      uint16_t pre[kSpanChunks + 2];
      int incl = 0;
      for (int lane = 0; lane <= kSpanChunks; ++lane) { pre[lane] = (uint16_t)incl; incl += mine[lane]; }
      const int total = incl;
      const long base = count;
      count += total;
      const long d = (long)j * per_group + (u - vs * per_group);
      dir[2 * d] = (uint32_t)base; dir[2 * d + 1] = (uint32_t)total;
      for (int k = 0; k < total; ++k) {
        int c = 0;
        for (int step = kSpanChunks / 2; step >= 1; step >>= 1)
          if ((int)pre[c + step] <= k) c += step;
        if (k - (int)pre[c] >= kHitCap) continue;
        const int h = (int)hit[c][k - (int)pre[c]];
        const bool rej = (h & 0x8000) != 0;
        const int n0 = (h & 0x7FFF) - 124;
        uint32_t words[11];
        int nbytes, crc_bad;
        decode_packet(&pd[4 * (size_t)(kGroupsPerChunk * c)], sp, crc4, n0, rej, words, nbytes, crc_bad);
        if (base + k < cap) fill_rec(out[base + k], j, ui.chunk0 + c, n0, nbytes, crc_bad, rej, words, sp, cap_base, n_int8);
      }
      for (int lane = 0; lane < ui.nch; ++lane) {          // step 4
        if (!sp.report_rejected || mine[lane] <= kHitCap) continue;
        const uint32_t *pdc = &pd[4 * (size_t)(kGroupsPerChunk * lane)];
        const long first = base + pre[lane];
        auto late = [&](int i, int n0, bool rej) {
          if (i < kHitCap || first + i >= cap) return;
          uint32_t words[11];
          int nbytes, crc_bad;
          decode_packet(pdc, sp, crc4, n0, rej, words, nbytes, crc_bad);
          fill_rec(out[first + i], j, ui.chunk0 + lane, n0, nbytes, crc_bad, rej, words, sp, cap_base, n_int8);
        };
        const int c0 = xh[2 * lane][kExactCap], c1 = xh[2 * lane + 1][kExactCap];
        if (c0 > kExactCap || c1 > kExactCap)
          chain_chunk(pdc, &cand[(size_t)kGroupsPerChunk * lane], &flagw[2 * (size_t)lane], sp, late);
        else
          chain_chunk_lists(pdc, xh[2 * lane], c0, xh[2 * lane + 1], c1, sp, late);
      }
    }
  }
  return count;
}

// prefilter_union of one cfg against prefilter_any of its StreamParams, for every (lo, hi) pair of the given words
extern "C" long emul_check_tapset(const btle_stream_cfg *cfg, const uint32_t *words, long n) {
  uint8_t wrow[48];
  make_whiten_row(cfg->channel, wrow);
  uint32_t ww[12];
  memcpy(ww, wrow, 48);
  StreamParams sp;
  make_params(*cfg, ww, sp);
  const TapSet ts = make_tapset(sp);
  long bad = 0;
  for (long i = 0; i + 8 <= n; i += 4)
    if (prefilter_union(words + i, words + i + 4, &ts, 1) != prefilter_any(words + i, words + i + 4, sp)) ++bad;
  return bad;
}
