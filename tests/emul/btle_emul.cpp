// Test-only CPU emulator of the CUDA kernels' logic.  It executes the SAME per-lane functions
// the sm_90a kernels use (btle_b200/csrc/btle_core.cuh, btle_params.h — compiled here for the
// host) in the same three passes the span kernel runs (phase words -> prefilter flags ->
// per-chunk resolve), one lane at a time.  It exists so that the kernel logic can be checked
// against the oracle in a container without a GPU; it is NOT part of the product and nothing
// under btle_b200/ links it.
#include <algorithm>
#include <cstring>
#include <vector>

#include "../../btle_b200/csrc/btle_params.h"

using namespace btle;

namespace {
struct HostEmit {
  btle_pkt_rec *out; long cap; long n; int stream, chunk; const StreamParams *sp;
  const int8_t *iq; long n_int8; long chunk_base_int8;
  void operator()(int n0, int nbytes, int crc_bad, const uint32_t words[11], bool rejected = false) {
    const long slot = n++;
    if (slot < cap) {
      btle_pkt_rec &r = out[slot];
      memset(&r, 0, sizeof r);
      r.stream = stream; r.chunk = chunk; r.n0 = n0;
      r.channel = (uint8_t)sp->channel; r.n_bytes = (uint8_t)nbytes; r.crc_bad = (uint8_t)crc_bad;
      r.flags = (uint8_t)((sp->raw ? 1 : 0) | (sp->adv ? 2 : 0) | (rejected ? 4 : 0));
      r.access_addr = sp->aa;
      if (sp->rssi) {
        uint32_t mag = 0;
        for (int k = 0; k < 128; ++k)
          for (int c = 0; c < 2; ++c) {
            long a = chunk_base_int8 + 2L * (n0 + k) + c;
            int v = (a >= 0 && a < n_int8) ? iq[a] : 0;
            mag += (uint32_t)(v < 0 ? -v : v);
          }
        r.mag_sum = (uint16_t)mag;
      }
      memcpy(r.bytes, words, 42);
    }
  }
};
}  // namespace

extern "C" long emul_rx_stream(const int8_t *iq, long n_int8, const btle_stream_cfg *cfg, int stream, int span_chunks,
                               btle_pkt_rec *out, long cap) {
  uint8_t wrow[48];
  make_whiten_row(cfg->channel, wrow);
  uint32_t ww[12];
  memcpy(ww, wrow, 48);
  StreamParams sp;
  make_params(*cfg, ww, sp);
  uint32_t crc4[1024];
  make_crc4(crc4);

  const long nchunks = n_int8 / kChunkInt8;
  HostEmit emit{out, cap, 0, stream, 0, &sp, iq, n_int8, 0};
  auto word_at = [&](long byte_off) -> uint32_t {   // 4 bytes little-endian, zero outside the capture
    uint32_t w = 0;
    for (int b = 0; b < 4; ++b) {
      long a = byte_off + b;
      if (a >= 0 && a < n_int8) w |= (uint32_t)(uint8_t)iq[a] << (8 * b);
    }
    return w;
  };
  for (long c0 = 0; c0 < nchunks; c0 += span_chunks) {
    const int nch = (int)std::min<long>(span_chunks, nchunks - c0);
    const int G = kGroupsPerChunk * nch + kHaloGroups;
    std::vector<uint32_t> pd(4 * (size_t)(G + 1), 0u);
    const long base = c0 * kChunkInt8;
    // pass A: one lane per group, walking its 128 samples from the end
    for (int g = 0; g < G; ++g) {
      uint32_t acc[4] = {0, 0, 0, 0};
      const long goff = base + 256L * g;
      uint32_t carry = word_at(goff + 256);
      for (int c = 15; c >= 0; --c) {
        uint32_t w0 = word_at(goff + 16 * c), w1 = word_at(goff + 16 * c + 4), w2 = word_at(goff + 16 * c + 8),
                 w3 = word_at(goff + 16 * c + 12);
        dbits8(w0, w1, w2, w3, carry, acc);
        carry = w0;
      }
      for (int ph = 0; ph < 4; ++ph) pd[4 * g + ph] = acc[ph];
    }
    // pass B: candidate words + group flags (dense warps do lanes 0..30, the resolver warp
    // fixes up lane 31 of every tile; the emulator just does all groups)
    std::vector<uint32_t> cand((size_t)G + 1, 0u);
    std::vector<uint32_t> flagw(2 * (size_t)nch, 0u);
    for (int g = 0; g < kGroupsPerChunk * nch; ++g) {
      const uint32_t a = prefilter_any(&pd[4 * (size_t)g], &pd[4 * (size_t)(g + 1)], sp);
      cand[g] = a;
      if (a) flagw[g >> 5] |= 1u << (g & 31);
    }
    // pass C: one lane per chunk
    for (int c = 0; c < nch; ++c) {
      emit.chunk = (int)(c0 + c);
      emit.chunk_base_int8 = (c0 + c) * (long)kChunkInt8;
      // a chunk sees its own 76 groups (+1); the span array continues into the next chunk, which
      // is exactly the look-ahead the reference reads (btle_rx.c:2619-2637)
      resolve_chunk(&pd[4 * (size_t)(kGroupsPerChunk * c)], &cand[(size_t)kGroupsPerChunk * c], &flagw[2 * (size_t)c], sp,
                    crc4, emit);
    }
  }
  return emit.n;
}

// The kernel's unit decomposition and resolver passes, lane by lane: Plan / unit_info (last wave cut into pieces),
// chain pass into per-chunk hit rows, exclusive prefix, the decode pass's binary search for a packet's chunk,
// one block of the output per (cfg, unit) + directory entry.  cfg i decodes capture cfg_capture[i] (non-decreasing, at most
// kMaxCfgsPerCapture per capture), or capture i when cfg_capture is NULL (then n_cfgs == n_captures).  The kernel is
// launch_rx's choice:
//   - a list that maps cfg i to capture i for every capture: btle_rx_persistent_kernel<1>, prefilter_any on the cfg's
//     StreamParams, directory entry = unit;
//   - any other list: <kMaxCfgsPerCapture>.  The plan runs over capture GROUPS (the captures some cfg names); per unit the
//     phase words are built once, the candidate words are the union of the group's cfgs' prefilters (prefilter_union on
//     make_tapset), and the resolver passes run once per cfg, directory entry cfg * (units per group) + the unit's index in
//     its group.
// flags: bit 0 permutes the order in which units reserve their block (on the GPU that is the order they finish in),
// bit 1 takes the candidate walk for every chunk.  sym: the dense pass of the symbol-spaced variant (dbits_group_sym<false>,
// launch_rx's choice for cfgs with BTLE_CFG_SYMBOL_SPACED; bytes in front of the capture read 0, as rx_batch's launch
// without a lead), else dbits_group_dense.  Records carry stream = cfg index.  Returns the number of records (one
// block per (cfg, unit), stored in reservation order), or -1 for an invalid cfg_capture, an uneven plan under
// <kMaxCfgsPerCapture> or a directory that is too small.  dir: 2 words per entry; *n_dir_out = entries written.
// Mirrors btle_rx_persistent_kernel; keep in step with it.
extern "C" long emul_rx_units(const int8_t *iq, long n_captures, long stride, long n_int8, const btle_stream_cfg *cfgs,
                              const int32_t *cfg_capture, long n_cfgs, int grid, int flags, int sym, btle_pkt_rec *out, long cap,
                              uint32_t *dir, long dir_cap, long *n_dir_out) {
  const int reverse_units = flags & 1, force_walk = (flags >> 1) & 1;
  *n_dir_out = 0;
  std::vector<int> caps, cfg0, ncfg;                       // per capture group: its capture, first cfg, number of cfgs
  for (long i = 0; i < n_cfgs; ++i) {
    const int c = cfg_capture ? cfg_capture[i] : (int)i;
    if (c < 0 || c >= n_captures || (i && c < caps.back())) return -1;
    if (!i || c != caps.back()) { caps.push_back(c); cfg0.push_back((int)i); ncfg.push_back(0); }
    if (++ncfg.back() > kMaxCfgsPerCapture) return -1;
  }
  const bool single = (long)caps.size() == n_cfgs && n_cfgs == n_captures;
  const long nchunks = n_int8 / kChunkInt8;
  if (nchunks == 0 || caps.empty()) return 0;
  const Plan pl = make_plan((long long)caps.size(), nchunks, grid);
  const int per_group = pl.big_units ? pl.spans_per_stream : pl.spans_per_stream << pl.piece_shift;
  if (!single && (pl.tail_units || (pl.big_units && pl.big_units != pl.total_units) || per_group * (long)caps.size() != pl.total_units)) return -1;
  const long n_dir = single ? pl.total_units : (long)per_group * n_cfgs;
  if (n_dir > dir_cap) return -1;
  *n_dir_out = n_dir;
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
  constexpr int kHitCap = BTLE_MAX_PKTS_PER_CHUNK + kRejectedInHitRow + 1;    // the kernel's hit row; more hits are left to step 4
  long count = 0;
  for (int uu = 0; uu < pl.total_units; ++uu) {
    const int u = reverse_units ? pl.total_units - 1 - uu : uu;
    const UnitInfo ui = unit_info(u, pl);
    const int vs = ui.stream;
    const int8_t *cap_base = iq + (long)caps[vs] * stride;
    auto word_at = [&](long byte_off) -> uint32_t {
      uint32_t w = 0;
      for (int b = 0; b < 4; ++b) { long a = byte_off + b; if (a >= 0 && a < n_int8) w |= (uint32_t)(uint8_t)cap_base[a] << (8 * b); }
      return w;
    };
    // dense pass, once per unit whatever the number of cfgs
    const int G = ui.groups;
    std::vector<uint32_t> pd(4 * (size_t)(G + 1) + 4, 0u), cand((size_t)G + 4, 0u), flagw(2 * (size_t)kSpanChunks + 2, 0u);
    const long base_off = (long)ui.chunk0 * kChunkInt8;
    for (int g = 0; g < G; ++g) {
      // the dense warps' arithmetic (one dp2a per sample, sign bits added with dp2a; btle_core.cuh) on the PTX ISA's
      // semantics of prmt / dp2a; garbage in the accumulators first: the walk must shift all of it out
      uint32_t acc[4] = {0xDEADBEEFu, 0x12345678u, 0xFFFFFFFFu, 0x80000001u};
      const long goff = base_off + 256L * g;
      auto word = [&](int k) -> uint32_t { return word_at(goff + 4L * k); };
      if (sym) dbits_group_sym<false>(word, 0, 0, acc);
      else dbits_group_dense(word, acc);
      for (int ph = 0; ph < 4; ++ph) pd[4 * g + ph] = acc[ph];
    }
    TapSet taps[kMaxCfgsPerCapture];
    for (int j = 0; !single && j < ncfg[vs]; ++j) taps[j] = make_tapset(sps[cfg0[vs] + j]);
    for (int g = 0; g < kGroupsPerChunk * ui.nch; ++g) {
      const uint32_t *lo = &pd[4 * (size_t)g], *hi = &pd[4 * (size_t)(g + 1)];
      const uint32_t a = single ? prefilter_any(lo, hi, sps[cfg0[vs]]) : prefilter_union(lo, hi, taps, ncfg[vs]);
      cand[g] = a;
      if (a) flagw[g >> 5] |= 1u << (g & 31);
    }
    // resolver passes, once per cfg
    for (int jc = 0; jc < ncfg[vs]; ++jc) {
      const int j = cfg0[vs] + jc;
      const StreamParams &sp = sps[j];
      // exact hits per flag word (lane = flag word), then the chain pass (lane = chunk) on the lists — or, for degenerate
      // masks with more matches than a list holds, on the candidate words
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
        if (c0 > kExactCap || c1 > kExactCap || force_walk)
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
      const long d = single ? u : (long)j * per_group + (u - vs * per_group);
      dir[2 * d] = (uint32_t)base; dir[2 * d + 1] = (uint32_t)total;
      for (int k = 0; k < total; ++k) {
        int c = 0;
        for (int step = kSpanChunks / 2; step >= 1; step >>= 1)
          if ((int)pre[c + step] <= k) c += step;
        if (k - (int)pre[c] >= kHitCap) continue;           // behind the chunk's row: step 4
        const int h = (int)hit[c][k - (int)pre[c]];
        const bool rej = (h & 0x8000) != 0;
        const int n0 = (h & 0x7FFF) - 124;
        uint32_t words[11];
        int nbytes, crc_bad;
        decode_packet(&pd[4 * (size_t)(kGroupsPerChunk * c)], sp, crc4, n0, rej, words, nbytes, crc_bad);
        if (base + k < cap) {
          HostEmit e{out + base + k, 1, 0, j, ui.chunk0 + c, &sp, cap_base, n_int8, (long)(ui.chunk0 + c) * kChunkInt8};
          e(n0, nbytes, crc_bad, words, rej);
        }
      }
      // step 4: a chunk with more hits than its row holds runs its chain again and stores hits kHitCap.. itself
      for (int lane = 0; lane < ui.nch; ++lane) {
        if (!sp.report_rejected || mine[lane] <= kHitCap) continue;
        const uint32_t *pdc = &pd[4 * (size_t)(kGroupsPerChunk * lane)];
        const long first = base + pre[lane];
        auto late = [&](int i, int n0, bool rej) {
          if (i < kHitCap || first + i >= cap) return;
          uint32_t words[11];
          int nbytes, crc_bad;
          decode_packet(pdc, sp, crc4, n0, rej, words, nbytes, crc_bad);
          HostEmit e{out + first + i, 1, 0, j, ui.chunk0 + lane, &sp, cap_base, n_int8, (long)(ui.chunk0 + lane) * kChunkInt8};
          e(n0, nbytes, crc_bad, words, rej);
        };
        const int c0 = xh[2 * lane][kExactCap], c1 = xh[2 * lane + 1][kExactCap];
        if (c0 > kExactCap || c1 > kExactCap || force_walk)
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

extern "C" uint32_t emul_crc24_words(const uint8_t *bytes, int n, uint32_t init) {
  uint32_t crc4[1024];
  make_crc4(crc4);
  uint32_t words[11] = {0};
  memcpy(words, bytes, (size_t)n);
  return crc24_words(words, n, init, crc4);
}

extern "C" void emul_tables(uint8_t *whiten /*40*42*/, uint32_t *crc /*256*/) {
  for (int ch = 0; ch < 40; ++ch) { uint8_t row[48]; make_whiten_row(ch, row); memcpy(whiten + 42 * ch, row, 42); }
  for (uint32_t b = 0; b < 256; ++b) crc[b] = make_crc_entry(b);
}

// Plan / unit_info alone: (stream, chunk0, nch) of every unit of a launch shape
extern "C" long emul_plan(long n_streams, long nchunks, int grid, int32_t *units /*3 per unit*/, long cap) {
  const Plan pl = make_plan(n_streams, nchunks, grid);
  if (pl.total_units > cap) return -pl.total_units;
  for (int u = 0; u < pl.total_units; ++u) {
    const UnitInfo ui = unit_info(u, pl);
    units[3 * u] = ui.stream; units[3 * u + 1] = ui.chunk0; units[3 * u + 2] = ui.nch;
  }
  return pl.total_units;
}

// The dense arithmetic of the other variants alone: carrier-offset correction (dbits_group_rot, include/btle_b200.h,
// BTLE_MAX_OFFSET_HZ) and the symbol-spaced discriminator (dbits_group_sym, BTLE_CFG_SYMBOL_SPACED), plain and rotated.
// Phase words of ngroups groups of 128 samples: words[0 .. 64 ngroups] are the capture's IQ words (one more behind the last
// group); pd[4 g + ph] bit i = d[128 g + 4 i + ph] of the rotated discriminator with (c, s).
extern "C" void emul_rot_phase_words(const uint32_t *words, long ngroups, int c, int s, uint32_t *pd) {
  for (long g = 0; g < ngroups; ++g) {
    const uint32_t *w = words + 64 * g;
    auto word = [&](int k) { return w[k]; };
    uint32_t acc[4] = {0u, 0u, 0u, 0u};
    dbits_group_rot(word, c, s, acc);
    for (int ph = 0; ph < 4; ++ph) pd[4 * g + ph] = acc[ph];
  }
}

// Phase words of groups [g0, g0 + ngroups) of one capture of n_int8 bytes at `cap`: pd[4 (g - g0) + ph] bit i =
// d[128 g + 4 i + ph].  Bytes [-lead, n_int8) of the capture are readable, every other byte reads 0.  rot: rotated by (c, s).
extern "C" void emul_sym_phase_words(const int8_t *cap, long n_int8, long lead, long g0, long ngroups, int rot, int c, int s, uint32_t *pd) {
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
    if (rot) dbits_group_sym<true>(word, c, s, acc);
    else dbits_group_sym<false>(word, 0, 0, acc);
    for (int ph = 0; ph < 4; ++ph) pd[4 * (g - g0) + ph] = acc[ph];
  }
}

// Exhaustive check of the dense loop's discriminator (btle_core.cuh, dbits8_dense) on the modelled instruction semantics:
// for every (I0, Q0, I1, Q1) in int8^4 the sign of t = dp2a(a(I0, Q0), [I1, Q1], 127) equals the sign of
// v = Q0*I1 - I0*Q1 (btle_rx.c:1533, d = v < 0 in this orientation), |t| < 2^24 (byte 3 of t is its sign: the dp4a gather),
// both halves of a word give the same a-operand, and the two gathers add exactly the two sign bits for every step index.
// Returns the number of violations.
extern "C" long emul_check_discriminator(void) {
  long bad = 0;
  for (int i0 = -128; i0 < 128; ++i0)
    for (int q0 = -128; q0 < 128; ++q0) {
      const uint32_t w_lo = (uint32_t)(uint8_t)i0 | ((uint32_t)(uint8_t)q0 << 8);          // sample in bytes 0, 1
      const uint32_t w_hi = w_lo << 16;                                                       // the same sample in bytes 2, 3
      const int a = dp_a2<0>(w_lo ^ 0x00FF00FFu);
      if (a != dp_a2<1>(w_hi ^ 0x00FF00FFu)) ++bad;
      for (int i1 = -128; i1 < 128; ++i1)
        for (int q1 = -128; q1 < 128; ++q1) {
          const uint32_t nxt = (uint32_t)(uint8_t)i1 | ((uint32_t)(uint8_t)q1 << 8);
          const int t = __dp2a_lo(a, (int)nxt, 127);
          const int v = q0 * i1 - i0 * q1;
          if ((t < 0) != (v < 0) || t != 256 * v + 127 - q1 || t >= (1 << 24) || t < -(1 << 24)) ++bad;
        }
    }
  // the same through dbits8_dense itself (what the kernel calls): samples A, B, A, B, ... -> the 8 pairs of one step alternate
  // (A, B), (B, A); A = every int8 pair, B = the edge values and a few others; all four step indices
  {
    int edge[10] = {-128, -127, -64, -1, 0, 1, 2, 63, 126, 127};
    for (int i0 = -128; i0 < 128; ++i0)
      for (int q0 = -128; q0 < 128; ++q0)
        for (int bi = 0; bi < 10; ++bi)
          for (int bq = 0; bq < 10; ++bq) {
            const int i1 = edge[bi], q1 = edge[bq];
            const uint32_t A = (uint32_t)(uint8_t)i0 | ((uint32_t)(uint8_t)q0 << 8), B = (uint32_t)(uint8_t)i1 | ((uint32_t)(uint8_t)q1 << 8);
            const uint32_t w = A | (B << 16);                       // samples A, B in one word
            const uint32_t dab = (q0 * i1 - i0 * q1) < 0, dba = (q1 * i0 - i1 * q0) < 0;
            // sample n of the step -> phase n & 3, bit 2*CM + (n >> 2); even samples are A (pair A,B), odd ones B (pair B,A)
            uint32_t a0[4] = {0, 0, 0, 0}, a1[4] = {0, 0, 0, 0}, a2[4] = {0, 0, 0, 0}, a3[4] = {0, 0, 0, 0};
            dbits8_dense<0>(w, w, w, w, w, a0);
            dbits8_dense<1>(w, w, w, w, w, a1);
            dbits8_dense<2>(w, w, w, w, w, a2);
            dbits8_dense<3>(w, w, w, w, w, a3);
            for (int ph = 0; ph < 4; ++ph) {
              const uint32_t d = (ph & 1) ? dba : dab, two = d | (d << 1);
              if (a0[ph] != two || a1[ph] != (two << 2) || a2[ph] != (two << 4) || a3[ph] != (two << 6)) ++bad;
            }
          }
  }
  // the gathers: every step index, every sign pair, accumulators with a clear low byte
  const int tv[4] = {-1, -(1 << 23), 0, (1 << 23)};
  const uint32_t accs[3] = {0u, 0xABCDEF00u, 0xFFFFFF00u};
  for (int x = 0; x < 4; ++x)
    for (int y = 0; y < 4; ++y)
      for (uint32_t acc : accs) {
        const uint32_t sx = tv[x] < 0, sy = tv[y] < 0;
        if (add_bits<0>(acc, tv[x], tv[y]) != acc + (sx << 0) + (sy << 1)) ++bad;
        if (add_bits<1>(acc, tv[x], tv[y]) != acc + (sx << 2) + (sy << 3)) ++bad;
        if (add_bits<2>(acc, tv[x], tv[y]) != acc + (sx << 4) + (sy << 5)) ++bad;
        if (add_bits<3>(acc, tv[x], tv[y]) != acc + (sx << 6) + (sy << 7)) ++bad;
        if (add_bit4<1>(add_bit4<0>(acc, tv[x]), tv[y]) != acc + (sx << 0) + (sy << 1)) ++bad;
        if (add_bit4<3>(add_bit4<2>(acc, tv[x]), tv[y]) != acc + (sx << 2) + (sy << 3)) ++bad;
        if (add_bit4<5>(add_bit4<4>(acc, tv[x]), tv[y]) != acc + (sx << 4) + (sy << 5)) ++bad;
        if (add_bit4<7>(add_bit4<6>(acc, tv[x]), tv[y]) != acc + (sx << 6) + (sy << 7)) ++bad;
      }
  return bad;
}
