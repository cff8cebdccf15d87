// Test-only CPU emulator of the carrier-offset correction (include/btle_b200.h, BTLE_MAX_OFFSET_HZ): the rotated dense
// arithmetic the receive kernel's dense warps run (dbits_group_rot, btle_b200/csrc/btle_core.cuh, with the PTX-semantics
// models of prmt / dp2a) and the rotated recovery step (recover_packet<true>).  Not part of the product.
#include <cstring>

#include "../../btle_b200/csrc/btle_params.h"

using namespace btle;

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

// emul_recover_records (btle_recover_emul.cpp) with the symbol-spaced bits rotated by rot4[2 stream], rot4[2 stream + 1]
// = (C4, S4) of the record's capture.
extern "C" long emul_recover_records_rot(const int8_t *iq, long stride, long n_int8, const btle_stream_cfg *cfgs, const int32_t *rot4,
                                         btle_pkt_rec *recs, long n) {
  uint32_t crc4[1024];
  make_crc4(crc4);
  long replaced = 0;
  for (long k = 0; k < n; ++k) {
    btle_pkt_rec &r = recs[k];
    const btle_stream_cfg &cfg = cfgs[r.stream];
    uint8_t wrow[48];
    make_whiten_row(cfg.channel, wrow);
    uint32_t ww[12];
    memcpy(ww, wrow, 48);
    StreamParams sp;
    make_params(cfg, ww, sp);
    if (!sp.recover || !r.crc_bad || (r.flags & BTLE_REC_REJECTED)) continue;
    uint32_t words[11];
    int nbytes = r.n_bytes;
    const int q = recover_packet<true>(iq_window(iq + (long)r.stream * stride, n_int8, r.chunk), sp, crc4, r.n0, words, nbytes,
                                       rot4[2 * r.stream], rot4[2 * r.stream + 1]);
    if (q < 0) continue;
    memcpy(r.bytes, words, sizeof r.bytes);
    r.n_bytes = (uint8_t)nbytes;
    r.crc_bad = 0;
    r.flags = (uint8_t)(r.flags | recovered_flags(q));
    ++replaced;
  }
  return replaced;
}
