// Test-only CPU emulator of BTLE_CFG_CORRECT together with BTLE_CFG_RECOVER: repair_packet (btle_b200/csrc/btle_core.cuh),
// the function the receive kernel's resolver runs in steps 3b, 3c and 4, applied to records as the kernel's other passes
// store them.  Repairing one counted record depends only on that record's (stream, chunk, n0, bytes, n_bytes), its cfg and
// the capture, so running it over the records of the emulated passes (tests/emul/btle_emul.cpp) gives what the kernel
// stores.  Also the shared syndrome table and lookup.  Not part of the product.
#include <cstring>

#include "../../btle_b200/csrc/btle_params.h"

using namespace btle;

// recs[0..n): records of captures iq + stream * stride (n_int8 each) decoded with cfgs[stream] (the emulated passes apply
// neither BTLE_CFG_RECOVER nor BTLE_CFG_CORRECT); every CRC-failed counted record of a cfg with either flag (not raw) is
// replaced as repair_packet decides, if it repairs it.  rot4: NULL for the unrotated bits (repair_packet<false>), else
// (C4, S4) of the record's capture at rot4[2 stream], rot4[2 stream + 1] (repair_packet<true>, carrier-offset
// correction).  Returns the number of records replaced, -1 if the syndrome table cannot be built.
extern "C" long emul_repair_records(const int8_t *iq, long stride, long n_int8, const btle_stream_cfg *cfgs, const int32_t *rot4,
                                    btle_pkt_rec *recs, long n) {
  uint32_t crc4[1024];
  make_crc4(crc4);
  static uint64_t syn[kSyndromeSlots];
  if (make_syndrome_table(syn) != kCorrectPatterns) return -1;
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
    if (!(sp.recover || sp.correct) || !r.crc_bad || (r.flags & BTLE_REC_REJECTED)) continue;
    uint32_t words[11] = {0};
    memcpy(words, r.bytes, sizeof r.bytes);               // the primary decode (zero behind n_bytes)
    int nbytes = r.n_bytes;
    const IqWindow w = iq_window(iq + (long)r.stream * stride, n_int8, r.chunk);
    const uint32_t extra = rot4 ? repair_packet<true>(w, sp, crc4, syn, r.n0, words, nbytes, rot4[2 * r.stream], rot4[2 * r.stream + 1])
                                : repair_packet<false>(w, sp, crc4, syn, r.n0, words, nbytes);
    if (!extra) continue;
    memcpy(r.bytes, words, sizeof r.bytes);               // words are zero behind n_bytes (<= 42)
    r.n_bytes = (uint8_t)nbytes;
    r.crc_bad = 0;
    r.flags = (uint8_t)(r.flags | extra);
    ++replaced;
  }
  return replaced;
}

// BTLE_CFG_CORRECT's table as make_syndrome_table builds it (tab[kSyndromeSlots]); returns its number of patterns
extern "C" long emul_syndrome_table(uint64_t *tab) { return make_syndrome_table(tab); }

// syndrome_lookup of every s in [s0, s0 + n): code[k] for s0 + k (-1: none)
extern "C" void emul_syndrome_lookup(uint32_t s0, long n, int16_t *code) {
  static uint64_t syn[kSyndromeSlots];
  make_syndrome_table(syn);
  for (long k = 0; k < n; ++k) code[k] = (int16_t)syndrome_lookup(syn, s0 + (uint32_t)k);
}
