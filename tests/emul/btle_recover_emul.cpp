// Test-only CPU emulator of BTLE_CFG_RECOVER: recover_packet (btle_b200/csrc/btle_core.cuh), the function the receive
// kernel's resolver runs in steps 3b and 4, applied to records as the kernel's other passes store them.  Recovery of one
// counted record depends only on that record's (stream, chunk, n0), its cfg and the capture, so running it over the
// records of the emulated passes (tests/emul/btle_emul.cpp) gives what the kernel stores.  Not part of the product.
#include <cstring>

#include "../../btle_b200/csrc/btle_params.h"

using namespace btle;

// recs[0..n): records of captures iq + stream * stride (n_int8 each) decoded with cfgs[stream]; every CRC-failed counted
// record of a cfg with BTLE_CFG_RECOVER (not raw) is replaced by its first alternative with a good CRC, if any.  rot4:
// NULL for the unrotated bits (recover_packet<false>), else (C4, S4) of the record's capture at rot4[2 stream],
// rot4[2 stream + 1] (recover_packet<true>, carrier-offset correction).  Returns the number of records replaced.
extern "C" long emul_recover_records(const int8_t *iq, long stride, long n_int8, const btle_stream_cfg *cfgs, const int32_t *rot4,
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
    const IqWindow w = iq_window(iq + (long)r.stream * stride, n_int8, r.chunk);
    const int q = rot4 ? recover_packet<true>(w, sp, crc4, r.n0, words, nbytes, rot4[2 * r.stream], rot4[2 * r.stream + 1])
                       : recover_packet<false>(w, sp, crc4, r.n0, words, nbytes);
    if (q < 0) continue;
    memcpy(r.bytes, words, sizeof r.bytes);               // words are zero behind n_bytes (<= 42)
    r.n_bytes = (uint8_t)nbytes;
    r.crc_bad = 0;
    r.flags = (uint8_t)(r.flags | recovered_flags(q));
    ++replaced;
  }
  return replaced;
}
