// Test-only CPU emulator of discover_kernel's logic (connection discovery).  Like btle_emul.cpp it executes the SAME
// per-lane functions the sm_90a kernel uses (btle_b200/csrc/btle_core.cuh, btle_params.h — compiled here for the host),
// one lane at a time, so that the candidate rule can be checked against the numpy restatement (tests/discover_ref.py) in
// a container without a GPU.  It is NOT part of the product and nothing under btle_b200/ links it.
#include <cstring>
#include <vector>

#include "../../btle_b200/csrc/btle_params.h"

using namespace btle;

// Connection discovery on one capture, lane by lane: phase words of every group (dbits8, bytes outside the capture read
// as 0), then discover_kernel's per-group test — empty_pdu_windows / empty_pdu_inside / empty_pdu_fields / crc24_unwind
// (btle_core.cuh) — in (group, phase, window) order.  Writes btle_conn_cand records, returns how many there are.
extern "C" long emul_discover(const int8_t *iq, long n_int8, int channel, int stream, btle_conn_cand *out, long cap) {
  uint8_t wrow[48];
  make_whiten_row(channel, wrow);
  uint32_t ww[12];
  memcpy(ww, wrow, 48);
  const long n_samples = n_int8 / 2, G = n_samples / 128 + 1;
  auto word_at = [&](long byte_off) -> uint32_t {
    uint32_t w = 0;
    for (int b = 0; b < 4; ++b) { long a = byte_off + b; if (a >= 0 && a < n_int8) w |= (uint32_t)(uint8_t)iq[a] << (8 * b); }
    return w;
  };
  std::vector<uint32_t> pd(4 * (size_t)(G + 4), 0u);
  for (long g = 0; g < G; ++g) {
    uint32_t acc[4] = {0, 0, 0, 0};
    const long goff = 256L * g;
    uint32_t carry = word_at(goff + 256);
    for (int c = 15; c >= 0; --c) {
      dbits8(word_at(goff + 16 * c), word_at(goff + 16 * c + 4), word_at(goff + 16 * c + 8), word_at(goff + 16 * c + 12), carry, acc);
      carry = word_at(goff + 16 * c);
    }
    for (int ph = 0; ph < 4; ++ph) pd[4 * g + ph] = acc[ph];
  }
  long n = 0;
  for (long g = 0; g < G; ++g)
    for (int ph = 0; ph < 4; ++ph) {
      uint32_t w[5];
      for (int k = 0; k < 5; ++k) w[k] = (g - 1 + k >= 0 && g - 1 + k < G) ? pd[4 * (g - 1 + k) + ph] : 0u;
      uint32_t m = empty_pdu_windows(w, ww[0]) & empty_pdu_inside(g, ph, n_samples);
      while (m) {
        const int i = __builtin_ctz(m);
        m &= m - 1;
        uint32_t aa, header, crc_rx;
        empty_pdu_fields(w, i, ww[0], ww[1], aa, header, crc_rx);
        if (n < cap) {
          btle_conn_cand &r = out[n];
          memset(&r, 0, sizeof r);
          r.sample = 128 * g + 4 * i + ph; r.stream = stream; r.access_addr = aa;
          r.crc_init = crc_init_reorder(crc24_unwind(crc_rx, header, 16));
          r.channel = (uint8_t)channel; r.header[0] = (uint8_t)header; r.header[1] = (uint8_t)(header >> 8);
        }
        ++n;
      }
    }
  return n;
}

extern "C" uint32_t emul_crc24_unwind(uint32_t crc, uint32_t bits, int nbits) { return crc24_unwind(crc, bits, nbits); }
