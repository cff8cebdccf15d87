// Test-only CPU emulator of the symbol-spaced discriminator (BTLE_CFG_SYMBOL_SPACED, include/btle_b200.h): the dense
// arithmetic the receive kernel's dense warps run in that mode (dbits8_sym / dbits8_sym_rot through dbits_group_sym,
// btle_b200/csrc/btle_core.cuh, with the PTX-semantics models of prmt / dp2a), and the unit path of btle_emul.cpp with that
// dense pass (emul_rx_units_sym).  Not part of the product.
#include "../../btle_b200/csrc/btle_params.h"

// emul_rx_units_sym: btle_emul.cpp's emul_rx_units, compiled once more with its dense walk replaced by the symbol-spaced
// one (its word() reads 0 outside the capture, as rx_batch's launch: no lead)
#define dbits_group_dense(word, acc) dbits_group_sym<false>(word, 0, 0, acc)
#define emul_rx_units emul_rx_units_sym
#include "btle_emul.cpp"
#undef emul_rx_units
#undef dbits_group_dense

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
