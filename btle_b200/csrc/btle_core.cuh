// btle_core.cuh — per-lane arithmetic of the BLE receive path, written once and used by the
// sm_90a kernels (btle_rx_kernels.cu).  Everything here is `__host__ __device__` so that the
// exact same logic can also be executed lane-by-lane on a CPU by the test-only emulator
// (tests/emul/), which is how the kernels are debugged in a container without a GPU.  The
// product never runs this on the host.
//
// Data model (DESIGN.md §3).  An IQ capture is cut the way the reference's main() cuts its ring
// buffer (btle_rx.c:2619-2651): chunks of 8192 IQ samples, each decoded independently with a
// 1504-sample look-ahead.  A lane owns one GROUP = 128 consecutive samples = 32 symbols x 4
// sample phases and turns it into four 32-bit PHASE WORDS:
//     pd[g][ph] bit i  =  d[128 g + 4 i + ph],   d[n] = (I[n] Q[n+1] - I[n+1] Q[n]) > 0
// (btle_rx.c:1502,1533).  In that layout the 32 taps of the access-address correlator
// (search_unique_bits, btle_rx.c:1510-1562: stride-4 samples) and the bits of a packet
// (demod_byte, :1489-1508: stride-4 samples) are CONTIGUOUS bits of one phase stream, so
// matching and decoding are funnel shifts on words.
#pragma once
#include <stdint.h>

#include "../../include/btle_b200.h"

#if defined(__CUDACC__)
#define BTLE_HD __host__ __device__ __forceinline__
#define BTLE_HDM __host__ __device__ __forceinline__   // member functions
#else
#define BTLE_HD static inline
#define BTLE_HDM inline
#endif

namespace btle {

constexpr int kChunkSamples = 8192;        // LEN_BUF_IN_SAMPLE/2, btle_rx.c:223
constexpr int kChunkInt8 = 16384;
constexpr int kGroupSamples = 128;
constexpr int kGroupsPerChunk = 64;
constexpr int kHaloGroups = 12;            // 1536 samples >= 1504 look-ahead (btle_rx.c:237-238)
constexpr int kWinGroups = kGroupsPerChunk + kHaloGroups;   // 76 groups = 9728 samples >= 9696
constexpr int kWinInt8 = 19392;            // demod_buf_len, btle_rx.c:2193
constexpr int kSearchInt8 = 16632;         // buf_len given by main(): 248+16384, btle_rx.c:2651
#ifndef BTLE_MAX_TAPS
#define BTLE_MAX_TAPS 12
#endif
constexpr int kMaxTaps = BTLE_MAX_TAPS;    // prefilter taps of the dense pass
constexpr int kTapsOne = (2 * kMaxTaps) / 3;   // taps taken from the 1-bits of the access address when it has enough

// How one launch is cut into UNITS of work (a unit = what one ring slot holds and one resolver pass decodes).
// Units [0, big_units) are whole SPANS of kSpanChunks chunks of one capture, in (stream, chunk) order; the spans
// behind them are cut into 2^piece_shift pieces of `piece` chunks each (used for inputs with fewer spans than SMs,
// so that a small capture still spreads over the GPU).  Unit order == (stream, chunk) order == the order the
// reference emits packets in.
constexpr int kSpanChunks = 16;
struct Plan {
  int spans_per_stream, nchunks;     // 16-chunk spans per capture, chunks per capture
  int big_units, total_units;
  int piece_shift, piece;            // pieces per span = 1 << piece_shift, chunks per piece = kSpanChunks >> piece_shift
  // balanced last wave (tail_units > 0): the chunks behind the last full wave of spans, all inside capture `tail_stream`,
  // are dealt as tail_units units of tail_base (+1 for the first tail_rem) chunks, one per CTA
  int tail_units, tail_stream, tail_start, tail_base, tail_rem;
};
struct UnitInfo {
  int stream, chunk0, nch;           // nch may be 0 (a piece behind the end of a ragged capture): nothing to do
  int groups, tiles;
};
BTLE_HD UnitInfo unit_info(int u, const Plan &pl) {
  UnitInfo s;
  if (pl.tail_units > 0 && u >= pl.big_units) {
    const int j = u - pl.big_units;
    s.stream = pl.tail_stream;
    s.chunk0 = pl.tail_start + j * pl.tail_base + (j < pl.tail_rem ? j : pl.tail_rem);
    s.nch = pl.tail_base + (j < pl.tail_rem ? 1 : 0);
  } else {
    int span, sub = 0, len = kSpanChunks;
    if (u < pl.big_units) span = u;
    else {
      const int j = u - pl.big_units;
      span = pl.big_units + (j >> pl.piece_shift);
      sub = (j & ((1 << pl.piece_shift) - 1)) * pl.piece;
      len = pl.piece;
    }
    s.stream = span / pl.spans_per_stream;
    s.chunk0 = (span - s.stream * pl.spans_per_stream) * kSpanChunks + sub;
    int nch = pl.nchunks - s.chunk0;
    if (nch > len) nch = len;
    if (nch < 0) nch = 0;
    s.nch = nch;
  }
  s.groups = s.nch ? kGroupsPerChunk * s.nch + kHaloGroups : 0;
  s.tiles = (s.groups + 31) >> 5;
  return s;
}
// grid = number of persistent CTAs that will share the units round-robin
BTLE_HD Plan make_plan(long long n_streams, long long nchunks, int grid) {
  Plan pl;
  pl.nchunks = (int)nchunks;
  pl.spans_per_stream = (int)((nchunks + kSpanChunks - 1) / kSpanChunks);
  pl.tail_units = pl.tail_stream = pl.tail_start = pl.tail_base = pl.tail_rem = 0;
  const long long total = (long long)pl.spans_per_stream * n_streams;
  // Whole spans whenever there is at least one per CTA.  (Cutting the last wave into 4-chunk pieces does not pay: a small
  // unit still costs a resolver warp its full latency and drags its own 12-group look-ahead tile through a warp with 12 of
  // 32 lanes busy.)
  // Small inputs are cut into pieces so that they spread over more SMs.
  long long big = total;
  pl.piece_shift = 0;
#ifdef BTLE_SPLIT_LAST_WAVE                              // (A/B builds only)
  if (grid > 0 && total < 96ll * grid) { big = (total / grid - 1) * grid; if (big < 0) big = 0; pl.piece_shift = 2; }
#endif
  if (grid > 0 && total < grid) {
    big = 0;
    pl.piece_shift = (4 * total >= grid) ? 2 : 4;        // pieces of 4 chunks; single chunks for tiny inputs
  }
  pl.piece = kSpanChunks >> pl.piece_shift;
  pl.big_units = (int)big;
  pl.total_units = (int)(big + ((total - big) << pl.piece_shift));
#ifdef BTLE_BALANCED_TAIL                                 // NOT the default (see below)
  // Balanced last wave.  With few waves (one 1 GiB capture: 31 spans per CTA on 132 SMs) the CTAs that hold one span more
  // than the others finish ~one span later.  Here the spans behind the last FULL wave are re-cut into one unit per CTA of equal size
  // (+-1 chunk) — still in chunk order, still <= 16 chunks, one look-ahead tile per unit as before — when they all belong
  // to one capture.  An isolated launch gains from it, but back-to-back launches lose: with the uneven deal the CTAs that
  // hold one span fewer retire early and the next launch's CTAs start on their SMs while the others finish — its start-up
  // and this launch's resolver tail overlap; with an even deal everything ends, and starts, at once.  Throughput of a
  // stream of captures is what matters, so the uneven deal stays.
  if (grid > 0 && total >= grid && total < 96ll * grid && total % grid != 0) {
    const long long first = (total / grid) * grid;                       // first span of the partial wave
    const long long st = first / pl.spans_per_stream;
    if (st == (total - 1) / pl.spans_per_stream) {                        // the partial wave lies inside one capture
      const long long start = (first - st * pl.spans_per_stream) * kSpanChunks;
      const long long T = nchunks - start;                                // chunks to deal
      const long long units = T < grid ? T : grid;
      if (T > 0 && (T + units - 1) / units <= kSpanChunks) {
        pl.big_units = (int)first;
        pl.tail_units = (int)units;
        pl.tail_stream = (int)st;
        pl.tail_start = (int)start;
        pl.tail_base = (int)(T / units);
        pl.tail_rem = (int)(T % units);
        pl.total_units = (int)(first + units);
        pl.piece_shift = 0;
        pl.piece = kSpanChunks;
      }
    }
  }
#endif
  return pl;
}

// Per-stream parameters, derived on the host from btle_stream_cfg (see make_params()).
struct StreamParams {
  uint32_t aa;                // -a, bit p = p-th received AA bit (uint32_to_bit_array, :798)
  uint32_t mask;              // -m
  uint32_t crc_init;          // crc_init_reorder(-k), :1969
  int32_t channel;
  int32_t raw;                // -r
  int32_t adv;                // channel in {37,38,39}, :2202
  int32_t rssi;               // -R
  int16_t report_rejected;    // -v: hits the reference drops for their ADV length (:2291-2298) are reported too (not counted)
  int16_t centre_hits;        // BTLE_CFG_CENTRE_HITS: the chain moves each full-window hit to the centre of its run (centre_hit)
  int16_t recover;            // BTLE_CFG_RECOVER and not raw: CRC-failed counted packets are demodulated again (recover_packet)
  int16_t correct;            // BTLE_CFG_CORRECT and not raw: CRC-failed counted packets are corrected by syndrome (repair_packet)
  int32_t tz;                // min(31, index of lowest set bit of aa&mask (32 if none))
  int32_t ntaps;              // 0 => every group is flagged (mask == 0)
  int32_t typed;              // 1 => taps [0, kTapsOne) expect a 1 and taps [kTapsOne, kMaxTaps) expect a 0
  uint32_t tap_pos[kMaxTaps]; // prefilter tap positions p (mask bit set), padded by repetition
  uint32_t tap_xor[kMaxTaps]; // 0 if aa bit p is 1, ~0 if it is 0
  uint32_t whiten[12];        // scramble_table[channel][0..41] packed little-endian (+pad)
};
static_assert(sizeof(StreamParams) == 192, "a resolver warp loads a StreamParams with one coalesced load (load_params_warp)");

BTLE_HD uint32_t funnel_r(uint32_t lo, uint32_t hi, uint32_t s) {
#if defined(__CUDA_ARCH__)
  return __funnelshift_r(lo, hi, s);
#else
  s &= 31;
  return s ? ((lo >> s) | (hi << (32 - s))) : lo;
#endif
}

// (acc << 1) | (v < 0)
BTLE_HD uint32_t push_sign(uint32_t acc, int v) {
#if defined(__CUDA_ARCH__)
  return __funnelshift_l((uint32_t)v, acc, 1);
#else
  return (acc << 1) | ((uint32_t)v >> 31);
#endif
}

// sign-extended byte K of w
template <int K>
BTLE_HD int sext8(uint32_t w) {
#if defined(__CUDA_ARCH__)
  int r;
  // prmt default mode: selector nibble bit3 = replicate the sign of the selected byte
  asm("prmt.b32 %0, %1, 0, %2;" : "=r"(r) : "r"(w), "n"(K | ((8 | K) << 4) | ((8 | K) << 8) | ((8 | K) << 12)));
  return r;
#else
  return (int)(int8_t)(w >> (8 * K));
#endif
}

// Discriminator bits of 8 consecutive samples held in w[0..3] (2 samples per word: I,Q,I,Q) plus
// the first sample of `wnext`; pushes them, LAST sample first, into the four phase accumulators
// so that after the caller has walked a group from its end to its start bit i of acc[ph] is
// d[4i+ph].  v = Q0*I1 - I0*Q1 = -(I0*Q1 - I1*Q0): d = 1  <=>  v < 0  (strict, btle_rx.c:1533).
//
// Device form (PRMT/SHF/LOP3 issue on one pipe, IMAD/IDP on another, tools/pipe_probe.cu; the ALU
// pipe is the one to unload): per sample ONE
// byte-permute builds a = [sext16(Q0) | sext16(~I0)] from the word with its I bytes complemented;
// IDP.2A against the RAW bytes [I1, Q1] of the next sample (half-word select is free) gives
// Q0*I1 + (~I0)*Q1 = v - Q1, and the missing Q1 comes from a second IDP.2A with the constant
// a = [0 | 1] chained through the accumulator — exact for every int8 input, I0 = -128 included.
#if defined(__CUDA_ARCH__)
template <int HALF>   // a-operand of the sample in bytes (2*HALF, 2*HALF+1) of the I-complemented word
__device__ __forceinline__ int dp_a(uint32_t wc) {
  int r;
  // selector nibbles, low to high: Q byte, sign(Q), ~I byte, sign(~I)
  asm("prmt.b32 %0, %1, 0, %2;" : "=r"(r) : "r"(wc), "n"(HALF ? 0xA2B3 : 0x8091));
  return r;
}
__device__ __forceinline__ int dp_lo(int a, uint32_t b) { return __dp2a_lo(a, (int)b, __dp2a_lo(0x00010000, (int)b, 0)); }
__device__ __forceinline__ int dp_hi(int a, uint32_t b) { return __dp2a_hi(a, (int)b, __dp2a_hi(0x00010000, (int)b, 0)); }
#endif
BTLE_HD void dbits8(uint32_t w0, uint32_t w1, uint32_t w2, uint32_t w3, uint32_t wnext, uint32_t acc[4]) {
#if defined(__CUDA_ARCH__)
  const uint32_t c0 = w0 ^ 0x00FF00FFu, c1 = w1 ^ 0x00FF00FFu, c2 = w2 ^ 0x00FF00FFu, c3 = w3 ^ 0x00FF00FFu;
  acc[3] = push_sign(acc[3], dp_lo(dp_a<1>(c3), wnext));
  acc[2] = push_sign(acc[2], dp_hi(dp_a<0>(c3), w3));
  acc[1] = push_sign(acc[1], dp_lo(dp_a<1>(c2), w3));
  acc[0] = push_sign(acc[0], dp_hi(dp_a<0>(c2), w2));
  acc[3] = push_sign(acc[3], dp_lo(dp_a<1>(c1), w2));
  acc[2] = push_sign(acc[2], dp_hi(dp_a<0>(c1), w1));
  acc[1] = push_sign(acc[1], dp_lo(dp_a<1>(c0), w1));
  acc[0] = push_sign(acc[0], dp_hi(dp_a<0>(c0), w0));
#else
  const int i0 = sext8<0>(w0), q0 = sext8<1>(w0), i1 = sext8<2>(w0), q1 = sext8<3>(w0);
  const int i2 = sext8<0>(w1), q2 = sext8<1>(w1), i3 = sext8<2>(w1), q3 = sext8<3>(w1);
  const int i4 = sext8<0>(w2), q4 = sext8<1>(w2), i5 = sext8<2>(w2), q5 = sext8<3>(w2);
  const int i6 = sext8<0>(w3), q6 = sext8<1>(w3), i7 = sext8<2>(w3), q7 = sext8<3>(w3);
  const int i8 = sext8<0>(wnext), q8 = sext8<1>(wnext);
  acc[3] = push_sign(acc[3], q7 * i8 - i7 * q8);
  acc[2] = push_sign(acc[2], q6 * i7 - i6 * q7);
  acc[1] = push_sign(acc[1], q5 * i6 - i5 * q6);
  acc[0] = push_sign(acc[0], q4 * i5 - i4 * q5);
  acc[3] = push_sign(acc[3], q3 * i4 - i3 * q4);
  acc[2] = push_sign(acc[2], q2 * i3 - i2 * q3);
  acc[1] = push_sign(acc[1], q1 * i2 - i1 * q2);
  acc[0] = push_sign(acc[0], q0 * i1 - i0 * q1);
#endif
}

// The dense loop's form of dbits8() (one IDP.2A per sample, sign bits gathered on the IDP pipe instead of the ALU pipe).
//   v:  a = [Q0 << 8 | ((~I0) << 8 | 0xFF)] as two signed half-words, b = raw [I1, Q1], accumulator 127:
//       t = 256*Q0*I1 + (256*(~I0) + 255)*Q1 + 127 = 256*v + (127 - Q1), and 0 <= 127 - Q1 <= 255, so t < 0 <=> v < 0
//       for every int8 input (|256 v| < 2^24).
//   bits: the two samples of one phase in this call (bits 2c, 2c+1 of the phase word, c = call index inside the group)
//       become a = [sign16(t_lo) | sign16(t_hi)] = [-1 or 0 | -1 or 0] with one byte-permute, and IDP.2A against
//       [-2^(2c%8), -2^(2c%8+1)] adds their bits into the phase word's current byte; CM = c % 4; the caller shifts
//       the four words left by 8 before the calls with CM == 3 (it walks the group from its end).
// Under nvcc the primitives are the instructions; for the CPU emulator (tests/emul, g++) they are the PTX ISA's published
// semantics of prmt.b32 (default mode) / dp2a / dp4a, so the emulator tests run this very arithmetic against the oracle.
#if defined(__CUDACC__)
#define BTLE_DENSE __device__ __forceinline__
template <int HALF>
__device__ __forceinline__ int dp_a2(uint32_t wc) {
  int r;
  // result bytes, low to high: 0x00, Q, 0xFF, ~I   (second source 0x0000FF00: byte 4 = 0x00, byte 5 = 0xFF)
  asm("prmt.b32 %0, %1, %2, %3;" : "=r"(r) : "r"(wc), "r"(0x0000FF00u), "n"(HALF ? 0x2534 : 0x0514));
  return r;
}
__device__ __forceinline__ int sign_pair(int t_lo, int t_hi) {
  int r;
  asm("prmt.b32 %0, %1, %2, %3;" : "=r"(r) : "r"(t_lo), "r"(t_hi), "n"(0xFFBB));
  return r;
}
#else
#define BTLE_DENSE inline
// prmt.b32 d, a, b, c (default mode): result byte i = byte (c >> 4i) & 7 of {b, a}, or that byte's sign replicated if bit 3 of the nibble is set
inline uint32_t prmt_b32(uint32_t a, uint32_t b, uint32_t sel) {
  const uint64_t src = ((uint64_t)b << 32) | a;
  uint32_t r = 0;
  for (int i = 0; i < 4; ++i) {
    const uint32_t n = (sel >> (4 * i)) & 0xFu;
    uint32_t byte = (uint32_t)(src >> (8 * (n & 7u))) & 0xFFu;
    if (n & 8u) byte = (byte & 0x80u) ? 0xFFu : 0x00u;
    r |= byte << (8 * i);
  }
  return r;
}
// dp2a.{lo,hi}.s32.s32: c + a.lo16 * b.byte{0|2} + a.hi16 * b.byte{1|3}  (all signed);  dp4a.s32.s32: c + sum of the four signed byte products
inline int idp2a_model(int a, int b, int c, int hi) {
  const int a0 = (int16_t)(uint16_t)((uint32_t)a & 0xFFFFu), a1 = (int16_t)(uint16_t)((uint32_t)a >> 16);
  const int b0 = (int8_t)(uint8_t)((uint32_t)b >> (hi ? 16 : 0)), b1 = (int8_t)(uint8_t)((uint32_t)b >> (hi ? 24 : 8));
  return (int)((uint32_t)c + (uint32_t)(a0 * b0) + (uint32_t)(a1 * b1));
}
inline int __dp2a_lo(int a, int b, int c) { return idp2a_model(a, b, c, 0); }
inline int __dp2a_hi(int a, int b, int c) { return idp2a_model(a, b, c, 1); }
inline int __dp4a(int a, int b, int c) {
  uint32_t r = (uint32_t)c;
  for (int i = 0; i < 4; ++i) r += (uint32_t)((int)(int8_t)(uint8_t)((uint32_t)a >> (8 * i)) * (int)(int8_t)(uint8_t)((uint32_t)b >> (8 * i)));
  return (int)r;
}
template <int HALF>
inline int dp_a2(uint32_t wc) { return (int)prmt_b32(wc, 0x0000FF00u, HALF ? 0x2534 : 0x0514); }
inline int sign_pair(int t_lo, int t_hi) { return (int)prmt_b32((uint32_t)t_lo, (uint32_t)t_hi, 0xFFBB); }
#endif
template <int CM>
BTLE_DENSE uint32_t add_bits(uint32_t acc, int t_lo, int t_hi) {
  const int a = sign_pair(t_lo, t_hi);
  if (CM == 0) return (uint32_t)__dp2a_lo(a, (int)0xF8FCFEFFu, (int)acc);   // bytes -1, -2
  if (CM == 1) return (uint32_t)__dp2a_hi(a, (int)0xF8FCFEFFu, (int)acc);   //       -4, -8
  if (CM == 2) return (uint32_t)__dp2a_lo(a, (int)0x80C0E0F0u, (int)acc);   //       -16, -32
  return (uint32_t)__dp2a_hi(a, (int)0x80C0E0F0u, (int)acc);                //       -64, -128
}
// Variant (-DBTLE_GATHER_4A): |t| < 2^24, so byte 3 of t is 0xFF / 0x00 = -1 / 0 as a signed byte, and IDP.4A of t itself
// against [0, 0, 0, -2^j] adds bit j without any byte-permute (one IDP per bit, nothing on the ALU pipe).
template <int J>
BTLE_DENSE uint32_t add_bit4(uint32_t acc, int t) {
  return (uint32_t)__dp4a(t, (int)((0x100u - (1u << J)) << 24), (int)acc);
}
template <int CM>
BTLE_DENSE void dbits8_dense(uint32_t w0, uint32_t w1, uint32_t w2, uint32_t w3, uint32_t wnext, uint32_t acc[4]) {
  const uint32_t c0 = w0 ^ 0x00FF00FFu, c1 = w1 ^ 0x00FF00FFu, c2 = w2 ^ 0x00FF00FFu, c3 = w3 ^ 0x00FF00FFu;
  const int t0 = __dp2a_hi(dp_a2<0>(c0), (int)w0, 127), t1 = __dp2a_lo(dp_a2<1>(c0), (int)w1, 127);
  const int t2 = __dp2a_hi(dp_a2<0>(c1), (int)w1, 127), t3 = __dp2a_lo(dp_a2<1>(c1), (int)w2, 127);
  const int t4 = __dp2a_hi(dp_a2<0>(c2), (int)w2, 127), t5 = __dp2a_lo(dp_a2<1>(c2), (int)w3, 127);
  const int t6 = __dp2a_hi(dp_a2<0>(c3), (int)w3, 127), t7 = __dp2a_lo(dp_a2<1>(c3), (int)wnext, 127);
#ifdef BTLE_GATHER_4A
  acc[0] = add_bit4<2 * CM + 1>(add_bit4<2 * CM>(acc[0], t0), t4);
  acc[1] = add_bit4<2 * CM + 1>(add_bit4<2 * CM>(acc[1], t1), t5);
  acc[2] = add_bit4<2 * CM + 1>(add_bit4<2 * CM>(acc[2], t2), t6);
  acc[3] = add_bit4<2 * CM + 1>(add_bit4<2 * CM>(acc[3], t3), t7);
#else
  acc[0] = add_bits<CM>(acc[0], t0, t4);
  acc[1] = add_bits<CM>(acc[1], t1, t5);
  acc[2] = add_bits<CM>(acc[2], t2, t6);
  acc[3] = add_bits<CM>(acc[3], t3, t7);
#endif
}
// one group (128 samples = 16 steps of 8) walked from its end, as the dense warps do it: acc[ph] bit i = d[4i + ph]
// word(k) = IQ word k of the group (k = 0..63), word(64) = first word behind it
template <class WordAt>
BTLE_DENSE void dbits_group_dense(WordAt &word, uint32_t acc[4]) {
  uint32_t carry = word(64);
#define BTLE_DENSE_STEP(C) do { const uint32_t w0 = word(4 * (C)), w1 = word(4 * (C) + 1), w2 = word(4 * (C) + 2), w3 = word(4 * (C) + 3); \
    if (((C) & 3) == 3) { acc[0] <<= 8; acc[1] <<= 8; acc[2] <<= 8; acc[3] <<= 8; } \
    dbits8_dense<(C) & 3>(w0, w1, w2, w3, carry, acc); carry = w0; } while (0)
  BTLE_DENSE_STEP(15); BTLE_DENSE_STEP(14); BTLE_DENSE_STEP(13); BTLE_DENSE_STEP(12);
  BTLE_DENSE_STEP(11); BTLE_DENSE_STEP(10); BTLE_DENSE_STEP(9); BTLE_DENSE_STEP(8);
  BTLE_DENSE_STEP(7); BTLE_DENSE_STEP(6); BTLE_DENSE_STEP(5); BTLE_DENSE_STEP(4);
  BTLE_DENSE_STEP(3); BTLE_DENSE_STEP(2); BTLE_DENSE_STEP(1); BTLE_DENSE_STEP(0);
#undef BTLE_DENSE_STEP
}

// ---- carrier-offset correction (the *_offset entry points, include/btle_b200.h) -----------------------------------------
// d[n] = C (I0 Q1 - I1 Q0) - S (I0 I1 + Q0 Q1) > 0, (C, S) = round(2^14 (cos, sin) phi).  As a sign: d = 1 <=> u < 0 with
// u = C v + S r, v = Q0 I1 - I0 Q1, r = I0 I1 + Q0 Q1.  |v|, |r| <= 2^15 and |C|, |S| <= 2^14, so |u| < 2^30: exact in int32.
BTLE_HD int rot_disc(int i0, int q0, int i1, int q1, int c, int s) { return c * (q0 * i1 - i0 * q1) + s * (i0 * i1 + q0 * q1); }
// Dense form, per sample: v as dbits8() builds it (one byte-permute of the I-complemented word, two IDP.2A against the raw
// bytes of the next sample), r from one byte-permute of the raw word ([sext16 I | sext16 Q]) and one IDP.2A, then two
// integer multiply-adds; the sign bits are gathered as in dbits8_dense (add_bits reads only the sign of u).
#if defined(__CUDACC__)
template <unsigned SEL>
__device__ __forceinline__ int prmt1(uint32_t w) {
  int r;
  asm("prmt.b32 %0, %1, 0, %2;" : "=r"(r) : "r"(w), "n"(SEL));
  return r;
}
#else
template <unsigned SEL>
inline int prmt1(uint32_t w) { return (int)prmt_b32(w, 0u, SEL); }
#endif
// u of the sample in bytes (2 HALF, 2 HALF + 1) of w (wc = w with its I bytes complemented); b holds the next sample in
// its bytes (0, 1) when HALF is 1 and (2, 3) when HALF is 0
template <int HALF>
BTLE_DENSE int rot_u(uint32_t w, uint32_t wc, uint32_t b, int c, int s) {
  const int a_im = prmt1<HALF ? 0xA2B3u : 0x8091u>(wc), a_re = prmt1<HALF ? 0xB3A2u : 0x9180u>(w);
  const int v = HALF ? __dp2a_lo(a_im, (int)b, __dp2a_lo(0x00010000, (int)b, 0)) : __dp2a_hi(a_im, (int)b, __dp2a_hi(0x00010000, (int)b, 0));
  const int r = HALF ? __dp2a_lo(a_re, (int)b, 0) : __dp2a_hi(a_re, (int)b, 0);
  return c * v + s * r;
}
template <int CM>
BTLE_DENSE void dbits8_rot(uint32_t w0, uint32_t w1, uint32_t w2, uint32_t w3, uint32_t wnext, int c, int s, uint32_t acc[4]) {
  const uint32_t c0 = w0 ^ 0x00FF00FFu, c1 = w1 ^ 0x00FF00FFu, c2 = w2 ^ 0x00FF00FFu, c3 = w3 ^ 0x00FF00FFu;
  const int t0 = rot_u<0>(w0, c0, w0, c, s), t1 = rot_u<1>(w0, c0, w1, c, s);
  const int t2 = rot_u<0>(w1, c1, w1, c, s), t3 = rot_u<1>(w1, c1, w2, c, s);
  const int t4 = rot_u<0>(w2, c2, w2, c, s), t5 = rot_u<1>(w2, c2, w3, c, s);
  const int t6 = rot_u<0>(w3, c3, w3, c, s), t7 = rot_u<1>(w3, c3, wnext, c, s);
  acc[0] = add_bits<CM>(acc[0], t0, t4);
  acc[1] = add_bits<CM>(acc[1], t1, t5);
  acc[2] = add_bits<CM>(acc[2], t2, t6);
  acc[3] = add_bits<CM>(acc[3], t3, t7);
}
// dbits_group_dense() with the rotated discriminator
template <class WordAt>
BTLE_DENSE void dbits_group_rot(WordAt &word, int c, int s, uint32_t acc[4]) {
  uint32_t carry = word(64);
  for (int C = 15; C >= 0; --C) {
    const uint32_t w0 = word(4 * C), w1 = word(4 * C + 1), w2 = word(4 * C + 2), w3 = word(4 * C + 3);
    if ((C & 3) == 3) { acc[0] <<= 8; acc[1] <<= 8; acc[2] <<= 8; acc[3] <<= 8; }
    switch (C & 3) {
      case 3: dbits8_rot<3>(w0, w1, w2, w3, carry, c, s, acc); break;
      case 2: dbits8_rot<2>(w0, w1, w2, w3, carry, c, s, acc); break;
      case 1: dbits8_rot<1>(w0, w1, w2, w3, carry, c, s, acc); break;
      default: dbits8_rot<0>(w0, w1, w2, w3, carry, c, s, acc); break;
    }
    carry = w0;
  }
}

// ---- symbol-spaced bits (BTLE_CFG_SYMBOL_SPACED, include/btle_b200.h) --------------------------------------------------
// d[n] = I[n-2] Q[n+2] - I[n+2] Q[n-2] > 0.  Samples n - 2 and n + 2 sit in the words in front of and behind sample n's word,
// at its byte position, so dbits8_dense's identity t = 256 v + (127 - Q1) carries over with the a-operand built from the
// word in front and the b-operand taken from the same half of the word behind: one byte-permute and one IDP.2A per sample.
// wprev = the IQ word in front of w0, wnext the word behind w3; the bits of the step's 8 samples go where dbits8_dense puts them.
template <int CM>
BTLE_DENSE void dbits8_sym(uint32_t wprev, uint32_t w0, uint32_t w1, uint32_t w2, uint32_t w3, uint32_t wnext, uint32_t acc[4]) {
  const uint32_t cp = wprev ^ 0x00FF00FFu, c0 = w0 ^ 0x00FF00FFu, c1 = w1 ^ 0x00FF00FFu, c2 = w2 ^ 0x00FF00FFu;
  const int t0 = __dp2a_lo(dp_a2<0>(cp), (int)w1, 127), t1 = __dp2a_hi(dp_a2<1>(cp), (int)w1, 127);
  const int t2 = __dp2a_lo(dp_a2<0>(c0), (int)w2, 127), t3 = __dp2a_hi(dp_a2<1>(c0), (int)w2, 127);
  const int t4 = __dp2a_lo(dp_a2<0>(c1), (int)w3, 127), t5 = __dp2a_hi(dp_a2<1>(c1), (int)w3, 127);
  const int t6 = __dp2a_lo(dp_a2<0>(c2), (int)wnext, 127), t7 = __dp2a_hi(dp_a2<1>(c2), (int)wnext, 127);
  acc[0] = add_bits<CM>(acc[0], t0, t4);
  acc[1] = add_bits<CM>(acc[1], t1, t5);
  acc[2] = add_bits<CM>(acc[2], t2, t6);
  acc[3] = add_bits<CM>(acc[3], t3, t7);
}
// rot_u with the second sample in the SAME half of b as the first one in w (rotated symbol-spaced bit, (c, s) = (C4, S4))
template <int HALF>
BTLE_DENSE int rot_u_sym(uint32_t w, uint32_t wc, uint32_t b, int c, int s) {
  const int a_im = prmt1<HALF ? 0xA2B3u : 0x8091u>(wc), a_re = prmt1<HALF ? 0xB3A2u : 0x9180u>(w);
  const int v = HALF ? __dp2a_hi(a_im, (int)b, __dp2a_hi(0x00010000, (int)b, 0)) : __dp2a_lo(a_im, (int)b, __dp2a_lo(0x00010000, (int)b, 0));
  const int r = HALF ? __dp2a_hi(a_re, (int)b, 0) : __dp2a_lo(a_re, (int)b, 0);
  return c * v + s * r;
}
template <int CM>
BTLE_DENSE void dbits8_sym_rot(uint32_t wprev, uint32_t w0, uint32_t w1, uint32_t w2, uint32_t w3, uint32_t wnext, int c, int s,
                               uint32_t acc[4]) {
  const uint32_t cp = wprev ^ 0x00FF00FFu, c0 = w0 ^ 0x00FF00FFu, c1 = w1 ^ 0x00FF00FFu, c2 = w2 ^ 0x00FF00FFu;
  const int t0 = rot_u_sym<0>(wprev, cp, w1, c, s), t1 = rot_u_sym<1>(wprev, cp, w1, c, s);
  const int t2 = rot_u_sym<0>(w0, c0, w2, c, s), t3 = rot_u_sym<1>(w0, c0, w2, c, s);
  const int t4 = rot_u_sym<0>(w1, c1, w3, c, s), t5 = rot_u_sym<1>(w1, c1, w3, c, s);
  const int t6 = rot_u_sym<0>(w2, c2, wnext, c, s), t7 = rot_u_sym<1>(w2, c2, wnext, c, s);
  acc[0] = add_bits<CM>(acc[0], t0, t4);
  acc[1] = add_bits<CM>(acc[1], t1, t5);
  acc[2] = add_bits<CM>(acc[2], t2, t6);
  acc[3] = add_bits<CM>(acc[3], t3, t7);
}
// one step of the symbol-spaced walk; ROT: rotated by (c, s) = (C4, S4)
template <bool ROT>
BTLE_DENSE void dbits8_sym_step(int cm, uint32_t wprev, uint32_t w0, uint32_t w1, uint32_t w2, uint32_t w3, uint32_t wnext, int c, int s,
                                uint32_t acc[4]) {
  if constexpr (ROT) {
    switch (cm) {
      case 3: dbits8_sym_rot<3>(wprev, w0, w1, w2, w3, wnext, c, s, acc); break;
      case 2: dbits8_sym_rot<2>(wprev, w0, w1, w2, w3, wnext, c, s, acc); break;
      case 1: dbits8_sym_rot<1>(wprev, w0, w1, w2, w3, wnext, c, s, acc); break;
      default: dbits8_sym_rot<0>(wprev, w0, w1, w2, w3, wnext, c, s, acc); break;
    }
  } else {
    switch (cm) {
      case 3: dbits8_sym<3>(wprev, w0, w1, w2, w3, wnext, acc); break;
      case 2: dbits8_sym<2>(wprev, w0, w1, w2, w3, wnext, acc); break;
      case 1: dbits8_sym<1>(wprev, w0, w1, w2, w3, wnext, acc); break;
      default: dbits8_sym<0>(wprev, w0, w1, w2, w3, wnext, acc); break;
    }
  }
}
// dbits_group_dense() with the symbol-spaced discriminator: word(-1) .. word(64) are read
template <bool ROT, class WordAt>
BTLE_DENSE void dbits_group_sym(WordAt &word, int c, int s, uint32_t acc[4]) {
  uint32_t carry = word(64);
  for (int C = 15; C >= 0; --C) {
    const uint32_t w0 = word(4 * C), w1 = word(4 * C + 1), w2 = word(4 * C + 2), w3 = word(4 * C + 3);
    if ((C & 3) == 3) { acc[0] <<= 8; acc[1] <<= 8; acc[2] <<= 8; acc[3] <<= 8; }
    dbits8_sym_step<ROT>(C & 3, word(4 * C - 1), w0, w1, w2, w3, carry, c, s, acc);
    carry = w0;
  }
}

// ---- low-pass in front of the symbol-spaced bits (BTLE_CFG_LOWPASS, include/btle_b200.h) ---------------------------------
// F[n] = (x[n-1] + 2 x[n] + x[n+1]) >> 2 per rail = avg(avg(x[n-1], x[n+1]), x[n]) with avg(a, b) = floor((a + b) / 2) (the
// nested floors are exact).  A signed per-byte avg is the unsigned one in offset binary (bytes XOR 0x80), and the unsigned one
// is (x & y) + (((x ^ y) >> 1) & 0x7F7F7F7F), which never carries across bytes.
BTLE_HD uint32_t avg_u8x4(uint32_t x, uint32_t y) { return (x & y) + (((x ^ y) >> 1) & 0x7F7F7F7Fu); }
// the filtered IQ word of w (samples 2k, 2k + 1) from the words in front of (wprev) and behind (wnext) it
BTLE_HD uint32_t lp_word(uint32_t wprev, uint32_t w, uint32_t wnext) {
  const uint32_t p = wprev ^ 0x80808080u, c = w ^ 0x80808080u, n = wnext ^ 0x80808080u;
  const uint32_t l = funnel_r(p, c, 16u), r = funnel_r(c, n, 16u);   // samples 2k - 1, 2k and 2k + 1, 2k + 2
  return avg_u8x4(avg_u8x4(l, r), c) ^ 0x80808080u;
}
// dbits_group_sym() on the filtered words: word(-2) .. word(65) are read
template <bool ROT, class WordAt>
BTLE_DENSE void dbits_group_lowpass(WordAt &word, int c, int s, uint32_t acc[4]) {
  auto fword = [&](int k) { return lp_word(word(k - 1), word(k), word(k + 1)); };
  dbits_group_sym<ROT>(fword, c, s, acc);
}

// Dense-pass prefilter: bit i of the result is 1 iff the window starting at symbol i of `lo`
// agrees with the access address on the (<=16) prefilter taps.  A superset of the true matches;
// the sparse pass re-checks every candidate exactly (search_from()).
BTLE_HD uint32_t prefilter(uint32_t lo, uint32_t hi, const StreamParams &sp) {
  uint32_t m = 0xFFFFFFFFu;
#pragma unroll
  for (int t = 0; t < kMaxTaps; ++t) m &= funnel_r(lo, hi, sp.tap_pos[t]) ^ sp.tap_xor[t];
  return m;
}
// Same predicate when the taps are typed (sp.typed): no per-tap XOR operand, so two taps fold into one
// three-input logic op (m & a & b, m & ~a & ~b) — 6 LOP3 instead of 12 per phase word for 8 + 4 taps.
BTLE_HD uint32_t prefilter_typed(uint32_t lo, uint32_t hi, const StreamParams &sp) {
  uint32_t m = 0xFFFFFFFFu;
#pragma unroll
  for (int t = 0; t < kTapsOne; ++t) m &= funnel_r(lo, hi, sp.tap_pos[t]);
#pragma unroll
  for (int t = kTapsOne; t < kMaxTaps; ++t) m &= ~funnel_r(lo, hi, sp.tap_pos[t]);
  return m;
}

// Candidate word of one group: bit i set iff the window starting at symbol i passed the prefilter
// on at least one of the four sample phases.
BTLE_HD uint32_t prefilter_any(const uint32_t lo[4], const uint32_t hi[4], const StreamParams &sp) {
  if (sp.typed)
    return prefilter_typed(lo[0], hi[0], sp) | prefilter_typed(lo[1], hi[1], sp) | prefilter_typed(lo[2], hi[2], sp) |
           prefilter_typed(lo[3], hi[3], sp);
  if (sp.ntaps == 0) return 0xFFFFFFFFu;               // mask == 0: every window matches
  return prefilter(lo[0], hi[0], sp) | prefilter(lo[1], hi[1], sp) | prefilter(lo[2], hi[2], sp) |
         prefilter(lo[3], hi[3], sp);
}

// ---- several access addresses on one capture (btle_b200_rx_multi) ------------------------------------------------------
// The dense pass of a capture read by up to kMaxCfgsPerCapture cfgs keeps, per cfg, only what its prefilter reads: the 12
// tap positions and their expected bits, 16 bytes instead of a whole StreamParams.  The candidate word of a group is the
// OR of the cfgs' candidate words, so it stays a superset of every cfg's exact matches; the resolver re-checks each
// candidate exactly against each cfg's own access address and mask.
constexpr int kMaxCfgsPerCapture = 8;      // BTLE_MAX_CFGS_PER_CAPTURE
struct TapSet {
  uint32_t pos[3];                         // byte t (t = 0..11) = tap_pos[t]
  uint32_t flags;                          // bit t: tap t expects a 0 (tap_xor[t] == ~0); kTapsAll: every window passes (mask 0)
};
constexpr uint32_t kTapsAll = 1u << 16;
BTLE_HD TapSet make_tapset(const StreamParams &sp) {
  TapSet ts;
  ts.pos[0] = ts.pos[1] = ts.pos[2] = 0u;
  ts.flags = sp.ntaps == 0 ? kTapsAll : 0u;
  for (int t = 0; t < kMaxTaps; ++t) {
    ts.pos[t >> 2] |= (sp.tap_pos[t] & 31u) << (8 * (t & 3));
    if (sp.tap_xor[t]) ts.flags |= 1u << t;
  }
  return ts;
}
// == prefilter_any() of the StreamParams the TapSet was made from (typed taps are a special case of the per-tap XOR)
BTLE_HD uint32_t prefilter_tapset(const uint32_t lo[4], const uint32_t hi[4], const TapSet &ts) {
  if (ts.flags & kTapsAll) return 0xFFFFFFFFu;
  uint32_t m[4] = {0xFFFFFFFFu, 0xFFFFFFFFu, 0xFFFFFFFFu, 0xFFFFFFFFu};
#pragma unroll
  for (int t = 0; t < kMaxTaps; ++t) {
    const uint32_t s = ts.pos[t >> 2] >> (8 * (t & 3)), x = 0u - ((ts.flags >> t) & 1u);
#pragma unroll
    for (int ph = 0; ph < 4; ++ph) m[ph] &= funnel_r(lo[ph], hi[ph], s) ^ x;   // funnel shifts read bits 0..4 of s
  }
  return m[0] | m[1] | m[2] | m[3];
}
// candidate word of a group for n cfgs: bit i set iff the window at symbol i passed at least one cfg's prefilter
BTLE_HD uint32_t prefilter_union(const uint32_t lo[4], const uint32_t hi[4], const TapSet *ts, int n) {
  uint32_t a = 0u;
  for (int j = 0; j < n; ++j) a |= prefilter_tapset(lo, hi, ts[j]);
  return a;
}

// 32 consecutive bits of phase stream `ph` starting at symbol s0 (may be negative or run past the
// window: missing words read as 0).  pd points at the chunk's first group, 4 words per group.
BTLE_HD uint32_t win32(const uint32_t *pd, int ph, int s0, int ngroups) {
  const int g = s0 >> 5;
  const uint32_t lo = (g >= 0 && g < ngroups) ? pd[4 * g + ph] : 0u;
  const uint32_t hi = (g + 1 >= 0 && g + 1 < ngroups) ? pd[4 * (g + 1) + ph] : 0u;
  return funnel_r(lo, hi, (uint32_t)(s0 & 31));
}

// Whitening bytes [off, off+4) of the channel as a little-endian word (off <= 40).
BTLE_HD uint32_t whiten32(const StreamParams &sp, int off) {
  return funnel_r(sp.whiten[off >> 2], sp.whiten[(off >> 2) + 1], (uint32_t)(8 * (off & 3)));
}

BTLE_HD int ctz32(uint32_t x) {
#if defined(__CUDA_ARCH__)
  return __ffs((int)x) - 1;
#else
  return __builtin_ctz(x);
#endif
}

// search_unique_bits (btle_rx.c:1510-1562) restated on phase words: first window start n0, in
// visiting order, that matches when the search (re)starts at sample R with a ZEROED 32-symbol
// history (:1518) and may place window ends below n0_lim+124 (SURVEY.md App. A.1-A.2).
//   part A: windows starting up to 4*tz samples BEFORE R; taps older than R read 0, so they can
//           only match if the access address' lowest masked bits are 0;
//   part B: full windows, n0 >= R.  Candidates come from the dense pass: flagw (bit g%32 of word
//           g/32) marks groups with candidates, cand[g] bit i marks symbol offsets whose window
//           passed the prefilter on at least one phase; each candidate is re-checked exactly.
//           Groups > g_cap are never window starts.
// part A alone: 1 = hit (n0_out), 0 = no hit here (go on with part B), -1 = the search is over (window ends ran past the limit)
BTLE_HD int search_zero_history(const uint32_t *pd, int R, int n0_lim, const StreamParams &sp, int &n0_out) {
  if (sp.tz > 0) {
    // part A.  A window that starts pz symbols before the first symbol >= R of its phase sees
    // zeros on taps [0,pz) and the stream from that symbol on taps [pz,32).  Candidates in
    // visiting order: pz = tz..1, and for each pz the four phases starting with phase R&3.
    uint32_t wph[4];
#pragma unroll
    for (int q = 0; q < 4; ++q) {                        // window at the first symbol >= R, phase (R+q)&3
      const int n = R + q, s = n >> 2;
      const uint32_t *p = pd + 4 * (s >> 5) + (n & 3);   // R >= 0 and s <= 2080: always inside pd
      wph[q] = funnel_r(p[0], p[4], (uint32_t)(s & 31));
    }
    for (int pz = sp.tz; pz >= 1; --pz) {
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const int c = R + q - 4 * pz;
        if (c >= n0_lim) return -1;                      // window ends only grow from here on
        if ((((wph[q] << pz) ^ sp.aa) & sp.mask) == 0u) { n0_out = c; return 1; }
      }
    }
  }
  return n0_lim <= 0 ? -1 : 0;
}

BTLE_HD bool search_from(const uint32_t *pd, const uint32_t *cand, const uint32_t *flagw, int R, int n0_lim,
                         const StreamParams &sp, int ngroups, int g_cap, int &n0_out) {
  const int za = search_zero_history(pd, R, n0_lim, sp, n0_out);
  if (za) return za > 0;
  int g_last = (n0_lim - 1) >> 7;
  if (g_last > g_cap) g_last = g_cap;
  for (int g = R >> 7; g <= g_last; ++g) {
    const uint32_t fw = flagw[g >> 5] >> (g & 31);
    if (!fw) { g |= 31; continue; }                      // rest of this flag word is empty
    if (!(fw & 1u)) { g += ctz32(fw) - 1; continue; }    // jump to the next flagged group
    uint32_t a = cand[g];
    while (a) {
      const int i = ctz32(a);
      a &= a - 1;
#pragma unroll
      for (int ph = 0; ph < 4; ++ph) {
        const int c = 128 * g + 4 * i + ph;
        if (c >= n0_lim) return false;                   // visiting order is increasing in c
        if (c < R) continue;
        const uint32_t hi = (g + 1 < ngroups) ? pd[4 * (g + 1) + ph] : 0u;
        const uint32_t w = funnel_r(pd[4 * g + ph], hi, (uint32_t)i);
        if (((w ^ sp.aa) & sp.mask) == 0u) { n0_out = c; return true; }    // btle_rx.c:1537-1543
      }
    }
  }
  return false;
}

// Reflected CRC-24 over `nbody` bytes held little-endian in words[0..9], four bytes per step
// ("slicing-by-4"): crc4[k][b] is the register after byte b followed by k zero bytes, so
// crc4[0] == crc_table (btle_rx.c:971-1004) and the result equals crc_update (:1211-1222).
BTLE_HD uint32_t crc24_words(const uint32_t words[11], int nbody, uint32_t crc, const uint32_t *crc4) {
  const int nw = nbody >> 2, rem = nbody & 3;
#pragma unroll
  for (int j = 0; j < 10; ++j) {
    if (j < nw) {
      const uint32_t x = crc ^ words[j];
      crc = crc4[768 + (x & 0xFFu)] ^ crc4[512 + ((x >> 8) & 0xFFu)] ^ crc4[256 + ((x >> 16) & 0xFFu)] ^ crc4[x >> 24];
    } else if (j == nw) {
      const uint32_t w = words[j];
      if (rem > 0) crc = crc4[(crc ^ w) & 0xFFu] ^ (crc >> 8);
      if (rem > 1) crc = crc4[(crc ^ (w >> 8)) & 0xFFu] ^ (crc >> 8);
      if (rem > 2) crc = crc4[(crc ^ (w >> 16)) & 0xFFu] ^ (crc >> 8);
    }
  }
  return crc;
}

// The reference's receiver() for ONE chunk (btle_rx.c:2188-2391), restated on phase words, in two parts.
//   pd       phase words of the chunk's kWinGroups groups (chunk + look-ahead) and one group more
//   cand     per-group candidate words, flagw 2 flag words (see search_from)
//
// chain_chunk(): the greedy control flow only — search, header length, the three length guards — i.e.
// everything that decides WHICH hits the reference counts (pkt_count++, :2274 / :2319).  hit(i, n0, rejected) is
// called for the i-th counted packet, in the reference's order (rejected = true: an ADV header with an impossible
// length, reported only when sp.report_rejected); returns their number.  What a counted packet
// contains does not influence the chain, so payload decode and CRC are left to decode_packet(), which the
// kernel runs afterwards for all packets of a span at once (one lane per packet, converged).
// With report_rejected a chunk reports up to BTLE_MAX_RECS_PER_CHUNK hits (include/btle_b200.h), without it at most
// BTLE_MAX_PKTS_PER_CHUNK.
// Rejected hits the resolver's per-chunk hit row holds on top of BTLE_MAX_PKTS_PER_CHUNK counted packets.  NOT a limit on
// what is reported: a chunk with more hits is finished by its own lane (btle_rx_kernels.cu, resolver step 4).
constexpr int kRejectedInHitRow = 16;
constexpr int kMaxRejectedPerChunk = kRejectedInHitRow;   // former name of the same constant, kept so code using it still builds
// BTLE_CFG_CENTRE_HITS (include/btle_b200.h): hit n of the search restarted at R moved to the centre of its run of matching
// window starts n, n + 1, .. (at most 4, below n0_lim and the chunk's 8192 window starts).  A hit through the zeroed
// history (n < R) stays.  Reads the phase words with win32, so the exact-hit lists and the candidate walk agree.
BTLE_HD int centre_hit(const uint32_t *pd, const StreamParams &sp, int R, int n0_lim, int n) {
  if (n < R) return n;
  int run = 1;
  for (; run < 4; ++run) {
    const int c = n + run;
    if (c >= n0_lim || c >= kChunkSamples) break;
    if (((win32(pd, c & 3, c >> 2, kWinGroups + 1) ^ sp.aa) & sp.mask) != 0u) break;
  }
  return n + ((run - 1) >> 1);
}

// search(R, n0_lim, n0&) -> bool: the reference's search_unique_bits restarted at sample R (see search_from)
template <class Search, class Hit>
BTLE_HD int chain_with(const uint32_t *pd, const StreamParams &sp, Search &search, Hit &hit) {
  int E = 0;                         // buf_len_eaten (int8 units), :2214
  int left = kSearchInt8 / 8;        // num_symbol_left, :2200
  int count = 0;
  for (;;) {
    if (left <= 0) break;            // search loop would not run -> -1 -> break, :2218
    const int R = E >> 1;            // restart sample
    const int n0_lim = R + 4 * left - 124;   // window end n0+124 must stay < R + 4*left
    int n0 = 0;
    if (!search(R, n0_lim, n0)) break;                   // :2218
    if (sp.centre_hits) n0 = centre_hit(pd, sp, R, n0_lim, n0);   // uniform per cfg
    E = 2 * n0 + 256;                                    // :2226, :2231
    E += 64 * (sp.raw ? 42 : 2);                         // :2254-2257
    if (E > kWinInt8) break;                             // :2259-2263
    left = (kSearchInt8 - E) / 8;                        // :2269
    if (!sp.raw) {
      const int ph = n0 & 3, hs = (n0 >> 2) + 32;        // first header symbol (>= 1)
      const uint32_t *p = pd + 4 * (hs >> 5) + ph;
      const uint32_t w0 = funnel_r(p[0], p[4], (uint32_t)(hs & 31)) ^ sp.whiten[0];   // :2265-2267
      int plen;
      if (sp.adv) {
        plen = (int)((w0 >> 8) & 0x3Fu);                 // :1962
        if (plen < 6 || plen > 37) {                     // :2291-2298 (cursor stays behind the header; not counted)
          if (sp.report_rejected) { hit(count, n0, true); ++count; }   // -v "PktBAD"
          continue;
        }
      } else {
        plen = (int)((w0 >> 8) & 0x1Fu);                 // :1944
      }
      E += 64 * (plen + 3);                              // :2305
      if (E > kWinInt8) break;                           // :2308-2311
      left = (kSearchInt8 - E) / 8;                      // :2316
    }
    hit(count, n0, false);
    ++count;                                             // pkt_count++, :2274 / :2319
  }
  return count;
}

template <class Hit>
BTLE_HD int chain_chunk(const uint32_t *pd, const uint32_t *cand, const uint32_t *flagw, const StreamParams &sp, Hit &hit) {
  struct Walk {
    const uint32_t *pd, *cand, *flagw; const StreamParams &sp;
    BTLE_HDM bool operator()(int R, int n0_lim, int &n0) { return search_from(pd, cand, flagw, R, n0_lim, sp, kWinGroups + 1, kGroupsPerChunk - 1, n0); }
  } walk{pd, cand, flagw, sp};
  return chain_with(pd, sp, walk, hit);
}

// ---- the same chain on pre-computed EXACT hits -------------------------------------------------------------------------
// The candidate walk of search_from() is the only part of the chain whose cost depends on the data, and it is the
// same for every restart point: which window starts of the chunk match the access address exactly.  The kernel
// therefore enumerates them once per unit with all 32 lanes (one flag word = 32 groups = 4096 samples per lane,
// enumerate_exact_hits), and the per-chunk chain only walks two short sorted lists with a cursor that never moves back.
constexpr int kExactCap = 15;              // exact hits kept per flag word; more (degenerate masks) -> the chunk falls back to search_from()
// hits of flag word `t` of a unit (groups 32t .. 32t+31 of the unit's pd / cand arrays): list[k] = sample offset inside
// the word (0..4095), ascending; returns their number, kExactCap + 1 meaning "too many"
BTLE_HD int enumerate_exact_hits(const uint32_t *pd, const uint32_t *cand, uint32_t fw, int t, const StreamParams &sp, uint16_t *list) {
  int n = 0;
  while (fw) {
    const int gl = ctz32(fw);
    fw &= fw - 1;
    const int g = 32 * t + gl;
    uint32_t a = cand[g];
    while (a) {
      const int i = ctz32(a);
      a &= a - 1;
#pragma unroll
      for (int ph = 0; ph < 4; ++ph) {
        const uint32_t w = funnel_r(pd[4 * g + ph], pd[4 * (g + 1) + ph], (uint32_t)i);   // the unit's pd has one group more than it has groups
        if (((w ^ sp.aa) & sp.mask) == 0u) {                                              // btle_rx.c:1537-1543
          if (n >= kExactCap) return kExactCap + 1;
          list[n++] = (uint16_t)(128 * gl + 4 * i + ph);
        }
      }
    }
  }
  return n;
}

// chain of one chunk from the lists of its two flag words (l0 / l1, counts n0cnt / n1cnt <= kExactCap)
template <class Hit>
BTLE_HD int chain_chunk_lists(const uint32_t *pd, const uint16_t *l0, int c0, const uint16_t *l1, int c1, const StreamParams &sp, Hit &hit) {
  struct Walk {
    const uint32_t *pd; const uint16_t *l0, *l1; int c0, c1, k; const StreamParams &sp;
    BTLE_HDM bool operator()(int R, int n0_lim, int &n0) {
      const int za = search_zero_history(pd, R, n0_lim, sp, n0);
      if (za) return za > 0;
      for (; k < c0 + c1; ++k) {                         // restart points only grow: entries before the cursor stay behind
        const int c = k < c0 ? (int)l0[k] : 4096 + (int)l1[k - c0];
        if (c < R) continue;
        if (c >= n0_lim) return false;
        n0 = c;
        return true;                                     // (the cursor stays: the next restart point lies behind this hit)
      }
      return false;
    }
  } walk{pd, l0, l1, c0, c1, 0, sp};
  return chain_with(pd, sp, walk, hit);
}

// The bytes of one counted packet whose access address starts at sample n0 of the chunk: tmp_byte[]
// of the reference (:2265-2267, :2313-2314) as 11 little-endian words (zero beyond n_bytes), and crc_check()
// (:1994-2016).  crc4 = 4 x 256 CRC tables (crc24_words).  Reads stay inside the chunk's 77 groups.
// header_only: a rejected hit (kRejectedHit) — just the two dewhitened header bytes, no CRC.
BTLE_HD void decode_packet(const uint32_t *pd, const StreamParams &sp, const uint32_t *crc4, int n0, bool header_only,
                           uint32_t words[11], int &nbytes_out, int &crc_bad_out) {
  const int ph = n0 & 3, hs = (n0 >> 2) + 32;
  // the packet is a contiguous run of phase stream `ph` starting at symbol hs
  const uint32_t *p = pd + 4 * (hs >> 5) + ph;
  const uint32_t o = (uint32_t)(hs & 31);
  uint32_t prev = p[0], cur = p[4];
  words[0] = funnel_r(prev, cur, o);
  int nbytes = 42, crc_bad = 0;
  if (!sp.raw) {
    words[0] ^= sp.whiten[0];
    const int plen = (int)((words[0] >> 8) & (sp.adv ? 0x3Fu : 0x1Fu));
    nbytes = header_only ? 2 : plen + 5;
  }
  const int nw = (nbytes + 3) >> 2;                      // words that hold packet bytes
  // bytes past n_bytes are zero (the reference's tmp_byte is only defined up to there)
  const uint32_t last_mask = (nbytes & 3) ? ((1u << (8 * (nbytes & 3))) - 1u) : 0xFFFFFFFFu;
  if (nw == 1) words[0] &= last_mask;
#pragma unroll
  for (int j = 1; j < 11; ++j) {
    words[j] = 0u;
    if (j < nw) {
      prev = cur;
      cur = p[4 * (j + 1)];
      uint32_t w = funnel_r(prev, cur, o);
      if (!sp.raw) w ^= sp.whiten[j];
      if (j == nw - 1) w &= last_mask;
      words[j] = w;
    }
  }
  if (!sp.raw && !header_only) {                         // crc_check, :1994-2016
    const int body = nbytes - 3;
    const uint32_t crc = crc24_words(words, body, sp.crc_init, crc4);
    const uint32_t rx = (win32(pd, ph, hs + 8 * body, kWinGroups + 1) ^ whiten32(sp, body)) & 0xFFFFFFu;
    crc_bad = (crc != rx);
  }
  nbytes_out = nbytes;
  crc_bad_out = crc_bad;
}

// ---- syndrome correction of CRC-failed packets (BTLE_CFG_CORRECT, include/btle_b200.h) -----------------------------------
// A packet of n_bytes bytes is N = 8 n_bytes bits in the order sent (body, then CRC).  The bit u places from the end (u = 0:
// the last CRC bit) is bit N - 1 - u.  An error there changes crc24(body) XOR received CRC by the syndrome
//   u < 24   1 << (23 - u)  (a CRC bit);
//   u >= 24  the CRC register (crc24_words convention) from 0 after a 1 and u - 24 zero bits (the CRC is linear, and zero
//            bits in front of the error leave a zero register where it starts),
// which depends on u alone, so one table serves every packet length.  Pattern code 2 u + w - 1: w = 1 the single bit u,
// w = 2 the adjacent pair u, u - 1 (u >= 1).  The table holds every pattern of the longest body (39 bytes).
constexpr int kCorrectMaxBits = 8 * 42;                      // 312 body bits of a 39-byte body + 24 CRC bits
constexpr int kCorrectPatterns = 2 * kCorrectMaxBits - 1;    // 336 single bits + 335 adjacent pairs = 671
// open addressing: slot = syndrome_slot(s) + k, k < kSyndromeProbes; entry = s << 32 | code, 0 = empty (no syndrome is 0)
constexpr int kSyndromeSlots = 4096;
constexpr int kSyndromeProbes = 6;
BTLE_HD uint32_t syndrome_slot(uint32_t s) { return (s * 0x9E3779B1u) >> 20; }
// syndrome of pattern `code`
BTLE_HD uint32_t pattern_syndrome(int code) {
  const int u = code >> 1, w = (code & 1) + 1;
  uint32_t s = 0u;
  for (int b = u - w + 1; b <= u; ++b) {
    uint32_t c = 1u << 23;
    if (b >= 24) {
      c = 0xDA6000u;                                         // a 1 into the zero register
      for (int z = 24; z < b; ++z) c = (c >> 1) ^ ((c & 1u) ? 0xDA6000u : 0u);
    } else {
      c >>= b;
    }
    s ^= c;
  }
  return s;
}
// Fills tab[kSyndromeSlots] with the kCorrectPatterns patterns; returns their number, or -1 if two share a syndrome, a
// syndrome is 0, or a pattern would lie kSyndromeProbes or more slots behind its own (none of which happens: tests).
BTLE_HD int make_syndrome_table(uint64_t *tab) {
  for (int i = 0; i < kSyndromeSlots; ++i) tab[i] = 0ull;
  int n = 0;
  for (int code = 0; code < kCorrectPatterns + 1; ++code) {
    if (code == 1) continue;                                 // (u = 0, w = 2) is no pattern
    const uint32_t s = pattern_syndrome(code);
    if (s == 0u) return -1;
    const uint32_t h = syndrome_slot(s);
    int k = 0;
    for (; k < kSyndromeProbes; ++k) {
      const uint64_t e = tab[(h + k) & (kSyndromeSlots - 1)];
      if (e == 0ull) break;
      if ((uint32_t)(e >> 32) == s) return -1;
    }
    if (k == kSyndromeProbes) return -1;
    tab[(h + k) & (kSyndromeSlots - 1)] = ((uint64_t)s << 32) | (uint32_t)code;
    ++n;
  }
  return n;
}
// code of the pattern whose syndrome is s, -1 if none: at most kSyndromeProbes read-only loads
BTLE_HD int syndrome_lookup(const uint64_t *tab, uint32_t s) {
  const uint32_t h = syndrome_slot(s);
#pragma unroll
  for (int k = 0; k < kSyndromeProbes; ++k) {
    const uint64_t *p = tab + ((h + k) & (kSyndromeSlots - 1));
#if defined(__CUDA_ARCH__)
    const uint64_t e = __ldg(reinterpret_cast<const unsigned long long *>(p));
#else
    const uint64_t e = *p;
#endif
    if (e == 0ull) return -1;
    if ((uint32_t)(e >> 32) == s) return (int)(uint32_t)e;
  }
  return -1;
}
// Packet (words[11] as decode_packet returns them, n_bytes) whose syndrome is s != 0: if s is the syndrome of a pattern
// that lies inside the packet and does not touch the header's length field (bits 8..13 on advertising channels, 8..12
// on data channels), flips its bits and returns true; else returns false and leaves words untouched.
BTLE_HD bool correct_words(uint32_t words[11], int nbytes, const StreamParams &sp, uint32_t s, const uint64_t *tab) {
  const int code = syndrome_lookup(tab, s);
  if (code < 0) return false;
  const int w = (code & 1) + 1, i = 8 * nbytes - 1 - (code >> 1);   // flips bits i .. i + w - 1
  if (i < 0) return false;                                           // further from the end than this packet is long
  if (i + w > 8 && i < (sp.adv ? 14 : 13)) return false;             // the length field
  const uint32_t m = w == 2 ? 3u : 1u;
#pragma unroll
  for (int j = 0; j < 11; ++j) {                                     // no dynamic index: words stays in registers
    const int lo = i - 32 * j;
    if (lo >= 0 && lo < 32) words[j] ^= m << lo;
    else if (lo == -1) words[j] ^= m >> 1;                           // the second bit of a pair that straddles a word
  }
  return true;
}
// The primary decode (words, n_bytes) of a counted, CRC-failed packet, corrected by correct_words if its syndrome allows
// (returns true).  The syndrome is the one decode_packet compares: crc24(body) XOR the received (dewhitened) CRC bytes.
BTLE_HD bool correct_packet(uint32_t words[11], int nbytes, const StreamParams &sp, const uint32_t *crc4, const uint64_t *tab) {
  const int body = nbytes - 3, at = 8 * body;
  uint32_t lo = 0u, hi = 0u;
#pragma unroll
  for (int j = 0; j < 11; ++j) {
    if (j == (at >> 5)) lo = words[j];
    if (j == (at >> 5) + 1) hi = words[j];
  }
  const uint32_t rx = funnel_r(lo, hi, (uint32_t)(at & 31)) & 0xFFFFFFu;
  const uint32_t s = crc24_words(words, body, sp.crc_init, crc4) ^ rx;
  return s != 0u && correct_words(words, nbytes, sp, s, tab);
}

// ---- recovery of CRC-failed packets (BTLE_CFG_RECOVER, include/btle_b200.h) --------------------------------------------
// The capture samples one chunk's recovery may read: sample s (relative to the chunk) is iq[2s], iq[2s+1] for 0 <= s < n,
// n = what the capture holds of the chunk's receiver() window [0, kWinInt8 / 2); every other sample reads 0.
// BTLE_CFG_LOWPASS reads the filtered samples F[s] (lp_at) under the same window rule; their neighbours x[s - 1], x[s + 1]
// come from the capture, readable for lo <= s < hi (`lead` bytes in front of the capture, nothing behind its end).
struct IqWindow {
  const int8_t *iq;            // the chunk's first sample
  int n;
  int lo, hi;
};
BTLE_HD IqWindow iq_window(const int8_t *capture, long long n_int8, long long chunk, long long lead = 0) {
  const long long base = chunk * kChunkInt8, avail = (n_int8 - base) >> 1;
  IqWindow w;
  w.iq = capture + base;
  w.n = avail < 0 ? 0 : (avail > kWinInt8 / 2 ? kWinInt8 / 2 : (int)avail);
  w.lo = (base + lead) >= 2 ? -1 : 0;
  w.hi = avail < 0 ? 0 : (avail > kWinInt8 / 2 + 1 ? kWinInt8 / 2 + 1 : (int)avail);
  return w;
}
// I and Q of sample s (0 outside the window)
BTLE_HD void iq_at(const IqWindow &w, int s, int &i, int &q) {
  i = q = 0;
  if (s >= 0 && s < w.n) { i = w.iq[2 * s]; q = w.iq[2 * s + 1]; }
}
// I and Q of the filtered sample F[s] (0 outside the window)
BTLE_HD void lp_at(const IqWindow &w, int s, int &i, int &q) {
  i = q = 0;
  if (s < 0 || s >= w.n) return;
  int im = 0, qm = 0, ip = 0, qp = 0;
  if (s - 1 >= w.lo) { im = w.iq[2 * s - 2]; qm = w.iq[2 * s - 1]; }
  if (s + 1 < w.hi) { ip = w.iq[2 * s + 2]; qp = w.iq[2 * s + 3]; }
  i = (im + 2 * w.iq[2 * s] + ip) >> 2;
  q = (qm + 2 * w.iq[2 * s + 1] + qp) >> 2;
}
// Symbol-spaced discriminator bits: bit k of the result is e[s0 + 4k], e[s] = (I[s] Q[s+4] - I[s+4] Q[s]) > 0.
// ROT: e[s] = C4 (I[s] Q[s+4] - I[s+4] Q[s]) - S4 (I[s] I[s+4] + Q[s] Q[s+4]) > 0 (rot_disc with the 4-sample rotation).
// LP (BTLE_CFG_LOWPASS): the same bits of the filtered samples.
template <bool ROT = false, bool LP = false>
BTLE_HD uint32_t sym_bits32(const IqWindow &w, int s0, int c4 = 0, int s4 = 0) {
  int i0, q0;
  if constexpr (LP) lp_at(w, s0, i0, q0);
  else iq_at(w, s0, i0, q0);
  uint32_t r = 0u;
#pragma unroll 4
  for (int k = 0; k < 32; ++k) {
    int i1, q1;
    if constexpr (LP) lp_at(w, s0 + 4 * k + 4, i1, q1);
    else iq_at(w, s0 + 4 * k + 4, i1, q1);
    if constexpr (ROT) r |= (uint32_t)(rot_disc(i0, q0, i1, q1, c4, s4) < 0) << k;
    else r |= (uint32_t)(i0 * q1 - i1 * q0 > 0) << k;
    i0 = i1;
    q0 = q1;
  }
  return r;
}
// One counted packet whose access address starts at sample n0 and whose primary decode failed the CRC: alternatives
// q = 0..3 (packet bit j = e[n0 + 4j + q - 2]) in order; the first whose CRC is good wins.  Returns q and writes that
// alternative's bytes (words[11], zero behind n_bytes, as decode_packet) and n_bytes; returns -1 and leaves both
// untouched when none passes.  Not for raw mode (sp.recover is 0 there).  ROT: the bits of sym_bits32<true>(.., c4, s4);
// LP: of the filtered samples (BTLE_CFG_LOWPASS).
// tab (BTLE_CFG_CORRECT; words, nbytes_out: the primary decode): when no alternative passes, steps on in repair_packet's
// order: returns 4 when correct_packet corrects the primary decode in words, else 5 + q for the first alternative q that
// correct_words corrects.  One loop for both, so that the kernel holds one alternative's words, not two.
template <bool ROT = false, bool LP = false>
BTLE_HD int recover_packet(const IqWindow &w, const StreamParams &sp, const uint32_t *crc4, int n0, uint32_t words[11], int &nbytes_out,
                           int c4 = 0, int s4 = 0, const uint64_t *tab = nullptr) {
  const int steps = tab ? 9 : 4;
  for (int t = 0; t < steps; ++t) {
    if (t == 4) {
      if (correct_packet(words, nbytes_out, sp, crc4, tab)) return 4;
      continue;
    }
    const int q = t < 4 ? t : t - 5;                     // exact, then corrected
    const int s0 = n0 + 4 * 32 + q - 2;                  // packet bit 32: the first header bit
    uint32_t alt[11];
    alt[0] = sym_bits32<ROT, LP>(w, s0, c4, s4) ^ sp.whiten[0];
    const int plen = (int)((alt[0] >> 8) & (sp.adv ? 0x3Fu : 0x1Fu));
    if (sp.adv && (plen < 6 || plen > 37)) continue;
    const int nbytes = plen + 5, nw = (nbytes + 3) >> 2, body = nbytes - 3;
    const uint32_t last_mask = (nbytes & 3) ? ((1u << (8 * (nbytes & 3))) - 1u) : 0xFFFFFFFFu;
#pragma unroll
    for (int j = 1; j < 11; ++j) alt[j] = j < nw ? sym_bits32<ROT, LP>(w, s0 + 4 * 32 * j, c4, s4) ^ sp.whiten[j] : 0u;
#pragma unroll
    for (int j = 0; j < 11; ++j)
      if (j == nw - 1) alt[j] &= last_mask;
    const uint32_t crc = crc24_words(alt, body, sp.crc_init, crc4);
    const uint32_t rx = (sym_bits32<ROT, LP>(w, s0 + 4 * 8 * body, c4, s4) ^ whiten32(sp, body)) & 0xFFFFFFu;
    if (t < 4 ? crc == rx : correct_words(alt, nbytes, sp, crc ^ rx, tab)) {
#pragma unroll
      for (int j = 0; j < 11; ++j) words[j] = alt[j];
      nbytes_out = nbytes;
      return t;
    }
  }
  return -1;
}
// flags bits a recovered record carries on top of the primary decode's (alternative q)
BTLE_HD uint32_t recovered_flags(int q) { return q < 0 ? 0u : (uint32_t)(BTLE_REC_RECOVERED | (q << 4)); }

// BTLE_CFG_RECOVER and BTLE_CFG_CORRECT on one counted packet whose primary decode (words, nbytes) failed the CRC, in the
// order of include/btle_b200.h (fewer assumed errors win): the alternatives exact, the primary decode corrected, the
// alternatives corrected.  Returns the flags bits the record gets on top of the primary decode's, with the winner's bytes
// in words and its n_bytes in nbytes; 0 when nothing passes (words and nbytes untouched).
template <bool ROT = false, bool LP = false>
BTLE_HD uint32_t repair_packet(const IqWindow &w, const StreamParams &sp, const uint32_t *crc4, const uint64_t *tab, int n0,
                               uint32_t words[11], int &nbytes, int c4 = 0, int s4 = 0) {
  if (!sp.recover) return (sp.correct && correct_packet(words, nbytes, sp, crc4, tab)) ? (uint32_t)BTLE_REC_CORRECTED : 0u;
  const int t = recover_packet<ROT, LP>(w, sp, crc4, n0, words, nbytes, c4, s4, sp.correct ? tab : nullptr);
  if (t < 4) return recovered_flags(t);                                   // -1: nothing passes
  return t == 4 ? (uint32_t)BTLE_REC_CORRECTED : recovered_flags(t - 5) | BTLE_REC_CORRECTED;
}

// Both parts back to back for one chunk (what the test-only CPU emulator runs, lane by lane):
// emit(n0, n_bytes, crc_bad, words[11], rejected) per counted (or, with report_rejected, rejected) hit, in the reference's order.
template <class Emit>
BTLE_HD int resolve_chunk(const uint32_t *pd, const uint32_t *cand, const uint32_t *flagw, const StreamParams &sp,
                          const uint32_t *crc4, Emit &emit) {
  struct Each {
    const uint32_t *pd; const StreamParams &sp; const uint32_t *crc4; Emit &emit;
    BTLE_HDM void operator()(int, int n0, bool rej) {
      uint32_t words[11];
      int nbytes, crc_bad;
      decode_packet(pd, sp, crc4, n0, rej, words, nbytes, crc_bad);
      emit(n0, nbytes, crc_bad, words, rej);
    }
  } each{pd, sp, crc4, emit};
  return chain_chunk(pd, cand, flagw, sp, each);
}

// ---- connection discovery: the empty-PDU candidate rule (DESIGN.md §6.2) ------------------------------------------------
// A window start n0 = 128 g + 4 i + ph of a data-channel capture is a CANDIDATE iff, on phase stream ph (symbol s0 = 32 g + i):
//   preamble  S[s0-8 .. s0] alternate (8 inequalities: 0x55 and 0xAA both pass);
//   header    the 16 symbols S[s0+32 .. s0+47] dewhitened with the first 16 whitening bits of the channel have LLID 1 and
//             byte 1 == 0 (length 0, RFU 0); NESN, SN, MD and the byte-0 RFU bits are free;
//   inside    every d[n] read lies in the capture (empty_pdu_inside).
// w[0..4] = phase words of groups g-1 .. g+3 on phase ph; wh0 = whitening bits 0..31 of the channel (StreamParams::whiten[0]).
// Bit i of the result: the window starting at symbol i of group g passes the preamble and header tests.
constexpr uint32_t kEmptyPduFixed = 0xFF03u;        // header bits the rule pins: LLID (bits 0, 1) and byte 1
BTLE_HD uint32_t empty_pdu_windows(const uint32_t w[5], uint32_t wh0) {
  uint32_t m = 0xFFFFFFFFu;
  uint32_t prev = funnel_r(w[0], w[1], 24u);                         // bit i = S[s0 - 8]
#pragma unroll
  for (int j = 1; j <= 8; ++j) {
    const uint32_t cur = j < 8 ? funnel_r(w[0], w[1], (uint32_t)(24 + j)) : w[1];
    m &= prev ^ cur;
    prev = cur;
  }
  const uint32_t need = (wh0 ^ 1u) & kEmptyPduFixed;                 // received header bits: whitening ^ (LLID 1, all else 0)
#pragma unroll
  for (int j = 0; j < 16; ++j) {
    if (!((kEmptyPduFixed >> j) & 1u)) continue;
    m &= funnel_r(w[2], w[3], (uint32_t)j) ^ (((need >> j) & 1u) - 1u);   // keep bit i iff S[s0+32+j] == need bit j
  }
  return m;
}
// Window starts i of group g (phase ph) whose reads lie inside a capture of n_samples samples: n0 - 32 >= 0 and
// n0 + 284 + 1 < n_samples (d[n] needs samples n and n+1).
BTLE_HD uint32_t empty_pdu_inside(long long g, int ph, long long n_samples) {
  const long long base = 128 * g + ph, lo = 32 - base, hi = n_samples - 286 - base;
  if (hi < 0) return 0u;
  const long long i_lo = lo <= 0 ? 0 : (lo + 3) / 4, i_hi = hi / 4 < 31 ? hi / 4 : 31;
  if (i_lo > i_hi) return 0u;
  const uint32_t upto = i_hi == 31 ? 0xFFFFFFFFu : ((1u << (i_hi + 1)) - 1u);
  return upto & ~((1u << i_lo) - 1u);
}
// Fields of the window at symbol i: access address, dewhitened header (16 bits) and the received CRC (24 bits, dewhitened
// with whitening bits 16..39); wh1 = whitening bits 32..63.
BTLE_HD void empty_pdu_fields(const uint32_t w[5], int i, uint32_t wh0, uint32_t wh1, uint32_t &aa, uint32_t &header,
                              uint32_t &crc_rx) {
  aa = funnel_r(w[1], w[2], (uint32_t)i);
  const uint32_t a = funnel_r(w[2], w[3], (uint32_t)i), b = funnel_r(w[3], w[4], (uint32_t)i);
  header = (a ^ wh0) & 0xFFFFu;
  crc_rx = (((a >> 16) | (b << 16)) ^ ((wh0 >> 16) | (wh1 << 16))) & 0xFFFFFFu;
}
// The CRC-24 register (crc24_words convention) from which `nbits` message bits (bit j = j-th bit sent) lead to `crc`.
// One step of the LFSR is  c' = (c >> 1) ^ (f ? 0xDA6000 : 0), f = (c ^ bit) & 1;  bit 23 of c' is f, so every step can be
// undone and the result is unique.  crc_init_reorder() of it is the -k value.
BTLE_HD uint32_t crc24_unwind(uint32_t crc, uint32_t bits, int nbits) {
  for (int j = nbits - 1; j >= 0; --j) {
    const uint32_t f = (crc >> 23) & 1u;
    crc = (((crc ^ (f ? 0xDA6000u : 0u)) << 1) | (f ^ ((bits >> j) & 1u))) & 0xFFFFFFu;
  }
  return crc;
}

// ---- the merge of BTLE_CFG_OFFSET_SEARCH's hypotheses (include/btle_b200.h, rule 2) --------------------------------------
// One record of a chunk's merged list: its n0, whether it is a counted CRC-ok record, and the caller's reference to it.
struct OsEnt {
  int32_t n0;
  uint32_t ok;    // 1: counted with crc_bad == 0 (the records that stay and that hypotheses 1..6 may add)
  uint32_t ref;
};
BTLE_HD uint32_t os_ok(uint8_t flags, uint8_t crc_bad) { return !(flags & (BTLE_REC_REJECTED | 1u)) && crc_bad == 0; }
// One step of the merge: hypothesis h >= 1's record r (r.ok, else the caller skips it) against the list b[0, nb), which is
// in n0 order.  Returns the new length: r dropped (a CRC-ok record within 8 samples), or the CRC-failed and rejected records
// within 8 samples removed and r inserted in n0 order.  No entry left in b has r's n0, so the place is unique.
BTLE_HD int os_merge_step(OsEnt *b, int nb, const OsEnt &r) {
  for (int i = 0; i < nb; ++i) {
    const int d = b[i].n0 - r.n0;
    if (b[i].ok && d >= -8 && d <= 8) return nb;
  }
  int w = 0;
  for (int i = 0; i < nb; ++i) {
    const int d = b[i].n0 - r.n0;
    if (d >= -8 && d <= 8) continue;
    b[w++] = b[i];
  }
  int at = w;
  while (at > 0 && b[at - 1].n0 > r.n0) { b[at] = b[at - 1]; --at; }
  b[at] = r;
  return w + 1;
}

}  // namespace btle
