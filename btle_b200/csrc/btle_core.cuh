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
  int32_t report_rejected;    // -v: hits the reference drops for their ADV length (:2291-2298) are reported too (not counted)
  int32_t tz;                 // min(31, index of lowest set bit of aa&mask (32 if none))
  int32_t ntaps;              // 0 => every group is flagged (mask == 0)
  int32_t typed;              // 1 => taps [0, kTapsOne) expect a 1 and taps [kTapsOne, kMaxTaps) expect a 0
  uint32_t tap_pos[kMaxTaps]; // prefilter tap positions p (mask bit set), padded by repetition
  uint32_t tap_xor[kMaxTaps]; // 0 if aa bit p is 1, ~0 if it is 0
  uint32_t whiten[12];        // scramble_table[channel][0..41] packed little-endian (+pad)
};

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

}  // namespace btle
