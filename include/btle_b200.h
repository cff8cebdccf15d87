/* btle_b200 — C-ABI of the CUDA-native (H100, sm_90a) BLE receive baseband.
 *
 * Drop-in boundary for ONE path of JiaoXianjun/BTLE: the btle_rx receive chain
 *   int8 IQ @4 Msps -> GFSK differential demod -> 4:1 bit decision -> 32-bit masked
 *   access-address sliding match -> dewhiten -> header parse -> CRC-24
 * (reference: host/btle-tools/src/btle_rx.c:1489-1562, 1969-2016, 2188-2391).
 *
 * The reference has no library/FFI layer (btle_rx is one translation unit,
 * src/CMakeLists.txt:34); its only function seam for this path is
 *   void receiver(IQ_TYPE *rxp_in, int buf_len, int channel_number, uint32_t access_addr,
 *                 uint32_t crc_init, int verbose_flag, int raw_flag)        btle_rx.c:2188
 * called by main() once per 16384-int8 half of its ring buffer (btle_rx.c:2619-2651), with the
 * mask, filters and sinks passed through globals.  btle_b200_rx*() replaces that call for a
 * whole capture (or a batch of captures) at once and RETURNS the packets receiver() would
 * have counted, in the same order, instead of printing them.  See INTEGRATION.md for the
 * binding a maintainer of the reference would add.
 *
 * Plain C: pointers and sizes only.  Every function returns 0 or a negative BTLE_E* code and
 * never exits the process.  A context is bound to one CUDA device and is not thread-safe;
 * use one context per thread.  There is NO CPU fallback: without a CUDA device
 * btle_b200_create() fails with BTLE_ENODEV.
 */
#ifndef BTLE_B200_H
#define BTLE_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define BTLE_OK 0
#define BTLE_EINVAL (-1)   /* bad argument (channel > 39, misaligned device pointer, ...)   */
#define BTLE_ENODEV (-2)   /* no usable CUDA device                                          */
#define BTLE_ENOMEM (-3)   /* device or host allocation failed                               */
#define BTLE_ECUDA (-4)    /* a CUDA call failed; see btle_b200_last_error()                 */
#define BTLE_EOVERFLOW (-5)/* more packets than `cap`; *n_out holds the number found          */
/* btle_b200_search_unique_bits() returns sample indices (even values >= -248, or -1 = no match, like the
 * reference's function), so its errors are moved out of that range: BTLE_SEARCH_ERR(BTLE_ECUDA) == -1004. */
#define BTLE_SEARCH_ERR(code) ((code) - 1000)

#define BTLE_CHUNK_INT8 16384      /* LEN_BUF/2, btle_rx.c:223-224                           */
#define BTLE_LOOKAHEAD_INT8 3008   /* LEN_BUF_MAX_NUM_PHY_SAMPLE, btle_rx.c:237-238          */
/* Upper bound of packets receiver() can count in one chunk.  A packet moves buf_len_eaten on by at least
 * 2*n0' + 256 + 64*2 + 64*3 int8 (:2226-2232, :2259, :2305) where n0' >= -4*ctz(access_addr & mask) relative to
 * the restart point (zeroed history, :1518), and a new search starts only while buf_len_eaten < 16632 (:2218):
 * 34 per chunk when bit 0 of the masked access address is set, 51 in the degenerate case mask == 0.  Real
 * captures hold a few; callers may size `cap` smaller and grow it on BTLE_EOVERFLOW (*n_out = needed). */
#define BTLE_MAX_PKTS_PER_CHUNK 51
/* Upper bound of records one chunk can return when BTLE_CFG_REPORT_REJECTED is set.  A rejected hit moves
 * buf_len_eaten on by at least 2*n0' + 256 + 64*2 >= -248 + 384 = 136 int8 (the header is demodulated, then the
 * search restarts behind it, :2291-2298), a counted packet by more, and hits start only while buf_len_eaten <= 16624
 * (:2218): at most 16624/136 + 1 = 123 hits.  Mask 0 on an all-zero capture reaches it on channels 38 and 39: every
 * window matches through the zeroed history, and every header is the channel's whitening sequence, whose length
 * field is outside 6..37 there, so all 123 hits of a chunk are rejected. */
#define BTLE_MAX_RECS_PER_CHUNK 123

/* Per-capture receiver parameters == btle_rx's -c / -a / -m / -k / -r / -R options
 * (parse_commandline, btle_rx.c:1244-1458; defaults :1271-1301). */
typedef struct {
  int32_t channel;       /* -c  0..39; 37..39 select the advertising-PDU header parser       */
  uint32_t access_addr;  /* -a  default 0x8E89BED6                                           */
  uint32_t access_mask;  /* -m  default 0xFFFFFFFF; bit p = compare p-th received AA bit     */
  uint32_t crc_init;     /* -k  default 0x555555, NOT reordered (crc_init_reorder is ours)   */
  int32_t raw;           /* -r  1: 42 un-dewhitened bytes after each AA hit (btle_rx.c:2254) */
  int32_t rssi;          /* flag bits: BTLE_CFG_RSSI (-R) 1: also return sum|I|+|Q| over the AA samples
                            (:2234-2243); BTLE_CFG_REPORT_REJECTED (-v) 2: advertising-channel hits whose header
                            length is outside 6..37 — the reference prints "PktBAD" for them under -v and does not
                            count them (:2291-2298) — come back as records with BTLE_REC_REJECTED set, every one
                            of them, in the reference's order (up to BTLE_MAX_RECS_PER_CHUNK records per chunk);
                            BTLE_CFG_RECOVER 4: CRC-failed packets are demodulated once more (below);
                            BTLE_CFG_SYMBOL_SPACED 16: the symbol-spaced discriminator (below);
                            BTLE_CFG_CENTRE_HITS 64: each hit centred on its run of matching phases (below);
                            BTLE_CFG_CORRECT 256: one-bit and adjacent-pair errors corrected by the CRC (below);
                            BTLE_CFG_LOWPASS 512: a [1, 2, 1] low-pass in front of the symbol-spaced bits (below);
                            BTLE_CFG_OFFSET_SEARCH 1024: a bank of seven carrier-offset hypotheses (below)  */
} btle_stream_cfg;
#define BTLE_CFG_RSSI 1
#define BTLE_CFG_REPORT_REJECTED 2
/* BTLE_CFG_RECOVER: opt-in recovery of packets that fail the CRC.  Not part of the reference's receiver; without it the
 * records are the reference's, bit for bit.
 * The chain (which hits are counted or rejected, their n0, restart points and length guards) is exactly the
 * reference's, computed from the primary decode.  Then every COUNTED record with crc_bad == 1 of a cfg with the flag
 * and raw == 0 is demodulated again:
 *   1. window   capture samples are read only inside [8192 chunk, 8192 chunk + 9696) (receiver()'s demod_buf_len,
 *               19392 int8); samples behind that range, or behind the capture's end, read as 0.  So the result does not
 *               depend on how a capture was cut into batches, segments or sets.
 *   2. bits     symbol-spaced: e[s] = (I[s] Q[s+4] - I[s+4] Q[s]) > 0, s relative to the chunk, products in int32.
 *   3. alternatives q = 0, 1, 2, 3, tried in that order.  Packet bit j of alternative q (j = 0: first access-address
 *               bit) is e[n0 + 4j + q - 2].  Bits j >= 32 are read into bytes, LSB first, and dewhitened with the
 *               channel's table (as the primary decode).  The header length comes from the alternative's own header:
 *               6 bits on channels 37..39, 5 bits on 0..36.  On advertising channels an alternative whose length is
 *               outside 6..37 is skipped.  Otherwise n_bytes = length + 5 and the CRC is checked as crc_check() does.
 *   4. result   the first alternative with a good CRC replaces the record's bytes (zero behind n_bytes) and n_bytes,
 *               with crc_bad = 0; flags gets BTLE_REC_RECOVERED and q in bits 4..5.  stream, chunk, n0, channel,
 *               access_addr and mag_sum stay.  If no alternative passes, the record is the reference's, byte for byte.
 * Rejected (BTLE_CFG_REPORT_REJECTED) records, raw-mode records and CRC-ok records are never touched; the flag does
 * nothing in raw mode. */
#define BTLE_CFG_RECOVER 4
/* BTLE_CFG_CORRECT: opt-in CRC-24 syndrome decoding of packets that fail the CRC.  Not part of the reference's receiver;
 * without it the records are the reference's (or the current mode's), bit for bit.  It applies only to a COUNTED record
 * with crc_bad == 1 of a cfg with the flag and raw == 0:
 *   1. chain     which hits are counted or rejected, their n0, the restart points, the length guards and n_bytes are
 *                unchanged.  The header's length field is never corrected (another length would move the CRC field).
 *   2. patterns  the packet bits in the order sent (the dewhitened bytes, LSB first): body bits 0 .. 8 (n_bytes - 3) - 1,
 *                then the 24 CRC bits.  The patterns are every single bit and every pair of adjacent bits, except those
 *                touching the length field: header bits 8..13 on channels 37..39, 8..12 on channels 0..36.  (Whitening is
 *                an XOR, so an error in the air is an error at the same place in the dewhitened bits.)
 *   3. syndrome  s = crc24(body) XOR the received CRC.  It depends only on an error's distance from the packet's end, so
 *                one table of the 671 patterns of the longest body (39 bytes) serves every length; their syndromes are
 *                distinct and non-zero.  If s is the syndrome of exactly one allowed pattern, that pattern's bits are
 *                flipped in bytes, crc_bad = 0 and flags gets BTLE_REC_CORRECTED.  Otherwise the record stays as it was.
 *                stream, chunk, n0, channel, n_bytes, access_addr and mag_sum never change.
 *   4. order     with BTLE_CFG_RECOVER too, fewer assumed errors win: the primary decode exact (the reference), then
 *                BTLE_CFG_RECOVER's alternatives q = 0..3 exact (a record identical to a RECOVER-only run), then the
 *                primary decode corrected, then the alternatives q = 0..3 corrected (first q wins; flags gets
 *                BTLE_REC_RECOVERED, q in bits 4..5 and BTLE_REC_CORRECTED; n_bytes is the alternative's).
 * A CRC-failed packet with no allowed pattern is "corrected" to wrong bytes when its syndrome happens to equal one of the
 * allowed ones: about 671 / 2^24 = 4.0e-5 of such packets if their syndromes were uniform.  The flag works in every
 * discriminator mode, with and without carrier-offset correction and BTLE_CFG_CENTRE_HITS; it is per cfg (like
 * BTLE_CFG_RECOVER).  btle_rx_ber_cfg.flags accepts it too. */
#define BTLE_CFG_CORRECT 256
/* BTLE_CFG_SYMBOL_SPACED: opt-in symbol-spaced discriminator.  Not part of the reference's receiver; without it the records
 * are the reference's, bit for bit.  With it every discriminator bit of the capture is
 *     d[n] = I[n-2] Q[n+2] - I[n+2] Q[n-2] > 0      (int32; x[n] = sample n of the capture)
 * a phase step over one symbol (+-pi/2 nominal) instead of a quarter symbol, centred on n as the reference's bit is centred
 * on n + 1/2, so n0, mag_sum, the BER scorer's +-3-sample match and btle_b200_rec_offset keep their meaning.  Samples in
 * front of the capture read as 0 unless the launch makes them readable (the stream sessions keep 256 bytes of the previous
 * segment set in front of each set), samples behind its end read as 0: a chunk's bits are a function of the capture, not
 * of how it was cut.  d[n] equals BTLE_CFG_RECOVER's alternative q = 0 bit e[n - 2] (which reads only its chunk window).
 * With carrier-offset correction (the *_offset entry points) the bit is rotated by (C4, S4) from 4 phi:
 *     d[n] = C4 (I[n-2] Q[n+2] - I[n+2] Q[n-2]) - S4 (I[n-2] I[n+2] + Q[n-2] Q[n+2]) > 0.
 * Everything the chain derives from d follows unchanged: the access-address search, the greedy chain and its length guards,
 * dewhitening, the CRC, -v rejected hits, BTLE_MAX_RECS_PER_CHUNK; BTLE_CFG_RECOVER keeps its own alternatives.
 * One mode per launch: every cfg of one rx_batch / rx_multi / device call must agree on this flag, else BTLE_EINVAL (with
 * last_error set).  A stream session's mode is that of the cfgs given to streams_open; a set_cfg or add_cfg with the other
 * value is BTLE_EINVAL.  btle_rx_ber_cfg.flags accepts it too. */
#define BTLE_CFG_SYMBOL_SPACED 16
/* BTLE_CFG_LOWPASS: opt-in low-pass filter in front of the symbol-spaced discriminator.  Valid only together with
 * BTLE_CFG_SYMBOL_SPACED.  Each discriminator bit of a raw sample reads the full 4-MHz noise band while a 1-Mbps GFSK signal
 * fills little more than 1 MHz of it; with the flag every bit reads filtered samples instead:
 *     F[n] = (x[n-1] + 2 x[n] + x[n+1]) >> 2       per rail (I and Q), arithmetic shift (floor); always -128..127
 *     d[n] = FI[n-2] FQ[n+2] - FI[n+2] FQ[n-2] > 0  (rotated by (C4, S4) with the *_offset entry points, as above)
 * The filter is symmetric, so n0 keeps its meaning.  x outside the capture reads 0 and the launch's lead bytes are readable,
 * exactly as for the symbol-spaced bits, so F and every chunk's bits are a function of the whole capture, not of how it was
 * cut.  BTLE_CFG_RECOVER's alternatives read F in place of x, e[s] = FI[s] FQ[s+4] - FI[s+4] FQ[s] > 0, under its window
 * rule: F[s] reads 0 outside [8192 chunk, 8192 chunk + 9696) and behind the capture's end, and inside it is computed from
 * the capture (x[s - 1] and x[s + 1] may lie outside the window).  mag_sum, btle_b200_rec_offset and discovery read the raw
 * samples; the search, BTLE_CFG_CENTRE_HITS, the chain and its guards, decode, the CRC, BTLE_CFG_CORRECT, -v and the record
 * caps are unchanged.  One mode per launch and per session, as for BTLE_CFG_SYMBOL_SPACED: mixed cfgs in one launch, a
 * session set_cfg or add_cfg with the other value, and the flag without BTLE_CFG_SYMBOL_SPACED are BTLE_EINVAL (with
 * last_error set).  btle_rx_ber_cfg.flags accepts it under the same pairing rule. */
#define BTLE_CFG_LOWPASS 512
/* BTLE_CFG_CENTRE_HITS: opt-in hit rule of the greedy chain.  Not part of the reference's receiver; without it the records
 * are the reference's (or the current mode's), bit for bit.  An access address stays matched for about a symbol around the
 * eye, so the search's first matching window start lies up to a few samples before the centre; with the flag the chain
 * moves each such hit to the centre of its run of matching sample phases:
 *   1. which hits  the search restarted at sample R (window-start limit n0_lim = R + 4 num_symbol_left - 124) returns n.
 *                  Only a full-window hit, n >= R, moves; a hit through the zeroed history (n < R) stays.
 *   2. the run     L = 1 + k, k = the number of consecutive q = 1, 2, 3 (in that order) with n + q < n0_lim, n + q < 8192
 *                  (a window start of the chunk) and the 32 bits d[n + q + 4j], j = 0..31, matching the access address
 *                  under the mask exactly as the search compares them.
 *   3. the hit     n0' = n + floor((L - 1) / 2): L = 1 or 2 keeps n, L = 3 or 4 gives n + 1.
 * Everything the chain derives from a hit then uses n0': the header and its length, the three length guards, the -v
 * rejected record, the restart point (buf_len_eaten = 2 n0' + 256 + ...), the bytes and the CRC, mag_sum and
 * BTLE_CFG_RECOVER's alternatives.  A record's n0 is n0', in -124..8191 as always.  The rule reads only the bits d of the
 * launch's mode, so it applies with and without BTLE_CFG_SYMBOL_SPACED, with and without carrier-offset correction, and in
 * raw mode; it reads nothing outside the chunk's window.  Since n0' >= n, every restart point lies at or behind the
 * reference's for the same hit, so the counting arguments of BTLE_MAX_PKTS_PER_CHUNK and BTLE_MAX_RECS_PER_CHUNK hold
 * unchanged.  The flag is per cfg (like BTLE_CFG_RECOVER): the cfgs of one launch, rx_multi capture or stream session
 * may mix it freely.  btle_rx_ber_cfg.flags accepts it too. */
#define BTLE_CFG_CENTRE_HITS 64
/* Carrier-offset correction: the *_offset entry points take one float offset_hz per capture, the received carrier minus
 * the nominal one in Hz (the sign of btle_rx_ber_cfg.cfo_hz: correcting by cfo_hz undoes that impairment).  Not part of the
 * reference's receiver.  With phi = 2 pi offset_hz / 4 MHz and C = round(2^14 cos phi), S = round(2^14 sin phi) (nearest,
 * ties to even; computed in double on the host), every discriminator bit becomes
 *     d[n] = C (I[n] Q[n+1] - I[n+1] Q[n]) - S (I[n] I[n+1] + Q[n] Q[n+1]) > 0      (int32, |each product sum| <= 2^15)
 * i.e. the sign of Im(conj(x[n]) x[n+1] e^(-j phi)).  The samples are not changed.  Everything the chain derives from these
 * bits — the access-address search, the greedy chain, the length guards, the bytes, the CRC, -v rejected hits — follows
 * unchanged.  For offset 0, (C, S) = (16384, 0) and every record equals the reference's, bit for bit; a non-NULL offset_hz
 * always takes the rotated kernel, also when every value is 0.  BTLE_CFG_RECOVER's symbol-spaced bits use the rotation
 * over 4 samples: (C4, S4) from 4 phi in the same formula, e[s] = C4 (I[s] Q[s+4] - I[s+4] Q[s]) - S4 (I[s] I[s+4] +
 * Q[s] Q[s+4]) > 0.  mag_sum (RSSI) reads the raw samples and is unaffected.  In rx_multi the cfgs of one capture share
 * its offset.  Values that are not finite, or with |offset_hz| > BTLE_MAX_OFFSET_HZ, are BTLE_EINVAL. */
#define BTLE_MAX_OFFSET_HZ 500000
/* BTLE_CFG_OFFSET_SEARCH: opt-in bank of carrier-offset hypotheses, so that transmitters at different offsets in one capture
 * are all received (every advertiser transmits from its own crystal, up to +-150 kHz off).  Not part of the reference's
 * receiver; without it every record is unchanged, bit for bit.  f_c is capture c's offset (offset_hz[c] of the *_offset
 * entry points and sessions, else 0).
 *   1. hypotheses  h = 0..6 decodes capture c at f_c + delta_h, delta = 0, -50, +50, -100, +100, -150, +150 kHz in that order
 *                  (BTLE_OFFSET_SEARCH_HZ), with every cfg of c, in the launch's discriminator mode, by the rotated kernel's
 *                  definition above.  Hypothesis 0 is the call without the flag at the same offsets.  The 50-kHz step
 *                  leaves at most 25 kHz of residual offset inside +-150 kHz.
 *   2. merge       per (cfg j, chunk k), independently of every other chunk: B starts as hypothesis 0's records of (j, k).
 *                  Then for h = 1..6 in order, for each of h's records r of (j, k) in n0 order that is counted with
 *                  crc_bad == 0 (CRC-ok as decoded or after BTLE_CFG_RECOVER / BTLE_CFG_CORRECT): if B holds a counted
 *                  CRC-ok record with |n0 - r.n0| <= 8 (two symbols), r is dropped; otherwise every CRC-failed or rejected
 *                  record of B with |n0 - r.n0| <= 8 is removed and r is inserted with flags |= BTLE_REC_OFFSET_SEARCH.
 *                  CRC-failed and rejected records of h >= 1 are never added.  The result is in (j, chunk, n0) order,
 *                  stream = j, and every field of a kept hypothesis-0 record is unchanged.
 *   3. so          the call returns every CRC-ok record of the call without the flag, unchanged; every other record it
 *                  returns carries BTLE_REC_OFFSET_SEARCH and crc_bad 0; CRC-failed and rejected records can only
 *                  disappear.  Duplicates across a chunk boundary (one packet found in chunk k by one hypothesis and in
 *                  k + 1 by another) are not merged.  btle_b200_rec_offset estimates a BTLE_REC_OFFSET_SEARCH record's
 *                  offset (it reads the raw samples, so it returns the packet's full offset, not the residual).
 *   4. mode        one mode per launch and per session, as BTLE_CFG_SYMBOL_SPACED: mixed cfgs in one launch, a session set_cfg
 *                  or add_cfg with the other value, the flag with raw (raw records have no CRC verdict) and |f_c| + 150 kHz >
 *                  BTLE_MAX_OFFSET_HZ are BTLE_EINVAL with last_error set.  btle_rx_ber_cfg.flags accepts it.
 *   5. capacity    the directory has the entries and layout of the call without the flag (btle_b200_rx_units and
 *                  btle_b200_rx_multi_units are unchanged).  The seven hypotheses are decoded into context-owned scratch of
 *                  `cap` records.  When they find more than that (T > cap), nothing is merged: *d_count / *n_out is T (the
 *                  merged count is never larger), the directory entries sum to T and their blocks hold no records, and the
 *                  host entry points return BTLE_EOVERFLOW.  A second call with cap >= T returns the whole result.  Flagged
 *                  launches of one context on different CUDA streams are ordered one after the other through the scratch. */
#define BTLE_CFG_OFFSET_SEARCH 1024
#define BTLE_OFFSET_SEARCH_HYPS 7
#define BTLE_OFFSET_SEARCH_HZ {0.0f, -50e3f, 50e3f, -100e3f, 100e3f, -150e3f, 150e3f}
#define BTLE_OFFSET_SEARCH_SPAN_HZ 150000
/* Records one chunk of one cfg can return with BTLE_CFG_OFFSET_SEARCH: hypothesis 0 contributes at most
 * BTLE_MAX_RECS_PER_CHUNK, each of hypotheses 1..6 inserts at most its counted packets (BTLE_MAX_PKTS_PER_CHUNK), and no
 * other step adds a record: 123 + 6 * 51 = 429. */
#define BTLE_MAX_MERGED_RECS_PER_CHUNK (BTLE_MAX_RECS_PER_CHUNK + (BTLE_OFFSET_SEARCH_HYPS - 1) * BTLE_MAX_PKTS_PER_CHUNK)

/* One packet the reference would have counted (pkt_count++, btle_rx.c:2274/:2319). 64 bytes. */
typedef struct {
  int32_t stream;        /* index of the capture in the batch                                */
  int32_t chunk;         /* index of the 16384-int8 chunk receiver() would have been given    */
  int32_t n0;            /* first IQ sample of the access address, relative to that chunk
                            (-124..8191; == hit_idx/2 accumulated, btle_rx.c:2226)            */
  uint8_t channel;
  uint8_t n_bytes;       /* 42 in raw mode, else 2 + payload_len + 3                          */
  uint8_t crc_bad;       /* crc_check() verdict, 1 = mismatch (btle_rx.c:2015); 0 in raw mode */
  uint8_t flags;         /* bit0 raw, bit1 advertising channel, bit2 BTLE_REC_REJECTED: not a packet the
                            reference counts — only bytes[0..1] (the header) are valid, n_bytes = 2;
                            bit3 BTLE_REC_RECOVERED: bytes from alternative q = bits 4..5 (BTLE_CFG_RECOVER);
                            bit6 BTLE_REC_CORRECTED: bytes corrected by the CRC syndrome (BTLE_CFG_CORRECT);
                            bit7 BTLE_REC_OFFSET_SEARCH: found by offset hypothesis 1..6 (BTLE_CFG_OFFSET_SEARCH) */
  uint32_t access_addr;
  uint16_t mag_sum;      /* sum |I|+|Q| over the 128 AA samples if cfg.rssi, else 0           */
  uint8_t bytes[42];     /* == reference tmp_byte[] (btle_rx.c:1485): dewhitened header,
                            payload, CRC; zero beyond n_bytes                                 */
} btle_pkt_rec;

#define BTLE_REC_REJECTED 4
#define BTLE_REC_RECOVERED 8
#define BTLE_REC_RECOVERED_Q(flags) (((flags) >> 4) & 3)
#define BTLE_REC_CORRECTED 64
#define BTLE_REC_OFFSET_SEARCH 128

typedef struct btle_b200_ctx btle_b200_ctx;

/* ---- context -------------------------------------------------------------------------- */
int btle_b200_create(btle_b200_ctx **out, int cuda_device);
void btle_b200_destroy(btle_b200_ctx *ctx);
const char *btle_b200_last_error(const btle_b200_ctx *ctx);
const char *btle_b200_strerror(int code);
/* Host placement for the host-buffer entry points: binds the CALLING THREAD to the CPUs of the NUMA node the GPU's
 * PCIe root hangs off (sysfs numa_node / cpulist, intersected with the current affinity) and makes that node the
 * preferred one for its page allocations.  Call it before allocating (page-locked) IQ buffers: on a two-socket box
 * host->device copies from the far socket cross the inter-socket link and the 8 GPUs' copies then share it.
 * *node_out = the node, or -1 if the machine does not expose one (then nothing is changed). */
int btle_b200_bind_host_numa(int cuda_device, int *node_out);
/* library/ABI version, (major<<16)|minor */
uint32_t btle_b200_version(void);

/* ---- the hot path --------------------------------------------------------------------- */
/* Host buffers in, host records out (what a reference-side caller uses; replaces the
 * main()->receiver() loop, btle_rx.c:2610-2662).  `iq` holds n_streams captures; capture s
 * starts at iq + s*stream_stride_int8 and is n_int8 long (interleaved I,Q int8, as written
 * by rx_callback, btle_rx.c:531-540).  Chunk k of a capture exists while 16384(k+1) <= n_int8;
 * bytes past the end of a capture read as 0 (the reference would wait for the radio).
 * Records come back sorted by (stream, chunk, n0) == the order receiver() emits them.
 * `iq` may be page-locked (cudaHostAlloc / cudaHostRegister: copied by DMA directly) or ordinary pageable
 * memory (moved through the context's page-locked staging buffers in 32 MiB segments, CPU copy of one
 * segment overlapping the DMA of the previous one). */
int btle_b200_rx_batch(btle_b200_ctx *ctx, const int8_t *iq, size_t n_streams, size_t stream_stride_int8,
                       size_t n_int8, const btle_stream_cfg *cfgs, btle_pkt_rec *out, size_t cap,
                       size_t *n_out);
/* The same with carrier-offset correction (BTLE_MAX_OFFSET_HZ above): offset_hz[s] for capture s; NULL: as btle_b200_rx_batch. */
int btle_b200_rx_batch_offset(btle_b200_ctx *ctx, const int8_t *iq, size_t n_streams, size_t stream_stride_int8, size_t n_int8,
                              const btle_stream_cfg *cfgs, const float *offset_hz, btle_pkt_rec *out, size_t cap, size_t *n_out);
/* Single capture convenience wrapper. */
int btle_b200_rx(btle_b200_ctx *ctx, const int8_t *iq, size_t n_int8, const btle_stream_cfg *cfg,
                 btle_pkt_rec *out, size_t cap, size_t *n_out);

/* Device-resident variant: `d_iq` (16-byte aligned; stride a multiple of 16 and >= n_int8 when n_streams > 1), `d_out`, `d_count`
 * and `d_dir` are device pointers usable from the context's device (local HBM or PEER memory of another GPU —
 * that is how the multi-GPU gather works: every rank's kernel stores its records straight into rank 0's buffer
 * over NVLink); work is enqueued on `cuda_stream` (a cudaStream_t, may be NULL) and NOT synchronised.
 *
 * Output layout.  A launch is cut into btle_b200_rx_units() UNITS of work (16 chunks of one capture, or a few
 * chunks in the last wave of the persistent grid), numbered in (stream, chunk) order.  Each unit reserves ONE
 * contiguous block of d_out (one atomic per unit on *d_count) and writes its records there in the reference's
 * order, and fills d_dir[unit] = {first record, number of records}.  So:
 *   - walking d_dir in index order visits all records in the order receiver() emits them (no sort needed);
 *     btle_b200_gather_ordered() does that walk on host copies;
 *   - sum(d_dir[u].count) == *d_count == packets found, also when that exceeds `cap` (records beyond cap are
 *     not stored);
 *   - blocks themselves follow each other in the order the units finished, i.e. d_out as a whole is NOT sorted.
 * *d_count (uint32) is zeroed by the call; every d_dir entry of the launch is written (no memset needed).
 * btle_b200_rx_device_dir() accepts d_count == NULL: the block reservations then run on a context-owned counter (a ring
 * of them, each cleared by an earlier launch) and no memset is enqueued in front of the kernel — for callers that take
 * the packet count from the directory.
 * Streams: the launches of one context may go to different CUDA streams (this call, btle_b200_rx_device,
 * btle_b200_discover_device and btle_b200_synth_streams_device share the context's cached parameter arrays, and d_count
 * == NULL launches share its counter ring).  Each launch is ordered after what it depends on — the upload of the
 * parameters it reads, and the earlier ring launch that cleared its counter — without serialising the streams' kernels:
 * a launch never waits for another stream's kernel that reads the same parameters, and launches on one stream, or
 * alternating strictly between two, add no cross-stream wait.  Ordering the caller's own buffers is the caller's part. */
typedef struct { uint32_t base, count; } btle_unit_dir;
size_t btle_b200_rx_units(const btle_b200_ctx *ctx, size_t n_streams, size_t n_int8);
int btle_b200_rx_device_dir(btle_b200_ctx *ctx, const int8_t *d_iq, size_t n_streams, size_t stream_stride_int8,
                            size_t n_int8, const btle_stream_cfg *cfgs, btle_pkt_rec *d_out, size_t cap,
                            uint32_t *d_count, btle_unit_dir *d_dir, size_t dir_cap, void *cuda_stream);
int btle_b200_rx_device_dir_offset(btle_b200_ctx *ctx, const int8_t *d_iq, size_t n_streams, size_t stream_stride_int8,
                                   size_t n_int8, const btle_stream_cfg *cfgs, const float *offset_hz, btle_pkt_rec *d_out, size_t cap,
                                   uint32_t *d_count, btle_unit_dir *d_dir, size_t dir_cap, void *cuda_stream);
/* Same with the directory kept in context-owned scratch: for callers that only want the set of records
 * (btle_b200_sort_records() on the host copy gives reference order). */
int btle_b200_rx_device(btle_b200_ctx *ctx, const int8_t *d_iq, size_t n_streams, size_t stream_stride_int8,
                        size_t n_int8, const btle_stream_cfg *cfgs, btle_pkt_rec *d_out, size_t cap,
                        uint32_t *d_count, void *cuda_stream);
void btle_b200_sort_records(btle_pkt_rec *recs, size_t n);
/* ---- several access addresses per capture, one read of the IQ --------------------------------------------------------
 * cfg j decodes capture cfg_capture[j].  cfg_capture is non-decreasing and lies in [0, n_captures), with at most
 * BTLE_MAX_CFGS_PER_CAPTURE cfgs per capture; a capture that no cfg names is not read.  Every cfg field applies per cfg
 * (two cfgs of one capture may differ in any of them, the access address included or not).  The result equals
 * btle_b200_rx_batch() on a batch whose stream j is a copy of capture cfg_capture[j] decoded with cfgs[j]: every record
 * field is equal, stream == j included, in (j, chunk, n0) order.  Each capture's IQ is turned into discriminator bits
 * once, whatever the number of cfgs reading it; the prefilter flags the union of the cfgs' candidates, and every
 * candidate is re-checked exactly per cfg.  Argument errors (a cfg_capture that decreases, leaves the range or names one
 * capture more than BTLE_MAX_CFGS_PER_CAPTURE times; the alignment and stride rules of the calls above) are BTLE_EINVAL
 * with btle_b200_last_error() set, and the context stays usable; BTLE_EOVERFLOW reports the needed count in *n_out.
 * A cfg_capture that maps cfg j to capture j for every capture is the launch of btle_b200_rx_batch / _rx_device_dir (same
 * kernel, same directory); btle_b200_rx_multi copies only the captures named, so there a list that names each of them
 * once is that launch too. */
#define BTLE_MAX_CFGS_PER_CAPTURE 8
int btle_b200_rx_multi(btle_b200_ctx *ctx, const int8_t *iq, size_t n_captures, size_t stream_stride_int8, size_t n_int8,
                       const btle_stream_cfg *cfgs, const int32_t *cfg_capture, size_t n_cfgs, btle_pkt_rec *out, size_t cap,
                       size_t *n_out);
/* with carrier-offset correction: offset_hz[c] for capture c (host array of n_captures), shared by capture c's cfgs */
int btle_b200_rx_multi_offset(btle_b200_ctx *ctx, const int8_t *iq, size_t n_captures, size_t stream_stride_int8, size_t n_int8,
                              const btle_stream_cfg *cfgs, const int32_t *cfg_capture, size_t n_cfgs, const float *offset_hz,
                              btle_pkt_rec *out, size_t cap, size_t *n_out);
/* directory entries of an rx_multi launch of this shape (0 for an invalid cfg_capture) */
size_t btle_b200_rx_multi_units(const btle_b200_ctx *ctx, size_t n_captures, const int32_t *cfg_capture, size_t n_cfgs, size_t n_int8);
/* device-resident form; directory, d_count (may be NULL: counter ring) and streams exactly as btle_b200_rx_device_dir():
 * walking d_dir in index order gives the records in (j, chunk, n0) order, so btle_b200_gather_ordered() applies. */
int btle_b200_rx_multi_device_dir(btle_b200_ctx *ctx, const int8_t *d_iq, size_t n_captures, size_t stream_stride_int8,
                                  size_t n_int8, const btle_stream_cfg *cfgs, const int32_t *cfg_capture, size_t n_cfgs,
                                  btle_pkt_rec *d_out, size_t cap, uint32_t *d_count, btle_unit_dir *d_dir, size_t dir_cap,
                                  void *cuda_stream);
int btle_b200_rx_multi_device_dir_offset(btle_b200_ctx *ctx, const int8_t *d_iq, size_t n_captures, size_t stream_stride_int8,
                                         size_t n_int8, const btle_stream_cfg *cfgs, const int32_t *cfg_capture, size_t n_cfgs,
                                         const float *offset_hz, btle_pkt_rec *d_out, size_t cap, uint32_t *d_count, btle_unit_dir *d_dir,
                                         size_t dir_cap, void *cuda_stream);
/* Per-packet carrier-offset estimate, one float per record (the record itself is not changed).  Record r's capture is
 * `stream` (records of btle_b200_rx_batch / rx_device_dir over the same captures); its samples are read with recovery's
 * window rule (outside [8192 chunk, 8192 chunk + 9696) or outside the capture: 0).  With z[n] = conj(x[n]) x[n+1]:
 *     hz[r] = 4e6 / (2 pi 156) * sum_{n = n0-32 .. n0+123} (atan2(Im z[n], Re z[n]) - ref[n - n0])
 * ref = the same turns of the noiseless btle_tx waveform (the 4-sps modulator of btle_b200_tx_modulate_device, int8 table
 * samples) of the packet's preamble and access address, tx sample BTLE_RX_BER_AA_OFFSET at n0: the preamble and access
 * address, up to 4 samples before the header, whose first bit the Gaussian filter lets into later turns.  So a noiseless
 * packet of the project's own transmitter, aligned, estimates 0.  Device form: d_iq (captures stride apart), d_recs and
 * d_hz device pointers, enqueued on cuda_stream, one warp per record; a record with chunk < 0 reads no sample (every
 * sample 0), so it never reads in front of its capture.  Host form: host buffers, synchronised; BTLE_EINVAL (and
 * btle_b200_last_error set) for a record whose stream is outside [0, n_streams) or whose chunk is negative. */
int btle_b200_rec_offset_device(btle_b200_ctx *ctx, const int8_t *d_iq, size_t stream_stride_int8, size_t n_int8, const btle_pkt_rec *d_recs,
                                size_t n, float *d_hz, void *cuda_stream);
int btle_b200_rec_offset(btle_b200_ctx *ctx, const int8_t *iq, size_t n_streams, size_t stream_stride_int8, size_t n_int8,
                         const btle_pkt_rec *recs, size_t n, float *hz);
/* Host helper: recs[0..n_recs) and dir[0..n_units) are host copies of a launch's d_out / d_dir; copies the
 * records into out[] in reference order.  *n_out = sum of the directory counts; BTLE_EOVERFLOW if that exceeds
 * `cap` or if blocks were cut off by n_recs (out then holds what was available, still in order). */
int btle_b200_gather_ordered(const btle_pkt_rec *recs, size_t n_recs, const btle_unit_dir *dir, size_t n_units,
                             btle_pkt_rec *out, size_t cap, size_t *n_out);
/* ---- streaming session: ONE capture of unbounded length (file, pipe, radio), pushed in pieces -------------------
 * The library cuts the stream into segments of `segment_chunks` chunks (0 = default 4096 = 64 MiB) and double-buffers
 * them: while the GPU copies / decodes segment i out of one page-locked buffer, the caller fills the other with
 * segment i+1 (btle_b200_stream_acquire() hands out that buffer directly, so a file can be read() straight into
 * page-locked memory; btle_b200_stream_push() is the copying convenience form).  Capture size is therefore bounded
 * neither by host RAM nor by HBM.  Records come back in the reference's order, `chunk` counted from the start of the
 * stream, as segments complete (the calls return how many they stored; they never block on the segment just handed
 * over).  Chunk semantics are the batch entry points': a chunk exists once its 16384 int8 are there, decode reads up
 * to 3008 int8 behind it, bytes behind the end of the stream read as 0. */
typedef struct btle_b200_stream btle_b200_stream;
int btle_b200_stream_open(btle_b200_ctx *ctx, const btle_stream_cfg *cfg, size_t segment_chunks, btle_b200_stream **out);
int btle_b200_stream_acquire(btle_b200_stream *s, int8_t **buf, size_t *space);       /* where to put the next bytes    */
int btle_b200_stream_commit(btle_b200_stream *s, size_t n_int8, btle_pkt_rec *out, size_t cap, size_t *n_out);
int btle_b200_stream_push(btle_b200_stream *s, const int8_t *iq, size_t n_int8, btle_pkt_rec *out, size_t cap, size_t *n_out);
/* retune: channel / access address / CRC init used from the next segment on (hop following on a live stream) */
int btle_b200_stream_set_cfg(btle_b200_stream *s, const btle_stream_cfg *cfg);
/* carrier-offset correction (BTLE_MAX_OFFSET_HZ) of the capture, from the next submitted segment on: btle_b200_streams_set_offset */
int btle_b200_stream_set_offset(btle_b200_stream *s, float offset_hz);
/* end of stream: decodes the tail, returns what is left (BTLE_EOVERFLOW: call again, more records are waiting) */
int btle_b200_stream_finish(btle_b200_stream *s, btle_pkt_rec *out, size_t cap, size_t *n_out);
void btle_b200_stream_close(btle_b200_stream *s);

/* ---- streaming session over N time-aligned captures (one per radio / channel), each pushed in pieces ---------------
 * Defined to equal btle_b200_rx_batch() on the same captures, each cut to the length of the shortest.  The captures are
 * cut into segment SETS: `segment_chunks` chunks of every capture (0 = default max(16, round_up(4096 / n_streams, 16)),
 * so that one half holds about 64 MiB whatever N is).  A set is decoded, in ONE batched launch over the N captures, once
 * every capture has filled its part (its segment plus the look-ahead); while the GPU decodes it, the caller fills the
 * other half.  btle_b200_streams_acquire() hands out where capture `stream`'s next bytes go (page-locked memory, so a
 * file or FIFO can be read() straight into it); *space == 0 means that capture's part is complete and the session waits
 * for the others.  Records come back per set in (stream, chunk, n0) order, `stream` = index in the session, `chunk`
 * counted from the start of the capture; records that do not fit `cap` wait for the next call (none are dropped).
 * btle_b200_streams_finish() decodes the complete chunks up to the SHORTEST capture's end; in that last set bytes behind
 * that length read as 0 for every capture.  It returns BTLE_EOVERFLOW while records are still waiting: call it again.
 * btle_b200_streams_set_cfg() applies from the next set that is submitted.  BTLE_EINVAL (with btle_b200_last_error()
 * set) for n_streams == 0, a stream index out of range, a commit of more bytes than acquired and a bad cfg; the session
 * stays usable after the last three.  btle_b200_stream_* above is this session with one capture. */
typedef struct btle_b200_streams btle_b200_streams;
int btle_b200_streams_open(btle_b200_ctx *ctx, const btle_stream_cfg *cfgs, size_t n_streams, size_t segment_chunks,
                           btle_b200_streams **out);
int btle_b200_streams_acquire(btle_b200_streams *s, size_t stream, int8_t **buf, size_t *space);
int btle_b200_streams_commit(btle_b200_streams *s, size_t stream, size_t n_int8, btle_pkt_rec *out, size_t cap, size_t *n_out);
int btle_b200_streams_set_cfg(btle_b200_streams *s, size_t stream, const btle_stream_cfg *cfg);
/* Carrier-offset correction (BTLE_MAX_OFFSET_HZ) of capture `capture`, shared by all its cfgs, used from the next submitted
 * segment set on, like set_cfg.  From the first call on, every set of the session is decoded by the rotated kernel (the
 * other captures at offset 0, which returns the default kernel's records), and a set keeps the offsets it was submitted
 * with, also for a backfill of cfgs added later.  So a record of chunk k equals that of btle_b200_rx_batch_offset on the
 * whole captures at the offsets in force when the set holding chunk k was submitted. */
int btle_b200_streams_set_offset(btle_b200_streams *s, size_t capture, float offset_hz);
int btle_b200_streams_finish(btle_b200_streams *s, btle_pkt_rec *out, size_t cap, size_t *n_out);
void btle_b200_streams_close(btle_b200_streams *s);

/* ---- connection discovery: empty-PDU candidates on data-channel captures, no access address given ------------------
 * Connections whose CONNECT_REQ was not captured are found from their data packets: every idle connection event carries
 * an empty PDU, whose header is fixed but for 3 bits and which is never encrypted.  Sample n0 of a capture on data
 * channel `ch` (0..36) is a CANDIDATE iff, with d[n] = (I[n]Q[n+1] - I[n+1]Q[n]) > 0:
 *   - the 9 bits d[n0 - 32 + 4j] (j = 0..7) and d[n0] alternate (preamble 0x55 or 0xAA);
 *   - the 16 bits d[n0 + 4(32 + j)] (j = 0..15), LSB first, dewhitened with the first 16 whitening bits of `ch`, have
 *     LLID 1 (bits 0..1) and byte 1 == 0 (length 0, RFU 0);
 *   - every d[n] read lies inside the capture: n0 >= 32 and n0 + 285 < n_int8 / 2.
 * Every sample index is tested; one packet usually gives 2-3 candidates at adjacent n0.  access_addr = d[n0 + 4i]
 * (i = 0..31) LSB first; crc_init is the unique -k value for which the CRC-24 of the two header bytes equals the
 * received CRC d[n0 + 4(48 + j)] (j = 0..23) dewhitened with whitening bits 16..39 (the LFSR is run backwards).
 * For a packet that btle_b200_rx_batch() decodes with that access address and CRC init, sample == chunk * 8192 + n0
 * of its record. */
typedef struct {
  int64_t sample;        /* n0: first IQ sample of the access address, from the start of the capture            */
  int32_t stream;
  uint32_t access_addr;
  uint32_t crc_init;     /* -k convention (not reordered)                                                      */
  uint8_t channel;
  uint8_t header[2];     /* dewhitened: LLID 1, length 0                                                       */
  uint8_t reserved[9];
} btle_conn_cand;        /* 32 bytes */
/* device: `d_iq` 16-byte aligned, stride a multiple of 16 and >= n_int8 when n_streams > 1; channels[s] (host array) is
 * the data channel of capture s.  Candidates are unordered; *d_count (zeroed by the call) = number found,
 * d_out[0..min(count, cap)) holds them.  Enqueued on cuda_stream, not synchronised.  n_streams == 0 and captures too
 * short for one window give 0 candidates.  A channel outside 0..36, a misaligned pointer or stride or a missing buffer
 * is BTLE_EINVAL with btle_b200_last_error() set. */
int btle_b200_discover_device(btle_b200_ctx *ctx, const int8_t *d_iq, size_t n_streams, size_t stream_stride_int8,
                              size_t n_int8, const int32_t *channels, btle_conn_cand *d_out, size_t cap,
                              uint32_t *d_count, void *cuda_stream);
/* host buffers (page-locked or pageable, as btle_b200_rx_batch); out sorted by (stream, sample).  BTLE_EOVERFLOW with
 * *n_out = the number found when that exceeds cap (out then holds cap of them, not necessarily the first ones). */
int btle_b200_discover(btle_b200_ctx *ctx, const int8_t *iq, size_t n_streams, size_t stream_stride_int8, size_t n_int8,
                       const int32_t *channels, btle_conn_cand *out, size_t cap, size_t *n_out);

/* ---- LE Coded PHY (long range, BLE 5): a receiver beside the 1M one, on the same 4-Msps int8 captures --------------
 * Not part of the reference.  The coded PHY sends the same 1 Msym/s GFSK on the same channels; its access address is
 * convolutionally coded and spread, so the 1M search never matches it.  Transmitter (Core Spec v5.x, Vol 6 Part B
 * §2.2, §3.3; btle_b200/synth.py coded_symbols):
 *   preamble  80 symbols, 10 x 0,0,1,1,1,1,0,0 in transmit order
 *   block 1   access address (32 bits, LSB first), CI (2 bits, LSB first: 0 S=8, 1 S=2, 2 and 3 reserved), TERM1 (3 zero
 *             bits); always S=8: 37 bits -> 74 coded bits -> 296 symbols
 *   block 2   PDU (16-bit header, byte 1 = length L, 8 bits; then L = 0..255 payload bytes), CRC-24, TERM2 (3 zero bits),
 *             at the S given by CI: (16 + 8L + 27) * S symbols
 *   order     CRC over the PDU, whitening of PDU + CRC (channel LFSR, as for 1M), FEC, pattern mapping; AA, CI and TERM are
 *             not whitened
 *   FEC       K = 4, rate 1/2, G0 = 1 + x + x^2 + x^3, G1 = 1 + x^2 + x^3; per input bit a0 is sent, then a1.  The state is
 *             zero at the start of block 1, and TERM1 returns it to zero for block 2
 *   mapper    S=8: coded bit 0 -> 0,0,1,1 and 1 -> 1,1,0,0; S=2: the coded bit as it is
 * Receiver (btle_b200_rx_coded*).  Positions are absolute samples of the capture; x outside the capture reads 0.
 *   discriminator  the BTLE_CFG_SYMBOL_SPACED | BTLE_CFG_LOWPASS one, always rotated: F[n] = (x[n-1] + 2 x[n] + x[n+1]) >> 2
 *             per rail, v[n] = C4 (FI[n-2] FQ[n+2] - FI[n+2] FQ[n-2]) - S4 (FI[n-2] FI[n+2] + FQ[n-2] FQ[n+2]) (int32), (C4,
 *             S4) from the capture's offset_hz as for the *_offset entry points ((16384, 0) without one).  Hard bit h[n] =
 *             v[n] > 0, soft value y[n] = clamp(v[n] >> 22, -127, 127).  There are no mode flags.
 *   symbols   symbol j relative to the access address is read at n0 + 4j; the preamble is j = -80..-1.
 *   search    P = the 336 known symbols j = -80..255: the preamble and the block-1 coding of the cfg's access address
 *             (fixed: the encoder starts at zero).  D(n0) = #{j = -80..255 : h[n0 + 4j] != P[j]}, defined only where
 *             the window lies inside the capture: n0 >= 323 and n0 + 1023 < n_samples.  n0 is a HIT iff D(n0) <=
 *             BTLE_CODED_MAX_DIST, D(n0) < D(m) for every defined m in [n0 - 8, n0 - 1] and D(n0) <= D(m) for every
 *             defined m in [n0 + 1, n0 + 8].  Each hit gives exactly one record (two hits are at least 9 samples apart).
 *   CI        from the state after the access address (its last 3 bits), code (c0, c1, 0, 0, 0) for c = 0..3 into the
 *             40 symbols j = 256..295; M(c) = sum (2 sym - 1) y.  The largest M wins, the lower c on a tie.  c >= 2: a
 *             record flagged BTLE_CODED_CI_RESERVED with s = 0, n_bytes = 0, crc_bad = 1.
 *   soft bits block 2 starts at j = 296.  Coded bit k reads 1 symbol (S=2: L = y) or 4 (S=8: L = y0 + y1 - y2 - y3).
 *   Viterbi   branch metric (2 a0 - 1) L0 + (2 a1 - 1) L1, maximised; state s = b[t-1] | b[t-2] << 1 | b[t-3] << 2; on
 *             equal metrics the predecessor with the lower index wins.  int32 metrics (|metric| <= 2.2e6; the states not
 *             yet reachable start at -2^29).
 *   header    Viterbi over info bits 0..39 from state 0, traced back from the best final state (lowest index on a tie);
 *             bits 0..15 dewhitened give the header, L = byte 1.
 *   full      Viterbi over 16 + 8L + 27 info bits from state 0, traced back from state 0; the bits dewhitened give header +
 *             payload + CRC, n_bytes = L + 5; crc_bad compares the CRC-24 (crc_init, -k convention) with the received CRC.
 *             The first 40 steps are the header pass's, so one trellis serves both.
 *   truncated a record whose symbols (up to j = 295 when CI is reserved, else the last of block 2) read a sample at or past
 *             the capture's end (n0 + 4 j + 3 >= n_samples) is flagged BTLE_CODED_TRUNCATED; those samples read 0.
 * Conformance rests on these rules: no third-party coded-PHY test vector was available.  tests/test_coded.py pins the
 * encoder's impulse response and a hand-checked preamble and block-1 layout. */
#define BTLE_CODED_MAX_DIST 96
#define BTLE_CODED_CI_RESERVED 1   /* btle_coded_rec.flags: CI 2 or 3, nothing decoded                                  */
#define BTLE_CODED_TRUNCATED 2     /* btle_coded_rec.flags: the packet runs past the capture's end (read as 0)          */
#define BTLE_CODED_MAX_BYTES 260   /* header + 255 payload bytes + CRC                                                */
typedef struct {
  int64_t sample;        /* n0: first sample of the access address (symbol j = 0), from the start of the capture        */
  int32_t stream;
  uint32_t access_addr;
  uint8_t channel;
  uint8_t s;             /* 8 or 2; 0 when CI is reserved                                                             */
  uint8_t ci;            /* 0..3                                                                                       */
  uint8_t crc_bad;
  uint8_t flags;         /* BTLE_CODED_CI_RESERVED, BTLE_CODED_TRUNCATED                                              */
  uint8_t reserved0;
  uint16_t n_bytes;      /* L + 5, 0 when CI is reserved                                                              */
  int32_t dist;          /* D(n0)                                                                                     */
  int32_t metric;        /* final metric of the full pass (state 0)                                                   */
  uint32_t mag_sum;      /* sum |I| + |Q| over samples n0 .. n0 + 1023 with BTLE_CFG_RSSI, else 0                       */
  uint8_t bytes[BTLE_CODED_MAX_BYTES];   /* dewhitened header + payload + CRC, zero beyond n_bytes                    */
  uint8_t reserved[8];
} btle_coded_rec;        /* 304 bytes */
/* device: `d_iq` 16-byte aligned, stride a multiple of 16 and >= n_int8 when n_streams > 1; cfgs[s] (host array) is the
 * access address, CRC init and channel of capture s; offset_hz (host array, NULL = 0) its carrier offset.  Records are
 * unordered; *d_count (zeroed by the call) = the number found, d_out[0 .. min(count, cap)) holds that many of them (not
 * necessarily the first ones: d_out also holds the hits between the two kernels, so no hit is dropped unseen).
 * Enqueued on cuda_stream, not synchronised.  BTLE_EINVAL with btle_b200_last_error() set: a channel outside 0..39, raw,
 * access_mask != 0xFFFFFFFF, an rssi flag other than BTLE_CFG_RSSI (the 1M opt-in flags mean nothing here and are
 * refused), an offset that is not finite or exceeds BTLE_MAX_OFFSET_HZ, a misaligned pointer or stride, a missing
 * buffer. */
int btle_b200_rx_coded_device(btle_b200_ctx *ctx, const int8_t *d_iq, size_t n_streams, size_t stream_stride_int8,
                              size_t n_int8, const btle_stream_cfg *cfgs, const float *offset_hz, btle_coded_rec *d_out,
                              size_t cap, uint32_t *d_count, void *cuda_stream);
/* host buffers (page-locked or pageable, as btle_b200_rx_batch); out sorted by (stream, sample) on the device before the
 * copy.  BTLE_EOVERFLOW with *n_out = the number found when that exceeds cap (out then holds cap of them); a second call
 * with cap >= *n_out returns them all. */
int btle_b200_rx_coded(btle_b200_ctx *ctx, const int8_t *iq, size_t n_streams, size_t stream_stride_int8, size_t n_int8,
                       const btle_stream_cfg *cfgs, const float *offset_hz, btle_coded_rec *out, size_t cap, size_t *n_out);
/* Several cfgs per capture, each capture read once (as btle_b200_rx_multi for 1M): cfg j decodes capture cfg_capture[j]
 * (non-decreasing, in range, at most BTLE_MAX_CFGS_PER_CAPTURE cfgs per capture; captures no cfg names are not read).
 * offset_hz (host array, NULL = 0) has one entry per capture, shared by all cfgs of that capture.  The result equals
 * btle_b200_rx_coded on a batch whose stream j is a copy of capture cfg_capture[j], decoded with cfgs[j] and
 * offset_hz[cfg_capture[j]]: every field of every record is equal, and `stream` is the cfg index j.  The device form
 * returns the records unordered with the exact count in *d_count, as btle_b200_rx_coded_device; the host form copies
 * only the captures some cfg names and returns the records in (j, sample) order, BTLE_EOVERFLOW with the exact count as
 * btle_b200_rx_coded.  Each cfg is checked as in btle_b200_rx_coded_device, and a bad cfg_capture is BTLE_EINVAL too.
 * btle_b200_rx_coded and _rx_coded_device are these calls with cfg_capture[j] = j. */
int btle_b200_rx_coded_multi(btle_b200_ctx *ctx, const int8_t *iq, size_t n_captures, size_t stream_stride_int8, size_t n_int8,
                             const btle_stream_cfg *cfgs, const int32_t *cfg_capture, size_t n_cfgs, const float *offset_hz,
                             btle_coded_rec *out, size_t cap, size_t *n_out);
int btle_b200_rx_coded_multi_device(btle_b200_ctx *ctx, const int8_t *d_iq, size_t n_captures, size_t stream_stride_int8,
                                    size_t n_int8, const btle_stream_cfg *cfgs, const int32_t *cfg_capture, size_t n_cfgs,
                                    const float *offset_hz, btle_coded_rec *d_out, size_t cap, uint32_t *d_count,
                                    void *cuda_stream);

/* ---- Coded connection discovery: empty coded PDUs on data-channel captures, no access address given -----------------
 * Not part of the reference.  The coded connections whose AUX_CONNECT_REQ was not captured are found from the empty PDUs
 * of their idle events, as btle_b200_discover finds 1M ones.  Discriminator, positions, hard bits h, soft values y and
 * the trellis are the coded receiver's ("LE Coded PHY" above).  On a capture of n_samples samples:
 *   search    for every n0 with 323 <= n0 and n0 + 1184 <= n_samples (the preamble and block 1 inside the capture):
 *             Dpre(n0) = #{j = -80..-1 : h[n0 + 4j] != preamble[j]}; C(n0) = sum over the 74 groups k = 0..73 of block 1
 *             (symbols j = 4k..4k+3, s0..s3) of the Hamming distance to the nearer of 0,0,1,1 and 1,1,0,0, i.e.
 *             [s0 != s1] + [s2 != s3] + 2 [s0 = s1 = s2 = s3] (no access address needed); Q(n0) = Dpre(n0) + C(n0).
 *   hit       Dpre(n0) <= BTLE_CODED_DISC_T_PRE, Q(n0) <= BTLE_CODED_DISC_T_Q, Q(n0) < Q(m) for every defined m in
 *             [n0 - W, n0 - 1] and Q(n0) <= Q(m) for every defined m in [n0 + 1, n0 + W], W = BTLE_CODED_DISC_W.  The
 *             preamble repeats every 8 symbols (32 samples) and the S=8 mapper looks the same at every 4-symbol step, so
 *             one packet makes a ladder of low Q every 32 samples; W spans it.  Two hits are more than W samples apart.
 *   align     for k = -K..K (K = BTLE_CODED_DISC_K), m = n0 + 32k with m inside the search range: score(m) = the soft
 *             correlation sum_{j=-80..-1} (2 preamble[j] - 1) y[m + 4j] plus the metric of state 0 after the 37 block-1
 *             steps (S=8 soft values of symbols 0..295, the trellis from state 0; TERM1 ends block 1 in state 0).  The
 *             largest score wins, the lowest k on a tie.  Its traceback from state 0 gives the access address (info bits
 *             0..31) and CI (bits 32..33).  CI 2 or 3: no candidate.  2 * 32 K < W + 1, so two hits never give one m.
 *   PDU       block 2 at the S of CI: 43 steps (16 header + 24 CRC + 3 TERM bits) from state 0, traced back from state
 *             0; bits 0..39 dewhitened with the channel's whitening bits 0..39 are the header and the received CRC.
 *             Every sample read must lie inside the capture (m + 4 (296 + 86 S/2 - 1) + 3 < n_samples with S/2 the
 *             symbols per coded bit over 2: 4 at S=8, 1 at S=2) or there is no candidate.  A CANDIDATE needs LLID 1 and
 *             byte 1 == 0 (btle_b200_discover's header rule); crc_init is the unique -k value whose CRC-24 of the two
 *             header bytes equals the received CRC.
 * For a noiseless coded empty PDU of the project's transmitter, sample is the n0 of btle_b200_rx_coded's record. */
#define BTLE_CODED_DISC_T_PRE 24
#define BTLE_CODED_DISC_T_Q 80
#define BTLE_CODED_DISC_W 256
#define BTLE_CODED_DISC_K 4
typedef struct {
  int64_t sample;        /* m: first sample of the access address (symbol j = 0), from the start of the capture         */
  int32_t stream;
  uint32_t access_addr;
  uint32_t crc_init;     /* -k convention (not reordered)                                                              */
  uint8_t channel;
  uint8_t header[2];     /* dewhitened: LLID 1, length 0                                                               */
  uint8_t s;             /* 8 or 2                                                                                     */
  int16_t dist;          /* Q of the hit                                                                               */
  int8_t shift;          /* the chosen k: sample = hit + 32 k                                                          */
  uint8_t reserved;
  int32_t metric;        /* metric of state 0 after block 2's 43 steps                                                 */
} btle_coded_cand;       /* 32 bytes; its first 23 bytes are laid out as btle_conn_cand's */
/* device: d_iq 16-byte aligned, stride a multiple of 16 and >= n_int8 when n_streams > 1; channels[s] (host array) the
 * data channel of capture s (0..36); offset_hz (host array, NULL = 0) its carrier offset (<= BTLE_MAX_OFFSET_HZ).
 * Candidates are unordered; *d_count (zeroed by the call) = the number found, d_out[0 .. min(count, cap)) holds that many
 * (not necessarily the first ones).  Enqueued on cuda_stream, not synchronised; the cfg cache is shared with the other
 * launches as described for btle_b200_rx_device_dir.  BTLE_EINVAL with btle_b200_last_error() set: a channel outside
 * 0..36, an offset that is not finite or too large, a misaligned pointer or stride, a missing buffer. */
int btle_b200_discover_coded_device(btle_b200_ctx *ctx, const int8_t *d_iq, size_t n_streams, size_t stream_stride_int8,
                                    size_t n_int8, const int32_t *channels, const float *offset_hz, btle_coded_cand *d_out,
                                    size_t cap, uint32_t *d_count, void *cuda_stream);
/* host buffers (page-locked or pageable); out sorted by (stream, sample) on the device before the copy.  BTLE_EOVERFLOW
 * with *n_out = the number found when that exceeds cap; a second call with cap >= *n_out returns them all. */
int btle_b200_discover_coded(btle_b200_ctx *ctx, const int8_t *iq, size_t n_streams, size_t stream_stride_int8, size_t n_int8,
                             const int32_t *channels, const float *offset_hz, btle_coded_cand *out, size_t cap, size_t *n_out);

/* ---- connections on a streaming session (btle_b200_streams_*): per-capture cfg lists, backfill, discovery -----------
 * Every cfg of a session has a stable index, never reused: the n_streams cfgs of btle_b200_streams_open are 0..n-1 (cfg
 * i decodes capture i), each added cfg gets the next one.  A record's `stream` is that index.  The records of cfg j equal
 * btle_b200_rx_batch() on cfg j's capture (cut to the shortest capture) decoded with cfg j, kept for
 * from_chunk <= chunk < until_chunk; each is returned exactly once, per set in (j, chunk, n0) order.
 * A set's live cfgs are sorted by capture and decoded in rounds of at most BTLE_MAX_CFGS_PER_CAPTURE cfgs per capture,
 * one btle_b200_rx_multi_device_dir launch per round (so a round of one cfg per capture in capture order, as every set
 * of a session whose cfg list never changed has, is the single-cfg launch described above).  A capture no live cfg names
 * is not read by the kernel.
 * BACKFILL: the two most recent sets stay on the device (the one whose records were handed out last, and the one in
 * flight).  add_cfg accepts any from_chunk >= btle_b200_streams_resident(); the next commit or finish call decodes every
 * cfg added since the last one over the resident sets that hold chunks >= its from_chunk (rounds of at most
 * BTLE_MAX_CFGS_PER_CAPTURE cfgs per capture, one launch each), and those records are handed out by that call or, for
 * the set in flight, with it (finish returns them until none wait; btle_b200_last_launches counts these launches too).
 * add_cfg does no GPU work: it fails only on bad arguments, and then adds nothing.  from_chunk < resident() is
 * BTLE_EINVAL, the session stays usable.  Device record buffers are sized per launch for BTLE_MAX_RECS_PER_CHUNK records
 * per chunk and cfg and reused by later launches; page-locked host memory holds only the records found. */
int btle_b200_streams_add_cfg(btle_b200_streams *s, size_t capture, const btle_stream_cfg *cfg, int64_t from_chunk, size_t *index);
/* cfg `index` decodes no chunk from the next submitted set on; *until_chunk = first chunk it no longer decodes.
 * An index out of range or already removed is BTLE_EINVAL. */
int btle_b200_streams_remove_cfg(btle_b200_streams *s, size_t index, int64_t *until_chunk);
/* first chunk of the oldest set whose IQ is still on the device: the smallest from_chunk add_cfg accepts */
int btle_b200_streams_resident(const btle_b200_streams *s, int64_t *first_chunk);
/* DISCOVERY: channels[i] = data channel 0..36 of capture i, or -1 (not scanned); applies from the next submitted set.
 * Each set's scanned parts (lead, segment and look-ahead) go through discover_kernel; the candidates whose window starts
 * in the segment are kept, with `sample` counted from the capture's start and `stream` = capture index.  The union over
 * the sets equals btle_b200_discover() on the whole captures cut to the shortest one; no candidate is dropped. */
int btle_b200_streams_set_discover(btle_b200_streams *s, const int32_t *channels);
/* candidates of the sets handed out so far, per set sorted by (stream, sample); taken ones are not returned again.
 * BTLE_EOVERFLOW when more wait than `cap` holds: call again. */
int btle_b200_streams_take_cands(btle_b200_streams *s, btle_conn_cand *out, size_t cap, size_t *n_out);

/* number of kernels the last rx call launched (bench.py's gpu_launches) */
int btle_b200_last_launches(const btle_b200_ctx *ctx);

/* ---- leaf functions with the reference's signatures (unit parity; each runs on the GPU) ---- */
/* search_unique_bits, btle_rx.c:1510: returns the int8 index of the first AA sample of the
 * first match when scanning `search_len` symbols from rxp with a zeroed history, or -1.
 * unique_bits / unique_bits_mask are 32 bytes of 0/1, LSB first (uint32_to_bit_array, :798).
 * A masked position whose unique_bits value is neither 0 nor 1 never matches a demodulated bit (:1539), so the
 * result is then -1.  Reads rxp[0 .. 8*search_len+1]; search_len <= 4096.  Errors: BTLE_SEARCH_ERR(BTLE_E*) (<= -1001). */
int btle_b200_search_unique_bits(btle_b200_ctx *ctx, const int8_t *rxp, int search_len,
                                 const uint8_t *unique_bits, const uint8_t *unique_bits_mask, int num_bits);
/* demod_byte, btle_rx.c:1489: num_byte <= 64 bytes from rxp[0 .. 64*num_byte+3]. */
int btle_b200_demod_byte(btle_b200_ctx *ctx, const int8_t *rxp, int num_byte, uint8_t *out_byte);
/* scramble_byte with scramble_table[channel]+table_offset, btle_rx.c:1232 / scramble_table.h:4. */
int btle_b200_scramble_byte(btle_b200_ctx *ctx, const uint8_t *byte_in, int num_byte, int channel,
                            int table_offset, uint8_t *byte_out);
/* crc24_byte, btle_rx.c:1224 (init_hex already reordered), and crc_init_reorder, :1969.  Any 32-bit init_hex behaves
 * as in the reference: the first byte's step starts from all 32 bits, so bits 24..31 of init_hex fold into bits 16..23,
 * and every step masks to 24 bits; with num_byte 0 the result is init_hex & 0xFFFFFF.  num_byte <= 4096. */
int btle_b200_crc24_byte(btle_b200_ctx *ctx, const uint8_t *byte_in, int num_byte, uint32_t init_hex,
                         uint32_t *crc_out);
uint32_t btle_b200_crc_init_reorder(uint32_t crc_init);
/* parse_adv_pdu_header_byte :1947 / parse_ll_pdu_header_byte :1939 (host-side, pure bit ops). */
void btle_b200_parse_adv_pdu_header_byte(const uint8_t *byte_in, int *pdu_type, int *tx_add, int *rx_add,
                                         int *payload_len);
void btle_b200_parse_ll_pdu_header_byte(const uint8_t *byte_in, int *llid, int *nesn, int *sn, int *md,
                                        int *payload_len);
/* Discriminator bits d[n] = (I[n]Q[n+1]-I[n+1]Q[n]) > 0 for n < n_samples (one byte 0/1 each);
 * reads iq[0 .. 2*n_samples+1] (host pointers). */
int btle_b200_dbits(btle_b200_ctx *ctx, const int8_t *iq, size_t n_samples, uint8_t *d_out);

/* ---- leaf functions with the signatures of the reference's bit-true Python model
 *      (python/btlelib.py; arrays of 0/1 int8 "bits", int16 samples at symbol rate) ------------- */
/* gfsk_demodulation_fixed_point(i, q), btlelib.py:395-400: for k < n-1
 *   signal[k] = int32(i[k])*int32(q[k+1]) - int32(i[k+1])*int32(q[k]),  bit[k] = signal[k] > 0. */
int btle_b200_gfsk_demod_i16(btle_b200_ctx *ctx, const int16_t *i, const int16_t *q, size_t n, int8_t *bit_out,
                             int32_t *signal_out);
/* search_unique_bit_sequence(bit, bit_sequence), btlelib.py:402-412: first index where the
 * sequence occurs, or -1 (also the function's return; errors are <= -2... see BTLE_E*).  Any length m: m == 0
 * returns 0 (the empty window at index 0 matches, also when n == 0), n < m returns -1. */
long btle_b200_search_bit_sequence(btle_b200_ctx *ctx, const int8_t *bit, size_t n, const int8_t *seq, size_t m);
/* crc24_core(bit_in, state_init_bit), btlelib.py:191-219: bit-serial CRC-24 LFSR, 24 result bits. */
int btle_b200_crc24_bits(btle_b200_ctx *ctx, const int8_t *bit_in, size_t n, const int8_t *state_init_bit,
                         int8_t *crc_bits_out);
/* scramble_core(bit_in, channel_number), btlelib.py:226-263: whitening of a bit array.  Any int channel: the
 * register is seeded from channel & 63, as the reference takes bits 5..0 of the integer (64 acts as 0, -1 as 63). */
int btle_b200_scramble_bits(btle_b200_ctx *ctx, const int8_t *bit_in, size_t n, int channel, int8_t *bit_out);

/* ---- the Python model's receiver, batched (BER sweep, BASELINE.json configs[3]) ----------------
 * btlelib.btle_rx(i, q, channel, crc_init_bits, aa_hex) (btlelib.py:414-541) for n_packets
 * windows of n_samples int16 samples each (n_samples a multiple of sps, n_samples/sps <= 2048):
 * symbol-spaced differential demod on each of the `sps` sample phases, exact 32-bit access
 * address search (first index), dewhitening from the PDU on, payload length from 6 (adv) or 5
 * bits, CRC-24 with the reference's clamp of the CRC position, first phase with CRC ok wins,
 * otherwise the values of the last phase that found the access address.  One warp per packet. */
typedef struct {
  int32_t start;         /* symbol index of the access address on the reported phase, -1 = never found */
  uint16_t n_pdu_bits;   /* len(pdu_bit)                                                              */
  uint8_t crc_ok;
  uint8_t phase;         /* sample_phase_idx as returned by btle_rx                                  */
  uint8_t payload_len;   /* num_byte_payload                                                         */
  uint8_t found;         /* 0: access address found on no phase; else 1 + the last phase it was found on
                            (== phase + 1 when crc_ok)                                                 */
  uint8_t pdu[70];       /* pdu_bit packed LSB first                                                 */
} btle_model_rx_rec;     /* 80 bytes */
int btle_b200_model_rx_batch_device(btle_b200_ctx *ctx, const int16_t *d_i, const int16_t *d_q, size_t n_packets,
                                    size_t n_samples, int sps, int channel, uint32_t crc_init, uint32_t access_addr,
                                    btle_model_rx_rec *d_out, void *cuda_stream);
int btle_b200_model_rx_batch(btle_b200_ctx *ctx, const int16_t *i, const int16_t *q, size_t n_packets, size_t n_samples,
                             int sps, int channel, uint32_t crc_init, uint32_t access_addr, btle_model_rx_rec *out);

/* ---- the Python model's receiver as a STREAMING mode over an 8-Msps capture (SURVEY.md §8f-3) -------------------
 * Input: interleaved int16 I,Q at 8 samples per symbol — the format `btle_ll -q` writes (firmware/btle_ll.c:50-51) and
 * python/test_btle_rx_by_captured_iq.py:71-78 reads.  btlelib.btle_rx works on one hand-cut window per packet; here the
 * windows are found on the GPU:
 *   1. sps8_hits_kernel: symbol-spaced differential bits on all 8 ABSOLUTE sample phases (phase = sample index mod 8)
 *      and every position where 32 of them equal the access address (HBM-bound, 4 bytes per sample);
 *   2. hits closer than BTLE_SPS8_MIN_PACKET_SYMBOLS symbols form one cluster (one packet seen on neighbouring
 *      phases); the first hit h of a cluster defines the window [w0, w0 + BTLE_SPS8_WINDOW), w0 = 8 (h / 8 -
 *      BTLE_SPS8_MARGIN_SYMBOLS) clamped to 0 — aligned to 8 samples, so the window's phases are the absolute ones;
 *      clusters whose window does not fit into the capture are dropped;
 *   3. the model receiver (8 phases, first CRC-ok phase wins; one warp per window) on every window, straight out of
 *      the capture;
 *   4. in time order, a window that starts inside the packet accepted before it is skipped.
 * rx == what btlelib.btle_rx returns for that window.  The CPU restatement oracle/btlelib_port.py follows the same four
 * steps and is pinned to the reference's btlelib window by window. */
#define BTLE_SPS8_WINDOW 3072              /* samples = 384 symbols: margin + AA + longest ADV PDU + CRC + slack        */
#define BTLE_SPS8_MARGIN_SYMBOLS 2
#define BTLE_SPS8_MIN_PACKET_SYMBOLS 72    /* access address + header + CRC                                           */
typedef struct {
  int64_t sample;          /* first sample of the access address on the reported phase (absolute, 8 Msps)            */
  int64_t window;          /* first sample of the window the model receiver ran on                                   */
  btle_model_rx_rec rx;
} btle_sps8_rec;           /* 96 bytes */
int btle_b200_rx_sps8(btle_b200_ctx *ctx, const int16_t *iq16, size_t n_samples, int channel, uint32_t crc_init,
                      uint32_t access_addr, btle_sps8_rec *out, size_t cap, size_t *n_out);
/* step 1 alone on a device-resident capture: *d_count (zeroed by the call) = number of hits, d_hits[0..min(count, cap)) =
 * their sample indices in no particular order; enqueued on cuda_stream, not synchronised.  `d_iq16` must be 16-byte
 * aligned (the kernel copies the capture in 16-byte vectors): anything else is BTLE_EINVAL. */
int btle_b200_sps8_hits_device(btle_b200_ctx *ctx, const int16_t *d_iq16, size_t n_samples, uint32_t access_addr,
                               int64_t *d_hits, size_t cap, uint32_t *d_count, void *cuda_stream);

/* ---- BER flow of python/test_btle_ber.py, entirely on the device (BASELINE.json configs[3]) ----------------------
 * n_packets packets of the 39-byte ADV PDU of test_btle_ber.py:27 with random payload bits (:49): CRC-24, whitening,
 * the Python model's 8-sps modulator, add_freq_sampling_error(ppm) (btlelib.py:823-857), add_noise(snr) (:859-871),
 * np.int16() truncation [ber_synth_kernel] -> the model's receiver, one warp per packet [model_rx_batch_kernel] ->
 * the script's error accounting (:62-72: bit errors only in CRC-failed packets) [ber_score_kernel].  Randomness is a
 * hash of (seed, packet, sample), so a run is reproducible and packet k is the same whatever the batch size. */
typedef struct {
  uint64_t seed;
  float snr_db;            /* NaN: BTLE_EINVAL                                                                     */
  float ppm;               /* 0, or -50..50 like test_btle_ber.py; not finite or |ppm| >= 1e6: BTLE_EINVAL         */
  int32_t channel;
  uint32_t crc_init;       /* as -k: 0x555555                                                                      */
  uint32_t access_addr;
  uint32_t reserved;
} btle_ber_cfg;
typedef struct {
  uint64_t packets, pkt_err, bit_err, bit_total, aa_miss;   /* aa_miss: CRC-failed packets whose access address was never found */
  double seconds;          /* device time of the run (CUDA events)                                                 */
} btle_ber_result;
int btle_b200_ber_run(btle_b200_ctx *ctx, const btle_ber_cfg *cfg, size_t n_packets, btle_ber_result *out);
/* the packet source and channel of btle_b200_ber_run alone, for packets first_packet .. first_packet + n_packets - 1 of
 * the run `cfg` describes (the same packets ber_run draws): d_i / d_q [n_packets][BTLE_BER_SAMPLES] int16 (planar, ready
 * for btle_b200_model_rx_batch_device with sps 8), d_truth [n_packets][40] the 39 PDU bytes as sent (byte 39 is not
 * written).  Device pointers; enqueued on cuda_stream, not synchronised. */
#define BTLE_BER_SAMPLES 3024      /* 8 sps x 8 x (1 + 4 + 39 + 3) air bytes + 16 */
int btle_b200_ber_synth_device(btle_b200_ctx *ctx, const btle_ber_cfg *cfg, uint64_t first_packet, size_t n_packets, int16_t *d_i,
                               int16_t *d_q, uint8_t *d_truth, void *cuda_stream);

/* ---- error rates of the 4-Msps receive chain (btle_rx_persistent_kernel), impaired captures scored on the device -----
 * Packet k of a run (k = 0, 1, ...); every draw is a hash of (seed, k, ...), so packet k is the same whatever the batch:
 *   PDU      channels 37..39: header 42 25 + 37 random bytes drawn as btle_b200_ber_run draws them (same truth for the same
 *            seed); channels 0..36: an LL data PDU, header 02 1B (LLID 2, length 27) + 27 random bytes, drawn the same way.
 *   IQ       preamble, access address, PDU + CRC-24 whitened for the channel (cfg's access address / CRC init), the btle_tx
 *            PHY at 4 sps (btle_b200_tx_modulate_device, sps 4): L = 32 * air bytes + 16 samples, times amplitude / 127.
 *   channel  in this order, at packet sample m = 0 .. L-1:
 *            1. clock and carrier error at ppm as btle_b200_ber_run applies it: the waveform read at (m - delta_k)(1 + e),
 *               e = ppm 1e-6, linear interpolation clamped to the first / last sample, then a rotation by
 *               e 2450e6 (1 + e) / 4e6 turns per sample; delta_k = j_k / 4, j_k drawn from 0..3 per packet;
 *            2. an extra carrier offset of cfo_hz / 4e6 turns per sample (1. and 2. are one rotation, turns summed);
 *            3. AWGN, sigma = amplitude / 10^(snr_db / 20) / sqrt 2 per rail, on every sample of the capture;
 *            4. rintf, then saturation to -128..127 (what a radio's int8 ADC delivers).
 *   capture  slot k holds samples [k S, (k+1) S), S = slot_samples >= L; packet k's L samples start at a drawn offset
 *            0 .. S - L of its slot.  Every other sample is noise alone, rounded and saturated the same way.  The capture
 *            of packets first .. first+n-1 starts with slot `first` at sample 0 and is BTLE_RX_BER_CAPTURE_INT8(n, S) int8
 *            long: whole 8192-sample chunks, samples behind slot first+n-1 carrying noise only.
 *   receiver btle_rx_persistent_kernel<1> (btle_b200_rx_device_dir) with BTLE_CFG_REPORT_REJECTED | cfg.flags, mask
 *            0xFFFFFFFF.
 *   scoring  packet k's record is the first record in reference order whose access-address sample chunk * 8192 + n0
 *            lies within +-3 of aa_sample (the synthesiser's access-address position, rounded).  pkt_err: no CRC-ok
 *            counted record; bit errors only in those packets, over the PDU bytes the record and the truth have in common
 *            (a counted record's PDU is its n_bytes - 3 bytes, a rejected one's its 2 header bytes), all 8 n_bytes bits
 *            when there is no record (test_btle_ber.py:62-72, as ber_score_kernel applies them). */
#define BTLE_RX_BER_AA_OFFSET 39       /* tx sample of the first access-address sample the receiver reports (n0)          */
#define BTLE_RX_BER_MATCH 3            /* +- samples between a record's access address and the truth's                     */
#define BTLE_RX_BER_MAX_SLOT 12000     /* largest slot_samples: a run's batches hold whole slots and whole chunks        */
#define BTLE_RX_BER_MAX_UNITS 12272    /* largest unit directory btle_b200_rx_ber_score_device takes                      */
#define BTLE_RX_BER_CAPTURE_INT8(n_packets, slot_samples) \
  ((((uint64_t)(n_packets) * (uint64_t)(slot_samples) + 8191u) / 8192u) * 16384u)
typedef struct {
  uint64_t seed;
  float snr_db;            /* NaN or infinite: BTLE_EINVAL                                                          */
  float ppm;               /* not finite or |ppm| >= 1e6: BTLE_EINVAL                                               */
  float cfo_hz;            /* extra carrier offset; not finite: BTLE_EINVAL                                         */
  int32_t amplitude;       /* 1..127: the transmitted waveform's scale, amplitude / 127                             */
  int32_t slot_samples;    /* L (1520 on channels 37..39, 1200 on 0..36) .. BTLE_RX_BER_MAX_SLOT                   */
  int32_t channel;         /* 0..39                                                                                 */
  uint32_t access_addr;
  uint32_t crc_init;       /* as -k                                                                                 */
  uint32_t flags;          /* any of BTLE_CFG_RECOVER, BTLE_CFG_SYMBOL_SPACED, BTLE_CFG_CENTRE_HITS, BTLE_CFG_CORRECT,
                              BTLE_CFG_LOWPASS and BTLE_CFG_OFFSET_SEARCH (given to the receiver); any other bit:
                              BTLE_EINVAL                                                                             */
  uint32_t reserved;       /* 0                                                                                     */
} btle_rx_ber_cfg;         /* 48 bytes */
typedef struct {
  int64_t aa_sample;       /* first access-address sample, from the start of the capture: slot start + offset +
                              round(BTLE_RX_BER_AA_OFFSET / (1 + e) + delta)                                          */
  int32_t offset;          /* first sample of the packet's L samples in its slot                                    */
  uint32_t clipped;        /* samples of the slot whose I or Q saturated                                            */
  uint8_t n_bytes;         /* PDU bytes: 39 (channels 37..39) or 29                                                  */
  uint8_t delta4;          /* 4 delta_k, 0..3                                                                         */
  uint8_t pdu[39];         /* the PDU as sent (before CRC and whitening); zero behind n_bytes                        */
  uint8_t reserved[7];
} btle_rx_ber_truth;       /* 64 bytes */
typedef struct {
  uint64_t packets, pkt_err, bit_err, bit_total;
  uint64_t aa_miss;        /* no record matched                                                                      */
  uint64_t len_reject;     /* only a BTLE_REC_REJECTED record matched (header length outside 6..37)                  */
  uint64_t crc_ok_wrong;   /* CRC ok, but the PDU differs from the truth (not a packet error, as in the model flow)   */
  uint64_t extra_recs;     /* records matched to no packet                                                           */
  uint64_t extra_crc_ok;   /* of those, counted records with a good CRC                                              */
  uint64_t clipped;        /* saturated samples (I or Q) in the packets' slots                                       */
  double seconds;          /* device time of the run (CUDA events)                                                   */
} btle_rx_ber_result;      /* 88 bytes */
/* n_packets packets 0 .. n_packets-1, in batches sized from free device memory; the result is independent of the batch
 * size (every batch starts on a chunk and slot boundary, and its look-ahead behind the last chunk is the next slots'; with
 * BTLE_CFG_SYMBOL_SPACED a batch also reads the 2 samples in front of it and 2 more behind its look-ahead, with
 * BTLE_CFG_LOWPASS 3 and 3).
 * BTLE_EINVAL with btle_b200_last_error() for: snr_db, ppm or cfo_hz NaN or infinite, |ppm| >= 1e6, amplitude outside
 * 1..127, slot_samples below L or above BTLE_RX_BER_MAX_SLOT, channel > 39, a flags bit other than BTLE_CFG_RECOVER,
 * BTLE_CFG_SYMBOL_SPACED, BTLE_CFG_CENTRE_HITS, BTLE_CFG_CORRECT, BTLE_CFG_LOWPASS and BTLE_CFG_OFFSET_SEARCH, BTLE_CFG_LOWPASS without
 * BTLE_CFG_SYMBOL_SPACED;
 * the context stays usable. */
int btle_b200_rx_ber_run(btle_b200_ctx *ctx, const btle_rx_ber_cfg *cfg, size_t n_packets, btle_rx_ber_result *out);
/* the capture and truth of packets first_packet .. first_packet + n_packets - 1 alone: d_iq (16-byte aligned) receives
 * BTLE_RX_BER_CAPTURE_INT8(n_packets, slot_samples) int8, d_truth n_packets rows.  Device pointers; enqueued on
 * cuda_stream, not synchronised. */
int btle_b200_rx_ber_synth_device(btle_b200_ctx *ctx, const btle_rx_ber_cfg *cfg, uint64_t first_packet, size_t n_packets, int8_t *d_iq,
                                  btle_rx_ber_truth *d_truth, void *cuda_stream);
/* scores the records of one btle_b200_rx_device_dir launch over such a capture (d_recs with room for n_recs records,
 * d_dir its n_units entries, n_units <= BTLE_RX_BER_MAX_UNITS) against d_truth[0 .. n_packets): ADDS this call's counts
 * to the counters of the device struct *d_result (`seconds` is not touched; zero it before the first call).  Records
 * past n_recs count as not returned.  Enqueued on cuda_stream, not synchronised. */
int btle_b200_rx_ber_score_device(btle_b200_ctx *ctx, const btle_rx_ber_truth *d_truth, size_t n_packets, const btle_pkt_rec *d_recs,
                                  size_t n_recs, const btle_unit_dir *d_dir, size_t n_units, btle_rx_ber_result *d_result,
                                  void *cuda_stream);

/* ---- 16-bit IQ ingest (SURVEY.md §8f-3) ------------------------------------------------------------
 * bladeRF SC16Q11 samples are reduced to the receive chain's int8 exactly as the reference's
 * stream_callback does: out = (in >> shift) & 0xFF, shift = 4 (btle_rx.c:307-308).  Host buffers;
 * the conversion runs on the GPU, then the capture goes through the same path as btle_b200_rx(). */
int btle_b200_rx_iq16(btle_b200_ctx *ctx, const int16_t *iq16, size_t n_int16, int shift, const btle_stream_cfg *cfg,
                      btle_pkt_rec *out, size_t cap, size_t *n_out);

/* ---- packet synthesiser (SURVEY.md §8f-1): the transmit PHY as a GPU kernel ---------------------
 * Integer GFSK modulation of n_packets packets given as air bytes (preamble, access address,
 * whitened PDU+CRC; bits LSB first), d_air [n_packets][max_bytes], d_nbytes [n_packets].
 *   sps == 4: gen_sample_from_phy_bit (host/btle-tools/src/btle_tx.c:1022-1063): +-1 impulses every
 *             4th sample, taps {2,11,32,53,60,53,32,11,2}, phase mod 1024, round(127 cos/sin).
 *             d_out_i receives interleaved int8 I,Q: [n_packets][2*(32*max_bytes+16)]; d_out_q unused.
 *   sps == 8: gfsk_modulation_fixed_point (python/btlelib.py:146-189): NRZ preceded by 17 samples of
 *             -1, 17 integer taps, >>1, phase mod 2048.  d_out_i / d_out_q: planar int8
 *             [n_packets][64*max_bytes+16].
 * Samples behind a packet's own 8*nbytes*sps+16 samples are written as 0.  Each d_nbytes[k] is clamped to
 * 0..max_bytes: a longer row is modulated as max_bytes bytes, a negative one as 0 bytes (16 samples).
 * Device pointers; enqueued on cuda_stream, not synchronised. */
int btle_b200_tx_modulate_device(btle_b200_ctx *ctx, const uint8_t *d_air, const int32_t *d_nbytes, size_t n_packets,
                                 size_t max_bytes, int sps, int8_t *d_out_i, int8_t *d_out_q, void *cuda_stream);

/* ---- host-side functions the reference keeps next to receiver(): payload parsers, receiver_status and the
 *      connection follower (btle_b200/csrc/btle_host.cpp; no CUDA involved) ----------------------------------
 * Same argument meaning, return values (0 / -1, control opcode) and printed messages as
 *   int parse_adv_pdu_payload_byte(uint8_t*, int, ADV_PDU_TYPE, void*)   btle_rx.c:1564
 *   int parse_ll_pdu_payload_byte(uint8_t*, int, LL_PDU_TYPE, void*)     btle_rx.c:1741
 * `out` points at the struct matching the PDU type; layouts == the reference's typedefs (:1078-1210). */
typedef struct { uint8_t AdvA[6]; uint8_t Data[31]; } btle_adv_payload_0_2_4_6;      /* ADV_PDU_PAYLOAD_TYPE_0_2_4_6 */
typedef struct { uint8_t A0[6]; uint8_t A1[6]; } btle_adv_payload_1_3;               /* ADV_PDU_PAYLOAD_TYPE_1_3     */
typedef struct {
  uint8_t InitA[6]; uint8_t AdvA[6]; uint8_t AA[4]; uint32_t CRCInit; uint8_t WinSize;
  uint16_t WinOffset, Interval, Latency, Timeout; uint8_t ChM[5]; uint8_t Hop; uint8_t SCA;
} btle_adv_payload_5;                                                                /* ADV_PDU_PAYLOAD_TYPE_5       */
typedef struct { uint8_t payload_byte[40]; } btle_adv_payload_r;                     /* ADV_PDU_PAYLOAD_TYPE_R       */
typedef union { btle_adv_payload_0_2_4_6 t0246; btle_adv_payload_1_3 t13; btle_adv_payload_5 t5; btle_adv_payload_r r; } btle_adv_payload;
typedef struct { uint8_t Data[40]; } btle_ll_data_payload;                           /* LL_DATA_PDU_PAYLOAD_TYPE     */
typedef struct { uint8_t Opcode, WinSize; uint16_t WinOffset, Interval, Latency, Timeout, Instant; } btle_ll_ctrl_payload_0;
typedef struct { uint8_t Opcode; uint8_t ChM[5]; uint16_t Instant; } btle_ll_ctrl_payload_1;
typedef struct { uint8_t Opcode, ErrorCode; } btle_ll_ctrl_payload_2_7_13;
typedef struct { uint8_t Opcode; uint8_t Rand[8]; uint8_t EDIV[2]; uint8_t SKDm[8]; uint8_t IVm[4]; } btle_ll_ctrl_payload_3;
typedef struct { uint8_t Opcode; uint8_t SKDs[8]; uint8_t IVs[4]; } btle_ll_ctrl_payload_4;
typedef struct { uint8_t Opcode; } btle_ll_ctrl_payload_5_6_10_11;
typedef struct { uint8_t Opcode; uint8_t FeatureSet[8]; } btle_ll_ctrl_payload_8_9;
typedef struct { uint8_t Opcode, VersNr; uint16_t CompId, SubVersNr; } btle_ll_ctrl_payload_12;
typedef struct { uint8_t Opcode; uint8_t payload_byte[40]; } btle_ll_ctrl_payload_r;
typedef union {
  btle_ll_data_payload data; btle_ll_ctrl_payload_0 c0; btle_ll_ctrl_payload_1 c1; btle_ll_ctrl_payload_2_7_13 c2; btle_ll_ctrl_payload_3 c3;
  btle_ll_ctrl_payload_4 c4; btle_ll_ctrl_payload_5_6_10_11 c5; btle_ll_ctrl_payload_8_9 c8; btle_ll_ctrl_payload_12 c12; btle_ll_ctrl_payload_r r;
} btle_ll_payload;
int btle_b200_parse_adv_pdu_payload_byte(const uint8_t *payload_byte, int num_payload_byte, int pdu_type, void *adv_pdu_payload);
/* returns -1 (drop), else the control opcode (0 for data PDUs, where the reference's return value is undefined) */
int btle_b200_parse_ll_pdu_payload_byte(const uint8_t *payload_byte, int num_payload_byte, int pdu_type, void *ll_pdu_payload);
uint64_t btle_b200_get_freq_by_channel_number(int channel_number);                   /* btle_rx.c:1006 */
int btle_b200_chm_is_full_map(const uint8_t *chm);                                    /* btle_rx.c:2395 */

/* RECV_STATUS (btle_rx.c:1462-1471) — process-wide like the reference's global `receiver_status`: written by the
 * payload parsers (CONNECT_REQ, LL_CONNECTION_UPDATE_REQ, LL_CHANNEL_MAP_REQ) and by btle_b200_note_packet(),
 * read by btle_b200_receiver_controller(). */
typedef struct {
  int pkt_avaliable;
  int hop;               /* -1 until a CONNECT_REQ was parsed */
  int new_chm_flag;
  int interval;
  uint32_t access_addr;
  uint32_t crc_init;
  int crc_ok;            /* CRC verdict of the most recent counted packet (bool in the reference)            */
  uint8_t chm[5];
  uint8_t reserved;
} btle_receiver_status;
btle_receiver_status *btle_b200_receiver_status(void);
/* what receiver() does to receiver_status for every packet it counts (btle_rx.c:2320-2321) */
void btle_b200_note_packet(const btle_pkt_rec *rec);

/* receiver_controller (btle_rx.c:2403): the connection-following state machine, same signature.  Call it once per
 * processed chunk.  0 wait for a CRC-ok CONNECT_REQ with a full channel map -> 1 wait for the first CRC-ok data
 * packet -> 2 hop `interval - 7 ms` after the last mark -> 3 wait for a packet on the new channel, "skip" after
 * `interval - 4 ms`.  The reference reads the wall clock and retunes its radio from inside; here both are hooks,
 * so the same machine runs on sample time over per-channel captures (the btle_rx_b200 program does that). */
typedef struct {
  int64_t ts_us;
  char event[16];        /* track_start / track_drop / chan_change (btj_emit_hop, btle_json.c:132)               */
  int state_from, state_to, ch, freq_mhz;
  uint32_t access_addr, crc_init;
  int interval_us, hop;
  uint8_t chm[5];
} btle_hop_event;
typedef struct {
  int64_t (*now_us)(void *user);                          /* gettimeofday() of the reference                      */
  int (*set_freq)(void *user, uint64_t freq_hz);          /* board_set_freq(); non-zero = failure (-> returns -1) */
  void (*event)(void *user, const btle_hop_event *ev);    /* btj_emit_hop()                                       */
  void *user;
  int quiet_text;                                         /* quiet_text_flag: no "Hop: ..." lines on stdout       */
} btle_hop_hooks;
void btle_b200_set_hop_hooks(const btle_hop_hooks *hooks);
void btle_b200_hop_reset(void);                           /* state 0, receiver_status as main() initialises it    */
int btle_b200_receiver_controller(void *rf_dev, int verbose_flag, int *chan, uint32_t *access_addr, uint32_t *crc_init_internal);

/* ---- capture synthesiser (benchmark / test input; SURVEY.md §8d C2-C5) -----------------------------------
 * Fills n_streams device captures with a noise floor and one burst per `slot_samples` slot: an ADV_IND (TxAdd = 1,
 * AdvA = slot | stream << 32, 0..31 bytes of AdvData) on channels 37..39, an LL data PDU (0..27 bytes) elsewhere,
 * with the stream's access address / CRC init, CRC-24 + whitening + the btle_tx PHY (btle_tx.c:1022-1063) at
 * `amplitude`/127, added to the floor with saturation.  Every `corrupt_every`-th burst gets one flipped bit (its
 * CRC must fail), every `straddle_every`-th is placed ACROSS an 8192-sample chunk boundary (its decode needs the
 * look-ahead behind the chunk).  All randomness is a hash of (seed, stream, position): reproducible, no state.
 * d_truth (optional, [n_streams][n_slots]) receives what was sent. */
typedef struct {
  uint64_t seed;
  int32_t slot_samples;    /* >= 1600 (>= 3200 when straddle_every > 0)                                  */
  int32_t amplitude;       /* 0..127; 0 = no bursts                                                      */
  int32_t corrupt_every;   /* 0 = never                                                                  */
  int32_t straddle_every;  /* 0 = never, else >= 2                                                       */
  int32_t noise;           /* 0: floor of the reference capture (sigma 0.8 LSB, mean -0.3, clip -7..6);
                              1: full-scale uniform int8 (hot interferer); 2: none                       */
  int32_t reserved;
} btle_synth_cfg;
typedef struct {
  int64_t start_sample;    /* first sample of the preamble; the access address starts 39 samples later
                              at the receiver (32 preamble samples + modulator delay)                     */
  int32_t stream, slot;
  uint8_t n_air_bytes, corrupt, straddle, pdu_len;
  uint8_t pdu[44];         /* header + payload as sent (before CRC and whitening)                         */
} btle_synth_truth;        /* 64 bytes */
int btle_b200_synth_streams_device(btle_b200_ctx *ctx, int8_t *d_iq, size_t n_streams, size_t stream_stride_int8,
                                   size_t n_int8, const btle_stream_cfg *cfgs, const btle_synth_cfg *sc,
                                   btle_synth_truth *d_truth, size_t truth_cap, size_t *n_slots_out, void *cuda_stream);

#ifdef __cplusplus
}
#endif
#endif /* BTLE_B200_H */
