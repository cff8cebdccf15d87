/* oracle/_ref wrapper: compiles the UNMODIFIED reference receiver
 * (the reference's host/btle-tools/src/btle_rx.c, found through -I at build
 * time; nothing is copied into this repo) into libbtle_ref.so and exposes a
 * small driver API around its `receiver()` (btle_rx.c:2188).
 *
 * TEST INFRASTRUCTURE ONLY.  Only tests/, __graft_entry__.smoke() and the
 * cpu_baseline / --impl reference legs of bench.py may run this.
 *
 * How records are captured without touching the reference source:
 *   - `-Dgettimeofday=oracle_hook_gettimeofday` (Makefile): the reference calls
 *     gettimeofday() exactly once per counted packet, right after crc_check()
 *     and `pkt_count++` (btle_rx.c:2274 raw, :2323 normal), so the hook sees
 *     the finished packet in the reference's own globals `tmp_byte`
 *     (btle_rx.c:1485) and `receiver_status` (:1487).
 *   - the library is built -fPIC with default (interposable) visibility, so the
 *     call receiver()->demod_byte() (btle_rx.c:2265) goes through the PLT and the
 *     driver executable interposes it to learn where the header was demodulated
 *     (=> AA start sample n0 = header sample - 128).
 */
#define ORACLE_HOOK_SET_FREQ
#define main btle_rx_reference_main
#include "btle_rx.c"
#undef main

#include <stdint.h>

typedef struct {
  int32_t chunk;     /* chunk index k (16384-int8 halves, SURVEY.md App. A.4) */
  int32_t n0;        /* AA first sample, relative to chunk start; INT32_MIN if unknown */
  int32_t nbytes;    /* bytes valid in `bytes`: 42 raw, else 2+plen+3 */
  int32_t crc_bad;   /* crc_check() verdict (1 = bad); 0 in raw mode */
  uint8_t bytes[48];
} ref_rec;

static ref_rec *g_out = 0;
static long g_cap = 0, g_n = 0;
static int g_chunk = 0, g_raw = 0, g_adv = 0;
static const int8_t *g_chunk_base = 0;
static const int8_t *g_hdr_ptr = 0;

static int g_report_rejected = 0;
void ref_report_rejected(int on) { g_report_rejected = on; }

/* A header was demodulated and no packet was counted behind it: either receiver() rejected it for its ADV length
 * (:2291-2298, printed as PktBAD under -v, the search goes on) or the length guard ended the chunk (:2308-2311).
 * Called before the next header is demodulated and at the end of the chunk, when tmp_byte[0..1] still holds the
 * dewhitened header; records the rejected ones (nbytes 2, the two header bytes) when asked to. */
static void note_uncounted_header(void) {
  if (!g_report_rejected || !g_hdr_ptr || g_raw || !g_adv) return;
  const int plen = tmp_byte[1] & 0x3F;
  if (plen >= 6 && plen <= 37) return;                 /* the length-guard break */
  if (g_out && g_n < g_cap) {
    ref_rec *r = &g_out[g_n];
    memset(r, 0, sizeof(*r));
    r->chunk = g_chunk;
    r->n0 = (int32_t)((g_hdr_ptr - g_chunk_base) / 2 - 128);
    r->nbytes = 2;
    memcpy(r->bytes, tmp_byte, 2);
  }
  g_n++;
}

/* called by the interposed demod_byte() in the driver executable */
void ref_note_demod(const int8_t *rxp, int num_byte) {
  if (num_byte == 2 || (g_raw && num_byte == 42)) {
    note_uncounted_header();
    g_hdr_ptr = rxp;
  }
}

static long long g_virtual_us = 0;       /* hop mode: the time at which the chunk being processed was complete */
static uint64_t g_last_freq = 0;
int oracle_hook_set_freq(uint64_t freq_hz) { g_last_freq = freq_hz; return 0; }

int oracle_hook_gettimeofday(struct timeval *tv, void *tz) {
  (void)tz;
  if (tv) { tv->tv_sec = (long)(g_virtual_us / 1000000); tv->tv_usec = (long)(g_virtual_us % 1000000); }
  if (!g_chunk_base) return 0;
  /* a packet was just counted iff raw-mode header demod happened, or
     receiver_status.pkt_avaliable was raised (btle_rx.c:2320) */
  int counted = g_raw ? (g_hdr_ptr != 0) : (receiver_status.pkt_avaliable == 1);
  if (!counted) return 0;
  if (g_out && g_n < g_cap) {
    ref_rec *r = &g_out[g_n];
    memset(r, 0, sizeof(*r));
    r->chunk = g_chunk;
    r->n0 = g_hdr_ptr ? (int32_t)((g_hdr_ptr - g_chunk_base) / 2 - 128) : INT32_MIN;
    if (g_raw) {
      r->nbytes = 42; r->crc_bad = 0;
    } else {
      int plen = g_adv ? (tmp_byte[1] & 0x3F) : (tmp_byte[1] & 0x1F);
      r->nbytes = plen + 5;
      r->crc_bad = receiver_status.crc_ok ? 0 : 1;
    }
    memcpy(r->bytes, tmp_byte, (size_t)r->nbytes);
  }
  g_n++;
  receiver_status.pkt_avaliable = 0;
  g_hdr_ptr = 0;
  return 0;
}

uint32_t ref_crc_init_reorder(uint32_t crc_init) { return crc_init_reorder(crc_init); }

/* Replays main()'s chunking (btle_rx.c:2619-2651) over a linear buffer:
 * for k in [k0,k1): receiver(iq + 16384k, 248+16384, ...).  The caller must keep
 * >= 3010 readable int8 behind the last chunk.  Returns the number of packets
 * the reference counted (may exceed cap; only cap are stored), plus the rejected
 * hits after ref_report_rejected(1). */
long ref_run_chunks(const int8_t *iq, long k0, long k1, int channel,
                    uint32_t access_addr, uint32_t access_mask, uint32_t crc_init,
                    int raw, ref_rec *out, long cap) {
  quiet_text_flag = 1; json_flag = 0; rssi_est_flag = 0; filename_pcap = NULL;
  filter_adva_set = 0; filter_pdu_mask = 0xFFFF;
  uint32_to_bit_array(access_mask, access_bit_mask);          /* btle_rx.c:2561 */
  uint32_t crc_internal = crc_init_reorder(crc_init);           /* btle_rx.c:2604 */
  g_out = out; g_cap = cap; g_n = 0; g_raw = raw;
  g_adv = (channel == 37 || channel == 38 || channel == 39);
  for (long k = k0; k < k1; k++) {
    g_chunk = (int)k;
    g_chunk_base = iq + 16384 * k;
    g_hdr_ptr = 0;
    receiver_status.pkt_avaliable = 0;
    receiver((IQ_TYPE *)g_chunk_base, (LEN_DEMOD_BUF_ACCESS - 1) * 2 * SAMPLE_PER_SYMBOL + (LEN_BUF) / 2,
             channel, access_addr, crc_internal, 0, raw);      /* btle_rx.c:2651 */
    note_uncounted_header();
    g_hdr_ptr = 0;
  }
  g_chunk_base = 0;
  return g_n;
}

/* Same replay, but with the reference's own sinks switched on: text lines on stdout
 * (quiet=0), NDJSON (json=1), pcap (filename != NULL), RSSI (-R), filters as given.
 * Time stamps come from the hooked gettimeofday() and are therefore all zero. */
long ref_run_sinks(const int8_t *iq, long k0, long k1, int channel, uint32_t access_addr, uint32_t access_mask,
                   uint32_t crc_init, int raw, int quiet, int json, int rssi, const char *pcap_name,
                   const char *filter_adva_str, const char *filter_pdu_csv, int verbose) {
  quiet_text_flag = quiet; json_flag = json; rssi_est_flag = rssi;
  btj_init(json);
  filename_pcap = (char *)pcap_name;
  if (filename_pcap) init_pcap_file();
  filter_adva_set = 0; filter_pdu_mask = 0xFFFF;
  if (filter_adva_str && parse_mac_string(filter_adva_str, filter_adva) == 0) filter_adva_set = 1;
  if (filter_pdu_csv) parse_pdu_type_csv(filter_pdu_csv, &filter_pdu_mask);
  uint32_to_bit_array(access_mask, access_bit_mask);
  uint32_t crc_internal = crc_init_reorder(crc_init);
  g_out = 0; g_cap = 0; g_n = 0; g_raw = raw;
  g_adv = (channel == 37 || channel == 38 || channel == 39);
  for (long k = k0; k < k1; k++) {
    g_chunk = (int)k; g_chunk_base = iq + 16384 * k; g_hdr_ptr = 0;
    receiver_status.pkt_avaliable = 0;
    receiver((IQ_TYPE *)g_chunk_base, (LEN_DEMOD_BUF_ACCESS - 1) * 2 * SAMPLE_PER_SYMBOL + (LEN_BUF) / 2,
             channel, access_addr, crc_internal, verbose, raw);
  }
  g_chunk_base = 0;
  fflush(stdout);
  if (filename_pcap) { fclose(fh_pcap_store); fh_pcap_store = NULL; filename_pcap = NULL; }
  return g_n;
}

/* The reference's OWN connection follower on a virtual radio: main()'s loop (btle_rx.c:2610-2662) over 40 time-aligned
 * per-channel captures, receiver() on the capture of the channel the "radio" is tuned to, then receiver_controller()
 * (btle_rx.c:2403) exactly as main() calls it; board_set_freq() lands in oracle_hook_set_freq(), gettimeofday() shows
 * the time at which the chunk (and its look-ahead) was complete.  Text / NDJSON go to stdout through the reference's
 * own sinks. */
long ref_run_hop(const int8_t *const caps[40], long nchunks, int chan0, uint32_t access_addr, uint32_t access_mask, uint32_t crc_init,
                 int quiet, int json, int verbose) {
  quiet_text_flag = quiet; json_flag = json; rssi_est_flag = 0; filename_pcap = NULL;
  btj_init(json);
  filter_adva_set = 0; filter_pdu_mask = 0xFFFF;
  uint32_to_bit_array(access_mask, access_bit_mask);
  uint32_t crc_internal = crc_init_reorder(crc_init);
  int chan = chan0;
  receiver_status.pkt_avaliable = 0; receiver_status.hop = -1; receiver_status.new_chm_flag = 0; receiver_status.interval = 0;
  receiver_status.access_addr = 0; receiver_status.crc_init = 0; receiver_status.crc_ok = false;
  memset(receiver_status.chm, 0, 5);
  g_out = 0; g_cap = 0; g_n = 0; g_raw = 0;
  for (long k = 0; k < nchunks; k++) {
    if (!caps[chan]) break;
    g_adv = (chan == 37 || chan == 38 || chan == 39);
    g_chunk = (int)k; g_chunk_base = caps[chan] + 16384 * k; g_hdr_ptr = 0;
    g_virtual_us = ((k + 1) * 8192ll + LEN_BUF_MAX_NUM_PHY_SAMPLE / 2) / 4;
    receiver_status.pkt_avaliable = 0;
    receiver((IQ_TYPE *)g_chunk_base, (LEN_DEMOD_BUF_ACCESS - 1) * 2 * SAMPLE_PER_SYMBOL + (LEN_BUF) / 2, chan, access_addr, crc_internal,
             verbose, 0);
    fflush(stdout);
    if (receiver_controller(NULL, verbose, &chan, &access_addr, &crc_internal) != 0) break;
  }
  g_chunk_base = 0;
  g_virtual_us = 0;
  fflush(stdout);
  return g_n;
}

/* leaf functions for unit parity */
int ref_search_unique_bits(const int8_t *rxp, int search_len, uint32_t aa, uint32_t mask) {
  uint8_t bits[32], mbits[32];
  uint32_to_bit_array(aa, bits);
  uint32_to_bit_array(mask, mbits);
  return search_unique_bits((IQ_TYPE *)rxp, search_len, bits, mbits, LEN_DEMOD_BUF_ACCESS);
}
void ref_demod_byte(const int8_t *rxp, int num_byte, uint8_t *out) { demod_byte((IQ_TYPE *)rxp, num_byte, out); }
uint32_t ref_crc24_byte(const uint8_t *b, int n, uint32_t init) { return (uint32_t)crc24_byte((uint8_t *)b, n, init); }
const uint8_t *ref_scramble_table(int ch) { return scramble_table[ch]; }
uint32_t ref_crc_table(int i) { return (uint32_t)crc_table[i]; }
