/* CPU restatement of the reference BLE receive path — TEST INFRASTRUCTURE ONLY.
 *
 * Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline leg may link
 * or call this.  The shipped product path (btle_b200/csrc) never does; it fails
 * loudly when the CUDA library is missing.
 *
 * Parity status: PINNED.  Checked bit-for-bit against the reference's own
 * receiver() compiled from the reference sources (oracle/_ref, see oracle/Makefile)
 * on matlab/sample_iq_4msps.txt, reference-generated TX->RX loopbacks and
 * adversarial fuzz (tests/test_oracle_vs_ref.py), and against the committed
 * golden vectors under tests/golden/ (tests/test_oracle_golden.py).
 */
#ifndef BTLE_ORACLE_H
#define BTLE_ORACLE_H
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* Same 64-byte layout as btle_pkt_rec in include/btle_b200.h. */
typedef struct {
  int32_t stream;
  int32_t chunk;       /* index of the 16384-int8 chunk inside the stream            */
  int32_t n0;          /* first IQ sample of the access address, relative to chunk   */
  uint8_t channel;
  uint8_t n_bytes;     /* 42 in raw mode, else 2 + payload_len + 3                    */
  uint8_t crc_bad;     /* verdict of the reference's crc_check(): 1 = mismatch        */
  uint8_t flags;       /* bit0 raw, bit1 advertising channel, bit2 rejected hit        */
  uint32_t access_addr;
  uint16_t mag_sum;    /* sum |I|+|Q| over the 128 AA samples (RSSI, App. A.6)        */
  uint8_t bytes[42];   /* dewhitened header+payload+crc (raw mode: still whitened)    */
} orc_rec;

typedef struct {
  int32_t channel;      /* 0..39 */
  uint32_t access_addr; /* as -a */
  uint32_t access_mask; /* as -m */
  uint32_t crc_init;    /* as -k (NOT reordered) */
  int32_t raw;          /* as -r */
} orc_cfg;

uint32_t orc_crc_init_reorder(uint32_t crc_init);
uint32_t orc_crc24(const uint8_t *bytes, int n, uint32_t init_reordered);
uint8_t orc_whiten_byte(int channel, int idx);
void orc_dbits(const int8_t *x, long n_samples, uint8_t *d);
int orc_search(const uint8_t *d, int R, int left, uint32_t aa, uint32_t mask, int *n0_out);
void orc_demod_bytes(const uint8_t *d, int n_first, int num_byte, uint8_t *out);
int orc_receiver_chunk(const int8_t *win, const orc_cfg *cfg, orc_rec *out, int cap, int32_t stream, int32_t chunk);
long orc_rx_stream(const int8_t *iq, long n_int8, const orc_cfg *cfg, int32_t stream, orc_rec *out, long cap);
/* The same with -v: report_rejected != 0 returns the ADV hits whose header length is outside 6..37 too
 * (printed as PktBAD, btle_rx.c:2291-2298), as records with flags bit2 set, n_bytes 2, the two header bytes. */
int orc_receiver_chunk_ex(const int8_t *win, const orc_cfg *cfg, int report_rejected, orc_rec *out, int cap, int32_t stream,
                          int32_t chunk);
long orc_rx_stream_ex(const int8_t *iq, long n_int8, const orc_cfg *cfg, int report_rejected, int32_t stream, orc_rec *out,
                      long cap);

#ifdef __cplusplus
}
#endif
#endif
