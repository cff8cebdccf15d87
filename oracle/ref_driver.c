/* Driver executable around oracle/_ref/libbtle_ref.so (the unmodified reference
 * receiver).  TEST INFRASTRUCTURE ONLY — see oracle/ref_wrap.c.
 *
 *   btle_ref_driver run  <iq.bin> <chan> <aa_hex> <crcinit_hex> <mask_hex> <raw> <out.rec> [rejected]
 *                                 ("rejected": also one record per hit rejected for its ADV header length, the
 *                                  hits -v prints as PktBAD: nbytes 2, the two dewhitened header bytes)
 *   btle_ref_driver time <iq.bin> <chan> <aa_hex> <crcinit_hex> <mask_hex> <raw> <procs> <reps>
 *   btle_ref_driver sinks <iq.bin> <chan> <aa> <crcinit> <mask> <raw> <quiet> <json> <rssi> <pcap|-> <fadva|-> <fpdu|-> [verbose]
 *                                 (the reference's own text / NDJSON / pcap output for the capture)
 *   btle_ref_driver hop  <dir>    <chan> <aa> <crcinit> <mask> <quiet> <json> <verbose>
 *                                 (dir/chNN.bin = time-aligned per-channel captures; the reference's receiver() +
 *                                  receiver_controller() on a virtual radio, its own text / NDJSON on stdout)
 *   btle_ref_driver kat           (prints table / leaf known answers as JSON)
 *
 * `run` writes one 64-byte ref_rec per packet.  `time` forks <procs> workers,
 * each replaying a contiguous range of chunks <reps> times through the
 * reference receiver() (it is not re-entrant, hence processes), and prints one
 * JSON line with IQ samples/s and packets/s.  The workers warm up with one
 * untimed pass, wait at a shared-memory barrier and time their own chunk loops
 * (clock_gettime MONOTONIC); the reported wall time is latest stop - earliest
 * start, so process creation, file read and exit are not in it.
 */
#define _GNU_SOURCE
#include <dlfcn.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <time.h>
#include <unistd.h>
#include <sys/wait.h>
#include <sys/mman.h>

typedef struct { int32_t chunk, n0, nbytes, crc_bad; uint8_t bytes[48]; } ref_rec;

extern void ref_note_demod(const int8_t *rxp, int num_byte);
extern void ref_report_rejected(int on);
extern long ref_run_chunks(const int8_t *iq, long k0, long k1, int channel, uint32_t aa, uint32_t mask,
                           uint32_t crc_init, int raw, ref_rec *out, long cap);
extern long ref_run_sinks(const int8_t *iq, long k0, long k1, int channel, uint32_t aa, uint32_t mask, uint32_t crc_init,
                          int raw, int quiet, int json, int rssi, const char *pcap, const char *fa, const char *ft, int verbose);
extern long ref_run_hop(const int8_t *const caps[40], long nchunks, int chan0, uint32_t aa, uint32_t mask, uint32_t crc_init, int quiet,
                        int json, int verbose);
extern uint32_t ref_crc_init_reorder(uint32_t);
extern const uint8_t *ref_scramble_table(int ch);
extern uint32_t ref_crc_table(int i);

/* Interposes the reference's demod_byte (btle_rx.c:1489): same signature. */
typedef void (*demod_fn)(int8_t *, int, uint8_t *);
void demod_byte(int8_t *rxp, int num_byte, uint8_t *out_byte) {
  static demod_fn real = 0;
  if (!real) real = (demod_fn)dlsym(RTLD_NEXT, "demod_byte");
  ref_note_demod(rxp, num_byte);
  real(rxp, num_byte, out_byte);
}

static int8_t *load_iq(const char *path, long *n_int8) {
  FILE *f = fopen(path, "rb");
  if (!f) { perror(path); exit(2); }
  fseek(f, 0, SEEK_END); long n = ftell(f); fseek(f, 0, SEEK_SET);
  int8_t *buf = (int8_t *)calloc((size_t)n + 8192, 1);   /* zero tail >= 3010 (App. A.4) */
  if (fread(buf, 1, (size_t)n, f) != (size_t)n) { perror("fread"); exit(2); }
  fclose(f);
  *n_int8 = n;
  return buf;
}

static double now_s(void) { struct timespec t; clock_gettime(CLOCK_MONOTONIC, &t); return t.tv_sec + 1e-9 * t.tv_nsec; }

int main(int argc, char **argv) {
  if (argc >= 2 && !strcmp(argv[1], "kat")) {
    printf("{\"crc_init_reorder\":{\"555555\":\"%06x\",\"a77b22\":\"%06x\",\"123456\":\"%06x\"},",
           ref_crc_init_reorder(0x555555), ref_crc_init_reorder(0xA77B22), ref_crc_init_reorder(0x123456));
    printf("\"crc_table\":[");
    for (int i = 0; i < 256; i++) printf("%u%s", ref_crc_table(i), i == 255 ? "" : ",");
    printf("],\"scramble_table\":[");
    for (int c = 0; c < 40; c++) {
      printf("[");
      for (int i = 0; i < 42; i++) printf("%u%s", ref_scramble_table(c)[i], i == 41 ? "" : ",");
      printf("]%s", c == 39 ? "" : ",");
    }
    printf("]}\n");
    return 0;
  }
  if (argc >= 10 && !strcmp(argv[1], "hop")) {
    const int8_t *caps[40];
    long n_min = -1;
    for (int c = 0; c < 40; c++) {
      char name[1024];
      snprintf(name, sizeof name, "%s/ch%02d.bin", argv[2], c);
      caps[c] = 0;
      if (access(name, R_OK) == 0) {
        long n; caps[c] = load_iq(name, &n);
        if (n_min < 0 || n < n_min) n_min = n;
      }
    }
    if (n_min < 0) { fprintf(stderr, "no captures in %s\n", argv[2]); return 2; }
    ref_run_hop(caps, n_min / 16384, atoi(argv[3]), (uint32_t)strtoul(argv[4], 0, 16), (uint32_t)strtoul(argv[6], 0, 16),
                (uint32_t)strtoul(argv[5], 0, 16), atoi(argv[7]), atoi(argv[8]), atoi(argv[9]));
    return 0;
  }
  if (argc < 9) { fprintf(stderr, "usage: see oracle/ref_driver.c\n"); return 2; }
  const char *mode = argv[1];
  long n_int8; int8_t *iq = load_iq(argv[2], &n_int8);
  int chan = atoi(argv[3]);
  uint32_t aa = (uint32_t)strtoul(argv[4], 0, 16), crc = (uint32_t)strtoul(argv[5], 0, 16);
  uint32_t mask = (uint32_t)strtoul(argv[6], 0, 16);
  int raw = atoi(argv[7]);
  long nchunks = n_int8 / 16384;
  if (!strcmp(mode, "run")) {
    long cap = nchunks * 123 + 16;  /* worst case is 123 per chunk (BTLE_MAX_RECS_PER_CHUNK, include/btle_b200.h) */
    ref_rec *out = (ref_rec *)calloc((size_t)cap, sizeof(ref_rec));
    ref_report_rejected(argc > 9 && !strcmp(argv[9], "rejected"));
    long n = ref_run_chunks(iq, 0, nchunks, chan, aa, mask, crc, raw, out, cap);
    FILE *f = fopen(argv[8], "wb");
    fwrite(out, sizeof(ref_rec), (size_t)(n < cap ? n : cap), f);
    fclose(f);
    fprintf(stderr, "ref: %ld chunks, %ld packets\n", nchunks, n);
    return 0;
  }
  if (!strcmp(mode, "sinks")) {
    /* sinks <iq> <chan> <aa> <crc> <mask> <raw> <quiet> <json> <rssi> <pcap|-> <filter_adva|-> <filter_pdu|-> */
    if (argc < 14) return 2;
    const char *pc = strcmp(argv[11], "-") ? argv[11] : 0, *fa = strcmp(argv[12], "-") ? argv[12] : 0,
               *ft = strcmp(argv[13], "-") ? argv[13] : 0;
    ref_run_sinks(iq, 0, nchunks, chan, aa, mask, crc, raw, atoi(argv[8]), atoi(argv[9]), atoi(argv[10]), pc, fa, ft, argc > 14 ? atoi(argv[14]) : 0);
    return 0;
  }
  if (!strcmp(mode, "time")) {
    /* All workers are forked first, run ONE untimed warm-up pass (page faults, copy-on-write,
     * caches), then meet at a barrier in shared memory; each worker stamps its own start/stop
     * around its timed passes.  Wall time = latest stop - earliest start after the barrier, so
     * fork()/exit()/wait() are outside the timed region. */
    int procs = atoi(argv[8]); int reps = argc > 9 ? atoi(argv[9]) : 1;
    if (procs < 1) procs = 1;
    if (procs > nchunks && nchunks > 0) procs = (int)nchunks;
    typedef struct { long packets; double t0, t1; int ok; } wstat;
    size_t shm_bytes = sizeof(int) * 16 + sizeof(wstat) * (size_t)procs;
    char *shm = (char *)mmap(0, shm_bytes, PROT_READ | PROT_WRITE, MAP_SHARED | MAP_ANONYMOUS, -1, 0);
    if (shm == MAP_FAILED) { perror("mmap"); return 2; }
    volatile int *arrived = (volatile int *)shm;          /* workers that finished warming up */
    volatile int *go = arrived + 1;                        /* set by the parent: start / abort */
    wstat *ws = (wstat *)(shm + sizeof(int) * 16);
    int started = 0;
    for (int p = 0; p < procs; p++) {
      pid_t pid = fork();
      if (pid < 0) { perror("fork"); break; }
      if (pid == 0) {
        long k0 = nchunks * p / procs, k1 = nchunks * (p + 1) / procs, tot = 0;
        ref_run_chunks(iq, k0, k1, chan, aa, mask, crc, raw, 0, 0);          /* warm-up, untimed */
        __sync_fetch_and_add((int *)arrived, 1);
        while (!*go) { struct timespec ts = {0, 50000}; nanosleep(&ts, 0); }
        if (*go < 0) _exit(3);
        ws[p].t0 = now_s();
        for (int r = 0; r < reps; r++) tot += ref_run_chunks(iq, k0, k1, chan, aa, mask, crc, raw, 0, 0);
        ws[p].t1 = now_s();
        ws[p].packets = tot;
        ws[p].ok = 1;
        _exit(0);
      }
      started++;
    }
    if (started < procs) {                                  /* a fork failed: do not report a partial run */
      *go = -1;
      for (int p = 0; p < started; p++) { int st; wait(&st); }
      fprintf(stderr, "ref_driver: only %d of %d workers could be started\n", started, procs);
      return 3;
    }
    while (*arrived < procs) { struct timespec ts = {0, 200000}; nanosleep(&ts, 0); }
    *go = 1;
    for (int p = 0; p < procs; p++) { int st; wait(&st); }
    long tot = 0; double t0 = 1e300, t1 = 0, sum_busy = 0; int ok = 0;
    for (int p = 0; p < procs; p++) {
      ok += ws[p].ok; tot += ws[p].packets;
      if (ws[p].t0 < t0) t0 = ws[p].t0;
      if (ws[p].t1 > t1) t1 = ws[p].t1;
      sum_busy += ws[p].t1 - ws[p].t0;
    }
    if (ok != procs) { fprintf(stderr, "ref_driver: %d of %d workers finished\n", ok, procs); return 3; }
    double dt = t1 - t0;
    double samples = (double)nchunks * 8192.0 * reps;
    printf("{\"seconds\":%.6f,\"iq_samples\":%.0f,\"packets\":%ld,\"msamples_per_s\":%.3f,\"packets_per_s\":%.1f,"
           "\"procs\":%d,\"reps\":%d,\"msamples_per_s_per_core\":%.3f,\"mean_worker_seconds\":%.6f}\n",
           dt, samples, tot, samples / dt / 1e6, tot / dt, procs, reps, samples / dt / 1e6 / procs, sum_busy / procs);
    return 0;
  }
  return 2;
}
