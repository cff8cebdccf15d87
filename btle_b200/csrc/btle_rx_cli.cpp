// btle_rx_b200 — btle_rx-compatible host program on top of the C-ABI (include/btle_b200.h).
//
// Keeps the option surface, text lines, NDJSON v1 events and pcap format of the reference's
// btle_rx (host/btle-tools/src/btle_rx.c: parse_commandline :1244-1458, receiver() sinks
// :2330-2389, pcap :110,:167-207; btle_json.c) so that its consumers (btle_cli: rx_proc.py:64-81,
// pcap_loader.py:93-144) keep working, but takes the IQ from a capture file instead of a radio and
// runs the whole receive chain on the GPU in one call.  Host-side work here is only what the
// reference does AFTER crc_check(): payload field re-ordering, the drop rules, the filters and the
// three sinks.
//
// Differences, on purpose:
//   * IQ source instead of an SDR (without one the program exits with status 1, the reference's "board failure"
//     code, :2586):
//       -i/--iq-file FILE[:CH[:AA[:CRCINIT[:HZ]]]]  (repeatable) raw interleaved int8 (what rx_callback writes,
//                                btle_rx.c:531-540), files or FIFOs, '-' = stdin for one of them; several -i are
//                                time-aligned captures, each with its own channel / access address / CRC init.  One session
//                                (btle_b200_streams_*) serves any number of -i: poll() across the inputs, read() into
//                                page-locked segments, each segment set decoded in one batched launch while the next is
//                                read (a capture may be larger than host RAM or HBM), up to the shortest capture's end.
//                                Packets are printed in time order, except that each capture's keep their own order
//                                (print_in_order): one capture's output is the reference's processing order.
//       --iq-dir DIR             DIR/ch00.bin .. DIR/ch39.bin, time-aligned captures of the BLE channels (missing
//                                files are skipped).  Without -o: like 40 -i entries.  With -o: see below.
//       --iq-txt FILE / --iq-sc16 FILE   text format of save_phy_sample (btle_rx.c:896-915) / int16 bladeRF samples.
//   * -o (hop) with --iq-dir: the reference retunes its ONE radio; here a virtual radio walks the per-channel captures
//     chunk by chunk with the reference's own state machine (btle_b200_receiver_controller == receiver_controller,
//     btle_rx.c:2403) on sample time: CONNECT_REQ on -c -> data channel (hop) -> hop every interval.  The decode for
//     every channel the radio could be on is done up front in two batched launches (advertising capture; then all 37
//     data captures with the connection's access address), the walk only picks what the radio would have seen.
//   * --connections with --iq-dir (not with -o): every connection at once instead of the reference's one radio.  The
//     session decodes the advertising captures; each CONNECT_REQ, and each connection found from its empty PDUs on the
//     data captures (discovery, no CONNECT_REQ needed), gets its access address / CRC init on all 37 data captures from
//     the oldest segment set still on the GPU on (the policy of btle_b200.hop.ConnectionMonitor).
//   * time stamps are sample time (4 Msps) from the start of the capture, not wall clock; in hop mode the state
//     machine's clock is the time at which a chunk (with its look-ahead) is complete.
#include <fcntl.h>
#include <getopt.h>
#include <poll.h>
#include <sys/stat.h>
#include <signal.h>
#include <unistd.h>

#include <algorithm>
#include <cerrno>

#include <climits>
#include <cmath>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <map>
#include <memory>
#include <set>
#include <string>
#include <vector>

#include "btle_b200.h"

namespace {

const char *ADV_NAME[16] = {"ADV_IND", "ADV_DIRECT_IND", "ADV_NONCONN_IND", "SCAN_REQ", "SCAN_RSP", "CONNECT_REQ",
                            "ADV_SCAN_IND", "RESERVED0", "RESERVED1", "RESERVED2", "RESERVED3", "RESERVED4",
                            "RESERVED5", "RESERVED6", "RESERVED7", "RESERVED8"};          // btle_rx.c:1153-1170
const char *LL_NAME[4] = {"LL_RESERVED", "LL_DATA1", "LL_DATA2", "LL_CTRL"};              // :1031-1036
const char *CTRL_NAME[15] = {"LL_CONNECTION_UPDATE_REQ", "LL_CHANNEL_MAP_REQ", "LL_TERMINATE_IND", "LL_ENC_REQ",
                             "LL_ENC_RSP", "LL_START_ENC_REQ", "LL_START_ENC_RSP", "LL_UNKNOWN_RSP", "LL_FEATURE_REQ",
                             "LL_FEATURE_RSP", "LL_PAUSE_ENC_REQ", "LL_PAUSE_ENC_RSP", "LL_VERSION_IND",
                             "LL_REJECT_IND", "LL_RESERVED"};                              // :1060-1076

struct Options {
  int chan = 37, gain = 6, lna = 32, amp = 0, verbose = 0, raw = 0, hop = 0, json = 0, quiet = 0, rssi = 0, recover = 0, symbol_spaced = 0, centre_hits = 0,
      correct = 0, lowpass = 0, offset_search = 0;
  uint32_t aa = 0x8E89BED6u, crc_init = 0x555555u, mask = 0xFFFFFFFFu;
  uint64_t freq_hz = 123;
  const char *pcap = nullptr, *iq_txt = nullptr, *iq_sc16 = nullptr, *iq_dir = nullptr, *iq_bin16 = nullptr;
  std::vector<std::string> iq_files;            // -i, possibly FILE:CH[:AA[:CRCINIT[:HZ]]] (HZ: --offset)
  size_t segment_chunks = 0;                    // 0: the session default
  int filter_adva_set = 0;
  uint8_t filter_adva[6] = {0, 0, 0, 0, 0, 0};
  uint16_t filter_pdu_mask = 0xFFFF;
  int device = 0;
  int connections = 0;                          // --connections
  int offset_set = 0, offset_auto = 0;          // --offset HZ / --offset auto
  float offset_hz = 0.0f;
};

void usage() {
  printf(
      "Usage:\n"
      "    -h --help\n      Print this help screen\n"
      "    -i --iq-file FILE[:CH[:AA[:CRCINIT]]]\n      raw interleaved int8 I,Q capture at 4 Msps ('-' = stdin)   [this build: no SDR]\n"
      "      repeatable: several time-aligned captures (files or FIFOs; '-' for at most one), each with its own channel /\n"
      "      access address / CRC init, streamed through one session; packets in time order up to the shortest capture's end\n"
      "       --iq-dir DIR\n      DIR/ch00.bin .. DIR/ch39.bin (time-aligned per-channel captures), streamed like several -i;\n"
      "      with -o the connection is followed across them (whole files)\n"
      "       --connections\n      with --iq-dir (all 40 captures; not with -o): decode every connection live, CONNECT_REQ or found from its\n"
      "      empty PDUs, on all data captures; packets of all connections in time order; per connection start one line\n"
      "        T Connection AA:aaaaaaaa CRCInit:cccccc SRC Interval:Nus Hop:H ChC FromChunk:K\n"
      "      (T: seconds of sample time of the CONNECT_REQ / first empty PDU; SRC: CONNECT_REQ or discovered; Interval -1 and\n"
      "      Hop -1 when the channel sequence is not CSA#1 on a full map; C: first data channel; K: first decoded chunk);\n"
      "      with -j a `hop` track_start event per connection whose sequence is known\n"
      "       --iq-bin16 FILE\n      interleaved int16 I,Q at 8 Msps (8 samples per symbol): a `btle_ll -q` capture; decoded with the 8-phase\n"
      "      CRC-select receiver of the reference's Python / Verilog model (first sample phase whose CRC is ok wins)\n"
      "       --segment-chunks N\n      chunks (16384 int8) per streamed segment of each capture (0 / default: 4096 = 64 MiB for one\n"
      "      capture, max(16, 4096 / N rounded up to 16) for N captures)\n"
      "       --iq-txt FILE\n      capture in the text format written by save_phy_sample()\n"
      "       --iq-sc16 FILE\n      raw interleaved int16 I,Q (bladeRF SC16Q11); reduced with >>4 like btle_rx's bladeRF build\n"
      "    -c --chan\n      Channel number. default 37. valid range 0~39\n"
      "    -g --gain / -l --lnaGain / -b --amp / -f --freq_hz\n      accepted for compatibility; no radio is driven\n"
      "    -a --access\n      Access address. 4 bytes. Hex format (like 89ABCDEF). Default 8e89bed6\n"
      "    -k --crcinit\n      CRC init value. 3 bytes. Hex format (like 555555). Default 555555\n"
      "    -m --access_mask\n      Access address bit mask. Hex. Default ffffffff\n"
      "    -v --verbose / -r --raw / -o --hop\n"
      "    -s --filename\n      Store packets to pcap file (DLT 256, LE LL with PHDR)\n"
      "    -j --json / -Q --quiet-text / -R --rssi-est\n"
      "       --recover\n      packets whose CRC fails are demodulated once more, symbol-spaced on four sample phases; the first\n"
      "      phase whose CRC is ok replaces the packet (printed as CRC0; NDJSON adds \"recovered\":q).  Not with -o or --iq-bin16\n"
      "       --correct\n      a packet whose CRC fails and whose CRC syndrome is that of one wrong bit or two adjacent wrong bits\n"
      "      (not in the length field) is corrected (printed as CRC0; NDJSON adds \"corrected\":true); with --recover after\n"
      "      its exact phases.  Applies to every cfg, --connections included.  Not with -o or --iq-bin16\n"
      "       --offset HZ|auto\n      carrier-offset correction of every capture, HZ = received minus nominal carrier (|HZ| <= 500000); a capture\n"
      "      given as FILE:CH:AA:CRCINIT:HZ takes its own.  auto (regular files only): a first pass without correction, the\n"
      "      median offset estimate of its CRC-ok packets printed on stderr, then the decode with it.  Not with --iq-bin16\n"
      "       --symbol-spaced\n      every discriminator bit compares samples one symbol apart (n-2, n+2) instead of a quarter symbol:\n"
      "      weaker packets are received; not the reference's receiver.  Applies to every capture.  Not with --iq-bin16\n"
      "       --lowpass\n      with --symbol-spaced: every discriminator bit reads [1, 2, 1] low-pass filtered samples (less noise per\n"
      "      bit); not the reference's receiver.  Applies to every capture, --recover's phases and the --offset auto pass\n"
      "      included.  Only with --symbol-spaced, not with --iq-bin16\n"
      "       --centre-hits\n      each access-address hit is moved to the centre of its run of matching sample phases before the\n"
      "      packet is read: fewer length rejects and CRC failures; not the reference's receiver.  Applies to every cfg,\n"
      "      --connections and the --offset auto pass included.  Not with --iq-bin16\n"
      "       --offset-search\n      every capture is decoded at seven carrier offsets around its own (0, +-50, +-100, +-150 kHz from the\n"
      "      --offset value or the capture's HZ field) and the packets merged: transmitters at different offsets are all\n"
      "      received; not the reference's receiver.  NDJSON adds \"offset_search\":true to packets the centre offset missed.\n"
      "      Applies to every cfg, --connections and the --offset auto pass included.  Not with -r or --iq-bin16\n"
      "    -F --filter-adva AA:BB:CC:DD:EE:FF / -T --filter-pdu-type 0,3,4\n"
      "    -d --device N   CUDA device (default 0)\n");
}

int parse_mac(const char *s, uint8_t out[6]) {        // btle_rx.c:126-146
  if (!s) return -1;
  if (strchr(s, ':')) return sscanf(s, "%2hhx:%2hhx:%2hhx:%2hhx:%2hhx:%2hhx", &out[0], &out[1], &out[2], &out[3], &out[4], &out[5]) == 6 ? 0 : -1;
  if (strlen(s) != 12) return -1;
  for (int i = 0; i < 6; ++i)
    if (sscanf(s + 2 * i, "%2hhx", &out[i]) != 1) return -1;
  return 0;
}

int parse_pdu_csv(const char *s, uint16_t *mask) {    // btle_rx.c:149-165
  if (!s) return -1;
  uint16_t m = 0;
  const char *p = s;
  while (*p) {
    char *end;
    long v = strtol(p, &end, 10);
    if (end == p || v < 0 || v > 15) return -1;
    m |= (uint16_t)(1u << v);
    p = end;
    if (*p == ',') ++p; else if (*p) return -1;
  }
  if (!m) return -1;
  *mask = m;
  return 0;
}

[[noreturn]] void bad_args() {
  usage();
  exit(-1);                                           // btle_rx.c:1455-1457
}

Options parse_commandline(int argc, char **argv) {
  Options o;
  static struct option longopts[] = {
      {"help", no_argument, 0, 'h'}, {"chan", required_argument, 0, 'c'}, {"gain", required_argument, 0, 'g'},
      {"lnaGain", required_argument, 0, 'l'}, {"amp", no_argument, 0, 'b'}, {"access", required_argument, 0, 'a'},
      {"crcinit", required_argument, 0, 'k'}, {"verbose", no_argument, 0, 'v'}, {"raw", no_argument, 0, 'r'},
      {"freq_hz", required_argument, 0, 'f'}, {"access_mask", required_argument, 0, 'm'}, {"hop", no_argument, 0, 'o'},
      {"filename", required_argument, 0, 's'}, {"json", no_argument, 0, 'j'}, {"quiet-text", no_argument, 0, 'Q'},
      {"rssi-est", no_argument, 0, 'R'}, {"filter-adva", required_argument, 0, 'F'},
      {"filter-pdu-type", required_argument, 0, 'T'}, {"iq-file", required_argument, 0, 'i'},
      {"iq-txt", required_argument, 0, 1000}, {"iq-sc16", required_argument, 0, 1001}, {"device", required_argument, 0, 'd'},
      {"iq-dir", required_argument, 0, 1002}, {"segment-chunks", required_argument, 0, 1003}, {"iq-bin16", required_argument, 0, 1004},
      {"connections", no_argument, 0, 1005}, {"recover", no_argument, 0, 1006}, {"correct", no_argument, 0, 1010},
      {"offset", required_argument, 0, 1007}, {"symbol-spaced", no_argument, 0, 1008},
      {"centre-hits", no_argument, 0, 1009}, {"lowpass", no_argument, 0, 1011},
      {"offset-search", no_argument, 0, 1012}, {0, 0, 0, 0}};
  for (;;) {
    int idx = 0;
    const int c = getopt_long(argc, argv, "hc:g:l:ba:k:vrf:m:os:jQRF:T:i:d:", longopts, &idx);   // + i:, d:
    if (c == -1) break;
    char *endp;
    switch (c) {
      case 'v': o.verbose = 1; break;
      case 'r': o.raw = 1; break;
      case 'o': o.hop = 1; break;
      case 'c': o.chan = (int)strtol(optarg, &endp, 10); break;
      case 'g': o.gain = (int)strtol(optarg, &endp, 10); break;
      case 'l': o.lna = (int)strtol(optarg, &endp, 10); break;
      case 'b': o.amp = 1; break;
      case 'f': o.freq_hz = (uint64_t)strtol(optarg, &endp, 10); break;
      case 'a': o.aa = (uint32_t)strtol(optarg, &endp, 16); break;
      case 'm': o.mask = (uint32_t)strtol(optarg, &endp, 16); break;
      case 'k': o.crc_init = (uint32_t)strtol(optarg, &endp, 16); break;
      case 's': o.pcap = optarg; break;
      case 'j': o.json = 1; break;
      case 'Q': o.quiet = 1; break;
      case 'R': o.rssi = 1; break;
      case 'i': o.iq_files.push_back(optarg); break;
      case 1002: o.iq_dir = optarg; break;
      case 1004: o.iq_bin16 = optarg; break;
      case 1005: o.connections = 1; break;
      case 1006: o.recover = 1; break;
      case 1010: o.correct = 1; break;
      case 1008: o.symbol_spaced = 1; break;
      case 1009: o.centre_hits = 1; break;
      case 1011: o.lowpass = 1; break;
      case 1012: o.offset_search = 1; break;
      case 1007:
        o.offset_set = 1;
        if (!strcmp(optarg, "auto")) { o.offset_auto = 1; break; }
        o.offset_hz = strtof(optarg, &endp);
        if (endp == optarg || *endp || !std::isfinite(o.offset_hz) || std::fabs(o.offset_hz) > (float)BTLE_MAX_OFFSET_HZ) {
          printf("Invalid --offset value: %s (expect Hz within +-%d, or auto)\n", optarg, BTLE_MAX_OFFSET_HZ);
          bad_args();
        }
        break;
      case 1003: o.segment_chunks = (size_t)strtoul(optarg, &endp, 10); break;
      case 1000: o.iq_txt = optarg; break;
      case 1001: o.iq_sc16 = optarg; break;
      case 'd': o.device = (int)strtol(optarg, &endp, 10); break;
      case 'F':
        if (parse_mac(optarg, o.filter_adva)) {
          printf("Invalid --filter-adva value: %s (expect AA:BB:CC:DD:EE:FF or 12 hex chars)\n", optarg);
          bad_args();
        }
        o.filter_adva_set = 1;
        break;
      case 'T':
        if (parse_pdu_csv(optarg, &o.filter_pdu_mask)) {
          printf("Invalid --filter-pdu-type value: %s (expect CSV of ints 0..15, e.g. 0,3,4)\n", optarg);
          bad_args();
        }
        break;
      default: bad_args();                            // 'h', '?', anything else
    }
  }
  if (o.chan < 0 || o.chan > 39) { printf("channel number must be within 0~%d!\n", 39); bad_args(); }   // :1432
  if (o.gain < 0 || o.gain > 62) { printf("rx gain must be within 0~%d!\n", 62); bad_args(); }            // :1437
  if (o.lna < 0 || o.lna > 40) { printf("lna gain must be within 0~%d!\n", 40); bad_args(); }            // :1442
  if (optind < argc) { printf("Error: unknown/extra arguments specified on command line!\n"); bad_args(); }
  if (o.connections && (!o.iq_dir || o.hop)) { printf("--connections needs --iq-dir and cannot be combined with -o\n"); bad_args(); }
  // -o follows as the reference's follower does, from the reference's records; --iq-bin16 has a receiver of its own
  if (o.recover && (o.hop || o.iq_bin16)) { printf("--recover cannot be combined with -o or --iq-bin16\n"); bad_args(); }
  if (o.correct && (o.hop || o.iq_bin16)) { printf("--correct cannot be combined with -o or --iq-bin16\n"); bad_args(); }
  // the 8-sps model receiver has no carrier-offset correction
  if (o.offset_set && o.iq_bin16) { printf("--offset cannot be combined with --iq-bin16 (the 8-sps receiver has no offset correction)\n"); bad_args(); }
  if (o.symbol_spaced && o.iq_bin16) { printf("--symbol-spaced cannot be combined with --iq-bin16 (the 8-sps receiver has its own discriminator)\n"); bad_args(); }
  if (o.centre_hits && o.iq_bin16) { printf("--centre-hits cannot be combined with --iq-bin16 (the 8-sps receiver has its own hit rule)\n"); bad_args(); }
  if (o.lowpass && (!o.symbol_spaced || o.iq_bin16)) { printf("--lowpass needs --symbol-spaced and cannot be combined with --iq-bin16\n"); bad_args(); }
  // raw records have no CRC verdict to merge the hypotheses by
  if (o.offset_search && (o.raw || o.iq_bin16)) { printf("--offset-search cannot be combined with -r or --iq-bin16\n"); bad_args(); }
  return o;
}

uint64_t freq_by_channel(int ch) {                    // get_freq_by_channel_number, btle_rx.c:1006
  if (ch == 37) return 2402000000ull;
  if (ch == 38) return 2426000000ull;
  if (ch == 39) return 2480000000ull;
  if (ch <= 10) return 2404000000ull + (uint64_t)ch * 2000000ull;
  return 2428000000ull + (uint64_t)(ch - 11) * 2000000ull;
}

bool load_txt(const char *name, std::vector<int8_t> &iq) {   // numbers separated by ", " (save_phy_sample): one pass over the file
  FILE *f = fopen(name, "r");
  if (!f) { perror(name); return false; }
  std::vector<char> buf(1 << 20);
  long v = 0;
  bool in_num = false, neg = false;
  size_t n;
  while ((n = fread(buf.data(), 1, buf.size(), f)) > 0)
    for (size_t k = 0; k < n; ++k) {
      const char c = buf[k];
      if (c >= '0' && c <= '9') { v = v * 10 + (c - '0'); in_num = true; }
      else {
        if (in_num) { iq.push_back((int8_t)(neg ? -v : v)); v = 0; in_num = false; neg = false; }
        if (c == '-') neg = true;
      }
    }
  if (in_num) iq.push_back((int8_t)(neg ? -v : v));
  fclose(f);
  return true;
}

bool load_raw(const char *name, std::vector<int8_t> &iq) {
  FILE *f = strcmp(name, "-") ? fopen(name, "rb") : stdin;
  if (!f) { perror(name); return false; }
  if (f != stdin && fseek(f, 0, SEEK_END) == 0) {
    const long sz = ftell(f);
    fseek(f, 0, SEEK_SET);
    if (sz > 0) {
      iq.resize((size_t)sz);
      const size_t got = fread(iq.data(), 1, (size_t)sz, f);
      iq.resize(got);
      fclose(f);
      return true;
    }
  }
  char buf[1 << 16];
  size_t n;
  while ((n = fread(buf, 1, sizeof buf, f)) > 0) iq.insert(iq.end(), buf, buf + n);
  if (f != stdin) fclose(f);
  return true;
}

// ---- owners: what a mode opens is closed on every return -------------------------------------------------------------
struct CtxClose { void operator()(btle_b200_ctx *c) const { btle_b200_destroy(c); } };
struct StreamsClose { void operator()(btle_b200_streams *s) const { btle_b200_streams_close(s); } };
struct FileClose { void operator()(FILE *f) const { fclose(f); } };
struct Inputs {                                       // the session's input descriptors; 0 (stdin) is left open
  std::vector<int> fds;
  ~Inputs() { for (int fd : fds) if (fd > 0) close(fd); }
};

// ---- sinks ----------------------------------------------------------------------------------------
void put_be32(FILE *f, uint32_t v) { const uint8_t b[4] = {(uint8_t)(v >> 24), (uint8_t)(v >> 16), (uint8_t)(v >> 8), (uint8_t)v}; fwrite(b, 1, 4, f); }

FILE *pcap_open(const char *name) {                   // init_pcap_file + PCAP_HDR_TCPDUMP, btle_rx.c:110,:167
  FILE *f = fopen(name, "wb");
  if (!f) return nullptr;
  put_be32(f, 0xA1B2C3D4u);                           // magic, big-endian file
  const uint8_t ver[4] = {0, 2, 0, 4};
  fwrite(ver, 1, 4, f);
  put_be32(f, 0); put_be32(f, 0);                     // thiszone, sigfigs
  put_be32(f, 1500);                                  // snaplen 0x5DC
  put_be32(f, 256);                                   // DLT_BLUETOOTH_LE_LL_WITH_PHDR
  return f;
}

void pcap_write(FILE *f, double t, const uint8_t *pkt, int len, int ch, uint32_t aa, int rssi) {   // :184-207
  const uint32_t sec = (uint32_t)t, usec = (uint32_t)((t - sec) * 1e6);
  put_be32(f, sec); put_be32(f, usec);
  put_be32(f, 10 + 4 + (uint32_t)len); put_be32(f, 10 + 4 + (uint32_t)len);
  int8_t sig = -127;
  if (rssi != INT_MIN) sig = (int8_t)(rssi > 20 ? 20 : (rssi < -126 ? -126 : rssi));
  const uint8_t phdr[10] = {(uint8_t)ch, (uint8_t)sig, 0, 0, 0, 0, 0, 0, 1, 0};
  fwrite(phdr, 1, 10, f);
  const uint8_t aab[4] = {(uint8_t)aa, (uint8_t)(aa >> 8), (uint8_t)(aa >> 16), (uint8_t)(aa >> 24)};   // host order of the reference (LE)
  fwrite(aab, 1, 4, f);
  fwrite(pkt, 1, (size_t)len, f);
}

void hex(const uint8_t *b, int n) { for (int i = 0; i < n; ++i) printf("%02x", b[i]); }
void hex_rev(const uint8_t *b, int n) { for (int i = n - 1; i >= 0; --i) printf("%02x", b[i]); }   // fields printed MSB first
uint32_t le16(const uint8_t *p) { return (uint32_t)p[0] | ((uint32_t)p[1] << 8); }

// AdvA for the filter / JSON (extract_adv_a, :1720-1739): MSB-first; false = not available
bool adv_a(const uint8_t *p, int type, uint8_t out[6]) {
  int off;
  if (type == 0 || type == 2 || type == 4 || type == 6 || type == 1 || type == 3) off = 0;
  else if (type == 5) off = 6;
  else return false;
  for (int i = 0; i < 6; ++i) out[i] = p[off + 5 - i];
  return true;
}
void print_adv_payload(const uint8_t *p, int type, int plen, int crc_bad) {     // print_adv_pdu_payload, :2131-2185
  if (type == 0 || type == 2 || type == 4 || type == 6) {
    printf("AdvA:"); hex_rev(p, 6);
    printf(" Data:"); hex(p + 6, plen - 6);
  } else if (type == 1 || type == 3) {
    printf("A0:"); hex_rev(p, 6);
    printf(" A1:"); hex_rev(p + 6, 6);
  } else if (type == 5) {
    printf("InitA:"); hex_rev(p, 6);
    printf(" AdvA:"); hex_rev(p + 6, 6);
    printf(" AA:"); hex_rev(p + 12, 4);
    const uint32_t crcinit = ((uint32_t)p[16] << 16) | ((uint32_t)p[17] << 8) | p[18];
    printf(" CRCInit:%06x WSize:%02x WOffset:%04x Itrvl:%04x Ltncy:%04x Timot:%04x", crcinit, p[19], le16(p + 20), le16(p + 22), le16(p + 24), le16(p + 26));
    printf(" ChM:"); hex_rev(p + 28, 5);
    printf(" Hop:%d SCA:%d", p[33] & 0x1F, (p[33] >> 5) & 7);
  } else {
    printf("Byte:"); hex(p, plen);
  }
  printf(" CRC%d\n", crc_bad);
}

void print_ll_payload(const uint8_t *p, int llid, int op, int plen, int crc_bad) {   // print_ll_pdu_payload, :2018-2129
  if (plen == 0) { printf("CRC%d\n", crc_bad); return; }
  if (llid != 3) {
    printf("LL_Data:"); hex(p, plen);
  } else if (op == 0) {
    printf("Op%02x(%s) WSize:%02x WOffset:%04x Itrvl:%04x Ltncy:%04x Timot:%04x Inst:%04x", op, CTRL_NAME[op], p[1], le16(p + 2), le16(p + 4), le16(p + 6), le16(p + 8), le16(p + 10));
  } else if (op == 1) {
    printf("Op%02x(%s)", op, CTRL_NAME[op]); printf(" ChM:"); hex_rev(p + 1, 5); printf(" Inst:%04x", le16(p + 6));
  } else if (op == 2 || op == 7 || op == 13) {
    printf("Op%02x(%s) Err:%02x", op, CTRL_NAME[op], p[1]);
  } else if (op == 3) {
    printf("Op%02x(%s)", op, CTRL_NAME[op]);
    printf(" Rand:"); hex_rev(p + 1, 8); printf(" EDIV:"); hex_rev(p + 9, 2);
    printf(" SKDm:"); hex_rev(p + 11, 8); printf(" IVm:"); hex_rev(p + 19, 4);
  } else if (op == 4) {
    printf("Op%02x(%s)", op, CTRL_NAME[op]); printf(" SKDs:"); hex_rev(p + 1, 8); printf(" IVs:"); hex_rev(p + 9, 4);
  } else if (op == 5 || op == 6 || op == 10 || op == 11) {
    printf("Op%02x(%s)", op, CTRL_NAME[op]);
  } else if (op == 8 || op == 9) {
    printf("Op%02x(%s)", op, CTRL_NAME[op]); printf(" FteurSet:"); hex_rev(p + 1, 8);
  } else if (op == 12) {
    printf("Op%02x(%s) Ver:%02x CompId:%04x SubVer:%04x", op, CTRL_NAME[op], p[1], le16(p + 2), le16(p + 4));
  } else {
    printf("Op%02x(%s)", op, CTRL_NAME[op > 13 ? 14 : op]); printf(" Byte:"); hex(p + 1, plen - 1);
  }
  printf(" CRC%d\n", crc_bad);
}

void json_hex(const uint8_t *b, int n) { putchar('"'); hex(b, n); putchar('"'); }
void json_status(double ts, const char *event, const Options &o) {               // btj_emit_status
  printf("{\"v\":1,\"t\":\"status\",\"ts\":%.6f,\"event\":\"%s\",\"board\":\"B200-file\",\"ch\":%d,\"freq_hz\":%llu,\"gain\":%d,\"lna\":%d,\"amp\":%d,\"filter_adva\":",
         ts, event, o.chan, (unsigned long long)o.freq_hz, o.gain, o.lna, o.amp);
  if (o.filter_adva_set) printf("\"%02x:%02x:%02x:%02x:%02x:%02x\"", o.filter_adva[0], o.filter_adva[1], o.filter_adva[2], o.filter_adva[3], o.filter_adva[4], o.filter_adva[5]);
  else printf("null");
  printf(",\"msg\":null}\n");
  fflush(stdout);
}

int rssi_from_mag(unsigned mag_sum) {                 // btle_rx.c:2244-2249
  double mean = (double)mag_sum / 128.0;
  if (mean < 1.0) mean = 1.0;
  int r = (int)(20.0 * log10(mean / 256.0) - 50.0);
  if (r < -127) r = -127;
  if (r > 20) r = 20;
  return r;
}

// ---- what receiver() does with a counted packet after crc_check(): filters, sinks (btle_rx.c:2318-2389) -----------
struct Sinks {
  const Options &o;
  std::unique_ptr<FILE, FileClose> pcap;
  int pkt_count = 0;
  double t_prev = 0.0;
  explicit Sinks(const Options &opt) : o(opt) {}

  void packet(const btle_pkt_rec &r, double t) {
    const uint8_t *b = r.bytes;
    const int ch = r.channel;
    const uint32_t aa = r.access_addr;
    const bool adv = (ch == 37 || ch == 38 || ch == 39);                        // :2202
    if (r.flags & BTLE_REC_REJECTED) {                                          // :2291-2298, only with -v
      int type, tx, rx, plen;
      btle_b200_parse_adv_pdu_header_byte(b, &type, &tx, &rx, &plen);
      printf("XXXus PktBAD Ch%d AA:%08x ", ch, aa);
      printf("ADV_PDU_t%d:%s T%d R%d PloadL%d ", type, ADV_NAME[type], tx, rx, plen);
      printf("Error: ADV payload length should be 6~37!\n");
      return;
    }
    ++pkt_count;                                                                // :2274 / :2319
    btle_b200_note_packet(&r);                                                  // receiver_status.crc_ok, :2320-2321
    // A hit through the zeroed history of chunk k+1 (n0 < 0) can start before the previous packet of chunk k.  The
    // reference stamps packets when it processes them (gettimeofday, :2323), so its clock never runs backwards.
    if (t < t_prev) t = t_prev;
    const int time_diff = (int)llround((t - t_prev) * 1e6);
    t_prev = t;
    const int rssi = o.rssi ? rssi_from_mag(r.mag_sum) : INT_MIN;
    if (r.flags & 1) {                                                          // raw, :2271-2286
      const long sec = (long)t;
      printf("%ld.%06ld Pkt%d Ch%d AA:%08x Raw:", sec, (long)((t - sec) * 1e6), pkt_count, ch, aa);
      hex(b, 42);
      printf("\n");
      return;
    }
    const int crc_bad = r.crc_bad;
    if (adv) {
      int type, tx, rx, plen;
      btle_b200_parse_adv_pdu_header_byte(b, &type, &tx, &rx, &plen);
      if (!(o.filter_pdu_mask & (1u << (type & 15)))) return;                   // :2332-2334
      btle_adv_payload parsed;
      if (btle_b200_parse_adv_pdu_payload_byte(b + 2, plen, type, &parsed)) return;   // :2336-2339 (also feeds receiver_status)
      uint8_t a[6];
      const bool has_a = adv_a(b + 2, type, a);
      if (o.filter_adva_set && has_a && memcmp(a, o.filter_adva, 6)) return;    // :2345-2348
      if (pcap) pcap_write(pcap.get(), t, b, plen + 2, ch, aa, rssi);           // :2361-2362
      if (!o.quiet) {
        printf("%07dus Pkt%03d Ch%d AA:%08x ", time_diff, pkt_count, ch, aa);
        printf("ADV_PDU_t%d:%s T%d R%d PloadL%d ", type, ADV_NAME[type], tx, rx, plen);
        print_adv_payload(b + 2, type, plen, crc_bad);
      }
      if (o.json) {                                                             // btj_emit_pkt_adv
        printf("{\"v\":1,\"t\":\"pkt\",\"ts\":%.6f,\"pkt\":%d,\"ch\":%d,\"aa\":\"%08x\",\"crc_ok\":%s,\"kind\":\"adv\",\"pdu_type\":%d,\"pdu_name\":\"%s\"",
               t, pkt_count, ch, aa, crc_bad ? "false" : "true", type, ADV_NAME[type]);
        printf(",\"tx_add\":%d,\"rx_add\":%d,\"plen\":%d,\"adv_a\":", tx, rx, plen);
        if (has_a) printf("\"%02x:%02x:%02x:%02x:%02x:%02x\"", a[0], a[1], a[2], a[3], a[4], a[5]); else printf("null");
        printf(",\"payload_hex\":"); json_hex(b + 2, plen);
        if (rssi == INT_MIN) printf(",\"rssi_est\":null"); else printf(",\"rssi_est\":%d", rssi);
        if (r.flags & BTLE_REC_RECOVERED) printf(",\"recovered\":%d", BTLE_REC_RECOVERED_Q(r.flags));
        if (r.flags & BTLE_REC_CORRECTED) printf(",\"corrected\":true");
        if (r.flags & BTLE_REC_OFFSET_SEARCH) printf(",\"offset_search\":true");
        printf("}\n");
      }
    } else {
      int llid, nesn, sn, md, plen;
      btle_b200_parse_ll_pdu_header_byte(b, &llid, &nesn, &sn, &md, &plen);
      btle_ll_payload parsed;
      const int op = btle_b200_parse_ll_pdu_payload_byte(b + 2, plen, llid, &parsed);
      if (op < 0) return;                                                       // :2350-2353
      if (o.filter_adva_set) return;                                            // :2355-2357
      if (pcap) pcap_write(pcap.get(), t, b, plen + 2, ch, aa, rssi);
      if (!o.quiet) {
        printf("%07dus Pkt%03d Ch%d AA:%08x ", time_diff, pkt_count, ch, aa);
        printf("LL_PDU_t%d:%s NESN%d SN%d MD%d PloadL%d ", llid, LL_NAME[llid], nesn, sn, md, plen);
        print_ll_payload(b + 2, llid, op, plen, crc_bad);
      }
      if (o.json) {                                                             // btj_emit_pkt_data
        printf("{\"v\":1,\"t\":\"pkt\",\"ts\":%.6f,\"pkt\":%d,\"ch\":%d,\"aa\":\"%08x\",\"crc_ok\":%s,\"kind\":\"data\",\"ll_pdu_type\":%d,\"ll_pdu_name\":\"%s\"",
               t, pkt_count, ch, aa, crc_bad ? "false" : "true", llid, LL_NAME[llid]);
        printf(",\"nesn\":%d,\"sn\":%d,\"md\":%d,\"plen\":%d,\"payload_hex\":", nesn, sn, md, plen);
        json_hex(b + 2, plen);
        if (rssi == INT_MIN) printf(",\"rssi_est\":null"); else printf(",\"rssi_est\":%d", rssi);
        if (r.flags & BTLE_REC_RECOVERED) printf(",\"recovered\":%d", BTLE_REC_RECOVERED_Q(r.flags));
        if (r.flags & BTLE_REC_CORRECTED) printf(",\"corrected\":true");
        if (r.flags & BTLE_REC_OFFSET_SEARCH) printf(",\"offset_search\":true");
        printf("}\n");
      }
    }
  }
};

double rec_time(const btle_pkt_rec &r) { return ((double)r.chunk * 8192.0 + r.n0) / 4.0e6; }   // sample time of the access address

// Prints a session's pending records in sample-time order (chunk × 8192 + n0, ties to the lower stream) while that lies
// before `safe`, except that each stream's records keep the order the session handed them out in, chunk by chunk.  That
// is the reference's processing order, in which a hit at n0 < 0 in chunk k+1 can start before a late packet of chunk k
// (Sinks::packet); so a record sorts at the latest time among its stream's records up to it.  Returns how many it printed.
size_t print_in_order(std::vector<btle_pkt_rec> &pending, Sinks &sinks, long long safe) {
  const auto before_safe = [&](const btle_pkt_rec &r) { return (long long)r.chunk * 8192 + r.n0 < safe; };
  if (std::none_of(pending.begin(), pending.end(), before_safe)) return 0;   // a sort time is never before the record's own
  std::stable_sort(pending.begin(), pending.end(), [](const btle_pkt_rec &a, const btle_pkt_rec &b) {
    return a.stream != b.stream ? a.stream < b.stream : a.chunk < b.chunk;
  });
  std::vector<long long> t(pending.size());
  std::vector<size_t> idx(pending.size());
  for (size_t i = 0; i < pending.size(); ++i) {
    const long long own = (long long)pending[i].chunk * 8192 + pending[i].n0;
    t[i] = i && pending[i - 1].stream == pending[i].stream ? std::max(own, t[i - 1]) : own;
    idx[i] = i;
  }
  std::stable_sort(idx.begin(), idx.end(), [&](size_t a, size_t b) { return t[a] != t[b] ? t[a] < t[b] : pending[a].stream < pending[b].stream; });
  size_t n = 0;
  for (; n < idx.size() && t[idx[n]] < safe; ++n) sinks.packet(pending[idx[n]], rec_time(pending[idx[n]]));
  std::vector<btle_pkt_rec> rest;
  for (size_t k = n; k < idx.size(); ++k) rest.push_back(pending[idx[k]]);
  pending.swap(rest);
  return n;
}

volatile sig_atomic_t g_stop = 0;
void on_sigint(int) { g_stop = 1; }                                             // btle_rx.c:100-104

struct Capture { std::string file; int chan; uint32_t aa, crc_init; float hz; bool own_hz; };

// a whole decimal number of Hz within the correction's range
bool parse_hz(const std::string &f, float *hz) {
  char *e = nullptr;
  const float v = strtof(f.c_str(), &e);
  if (f.empty() || *e || !std::isfinite(v) || std::fabs(v) > (float)BTLE_MAX_OFFSET_HZ) return false;
  *hz = v;
  return true;
}

// "FILE[:CH[:AA[:CRCINIT[:HZ]]]]"
Capture parse_capture(const std::string &spec, const Options &o) {
  Capture c{spec, o.chan, o.aa, o.crc_init, o.offset_hz, false};
  std::vector<std::string> parts;
  size_t pos = 0;
  for (;;) {
    const size_t q = spec.find(':', pos);
    parts.push_back(spec.substr(pos, q == std::string::npos ? q : q - pos));
    if (q == std::string::npos) break;
    pos = q + 1;
  }
  // FILE:CH:AA:CRCINIT:HZ: the fifth field is the capture's carrier offset (may be negative)
  if (parts.size() >= 5) {
    float hz;
    bool hexes = true;
    for (size_t k = parts.size() - 4; k < parts.size() - 1; ++k)
      hexes &= !parts[k].empty() && parts[k].find_first_not_of("0123456789abcdefABCDEF") == std::string::npos;
    if (hexes && parse_hz(parts.back(), &hz)) {
      c.hz = hz;
      c.own_hz = true;
      parts.pop_back();
    }
  }
  // a ':' inside a path: only trailing fields that look like numbers are taken as parameters
  size_t nfield = 0;
  while (nfield < 3 && parts.size() > 1 + nfield) {
    const std::string &f = parts[parts.size() - 1 - nfield];
    if (f.empty() || f.find_first_not_of("0123456789abcdefABCDEF") != std::string::npos) break;
    ++nfield;
  }
  // fields are CH, then AA, then CRCINIT: with 1 field it is CH, with 2 CH:AA, with 3 CH:AA:CRCINIT
  const size_t first = parts.size() - nfield;
  if (nfield >= 1) c.chan = (int)strtol(parts[first].c_str(), nullptr, 10);
  if (nfield >= 2) c.aa = (uint32_t)strtoul(parts[first + 1].c_str(), nullptr, 16);
  if (nfield >= 3) c.crc_init = (uint32_t)strtoul(parts[first + 2].c_str(), nullptr, 16);
  c.file.clear();
  for (size_t k = 0; k < first; ++k) c.file += (k ? ":" : "") + parts[k];
  return c;
}

int cfg_flags(const Options &o) {
  return (o.rssi ? BTLE_CFG_RSSI : 0) | (o.verbose ? BTLE_CFG_REPORT_REJECTED : 0) | (o.recover ? BTLE_CFG_RECOVER : 0) |
         (o.symbol_spaced ? BTLE_CFG_SYMBOL_SPACED : 0) | (o.centre_hits ? BTLE_CFG_CENTRE_HITS : 0) |
         (o.correct ? BTLE_CFG_CORRECT : 0) | (o.lowpass ? BTLE_CFG_LOWPASS : 0) | (o.offset_search ? BTLE_CFG_OFFSET_SEARCH : 0);
}

int fail(btle_b200_ctx *ctx, int rc, const char *what) {
  printf("%s: %s (%s)\n", what, btle_b200_strerror(rc), btle_b200_last_error(ctx));
  return 1;
}

// rx_batch with a capacity that is grown once if the library asks; offset_hz: one per capture, or NULL (no correction)
int rx_batch_grow(btle_b200_ctx *ctx, const int8_t *iq, size_t ns, size_t stride, size_t n, const btle_stream_cfg *cfgs,
                  std::vector<btle_pkt_rec> &recs, const float *offset_hz = nullptr) {
  size_t cap = ns * (n / BTLE_CHUNK_INT8) * 4 + 1024, got = 0;
  int rc = 0;
  for (int attempt = 0; attempt < 2; ++attempt) {
    recs.resize(cap);
    rc = btle_b200_rx_batch_offset(ctx, iq, ns, stride, n, cfgs, offset_hz, recs.data(), cap, &got);
    if (rc != BTLE_EOVERFLOW) break;
    cap = got;
  }
  recs.resize(rc ? 0 : got);
  return rc;
}

// --offset auto: the median of btle_b200_rec_offset over the CRC-ok counted packets of a first pass without correction
// (not raw, no flags but cfg's discriminator mode, hit rule and offset bank), 0 when no packet passes; printed on stderr under `name`.
// Returns the exit status.
int estimate_offset(btle_b200_ctx *ctx, const std::vector<int8_t> &iq, btle_stream_cfg cfg, const char *name, float *hz) {
  cfg.raw = 0;
  cfg.rssi &= BTLE_CFG_SYMBOL_SPACED | BTLE_CFG_LOWPASS | BTLE_CFG_CENTRE_HITS | BTLE_CFG_OFFSET_SEARCH;
  std::vector<btle_pkt_rec> recs;
  int rc = rx_batch_grow(ctx, iq.data(), 1, iq.size(), iq.size(), &cfg, recs);
  recs.erase(std::remove_if(recs.begin(), recs.end(), [](const btle_pkt_rec &r) { return r.crc_bad || (r.flags & BTLE_REC_REJECTED); }),
             recs.end());
  std::vector<float> e(recs.size());
  if (!rc && !e.empty()) rc = btle_b200_rec_offset(ctx, iq.data(), 1, iq.size(), iq.size(), recs.data(), recs.size(), e.data());
  if (rc) return fail(ctx, rc, "--offset auto");
  std::sort(e.begin(), e.end());
  const size_t m = e.size() / 2;
  *hz = e.empty() ? 0.0f : e.size() & 1 ? e[m] : 0.5f * (e[m - 1] + e[m]);
  fprintf(stderr, "offset estimate %s: %.1f Hz (%zu CRC-ok packets)\n", name, *hz, e.size());
  return 0;
}

// ---- hop mode: a virtual radio over per-channel captures (receiver_controller semantics) -------------------------
struct HopRun {
  const Options *o;
  int64_t now = 0;
  int retunes = 0;
};
int64_t hop_now(void *u) { return static_cast<HopRun *>(u)->now; }
int hop_set_freq(void *u, uint64_t) { ++static_cast<HopRun *>(u)->retunes; return 0; }
void hop_event(void *u, const btle_hop_event *e) {                              // btj_emit_hop, btle_json.c:132-160
  const HopRun *h = static_cast<HopRun *>(u);
  if (!h->o->json) return;
  printf("{\"v\":1,\"t\":\"hop\",\"ts\":%.6f,\"event\":\"%s\",\"state_from\":%d,\"state_to\":%d,\"ch\":%d,\"freq_mhz\":%d,"
         "\"aa\":\"%08x\",\"crc_init\":\"%06x\",\"interval_us\":%d,\"hop\":%d,\"chm\":\"%02x%02x%02x%02x%02x\"}\n",
         (double)e->ts_us / 1e6, e->event, e->state_from, e->state_to, e->ch, e->freq_mhz, e->access_addr, e->crc_init & 0xFFFFFFu,
         e->interval_us, e->hop, e->chm[0], e->chm[1], e->chm[2], e->chm[3], e->chm[4]);
}
// time at which chunk k and its look-ahead are complete: what the reference's wall clock shows when it runs receiver() on it
int64_t chunk_done_us(long long k) { return (int64_t)(((k + 1) * 8192ll + BTLE_LOOKAHEAD_INT8 / 2) / 4); }

// ---- --connections: btle_b200.hop.ConnectionMonitor's policy over a 40-capture session (capture i = channel i) ----------
struct ConnMonitor {
  static constexpr double kEventSpan = 3.75e-3;        // hop.EVENT_SPAN_S
  static constexpr int kMinEvents = 4;                 // discover_connections(min_events=4)
  static constexpr double kGroupS = 8.0;               // ConnectionMonitor(group_s=8.0)
  double t_now = 0.0;
  btle_b200_streams *ss;
  const Options &o;
  struct Conn {
    uint32_t aa, crc_init;
    bool discovered, tracked = false, announced_start = false, stopped = false;
    int interval = 0, hop = 0, first_ch = 0;           // interval in 1.25 ms units
    double ts = 0.0;                                   // CONNECT_REQ time or first empty PDU
    long long from = 0;
    std::vector<size_t> cfgs;
  };
  struct Group { std::vector<std::pair<double, int>> ev; int conn = -1; };
  std::vector<Conn> conns;
  std::map<std::pair<uint32_t, uint32_t>, Group> groups;
  std::set<uint32_t> announced;
  int added = 0;                                       // cfgs added by the last hand_out
  int rc = 0;

  ConnMonitor(btle_b200_streams *s, const Options &opt) : ss(s), o(opt) {}

  int begin() {
    int64_t until;
    for (size_t c = 0; c < 37 && !rc; ++c) rc = btle_b200_streams_remove_cfg(ss, c, &until);
    std::vector<int32_t> ch(40, -1);
    for (int c = 0; c < 37; ++c) ch[c] = c;
    if (!rc) rc = btle_b200_streams_set_discover(ss, ch.data());
    return rc;
  }
  void start(Conn &c) {
    int64_t from = 0;
    btle_b200_streams_resident(ss, &from);
    c.from = from;
    for (int ch = 0; ch < 37 && !rc; ++ch) {
      const btle_stream_cfg cfg{ch, c.aa, 0xFFFFFFFFu, c.crc_init, 0,
                                (o.rssi ? BTLE_CFG_RSSI : 0) | (o.recover ? BTLE_CFG_RECOVER : 0) | (o.symbol_spaced ? BTLE_CFG_SYMBOL_SPACED : 0) |
                                    (o.centre_hits ? BTLE_CFG_CENTRE_HITS : 0) | (o.correct ? BTLE_CFG_CORRECT : 0) |
                                    (o.lowpass ? BTLE_CFG_LOWPASS : 0) | (o.offset_search ? BTLE_CFG_OFFSET_SEARCH : 0)};
      size_t j = 0;
      rc = btle_b200_streams_add_cfg(ss, (size_t)ch, &cfg, from, &j);
      c.cfgs.push_back(j);
      ++added;
    }
    if (!o.quiet)
      printf("%.6f Connection AA:%08x CRCInit:%06x %s Interval:%dus Hop:%d Ch%d FromChunk:%lld\n", c.ts, c.aa, c.crc_init & 0xFFFFFFu,
             c.discovered ? "discovered" : "CONNECT_REQ", c.tracked ? c.interval * 1250 : -1, c.tracked ? c.hop : -1, c.first_ch, c.from);
    note_tracked(c);
  }
  void note_tracked(Conn &c) {                         // one hop track_start line, as hop.hop_events() forms it
    if (!o.json || !c.tracked || c.announced_start) return;
    c.announced_start = true;
    printf("{\"v\":1,\"t\":\"hop\",\"ts\":%.6f,\"event\":\"track_start\",\"state_from\":0,\"state_to\":1,\"ch\":%d,\"freq_mhz\":%d,"
           "\"aa\":\"%08x\",\"crc_init\":\"%06x\",\"interval_us\":%d,\"hop\":%d,\"chm\":\"1fffffffff\"}\n",
           c.ts, c.first_ch, (int)(freq_by_channel(c.first_ch) / 1000000), c.aa, c.crc_init & 0xFFFFFFu, c.interval * 1250, c.hop);
  }
  void stop(Conn &c) {
    int64_t until;
    for (size_t j : c.cfgs) if (!rc) rc = btle_b200_streams_remove_cfg(ss, j, &until);
    c.cfgs.clear();
    c.stopped = true;
  }
  // hop._connection_from_events: interval = GCD of the gaps in 1.25 ms units, hop = dch * m^-1 (mod 37)
  static void from_events(Conn &c, const std::vector<std::pair<double, int>> &ev) {
    long long interval = 0;
    std::vector<long long> units;
    for (size_t i = 1; i < ev.size(); ++i) {
      units.push_back((long long)std::nearbyint((ev[i].first - ev[i - 1].first) / 1.25e-3));   // round half to even, as Python
      long long a = interval, b = std::llabs(units.back());
      while (b) { const long long t = a % b; a = b; b = t; }
      interval = a;
    }
    bool ok = interval >= 6 && interval <= 3200;
    std::set<int> hops;
    if (ok)
      for (size_t i = 1; i < ev.size(); ++i) {
        const int m = (int)(((units[i - 1] / interval) % 37 + 37) % 37);
        if (m == 0) { ok = ok && ev[i].second == ev[i - 1].second; continue; }
        int inv = 1;
        while (inv * m % 37 != 1) ++inv;
        hops.insert((((ev[i].second - ev[i - 1].second) * inv) % 37 + 37) % 37);
      }
    ok = ok && hops.size() == 1 && !hops.count(0);
    c.tracked = ok;
    c.interval = ok ? (int)interval : 0;
    c.hop = ok ? *hops.begin() : 0;
    c.ts = ev[0].first;
    c.first_ch = ev[0].second;
  }
  // records just handed out (and the candidates of the same sets)
  void hand_out(const btle_pkt_rec *r, size_t n) {
    added = 0;
    for (size_t i = 0; i < n && !rc; ++i) {
      const uint8_t *b = r[i].bytes, *p = b + 2;
      t_now = std::max(t_now, rec_time(r[i]));
      if (r[i].stream < 37 || r[i].stream >= 40 || r[i].crc_bad || (b[0] & 0x0F) != 5 || (b[1] & 0x3F) != 34) continue;
      Conn c{};
      c.aa = (uint32_t)p[12] | (uint32_t)p[13] << 8 | (uint32_t)p[14] << 16 | (uint32_t)p[15] << 24;
      c.crc_init = (uint32_t)p[16] << 16 | (uint32_t)p[17] << 8 | p[18];
      c.interval = p[22] | p[23] << 8;
      c.hop = p[33] & 0x1F;
      c.tracked = p[28] == 0xFF && p[29] == 0xFF && p[30] == 0xFF && p[31] == 0xFF && p[32] == 0x1F && c.interval > 0;
      c.discovered = false;
      c.ts = rec_time(r[i]);
      c.first_ch = c.hop % 37;
      announced.insert(c.aa);
      for (Conn &d : conns)                            // announced after all: the CONNECT_REQ connection takes it over
        if (d.discovered && d.aa == c.aa && !d.stopped) stop(d);
      conns.push_back(c);
      start(conns.back());
    }
    std::vector<btle_conn_cand> cand(4096);
    std::vector<btle_conn_cand> all;
    for (;;) {
      size_t got = 0;
      const int q = btle_b200_streams_take_cands(ss, cand.data(), cand.size(), &got);
      all.insert(all.end(), cand.begin(), cand.begin() + (long)got);
      if (q != BTLE_EOVERFLOW) break;
    }
    std::stable_sort(all.begin(), all.end(), [](const btle_conn_cand &a, const btle_conn_cand &b) {
      if (a.access_addr != b.access_addr) return a.access_addr < b.access_addr;
      if (a.crc_init != b.crc_init) return a.crc_init < b.crc_init;
      return a.sample < b.sample;
    });
    for (const btle_conn_cand &c : all) {
      auto &ev = groups[{c.access_addr, c.crc_init}].ev;
      const double t = (double)c.sample / 4.0e6;
      if (!ev.empty() && c.channel == ev.back().second && t - ev.back().first < kEventSpan) continue;
      ev.push_back({t, (int)c.channel});
    }
    for (const btle_conn_cand &c : all) t_now = std::max(t_now, (double)c.sample / 4.0e6);
    for (auto it = groups.begin(); it != groups.end();)     // noise groups that stopped: forgotten (ConnectionMonitor.group_s)
      it = it->second.conn < 0 && (int)it->second.ev.size() < kMinEvents && t_now - it->second.ev.back().first > kGroupS ? groups.erase(it) : std::next(it);
    for (auto &kv : groups) {
      Group &g = kv.second;
      if ((int)g.ev.size() < kMinEvents || announced.count(kv.first.first) || rc) continue;
      if (g.conn < 0) {
        Conn c{};
        c.aa = kv.first.first; c.crc_init = kv.first.second; c.discovered = true;
        from_events(c, g.ev);
        g.conn = (int)conns.size();
        conns.push_back(c);
        start(conns.back());
      } else if (!conns[(size_t)g.conn].stopped) {
        from_events(conns[(size_t)g.conn], g.ev);
        note_tracked(conns[(size_t)g.conn]);
      }
    }
  }
};

// The raw captures: every -i, then DIR/chNN.bin of --iq-dir, with their carrier offsets (--offset auto: estimated here
// from a first pass).  *use_off: some capture has a correction.  Returns the exit status.
int load_captures(btle_b200_ctx *ctx, const Options &o, std::vector<Capture> &caps, bool *use_off) {
  for (const std::string &f : o.iq_files) caps.push_back(parse_capture(f, o));
  if (o.iq_dir) {
    for (int ch = 0; ch < 40; ++ch) {
      char name[512];
      snprintf(name, sizeof name, "%s/ch%02d.bin", o.iq_dir, ch);
      if (access(name, R_OK) != 0) continue;
      const bool adv = ch >= 37;
      caps.push_back(Capture{name, ch, adv ? 0x8E89BED6u : o.aa, adv ? 0x555555u : o.crc_init, o.offset_hz, false});
    }
    if (caps.empty()) { printf("no chNN.bin capture found in %s\n", o.iq_dir); return 1; }
  }
  for (const Capture &c : caps)
    if (c.chan < 0 || c.chan > 39) { printf("channel number must be within 0~%d!\n", 39); return 1; }
  if (o.connections && caps.size() != 40) { printf("--connections needs all 40 chNN.bin captures in %s\n", o.iq_dir); return 1; }
  // carrier-offset correction: --offset HZ for every capture, FILE:CH:AA:CRCINIT:HZ for one, --offset auto from a first pass
  *use_off = o.offset_set;
  for (const Capture &c : caps) *use_off |= c.own_hz;
  if (!o.offset_auto) return 0;
  for (Capture &c : caps) {
    if (c.own_hz) continue;
    struct stat sb;
    if (c.file == "-" || stat(c.file.c_str(), &sb) != 0 || !S_ISREG(sb.st_mode)) {
      printf("--offset auto needs regular files (%s is not one)\n", c.file.c_str());
      return 1;
    }
    std::vector<int8_t> iq;
    if (!load_raw(c.file.c_str(), iq)) return 1;
    if (estimate_offset(ctx, iq, btle_stream_cfg{c.chan, c.aa, o.mask, c.crc_init, 0, cfg_flags(o)}, c.file.c_str(), &c.hz)) return 1;
  }
  return 0;
}

// Each mode returns the exit status and, when it is 0, the sample time at which the input ended (*t_end).

// ---- --iq-bin16: 8 samples per symbol, the Python / Verilog model's receiver over the capture ------------------------------
int run_sps8(btle_b200_ctx *ctx, const Options &o, Sinks &sinks, double *t_end) {
  std::vector<int8_t> raw;
  if (!load_raw(o.iq_bin16, raw)) return 1;
  const size_t n_samples = raw.size() / 4;
  std::vector<btle_sps8_rec> recs(n_samples / 576 + 16);
  size_t n = 0;
  const int rc = btle_b200_rx_sps8(ctx, reinterpret_cast<const int16_t *>(raw.data()), n_samples, o.chan, o.crc_init, o.aa, recs.data(), recs.size(), &n);
  if (rc) return fail(ctx, rc, "btle_b200_rx_sps8");
  const bool adv = (o.chan == 37 || o.chan == 38 || o.chan == 39);
  for (size_t i = 0; i < n && !g_stop; ++i) {
    const btle_model_rx_rec &m = recs[i].rx;
    if (!m.found || m.n_pdu_bits < 16) continue;         // no header decoded: nothing the sinks could show
    btle_pkt_rec r;
    memset(&r, 0, sizeof r);
    const int have = m.n_pdu_bits / 8;                    // header + payload bytes that were decoded (CRC clamp, btlelib.py:488-490)
    memcpy(r.bytes, m.pdu, (size_t)std::min(have, 39));
    const int plen = std::min(have - 2, (int)(r.bytes[1] & (adv ? 0x3F : 0x1F)));
    r.bytes[1] = (uint8_t)((r.bytes[1] & (adv ? 0xC0 : 0xE0)) | plen);
    r.channel = (uint8_t)o.chan; r.access_addr = o.aa; r.flags = adv ? 2 : 0;
    r.crc_bad = m.crc_ok ? 0 : 1;
    r.n_bytes = (uint8_t)(plen + 5);
    sinks.packet(r, (double)recs[i].sample / 8.0e6);
  }
  *t_end = (double)n_samples / 8.0e6;
  return 0;
}

// ---- -o with --iq-dir: connection following over per-channel captures -------------------------------------------------
int run_hop(btle_b200_ctx *ctx, const Options &o, const std::vector<Capture> &caps, bool use_off, Sinks &sinks, double *t_end) {
  std::vector<std::vector<int8_t>> iq(40);
  std::vector<float> hz_of(40, 0.0f);                        // the offset of each channel's capture
  size_t n = SIZE_MAX;
  for (const Capture &c : caps) {
    if (!load_raw(c.file.c_str(), iq[c.chan])) return 1;
    n = std::min(n, iq[c.chan].size());
    hz_of[c.chan] = c.hz;
  }
  if (iq[o.chan].empty()) { printf("no capture of the start channel %d in %s\n", o.chan, o.iq_dir); return 1; }
  const long long nchunks = (long long)(n / BTLE_CHUNK_INT8);
  HopRun run{&o};
  btle_hop_hooks hooks{hop_now, hop_set_freq, hop_event, &run, o.quiet};
  btle_b200_set_hop_hooks(&hooks);
  int chan = o.chan;
  uint32_t aa = o.aa, crc_internal = btle_b200_crc_init_reorder(o.crc_init);
  // pass A: the start channel with the command line's access address, all chunks
  std::vector<btle_pkt_rec> recs;
  btle_stream_cfg cfg0{o.chan, o.aa, o.mask, o.crc_init, o.raw, cfg_flags(o)};
  int rc = rx_batch_grow(ctx, iq[o.chan].data(), 1, n, n, &cfg0, recs, use_off ? &hz_of[o.chan] : nullptr);
  if (rc) return fail(ctx, rc, "btle_b200_rx_batch");
  size_t ri = 0;
  long long k = 0;
  for (; k < nchunks && !g_stop; ++k) {
    for (; ri < recs.size() && recs[ri].chunk == k; ++ri) sinks.packet(recs[ri], rec_time(recs[ri]));
    run.now = chunk_done_us(k);
    if (btle_b200_receiver_controller(nullptr, o.verbose, &chan, &aa, &crc_internal) != 0) break;   // :2655-2658
    if (chan != o.chan) { ++k; break; }                    // track start: the radio now sits on a data channel
  }
  if (chan != o.chan && k < nchunks) {
    // pass B: every data channel from chunk k on, with the connection's parameters, one batched launch
    const btle_receiver_status *st = btle_b200_receiver_status();
    const size_t off = (size_t)k * BTLE_CHUNK_INT8, n2 = n - off, stride = (n2 + 15) & ~size_t(15);
    std::vector<int> chan_of;
    for (int c = 0; c < 37; ++c) if (!iq[c].empty()) chan_of.push_back(c);
    std::vector<int8_t> stage(stride * chan_of.size());
    std::vector<btle_stream_cfg> cfgs;
    std::vector<float> hz;
    for (size_t s_ = 0; s_ < chan_of.size(); ++s_) {
      memcpy(stage.data() + s_ * stride, iq[chan_of[s_]].data() + off, n2);
      cfgs.push_back(btle_stream_cfg{chan_of[s_], st->access_addr, o.mask, st->crc_init, o.raw, cfg_flags(o)});
      hz.push_back(hz_of[chan_of[s_]]);
    }
    std::vector<btle_pkt_rec> data;
    rc = rx_batch_grow(ctx, stage.data(), chan_of.size(), stride, n2, cfgs.data(), data, use_off ? hz.data() : nullptr);
    if (rc) return fail(ctx, rc, "btle_b200_rx_batch");
    // index: first record of every (stream, chunk)
    std::vector<size_t> first(chan_of.size() * (size_t)(nchunks - k) + 1, 0);
    {
      size_t p = 0;
      for (size_t b = 0; b + 1 < first.size(); ++b) {
        const int s_ = (int)(b / (size_t)(nchunks - k)), c = (int)(b % (size_t)(nchunks - k));
        while (p < data.size() && (data[p].stream < s_ || (data[p].stream == s_ && data[p].chunk < c))) ++p;
        first[b] = p;
      }
      first.back() = data.size();
    }
    std::vector<int> stream_of(40, -1);
    for (size_t s_ = 0; s_ < chan_of.size(); ++s_) stream_of[chan_of[s_]] = (int)s_;
    for (; k < nchunks && !g_stop; ++k) {
      const int s_ = stream_of[chan];
      if (s_ >= 0) {
        const size_t b = (size_t)s_ * (size_t)(nchunks - (long long)(off / BTLE_CHUNK_INT8)) + (size_t)(k - (long long)(off / BTLE_CHUNK_INT8));
        for (size_t p = first[b]; p < first[b + 1]; ++p) {
          btle_pkt_rec r = data[p];
          r.chunk += (int32_t)(off / BTLE_CHUNK_INT8);
          sinks.packet(r, rec_time(r));
        }
      }
      run.now = chunk_done_us(k);
      if (btle_b200_receiver_controller(nullptr, o.verbose, &chan, &aa, &crc_internal) != 0) break;
    }
  }
  btle_b200_set_hop_hooks(nullptr);
  *t_end = (double)(n / 2) / 4.0e6;
  return 0;
}

// ---- --iq-txt / --iq-sc16: whole-file formats, one rx_batch call ----------------------------------------------------
int run_whole_file(btle_b200_ctx *ctx, const Options &o, Sinks &sinks, double *t_end) {
  std::vector<int8_t> iq;
  if (o.iq_sc16 ? !load_raw(o.iq_sc16, iq) : !load_txt(o.iq_txt, iq)) return 1;
  if (o.iq_sc16) {                                           // SC16Q11 to int8 as btle_rx's bladeRF build does, btle_rx.c:307-308
    const int16_t *p16 = reinterpret_cast<const int16_t *>(iq.data());
    std::vector<int8_t> r(iq.size() / 2);
    for (size_t i = 0; i < r.size(); ++i) r[i] = (int8_t)((p16[i] >> 4) & 0xFF);
    iq.swap(r);
  }
  btle_stream_cfg cfg{o.chan, o.aa, o.mask, o.crc_init, o.raw, cfg_flags(o)};
  float hz = o.offset_hz;
  if (o.offset_auto && estimate_offset(ctx, iq, cfg, o.iq_txt ? o.iq_txt : "capture", &hz)) return 1;
  std::vector<btle_pkt_rec> recs;
  const int rc = rx_batch_grow(ctx, iq.data(), 1, iq.size(), iq.size(), &cfg, recs, o.offset_set ? &hz : nullptr);
  if (rc) return fail(ctx, rc, "btle_b200_rx");
  for (size_t i = 0; i < recs.size() && !g_stop; ++i) sinks.packet(recs[i], rec_time(recs[i]));
  *t_end = (double)(iq.size() / 2) / 4.0e6;
  return 0;
}

// ---- raw captures (every -i, --iq-dir without -o), streamed through one session (btle_b200_streams_*): poll() across the
//      inputs, read() into whichever capture has data and room, one batched launch per segment set --------------------------
int run_session(btle_b200_ctx *ctx, const Options &o, const std::vector<Capture> &caps, bool use_off, Sinks &sinks, double *t_end) {
  const size_t ns = caps.size();
  Inputs in;
  size_t n_stdin = 0;
  for (const Capture &c : caps) {
    if (c.file == "-") {
      if (n_stdin++) { printf("'-' (stdin) can be the input of one capture only\n"); return 1; }
      in.fds.push_back(0);
      continue;
    }
    in.fds.push_back(open(c.file.c_str(), O_RDONLY));         // a FIFO: waits here until its writer has opened it
    if (in.fds.back() < 0) { perror(c.file.c_str()); return 1; }
  }
  std::vector<btle_stream_cfg> cfgs;
  for (const Capture &c : caps) cfgs.push_back(btle_stream_cfg{c.chan, c.aa, o.mask, c.crc_init, o.raw, cfg_flags(o)});
  btle_b200_streams *ss = nullptr;
  int rc = btle_b200_streams_open(ctx, cfgs.data(), ns, o.segment_chunks, &ss);
  const std::unique_ptr<btle_b200_streams, StreamsClose> session(ss);
  if (rc) return fail(ctx, rc, "btle_b200_streams_open");
  for (size_t s_ = 0; s_ < ns && use_off && !rc; ++s_) rc = btle_b200_streams_set_offset(ss, s_, caps[s_].hz);
  if (rc) return fail(ctx, rc, "btle_b200_streams_set_offset");
  ConnMonitor mon(ss, o);
  if (o.connections && mon.begin()) return fail(ctx, mon.rc, "--connections");
  std::vector<btle_pkt_rec> recs(65536), pending;
  long long max_chunk = -1;
  // A record is printed once no record still to come can sort in front of it: every such record lies in a chunk behind
  // max_chunk, and a hit starts at most 124 samples before its chunk.
  auto emit = [&](bool all) {
    long long safe = (max_chunk + 1) * 8192 - 124;
    if (o.connections) {                                     // a backfilled record can lie anywhere in the resident sets
      int64_t res = 0;
      btle_b200_streams_resident(ss, &res);
      safe = std::min<long long>(safe, (long long)res * 8192 - 124);
    }
    if (print_in_order(pending, sinks, all ? LLONG_MAX : safe)) fflush(stdout);
  };
  auto keep = [&](size_t n) {
    for (size_t i = 0; i < n; ++i) { pending.push_back(recs[i]); max_chunk = std::max<long long>(max_chunk, recs[i].chunk); }
    if (o.connections) { mon.hand_out(recs.data(), n); if (mon.rc && !rc) rc = mon.rc; }
  };
  std::vector<size_t> total(ns, 0);
  std::vector<char> eof(ns, 0);
  size_t shortest = SIZE_MAX;                                 // length of the shortest capture once one has ended
  while (!g_stop && rc == 0) {
    std::vector<pollfd> pf;
    std::vector<size_t> who;
    for (size_t s_ = 0; s_ < ns; ++s_) {
      if (eof[s_] || total[s_] >= shortest) continue;         // bytes behind the shortest capture are not decoded
      int8_t *buf; size_t space;
      btle_b200_streams_acquire(ss, s_, &buf, &space);
      if (space) { pf.push_back(pollfd{in.fds[s_], POLLIN, 0}); who.push_back(s_); }   // else: waits for the other captures
    }
    if (pf.empty()) break;
    if (poll(pf.data(), pf.size(), -1) < 0) {
      if (errno == EINTR) continue;
      perror("poll");
      break;
    }
    for (size_t k = 0; k < pf.size() && rc == 0; ++k) {
      if (!(pf[k].revents & (POLLIN | POLLHUP | POLLERR))) continue;
      const size_t s_ = who[k];
      int8_t *buf; size_t space;
      btle_b200_streams_acquire(ss, s_, &buf, &space);
      const ssize_t got = read(in.fds[s_], buf, std::min(space, size_t(8) << 20));
      if (got < 0 && errno == EINTR) continue;
      if (got <= 0) {
        if (got < 0) perror(caps[s_].file.c_str());
        eof[s_] = 1;
        shortest = std::min(shortest, total[s_]);
        continue;
      }
      total[s_] += (size_t)got;
      size_t n = 0;
      rc = btle_b200_streams_commit(ss, s_, (size_t)got, recs.data(), recs.size(), &n);
      keep(n);
      while (rc == 0 && n == recs.size()) { rc = btle_b200_streams_commit(ss, s_, 0, recs.data(), recs.size(), &n); keep(n); }
      emit(false);
    }
  }
  if (rc) return fail(ctx, rc, "btle_b200_streams_commit");
  for (bool more = true; more && rc == 0;) {                 // end of input or SIGINT: decode up to the shortest capture
    more = false;
    for (;;) {
      size_t n = 0;
      rc = btle_b200_streams_finish(ss, recs.data(), recs.size(), &n);
      keep(n);
      more |= o.connections && mon.added > 0;                // new connections: their backfill comes from the next finish
      if (rc != BTLE_EOVERFLOW) break;
    }
  }
  if (rc) return fail(ctx, rc, "btle_b200_streams_finish");
  const size_t n_read = *std::min_element(total.begin(), total.end());
  if (g_stop) {
    // stopped mid-stream: print only what a full run prints first — the chunks whose look-ahead had arrived on every
    // capture (the tail decode read zeros behind them), up to where a later chunk's hit could sort in front
    const long long done = n_read >= (size_t)BTLE_LOOKAHEAD_INT8 ? (long long)((n_read - BTLE_LOOKAHEAD_INT8) / BTLE_CHUNK_INT8) : 0;
    pending.erase(std::remove_if(pending.begin(), pending.end(), [&](const btle_pkt_rec &r) { return r.chunk >= done; }), pending.end());
    max_chunk = done - 1;
    emit(false);
  } else {
    emit(true);
  }
  *t_end = (double)(n_read / 2) / 4.0e6;
  return 0;
}

}  // namespace

int main(int argc, char **argv) {
  printf("BLE sniffer (B200 offline receive chain; option surface of btle_rx by Xianjun Jiao)\n\n");
  Options o = parse_commandline(argc, argv);
  if (o.freq_hz == 123) o.freq_hz = freq_by_channel(o.chan);                    // btle_rx.c:2558
  if (!o.quiet)
    printf("Cmd line input: chan %d, freq %ldMHz, access addr %08x, crc init %06x raw %d verbose %d rx %ddB (%s) file=%s\n", o.chan,
           (long)(o.freq_hz / 1000000), o.aa, o.crc_init, o.raw, o.verbose, o.gain, "B200-file", o.pcap ? o.pcap : "(null)");
  Sinks sinks(o);
  if (o.pcap) {
    if (!o.quiet) printf("will store packets to: %s\n", o.pcap);
    sinks.pcap.reset(pcap_open(o.pcap));
    if (!sinks.pcap) { perror(o.pcap); return 1; }
  }
  if (o.json) json_status(0.0, "start", o);
  if (o.iq_files.empty() && !o.iq_txt && !o.iq_sc16 && !o.iq_dir && !o.iq_bin16) {
    printf("open_board: no SDR support in this build; give a capture with -i/--iq-file\n");
    if (o.json) json_status(0.0, "stop", o);
    return 1;                                                                   // btle_rx.c:2586
  }
  struct sigaction sa;
  memset(&sa, 0, sizeof sa);
  sa.sa_handler = on_sigint;
  sigaction(SIGINT, &sa, nullptr);
  sigaction(SIGTERM, &sa, nullptr);

  btle_b200_bind_host_numa(o.device, nullptr);                                  // page-locked buffers next to the GPU
  btle_b200_ctx *created = nullptr;
  const int rc = btle_b200_create(&created, o.device);
  const std::unique_ptr<btle_b200_ctx, CtxClose> ctx(created);
  if (rc) { printf("btle_b200_create: %s\n", btle_b200_strerror(rc)); return 1; }
  btle_b200_hop_reset();
  std::vector<Capture> caps;
  bool use_off = false;
  if (const int st = load_captures(ctx.get(), o, caps, &use_off)) return st;

  double t_end = 0.0;
  int st;
  if (o.iq_bin16) st = run_sps8(ctx.get(), o, sinks, &t_end);
  else if (o.hop && o.iq_dir) st = run_hop(ctx.get(), o, caps, use_off, sinks, &t_end);
  else if ((o.iq_txt || o.iq_sc16) && !o.iq_dir && caps.size() <= 1) st = run_whole_file(ctx.get(), o, sinks, &t_end);
  else st = run_session(ctx.get(), o, caps, use_off, sinks, &t_end);
  if (st) return st;

  fflush(stdout);
  if (!o.quiet) printf("Exit main loop ...\n");                                 // :2664
  if (o.json) json_status(t_end, "stop", o);
  return 0;
}
