// btle_rx_kernels.cu — sm_90a kernels of the BLE receive path + the C-ABI (include/btle_b200.h).
//
// btle_rx_persistent_kernel does the whole receive chain of the reference's receiver()
// (btle_rx.c:2188-2391): one persistent, warp-specialised CTA per SM.
//   dense warps     IQ tile (one TMA box, 128B swizzle) -> per-lane discriminator bits packed into
//                   phase words (btle_core.cuh: 1 PRMT + 2 IDP.2A + 1 SHF per sample) -> 12-tap
//                   bit-parallel prefilter of the 32-tap access-address match against the neighbour
//                   lane's words (__shfl_down_sync) -> candidate words + group flags (ballot)
//   resolver warps  one lane per chunk replays the reference's greedy loop on the phase words:
//                   zero-history partial windows, exact re-check of candidates, dewhiten, header
//                   parse, length guards, CRC-24 (4 bytes per step), 64-byte record appended
//   ring            4 span slots between them, mbarrier full/empty protocol
// Also here: leaf kernels with the reference's function signatures (unit parity), the Python
// model's receiver batched one warp per packet, and the transmit PHY (one 4- and 8-sps modulator block,
// gfsk_block, shared by the modulator, capture-synthesiser and BER kernels).
// No tensor cores: the path has no dense contraction (integer compare / bit work on a stream).
#include <cuda.h>
#include <cuda_runtime.h>

#include <sched.h>
#include <sys/syscall.h>
#include <unistd.h>

#include <algorithm>
#include <climits>
#include <cmath>
#include <cstdio>
#include <cstring>
#include <memory>
#include <new>
#include <string>
#include <thread>
#include <type_traits>
#include <vector>

#include "../../include/btle_b200.h"
#include "btle_core.cuh"
#include "btle_params.h"

using namespace btle;

// ----------------------------------------------------------------------------------------------
// protocol tables in constant memory (generated at context creation, verified against the
// reference's scramble_table.h / crc_table in tests)
__constant__ uint32_t c_whiten_words[40][12];
__constant__ uint32_t c_crc4[1024];
__constant__ int8_t c_cos1024[1024], c_sin1024[1024];   // round(127 cos/sin(2 pi k/1024)), gauss_cos_sin_table.h
__constant__ int8_t c_cos2048[2048], c_sin2048[2048];   // btlelib.py:52-66 (sin_cos_gen)
__constant__ int c_gauss4[9] = {2, 11, 32, 53, 60, 53, 32, 11, 2};                       // btle_tx.c gauss_coef_int8[4..12]
__constant__ int c_gauss8[17] = {0, 0, 0, 1, 4, 9, 15, 22, 24, 22, 15, 9, 4, 1, 0, 0, 0};  // btlelib.py:146-160   // c_crc4[0..255] == crc_table (btle_rx.c:971-1004)

static_assert(sizeof(btle_pkt_rec) == 64, "record must be 64 bytes");
static_assert(sizeof(btle_stream_cfg) == 24, "cfg must be 24 bytes");
static_assert(sizeof(btle_model_rx_rec) == 80, "model rx record must be 80 bytes");
static_assert(sizeof(btle_synth_truth) == 64, "synth truth record must be 64 bytes");
static_assert(sizeof(btle_sps8_rec) == 96, "sps8 record must be 96 bytes");

#ifdef BTLE_TIMING
// diagnostic builds only (tools/diag_timing.py): per-CTA time stamps in ns
__device__ unsigned long long g_timing[132 * 16];
__device__ __forceinline__ unsigned long long gtime() { unsigned long long t; asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t)); return t; }
#define BTLE_STAMP(slot) do { if (lane == 0) atomicMax(&g_timing[(blockIdx.x % 132) * 16 + (slot)], gtime()); } while (0)
#define BTLE_STAMP_MIN(slot) do { if (lane == 0) atomicMin(&g_timing[(blockIdx.x % 132) * 16 + (slot)], gtime()); } while (0)
// cumulative SM cycles of one warp (slots 12..15: dense TMA waits, dense `empty` waits, resolver `full` waits, dense total)
struct WaitClock {
  long long t0 = 0, sum = 0;
  __device__ __forceinline__ void begin() { t0 = clock64(); }
  __device__ __forceinline__ void end() { sum += clock64() - t0; }
};
#define BTLE_WAIT_SUM(slot, v) do { if (lane == 0) atomicAdd(&g_timing[(blockIdx.x % 132) * 16 + (slot)], (unsigned long long)(v)); } while (0)
extern "C" void btle_b200_debug_timing(unsigned long long *dst, int reset) {
  if (reset) { static unsigned long long z[132 * 16]; for (int i = 0; i < 132 * 16; ++i) z[i] = (i % 16 == 0 || i % 16 == 2) ? ~0ull : 0ull; cudaMemcpyToSymbol(g_timing, z, sizeof z); }
  else cudaMemcpyFromSymbol(dst, g_timing, sizeof(unsigned long long) * 132 * 16);
}
#else
#define BTLE_STAMP(slot) do { } while (0)
#define BTLE_STAMP_MIN(slot) do { } while (0)
struct WaitClock {
  long long sum = 0;
  __device__ __forceinline__ void begin() {}
  __device__ __forceinline__ void end() {}
};
#define BTLE_WAIT_SUM(slot, v) do { } while (0)
#endif

namespace {

// ---- launch shape -----------------------------------------------------------------------------
#ifndef BTLE_DENSE_WARPS
#define BTLE_DENSE_WARPS 16
#endif
#ifndef BTLE_RESOLVE_WARPS
#define BTLE_RESOLVE_WARPS 3
#endif
#ifndef BTLE_SLOTS
#define BTLE_SLOTS 4
#endif
#ifndef BTLE_CTAS_PER_SM
#define BTLE_CTAS_PER_SM 1     // (A/B builds: 2 CTAs of 7 dense + 2 resolver warps and 2 slots share one SM)
#endif
constexpr int kCtasPerSm = BTLE_CTAS_PER_SM;
constexpr int kDenseWarps = BTLE_DENSE_WARPS;  // producers: IQ -> phase words + candidate words
constexpr int kResolveWarps = BTLE_RESOLVE_WARPS;   // consumers: per-chunk greedy decode (alternate spans)
constexpr int kThreads = (kDenseWarps + kResolveWarps) * 32;
// kSpanChunks = 16 chunks per span (btle_core.cuh): one resolver lane per chunk in the chain pass
constexpr int kSlots = BTLE_SLOTS;             // ring of span buffers between producers and consumers
constexpr int kSpanGroups = kGroupsPerChunk * kSpanChunks + kHaloGroups;   // 1036
constexpr int kStageBytes = 8192;              // one warp tile (32 groups = 4096 samples), one TMA box
constexpr int kHaloRows = kHaloGroups;         // rows of the last (look-ahead) tile of a span: always 12

// The cfgs of the capture a slot's unit reads, when several may read one capture (btle_b200_rx_multi): their prefilter
// taps for the dense warps; each resolver pass loads one cfg's full StreamParams (Smem::rsp).
struct MultiCfg {
  TapSet taps[kMaxCfgsPerCapture];
  int cfg0, ncfg, pad[2];                      // cfgs cfg0 .. cfg0 + ncfg - 1
};
// KC = most cfgs per capture the kernel instantiation decodes: 1 (btle_b200_rx_batch and friends) or kMaxCfgsPerCapture
template <int KC>
struct Slot {
  uint4 pd[kSpanGroups + 1];                   // phase words (+1 zero group behind the data)
  uint32_t cand[kSpanGroups + 4];              // candidate word per group (prefilter, any phase, any cfg)
  uint32_t flagw[2 * kSpanChunks + 2];         // bit l of word t: group 32t+l has candidates
  std::conditional_t<KC == 1, StreamParams, MultiCfg> sp;
};

// Hits the chain pass keeps per chunk (68 x u16): every counted packet fits.  With report_rejected a chunk may have up to
// BTLE_MAX_RECS_PER_CHUNK hits; rows of that size would not fit next to the ring, so the hits behind the row are decoded by
// the chunk's own lane, which runs the chain once more (resolver step 4).
constexpr int kHitCap = BTLE_MAX_PKTS_PER_CHUNK + kRejectedInHitRow + 1;
static_assert(kHitCap >= BTLE_MAX_PKTS_PER_CHUNK && kSpanChunks * BTLE_MAX_RECS_PER_CHUNK < 0x10000, "hit rows / u16 prefix");
struct ResolveScratch {                        // per resolver warp, between the chain pass and the decode pass
  uint16_t hit[kSpanChunks][kHitCap];          // n0 + 124 of the chunk's first kHitCap hits, in the reference's order
  uint16_t pre[kSpanChunks + 2];               // exclusive prefix of the per-chunk counts; [kSpanChunks] = total
  uint16_t xh[2 * kSpanChunks][kExactCap + 1]; // exact access-address hits per flag word (offsets inside the word); [kExactCap] = count
};

template <int KC>
struct SmemBase {
  Slot<KC> slot[kSlots];
  uint32_t crc4[1024];
  ResolveScratch rs[kResolveWarps];
  alignas(1024) unsigned char stage[kDenseWarps][kStageBytes];
  alignas(8) unsigned long long mbar[kDenseWarps];       // TMA completion, one per dense warp
  unsigned long long full[kSlots];                        // kDenseWarps arrivals: span published
  unsigned long long empty[kSlots];                       // 1 arrival: span consumed
};
template <int KC> struct Smem : SmemBase<KC> {};
template <> struct Smem<kMaxCfgsPerCapture> : SmemBase<kMaxCfgsPerCapture> {
  StreamParams rsp[kResolveWarps];                        // the cfg a resolver warp is decoding
};

static_assert(sizeof(Smem<1>) <= (kCtasPerSm == 1 ? 232448 : 116224 - 1024), "Smem exceeds what a CTA can have on sm_90");
static_assert(sizeof(Smem<kMaxCfgsPerCapture>) <= (kCtasPerSm == 1 ? 232448 : 116224 - 1024), "Smem exceeds what a CTA can have on sm_90");
static_assert(kMaxCfgsPerCapture == BTLE_MAX_CFGS_PER_CAPTURE && kMaxCfgsPerCapture <= 32, "one lane per cfg loads the taps");

__device__ __forceinline__ uint32_t smem_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(unsigned long long *bar, int count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
// Ring barriers may stay closed for microseconds: poll politely so the spin does not eat issue slots.
__device__ __forceinline__ void mbar_wait_backoff(unsigned long long *bar, uint32_t parity) {
  uint32_t done = 0;
  for (;;) {
#ifdef BTLE_WAIT_HINT
    // suspend-time hint: the warp sleeps inside the barrier unit and is woken by the phase change, instead of polling
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2, %3;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(done) : "r"(smem_u32(bar)), "r"(parity), "r"(4000u) : "memory");
    if (done) break;
    __nanosleep(500);
#else
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(done) : "r"(smem_u32(bar)), "r"(parity) : "memory");
    if (done) break;
    __nanosleep(200);
#endif
  }
}
__device__ __forceinline__ void mbar_arrive(unsigned long long *bar) {
  asm volatile("mbarrier.arrive.release.cta.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(unsigned long long *bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(unsigned long long *bar, uint32_t parity) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "WAIT_%=:\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
      "@p bra DONE_%=;\n\t"
      "bra WAIT_%=;\n\t"
      "DONE_%=:\n\t}"
      ::"r"(smem_u32(bar)), "r"(parity) : "memory");
}
// TMA tiled copy (cp.async.bulk.tensor, SASS UTMALDG): box {128 B, rows, 2 halves, 1 stream} of the
// IQ tensor {128 B, 256-byte runs, 2 halves, streams} -> shared, 128B-swizzled, completion counted
// in bytes on an mbarrier.
__device__ __forceinline__ void tma_load_tile(void *smem_dst, const CUtensorMap *map, int run, int stream, unsigned long long *bar) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3, %4, %5}], [%6];"
      ::"r"(smem_u32(smem_dst)), "l"(map), "r"(0), "r"(run), "r"(0), "r"(stream), "r"(smem_u32(bar)) : "memory");
}
// Writes one packet record.  Reads the raw IQ only when the caller asked for RSSI.
// `extra`: flags bits on top of raw / advertising / rejected (recovered_flags()).
__device__ __forceinline__ void store_record(btle_pkt_rec *dst, int stream, int chunk, int n0, int nbytes, int crc_bad, bool rejected,
                                             const uint32_t words[11], const StreamParams &sp, const int8_t *iq,
                                             long long n_int8, long long lead, uint32_t extra = 0u) {
  uint32_t mag = 0;
  if (sp.rssi) {                                            // btle_rx.c:2234-2243
    const long long first = (long long)chunk * kChunkInt8 + 2ll * n0;
    for (int k = 0; k < 256; ++k) {
      const long long a = first + k;
      int v = (a >= -lead && a < n_int8) ? (int)iq[a] : 0;     // `lead` bytes in front of the capture are readable (stream segments)
      mag += (uint32_t)(v < 0 ? -v : v);
    }
  }
  uint32_t r[16];
  r[0] = (uint32_t)stream;
  r[1] = (uint32_t)chunk;
  r[2] = (uint32_t)n0;
  r[3] = (uint32_t)sp.channel | ((uint32_t)nbytes << 8) | ((uint32_t)crc_bad << 16) |
         ((uint32_t)((sp.raw ? 1 : 0) | (sp.adv ? 2 : 0) | (rejected ? BTLE_REC_REJECTED : 0) | extra) << 24);
  r[4] = sp.aa;
  r[5] = (mag & 0xFFFFu) | (words[0] << 16);                // mag_sum, bytes[0..1]
#pragma unroll
  for (int j = 1; j < 11; ++j) r[5 + j] = (words[j - 1] >> 16) | (words[j] << 16);
  uint4 *d4 = reinterpret_cast<uint4 *>(dst);
#pragma unroll
  for (int q = 0; q < 4; ++q) d4[q] = make_uint4(r[4 * q], r[4 * q + 1], r[4 * q + 2], r[4 * q + 3]);
}

// BTLE_CFG_RECOVER: stores the record of a counted packet whose primary decode failed the CRC when one of its
// alternatives passes (recover_packet) and returns true; false: nothing stored, the caller stores the primary decode.
// Out of line, so that the decode pass keeps its registers and the launches of cfgs without the flag pay one branch.
// ROT: the symbol-spaced bits are rotated by (c4, s4) (carrier-offset correction).
template <bool ROT>
__device__ __forceinline__ bool store_recovered(btle_pkt_rec *dst, int stream, int chunk, int n0, const StreamParams &sp, const uint32_t *crc4,
                                             const int8_t *iq, long long n_int8, long long lead, int c4 = 0, int s4 = 0) {
  uint32_t words[11];
  int nbytes = 0;
  const int q = recover_packet<ROT>(iq_window(iq, n_int8, chunk), sp, crc4, n0, words, nbytes, c4, s4);
  if (q < 0) return false;
  store_record(dst, stream, chunk, n0, nbytes, 0, false, words, sp, iq, n_int8, lead, recovered_flags(q));
  return true;
}

// Copy one stream's parameters (built on the host by make_params(), uploaded next to the cfg array) into a ring slot:
// one coalesced load of sizeof(StreamParams) = 192 bytes by a warp, no dependent look-ups.
constexpr int kParamWords = (int)(sizeof(StreamParams) / 4);
static_assert(sizeof(StreamParams) % 4 == 0 && kParamWords <= 64, "StreamParams is copied as <= 2 words per lane");
__device__ __forceinline__ void load_params_warp(const StreamParams *__restrict__ src, StreamParams &dst, int lane) {
  const uint32_t *s = reinterpret_cast<const uint32_t *>(src);
  uint32_t *d = reinterpret_cast<uint32_t *>(&dst);
  const uint32_t a = __ldg(s + lane);
  uint32_t b = 0;
  if (lane + 32 < kParamWords) b = __ldg(s + lane + 32);
  d[lane] = a;
  if (lane + 32 < kParamWords) d[lane + 32] = b;
}
// The cfgs of capture group `vs` (vmap[vs] = {capture, first cfg, number of cfgs}) into a slot: lane j builds cfg j's taps.
__device__ __forceinline__ void load_multi_warp(const StreamParams *__restrict__ params, const int4 *__restrict__ vmap, int vs,
                                                MultiCfg &dst, int lane) {
  const int4 v = __ldg(vmap + vs);
  if (lane < v.z) dst.taps[lane] = make_tapset(params[v.y + lane]);
  if (lane == 0) { dst.cfg0 = v.y; dst.ncfg = v.z; }
}

// One persistent CTA per SM.  Units of work (a span of 16 chunks of one capture, or a 4-chunk piece of one in the
// last wave — Plan, btle_core.cuh) are dealt round-robin to CTAs.
// Warps 0..15 (dense): per 4096-sample tile, one TMA box brings the tile into 128B-swizzled shared rows;
//   each lane turns its 128 samples into 4 phase words, prefilters the access-address match against
//   the neighbour lane's words (warp shuffle) and publishes both in the unit's ring slot.
// Warps 16..18 (resolvers, units k = r, r+3, ...): when a unit is complete,
//   1. chain pass, one lane per chunk: the reference's greedy receiver() control flow (search, header length,
//      guards) on the phase words -> positions of the packets the reference counts;
//   2. one warp scan + ONE atomic reserve the unit's block of the output and fill the unit's directory entry;
//   3. decode pass, one lane per PACKET (converged): bytes, dewhitening, CRC-24, 64-byte record stored at its
//      final position — records of a unit are contiguous and in the reference's order.
// Producers and consumers are decoupled through a 4-slot ring with full/empty mbarriers, so the sparse
// passes of unit k overlap the dense pass of units k+1 .. k+3.
// KC > 1 (btle_b200_rx_multi): the plan's streams are capture GROUPS, vmap[g] = {capture, first cfg, number of cfgs}.  A
// capture's IQ still becomes phase words once; the candidate words are the union of its cfgs' prefilters, and the resolver
// runs steps 1a-4 once per cfg, each run with its own directory entry: cfg j's units sit at j * (units per group) + the
// unit's index inside its group, so the directory walks in (cfg, chunk, n0) order.  Records carry stream = cfg index.
// ROT (the *_offset entry points): rot[i] = {C, S, C4, S4} of cfg i (make_rot); the dense warps build the phase words from
// the rotated discriminator (dbits8_rot, with the rotation of the capture's first cfg) and recovery rotates its
// symbol-spaced bits by (C4, S4).  Without ROT, rot is not read.
template <int KC, bool ROT>
__global__ void __launch_bounds__(kThreads, kCtasPerSm)
btle_rx_persistent_kernel(const __grid_constant__ CUtensorMap map32, const __grid_constant__ CUtensorMap map12,
                          const int8_t *__restrict__ iq, long long stream_stride, long long n_int8,
                          const StreamParams *__restrict__ params, const Plan plan,
                          btle_pkt_rec *__restrict__ out, unsigned cap, unsigned *__restrict__ count,
                          uint2 *__restrict__ dir, unsigned *__restrict__ zero_next, long long lead,
                          const int4 *__restrict__ vmap, const int4 *__restrict__ rot) {
  extern __shared__ __align__(128) unsigned char smem_raw[];
  Smem<KC> &M = *reinterpret_cast<Smem<KC> *>(smem_raw);
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int total_units = plan.total_units;
  // capture that group `vs` reads
  auto capture_of = [&](int vs) -> int {
    if constexpr (KC == 1) return vs;
    else return __ldg(&vmap[vs].x);
  };

  BTLE_STAMP_MIN(0);
  // context-owned allocation counters rotate through a ring: this launch clears the one a launch half a ring later will use
  if (zero_next && blockIdx.x == 0 && tid == 0) *zero_next = 0u;
  // ---- dense warps: (span, tile) iterator and TMA request helpers -------------------------------------
  // Each warp walks its own sequence of tiles (tile j of the CTA goes to warp j % 16, across
  // unit boundaries).  A tile is fetched as ONE TMA box: row r of half h (the lower / upper 128
  // bytes of the 256-byte run of group r) lands at (h * rows + r) * 128 B, 128B-swizzled.  As soon
  // as the tile has been consumed the warp's NEXT tile is requested into the buffer; the other 15
  // dense warps' copies are in flight meanwhile.
  unsigned char *stage = M.stage[warp < kDenseWarps ? warp : 0];
  unsigned long long *mbar = &M.mbar[warp < kDenseWarps ? warp : 0];
  // How a tile's bytes get into shared memory.  The tensor map has n_int8/256 rows per capture; rows behind them read
  // as ZERO through TMA (out-of-bounds fill), which is exactly what the reference-equivalent semantics want for the
  // look-ahead behind the end of a capture.  Only a capture whose length is not a multiple of 256 has one partial row
  // that TMA would zero as a whole: the tile that holds it is filled by hand.  A tile entirely behind the capture
  // (the look-ahead tile of a capture's last span) is zeroed in place.
  const int runs = (int)(n_int8 >> 8);
  const bool ragged = (n_int8 & 255) != 0;
  auto tile_mode = [&](int run0, int rows) {              // 0 TMA, 1 by hand, 2 zeros
    if (run0 >= runs + (ragged ? 1 : 0)) return 2;
    return (ragged && runs < run0 + rows) ? 1 : 0;
  };
  struct Cursor {                                         // (unit, tile) iterator of this warp
    int unit, t, rot, tiles, groups, chunk0, stream;
    bool valid;
  };
  auto enter_unit = [&](Cursor &c) {
    c.valid = c.unit < total_units;
    if (c.valid) {
      const UnitInfo ui = unit_info(c.unit, plan);
      c.tiles = ui.tiles; c.groups = ui.groups; c.chunk0 = ui.chunk0; c.stream = capture_of(ui.stream);
      c.t = warp - c.rot;
      if (c.t < 0) c.t += kDenseWarps;
    }
  };
  auto next_unit = [&](Cursor &c) {
    c.rot = (c.rot + c.tiles) % kDenseWarps;
    c.unit += gridDim.x;
    enter_unit(c);
  };
  auto next_tile = [&](Cursor &c) {                       // next tile of this warp, skipping empty units
    c.t += kDenseWarps;
    while (c.valid && c.t >= c.tiles) next_unit(c);
  };
  // descriptor of the tile under the prefetch cursor, refreshed once per tile
  int nx_run0 = 0, nx_stream = 0;
  uint32_t nx_bytes = 0;                                  // bytes of the tile; 0 = nothing to request by TMA
  const CUtensorMap *nx_map = &map32;
  auto describe = [&](const Cursor &c) {
    nx_bytes = 0;
    if (!c.valid) return;
    const int rows = min(32, c.groups - c.t * 32);
    nx_run0 = c.chunk0 * 64 + c.t * 32;
    nx_stream = c.stream;
    nx_map = (rows == 32) ? &map32 : &map12;
    if (tile_mode(nx_run0, rows) == 0) nx_bytes = (uint32_t)rows * 256u;   // else: filled by the consumer itself
  };
  auto request = [&]() {                                  // the described tile
    if (lane == 0 && nx_bytes) {
      mbar_expect_tx(mbar, nx_bytes);
      tma_load_tile(stage, nx_map, nx_run0, nx_stream, mbar);
    }
  };
  Cursor pf;                                              // the tile to request next
  pf.unit = blockIdx.x; pf.rot = 0; pf.valid = false; pf.t = 0; pf.tiles = 0; pf.groups = 0; pf.chunk0 = 0; pf.stream = 0;

  // Start-up.  Warps 0..3 fetch the parameters of the CTA's first four units; their loads are issued BEFORE the tile
  // requests (132 CTAs x 16 warps x 8 KB of TMA traffic would otherwise sit in front of them in the memory system)
  // and consumed after, so both round trips overlap.
  uint32_t pw0 = 0, pw1 = 0;
  const int first_unit = blockIdx.x + warp * gridDim.x;
  const bool has_params = warp < kSlots && first_unit < total_units;
  if (KC == 1 && has_params) {
    const uint32_t *src = reinterpret_cast<const uint32_t *>(params + unit_info(first_unit, plan).stream);
    pw0 = __ldg(src + lane);
    if (lane + 32 < kParamWords) pw1 = __ldg(src + lane + 32);
  }
  if (warp < kDenseWarps) {
    // the first tile is requested right away: its HBM round trip overlaps the rest of the start-up
    if (lane == 0) {
      mbar_init(mbar, 1);
      asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncwarp();
    enter_unit(pf);
    while (pf.valid && pf.t >= pf.tiles) next_unit(pf);
    describe(pf);
    request();
    next_tile(pf);
    describe(pf);
    BTLE_STAMP(10);
  }
  if (tid < kSlots) { mbar_init(&M.full[tid], kDenseWarps); mbar_init(&M.empty[tid], 1); }
  if (has_params) {
    if constexpr (KC == 1) {
      uint32_t *d = reinterpret_cast<uint32_t *>(&M.slot[warp].sp);
      d[lane] = pw0;
      if (lane + 32 < kParamWords) d[lane + 32] = pw1;
    } else {
      load_multi_warp(params, vmap, unit_info(first_unit, plan).stream, M.slot[warp].sp, lane);
    }
    BTLE_STAMP(11);
  }
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  __syncthreads();
  BTLE_STAMP(1);

  if (warp < kDenseWarps) {
    // =============================== dense producers ===============================
    uint32_t tma_phase = 0;                               // parity to wait for on the tile's mbarrier
    int rot_w = 0, k = 0;
    WaitClock w_all, w_tma, w_empty;
    w_all.begin();
    for (int unit = blockIdx.x; unit < total_units; unit += gridDim.x, ++k) {
      const int b = k % kSlots;
      auto &S = M.slot[b];
      const uint32_t use = (uint32_t)(k / kSlots);
      w_empty.begin();
      if (use > 0) mbar_wait_backoff(&M.empty[b], (use - 1) & 1u);   // resolver released the slot's previous unit
      w_empty.end();
      const UnitInfo si = unit_info(unit, plan);
      const int8_t *cap_base = iq + (long long)capture_of(si.stream) * stream_stride;
      int rc = 0, rs = 0;                                 // (C, S) of the capture
      if constexpr (ROT) {
        const int4 r = __ldg(rot + (KC == 1 ? si.stream : __ldg(&vmap[si.stream].y)));
        rc = r.x;
        rs = r.y;
      }
      int t = warp - rot_w;
      if (t < 0) t += kDenseWarps;
      for (; t < si.tiles; t += kDenseWarps) {
        const int rows = min(32, si.groups - t * 32);
        const int run0 = si.chunk0 * 64 + t * 32;
        const long long tile_off = (long long)run0 * 256;
        const int mode = tile_mode(run0, rows);
        const bool tma = mode == 0;
        // first IQ word behind the tile: the sample after the last row's run
        uint32_t tail = 0;
        if (lane == rows - 1) {
          const long long o = tile_off + (long long)rows * 256;
          if (o + 4 <= n_int8) tail = __ldg(reinterpret_cast<const uint32_t *>(cap_base + o));
          else
            for (int bb = 0; bb < 4; ++bb)
              if (o + bb < n_int8) tail |= (uint32_t)(uint8_t)cap_base[o + bb] << (8 * bb);
        }
        if (tma) {
          w_tma.begin();
          mbar_wait(mbar, tma_phase);
          w_tma.end();
          tma_phase ^= 1u;
        } else if (mode == 2) {
          if (lane < rows) {
#pragma unroll
            for (int cc = 0; cc < 16; ++cc)
              *reinterpret_cast<uint4 *>(stage + (((cc >> 3) * rows + lane) << 7) + ((cc & 7) << 4)) = make_uint4(0u, 0u, 0u, 0u);
          }
          __syncwarp();
        } else {
          // the capture's partial last row: bytes past n_int8 read as 0 (same swizzled layout, generic stores)
          if (lane < rows) {
            for (int half = 0; half < 2; ++half) {
              const long long row_off = tile_off + (long long)lane * 256 + 128 * half;
              const int r = half * rows + lane;
              for (int wi = 0; wi < 32; ++wi) {
                const long long o = row_off + 4ll * wi;
                uint32_t w = 0;
                if (o + 4 <= n_int8) w = *reinterpret_cast<const uint32_t *>(cap_base + o);
                else
                  for (int bb = 0; bb < 4; ++bb)
                    if (o + bb < n_int8) w |= (uint32_t)(uint8_t)cap_base[o + bb] << (8 * bb);
                reinterpret_cast<uint32_t *>(stage + (r << 7) + ((((wi >> 2) ^ (r & 7))) << 4))[wi & 3] = w;
              }
            }
          }
          __syncwarp();
        }
        uint32_t acc[4] = {0u, 0u, 0u, 0u};
        uint32_t carry = 0u, wtop = 0u;
        int vtop = 0;
#pragma unroll 1
        for (int half = 1; half >= 0; --half) {
          // 16-byte chunk cc of box row r sits at cc ^ (r & 7) (TMA SWIZZLE_128B): the 8 lanes of a quarter-warp
          // hit 8 different bank groups -> conflict-free LDS.128
          const int r = half * rows + lane;
          const unsigned char *row = stage + (r << 7);
          const uint32_t sw = (uint32_t)(r & 7);
          if (half == 0) {
            // now the neighbour's first word is here: redo the one bit that needed it (sample 127)
            const uint32_t first = reinterpret_cast<const uint4 *>(row + (sw << 4))->x;
            uint32_t nb = __shfl_down_sync(0xFFFFFFFFu, first, 1);
            if (lane == rows - 1) nb = tail;
            if constexpr (ROT) vtop = rot_disc(sext8<2>(wtop), sext8<3>(wtop), sext8<0>(nb), sext8<1>(nb), rc, rs);
            else vtop = sext8<3>(wtop) * sext8<0>(nb) - sext8<2>(wtop) * sext8<1>(nb);
          }
          if (lane < rows) {
#pragma unroll
            for (int cc = 7; cc >= 0; --cc) {
              const uint4 w = *reinterpret_cast<const uint4 *>(row + ((((uint32_t)cc ^ sw)) << 4));
              if (half == 1 && cc == 7) wtop = w.w;
              if constexpr (ROT) {
                if ((cc & 3) == 3) {
#pragma unroll
                  for (int ph = 0; ph < 4; ++ph) acc[ph] <<= 8;
                }
                switch (cc & 3) {
                  case 3: dbits8_rot<3>(w.x, w.y, w.z, w.w, carry, rc, rs, acc); break;
                  case 2: dbits8_rot<2>(w.x, w.y, w.z, w.w, carry, rc, rs, acc); break;
                  case 1: dbits8_rot<1>(w.x, w.y, w.z, w.w, carry, rc, rs, acc); break;
                  default: dbits8_rot<0>(w.x, w.y, w.z, w.w, carry, rc, rs, acc); break;
                }
                carry = w.x;
                continue;
              }
#ifdef BTLE_DBITS_PUSH
              dbits8(w.x, w.y, w.z, w.w, carry, acc);
#else
              if ((cc & 3) == 3) {                          // next byte of the phase words (the walk goes downwards)
#pragma unroll
                for (int ph = 0; ph < 4; ++ph) acc[ph] <<= 8;
              }
              switch (cc & 3) {
                case 3: dbits8_dense<3>(w.x, w.y, w.z, w.w, carry, acc); break;
                case 2: dbits8_dense<2>(w.x, w.y, w.z, w.w, carry, acc); break;
                case 1: dbits8_dense<1>(w.x, w.y, w.z, w.w, carry, acc); break;
                default: dbits8_dense<0>(w.x, w.y, w.z, w.w, carry, acc); break;
              }
#endif
              carry = w.x;
            }
            // sample 127 was pushed first, so after all 32 pushes it is bit 31 of phase 3
            if (half == 0) acc[3] = (acc[3] & 0x7FFFFFFFu) | ((uint32_t)vtop & 0x80000000u);
          }
        }
        __syncwarp();                                     // everyone is done reading the buffer
        request();                                        // the warp's next tile
        next_tile(pf);
        describe(pf);
        BTLE_STAMP_MIN(2);
        if (lane < rows) S.pd[t * 32 + lane] = make_uint4(acc[0], acc[1], acc[2], acc[3]);
        // candidate words: lanes 0..30 see the next group's words through the warp; lane 31 of
        // a full tile is completed by the resolver (its neighbour group belongs to another warp)
        uint32_t hi[4];
#pragma unroll
        for (int ph = 0; ph < 4; ++ph) hi[ph] = __shfl_down_sync(0xFFFFFFFFu, acc[ph], 1);
        uint32_t a = 0u;
        if (t < 2 * si.nch && lane < 31) {
          if constexpr (KC == 1) a = prefilter_any(acc, hi, S.sp);
          else a = prefilter_union(acc, hi, S.sp.taps, S.sp.ncfg);
        }
        const uint32_t fw = __ballot_sync(0xFFFFFFFFu, a != 0u);
        if (lane < rows) S.cand[t * 32 + lane] = a;
        if (lane == 0) {
          S.flagw[t] = fw;
          if (t == si.tiles - 1) S.pd[si.groups] = make_uint4(0u, 0u, 0u, 0u);
        }
      }
      rot_w = (rot_w + si.tiles) % kDenseWarps;
      __syncwarp();
      if (lane == 0) mbar_arrive(&M.full[b]);             // release: this warp's share of the unit is published
      BTLE_STAMP(3);
    }
    w_all.end();
    BTLE_WAIT_SUM(12, w_tma.sum);
    BTLE_WAIT_SUM(13, w_empty.sum);
    BTLE_WAIT_SUM(15, w_all.sum);
  } else {
    // ================================== resolvers ==================================
    // the CRC tables are only needed here: built by the resolver warps while the first unit is in flight
    // (crc4[0..255] = crc_table, btle_rx.c:971-1004; [256k..] = the same followed by k zero bytes)
    {
      const int rt = tid - kDenseWarps * 32, rn = kResolveWarps * 32;
      for (int i = rt; i < 256; i += rn) M.crc4[i] = make_crc_entry((uint32_t)i);
      asm volatile("bar.sync 1, %0;" ::"r"(rn) : "memory");
      for (int kk = 1; kk < 4; ++kk) {
        for (int i = rt; i < 256; i += rn) { const uint32_t x = M.crc4[(kk - 1) * 256 + i]; M.crc4[kk * 256 + i] = M.crc4[x & 0xFFu] ^ (x >> 8); }
        asm volatile("bar.sync 1, %0;" ::"r"(rn) : "memory");
      }
    }
    // resolver warp r takes this CTA's units k = r, r + kResolveWarps, ...
    ResolveScratch &RS = M.rs[warp - kDenseWarps];
    int k = warp - kDenseWarps;
    WaitClock w_full;
    for (int unit = blockIdx.x + k * gridDim.x; unit < total_units; unit += kResolveWarps * gridDim.x, k += kResolveWarps) {
      const int b = k % kSlots;
      auto &S = M.slot[b];
      w_full.begin();
      mbar_wait_backoff(&M.full[b], (uint32_t)(k / kSlots) & 1u);   // all tiles of the unit are published
      w_full.end();
      BTLE_STAMP(4);
      const UnitInfo si = unit_info(unit, plan);
      const int8_t *cap_base = iq + (long long)capture_of(si.stream) * stream_stride;
      for (int t = lane; t < 2 * si.nch; t += 32) {       // lane 31 of every full tile
        const int g = 32 * t + 31;
        const uint4 lo = S.pd[g], hi = S.pd[g + 1];
        const uint32_t l4[4] = {lo.x, lo.y, lo.z, lo.w}, h4[4] = {hi.x, hi.y, hi.z, hi.w};
        uint32_t a;
        if constexpr (KC == 1) a = prefilter_any(l4, h4, S.sp);
        else a = prefilter_union(l4, h4, S.sp.taps, S.sp.ncfg);
        S.cand[g] = a;
        if (a) S.flagw[t] |= 0x80000000u;
      }
      __syncwarp();
      BTLE_STAMP(6);
      // steps 1a-4 once per cfg of the unit's capture (KC == 1: once, with the slot's parameters)
      int ncfg = 1, cfg0 = 0, per_group = 0, local = 0;
      if constexpr (KC > 1) {
        ncfg = S.sp.ncfg;
        cfg0 = S.sp.cfg0;
        per_group = plan.big_units ? plan.spans_per_stream : plan.spans_per_stream << plan.piece_shift;   // the host plans evenly
        local = unit - si.stream * per_group;
      }
      for (int jc = 0; jc < ncfg; ++jc) {
        const StreamParams *spp;
        if constexpr (KC == 1) spp = &S.sp;
        else {
          spp = &M.rsp[warp - kDenseWarps];
          load_params_warp(params + cfg0 + jc, M.rsp[warp - kDenseWarps], lane);
          __syncwarp();
        }
        const StreamParams &sp = *spp;
        const int rec_stream = KC == 1 ? si.stream : cfg0 + jc;
        int c4 = 0, s4 = 0;                                 // (C4, S4) of the cfg: recovery's rotation
        if constexpr (ROT) {
          const int4 r = __ldg(rot + rec_stream);
          c4 = r.z;
          s4 = r.w;
        }
        const int dir_at = KC == 1 ? unit : (cfg0 + jc) * per_group + local;
        // 1a. exact access-address hits of the unit, all lanes (lane = flag word = 32 groups): the only data-dependent search
        for (int t = lane; t < 2 * si.nch; t += 32)
          RS.xh[t][kExactCap] = (uint16_t)enumerate_exact_hits(reinterpret_cast<const uint32_t *>(S.pd), S.cand, S.flagw[t], t, sp, RS.xh[t]);
        __syncwarp();
        // 1b. chain pass: which hits does the reference count?  (lane = chunk; walks the chunk's two hit lists)
        int mine = 0;
        if (lane < si.nch) {
          struct Note {
            uint16_t *row;
            __device__ __forceinline__ void operator()(int i, int n0, bool rej) {
              if (i < kHitCap) row[i] = (uint16_t)((n0 + 124) | (rej ? 0x8000 : 0));
            }
          } note{RS.hit[lane]};
          const uint32_t *pdc = reinterpret_cast<const uint32_t *>(&S.pd[kGroupsPerChunk * lane]);
          const int c0 = RS.xh[2 * lane][kExactCap], c1 = RS.xh[2 * lane + 1][kExactCap];
          if (c0 > kExactCap || c1 > kExactCap)              // degenerate mask: too many matches to list, walk the candidates instead
            mine = chain_chunk(pdc, &S.cand[kGroupsPerChunk * lane], &S.flagw[2 * lane], sp, note);
          else
            mine = chain_chunk_lists(pdc, RS.xh[2 * lane], c0, RS.xh[2 * lane + 1], c1, sp, note);
        }
        BTLE_STAMP(7);
        // 2. the unit's block of the output: exclusive scan of the per-chunk counts, one atomic for the unit
        int incl = mine;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) { const int v = __shfl_up_sync(0xFFFFFFFFu, incl, d); if (lane >= d) incl += v; }
        const int total = __shfl_sync(0xFFFFFFFFu, incl, 31);
        if (lane <= kSpanChunks) RS.pre[lane] = (uint16_t)(incl - mine);   // lanes >= nch hold `total`
        unsigned my_base = 0;
        if (lane == 0) {
          if (total) my_base = atomicAdd(count, (unsigned)total);
          dir[dir_at] = make_uint2(my_base, (unsigned)total);
        }
        __syncwarp();
        BTLE_STAMP(8);
        // 3. decode pass: one lane per packet, all lanes on the same instruction stream.  The reservation's result is
        //    only needed when the records are stored, so the atomic's round trip to L2 overlaps the decode.
        for (int j0 = 0; j0 < total; j0 += 32) {
          const int j = j0 + lane;
          uint32_t words[11];
          int nbytes = 0, crc_bad = 0, n0 = 0, c = 0;
          bool rej = false, live = false;
          if (j < total) {
            // chunk of packet j: pre[c] <= j < pre[c + 1]
#pragma unroll
            for (int step = kSpanChunks / 2; step >= 1; step >>= 1)
              if ((int)RS.pre[c + step] <= j) c += step;
            const int i = j - (int)RS.pre[c];
            live = i < kHitCap;                               // hits behind the chunk's row are left to step 4
            if (live) {
              const int h = (int)RS.hit[c][i];
              rej = (h & 0x8000) != 0;
              n0 = (h & 0x7FFF) - 124;
              decode_packet(reinterpret_cast<const uint32_t *>(&S.pd[kGroupsPerChunk * c]), sp, M.crc4, n0, rej, words, nbytes, crc_bad);
            }
          }
          // 3b. BTLE_CFG_RECOVER (uniform per cfg): a counted packet whose CRC failed is demodulated again from the
          //     capture's IQ, symbol-spaced on four sample phases; the lanes that need it run it together
          const unsigned base = __shfl_sync(0xFFFFFFFFu, my_base, 0);
          bool stored = false;
          if (sp.recover) {
            if (live && crc_bad && !rej && base + (unsigned)j < cap)
              stored = store_recovered<ROT>(out + base + j, rec_stream, si.chunk0 + c, n0, sp, M.crc4, cap_base, n_int8, lead, c4, s4);
          }
          if (live && !stored && base + (unsigned)j < cap)
            store_record(out + base + j, rec_stream, si.chunk0 + c, n0, nbytes, crc_bad, rej, words, sp, cap_base, n_int8, lead);
        }
        // 4. only with report_rejected can a chunk have more hits than its row holds (degenerate masks, up to
        //    BTLE_MAX_RECS_PER_CHUNK): the chunk's lane runs the same chain again and decodes and stores hits kHitCap.. itself
        if (sp.report_rejected) {
          const unsigned base = __shfl_sync(0xFFFFFFFFu, my_base, 0);
          if (mine > kHitCap) {
            struct Late {
              const uint32_t *pd; const StreamParams &sp; const uint32_t *crc4;
              btle_pkt_rec *out; unsigned first, cap; int stream, chunk; const int8_t *iq; long long n_int8, lead; int c4, s4;
              __device__ __forceinline__ void operator()(int i, int n0, bool rej) {
                if (i < kHitCap || first + (unsigned)i >= cap) return;
                uint32_t words[11];
                int nbytes, crc_bad;
                decode_packet(pd, sp, crc4, n0, rej, words, nbytes, crc_bad);
                if (sp.recover && crc_bad && !rej && store_recovered<ROT>(out + first + i, stream, chunk, n0, sp, crc4, iq, n_int8, lead, c4, s4))
                  return;                                             // as step 3b
                store_record(out + first + i, stream, chunk, n0, nbytes, crc_bad, rej, words, sp, iq, n_int8, lead);
              }
            };
            const uint32_t *pdc = reinterpret_cast<const uint32_t *>(&S.pd[kGroupsPerChunk * lane]);
            Late late{pdc, sp, M.crc4, out, base + RS.pre[lane], cap, rec_stream, si.chunk0 + lane, cap_base, n_int8, lead, c4, s4};
            const int c0 = RS.xh[2 * lane][kExactCap], c1 = RS.xh[2 * lane + 1][kExactCap];
            if (c0 > kExactCap || c1 > kExactCap)
              chain_chunk(pdc, &S.cand[kGroupsPerChunk * lane], &S.flagw[2 * lane], sp, late);
            else
              chain_chunk_lists(pdc, RS.xh[2 * lane], c0, RS.xh[2 * lane + 1], c1, sp, late);
          }
        }
        BTLE_STAMP(9);
        __syncwarp();                                       // (KC > 1: the next cfg's run reuses RS and rsp)
      }
      // the slot is reused by unit k + kSlots of this CTA: refresh its parameters if the stream changes
      const int next = unit + kSlots * gridDim.x;
      if (next < total_units) {
        const int ns = unit_info(next, plan).stream;
        if constexpr (KC == 1) {
          if (ns != si.stream) load_params_warp(params + ns, S.sp, lane);
        } else {
          if (ns != si.stream) load_multi_warp(params, vmap, ns, S.sp, lane);
        }
      }
      __syncwarp();
      if (lane == 0) mbar_arrive(&M.empty[b]);            // release the slot to the producers
      BTLE_STAMP(5);
    }
    BTLE_WAIT_SUM(14, w_full.sum);
  }
}

// ---- leaf kernels (unit parity through the C-ABI; not performance paths) ------------------------
__global__ void dbits_kernel(const int8_t *iq, long long n_samples, uint8_t *d) {
  const long long n = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (n >= n_samples) return;
  const int i0 = iq[2 * n], q0 = iq[2 * n + 1], i1 = iq[2 * n + 2], q1 = iq[2 * n + 3];
  d[n] = (uint8_t)((i0 * q1 - i1 * q0) > 0);            // btle_rx.c:1533
}

// search_unique_bits (btle_rx.c:1510): one CTA; phase words and candidate words for the searched
// range, then lane 0 runs search_from() with R = 0.  ngroups*128 samples must be readable (+1).
__global__ void search_kernel(const int8_t *iq, int search_len, btle_stream_cfg cfg, int ngroups, uint32_t *pd,
                              uint32_t *cand, int *result) {
  __shared__ StreamParams sp;
  __shared__ uint32_t flagw[8];
  if (threadIdx.x == 0) make_params(cfg, c_whiten_words[cfg.channel], sp);
  if (threadIdx.x < 8) flagw[threadIdx.x] = 0u;
  for (int g = threadIdx.x; g < ngroups + 1; g += blockDim.x) {
    uint32_t acc[4] = {0u, 0u, 0u, 0u};
    if (g < ngroups) {
      const uint32_t *w = reinterpret_cast<const uint32_t *>(iq) + 64 * (long long)g;
      uint32_t carry = w[64];
      for (int c = 15; c >= 0; --c) {
        dbits8(w[4 * c], w[4 * c + 1], w[4 * c + 2], w[4 * c + 3], carry, acc);
        carry = w[4 * c];
      }
    }
    for (int ph = 0; ph < 4; ++ph) pd[4 * g + ph] = acc[ph];
  }
  __syncthreads();
  for (int g = threadIdx.x; g < ngroups; g += blockDim.x) {
    const uint32_t a = prefilter_any(&pd[4 * g], &pd[4 * (g + 1)], sp);
    cand[g] = a;
    if (a) atomicOr(&flagw[g >> 5], 1u << (g & 31));
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    int n0 = 0;
    const bool hit = search_from(pd, cand, flagw, 0, 4 * search_len - 124, sp, ngroups + 1, ngroups - 1, n0);
    *result = hit ? 2 * n0 : -1;                          // return value, btle_rx.c:1550/:1561
  }
}

__global__ void demod_byte_kernel(const int8_t *rxp, int num_byte, uint8_t *out) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= num_byte) return;
  uint32_t b = 0;
  for (int j = 0; j < 8; ++j) {                           // btle_rx.c:1496-1506
    const int8_t *p = rxp + 8 * (8 * k + j);
    b |= (uint32_t)(((int)p[0] * p[3] - (int)p[2] * p[1]) > 0) << j;
  }
  out[k] = (uint8_t)b;
}

__global__ void scramble_kernel(const uint8_t *in, int n, int channel, int off, uint8_t *out) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int t = off + i;
  out[i] = in[i] ^ (uint8_t)(c_whiten_words[channel][t >> 2] >> (8 * (t & 3)));   // btle_rx.c:1232-1237
}

// CRC-24 register after the bytes p[0..n), one table step per byte (btle_rx.c:1215-1218)
__device__ __forceinline__ uint32_t crc24_bytes(uint32_t crc, const uint8_t *p, int n) {
  for (int i = 0; i < n; ++i) crc = c_crc4[(crc ^ p[i]) & 0xFFu] ^ (crc >> 8);
  return crc;
}

// crc24_byte (btle_rx.c:1224): crc_update starts from the full 32-bit init_hex and masks to 24 bits only after each
// byte, so bits 24..31 of the init land in bits 16..23 on the first byte; with no byte the result is init & 0xFFFFFF
__global__ void crc24_kernel(const uint8_t *in, int n, uint32_t init, uint32_t *out) {
  if (n == 0) { *out = init & 0xFFFFFFu; return; }
  const uint32_t crc = (c_crc4[(init ^ in[0]) & 0xFFu] ^ (init >> 8)) & 0xFFFFFFu;
  *out = crc24_bytes(crc, in + 1, n - 1);
}

// stream_callback's sample reduction (btle_rx.c:307-308): int16 -> (x >> shift) & 0xFF
__global__ void iq16_to_iq8_kernel(const int16_t *__restrict__ in, long long n, int shift, int8_t *__restrict__ out) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
    out[i] = (int8_t)((in[i] >> shift) & 0xFF);
}

// ---- btlelib.py leaf kernels (python/btlelib.py) ------------------------------------------------
__global__ void gfsk_demod_i16_kernel(const int16_t *i, const int16_t *q, long long n, int8_t *bit, int32_t *sig) {
  const long long k = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (k + 1 >= n) return;
  // int32 products with numpy's wrap-around semantics (btlelib.py:396)
  const uint32_t s = (uint32_t)((int32_t)i[k] * (int32_t)q[k + 1]) - (uint32_t)((int32_t)i[k + 1] * (int32_t)q[k]);
  sig[k] = (int32_t)s;
  bit[k] = (int8_t)((int32_t)s > 0);
}

__global__ void search_seq_kernel(const int8_t *bit, long long n, const int8_t *seq, long long m, long long *first) {
  const long long s0 = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (s0 + m > n) return;
  for (long long j = 0; j < m; ++j)
    if (bit[s0 + j] != seq[j]) return;                    // btlelib.py:408
  atomicMin(reinterpret_cast<unsigned long long *>(first), (unsigned long long)s0);
}

// crc24_core, btlelib.py:191-219: 24-stage LFSR, feedback = stage 23 ^ input, taps into stages
// 0,1,3,4,6,9,10; the result is the register read from stage 23 down to 0.
__global__ void crc24_bits_kernel(const int8_t *in, long long n, const int8_t *init, int8_t *out) {
  uint32_t st = 0;                                         // bit k = stage k
  for (int k = 0; k < 24; ++k) st |= (uint32_t)(init[k] & 1) << k;
  for (long long t = 0; t < n; ++t) {
    const uint32_t fb = ((st >> 23) ^ (uint32_t)in[t]) & 1u;
    st = (st << 1) & 0xFFFFFFu;
    if (fb) st ^= 0x00065Bu;                               // stages 0,1,3,4,6,9,10
  }
  for (int k = 0; k < 24; ++k) out[k] = (int8_t)((st >> (23 - k)) & 1u);
}

// scramble_core, btlelib.py:226-263: same LFSR as scramble_table.h, applied bit by bit.
__global__ void scramble_bits_kernel(const int8_t *in, long long n, int channel, int8_t *out) {
  uint32_t reg = whiten_seed(channel);
  for (long long t = 0; t < n; ++t) out[t] = (int8_t)((whiten_step(reg) + (uint32_t)in[t]) & 1u);
}

// Transmit PHY, run by one CTA per packet: the GFSK modulator of the air bits sb[0..nbit) (LSB first), nsamp = nbit * SPS
// + 16 samples.  Each pass covers 8 samples per thread of the block, 8 consecutive ones per thread: frequency word per
// sample from the (at most 3 / 17) filter taps that see an impulse, block-wide inclusive scan for the phase, carried from
// pass to pass.  THREADS is the block size, or 0 to read it from blockDim.x.  (On an H100 80GB HBM3 at 700 W, a constant
// made ber_synth_kernel about 15 % faster than reading blockDim.x, and tx_modulate_kernel<8> about 10 % slower.)
// sink(m, ph) is called with the phase-table index of every sample m < n_out (words past the packet are 0).
//   SPS 4 (btle_tx.c:1022-1063): sample m takes the phase before word m, modulo 1024
//   SPS 8 (btlelib.py:146-189): sample m takes the phase including word m, modulo 2048
// Every thread of the block must call it; it ends with a block barrier, so the sink's shared-memory writes are visible.
template <int SPS, int THREADS, class Sink>
__device__ __forceinline__ void gfsk_block(const uint8_t *sb, int nbit, int n_out, Sink sink) {
  __shared__ int warp_tot[THREADS ? THREADS / 32 : 32];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const unsigned nthreads = THREADS ? THREADS : blockDim.x;
  const int nsamp = nbit * SPS + 16;
  auto pm1 = [&](int k) { return ((sb[k >> 3] >> (k & 7)) & 1) ? 1 : -1; };
  int run = 0;                                             // phase carried through the whole packet
  for (int base = 0; base < n_out; base += 8 * nthreads) {
    const int s0 = base + 8 * tid;
    int f[8];
#pragma unroll
    for (int u = 0; u < 8; ++u) {
      const int m = s0 + u;                                // frequency word whose running sum is the phase
      int acc = 0;
      if (SPS == 4) {
        // acc_m = sum_{j=3..11} g[15-j] * os[m+j], impulse of symbol k at os[15+4k] (btle_tx.c:1052-1056)
        if (m < nsamp - 1) {
#pragma unroll
          for (int j = 3; j <= 11; ++j) {
            const int idx = m + j - 15;
            if (idx >= 0 && (idx & 3) == 0 && (idx >> 2) < nbit) acc += c_gauss4[j - 3] * pm1(idx >> 2);
          }
        }
      } else {
        // y[m] = sum_j taps[j] * x[17 - j + m], x = 17 x (-1), then the NRZ waveform (btlelib.py:163-167)
        if (m < nsamp) {
          int y = 0;
#pragma unroll
          for (int j = 3; j <= 13; ++j) {                  // taps outside 3..13 are zero
            const int xi = 17 - j + m;
            int x = 0;
            if (xi < 17) x = -1; else if (xi - 17 < 8 * nbit) x = pm1((xi - 17) >> 3);
            y += c_gauss8[j] * x;
          }
          acc = y >> 1;                                    // btlelib.py:177
        }
      }
      f[u] = acc;
    }
    int loc = 0;
#pragma unroll
    for (int u = 0; u < 8; ++u) { loc += f[u]; f[u] = loc; }               // inclusive within the thread
    int incl = loc;                                        // inclusive scan of thread totals across the block
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
      const int v = __shfl_up_sync(0xFFFFFFFFu, incl, d);
      if (lane >= d) incl += v;
    }
    if (lane == 31) warp_tot[warp] = incl;
    __syncthreads();
    int woff = 0, tot = 0;
    for (int w = 0; w < (int)(nthreads >> 5); ++w) { if (w < warp) woff += warp_tot[w]; tot += warp_tot[w]; }
    const int excl = run + woff + incl - loc;              // sum of all frequency words before this thread's first
#pragma unroll
    for (int u = 0; u < 8; ++u) {
      const int m = s0 + u;
      if (m >= n_out) break;
      if (SPS == 4) sink(m, (excl + (u ? f[u - 1] : 0)) & 1023);   // sample[0] = table[0] (btle_tx.c:1046-1061)
      else sink(m, (excl + f[u]) & 2047);                          // cumsum includes the current word (btlelib.py:97)
    }
    run += tot;
    __syncthreads();
  }
}

// Air bytes of one packet into sb[0..n_sb): preamble (0x55 / 0xAA by the access address's first bit), the access address
// little-endian, then PDU + CRC-24 whitened for the channel, zeros behind.  crc_init is the reordered register
// (crc_init_reorder).  corrupt_bit >= 0 flips that bit of PDU + CRC after the CRC is computed, so the packet fails it.
__device__ __forceinline__ void build_air(const uint8_t *pdu, int pdu_len, uint32_t aa, uint32_t crc_init, int channel, int corrupt_bit,
                                          uint8_t *sb, int n_sb) {
  const uint32_t crc = crc24_bytes(crc_init, pdu, pdu_len);
  sb[0] = (aa & 1u) ? 0x55 : 0xAA;
  for (int b = 0; b < 4; ++b) sb[1 + b] = (uint8_t)(aa >> (8 * b));
  for (int b = 0; b < pdu_len + 3; ++b) {
    uint8_t v = b < pdu_len ? pdu[b] : (uint8_t)(crc >> (8 * (b - pdu_len)));
    if (corrupt_bit >= 0 && b == corrupt_bit >> 3) v ^= (uint8_t)(1u << (corrupt_bit & 7));
    sb[5 + b] = v ^ (uint8_t)(c_whiten_words[channel][b >> 2] >> (8 * (b & 3)));
  }
  for (int b = 5 + pdu_len + 3; b < n_sb; ++b) sb[b] = 0;
}

// ---- per-packet carrier-offset estimate (btle_b200_rec_offset_device; definition in include/btle_b200.h) -------------
// One warp per record.  Turn k (k = 0 .. kOffTurns-1) is arg(conj(x[n]) x[n+1]), n = n0 - 32 + k, read through the record's
// chunk window (iq_window); the reference turn is the same over the btle_tx waveform (gfsk_block<4>: phase before
// frequency word m, int8 table samples) of the preamble and access address alone, tx sample m = n - n0 +
// BTLE_RX_BER_AA_OFFSET.  The turns end 4 samples before the header: later ones see its first bit through the filter.
constexpr int kOffLead = 32, kOffTurns = 156;
__device__ __forceinline__ int tx4_freq(const uint8_t *sb, int nbit, int m) {   // frequency word m of gfsk_block<4>
  int acc = 0;
#pragma unroll
  for (int j = 3; j <= 11; ++j) {
    const int idx = m + j - 15;
    if (idx >= 0 && (idx & 3) == 0 && (idx >> 2) < nbit) acc += c_gauss4[j - 3] * (((sb[idx >> 5] >> ((idx >> 2) & 7)) & 1) ? 1 : -1);
  }
  return acc;
}
__global__ void rec_offset_kernel(const int8_t *__restrict__ iq, long long stride, long long n_int8, const btle_pkt_rec *__restrict__ recs,
                                  long long n, float *__restrict__ hz) {
  const long long r = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (r >= n) return;
  const int stream = recs[r].stream, chunk = recs[r].chunk, n0 = recs[r].n0;
  const uint32_t aa = recs[r].access_addr;
  const uint8_t sb[5] = {(uint8_t)((aa & 1u) ? 0x55 : 0xAA), (uint8_t)aa, (uint8_t)(aa >> 8), (uint8_t)(aa >> 16), (uint8_t)(aa >> 24)};
  const IqWindow w = iq_window(iq + (long long)stream * stride, n_int8, chunk);
  const int m_first = BTLE_RX_BER_AA_OFFSET - kOffLead;
  int ph = 0, m = 0;                                        // phase before frequency word m of the reference
  float sum = 0.0f;
  for (int k = lane; k < kOffTurns; k += 32) {
    for (; m < m_first + k; ++m) ph += tx4_freq(sb, 40, m);
    const int p1 = ph + tx4_freq(sb, 40, m);
    const int ri0 = c_cos1024[ph & 1023], rq0 = c_sin1024[ph & 1023], ri1 = c_cos1024[p1 & 1023], rq1 = c_sin1024[p1 & 1023];
    int i0, q0, i1, q1;
    iq_at(w, n0 - kOffLead + k, i0, q0);
    iq_at(w, n0 - kOffLead + k + 1, i1, q1);
    sum += atan2f((float)(i0 * q1 - q0 * i1), (float)(i0 * i1 + q0 * q1)) -
           atan2f((float)(ri0 * rq1 - rq0 * ri1), (float)(ri0 * ri1 + rq0 * rq1));
  }
#pragma unroll
  for (int d = 16; d >= 1; d >>= 1) sum += __shfl_xor_sync(0xFFFFFFFFu, sum, d);
  if (lane == 0) hz[r] = sum * (float)(4e6 / (6.283185307179586 * kOffTurns));
}

// The transmit PHY on a batch of air-byte rows: samples past a packet's own, up to the longest row's, are zero.
// A row's length is clamped to 0..max_bytes, so it never reads another row's bytes or past the batch.
template <int SPS>
__global__ void __launch_bounds__(512)
tx_modulate_kernel(const uint8_t *__restrict__ air, const int32_t *__restrict__ nbytes, int max_bytes,
                   int8_t *__restrict__ out_i, int8_t *__restrict__ out_q) {
  __shared__ uint8_t sb[128];
  const int pkt = blockIdx.x;
  const int nb = min(max(nbytes[pkt], 0), max_bytes);
  for (int i = threadIdx.x; i < 128; i += blockDim.x) sb[i] = (i < nb) ? air[(size_t)pkt * max_bytes + i] : 0;
  __syncthreads();
  const int nsamp = 8 * nb * SPS + 16, nsamp_max = 8 * max_bytes * SPS + 16;
  gfsk_block<SPS, 0>(sb, 8 * nb, nsamp_max, [&](int m, int ph) {
    const bool on = m < nsamp;
    if (SPS == 4) {
      out_i[((size_t)pkt * nsamp_max + m) * 2] = on ? c_cos1024[ph] : 0;
      out_i[((size_t)pkt * nsamp_max + m) * 2 + 1] = on ? c_sin1024[ph] : 0;
    } else {
      out_i[(size_t)pkt * nsamp_max + m] = on ? c_cos2048[ph] : 0;
      out_q[(size_t)pkt * nsamp_max + m] = on ? c_sin2048[ph] : 0;
    }
  });
}

// ---- capture synthesiser (test / benchmark input, SURVEY.md §8d C2-C5): noise floor + one burst per slot, all on
// the device.  Counter-based randomness (a 64-bit mix of seed, stream, position), so every byte of every capture is
// a pure function of (seed, stream, index) and a slot can be regenerated on its own.
__constant__ uint32_t c_noise_thr[13];     // P(round(N(-0.3, 0.8)) <= v) * 2^32 for v = -7 .. 5
__device__ __forceinline__ uint64_t mix64(uint64_t x) {          // splitmix64 finaliser
  x += 0x9E3779B97F4A7C15ull;
  x = (x ^ (x >> 30)) * 0xBF58476D1CE4E5B9ull;
  x = (x ^ (x >> 27)) * 0x94D049BB133111EBull;
  return x ^ (x >> 31);
}
__device__ __forceinline__ uint64_t draw(uint64_t seed, uint64_t stream, uint64_t a, uint64_t k) {
  return mix64(mix64(seed ^ (stream * 0xD1B54A32D192ED03ull)) ^ (a * 0x9E3779B97F4A7C15ull) ^ (k << 56));
}
__device__ __forceinline__ int noise_floor_value(uint32_t u) {
  int v = -7;
#pragma unroll
  for (int k = 0; k < 13; ++k) v += (u >= c_noise_thr[k]);
  return v;
}
// kind 0: integer noise floor of the reference capture (sigma 0.8 LSB, mean -0.3, clipped to [-7, 6]);
// kind 1: full-scale uniform int8 (a hot interferer: discriminator bits are 50/50); kind 2: zeros
__global__ void synth_noise_kernel(int8_t *__restrict__ iq, long long stride, long long n_int8, int n_streams, uint64_t seed, int kind) {
  const long long per = (n_int8 + 15) >> 4;                 // 16-byte pieces per capture
  const long long total = per * n_streams;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const long long s = i / per, p = i - s * per;
    uint32_t w[4] = {0u, 0u, 0u, 0u};
    if (kind == 0) {
#pragma unroll
      for (int q = 0; q < 8; ++q) {
        const uint64_t r = draw(seed, (uint64_t)s, (uint64_t)p * 8 + q, 1);
        const uint32_t b0 = (uint32_t)noise_floor_value((uint32_t)r) & 0xFFu, b1 = (uint32_t)noise_floor_value((uint32_t)(r >> 32)) & 0xFFu;
        w[q >> 1] |= (b0 | (b1 << 8)) << (16 * (q & 1));
      }
    } else if (kind == 1) {
      const uint64_t r0 = draw(seed, (uint64_t)s, (uint64_t)p * 2, 1), r1 = draw(seed, (uint64_t)s, (uint64_t)p * 2 + 1, 1);
      w[0] = (uint32_t)r0; w[1] = (uint32_t)(r0 >> 32); w[2] = (uint32_t)r1; w[3] = (uint32_t)(r1 >> 32);
    }
    int8_t *dst = iq + s * stride + 16 * p;
    if (16 * p + 16 <= n_int8 && ((reinterpret_cast<uintptr_t>(dst) & 15) == 0)) *reinterpret_cast<uint4 *>(dst) = make_uint4(w[0], w[1], w[2], w[3]);
    else
      for (int b = 0; b < 16; ++b)
        if (16 * p + b < n_int8) dst[b] = (int8_t)(w[b >> 2] >> (8 * (b & 3)));
  }
}

struct SynthSlot { long long start; int n_air, pdu_len, corrupt_bit, straddle; };
// Placement and length of the burst of (stream, slot): needs only hashes, so a slot can ask about its predecessor.
__device__ SynthSlot synth_slot_geometry(const btle_synth_cfg &sc, const btle_stream_cfg &cfg, int stream, long long slot, long long n_samples,
                                         bool look_back) {
  SynthSlot g;
  const bool adv = cfg.channel >= 37;
  const uint64_t r = draw(sc.seed, (uint64_t)stream, (uint64_t)slot, 2);
  g.pdu_len = adv ? 2 + 6 + (int)(r % 32) : 2 + (int)(r % 28);               // ADV_IND: AdvA + 0..31 B; LL data: 0..27 B
  g.n_air = 1 + 4 + g.pdu_len + 3;
  const int n_s = 32 * g.n_air + 16;
  g.corrupt_bit = -1;
  if (sc.corrupt_every > 0 && slot % sc.corrupt_every == sc.corrupt_every - 1)
    g.corrupt_bit = g.pdu_len > 2 ? 16 + (int)((r >> 16) % (uint64_t)(8 * g.pdu_len - 16)) : 8 * g.pdu_len + 3;
  const long long S = sc.slot_samples;
  long long lo = slot * S;
  if (look_back && slot > 0 && sc.straddle_every > 0) {                       // a straddling predecessor spills into this slot
    const SynthSlot pv = synth_slot_geometry(sc, cfg, stream, slot - 1, n_samples, false);
    if (pv.straddle && pv.start + 32 * pv.n_air + 16 + 32 > lo) lo = pv.start + 32 * pv.n_air + 16 + 32;
  }
  long long hi = (slot + 1) * S - n_s;                                        // last start that keeps the burst in its slot
  if (hi < lo) hi = lo;
  g.start = lo + (long long)((r >> 32) % (uint64_t)(hi - lo + 1));
  g.straddle = 0;
  if (sc.straddle_every > 0 && slot % sc.straddle_every == sc.straddle_every - 1) {
    const long long edge = (slot * S / kChunkSamples + 1) * (long long)kChunkSamples;   // next chunk boundary behind the slot start
    const long long first = max(slot * S, edge - n_s + 1);
    if (first < edge && edge <= (slot + 1) * S && edge + n_s < n_samples) {
      g.start = first + (long long)((r >> 40) % (uint64_t)(edge - first));      // the boundary falls strictly inside the burst
      g.straddle = 1;
    }
  }
  return g;
}

// One CTA per (stream, slot): PDU from hashes -> build_air -> the 4-sps transmit PHY (gfsk_block) -> scaled by
// amplitude/127 (floor) and added to the floor with saturation.
__global__ void __launch_bounds__(256)
synth_bursts_kernel(int8_t *__restrict__ iq, long long stride, long long n_int8, const btle_stream_cfg *__restrict__ cfgs,
                    const btle_synth_cfg sc, long long n_slots, btle_synth_truth *__restrict__ truth) {
  __shared__ uint8_t sb[64];
  __shared__ SynthSlot G;
  const long long gid = blockIdx.x;
  const int stream = (int)(gid / n_slots);
  const long long slot = gid - (long long)stream * n_slots;
  const btle_stream_cfg cfg = cfgs[stream];
  const long long n_samples = n_int8 / 2;
  if (threadIdx.x == 0) {
    G = synth_slot_geometry(sc, cfg, stream, slot, n_samples, true);
    const bool adv = cfg.channel >= 37;
    uint8_t pdu[48];
    const int plen = G.pdu_len - 2;
    if (adv) {
      pdu[0] = 0x40; pdu[1] = (uint8_t)plen;                                  // ADV_IND, TxAdd = 1
      const uint64_t adva = (uint64_t)slot | ((uint64_t)(stream & 0xFFFF) << 32);
      for (int b = 0; b < 6; ++b) pdu[2 + b] = (uint8_t)(adva >> (8 * b));
      for (int b = 6; b < plen; ++b) pdu[2 + b] = (uint8_t)(draw(sc.seed, (uint64_t)stream, (uint64_t)slot, 3 + (b >> 3)) >> (8 * (b & 7)));
    } else {
      const uint64_t r = draw(sc.seed, (uint64_t)stream, (uint64_t)slot, 2);
      pdu[0] = (uint8_t)((1 + ((r >> 8) & 1)) | ((slot & 1) << 2) | (((slot >> 1) & 1) << 3));   // LLID 1/2, NESN, SN
      pdu[1] = (uint8_t)plen;
      for (int b = 0; b < plen; ++b) pdu[2 + b] = (uint8_t)(draw(sc.seed, (uint64_t)stream, (uint64_t)slot, 3 + (b >> 3)) >> (8 * (b & 7)));
    }
    build_air(pdu, G.pdu_len, cfg.access_addr, crc_init_reorder(cfg.crc_init), cfg.channel, G.corrupt_bit, sb, 64);
    if (truth) {
      btle_synth_truth t;
      memset(&t, 0, sizeof t);
      t.start_sample = G.start; t.stream = stream; t.slot = (int32_t)slot;
      t.n_air_bytes = (uint8_t)G.n_air; t.corrupt = (uint8_t)(G.corrupt_bit >= 0); t.straddle = (uint8_t)G.straddle; t.pdu_len = (uint8_t)G.pdu_len;
      for (int b = 0; b < G.pdu_len; ++b) t.pdu[b] = pdu[b];
      truth[gid] = t;
    }
  }
  __syncthreads();
  // 256 threads x 8 samples >= 1520 samples: one pass.  Samples behind the capture's last whole sample are not written.
  int8_t *cap = iq + (long long)stream * stride + 2 * G.start;
  const int nbit = 8 * G.n_air;
  gfsk_block<4, 256>(sb, nbit, (int)min((long long)(4 * nbit + 16), n_samples - G.start), [&](int m, int ph) {
    auto addsat = [&](int8_t &s, int wave) {
      const int p = wave * sc.amplitude;
      const int scaled = p >= 0 ? p / 127 : -((-p + 126) / 127);              // floor division, like the numpy generator
      const int v = (int)s + scaled;
      s = (int8_t)(v > 127 ? 127 : (v < -128 ? -128 : v));
    };
    addsat(cap[2 * m], c_cos1024[ph]);
    addsat(cap[2 * m + 1], c_sin1024[ph]);
  });
}

// ---- 8 samples per symbol, streaming (SURVEY.md 8f-3): where does the access address occur, on which sample phase? ----
// Phase ph of an 8-Msps capture is the symbol-rate stream n = 8 s + ph; its bits are the Python model's
// gfsk_demodulation_fixed_point on samples 8 symbols apart (btlelib.py:395-400).  One CTA = 32 groups of 32 symbols
// (8192 samples, 32 KB of int16 IQ) + 8 samples of the next group:
//   load     the tile goes to shared memory with coalesced 16-byte loads (4 samples each), all of a thread's loads in
//            flight at once; a group's 256 sample words are stored 264 words apart, so that the compute phase — whose
//            warp reads 8 consecutive phases of 4 groups — touches 32 different banks
//   pack     thread (g, ph) packs the 32 bits of group g on phase ph into a word
//   match    and compares the 32 windows starting in its word against the access address (funnel shift with the next
//            group's word of the same phase)
constexpr int kSps8Groups = 32;
constexpr int kSps8Pitch = 264;                                             // words per group row in shared memory
constexpr int kSps8TileWords = (kSps8Groups + 1) * kSps8Pitch;
constexpr int kSps8Vec = (kSps8Groups + 1) * 64;                            // 16-byte vectors per tile (33 rows x 256 samples)
#ifndef BTLE_SPS8_BUFS
#define BTLE_SPS8_BUFS 1   // 1: one tile per CTA, 6 CTAs per SM hide each other's load phase;
#endif                     // 2: persistent CTAs, next tile in flight while the current one is packed (half the warps per SM)
constexpr int kSps8Bufs = BTLE_SPS8_BUFS;
constexpr size_t kSps8Smem = (kSps8Bufs * kSps8TileWords + (kSps8Groups + 1) * 8) * sizeof(uint32_t);   // tile buffer(s) + the bit words
__device__ __forceinline__ void cp_async16(void *smem_dst, const void *gsrc) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(smem_u32(smem_dst)), "l"(gsrc) : "memory");
}
// Tiles are copied global -> shared with cp.async (SASS LDGSTS).  The kernel body is written as a loop over tiles with
// kSps8Bufs buffers; the shipped configuration is one buffer and one tile per CTA (see BTLE_SPS8_BUFS).
__global__ void __launch_bounds__(256)
sps8_hits_kernel(const int16_t *__restrict__ iq, long long n_samples, long long n_tiles, uint32_t aa, long long *__restrict__ hits, unsigned cap,
                 unsigned *__restrict__ count) {
  extern __shared__ __align__(16) uint32_t sps8_smem[];
  // one word = (I, Q) of one sample.  (Buffer addresses are computed, not kept in an array: an indexed array of pointers
  // ends up in local memory and the tile accesses become generic loads instead of LDS.)
  auto tile_buf = [&](int b) -> uint32_t * { return sps8_smem + (kSps8Bufs > 1 ? b : 0) * kSps8TileWords; };
  uint32_t(*W)[8] = reinterpret_cast<uint32_t(*)[8]>(sps8_smem + kSps8Bufs * kSps8TileWords);
  const uint32_t *s32 = reinterpret_cast<const uint32_t *>(iq);
  const uint4 *s128 = reinterpret_cast<const uint4 *>(iq);                 // iq is 16-byte aligned
  // tile = 32 groups x 256 samples + the first 256 samples of the next group (only its first 8 are used, for bit 31 of the
  // last group; the full row keeps the copy regular)
  // a tile whose 33 staged rows and the one sample behind them lie inside the capture needs no range checks at all
  auto interior = [&](long long tile) { return (tile + 1) * (kSps8Groups * 256ll) + 256 + 8 <= n_samples; };
  auto issue = [&](uint32_t *T, long long tile) {
    const long long base = tile * (kSps8Groups * 256ll);
    if (interior(tile)) {
      const uint4 *src = s128 + base / 4 + threadIdx.x;
      uint32_t *dst = &T[(threadIdx.x >> 6) * kSps8Pitch + 4 * (threadIdx.x & 63)];
#pragma unroll
      for (int r = 0; r < 8; ++r) cp_async16(dst + r * 4 * kSps8Pitch, src + 256 * r);      // 256 vectors = 4 rows per step
      if (threadIdx.x < kSps8Vec - 2048) cp_async16(dst + 8 * 4 * kSps8Pitch, src + 2048);
    } else {
#pragma unroll 1
      for (int r = 0; r < 9; ++r) {
        const int k = threadIdx.x + 256 * r;
        if (k < kSps8Vec) {
          uint32_t *dst = &T[(k >> 6) * kSps8Pitch + 4 * (k & 63)];
          const long long n = base + 4ll * k;
          if (n + 4 <= n_samples) cp_async16(dst, s128 + base / 4 + k);
          else {                                                            // behind the capture / its last, partial vector
            uint32_t w[4] = {0u, 0u, 0u, 0u};
            for (int q = 0; q < 4; ++q) if (n + q < n_samples) w[q] = __ldg(s32 + n + q);
            *reinterpret_cast<uint4 *>(dst) = make_uint4(w[0], w[1], w[2], w[3]);
          }
        }
      }
    }
    asm volatile("cp.async.commit_group;" ::: "memory");
  };
  const int ph = threadIdx.x & 7, gl = threadIdx.x >> 3;
  int buf = 0;
  long long tile = blockIdx.x;
  if (tile < n_tiles) issue(tile_buf(0), tile);
  for (; tile < n_tiles; tile += gridDim.x, buf ^= 1) {
    const long long next = tile + gridDim.x;
    if (kSps8Bufs > 1 && next < n_tiles) {
      issue(tile_buf(buf ^ 1), next);
      asm volatile("cp.async.wait_group 1;" ::: "memory");                 // the current tile has landed, the next may still fly
    } else {
      asm volatile("cp.async.wait_group 0;" ::: "memory");
    }
    __syncthreads();
    const uint32_t *T = tile_buf(buf);
    const long long g0 = tile * kSps8Groups;
    auto bit = [](uint32_t cur, uint32_t nxt) -> uint32_t {
      const int i0 = (int16_t)(cur & 0xFFFF), q0 = (int16_t)(cur >> 16), i1 = (int16_t)(nxt & 0xFFFF), q1 = (int16_t)(nxt >> 16);
      // btlelib.py:396 computes i0*q1 - i1*q0 in int32; for int16 inputs the difference cannot wrap (|products| <= 2^30),
      // so its sign is the comparison of the two products
      return (uint32_t)(i0 * q1 > i1 * q0);
    };
    const bool inside = interior(tile);
    for (int gg = gl; gg <= kSps8Groups; gg += 32) {
      const long long n0 = (g0 + gg) * 256 + ph;
      const uint32_t *row = &T[gg * kSps8Pitch + ph];
      uint32_t w = 0, cur = row[0];
      if (gg < kSps8Groups) {
#pragma unroll
        for (int k = 0; k < 32; ++k) {
          const uint32_t nxt = (k < 31) ? row[8 * (k + 1)] : T[(gg + 1) * kSps8Pitch + ph];
          w |= bit(cur, nxt) << k;
          cur = nxt;
        }
      } else {
        // the look-ahead group's word (needed by windows that start in the tile's last group): 32 of its samples are in the
        // staged 33rd row, the last one belongs to the group behind it (L2: the next tile)
        const uint32_t behind = (n0 + 256 < n_samples) ? __ldg(s32 + n0 + 256) : 0u;
#pragma unroll
        for (int k = 0; k < 32; ++k) {
          const uint32_t nxt = (k < 31) ? row[8 * (k + 1)] : behind;
          w |= bit(cur, nxt) << k;
          cur = nxt;
        }
      }
      if (!inside) {                                                        // bit k needs samples n0 + 8k and n0 + 8(k+1) inside the capture
        const long long room = (n_samples - 1 - n0) / 8;
        if (room < 32) w = room <= 0 ? 0u : (w & ((1u << room) - 1u));
      }
      W[gg][ph] = w;
    }
    __syncthreads();
    const uint32_t lo = W[gl][ph], hi = W[gl + 1][ph];
    // all 32 window starts at once: bit i of m survives if the window starting at bit i agrees with the access address on 8
    // of its 32 bits (every 4th), then the few survivors are compared exactly
    uint32_t m = 0xFFFFFFFFu;
#pragma unroll
    for (int p = 0; p < 32; p += 4) {
      const uint32_t f = funnel_r(lo, hi, (uint32_t)p);                     // bit i = stream bit i + p
      m &= ((aa >> p) & 1u) ? f : ~f;
    }
    while (m) {
      const int i = __ffs((int)m) - 1;
      m &= m - 1;
      if (funnel_r(lo, hi, (uint32_t)i) == aa) {
        const long long n = (g0 + gl) * 256 + 8ll * i + ph;                // first sample of the access address
        if (n + 8ll * 32 < n_samples) {                                    // all 32 bits lie inside the capture
          const unsigned k = atomicAdd(count, 1u);
          if (k < cap) hits[k] = n;
        }
      }
    }
    __syncthreads();                                                        // W and the consumed buffer are free again
    if (kSps8Bufs == 1 && next < n_tiles) issue(tile_buf(0), next);
  }
}

// ---- connection discovery: empty-PDU candidates with no access address given (btle_b200_discover*) --------------------
// One CTA = kDiscGroups groups of window starts of one capture.  The rule (btle_core.cuh, empty_pdu_windows) reads the
// phase words of one group in front of a window's group and three behind it, so the CTA stages kDiscThreads + 1 groups:
//   load   cp.async of the groups' IQ (16-byte vectors, coalesced) into rows of kDiscPitch words: a lane's 16-byte reads
//          of its own row are conflict-free within each quarter warp; bytes outside the capture read as 0
//   pack   lane j turns group j into its four phase words (the dense receive loop, dbits_group_dense)
//   test   lane j < kDiscGroups tests the 32 window starts of its group on each phase against the rule at once (funnel
//          shifts of the neighbours' words); the rare survivor gets its access address, header and CRC-init (16 reverse
//          LFSR steps) and one atomic on the counter places its 32-byte record
// Like sps8_hits_kernel one tile per CTA: six CTAs per SM hide each other's load phase.
constexpr int kDiscThreads = 128;
constexpr int kDiscGroups = kDiscThreads - 4;                              // window-start groups per CTA
constexpr int kDiscRows = kDiscThreads + 1;                                // staged groups (the last one for its first sample only)
constexpr int kDiscPitch = 68;                                             // words per staged row (64 + 4 of padding)
constexpr size_t kDiscSmem = ((size_t)kDiscRows * kDiscPitch + 4 * kDiscThreads) * sizeof(uint32_t);
static_assert(sizeof(btle_conn_cand) == 32, "candidate record must be 32 bytes");
__global__ void __launch_bounds__(kDiscThreads, 6)
discover_kernel(const int8_t *__restrict__ iq, long long stride, long long n_int8, long long tiles_per_stream,
                const StreamParams *__restrict__ params, btle_conn_cand *__restrict__ out, unsigned cap, unsigned *__restrict__ count) {
  extern __shared__ __align__(16) uint32_t disc_smem[];
  uint4 *pdw = reinterpret_cast<uint4 *>(disc_smem + kDiscRows * kDiscPitch);   // phase words of staged group j
  const long long stream = blockIdx.x / tiles_per_stream, tile = blockIdx.x - stream * tiles_per_stream;
  const int8_t *cap_base = iq + stream * stride;
  const long long row0 = (tile * kDiscGroups - 1) * 256;                   // first byte of staged group 0
  const bool interior = row0 >= 0 && row0 + kDiscRows * 256ll <= n_int8;
  for (int k = threadIdx.x; k < kDiscThreads * 16 + 1; k += kDiscThreads) {   // 16 vectors per row, 1 of the last row
    uint32_t *dst = disc_smem + (k >> 4) * kDiscPitch + 4 * (k & 15);
    const long long b = row0 + 16ll * k;
    if (interior || (b >= 0 && b + 16 <= n_int8)) {
      cp_async16(dst, cap_base + b);
    } else {
      uint32_t v[4] = {0u, 0u, 0u, 0u};
      for (int q = 0; q < 16; ++q)
        if (b + q >= 0 && b + q < n_int8) v[q >> 2] |= (uint32_t)(uint8_t)cap_base[b + q] << (8 * (q & 3));
      *reinterpret_cast<uint4 *>(dst) = make_uint4(v[0], v[1], v[2], v[3]);
    }
  }
  asm volatile("cp.async.commit_group;\n\tcp.async.wait_group 0;" ::: "memory");
  __syncthreads();
  {
    const uint4 *row = reinterpret_cast<const uint4 *>(disc_smem + threadIdx.x * kDiscPitch);
    auto word = [&](int k) -> uint32_t {
      if (k == 64) return row[kDiscPitch / 4].x;                            // first sample of the next group
      const uint4 v = row[k >> 2];
      return (k & 3) == 0 ? v.x : (k & 3) == 1 ? v.y : (k & 3) == 2 ? v.z : v.w;
    };
    uint32_t acc[4] = {0u, 0u, 0u, 0u};
    dbits_group_dense(word, acc);
    pdw[threadIdx.x] = make_uint4(acc[0], acc[1], acc[2], acc[3]);
  }
  __syncthreads();
  const int j = threadIdx.x;
  const long long g = tile * kDiscGroups + j, n_samples = n_int8 / 2;
  if (j >= kDiscGroups || 128 * g > n_samples - 286) return;               // no window start of this group lies inside
  const bool edge = g == 0 || 128 * g + 127 > n_samples - 286;
  const uint32_t wh0 = __ldg(&params[stream].whiten[0]), wh1 = __ldg(&params[stream].whiten[1]);
  const uint4 p0 = pdw[j], p1 = pdw[j + 1], p2 = pdw[j + 2], p3 = pdw[j + 3], p4 = pdw[j + 4];
#pragma unroll
  for (int ph = 0; ph < 4; ++ph) {
    auto at = [&](const uint4 &p) { return ph == 0 ? p.x : ph == 1 ? p.y : ph == 2 ? p.z : p.w; };
    const uint32_t w[5] = {at(p0), at(p1), at(p2), at(p3), at(p4)};
    uint32_t m = empty_pdu_windows(w, wh0);
    if (edge) m &= empty_pdu_inside(g, ph, n_samples);
    while (m) {
      const int i = __ffs((int)m) - 1;
      m &= m - 1;
      uint32_t aa, header, crc_rx;
      empty_pdu_fields(w, i, wh0, wh1, aa, header, crc_rx);
      const uint32_t crc_init = crc_init_reorder(crc24_unwind(crc_rx, header, 16));
      const unsigned k = atomicAdd(count, 1u);
      if (k < cap) {
        const long long n0 = 128 * g + 4 * i + ph;
        uint4 *d = reinterpret_cast<uint4 *>(out + k);
        d[0] = make_uint4((uint32_t)n0, (uint32_t)(n0 >> 32), (uint32_t)stream, aa);
        d[1] = make_uint4(crc_init, (uint32_t)__ldg(&params[stream].channel) | (header << 8), 0u, 0u);
      }
    }
  }
}

// ---- BER flow of python/test_btle_ber.py on the device: packet source + channel + int16 truncation --------------------
// One CTA per packet: 37 random payload bytes behind the fixed header 42 25 (test_btle_ber.py:27,:49), build_air,
// the Python model's 8-sps modulator (gfsk_block<8>), add_freq_sampling_error (linear
// resampling at 1 + ppm/1e6 and the matching carrier rotation at 2450 MHz, btlelib.py:823-857), add_noise (AWGN,
// sigma = 127 / 10^(snr/20) / sqrt 2 per rail, :859-871), np.int16() truncation.  Counter-based randomness.
constexpr int kBerPduBytes = 39, kBerAirBytes = 1 + 4 + kBerPduBytes + 3, kBerSamples = 8 * 8 * kBerAirBytes + 16;   // 3024
__device__ __forceinline__ float2 gauss_pair(uint64_t r) {                 // Box-Muller on two 32-bit uniforms
  const float u1 = ((float)(uint32_t)r + 0.5f) * 2.3283064365386963e-10f;    // (0, 1)
  const float u2 = (float)(uint32_t)(r >> 32) * 2.3283064365386963e-10f;
  const float rad = sqrtf(-2.0f * __logf(u1));
  float sn, cs;
  sincospif(2.0f * u2, &sn, &cs);
  return make_float2(rad * cs, rad * sn);
}
__global__ void __launch_bounds__(384)
ber_synth_kernel(const btle_ber_cfg cfg, unsigned long long first_packet, int n_packets, int16_t *__restrict__ out_i, int16_t *__restrict__ out_q,
                 uint8_t *__restrict__ truth /*[n][40]*/) {
  __shared__ uint8_t sb[64];
  __shared__ float txi[kBerSamples + 8], txq[kBerSamples + 8];
  const int pkt = blockIdx.x, tid = threadIdx.x;
  if (pkt >= n_packets) return;
  const unsigned long long gp = first_packet + (unsigned long long)pkt;
  if (tid == 0) {
    uint8_t pdu[kBerPduBytes];
    pdu[0] = 0x42; pdu[1] = 0x25;
    for (int b = 2; b < kBerPduBytes; ++b) pdu[b] = (uint8_t)(draw(cfg.seed, gp, (uint64_t)(b >> 3), 9) >> (8 * (b & 7)));
    build_air(pdu, kBerPduBytes, cfg.access_addr, crc_init_reorder(cfg.crc_init), cfg.channel, -1, sb, 64);
    for (int b = 0; b < kBerPduBytes; ++b) truth[(size_t)pkt * 40 + b] = pdu[b];
  }
  __syncthreads();
  // 384 threads x 8 samples >= 3024 samples: one pass
  gfsk_block<8, 384>(sb, 8 * kBerAirBytes, kBerSamples, [&](int m, int ph) {
    txi[m] = (float)c_cos2048[ph];
    txq[m] = (float)c_sin2048[ph];
  });
  const double e = (double)cfg.ppm * 1e-6;
  const float sigma = 127.0f / exp10f(cfg.snr_db / 20.0f) * 0.70710678f;
  // carrier offset fo = e * 2450e6 Hz at the new sampling time (1/8 us) * (1 + e): cycles per sample
  const double cyc = e * 2450e6 * (0.125e-6 * (1.0 + e));
  for (int m = tid; m < kBerSamples; m += blockDim.x) {
    float vi = txi[m], vq = txq[m];
    if (cfg.ppm != 0.0f) {
      const double x = (double)m * (1.0 + e);                // np.interp(x, xp, i): linear, clamped to the last sample
      int k = (int)x;
      if (k >= kBerSamples - 1) { vi = txi[kBerSamples - 1]; vq = txq[kBerSamples - 1]; }
      else {
        const float fr = (float)(x - (double)k);
        vi = txi[k] + (txi[k + 1] - txi[k]) * fr;
        vq = txq[k] + (txq[k + 1] - txq[k]) * fr;
      }
      double turns = cyc * (double)m;
      turns -= floor(turns);
      float sn, cs;
      sincospif(2.0f * (float)turns, &sn, &cs);
      const float ri = vi * cs - vq * sn, rq = vi * sn + vq * cs;
      vi = ri; vq = rq;
    }
    const float2 g = gauss_pair(draw(cfg.seed, gp, (uint64_t)m, 10));
    out_i[(size_t)pkt * kBerSamples + m] = (int16_t)(vi + sigma * g.x);     // np.int16(): truncation toward zero
    out_q[(size_t)pkt * kBerSamples + m] = (int16_t)(vq + sigma * g.y);
  }
}

// test_btle_ber.py:62-72: bit errors are counted only in packets whose CRC failed; an empty rx_pdu_bit counts all 312 bits
__global__ void ber_score_kernel(const btle_model_rx_rec *__restrict__ rec, const uint8_t *__restrict__ truth, int n,
                                 unsigned long long *__restrict__ acc /*pkt_err, bit_err, aa_miss*/) {
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  unsigned err = 0, perr = 0, miss = 0;
  if (p < n) {
    const btle_model_rx_rec &r = rec[p];
    if (!r.crc_ok) {
      perr = 1;
      miss = r.found ? 0u : 1u;
      const int nb = r.n_pdu_bits;
      if (nb == 0) err = 8 * kBerPduBytes;
      else {
        const int common = min(nb, 8 * kBerPduBytes);
        for (int b = 0; b < (common + 7) / 8; ++b) {
          uint32_t d = (uint32_t)(r.pdu[b] ^ truth[(size_t)p * 40 + b]);
          const int rem = common - 8 * b;
          if (rem < 8) d &= (1u << rem) - 1u;
          err += __popc(d);
        }
      }
    }
  }
  // warp-level reduction, one atomic per warp and counter
  for (int d = 16; d; d >>= 1) { err += __shfl_down_sync(0xFFFFFFFFu, err, d); perr += __shfl_down_sync(0xFFFFFFFFu, perr, d); miss += __shfl_down_sync(0xFFFFFFFFu, miss, d); }
  if ((threadIdx.x & 31) == 0) {
    if (perr) atomicAdd(&acc[0], (unsigned long long)perr);
    if (err) atomicAdd(&acc[1], (unsigned long long)err);
    if (miss) atomicAdd(&acc[2], (unsigned long long)miss);
  }
}

// ---- error rates of the 4-Msps receive chain (btle_b200_rx_ber_*; the definition is in include/btle_b200.h) -----------
// One CTA per slot of the capture: the packet from hashes (build_air), the btle_tx PHY at 4 sps (gfsk_block<4>) scaled
// into shared memory, then every sample of the slot: resampling at (m - delta)(1 + e), the carrier rotation, AWGN, rintf
// and int8 saturation, stored straight into the capture.  Slots at or behind n_live (global index) and samples at or
// behind n_samples are not packets; slots from n_truth on (relative to the capture) write no truth row.
constexpr int kRxBerPduAdv = 39, kRxBerPduData = 29, kRxBerMaxL = 32 * (1 + 4 + kRxBerPduAdv + 3) + 16;   // 1520
__host__ __device__ __forceinline__ int rx_ber_pdu_bytes(int channel) { return channel >= 37 ? kRxBerPduAdv : kRxBerPduData; }
__host__ __device__ __forceinline__ int rx_ber_len(int channel) { return 32 * (1 + 4 + rx_ber_pdu_bytes(channel) + 3) + 16; }
__global__ void __launch_bounds__(256)
rx_ber_synth_kernel(const btle_rx_ber_cfg cfg, unsigned long long first, unsigned long long n_live, long long n_samples,
                    long long n_truth, int8_t *__restrict__ iq, btle_rx_ber_truth *__restrict__ truth) {
  __shared__ uint8_t sb[64];
  __shared__ float txi[kRxBerMaxL], txq[kRxBerMaxL];
  __shared__ int s_off, s_delta4;
  __shared__ unsigned s_clipped;
  const long long slot = blockIdx.x;
  const unsigned long long gk = first + (unsigned long long)slot;
  const int S = cfg.slot_samples, L = rx_ber_len(cfg.channel), tid = threadIdx.x;
  const bool live = gk < n_live;
  if (tid == 0) {
    s_clipped = 0;
    const uint64_t r = draw(cfg.seed, gk, 0, 12);
    s_off = (int)(r % (uint64_t)(S - L + 1));
    s_delta4 = (int)((r >> 32) & 3);
    if (live) {
      const int nb = rx_ber_pdu_bytes(cfg.channel);
      uint8_t pdu[kRxBerPduAdv];
      if (cfg.channel >= 37) { pdu[0] = 0x42; pdu[1] = 0x25; }          // the PDU of btle_b200_ber_run
      else { pdu[0] = 0x02; pdu[1] = kRxBerPduData - 2; }                 // LL data, LLID 2, length 27
      for (int b = 2; b < nb; ++b) pdu[b] = (uint8_t)(draw(cfg.seed, gk, (uint64_t)(b >> 3), 9) >> (8 * (b & 7)));
      build_air(pdu, nb, cfg.access_addr, crc_init_reorder(cfg.crc_init), cfg.channel, -1, sb, 64);
      if (slot < n_truth) {
        btle_rx_ber_truth t;
        memset(&t, 0, sizeof t);
        const double e = (double)cfg.ppm * 1e-6;
        t.aa_sample = slot * S + s_off + (long long)floor(BTLE_RX_BER_AA_OFFSET / (1.0 + e) + 0.25 * s_delta4 + 0.5);
        t.offset = s_off;
        t.n_bytes = (uint8_t)nb;
        t.delta4 = (uint8_t)s_delta4;
        for (int b = 0; b < nb; ++b) t.pdu[b] = pdu[b];
        truth[slot] = t;
      }
    }
  }
  __syncthreads();
  const float scale = (float)cfg.amplitude / 127.0f;
  if (live) {                                                  // 256 threads x 8 samples >= 1520 samples: one pass
    gfsk_block<4, 256>(sb, (L - 16) / 4, L, [&](int m, int ph) {
      txi[m] = (float)c_cos1024[ph] * scale;
      txq[m] = (float)c_sin1024[ph] * scale;
    });
  }
  const double e = (double)cfg.ppm * 1e-6, delta = 0.25 * s_delta4;
  // turns per sample: the ppm's carrier error at the new sampling time (1 + e) / 4 Msps, plus the extra offset
  const double rate = e * 2450e6 * (0.25e-6 * (1.0 + e)) + (double)cfg.cfo_hz / 4e6;
  const float sigma = (float)cfg.amplitude / exp10f(cfg.snr_db / 20.0f) * 0.70710678f;
  const int off = s_off;
  const long long s0 = slot * S;
  const int n_here = (int)min((long long)S, n_samples - s0);
  unsigned clipped = 0;
  for (int j = tid; j < n_here; j += blockDim.x) {
    float vi = 0.0f, vq = 0.0f;
    const int m = j - off;
    if (live && m >= 0 && m < L) {
      const double x = ((double)m - delta) * (1.0 + e);
      if (x <= 0.0) { vi = txi[0]; vq = txq[0]; }                   // np.interp: clamped at both ends
      else {
        const int k = (int)x;
        if (k >= L - 1) { vi = txi[L - 1]; vq = txq[L - 1]; }
        else {
          const float fr = (float)(x - (double)k);
          vi = txi[k] + (txi[k + 1] - txi[k]) * fr;
          vq = txq[k] + (txq[k + 1] - txq[k]) * fr;
        }
      }
      if (rate != 0.0) {
        double turns = rate * (double)m;
        turns -= floor(turns);
        float sn, cs;
        sincospif(2.0f * (float)turns, &sn, &cs);
        const float ri = vi * cs - vq * sn, rq = vi * sn + vq * cs;
        vi = ri; vq = rq;
      }
    }
    const float2 g = gauss_pair(draw(cfg.seed, gk, (uint64_t)j, 11));
    const float ri = rintf(vi + sigma * g.x), rq = rintf(vq + sigma * g.y);
    const int ii = (int)fminf(fmaxf(ri, -128.0f), 127.0f), qq = (int)fminf(fmaxf(rq, -128.0f), 127.0f);
    clipped += (ri < -128.0f || ri > 127.0f || rq < -128.0f || rq > 127.0f) ? 1u : 0u;
    reinterpret_cast<uint16_t *>(iq)[s0 + j] = (uint16_t)((uint32_t)(ii & 0xFF) | ((uint32_t)(qq & 0xFF) << 8));
  }
  if (live && slot < n_truth) {
    for (int d = 16; d; d >>= 1) clipped += __shfl_down_sync(0xFFFFFFFFu, clipped, d);
    if ((tid & 31) == 0 && clipped) atomicAdd(&s_clipped, clipped);
    __syncthreads();
    if (tid == 0) truth[slot].clipped = s_clipped;
  }
}

// One thread per packet: its record is found in the launch's records through the unit directory, whose walk is the
// reference order, (chunk, n0): an exclusive prefix of the directory counts in shared memory maps a position of that
// order to its unit, a binary search finds the first record of the lowest chunk that can hold a match, and the records
// from there on are read until the highest one.  The CTAs also share a pass over the stored records, which counts the
// records and the CRC-ok ones; matched ones are taken off, so extra_recs / extra_crc_ok add up without a per-record
// match table.  One atomic per warp and counter, as ber_score_kernel.
__global__ void __launch_bounds__(256)
rx_ber_score_kernel(const btle_rx_ber_truth *__restrict__ truth, int n, const btle_pkt_rec *__restrict__ recs, unsigned long long n_recs,
                    const uint2 *__restrict__ dir, int n_units, unsigned long long *__restrict__ acc /* btle_rx_ber_result */) {
  extern __shared__ unsigned rx_ber_pre[];                    // [n_units + 1]: records before unit u in the walk
  __shared__ unsigned warp_sum[8];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  {
    const int per = (n_units + 255) / 256, u0 = min(n_units, tid * per), u1 = min(n_units, u0 + per);
    unsigned s = 0;
    for (int u = u0; u < u1; ++u) s += __ldg(&dir[u].y);
    unsigned incl = s;
    for (int d = 1; d < 32; d <<= 1) {
      const unsigned v = __shfl_up_sync(0xFFFFFFFFu, incl, d);
      if (lane >= d) incl += v;
    }
    if (lane == 31) warp_sum[warp] = incl;
    __syncthreads();
    unsigned run = incl - s;
    for (int w = 0; w < warp; ++w) run += warp_sum[w];
    for (int u = u0; u < u1; ++u) { rx_ber_pre[u] = run; run += __ldg(&dir[u].y); }
    if (tid == 255) rx_ber_pre[n_units] = run;
    __syncthreads();
  }
  const unsigned total = rx_ber_pre[n_units];
  // position i of the walk -> index into recs (or ~0ull when that record was not stored)
  auto at = [&](unsigned i) -> unsigned long long {
    int lo = 0, hi = n_units - 1;                            // last unit with pre <= i
    while (lo < hi) {
      const int mid = (lo + hi + 1) >> 1;
      if (rx_ber_pre[mid] <= i) lo = mid; else hi = mid - 1;
    }
    const unsigned long long r = (unsigned long long)__ldg(&dir[lo].x) + (i - rx_ber_pre[lo]);
    return r < n_recs ? r : ~0ull;
  };
  unsigned long long c[10] = {0, 0, 0, 0, 0, 0, 0, 0, 0, 0};   // btle_rx_ber_result's counters, in its order
  long long matched = 0, matched_ok = 0;
  const int p = blockIdx.x * blockDim.x + tid;
  if (p < n) {
    const btle_rx_ber_truth &t = truth[p];
    const long long a = t.aa_sample;
    const int nb = t.n_bytes;
    const long long c_lo = (a - BTLE_RX_BER_MATCH) / kChunkSamples;                     // n0 <= 8191
    const long long c_hi = (a + BTLE_RX_BER_MATCH + 124) / kChunkSamples;               // n0 >= -124
    unsigned lo = 0, hi = total;                               // first position whose chunk >= c_lo
    while (lo < hi) {
      const unsigned mid = (lo + hi) >> 1;
      const unsigned long long r = at(mid);
      if (r != ~0ull && recs[r].chunk < c_lo) lo = mid + 1; else hi = mid;
    }
    const btle_pkt_rec *m = nullptr;
    for (unsigned i = lo; i < total; ++i) {
      const unsigned long long r = at(i);
      if (r == ~0ull) break;
      const btle_pkt_rec &x = recs[r];
      if (x.chunk > c_hi) break;
      const long long pos = (long long)x.chunk * kChunkSamples + x.n0;
      if (pos >= a - BTLE_RX_BER_MATCH && pos <= a + BTLE_RX_BER_MATCH) { m = &x; break; }
    }
    c[0] = 1;
    c[3] = 8ull * nb;
    c[9] = t.clipped;
    const bool rejected = m && (m->flags & BTLE_REC_REJECTED);
    const bool ok = m && !rejected && !m->crc_bad;
    int common = 0;
    if (m) {
      ++matched;
      common = min(rejected ? 2 : (int)m->n_bytes - 3, nb);
      if (common < 0) common = 0;
    }
    if (ok) {
      ++matched_ok;
      bool same = (int)m->n_bytes - 3 == nb;
      for (int b = 0; b < nb && same; ++b) same = m->bytes[b] == t.pdu[b];
      c[6] = same ? 0 : 1;
    } else {
      c[1] = 1;
      if (!m) { c[4] = 1; c[2] = 8ull * nb; }
      else {
        c[5] = rejected ? 1 : 0;
        unsigned err = 0;
        for (int b = 0; b < common; ++b) err += __popc((unsigned)(m->bytes[b] ^ t.pdu[b]));
        c[2] = err;
      }
    }
  }
  // every stored record once, over the CTAs: counted here, matched ones taken off above
  const unsigned long long stored = min((unsigned long long)total, n_recs);
  long long nrec = 0, nok = 0;
  for (unsigned long long r = (unsigned long long)blockIdx.x * blockDim.x + tid; r < stored; r += (unsigned long long)gridDim.x * blockDim.x) {
    ++nrec;
    if (!(recs[r].flags & BTLE_REC_REJECTED) && !recs[r].crc_bad) ++nok;
  }
  c[7] = (unsigned long long)(nrec - matched);                 // may be "negative" per thread; the sums are exact modulo 2^64
  c[8] = (unsigned long long)(nok - matched_ok);
#pragma unroll
  for (int k = 0; k < 10; ++k) {
    unsigned long long v = c[k];
    for (int d = 16; d; d >>= 1) v += __shfl_down_sync(0xFFFFFFFFu, v, d);
    if (lane == 0 && v) atomicAdd(&acc[k], v);
  }
}

// btlelib.btle_rx for a batch of packet windows: one warp per packet (see include/btle_b200.h).
constexpr int kModelMaxWords = 64;                        // <= 2048 symbols per window
// Sample a of packet p sits at g{i,q}[(base(p) + a) * elem_stride], base(p) = win_off ? win_off[p] : p * n_samples:
// a planar batch (elem_stride 1) or windows cut out of one interleaved int16 capture (gi = iq, gq = iq + 1, elem_stride 2).
__global__ void __launch_bounds__(128)
model_rx_batch_kernel(const int16_t *__restrict__ gi, const int16_t *__restrict__ gq, long long elem_stride,
                      const long long *__restrict__ win_off, int n_packets, int n_samples, int sps,
                      int adv, int channel, uint32_t aa, uint32_t crc_init, btle_model_rx_rec *__restrict__ out) {
  __shared__ uint32_t wh[26];                              // whitening stream, 800 bits (+pad)
  __shared__ uint32_t crc_tab[256];
  __shared__ uint32_t bw[4][kModelMaxWords + 2];           // demodulated bits of the current phase
  __shared__ uint32_t pw[4][20];                           // pdu words of the last phase that found the AA
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (int i = threadIdx.x; i < 256; i += blockDim.x) crc_tab[i] = c_crc4[i];
  if (threadIdx.x == 0) {                                  // scramble_core's LFSR (btlelib.py:226-263)
    uint32_t reg = whiten_seed(channel);
    for (int w = 0; w < 26; ++w) {
      uint32_t v = 0;
      for (int b = 0; b < 32; ++b) v |= whiten_step(reg) << b;
      wh[w] = v;
    }
  }
  __syncthreads();
  const int pkt = blockIdx.x * 4 + warp;
  if (pkt >= n_packets) return;
  const long long base = win_off ? win_off[pkt] : (long long)pkt * n_samples;
  const int16_t *pi = gi + base * elem_stride, *pq = gq + base * elem_stride;
  const long long es = elem_stride;
  const int num_bit = n_samples / sps - 1;                 // btlelib.py:444 (n_samples % sps == 0)
  const int nw = (num_bit + 31) >> 5;
  uint32_t *B = bw[warp], *P = pw[warp];
  auto sbits = [&](int p) {                                // 32 stream bits from position p (p >= 0)
    return funnel_r(B[p >> 5], B[(p >> 5) + 1], (uint32_t)(p & 31));
  };
  auto wbits = [&](int p) { return funnel_r(wh[p >> 5], wh[(p >> 5) + 1], (uint32_t)(p & 31)); };
  int r_start = -1, r_plen = 0, r_npdu = 0, r_ok = 0, r_found = 0, r_phase = sps - 1;
  for (int w = lane; w < 20; w += 32) P[w] = 0u;
  for (int ph = 0; ph < sps; ++ph) {
    // gfsk_demodulation_fixed_point on i[ph::sps], q[ph::sps] (btlelib.py:395-400,461)
    for (int j = 0; j < nw; ++j) {
      const int k = 32 * j + lane;
      bool bit = false;
      if (k < num_bit) {
        const long long a = (long long)(ph + sps * k) * es, b2 = (long long)(ph + sps * k + sps) * es;
        const uint32_t sd = (uint32_t)((int)pi[a] * (int)pq[b2]) - (uint32_t)((int)pi[b2] * (int)pq[a]);
        bit = (int32_t)sd > 0;
      }
      const uint32_t W = __ballot_sync(0xFFFFFFFFu, bit);
      if (lane == 0) B[j] = W;
    }
    if (lane == 0) { B[nw] = 0u; B[nw + 1] = 0u; }
    __syncwarp();
    // search_unique_bit_sequence: first index whose 32 bits equal the access address (btlelib.py:402-412)
    int start = -1;
    for (int j = 0; j < nw && start < 0; ++j) {
      const int s = 32 * j + lane;
      const bool ok = (s + 32 <= num_bit) && (sbits(s) == aa);
      const uint32_t m = __ballot_sync(0xFFFFFFFFu, ok);
      if (m) start = 32 * j + __ffs((int)m) - 1;
    }
    if (start >= 0) {
      r_found = 1 + ph;                                    // 1 + the last phase the access address was found on
      r_start = start;
      const int len_info = 8 + num_bit - start;            // 8 zero bits are prepended (btlelib.py:474)
      const uint32_t hdr = sbits(start + 32) ^ wbits(0);   // info[40:] is dewhitened (btlelib.py:265-268)
      const int plen = (int)((hdr >> 8) & (adv ? 0x3Fu : 0x1Fu));        // btlelib.py:477-483
      int crc_start = 40 + 16 + 8 * plen;
      if (crc_start + 24 > len_info) crc_start = len_info - 24;          // btlelib.py:488-490
      const int npdu = crc_start > 40 ? crc_start - 40 : 0;
      r_plen = plen;
      r_npdu = npdu;
      __syncwarp();
      if (lane < 20) {                                     // pdu_bit = info[40:crc_start]
        uint32_t w = 0u;
        const int rem = npdu - 32 * lane;
        if (rem > 0) {
          w = sbits(start + 32 + 32 * lane) ^ wbits(32 * lane);
          if (rem < 32) w &= (1u << rem) - 1u;
        }
        P[lane] = w;
      }
      __syncwarp();
      int ok = 0;
      if (lane == 0) {
        // crc24_core over pdu_bit (btlelib.py:191-219) == reflected CRC-24 on the LSB-first bit stream
        uint32_t crc = crc_init;
        const int nbytes = npdu >> 3;
        for (int b = 0; b < nbytes; ++b) crc = crc_tab[(crc ^ (P[b >> 2] >> (8 * (b & 3)))) & 0xFFu] ^ (crc >> 8);
        for (int b = 8 * nbytes; b < npdu; ++b) {
          const uint32_t fb = (crc ^ (P[b >> 5] >> (b & 31))) & 1u;
          crc = (crc >> 1) ^ (fb ? 0xDA6000u : 0u);
        }
        uint32_t rx = 0;
        if (crc_start >= 40) {
          rx = (sbits(start + crc_start - 8) ^ wbits(crc_start - 40)) & 0xFFFFFFu;
        } else {                                           // CRC window reaches back into the AA / zero bits
          for (int t = 0; t < 24; ++t) {
            const int idx = crc_start + t;
            uint32_t bit = 0;
            if (idx >= 8) bit = (B[(start + idx - 8) >> 5] >> ((start + idx - 8) & 31)) & 1u;
            if (idx >= 40) bit ^= (wh[(idx - 40) >> 5] >> ((idx - 40) & 31)) & 1u;
            rx |= bit << t;
          }
        }
        ok = (crc == rx);
      }
      ok = __shfl_sync(0xFFFFFFFFu, ok, 0);
      r_ok = ok;
      if (ok) { r_phase = ph; break; }                     // btlelib.py:517
    }
    __syncwarp();
  }
  btle_model_rx_rec *o = out + pkt;
  if (lane == 0) {
    o->start = r_start; o->n_pdu_bits = (uint16_t)r_npdu; o->crc_ok = (uint8_t)r_ok; o->phase = (uint8_t)r_phase;
    o->payload_len = (uint8_t)r_plen; o->found = (uint8_t)r_found;
  }
  __syncwarp();
  for (int b = lane; b < 70; b += 32) o->pdu[b] = (uint8_t)(P[b >> 2] >> (8 * (b & 3)));
}

}  // namespace

// ================================================================================================
// C-ABI
// ================================================================================================
constexpr unsigned kCountRing = 64;  // context-owned allocation counters (launch_rx)
constexpr int kSlotUsers = 4;        // streams whose last launch is tracked per cfg slot (more share one entry, see note_use)

// `n` elements of T in memory the buffer owns: device memory, or page-locked host memory (kHost).  It is released
// through cudaFree / cudaFreeHost, which wait for work still using it, so a buffer may be regrown or dropped while a
// launch that reads it is held on another stream.  The owner selects the context's device before that.
template <class T, bool kHost = false>
struct Buf {
  T *p = nullptr;
  size_t n = 0;
  Buf() = default;
  Buf(const Buf &) = delete;
  Buf &operator=(const Buf &) = delete;
  ~Buf() { release(); }
  operator T *() const { return p; }
  void release() {
    if (p) { if (kHost) cudaFreeHost(p); else cudaFree(p); }
    p = nullptr;
    n = 0;
  }
  int alloc(btle_b200_ctx *ctx, size_t count);             // exactly `count` elements; the old ones are dropped
  int reserve(btle_b200_ctx *ctx, size_t count) {          // at least `count`, with room to grow
    return p && n >= count ? BTLE_OK : alloc(ctx, count + count / 8 + 4096 / sizeof(T));
  }
};
template <class T> using HostBuf = Buf<T, true>;

struct StreamUse {                   // the last launch a stream enqueued: CUDA's id of the stream + an event behind it
  unsigned long long stream = 0;
  cudaEvent_t ev = nullptr;
  unsigned long long stamp = 0;      // 0: no launch recorded
};
struct CfgSlot {                     // one uploaded btle_stream_cfg array + the per-stream parameters derived from it
  Buf<btle_stream_cfg> d;            // (small LRU cache, see upload_cfgs)
  Buf<StreamParams> d_params;
  HostBuf<btle_stream_cfg> h; HostBuf<StreamParams> h_params;   // page-locked sources of the upload
  size_t n = 0;                      // entries of the cached array (0: empty)
  // btle_b200_rx_multi: the cfgs' capture indices are part of the key, and the capture groups derived from them
  // ({capture, first cfg, number of cfgs} per capture read) are uploaded with the parameters
  bool multi = false;
  std::vector<int32_t> cfg_capture;
  Buf<int4> d_vmap;
  HostBuf<int4> h_vmap;
  size_t n_vmap = 0;
  // the *_offset entry points: {C, S, C4, S4} per cfg (make_rot), part of the key; empty: the launch is not rotated
  std::vector<int4> rot;
  Buf<int4> d_rot;
  HostBuf<int4> h_rot;
  unsigned long long up_stream = 0;  // stream the upload was enqueued on
  cudaEvent_t uploaded = nullptr;    // recorded behind the upload's two copies
  StreamUse use[kSlotUsers];         // last launch of each stream that read this upload
  unsigned long long stamp = 0;
};
struct MapSlot {                     // encoded TMA tensor maps of one (pointer, shape) combination
  const void *ptr = nullptr; size_t n_streams = 0, stride = 0, n_int8 = 0;
  CUtensorMap map32, map12;
  unsigned long long stamp = 0;
};
struct btle_b200_ctx {
  int device = 0;
  cudaStream_t stream = nullptr;
  std::string err;
  int last_launches = 0;
  int num_sms = 0;                  // cudaDevAttrMultiProcessorCount, read at creation
  void *encode_tiled = nullptr;     // cuTensorMapEncodeTiled, fetched through the runtime
  unsigned long long tick = 0;
  CfgSlot cfg_slot[4];
  MapSlot map_slot[4];
  // scratch owned by the context (host-buffer entry points)
  Buf<int8_t> d_iq;
  Buf<btle_pkt_rec> d_out;
  Buf<btle_unit_dir> d_dir;
  Buf<float> d_hz;                      // btle_b200_rec_offset's estimates
  Buf<unsigned> d_count;
  Buf<unsigned> d_count_ring;       // kCountRing allocation counters for launches that do not hand in their own (no memset node)
  unsigned ring_pos = 0;
  StreamUse ring_last[kCountRing / 2];   // [ring_pos % (kCountRing/2)]: the ring launch that next launch depends on (launch_rx)
  HostBuf<unsigned> h_count;
  HostBuf<btle_pkt_rec> h_recs;     // staging for records
  HostBuf<btle_unit_dir> h_dir;     // staging for the unit directory
  HostBuf<int8_t> h_stage[2];       // staging for pageable callers
  cudaEvent_t stage_free[2] = {nullptr, nullptr};
  Buf<uint8_t> d_leaf;              // scratch of the leaf entry points (leaf_layout)
  Buf<btle_conn_cand> d_cand;       // device candidates of btle_b200_discover
};

template <class T, bool kHost>
int Buf<T, kHost>::alloc(btle_b200_ctx *ctx, size_t count) {
  release();
  void *q = nullptr;
  const cudaError_t e = kHost ? cudaHostAlloc(&q, count * sizeof(T), cudaHostAllocDefault) : cudaMalloc(&q, count * sizeof(T));
  if (e != cudaSuccess) {
    cudaGetLastError();
    ctx->err = kHost ? "cudaHostAlloc failed" : "cudaMalloc failed";
    return BTLE_ENOMEM;
  }
  p = static_cast<T *>(q);
  n = count;
  return BTLE_OK;
}

namespace {

#define BTLE_CUDA(ctx, call)                                                              \
  do {                                                                                    \
    cudaError_t e_ = (call);                                                              \
    if (e_ != cudaSuccess) {                                                              \
      (ctx)->err = std::string(#call) + ": " + cudaGetErrorString(e_);                    \
      return BTLE_ECUDA;                                                                  \
    }                                                                                     \
  } while (0)

// Lays the leaf entry points' scratch out in ctx->d_leaf: piece(p, n) stands for n elements of T, and each piece starts
// on a 256-byte boundary.  leaf_layout(ctx, piece(a, na), piece(b, nb), ...) reserves the whole and sets a, b, ...
template <class T> struct Piece { T *&p; size_t n; };
template <class T> Piece<T> piece(T *&p, size_t n) { return {p, n}; }
constexpr size_t piece_bytes(size_t bytes) { return (bytes + 255) & ~size_t(255); }
template <class... T>
int leaf_layout(btle_b200_ctx *ctx, Piece<T>... pieces) {
  const int rc = ctx->d_leaf.reserve(ctx, (piece_bytes(pieces.n * sizeof(T)) + ...));
  if (rc) return rc;
  uint8_t *at = ctx->d_leaf;
  ((pieces.p = reinterpret_cast<T *>(at), at += piece_bytes(pieces.n * sizeof(T))), ...);
  return BTLE_OK;
}

// The end of a leaf entry point: its kernel's launch checked, `bytes` of the kernel's output copied to `dst`, waited for.
int leaf_result(btle_b200_ctx *ctx, void *dst, const void *src, size_t bytes) {
  BTLE_CUDA(ctx, cudaGetLastError());
  BTLE_CUDA(ctx, cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDeviceToHost, ctx->stream));
  BTLE_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  return BTLE_OK;
}

int validate_cfgs(btle_b200_ctx *ctx, const btle_stream_cfg *cfgs, size_t n) {
  for (size_t i = 0; i < n; ++i)
    if (cfgs[i].channel < 0 || cfgs[i].channel > 39) {   // same range check as btle_rx.c:1432-1435
      ctx->err = "channel number must be within 0~39";
      return BTLE_EINVAL;
    }
  return BTLE_OK;
}

// CUDA's id of a stream: unique for the life of the process (a handle can be re-used by a stream created later).
int stream_id(btle_b200_ctx *ctx, cudaStream_t st, unsigned long long *sid) {
  BTLE_CUDA(ctx, cudaStreamGetId(st, sid));
  return BTLE_OK;
}

// The cfg array of a launch must live on the device while the kernel runs.  Uploaded arrays are kept in a small LRU
// cache keyed by content, shared by launches on any stream.  Two orders keep it right without host or device-wide
// synchronisation:
//   - a launch that finds its array in the cache waits for the upload when the upload went to another stream and this
//     stream has not launched with it since (in steady state the event has long completed, and the wait is made once);
//   - the upload that evicts a slot waits for the slot's previous upload and for the last launch of EVERY stream that
//     read it (note_use), so a launch still held on one stream keeps its parameters.
// A launch never waits for another stream's kernel: two pipes that alternate over the same arrays still overlap.
// The copies come from page-locked staging, so enqueueing them never blocks the host behind a busy stream; the host
// waits only when it must rewrite a staging buffer whose previous copy has not run yet.
// cfg_capture (btle_b200_rx_multi, else nullptr): cfg i decodes capture cfg_capture[i]; already validated.
// rot (the *_offset entry points, else nullptr): n rotations, uploaded with the parameters and part of the key.
int upload_cfgs(btle_b200_ctx *ctx, const btle_stream_cfg *cfgs, size_t n, cudaStream_t st, unsigned long long sid, CfgSlot **slot_out,
                const int32_t *cfg_capture = nullptr, const int4 *rot = nullptr) {
  CfgSlot *pick = nullptr;
  for (CfgSlot &c : ctx->cfg_slot)
    if (c.n == n && c.multi == (cfg_capture != nullptr) && !memcmp(c.h, cfgs, n * sizeof(btle_stream_cfg)) &&
        (!cfg_capture || !memcmp(c.cfg_capture.data(), cfg_capture, n * sizeof(int32_t))) &&
        c.rot.empty() == (rot == nullptr) && (!rot || !memcmp(c.rot.data(), rot, n * sizeof(int4)))) { pick = &c; break; }
  if (pick) {
    bool seen = pick->up_stream == sid;
    for (const StreamUse &u : pick->use) seen |= u.stamp && u.stream == sid;
    if (!seen) BTLE_CUDA(ctx, cudaStreamWaitEvent(st, pick->uploaded, 0));
  } else {
    pick = &ctx->cfg_slot[0];
    for (CfgSlot &c : ctx->cfg_slot) if (c.stamp < pick->stamp) pick = &c;
    if (!pick->uploaded) BTLE_CUDA(ctx, cudaEventCreateWithFlags(&pick->uploaded, cudaEventDisableTiming));
    if (pick->n) {
      if (pick->up_stream != sid) BTLE_CUDA(ctx, cudaStreamWaitEvent(st, pick->uploaded, 0));
      for (const StreamUse &u : pick->use)
        if (u.stamp && u.stream != sid) BTLE_CUDA(ctx, cudaStreamWaitEvent(st, u.ev, 0));
    }
    // Staging that is kept still feeds the previous upload's copies; arrays that grow are freed by cudaFree /
    // cudaFreeHost, which wait for the work that still uses them.
    if (pick->n && pick->h.n >= n && pick->h_params.n >= n) BTLE_CUDA(ctx, cudaEventSynchronize(pick->uploaded));
    pick->n = 0;
    if (pick->d.reserve(ctx, n) || pick->d_params.reserve(ctx, n) || pick->h.reserve(ctx, n) || pick->h_params.reserve(ctx, n))
      return BTLE_ENOMEM;
    // (h_vmap grows in step with h: when it is kept, so is h, and the wait above covered its previous copy)
    if (cfg_capture && (pick->d_vmap.reserve(ctx, n) || pick->h_vmap.reserve(ctx, n))) return BTLE_ENOMEM;
    if (rot && (pick->d_rot.reserve(ctx, n) || pick->h_rot.reserve(ctx, n))) return BTLE_ENOMEM;
    for (StreamUse &u : pick->use) u.stamp = 0;              // ordered before the new copies by the waits above
    memcpy(pick->h, cfgs, n * sizeof(btle_stream_cfg));
    for (size_t i = 0; i < n; ++i) {                         // make_params(): btle_params.h, the same code the CPU emulator runs
      uint8_t row[48];
      make_whiten_row(cfgs[i].channel, row);
      uint32_t ww[12];
      memcpy(ww, row, 48);
      make_params(cfgs[i], ww, pick->h_params[i]);
    }
    BTLE_CUDA(ctx, cudaMemcpyAsync(pick->d, pick->h, n * sizeof(btle_stream_cfg), cudaMemcpyHostToDevice, st));
    BTLE_CUDA(ctx, cudaMemcpyAsync(pick->d_params, pick->h_params, n * sizeof(StreamParams), cudaMemcpyHostToDevice, st));
    pick->multi = cfg_capture != nullptr;
    pick->n_vmap = 0;
    if (cfg_capture) {
      pick->cfg_capture.assign(cfg_capture, cfg_capture + n);
      for (size_t i = 0; i < n; ++i) {
        if (!i || cfg_capture[i] != cfg_capture[i - 1]) pick->h_vmap[pick->n_vmap++] = make_int4(cfg_capture[i], (int)i, 0, 0);
        ++pick->h_vmap[pick->n_vmap - 1].z;
      }
      BTLE_CUDA(ctx, cudaMemcpyAsync(pick->d_vmap, pick->h_vmap, pick->n_vmap * sizeof(int4), cudaMemcpyHostToDevice, st));
    }
    pick->rot.assign(rot ? rot : nullptr, rot ? rot + n : nullptr);
    if (rot) {
      memcpy(pick->h_rot, rot, n * sizeof(int4));
      BTLE_CUDA(ctx, cudaMemcpyAsync(pick->d_rot, pick->h_rot, n * sizeof(int4), cudaMemcpyHostToDevice, st));
    }
    BTLE_CUDA(ctx, cudaEventRecord(pick->uploaded, st));
    pick->up_stream = sid;
    pick->n = n;
  }
  pick->stamp = ++ctx->tick;
  *slot_out = pick;
  return BTLE_OK;
}

// After a launch on `st` that read `slot`: the event of st's entry now stands behind it.  With more than kSlotUsers
// streams on one slot, the least recent entry is taken over, and st first waits for the launch it stood for, so the
// entry still covers both (that orders st's LATER work behind the other stream; the launch just made runs freely).
int note_use(btle_b200_ctx *ctx, CfgSlot *slot, cudaStream_t st, unsigned long long sid) {
  StreamUse *u = nullptr;
  for (StreamUse &x : slot->use) if (x.stamp && x.stream == sid) { u = &x; break; }
  if (!u) {
    u = &slot->use[0];
    for (StreamUse &x : slot->use) if (x.stamp < u->stamp) u = &x;
    if (!u->ev) BTLE_CUDA(ctx, cudaEventCreateWithFlags(&u->ev, cudaEventDisableTiming));
    if (u->stamp) BTLE_CUDA(ctx, cudaStreamWaitEvent(st, u->ev, 0));
  }
  BTLE_CUDA(ctx, cudaEventRecord(u->ev, st));
  u->stream = sid;
  u->stamp = ++ctx->tick;
  return BTLE_OK;
}

// IQ as a 4-D byte tensor {128 B, 256-byte runs, 2 halves, streams}; a box is `rows` consecutive runs, both
// halves, so each lane's 256-byte run lands as two conflict-free 128-byte rows (row r of half h at h * rows + r).
// Encoded maps are cached per (pointer, shape): a streaming caller alternates between a few buffers.
int get_maps(btle_b200_ctx *ctx, const int8_t *d_iq, size_t n_streams, size_t stride, size_t n_int8, const MapSlot **out) {
  MapSlot *pick = nullptr;
  for (MapSlot &m : ctx->map_slot)
    if (m.stamp && m.ptr == d_iq && m.n_streams == n_streams && m.stride == stride && m.n_int8 == n_int8) { pick = &m; break; }
  if (!pick) {
    pick = &ctx->map_slot[0];
    for (MapSlot &m : ctx->map_slot) if (m.stamp < pick->stamp) pick = &m;
    typedef CUresult (*encode_fn)(CUtensorMap *, CUtensorMapDataType, cuuint32_t, void *, const cuuint64_t *,
                                  const cuuint64_t *, const cuuint32_t *, const cuuint32_t *, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
    encode_fn enc = reinterpret_cast<encode_fn>(ctx->encode_tiled);
    const cuuint64_t runs = (cuuint64_t)(n_int8 / 256);
    const cuuint64_t dims[4] = {128, runs, 2, (cuuint64_t)n_streams};
    const cuuint64_t strides[3] = {256, 128, (cuuint64_t)(n_streams > 1 ? stride : ((n_int8 + 255) & ~size_t(255)))};
    const cuuint32_t estr[4] = {1, 1, 1, 1};
    for (int which = 0; which < 2; ++which) {
      const cuuint32_t box[4] = {128, (cuuint32_t)(which ? kHaloRows : 32), 2, 1};
      const CUresult r = enc(which ? &pick->map12 : &pick->map32, CU_TENSOR_MAP_DATA_TYPE_UINT8, 4, const_cast<int8_t *>(d_iq), dims,
                             strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                             CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
      if (r != CUDA_SUCCESS) { pick->stamp = 0; ctx->err = "cuTensorMapEncodeTiled failed (" + std::to_string((int)r) + ")"; return BTLE_ECUDA; }
    }
    pick->ptr = d_iq; pick->n_streams = n_streams; pick->stride = stride; pick->n_int8 = n_int8;
  }
  pick->stamp = ++ctx->tick;
  *out = pick;
  return BTLE_OK;
}

Plan plan_for(const btle_b200_ctx *ctx, size_t n_streams, size_t n_int8) {
  return make_plan((long long)n_streams, (long long)(n_int8 / kChunkInt8), ctx->num_sms * kCtasPerSm);
}

// Several cfgs per capture (btle_b200_rx_multi): cfg i decodes capture cfg_capture[i] (non-decreasing, in range, at most
// kMaxCfgsPerCapture per capture; else BTLE_EINVAL).  *groups = number of distinct captures named.
int check_cfg_capture(btle_b200_ctx *ctx, size_t n_captures, const int32_t *cfg_capture, size_t n_cfgs, size_t *groups) {
  *groups = 0;
  size_t run = 0;
  for (size_t i = 0; i < n_cfgs; ++i) {
    const int32_t c = cfg_capture[i];
    if (c < 0 || (size_t)c >= n_captures) { ctx->err = "rx_multi: cfg_capture out of range"; return BTLE_EINVAL; }
    if (i && c < cfg_capture[i - 1]) { ctx->err = "rx_multi: cfg_capture must be non-decreasing"; return BTLE_EINVAL; }
    run = (i && c == cfg_capture[i - 1]) ? run + 1 : 1;
    if (run == 1) ++*groups;
    if (run > (size_t)kMaxCfgsPerCapture) { ctx->err = "rx_multi: more than BTLE_MAX_CFGS_PER_CAPTURE cfgs on one capture"; return BTLE_EINVAL; }
  }
  return BTLE_OK;
}
// Directory entries of a launch of n_cfgs cfgs over the `groups` captures they name: the plan's units over those
// captures, or with several cfgs on a capture every capture's (equal) share of them once per cfg
size_t rx_units(const btle_b200_ctx *ctx, size_t groups, size_t n_cfgs, size_t n_int8) {
  if (!groups || n_int8 < (size_t)kChunkInt8) return 0;
  const size_t total = (size_t)plan_for(ctx, groups, n_int8).total_units;
  return n_cfgs == groups ? total : n_cfgs * (total / groups);
}

// {C, S, C4, S4} of a carrier offset (include/btle_b200.h): round(2^14 (cos, sin)) of phi and of 4 phi, phi = 2 pi hz / 4 MHz
int4 make_rot(float hz) {
  const double ph = 6.283185307179586476925286766559 * (double)hz / 4e6;
  return make_int4((int)lrint(16384.0 * cos(ph)), (int)lrint(16384.0 * sin(ph)), (int)lrint(16384.0 * cos(4.0 * ph)),
                   (int)lrint(16384.0 * sin(4.0 * ph)));
}
// rotations of n cfgs from one offset per capture (cfg i reads capture cap_of[i], or i when cap_of is nullptr)
int make_rots(btle_b200_ctx *ctx, const float *offset_hz, size_t n_captures, const int32_t *cap_of, size_t n, std::vector<int4> &rot) {
  for (size_t c = 0; c < n_captures; ++c)
    if (!std::isfinite(offset_hz[c]) || std::fabs(offset_hz[c]) > (float)BTLE_MAX_OFFSET_HZ) {
      ctx->err = "offset_hz must be finite and within +-BTLE_MAX_OFFSET_HZ";
      return BTLE_EINVAL;
    }
  rot.resize(n);
  for (size_t i = 0; i < n; ++i) rot[i] = make_rot(offset_hz[cap_of ? cap_of[i] : i]);
  return BTLE_OK;
}

template <int KC, bool ROT>
void enqueue_rx(unsigned grid, cudaStream_t st, const MapSlot *ms, const int8_t *d_iq, size_t stride, size_t n_int8, const CfgSlot *cs,
                const Plan &plan, btle_pkt_rec *d_out, unsigned cap32, unsigned *d_count, btle_unit_dir *d_dir, unsigned *zero_next,
                long long lead) {
  btle_rx_persistent_kernel<KC, ROT><<<grid, kThreads, sizeof(Smem<KC>), st>>>(
      ms->map32, ms->map12, d_iq, (long long)stride, (long long)n_int8, cs->d_params, plan, d_out, cap32, d_count,
      reinterpret_cast<uint2 *>(d_dir), zero_next, lead, KC > 1 ? cs->d_vmap.p : nullptr, ROT ? cs->d_rot.p : nullptr);
}

// Enqueue the persistent kernel for device-resident inputs: n_cfgs cfgs on n_streams captures, cfg i decoding capture
// cfg_capture[i] (checked by check_cfg_capture), or capture i when cfg_capture is nullptr (then n_cfgs == n_streams).
// A list that maps cfg i to capture i for every capture runs btle_rx_persistent_kernel<1>, the directory in unit order;
// any other list runs <kMaxCfgsPerCapture> over the captures it names, the directory in (cfg, chunk) order.
// rot != nullptr: one rotation per cfg (make_rot), the rotated kernel variant.  `lead`: bytes readable in front of each
// capture (the stream session's lead: RSSI of hits at a segment's very start).
int launch_rx(btle_b200_ctx *ctx, const int8_t *d_iq, size_t n_streams, size_t stride, size_t n_int8, const btle_stream_cfg *cfgs,
              const int32_t *cfg_capture, size_t n_cfgs, const int4 *rot, btle_pkt_rec *d_out, size_t cap, unsigned *d_count,
              btle_unit_dir *d_dir, cudaStream_t st, long long lead) {
  ctx->last_launches = 0;
  unsigned *zero_next = nullptr;
  if (d_count) BTLE_CUDA(ctx, cudaMemsetAsync(d_count, 0, sizeof(unsigned), st));
  const long long nchunks = (long long)(n_int8 / kChunkInt8);
  if (nchunks == 0 || n_streams == 0 || n_cfgs == 0) return BTLE_OK;
  size_t groups = n_streams;                                  // captures the launch reads
  if (cfg_capture) {
    groups = 0;
    for (size_t i = 0; i < n_cfgs; ++i) groups += !i || cfg_capture[i] != cfg_capture[i - 1];
    if (groups == n_cfgs && n_cfgs == n_streams) cfg_capture = nullptr;   // cfg i on capture i
  }
  const bool multi = cfg_capture != nullptr;
  unsigned long long sid = 0;
  int rc = stream_id(ctx, st, &sid);
  if (rc) return rc;
  const long long spans = (nchunks + kSpanChunks - 1) / kSpanChunks;
  if (spans * (long long)n_cfgs > 0x07FFFFFFll || nchunks > 0x7FFFFFFFll) { ctx->err = "batch too large for one launch"; return BTLE_EINVAL; }
  const Plan plan = plan_for(ctx, groups, n_int8);
  if (multi && (plan.tail_units || (plan.big_units && plan.big_units != plan.total_units))) {
    ctx->err = "rx_multi: this build's unit plan is not the same for every capture";   // (A/B builds with a re-cut last wave)
    return BTLE_EINVAL;
  }
  CfgSlot *cs = nullptr;
  rc = upload_cfgs(ctx, cfgs, n_cfgs, st, sid, &cs, cfg_capture, rot);
  if (rc) return rc;
  const MapSlot *ms = nullptr;
  rc = get_maps(ctx, d_iq, n_streams, stride, n_int8, &ms);
  if (rc) return rc;
  StreamUse *ring = nullptr;
  if (!d_count) {
    // No counter from the caller (it reads the unit directory): take the next one of the context's ring, with no
    // memset node in front of the kernel.  Launch i (counted over the ring launches that ran) takes counter i % 64,
    // which launch i - 32 cleared, and clears counter (i + 32) % 64, which launch i - 32 used.  So launch i depends on
    // launch i - 32 alone (and through it on all earlier ones).  On the same stream that order is given; on another
    // stream this launch waits for its event.  One stream, or two in strict alternation, never waits.
    ring = &ctx->ring_last[ctx->ring_pos % (kCountRing / 2)];
    if (!ring->ev) BTLE_CUDA(ctx, cudaEventCreateWithFlags(&ring->ev, cudaEventDisableTiming));
    if (ring->stamp && ring->stream != sid) BTLE_CUDA(ctx, cudaStreamWaitEvent(st, ring->ev, 0));
    d_count = ctx->d_count_ring + ctx->ring_pos;
    zero_next = ctx->d_count_ring + (ctx->ring_pos + kCountRing / 2) % kCountRing;
  }
  const unsigned grid = (unsigned)std::min<long long>(plan.total_units, (long long)ctx->num_sms * kCtasPerSm);   // one persistent CTA per SM
  const auto enqueue = multi ? (rot ? enqueue_rx<kMaxCfgsPerCapture, true> : enqueue_rx<kMaxCfgsPerCapture, false>)
                             : (rot ? enqueue_rx<1, true> : enqueue_rx<1, false>);
  enqueue(grid, st, ms, d_iq, stride, n_int8, cs, plan, d_out, (unsigned)std::min<size_t>(cap, 0xFFFFFFFFu), d_count, d_dir, zero_next, lead);
  BTLE_CUDA(ctx, cudaGetLastError());
  if (ring) {                                                 // the position is taken only by a launch that was enqueued
    ctx->ring_pos = (ctx->ring_pos + 1) % kCountRing;
    BTLE_CUDA(ctx, cudaEventRecord(ring->ev, st));
    ring->stream = sid;
    ring->stamp = ++ctx->tick;
  }
  rc = note_use(ctx, cs, st, sid);
  if (rc) return rc;
  ctx->last_launches = 1;
  return BTLE_OK;
}

bool rec_less(const btle_pkt_rec &a, const btle_pkt_rec &b) {
  if (a.stream != b.stream) return a.stream < b.stream;
  if (a.chunk != b.chunk) return a.chunk < b.chunk;
  return a.n0 < b.n0;
}

// memcpy with a few threads: one core moves ~10 GB/s, a PCIe 5 x16 link takes ~55 GB/s
void par_memcpy(void *dst, const void *src, size_t n) {
  const size_t kMin = size_t(4) << 20;
  unsigned t = std::thread::hardware_concurrency();
  t = t >= 16 ? 6 : (t >= 4 ? 2 : 1);
  if (n < 2 * kMin || t < 2) { memcpy(dst, src, n); return; }
  std::vector<std::thread> th;
  const size_t per = ((n / t) + 4095) & ~size_t(4095);
  for (unsigned i = 1; i < t; ++i) {
    const size_t o = std::min(n, i * per), e = std::min(n, (i + 1) * per);
    if (e > o) th.emplace_back([=] { memcpy(static_cast<char *>(dst) + o, static_cast<const char *>(src) + o, e - o); });
  }
  memcpy(dst, src, std::min(n, per));
  for (auto &x : th) x.join();
}

bool is_pinned(const void *p) {
  cudaPointerAttributes a;
  if (cudaPointerGetAttributes(&a, p) != cudaSuccess) { cudaGetLastError(); return false; }
  return a.type == cudaMemoryTypeHost || a.type == cudaMemoryTypeManaged;
}

// Host -> device copy of `rows` rows of `width` bytes.  Page-locked sources go straight to the DMA engine; pageable
// sources are moved through two page-locked staging buffers in segments, the CPU copy of segment i+1 overlapping
// the DMA of segment i (cudaMemcpyAsync on pageable memory would stage synchronously at a fraction of the link rate).
int h2d_rows(btle_b200_ctx *ctx, int8_t *dst, size_t dpitch, const int8_t *src, size_t spitch, size_t width, size_t rows,
             cudaStream_t st) {
  if (!width || !rows) return BTLE_OK;
  if (is_pinned(src)) {
    if (rows == 1 || (dpitch == spitch && dpitch == width)) BTLE_CUDA(ctx, cudaMemcpyAsync(dst, src, width * rows, cudaMemcpyHostToDevice, st));
    else BTLE_CUDA(ctx, cudaMemcpy2DAsync(dst, dpitch, src, spitch, width, rows, cudaMemcpyHostToDevice, st));
    return BTLE_OK;
  }
  const size_t seg = size_t(32) << 20;
  for (int b = 0; b < 2; ++b) {
    if (ctx->h_stage[b].n < seg) {
      const int rc = ctx->h_stage[b].alloc(ctx, seg);
      if (rc) return rc;
    }
    if (!ctx->stage_free[b]) BTLE_CUDA(ctx, cudaEventCreateWithFlags(&ctx->stage_free[b], cudaEventDisableTiming));
  }
  int b = 0;
  bool used[2] = {false, false};
  for (size_t r = 0; r < rows; ++r)
    for (size_t o = 0; o < width; o += seg) {
      const size_t n = std::min(seg, width - o);
      if (used[b]) BTLE_CUDA(ctx, cudaEventSynchronize(ctx->stage_free[b]));
      par_memcpy(ctx->h_stage[b], src + r * spitch + o, n);
      BTLE_CUDA(ctx, cudaMemcpyAsync(dst + r * dpitch + o, ctx->h_stage[b], n, cudaMemcpyHostToDevice, st));
      BTLE_CUDA(ctx, cudaEventRecord(ctx->stage_free[b], st));
      used[b] = true;
      b ^= 1;
    }
  return BTLE_OK;
}

// Host captures (n_captures rows `stride` bytes apart, page-locked or pageable) -> ctx->d_iq, rows `*pitch` bytes apart:
// captures caps[0, n_read) (ascending; nullptr: captures 0 .. n_read - 1) one after the other, one copy per run of
// consecutive captures.  Exactly the caller's bytes are read: n_int8 per capture, never the padding behind the last one.
int ingest(btle_b200_ctx *ctx, const int8_t *iq, size_t n_captures, size_t stride, size_t n_int8, const int32_t *caps, size_t n_read,
           size_t *pitch) {
  if (n_captures > 1 && stride < n_int8) { ctx->err = "stream stride smaller than stream length"; return BTLE_EINVAL; }
  *pitch = (n_int8 + 15) & ~size_t(15);
  const size_t spitch = n_captures > 1 ? stride : n_int8;
  int rc = ctx->d_iq.reserve(ctx, std::max<size_t>(*pitch * n_read, 16));
  if (rc) return rc;
  for (size_t g = 0; g < n_read;) {
    size_t e = caps ? g + 1 : n_read;
    while (e < n_read && caps[e] == caps[e - 1] + 1) ++e;
    if (g) BTLE_CUDA(ctx, cudaStreamSynchronize(ctx->stream));   // a new copy may reuse the page-locked staging of the last one
    rc = h2d_rows(ctx, ctx->d_iq + g * *pitch, *pitch, iq + (caps ? (size_t)caps[g] : 0) * spitch, spitch, n_int8, e - g, ctx->stream);
    if (rc) return rc;
    g = e;
  }
  return BTLE_OK;
}

// After a launch on `st` that counted its results in ctx->d_count: the count to the host and a wait (*found = the
// count); then, when n = min(count, cap) > 0, copy(n) enqueues the copies of the first n results and they are waited for.
template <class Copy>
int fetch_counted(btle_b200_ctx *ctx, cudaStream_t st, size_t cap, size_t *found, Copy &&copy) {
  BTLE_CUDA(ctx, cudaMemcpyAsync(ctx->h_count, ctx->d_count, sizeof(unsigned), cudaMemcpyDeviceToHost, st));
  BTLE_CUDA(ctx, cudaStreamSynchronize(st));
  *found = *ctx->h_count;
  const size_t n = std::min(*found, cap);
  if (!n) return BTLE_OK;
  const int rc = copy(n);
  if (rc) return rc;
  BTLE_CUDA(ctx, cudaStreamSynchronize(st));
  return BTLE_OK;
}

// After a launch on `st`: count, records and unit directory to the host; records copied into `out` in reference
// order (walk of the directory).  *n_out = packets found (may exceed cap -> BTLE_EOVERFLOW).
int fetch_ordered(btle_b200_ctx *ctx, const btle_pkt_rec *d_out, const btle_unit_dir *d_dir, size_t n_units, btle_pkt_rec *out,
                  size_t cap, size_t *n_out, cudaStream_t st) {
  const int rc = fetch_counted(ctx, st, cap, n_out, [&](size_t n) {
    if (ctx->h_recs.reserve(ctx, n) || ctx->h_dir.reserve(ctx, n_units)) return BTLE_ENOMEM;
    BTLE_CUDA(ctx, cudaMemcpyAsync(ctx->h_recs, d_out, n * sizeof(btle_pkt_rec), cudaMemcpyDeviceToHost, st));
    BTLE_CUDA(ctx, cudaMemcpyAsync(ctx->h_dir, d_dir, n_units * sizeof(btle_unit_dir), cudaMemcpyDeviceToHost, st));
    return BTLE_OK;
  });
  if (rc) return rc;
  if (const size_t n = std::min(*n_out, cap)) {
    size_t got = 0;
    btle_b200_gather_ordered(ctx->h_recs, n, ctx->h_dir, n_units, out, cap, &got);
  }
  if (*n_out > cap) { ctx->err = "output capacity too small"; return BTLE_EOVERFLOW; }
  return BTLE_OK;
}

// The receive entry points: cfg i decodes capture cfg_capture[i], or capture i when cfg_capture is nullptr (then
// n_cfgs == n_captures).  rx_device_path checks and enqueues a launch on device-resident captures.
int rx_device_path(btle_b200_ctx *ctx, const int8_t *d_iq, size_t n_captures, size_t stride, size_t n_int8, const btle_stream_cfg *cfgs,
                   const int32_t *cfg_capture, size_t n_cfgs, const float *offset_hz, btle_pkt_rec *d_out, size_t cap, uint32_t *d_count,
                   btle_unit_dir *d_dir, size_t dir_cap, void *cuda_stream) {
  if (!ctx) return BTLE_EINVAL;
  if ((!d_out && cap) || (!cfgs && n_cfgs) || !d_dir) { ctx->err = "rx: missing buffer"; return BTLE_EINVAL; }
  if ((reinterpret_cast<uintptr_t>(d_iq) & 15) || (n_captures > 1 && (stride & 15))) { ctx->err = "device IQ must be 16-byte aligned"; return BTLE_EINVAL; }
  if (n_captures > 1 && stride < n_int8) { ctx->err = "stream stride smaller than stream length"; return BTLE_EINVAL; }
  size_t groups = n_cfgs;
  int rc = cfg_capture ? check_cfg_capture(ctx, n_captures, cfg_capture, n_cfgs, &groups) : BTLE_OK;
  if (rc) return rc;
  if (dir_cap < rx_units(ctx, groups, n_cfgs, n_int8)) { ctx->err = "unit directory too small (btle_b200_rx_units / _rx_multi_units)"; return BTLE_EINVAL; }
  rc = validate_cfgs(ctx, cfgs, n_cfgs);
  if (rc) return rc;
  std::vector<int4> rot;
  if (offset_hz && (rc = make_rots(ctx, offset_hz, n_captures, cfg_capture, n_cfgs, rot))) return rc;
  BTLE_CUDA(ctx, cudaSetDevice(ctx->device));
  return launch_rx(ctx, d_iq, n_captures, stride, n_int8, cfgs, cfg_capture, n_cfgs, offset_hz ? rot.data() : nullptr, d_out, cap, d_count,
                   d_dir, reinterpret_cast<cudaStream_t>(cuda_stream), 0);
}

// Host captures in, records out in reference order: only the captures some cfg reads are copied, one after the other,
// and the list is renumbered to match (a list that names each capture it reads once is then cfg i on capture i).
int rx_host_path(btle_b200_ctx *ctx, const int8_t *iq, size_t n_captures, size_t stride, size_t n_int8, const btle_stream_cfg *cfgs,
                 const int32_t *cfg_capture, size_t n_cfgs, const float *offset_hz, btle_pkt_rec *out, size_t cap, size_t *n_out) {
  if (!ctx) return BTLE_EINVAL;
  if (!n_out || (!out && cap) || (!cfgs && n_cfgs) || (!iq && n_captures && n_int8)) { ctx->err = "rx: missing buffer"; return BTLE_EINVAL; }
  *n_out = 0;
  size_t groups = n_cfgs;
  int rc = cfg_capture ? check_cfg_capture(ctx, n_captures, cfg_capture, n_cfgs, &groups) : BTLE_OK;
  if (rc) return rc;
  rc = validate_cfgs(ctx, cfgs, n_cfgs);
  if (rc) return rc;
  std::vector<int4> rot;
  if (offset_hz && (rc = make_rots(ctx, offset_hz, n_captures, cfg_capture, n_cfgs, rot))) return rc;
  BTLE_CUDA(ctx, cudaSetDevice(ctx->device));
  std::vector<int32_t> caps, local;                          // the captures read, in order; cfg i reads caps[local[i]]
  for (size_t i = 0; cfg_capture && i < n_cfgs; ++i) {
    if (!i || cfg_capture[i] != cfg_capture[i - 1]) caps.push_back(cfg_capture[i]);
    local.push_back((int32_t)caps.size() - 1);
  }
  size_t pitch = 0;
  rc = ingest(ctx, iq, n_captures, stride, n_int8, cfg_capture ? caps.data() : nullptr, groups, &pitch);
  if (rc) return rc;
  const size_t units = rx_units(ctx, groups, n_cfgs, n_int8);
  if (ctx->d_out.reserve(ctx, std::max<size_t>(cap, 1)) || ctx->d_dir.reserve(ctx, std::max<size_t>(units, 1))) return BTLE_ENOMEM;
  rc = launch_rx(ctx, ctx->d_iq, groups, pitch, n_int8, cfgs, cfg_capture ? local.data() : nullptr, n_cfgs, offset_hz ? rot.data() : nullptr,
                 ctx->d_out, cap, ctx->d_count, ctx->d_dir, ctx->stream, 0);
  if (rc) return rc;
  return fetch_ordered(ctx, ctx->d_out, ctx->d_dir, units, out, cap, n_out, ctx->stream);
}

int launch_sps8_hits(btle_b200_ctx *ctx, const int16_t *d_iq16, size_t n_samples, uint32_t aa, long long *d_hits, size_t cap, unsigned *d_count,
                     cudaStream_t st) {
  const long long groups = ((long long)n_samples + 255) / 256, tiles = (groups + kSps8Groups - 1) / kSps8Groups;
  const unsigned grid = kSps8Bufs > 1 ? (unsigned)std::min<long long>(tiles, 3ll * ctx->num_sms) : (unsigned)std::min<long long>(tiles, 0x7FFFFFFF);
  sps8_hits_kernel<<<grid, 256, kSps8Smem, st>>>(d_iq16, (long long)n_samples, tiles, aa, d_hits, (unsigned)cap, d_count);
  BTLE_CUDA(ctx, cudaGetLastError());
  return BTLE_OK;
}

// Checks and launch of discover_kernel (the counter is zeroed here).  The channels travel as btle_stream_cfg through the
// cfg cache, so the kernel reads each capture's whitening words from its StreamParams.
int check_data_channels(btle_b200_ctx *ctx, const int32_t *channels, size_t n_streams) {
  if (!channels && n_streams) { ctx->err = "discover: missing channel array"; return BTLE_EINVAL; }
  for (size_t s = 0; s < n_streams; ++s)
    if (channels[s] < 0 || channels[s] > 36) { ctx->err = "discover: data channel must be within 0~36"; return BTLE_EINVAL; }
  return BTLE_OK;
}

int launch_discover(btle_b200_ctx *ctx, const int8_t *d_iq, size_t n_streams, size_t stride, size_t n_int8, const int32_t *channels,
                    btle_conn_cand *d_out, size_t cap, unsigned *d_count, cudaStream_t st) {
  if (!d_count || (!d_out && cap) || (!d_iq && n_streams && n_int8)) { ctx->err = "discover: missing buffer"; return BTLE_EINVAL; }
  if ((reinterpret_cast<uintptr_t>(d_iq) & 15) || (n_streams > 1 && (stride & 15))) { ctx->err = "device IQ must be 16-byte aligned"; return BTLE_EINVAL; }
  if (n_streams > 1 && stride < n_int8) { ctx->err = "stream stride smaller than stream length"; return BTLE_EINVAL; }
  int rc = check_data_channels(ctx, channels, n_streams);
  if (rc) return rc;
  BTLE_CUDA(ctx, cudaSetDevice(ctx->device));
  ctx->last_launches = 0;
  BTLE_CUDA(ctx, cudaMemsetAsync(d_count, 0, sizeof(unsigned), st));
  const long long n_samples = (long long)(n_int8 / 2);
  if (!n_streams || n_samples < 32 + 286) return BTLE_OK;                  // no window fits
  const long long groups = (n_samples - 286) / 128 + 1;                    // groups holding a window start inside the capture
  const long long tiles = (groups + kDiscGroups - 1) / kDiscGroups;
  if (tiles * (long long)n_streams > 0x7FFFFFFFll) { ctx->err = "batch too large for one launch"; return BTLE_EINVAL; }
  std::vector<btle_stream_cfg> cfgs(n_streams);
  for (size_t s = 0; s < n_streams; ++s) cfgs[s] = btle_stream_cfg{channels[s], 0x8E89BED6u, 0xFFFFFFFFu, 0x555555u, 0, 0};
  unsigned long long sid = 0;
  rc = stream_id(ctx, st, &sid);
  if (rc) return rc;
  CfgSlot *cs = nullptr;
  rc = upload_cfgs(ctx, cfgs.data(), n_streams, st, sid, &cs);
  if (rc) return rc;
  discover_kernel<<<(unsigned)(tiles * (long long)n_streams), kDiscThreads, kDiscSmem, st>>>(
      d_iq, (long long)stride, (long long)n_int8, tiles, cs->d_params, d_out, (unsigned)std::min<size_t>(cap, 0xFFFFFFFFu), d_count);
  BTLE_CUDA(ctx, cudaGetLastError());
  rc = note_use(ctx, cs, st, sid);
  if (rc) return rc;
  ctx->last_launches = 1;
  return BTLE_OK;
}

}  // namespace

extern "C" {

uint32_t btle_b200_version(void) { return (0u << 16) | 3u; }

const char *btle_b200_strerror(int code) {
  switch (code) {
    case BTLE_OK: return "ok";
    case BTLE_EINVAL: return "invalid argument";
    case BTLE_ENODEV: return "no usable CUDA device";
    case BTLE_ENOMEM: return "out of memory";
    case BTLE_ECUDA: return "CUDA error";
    case BTLE_EOVERFLOW: return "more packets than the output capacity";
    default: return "unknown error";
  }
}

const char *btle_b200_last_error(const btle_b200_ctx *ctx) { return ctx ? ctx->err.c_str() : "null context"; }
int btle_b200_last_launches(const btle_b200_ctx *ctx) { return ctx ? ctx->last_launches : 0; }

int btle_b200_bind_host_numa(int cuda_device, int *node_out) {
  if (node_out) *node_out = -1;
  char bus[64] = {0};
  if (cudaDeviceGetPCIBusId(bus, (int)sizeof bus, cuda_device) != cudaSuccess) { cudaGetLastError(); return BTLE_ENODEV; }
  for (char *c = bus; *c; ++c) if (*c >= 'A' && *c <= 'F') *c = (char)(*c - 'A' + 'a');
  char path[256];
  snprintf(path, sizeof path, "/sys/bus/pci/devices/%s/numa_node", bus);
  int node = -1;
  if (FILE *f = fopen(path, "r")) { if (fscanf(f, "%d", &node) != 1) node = -1; fclose(f); }
  if (node < 0) return BTLE_OK;                            // single-node machine or not exposed: nothing to bind
  snprintf(path, sizeof path, "/sys/devices/system/node/node%d/cpulist", node);
  cpu_set_t want, have, both;
  CPU_ZERO(&want);
  if (FILE *f = fopen(path, "r")) {                        // "0-47,96-143"
    int a, b;
    while (fscanf(f, "%d", &a) == 1) {
      b = a;
      int ch = fgetc(f);
      if (ch == '-') { if (fscanf(f, "%d", &b) != 1) b = a; ch = fgetc(f); }
      for (int c = a; c <= b && c < CPU_SETSIZE; ++c) CPU_SET(c, &want);
      if (ch != ',') break;
    }
    fclose(f);
  }
  if (sched_getaffinity(0, sizeof have, &have) == 0) {
    CPU_AND(&both, &want, &have);                          // never widen what a cpuset / taskset allowed
    if (CPU_COUNT(&both) > 0) sched_setaffinity(0, sizeof both, &both);
  }
  if (node < 1024) {                                       // MPOL_PREFERRED: pages this thread touches (and pins) come from `node`
    unsigned long mask[16] = {0};
    mask[node / (8 * sizeof(unsigned long))] |= 1ul << (node % (8 * sizeof(unsigned long)));
    syscall(SYS_set_mempolicy, 1 /* MPOL_PREFERRED */, mask, (unsigned long)(8 * sizeof mask));
  }
  if (node_out) *node_out = node;
  return BTLE_OK;
}

int btle_b200_create(btle_b200_ctx **out, int cuda_device) {
  if (!out) return BTLE_EINVAL;
  *out = nullptr;
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev <= 0 || cuda_device < 0 || cuda_device >= ndev) {
    cudaGetLastError();
    return BTLE_ENODEV;   // no CPU fallback, by design
  }
  btle_b200_ctx *ctx = new (std::nothrow) btle_b200_ctx();
  if (!ctx) return BTLE_ENOMEM;
  ctx->device = cuda_device;
  if (cudaSetDevice(cuda_device) != cudaSuccess) { delete ctx; return BTLE_ENODEV; }
  // protocol tables -> constant memory
  uint32_t ww[40][12];
  for (int ch = 0; ch < 40; ++ch) { uint8_t row[48]; make_whiten_row(ch, row); memcpy(ww[ch], row, 48); }
  uint32_t crc[1024];
  make_crc4(crc);
  if (cudaDeviceGetAttribute(&ctx->num_sms, cudaDevAttrMultiProcessorCount, cuda_device) != cudaSuccess || ctx->num_sms < 1) {
    cudaGetLastError();
    delete ctx;
    return BTLE_ECUDA;
  }
  if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &ctx->encode_tiled, cudaEnableDefault, nullptr) != cudaSuccess ||
      !ctx->encode_tiled) {
    cudaGetLastError();
    delete ctx;
    return BTLE_ENODEV;
  }
  {
    static int8_t c1[1024], s1[1024], c2[2048], s2[2048];
    const double two_pi = 6.283185307179586476925286766559;
    for (int k = 0; k < 1024; ++k) { c1[k] = (int8_t)nearbyint(127.0 * cos(two_pi * k / 1024.0)); s1[k] = (int8_t)nearbyint(127.0 * sin(two_pi * k / 1024.0)); }
    for (int k = 0; k < 2048; ++k) { c2[k] = (int8_t)nearbyint(127.0 * cos(two_pi * k / 2048.0)); s2[k] = (int8_t)nearbyint(127.0 * sin(two_pi * k / 2048.0)); }
    if (cudaMemcpyToSymbol(c_cos1024, c1, sizeof c1) != cudaSuccess || cudaMemcpyToSymbol(c_sin1024, s1, sizeof s1) != cudaSuccess ||
        cudaMemcpyToSymbol(c_cos2048, c2, sizeof c2) != cudaSuccess || cudaMemcpyToSymbol(c_sin2048, s2, sizeof s2) != cudaSuccess) {
      cudaGetLastError();
      btle_b200_destroy(ctx);
      return BTLE_ECUDA;
    }
  }
  uint32_t thr[13];
  for (int k = 0; k < 13; ++k) {                         // P(round(N(-0.3, 0.8)) <= v), v = -7 + k
    const double p = 0.5 * erfc(-(((double)(-7 + k) + 0.5 + 0.3) / 0.8) / sqrt(2.0));
    thr[k] = (uint32_t)std::min(4294967295.0, p * 4294967296.0);
  }
  if (cudaMemcpyToSymbol(c_noise_thr, thr, sizeof thr) != cudaSuccess ||
      cudaMemcpyToSymbol(c_whiten_words, ww, sizeof ww) != cudaSuccess ||
      cudaMemcpyToSymbol(c_crc4, crc, sizeof crc) != cudaSuccess ||
      cudaFuncSetAttribute(btle_rx_persistent_kernel<1, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(Smem<1>)) != cudaSuccess ||
      cudaFuncSetAttribute(btle_rx_persistent_kernel<kMaxCfgsPerCapture, false>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                           (int)sizeof(Smem<kMaxCfgsPerCapture>)) != cudaSuccess ||
      cudaFuncSetAttribute(btle_rx_persistent_kernel<1, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(Smem<1>)) != cudaSuccess ||
      cudaFuncSetAttribute(btle_rx_persistent_kernel<kMaxCfgsPerCapture, true>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                           (int)sizeof(Smem<kMaxCfgsPerCapture>)) != cudaSuccess ||
      cudaFuncSetAttribute(sps8_hits_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kSps8Smem) != cudaSuccess ||
      cudaFuncSetAttribute(discover_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kDiscSmem) != cudaSuccess ||
      cudaStreamCreateWithFlags(&ctx->stream, cudaStreamNonBlocking) != cudaSuccess ||
      ctx->d_count.alloc(ctx, 1) || ctx->d_count_ring.alloc(ctx, kCountRing) ||
      cudaMemset(ctx->d_count_ring, 0, kCountRing * sizeof(unsigned)) != cudaSuccess || ctx->h_count.alloc(ctx, 1)) {
    cudaGetLastError();
    btle_b200_destroy(ctx);
    return BTLE_ECUDA;
  }
  *out = ctx;
  return BTLE_OK;
}

void btle_b200_destroy(btle_b200_ctx *ctx) {
  if (!ctx) return;
  cudaSetDevice(ctx->device);
  if (ctx->stream) cudaStreamDestroy(ctx->stream);
  for (CfgSlot &c : ctx->cfg_slot) {
    if (c.uploaded) cudaEventDestroy(c.uploaded);
    for (StreamUse &u : c.use) if (u.ev) cudaEventDestroy(u.ev);
  }
  for (StreamUse &u : ctx->ring_last) if (u.ev) cudaEventDestroy(u.ev);
  for (cudaEvent_t e : ctx->stage_free) if (e) cudaEventDestroy(e);
  delete ctx;                                               // frees the buffers
}

size_t btle_b200_rx_units(const btle_b200_ctx *ctx, size_t n_streams, size_t n_int8) {
  return ctx ? rx_units(ctx, n_streams, n_streams, n_int8) : 0;
}

int btle_b200_rx_device_dir_offset(btle_b200_ctx *ctx, const int8_t *d_iq, size_t n_streams, size_t stride, size_t n_int8,
                                   const btle_stream_cfg *cfgs, const float *offset_hz, btle_pkt_rec *d_out, size_t cap, uint32_t *d_count,
                                   btle_unit_dir *d_dir, size_t dir_cap, void *cuda_stream) {
  return rx_device_path(ctx, d_iq, n_streams, stride, n_int8, cfgs, nullptr, n_streams, offset_hz, d_out, cap, d_count, d_dir, dir_cap,
                        cuda_stream);
}

int btle_b200_rx_device_dir(btle_b200_ctx *ctx, const int8_t *d_iq, size_t n_streams, size_t stride, size_t n_int8,
                            const btle_stream_cfg *cfgs, btle_pkt_rec *d_out, size_t cap, uint32_t *d_count,
                            btle_unit_dir *d_dir, size_t dir_cap, void *cuda_stream) {
  return rx_device_path(ctx, d_iq, n_streams, stride, n_int8, cfgs, nullptr, n_streams, nullptr, d_out, cap, d_count, d_dir, dir_cap,
                        cuda_stream);
}

int btle_b200_rx_device(btle_b200_ctx *ctx, const int8_t *d_iq, size_t n_streams, size_t stride, size_t n_int8,
                        const btle_stream_cfg *cfgs, btle_pkt_rec *d_out, size_t cap, uint32_t *d_count,
                        void *cuda_stream) {
  if (!ctx) return BTLE_EINVAL;
  BTLE_CUDA(ctx, cudaSetDevice(ctx->device));
  // the directory goes to context-owned scratch (callers of this entry point sort the records themselves)
  const int rc = ctx->d_dir.reserve(ctx, std::max<size_t>(btle_b200_rx_units(ctx, n_streams, n_int8), 1));
  if (rc) return rc;
  return rx_device_path(ctx, d_iq, n_streams, stride, n_int8, cfgs, nullptr, n_streams, nullptr, d_out, cap, d_count, ctx->d_dir,
                        ctx->d_dir.n, cuda_stream);
}

void btle_b200_sort_records(btle_pkt_rec *recs, size_t n) { std::sort(recs, recs + n, rec_less); }

int btle_b200_gather_ordered(const btle_pkt_rec *recs, size_t n_recs, const btle_unit_dir *dir, size_t n_units,
                             btle_pkt_rec *out, size_t cap, size_t *n_out) {
  if ((!recs && n_recs) || (!dir && n_units) || (!out && cap) || !n_out) return BTLE_EINVAL;
  size_t pos = 0, total = 0;
  for (size_t u = 0; u < n_units; ++u) {
    const size_t base = dir[u].base, cnt = dir[u].count;
    total += cnt;
    if (base >= n_recs) continue;                           // block was cut off by the producer's capacity
    const size_t take = std::min(std::min(cnt, n_recs - base), cap - pos);
    if (take) memcpy(out + pos, recs + base, take * sizeof(btle_pkt_rec));
    pos += take;
  }
  *n_out = total;
  return total > cap || pos < total ? BTLE_EOVERFLOW : BTLE_OK;
}

int btle_b200_rx_batch_offset(btle_b200_ctx *ctx, const int8_t *iq, size_t n_streams, size_t stride, size_t n_int8,
                              const btle_stream_cfg *cfgs, const float *offset_hz, btle_pkt_rec *out, size_t cap, size_t *n_out) {
  return rx_host_path(ctx, iq, n_streams, stride, n_int8, cfgs, nullptr, n_streams, offset_hz, out, cap, n_out);
}

int btle_b200_rx_batch(btle_b200_ctx *ctx, const int8_t *iq, size_t n_streams, size_t stride, size_t n_int8,
                       const btle_stream_cfg *cfgs, btle_pkt_rec *out, size_t cap, size_t *n_out) {
  return rx_host_path(ctx, iq, n_streams, stride, n_int8, cfgs, nullptr, n_streams, nullptr, out, cap, n_out);
}

int btle_b200_rec_offset_device(btle_b200_ctx *ctx, const int8_t *d_iq, size_t stride, size_t n_int8, const btle_pkt_rec *d_recs, size_t n,
                                float *d_hz, void *cuda_stream) {
  if (!ctx) return BTLE_EINVAL;
  if (n && (!d_recs || !d_hz || (!d_iq && n_int8))) { ctx->err = "rec_offset: missing buffer"; return BTLE_EINVAL; }
  if (!n) return BTLE_OK;
  BTLE_CUDA(ctx, cudaSetDevice(ctx->device));
  const long long blocks = ((long long)n + 7) / 8;                 // 8 warps (records) per block
  if (blocks > 0x7FFFFFFFll) { ctx->err = "rec_offset: too many records"; return BTLE_EINVAL; }
  rec_offset_kernel<<<(unsigned)blocks, 256, 0, reinterpret_cast<cudaStream_t>(cuda_stream)>>>(d_iq, (long long)stride, (long long)n_int8, d_recs,
                                                                                           (long long)n, d_hz);
  BTLE_CUDA(ctx, cudaGetLastError());
  return BTLE_OK;
}

int btle_b200_rec_offset(btle_b200_ctx *ctx, const int8_t *iq, size_t n_streams, size_t stride, size_t n_int8, const btle_pkt_rec *recs, size_t n,
                         float *hz) {
  if (!ctx || (n && (!recs || !hz)) || (!iq && n_streams && n_int8)) return BTLE_EINVAL;
  for (size_t i = 0; i < n; ++i)
    if (recs[i].stream < 0 || (size_t)recs[i].stream >= n_streams) { ctx->err = "rec_offset: record stream out of range"; return BTLE_EINVAL; }
  if (!n) return BTLE_OK;
  BTLE_CUDA(ctx, cudaSetDevice(ctx->device));
  cudaStream_t st = ctx->stream;
  size_t pitch = 0;
  int rc = ingest(ctx, iq, n_streams, stride, n_int8, nullptr, n_streams, &pitch);
  if (rc) return rc;
  if (ctx->d_out.reserve(ctx, n) || ctx->d_hz.reserve(ctx, n)) return BTLE_ENOMEM;
  BTLE_CUDA(ctx, cudaMemcpyAsync(ctx->d_out, recs, n * sizeof(btle_pkt_rec), cudaMemcpyHostToDevice, st));
  rc = btle_b200_rec_offset_device(ctx, ctx->d_iq, pitch, n_int8, ctx->d_out, n, ctx->d_hz, st);
  if (rc) return rc;
  BTLE_CUDA(ctx, cudaMemcpyAsync(hz, ctx->d_hz, n * sizeof(float), cudaMemcpyDeviceToHost, st));
  BTLE_CUDA(ctx, cudaStreamSynchronize(st));
  return BTLE_OK;
}

int btle_b200_rx_iq16(btle_b200_ctx *ctx, const int16_t *iq16, size_t n_int16, int shift, const btle_stream_cfg *cfg,
                      btle_pkt_rec *out, size_t cap, size_t *n_out) {
  if (!ctx || (!iq16 && n_int16) || !cfg || !n_out || (!out && cap) || shift < 0 || shift > 8) return BTLE_EINVAL;
  *n_out = 0;
  BTLE_CUDA(ctx, cudaSetDevice(ctx->device));
  cudaStream_t st = ctx->stream;
  const size_t pitch = (n_int16 + 255) & ~size_t(255);
  if (ctx->d_iq.reserve(ctx, pitch + 2 * n_int16 + 512) || ctx->d_out.reserve(ctx, std::max<size_t>(cap, 1))) return BTLE_ENOMEM;
  int16_t *d16 = reinterpret_cast<int16_t *>(ctx->d_iq + pitch + 256);      // behind the int8 capture
  if (n_int16) {
    const int rc = h2d_rows(ctx, reinterpret_cast<int8_t *>(d16), 2 * n_int16, reinterpret_cast<const int8_t *>(iq16), 2 * n_int16, 2 * n_int16, 1, st);
    if (rc) return rc;
    iq16_to_iq8_kernel<<<(unsigned)std::min<size_t>((n_int16 + 255) / 256, (size_t)ctx->num_sms * 16), 256, 0, st>>>(d16, (long long)n_int16, shift, ctx->d_iq);
    BTLE_CUDA(ctx, cudaGetLastError());
  }
  const int rc = btle_b200_rx_device(ctx, ctx->d_iq, 1, pitch, n_int16, cfg, ctx->d_out, cap, ctx->d_count, st);
  if (rc) return rc;
  return fetch_ordered(ctx, ctx->d_out, ctx->d_dir, btle_b200_rx_units(ctx, 1, n_int16), out, cap, n_out, st);
}

int btle_b200_rx(btle_b200_ctx *ctx, const int8_t *iq, size_t n_int8, const btle_stream_cfg *cfg, btle_pkt_rec *out,
                 size_t cap, size_t *n_out) {
  return rx_host_path(ctx, iq, 1, n_int8, n_int8, cfg, nullptr, 1, nullptr, out, cap, n_out);
}

// ---- several cfgs per capture -------------------------------------------------------------------------------------
size_t btle_b200_rx_multi_units(const btle_b200_ctx *ctx, size_t n_captures, const int32_t *cfg_capture, size_t n_cfgs, size_t n_int8) {
  if (!ctx || !n_cfgs || !cfg_capture) return 0;
  size_t groups = 0;
  btle_b200_ctx *c = const_cast<btle_b200_ctx *>(ctx);
  const std::string keep = c->err;                        // a query: leaves last_error as it was
  const int rc = check_cfg_capture(c, n_captures, cfg_capture, n_cfgs, &groups);
  c->err = keep;
  return rc ? 0 : rx_units(ctx, groups, n_cfgs, n_int8);
}

int btle_b200_rx_multi_device_dir_offset(btle_b200_ctx *ctx, const int8_t *d_iq, size_t n_captures, size_t stride, size_t n_int8,
                                         const btle_stream_cfg *cfgs, const int32_t *cfg_capture, size_t n_cfgs, const float *offset_hz,
                                         btle_pkt_rec *d_out, size_t cap, uint32_t *d_count, btle_unit_dir *d_dir, size_t dir_cap,
                                         void *cuda_stream) {
  if (ctx && n_cfgs && !cfg_capture) { ctx->err = "rx_multi: missing cfg_capture"; return BTLE_EINVAL; }
  return rx_device_path(ctx, d_iq, n_captures, stride, n_int8, cfgs, cfg_capture, n_cfgs, offset_hz, d_out, cap, d_count, d_dir, dir_cap,
                        cuda_stream);
}

int btle_b200_rx_multi_device_dir(btle_b200_ctx *ctx, const int8_t *d_iq, size_t n_captures, size_t stride, size_t n_int8,
                                  const btle_stream_cfg *cfgs, const int32_t *cfg_capture, size_t n_cfgs, btle_pkt_rec *d_out,
                                  size_t cap, uint32_t *d_count, btle_unit_dir *d_dir, size_t dir_cap, void *cuda_stream) {
  return btle_b200_rx_multi_device_dir_offset(ctx, d_iq, n_captures, stride, n_int8, cfgs, cfg_capture, n_cfgs, nullptr, d_out, cap, d_count,
                                              d_dir, dir_cap, cuda_stream);
}

int btle_b200_rx_multi(btle_b200_ctx *ctx, const int8_t *iq, size_t n_captures, size_t stride, size_t n_int8, const btle_stream_cfg *cfgs,
                       const int32_t *cfg_capture, size_t n_cfgs, btle_pkt_rec *out, size_t cap, size_t *n_out) {
  return btle_b200_rx_multi_offset(ctx, iq, n_captures, stride, n_int8, cfgs, cfg_capture, n_cfgs, nullptr, out, cap, n_out);
}

int btle_b200_rx_multi_offset(btle_b200_ctx *ctx, const int8_t *iq, size_t n_captures, size_t stride, size_t n_int8, const btle_stream_cfg *cfgs,
                              const int32_t *cfg_capture, size_t n_cfgs, const float *offset_hz, btle_pkt_rec *out, size_t cap, size_t *n_out) {
  if (ctx && n_cfgs && !cfg_capture) { ctx->err = "rx_multi: missing cfg_capture"; return BTLE_EINVAL; }
  return rx_host_path(ctx, iq, n_captures, stride, n_int8, cfgs, cfg_capture, n_cfgs, offset_hz, out, cap, n_out);
}

// ---- streaming sessions: N time-aligned captures of unbounded length, pushed in pieces ----------------------------
}  // extern "C"

// One segment SET = `seg_chunks` chunks of every capture.  Capture i's part of a set sits at i * stride in the half's
// buffers: kLead bytes of the previous set, the segment, kLook look-ahead bytes (the start of the next set).  Once every
// capture has filled its own, a set's live cfgs are decoded in rounds of at most kMaxCfgsPerCapture cfgs per capture,
// one launch of the persistent kernel each (launch_rx: the single-cfg kernel for a round of one cfg per capture in
// capture order, as every set of a session whose cfg list never changed is).  A cfg added for chunks that are still
// resident is decoded over them by one more round on the half that holds them (backfill).
struct btle_b200_streams {
  btle_b200_ctx *ctx = nullptr;
  size_t n = 0;                                            // captures in the session
  struct Entry {                                           // stable cfg index j: decodes `capture` for chunks [from, until)
    btle_stream_cfg cfg; size_t capture; long long from, until;
  };
  std::vector<Entry> entries;                              // [0, n): the cfgs of streams_open
  std::vector<size_t> backfill;                            // cfgs added since the last commit / finish (streams_backfill)
  int call_launches = 0;                                   // launches of the current commit / finish call
  std::vector<int32_t> disc;                               // data channel scanned per capture, -1: none (set_discover)
  std::vector<float> offset;                               // carrier offset per capture (set_offset); empty: never set, default kernel
  std::vector<btle_conn_cand> cands;                       // candidates of the sets handed out, not yet taken
  size_t seg_chunks = 0, seg_bytes = 0, buf_bytes = 0;     // a part = seg_chunks chunks (+ kLook look-ahead bytes behind it)
  size_t stride = 0;                                       // kLead + buf_bytes: bytes from one capture's part to the next
  static constexpr size_t kLook = 4096;                    // >= 3008 + the kernel's 12-group tile (3072 + 4)
  static constexpr size_t kLead = 256;                     // bytes of the previous set kept in front (a hit may start up to 124 samples
                                                           // before its chunk; the RSSI sum reads the raw IQ there)
  struct Job {                                             // one round's launch on a half's IQ, collected with the half
    std::vector<size_t> index;                             // launch position -> stable cfg index
    size_t units = 0, cap = 0;
    Buf<btle_pkt_rec> d_out; Buf<btle_unit_dir> d_dir; Buf<unsigned> d_count;
    HostBuf<unsigned> h_count; HostBuf<btle_unit_dir> h_dir;
  };
  struct Scan {                                            // one discover launch over captures [first, first + count)
    size_t first = 0, count = 0, off = 0, cap = 0;         // candidates at d_cand[off, off + cap)
  };
  struct Half {
    HostBuf<int8_t> h; Buf<int8_t> d;                      // page-locked host / device IQ buffers, n parts of `stride` bytes
    size_t n_submitted = 0;
    long long first_chunk = 0;
    std::vector<float> offset;                             // the session's offsets when the set was submitted (backfill reuses them)
    cudaStream_t st = nullptr;
    bool resident = false;                                 // d holds the set at first_chunk (lead, n_submitted bytes)
    std::vector<std::unique_ptr<Job>> jobs;                // jobs[0, n_jobs) wait to be collected (grown, then reused)
    size_t n_jobs = 0;
    HostBuf<btle_pkt_rec> h_jrecs;                         // their records, grown to what they found
    std::vector<Scan> scans;                               // discover launches waiting to be collected
    std::vector<int32_t> scan_ch;                          // the channels they scanned, per capture
    size_t scan_samples = 0;                               // window starts kept: local samples [128, 128 + scan_samples)
    size_t scan_bytes = 0;                                 // bytes each scanned part was read with (lead included)
    Buf<btle_conn_cand> d_cand; Buf<unsigned> d_ccount; HostBuf<unsigned> h_ccount; HostBuf<btle_conn_cand> h_cand;
  } half[2];
  std::vector<size_t> fill;                                // bytes in each capture's part of the half being filled
  size_t n_full = 0;                                       // captures whose part of that half is complete
  int cur = 0;                                             // half being filled
  long long next_chunk = 0;                                // stream-wide index of the first chunk of the half being filled
  std::vector<btle_pkt_rec> ready;                         // decoded, not yet handed out
  size_t ready_pos = 0;
};

// the single-capture session is a one-capture btle_b200_streams
struct btle_b200_stream {
  btle_b200_streams *m = nullptr;
};

namespace {
using Streams = btle_b200_streams;

// One round's launch over half b's set, enqueued behind whatever its stream holds: cfgs `idx` (stable indices, sorted
// by capture, at most kMaxCfgsPerCapture per capture) on the set's n_submitted bytes.  Buffers, strides and cfgs are the
// session's own, checked when made.  Collected by streams_collect.
int streams_job(Streams *s, int b, const std::vector<size_t> &idx) {
  btle_b200_ctx *ctx = s->ctx;
  auto &H = s->half[b];
  if (H.n_jobs == H.jobs.size()) {
    H.jobs.emplace_back(new (std::nothrow) Streams::Job());
    if (!H.jobs.back()) { H.jobs.pop_back(); return BTLE_ENOMEM; }
  }
  Streams::Job &J = *H.jobs[H.n_jobs];
  const size_t k = idx.size(), nch = H.n_submitted / kChunkInt8;
  std::vector<btle_stream_cfg> cfgs(k);
  std::vector<int32_t> cc(k);
  size_t groups = 0;                                         // captures the round reads
  std::vector<int4> rot;                                     // H.offset non-empty: the rotated kernel, capture cc[i]'s offset
  for (size_t i = 0; i < k; ++i) {
    cfgs[i] = s->entries[idx[i]].cfg;
    cc[i] = (int32_t)s->entries[idx[i]].capture;
    groups += !i || cc[i] != cc[i - 1];
    if (!H.offset.empty()) rot.push_back(make_rot(H.offset[cc[i]]));
  }
  const size_t units = std::max<size_t>(rx_units(ctx, groups, k, H.n_submitted), 1);
  const size_t cap = k * nch * BTLE_MAX_RECS_PER_CHUNK;      // the most a launch can find: never an overflow
  if (J.d_out.reserve(ctx, cap) || J.d_dir.reserve(ctx, units) || J.h_dir.reserve(ctx, units) ||
      (!J.d_count && (J.d_count.alloc(ctx, 1) || J.h_count.alloc(ctx, 1))))
    return BTLE_ENOMEM;
  const int rc = launch_rx(ctx, H.d + Streams::kLead, s->n, s->stride, H.n_submitted, cfgs.data(), cc.data(), k,
                           rot.empty() ? nullptr : rot.data(), J.d_out, cap, J.d_count, J.d_dir, H.st, Streams::kLead);
  if (rc) return rc;
  BTLE_CUDA(ctx, cudaMemcpyAsync(J.h_count, J.d_count, sizeof(unsigned), cudaMemcpyDeviceToHost, H.st));
  BTLE_CUDA(ctx, cudaMemcpyAsync(J.h_dir, J.d_dir, units * sizeof(btle_unit_dir), cudaMemcpyDeviceToHost, H.st));
  J.index = idx;
  J.units = units;
  J.cap = cap;
  ++H.n_jobs;
  return BTLE_OK;
}

// Those of the cfgs `cand` that decode some chunk of half b's set, sorted by capture, in rounds of at most
// kMaxCfgsPerCapture per capture: one streams_job per round.  A capture no such cfg names is not read.  *launches counts
// the launches.
int streams_rounds(Streams *s, int b, const std::vector<size_t> &cand, int *launches) {
  auto &H = s->half[b];
  const long long lo = H.first_chunk, hi = lo + (long long)(H.n_submitted / kChunkInt8);
  std::vector<size_t> live;
  for (size_t j : cand)
    if (s->entries[j].from < hi && s->entries[j].until > lo) live.push_back(j);
  std::stable_sort(live.begin(), live.end(), [&](size_t x, size_t y) { return s->entries[x].capture < s->entries[y].capture; });
  for (size_t r = 0;; ++r) {
    std::vector<size_t> idx;
    for (size_t i = 0; i < live.size();) {                  // [i, e): the live cfgs of one capture
      size_t e = i;
      while (e < live.size() && s->entries[live[e]].capture == s->entries[live[i]].capture) ++e;
      for (size_t q = i + r * kMaxCfgsPerCapture; q < std::min(e, i + (r + 1) * kMaxCfgsPerCapture); ++q) idx.push_back(live[q]);
      i = e;
    }
    if (idx.empty()) return BTLE_OK;
    const int rc = streams_job(s, b, idx);
    if (rc) return rc;
    ++*launches;
  }
}

// discover_kernel over every scanned capture's part of half b: `bytes` bytes from the start of its lead.  One launch
// per run of adjacent scanned captures, each with its own counter and part of d_cand.
int streams_scan(Streams *s, int b, size_t bytes, size_t keep_samples, int *launches) {
  btle_b200_ctx *ctx = s->ctx;
  auto &H = s->half[b];
  H.scans.clear();
  size_t total = 0;
  for (size_t i = 0; i < s->n;) {
    if (s->disc[i] < 0) { ++i; continue; }
    size_t e = i + 1;
    while (e < s->n && s->disc[e] >= 0) ++e;
    Streams::Scan sc;
    sc.first = i; sc.count = e - i; sc.off = total; sc.cap = sc.count * (bytes / kChunkInt8 + 1) * 8 + 256;
    total += sc.cap;
    H.scans.push_back(sc);
    i = e;
  }
  if (H.scans.empty()) return BTLE_OK;
  H.scan_ch = s->disc;
  H.scan_bytes = bytes;
  H.scan_samples = keep_samples;
  if (H.d_cand.reserve(ctx, total) || H.d_ccount.reserve(ctx, H.scans.size()) || H.h_ccount.reserve(ctx, H.scans.size())) return BTLE_ENOMEM;
  for (size_t r = 0; r < H.scans.size(); ++r) {
    const Streams::Scan &sc = H.scans[r];
    const int rc = launch_discover(ctx, H.d + sc.first * s->stride, sc.count, s->stride, bytes, H.scan_ch.data() + sc.first,
                                   H.d_cand + sc.off, sc.cap, H.d_ccount + r, H.st);
    if (rc) return rc;
    BTLE_CUDA(ctx, cudaMemcpyAsync(H.h_ccount + r, H.d_ccount + r, sizeof(unsigned), cudaMemcpyDeviceToHost, H.st));
    ++*launches;
  }
  return BTLE_OK;
}

// decode the first n_int8 bytes of every capture's part of half b (bytes behind n_int8 read as 0); `last`: the end of the
// captures, so discovery keeps every window start of the n_int8 bytes instead of those of the segment
int streams_submit(Streams *s, int b, size_t n_int8, bool last = false) {
  btle_b200_ctx *ctx = s->ctx;
  auto &H = s->half[b];
  H.n_submitted = n_int8;
  H.first_chunk = s->next_chunk;
  H.offset = s->offset;
  const bool scan = std::any_of(s->disc.begin(), s->disc.end(), [](int32_t c) { return c >= 0; });
  if (n_int8 < (size_t)kChunkInt8 && !(scan && n_int8)) { H.resident = false; return BTLE_OK; }
  constexpr size_t L = btle_b200_streams::kLead;
  if (L + n_int8 == s->stride || s->n == 1)
    BTLE_CUDA(ctx, cudaMemcpyAsync(H.d, H.h, (s->n - 1) * s->stride + L + n_int8, cudaMemcpyHostToDevice, H.st));
  else
    BTLE_CUDA(ctx, cudaMemcpy2DAsync(H.d, s->stride, H.h, s->stride, L + n_int8, s->n, cudaMemcpyHostToDevice, H.st));
  H.resident = true;
  int &launches = s->call_launches, rc = BTLE_OK;
  if (n_int8 >= (size_t)kChunkInt8) {
    std::vector<size_t> all(s->entries.size());
    for (size_t j = 0; j < all.size(); ++j) all[j] = j;
    rc = streams_rounds(s, b, all, &launches);
    if (rc) return rc;
  }
  if (scan) {
    rc = streams_scan(s, b, L + n_int8, (last ? n_int8 : s->seg_bytes) / 2, &launches);
    if (rc) return rc;
  }
  return BTLE_OK;
}

// Backfill of the cfgs added since the last call (s->backfill): on each resident set that holds chunks at or behind their
// from_chunk, one streams_rounds pass over all of them (at most kMaxCfgsPerCapture per capture per launch), on that
// half's stream.  Runs at the start of the next commit / finish, before any set is collected or submitted, so the
// halves still hold the sets add_cfg saw.
int streams_backfill(Streams *s) {
  if (s->backfill.empty()) return BTLE_OK;
  std::vector<size_t> cand;
  cand.swap(s->backfill);
  for (int b = 0; b < 2; ++b) {
    const auto &H = s->half[b];
    if (!H.resident || H.n_submitted < (size_t)kChunkInt8) continue;
    const int rc = streams_rounds(s, b, cand, &s->call_launches);
    if (rc) return rc;
  }
  return BTLE_OK;
}
// the number of launches a commit / finish call made, when it made any
void streams_note_launches(Streams *s) {
  if (s->call_launches) s->ctx->last_launches = s->call_launches;
}

// the records of half b's jobs: stable cfg index in `stream`, stream-wide chunks, each cfg's [from, until) kept, in
// (cfg, chunk, n0) order, appended to s->ready.  A job gathers in (launch position, chunk, n0) order, which is already
// that order when positions map to ascending cfgs (always, while the cfg list is unchanged): only other orders are sorted.
int streams_collect_jobs(Streams *s, int b) {
  btle_b200_ctx *ctx = s->ctx;
  auto &H = s->half[b];
  size_t total = 0;
  for (size_t q = 0; q < H.n_jobs; ++q) {
    const Streams::Job &J = *H.jobs[q];
    if (*J.h_count > J.cap) { ctx->err = "stream segment produced more records than BTLE_MAX_RECS_PER_CHUNK allows"; return BTLE_EOVERFLOW; }
    total += *J.h_count;
  }
  const size_t n_jobs = H.n_jobs;
  H.n_jobs = 0;
  if (!total) return BTLE_OK;
  if (H.h_jrecs.reserve(ctx, total)) return BTLE_ENOMEM;
  for (size_t q = 0, at = 0; q < n_jobs; at += *H.jobs[q]->h_count, ++q)
    if (*H.jobs[q]->h_count)
      BTLE_CUDA(ctx, cudaMemcpyAsync(H.h_jrecs + at, H.jobs[q]->d_out, *H.jobs[q]->h_count * sizeof(btle_pkt_rec), cudaMemcpyDeviceToHost, H.st));
  BTLE_CUDA(ctx, cudaStreamSynchronize(H.st));
  const size_t at0 = s->ready.size();
  s->ready.resize(at0 + total);
  size_t end = at0;                                          // the records kept so far: s->ready[at0, end)
  for (size_t q = 0, at = 0; q < n_jobs; ++q) {
    const Streams::Job &J = *H.jobs[q];
    const size_t found = *J.h_count;
    btle_pkt_rec *got = s->ready.data() + end;               // filtered in place: a record is written at or before its slot
    size_t n_got = 0;
    btle_b200_gather_ordered(H.h_jrecs + at, found, J.h_dir, J.units, got, found, &n_got);
    for (size_t i = 0; i < found; ++i) {
      btle_pkt_rec r = got[i];
      const size_t j = J.index[(size_t)r.stream];
      const long long chunk = r.chunk + H.first_chunk;
      if (chunk < s->entries[j].from || chunk >= s->entries[j].until) continue;
      r.stream = (int32_t)j;
      r.chunk = (int32_t)chunk;
      s->ready[end++] = r;
    }
    at += found;
  }
  s->ready.resize(end);
  const auto by_cfg = [](const btle_pkt_rec &x, const btle_pkt_rec &y) { return x.stream < y.stream; };
  if (!std::is_sorted(s->ready.begin() + at0, s->ready.end(), by_cfg)) std::stable_sort(s->ready.begin() + at0, s->ready.end(), by_cfg);
  return BTLE_OK;
}

// the candidates of half b's discover launches: window starts inside the set's segment, stream-wide samples, capture
// index in `stream`, sorted by (stream, sample), appended to s->cands.  A launch whose buffer overflowed is run again
// on the still-resident set with room for all it found.
int streams_collect_scans(Streams *s, int b) {
  btle_b200_ctx *ctx = s->ctx;
  auto &H = s->half[b];
  if (H.scans.empty()) return BTLE_OK;
  std::vector<Streams::Scan> scans;
  scans.swap(H.scans);
  std::vector<size_t> found(scans.size());
  size_t total = 0;
  for (size_t r = 0; r < scans.size(); ++r) total += (found[r] = H.h_ccount[r]);
  if (H.h_cand.reserve(ctx, std::max<size_t>(total, 1))) return BTLE_ENOMEM;
  for (size_t r = 0, at = 0; r < scans.size(); at += found[r], ++r)
    if (found[r] && found[r] <= scans[r].cap)
      BTLE_CUDA(ctx, cudaMemcpyAsync(H.h_cand + at, H.d_cand + scans[r].off, found[r] * sizeof(btle_conn_cand), cudaMemcpyDeviceToHost, H.st));
  BTLE_CUDA(ctx, cudaStreamSynchronize(H.st));
  for (size_t r = 0, at = 0; r < scans.size(); at += found[r], ++r) {
    if (found[r] <= scans[r].cap) continue;
    if (H.d_cand.reserve(ctx, found[r])) return BTLE_ENOMEM;   // (the other launches' candidates are on the host already)
    const int rc = launch_discover(ctx, H.d + scans[r].first * s->stride, scans[r].count, s->stride, H.scan_bytes,
                                   H.scan_ch.data() + scans[r].first, H.d_cand, found[r], H.d_ccount, H.st);
    if (rc) return rc;
    BTLE_CUDA(ctx, cudaMemcpyAsync(H.h_cand + at, H.d_cand, found[r] * sizeof(btle_conn_cand), cudaMemcpyDeviceToHost, H.st));
    BTLE_CUDA(ctx, cudaStreamSynchronize(H.st));
  }
  const long long lead = (long long)(Streams::kLead / 2), base = H.first_chunk * (long long)(kChunkInt8 / 2) - lead;
  const size_t at0 = s->cands.size();
  for (size_t r = 0, at = 0; r < scans.size(); at += found[r], ++r)
    for (size_t i = at; i < at + found[r]; ++i) {
      btle_conn_cand c = H.h_cand[i];
      if (c.sample < lead || c.sample >= lead + (long long)H.scan_samples || base + c.sample < 32) continue;
      c.sample += base;
      c.stream += (int32_t)scans[r].first;
      s->cands.push_back(c);
    }
  std::sort(s->cands.begin() + at0, s->cands.end(), [](const btle_conn_cand &x, const btle_conn_cand &y) {
    return x.stream != y.stream ? x.stream < y.stream : x.sample < y.sample;
  });
  return BTLE_OK;
}

// wait for half b's launches; append its records ((stream, chunk, n0) order, stream-wide chunk numbers) to s->ready and
// its candidates to s->cands
int streams_collect(Streams *s, int b) {
  btle_b200_ctx *ctx = s->ctx;
  auto &H = s->half[b];
  if (!H.n_jobs && H.scans.empty()) return BTLE_OK;
  BTLE_CUDA(ctx, cudaStreamSynchronize(H.st));
  int rc = streams_collect_jobs(s, b);
  if (rc) return rc;
  return streams_collect_scans(s, b);
}
// first chunk of the oldest set whose IQ is still on the device (the next set's first chunk when none is)
long long streams_resident(const Streams *s) {
  long long r = s->next_chunk;
  for (const auto &H : s->half)
    if (H.resident) r = std::min(r, H.first_chunk);
  return r;
}
size_t streams_take(btle_b200_streams *s, btle_pkt_rec *out, size_t cap) {
  const size_t n = std::min(cap, s->ready.size() - s->ready_pos);
  if (n) memcpy(out, s->ready.data() + s->ready_pos, n * sizeof(btle_pkt_rec));
  s->ready_pos += n;
  if (s->ready_pos == s->ready.size()) { s->ready.clear(); s->ready_pos = 0; }
  return n;
}
int streams_index(btle_b200_streams *s, size_t stream) {
  if (stream < s->n) return BTLE_OK;
  s->ctx->err = "stream index out of range";
  return BTLE_EINVAL;
}
}  // namespace

extern "C" {

int btle_b200_streams_open(btle_b200_ctx *ctx, const btle_stream_cfg *cfgs, size_t n_streams, size_t segment_chunks,
                           btle_b200_streams **out) {
  if (!ctx || !out) return BTLE_EINVAL;
  *out = nullptr;
  if (n_streams == 0) { ctx->err = "streams_open: no captures"; return BTLE_EINVAL; }
  if (!cfgs) return BTLE_EINVAL;
  int rc = validate_cfgs(ctx, cfgs, n_streams);
  if (rc) return rc;
  // default: about 4096 chunks (64 MiB = 8.4 s of air of one capture) per half over all captures, so the footprint does
  // not grow with the number of captures; at least 16 chunks per capture
  if (segment_chunks == 0) segment_chunks = std::max<size_t>(16, (4096 / n_streams + 15) & ~size_t(15));
  if (segment_chunks > (1u << 20)) { ctx->err = "segment too large"; return BTLE_EINVAL; }
  BTLE_CUDA(ctx, cudaSetDevice(ctx->device));
  btle_b200_streams *s = new (std::nothrow) btle_b200_streams();
  if (!s) return BTLE_ENOMEM;
  s->ctx = ctx; s->n = n_streams; s->fill.assign(n_streams, 0);
  for (size_t i = 0; i < n_streams; ++i) s->entries.push_back({cfgs[i], i, 0, LLONG_MAX});
  s->disc.assign(n_streams, -1);
  s->seg_chunks = segment_chunks; s->seg_bytes = segment_chunks * (size_t)kChunkInt8;
  s->buf_bytes = s->seg_bytes + btle_b200_streams::kLook;
  s->stride = btle_b200_streams::kLead + s->buf_bytes;     // a multiple of 16, as the batched kernel needs
  // each half's first job and h_jrecs are sized for a round of one cfg per capture, so a session whose cfg list never
  // changes allocates nothing after this.  A short tail can be cut into more units than a full set (make_plan: down to
  // one chunk per unit, over whole 16-chunk spans), so the directory holds the most any such launch can have.
  const size_t cap = n_streams * segment_chunks * BTLE_MAX_RECS_PER_CHUNK;
  const size_t units = n_streams * ((segment_chunks + 15) & ~size_t(15));
  for (auto &H : s->half) {
    H.jobs.emplace_back(new (std::nothrow) Streams::Job());
    Streams::Job *J = H.jobs.back().get();
    if (!J || H.h.alloc(ctx, n_streams * s->stride) || H.d.alloc(ctx, n_streams * s->stride) || J->d_out.alloc(ctx, cap) ||
        J->d_dir.alloc(ctx, units) || J->d_count.alloc(ctx, 1) || J->h_count.alloc(ctx, 1) || J->h_dir.alloc(ctx, units) ||
        H.h_jrecs.alloc(ctx, cap) || cudaStreamCreateWithFlags(&H.st, cudaStreamNonBlocking) != cudaSuccess) {
      cudaGetLastError();
      ctx->err = "streams_open: allocation failed";
      btle_b200_streams_close(s);
      return BTLE_ENOMEM;
    }
    for (size_t i = 0; i < n_streams; ++i) memset(H.h + i * s->stride, 0, btle_b200_streams::kLead);   // nothing before the start
  }
  *out = s;
  return BTLE_OK;
}

void btle_b200_streams_close(btle_b200_streams *s) {
  if (!s) return;
  cudaSetDevice(s->ctx->device);
  for (auto &H : s->half)
    if (H.st) { cudaStreamSynchronize(H.st); cudaStreamDestroy(H.st); }
  delete s;                                                 // frees the halves' buffers
}

int btle_b200_streams_set_cfg(btle_b200_streams *s, size_t stream, const btle_stream_cfg *cfg) {
  if (!s || !cfg) return BTLE_EINVAL;
  int rc = streams_index(s, stream);
  if (rc) return rc;
  rc = validate_cfgs(s->ctx, cfg, 1);
  if (rc) return rc;
  s->entries[stream].cfg = *cfg;                            // used from the next submitted segment set on
  return BTLE_OK;
}

int btle_b200_streams_set_offset(btle_b200_streams *s, size_t capture, float offset_hz) {
  if (!s) return BTLE_EINVAL;
  int rc = streams_index(s, capture);
  if (rc) return rc;
  std::vector<int4> rot;
  if ((rc = make_rots(s->ctx, &offset_hz, 1, nullptr, 1, rot))) return rc;
  if (s->offset.empty()) s->offset.assign(s->n, 0.0f);    // from now on every set takes the rotated kernel
  s->offset[capture] = offset_hz;                           // used from the next submitted segment set on
  return BTLE_OK;
}

int btle_b200_streams_acquire(btle_b200_streams *s, size_t stream, int8_t **buf, size_t *space) {
  if (!s || !buf || !space) return BTLE_EINVAL;
  const int rc = streams_index(s, stream);
  if (rc) return rc;
  auto &H = s->half[s->cur];
  *buf = H.h + stream * s->stride + btle_b200_streams::kLead + s->fill[stream];
  *space = s->buf_bytes - s->fill[stream];                  // 0: this capture's part is complete, the others are behind
  return BTLE_OK;
}

int btle_b200_streams_commit(btle_b200_streams *s, size_t stream, size_t n_int8, btle_pkt_rec *out, size_t cap, size_t *n_out) {
  if (!s || !n_out || (!out && cap)) return BTLE_EINVAL;
  *n_out = 0;
  int rc = streams_index(s, stream);
  if (rc) return rc;
  if (n_int8 > s->buf_bytes - s->fill[stream]) { s->ctx->err = "stream_commit: more bytes than acquired"; return BTLE_EINVAL; }
  BTLE_CUDA(s->ctx, cudaSetDevice(s->ctx->device));
  s->call_launches = 0;
  rc = streams_backfill(s);
  if (rc) return rc;
  rc = streams_collect(s, s->cur);                          // backfill launches on the set the filling half still holds
  if (rc) return rc;
  s->fill[stream] += n_int8;
  if (n_int8 && s->fill[stream] == s->buf_bytes) ++s->n_full;
  if (s->n_full == s->n) {                                  // every part + look-ahead complete: hand the set to the GPU
    const int b = s->cur, o = b ^ 1;
    rc = streams_collect(s, o);                             // the other half's previous set must be done before its buffers are reused
    if (rc) return rc;
    rc = streams_submit(s, b, s->buf_bytes);
    if (rc) return rc;
    // the look-ahead bytes are the beginning of the next set, the bytes in front of them its lead
    for (size_t i = 0; i < s->n; ++i) {
      memcpy(s->half[o].h + i * s->stride, s->half[b].h + i * s->stride + s->seg_bytes,
             btle_b200_streams::kLead + btle_b200_streams::kLook);
      s->fill[i] = btle_b200_streams::kLook;
    }
    s->n_full = 0;
    s->next_chunk += (long long)s->seg_chunks;
    s->cur = o;
  }
  streams_note_launches(s);
  *n_out = streams_take(s, out, cap);
  return BTLE_OK;
}

int btle_b200_streams_finish(btle_b200_streams *s, btle_pkt_rec *out, size_t cap, size_t *n_out) {
  if (!s || !n_out || (!out && cap)) return BTLE_EINVAL;
  *n_out = 0;
  BTLE_CUDA(s->ctx, cudaSetDevice(s->ctx->device));
  const int b = s->cur, o = b ^ 1;
  s->call_launches = 0;
  int rc = streams_backfill(s);
  if (rc) return rc;
  rc = streams_collect(s, b);                               // backfill launches
  if (rc) return rc;
  rc = streams_collect(s, o);
  if (rc) return rc;
  // the tail: complete chunks of the SHORTEST capture; behind that length every capture reads as 0 (rx_batch's common n_int8)
  const size_t n_int8 = *std::min_element(s->fill.begin(), s->fill.end());
  const bool scan = std::any_of(s->disc.begin(), s->disc.end(), [](int32_t c) { return c >= 0; });
  if (n_int8 >= (size_t)kChunkInt8 || (scan && n_int8)) {   // (discovery reads the windows of a tail shorter than a chunk)
    rc = streams_submit(s, b, n_int8, true);
    if (rc) return rc;
    rc = streams_collect(s, b);
    if (rc) return rc;
    s->next_chunk += (long long)(n_int8 / kChunkInt8);
  }
  std::fill(s->fill.begin(), s->fill.end(), size_t(0));
  s->n_full = 0;
  streams_note_launches(s);
  *n_out = streams_take(s, out, cap);
  return (s->ready.size() > s->ready_pos) ? BTLE_EOVERFLOW : BTLE_OK;   // call again with more room
}

int btle_b200_streams_resident(const btle_b200_streams *s, int64_t *first_chunk) {
  if (!s || !first_chunk) return BTLE_EINVAL;
  *first_chunk = streams_resident(s);
  return BTLE_OK;
}

int btle_b200_streams_add_cfg(btle_b200_streams *s, size_t capture, const btle_stream_cfg *cfg, int64_t from_chunk, size_t *index) {
  if (!s || !cfg || !index) return BTLE_EINVAL;
  int rc = streams_index(s, capture);
  if (rc) return rc;
  rc = validate_cfgs(s->ctx, cfg, 1);
  if (rc) return rc;
  if (from_chunk < streams_resident(s)) {
    s->ctx->err = "streams_add_cfg: from_chunk lies before the first resident chunk (btle_b200_streams_resident)";
    return BTLE_EINVAL;
  }
  // backfill over the resident sets is enqueued by the next commit / finish, batched with every cfg added until then
  const size_t j = s->entries.size();
  s->entries.push_back({*cfg, capture, (long long)from_chunk, LLONG_MAX});
  s->backfill.push_back(j);
  *index = j;
  return BTLE_OK;
}

int btle_b200_streams_remove_cfg(btle_b200_streams *s, size_t index, int64_t *until_chunk) {
  if (!s || !until_chunk) return BTLE_EINVAL;
  if (index >= s->entries.size()) { s->ctx->err = "streams_remove_cfg: cfg index out of range"; return BTLE_EINVAL; }
  auto &e = s->entries[index];
  if (e.until != LLONG_MAX) { s->ctx->err = "streams_remove_cfg: cfg already removed"; return BTLE_EINVAL; }
  e.until = std::max(e.from, s->next_chunk);                // the next submitted set starts at next_chunk
  *until_chunk = e.until;
  return BTLE_OK;
}

int btle_b200_streams_set_discover(btle_b200_streams *s, const int32_t *channels) {
  if (!s || !channels) return BTLE_EINVAL;
  for (size_t i = 0; i < s->n; ++i)
    if (channels[i] < -1 || channels[i] > 36) { s->ctx->err = "streams_set_discover: data channel must be within 0~36 or -1"; return BTLE_EINVAL; }
  s->disc.assign(channels, channels + s->n);
  return BTLE_OK;
}

int btle_b200_streams_take_cands(btle_b200_streams *s, btle_conn_cand *out, size_t cap, size_t *n_out) {
  if (!s || !n_out || (!out && cap)) return BTLE_EINVAL;
  const size_t n = std::min(cap, s->cands.size());
  if (n) memcpy(out, s->cands.data(), n * sizeof(btle_conn_cand));
  s->cands.erase(s->cands.begin(), s->cands.begin() + n);
  *n_out = n;
  return s->cands.empty() ? BTLE_OK : BTLE_EOVERFLOW;       // call again with more room
}

// ---- single capture: a one-capture session ----
int btle_b200_stream_open(btle_b200_ctx *ctx, const btle_stream_cfg *cfg, size_t segment_chunks, btle_b200_stream **out) {
  if (!ctx || !cfg || !out) return BTLE_EINVAL;
  *out = nullptr;
  btle_b200_stream *w = new (std::nothrow) btle_b200_stream();
  if (!w) return BTLE_ENOMEM;
  const int rc = btle_b200_streams_open(ctx, cfg, 1, segment_chunks, &w->m);
  if (rc) { delete w; return rc; }
  *out = w;
  return BTLE_OK;
}

void btle_b200_stream_close(btle_b200_stream *s) {
  if (!s) return;
  btle_b200_streams_close(s->m);
  delete s;
}

int btle_b200_stream_set_cfg(btle_b200_stream *s, const btle_stream_cfg *cfg) {
  return s ? btle_b200_streams_set_cfg(s->m, 0, cfg) : BTLE_EINVAL;
}

int btle_b200_stream_set_offset(btle_b200_stream *s, float offset_hz) {
  return s ? btle_b200_streams_set_offset(s->m, 0, offset_hz) : BTLE_EINVAL;
}

int btle_b200_stream_acquire(btle_b200_stream *s, int8_t **buf, size_t *space) {
  return s ? btle_b200_streams_acquire(s->m, 0, buf, space) : BTLE_EINVAL;
}

int btle_b200_stream_commit(btle_b200_stream *s, size_t n_int8, btle_pkt_rec *out, size_t cap, size_t *n_out) {
  return s ? btle_b200_streams_commit(s->m, 0, n_int8, out, cap, n_out) : BTLE_EINVAL;
}

int btle_b200_stream_push(btle_b200_stream *s, const int8_t *iq, size_t n_int8, btle_pkt_rec *out, size_t cap, size_t *n_out) {
  if (!s || (!iq && n_int8) || !n_out || (!out && cap)) return BTLE_EINVAL;
  *n_out = 0;
  size_t done = 0;
  while (done < n_int8) {
    int8_t *buf; size_t space;
    btle_b200_stream_acquire(s, &buf, &space);
    const size_t n = std::min(space, n_int8 - done);
    memcpy(buf, iq + done, n);
    done += n;
    size_t got = 0;
    const int rc = btle_b200_stream_commit(s, n, out + *n_out, cap - *n_out, &got);
    *n_out += got;
    if (rc) return rc;
  }
  return BTLE_OK;
}

int btle_b200_stream_finish(btle_b200_stream *s, btle_pkt_rec *out, size_t cap, size_t *n_out) {
  return s ? btle_b200_streams_finish(s->m, out, cap, n_out) : BTLE_EINVAL;
}

// ---- leaf functions ------------------------------------------------------------------------------
int btle_b200_dbits(btle_b200_ctx *ctx, const int8_t *iq, size_t n_samples, uint8_t *d_out) {
  if (!ctx || !iq || !d_out) return BTLE_EINVAL;
  if (n_samples == 0) return BTLE_OK;
  BTLE_CUDA(ctx, cudaSetDevice(ctx->device));
  const size_t in_bytes = 2 * n_samples + 2;
  int8_t *d_in;
  uint8_t *d_d;
  const int rc = leaf_layout(ctx, piece(d_in, in_bytes), piece(d_d, n_samples));
  if (rc) return rc;
  BTLE_CUDA(ctx, cudaMemcpyAsync(d_in, iq, in_bytes, cudaMemcpyHostToDevice, ctx->stream));
  dbits_kernel<<<(unsigned)((n_samples + 255) / 256), 256, 0, ctx->stream>>>(d_in, (long long)n_samples, d_d);
  return leaf_result(ctx, d_out, d_d, n_samples);
}

// body of btle_b200_search_unique_bits: a BTLE_* code, the hit (or -1) in *res
static int search_unique_bits(btle_b200_ctx *ctx, const int8_t *rxp, int search_len, const btle_stream_cfg &cfg, int *res) {
  BTLE_CUDA(ctx, cudaSetDevice(ctx->device));
  const size_t valid = 8 * (size_t)search_len + 2;          // int8 the reference reads (:1528-1529)
  const int ngroups = (int)((4 * (size_t)search_len + 127) / 128);
  const size_t in_bytes = ((size_t)ngroups + 1) * 256;      // ngroups * 128 samples + the carry word, zero behind `valid`
  int8_t *d_in;
  uint32_t *d_pd, *d_cand;
  int *d_res;
  const int rc = leaf_layout(ctx, piece(d_in, in_bytes), piece(d_pd, 4 * ((size_t)ngroups + 1)), piece(d_cand, (size_t)ngroups + 1),
                             piece(d_res, 1));
  if (rc) return rc;
  BTLE_CUDA(ctx, cudaMemsetAsync(d_in, 0, in_bytes, ctx->stream));
  BTLE_CUDA(ctx, cudaMemcpyAsync(d_in, rxp, valid, cudaMemcpyHostToDevice, ctx->stream));
  search_kernel<<<1, 128, 0, ctx->stream>>>(d_in, search_len, cfg, ngroups, d_pd, d_cand, d_res);
  return leaf_result(ctx, res, d_res, sizeof(int));
}

int btle_b200_search_unique_bits(btle_b200_ctx *ctx, const int8_t *rxp, int search_len, const uint8_t *unique_bits,
                                 const uint8_t *unique_bits_mask, int num_bits) {
  // hits are even values >= -248 and -1 means "none" (btle_rx.c:1550/:1561): errors are reported as
  // BTLE_SEARCH_ERR(code) = code - 1000 so that no error can be mistaken for a result
  if (!ctx || !rxp || !unique_bits || !unique_bits_mask || num_bits != 32 || search_len < 0 || search_len > 4096)
    return BTLE_SEARCH_ERR(BTLE_EINVAL);      // the reference only ever passes LEN_DEMOD_BUF_ACCESS = 32
  if (search_len == 0) return -1;
  btle_stream_cfg cfg{};
  cfg.channel = 37;
  for (int p = 0; p < 32; ++p) {
    // the reference compares a demodulated 0/1 with unique_bits[p] (:1539): a masked value other than 0 or 1 never matches
    if (unique_bits_mask[p] && unique_bits[p] > 1) return -1;
    cfg.access_addr |= (uint32_t)(unique_bits[p] & 1u) << p;
    cfg.access_mask |= (uint32_t)(unique_bits_mask[p] ? 1u : 0u) << p;
  }
  int res = -1;
  const int rc = search_unique_bits(ctx, rxp, search_len, cfg, &res);
  return rc ? BTLE_SEARCH_ERR(rc) : res;
}

int btle_b200_demod_byte(btle_b200_ctx *ctx, const int8_t *rxp, int num_byte, uint8_t *out_byte) {
  if (!ctx || !rxp || !out_byte || num_byte < 0 || num_byte > 64) return BTLE_EINVAL;
  if (num_byte == 0) return BTLE_OK;
  BTLE_CUDA(ctx, cudaSetDevice(ctx->device));
  const size_t in_bytes = 64 * (size_t)num_byte - 4;       // last read index: 8*(8n-1)+3
  int8_t *d_in;
  uint8_t *d_o;
  const int rc = leaf_layout(ctx, piece(d_in, in_bytes), piece(d_o, num_byte));
  if (rc) return rc;
  BTLE_CUDA(ctx, cudaMemcpyAsync(d_in, rxp, in_bytes, cudaMemcpyHostToDevice, ctx->stream));
  demod_byte_kernel<<<1, 64, 0, ctx->stream>>>(d_in, num_byte, d_o);
  return leaf_result(ctx, out_byte, d_o, num_byte);
}

int btle_b200_scramble_byte(btle_b200_ctx *ctx, const uint8_t *byte_in, int num_byte, int channel, int table_offset,
                            uint8_t *byte_out) {
  if (!ctx || !byte_in || !byte_out || num_byte < 0 || channel < 0 || channel > 39 || table_offset < 0 ||
      table_offset + num_byte > 42)
    return BTLE_EINVAL;
  if (num_byte == 0) return BTLE_OK;
  BTLE_CUDA(ctx, cudaSetDevice(ctx->device));
  uint8_t *d_in, *d_o;
  const int rc = leaf_layout(ctx, piece(d_in, num_byte), piece(d_o, num_byte));
  if (rc) return rc;
  BTLE_CUDA(ctx, cudaMemcpyAsync(d_in, byte_in, num_byte, cudaMemcpyHostToDevice, ctx->stream));
  scramble_kernel<<<1, 64, 0, ctx->stream>>>(d_in, num_byte, channel, table_offset, d_o);
  return leaf_result(ctx, byte_out, d_o, num_byte);
}

int btle_b200_crc24_byte(btle_b200_ctx *ctx, const uint8_t *byte_in, int num_byte, uint32_t init_hex, uint32_t *crc_out) {
  if (!ctx || (!byte_in && num_byte) || !crc_out || num_byte < 0 || num_byte > 4096) return BTLE_EINVAL;
  BTLE_CUDA(ctx, cudaSetDevice(ctx->device));
  uint8_t *d_in;
  uint32_t *d_o;
  const int rc = leaf_layout(ctx, piece(d_in, num_byte), piece(d_o, 1));
  if (rc) return rc;
  if (num_byte) BTLE_CUDA(ctx, cudaMemcpyAsync(d_in, byte_in, num_byte, cudaMemcpyHostToDevice, ctx->stream));
  crc24_kernel<<<1, 1, 0, ctx->stream>>>(d_in, num_byte, init_hex, d_o);
  return leaf_result(ctx, crc_out, d_o, sizeof(uint32_t));
}

uint32_t btle_b200_crc_init_reorder(uint32_t crc_init) { return crc_init_reorder(crc_init); }

int btle_b200_tx_modulate_device(btle_b200_ctx *ctx, const uint8_t *d_air, const int32_t *d_nbytes, size_t n_packets,
                                 size_t max_bytes, int sps, int8_t *d_out_i, int8_t *d_out_q, void *cuda_stream) {
  if (!ctx || !d_air || !d_nbytes || !d_out_i || (sps != 4 && sps != 8) || (sps == 8 && !d_out_q) || max_bytes == 0 ||
      max_bytes > 128 || n_packets > 0x7FFFFFFFu)
    return BTLE_EINVAL;
  if (n_packets == 0) return BTLE_OK;
  BTLE_CUDA(ctx, cudaSetDevice(ctx->device));
  cudaStream_t st = reinterpret_cast<cudaStream_t>(cuda_stream);
  if (sps == 4) tx_modulate_kernel<4><<<(unsigned)n_packets, 256, 0, st>>>(d_air, d_nbytes, (int)max_bytes, d_out_i, d_out_q);
  else tx_modulate_kernel<8><<<(unsigned)n_packets, 512, 0, st>>>(d_air, d_nbytes, (int)max_bytes, d_out_i, d_out_q);
  BTLE_CUDA(ctx, cudaGetLastError());
  return BTLE_OK;
}

int btle_b200_synth_streams_device(btle_b200_ctx *ctx, int8_t *d_iq, size_t n_streams, size_t stride, size_t n_int8,
                                   const btle_stream_cfg *cfgs, const btle_synth_cfg *sc, btle_synth_truth *d_truth,
                                   size_t truth_cap, size_t *n_slots_out, void *cuda_stream) {
  if (!ctx || !d_iq || !cfgs || !sc || n_streams == 0 || (n_streams > 1 && stride < n_int8)) return BTLE_EINVAL;
  if (sc->slot_samples < 1600 || sc->amplitude < 0 || sc->amplitude > 127 || sc->noise < 0 || sc->noise > 2 || sc->corrupt_every < 0 ||
      sc->straddle_every < 0 || (sc->straddle_every > 0 && (sc->straddle_every < 2 || sc->slot_samples < 3200))) {
    ctx->err = "synth: slot_samples >= 1600 (>= 3200 and straddle_every >= 2 with straddling), amplitude 0..127, noise 0..2";
    return BTLE_EINVAL;
  }
  int rc = validate_cfgs(ctx, cfgs, n_streams);
  if (rc) return rc;
  const size_t n_slots = (n_int8 / 2) / (size_t)sc->slot_samples;
  if (n_slots_out) *n_slots_out = n_slots;
  if (d_truth && truth_cap < n_slots * n_streams) { ctx->err = "synth: truth buffer too small"; return BTLE_EINVAL; }
  if (n_slots * n_streams > 0x7FFFFFFFull) { ctx->err = "synth: too many slots for one launch"; return BTLE_EINVAL; }
  BTLE_CUDA(ctx, cudaSetDevice(ctx->device));
  cudaStream_t st = reinterpret_cast<cudaStream_t>(cuda_stream);
  unsigned long long sid = 0;
  rc = stream_id(ctx, st, &sid);
  if (rc) return rc;
  CfgSlot *cs = nullptr;
  rc = upload_cfgs(ctx, cfgs, n_streams, st, sid, &cs);
  if (rc) return rc;
  synth_noise_kernel<<<ctx->num_sms * 8, 256, 0, st>>>(d_iq, (long long)stride, (long long)n_int8, (int)n_streams, sc->seed, sc->noise);
  BTLE_CUDA(ctx, cudaGetLastError());
  if (n_slots && sc->amplitude > 0) {
    synth_bursts_kernel<<<(unsigned)(n_slots * n_streams), 256, 0, st>>>(d_iq, (long long)stride, (long long)n_int8, cs->d, *sc,
                                                                          (long long)n_slots, d_truth);
    BTLE_CUDA(ctx, cudaGetLastError());
  }
  return note_use(ctx, cs, st, sid);
}

int btle_b200_model_rx_batch_device(btle_b200_ctx *ctx, const int16_t *d_i, const int16_t *d_q, size_t n_packets,
                                    size_t n_samples, int sps, int channel, uint32_t crc_init, uint32_t access_addr,
                                    btle_model_rx_rec *d_out, void *cuda_stream) {
  if (!ctx || !d_i || !d_q || !d_out || sps < 1 || sps > 64 || channel < 0 || channel > 39 || n_samples % (size_t)sps ||
      n_samples / (size_t)sps < 34 || n_samples / (size_t)sps > 32u * kModelMaxWords || n_packets > 0x7FFFFFFFu / 4 * 4)
    return BTLE_EINVAL;
  if (n_packets == 0) return BTLE_OK;
  BTLE_CUDA(ctx, cudaSetDevice(ctx->device));
  const int adv = (channel >= 37 && channel <= 39);
  model_rx_batch_kernel<<<(unsigned)((n_packets + 3) / 4), 128, 0, reinterpret_cast<cudaStream_t>(cuda_stream)>>>(
      d_i, d_q, 1, nullptr, (int)n_packets, (int)n_samples, sps, adv, channel, access_addr, crc_init_reorder(crc_init), d_out);
  BTLE_CUDA(ctx, cudaGetLastError());
  return BTLE_OK;
}

int btle_b200_model_rx_batch(btle_b200_ctx *ctx, const int16_t *i, const int16_t *q, size_t n_packets, size_t n_samples,
                             int sps, int channel, uint32_t crc_init, uint32_t access_addr, btle_model_rx_rec *out) {
  if (!ctx || !i || !q || !out) return BTLE_EINVAL;
  if (n_packets == 0) return BTLE_OK;
  BTLE_CUDA(ctx, cudaSetDevice(ctx->device));
  const size_t nb = n_packets * n_samples * 2;
  int16_t *d_i, *d_q;
  btle_model_rx_rec *d_o;
  int rc = leaf_layout(ctx, piece(d_i, n_packets * n_samples), piece(d_q, n_packets * n_samples), piece(d_o, n_packets));
  if (rc) return rc;
  BTLE_CUDA(ctx, cudaMemcpyAsync(d_i, i, nb, cudaMemcpyHostToDevice, ctx->stream));
  BTLE_CUDA(ctx, cudaMemcpyAsync(d_q, q, nb, cudaMemcpyHostToDevice, ctx->stream));
  rc = btle_b200_model_rx_batch_device(ctx, d_i, d_q, n_packets, n_samples, sps, channel, crc_init, access_addr, d_o, ctx->stream);
  if (rc) return rc;
  BTLE_CUDA(ctx, cudaMemcpyAsync(out, d_o, n_packets * sizeof(btle_model_rx_rec), cudaMemcpyDeviceToHost, ctx->stream));
  BTLE_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  return BTLE_OK;
}

int btle_b200_sps8_hits_device(btle_b200_ctx *ctx, const int16_t *d_iq16, size_t n_samples, uint32_t access_addr, int64_t *d_hits, size_t cap,
                               uint32_t *d_count, void *cuda_stream) {
  if (!ctx || !d_iq16 || !d_count || (!d_hits && cap)) return BTLE_EINVAL;
  if (reinterpret_cast<uintptr_t>(d_iq16) & 15) {          // sps8_hits_kernel copies the capture in 16-byte vectors
    ctx->err = "sps8_hits_device: the capture must be 16-byte aligned";
    return BTLE_EINVAL;
  }
  BTLE_CUDA(ctx, cudaSetDevice(ctx->device));
  cudaStream_t st = reinterpret_cast<cudaStream_t>(cuda_stream);
  BTLE_CUDA(ctx, cudaMemsetAsync(d_count, 0, sizeof(unsigned), st));
  if (!n_samples) return BTLE_OK;
  const int rc = launch_sps8_hits(ctx, d_iq16, n_samples, access_addr, reinterpret_cast<long long *>(d_hits), std::min<size_t>(cap, 0xFFFFFFFFu), d_count, st);
  if (rc) return rc;
  ctx->last_launches = 1;
  return BTLE_OK;
}

int btle_b200_discover_device(btle_b200_ctx *ctx, const int8_t *d_iq, size_t n_streams, size_t stride, size_t n_int8,
                              const int32_t *channels, btle_conn_cand *d_out, size_t cap, uint32_t *d_count, void *cuda_stream) {
  if (!ctx) return BTLE_EINVAL;
  return launch_discover(ctx, d_iq, n_streams, stride, n_int8, channels, d_out, cap, d_count, reinterpret_cast<cudaStream_t>(cuda_stream));
}

int btle_b200_discover(btle_b200_ctx *ctx, const int8_t *iq, size_t n_streams, size_t stride, size_t n_int8, const int32_t *channels,
                       btle_conn_cand *out, size_t cap, size_t *n_out) {
  if (!ctx) return BTLE_EINVAL;
  if (!n_out || (!out && cap) || (!iq && n_streams && n_int8)) { ctx->err = "discover: missing buffer"; return BTLE_EINVAL; }
  *n_out = 0;
  int rc = check_data_channels(ctx, channels, n_streams);                  // before any byte is copied
  if (rc) return rc;
  BTLE_CUDA(ctx, cudaSetDevice(ctx->device));
  cudaStream_t st = ctx->stream;
  size_t pitch = 0;
  rc = ingest(ctx, iq, n_streams, stride, n_int8, nullptr, n_streams, &pitch);
  if (rc) return rc;
  rc = ctx->d_cand.reserve(ctx, std::max<size_t>(cap, 1));
  if (rc) return rc;
  rc = launch_discover(ctx, ctx->d_iq, n_streams, pitch, n_int8, channels, ctx->d_cand, cap, ctx->d_count, st);
  if (rc) return rc;
  rc = fetch_counted(ctx, st, cap, n_out, [&](size_t n) {
    BTLE_CUDA(ctx, cudaMemcpyAsync(out, ctx->d_cand, n * sizeof(btle_conn_cand), cudaMemcpyDeviceToHost, st));
    return BTLE_OK;
  });
  if (rc) return rc;
  std::sort(out, out + std::min(*n_out, cap), [](const btle_conn_cand &a, const btle_conn_cand &b) {
    return a.stream != b.stream ? a.stream < b.stream : a.sample < b.sample;
  });
  if (*n_out > cap) { ctx->err = "output capacity too small"; return BTLE_EOVERFLOW; }
  return BTLE_OK;
}

// Streaming form of the Python model's receiver over an 8-Msps interleaved int16 capture (see include/btle_b200.h).
int btle_b200_rx_sps8(btle_b200_ctx *ctx, const int16_t *iq16, size_t n_samples, int channel, uint32_t crc_init, uint32_t access_addr,
                      btle_sps8_rec *out, size_t cap, size_t *n_out) {
  if (!ctx || (!iq16 && n_samples) || !n_out || (!out && cap) || channel < 0 || channel > 39) return BTLE_EINVAL;
  *n_out = 0;
  if (n_samples < (size_t)BTLE_SPS8_WINDOW) return BTLE_OK;
  BTLE_CUDA(ctx, cudaSetDevice(ctx->device));
  cudaStream_t st = ctx->stream;
  const size_t bytes = n_samples * 4, hit_cap = n_samples / 256 + 4096;
  int rc = ctx->d_iq.reserve(ctx, bytes + 256);
  if (rc) return rc;
  long long *d_hits;
  rc = leaf_layout(ctx, piece(d_hits, hit_cap));
  if (rc) return rc;
  const int16_t *d_iq = reinterpret_cast<const int16_t *>(ctx->d_iq.p);
  rc = h2d_rows(ctx, ctx->d_iq, bytes, reinterpret_cast<const int8_t *>(iq16), bytes, bytes, 1, st);
  if (rc) return rc;
  BTLE_CUDA(ctx, cudaMemsetAsync(ctx->d_count, 0, sizeof(unsigned), st));
  rc = launch_sps8_hits(ctx, d_iq, n_samples, access_addr, d_hits, hit_cap, ctx->d_count, st);
  if (rc) return rc;
  ctx->last_launches = 1;
  size_t n_hits = 0;
  std::vector<long long> hits;
  rc = fetch_counted(ctx, st, hit_cap, &n_hits, [&](size_t n) {
    if (n_hits > hit_cap) { ctx->err = "rx_sps8: more access-address hits than the hit buffer holds"; return BTLE_EOVERFLOW; }
    hits.resize(n);
    BTLE_CUDA(ctx, cudaMemcpyAsync(hits.data(), d_hits, n * 8, cudaMemcpyDeviceToHost, st));
    return BTLE_OK;
  });
  if (rc) return rc;
  if (hits.empty()) return BTLE_OK;
  std::sort(hits.begin(), hits.end());
  // candidates: the first hit of every cluster (hits closer than the shortest possible packet belong to one packet: the same
  // access address seen on neighbouring sample phases), with its window
  std::vector<long long> cand, win;
  long long last = -(1ll << 60);
  for (long long h : hits) {
    if (h < last + 8ll * BTLE_SPS8_MIN_PACKET_SYMBOLS) continue;
    last = h;
    long long w0 = 8 * (h / 8 - BTLE_SPS8_MARGIN_SYMBOLS);
    if (w0 < 0) w0 = 0;
    if (w0 + BTLE_SPS8_WINDOW > (long long)n_samples) continue;             // the window must lie inside the capture
    cand.push_back(h);
    win.push_back(w0);
  }
  if (cand.empty()) return BTLE_OK;
  const size_t nc = cand.size();
  long long *d_win;                                         // the hits are consumed: windows and records take their place
  btle_model_rx_rec *d_rec;
  rc = leaf_layout(ctx, piece(d_win, nc), piece(d_rec, nc));
  if (rc) return rc;
  BTLE_CUDA(ctx, cudaMemcpyAsync(d_win, win.data(), nc * 8, cudaMemcpyHostToDevice, st));
  const int adv = (channel >= 37 && channel <= 39);
  model_rx_batch_kernel<<<(unsigned)((nc + 3) / 4), 128, 0, st>>>(d_iq, d_iq + 1, 2, d_win, (int)nc, BTLE_SPS8_WINDOW, 8, adv, channel, access_addr,
                                                                  crc_init_reorder(crc_init), d_rec);
  BTLE_CUDA(ctx, cudaGetLastError());
  std::vector<btle_model_rx_rec> recs(nc);
  BTLE_CUDA(ctx, cudaMemcpyAsync(recs.data(), d_rec, nc * sizeof(btle_model_rx_rec), cudaMemcpyDeviceToHost, st));
  BTLE_CUDA(ctx, cudaStreamSynchronize(st));
  ctx->last_launches = 2;
  // greedy: a candidate inside the packet accepted before it is part of that packet
  long long cursor = -1;
  size_t n = 0;
  for (size_t k = 0; k < nc; ++k) {
    if (cand[k] < cursor) continue;
    const btle_model_rx_rec &r = recs[k];
    long long at = cand[k];
    if (r.found) at = win[k] + 8ll * r.start + (r.crc_ok ? r.phase : r.found - 1);
    const int plen = r.found ? r.payload_len : 0;
    cursor = at + 8ll * (32 + 16 + 8 * plen + 24);
    if (n < cap) { out[n].sample = at; out[n].window = win[k]; out[n].rx = r; }
    ++n;
  }
  *n_out = n;
  if (n > cap) { ctx->err = "output capacity too small"; return BTLE_EOVERFLOW; }
  return BTLE_OK;
}

// ber_synth_kernel reads sample (int)(m * (1 + ppm 1e-6)) of its packet: ppm must be finite and above -1e6 (the
// reference's script uses -50..50), and the SNR must be a number
static int check_ber_cfg(btle_b200_ctx *ctx, const btle_ber_cfg *cfg) {
  if (cfg->channel < 0 || cfg->channel > 39) { ctx->err = "ber: channel must be 0..39"; return BTLE_EINVAL; }
  if (!std::isfinite(cfg->ppm) || std::fabs(cfg->ppm) >= 1e6f) { ctx->err = "ber: ppm must be finite with |ppm| < 1e6"; return BTLE_EINVAL; }
  if (std::isnan(cfg->snr_db)) { ctx->err = "ber: snr_db is NaN"; return BTLE_EINVAL; }
  return BTLE_OK;
}

int btle_b200_ber_run(btle_b200_ctx *ctx, const btle_ber_cfg *cfg, size_t n_packets, btle_ber_result *out) {
  if (!ctx || !cfg || !out) return BTLE_EINVAL;
  memset(out, 0, sizeof *out);
  int rc = check_ber_cfg(ctx, cfg);
  if (rc) return rc;
  if (!n_packets) return BTLE_OK;
  BTLE_CUDA(ctx, cudaSetDevice(ctx->device));
  cudaStream_t st = ctx->stream;
  const size_t B = std::min<size_t>(n_packets, 32768);
  int16_t *d_i, *d_q;
  uint8_t *d_truth;
  btle_model_rx_rec *d_rec;
  unsigned long long *d_acc;
  rc = leaf_layout(ctx, piece(d_i, B * kBerSamples), piece(d_q, B * kBerSamples), piece(d_truth, B * 40), piece(d_rec, B), piece(d_acc, 3));
  if (rc) return rc;
  BTLE_CUDA(ctx, cudaMemsetAsync(d_acc, 0, 3 * sizeof(unsigned long long), st));
  struct Timing {                                           // the two events are destroyed on every return
    cudaEvent_t e0 = nullptr, e1 = nullptr;
    ~Timing() { if (e0) cudaEventDestroy(e0); if (e1) cudaEventDestroy(e1); }
  } t;
  BTLE_CUDA(ctx, cudaEventCreate(&t.e0));
  BTLE_CUDA(ctx, cudaEventCreate(&t.e1));
  BTLE_CUDA(ctx, cudaEventRecord(t.e0, st));
  const int adv = (cfg->channel >= 37);
  int launches = 0;
  for (size_t done = 0; done < n_packets; done += B) {
    const int n = (int)std::min(B, n_packets - done);
    ber_synth_kernel<<<n, 384, 0, st>>>(*cfg, (unsigned long long)done, n, d_i, d_q, d_truth);
    model_rx_batch_kernel<<<(n + 3) / 4, 128, 0, st>>>(d_i, d_q, 1, nullptr, n, kBerSamples, 8, adv, cfg->channel, cfg->access_addr,
                                                      crc_init_reorder(cfg->crc_init), d_rec);
    ber_score_kernel<<<(n + 255) / 256, 256, 0, st>>>(d_rec, d_truth, n, d_acc);
    launches += 3;
  }
  BTLE_CUDA(ctx, cudaGetLastError());
  BTLE_CUDA(ctx, cudaEventRecord(t.e1, st));
  unsigned long long acc[3];
  BTLE_CUDA(ctx, cudaMemcpyAsync(acc, d_acc, sizeof acc, cudaMemcpyDeviceToHost, st));
  BTLE_CUDA(ctx, cudaStreamSynchronize(st));
  float ms = 0;
  BTLE_CUDA(ctx, cudaEventElapsedTime(&ms, t.e0, t.e1));
  out->packets = n_packets; out->pkt_err = acc[0]; out->bit_err = acc[1]; out->aa_miss = acc[2];
  out->bit_total = (uint64_t)n_packets * 8 * kBerPduBytes;
  out->seconds = ms * 1e-3;
  ctx->last_launches = launches;
  return BTLE_OK;
}

static_assert(kBerSamples == BTLE_BER_SAMPLES, "include/btle_b200.h documents the BER packet length");
int btle_b200_ber_synth_device(btle_b200_ctx *ctx, const btle_ber_cfg *cfg, uint64_t first_packet, size_t n_packets, int16_t *d_i,
                               int16_t *d_q, uint8_t *d_truth, void *cuda_stream) {
  if (!ctx || !cfg || !d_i || !d_q || !d_truth || n_packets > 0x7FFFFFFFu) return BTLE_EINVAL;
  int rc = check_ber_cfg(ctx, cfg);
  if (rc) return rc;
  if (!n_packets) return BTLE_OK;
  BTLE_CUDA(ctx, cudaSetDevice(ctx->device));
  ber_synth_kernel<<<(unsigned)n_packets, 384, 0, reinterpret_cast<cudaStream_t>(cuda_stream)>>>(
      *cfg, (unsigned long long)first_packet, (int)n_packets, d_i, d_q, d_truth);
  BTLE_CUDA(ctx, cudaGetLastError());
  ctx->last_launches = 1;
  return BTLE_OK;
}

static_assert(sizeof(btle_rx_ber_cfg) == 48 && sizeof(btle_rx_ber_truth) == 64 && sizeof(btle_rx_ber_result) == 88,
              "include/btle_b200.h documents these sizes");
static_assert(kRxBerMaxL == 1520 && BTLE_RX_BER_MAX_SLOT / 16 * 16 + 16 <= BTLE_RX_BER_MAX_UNITS,
              "a run's smallest batch (lcm(slot, 8192) samples) has a directory rx_ber_score_kernel takes");
static int check_rx_ber_cfg(btle_b200_ctx *ctx, const btle_rx_ber_cfg *cfg) {
  if (cfg->channel < 0 || cfg->channel > 39) { ctx->err = "rx_ber: channel must be 0..39"; return BTLE_EINVAL; }
  if (!std::isfinite(cfg->snr_db) || !std::isfinite(cfg->ppm) || !std::isfinite(cfg->cfo_hz)) {
    ctx->err = "rx_ber: snr_db, ppm and cfo_hz must be finite";
    return BTLE_EINVAL;
  }
  if (std::fabs(cfg->ppm) >= 1e6f) { ctx->err = "rx_ber: ppm must have |ppm| < 1e6"; return BTLE_EINVAL; }
  if (cfg->amplitude < 1 || cfg->amplitude > 127) { ctx->err = "rx_ber: amplitude must be 1..127"; return BTLE_EINVAL; }
  if (cfg->flags & ~(uint32_t)BTLE_CFG_RECOVER) { ctx->err = "rx_ber: flags may only hold BTLE_CFG_RECOVER"; return BTLE_EINVAL; }
  if (cfg->slot_samples < rx_ber_len(cfg->channel) || cfg->slot_samples > BTLE_RX_BER_MAX_SLOT) {
    ctx->err = "rx_ber: slot_samples must hold the packet (" + std::to_string(rx_ber_len(cfg->channel)) + " samples on this channel) and be at most " +
               std::to_string(BTLE_RX_BER_MAX_SLOT);
    return BTLE_EINVAL;
  }
  return BTLE_OK;
}

// capture of `n_samples` samples from slot `first` on (packets while the global slot index is below n_live, truth rows
// for the first n_truth slots)
static int launch_rx_ber_synth(btle_b200_ctx *ctx, const btle_rx_ber_cfg &cfg, uint64_t first, uint64_t n_live, long long n_samples,
                               long long n_truth, int8_t *d_iq, btle_rx_ber_truth *d_truth, cudaStream_t st) {
  const long long slots = (n_samples + cfg.slot_samples - 1) / cfg.slot_samples;
  if (slots > 0x7FFFFFFFll) { ctx->err = "rx_ber: too many slots for one launch"; return BTLE_EINVAL; }
  rx_ber_synth_kernel<<<(unsigned)slots, 256, 0, st>>>(cfg, first, n_live, n_samples, n_truth, d_iq, d_truth);
  BTLE_CUDA(ctx, cudaGetLastError());
  return BTLE_OK;
}

static int launch_rx_ber_score(btle_b200_ctx *ctx, const btle_rx_ber_truth *d_truth, size_t n_packets, const btle_pkt_rec *d_recs, size_t n_recs,
                               const btle_unit_dir *d_dir, size_t n_units, btle_rx_ber_result *d_result, cudaStream_t st) {
  const unsigned grid = (unsigned)std::max<size_t>(1, (n_packets + 255) / 256);
  rx_ber_score_kernel<<<grid, 256, (n_units + 1) * sizeof(unsigned), st>>>(d_truth, (int)n_packets, d_recs, (unsigned long long)n_recs,
                                                                         reinterpret_cast<const uint2 *>(d_dir), (int)n_units,
                                                                         reinterpret_cast<unsigned long long *>(d_result));
  BTLE_CUDA(ctx, cudaGetLastError());
  return BTLE_OK;
}

int btle_b200_rx_ber_synth_device(btle_b200_ctx *ctx, const btle_rx_ber_cfg *cfg, uint64_t first_packet, size_t n_packets, int8_t *d_iq,
                                  btle_rx_ber_truth *d_truth, void *cuda_stream) {
  if (!ctx) return BTLE_EINVAL;
  if (!cfg || (n_packets && (!d_iq || !d_truth))) { ctx->err = "rx_ber_synth: missing buffer"; return BTLE_EINVAL; }
  int rc = check_rx_ber_cfg(ctx, cfg);
  if (rc) return rc;
  if (reinterpret_cast<uintptr_t>(d_iq) & 15) { ctx->err = "device IQ must be 16-byte aligned"; return BTLE_EINVAL; }
  if (!n_packets) return BTLE_OK;
  BTLE_CUDA(ctx, cudaSetDevice(ctx->device));
  const long long n_samples = (long long)(BTLE_RX_BER_CAPTURE_INT8(n_packets, cfg->slot_samples) / 2);
  rc = launch_rx_ber_synth(ctx, *cfg, first_packet, first_packet + n_packets, n_samples, (long long)n_packets, d_iq, d_truth,
                           reinterpret_cast<cudaStream_t>(cuda_stream));
  if (rc) return rc;
  ctx->last_launches = 1;
  return BTLE_OK;
}

int btle_b200_rx_ber_score_device(btle_b200_ctx *ctx, const btle_rx_ber_truth *d_truth, size_t n_packets, const btle_pkt_rec *d_recs,
                                  size_t n_recs, const btle_unit_dir *d_dir, size_t n_units, btle_rx_ber_result *d_result,
                                  void *cuda_stream) {
  if (!ctx) return BTLE_EINVAL;
  if (!d_result || (n_packets && !d_truth) || (n_recs && !d_recs) || (n_units && !d_dir)) { ctx->err = "rx_ber_score: missing buffer"; return BTLE_EINVAL; }
  if (n_units > BTLE_RX_BER_MAX_UNITS) { ctx->err = "rx_ber_score: more than BTLE_RX_BER_MAX_UNITS directory entries"; return BTLE_EINVAL; }
  if (n_packets > 0x7FFFFFFFu) { ctx->err = "rx_ber_score: too many packets for one launch"; return BTLE_EINVAL; }
  if (!n_packets && !n_units) return BTLE_OK;
  BTLE_CUDA(ctx, cudaSetDevice(ctx->device));
  const int rc = launch_rx_ber_score(ctx, d_truth, n_packets, d_recs, n_recs, d_dir, n_units, d_result, reinterpret_cast<cudaStream_t>(cuda_stream));
  if (rc) return rc;
  ctx->last_launches = 1;
  return BTLE_OK;
}

// Batches of B packets, B a multiple of 8192 / gcd(S, 8192): every batch but the last covers whole chunks and ends on a
// slot boundary, so its capture is the run's one long capture from its first chunk on, and its look-ahead behind the last
// chunk (BTLE_LOOKAHEAD_INT8) is written with the slots that follow.  The receiver decodes a chunk from that chunk and its
// look-ahead alone (zeroed history at each chunk), so every batch's records are the long capture's records of its
// chunks, and the counts do not depend on B.
int btle_b200_rx_ber_run(btle_b200_ctx *ctx, const btle_rx_ber_cfg *cfg, size_t n_packets, btle_rx_ber_result *out) {
  if (!ctx) return BTLE_EINVAL;
  if (!cfg || !out) { ctx->err = "rx_ber_run: missing argument"; return BTLE_EINVAL; }
  memset(out, 0, sizeof *out);
  int rc = check_rx_ber_cfg(ctx, cfg);
  if (rc) return rc;
  if (!n_packets) return BTLE_OK;
  BTLE_CUDA(ctx, cudaSetDevice(ctx->device));
  cudaStream_t st = ctx->stream;
  const long long S = cfg->slot_samples;
  long long g = kChunkSamples, b = S;
  while (b) { const long long t = g % b; g = b; b = t; }
  const long long q = kChunkSamples / g;                     // packets of the smallest batch: lcm(S, 8192) / S
  size_t free_b = 0, total_b = 0;
  BTLE_CUDA(ctx, cudaMemGetInfo(&free_b, &total_b));
  const size_t per_chunk = kChunkInt8 + BTLE_MAX_RECS_PER_CHUNK * sizeof(btle_pkt_rec) + 8 * sizeof(btle_rx_ber_truth);
  const long long want_chunks = (long long)std::min<size_t>(8192, std::max<size_t>(1, free_b / 2 / per_chunk));
  const long long B = std::max(1ll, want_chunks * kChunkSamples / (q * S)) * q;
  const size_t max_b = std::min<size_t>(n_packets, (size_t)B);
  const long long max_chunks = ((long long)max_b * S + kChunkSamples - 1) / kChunkSamples;
  const size_t max_int8 = (size_t)max_chunks * kChunkInt8 + BTLE_LOOKAHEAD_INT8, max_recs = (size_t)max_chunks * BTLE_MAX_RECS_PER_CHUNK;
  if (ctx->d_iq.reserve(ctx, max_int8) || ctx->d_out.reserve(ctx, max_recs) ||
      ctx->d_dir.reserve(ctx, (size_t)(max_chunks + kSpanChunks - 1) / kSpanChunks * kSpanChunks))   // >= units of any batch
    return BTLE_ENOMEM;
  btle_rx_ber_truth *d_truth;
  btle_rx_ber_result *d_res;
  rc = leaf_layout(ctx, piece(d_truth, max_b), piece(d_res, 1));
  if (rc) return rc;
  BTLE_CUDA(ctx, cudaMemsetAsync(d_res, 0, sizeof(btle_rx_ber_result), st));
  struct Timing {                                           // the two events are destroyed on every return
    cudaEvent_t e0 = nullptr, e1 = nullptr;
    ~Timing() { if (e0) cudaEventDestroy(e0); if (e1) cudaEventDestroy(e1); }
  } t;
  BTLE_CUDA(ctx, cudaEventCreate(&t.e0));
  BTLE_CUDA(ctx, cudaEventCreate(&t.e1));
  BTLE_CUDA(ctx, cudaEventRecord(t.e0, st));
  const btle_stream_cfg scfg{cfg->channel, cfg->access_addr, 0xFFFFFFFFu, cfg->crc_init, 0, (int32_t)(BTLE_CFG_REPORT_REJECTED | cfg->flags)};
  int launches = 0;
  for (size_t done = 0; done < n_packets; done += max_b) {
    const size_t n = std::min(max_b, n_packets - done);
    const bool last = done + n == n_packets;
    const long long chunks = ((long long)n * S + kChunkSamples - 1) / kChunkSamples;
    const size_t n_int8 = (size_t)chunks * kChunkInt8 + (last ? 0 : BTLE_LOOKAHEAD_INT8);
    rc = launch_rx_ber_synth(ctx, *cfg, done, n_packets, (long long)(n_int8 / 2), (long long)n, ctx->d_iq, d_truth, st);
    if (rc) return rc;
    const size_t cap = (size_t)chunks * BTLE_MAX_RECS_PER_CHUNK, units = btle_b200_rx_units(ctx, 1, n_int8);
    rc = launch_rx(ctx, ctx->d_iq, 1, n_int8, n_int8, &scfg, nullptr, 1, nullptr, ctx->d_out, cap, ctx->d_count, ctx->d_dir, st, 0);
    if (rc) return rc;
    rc = launch_rx_ber_score(ctx, d_truth, n, ctx->d_out, cap, ctx->d_dir, units, d_res, st);
    if (rc) return rc;
    launches += 3;
  }
  BTLE_CUDA(ctx, cudaEventRecord(t.e1, st));
  btle_rx_ber_result res;
  BTLE_CUDA(ctx, cudaMemcpyAsync(&res, d_res, sizeof res, cudaMemcpyDeviceToHost, st));
  BTLE_CUDA(ctx, cudaStreamSynchronize(st));
  float ms = 0;
  BTLE_CUDA(ctx, cudaEventElapsedTime(&ms, t.e0, t.e1));
  *out = res;
  out->seconds = ms * 1e-3;
  ctx->last_launches = launches;
  return BTLE_OK;
}

int btle_b200_gfsk_demod_i16(btle_b200_ctx *ctx, const int16_t *i, const int16_t *q, size_t n, int8_t *bit_out,
                             int32_t *signal_out) {
  if (!ctx || !i || !q || !bit_out || !signal_out) return BTLE_EINVAL;
  if (n < 2) return BTLE_OK;
  BTLE_CUDA(ctx, cudaSetDevice(ctx->device));
  int16_t *d_i, *d_q;
  int32_t *d_s;
  int8_t *d_b;
  const int rc = leaf_layout(ctx, piece(d_i, n), piece(d_q, n), piece(d_s, n), piece(d_b, n));
  if (rc) return rc;
  BTLE_CUDA(ctx, cudaMemcpyAsync(d_i, i, 2 * n, cudaMemcpyHostToDevice, ctx->stream));
  BTLE_CUDA(ctx, cudaMemcpyAsync(d_q, q, 2 * n, cudaMemcpyHostToDevice, ctx->stream));
  gfsk_demod_i16_kernel<<<(unsigned)((n + 255) / 256), 256, 0, ctx->stream>>>(d_i, d_q, (long long)n, d_b, d_s);
  BTLE_CUDA(ctx, cudaGetLastError());
  BTLE_CUDA(ctx, cudaMemcpyAsync(bit_out, d_b, n - 1, cudaMemcpyDeviceToHost, ctx->stream));
  BTLE_CUDA(ctx, cudaMemcpyAsync(signal_out, d_s, 4 * (n - 1), cudaMemcpyDeviceToHost, ctx->stream));
  BTLE_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  return BTLE_OK;
}

// body of btle_b200_search_bit_sequence: a BTLE_* code, the first match (or -1) in *first
static int search_bit_sequence(btle_b200_ctx *ctx, const int8_t *bit, size_t n, const int8_t *seq, size_t m, long long *first) {
  BTLE_CUDA(ctx, cudaSetDevice(ctx->device));
  int8_t *d_b, *d_s;
  long long *d_first;
  const int rc = leaf_layout(ctx, piece(d_b, n), piece(d_s, m), piece(d_first, 1));
  if (rc) return rc;
  *first = -1;                                              // all ones == "none" for the unsigned atomicMin
  BTLE_CUDA(ctx, cudaMemcpyAsync(d_b, bit, n, cudaMemcpyHostToDevice, ctx->stream));
  BTLE_CUDA(ctx, cudaMemcpyAsync(d_s, seq, m, cudaMemcpyHostToDevice, ctx->stream));
  BTLE_CUDA(ctx, cudaMemcpyAsync(d_first, first, 8, cudaMemcpyHostToDevice, ctx->stream));
  search_seq_kernel<<<(unsigned)((n + 255) / 256), 256, 0, ctx->stream>>>(d_b, (long long)n, d_s, (long long)m, d_first);
  return leaf_result(ctx, first, d_first, 8);
}

long btle_b200_search_bit_sequence(btle_b200_ctx *ctx, const int8_t *bit, size_t n, const int8_t *seq, size_t m) {
  if (!ctx || (!bit && n) || (!seq && m)) return BTLE_EINVAL - 1;     // -2: errors never collide with "-1 = not found"
  if (m == 0) return 0;                                     // btlelib.py:408: the empty window at i = 0 matches
  if (n < m) return -1;
  long long first = -1;
  const int rc = search_bit_sequence(ctx, bit, n, seq, m, &first);
  return rc ? rc - 1 : (long)first;
}

int btle_b200_crc24_bits(btle_b200_ctx *ctx, const int8_t *bit_in, size_t n, const int8_t *state_init_bit, int8_t *crc_bits_out) {
  if (!ctx || (!bit_in && n) || !state_init_bit || !crc_bits_out) return BTLE_EINVAL;
  BTLE_CUDA(ctx, cudaSetDevice(ctx->device));
  int8_t *d_b, *d_i, *d_o;
  const int rc = leaf_layout(ctx, piece(d_b, n), piece(d_i, 24), piece(d_o, 24));
  if (rc) return rc;
  if (n) BTLE_CUDA(ctx, cudaMemcpyAsync(d_b, bit_in, n, cudaMemcpyHostToDevice, ctx->stream));
  BTLE_CUDA(ctx, cudaMemcpyAsync(d_i, state_init_bit, 24, cudaMemcpyHostToDevice, ctx->stream));
  crc24_bits_kernel<<<1, 1, 0, ctx->stream>>>(d_b, (long long)n, d_i, d_o);
  return leaf_result(ctx, crc_bits_out, d_o, 24);
}

int btle_b200_scramble_bits(btle_b200_ctx *ctx, const int8_t *bit_in, size_t n, int channel, int8_t *bit_out) {
  if (!ctx || (!bit_in && n) || (!bit_out && n)) return BTLE_EINVAL;
  if (n == 0) return BTLE_OK;
  BTLE_CUDA(ctx, cudaSetDevice(ctx->device));
  int8_t *d_b, *d_o;
  const int rc = leaf_layout(ctx, piece(d_b, n), piece(d_o, n));
  if (rc) return rc;
  BTLE_CUDA(ctx, cudaMemcpyAsync(d_b, bit_in, n, cudaMemcpyHostToDevice, ctx->stream));
  // btlelib.py:238-243 seeds the register from bits 5..0 of any integer channel
  scramble_bits_kernel<<<1, 1, 0, ctx->stream>>>(d_b, (long long)n, channel & 63, d_o);
  return leaf_result(ctx, bit_out, d_o, n);
}

void btle_b200_parse_adv_pdu_header_byte(const uint8_t *b, int *pdu_type, int *tx_add, int *rx_add, int *payload_len) {
  *pdu_type = b[0] & 0x0F;             // btle_rx.c:1950
  *tx_add = (b[0] & 0x40) != 0;        // :1955
  *rx_add = (b[0] & 0x80) != 0;        // :1959
  *payload_len = b[1] & 0x3F;          // :1962
}

void btle_b200_parse_ll_pdu_header_byte(const uint8_t *b, int *llid, int *nesn, int *sn, int *md, int *payload_len) {
  *llid = b[0] & 0x03;                 // btle_rx.c:1940
  *nesn = (b[0] & 0x04) != 0;
  *sn = (b[0] & 0x08) != 0;
  *md = (b[0] & 0x10) != 0;
  *payload_len = b[1] & 0x1F;          // :1944
}

}  // extern "C"
