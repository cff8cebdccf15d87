// Feed probe for btle_rx_persistent_kernel (run by tools/probe_feed.py, kept outside the library like pipe_probe.cu).
//
// The probe kernels walk a capture the way the receive kernel's dense warps do: one CTA per SM, spans of 16 chunks
// (1024 groups of 256 bytes) plus a 12-group look-ahead tile dealt round-robin to CTAs, tile j of a CTA (32 groups,
// 8 KB) on dense warp j % W, TMA boxes with SWIZZLE_128B and L2_PROMOTION_L2_256B.  Only the way tiles are fetched
// changes between variants; the arithmetic is either the receive kernel's dense loop (dbits8_dense) or a cheap XOR of
// the words, so the feed can be seen with and without the SM work it has to hide.
//
//   halves<W, NB, PF, T>  a warp's tiles as a sequence of 4 KB half boxes (upper half first) through a ring of NB half
//                         buffers; a buffer is requested again as soon as its half has been consumed.  W = 16, NB = 2,
//                         T = 33 is the receive kernel's earlier feed.  PF: also prefetch the warp's tile after next into L2
//                         (cp.async.bulk.prefetch.tensor).  T = 32: no look-ahead tile (its bytes and its iteration).
//   tiles<W, NT>          one 8 KB box per tile (tensor dims {128 B, runs, halves, streams}: half h lands at h x rows x
//                         128 B in the same swizzled layout) through NT tile buffers, one mbarrier per tile.  W = 16, NT = 1 is the
//                         receive kernel's feed since the probe picked it (DESIGN.md, section 4.1).
#include <cuda.h>
#include <cuda_runtime.h>

#include <cstdint>
#include <cstdio>
#include <string_view>

#include "../btle_b200/csrc/btle_core.cuh"

using namespace btle;

namespace {

constexpr int kRunsPerSpan = kSpanChunks * kGroupsPerChunk;   // 1024 groups of 256 bytes
constexpr int kSmemBytes = 200 * 1024;                        // one CTA per SM, as the receive kernel

__device__ __forceinline__ uint32_t smem_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(unsigned long long *bar, int count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
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
      "DONE_%=:\n\t}" ::"r"(smem_u32(bar)),
      "r"(parity)
      : "memory");
}
__device__ __forceinline__ void tma_load(void *dst, const CUtensorMap *map, int c1, int c2, unsigned long long *bar) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3, %4, %5}], [%6];" ::"r"(
          smem_u32(dst)),
      "l"(map), "r"(0), "r"(c1), "r"(c2), "r"(0), "r"(smem_u32(bar))
      : "memory");
}
__device__ __forceinline__ void tma_prefetch(const CUtensorMap *map, int c1, int c2) {
  asm volatile("cp.async.bulk.prefetch.tensor.4d.L2.global.tile [%0, {%1, %2, %3, %4}];" ::"l"(map), "r"(0), "r"(c1), "r"(c2), "r"(0)
               : "memory");
}

// tile i of warp w: (run0, rows), or rows = 0 behind the CTA's last unit
template <int W, int T>
__device__ __forceinline__ int tile_of(int w, int i, int units, int &run0) {
  const int j = w + i * W, k = j / T, t = j - k * T;
  const int unit = blockIdx.x + k * gridDim.x;
  if (unit >= units) return 0;
  run0 = unit * kRunsPerSpan + t * 32;
  return t < 32 ? 32 : kHaloGroups;
}

// consume one 128-byte swizzled row (the 16-byte chunk cc sits at cc ^ sw)
template <bool DENSE>
__device__ __forceinline__ void consume_row(const unsigned char *row, uint32_t sw, uint32_t acc[4], uint32_t &carry) {
#pragma unroll
  for (int cc = 7; cc >= 0; --cc) {
    const uint4 w = *reinterpret_cast<const uint4 *>(row + ((((uint32_t)cc ^ sw)) << 4));
    if (DENSE) {
      if ((cc & 3) == 3) {
#pragma unroll
        for (int ph = 0; ph < 4; ++ph) acc[ph] <<= 8;
      }
      switch (cc & 3) {
        case 3: dbits8_dense<3>(w.x, w.y, w.z, w.w, carry, acc); break;
        case 2: dbits8_dense<2>(w.x, w.y, w.z, w.w, carry, acc); break;
        case 1: dbits8_dense<1>(w.x, w.y, w.z, w.w, carry, acc); break;
        default: dbits8_dense<0>(w.x, w.y, w.z, w.w, carry, acc); break;
      }
    } else {
      acc[0] ^= w.x; acc[1] ^= w.y; acc[2] ^= w.z; acc[3] ^= w.w;
    }
    carry = w.x;
  }
}

template <int W, int NB, bool PF, int T, bool DENSE>
__global__ void __launch_bounds__(W * 32, 1)
feed_halves(const __grid_constant__ CUtensorMap map32, const __grid_constant__ CUtensorMap map12, int units, uint32_t *sink) {
  extern __shared__ __align__(1024) unsigned char smem[];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  unsigned char *stage = smem + warp * NB * 4096;
  unsigned long long *mbar = reinterpret_cast<unsigned long long *>(smem + W * NB * 4096) + warp * NB;
  if (lane == 0) {
    for (int b = 0; b < NB; ++b) mbar_init(&mbar[b], 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncwarp();
  // half q of the warp's sequence: tile q >> 1, upper half first
  auto request = [&](int q) {
    int run0 = 0;
    const int rows = tile_of<W, T>(warp, q >> 1, units, run0);
    if (lane != 0 || rows == 0) return;
    const int half = 1 - (q & 1);
    const CUtensorMap *map = rows == 32 ? &map32 : &map12;
    unsigned long long *bar = &mbar[q % NB];
    mbar_expect_tx(bar, (uint32_t)rows * 128u);
    tma_load(stage + (q % NB) * 4096, map, half, run0, bar);
    if (PF && half == 1) {                                  // the warp's tile after this one, into L2
      int pr = 0;
      const int prow = tile_of<W, T>(warp, (q >> 1) + 1, units, pr);
      if (prow) {
        const CUtensorMap *pm = prow == 32 ? &map32 : &map12;
        tma_prefetch(pm, 0, pr);
        tma_prefetch(pm, 1, pr);
      }
    }
  };
  for (int q = 0; q < NB; ++q) request(q);
  uint32_t acc[4] = {0u, 0u, 0u, 0u}, carry = 0u, out = 0u;
  for (int q = 0;; ++q) {
    int run0 = 0;
    const int rows = tile_of<W, T>(warp, q >> 1, units, run0);
    if (rows == 0) break;
    mbar_wait(&mbar[q % NB], (uint32_t)(q / NB) & 1u);
    if (lane < rows) consume_row<DENSE>(stage + (q % NB) * 4096 + (lane << 7), (uint32_t)(lane & 7), acc, carry);
    __syncwarp();
    request(q + NB);
    if (q & 1) out ^= acc[0] ^ acc[1] ^ acc[2] ^ acc[3];
  }
  sink[blockIdx.x * blockDim.x + threadIdx.x] = out;
}

template <int W, int NT, bool DENSE>
__global__ void __launch_bounds__(W * 32, 1)
feed_tiles(const __grid_constant__ CUtensorMap map32, const __grid_constant__ CUtensorMap map12, int units, uint32_t *sink) {
  constexpr int T = 33;
  extern __shared__ __align__(1024) unsigned char smem[];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  unsigned char *stage = smem + warp * NT * 8192;
  unsigned long long *mbar = reinterpret_cast<unsigned long long *>(smem + W * NT * 8192) + warp * NT;
  if (lane == 0) {
    for (int b = 0; b < NT; ++b) mbar_init(&mbar[b], 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncwarp();
  auto request = [&](int i) {
    int run0 = 0;
    const int rows = tile_of<W, T>(warp, i, units, run0);
    if (lane != 0 || rows == 0) return;
    unsigned long long *bar = &mbar[i % NT];
    mbar_expect_tx(bar, (uint32_t)rows * 256u);
    tma_load(stage + (i % NT) * 8192, rows == 32 ? &map32 : &map12, run0, 0, bar);
  };
  for (int i = 0; i < NT; ++i) request(i);
  uint32_t acc[4] = {0u, 0u, 0u, 0u}, carry = 0u, out = 0u;
  for (int i = 0;; ++i) {
    int run0 = 0;
    const int rows = tile_of<W, T>(warp, i, units, run0);
    if (rows == 0) break;
    mbar_wait(&mbar[i % NT], (uint32_t)(i / NT) & 1u);
    if (lane < rows) {
      const unsigned char *buf = stage + (i % NT) * 8192;
#pragma unroll 1
      for (int h = 1; h >= 0; --h) {                        // row h * rows + lane of the box
        const int r = h * rows + lane;
        consume_row<DENSE>(buf + (r << 7), (uint32_t)(r & 7), acc, carry);
      }
    }
    __syncwarp();
    request(i + NT);
    out ^= acc[0] ^ acc[1] ^ acc[2] ^ acc[3];
  }
  sink[blockIdx.x * blockDim.x + threadIdx.x] = out;
}

typedef CUresult (*encode_fn)(CUtensorMap *, CUtensorMapDataType, cuuint32_t, void *, const cuuint64_t *, const cuuint64_t *,
                              const cuuint32_t *, const cuuint32_t *, CUtensorMapInterleave, CUtensorMapSwizzle,
                              CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

// whole_tiles = 0: {128 B, 2 halves, runs, 1}, box {128, 1, rows, 1};  1: {128 B, runs, 2 halves, 1}, box {128, rows, 2, 1}
int encode(const int8_t *iq, long long n_int8, int whole_tiles, CUtensorMap *m32, CUtensorMap *m12) {
  static encode_fn enc = nullptr;
  if (!enc) {
    void *p = nullptr;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, nullptr) != cudaSuccess || !p) return -1;
    enc = reinterpret_cast<encode_fn>(p);
  }
  const cuuint64_t runs = (cuuint64_t)(n_int8 / 256);
  const cuuint64_t dims0[4] = {128, 2, runs, 1}, dims1[4] = {128, runs, 2, 1};
  const cuuint64_t str0[3] = {128, 256, (cuuint64_t)n_int8}, str1[3] = {256, 128, (cuuint64_t)n_int8};
  const cuuint32_t estr[4] = {1, 1, 1, 1};
  for (int which = 0; which < 2; ++which) {
    const cuuint32_t rows = which ? kHaloGroups : 32;
    const cuuint32_t box0[4] = {128, 1, rows, 1}, box1[4] = {128, rows, 2, 1};
    const CUresult r = enc(which ? m12 : m32, CU_TENSOR_MAP_DATA_TYPE_UINT8, 4, const_cast<int8_t *>(iq), whole_tiles ? dims1 : dims0,
                           whole_tiles ? str1 : str0, whole_tiles ? box1 : box0, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                           CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) return -2;
  }
  return 0;
}

template <class K>
int launch(K kernel, int threads, int whole_tiles, const int8_t *iq, long long n_int8, uint32_t *sink, int grid, cudaStream_t st) {
  CUtensorMap m32, m12;
  if (encode(iq, n_int8, whole_tiles, &m32, &m12)) return -2;
  if (cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmemBytes) != cudaSuccess) return -3;
  const int units = (int)(n_int8 / ((long long)kRunsPerSpan * 256));
  kernel<<<grid, threads, kSmemBytes, st>>>(m32, m12, units, sink);
  return cudaGetLastError() == cudaSuccess ? 0 : -4;
}

}  // namespace

// Variants by name: see tools/probe_feed.py.  Returns 0, or a negative code (-1 unknown variant).
extern "C" int probe_feed_launch(const char *name, int dense, const int8_t *iq, long long n_int8, uint32_t *sink, int grid,
                                 cudaStream_t st) {
  const std::string_view v(name);
#define PROBE_HALVES(NAME, W, NB, PF, T)                                                                                    \
  if (v == NAME)                                                                                                            \
    return dense ? launch(feed_halves<W, NB, PF, T, true>, W * 32, 0, iq, n_int8, sink, grid, st)                        \
                 : launch(feed_halves<W, NB, PF, T, false>, W * 32, 0, iq, n_int8, sink, grid, st);
#define PROBE_TILES(NAME, W, NT)                                                                                            \
  if (v == NAME)                                                                                                            \
    return dense ? launch(feed_tiles<W, NT, true>, W * 32, 1, iq, n_int8, sink, grid, st)                                \
                 : launch(feed_tiles<W, NT, false>, W * 32, 1, iq, n_int8, sink, grid, st);
  PROBE_HALVES("A", 16, 2, false, 33)            // the earlier feed: two half boxes per tile
  PROBE_TILES("B", 16, 1)                        // one box per tile, one tile buffer per warp (the receive kernel's feed)
  PROBE_TILES("B2", 8, 2)                        // one box per tile, two tile buffers per warp (same 128 KB)
  PROBE_HALVES("C3w12", 12, 3, false, 33)        // three halves per warp, 12 warps (144 KB)
  PROBE_HALVES("C4w8", 8, 4, false, 33)          // four halves per warp, 8 warps (128 KB)
  PROBE_HALVES("C3w16", 16, 3, false, 33)        // three halves per warp, 16 warps (192 KB: needs a smaller ring)
  PROBE_HALVES("Cpf", 16, 2, true, 33)           // A + L2 prefetch of the warp's tile after next
  PROBE_HALVES("D", 16, 2, false, 32)            // A without the look-ahead tile
#undef PROBE_HALVES
#undef PROBE_TILES
  return -1;
}
