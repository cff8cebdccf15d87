// The CPU emulator's BTLE_CFG_OFFSET_SEARCH merge: the kernel's per-chunk step (os_merge_step, btle_core.cuh) over the
// hypotheses' records of one cfg, chunk by chunk, as btle_offset_merge_kernel runs it.
#include <algorithm>
#include <cstdint>
#include <vector>

#include "../../btle_b200/csrc/btle_core.cuh"

using namespace btle;

// n records of one cfg, in (hyp, chunk, n0) order as the hypotheses' launch stores them: hyp[i] in 0..6, chunk[i], n0[i],
// flags[i], crc_bad[i].  Writes the merged list's record indices to out (chunk by chunk, ascending) and returns its length;
// a record inserted by hypothesis 1..6 gets bit 31 set in out.
extern "C" long emul_os_merge(const int32_t *hyp, const int32_t *chunk, const int32_t *n0, const uint8_t *flags, const uint8_t *crc_bad,
                              long n, int32_t *out) {
  std::vector<int32_t> chunks;
  for (long i = 0; i < n; ++i) chunks.push_back(chunk[i]);
  std::vector<int32_t> order(chunks);
  std::sort(order.begin(), order.end());
  order.erase(std::unique(order.begin(), order.end()), order.end());
  std::vector<OsEnt> b(BTLE_MAX_MERGED_RECS_PER_CHUNK + 1);
  long m = 0;
  for (int32_t k : order) {
    int nb = 0;
    for (long i = 0; i < n; ++i)
      if (hyp[i] == 0 && chunk[i] == k) b[nb++] = OsEnt{n0[i], os_ok(flags[i], crc_bad[i]), (uint32_t)i};
    for (int h = 1; h < BTLE_OFFSET_SEARCH_HYPS; ++h)
      for (long i = 0; i < n; ++i)
        if (hyp[i] == h && chunk[i] == k && os_ok(flags[i], crc_bad[i]))
          nb = os_merge_step(b.data(), nb, OsEnt{n0[i], 1u, (uint32_t)i | 0x80000000u});
    for (int i = 0; i < nb; ++i) out[m++] = (int32_t)b[i].ref;
  }
  return m;
}
