// Host build of the MSM's digit sort (spectre_b200/csrc/msm.cuh) for tests/test_hostemu_msm_sort.py: the per-thread bodies
// of the digit and offsets kernels around a serial stable sort (the device runs an LSD radix sort, which is stable too),
// next to the counting sort (histogram, exclusive scan, scatter at a cursor) that the library ran before, on the same scalars.
#include "../../spectre_b200/csrc/msm.cuh"
#include <algorithm>
#include <string.h>
#include <vector>
using namespace spb;

static MsmGeom geometry(uint64_t n, uint32_t c, int precomp) { return msm_make_geometry(c, precomp != 0, (uint32_t)n); }

extern "C" {
uint64_t he_sort_buckets(uint32_t c, int precomp) { MsmGeom g = geometry(1, c, precomp); return (uint64_t)g.BW * g.B; }
int he_sort_key_bits(uint32_t c, int precomp) { return msm_key_bits(geometry(1, c, precomp)); }

// counting sort: offsets (nb + 1) and entries (n * W) -> M
uint64_t he_sort_counting(const Fr* scalars, uint64_t n, uint32_t c, int precomp, uint32_t* offsets, MsmEntry* ent) {
  const MsmGeom g = geometry(n, c, precomp);
  const uint64_t nb = (uint64_t)g.BW * g.B;
  std::vector<uint32_t> counts(nb + 1, 0);
  for (uint64_t t = 0; t < n; t++) msm_count_thread(t, n, scalars, g, counts.data());
  uint64_t run = 0;
  for (uint64_t i = 0; i <= nb; i++) { offsets[i] = (uint32_t)run; run += counts[i]; }
  std::vector<uint32_t> cursor(offsets, offsets + nb + 1);
  for (uint64_t t = 0; t < n; t++) msm_scatter_thread(t, n, scalars, g, cursor.data(), ent);
  return offsets[nb];
}

// digits -> stable sort by key -> offsets: the library's steps 1-3. The offsets array is filled with a marker first, so an
// offset the bodies leave unwritten shows.
uint64_t he_sort_radix(const Fr* scalars, uint64_t n, uint32_t c, int precomp, uint32_t* offsets, MsmEntry* ent) {
  const MsmGeom g = geometry(n, c, precomp);
  const uint64_t nb = (uint64_t)g.BW * g.B;
  uint32_t total = 0;
  for (uint64_t t = 0; t < n; t++) msm_digits_thread(t, n, scalars, g, &total, ent);
  std::stable_sort(ent, ent + total, [](const MsmEntry& a, const MsmEntry& b) { return a.key < b.key; });
  memset(offsets, 0xAB, (nb + 1) * sizeof(uint32_t));
  for (uint64_t k = 0; k <= nb + 1; k++) msm_offsets_thread(k, nb, total, ent, offsets);   // one thread past the end: no write
  return total;
}
}
