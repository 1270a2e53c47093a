// TEST HARNESS ONLY: the merge of a hashed GROUP BY's gathered rank tables (hash_merge.cuh) on the CPU, for
// tests/test_hash_merge_core.py.  The record addressing, the fold and the per-cell combine are the device's own code; a
// std::stable_sort of the wide ids stands in for the device's LSD radix sort (both stable).  Never linked into
// libparseable_b200.so.
#include <algorithm>
#include <cstdint>
#include <cstring>
#include <numeric>
#include <vector>

#include "hash_merge.cuh"
using namespace pqb;

extern "C" {
// recv: nranks blocks of (1 + cells) planes of e_max words (wide ids, then the cell planes); listed[r]: rank r's listed
// records.  acc_init[a]: the combine of plane 1 + a (0 wrapping add, 1 f64 add, 2 signed min, 3 signed max).  Writes the
// merged groups to wide_out[G] and acc_out[c * cap + g] with cap = the listed records of every rank; returns G.
uint32_t hm_merge(uint32_t nranks, uint64_t e_max, uint32_t cells, uint32_t n_acc, const uint8_t* acc_init, const uint64_t* recv,
                  const uint64_t* listed, uint64_t* acc_out, uint64_t* wide_out) {
  std::vector<unsigned long long> pre(nranks + 1, 0);
  for (uint32_t r = 0; r < nranks; r++) pre[r + 1] = pre[r] + listed[r];
  const uint32_t n = uint32_t(pre[nranks]);
  HashMergeArgs a{};
  a.recv = reinterpret_cast<const unsigned long long*>(recv);
  a.pre = pre.data();
  a.e_max = e_max;
  a.nranks = nranks;
  a.n = n;
  a.cap = n;
  a.cells = cells;
  a.n_acc = n_acc;
  std::memcpy(a.acc_init, acc_init, std::min<size_t>(n_acc, sizeof(a.acc_init)));
  std::vector<unsigned long long> ids(n);
  for (uint32_t p = 0; p < n; p++) ids[p] = hm_word(a, p, 0);
  std::vector<uint32_t> sorted(n);
  std::iota(sorted.begin(), sorted.end(), 0u);
  std::stable_sort(sorted.begin(), sorted.end(), [&](uint32_t x, uint32_t y) { return ids[x] < ids[y]; });
  a.ids = ids.data();
  a.sorted = sorted.data();
  a.acc = reinterpret_cast<unsigned long long*>(acc_out);
  a.wide = reinterpret_cast<unsigned long long*>(wide_out);
  uint32_t g = 0;
  for (uint32_t q = 0; q < n;) {
    uint32_t q1 = q + 1;
    while (q1 < n && ids[sorted[q1]] == ids[sorted[q]]) q1++;
    hm_fold(a, q, q1, g++);
    q = q1;
  }
  return g;
}

uint64_t hm_combine_host(uint64_t acc, uint64_t v, uint32_t how) { return hm_combine(acc, v, how); }
}
