// Hashed GROUP BY under PQ_QUERY_ALLREDUCE: the pure (host + device) pieces of the merge of every rank's groups.
//
// Each rank lists the cells of its hash table that hold rows (count > 0) and packs them into E_max records (E_max: the
// most any rank listed); one all-gather hands every rank the same N blocks, in rank order.  Rank r's block holds
// 1 + cells planes of E_max words: the wide group ids, then the cell planes in the order d_acc keeps them (count, the
// accumulators, the non-null counters).  Its first E_r records are listed cells, the rest padding.
//
// The listed records, numbered p = pre[r] + j (ranks in order), are sorted by wide id with a stable sort, so the records
// of one group sit together in rank order.  One thread per group folds them into one merged cell per plane:
//   count, COUNT, non-null counters, Int64 SUM   wrapping add
//   Float64 SUM / AVG                            f64 add in rank order: ((r0 + r1) + r2) ...
//   MIN / MAX                                    signed min / max of the cell encoding (totalOrder for Float64, ranks in
//                                                the agreed numbering for Utf8, bits for Boolean)
// Every rank holds the same bytes and folds them the same way, so every rank's table is the same bit for bit.
//
// Free of CUDA-only constructs: tests/test_hash_merge_core.py runs the same code on the CPU through
// tools/hash_merge_host.cpp.
#pragma once
#include <cstdint>
#include <cstring>

#include "decode_core.cuh"   // PQ_HD
#include "device_structs.hpp"
#ifdef __CUDACC__
#include "egress_kernels.cuh"   // kSlotTile
#endif

namespace pqb {

// the exchange record every rank sends before the cells: what decides, alike on every rank, whether the merge runs
enum : uint32_t { kMergeListed = 0, kMergeFull = 1, kMergeCorrupt = 2, kMergeBudget = 3, kMergeRecWords = 4 };

struct HashMergeArgs {
  const unsigned long long* recv;   // nranks blocks of (1 + cells) planes of e_max words
  const unsigned long long* pre;    // [nranks + 1]: the first listed record of every rank, and the total
  const unsigned long long* ids;    // the wide id of every listed record p
  const uint32_t* sorted;           // the listed records in ascending wide id, equal ids in rank order
  const unsigned long long* tile_base;   // merged slot of the first group head of every tile of sorted positions
  unsigned long long* acc;          // the merged table: cells planes of cap words
  unsigned long long* wide;         // its wide group ids [cap]
  uint64_t e_max;
  uint32_t nranks, n, cap, cells, n_acc;
  uint8_t acc_init[kMaxAggs * 2];   // the combine of accumulator plane 1 + a (DevPlan::acc_init)
};

PQ_HD uint64_t hm_f64_add(uint64_t a, uint64_t b) {
#ifdef __CUDA_ARCH__
  return (uint64_t)__double_as_longlong(__dadd_rn(__longlong_as_double((long long)a), __longlong_as_double((long long)b)));
#else
  double x, y;
  std::memcpy(&x, &a, 8);
  std::memcpy(&y, &b, 8);
  x += y;
  std::memcpy(&a, &x, 8);
  return a;
#endif
}

// one cell of rank r folded into the cells of ranks before it.  how: 0 wrapping add, 1 f64 add, 2 signed min, 3 signed max
PQ_HD uint64_t hm_combine(uint64_t acc, uint64_t v, uint32_t how) {
  if (how == 0) return acc + v;
  if (how == 1) return hm_f64_add(acc, v);
  if (how == 2) return int64_t(v) < int64_t(acc) ? v : acc;
  return int64_t(v) > int64_t(acc) ? v : acc;
}

// the combine of plane c: count (0) and the non-null counters add, the accumulators as DevPlan::acc_init says
PQ_HD uint32_t hm_how(const HashMergeArgs& a, uint32_t c) { return (c >= 1 && c < 1 + a.n_acc) ? a.acc_init[c - 1] : 0u; }

// the rank whose listed records hold record p: pre[r] <= p < pre[r + 1] (a rank may list none)
PQ_HD uint32_t hm_rank_of(const HashMergeArgs& a, uint64_t p) {
  uint32_t lo = 0, hi = a.nranks - 1;
  while (lo < hi) {
    const uint32_t mid = (lo + hi + 1) / 2;
    if (a.pre[mid] <= p) lo = mid;
    else hi = mid - 1;
  }
  return lo;
}

// word `plane` of listed record p (plane 0: the wide id, 1 + c: cell plane c)
PQ_HD uint64_t hm_word(const HashMergeArgs& a, uint64_t p, uint32_t plane) {
  const uint32_t r = hm_rank_of(a, p);
  return a.recv[(uint64_t(r) * (1 + a.cells) + plane) * a.e_max + (p - a.pre[r])];
}

// merged slot g: the group whose records sit at sorted positions [q0, q1), folded in rank order
PQ_HD void hm_fold(const HashMergeArgs& a, uint32_t q0, uint32_t q1, uint32_t g) {
  a.wide[g] = a.ids[a.sorted[q0]];
  for (uint32_t c = 0; c < a.cells; c++) {
    const uint32_t how = hm_how(a, c);
    uint64_t v = hm_word(a, a.sorted[q0], 1 + c);
    for (uint32_t q = q0 + 1; q < q1; q++) v = hm_combine(v, hm_word(a, a.sorted[q], 1 + c), how);
    a.acc[uint64_t(c) * a.cap + g] = v;
  }
}

#ifdef __CUDACC__
// ---- the kernels (query.cu runs them after k_flat_agg, in place of the grouped all-reduce):
//   k_merge_record   this rank's exchange record: listed cells, table full, corrupt code, merge budget
//   k_hash_pack      the listed cells (out_slot, slot order) into the send block of e_max records
//   k_merge_list     the wide id of every listed record of the gathered blocks, ranks in order: the sort's keys
//   (RadixSort)      query.cu's LSD radix sort of those ids, stable
//   k_merge_heads    group heads (the sorted id changes) per tile of kSlotTile sorted positions
//   k_item_prefix    the merged slot of every tile's first head, and G
//   k_merge_fold     one thread per group: hm_fold of its records into merged slot = heads before it
__global__ void k_merge_record(unsigned long long* __restrict__ rec, const unsigned long long* __restrict__ listed,
                               const unsigned long long* __restrict__ counters, unsigned long long budget) {
  const unsigned long long code = counters[1];   // 100: agg_hash_slot found the table full; anything else: a corrupt page
  rec[kMergeListed] = *listed;
  rec[kMergeFull] = code == 100ull ? 1ull : 0ull;
  rec[kMergeCorrupt] = code == 100ull ? 0ull : code;
  rec[kMergeBudget] = budget;
}

__global__ void k_hash_pack(const unsigned long long* __restrict__ acc, const unsigned long long* __restrict__ hkeys, uint32_t nslots,
                            uint32_t cells, const uint32_t* __restrict__ out_slot, uint32_t listed, uint64_t e_max,
                            unsigned long long* __restrict__ send) {
  for (uint32_t j = blockIdx.x * blockDim.x + threadIdx.x; j < listed; j += gridDim.x * blockDim.x) {
    const uint32_t s = out_slot[j];
    send[j] = hkeys[s];
    for (uint32_t c = 0; c < cells; c++) send[(1 + uint64_t(c)) * e_max + j] = acc[uint64_t(c) * nslots + s];
  }
}

__global__ void k_merge_list(const HashMergeArgs a, unsigned long long* __restrict__ ids) {
  for (uint32_t p = blockIdx.x * blockDim.x + threadIdx.x; p < a.n; p += gridDim.x * blockDim.x) ids[p] = hm_word(a, p, 0);
}

__device__ __forceinline__ bool hm_head(const HashMergeArgs& a, uint32_t q) {
  return q < a.n && (q == 0 || a.ids[a.sorted[q]] != a.ids[a.sorted[q - 1]]);
}

__global__ void k_merge_heads(const HashMergeArgs a, uint32_t* __restrict__ tile_counts) {
  __shared__ uint32_t ws[8];
  const uint32_t q0 = blockIdx.x * kSlotTile;
  uint32_t c = 0;
  for (uint32_t i = threadIdx.x; i < (uint32_t)kSlotTile; i += blockDim.x) c += hm_head(a, q0 + i) ? 1u : 0u;
  c = __reduce_add_sync(0xffffffffu, c);
  if ((threadIdx.x & 31) == 0) ws[threadIdx.x >> 5] = c;
  __syncthreads();
  if (threadIdx.x == 0) {
    uint32_t t = 0;
    for (uint32_t w = 0; w < blockDim.x / 32; w++) t += ws[w];
    tile_counts[blockIdx.x] = t;
  }
}

// 256 threads x 4 consecutive sorted positions per tile, as k_slot_compact
__global__ void __launch_bounds__(256) k_merge_fold(const HashMergeArgs a) {
  __shared__ uint32_t ws[8];
  const uint32_t q0 = blockIdx.x * kSlotTile + threadIdx.x * 4;
  uint32_t f[4], c = 0;
#pragma unroll
  for (int k = 0; k < 4; k++) { f[k] = hm_head(a, q0 + k) ? 1u : 0u; c += f[k]; }
  uint32_t incl = c;
  const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (int o = 1; o < 32; o <<= 1) {
    const uint32_t t = __shfl_up_sync(0xffffffffu, incl, o);
    if ((int)lane >= o) incl += t;
  }
  if (lane == 31) ws[warp] = incl;
  __syncthreads();
  uint32_t wbase = 0;
  for (uint32_t w = 0; w < warp; w++) wbase += ws[w];
  uint32_t g = uint32_t(a.tile_base[blockIdx.x]) + wbase + incl - c;
#pragma unroll
  for (int k = 0; k < 4; k++) {
    if (!f[k]) continue;
    const uint32_t q = q0 + k;
    uint32_t q1 = q + 1;   // at most one record per rank
    while (q1 < a.n && !hm_head(a, q1)) q1++;
    hm_fold(a, q, q1, g++);
  }
}
#endif

}  // namespace pqb
