// MEDIAN / PERCENTILE_CONT after the scan.  k_flat_agg (its PCT instantiations) appended one (group slot, order key)
// pair per non-NULL selected row of every percentile column; per column:
//
//   k_pct_stage   the pairs as two ORDER BY terms (slot, key) in the layout order_sort reads ([2][n] values, no NULLs),
//                 and the value range of both terms
//   order_sort    (query.cu) the existing ORDER BY sort: the pair positions in (slot, key) order
//   k_pct_pick    one thread per non-empty group (out_slot): binary search of the group's run of sorted pairs, then the
//                 median / percentile of each aggregate over that run (percentile_core.cuh), written as the output bits
//                 into the aggregate's accumulator cell (replica 0 of acc).  agg_output_value reads it from there, so
//                 k_agg_finish and k_order_encode (ORDER BY on a percentile) need nothing else.
#pragma once
#include <cuda_runtime.h>

#include "device_structs.hpp"
#include "order_keys.cuh"
#include "percentile_core.cuh"

namespace pqb {

__global__ void __launch_bounds__(256) k_pct_stage(const uint32_t* __restrict__ slots, const unsigned long long* __restrict__ keys,
                                                   uint32_t n, unsigned long long* __restrict__ vals, uint8_t* __restrict__ nulls,
                                                   OrderRange* __restrict__ ranges) {
  unsigned long long smin = ~0ull, smax = 0ull, kmin = ~0ull, kmax = 0ull;
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const unsigned long long s = slots[i], k = keys[i];
    vals[i] = s;
    vals[size_t(n) + i] = k;
    nulls[i] = 0;
    nulls[size_t(n) + i] = 0;
    smin = min(smin, s); smax = max(smax, s);
    kmin = min(kmin, k); kmax = max(kmax, k);
  }
  for (int o = 16; o > 0; o >>= 1) {
    smin = min(smin, __shfl_xor_sync(0xffffffffu, smin, o));
    smax = max(smax, __shfl_xor_sync(0xffffffffu, smax, o));
    kmin = min(kmin, __shfl_xor_sync(0xffffffffu, kmin, o));
    kmax = max(kmax, __shfl_xor_sync(0xffffffffu, kmax, o));
  }
  if ((threadIdx.x & 31) == 0 && smin <= smax) {
    atomicMin(&ranges[0].min, smin);
    atomicMax(&ranges[0].max, smax);
    atomicOr(&ranges[0].has_value, 1u);
    atomicMin(&ranges[1].min, kmin);
    atomicMax(&ranges[1].max, kmax);
    atomicOr(&ranges[1].has_value, 1u);
  }
}

struct PctPickAgg {
  double p;              // PERCENTILE_CONT: the fraction
  uint8_t median;        // 1: MEDIAN
  uint8_t acc_slot;      // the aggregate's accumulator array
  uint8_t _pad[6];
};
struct PctPickArgs {
  const unsigned long long* vals;   // [2][n]: group slot, order key (k_pct_stage)
  const uint32_t* order;            // pair positions in (slot, key) order; nullptr: the positions are in order already
  const uint32_t* out_slot;         // the non-empty group slots
  unsigned long long* acc;
  uint32_t n, n_out, nslots, naggs, f64;
  uint32_t _pad;
  PctPickAgg a[kMaxAggs];
};

__global__ void __launch_bounds__(256) k_pct_pick(const __grid_constant__ PctPickArgs a) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= a.n_out) return;
  const uint32_t slot = a.out_slot[i];
  auto at = [&](uint32_t r) { return a.order ? a.order[r] : r; };
  // [lo, hi): the sorted positions holding this group's pairs
  uint32_t lo = 0, hi = a.n;
  while (lo < hi) {
    const uint32_t m = lo + ((hi - lo) >> 1);
    if (a.vals[at(m)] < slot) lo = m + 1; else hi = m;
  }
  uint32_t end = a.n;
  hi = lo;
  while (hi < end) {
    const uint32_t m = hi + ((end - hi) >> 1);
    if (a.vals[at(m)] <= slot) hi = m + 1; else end = m;
  }
  if (hi == lo) return;   // every input of the group was NULL: agg_output_value reports NULL from the non-NULL count
  const unsigned long long* keys = a.vals + a.n;
  auto key = [&](uint64_t r) { return uint64_t(keys[at(lo + uint32_t(r))]); };
  for (uint32_t g = 0; g < a.naggs; g++) {
    const PctPickAgg& pa = a.a[g];
    a.acc[size_t(1 + pa.acc_slot) * a.nslots + slot] = pct_pick(key, hi - lo, pa.median != 0, pa.p, a.f64 != 0);
  }
}

}  // namespace pqb
