// MEDIAN / PERCENTILE_CONT: the pure (host + device) pieces.  A value travels as its ORDER BY key (order_keys.cuh:
// order_encode, ascending) so that sorting (group slot, key) pairs sorts every group's values in the query's value
// order; k_pct_pick decodes the keys at the ranks it needs and computes the result with the functions below.
//
// Rules restated from DataFusion 53 (not vendored here, so not checked):
//   median(x)            n odd: the middle value.  n even: Int64 (lo + hi) wrapping, / 2 truncating toward zero
//                        (add_wrapping(..).div_wrapping(2)); Float64 (lo + hi) / 2.  Output type = input type.
//   percentile_cont(x,p) h = p * (n - 1), lo = floor(h), f = h - lo over the values as f64: v[lo] when f == 0, else
//                        v[lo] + f * (v[lo + 1] - v[lo]).  Output Float64.
// Float64 operations on NaN follow x86-64 SSE, where DataFusion usually runs: a NaN operand comes back quieted (the
// first one when both are), an invalid operation (inf - inf, 0 * inf) gives the default NaN 0xfff8000000000000.  The
// device's own NaN rule differs (one canonical NaN), so the operations are spelled out here and the GPU and a CPU agree
// bit for bit.  Every product and sum is rounded on its own (no FMA contraction).
//
// Free of CUDA-only constructs: tests/test_percentile_core.py runs the same code on the CPU through
// tools/order_keys_host.cpp.
#pragma once
#include <cmath>
#include <cstdint>
#include <cstring>

#include "order_keys.cuh"

namespace pqb {

constexpr uint64_t kF64QuietBit = 1ull << 51;
constexpr uint64_t kF64DefaultNaN = 0xfff8000000000000ull;   // x86-64's "real indefinite"

PQ_HD double pct_f64(uint64_t b) {
#ifdef __CUDA_ARCH__
  return __longlong_as_double((long long)b);
#else
  double d;
  std::memcpy(&d, &b, 8);
  return d;
#endif
}
PQ_HD uint64_t pct_bits(double d) {
#ifdef __CUDA_ARCH__
  return (uint64_t)__double_as_longlong(d);
#else
  uint64_t b;
  std::memcpy(&b, &d, 8);
  return b;
#endif
}
PQ_HD bool pct_is_nan(uint64_t b) { return (b & 0x7fffffffffffffffull) > 0x7ff0000000000000ull; }

// a op b with x86-64 SSE NaN results; op: 0 add, 1 sub, 2 mul, 3 div
PQ_HD uint64_t pct_f64_op(uint64_t a, uint64_t b, int op) {
  if (pct_is_nan(a)) return a | kF64QuietBit;
  if (pct_is_nan(b)) return b | kF64QuietBit;
  const double x = pct_f64(a), y = pct_f64(b);
  double r;
#ifdef __CUDA_ARCH__
  r = op == 0 ? __dadd_rn(x, y) : op == 1 ? __dsub_rn(x, y) : op == 2 ? __dmul_rn(x, y) : __ddiv_rn(x, y);
#else
  r = op == 0 ? x + y : op == 1 ? x - y : op == 2 ? x * y : x / y;
#endif
  const uint64_t rb = pct_bits(r);
  return pct_is_nan(rb) ? kF64DefaultNaN : rb;
}

// an ascending order key (order_encode(bits, enc, false)) back to the value's bits
PQ_HD uint64_t pct_key_bits(uint64_t key, bool f64) {
  const uint64_t v = key ^ (1ull << 63);
  return f64 ? f64_from_order_key(int64_t(v)) : v;
}
// the value as f64 bits (Int64 converted, rounding to nearest)
PQ_HD uint64_t pct_as_f64(uint64_t bits, bool f64) {
  return f64 ? bits : pct_bits(double(int64_t(bits)));
}

// median of an even number of values: lo / hi the two middle ones (value bits)
PQ_HD uint64_t pct_median_even(uint64_t lo, uint64_t hi, bool f64) {
  if (f64) return pct_f64_op(pct_f64_op(lo, hi, 0), pct_bits(2.0), 3);
  const int64_t s = int64_t(lo + hi);   // wrapping add
  return uint64_t(s / 2);               // C++ division truncates toward zero
}

// rank of percentile p over n > 0 values: lo and the fraction f (bits of the f64)
PQ_HD void pct_rank(double p, uint64_t n, uint64_t& lo, double& f) {
  const double nm1 = double(n - 1);
#ifdef __CUDA_ARCH__
  const double h = __dmul_rn(p, nm1);
  const double fl = floor(h);
  f = __dsub_rn(h, fl);
#else
  const double h = p * nm1;
  const double fl = std::floor(h);
  f = h - fl;
#endif
  lo = uint64_t(fl);
  if (lo >= n) { lo = n - 1; f = 0.0; }   // p * (n - 1) never rounds above n - 1; kept as a bound for the reads
}

// v[lo] + f * (v[lo + 1] - v[lo]), all f64 bits; f == 0 returns vlo (no inf - inf at an exact rank)
PQ_HD uint64_t pct_interpolate(uint64_t vlo, uint64_t vhi, double f) {
  if (f == 0.0) return vlo;
  const uint64_t d = pct_f64_op(vhi, vlo, 1);
  const uint64_t t = pct_f64_op(pct_bits(f), d, 2);
  return pct_f64_op(vlo, t, 0);
}

// one aggregate of one group: n > 0 ascending keys, key(i) reads the i-th.  MEDIAN (p unused) -> value bits of the
// input type, PERCENTILE_CONT -> f64 bits.  k_pct_pick runs this per group; the CPU tests run it on edge vectors.
template <typename KeyAt>
PQ_HD uint64_t pct_pick(const KeyAt& key, uint64_t n, bool median, double p, bool f64) {
  if (median) {
    const uint64_t lo = pct_key_bits(key((n - 1) / 2), f64);
    if (n & 1) return lo;
    return pct_median_even(lo, pct_key_bits(key(n / 2), f64), f64);
  }
  uint64_t r;
  double f;
  pct_rank(p, n, r, f);
  const uint64_t vlo = pct_as_f64(pct_key_bits(key(r), f64), f64);
  if (f == 0.0) return vlo;
  return pct_interpolate(vlo, pct_as_f64(pct_key_bits(key(r + 1), f64), f64), f);
}

}  // namespace pqb
