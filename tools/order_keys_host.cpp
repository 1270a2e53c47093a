// TEST HARNESS ONLY: exposes the pure host/device ORDER BY key functions of order_keys.cuh to tests/test_order_keys.py,
// run in the same sequence as k_order_encode -> pack plan -> k_order_pack, and the MEDIAN / PERCENTILE_CONT arithmetic of
// percentile_core.cuh to tests/test_percentile_core.py.  Never linked into libparseable_b200.so.
#include <cstdint>
#include <cstring>
#include <vector>
#include "order_keys.cuh"
#include "percentile_core.cuh"
using namespace pqb;

extern "C" {
uint64_t ok_encode(uint64_t bits, uint32_t enc, int desc) { return order_encode(bits, enc, desc != 0); }

// raw[t * n + i]: the term's raw 64 bits (Int64, Float64 bits, or an unsigned rank); nulls[t * n + i] != 0: NULL.
// Writes words[i * kMaxOrderWords + k] and the plan as nwords, total_bits, then per term {pos, null_bit, value_bits};
// returns nwords.
int32_t ok_pack(uint32_t n, uint32_t nterms, const uint64_t* raw, const uint8_t* nulls, const uint8_t* enc, const uint8_t* desc,
                const uint8_t* nulls_first, uint64_t* words, uint32_t* plan_out) {
  if (nterms > uint32_t(kMaxOrder)) return -1;
  std::vector<uint64_t> vals(size_t(n) * nterms);
  std::vector<OrderRange> r(nterms, OrderRange{~0ull, 0ull, 0u, 0u});
  for (uint32_t t = 0; t < nterms; t++)
    for (uint32_t i = 0; i < n; i++) {
      const uint64_t v = order_encode(raw[size_t(t) * n + i], enc[t], desc[t] != 0);
      vals[size_t(t) * n + i] = v;
      if (nulls[size_t(t) * n + i]) { r[t].has_null = 1; continue; }
      r[t].has_value = 1;
      if (v < r[t].min) r[t].min = v;
      if (v > r[t].max) r[t].max = v;
    }
  OrderPack p{};
  order_pack_plan(r.data(), nulls_first, nterms, p);
  uint64_t v[kMaxOrder];
  uint8_t nl[kMaxOrder];
  for (uint32_t i = 0; i < n; i++) {
    for (uint32_t t = 0; t < nterms; t++) { v[t] = vals[size_t(t) * n + i]; nl[t] = nulls[size_t(t) * n + i]; }
    uint64_t* w = words + size_t(i) * kMaxOrderWords;
    std::memset(w, 0, kMaxOrderWords * 8);
    order_pack_row(p, v, nl, w);
  }
  plan_out[0] = p.nwords;
  plan_out[1] = p.total_bits;
  for (uint32_t t = 0; t < nterms; t++) {
    plan_out[2 + 3 * t] = p.t[t].pos;
    plan_out[3 + 3 * t] = p.t[t].null_bit;
    plan_out[4 + 3 * t] = p.t[t].value_bits;
  }
  return int32_t(p.nwords);
}

void ok_string_ranks(const uint32_t* offs, const uint8_t* bytes, uint32_t card, uint32_t* rank) {
  order_string_ranks(offs, bytes, card, rank);
}

uint32_t ok_max_words() { return kMaxOrderWords; }

// MEDIAN / PERCENTILE_CONT of one group as k_pct_pick computes it: keys[0, n) are the group's ascending order keys
// (ok_encode(bits, OE_I64 | OE_F64, 0)); median != 0: MEDIAN, else PERCENTILE_CONT(p).  Returns the result's bits.
uint64_t pk_pick(const uint64_t* keys, uint64_t n, int median, double p, int f64) {
  return pct_pick([&](uint64_t i) { return keys[i]; }, n, median != 0, p, f64 != 0);
}
uint64_t pk_key_bits(uint64_t key, int f64) { return pct_key_bits(key, f64 != 0); }
uint64_t pk_f64_op(uint64_t a, uint64_t b, int op) { return pct_f64_op(a, b, op); }
}
