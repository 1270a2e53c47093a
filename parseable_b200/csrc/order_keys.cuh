// ORDER BY over aggregate results: the pure (host + device) pieces.  Every sort term of an output row becomes one
// order-preserving unsigned 64-bit value (plus a NULL flag); the terms of a query are then packed MSB-first into as few
// 64-bit words as their value ranges need, so that comparing rows is comparing word tuples.
//
// Value order restated from arrow-ord's sort (what DataFusion's SortExec uses; not vendored here, so not checked):
//   Int64 / Timestamp(ms) signed; Float64 by IEEE totalOrder (-NaN < -inf < ... < -0.0 < +0.0 < ... < +inf < +NaN, the
//   f64_order_key the filters use); Utf8 bytewise, a prefix before any longer string; Boolean false < true; NULLs first
//   or last as the term asks, in either direction.
//
// Free of CUDA-only constructs: tests/test_order_keys.py runs the same code on the CPU through tools/order_keys_host.cpp.
#pragma once
#include <algorithm>
#include <cstdint>
#include <vector>

#include "decode_core.cuh"

namespace pqb {

constexpr int kMaxOrder = 8;                 // ORDER BY terms of one query
constexpr int kMaxOrderWords = 9;            // 8 terms x (64 value bits + 1 NULL bit) = 520 bits
constexpr uint32_t kOrderCta = 4096;         // results up to this many rows are sorted by one CTA in shared memory

// how a term's raw 64 bits become an order-preserving unsigned value
enum OrderEnc : uint8_t {
  OE_I64 = 0,   // signed 64-bit integer (Int64, Timestamp, COUNT, SUM of Int64)
  OE_F64 = 1,   // IEEE double bits (totalOrder)
  OE_RAW = 2    // already an unsigned rank (string rank, boolean, DATE_BIN bin number)
};

PQ_HD uint64_t order_encode(uint64_t bits, uint32_t enc, bool desc) {
  uint64_t v = bits;
  if (enc == OE_I64) v = bits ^ (1ull << 63);
  else if (enc == OE_F64) v = uint64_t(f64_order_key(bits)) ^ (1ull << 63);
  return desc ? ~v : v;
}

// the non-NULL values of a term range over [min, max] (after order_encode); has_value == 0: every row is NULL
struct OrderRange {
  unsigned long long min, max;
  uint32_t has_null, has_value;
};

// one term of the packed key: an optional NULL bit, then (value - min) in value_bits bits, starting `pos` bits below
// the most significant bit of word 0
struct OrderPackTerm {
  uint64_t min;
  uint32_t pos;
  uint8_t null_bit;      // 1: the term carries a NULL flag bit (it met a NULL)
  uint8_t value_bits;    // 0..64
  uint8_t nulls_first;
  uint8_t _pad;
};
struct OrderPack {
  uint32_t nterms, nwords, total_bits, _pad;
  OrderPackTerm t[kMaxOrder];
};

PQ_HD uint32_t order_bits_for(uint64_t span) {   // bits needed for 0..span
  uint32_t b = 0;
  while (b < 64 && (span >> b) != 0) b++;
  return b;
}

// terms in ORDER BY order, most significant first; nulls_first[t] as the query asks
PQ_HD void order_pack_plan(const OrderRange* r, const uint8_t* nulls_first, uint32_t nterms, OrderPack& p) {
  p.nterms = nterms;
  uint32_t pos = 0;
  for (uint32_t t = 0; t < nterms; t++) {
    OrderPackTerm& pt = p.t[t];
    pt.nulls_first = nulls_first[t];
    pt.null_bit = r[t].has_null ? 1 : 0;
    pt.min = r[t].has_value ? r[t].min : 0;
    pt.value_bits = uint8_t(r[t].has_value ? order_bits_for(r[t].max - r[t].min) : 0);
    pt.pos = pos;
    pt._pad = 0;
    pos += pt.null_bit + pt.value_bits;
  }
  p.total_bits = pos;
  p.nwords = (pos + 63) / 64;
  p._pad = 0;
}

// OR the low `w` bits of v into the word tuple, its most significant bit `pos` bits below the top of word 0; a field may
// straddle two words
PQ_HD void order_put_bits(uint64_t* words, uint32_t pos, uint32_t w, uint64_t v) {
  if (w == 0) return;
  const uint32_t wi = pos >> 6, off = pos & 63;
  if (off + w <= 64) {
    words[wi] |= v << (64 - off - w);
  } else {
    const uint32_t lo = off + w - 64;   // bits that spill into the next word
    words[wi] |= v >> lo;
    words[wi + 1] |= v << (64 - lo);
  }
}

// one row: encoded values and NULL flags of every term -> p.nwords words (the caller zeroes them)
PQ_HD void order_pack_row(const OrderPack& p, const uint64_t* vals, const uint8_t* nulls, uint64_t* words) {
  for (uint32_t t = 0; t < p.nterms; t++) {
    const OrderPackTerm& pt = p.t[t];
    const bool isnull = nulls[t] != 0;
    if (pt.null_bit) order_put_bits(words, pt.pos, 1, (isnull != (pt.nulls_first != 0)) ? 1u : 0u);
    if (!isnull) order_put_bits(words, pt.pos + pt.null_bit, pt.value_bits, vals[t] - pt.min);
  }
}

// host only: the bytewise rank of every value of a key dictionary (offsets[card + 1] into bytes), a shorter prefix
// first.  Group ids are numbered hot-first, not in value order; ORDER BY on a Utf8 key sorts by these ranks.
inline void order_string_ranks(const uint32_t* offs, const uint8_t* bytes, uint32_t card, uint32_t* rank) {
  std::vector<uint32_t> ids(card);
  for (uint32_t i = 0; i < card; i++) ids[i] = i;
  std::sort(ids.begin(), ids.end(), [&](uint32_t a, uint32_t b) {
    const int c = cmp_bytes(bytes + offs[a], offs[a + 1] - offs[a], bytes + offs[b], offs[b + 1] - offs[b]);
    return c != 0 ? c < 0 : a < b;
  });
  for (uint32_t i = 0; i < card; i++) rank[ids[i]] = i;
}

}  // namespace pqb
