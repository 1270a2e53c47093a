// Pure (host + device) pieces of the Parquet page decoder: RLE / bit-packed
// hybrid run walking, bit extraction, PLAIN value loads, order-preserving f64
// keys.  Restates, for one GPU thread at a time, what parquet 58.1.0's
// RleDecoder / BitReader / PlainDecoder do for the reference
// (SURVEY.md §8 row a10; format: Apache Parquet "Encodings" spec).
//
// Everything here is free of CUDA-only constructs so the same code is exercised
// on the CPU by tests/test_decode_core.py through tools/decode_core_host.cpp
// (test harness only; it is never linked into libparseable_b200.so).
#pragma once
#include <cmath>
#include <cstdint>
#include <cstring>

#include "device_structs.hpp"

#if defined(__CUDACC__)
#define PQ_HD __host__ __device__ __forceinline__
#else
#define PQ_HD inline
#endif

namespace pqb {

// One encoded stream of a page: either the definition levels (bw = 1) or the
// dictionary indices (bw = page bit width).  Offsets are arena byte offsets.
struct StreamState {
  uint64_t pos;            // next run header
  uint64_t end;            // end of the stream
  uint64_t data_pos;       // bit-packed run: first byte of the run's packed data
  uint32_t run_remaining;  // values left in the current run
  uint32_t run_consumed;   // values already taken from the current bit-packed run
  uint32_t rle_value;
  uint8_t kind;            // 0 RLE, 1 bit-packed
  uint8_t bw;
  uint16_t _pad;
};

// A staged copy of arena bytes [arena_base, arena_base + len) (shared memory on the GPU).
struct Window {
  const uint8_t* data;
  uint64_t arena_base;
  uint32_t len;
};

PQ_HD void stream_init(StreamState& s, uint64_t begin, uint64_t end, uint32_t bw) {
  s.pos = begin; s.end = end; s.data_pos = begin;
  s.run_remaining = 0; s.run_consumed = 0; s.rle_value = 0; s.kind = 0; s.bw = uint8_t(bw); s._pad = 0;
}

// First arena byte the stream still needs (where the next window must start).
PQ_HD uint64_t stream_window_start(const StreamState& s) {
  if (s.run_remaining != 0 && s.kind == 1)
    return s.data_pos + ((uint64_t(s.run_consumed) * s.bw) >> 3);
  return s.pos;
}

// Bytes a window must hold so that `rows` values of a bw-bit stream always fit,
// whatever the run structure: the worst legal case is one header + one value per
// run (RLE runs of length 1).
PQ_HD uint32_t stream_window_cap(uint32_t rows, uint32_t bw) {
  uint32_t per_value = 1 + ((bw + 7) >> 3);
  return ((rows * per_value + 64 + 15) & ~15u) + 16;
}

// Walk run headers until `need` values are covered, the directory is full or the
// window ends.  Appends DirEntry records; returns the values covered.
PQ_HD uint32_t walk_stream(StreamState& s, const Window& w, uint32_t need, DirEntry* dir,
                           uint32_t& nent, uint32_t max_ent) {
  // All arithmetic is 32-bit and window relative (windows are < 64 KiB); the 64-bit arena
  // offsets of the persistent state are rebuilt on exit.  rdata may wrap below the window for a
  // run whose data began before it (only the not-yet-consumed tail must be inside).
  uint32_t covered = 0;
  const uint32_t wlen = w.len;
  const uint32_t bw = s.bw;
  const uint64_t end_rel = s.end - w.arena_base;
  const uint32_t rend = end_rel > 0xffffffffull ? 0xffffffffu : uint32_t(end_rel);
  uint32_t rp = uint32_t(s.pos - w.arena_base);          // next header
  int32_t rdata = int32_t(int64_t(s.data_pos) - int64_t(w.arena_base));  // current bit-packed run's data
  uint32_t remaining = s.run_remaining, consumed = s.run_consumed, rle_value = s.rle_value, kind = s.kind;
  uint32_t chunks = nent ? uint32_t(dir[nent - 1].chunk0) + ((uint32_t(dir[nent - 1].count) + 31u) >> 5) : 0u;
  while (covered < need) {
    if (remaining == 0) {
      // parse the next header: ULEB128, at most 5 bytes for a 32-bit count
      uint32_t p = rp;
      if (p >= rend) break;  // stream exhausted (corrupt page or padding); caller flags it
      uint32_t h = 0;
      int shift = 0;
      bool ok = false;
      while (p < wlen && p < rend && shift < 35) {
        uint32_t b = w.data[p];
        p++;
        h |= (b & 0x7f) << shift;
        shift += 7;
        if (!(b & 0x80)) { ok = true; break; }
      }
      if (!ok) break;  // header straddles the window end
      if (h & 1) {
        uint32_t groups = h >> 1;
        kind = 1;
        remaining = groups * 8;
        consumed = 0;
        rdata = int32_t(p);
        rp = p + groups * bw;
        if (groups == 0) continue;
      } else {
        uint32_t vbytes = (bw + 7) >> 3;
        if (p + vbytes > wlen) break;
        uint32_t v = 0;
        for (uint32_t i = 0; i < vbytes; i++) v |= uint32_t(w.data[p + i]) << (8 * i);
        kind = 0;
        remaining = h >> 1;
        consumed = 0;
        rle_value = v;
        rp = p + vbytes;
        if (remaining == 0) continue;
      }
    }
    if (nent >= max_ent) break;
    uint32_t take = remaining;
    if (take > need - covered) take = need - covered;
    if (take > uint32_t(kDirEntryMaxValues)) take = kDirEntryMaxValues;
    DirEntry e;
    e.start = covered;
    if (kind == 1) {
      // the bits of values [consumed, consumed+take) must lie inside the window
      int32_t avail_bits = (int32_t(wlen) - rdata) * 8;   // rdata may be negative: more bits, all before `consumed`
      int32_t first_bit = int32_t(consumed * bw);
      if (int32_t((consumed + take) * bw) > avail_bits) {
        if (bw == 0 || avail_bits <= first_bit) break;
        uint32_t fit = uint32_t(avail_bits) / bw;
        if (fit <= consumed) break;
        take = fit - consumed;
      }
      e.kind = 1;
      e.payload = uint32_t(rdata * 8 + first_bit);   // >= 0: the window starts at or before the first unread bit
    } else {
      e.kind = 0;
      e.payload = rle_value;
    }
    e.count = uint16_t(take);
    e.chunk0 = uint8_t(chunks);
    e._pad = 0;
    chunks += (take + 31u) >> 5;
    dir[nent++] = e;
    covered += take;
    remaining -= take;
    consumed += take;
  }
  s.pos = w.arena_base + rp;
  s.data_pos = uint64_t(int64_t(w.arena_base) + rdata);
  s.run_remaining = remaining;
  s.run_consumed = consumed;
  s.rle_value = rle_value;
  s.kind = uint8_t(kind);
  return covered;
}

// ---- DELTA_BINARY_PACKED (Parseable's p_timestamp, streams.rs:587-590) ----------------------
// header: block size, miniblocks per block, total count, first value (zigzag); then per block:
// min delta (zigzag), one bit width per miniblock, miniblock bodies (values - min delta, bit packed).
struct DeltaState {
  int64_t last_value;       // running prefix: value of the last decoded row of this page
  int64_t min_delta;
  int64_t first_value;
  uint64_t pos;             // next unread structure (page header / block header / miniblock body)
  uint64_t end;
  uint64_t mini_data;       // body of the current miniblock
  uint32_t vals_per_mini;
  uint32_t n_mini;
  uint32_t mini_idx;        // next miniblock of the current block (== n_mini: a block header comes next)
  uint32_t mini_remaining;  // values left in the current miniblock
  uint32_t mini_consumed;
  uint32_t total_left;      // deltas left in the page
  uint8_t bws[8];
  uint8_t header_done;
  uint8_t first_pending;    // the page's first value has not been emitted yet
  uint8_t cur_bw;
  uint8_t bad;              // malformed / unsupported geometry
};

struct DeltaEntry {
  uint32_t start;      // first value (slab relative)
  uint16_t count;
  uint8_t bw;
  uint8_t kind;        // 0: packed deltas, 1: the page's first value (absolute, in min_delta)
  uint32_t bitoff;     // of the first value inside the window
  uint32_t _pad;
  int64_t min_delta;
};

PQ_HD void delta_init(DeltaState& s, uint64_t begin, uint64_t end) {
  s.last_value = 0; s.min_delta = 0; s.first_value = 0;
  s.pos = begin; s.end = end; s.mini_data = begin;
  s.vals_per_mini = 0; s.n_mini = 0; s.mini_idx = 0; s.mini_remaining = 0; s.mini_consumed = 0; s.total_left = 0;
  for (int i = 0; i < 8; i++) s.bws[i] = 0;
  s.header_done = 0; s.first_pending = 0; s.cur_bw = 0; s.bad = 0;
}

PQ_HD uint64_t delta_window_start(const DeltaState& s) {
  if (s.header_done && s.mini_remaining != 0) return s.mini_data + ((uint64_t(s.mini_consumed) * s.cur_bw) >> 3);
  return s.pos;
}

// ULEB128 inside a window; returns false when it runs past `lim`
PQ_HD bool win_varint(const Window& w, uint32_t& p, uint32_t lim, uint64_t& out) {
  uint64_t v = 0;
  for (int shift = 0; shift < 70; shift += 7) {
    if (p >= lim) return false;
    uint32_t b = w.data[p++];
    if (shift < 64) v |= uint64_t(b & 0x7f) << shift;
    if (!(b & 0x80)) { out = v; return true; }
  }
  return false;
}

PQ_HD uint32_t walk_delta(DeltaState& s, const Window& w, uint32_t need, DeltaEntry* dir, uint32_t& nent,
                          uint32_t max_ent) {
  uint32_t covered = 0;
  if (s.bad) return 0;
  const uint64_t end_rel = s.end - w.arena_base;
  const uint32_t lim = end_rel < w.len ? uint32_t(end_rel) : w.len;   // readable bytes of the stream in this window
  if (!s.header_done) {
    uint32_t p = uint32_t(s.pos - w.arena_base);
    uint64_t bs, nm, total, fz;
    if (!win_varint(w, p, lim, bs) || !win_varint(w, p, lim, nm) || !win_varint(w, p, lim, total) ||
        !win_varint(w, p, lim, fz))
      return 0;
    if (nm == 0 || nm > 8 || bs == 0 || bs % nm != 0 || bs > (1u << 20)) { s.bad = 1; return 0; }
    s.vals_per_mini = uint32_t(bs / nm);
    s.n_mini = uint32_t(nm);
    s.mini_idx = s.n_mini;
    s.first_value = int64_t(fz >> 1) ^ -int64_t(fz & 1);
    s.first_pending = total > 0;
    s.total_left = total > 0 ? uint32_t(total - 1) : 0;
    s.pos = w.arena_base + p;
    s.header_done = 1;
  }
  while (covered < need) {
    if (nent >= max_ent) break;
    if (s.first_pending) {
      DeltaEntry e;
      e.start = covered; e.count = 1; e.bw = 0; e.kind = 1; e.bitoff = 0; e._pad = 0; e.min_delta = s.first_value;
      dir[nent++] = e;
      s.first_pending = 0;
      covered++;
      continue;
    }
    if (s.mini_remaining == 0) {
      if (s.total_left == 0) break;
      uint32_t p = uint32_t(s.pos - w.arena_base);
      if (s.mini_idx >= s.n_mini) {  // block header
        uint64_t mz;
        uint32_t q = p;
        if (!win_varint(w, q, lim, mz) || q + s.n_mini > lim) break;
        s.min_delta = int64_t(mz >> 1) ^ -int64_t(mz & 1);
        for (uint32_t i = 0; i < s.n_mini; i++) s.bws[i] = w.data[q + i];
        p = q + s.n_mini;
        s.mini_idx = 0;
      }
      s.cur_bw = s.bws[s.mini_idx];
      if (s.cur_bw > 64) { s.bad = 1; break; }
      s.mini_data = w.arena_base + p;
      s.pos = s.mini_data + (uint64_t(s.vals_per_mini) * s.cur_bw) / 8;
      s.mini_consumed = 0;
      s.mini_remaining = s.vals_per_mini < s.total_left ? s.vals_per_mini : s.total_left;
      s.mini_idx++;
    }
    uint32_t take = s.mini_remaining;
    if (take > need - covered) take = need - covered;
    int64_t rdata = int64_t(s.mini_data) - int64_t(w.arena_base);
    int64_t avail_bits = (int64_t(w.len) - rdata) * 8;
    int64_t first_bit = int64_t(s.mini_consumed) * s.cur_bw;
    if (first_bit + int64_t(take) * s.cur_bw > avail_bits) {
      if (s.cur_bw == 0 || avail_bits <= first_bit) break;
      uint32_t fit = uint32_t((avail_bits - first_bit) / s.cur_bw);
      if (fit == 0) break;
      take = fit;
    }
    DeltaEntry e;
    e.start = covered; e.count = uint16_t(take); e.bw = s.cur_bw; e.kind = 0;
    e.bitoff = uint32_t(rdata * 8 + first_bit); e._pad = 0; e.min_delta = s.min_delta;
    dir[nent++] = e;
    covered += take;
    s.mini_remaining -= take;
    s.mini_consumed += take;
    s.total_left -= take;
  }
  return covered;
}

// bw <= 64; the window keeps 8 bytes of slack so the third word is readable
PQ_HD uint64_t bp_get64(const uint32_t* words, uint32_t bitoff, uint32_t bw, uint32_t j) {
  if (bw == 0) return 0;
  uint32_t bit = bitoff + j * bw;
  uint32_t wi = bit >> 5, sh = bit & 31;
  uint64_t lo = uint64_t(words[wi]) | (uint64_t(words[wi + 1]) << 32);
  uint64_t v = lo >> sh;
  if (sh && bw + sh > 64) v |= uint64_t(words[wi + 2]) << (64 - sh);
  return bw >= 64 ? v : (v & ((1ull << bw) - 1ull));
}

// Value j of a bit-packed run whose first value starts at bit `bitoff` of a
// 4-byte aligned word array.  bw <= 32.
PQ_HD uint32_t bp_get(const uint32_t* words, uint32_t bitoff, uint32_t bw, uint32_t j) {
  uint32_t bit = bitoff + j * bw;
  uint32_t wi = bit >> 5, sh = bit & 31;
  uint32_t lo = words[wi];
  uint32_t hi = words[wi + 1];
  uint64_t both = (uint64_t(hi) << 32) | lo;
  uint32_t v = uint32_t(both >> sh);
  return bw >= 32 ? v : (v & ((1u << bw) - 1u));
}

// Unaligned little-endian 8-byte load built from two aligned 8-byte loads.  The
// arena keeps 16 bytes of slack after every chunk, so the second load is in bounds.
PQ_HD uint64_t load_u64_unaligned(const uint8_t* p) {
  uintptr_t a = reinterpret_cast<uintptr_t>(p);
  const uint64_t* q = reinterpret_cast<const uint64_t*>(a & ~uintptr_t(7));
  uint32_t sh = uint32_t(a & 7) * 8;
  uint64_t lo = q[0];
  if (sh == 0) return lo;
  uint64_t hi = q[1];
  return (lo >> sh) | (hi << (64 - sh));
}
PQ_HD uint32_t load_u32_unaligned(const uint8_t* p) {
  uintptr_t a = reinterpret_cast<uintptr_t>(p);
  const uint32_t* q = reinterpret_cast<const uint32_t*>(a & ~uintptr_t(3));
  uint32_t sh = uint32_t(a & 3) * 8;
  uint32_t lo = q[0];
  if (sh == 0) return lo;
  uint32_t hi = q[1];
  return (lo >> sh) | (hi << (32 - sh));
}

// IEEE-754 totalOrder as a signed-integer order: DataFusion / arrow-ord compare
// and min/max floats this way (SURVEY §8 rows a11, a12): -NaN < -inf < ... < -0.0 <
// +0.0 < ... < +inf < +NaN.
PQ_HD int64_t f64_order_key(uint64_t bits) {
  int64_t b = int64_t(bits);
  return b ^ int64_t(uint64_t(b >> 63) >> 1);
}
PQ_HD uint64_t f64_from_order_key(int64_t k) {
  return uint64_t(k ^ int64_t(uint64_t(k >> 63) >> 1));
}

// ---- value pages (FK_FOR): numeric dictionary pages as bit-packed values ----
// An Int64 value v is stored as the w-bit offset v - base (64-bit wrapping: base + bits gives v back exactly).  A Float64
// value v is first written as an integer k with dec_decode_f64(k, e) == v bit for bit (|k| < 2^53), then stored like an
// Int64.  A value without such a k (NaN, infinities, -0.0, subnormals, most random doubles) refuses the encoding, and its
// chunk keeps the dictionary.
//
// The decode is k / 10^e rounded to nearest: the quotient through the correctly rounded reciprocal, plus one exact FMA
// correction step (q0 = k * r, rem = k - q0 * 10^e exactly, q = q0 + rem * r).  That is the IEEE quotient for decimal
// values (tests/test_agg_forms.py compares it with IEEE division), costs two FMAs and a multiply instead of the
// division's slow-path call -- which spilled the aggregate kernel's registers -- and, above all, the encoder accepts k
// only when THIS function gives v back, so no value ever changes whatever the rounding of a corner case.
constexpr uint32_t kForMaxExp = 9;      // decimal exponents 0 .. 9 are tried
constexpr uint32_t kForMaxBits = 32;    // a chunk whose offsets need more bits keeps the dictionary
struct DecScale { double p10, rinv; };
PQ_HD DecScale dec_scale(uint32_t e) {   // 10^e is exact for e <= 22
  double p = 1.0;
  for (uint32_t i = 0; i < e; i++) p *= 10.0;
  return DecScale{p, 1.0 / p};
}
PQ_HD double f64_of_bits(uint64_t b) { double d; memcpy(&d, &b, 8); return d; }
PQ_HD uint64_t bits_of_f64(double d) { uint64_t b; memcpy(&b, &d, 8); return b; }
PQ_HD uint64_t dec_decode_f64(int64_t k, DecScale s) {
  const double x = double(k), q0 = x * s.rinv;
  return bits_of_f64(fma(fma(-q0, s.p10, x), s.rinv, q0));
}
// false: v has no k at this exponent
PQ_HD bool dec_encode_f64(uint64_t bits, DecScale s, int64_t& k) {
  if (bits == 0x8000000000000000ull) return false;   // -0.0 would come back as +0.0
  const double v = f64_of_bits(bits);
  if (!(v - v == 0.0)) return false;                 // NaN, +-inf
  const double r = rint(v * s.p10);
  if (!(fabs(r) < 9007199254740992.0)) return false; // |k| < 2^53: double(k) is exact
  k = int64_t(r);
  return dec_decode_f64(k, s) == bits;
}
PQ_HD uint64_t for_encode(int64_t v, int64_t base) { return uint64_t(v) - uint64_t(base); }
PQ_HD int64_t for_decode(int64_t base, uint32_t bits) { return int64_t(uint64_t(base) + bits); }
PQ_HD uint32_t bit_width_u64(uint64_t x) {
  uint32_t n = 0;
  while (x) { n++; x >>= 1; }
  return n;
}

// compare with PqCmp codes: 0 EQ 1 NE 2 LT 3 LE 4 GT 5 GE
PQ_HD bool cmp_i64(int64_t a, int64_t b, uint32_t op) {
  switch (op) {
    case 0: return a == b;
    case 1: return a != b;
    case 2: return a < b;
    case 3: return a <= b;
    case 4: return a > b;
    default: return a >= b;
  }
}

// bytes: lexicographic unsigned compare (arrow-ord on Utf8), returns <0, 0, >0
PQ_HD int cmp_bytes(const uint8_t* a, uint32_t na, const uint8_t* b, uint32_t nb) {
  uint32_t n = na < nb ? na : nb;
  for (uint32_t i = 0; i < n; i++) {
    if (a[i] != b[i]) return a[i] < b[i] ? -1 : 1;
  }
  return na == nb ? 0 : (na < nb ? -1 : 1);
}
PQ_HD bool cmp_result(int c, uint32_t op) {
  switch (op) {
    case 0: return c == 0;
    case 1: return c != 0;
    case 2: return c < 0;
    case 3: return c <= 0;
    case 4: return c > 0;
    default: return c >= 0;
  }
}

// 64-bit mix (splitmix64 finaliser) and FNV-style byte hash for dictionary keys.
PQ_HD uint64_t mix64(uint64_t x) {
  x ^= x >> 30; x *= 0xbf58476d1ce4e5b9ull;
  x ^= x >> 27; x *= 0x94d049bb133111ebull;
  x ^= x >> 31;
  return x;
}
PQ_HD uint64_t hash_bytes(const uint8_t* p, uint32_t n) {
  uint64_t h = 0xcbf29ce484222325ull ^ (uint64_t(n) * 0x9e3779b97f4a7c15ull);
  for (uint32_t i = 0; i < n; i++) { h ^= p[i]; h *= 0x100000001b3ull; }
  return mix64(h);
}

// ---- SQL LIKE over raw bytes (arrow-string like.rs semantics: '%' any run, '_' one
// character, ESCAPE '\').  Patterns are classified on the host; the device sees the
// cooked needle.  kinds: 0 equals, 1 starts-with, 2 ends-with, 3 contains, 4 general.
enum LikeKind : uint32_t { LIKE_EQ = 0, LIKE_PREFIX = 1, LIKE_SUFFIX = 2, LIKE_CONTAINS = 3, LIKE_GENERAL = 4 };

PQ_HD uint8_t ascii_lower(uint8_t c) { return (c >= 'A' && c <= 'Z') ? uint8_t(c + 32) : c; }

PQ_HD bool bytes_eq_ci(const uint8_t* a, const uint8_t* b, uint32_t n, bool ci) {
  for (uint32_t i = 0; i < n; i++) {
    uint8_t x = a[i], y = b[i];
    if (ci) { x = ascii_lower(x); y = ascii_lower(y); }
    if (x != y) return false;
  }
  return true;
}

// utf-8 aware advance by one character
PQ_HD uint32_t utf8_next(const uint8_t* s, uint32_t i, uint32_t n) {
  i++;
  while (i < n && (s[i] & 0xc0) == 0x80) i++;
  return i;
}

// General matcher on the raw pattern (with escapes), iterative with single backtrack
// point (classic wildcard algorithm).
PQ_HD bool like_general(const uint8_t* s, uint32_t n, const uint8_t* p, uint32_t m, bool ci) {
  uint32_t si = 0, pi = 0;
  uint32_t star_p = 0xffffffffu, star_s = 0;
  while (si < n) {
    bool adv = false;
    if (pi < m) {
      uint8_t c = p[pi];
      if (c == '%') { star_p = ++pi; star_s = si; continue; }
      if (c == '_') { si = utf8_next(s, si, n); pi++; continue; }
      uint32_t lit = pi;
      if (c == '\\' && pi + 1 < m) lit = pi + 1;
      uint8_t x = s[si], y = p[lit];
      if (ci) { x = ascii_lower(x); y = ascii_lower(y); }
      if (x == y) { si++; pi = lit + 1; adv = true; }
    }
    if (adv) continue;
    if (star_p == 0xffffffffu) return false;
    star_s = utf8_next(s, star_s, n);
    si = star_s;
    pi = star_p;
  }
  while (pi < m && p[pi] == '%') pi++;
  return pi == m;
}

PQ_HD bool like_match(const uint8_t* s, uint32_t n, const uint8_t* needle, uint32_t m, uint32_t kind, bool ci) {
  switch (kind) {
    case LIKE_EQ: return n == m && bytes_eq_ci(s, needle, m, ci);
    case LIKE_PREFIX: return n >= m && bytes_eq_ci(s, needle, m, ci);
    case LIKE_SUFFIX: return n >= m && bytes_eq_ci(s + (n - m), needle, m, ci);
    case LIKE_CONTAINS: {
      if (m == 0) return true;
      if (n < m) return false;
      for (uint32_t i = 0; i + m <= n; i++)
        if (bytes_eq_ci(s + i, needle, m, ci)) return true;
      return false;
    }
    default: return like_general(s, n, needle, m, ci);
  }
}

}  // namespace pqb
