// The membership set of PQ_OP_IN: built on the host (query.cu, tools/in_set_host.cpp), probed on host and device.
//
// Blob layout (8-byte aligned where it sits in the literal pool):
//   InSetHeader                      16 bytes
//   numeric (kind 0): uint64_t slots[cap]    the values' 8 bytes (Int64 / Timestamp / Date32 widened, Float64 bits);
//                                            kInSetEmpty marks a free slot, and header.has_empty says whether that one
//                                            value is itself a member
//   bytes (kind 1):   InSetSlot slots[cap]   (hash_bytes, pool offset, length); length kInSetFree marks a free slot
//                     uint8_t pool[]         the members' bytes
// Open addressing with linear probing over a power-of-two table at most half full, so every probe ends at a free slot.
// The hashes are those of GROUP BY key interning (decode_core.cuh).
#pragma once
#include <cstdint>

#include <algorithm>
#include <cstring>
#include <vector>

#include "decode_core.cuh"

namespace pqb {

struct InSetHeader {
  uint32_t kind;        // 0 numeric, 1 bytes
  uint32_t mask;        // cap - 1
  uint32_t has_empty;   // numeric: kInSetEmpty is a member
  uint32_t pool_bytes;  // bytes: size of the pool behind the slots
};
struct InSetSlot {
  uint64_t hash;
  uint32_t off, len;
};
constexpr uint64_t kInSetEmpty = 0x7ff4a3c5e1b20d96ull;   // a NaN payload no writer is known to produce
constexpr uint32_t kInSetFree = 0xffffffffu;
constexpr uint32_t kInSetMaxElems = 1u << 20;
constexpr uint64_t kInSetMaxBytes = 64ull << 20;

PQ_HD uint64_t in_ld64(const uint64_t* p) {
#ifdef __CUDA_ARCH__
  return __ldg(reinterpret_cast<const unsigned long long*>(p));
#else
  return *p;
#endif
}
PQ_HD uint32_t in_ld32(const uint32_t* p) {
#ifdef __CUDA_ARCH__
  return __ldg(p);
#else
  return *p;
#endif
}

// Is the 8-byte value v a member of a numeric set?
PQ_HD bool in_set_has_u64(const uint8_t* blob, uint64_t v) {
  const uint32_t* h = reinterpret_cast<const uint32_t*>(blob);
  if (v == kInSetEmpty) return in_ld32(h + 2) != 0;
  const uint32_t mask = in_ld32(h + 1);
  const uint64_t* slots = reinterpret_cast<const uint64_t*>(blob + sizeof(InSetHeader));
  for (uint32_t i = uint32_t(mix64(v)) & mask;; i = (i + 1) & mask) {
    const uint64_t s = in_ld64(slots + i);
    if (s == v) return true;
    if (s == kInSetEmpty) return false;
  }
}

// Are the bytes s[0, n) a member of a bytes set?
PQ_HD bool in_set_has_bytes(const uint8_t* blob, const uint8_t* s, uint32_t n) {
  const uint32_t mask = in_ld32(reinterpret_cast<const uint32_t*>(blob) + 1);
  const InSetSlot* slots = reinterpret_cast<const InSetSlot*>(blob + sizeof(InSetHeader));
  const uint8_t* pool = blob + sizeof(InSetHeader) + (uint64_t(mask) + 1) * sizeof(InSetSlot);
  const uint64_t hs = hash_bytes(s, n);
  for (uint32_t i = uint32_t(hs) & mask;; i = (i + 1) & mask) {
    const uint32_t len = in_ld32(&slots[i].len);
    if (len == kInSetFree) return false;
    if (len == n && in_ld64(&slots[i].hash) == hs) {
      const uint8_t* p = pool + in_ld32(&slots[i].off);
      uint32_t k = 0;
      while (k < n && p[k] == s[k]) k++;
      if (k == n) return true;
    }
  }
}

// Either kind: a bytes set reads s[0, n), a numeric one reads v
PQ_HD bool in_set_has(const uint8_t* blob, const uint8_t* s, uint32_t n, uint64_t v) {
  return in_ld32(reinterpret_cast<const uint32_t*>(blob)) ? in_set_has_bytes(blob, s, n) : in_set_has_u64(blob, v);
}

// ---- building a set (host only) ----
// table size: the smallest power of two at least twice the number of distinct members (load factor <= 1/2)
inline uint32_t in_set_cap(size_t n) {
  uint32_t cap = 2;
  while (cap < 2 * n) cap <<= 1;
  return cap;
}

// A numeric set of the values v[0, n) (duplicates allowed)
inline std::vector<uint8_t> in_set_build_u64(const uint64_t* v, size_t n) {
  std::vector<uint64_t> u(v, v + n);
  std::sort(u.begin(), u.end());
  u.erase(std::unique(u.begin(), u.end()), u.end());
  InSetHeader hd{0, 0, 0, 0};
  const auto e = std::find(u.begin(), u.end(), kInSetEmpty);
  if (e != u.end()) { hd.has_empty = 1; u.erase(e); }
  const uint32_t cap = in_set_cap(u.size());
  hd.mask = cap - 1;
  std::vector<uint8_t> blob(sizeof(InSetHeader) + size_t(cap) * 8);
  std::memcpy(blob.data(), &hd, sizeof(hd));
  uint64_t* slots = reinterpret_cast<uint64_t*>(blob.data() + sizeof(InSetHeader));
  std::fill(slots, slots + cap, kInSetEmpty);
  for (uint64_t x : u) {
    uint32_t i = uint32_t(mix64(x)) & hd.mask;
    while (slots[i] != kInSetEmpty) i = (i + 1) & hd.mask;
    slots[i] = x;
  }
  return blob;
}

// A bytes set of the strings (p[k], len[k]), k < n (duplicates allowed)
inline std::vector<uint8_t> in_set_build_bytes(const uint8_t* const* p, const uint32_t* len, size_t n) {
  // distinct members first, so that the load factor counts them only
  std::vector<uint32_t> ord(n);
  for (uint32_t k = 0; k < n; k++) ord[k] = k;
  auto less = [&](uint32_t a, uint32_t b) {
    const int c = std::memcmp(p[a], p[b], std::min(len[a], len[b]));
    return c != 0 ? c < 0 : len[a] < len[b];
  };
  std::sort(ord.begin(), ord.end(), less);
  ord.erase(std::unique(ord.begin(), ord.end(), [&](uint32_t a, uint32_t b) { return !less(a, b) && !less(b, a); }), ord.end());
  uint64_t pool_bytes = 0;
  for (uint32_t k : ord) pool_bytes += len[k];
  const uint32_t cap = in_set_cap(ord.size());
  InSetHeader hd{1, cap - 1, 0, uint32_t(pool_bytes)};
  std::vector<uint8_t> blob(sizeof(InSetHeader) + size_t(cap) * sizeof(InSetSlot) + pool_bytes);
  std::memcpy(blob.data(), &hd, sizeof(hd));
  InSetSlot* slots = reinterpret_cast<InSetSlot*>(blob.data() + sizeof(InSetHeader));
  for (uint32_t i = 0; i < cap; i++) slots[i] = InSetSlot{0, 0, kInSetFree};
  uint8_t* pool = blob.data() + sizeof(InSetHeader) + size_t(cap) * sizeof(InSetSlot);
  uint32_t off = 0;
  for (uint32_t k : ord) {
    const uint64_t hs = hash_bytes(p[k], len[k]);
    uint32_t i = uint32_t(hs) & hd.mask;
    while (slots[i].len != kInSetFree) i = (i + 1) & hd.mask;
    slots[i] = InSetSlot{hs, off, len[k]};
    if (len[k]) std::memcpy(pool + off, p[k], len[k]);
    off += len[k];
  }
  return blob;
}

}  // namespace pqb
