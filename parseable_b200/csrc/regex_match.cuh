// The DFA walk of PQ_OP_REGEX, for host and device (regex_compile.cpp writes the blob).
//
// Blob layout (8-byte aligned where it sits in the literal pool):
//   RxHeader                         16 bytes
//   uint8_t  cls[256]                byte -> equivalence class
//   uint16_t next[nstates][nclasses] transitions
//   uint8_t  eot[(nstates + 7) / 8]  bit s: state s accepts at the end of the text ($, \z)
// State 0 is the dead state, state 1 the absorbing matched state: the walk stops at either.
#pragma once
#include <cstdint>

#ifndef PQ_HD
#ifdef __CUDACC__
#define PQ_HD __host__ __device__ __forceinline__
#else
#define PQ_HD inline
#endif
#endif

namespace pqb {

struct RxHeader {
  uint32_t nstates, nclasses, start, bytes;   // bytes: the whole blob
};
constexpr uint32_t kRxDead = 0, kRxMatched = 1;
constexpr uint32_t kRxClsOff = 16, kRxNextOff = 16 + 256;

PQ_HD uint32_t rx_ld8(const uint8_t* p) {
#ifdef __CUDA_ARCH__
  return __ldg(p);
#else
  return *p;
#endif
}
PQ_HD uint32_t rx_ld16(const uint16_t* p) {
#ifdef __CUDA_ARCH__
  return __ldg(p);
#else
  return *p;
#endif
}
PQ_HD uint32_t rx_ld32(const uint32_t* p) {
#ifdef __CUDA_ARCH__
  return __ldg(p);
#else
  return *p;
#endif
}

// TRUE when some substring of s[0, n) matches (the unanchored `.*?` prefix is part of the DFA)
PQ_HD bool regex_match(const uint8_t* s, uint32_t n, const uint8_t* blob) {
  const uint32_t* h = reinterpret_cast<const uint32_t*>(blob);
  const uint32_t nclasses = rx_ld32(h + 1);
  uint32_t st = rx_ld32(h + 2);
  const uint8_t* cls = blob + kRxClsOff;
  const uint16_t* next = reinterpret_cast<const uint16_t*>(blob + kRxNextOff);
  for (uint32_t i = 0; i < n && st > kRxMatched; i++) st = rx_ld16(next + st * nclasses + rx_ld8(cls + s[i]));
  if (st <= kRxMatched) return st == kRxMatched;
  const uint8_t* eot = blob + kRxNextOff + size_t(rx_ld32(h)) * nclasses * 2;
  return (rx_ld8(eot + (st >> 3)) >> (st & 7)) & 1u;
}

}  // namespace pqb
