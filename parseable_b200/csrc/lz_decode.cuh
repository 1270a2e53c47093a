// LZ4_RAW (codec 7), SNAPPY (codec 1) and stored (codec 0) page decoders: one warp decodes one page.  Every lane
// parses the (tiny) sequence headers redundantly -- the loads broadcast -- and the 32 lanes share the literal / match
// copies.  k_decompress_pages (decomp_kernels.cuh) calls one function per codec.
//
// The same source compiles for the host: there every copy runs its 32 lanes one after another over the same index
// arithmetic, in ascending order, or descending under LZ_LANES_DESCENDING.  Lanes of one copy never read what another
// lane of that copy writes, so both orders give the same bytes.  tools/lz_host.cpp exposes the decoders to
// tests/test_page_codecs.py, which checks them against pyarrow's codecs on the CPU.
//
// Every length is compared against what is left of the source and of the destination (`len > sn - sp`), never as a
// sum that could wrap (page sizes are below 2^31: Parquet page headers hold them as i32).  A decoder returns true
// only when the page decodes to exactly dn bytes; it writes nothing outside d[0 .. dn).  The literal copy reads up to
// 3 bytes past a literal's end and 3 bytes below an aligned word, so the source buffer needs that much slack (table.cu
// gives the staging buffer 256 bytes).
#pragma once
#include <cstdint>

#include "zstd_decode.cuh"   // ZS_FN, zs_funnel_r

#ifndef LZ_LANES_DESCENDING
#define LZ_LANES_DESCENDING 0
#endif

namespace pqb {

#if defined(__CUDA_ARCH__)
#define LZ_SYNC() __syncwarp()
#define LZ_UNROLL _Pragma("unroll")
#else
#define LZ_SYNC() ((void)0)
#define LZ_UNROLL
#endif

ZS_FN void lz_store16(uint8_t* d, uint32_t c, uint32_t x0, uint32_t x1, uint32_t x2, uint32_t x3) {   // d 16-byte aligned
#if defined(__CUDA_ARCH__)
  reinterpret_cast<uint4*>(d)[c] = make_uint4(x0, x1, x2, x3);
#else
  uint32_t* q = reinterpret_cast<uint32_t*>(d) + size_t(c) * 4;
  q[0] = x0; q[1] = x1; q[2] = x2; q[3] = x3;
#endif
}

// literal run: `len` bytes that do not overlap, any alignment of source and destination.  A page of incompressible
// bit-packed indices or PLAIN doubles is ONE literal run of 40-160 KB handled by one warp, so the copy must keep many
// bytes in flight: the destination is walked in aligned 16-byte chunks, every lane builds its chunk from five aligned
// source words with a funnel shift (the source sits at an arbitrary byte phase), four chunks per lane and trip.
ZS_FN void lz_literal_copy_lane(uint8_t* __restrict__ d, const uint8_t* __restrict__ s, uint32_t len, uint32_t lane) {
  uint32_t head = uint32_t(-reinterpret_cast<uintptr_t>(d)) & 15u;   // bytes until d is 16-byte aligned
  if (head > len) head = len;
  if (lane < head) d[lane] = s[lane];
  d += head; s += head; len -= head;
  const uint32_t n16 = len >> 4;
  if (n16) {
    const uint32_t sh = (uint32_t(reinterpret_cast<uintptr_t>(s)) & 3u) * 8u;
    const uint32_t* sw = reinterpret_cast<const uint32_t*>(reinterpret_cast<uintptr_t>(s) & ~uintptr_t(3));
    uint32_t c = lane;
    for (; c + 3 * 32 < n16; c += 4 * 32) {
      uint32_t w[4][5];
      LZ_UNROLL
      for (int k = 0; k < 4; k++)
        LZ_UNROLL
        for (int j = 0; j < 5; j++) w[k][j] = (j < 4 || sh) ? sw[(c + k * 32) * 4 + j] : 0u;   // the fifth word only when the phase needs it (it may lie past the source)
      LZ_UNROLL
      for (int k = 0; k < 4; k++)
        lz_store16(d, c + k * 32, zs_funnel_r(w[k][0], w[k][1], sh), zs_funnel_r(w[k][1], w[k][2], sh),
                   zs_funnel_r(w[k][2], w[k][3], sh), zs_funnel_r(w[k][3], w[k][4], sh));
    }
    for (; c < n16; c += 32) {
      uint32_t w[5];
      LZ_UNROLL
      for (int j = 0; j < 5; j++) w[j] = (j < 4 || sh) ? sw[c * 4 + j] : 0u;
      lz_store16(d, c, zs_funnel_r(w[0], w[1], sh), zs_funnel_r(w[1], w[2], sh), zs_funnel_r(w[2], w[3], sh), zs_funnel_r(w[3], w[4], sh));
    }
  }
  const uint32_t done = n16 << 4;
  if (done + lane < len) d[done + lane] = s[done + lane];   // < 16 bytes left
}

// match copy with LZ77 overlap semantics: the source pattern [dp-off, dp) already exists, bytes
// beyond it repeat with period `off`
ZS_FN void lz_match_copy_lane(uint8_t* d, uint32_t dp, uint32_t off, uint32_t len, uint32_t lane) {
  if (off >= len) {
    for (uint32_t i = lane; i < len; i += 32) d[dp + i] = d[dp - off + i];
  } else {
    for (uint32_t i = lane; i < len; i += 32) d[dp + i] = d[dp - off + (i % off)];
  }
}

// the copies of the whole warp: this thread's lane on the device, all 32 lanes in turn on the host
ZS_FN void lz_literal_copy(uint8_t* __restrict__ d, const uint8_t* __restrict__ s, uint32_t len) {
#if defined(__CUDA_ARCH__)
  lz_literal_copy_lane(d, s, len, threadIdx.x & 31u);
#else
  for (uint32_t k = 0; k < 32; k++) lz_literal_copy_lane(d, s, len, LZ_LANES_DESCENDING ? 31 - k : k);
#endif
}
ZS_FN void lz_match_copy(uint8_t* d, uint32_t dp, uint32_t off, uint32_t len) {
#if defined(__CUDA_ARCH__)
  lz_match_copy_lane(d, dp, off, len, threadIdx.x & 31u);
#else
  for (uint32_t k = 0; k < 32; k++) lz_match_copy_lane(d, dp, off, len, LZ_LANES_DESCENDING ? 31 - k : k);
#endif
}

// codec 0: the page is stored as is.  A size mismatch is refused before anything is written.
ZS_FN bool stored_decode(const uint8_t* s, uint32_t sn, uint8_t* d, uint32_t dn) {
  if (sn != dn) return false;
  lz_literal_copy(d, s, dn);
  return true;
}

// LZ4 length extension: bytes of 255 continue it, any other byte ends it.  False when the source ends inside it, or
// when the length passes `cap` (so the sum stays below cap + 256 and cannot wrap).
ZS_FN bool lz4_len_ext(const uint8_t* s, uint32_t sn, uint32_t& sp, uint32_t& len, uint32_t cap) {
  uint32_t b;
  do {
    if (sp >= sn || len > cap) return false;
    b = s[sp++];
    len += b;
  } while (b == 255);
  return true;
}

// ---- LZ4 block format: token | literal length ext | literals | offset(2) | match length ext ----
ZS_FN bool lz4_raw_decode(const uint8_t* s, uint32_t sn, uint8_t* d, uint32_t dn) {
  uint32_t sp = 0, dp = 0;
  while (sp < sn) {
    const uint32_t token = s[sp++];
    uint32_t lit = token >> 4;
    if (lit == 15 && !lz4_len_ext(s, sn, sp, lit, sn)) return false;
    if (lit > sn - sp || lit > dn - dp) return false;
    lz_literal_copy(d + dp, s + sp, lit);
    sp += lit;
    dp += lit;
    if (sp >= sn) break;  // the last sequence carries literals only
    if (2 > sn - sp) return false;
    const uint32_t off = uint32_t(s[sp]) | (uint32_t(s[sp + 1]) << 8);
    sp += 2;
    uint32_t ml = token & 15;
    if (ml == 15 && !lz4_len_ext(s, sn, sp, ml, dn)) return false;
    ml += 4;
    if (off == 0 || off > dp || ml > dn - dp) return false;
    LZ_SYNC();  // the literals just written may be the match source
    lz_match_copy(d, dp, off, ml);
    dp += ml;
    LZ_SYNC();
  }
  return dp == dn;
}

// ---- Snappy: varint uncompressed length, then tagged elements ----
ZS_FN bool snappy_decode(const uint8_t* s, uint32_t sn, uint8_t* d, uint32_t dn) {
  uint32_t sp = 0, dp = 0, ulen = 0;
  for (uint32_t shift = 0;; shift += 7) {
    if (sp >= sn) return false;
    const uint32_t b = s[sp++];
    if (shift == 28 && b > 15) return false;   // more than 32 bits
    ulen |= (b & 0x7fu) << shift;
    if (!(b & 0x80u)) break;
  }
  if (ulen != dn) return false;
  while (sp < sn) {
    const uint32_t tag = s[sp++];
    const uint32_t kind = tag & 3;
    if (kind == 0) {
      uint32_t lm1 = tag >> 2;   // length - 1
      if (lm1 >= 60) {
        const uint32_t nb = lm1 - 59;
        if (nb > sn - sp) return false;
        lm1 = 0;
        for (uint32_t k = 0; k < nb; k++) lm1 |= uint32_t(s[sp + k]) << (8 * k);
        sp += nb;
      }
      if (lm1 >= sn - sp || lm1 >= dn - dp) return false;
      const uint32_t len = lm1 + 1;
      lz_literal_copy(d + dp, s + sp, len);
      sp += len;
      dp += len;
      LZ_SYNC();
    } else {
      uint32_t len, off;
      if (kind == 1) {
        if (1 > sn - sp) return false;
        len = 4 + ((tag >> 2) & 7);
        off = ((tag >> 5) << 8) | s[sp];
        sp += 1;
      } else if (kind == 2) {
        if (2 > sn - sp) return false;
        len = (tag >> 2) + 1;
        off = uint32_t(s[sp]) | (uint32_t(s[sp + 1]) << 8);
        sp += 2;
      } else {
        if (4 > sn - sp) return false;
        len = (tag >> 2) + 1;
        off = uint32_t(s[sp]) | (uint32_t(s[sp + 1]) << 8) | (uint32_t(s[sp + 2]) << 16) | (uint32_t(s[sp + 3]) << 24);
        sp += 4;
      }
      if (off == 0 || off > dp || len > dn - dp) return false;
      LZ_SYNC();
      lz_match_copy(d, dp, off, len);
      dp += len;
      LZ_SYNC();
    }
  }
  return dp == dn;
}

}  // namespace pqb
