// GZIP pages (Parquet codec 2; `gzip` is a legal P_PARQUET_COMPRESSION_ALGO of the reference,
// /root/reference/src/option.rs:62-86; parquet 58.1.0 gets it from flate2): gzip members (RFC 1952) around
// DEFLATE streams (RFC 1951), written from the two RFCs.  One warp decodes one page, like the other codecs
// (decomp_kernels.cuh): the bit-serial part -- Huffman table construction and symbol decoding -- is walked by
// every lane redundantly (loads broadcast), match and stored-block copies are shared by the 32 lanes.
// The same source compiles for the host (one "lane"): tools/zstd_host.cpp exposes it to tests/test_zstd.py,
// which checks it against zlib on the CPU.
#pragma once
#include <cstdint>

#include "zstd_decode.cuh"   // ZS_FN / ZS_LANE / ZS_SYNC and the shared copies

namespace pqb {

constexpr int kInfFastBits = 10;
struct InflateWs {                // per-decoder scratch (global memory on the device: one per resident warp)
  uint16_t lcount[16], dcount[16];
  uint16_t lsym[288], dsym[32];
  uint16_t fast[1 << kInfFastBits];   // literal / length code of every 10-bit window: (symbol << 4) | length, 0: longer code
  uint8_t lens[352];               // [0, 19): code-length code; [32, 32 + 286 + 30): the two alphabets
};

struct InfBits {                  // LSB-first bit reader over src[0 .. n)
  const uint8_t* p;
  uint32_t n, pos;                // pos: next byte
  uint64_t buf;
  uint32_t cnt;
  bool bad;
};
ZS_FN void inf_fill(InfBits& b) {
  while (b.cnt <= 56 && b.pos < b.n) { b.buf |= uint64_t(b.p[b.pos++]) << b.cnt; b.cnt += 8; }
}
ZS_FN uint32_t inf_bits(InfBits& b, uint32_t k) {   // k <= 16
  if (b.cnt < k) { inf_fill(b); if (b.cnt < k) { b.bad = true; return 0; } }
  const uint32_t v = uint32_t(b.buf) & ((1u << k) - 1u);
  b.buf >>= k;
  b.cnt -= k;
  return v;
}

// canonical Huffman code from code lengths: count[len], symbols in code order.  Returns false for an over-subscribed
// set; an incomplete set is legal only for a single distance code (RFC 1951 3.2.7) -- decoding then rejects unused codes
ZS_FN_NOINLINE bool inf_build(const uint8_t* lens, uint32_t n, uint16_t* count, uint16_t* sym) {
  for (int i = 0; i < 16; i++) count[i] = 0;
  for (uint32_t i = 0; i < n; i++) count[lens[i]]++;
  int left = 1;
  for (int len = 1; len < 16; len++) {
    left <<= 1;
    left -= int(count[len]);
    if (left < 0) return false;
  }
  uint16_t offs[16];
  offs[1] = 0;
  for (int len = 1; len < 15; len++) offs[len + 1] = uint16_t(offs[len] + count[len]);
  for (uint32_t i = 0; i < n; i++)
    if (lens[i]) sym[offs[lens[i]]++] = uint16_t(i);
  return true;
}
// one symbol, bit by bit (codes are packed most significant bit first); -1: not a code / out of input
ZS_FN int32_t inf_decode_slow(InfBits& b, const uint16_t* count, const uint16_t* sym) {
  int32_t code = 0, first = 0, index = 0;
  for (int len = 1; len < 16; len++) {
    code |= int32_t(inf_bits(b, 1));
    if (b.bad) return -1;
    const int32_t c = count[len];
    if (code - c < first) return sym[index + (code - first)];
    index += c;
    first += c;
    first <<= 1;
    code <<= 1;
  }
  return -1;
}
// the literal / length table for windows of kInfFastBits bits (bit-reversed codes: the stream is read LSB first)
ZS_FN_NOINLINE void inf_build_fast(InflateWs& w) {
  for (uint32_t i = 0; i < (1u << kInfFastBits); i++) w.fast[i] = 0;
  uint32_t code = 0, index = 0;
  for (uint32_t len = 1; len <= uint32_t(kInfFastBits); len++) {
    for (uint32_t k = 0; k < w.lcount[len]; k++, code++, index++) {
      uint32_t rev = 0;
      for (uint32_t i = 0; i < len; i++) rev |= ((code >> i) & 1u) << (len - 1 - i);
      for (uint32_t hi = 0; hi < (1u << (kInfFastBits - len)); hi++) w.fast[rev | (hi << len)] = uint16_t((w.lsym[index] << 4) | len);
    }
    code <<= 1;
  }
}
ZS_FN int32_t inf_decode_litlen(InfBits& b, const InflateWs& w) {
  if (b.cnt < uint32_t(kInfFastBits)) inf_fill(b);
  if (b.cnt >= uint32_t(kInfFastBits)) {
    const uint32_t e = w.fast[uint32_t(b.buf) & ((1u << kInfFastBits) - 1u)];
    if (e) { b.buf >>= (e & 15u); b.cnt -= (e & 15u); return int32_t(e >> 4); }
  }
  return inf_decode_slow(b, w.lcount, w.lsym);
}

// one DEFLATE stream: dst[dp ..) grows; returns false when corrupt or the output would pass dn
ZS_FN_NOINLINE bool inflate_stream(InflateWs& w, InfBits& b, uint8_t* dst, uint64_t& dp, uint64_t dn) {
  const uint16_t lbase[29] = {3, 4, 5, 6, 7, 8, 9, 10, 11, 13, 15, 17, 19, 23, 27, 31, 35, 43, 51, 59, 67, 83, 99, 115, 131, 163, 195, 227, 258};
  const uint8_t lext[29] = {0, 0, 0, 0, 0, 0, 0, 0, 1, 1, 1, 1, 2, 2, 2, 2, 3, 3, 3, 3, 4, 4, 4, 4, 5, 5, 5, 5, 0};
  const uint16_t dbase[30] = {1, 2, 3, 4, 5, 7, 9, 13, 17, 25, 33, 49, 65, 97, 129, 193, 257, 385, 513, 769, 1025, 1537, 2049, 3073, 4097, 6145, 8193, 12289, 16385, 24577};
  const uint8_t dext[30] = {0, 0, 0, 0, 1, 1, 2, 2, 3, 3, 4, 4, 5, 5, 6, 6, 7, 7, 8, 8, 9, 9, 10, 10, 11, 11, 12, 12, 13, 13};
  const uint8_t clorder[19] = {16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15};
  for (;;) {
    const uint32_t last = inf_bits(b, 1), type = inf_bits(b, 2);
    if (b.bad) return false;
    if (type == 0) {
      // stored: to the byte boundary, LEN, ~LEN, bytes
      const uint32_t drop = b.cnt & 7u;
      b.buf >>= drop; b.cnt -= drop;
      const uint32_t len = inf_bits(b, 16), nlen = inf_bits(b, 16);
      if (b.bad || (len ^ 0xffffu) != nlen) return false;
      // whole bytes still in the bit buffer go back to the byte stream
      b.pos -= b.cnt >> 3; b.buf = 0; b.cnt = 0;
      if (uint64_t(b.pos) + len > b.n || dp + len > dn) return false;
      ZS_SYNC();
      zs_copy(dst + dp, b.p + b.pos, len);
      ZS_SYNC();
      b.pos += len;
      dp += len;
    } else if (type == 1 || type == 2) {
      ZS_SYNC();   // every lane is done with the previous block's tables
      bool ok = true;
      InfBits b0 = b;
      if (ZS_LANE == 0) {
        if (type == 1) {
          for (uint32_t i = 0; i < 144; i++) w.lens[i] = 8;
          for (uint32_t i = 144; i < 256; i++) w.lens[i] = 9;
          for (uint32_t i = 256; i < 280; i++) w.lens[i] = 7;
          for (uint32_t i = 280; i < 288; i++) w.lens[i] = 8;
          ok = inf_build(w.lens, 288, w.lcount, w.lsym);
          for (uint32_t i = 0; i < 30; i++) w.lens[i] = 5;
          ok = ok && inf_build(w.lens, 30, w.dcount, w.dsym);
        } else {
          const uint32_t nlen = inf_bits(b0, 5) + 257, ndist = inf_bits(b0, 5) + 1, ncode = inf_bits(b0, 4) + 4;
          ok = !b0.bad && nlen <= 286 && ndist <= 30;
          if (ok) {
            for (uint32_t i = 0; i < 19; i++) w.lens[i] = 0;
            for (uint32_t i = 0; i < ncode; i++) w.lens[clorder[i]] = uint8_t(inf_bits(b0, 3));
            ok = !b0.bad && inf_build(w.lens, 19, w.lcount, w.lsym);
            // the code lengths of both alphabets, run-length coded with the 19-symbol code
            uint32_t idx = 0;
            while (ok && idx < nlen + ndist) {
              const int32_t s = inf_decode_slow(b0, w.lcount, w.lsym);
              if (s < 0) { ok = false; break; }
              if (s < 16) w.lens[32 + idx++] = uint8_t(s);
              else {
                uint32_t prev = 0, rep;
                if (s == 16) { if (idx == 0) { ok = false; break; } prev = w.lens[32 + idx - 1]; rep = 3 + inf_bits(b0, 2); }
                else if (s == 17) rep = 3 + inf_bits(b0, 3);
                else rep = 11 + inf_bits(b0, 7);
                if (b0.bad || idx + rep > nlen + ndist) { ok = false; break; }
                while (rep--) w.lens[32 + idx++] = uint8_t(prev);
              }
            }
            ok = ok && w.lens[32 + 256] != 0;   // a block without an end code never ends
            if (ok) {
              // distance lengths first (the literal / length build overwrites nothing it needs)
              ok = inf_build(w.lens + 32 + nlen, ndist, w.dcount, w.dsym);
              ok = ok && inf_build(w.lens + 32, nlen, w.lcount, w.lsym);
            }
          }
        }
        if (ok) inf_build_fast(w);
      }
#if defined(__CUDA_ARCH__)
      ok = __shfl_sync(0xffffffffu, ok ? 1 : 0, 0) != 0;
      // every lane continues where lane 0's header parse ended
      b.pos = __shfl_sync(0xffffffffu, b0.pos, 0);
      b.cnt = __shfl_sync(0xffffffffu, b0.cnt, 0);
      b.buf = (uint64_t(__shfl_sync(0xffffffffu, uint32_t(b0.buf >> 32), 0)) << 32) | __shfl_sync(0xffffffffu, uint32_t(b0.buf), 0);
#else
      b = b0;
#endif
      if (!ok) return false;
      ZS_SYNC();
      for (;;) {
        const int32_t s = inf_decode_litlen(b, w);
        if (s < 0) return false;
        if (s < 256) {
          if (dp >= dn) return false;
          if (ZS_LANE == 0) dst[dp] = uint8_t(s);
          dp++;
        } else if (s == 256) break;
        else {
          const uint32_t li = uint32_t(s) - 257;
          if (li >= 29) return false;
          const uint32_t len = lbase[li] + inf_bits(b, lext[li]);
          const int32_t ds = inf_decode_slow(b, w.dcount, w.dsym);
          if (ds < 0 || ds >= 30) return false;
          const uint32_t dist = dbase[ds] + inf_bits(b, dext[ds]);
          if (b.bad || dist > dp || dp + len > dn) return false;
          ZS_SYNC();   // the literals just written may be the match source
          zs_match(dst, dp, dist, len);
          dp += len;
          ZS_SYNC();
        }
      }
    } else return false;
    if (last) break;
  }
  return true;
}

// src[0 .. sn) = one or more gzip members; dst must receive exactly dn bytes.  Every lane of the warp calls it with
// the same arguments.  CRC-32 / ISIZE trailers are skipped, not verified (the page header already says the size).
ZS_FN_NOINLINE bool gzip_decode(InflateWs& w, const uint8_t* src, uint32_t sn, uint8_t* dst, uint64_t dn) {
  uint64_t dp = 0;
  uint32_t sp = 0;
  while (sp < sn) {
    if (sp + 10 > sn || src[sp] != 0x1f || src[sp + 1] != 0x8b || src[sp + 2] != 8) return false;
    const uint32_t flg = src[sp + 3];
    if (flg & 0xe0u) return false;
    sp += 10;
    if (flg & 4u) {   // FEXTRA
      if (sp + 2 > sn) return false;
      const uint32_t xl = uint32_t(src[sp]) | (uint32_t(src[sp + 1]) << 8);
      sp += 2;
      if (uint64_t(sp) + xl > sn) return false;
      sp += xl;
    }
    for (uint32_t f = 8u; f <= 16u; f <<= 1)   // FNAME, FCOMMENT: zero-terminated
      if (flg & f) {
        while (sp < sn && src[sp]) sp++;
        if (sp >= sn) return false;
        sp++;
      }
    if (flg & 2u) sp += 2;   // FHCRC
    if (sp >= sn) return false;
    InfBits b{src + sp, sn - sp, 0, 0, 0, false};
    if (!inflate_stream(w, b, dst, dp, dn)) return false;
    // the unread whole bytes in the bit buffer belong to the trailer
    const uint32_t used = b.pos - (b.cnt >> 3);
    sp += used;
    if (sp + 8 > sn) return false;
    sp += 8;   // CRC-32, ISIZE
  }
  ZS_SYNC();
  return dp == dn;
}

// The workspace of one k_decompress_zstd warp (decomp_kernels.cuh): it decodes page after page, ZSTD and GZIP mixed,
// in the same memory.  Parquet codec 2 is GZIP, anything else reaching here is ZSTD (codec 6).
union HeavyWs {
  ZstdWs z;
  InflateWs g;
};
ZS_FN bool heavy_page_decode(HeavyWs& w, uint32_t codec, const uint8_t* src, uint32_t sn, uint8_t* dst, uint32_t dn) {
  return codec == 2u ? gzip_decode(w.g, src, sn, dst, dn) : zstd_decode(w.z, src, sn, dst, dn);
}

}  // namespace pqb
