// Zstandard frame decoder for Parquet pages (codec 6, a legal P_PARQUET_COMPRESSION_ALGO of the
// reference: /root/reference/src/option.rs:62-86; parquet 58.1.0 gets it from the zstd crate).
// Written from the format specification (RFC 8878): frames, raw / RLE / compressed blocks, raw / RLE /
// Huffman (1 or 4 streams, tree given directly or FSE-compressed, or reused) literals, sequences with
// predefined / RLE / FSE-described / repeated tables, repeat offsets, skippable frames, no dictionaries.
//
// One WARP decodes one page.  The serial part of the format -- table construction, the three
// interleaved FSE states of the sequence stream -- is walked by every lane redundantly (the loads
// broadcast, like the LZ4 decoder in decomp_kernels.cuh); the parallel parts are shared: the four
// Huffman streams of a literals section go to four lanes, literal and match copies to all 32.
// The same source compiles for the host (one "lane"): tools/zstd_host.cpp exposes it to
// tests/test_zstd.py, which checks it against pyarrow's zstd on the CPU, and tools/decomp_dev.cu runs the kernel
// itself over the same inputs on the GPU.
#pragma once
#include <cstdint>

#if defined(__CUDACC__)
#define ZS_FN __host__ __device__ __forceinline__
#define ZS_FN_NOINLINE __host__ __device__ __noinline__
#else
#define ZS_FN inline
#define ZS_FN_NOINLINE inline
#endif

namespace pqb {

constexpr uint32_t kZstdBlockMax = 128u * 1024u;
constexpr int kZsHufLog = 11, kZsLLLog = 9, kZsOFLog = 8, kZsMLLog = 9;

struct ZsFse {                 // one FSE decoding table
  uint16_t base[512];          // new_state_base
  uint8_t sym[512];
  uint8_t nbits[512];
  uint32_t log;                // accuracy log (0: RLE table, one state)
};
// per-decoder scratch (global memory on the device: one per resident warp)
struct ZstdWs {
  ZsFse ll, of, ml;
  ZsFse wt;                    // Huffman weights table (accuracy log <= 6); also scratch
  uint8_t huf_sym[1 << kZsHufLog];
  uint8_t huf_nb[1 << kZsHufLog];
  uint32_t huf_log;            // 0: no Huffman table yet
  uint32_t have_ll, have_of, have_ml;
  uint8_t weights[256];
  int16_t freq[256];
  uint8_t lit[kZstdBlockMax + 32];
};

// ---- lanes -----------------------------------------------------------------------------------
#if defined(__CUDA_ARCH__)
#define ZS_LANE (threadIdx.x & 31u)
#define ZS_LANES 32u
#define ZS_SYNC() __syncwarp()
#else
#define ZS_LANE 0u
#define ZS_LANES 1u
#define ZS_SYNC() ((void)0)
#endif

ZS_FN int zs_highbit(uint32_t v) {   // index of the highest set bit, v != 0
  int r = 0;
  while (v >>= 1) r++;
  return r;
}

// nbits (<= 32) bits starting at bit `bitoff` of p, little endian; the caller guarantees the bytes exist
ZS_FN uint64_t zs_bits_le(const uint8_t* p, uint32_t nbits, uint64_t bitoff) {
  if (!nbits) return 0;
  const uint8_t* q = p + (bitoff >> 3);
  const uint32_t sh = uint32_t(bitoff & 7u), need = (sh + nbits + 7u) >> 3;
  uint64_t v = 0;
  for (uint32_t i = 0; i < need; i++) v |= uint64_t(q[i]) << (8u * i);
  return (v >> sh) & ((1ull << nbits) - 1ull);
}
// Backward bit stream over p[0 .. len): `off` is the number of unread bits below the cursor (it may go negative at the
// very end: the bits below the start of the stream read as zero).  Reads go through a 64-bit window of the stream held
// in registers: one (aligned, on the device) load per ~64 bits consumed instead of a byte-wise assembly per field.
struct ZsR {
  const uint8_t* p;
  uint32_t len;
  int64_t off;
  uint64_t win;       // bits [wbase, wbase + 64) of the stream (fewer at a short stream's end)
  int64_t wbase;      // multiple of 8; -1: nothing loaded
};
ZS_FN uint32_t zs_funnel_r(uint32_t lo, uint32_t hi, uint32_t sh) {   // low word of (hi:lo) >> sh, sh in {0, 8, 16, 24}
#if defined(__CUDA_ARCH__)
  return __funnelshift_r(lo, hi, sh);
#else
  return sh ? (lo >> sh) | (hi << (32u - sh)) : lo;
#endif
}
ZS_FN uint64_t zs_load_window(const uint8_t* p, uint32_t len, uint64_t byte) {   // up to 8 bytes at p[byte ..], little endian
#if defined(__CUDA_ARCH__) || defined(ZS_TEST_ALIGNED)   // (the host build takes this path only in the test harness that checks it)
  if (byte + 12 <= len) {   // three aligned words hold the eight bytes, whatever the byte phase; they stay inside p[0 .. len) plus at most 3 bytes below p (the buffer's base is aligned)
    const uintptr_t a = reinterpret_cast<uintptr_t>(p + byte);
    const uint32_t* w = reinterpret_cast<const uint32_t*>(a & ~uintptr_t(3));
    const uint32_t sh = uint32_t(a & 3u) * 8u;
    const uint32_t w0 = w[0], w1 = w[1], w2 = w[2];
    return (uint64_t(zs_funnel_r(w1, w2, sh)) << 32) | zs_funnel_r(w0, w1, sh);
  }
#endif
  uint64_t v = 0;
  for (uint32_t i = 0; i < 8 && byte + i < len; i++) v |= uint64_t(p[byte + i]) << (8u * i);
  return v;
}
ZS_FN uint64_t zs_rbits(ZsR& r, uint32_t nbits) {   // nbits <= 32
  r.off -= int64_t(nbits);
  if (nbits == 0) return 0;
  if (r.off >= 0) {
    if (r.wbase < 0 || r.off < r.wbase || r.off + int64_t(nbits) > r.wbase + 64) {
      // reads walk downwards: a window that ends at the byte above this field serves the following ones too
      int64_t b = ((r.off + int64_t(nbits) + 7) & ~int64_t(7)) - 64;
      if (b < 0) b = 0;
      r.wbase = b;
      r.win = zs_load_window(r.p, r.len, uint64_t(b >> 3));
    }
    return (r.win >> uint32_t(r.off - r.wbase)) & ((1ull << nbits) - 1ull);
  }
  const int64_t real = int64_t(nbits) + r.off;   // bits that exist
  if (real <= 0) return 0;
  const uint64_t v = zs_bits_le(r.p, uint32_t(real), 0);
  return (-r.off) >= 64 ? 0 : (v << uint32_t(-r.off));
}
// start of a backward stream: position of the end mark in the last byte; off < 0: corrupt
ZS_FN ZsR zs_rstart(const uint8_t* p, uint32_t len) {
  ZsR r{p, len, -1, 0, -1};
  if (!len || p[len - 1] == 0) return r;
  r.off = int64_t(len) * 8 - (8 - zs_highbit(p[len - 1]));
  return r;
}

// ---- FSE ---------------------------------------------------------------------------------------
// normalised counts -> decoding table.  Returns false on a corrupt distribution.
ZS_FN_NOINLINE bool zs_fse_build(ZsFse& t, const int16_t* freq, uint32_t nsym, uint32_t log) {
  const uint32_t size = 1u << log;
  uint16_t next[256];
  uint32_t high = size;
  for (uint32_t s = 0; s < nsym; s++) {
    if (freq[s] == -1) { t.sym[--high] = uint8_t(s); next[s] = 1; }
    else next[s] = uint16_t(freq[s] > 0 ? freq[s] : 0);
  }
  const uint32_t step = (size >> 1) + (size >> 3) + 3, mask = size - 1;
  uint32_t pos = 0;
  for (uint32_t s = 0; s < nsym; s++) {
    if (freq[s] <= 0) continue;
    for (int i = 0; i < freq[s]; i++) {
      t.sym[pos] = uint8_t(s);
      do { pos = (pos + step) & mask; } while (pos >= high);
    }
  }
  if (pos != 0) return false;
  for (uint32_t i = 0; i < size; i++) {
    const uint32_t s = t.sym[i], d = next[s]++;
    if (d == 0) return false;
    const uint32_t nb = log - uint32_t(zs_highbit(d));
    t.nbits[i] = uint8_t(nb);
    t.base[i] = uint16_t((d << nb) - size);
  }
  t.log = log;
  return true;
}
ZS_FN void zs_fse_rle(ZsFse& t, uint8_t sym) {
  t.sym[0] = sym; t.nbits[0] = 0; t.base[0] = 0; t.log = 0;
}
// FSE table description (forward bit stream) -> freq[]; returns bytes consumed, 0: corrupt
ZS_FN_NOINLINE uint32_t zs_fse_header(const uint8_t* p, uint32_t len, int16_t* freq, uint32_t max_sym, uint32_t max_log,
                                      uint32_t& nsym, uint32_t& log) {
  if (!len) return 0;
  const uint64_t nbits_total = uint64_t(len) * 8;
  uint64_t bo = 0;
  auto rd = [&](uint32_t n, uint64_t& v) -> bool {
    if (bo + n > nbits_total) {   // the last fields may ask for more bits than the stream holds: the missing ones are zero
      const uint64_t have = bo < nbits_total ? nbits_total - bo : 0;
      v = have ? zs_bits_le(p, uint32_t(have), bo) : 0;
      bo += n;
      return bo <= nbits_total + 32;
    }
    v = zs_bits_le(p, n, bo);
    bo += n;
    return true;
  };
  uint64_t v;
  if (!rd(4, v)) return 0;
  log = 5 + uint32_t(v);
  if (log > max_log) return 0;
  int32_t remaining = 1 << log;
  uint32_t s = 0;
  while (remaining > 0 && s < max_sym) {
    const uint32_t bits = uint32_t(zs_highbit(uint32_t(remaining + 1))) + 1;
    if (!rd(bits, v)) return 0;
    uint32_t val = uint32_t(v);
    const uint32_t lower = (1u << (bits - 1)) - 1u, thresh = (1u << bits) - 1u - uint32_t(remaining + 1);
    if ((val & lower) < thresh) { bo -= 1; val &= lower; }
    else if (val > lower) val -= thresh;
    const int32_t proba = int32_t(val) - 1;
    remaining -= proba < 0 ? -proba : proba;
    freq[s++] = int16_t(proba);
    if (proba == 0) {
      for (;;) {
        if (!rd(2, v)) return 0;
        const uint32_t rep = uint32_t(v);
        for (uint32_t i = 0; i < rep && s < max_sym; i++) freq[s++] = 0;
        if (rep != 3) break;
        if (s >= max_sym) break;
      }
    }
  }
  if (remaining != 0 || bo > nbits_total) return 0;
  nsym = s;
  return uint32_t((bo + 7) >> 3);
}

// ---- Huffman literals --------------------------------------------------------------------------
// weights[0 .. n) (the last one already completed) -> decoding table of huf_log bits
ZS_FN_NOINLINE bool zs_huf_build(ZstdWs& w, uint32_t n) {
  uint32_t sum = 0;
  for (uint32_t i = 0; i + 1 < n; i++) {
    if (w.weights[i] > kZsHufLog) return false;
    sum += w.weights[i] ? (1u << (w.weights[i] - 1)) : 0u;
  }
  if (!sum) return false;
  const uint32_t maxbits = uint32_t(zs_highbit(sum)) + 1;
  if (maxbits > uint32_t(kZsHufLog)) return false;
  const uint32_t left = (1u << maxbits) - sum;
  if (left & (left - 1)) return false;
  w.weights[n - 1] = uint8_t(zs_highbit(left) + 1);
  uint32_t rank_count[kZsHufLog + 2];
  uint32_t rank_idx[kZsHufLog + 2];
  for (uint32_t i = 0; i <= uint32_t(kZsHufLog) + 1; i++) rank_count[i] = 0;
  for (uint32_t i = 0; i < n; i++) {
    const uint32_t b = w.weights[i] ? maxbits + 1 - w.weights[i] : 0;
    rank_count[b]++;
  }
  rank_idx[maxbits] = 0;
  for (uint32_t i = maxbits; i >= 1; i--) {
    rank_idx[i - 1] = rank_idx[i] + rank_count[i] * (1u << (maxbits - i));
    for (uint32_t k = rank_idx[i]; k < rank_idx[i - 1]; k++) w.huf_nb[k] = uint8_t(i);
  }
  if (rank_idx[0] != (1u << maxbits)) return false;
  for (uint32_t i = 0; i < n; i++) {
    if (!w.weights[i]) continue;
    const uint32_t b = maxbits + 1 - w.weights[i], len = 1u << (maxbits - b);
    for (uint32_t k = 0; k < len; k++) w.huf_sym[rank_idx[b] + k] = uint8_t(i);
    rank_idx[b] += len;
  }
  w.huf_log = maxbits;
  return true;
}
// Huffman tree description -> table; returns bytes consumed, 0: corrupt
ZS_FN_NOINLINE uint32_t zs_huf_tree(ZstdWs& w, const uint8_t* p, uint32_t len) {
  if (!len) return 0;
  const uint32_t hb = p[0];
  uint32_t n = 0, used;
  if (hb >= 128) {
    n = hb - 127;
    const uint32_t nb = (n + 1) / 2;
    if (1 + nb > len) return 0;
    for (uint32_t i = 0; i < n; i++) w.weights[i] = (i & 1u) ? (p[1 + i / 2] & 15u) : (p[1 + i / 2] >> 4);
    used = 1 + nb;
  } else {
    if (1 + hb > len || hb == 0) return 0;
    const uint8_t* q = p + 1;
    uint32_t nsym = 0, log = 0;
    const uint32_t hdr = zs_fse_header(q, hb, w.freq, 256, 6, nsym, log);
    if (!hdr || hdr >= hb) return 0;
    if (!zs_fse_build(w.wt, w.freq, nsym, log)) return 0;
    const uint8_t* bs = q + hdr;
    const uint32_t bl = hb - hdr;
    ZsR r = zs_rstart(bs, bl);
    if (r.off < 0) return 0;
    uint32_t s1 = uint32_t(zs_rbits(r, log)), s2 = uint32_t(zs_rbits(r, log));
    for (;;) {
      if (n >= 254) return 0;
      w.weights[n++] = w.wt.sym[s1];
      s1 = w.wt.base[s1] + uint32_t(zs_rbits(r, w.wt.nbits[s1]));
      if (r.off < 0) { w.weights[n++] = w.wt.sym[s2]; break; }
      if (n >= 254) return 0;
      w.weights[n++] = w.wt.sym[s2];
      s2 = w.wt.base[s2] + uint32_t(zs_rbits(r, w.wt.nbits[s2]));
      if (r.off < 0) { w.weights[n++] = w.wt.sym[s1]; break; }
    }
    used = 1 + hb;
  }
  if (n + 1 > 256) return 0;
  if (!zs_huf_build(w, n + 1)) return 0;
  return used;
}
// one Huffman stream -> exactly `n` literals
ZS_FN_NOINLINE bool zs_huf_stream(const ZstdWs& w, const uint8_t* p, uint32_t len, uint8_t* out, uint32_t n) {
  ZsR r = zs_rstart(p, len);
  if (r.off < 0) return false;
  const uint32_t L = w.huf_log, mask = (1u << L) - 1u;
  uint32_t st = uint32_t(zs_rbits(r, L));
  uint32_t i = 0;
  while (r.off > -int64_t(L)) {
    if (i >= n) return false;
    out[i++] = w.huf_sym[st];
    const uint32_t nb = w.huf_nb[st];
    st = ((st << nb) + uint32_t(zs_rbits(r, nb))) & mask;
  }
  return r.off == -int64_t(L) && i == n;
}

// ---- copies (shared by the lanes of the warp) ----------------------------------------------------
ZS_FN void zs_copy(uint8_t* d, const uint8_t* s, uint32_t n) {   // no overlap
  for (uint32_t i = ZS_LANE; i < n; i += ZS_LANES) d[i] = s[i];
}
ZS_FN void zs_match(uint8_t* d, uint64_t dp, uint32_t off, uint32_t n) {
  if (off >= n) { for (uint32_t i = ZS_LANE; i < n; i += ZS_LANES) d[dp + i] = d[dp - off + i]; }
  else { for (uint32_t i = ZS_LANE; i < n; i += ZS_LANES) d[dp + i] = d[dp - off + (i % off)]; }
}
ZS_FN void zs_fill(uint8_t* d, uint8_t v, uint32_t n) {
  for (uint32_t i = ZS_LANE; i < n; i += ZS_LANES) d[i] = v;
}

struct ZsSeqTabs { uint32_t dummy; };
// literal length / match length codes: baseline and extra bits
ZS_FN uint32_t zs_ll_base(uint32_t c) {
  return c < 16 ? c : (c < 20 ? 16 + (c - 16) * 2 : (c < 22 ? 24 + (c - 20) * 4 : (c < 24 ? 32 + (c - 22) * 8 : (c == 24 ? 48u : (1u << (c - 19))))));
}
ZS_FN uint32_t zs_ll_bits(uint32_t c) {
  return c < 16 ? 0 : (c < 20 ? 1 : (c < 22 ? 2 : (c < 24 ? 3 : (c == 24 ? 4u : c - 19))));
}
ZS_FN uint32_t zs_ml_base(uint32_t c) {
  if (c < 32) return c + 3;
  if (c < 36) return 35 + (c - 32) * 2;
  if (c < 38) return 43 + (c - 36) * 4;
  if (c < 40) return 51 + (c - 38) * 8;
  if (c < 42) return 67 + (c - 40) * 16;
  if (c == 42) return 99;
  return 3u + (1u << (c - 36));   // 43: 131, 44: 259, ... 52: 65539
}
ZS_FN uint32_t zs_ml_bits(uint32_t c) {
  if (c < 32) return 0;
  if (c < 36) return 1;
  if (c < 38) return 2;
  if (c < 40) return 3;
  if (c < 42) return 4;
  if (c == 42) return 5;
  return c - 36;   // 43: 7 ... 52: 16
}

// table of one sequence field per the block's compression mode.  Lane 0 builds (callers sync).  Returns bytes
// consumed (may be 0 for predefined / repeat), < 0: corrupt.
ZS_FN_NOINLINE int32_t zs_seq_table(ZsFse& t, uint32_t& have, uint32_t mode, const uint8_t* p, uint32_t len, int which, ZstdWs& w) {
  // which: 0 LL, 1 OF, 2 ML
  if (mode == 0) {
    const int16_t LL[36] = {4, 3, 2, 2, 2, 2, 2, 2, 2, 2, 2, 2, 2, 1, 1, 1, 2, 2, 2, 2, 2, 2, 2, 2, 2, 3, 2, 1, 1, 1, 1, 1, -1, -1, -1, -1};
    const int16_t OF[29] = {1, 1, 1, 1, 1, 1, 2, 2, 2, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, -1, -1, -1, -1, -1};
    const int16_t ML[53] = {1, 4, 3, 2, 2, 2, 2, 2, 2, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1,
                            1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, -1, -1, -1, -1, -1, -1, -1};
    bool ok;
    if (which == 0) ok = zs_fse_build(t, LL, 36, 6);
    else if (which == 1) ok = zs_fse_build(t, OF, 29, 5);
    else ok = zs_fse_build(t, ML, 53, 6);
    have = ok ? 1u : 0u;
    return ok ? 0 : -1;
  }
  const uint32_t max_sym = which == 0 ? 36u : (which == 1 ? 32u : 53u);
  if (mode == 1) {
    if (len < 1 || p[0] >= max_sym) return -1;
    zs_fse_rle(t, p[0]);
    have = 1;
    return 1;
  }
  if (mode == 2) {
    uint32_t nsym = 0, log = 0;
    const uint32_t max_log = which == 0 ? kZsLLLog : (which == 1 ? kZsOFLog : kZsMLLog);
    const uint32_t used = zs_fse_header(p, len, w.freq, max_sym, max_log, nsym, log);
    if (!used) return -1;
    if (!zs_fse_build(t, w.freq, nsym, log)) return -1;
    have = 1;
    return int32_t(used);
  }
  return have ? 0 : -1;   // repeat: the previous block's table
}

// ---- one compressed block ----------------------------------------------------------------------
// dst[0 .. dp) is everything decoded so far in this frame (the window); returns the new dp, or ~0ull: corrupt
ZS_FN_NOINLINE uint64_t zs_block(ZstdWs& w, const uint8_t* p, uint32_t len, uint8_t* dst, uint64_t dp, uint64_t dn, uint32_t* rep) {
  const uint64_t BAD = ~0ull;
  if (len < 1) return BAD;
  // ---- literals section ----
  const uint32_t ltype = p[0] & 3u, sf = (p[0] >> 2) & 3u;
  uint32_t hdr, regen, comp = 0, streams = 1;
  if (ltype < 2) {
    if ((sf & 1u) == 0) { hdr = 1; regen = p[0] >> 3; }
    else if (sf == 1) { if (len < 2) return BAD; hdr = 2; regen = (uint32_t(p[0]) | (uint32_t(p[1]) << 8)) >> 4; }
    else { if (len < 3) return BAD; hdr = 3; regen = (uint32_t(p[0]) | (uint32_t(p[1]) << 8) | (uint32_t(p[2]) << 16)) >> 4; }
  } else {
    if (sf < 2) {
      if (len < 3) return BAD;
      const uint32_t v = uint32_t(p[0]) | (uint32_t(p[1]) << 8) | (uint32_t(p[2]) << 16);
      hdr = 3; regen = (v >> 4) & 0x3ffu; comp = (v >> 14) & 0x3ffu; streams = sf == 0 ? 1 : 4;
    } else if (sf == 2) {
      if (len < 4) return BAD;
      const uint32_t v = uint32_t(p[0]) | (uint32_t(p[1]) << 8) | (uint32_t(p[2]) << 16) | (uint32_t(p[3]) << 24);
      hdr = 4; regen = (v >> 4) & 0x3fffu; comp = v >> 18; streams = 4;
    } else {
      if (len < 5) return BAD;
      const uint64_t v = uint64_t(p[0]) | (uint64_t(p[1]) << 8) | (uint64_t(p[2]) << 16) | (uint64_t(p[3]) << 24) | (uint64_t(p[4]) << 32);
      hdr = 5; regen = uint32_t((v >> 4) & 0x3ffffu); comp = uint32_t((v >> 22) & 0x3ffffu); streams = 4;
    }
  }
  if (regen > kZstdBlockMax) return BAD;
  const uint8_t* lit = nullptr;   // where the block's literals are read from
  uint32_t pos = hdr;
  if (ltype == 0) {
    if (pos + regen > len) return BAD;
    lit = p + pos;
    pos += regen;
  } else if (ltype == 1) {
    if (pos + 1 > len) return BAD;
    ZS_SYNC();
    zs_fill(w.lit, p[pos], regen);
    ZS_SYNC();
    lit = w.lit;
    pos += 1;
  } else {
    if (pos + comp > len) return BAD;
    const uint8_t* q = p + pos;
    uint32_t ql = comp;
    ZS_SYNC();   // everybody is done with the previous block's literals and tables
    uint32_t tree = 0;
    if (ltype == 2) {
      if (ZS_LANE == 0) tree = zs_huf_tree(w, q, ql);
#if defined(__CUDA_ARCH__)
      tree = __shfl_sync(0xffffffffu, tree, 0);
#endif
      if (!tree) return BAD;
      q += tree; ql -= tree;
    } else if (!w.huf_log) return BAD;
    ZS_SYNC();
    bool ok = true;
    if (streams == 1) {
      if (ZS_LANE == 0) ok = zs_huf_stream(w, q, ql, w.lit, regen);
    } else {
      if (ql < 6) return BAD;
      const uint32_t s1 = uint32_t(q[0]) | (uint32_t(q[1]) << 8), s2 = uint32_t(q[2]) | (uint32_t(q[3]) << 8), s3 = uint32_t(q[4]) | (uint32_t(q[5]) << 8);
      if (6ull + s1 + s2 + s3 > ql) return BAD;
      const uint32_t s4 = ql - 6 - s1 - s2 - s3, per = (regen + 3) / 4;
      if (3ull * per > regen) return BAD;
      const uint32_t so[4] = {6, 6 + s1, 6 + s1 + s2, 6 + s1 + s2 + s3}, sl[4] = {s1, s2, s3, s4};
#if defined(__CUDA_ARCH__)
      if (ZS_LANE < 4) {
        const uint32_t k = ZS_LANE;
        ok = zs_huf_stream(w, q + so[k], sl[k], w.lit + k * per, k < 3 ? per : regen - 3 * per);
      }
#else
      for (uint32_t k = 0; k < 4; k++) ok = ok && zs_huf_stream(w, q + so[k], sl[k], w.lit + k * per, k < 3 ? per : regen - 3 * per);
#endif
    }
#if defined(__CUDA_ARCH__)
    ok = __all_sync(0xffffffffu, ok);
#endif
    if (!ok) return BAD;
    ZS_SYNC();
    lit = w.lit;
    pos += comp;
  }
  // ---- sequences section ----
  if (pos >= len) return BAD;
  uint32_t nseq = p[pos++];
  if (nseq >= 128) {
    if (nseq == 255) {
      if (pos + 2 > len) return BAD;
      nseq = uint32_t(p[pos]) + (uint32_t(p[pos + 1]) << 8) + 0x7f00u;
      pos += 2;
    } else {
      if (pos + 1 > len) return BAD;
      nseq = ((nseq - 128) << 8) + p[pos];
      pos += 1;
    }
  }
  if (nseq == 0) {
    if (dp + regen > dn) return BAD;
    zs_copy(dst + dp, lit, regen);
    return dp + regen;
  }
  if (pos >= len) return BAD;
  const uint32_t modes = p[pos++];
  if (modes & 3u) return BAD;
  int32_t used[3] = {0, 0, 0};
  ZS_SYNC();
  if (ZS_LANE == 0) {
    used[0] = zs_seq_table(w.ll, w.have_ll, modes >> 6, p + pos, len - pos, 0, w);
    if (used[0] >= 0) used[1] = zs_seq_table(w.of, w.have_of, (modes >> 4) & 3u, p + pos + used[0], len - pos - used[0], 1, w);
    if (used[0] >= 0 && used[1] >= 0)
      used[2] = zs_seq_table(w.ml, w.have_ml, (modes >> 2) & 3u, p + pos + used[0] + used[1], len - pos - used[0] - used[1], 2, w);
  }
#if defined(__CUDA_ARCH__)
  for (int k = 0; k < 3; k++) used[k] = __shfl_sync(0xffffffffu, used[k], 0);
#endif
  if (used[0] < 0 || used[1] < 0 || used[2] < 0) return BAD;
  ZS_SYNC();
  pos += uint32_t(used[0] + used[1] + used[2]);
  if (pos >= len) return BAD;
  const uint8_t* bs = p + pos;
  const uint32_t bl = len - pos;
  ZsR r = zs_rstart(bs, bl);
  if (r.off < 0) return BAD;
  uint32_t sl = uint32_t(zs_rbits(r, w.ll.log)), so = uint32_t(zs_rbits(r, w.of.log)), sm = uint32_t(zs_rbits(r, w.ml.log));
  if (r.off < 0) return BAD;
  uint32_t lp = 0;   // literals consumed
  for (uint32_t i = 0; i < nseq; i++) {
    const uint32_t oc = w.of.sym[so], lc = w.ll.sym[sl], mc = w.ml.sym[sm];
    if (oc > 31 || lc > 35 || mc > 52) return BAD;
    const uint64_t ov = (1ull << oc) + zs_rbits(r, oc);
    const uint32_t mlen = zs_ml_base(mc) + uint32_t(zs_rbits(r, zs_ml_bits(mc)));
    const uint32_t llen = zs_ll_base(lc) + uint32_t(zs_rbits(r, zs_ll_bits(lc)));
    if (r.off < 0) return BAD;
    if (i + 1 < nseq) {
      sl = w.ll.base[sl] + uint32_t(zs_rbits(r, w.ll.nbits[sl]));
      sm = w.ml.base[sm] + uint32_t(zs_rbits(r, w.ml.nbits[sm]));
      so = w.of.base[so] + uint32_t(zs_rbits(r, w.of.nbits[so]));
      if (r.off < 0) return BAD;
    }
    uint64_t offset;
    if (ov > 3) {
      offset = ov - 3;
      rep[2] = rep[1]; rep[1] = rep[0]; rep[0] = uint32_t(offset);
    } else {
      uint32_t idx = uint32_t(ov);
      if (llen == 0) idx++;
      if (idx == 1) offset = rep[0];
      else {
        offset = idx < 4 ? rep[idx - 1] : rep[0] - 1;
        if (idx > 2) rep[2] = rep[1];
        rep[1] = rep[0];
        rep[0] = uint32_t(offset);
      }
    }
    if (offset == 0 || offset > 0xffffffffull) return BAD;
    if (lp + llen > regen || dp + llen + mlen > dn) return BAD;
    zs_copy(dst + dp, lit + lp, llen);
    lp += llen;
    dp += llen;
    if (offset > dp) return BAD;   // no dictionaries: a match cannot reach in front of the frame
    ZS_SYNC();                     // the literals just written may be the match source
    zs_match(dst, dp, uint32_t(offset), mlen);
    dp += mlen;
    ZS_SYNC();
  }
  if (r.off != 0) return BAD;
  const uint32_t rest = regen - lp;
  if (dp + rest > dn) return BAD;
  zs_copy(dst + dp, lit + lp, rest);
  return dp + rest;
}

// ---- frames --------------------------------------------------------------------------------------
// src[0 .. sn) = one or more zstd frames; dst must receive exactly dn bytes.  Every lane of the warp calls it with
// the same arguments.  Returns true when the page decoded to its declared size.
ZS_FN_NOINLINE bool zstd_decode(ZstdWs& w, const uint8_t* src, uint32_t sn, uint8_t* dst, uint64_t dn) {
  uint64_t dp = 0;
  uint32_t sp = 0;
  while (sp < sn) {
    if (sp + 4 > sn) return false;
    const uint32_t magic = uint32_t(src[sp]) | (uint32_t(src[sp + 1]) << 8) | (uint32_t(src[sp + 2]) << 16) | (uint32_t(src[sp + 3]) << 24);
    sp += 4;
    if ((magic & 0xfffffff0u) == 0x184d2a50u) {   // skippable frame
      if (sp + 4 > sn) return false;
      const uint32_t n = uint32_t(src[sp]) | (uint32_t(src[sp + 1]) << 8) | (uint32_t(src[sp + 2]) << 16) | (uint32_t(src[sp + 3]) << 24);
      sp += 4;
      if (uint64_t(sp) + n > sn) return false;
      sp += n;
      continue;
    }
    if (magic != 0xfd2fb528u) return false;
    if (sp + 1 > sn) return false;
    const uint32_t fhd = src[sp++];
    const uint32_t fcs_flag = fhd >> 6, single = (fhd >> 5) & 1u, checksum = (fhd >> 2) & 1u, did = fhd & 3u;
    if (fhd & 0x08u) return false;   // reserved bit
    if (!single) sp += 1;            // window descriptor: the whole page is the window here
    const uint32_t did_len = did == 3 ? 4u : did;
    if (did_len) {
      if (sp + did_len > sn) return false;
      uint32_t id = 0;
      for (uint32_t i = 0; i < did_len; i++) id |= uint32_t(src[sp + i]) << (8 * i);
      if (id) return false;          // a frame that needs a dictionary
      sp += did_len;
    }
    const uint32_t fcs_len = fcs_flag == 0 ? (single ? 1u : 0u) : (fcs_flag == 1 ? 2u : (fcs_flag == 2 ? 4u : 8u));
    sp += fcs_len;                   // the page header already says how many bytes come out
    if (sp > sn) return false;
    const uint64_t frame0 = dp;
    uint32_t rep[3] = {1, 4, 8};
    ZS_SYNC();
    if (ZS_LANE == 0) { w.huf_log = 0; w.have_ll = w.have_of = w.have_ml = 0; }
    ZS_SYNC();
    for (;;) {
      if (sp + 3 > sn) return false;
      const uint32_t bh = uint32_t(src[sp]) | (uint32_t(src[sp + 1]) << 8) | (uint32_t(src[sp + 2]) << 16);
      sp += 3;
      const uint32_t last = bh & 1u, type = (bh >> 1) & 3u, bsz = bh >> 3;
      if (type == 0) {
        if (uint64_t(sp) + bsz > sn || dp + bsz > dn) return false;
        zs_copy(dst + dp, src + sp, bsz);
        sp += bsz; dp += bsz;
      } else if (type == 1) {
        if (sp + 1 > sn || dp + bsz > dn) return false;
        zs_fill(dst + dp, src[sp], bsz);
        sp += 1; dp += bsz;
      } else if (type == 2) {
        if (uint64_t(sp) + bsz > sn || bsz > kZstdBlockMax) return false;
        // the window of a frame starts at the frame: hand the block the frame's output only
        const uint64_t r = zs_block(w, src + sp, bsz, dst + frame0, dp - frame0, dn - frame0, rep);
        if (r == ~0ull) return false;
        dp = frame0 + r;
        sp += bsz;
      } else return false;
      ZS_SYNC();
      if (last) break;
    }
    if (checksum) { if (sp + 4 > sn) return false; sp += 4; }   // xxh64 of the content: not verified (the reference's reader does not ask for it either)
  }
  return dp == dn;
}

}  // namespace pqb
