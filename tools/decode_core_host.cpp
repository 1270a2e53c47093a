// TEST HARNESS ONLY: exposes the pure host/device functions of decode_core.cuh to
// tests/test_decode_core.py so the run-walker / bit-unpacker are exercised on the
// CPU.  Never linked into libparseable_b200.so.
#include <cstdint>
#include <cstring>
#include <vector>
#include "decode_core.cuh"
using namespace pqb;

extern "C" {
// Decode `n` values of an RLE/bit-packed hybrid stream exactly as the scan kernel does: windows of
// `win_cap` bytes, slabs of `slab` values, directory of `max_ent` entries.  Returns values decoded.
int64_t dc_decode_hybrid(const uint8_t* stream, uint64_t len, uint32_t bw, uint32_t n, uint32_t slab,
                         uint32_t win_cap, uint32_t max_ent, uint32_t* out) {
  std::vector<uint8_t> padded(len + win_cap + 64, 0);
  std::memcpy(padded.data() + 16, stream, len);   // arena offset 16: unaligned start on purpose? no, 16-aligned
  StreamState st;
  stream_init(st, 16, 16 + len, bw);
  uint32_t done = 0;
  std::vector<DirEntry> dir(max_ent);
  std::vector<uint32_t> win((win_cap + 16) / 4 + 4);
  int guard = 0;
  while (done < n) {
    uint64_t s = stream_window_start(st) & ~15ull;
    std::memset(win.data(), 0, win.size() * 4);
    uint64_t avail = padded.size() - s;
    std::memcpy(win.data(), padded.data() + s, avail < win_cap ? avail : win_cap);
    Window w{reinterpret_cast<const uint8_t*>(win.data()), s, win_cap};
    uint32_t need = n - done < slab ? n - done : slab;
    uint32_t nent = 0;
    uint32_t got = walk_stream(st, w, need, dir.data(), nent, max_ent);
    if (got == 0) { if (++guard > 2) return -int64_t(done) - 1; continue; }
    guard = 0;
    for (uint32_t e = 0; e < nent; e++) {
      const DirEntry& d = dir[e];
      for (uint32_t j = 0; j < d.count; j++)
        out[done + d.start + j] = d.kind ? bp_get(win.data(), d.payload, bw, j) : d.payload;
    }
    done += got;
  }
  return done;
}
// DELTA_BINARY_PACKED page payload -> int64 values, through the kernel's window / directory geometry
int64_t dc_decode_delta(const uint8_t* stream, uint64_t len, uint32_t n, uint32_t slab, uint32_t win_cap,
                        uint32_t max_ent, int64_t* out) {
  std::vector<uint8_t> padded(len + win_cap + 64, 0);
  std::memcpy(padded.data() + 16, stream, len);
  DeltaState st;
  delta_init(st, 16, 16 + len);
  uint32_t done = 0;
  std::vector<DeltaEntry> dir(max_ent);
  std::vector<uint32_t> win((win_cap + 16) / 4 + 4);
  int guard = 0;
  while (done < n) {
    uint64_t s = delta_window_start(st) & ~15ull;
    std::memset(win.data(), 0, win.size() * 4);
    uint64_t avail = padded.size() - s;
    std::memcpy(win.data(), padded.data() + s, avail < win_cap ? avail : win_cap);
    Window w{reinterpret_cast<const uint8_t*>(win.data()), s, win_cap};
    uint32_t need = n - done < slab ? n - done : slab;
    uint32_t nent = 0;
    uint32_t got = walk_delta(st, w, need, dir.data(), nent, max_ent);
    if (got == 0) { if (++guard > 2 || st.bad) return -int64_t(done) - 1; continue; }
    guard = 0;
    for (uint32_t e = 0; e < nent; e++) {
      const DeltaEntry& d = dir[e];
      for (uint32_t j = 0; j < d.count; j++) {
        int64_t delta = d.kind ? d.min_delta : int64_t(uint64_t(d.min_delta) + bp_get64(win.data(), d.bitoff, d.bw, j));
        st.last_value = int64_t(uint64_t(st.last_value) + uint64_t(delta));
        out[done + d.start + j] = st.last_value;
      }
    }
    done += got;
  }
  return done;
}
// value pages: 1 and k when `bits` has an integer k at decimal exponent e, 0 when it refuses
int dc_dec_encode_f64(uint64_t bits, uint32_t e, int64_t* k) { return dec_encode_f64(bits, dec_scale(e), *k) ? 1 : 0; }
uint64_t dc_dec_decode_f64(int64_t k, uint32_t e) { return dec_decode_f64(k, dec_scale(e)); }
// n values at once (k[i] / 10^e -> out[i]): the tests compare millions of them with IEEE division
void dc_dec_decode_many(const int64_t* k, uint64_t n, uint32_t e, uint64_t* out) {
  const DecScale s = dec_scale(e);
  for (uint64_t i = 0; i < n; i++) out[i] = dec_decode_f64(k[i], s);
}
uint64_t dc_for_encode(int64_t v, int64_t base) { return for_encode(v, base); }
int64_t dc_for_decode(int64_t base, uint32_t bits) { return for_decode(base, bits); }
uint32_t dc_bit_width(uint64_t x) { return bit_width_u64(x); }
int64_t dc_f64_key(uint64_t bits) { return f64_order_key(bits); }
uint64_t dc_f64_from_key(int64_t k) { return f64_from_order_key(k); }
int dc_like(const uint8_t* s, uint32_t n, const uint8_t* p, uint32_t m, uint32_t kind, int ci) {
  return like_match(s, n, p, m, kind, ci != 0);
}
uint64_t dc_load_u64(const uint8_t* base, uint32_t off) { return load_u64_unaligned(base + off); }
}

// ---- replica of k_scan's per-slab run directory + the octet pass (TEST ONLY) --------------------
// k_scan's slab control and octet_leaf / fast_and_rows live in scan_kernel.cuh as device code; this is
// the same algorithm over one NULL-free dictionary page on the CPU (octet_leaf_replica is the device
// function's text with the funnel-shift intrinsic spelled out), so random run structures, every bit
// width, the directory budget, slabs shrunk to what the walker covered and the straddling-octet path
// are exercised without a GPU.
static inline uint32_t host_funnelshift_r(uint32_t lo, uint32_t hi, uint32_t sh) {
  const uint64_t both = (uint64_t(hi) << 32) | lo;
  return uint32_t(both >> (sh & 31));
}
constexpr int kLutCacheBytes = 2048;
static inline uint32_t octet_leaf_replica(const uint32_t* dirw, uint32_t nent, const uint32_t* win,
                                               uint32_t bw, uint32_t r, uint32_t need, bool smem_lut,
                                               const uint8_t* lut_s, const uint8_t* lut_g) {
  // directory entry holding row r: {start, count | kind << 16 | chunk0 << 24, payload}; two sentinel
  // entries (start = ~0) follow the last one
  uint32_t e = 0;
  if (nent > 6) {
    for (uint32_t step = 32; step; step >>= 1) {
      const uint32_t c = e + step;
      if (c < nent && dirw[c * kDirWords] <= r) e = c;
    }
  } else {
    while (dirw[(e + 1) * kDirWords] <= r) e++;
  }
  const uint32_t* A = dirw + e * kDirWords;
  const uint32_t start = A[0], meta = A[1], payload = A[2], next = A[kDirWords];
  const uint32_t vmask = bw >= 32 ? 0xffffffffu : ((1u << bw) - 1u);
  uint32_t m = 0;
  if (r + 8 <= next) {
    if (!(meta & 0x10000u)) {  // RLE run: one value answers the whole octet
      const uint32_t t = smem_lut ? lut_s[payload & (kLutCacheBytes - 1)] : lut_g[payload];
      return t ? 0xffu : 0u;
    }
    const uint32_t bit0 = payload + (r - start) * bw;
    if (bw <= 8) {
      // the octet is at most 64 bits: three words cover it at any bit phase
      const uint32_t wi = bit0 >> 5, sh = bit0 & 31;
      const uint32_t x0 = win[wi], x1 = win[wi + 1], x2 = win[wi + 2];
      const uint32_t lo = host_funnelshift_r(x0, x1, sh), hi = host_funnelshift_r(x1, x2, sh);
      if (smem_lut) {
        for (int k = 7; k >= 0; k--) {
          const uint32_t s = uint32_t(k) * bw;
          const uint32_t v = (s < 32 ? host_funnelshift_r(lo, hi, s) : (hi >> (s - 32))) & vmask;
          m = m * 2 + lut_s[v];
        }
      } else {
        for (int k = 7; k >= 0; k--) {
          const uint32_t s = uint32_t(k) * bw;
          const uint32_t v = (s < 32 ? host_funnelshift_r(lo, hi, s) : (hi >> (s - 32))) & vmask;
          m = m * 2 + (((need >> k) & 1) ? uint32_t(lut_g[v]) : 0u);
        }
      }
      return m;
    }
    for (int k = 7; k >= 0; k--) {
      uint32_t t = 0;
      if ((need >> k) & 1) {
        const uint32_t bit = bit0 + uint32_t(k) * bw;
        const uint32_t wi = bit >> 5;
        const uint32_t v = host_funnelshift_r(win[wi], win[wi + 1], bit & 31) & vmask;
        t = smem_lut ? lut_s[v & (kLutCacheBytes - 1)] : lut_g[v];
      }
      m = m * 2 + t;
    }
    return m;
  }
  // the octet straddles directory entries (short runs, e.g. a skewed `level` column): entry by entry,
  // an RLE run answers all its rows of the octet with one LUT probe
  uint32_t k = 0;
  while (k < 8) {
    while (dirw[(e + 1) * kDirWords] <= r + k) e++;
    const uint32_t* B = dirw + e * kDirWords;
    const uint32_t nx = B[kDirWords];
    const uint32_t kend = nx - r < 8u ? nx - r : 8u;      // first row of the octet past this entry
    const uint32_t seg = ((1u << kend) - 1u) & ~((1u << k) - 1u);
    if (need & seg) {
      if (!(B[1] & 0x10000u)) {
        const uint32_t t = smem_lut ? lut_s[B[2] & (kLutCacheBytes - 1)] : lut_g[B[2]];
        if (t) m |= seg;
      } else {
        uint32_t bit = B[2] + (r + k - B[0]) * bw;
        for (uint32_t j = k; j < kend; j++, bit += bw) {
          if (!((need >> j) & 1)) continue;
          const uint32_t wi = bit >> 5;
          const uint32_t v = host_funnelshift_r(win[wi], win[wi + 1], bit & 31) & vmask;
          const uint32_t t = smem_lut ? lut_s[v & (kLutCacheBytes - 1)] : lut_g[v];
          m |= (t ? 1u : 0u) << j;
        }
      }
    }
    k = kend;
  }
  return m;
}

// One page through k_scan's general path as MODE_FAST_AND runs it: per slab, issue_windows stages
// valwin_cap_for_bw(bw) bytes from the stream's window start, the walker builds the directory
// (kMaxDirEntries - 2 entries, two sentinels behind), and when it covers fewer rows than the slab's
// target, general_walk shrinks the slab to what it covered and walks again from the same cursor.  The
// octet pass then places the slab's selection bits in the page's bitmap the way fast_and_rows does.
// Returns the rows scanned (-1: the walker made no progress); *shrunk = slabs that were shrunk.
extern "C" int64_t dc_walk_octet_scan(const uint8_t* stream, uint64_t len, uint32_t bw, uint32_t n, const uint8_t* lut,
                                      uint32_t smem_lut, uint32_t* bitmap, uint32_t* shrunk) {
  const uint32_t cap = valwin_cap_for_bw(bw);
  std::vector<uint8_t> arena(16 + len + cap + 64, 0);
  std::memcpy(arena.data() + 16, stream, len);
  StreamState st;
  stream_init(st, 16, 16 + len, bw);
  std::vector<uint32_t> win(cap / 4 + 8);
  std::vector<DirEntry> dir(kMaxDirEntries);
  uint32_t r_item = 0;
  *shrunk = 0;
  while (r_item < n) {
    const uint32_t target = n - r_item < (uint32_t)kSlabRows ? n - r_item : (uint32_t)kSlabRows;
    const uint64_t base = stream_window_start(st) & ~15ull;        // issue_windows: the TMA copy of the window
    std::memset(win.data(), 0, win.size() * 4);
    std::memcpy(win.data(), arena.data() + base, cap);
    const Window w{reinterpret_cast<const uint8_t*>(win.data()), base, cap};
    const StreamState snap = st;
    uint32_t nent = 0;
    uint32_t R = walk_stream(st, w, target, dir.data(), nent, kMaxDirEntries - 2);
    if (R < target) {                                                 // general_walk: shrink, walk again
      if (R == 0) return -1;
      ++*shrunk;
      st = snap;
      nent = 0;
      if (walk_stream(st, w, R, dir.data(), nent, kMaxDirEntries - 2) != R) return -1;
    }
    DirEntry* d = dir.data();                                         // dir_sentinels
    d[nent].start = 0xffffffffu; d[nent].count = 0; d[nent].kind = 0; d[nent].chunk0 = 0; d[nent].payload = 0; d[nent]._pad = 0;
    d[nent + 1] = d[nent];
    const uint32_t* dirw = reinterpret_cast<const uint32_t*>(d);
    // fast_and_rows: 256 threads x 8 rows; byte stores when the slab starts on a byte, else 32-row words ORed in
    uint8_t sel[kSlabRows / 8];
    for (uint32_t t = 0; t < kSlabRows / 8; t++) {
      const uint32_t r8 = t * 8;
      uint32_t sel8 = r8 >= R ? 0u : (R - r8 >= 8 ? 0xffu : ((1u << (R - r8)) - 1u));
      if (sel8) sel8 &= octet_leaf_replica(dirw, nent, win.data(), bw, r8, sel8, smem_lut != 0, lut, lut);
      sel[t] = uint8_t(sel8);
    }
    if ((r_item & 7u) == 0) {
      for (uint32_t t = 0; t < kSlabRows / 8; t++)
        if (sel[t]) reinterpret_cast<uint8_t*>(bitmap)[(r_item + t * 8) >> 3] = sel[t];
    } else {
      for (uint32_t wd = 0; wd < (uint32_t)kSlabWords; wd++) {
        const uint32_t v = sel[4 * wd] | (sel[4 * wd + 1] << 8) | (sel[4 * wd + 2] << 16) | (uint32_t(sel[4 * wd + 3]) << 24);
        if (v == 0) continue;
        const uint32_t pos = r_item + wd * 32, sh = pos & 31;
        uint32_t* dst = bitmap + (pos >> 5);
        if (sh == 0) *dst = v;
        else {
          dst[0] |= v << sh;
          if (v >> (32 - sh)) dst[1] |= v >> (32 - sh);
        }
      }
    }
    r_item += R;
  }
  return n;
}
