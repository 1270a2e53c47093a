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
// hybrid stream -> flat bit-packed words (the slab index's copy of run-heavy pages), `slab` values per call
int64_t dc_transcode(const uint8_t* stream, uint64_t len, uint32_t bw, uint32_t n, uint32_t slab, uint32_t* out_words) {
  std::vector<uint8_t> padded(len + 64 + 16, 0);
  std::memcpy(padded.data() + 16, stream, len);
  StreamState st;
  stream_init(st, 16, 16 + len, bw);
  BitWriter b{out_words, 0, 0};
  uint32_t done = 0;
  while (done < n) {
    uint32_t need = n - done < slab ? n - done : slab;
    uint32_t got = transcode_values(st, padded.data(), need, b);
    done += got;
    if (got < need) return -int64_t(done) - 1;
  }
  bitwriter_flush(b);
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

// ---- replica of the slab index + the octet pass (TEST ONLY) ------------------------------------
// k_slab_index / k_flatten_pages / octet_leaf live in scan_kernel.cuh as device code; this is the
// same algorithm over one page on the CPU (octet_leaf_replica is the device function's text with the
// funnel-shift intrinsic spelled out), so random run structures, every bit width, the entry budget,
// the flat-copy fallback and the straddling-octet path are exercised without a GPU.
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

extern "C" int64_t dc_index_octet_scan(const uint8_t* stream, uint64_t len, uint32_t bw, uint32_t n, const uint8_t* lut,
                                       uint32_t smem_lut, uint32_t budget_per_slab, uint8_t* out_bytes, int32_t* used_flat) {
  const uint32_t cap = ((kSlabRows * bw / 8 + kSlabRows / 8 + 64) + 15u) & ~15u;   // valwin_cap_for_bw
  std::vector<uint8_t> arena(16 + len + cap + 64, 0);
  std::memcpy(arena.data() + 16, stream, len);
  const uint32_t nslabs = (n + kSlabRows - 1) / kSlabRows;
  struct Rec { const uint8_t* win; uint32_t nent, ent0; };
  std::vector<Rec> recs(nslabs);
  const uint32_t budget = nslabs * budget_per_slab;
  std::vector<DirEntry> dirs(budget + 3 * nslabs + 8);
  std::vector<uint32_t> side;
  StreamState st;
  stream_init(st, 16, 16 + len, bw);
  uint32_t used = 0, rows_left = n;
  bool flat = false;
  for (uint32_t k = 0; k < nslabs && !flat; k++) {      // k_slab_index
    const uint32_t R = rows_left < (uint32_t)kSlabRows ? rows_left : (uint32_t)kSlabRows;
    const uint64_t base = stream_window_start(st) & ~15ull;
    const Window w{arena.data() + base, base, cap};
    uint32_t m = 0, got = 0;
    if (used + 3 <= budget) {
      const uint32_t room = budget - used - 2;
      got = walk_stream(st, w, R, dirs.data() + used, m, room < uint32_t(kMaxDirEntries - 2) ? room : uint32_t(kMaxDirEntries - 2));
    }
    if (got < R || m == 0) { flat = true; break; }
    DirEntry* d = dirs.data() + used;
    d[m].start = 0xffffffffu; d[m].count = 0; d[m].kind = 0; d[m].chunk0 = 0; d[m].payload = 0; d[m]._pad = 0; d[m + 1] = d[m];
    recs[k] = {arena.data() + base, m, used};
    used += m + 2;
    rows_left -= R;
  }
  *used_flat = flat ? 1 : 0;
  if (flat) {                                           // k_flatten_pages
    side.assign(size_t(n) * (bw ? bw : 1) / 32 + cap / 4 + 64, 0);
    stream_init(st, 16, 16 + len, bw);
    BitWriter b{side.data(), 0, 0};
    rows_left = n;
    for (uint32_t k = 0; k < nslabs; k++) {
      const uint32_t R = rows_left < (uint32_t)kSlabRows ? rows_left : (uint32_t)kSlabRows;
      if (transcode_values(st, arena.data(), R, b) < R) return -1;
      DirEntry* d = dirs.data() + 3 * k;
      d[0].start = 0; d[0].count = uint16_t(R); d[0].kind = bw ? 1 : 0; d[0].chunk0 = 0; d[0].payload = 0; d[0]._pad = 0;
      d[1].start = 0xffffffffu; d[1].count = 0; d[1].kind = 0; d[1].chunk0 = 0; d[1].payload = 0; d[1]._pad = 0; d[2] = d[1];
      recs[k] = {reinterpret_cast<const uint8_t*>(side.data()) + size_t(k) * (kSlabRows / 8) * bw, 1, 3 * k};
      rows_left -= R;
    }
    bitwriter_flush(b);
  }
  // the octet pass over every slab: 256 "threads" x 8 rows, windows and directories staged like the TMA copies
  std::vector<uint32_t> win(cap / 4 + 8), dirw(size_t(kMaxDirEntries) * kDirWords);
  rows_left = n;
  for (uint32_t k = 0; k < nslabs; k++) {
    const uint32_t R = rows_left < (uint32_t)kSlabRows ? rows_left : (uint32_t)kSlabRows;
    std::memcpy(win.data(), recs[k].win, cap);
    std::memcpy(dirw.data(), dirs.data() + recs[k].ent0, (recs[k].nent + 2) * sizeof(DirEntry));
    for (uint32_t t = 0; t < 256; t++) {
      const uint32_t r8 = t * 8;
      uint32_t sel8 = r8 >= R ? 0u : (R - r8 >= 8 ? 0xffu : ((1u << (R - r8)) - 1u));
      if (sel8) sel8 &= octet_leaf_replica(dirw.data(), recs[k].nent, win.data(), bw, r8, sel8, smem_lut != 0, lut, lut);
      if (size_t(k) * 256 + t < (size_t(n) + 7) / 8) out_bytes[size_t(k) * 256 + t] = uint8_t(sel8);
    }
    rows_left -= R;
  }
  return n;
}
