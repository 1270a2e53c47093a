// Flat store: the scan-ready form of a resident table, built once when the table is opened.
//
// Parquet's RLE / bit-packed hybrid is the only sequential part of the format: run headers every
// <= 504 values, RLE runs in between.  A kernel that reads it pays a directory lookup and a
// straddle path per value (round 1: 3.6 warp-instructions per row, 6 % of the HBM roofline).  The
// hot tier therefore keeps every NULL-free dictionary-index page a second way: the same indices at
// the same bit width, LSB first, WITHOUT headers and with RLE runs expanded — value i of the page
// is bits [i*bw, (i+1)*bw).  Any 128-row boundary is 16-byte aligned, so the scan stages slabs with
// plain TMA bulk copies and a thread finds its rows with one multiply.  Size = rows*bw/8, the same
// as the bit-packed original to within the run headers.  PLAIN INT64 / DOUBLE pages and numeric
// dictionaries are copied to 16-byte aligned positions (the file keeps them at arbitrary offsets
// behind their Thrift headers); PLAIN BOOLEAN pages already are 1-bit flat.
//
// One warp per page.  The run headers are walked out of a shared-memory tile (tens of cycles per
// header instead of an L2 round trip); the runs of a tile are then expanded by all 32 lanes, one
// destination word per lane.
//
// Replaces nothing in the reference: it is the GPU analogue of keeping the hot tier decoded to
// Arrow in memory (src/hottier.rs), except that values stay dictionary-encoded and bit-packed.
#pragma once
#include <cuda_runtime.h>

#include <climits>

#include "decode_core.cuh"
#include "device_structs.hpp"

namespace pqb {

constexpr int kFlatTile = 4096;       // bytes of one staged tile of the hybrid stream
constexpr int kFlatTileRuns = 96;     // runs parsed per round

struct FlatRun { uint32_t row0, count, kind, payload; };   // kind 0 RLE (payload = value), 1 bit-packed (payload = tile bit offset)

// 32 bits starting at bit `bit` of a 4-byte aligned word array
__device__ __forceinline__ uint32_t bits32_at(const uint32_t* w, uint32_t bit) {
  const uint32_t i = bit >> 5, sh = bit & 31;
  return __funnelshift_r(w[i], w[i + 1], sh);
}

// OR `nbits` bits (starting at destination bit `db`) produced by gen(k) = the 32 bits that start at
// run-relative bit k; all lanes of the warp take part.  Interior words are plain stores (a
// destination word inside one run belongs to that run alone), the first and last word of a run are
// shared with its neighbours and merged atomically into the zeroed destination.
template <typename Gen>
__device__ __forceinline__ void emit_bits(uint32_t* __restrict__ dst, uint64_t db, uint64_t nbits, Gen gen) {
  if (nbits == 0) return;
  const uint64_t w0 = db >> 5, w1 = (db + nbits - 1) >> 5;
  for (uint64_t w = w0 + (threadIdx.x & 31); w <= w1; w += 32) {
    const uint64_t wb = w << 5;
    const uint64_t lo = wb > db ? wb : db;
    const uint64_t hi = wb + 32 < db + nbits ? wb + 32 : db + nbits;
    uint32_t v = gen(uint32_t(lo - db));
    const uint32_t n = uint32_t(hi - lo);
    if (n < 32) v &= (1u << n) - 1u;
    v <<= uint32_t(lo - wb);
    if (lo == wb && n == 32) dst[w] = v;
    else if (v) atomicOr(&dst[w], v);
  }
}

// every definition level of the page must be 1 (RLE runs of 1s, or bit-packed groups of 1s)
__device__ inline bool def_levels_all_valid(const uint8_t* __restrict__ p, uint32_t len, uint32_t rows) {
  uint32_t pos = 0, covered = 0;
  while (covered < rows) {
    uint32_t h = 0;
    int shift = 0;
    bool ok = false;
    while (pos < len && shift < 35) {
      const uint32_t b = p[pos++];
      h |= (b & 0x7f) << shift;
      shift += 7;
      if (!(b & 0x80)) { ok = true; break; }
    }
    if (!ok) return false;
    if (h & 1) {
      const uint32_t groups = h >> 1;
      if (pos + groups > len) return false;
      for (uint32_t g = 0; g < groups; g++) {
        const uint32_t left = rows - covered;
        const uint32_t need = left >= 8 ? 0xffu : ((1u << left) - 1u);
        if ((p[pos + g] & need) != need) return false;
        covered += left >= 8 ? 8 : left;
        if (covered >= rows) break;
      }
      pos += groups;
    } else {
      if (pos >= len) return false;
      const uint32_t v = p[pos++];
      const uint32_t cnt = h >> 1;
      if (cnt == 0) continue;
      if (!(v & 1)) return false;
      covered += cnt;
    }
  }
  return true;
}

enum FlatJobKind : uint32_t { FJ_HYBRID = 1, FJ_COPY8 = 2, FJ_BITS = 3, FJ_DICT8 = 4, FJ_VALID = 5, FJ_BYTES = 6, FJ_DICT4 = 7, FJ_WIDEN4 = 8 };
// FJ_HYBRID: RLE / bit-packed hybrid stream -> flat bits       (page)
// FJ_COPY8 : PLAIN 8-byte values -> aligned copy               (page)
// FJ_BITS  : PLAIN boolean bits -> aligned copy                (page)
// FJ_DICT8 : numeric dictionary (8-byte entries) -> aligned copy (src = arena offset, rows = entries)
// FJ_VALID : validity bitmap only (a DELTA page with NULLs: its values follow on demand, ensure_plain8)
// FJ_BYTES : PLAIN BYTE_ARRAY page (dictionary fallback, streams.rs:584-631) -> u32 start of every row's bytes
// FJ_DICT4 : Date32 dictionary (4-byte INT32 entries) -> sign-extended 8-byte copy, as FJ_DICT8 writes it
// FJ_WIDEN4: PLAIN Date32 page (4-byte INT32 values) -> sign-extended 8-byte values, as FJ_COPY8 writes them (FK_PLAIN8)
// A page with NULLs (vdst != ~0) also gets its validity bitmap (1 bit per ROW, from the definition
// levels) and its values EXPANDED to one slot per row (NULL rows hold 0), so that row r of the page
// is slot r whatever the NULLs: the scan needs no rank / prefix popcount.
struct FlatStoreJob {
  uint64_t src;      // FJ_DICT8: arena offset of the dictionary payload
  uint64_t dst;      // byte offset in the flat buffer (16-byte aligned)
  uint64_t vdst;     // validity bitmap in the flat buffer, or ~0: the page holds no NULLs
  uint64_t tmp;      // FJ_HYBRID with NULLs: scratch for the dense (non-null only) values, in the flat buffer
  uint32_t page;     // page index (page jobs)
  uint32_t kind;     // FlatJobKind
  uint32_t rows;     // FJ_DICT8: entries
  uint32_t _pad;
};

// 0: every definition level is 1; 1: the page holds NULLs; one thread per page
__global__ void k_page_has_nulls(const uint8_t* __restrict__ arena, const DevPage* __restrict__ pages, uint32_t n_pages,
                                 uint8_t* __restrict__ out) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_pages) return;
  const DevPage pg = pages[i];
  out[i] = (pg.def_len && !def_levels_all_valid(arena + pg.off + pg.def_off, pg.def_len, pg.num_rows)) ? 1 : 0;
}

// One RLE / bit-packed hybrid stream [s_begin, s_end) of `nvals` values at `bw` bits -> flat bits at dst
// (zeroed).  Warp cooperative; returns false for a stream the walker refuses.
__device__ __noinline__ bool flatten_hybrid(const uint8_t* __restrict__ arena, uint64_t s_begin, uint64_t s_end, uint32_t bw,
                                            uint32_t nvals, uint32_t* __restrict__ dst, uint8_t* tile, FlatRun* runs) {
  const uint32_t lane = threadIdx.x & 31;
  if (bw == 0 || nvals == 0) return true;   // a one-entry dictionary has no bits at all
  // walker state (lane 0 authoritative, broadcast every round)
  uint64_t p = s_begin;        // next unread stream byte: a run header, or the data of a bit-packed run in progress
  uint32_t row = 0;            // values emitted so far
  uint32_t bp_left = 0;        // groups of 8 left in the bit-packed run in progress
  uint32_t bad = 0;
  const uint32_t vbytes = (bw + 7) >> 3;
  while (row < nvals && !bad) {
    const uint64_t t0 = p & ~15ull;
    for (uint32_t o = lane * 16; o < uint32_t(kFlatTile) + 16; o += 32 * 16)
      *reinterpret_cast<uint4*>(tile + o) = *reinterpret_cast<const uint4*>(arena + t0 + o);
    __syncwarp();
    bool refill = false;
    while (row < nvals && !bad && !refill) {
      uint32_t nruns = 0;
      if (lane == 0) {
        while (row < nvals && nruns < uint32_t(kFlatTileRuns)) {
          uint32_t rel = uint32_t(p - t0);
          if (bp_left == 0) {
            if (p >= s_end) { bad = 1; break; }
            if (rel + 5 + vbytes > uint32_t(kFlatTile) && rel > 16) { refill = true; break; }
            uint32_t h = 0, q = rel;
            int shift = 0;
            bool okh = false;
            while (shift < 35 && t0 + q < s_end) {
              const uint32_t b = tile[q++];
              h |= (b & 0x7f) << shift;
              shift += 7;
              if (!(b & 0x80)) { okh = true; break; }
            }
            if (!okh) { bad = 1; break; }
            if (h & 1) {
              bp_left = h >> 1;
              p = t0 + q;
              if (bp_left == 0) continue;
              rel = q;
            } else {
              uint32_t v = 0;
              for (uint32_t i = 0; i < vbytes; i++) v |= uint32_t(tile[q + i]) << (8 * i);
              p = t0 + q + vbytes;
              uint32_t cnt = h >> 1;
              if (cnt == 0) continue;
              if (cnt > nvals - row) cnt = nvals - row;
              runs[nruns++] = FlatRun{row, cnt, 0u, bw >= 32 ? v : (v & ((1u << bw) - 1u))};
              row += cnt;
              continue;
            }
          }
          // bit-packed data at tile offset rel: whole groups of 8 values = bw bytes each
          uint32_t fit = (uint32_t(kFlatTile) - rel) / bw;
          if (fit == 0) { refill = true; break; }
          if (fit > bp_left) fit = bp_left;
          if (p + uint64_t(fit) * bw > s_end + 8) { bad = 1; break; }   // runs may be padded, never far past the page
          uint32_t cnt = fit * 8;
          if (cnt > nvals - row) cnt = nvals - row;
          runs[nruns++] = FlatRun{row, cnt, 1u, rel * 8};
          row += cnt;
          p += uint64_t(fit) * bw;
          bp_left -= fit;
          if (row >= nvals) bp_left = 0;
        }
      }
      nruns = __shfl_sync(0xffffffffu, nruns, 0);
      row = __shfl_sync(0xffffffffu, row, 0);
      bad = __shfl_sync(0xffffffffu, bad, 0);
      refill = __shfl_sync(0xffffffffu, refill ? 1u : 0u, 0) != 0;
      p = __shfl_sync(0xffffffffu, p, 0);
      bp_left = __shfl_sync(0xffffffffu, bp_left, 0);
      __syncwarp();
      const uint32_t* tw = reinterpret_cast<const uint32_t*>(tile);
      for (uint32_t r = 0; r < nruns; r++) {
        const FlatRun rn = runs[r];
        const uint64_t db = uint64_t(rn.row0) * bw, nb = uint64_t(rn.count) * bw;
        if (rn.kind) {
          const uint32_t sb = rn.payload;
          emit_bits(dst, db, nb, [&](uint32_t k) { return bits32_at(tw, sb + k); });
        } else if (rn.payload) {
          uint64_t rep = 0;
          for (uint32_t s = 0; s < 64; s += bw) rep |= uint64_t(rn.payload) << s;
          emit_bits(dst, db, nb, [&](uint32_t k) { return uint32_t(rep >> (k % bw)); });
        }
      }
      __syncwarp();
      if (nruns == 0 && !refill && !bad && row < nvals) bad = 1;   // no progress: corrupt stream
    }
  }
  return !bad;
}

// non-null values of a page = set bits of its validity bitmap (warp cooperative)
__device__ __forceinline__ uint32_t warp_count_valid(const uint32_t* __restrict__ valid, uint32_t rows) {
  const uint32_t lane = threadIdx.x & 31;
  uint32_t c = 0;
  for (uint32_t w = lane; w < (rows + 31) / 32; w += 32) {
    uint32_t x = valid[w];
    if (w * 32 + 32 > rows) x &= (1u << (rows - w * 32)) - 1u;
    c += __popc(x);
  }
  return __reduce_add_sync(0xffffffffu, c);
}

// Dense (non-null only) values -> one slot per row.  get(k) = k-th dense value; put(r, v) stores row r.
template <typename Get, typename Put>
__device__ __forceinline__ void expand_rows(const uint32_t* __restrict__ valid, uint32_t rows, Get get, Put put) {
  const uint32_t lane = threadIdx.x & 31;
  uint32_t base = 0;
  for (uint32_t r0 = 0; r0 < rows; r0 += 32) {
    const uint32_t r = r0 + lane;
    const uint32_t word = valid[r0 >> 5] & (rows - r0 >= 32 ? 0xffffffffu : ((1u << (rows - r0)) - 1u));
    const bool v = (word >> lane) & 1u;
    const uint32_t rank = base + __popc(word & ((1u << lane) - 1u));
    put(r, v, v ? get(rank) : 0ull, word);
    base += __popc(word);
  }
}

__global__ void __launch_bounds__(128) k_flat_store(const uint8_t* __restrict__ arena, const DevPage* __restrict__ pages,
                                                    const FlatStoreJob* __restrict__ jobs, uint32_t n_jobs,
                                                    uint8_t* __restrict__ flat, uint8_t* __restrict__ ok_out, uint32_t* __restrict__ maxlen_out) {
  __shared__ __align__(16) uint8_t tiles[4][kFlatTile + 16];
  __shared__ FlatRun runs_s[4][kFlatTileRuns];
  const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const uint32_t ji = blockIdx.x * 4 + warp;
  if (ji >= n_jobs) return;
  const FlatStoreJob job = jobs[ji];
  if (job.kind == FJ_DICT8 || job.kind == FJ_DICT4) {
    uint64_t* d = reinterpret_cast<uint64_t*>(flat + job.dst);
    if (job.kind == FJ_DICT8)
      for (uint32_t i = lane; i < job.rows; i += 32) d[i] = load_u64_unaligned(arena + job.src + uint64_t(i) * 8);
    else
      for (uint32_t i = lane; i < job.rows; i += 32) d[i] = uint64_t(int64_t(int32_t(load_u32_unaligned(arena + job.src + uint64_t(i) * 4))));
    if (lane == 0) ok_out[ji] = 1;
    return;
  }
  const DevPage pg = pages[job.page];
  uint8_t* tile = tiles[warp];
  FlatRun* runs = runs_s[warp];
  const bool has_nulls = job.vdst != ~0ull;
  const uint32_t rows = pg.num_rows;
  uint32_t* valid = reinterpret_cast<uint32_t*>(flat + job.vdst);
  uint32_t nn = rows;   // non-null values
  if (has_nulls) {
    // definition levels (bit width 1) -> validity bitmap, 1 bit per row
    if (!flatten_hybrid(arena, pg.off + pg.def_off, pg.off + pg.def_off + pg.def_len, 1, rows, valid, tile, runs)) {
      if (lane == 0) ok_out[ji] = 0;
      return;
    }
    __syncwarp();
    __threadfence_block();
    nn = warp_count_valid(valid, rows);
  }
  const uint8_t* vals = arena + pg.off + pg.val_off;
  if (job.kind == FJ_VALID) { if (lane == 0) ok_out[ji] = 1; return; }
  if (job.kind == FJ_BYTES) {
    // [len][bytes][len][bytes]...: a chain, walked by lane 0 out of shared-memory tiles; NULL rows own no bytes
    uint32_t* offs = reinterpret_cast<uint32_t*>(flat + job.dst);
    const uint64_t v0 = pg.off + pg.val_off, vend = pg.off + pg.len;
    uint64_t p = v0;
    uint32_t r = 0, bad = 0, maxlen = 0;
    while (r < rows && !bad) {
      const uint64_t t0 = p & ~15ull;
      for (uint32_t o = lane * 16; o < uint32_t(kFlatTile) + 16; o += 32 * 16)
        *reinterpret_cast<uint4*>(tile + o) = *reinterpret_cast<const uint4*>(arena + t0 + o);
      __syncwarp();
      if (lane == 0) {
        while (r < rows) {
          if (has_nulls && !((valid[r >> 5] >> (r & 31)) & 1u)) { offs[r++] = 0; continue; }
          if (p + 4 > vend) { bad = 1; break; }
          const uint32_t rel = uint32_t(p - t0);
          if (rel + 4 > uint32_t(kFlatTile)) break;   // next length prefix is outside this tile
          const uint32_t len = uint32_t(tile[rel]) | (uint32_t(tile[rel + 1]) << 8) | (uint32_t(tile[rel + 2]) << 16) | (uint32_t(tile[rel + 3]) << 24);
          if (p + 4 + uint64_t(len) > vend) { bad = 1; break; }
          if (len > maxlen) maxlen = len;
          offs[r++] = uint32_t(p + 4 - v0);
          p += 4 + uint64_t(len);
        }
      }
      r = __shfl_sync(0xffffffffu, r, 0);
      p = __shfl_sync(0xffffffffu, p, 0);
      bad = __shfl_sync(0xffffffffu, bad, 0);
      __syncwarp();
    }
    if (lane == 0) {
      ok_out[ji] = bad ? 0 : 1;
      if (maxlen_out) maxlen_out[ji] = maxlen;
    }
    return;
  }
  if (job.kind == FJ_COPY8) {
    if (uint64_t(pg.val_off) + uint64_t(nn) * 8 > pg.len) { if (lane == 0) ok_out[ji] = 0; return; }
    uint64_t* d = reinterpret_cast<uint64_t*>(flat + job.dst);
    if (!has_nulls) {
      for (uint32_t i = lane; i < rows; i += 32) d[i] = load_u64_unaligned(vals + uint64_t(i) * 8);
    } else {
      expand_rows(valid, rows, [&](uint32_t k) { return load_u64_unaligned(vals + uint64_t(k) * 8); },
                  [&](uint32_t r, bool, uint64_t v, uint32_t) { if (r < rows) d[r] = v; });
    }
    if (lane == 0) ok_out[ji] = 1;
    return;
  }
  if (job.kind == FJ_WIDEN4) {
    if (uint64_t(pg.val_off) + uint64_t(nn) * 4 > pg.len) { if (lane == 0) ok_out[ji] = 0; return; }
    uint64_t* d = reinterpret_cast<uint64_t*>(flat + job.dst);
    auto at = [&](uint32_t k) { return uint64_t(int64_t(int32_t(load_u32_unaligned(vals + uint64_t(k) * 4)))); };
    if (!has_nulls) {
      for (uint32_t i = lane; i < rows; i += 32) d[i] = at(i);
    } else {
      expand_rows(valid, rows, at, [&](uint32_t r, bool, uint64_t v, uint32_t) { if (r < rows) d[r] = v; });
    }
    if (lane == 0) ok_out[ji] = 1;
    return;
  }
  if (job.kind == FJ_BITS) {
    if (uint64_t(pg.val_off) + ((nn + 7) >> 3) > pg.len) { if (lane == 0) ok_out[ji] = 0; return; }
    uint32_t* d = reinterpret_cast<uint32_t*>(flat + job.dst);
    if (!has_nulls) {
      const uint32_t nw = (rows + 31) >> 5;
      for (uint32_t i = lane; i < nw; i += 32) d[i] = load_u32_unaligned(vals + uint64_t(i) * 4);
    } else {
      expand_rows(valid, rows, [&](uint32_t k) { return uint64_t((vals[k >> 3] >> (k & 7)) & 1u); },
                  [&](uint32_t r, bool v, uint64_t x, uint32_t) {
                    const uint32_t w = __ballot_sync(0xffffffffu, v && x);
                    if (lane == 0) d[r >> 5] = w;
                  });
    }
    if (lane == 0) ok_out[ji] = 1;
    return;
  }
  // ---- FJ_HYBRID ----
  const uint32_t bw = pg.bit_width;
  uint32_t* dst = reinterpret_cast<uint32_t*>(flat + job.dst);
  const uint64_t s_begin = pg.off + pg.val_off, s_end = pg.off + pg.len;
  bool ok;
  if (!has_nulls) ok = flatten_hybrid(arena, s_begin, s_end, bw, rows, dst, tile, runs);
  else {
    uint32_t* tmp = reinterpret_cast<uint32_t*>(flat + job.tmp);
    ok = flatten_hybrid(arena, s_begin, s_end, bw, nn, tmp, tile, runs);
    __syncwarp();
    __threadfence_block();
    if (ok && bw) {
      const uint32_t mask = bw >= 32 ? 0xffffffffu : ((1u << bw) - 1u);
      expand_rows(valid, rows, [&](uint32_t k) { return uint64_t(bits32_at(tmp, k * bw) & mask); },
                  [&](uint32_t r, bool v, uint64_t x, uint32_t) {
                    if (!v || !x) return;
                    const uint64_t bit = uint64_t(r) * bw;
                    const uint32_t sh = uint32_t(bit & 31);
                    atomicOr(&dst[bit >> 5], uint32_t(x) << sh);
                    if (sh + bw > 32) atomicOr(&dst[(bit >> 5) + 1], uint32_t(x) >> (32 - sh));
                  });
    }
  }
  if (lane == 0) ok_out[ji] = ok ? 1 : 0;
}

// Every dictionary index of the flat store against its dictionary's entry count, once per table: the reference's
// reader fails a file whose index leaves the dictionary, and nothing downstream has to trust the file after this
// (the scan kernels still clamp: a LUT is never left).  One warp per page; first_bad = lowest failing page index.
__global__ void __launch_bounds__(128) k_check_flat_indices(const uint8_t* __restrict__ flat, const FlatPageRec* __restrict__ fpages,
                                                            const uint32_t* __restrict__ dict_n, uint32_t n_pages, uint32_t* __restrict__ first_bad) {
  const uint32_t lane = threadIdx.x & 31;
  const uint32_t pi = blockIdx.x * 4 + (threadIdx.x >> 5);
  if (pi >= n_pages) return;
  const FlatPageRec fp = fpages[pi];
  if (fp.fkind != FK_INDEX || fp.bw == 0) return;
  const uint32_t limit = dict_n[pi] ? dict_n[pi] : 1u;             // NULL rows hold slot value 0
  if (fp.bw < 32 && limit >= (1u << fp.bw)) return;                 // every bw-bit value is an entry
  const uint32_t* w = reinterpret_cast<const uint32_t*>(flat + fp.off);
  const uint32_t mask = fp.bw >= 32 ? 0xffffffffu : ((1u << fp.bw) - 1u);
  bool bad = false;
  for (uint32_t i = lane; i < fp.rows; i += 32) bad |= (bits32_at(w, i * fp.bw) & mask) >= limit;
  if (__any_sync(0xffffffffu, bad) && lane == 0) atomicMin(first_bad, pi);
}

// ---- agg pages: what k_flat_agg reads instead of a dictionary index when the index only ever looks something up ----
// Built once per table column (Table::ensure_for_pages / ensure_id_pages) and kept with the table:
//   FK_FOR  value page of a numeric dictionary page: base + w-bit offset per row (decode_core.cuh: for_* / dec_*)
//   FK_IDS  id page of a GROUP BY key's dictionary page: the row's group id at bits(card - 1) bits
// Both follow the flat store's conventions: 16-byte aligned, row r at bits [r*w, (r+1)*w), NULL rows hold 0, the index
// page's validity bitmap is reused.
struct ForChunkJob { uint64_t dict8; uint32_t n; uint32_t f64; };
struct ForChunkInfo { int64_t base; uint32_t w; uint32_t e; uint32_t ok; uint32_t _pad; };

template <typename T, typename Op>
__device__ __forceinline__ T block_reduce_256(T v, T* s, Op op) {   // 256 threads; s holds 8 T
  for (int o = 16; o; o >>= 1) v = op(v, __shfl_xor_sync(0xffffffffu, v, o));
  __syncthreads();
  if ((threadIdx.x & 31) == 0) s[threadIdx.x >> 5] = v;
  __syncthreads();
  v = s[0];
  for (int w = 1; w < 8; w++) v = op(v, s[w]);
  return v;
}

// One block per chunk: can every dictionary entry be written as base + w bits (w <= 32)?  Float64: the smallest decimal
// exponent e at which every entry has its k.
__global__ void __launch_bounds__(256) k_for_classify(const uint8_t* __restrict__ flat, const ForChunkJob* __restrict__ jobs,
                                                      ForChunkInfo* __restrict__ out) {
  __shared__ long long s_ll[8];
  __shared__ uint32_t s_u[8];
  const ForChunkJob j = jobs[blockIdx.x];
  const uint64_t* __restrict__ d = reinterpret_cast<const uint64_t*>(flat + j.dict8);
  uint32_t e = 0;
  if (j.f64) {
    uint32_t fail = 0;   // bit e: some entry has no k at exponent e
    for (uint32_t i = threadIdx.x; i < j.n && fail != (2u << kForMaxExp) - 1u; i += 256) {
      const uint64_t b = d[i];
      for (uint32_t x = 0; x <= kForMaxExp; x++) {
        int64_t k;
        if (!((fail >> x) & 1u) && !dec_encode_f64(b, dec_scale(x), k)) fail |= 1u << x;
      }
    }
    fail = block_reduce_256<uint32_t>(fail, s_u, [](uint32_t a, uint32_t b) { return a | b; });
    e = __ffs(~fail) - 1;
    if (e > kForMaxExp) {
      if (threadIdx.x == 0) out[blockIdx.x] = ForChunkInfo{0, 0, 0, 0, 0};
      return;
    }
  }
  const DecScale p10 = dec_scale(e);
  long long lo = LLONG_MAX, hi = LLONG_MIN;
  for (uint32_t i = threadIdx.x; i < j.n; i += 256) {
    int64_t k = int64_t(d[i]);
    if (j.f64) dec_encode_f64(d[i], p10, k);
    lo = k < lo ? k : lo;
    hi = k > hi ? k : hi;
  }
  __syncthreads();
  lo = block_reduce_256<long long>(lo, s_ll, [](long long a, long long b) { return a < b ? a : b; });
  __syncthreads();
  hi = block_reduce_256<long long>(hi, s_ll, [](long long a, long long b) { return a > b ? a : b; });
  if (threadIdx.x == 0) {
    const uint32_t w = j.n ? bit_width_u64(for_encode(hi, lo)) : 0u;
    out[blockIdx.x] = ForChunkInfo{j.n ? lo : 0, w, e, (j.n && w <= kForMaxBits) ? 1u : 0u, 0};
  }
}

enum AggFormKind : uint32_t { AF_I64 = 0, AF_F64 = 1, AF_IDS = 2 };
struct AggFormJob {
  uint64_t src;      // the FK_INDEX page (flat offset)
  uint64_t dst;      // its agg page (flat offset, may wrap: a buffer of its own)
  uint64_t voff;     // validity bitmap of the index page, or ~0
  uint64_t table;    // AF_I64 / AF_F64: the chunk's 8-byte dictionary (flat offset); AF_IDS: device address of gid + lut_base
  int64_t base;
  uint32_t rows, sbw, dict_n, w, e, kind;
};
// One warp per page; a lane writes whole groups of 32 rows = w words, so no word is shared between lanes.
__global__ void __launch_bounds__(128) k_agg_form_pack(uint8_t* __restrict__ flat, const AggFormJob* __restrict__ jobs, uint32_t n_jobs) {
  const uint32_t lane = threadIdx.x & 31;
  const uint32_t ji = blockIdx.x * 4 + (threadIdx.x >> 5);
  if (ji >= n_jobs) return;
  const AggFormJob j = jobs[ji];
  const uint32_t* __restrict__ src = reinterpret_cast<const uint32_t*>(flat + j.src);
  const uint32_t* __restrict__ valid = j.voff != ~0ull ? reinterpret_cast<const uint32_t*>(flat + j.voff) : nullptr;
  const uint64_t* __restrict__ dict = reinterpret_cast<const uint64_t*>(flat + j.table);
  const uint32_t* __restrict__ gid = reinterpret_cast<const uint32_t*>(j.table);
  uint32_t* __restrict__ dst = reinterpret_cast<uint32_t*>(flat + j.dst);
  const uint32_t smask = j.sbw >= 32 ? 0xffffffffu : ((1u << j.sbw) - 1u), dict_max = j.dict_n ? j.dict_n - 1 : 0u;
  const DecScale p10 = dec_scale(j.e);
  for (uint32_t g = lane; g * 32 < j.rows; g += 32) {
    const uint32_t vw = valid ? valid[g] : 0xffffffffu;
    uint32_t* out = dst + size_t(g) * j.w;
    uint64_t acc = 0;
    uint32_t nacc = 0;
    for (uint32_t k = 0; k < 32; k++) {
      const uint32_t r = g * 32 + k;
      uint32_t x = 0;
      if (r < j.rows && ((vw >> k) & 1u)) {
        uint32_t idx = j.sbw ? (bits32_at(src, r * j.sbw) & smask) : 0u;
        idx = idx < dict_max ? idx : dict_max;   // as col_index: a corrupt index never leaves the dictionary
        if (j.kind == AF_IDS) x = gid[idx];
        else {
          int64_t v = int64_t(dict[idx]);
          if (j.kind == AF_F64) dec_encode_f64(dict[idx], p10, v);   // succeeds: k_for_classify tried every entry
          x = uint32_t(for_encode(v, j.base));
        }
      }
      acc |= uint64_t(x) << nacc;
      nacc += j.w;
      if (nacc >= 32) { *out++ = uint32_t(acc); acc >>= 32; nacc -= 32; }
    }
  }
}

// ---- tuple id pages: one id per GROUP BY key tuple (Table::ensure_tuple_pages) ----
// A job is a row range of one lead-column page over which every key column stays inside one page.  The row's group is
// the mixed radix of its keys' ids, exactly as k_flat_agg forms it from per-key pages (NULL and an absent chunk: id
// card).  k_tuple_count counts the rows of every group that occurs; k_tuple_pack writes each row's tuple id (the
// group's rank by count) into the lead page's tuple page at w bits, ORing into a zeroed buffer where jobs share a word.
struct TupleKeySrc {
  uint64_t src;        // the key's FK_INDEX page (flat offset)
  uint64_t voff;       // its validity bitmap, or ~0
  const uint32_t* gid; // gid LUT of the chunk (device address of gid + the row group's base); nullptr: chunk absent
  uint32_t row0, sbw, dict_n, _pad;
};
struct TupleJob {
  uint64_t dst;        // the lead page's tuple page (flat offset, may wrap: a buffer of its own)
  uint32_t row0, rows; // rows [row0, row0 + rows) of the lead page
  TupleKeySrc k[kMaxKeys];
};
struct TupleArgs {
  const TupleJob* jobs;
  uint32_t n_jobs, nkeys, w;
  uint32_t card[kMaxKeys], stride[kMaxKeys];
  unsigned int* counts;   // k_tuple_count: rows per mixed-radix id
  const uint32_t* rank;   // k_tuple_pack: tuple id per mixed-radix id
};
__device__ __forceinline__ uint32_t tuple_mixed(const uint8_t* __restrict__ flat, const TupleArgs& a, const TupleJob& j, uint32_t r) {
  uint32_t m = 0;
  for (uint32_t k = 0; k < a.nkeys; k++) {
    const TupleKeySrc& s = j.k[k];
    uint32_t id = a.card[k];
    const uint32_t rr = s.row0 + r;
    if (s.gid && (s.voff == ~0ull || ((reinterpret_cast<const uint32_t*>(flat + s.voff)[rr >> 5] >> (rr & 31)) & 1u))) {
      const uint32_t smask = s.sbw >= 32 ? 0xffffffffu : ((1u << s.sbw) - 1u), dict_max = s.dict_n ? s.dict_n - 1 : 0u;
      uint32_t idx = s.sbw ? (bits32_at(reinterpret_cast<const uint32_t*>(flat + s.src), rr * s.sbw) & smask) : 0u;
      idx = idx < dict_max ? idx : dict_max;   // as col_index: a corrupt index never leaves the dictionary
      id = s.gid[idx];
    }
    m += id * a.stride[k];
  }
  return m;
}
// one warp per job; lanes that meet the same group add once
__global__ void __launch_bounds__(128) k_tuple_count(const uint8_t* __restrict__ flat, const __grid_constant__ TupleArgs a) {
  const uint32_t lane = threadIdx.x & 31;
  const uint32_t ji = blockIdx.x * 4 + (threadIdx.x >> 5);
  if (ji >= a.n_jobs) return;
  const TupleJob& j = a.jobs[ji];
  for (uint32_t r0 = 0; r0 < j.rows; r0 += 32) {
    const uint32_t r = r0 + lane;
    const bool live = r < j.rows;
    const uint32_t m = live ? tuple_mixed(flat, a, j, r) : ~0u;
    const uint32_t peers = __match_any_sync(0xffffffffu, m);
    if (live && lane == uint32_t(__ffs(peers) - 1)) atomicAdd(a.counts + m, uint32_t(__popc(peers)));
  }
}
// one warp per job; a lane writes whole groups of 32 rows of the lead page (w words each)
__global__ void __launch_bounds__(128) k_tuple_pack(uint8_t* __restrict__ flat, const __grid_constant__ TupleArgs a) {
  const uint32_t lane = threadIdx.x & 31;
  const uint32_t ji = blockIdx.x * 4 + (threadIdx.x >> 5);
  if (ji >= a.n_jobs) return;
  const TupleJob& j = a.jobs[ji];
  uint32_t* __restrict__ dst = reinterpret_cast<uint32_t*>(flat + j.dst);
  const uint32_t g0 = j.row0 / 32, g1 = (j.row0 + j.rows + 31) / 32;
  for (uint32_t g = g0 + lane; g < g1; g += 32) {
    uint32_t* out = dst + size_t(g) * a.w;
    uint64_t acc = 0;
    uint32_t nacc = 0;
    for (uint32_t k = 0; k < 32; k++) {
      const uint32_t p = g * 32 + k;   // row of the lead page
      const uint32_t x = (p >= j.row0 && p < j.row0 + j.rows) ? a.rank[tuple_mixed(flat, a, j, p - j.row0)] : 0u;
      acc |= uint64_t(x) << nacc;
      nacc += a.w;
      if (nacc >= 32) {
        if (uint32_t(acc)) atomicOr(out, uint32_t(acc));
        out++;
        acc >>= 32;
        nacc -= 32;
      }
    }
  }
}

// ---- DELTA_BINARY_PACKED (Parseable's p_timestamp, streams.rs:587-590) -> aligned 8-byte values ----
// Only built when a query needs the VALUES of such a column (a time range that cuts a row group, a
// projection of p_timestamp): footer statistics decide the injected range for every other query and
// the column is then never read.  One warp per page: lane 0 walks the block headers (zigzag varints,
// one bit width per miniblock), the warp unpacks a miniblock's deltas in parallel and turns them into
// values with a shuffle scan carried across miniblocks.
struct DeltaJob { uint32_t page; uint32_t sext32 /* 1: an INT32 (Date32) stream, the low word sign-extended */; uint64_t dst; uint64_t vsrc /* validity bitmap of a page with NULLs (flat-base relative), or ~0 */; uint64_t tmp /* scratch for its dense values */; };

__device__ __forceinline__ bool rd_varint(const uint8_t* __restrict__ p, uint64_t& pos, uint64_t end, uint64_t& out) {
  uint64_t v = 0;
  for (int shift = 0; shift < 70; shift += 7) {
    if (pos >= end) return false;
    const uint32_t b = p[pos++];
    if (shift < 64) v |= uint64_t(b & 0x7f) << shift;
    if (!(b & 0x80)) { out = v; return true; }
  }
  return false;
}

// One DELTA_BINARY_PACKED stream starting at p[pos]: header <block size> <miniblocks per block> <total count> <first value>,
// then blocks of <min delta> <bit width per miniblock> <miniblocks>.  Warp cooperative; put(i, value) receives every
// value (64-bit wrapping arithmetic like the reference's decoder; an INT32 stream is the low word).  `want`: the count the
// caller expects, or ~0u to take the header's (returned through total_out, at most `cap`).  On return pos is the first
// byte after the stream: the last miniblock that holds values is stored in full, later ones not at all.
template <class Put>
__device__ __forceinline__ bool dbp_decode_warp(const uint8_t* __restrict__ p, uint64_t& pos, const uint64_t end, uint32_t want,
                                                uint32_t cap, uint32_t& total_out, Put put) {
  const uint32_t lane = threadIdx.x & 31;
  uint64_t bs = 0, nm = 0, total = 0, fz = 0;
  uint32_t bad = 0;
  if (lane == 0) {
    if (!rd_varint(p, pos, end, bs) || !rd_varint(p, pos, end, nm) || !rd_varint(p, pos, end, total) || !rd_varint(p, pos, end, fz)) bad = 1;
    if (!bad && (nm == 0 || bs == 0 || bs % nm != 0 || (bs / nm) % 32 != 0 || bs > (1u << 20))) bad = 1;
    if (!bad && (want != ~0u ? total != want : total > cap)) bad = 1;
  }
  bad = __shfl_sync(0xffffffffu, bad, 0);
  if (bad) return false;
  bs = __shfl_sync(0xffffffffu, bs, 0);
  nm = __shfl_sync(0xffffffffu, nm, 0);
  fz = __shfl_sync(0xffffffffu, fz, 0);
  pos = __shfl_sync(0xffffffffu, pos, 0);
  const uint32_t nvals = uint32_t(__shfl_sync(0xffffffffu, total, 0));
  total_out = nvals;
  const uint32_t vpm = uint32_t(bs / nm);   // values per miniblock, a multiple of 32
  int64_t last = int64_t(fz >> 1) ^ -int64_t(fz & 1);
  if (lane == 0 && nvals) put(0u, last);
  uint32_t done = 1;                        // values written
  while (done < nvals && !bad) {
    // block header: min delta + one bit width per miniblock (any number of miniblocks: the format only asks that a
    // miniblock hold a multiple of 32 values, and the Rust `parquet` crate or parquet-mr may write more than 32 of them)
    uint64_t mz = 0;
    if (lane == 0) { if (!rd_varint(p, pos, end, mz) || pos + nm > end) bad = 1; }
    bad = __shfl_sync(0xffffffffu, bad, 0);
    if (bad) break;
    mz = __shfl_sync(0xffffffffu, mz, 0);
    pos = __shfl_sync(0xffffffffu, pos, 0);
    const int64_t min_delta = int64_t(mz >> 1) ^ -int64_t(mz & 1);
    const uint64_t wpos = pos;
    pos += nm;
    for (uint32_t m = 0; m < nm && done < nvals; m++) {
      const uint32_t bw = p[wpos + m];   // the same byte for every lane: one broadcast load
      if (bw > 64 || pos + (uint64_t(vpm) * bw) / 8 > end + 8) { bad = 1; break; }
      const uint32_t take = nvals - done < vpm ? nvals - done : vpm;
      for (uint32_t v0 = 0; v0 < take; v0 += 32) {
        const uint32_t j = v0 + lane;
        uint64_t d = 0;
        if (bw && j < take) {
          const uint64_t bit = uint64_t(j) * bw;
          const uint8_t* q = p + pos + (bit >> 3);
          const uint32_t sh = uint32_t(bit & 7);
          d = load_u64_unaligned(q) >> sh;
          if (sh + bw > 64) d |= uint64_t(q[8]) << (64 - sh);
          if (bw < 64) d &= (1ull << bw) - 1ull;
        }
        uint64_t x = j < take ? uint64_t(min_delta) + d : 0ull, incl = x;
        for (int o = 1; o < 32; o <<= 1) {
          const uint64_t t = __shfl_up_sync(0xffffffffu, incl, o);
          if ((int)lane >= o) incl += t;
        }
        const uint64_t val = uint64_t(last) + incl;
        if (j < take) put(done + j, int64_t(val));
        last = int64_t(__shfl_sync(0xffffffffu, val, 31));
        if (take - v0 < 32) last = int64_t(__shfl_sync(0xffffffffu, val, (take - v0 - 1) & 31));
      }
      done += take;
      pos += (uint64_t(vpm) * bw) / 8;
    }
  }
  return !bad;
}

__global__ void __launch_bounds__(128) k_delta_to_plain8(const uint8_t* __restrict__ arena, const DevPage* __restrict__ pages,
                                                         const DeltaJob* __restrict__ jobs, uint32_t n_jobs, uint8_t* __restrict__ flat_base,
                                                         uint8_t* __restrict__ ok_out) {
  const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const uint32_t ji = blockIdx.x * 4 + warp;
  if (ji >= n_jobs) return;
  const DeltaJob job = jobs[ji];
  const DevPage pg = pages[job.page];
  // a page with NULLs holds only its non-null values: they are decoded densely, then spread over the row slots
  const bool has_nulls = job.vsrc != ~0ull;
  const uint32_t* valid = reinterpret_cast<const uint32_t*>(flat_base + job.vsrc);
  const uint32_t nvals = has_nulls ? warp_count_valid(valid, pg.num_rows) : pg.num_rows;
  const uint8_t* p = arena + pg.off;
  uint64_t pos = pg.val_off;
  int64_t* final_out = reinterpret_cast<int64_t*>(flat_base + job.dst);
  int64_t* out = has_nulls ? reinterpret_cast<int64_t*>(flat_base + job.tmp) : final_out;
  uint32_t total = 0;
  const bool ok = dbp_decode_warp(p, pos, uint64_t(pg.len), nvals, nvals, total,
                                  [&](uint32_t i, int64_t v) { out[i] = job.sext32 ? int64_t(int32_t(uint32_t(v))) : v; });
  if (has_nulls && ok) {
    __syncwarp();
    __threadfence_block();
    expand_rows(valid, pg.num_rows, [&](uint32_t k) { return uint64_t(out[k]); },
                [&](uint32_t r, bool, uint64_t v, uint32_t) { if (r < pg.num_rows) final_out[r] = int64_t(v); });
  }
  if (lane == 0) ok_out[ji] = ok ? 1 : 0;
}

// ---- DELTA_BYTE_ARRAY / DELTA_LENGTH_BYTE_ARRAY (the fallback encoding of Parseable's custom-partition columns,
// streams.rs:614-619) -> the same bytes as a PLAIN BYTE_ARRAY page ([u32 length][bytes]...), so that everything
// downstream sees one kind of string page.  Two passes, one warp per page:
//   k_dba_lengths     decodes the prefix / suffix length streams (DELTA_BINARY_PACKED INT32) into scratch and adds them up
//   k_dba_materialise writes the page: the level bytes as they are, then every value = the first <prefix> bytes of
//                     the previous value + its suffix (front coding is a chain: values one after the other, bytes in parallel)
__global__ void __launch_bounds__(128) k_dba_lengths(const uint8_t* __restrict__ arena, const DevPage* __restrict__ pages,
                                                     const DbaJob* __restrict__ jobs, uint32_t n_jobs, uint8_t* __restrict__ scratch,
                                                     DbaInfo* __restrict__ info) {
  const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const uint32_t ji = blockIdx.x * 4 + warp;
  if (ji >= n_jobs) return;
  const DbaJob job = jobs[ji];
  const DevPage pg = pages[job.page];
  const uint8_t* p = arena + pg.off;
  uint64_t pos = pg.val_off;
  uint32_t* plen = reinterpret_cast<uint32_t*>(scratch + job.len_tmp);
  uint32_t* slen = plen + pg.num_rows;
  uint32_t n = 0, n2 = 0;
  unsigned long long sum = 0;
  bool ok = true;
  if (pg.val_off >= pg.len) {   // an all-NULL page may carry no value bytes at all
    n = 0;
  } else {
    if (job.with_prefix) {
      ok = dbp_decode_warp(p, pos, uint64_t(pg.len), ~0u, pg.num_rows, n, [&](uint32_t i, int64_t v) { plen[i] = uint32_t(v); });
      if (ok) ok = dbp_decode_warp(p, pos, uint64_t(pg.len), n, n, n2, [&](uint32_t i, int64_t v) { slen[i] = uint32_t(v); });
    } else {
      ok = dbp_decode_warp(p, pos, uint64_t(pg.len), ~0u, pg.num_rows, n, [&](uint32_t i, int64_t v) { slen[i] = uint32_t(v); });
    }
    __syncwarp();
    __threadfence_block();
    if (ok) {
      // lengths are non-negative INT32; a prefix may not be longer than the previous value; suffix bytes must be in the page
      unsigned long long suf = 0;
      uint32_t bad = 0, prev_len = 0;
      for (uint32_t i0 = 0; i0 < n; i0 += 32) {
        const uint32_t i = i0 + lane;
        const uint32_t pl = (i < n && job.with_prefix) ? plen[i] : 0u, sl = i < n ? slen[i] : 0u;
        if ((pl | sl) & 0x80000000u) bad = 1;
        const uint32_t len = pl + sl;
        const uint32_t before = __shfl_up_sync(0xffffffffu, len, 1);
        if (i < n && pl > (lane ? before : prev_len)) bad = 1;
        prev_len = __shfl_sync(0xffffffffu, len, 31);
        sum += len;
        suf += sl;
      }
      for (int o = 16; o; o >>= 1) { sum += __shfl_xor_sync(0xffffffffu, sum, o); suf += __shfl_xor_sync(0xffffffffu, suf, o); }
      bad = __any_sync(0xffffffffu, bad);
      if (bad || pos + suf > pg.len) ok = false;
    }
  }
  if (lane == 0) info[ji] = {sum + 4ull * n, n, uint32_t(pos), ok ? 1u : 0u, 0u};
}

__global__ void __launch_bounds__(128) k_dba_materialise(const uint8_t* __restrict__ arena, const DevPage* __restrict__ pages,
                                                         const DbaJob* __restrict__ jobs, const DbaInfo* __restrict__ info, uint32_t n_jobs,
                                                         const uint8_t* __restrict__ scratch, uint8_t* __restrict__ mat) {
  const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const uint32_t ji = blockIdx.x * 4 + warp;
  if (ji >= n_jobs) return;
  const DbaJob job = jobs[ji];
  const DbaInfo in = info[ji];
  if (!in.ok) return;
  const DevPage pg = pages[job.page];
  const uint8_t* p = arena + pg.off;
  uint8_t* out = mat + job.dst;
  // level bytes first (the new page: definition levels at 0, values right after them)
  for (uint32_t i = lane; i < pg.def_len; i += 32) out[i] = p[pg.def_off + i];
  out += pg.def_len;
  const uint32_t* plen = reinterpret_cast<const uint32_t*>(scratch + job.len_tmp);
  const uint32_t* slen = plen + pg.num_rows;
  const uint8_t* src = p + in.data_pos;    // suffixes, back to back
  uint64_t o_base = 0, s_base = 0;         // bytes written / suffix bytes consumed before this group of 32 values
  uint64_t prev = 0;                       // where the previous value's bytes start in `out`
  for (uint32_t i0 = 0; i0 < in.nvals; i0 += 32) {
    const uint32_t i = i0 + lane;
    const uint32_t pl = (i < in.nvals && job.with_prefix) ? plen[i] : 0u, sl = i < in.nvals ? slen[i] : 0u;
    // exclusive scans: every value's place in the output and in the suffix bytes is known without the chain
    uint64_t o_inc = i < in.nvals ? uint64_t(pl) + sl + 4 : 0ull, s_inc = sl;
    for (int o = 1; o < 32; o <<= 1) {
      const uint64_t a = __shfl_up_sync(0xffffffffu, o_inc, o), b = __shfl_up_sync(0xffffffffu, s_inc, o);
      if ((int)lane >= o) { o_inc += a; s_inc += b; }
    }
    const uint64_t my_o = o_base + o_inc - (i < in.nvals ? uint64_t(pl) + sl + 4 : 0ull), my_s = s_base + s_inc - sl;
    if (i < in.nvals) {   // the length word and the suffix do not depend on the chain
      const uint32_t len = pl + sl;
      uint8_t* w = out + my_o;
      w[0] = uint8_t(len); w[1] = uint8_t(len >> 8); w[2] = uint8_t(len >> 16); w[3] = uint8_t(len >> 24);
    }
    const uint32_t cnt = in.nvals - i0 < 32 ? in.nvals - i0 : 32;
    for (uint32_t k = 0; k < cnt; k++) {
      const uint32_t kp = __shfl_sync(0xffffffffu, pl, k), ks = __shfl_sync(0xffffffffu, sl, k);
      const uint64_t ko = __shfl_sync(0xffffffffu, my_o, k) + 4, ksrc = __shfl_sync(0xffffffffu, my_s, k);
      for (uint32_t b = lane; b < ks; b += 32) out[ko + kp + b] = src[ksrc + b];
      if (kp) {
        __syncwarp();   // the previous value is complete (its prefix part was written one trip ago)
        for (uint32_t b = lane; b < kp; b += 32) out[ko + b] = out[prev + b];
      }
      prev = ko;
      __syncwarp();
    }
    o_base += __shfl_sync(0xffffffffu, o_inc, 31);
    s_base += __shfl_sync(0xffffffffu, s_inc, 31);
  }
}

}  // namespace pqb
