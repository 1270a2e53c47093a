// Dictionary-side kernels that run before the fused scan:
//   * string dictionary entry offsets (PLAIN BYTE_ARRAY = 4-byte length + bytes),
//   * leaf predicates evaluated once per DICTIONARY ENTRY into byte LUTs, so the
//     scan tests one byte per row instead of comparing strings / floats,
//   * GROUP BY key unification: every per-chunk dictionary entry is hashed into a
//     global open-addressing table; its dense group id lands in a per-entry LUT.
// This is where arrow-ord / arrow-string comparison kernels and DataFusion's
// GroupValues interning (SURVEY.md §8 rows a11, a12) are restated for the GPU.
#pragma once
#include <cuda_runtime.h>

#include "decode_core.cuh"
#include "device_structs.hpp"
#include "in_set.cuh"
#include "regex_match.cuh"

namespace pqb {

struct DevPrepArgs {
  const uint8_t* arena;
  const DevChunk* chunks;        // [table row group * ncols + slot]
  uint32_t n_chunks;             // row groups * ncols
  uint32_t ncols;
  const uint8_t* rg_live;        // per row group: 0 = pruned for this query (nullptr: all live)
  const uint64_t* ent[kMaxCols]; // per slot: arena offset of every dictionary entry of the column (string leaves only)
  uint8_t* luts;
  const uint8_t* lit_pool;
  unsigned long long* counters;  // [1] error flag
};

// one column chunk as the table-level side-table builders see it
struct EntChunk { uint64_t dict_off; uint32_t dict_len; uint32_t dict_n; uint32_t base; uint32_t present; };

// Arena offset of every dictionary entry of ONE column (all row groups): query independent, built on
// first use and kept with the table.
// One WARP per column chunk.  A PLAIN byte-array dictionary is a chain (each length prefix says where
// the next entry starts), so the walk is serial — but not at HBM/L2 latency: the warp stages the
// dictionary through shared memory in 4 KiB tiles (coalesced 16-byte loads) and lane 0 follows the
// chain there (tens of cycles per entry instead of ~600).
constexpr int kEntTile = 4096;
__global__ void __launch_bounds__(128) k_dict_entry_offsets(const uint8_t* __restrict__ arena, const EntChunk* __restrict__ chunks,
                                                            uint32_t n_chunks, uint32_t kind, uint64_t* __restrict__ ent_off,
                                                            unsigned int* __restrict__ err) {
  __shared__ __align__(16) uint8_t tiles[4][kEntTile + 16];
  const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const uint32_t ci = blockIdx.x * 4 + warp;
  if (ci >= n_chunks) return;
  const EntChunk ch = chunks[ci];
  if (!ch.present || ch.dict_n == 0) return;
  uint64_t* out = ent_off + ch.base;
  if (kind != DK_STR) {
    for (uint32_t i = lane; i < ch.dict_n; i += 32) out[i] = ch.dict_off + uint64_t(i) * 8;
    return;
  }
  uint8_t* tile = tiles[warp];
  const uint64_t end = ch.dict_off + ch.dict_len;
  uint64_t p = ch.dict_off;
  uint32_t i = 0, maxlen = 0;
  bool bad = false;
  while (i < ch.dict_n && !bad) {
    // stage [t0, t0 + kEntTile) with t0 = p rounded down to 16 (the arena is padded past every chunk)
    const uint64_t t0 = p & ~15ull;
    for (uint32_t o = lane * 16; o < (uint32_t)kEntTile; o += 32 * 16)
      *reinterpret_cast<uint4*>(tile + o) = *reinterpret_cast<const uint4*>(arena + t0 + o);
    __syncwarp();
    if (lane == 0) {
      while (i < ch.dict_n) {
        if (p + 4 > end) { bad = true; break; }
        const uint32_t rel = uint32_t(p - t0);
        if (rel + 4 > (uint32_t)kEntTile) break;   // next length prefix is outside this tile
        const uint32_t len = uint32_t(tile[rel]) | (uint32_t(tile[rel + 1]) << 8) | (uint32_t(tile[rel + 2]) << 16) |
                             (uint32_t(tile[rel + 3]) << 24);
        if (p + 4 + uint64_t(len) > end) { bad = true; break; }
        if (len > maxlen) maxlen = len;
        out[i++] = p + 4;
        p += 4 + uint64_t(len);
      }
    }
    i = __shfl_sync(0xffffffffu, i, 0);
    p = __shfl_sync(0xffffffffu, p, 0);
    bad = __shfl_sync(0xffffffffu, bad ? 1 : 0, 0) != 0;
    __syncwarp();
  }
  if (lane == 0 && maxlen) atomicMax(err + 1, maxlen);   // longest entry of the column (sizes projected string buffers)
  if (bad) {
    // a corrupt dictionary: the remaining entries read as empty strings at the dictionary start (never
    // out of bounds); the query that asked for this table fails with PQ_ERR_CORRUPT
    for (uint32_t k = i + lane; k < ch.dict_n; k += 32) out[k] = ch.dict_off + 4;
    if (lane == 0) atomicExch(err, 3u);
  }
}

__device__ __forceinline__ uint32_t entry_len(const uint8_t* arena, uint64_t off, uint8_t kind) {
  return kind == DK_STR ? load_u32_unaligned(arena + off - 4) : 8u;
}

// grid.x = chunk (row group x slot), grid.y = blocks over entries
__global__ void k_leaf_luts(DevPrepArgs a, const __grid_constant__ DevPlan plan) {
  uint32_t ci = blockIdx.x;
  const DevChunk ch = a.chunks[ci];
  uint32_t col = ci % a.ncols;
  if (!ch.present || ch.dict_n == 0) return;
  if (a.rg_live && !a.rg_live[ci / a.ncols]) return;
  const uint8_t kind = plan.cols[col].kind;
  for (uint32_t e = blockIdx.y * blockDim.x + threadIdx.x; e < ch.dict_n; e += gridDim.y * blockDim.x) {
    for (uint32_t l = 0; l < plan.nleaves; l++) {
      const DevLeaf& lf = plan.leaves[l];
      if (lf.col != col || !value_leaf(lf.kind)) continue;
      bool t;
      if (kind == DK_STR) {
        uint64_t off = a.ent[col][ch.lut_base + e];
        uint32_t len = load_u32_unaligned(a.arena + off - 4);
        const uint8_t* s = a.arena + off;
        const uint8_t* lit = a.lit_pool + lf.str_off;
        if (lf.kind == LK_CMP) t = cmp_result(cmp_bytes(s, len, lit, lf.str_len), lf.cmp);
        else if (lf.kind == LK_REGEX) t = regex_match(s, len, lit) != ((lf.flags & 1u) != 0);   // once per dictionary entry
        else if (lf.kind == LK_IN) t = in_set_has_bytes(lit, s, len);
        else {
          t = like_match(s, len, lit, lf.str_len, lf.cmp, (lf.flags & 2u) != 0);
          if (lf.flags & 1u) t = !t;
        }
      } else if (lf.kind == LK_IN) {   // Int64 / Float64: the entry's 8 bytes (Float64: its bits) in the set
        t = in_set_has_u64(a.lit_pool + lf.str_off, load_u64_unaligned(a.arena + ch.dict_off + uint64_t(e) * 8));
      } else if (kind == DK_I64) {
        t = cmp_i64((int64_t)load_u64_unaligned(a.arena + ch.dict_off + uint64_t(e) * 8), lf.lit_i64, lf.cmp);
      } else if (kind == DK_F64) {
        t = cmp_i64(f64_order_key(load_u64_unaligned(a.arena + ch.dict_off + uint64_t(e) * 8)),
                    f64_order_key((uint64_t)lf.lit_i64), lf.cmp);
      } else {
        t = false;
      }
      a.luts[lf.lut_off + ch.lut_base + e] = t ? 1 : 0;
    }
  }
}

// ---- GROUP BY key interning (per table column, query independent) ----
// "Entries" of a key column: the dictionary entries of every row group, then -- for columns with pages that have no
// dictionary (PLAIN fallback of an overflowed dictionary, PLAIN / DELTA numerics) -- every ROW of those pages.  An entry
// is where its value's bytes sit relative to the arena (a row's 8-byte slot of the flat store lies outside the arena:
// the offset wraps, arena + offset does not); ~0 marks a NULL row / padding.
struct EntView {
  const uint64_t* dict;   // [0, n_dict): dictionary entries
  const uint64_t* rows;   // [n_dict, ...): rows of the column's non-dictionary pages
  uint32_t n_dict;
};
__device__ __forceinline__ uint64_t ent_at(const EntView& v, uint32_t ge) { return ge < v.n_dict ? v.dict[ge] : v.rows[ge - v.n_dict]; }
constexpr uint64_t kNoEntry = ~0ull;

struct DevKeyTable {
  unsigned long long* slots;  // 0 empty, else (hash32 << 32) | (column entry index + 1)
  uint32_t* gid_of_slot;
  uint32_t* rep_of_gid;       // representative column entry index per group id
  uint32_t* counter;          // [0] distinct count, [1] overflow flag
  uint32_t cap_mask;
  uint32_t kind;              // DevKind
  EntView ent;                // entry offsets of the column
  uint32_t* gid;              // out: group id per column entry
};

__device__ __forceinline__ bool entry_equal(const uint8_t* arena, uint64_t oa, uint64_t ob, uint32_t len, uint8_t kind) {
  if (kind != DK_STR) return load_u64_unaligned(arena + oa) == load_u64_unaligned(arena + ob);
  if (load_u32_unaligned(arena + ob - 4) != len) return false;
  for (uint32_t i = 0; i < len; i++)
    if (arena[oa + i] != arena[ob + i]) return false;
  return true;
}

// mode 0: insert + number; mode 1: lookup -> gid[]
__device__ __forceinline__ void intern_entry(const uint8_t* __restrict__ arena, const DevKeyTable& t, uint32_t ge, int mode) {
  const uint64_t off = ent_at(t.ent, ge);
  if (off == kNoEntry) return;
  uint32_t len = entry_len(arena, off, (uint8_t)t.kind);
  uint64_t h = t.kind == DK_STR ? hash_bytes(arena + off, len) : mix64(load_u64_unaligned(arena + off));
  uint32_t h32 = uint32_t(h >> 32);
  unsigned long long word = ((unsigned long long)h32 << 32) | (unsigned long long)(ge + 1);
  uint32_t slot = uint32_t(h) & t.cap_mask;
  uint32_t probes = 0;
  for (;;) {
    unsigned long long cur = t.slots[slot];
    if (cur == 0 && mode == 0) {
      unsigned long long prev = atomicCAS(&t.slots[slot], 0ull, word);
      if (prev == 0) {
        uint32_t gid = atomicAdd(&t.counter[0], 1u);
        t.gid_of_slot[slot] = gid;
        t.rep_of_gid[gid] = ge;
        break;
      }
      cur = prev;
    }
    if (cur == 0) { atomicExch(&t.counter[1], 2u); break; }  // lookup miss: cannot happen
    if (uint32_t(cur >> 32) == h32) {
      uint32_t other = uint32_t(cur & 0xffffffffull) - 1;
      if (other == ge || entry_equal(arena, off, ent_at(t.ent, other), len, (uint8_t)t.kind)) {
        if (mode == 1) t.gid[ge] = t.gid_of_slot[slot];
        break;
      }
    }
    slot = (slot + 1) & t.cap_mask;
    if (++probes > t.cap_mask) { atomicExch(&t.counter[1], 1u); break; }
  }
}

// dictionary entries.  grid.x = column chunks in [c0, c0 + gridDim.x)
__global__ void k_key_intern(const uint8_t* __restrict__ arena, const EntChunk* __restrict__ chunks, uint32_t c0, DevKeyTable t, int mode) {
  const EntChunk ch = chunks[c0 + blockIdx.x];
  if (!ch.present || ch.dict_n == 0) return;
  for (uint32_t e = blockIdx.y * blockDim.x + threadIdx.x; e < ch.dict_n; e += gridDim.y * blockDim.x) intern_entry(arena, t, ch.base + e, mode);
}

// rows of the column's non-dictionary pages: where every row's value sits (k_row_entries), then the same interning
struct RowPage {
  uint64_t off;      // flat-store offset of the page's slots (FK_PLAIN8: 8 bytes per row; FK_BYTES: u32 per row, relative to `base`)
  uint64_t voff;     // validity bits, ~0: no NULLs
  uint64_t base;     // FK_BYTES: arena offset of the page's values section
  uint32_t rows;
  uint32_t ebase;    // first entry of the page inside EntView.rows (a multiple of 4: the id page is a TMA source)
  uint32_t fkind;
  uint32_t _pad;
};
__global__ void k_row_entries(const uint8_t* __restrict__ flat, const RowPage* __restrict__ rp, uint32_t n_pages, uint64_t flat_minus_arena,
                              uint64_t* __restrict__ out) {
  for (uint32_t p = blockIdx.x; p < n_pages; p += gridDim.x) {
    const RowPage pg = rp[p];
    const uint32_t* vw = pg.voff == ~0ull ? nullptr : reinterpret_cast<const uint32_t*>(flat + pg.voff);
    for (uint32_t r = threadIdx.x; r < pg.rows; r += blockDim.x) {
      const bool valid = !vw || ((vw[r >> 5] >> (r & 31)) & 1u);
      uint64_t e = kNoEntry;
      if (valid) e = pg.fkind == FK_PLAIN8 ? flat_minus_arena + pg.off + uint64_t(r) * 8 : pg.base + reinterpret_cast<const uint32_t*>(flat + pg.off)[r];
      out[pg.ebase + r] = e;
    }
  }
}
__global__ void k_row_intern(const uint8_t* __restrict__ arena, const RowPage* __restrict__ rp, uint32_t n_pages, DevKeyTable t, int mode) {
  for (uint32_t p = blockIdx.x; p < n_pages; p += gridDim.x) {
    const uint32_t rows = rp[p].rows, e0 = t.ent.n_dict + rp[p].ebase;
    for (uint32_t r = threadIdx.x; r < rows; r += blockDim.x) intern_entry(arena, t, e0 + r, mode);
  }
}

// renumber group ids: gid[e] = remap[gid[e]] for every entry of the column
__global__ void k_gid_remap(const uint32_t* __restrict__ gid_in, uint32_t* __restrict__ gid_out, uint32_t n_entries,
                            const uint32_t* __restrict__ remap, uint32_t card) {
  for (uint32_t e = blockIdx.x * blockDim.x + threadIdx.x; e < n_entries; e += gridDim.x * blockDim.x) {
    const uint32_t g = gid_in[e];
    gid_out[e] = g < card ? remap[g] : g;
  }
}

// MIN / MAX over Utf8, per group id g < card: ids[g] = rank[g] (64-bit), inv[rank[g]] = g (the group id of every rank)
__global__ void k_rank_ids(const uint32_t* __restrict__ rank, uint32_t card, uint64_t* __restrict__ ids, uint32_t* __restrict__ inv) {
  for (uint32_t g = blockIdx.x * blockDim.x + threadIdx.x; g < card; g += gridDim.x * blockDim.x) {
    ids[g] = rank[g];
    inv[rank[g]] = g;
  }
}
// ... and per dictionary entry: ent[e] = rank[gid[e]]
__global__ void k_rank_compose(const uint32_t* __restrict__ gid, uint32_t n_entries, const uint32_t* __restrict__ rank, uint32_t card,
                               uint64_t* __restrict__ ent) {
  for (uint32_t e = blockIdx.x * blockDim.x + threadIdx.x; e < n_entries; e += gridDim.x * blockDim.x) {
    const uint32_t g = gid[e];
    ent[e] = g < card ? rank[g] : 0u;
  }
}

// Occurrences of every group id over a sample of the key column's flat pages: the hot-first
// numbering of group ids (the flat aggregate kernel keeps slots < hot_slots in shared memory).
struct KeySamplePage { uint64_t off; uint32_t rows; uint32_t bw; uint32_t base; uint32_t dict_n; };
__global__ void k_key_sample(const uint8_t* __restrict__ flat, const KeySamplePage* __restrict__ sp, uint32_t n_pages,
                             const uint32_t* __restrict__ gid, uint32_t* __restrict__ counts) {
  const KeySamplePage p = sp[blockIdx.x];
  const uint32_t* w = reinterpret_cast<const uint32_t*>(flat + p.off);
  const uint32_t mask = p.bw >= 32 ? 0xffffffffu : ((1u << p.bw) - 1u);
  for (uint32_t r = threadIdx.x; r < p.rows; r += blockDim.x) {
    uint32_t v = 0;
    if (p.bw) {
      const uint32_t bit = r * p.bw, i = bit >> 5, sh = bit & 31;
      v = __funnelshift_r(w[i], w[i + 1], sh) & mask;
    }
    if (v >= p.dict_n) continue;
    atomicAdd(&counts[gid[p.base + v]], 1u);
  }
}

// accumulator table initialisation: rows / sums / nn = 0, MIN = INT64_MAX, MAX = INT64_MIN
__global__ void k_acc_init(unsigned long long* acc, uint32_t nslots, uint32_t n_acc, uint32_t cells, uint32_t replicas,
                           const __grid_constant__ DevPlan plan) {
  uint64_t n = uint64_t(nslots) * cells * replicas;
  for (uint64_t i = blockIdx.x * uint64_t(blockDim.x) + threadIdx.x; i < n; i += uint64_t(gridDim.x) * blockDim.x) {
    uint32_t arr = uint32_t((i / nslots) % cells);
    unsigned long long init = 0;
    if (arr >= 1 && arr < 1 + n_acc) {
      uint8_t k = plan.acc_init[arr - 1];
      init = k == 2 ? 0x7fffffffffffffffull : (k == 3 ? 0x8000000000000000ull : 0ull);
    }
    acc[i] = init;
  }
}

// compact non-empty groups: out_slot[n], out_cells[cell][n]
__global__ void k_agg_compact(const unsigned long long* acc, uint32_t nslots, uint32_t cells, uint32_t* out_count,
                              uint32_t* out_slot, unsigned long long* out_cells, uint32_t out_cap) {
  for (uint32_t s = blockIdx.x * blockDim.x + threadIdx.x; s < nslots; s += gridDim.x * blockDim.x) {
    if (acc[s] == 0) continue;
    uint32_t o = atomicAdd(out_count, 1u);
    if (o >= out_cap) continue;
    out_slot[o] = s;
    for (uint32_t c = 0; c < cells; c++) out_cells[uint64_t(c) * out_cap + o] = acc[uint64_t(c) * nslots + s];
  }
}

// ---- bitmap-driven stream compaction (arrow-select `filter` in the reference, SURVEY §8 a11) ----
// exclusive prefix of the per-item selected-row counts; one block
__global__ void k_item_prefix(const uint32_t* __restrict__ counts, uint32_t n, unsigned long long* __restrict__ base,
                              unsigned long long* __restrict__ total) {
  __shared__ unsigned long long warp_sums[32];
  __shared__ unsigned long long carry;
  if (threadIdx.x == 0) carry = 0;
  __syncthreads();
  const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = blockDim.x >> 5;
  for (uint32_t i0 = 0; i0 < n; i0 += blockDim.x) {
    uint32_t i = i0 + threadIdx.x;
    unsigned long long v = i < n ? counts[i] : 0, incl = v;
    for (int o = 1; o < 32; o <<= 1) {
      unsigned long long t = __shfl_up_sync(0xffffffffu, incl, o);
      if ((int)lane >= o) incl += t;
    }
    if (lane == 31) warp_sums[warp] = incl;
    __syncthreads();
    if (warp == 0) {
      unsigned long long w = lane < nwarps ? warp_sums[lane] : 0, wi = w;
      for (int o = 1; o < 32; o <<= 1) {
        unsigned long long t = __shfl_up_sync(0xffffffffu, wi, o);
        if ((int)lane >= o) wi += t;
      }
      warp_sums[lane] = wi - w;  // exclusive
    }
    __syncthreads();
    unsigned long long excl = carry + warp_sums[warp] + incl - v;
    if (i < n) base[i] = excl;
    __syncthreads();
    if (threadIdx.x == blockDim.x - 1) carry = excl + v;
    __syncthreads();
  }
  if (threadIdx.x == 0) *total = carry;
}

// one CTA per item (grid-strided): selection bitmap -> ascending global row ordinals
__global__ void k_compact_row_ids(const uint32_t* __restrict__ bitmap, const DevItem* __restrict__ items,
                                  const uint32_t* __restrict__ item_counts, const unsigned long long* __restrict__ base,
                                  uint32_t n_items, unsigned long long* __restrict__ out, unsigned long long out_cap) {
  __shared__ uint32_t warp_sums[32];
  __shared__ uint32_t carry;
  const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = blockDim.x >> 5;
  for (uint32_t it = blockIdx.x; it < n_items; it += gridDim.x) {
    if (item_counts[it] == 0) continue;  // uniform per block
    const DevItem item = items[it];
    const uint32_t nwords = (item.nrows + 31) >> 5;
    if (threadIdx.x == 0) carry = 0;
    __syncthreads();
    for (uint32_t w0 = 0; w0 < nwords; w0 += blockDim.x) {
      uint32_t w = w0 + threadIdx.x;
      uint32_t word = w < nwords ? bitmap[item.bitmap_word0 + w] : 0;
      uint32_t c = __popc(word), incl = c;
      for (int o = 1; o < 32; o <<= 1) {
        uint32_t t = __shfl_up_sync(0xffffffffu, incl, o);
        if ((int)lane >= o) incl += t;
      }
      if (lane == 31) warp_sums[warp] = incl;
      __syncthreads();
      if (warp == 0) {
        uint32_t s = lane < nwarps ? warp_sums[lane] : 0, si = s;
        for (int o = 1; o < 32; o <<= 1) {
          uint32_t t = __shfl_up_sync(0xffffffffu, si, o);
          if ((int)lane >= o) si += t;
        }
        warp_sums[lane] = si - s;
      }
      __syncthreads();
      unsigned long long pos = base[it] + carry + warp_sums[warp] + incl - c;
      unsigned long long row = item.global_row0 + uint64_t(w) * 32;
      while (word) {
        int b = __ffs(word) - 1;
        word &= word - 1;
        if (pos < out_cap) out[pos] = row + b;
        pos++;
      }
      __syncthreads();
      if (threadIdx.x == blockDim.x - 1) carry += warp_sums[warp] + incl;
      __syncthreads();
    }
  }
}

// key value export: lengths, then bytes at host-computed offsets
__global__ void k_key_lens(const uint8_t* arena, EntView ent, const uint32_t* rep_of_gid, uint32_t card,
                           uint8_t kind, uint32_t* lens) {
  uint32_t g = blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= card) return;
  lens[g] = entry_len(arena, ent_at(ent, rep_of_gid[g]), kind);
}
__global__ void k_key_bytes(const uint8_t* arena, EntView ent, const uint32_t* rep_of_gid, uint32_t card,
                            uint8_t kind, const uint32_t* offsets, uint8_t* out) {
  uint32_t g = blockIdx.x;
  if (g >= card) return;
  uint64_t off = ent_at(ent, rep_of_gid[g]);
  uint32_t len = entry_len(arena, off, kind);
  for (uint32_t i = threadIdx.x; i < len; i += blockDim.x) out[offsets[g] + i] = arena[off + i];
}

}  // namespace pqb
