// Result assembly on the device: the accumulator table of an aggregate query becomes the buffers of
// its Arrow result batches (values, validity bitmaps, string offsets + bytes of the group keys) in
// ONE device block that is copied to page-locked host memory once; the batches alias that block.
// Replaces, for the reference, AggregateExec(Final)'s output + the RecordBatch construction
// (DataFusion; results are what Query::execute returns, /root/reference/src/query/mod.rs:287-291).
#pragma once
#include <cuda_runtime.h>

#include "decode_core.cuh"
#include "device_structs.hpp"

namespace pqb {

constexpr int kSlotTile = 1024;

// The slot at list position p: order[p] (a permutation of the slots), or p itself when order is nullptr
__device__ __forceinline__ uint32_t slot_at(const uint32_t* __restrict__ order, uint32_t p) { return order ? order[p] : p; }

// non-empty groups per tile of kSlotTile list positions
__global__ void k_slot_tile_counts(const unsigned long long* __restrict__ rows, uint32_t nslots, uint32_t* __restrict__ tile_counts,
                                   const uint32_t* __restrict__ order) {
  __shared__ uint32_t ws[8];
  const uint32_t s0 = blockIdx.x * kSlotTile;
  uint32_t c = 0;
  for (uint32_t i = threadIdx.x; i < (uint32_t)kSlotTile; i += blockDim.x) c += (s0 + i < nslots && rows[slot_at(order, s0 + i)] != 0) ? 1u : 0u;
  c = __reduce_add_sync(0xffffffffu, c);
  if ((threadIdx.x & 31) == 0) ws[threadIdx.x >> 5] = c;
  __syncthreads();
  if (threadIdx.x == 0) {
    uint32_t t = 0;
    for (uint32_t w = 0; w < blockDim.x / 32; w++) t += ws[w];
    tile_counts[blockIdx.x] = t;
  }
}

// list order (ascending slot, or order[]): out_slot[base[tile] + rank inside the tile]; 256 threads x 4 consecutive positions
__global__ void __launch_bounds__(256) k_slot_compact(const unsigned long long* __restrict__ rows, uint32_t nslots,
                                                      const unsigned long long* __restrict__ tile_base, uint32_t* __restrict__ out_slot,
                                                      const uint32_t* __restrict__ order) {
  __shared__ uint32_t ws[8];
  const uint32_t s0 = blockIdx.x * kSlotTile + threadIdx.x * 4;
  uint32_t f[4], c = 0;
#pragma unroll
  for (int k = 0; k < 4; k++) { f[k] = (s0 + k < nslots && rows[slot_at(order, s0 + k)] != 0) ? 1u : 0u; c += f[k]; }
  uint32_t incl = c;
  const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (int o = 1; o < 32; o <<= 1) {
    const uint32_t t = __shfl_up_sync(0xffffffffu, incl, o);
    if ((int)lane >= o) incl += t;
  }
  if (lane == 31) ws[warp] = incl;
  __syncthreads();
  uint32_t wbase = 0;
  for (uint32_t w = 0; w < warp; w++) wbase += ws[w];
  unsigned long long pos = tile_base[blockIdx.x] + wbase + incl - c;
#pragma unroll
  for (int k = 0; k < 4; k++)
    if (f[k]) out_slot[pos++] = slot_at(order, s0 + k);
}

struct FinishKey {
  const uint32_t* kd_offs;     // key dictionary: offsets (group-id order)
  const uint8_t* kd_bytes;
  uint64_t val_off;            // 8-byte values | bit-packed booleans (per batch words) | int32 string offsets (n_out + 1)
  uint64_t valid_off;          // validity words, per batch
  uint64_t len_off;            // strings: u32 length per row (scratch, device only)
  uint64_t data_off;           // strings: bytes
  uint32_t stride, card;
  uint64_t wstride;            // stride in 64 bits (hashed group-by decodes the wide id)
  uint32_t kind;               // DevKind (DK_I32: a Date32 key, 4-byte values)
  uint32_t is_bin;             // DATE_BIN key: value = bin_base + group id * bin_width
  int64_t bin_base, bin_width;
};
// MIN / MAX over Utf8: the cell holds the winning rank; inv maps it to its group id in the numbering whose dictionary
// (kd_offs / kd_bytes) holds the bytes
struct FinishAggStr {
  const uint32_t* kd_offs;
  const uint8_t* kd_bytes;
  const uint32_t* inv;         // rank -> group id
  uint64_t len_off;            // u32 length per row (scratch, device only)
  uint64_t data_off;           // bytes
};
struct FinishArgs {
  const unsigned long long* acc;
  const unsigned long long* wide;   // hashed group-by: wide group id per slot (nullptr: the slot is the id)
  const uint32_t* out_slot;
  uint8_t* out;                // the result block
  uint32_t* nulls;             // [(nkeys + naggs) * nbatches] inside the block
  // n_dev == nullptr: n_out groups.  Otherwise the block was laid out before the group count came back to the host:
  // n_out is its capacity and the kernels read the count (min(*n_dev, n_out) groups) where k_item_prefix left it
  const unsigned long long* n_dev;
  uint32_t n_out, nslots, n_acc, naggs, nkeys;
  uint32_t batch_rows, words_per_batch, nbatches;
  DevAgg aggs[kMaxAggs];
  uint8_t nn_is_rows[kMaxAggs];
  // the output layout of each aggregate: DK_STR (MIN / MAX over Utf8: int32 offsets at val_off, bytes at astr.data_off),
  // DK_BOOL (MIN / MAX over Boolean: bit-packed values per batch at val_off), anything else 8-byte values
  uint8_t out_kind[kMaxAggs];   // (DK_I32: MIN / MAX over Date32, 4-byte values)
  uint64_t val_off[kMaxAggs], valid_off[kMaxAggs];
  FinishAggStr astr[kMaxAggs];
  FinishKey keys[kMaxKeys];
};

// The output value of one aggregate of one group slot: the bits of its Int64 / Float64 result, valid == false for NULL.
// k_agg_finish writes it and k_order_encode sorts by it, so an ORDER BY on an aggregate and its output cannot disagree.
__device__ __forceinline__ unsigned long long agg_output_value(const unsigned long long* __restrict__ acc, uint32_t nslots, uint32_t n_acc,
                                                               const DevAgg ag, uint8_t nn_is_rows, uint32_t slot,
                                                               unsigned long long rows, bool& valid) {
  unsigned long long nn = 0, cell = 0;
  if (ag.fn != AG_COUNT_STAR) nn = nn_is_rows ? rows : acc[size_t(1 + n_acc + ag.nn_slot) * nslots + slot];
  if (ag.fn >= AG_SUM) cell = acc[size_t(1 + ag.acc_slot) * nslots + slot];
  valid = true;
  unsigned long long v = 0;
  switch (ag.fn) {
    case AG_COUNT_STAR: v = rows; break;
    case AG_COUNT: v = nn; break;
    case AG_COUNT_DISTINCT: v = cell; break;   // first sightings of the group's values: 0 when every input was NULL
    case AG_SUM:
    case AG_MEDIAN:             // MEDIAN / PERCENTILE_CONT: the output bits k_pct_pick wrote
    case AG_PERCENTILE_CONT: valid = nn > 0; v = cell; break;
    case AG_AVG:
      valid = nn > 0;
      if (valid) v = (unsigned long long)__double_as_longlong(__longlong_as_double((long long)cell) / double(nn));
      break;
    default:
      valid = nn > 0;
      v = ag.kind == DK_F64 ? f64_from_order_key((int64_t)cell) : cell;
  }
  return v;
}

__device__ __forceinline__ uint32_t finish_rows(const FinishArgs& f) {
  return f.n_dev ? uint32_t(min(*f.n_dev, (unsigned long long)f.n_out)) : f.n_out;
}

// the group id of one GROUP BY key of a group slot (hashed GROUP BY: decoded from the slot's wide id); card: NULL
__device__ __forceinline__ uint32_t key_gid_of_slot(const unsigned long long* __restrict__ wide, uint32_t slot, uint64_t wstride, uint32_t card) {
  return uint32_t(((wide ? wide[slot] : uint64_t(slot)) / wstride) % (card + 1));
}

// one thread per output row: aggregate values + validity, numeric / boolean key values, string key lengths
__global__ void k_agg_finish(const __grid_constant__ FinishArgs f) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= finish_rows(f)) return;
  const uint32_t slot = f.out_slot[i];
  const uint32_t batch = i / f.batch_rows, pos = i - batch * f.batch_rows;
  const uint32_t word = batch * f.words_per_batch + (pos >> 5), bit = 1u << (pos & 31);
  const unsigned long long rows = f.acc[slot];
  for (uint32_t a = 0; a < f.naggs; a++) {
    bool valid;
    const unsigned long long v = agg_output_value(f.acc, f.nslots, f.n_acc, f.aggs[a], f.nn_is_rows[a], slot, rows, valid);
    if (f.out_kind[a] == DK_STR) {   // the winning rank's length; k_agg_str_gather copies its bytes
      const FinishAggStr& s = f.astr[a];
      const uint32_t g = valid ? s.inv[v] : 0u;
      reinterpret_cast<uint32_t*>(f.out + s.len_off)[i] = valid ? s.kd_offs[g + 1] - s.kd_offs[g] : 0u;
    } else if (f.out_kind[a] == DK_BOOL) {
      if (valid && v) atomicOr(reinterpret_cast<uint32_t*>(f.out + f.val_off[a]) + word, bit);
    } else if (f.out_kind[a] == DK_I32) {   // MIN / MAX over Date32: the low word of the sign-extended cell
      reinterpret_cast<uint32_t*>(f.out + f.val_off[a])[i] = valid ? uint32_t(v) : 0u;
    } else {
      reinterpret_cast<unsigned long long*>(f.out + f.val_off[a])[i] = valid ? v : 0ull;
    }
    if (valid) atomicOr(reinterpret_cast<uint32_t*>(f.out + f.valid_off[a]) + word, bit);
    else atomicAdd(&f.nulls[(f.nkeys + a) * f.nbatches + batch], 1u);
  }
  for (uint32_t k = 0; k < f.nkeys; k++) {
    const FinishKey& key = f.keys[k];
    const uint32_t gid = key_gid_of_slot(f.wide, slot, key.wstride, key.card);
    const bool valid = gid != key.card;   // NULL is its own group (field_stats.rs:1009-1037)
    if (valid) atomicOr(reinterpret_cast<uint32_t*>(f.out + key.valid_off) + word, bit);
    else atomicAdd(&f.nulls[k * f.nbatches + batch], 1u);
    if (key.kind == DK_STR) {
      reinterpret_cast<uint32_t*>(f.out + key.len_off)[i] = valid ? key.kd_offs[gid + 1] - key.kd_offs[gid] : 0u;
    } else if (key.kind == DK_BOOL) {
      if (valid && gid) atomicOr(reinterpret_cast<uint32_t*>(f.out + key.val_off) + word, bit);
    } else {
      unsigned long long v = 0;
      if (valid && key.is_bin) v = (unsigned long long)(key.bin_base + (long long)gid * key.bin_width);
      else if (valid) {
        const uint8_t* p = key.kd_bytes + key.kd_offs[gid];
        for (int b = 0; b < 8; b++) v |= (unsigned long long)p[b] << (8 * b);
      }
      if (key.kind == DK_I32) reinterpret_cast<uint32_t*>(f.out + key.val_off)[i] = uint32_t(v);   // Date32
      else reinterpret_cast<unsigned long long*>(f.out + key.val_off)[i] = v;
    }
  }
}

// exclusive scan of u32 lengths into int32 Arrow offsets (n + 1 entries); one block.  n_dev != nullptr: min(*n_dev, n)
// lengths (a result block laid out for n groups before the count was known)
__global__ void k_offsets_scan(const uint32_t* __restrict__ lens, uint32_t n, const unsigned long long* __restrict__ n_dev,
                               int32_t* __restrict__ offs) {
  if (n_dev) n = uint32_t(min(*n_dev, (unsigned long long)n));
  __shared__ unsigned long long warp_sums[32];
  __shared__ unsigned long long carry;
  if (threadIdx.x == 0) carry = 0;
  __syncthreads();
  const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = blockDim.x >> 5;
  for (uint32_t i0 = 0; i0 < n; i0 += blockDim.x) {
    const uint32_t i = i0 + threadIdx.x;
    unsigned long long v = i < n ? lens[i] : 0, incl = v;
    for (int o = 1; o < 32; o <<= 1) {
      const unsigned long long t = __shfl_up_sync(0xffffffffu, incl, o);
      if ((int)lane >= o) incl += t;
    }
    if (lane == 31) warp_sums[warp] = incl;
    __syncthreads();
    if (warp == 0) {
      unsigned long long w = lane < nwarps ? warp_sums[lane] : 0, wi = w;
      for (int o = 1; o < 32; o <<= 1) {
        const unsigned long long t = __shfl_up_sync(0xffffffffu, wi, o);
        if ((int)lane >= o) wi += t;
      }
      warp_sums[lane] = wi - w;
    }
    __syncthreads();
    const unsigned long long excl = carry + warp_sums[warp] + incl - v;
    if (i < n) offs[i] = int32_t(excl);
    __syncthreads();
    if (threadIdx.x == blockDim.x - 1) carry = excl + v;
    __syncthreads();
  }
  if (threadIdx.x == 0) offs[n] = int32_t(carry);
}

// the exact string bytes of key k over the output rows (for a result whose count-free bound is too large to allocate)
__global__ void k_key_bytes_total(const __grid_constant__ FinishArgs f, uint32_t k, unsigned long long* __restrict__ total) {
  const FinishKey& key = f.keys[k];
  unsigned long long s = 0;
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < finish_rows(f); i += gridDim.x * blockDim.x) {
    const uint32_t gid = key_gid_of_slot(f.wide, f.out_slot[i], key.wstride, key.card);
    if (gid != key.card) s += key.kd_offs[gid + 1] - key.kd_offs[gid];
  }
  for (int o = 16; o; o >>= 1) s += __shfl_down_sync(0xffffffffu, s, o);
  if ((threadIdx.x & 31) == 0 && s) atomicAdd(total, s);
}

// string key bytes: one warp per output row
__global__ void k_key_gather(const __grid_constant__ FinishArgs f, uint32_t k) {
  const uint32_t i = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (i >= finish_rows(f)) return;
  const FinishKey& key = f.keys[k];
  const uint32_t gid = uint32_t(((f.wide ? f.wide[f.out_slot[i]] : uint64_t(f.out_slot[i])) / key.wstride) % (key.card + 1));
  if (gid == key.card) return;
  const uint32_t a = key.kd_offs[gid], n = key.kd_offs[gid + 1] - a;
  uint8_t* dst = f.out + key.data_off + reinterpret_cast<const int32_t*>(f.out + key.val_off)[i];
  for (uint32_t b = lane; b < n; b += 32) dst[b] = key.kd_bytes[a + b];
}

// bytes of a MIN / MAX over Utf8 (aggregate a): one warp per output row
__global__ void k_agg_str_gather(const __grid_constant__ FinishArgs f, uint32_t a) {
  const uint32_t i = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (i >= finish_rows(f)) return;
  const FinishAggStr& s = f.astr[a];
  const uint32_t n = reinterpret_cast<const uint32_t*>(f.out + s.len_off)[i];
  if (n == 0) return;   // NULL, or the empty string
  const unsigned long long rank = f.acc[size_t(1 + f.aggs[a].acc_slot) * f.nslots + f.out_slot[i]];
  const uint32_t g = s.inv[rank];
  const uint8_t* src = s.kd_bytes + s.kd_offs[g];
  uint8_t* dst = f.out + s.data_off + reinterpret_cast<const int32_t*>(f.out + f.val_off[a])[i];
  for (uint32_t b = lane; b < n; b += 32) dst[b] = src[b];
}


// ---- projection: TableProvider::scan(projection, ...) (stream_schema_provider.rs:526-659, :114-189) ----
// Late materialisation: the filter kernels leave a selection bitmap; only the selected rows of the
// projected columns are decoded, straight out of the flat store (row r of a page is bits
// [r*bw, (r+1)*bw) / 8-byte slot r), dictionary values through the chunk's dictionary.  The buffers
// of every result batch are assembled in one device block, like the aggregate results above.
struct ProjCol {
  const uint64_t* ent;   // strings: arena offset of every dictionary entry of the column
  uint64_t val_off;      // 8-byte values | per-batch bit words (bool) | int32 offsets (n + 1) (strings)
  uint64_t valid_off;    // per-batch validity words
  uint64_t src_off;      // strings: u64 arena offset of the bytes per output row (device-only scratch)
  uint64_t len_off;      // strings: u32 length per output row (device-only scratch)
  uint64_t data_off;     // strings: bytes
  uint32_t slot;         // column slot of the plan (chunk table, item.page, item.poff); 0xffffffff: the __row_id column
  uint32_t kind;         // DevKind (DK_I32: a Date32 column, 4-byte values)
};
struct ProjArgs {
  const uint8_t* arena;
  const uint8_t* flat;
  const FlatPageRec* fpages;
  const DevChunk* chunks;
  const DevItem* items;
  const uint32_t* bitmap;
  const uint32_t* item_counts;
  const unsigned long long* item_base;
  uint8_t* out;
  uint32_t* nulls;       // [ncols * nbatches]
  unsigned long long n_out;   // output rows kept (LIMIT)
  uint32_t n_items, plan_ncols, ncols;
  uint32_t batch_rows, words_per_batch, nbatches;
  ProjCol cols[kMaxCols + 1];
};

__device__ __forceinline__ uint32_t flat_bits_at(const uint8_t* flat, uint64_t off, uint64_t bit, uint32_t bw) {
  if (bw == 0) return 0;
  const uint32_t* w = reinterpret_cast<const uint32_t*>(flat + off) + (bit >> 5);
  const uint32_t sh = uint32_t(bit & 31);
  const uint32_t v = __funnelshift_r(w[0], w[1], sh);
  return bw >= 32 ? v : (v & ((1u << bw) - 1u));
}

// Every selected row of the work items this CTA takes (one CTA per item, grid-strided; <= 256 threads), in scan order:
// fn(item, item index, row inside the item, position in the selection = item_base + the in-item prefix).  Every thread
// of the CTA returns from it.
template <class Fn>
__device__ __forceinline__ void for_each_selected(const DevItem* __restrict__ items, const uint32_t* __restrict__ bitmap,
                                                  const uint32_t* __restrict__ item_counts, const unsigned long long* __restrict__ item_base,
                                                  uint32_t n_items, Fn&& fn) {
  __shared__ uint32_t warp_sums[8];
  __shared__ uint32_t carry;
  const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = blockDim.x >> 5;
  for (uint32_t it = blockIdx.x; it < n_items; it += gridDim.x) {
    if (item_counts[it] == 0) continue;   // uniform per block
    const DevItem& item = items[it];
    const uint32_t nwords = (item.nrows + 31) >> 5;
    if (threadIdx.x == 0) carry = 0;
    __syncthreads();
    for (uint32_t w0 = 0; w0 < nwords; w0 += blockDim.x) {
      const uint32_t w = w0 + threadIdx.x;
      uint32_t word = w < nwords ? bitmap[item.bitmap_word0 + w] : 0;
      const uint32_t c = __popc(word);
      uint32_t incl = c;
      for (int o = 1; o < 32; o <<= 1) {
        const uint32_t t = __shfl_up_sync(0xffffffffu, incl, o);
        if ((int)lane >= o) incl += t;
      }
      if (lane == 31) warp_sums[warp] = incl;
      __syncthreads();
      if (warp == 0) {
        uint32_t s = lane < nwarps ? warp_sums[lane] : 0, si = s;
        for (int o = 1; o < 32; o <<= 1) {
          const uint32_t t = __shfl_up_sync(0xffffffffu, si, o);
          if ((int)lane >= o) si += t;
        }
        if (lane < nwarps) warp_sums[lane] = si - s;
      }
      __syncthreads();
      unsigned long long pos = item_base[it] + carry + warp_sums[warp] + incl - c;
      while (word) {
        const uint32_t b = __ffs(word) - 1;
        word &= word - 1;
        fn(item, it, w * 32 + b, pos);
        pos++;
      }
      __syncthreads();
      if (threadIdx.x == blockDim.x - 1) carry += warp_sums[warp] + incl;
      __syncthreads();
    }
  }
}

// The value of row r of a work item in one column slot, straight out of the flat store (row r of a page is bits
// [r*bw, (r+1)*bw) / 8-byte slot r); false for NULL (a NULL row, or the column is missing from the file).  v is the
// 8-byte value (Int64 / Timestamp / Float64 bits, a numeric dictionary through the chunk's aligned copy) or 0 / 1
// (Boolean).  Utf8: the arena offset of the value's bytes, their length in len; with IDS instead the value's id in the
// column's GROUP BY numbering (ensure_key): gid[entry] of a dictionary entry, or the u32 of an FK_IDS page.
template <bool IDS>
__device__ __forceinline__ bool flat_value_at(const uint8_t* __restrict__ arena, const uint8_t* __restrict__ flat,
                                              const FlatPageRec* __restrict__ fpages, const DevChunk* __restrict__ chunks,
                                              uint32_t plan_ncols, const DevItem& item, uint32_t slot, uint32_t kind,
                                              const uint64_t* __restrict__ ent, const uint32_t* __restrict__ gid, uint32_t r,
                                              unsigned long long& v, uint32_t& len) {
  if ((item.absent >> slot) & 1u) return false;
  const FlatPageRec fp = fpages[item.page[slot]];
  const uint64_t row = uint64_t(item.poff[slot]) + r;
  if (fp.voff != ~0ull && !((reinterpret_cast<const uint32_t*>(flat + fp.voff)[row >> 5] >> (row & 31)) & 1u)) return false;
  if (IDS && fp.fkind == FK_IDS) {
    v = reinterpret_cast<const uint32_t*>(flat + fp.off)[row];
  } else if (fp.fkind == FK_BYTES) {   // PLAIN byte array: the row's bytes inside the page
    const uint64_t e = fp.base + reinterpret_cast<const uint32_t*>(flat + fp.off)[row];
    v = e;
    len = load_u32_unaligned(arena + e - 4);
  } else if (fp.fkind == FK_PLAIN8) {
    v = reinterpret_cast<const unsigned long long*>(flat + fp.off)[row];
  } else if (fp.fkind == FK_BITS) {
    v = (reinterpret_cast<const uint32_t*>(flat + fp.off)[row >> 5] >> (row & 31)) & 1u;
  } else {
    const DevChunk& ch = chunks[item.rg * plan_ncols + slot];
    uint32_t idx = flat_bits_at(flat, fp.off, row * fp.bw, fp.bw);
    idx = idx < ch.dict_n ? idx : (ch.dict_n ? ch.dict_n - 1 : 0);
    if (kind == DK_STR && IDS) {
      v = gid[ch.lut_base + idx];
    } else if (kind == DK_STR) {
      const uint64_t e = ent[ch.lut_base + idx];
      v = e;
      len = load_u32_unaligned(arena + e - 4);
    } else {
      v = reinterpret_cast<const unsigned long long*>(flat + ch.dict8_off)[idx];
    }
  }
  return true;
}

// every projected column of one selected row (row r of `item`) at output position pos < n_out
__device__ __forceinline__ void project_row(const ProjArgs& f, const DevItem& item, uint32_t r, unsigned long long pos) {
  const uint32_t batch = uint32_t(pos / f.batch_rows), bp = uint32_t(pos - uint64_t(batch) * f.batch_rows);
  const uint32_t vword = batch * f.words_per_batch + (bp >> 5), vbit = 1u << (bp & 31);
  for (uint32_t ci = 0; ci < f.ncols; ci++) {
    const ProjCol& pc = f.cols[ci];
    if (pc.slot == 0xffffffffu) {   // __row_id: ordinal of the row in the scanned table
      reinterpret_cast<unsigned long long*>(f.out + pc.val_off)[pos] = item.global_row0 + r;
      continue;
    }
    unsigned long long v = 0;
    uint32_t len = 0;
    if (!flat_value_at<false>(f.arena, f.flat, f.fpages, f.chunks, f.plan_ncols, item, pc.slot, pc.kind, pc.ent, nullptr, r, v, len)) {
      atomicAdd(&f.nulls[ci * f.nbatches + batch], 1u);   // NULL: value slot stays 0, string length 0
      continue;
    }
    atomicOr(reinterpret_cast<uint32_t*>(f.out + pc.valid_off) + vword, vbit);
    if (pc.kind == DK_STR) {
      reinterpret_cast<unsigned long long*>(f.out + pc.src_off)[pos] = v;
      reinterpret_cast<uint32_t*>(f.out + pc.len_off)[pos] = len;
    } else if (pc.kind == DK_BOOL) {
      if (v) atomicOr(reinterpret_cast<uint32_t*>(f.out + pc.val_off) + vword, vbit);
    } else if (pc.kind == DK_I32) {   // Date32: the low word of the sign-extended value
      reinterpret_cast<uint32_t*>(f.out + pc.val_off)[pos] = uint32_t(v);
    } else {
      reinterpret_cast<unsigned long long*>(f.out + pc.val_off)[pos] = v;
    }
  }
}

// one CTA per work item (grid-strided): bitmap words -> output positions -> values of every projected column
__global__ void __launch_bounds__(256) k_project(const __grid_constant__ ProjArgs f) {
  for_each_selected(f.items, f.bitmap, f.item_counts, f.item_base, f.n_items,
                    [&](const DevItem& item, uint32_t, uint32_t r, unsigned long long pos) {
                      if (pos < f.n_out) project_row(f, item, r, pos);
                    });
}

// ORDER BY ... LIMIT on a scan: output row i is the selected row at position kept[i] of the selection (kept == nullptr:
// i), reached through its handle (item index << 32 | row inside the item); one thread per output row
__global__ void __launch_bounds__(256) k_project_rows(const __grid_constant__ ProjArgs f, const unsigned long long* __restrict__ handles,
                                                      const uint32_t* __restrict__ kept) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= f.n_out) return;
  const unsigned long long h = handles[kept ? kept[i] : i];
  project_row(f, f.items[uint32_t(h >> 32)], uint32_t(h), i);
}

// ORDER BY ... LIMIT on a scan under PQ_QUERY_ALLGATHER: output row i is this rank's row with handle owned[i], or
// another rank's (~0): its bytes stay zero here, so that the sum of every rank's block is the result
__global__ void __launch_bounds__(256) k_project_owned(const __grid_constant__ ProjArgs f, const unsigned long long* __restrict__ owned) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= f.n_out) return;
  const unsigned long long h = owned[i];
  if (h != ~0ull) project_row(f, f.items[uint32_t(h >> 32)], uint32_t(h), i);
}

// string bytes of one projected column: one warp per output row (owned != nullptr: the rows k_project_owned projected)
__global__ void k_project_bytes(const __grid_constant__ ProjArgs f, uint32_t ci, unsigned long long n_rows,
                                const unsigned long long* __restrict__ owned = nullptr) {
  const unsigned long long i = (blockIdx.x * uint64_t(blockDim.x) + threadIdx.x) >> 5;
  const uint32_t lane = threadIdx.x & 31;
  if (i >= n_rows || (owned && owned[i] == ~0ull)) return;
  const ProjCol& pc = f.cols[ci];
  const uint32_t n = reinterpret_cast<const uint32_t*>(f.out + pc.len_off)[i];
  const uint8_t* src = f.arena + reinterpret_cast<const unsigned long long*>(f.out + pc.src_off)[i];
  uint8_t* dst = f.out + pc.data_off + reinterpret_cast<const int32_t*>(f.out + pc.val_off)[i];
  for (uint32_t b = lane; b < n; b += 32) dst[b] = src[b];
}

}  // namespace pqb
