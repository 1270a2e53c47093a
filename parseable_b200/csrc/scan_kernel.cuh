// The fused scan kernel: Parquet page decode -> predicate bitmap -> (count /
// selection bitmap | hash group-by accumulation) in ONE pass over the encoded
// bytes.  Replaces, for the reference, the DataFusion operator chain
//   DataSourceExec(Parquet) -> FilterExec -> AggregateExec(Partial)
// that Query::execute drives (/root/reference/src/query/mod.rs:287;
// SURVEY.md §8 rows a10-a12).
//
// Shape: persistent CTAs pull work items (row ranges between page boundaries
// common to all referenced columns) from a queue.  Per 2048-row slab a CTA
//   1. waits for the TMA bulk copies (cp.async.bulk + mbarrier) that staged the
//      next window of every encoded stream in shared memory,
//   2. one lane per column (on different warps) walks the RLE/bit-packed run
//      headers — the only sequential part of the format — into a run directory,
//   3. issues the TMA copies for the NEXT slab (double buffered),
//   4. all warps unpack bit-packed dictionary indices straight into leaf-predicate
//      bits (dictionary LUT byte per value, warp ballot -> 32-row words); columns
//      that feed GROUP BY / aggregates also stage their indices,
//   5. PLAIN pages are compared straight from HBM with 8-byte loads,
//   6. words are combined with Kleene logic and either counted / stored as the
//      selection bitmap, or drive shared-memory (or L2) atomics into the
//      accumulator table.
// Columns with NULLs take the general path (validity bitmap, rank, expansion).
// HBM traffic = the encoded bytes once + the bitmap; nothing decoded is written back.
#pragma once
#include <cuda_runtime.h>

#include "decode_core.cuh"
#include "device_structs.hpp"
#include "ptx_utils.cuh"

namespace pqb {

// tuning knobs (make EXTRA=-DPQB_SCAN_THREADS=128 ...): threads per CTA and the occupancy the
// register allocator is asked to allow
#ifndef PQB_SCAN_THREADS
#define PQB_SCAN_THREADS 256
#endif
#ifndef PQB_SCAN_MIN_BLOCKS
#define PQB_SCAN_MIN_BLOCKS 4
#endif
constexpr int kScanThreads = PQB_SCAN_THREADS;
constexpr int kScanWarps = kScanThreads / 32;

// byte offsets of the dynamic shared-memory regions, computed on the host
struct SmemLayout {
  uint32_t defwin[kMaxCols][2];
  uint32_t valwin[kMaxCols][2];
  uint32_t defwin_cap[kMaxCols];
  uint32_t valwin_cap[kMaxCols];
  uint32_t valid[kMaxCols];   // uint32[kSlabWords + 2]
  uint32_t rank[kMaxCols];    // uint32[kSlabWords]
  uint32_t idx[kMaxCols];     // uint32[kSlabRows]  (0: indices of this column are never staged)
  uint32_t defdir[kMaxCols];  // DirEntry[kMaxDirEntries]
  uint32_t valdir[kMaxCols][2];  // DirEntry / DeltaEntry directory of the value stream, double buffered
  uint32_t leafT;             // uint32[nleaves][kSlabWords + 2]
  uint32_t sel;               // uint32[kSlabWords]
  uint32_t acc;               // shared accumulator table
  uint32_t lutc;              // uint8[nleaves][kLutCacheBytes]: leaf LUTs of the current row group (fast AND path)
  uint32_t total;
};
constexpr int kLeafWords = kSlabWords + 2;
constexpr int kLutCacheBytes = 2048;

// per-column cursor over the pages of one column chunk
struct ColCursor {
  StreamState def, val;
  DeltaState dl;            // value stream of a DELTA_BINARY_PACKED page
  uint64_t val_base;        // arena offset of the values section of the current page
  uint64_t defwin_base[2];  // arena base of the staged windows
  uint64_t valwin_base[2];
  uint32_t page;
  uint32_t page_end;        // one past the chunk's last page
  uint32_t page_rows_left;
  uint32_t vals_done;       // non-null values consumed in the current page
  uint32_t enc;
  uint32_t has_def;
  uint32_t present;
  uint32_t _pad;
};

// what the row phase needs to know about a column for the CURRENT slab
struct SlabCol {
  uint64_t val_base;
  uint64_t dict_off;
  uint32_t vals_done;
  uint32_t enc;
  uint32_t bw;
  uint32_t present;
  uint32_t all_valid;
  uint32_t nv;
  uint32_t ndef, nval;
  uint32_t lut_base;
  uint32_t _pad;
  int64_t _pad2;
};

enum SlabMode : uint32_t { MODE_GENERIC = 0, MODE_FAST_AND = 1, MODE_ROW_MAJOR = 2, MODE_GENERAL_WALK = 3 };

struct ScanCtl {
  uint64_t mbar[2];
  uint32_t item;
  uint32_t error;
  uint32_t sel_count;
  uint32_t rmin_all;     // min over columns of the rows the fast walk covered
  uint32_t any_nulls;    // some column of this slab has a NULL (general path)
  uint32_t target;       // rows the next slab should try to take
  uint32_t mode;         // row pass chosen by the control warp for the current slab
  uint32_t R;            // rows of the current slab
  uint32_t has_delta;    // some column of this slab is DELTA_BINARY_PACKED
  uint32_t rmin[kMaxCols];
  int64_t scan_tmp[kScanWarps];             // DELTA prefix scan: per-warp totals
  uint32_t wcur[kScanWarps][kMaxCols];      // fast row pass: per warp, per column run-directory cursor
  uint32_t stk[kScanWarps][2 * kPredStack]; // fast row pass: per warp Kleene stack (t, n) words
  uint32_t lut_smem[kMaxLeaves];            // fast AND path: leaf LUT of this item's row group is cached in smem
  ColCursor cur[kMaxCols];
  SlabCol slab[2][kMaxCols];                // per staging buffer
  int64_t dl_last[kMaxCols];                // DELTA pages: value of the last row decoded so far in the page (carried across slabs)
};

__device__ __forceinline__ void page_enter(ColCursor& c, const DevPage* pages, uint32_t pg) {
  const DevPage p = pages[pg];
  c.page = pg;
  c.page_rows_left = p.num_rows;
  c.vals_done = 0;
  c.enc = p.enc;
  c.has_def = p.def_len != 0;
  c.val_base = p.off + p.val_off;
  stream_init(c.def, p.off + p.def_off, p.off + p.def_off + p.def_len, 1);
  stream_init(c.val, p.off + p.val_off, p.off + p.len, p.bit_width);
  if (p.enc == DE_DELTA) delta_init(c.dl, p.off + p.val_off, p.off + p.len);
}

__device__ __forceinline__ uint64_t value_window_start(const ColCursor& c) {
  return c.enc == DE_DELTA ? delta_window_start(c.dl) : stream_window_start(c.val);
}

// thread 0: stage the windows every stream needs next into buffer `buf`, and publish the row
// target of the next slab
__device__ __forceinline__ void issue_windows(ScanCtl& ctl, const SmemLayout& L, uint8_t* smem,
                                              const uint8_t* arena, uint32_t ncols, uint32_t buf, uint32_t rows_left) {
  uint32_t bytes = 0;
  uint32_t target = rows_left < (uint32_t)kSlabRows ? rows_left : (uint32_t)kSlabRows;
  for (uint32_t c = 0; c < ncols; c++) {
    const ColCursor& cr = ctl.cur[c];
    if (!cr.present) continue;
    target = cr.page_rows_left < target ? cr.page_rows_left : target;
    if (cr.has_def) bytes += L.defwin_cap[c];
    if (PQB_ENC_HAS_WINDOW(cr.enc)) bytes += L.valwin_cap[c];
  }
  ctl.target = target;
  ctl.rmin_all = target;
  ctl.any_nulls = 0;
  mbar_arrive_expect_tx(&ctl.mbar[buf], bytes);
  for (uint32_t c = 0; c < ncols; c++) {
    ColCursor& cr = ctl.cur[c];
    if (!cr.present) continue;
    if (cr.has_def) {
      uint64_t s = stream_window_start(cr.def) & ~15ull;
      cr.defwin_base[buf] = s;
      tma_load_1d(smem + L.defwin[c][buf], arena + s, L.defwin_cap[c], &ctl.mbar[buf]);
    }
    if (PQB_ENC_HAS_WINDOW(cr.enc)) {
      uint64_t s = value_window_start(cr) & ~15ull;
      cr.valwin_base[buf] = s;
      tma_load_1d(smem + L.valwin[c][buf], arena + s, L.valwin_cap[c], &ctl.mbar[buf]);
    }
  }
}

// OR a 32-bit group of bits into a bitmap at an arbitrary bit position
__device__ __forceinline__ void or_bits(uint32_t* bm, uint32_t pos, uint32_t word) {
  uint32_t sh = pos & 31;
  if (sh == 0) { atomicOr(&bm[pos >> 5], word); return; }
  atomicOr(&bm[pos >> 5], word << sh);
  uint32_t hi = word >> (32 - sh);
  if (hi) atomicOr(&bm[(pos >> 5) + 1], hi);
}

// two sentinel entries (start = ~0) behind the last directory entry: the row pass may always look
// one and two entries ahead without a bounds test
__device__ __forceinline__ void dir_sentinels(DirEntry* dir, uint32_t n) {
  dir[n].start = 0xffffffffu; dir[n].count = 0; dir[n].kind = 0; dir[n].chunk0 = 0; dir[n].payload = 0; dir[n]._pad = 0;
  dir[n + 1] = dir[n];
}

// expand a run directory of 1-bit values into a bitmap (OR into pre-zeroed words)
__device__ __forceinline__ void dir_to_bitmap(const DirEntry* dir, uint32_t nent, const uint32_t* win,
                                              uint32_t* bm) {
  for (uint32_t e = warp_id(); e < nent; e += kScanWarps) {
    const DirEntry d = dir[e];
    for (uint32_t k = 0; k < d.count; k += 32) {
      uint32_t j = k + lane_id();
      uint32_t bit = 0;
      if (j < d.count) bit = d.kind ? bp_get(win, d.payload, 1, j) : (d.payload & 1);
      uint32_t word = __ballot_sync(0xffffffffu, bit);
      if (lane_id() == 0 && word) or_bits(bm, d.start + k, word);
    }
  }
}

// unpack a run directory of dictionary indices into idx[0..nv)
__device__ __forceinline__ void dir_to_idx(const DirEntry* dir, uint32_t nent, const uint32_t* win, uint32_t bw,
                                           uint32_t* idx) {
  for (uint32_t e = warp_id(); e < nent; e += kScanWarps) {
    const DirEntry d = dir[e];
    if (d.kind) {
      for (uint32_t j = lane_id(); j < d.count; j += 32) idx[d.start + j] = bp_get(win, d.payload, bw, j);
    } else {
      for (uint32_t j = lane_id(); j < d.count; j += 32) idx[d.start + j] = d.payload;
    }
  }
}

// Fused unpack -> leaf LUT -> ballot: no index staging.  Up to two leaves of the same column are
// evaluated from one unpacked index; bits land in VALUE space (== row space when the slab has no
// NULLs).  Work is dealt to warps in 32-value chunks (DirEntry.chunk0), not whole runs, so a slab
// with five 504-value runs still keeps all eight warps busy.
template <bool kTwo>
__device__ __forceinline__ void dir_to_leafbits(const DirEntry* dir, uint32_t nent, const uint32_t* win, uint32_t bw,
                                                const uint8_t* __restrict__ lut0, uint32_t* T0,
                                                const uint8_t* __restrict__ lut1, uint32_t* T1, uint32_t* idx) {
  if (nent == 0) return;
  const DirEntry last = dir[nent - 1];
  const uint32_t nchunks = uint32_t(last.chunk0) + ((uint32_t(last.count) + 31u) >> 5);
  const uint32_t lane = lane_id();
  uint32_t e = 0;
  DirEntry d = dir[0];
  uint32_t next0 = nent > 1 ? uint32_t(dir[1].chunk0) : 0xffffffffu;
  for (uint32_t q = warp_id(); q < nchunks; q += kScanWarps) {
    while (q >= next0) {  // warp uniform; chunks are visited in increasing order
      e++;
      d = dir[e];
      next0 = e + 1 < nent ? uint32_t(dir[e + 1].chunk0) : 0xffffffffu;
    }
    const uint32_t k = (q - d.chunk0) * 32;
    const uint32_t j = k + lane;
    const bool in = j < d.count;
    const uint32_t v = d.kind ? (in ? bp_get(win, d.payload, bw, j) : 0u) : d.payload;
    if (idx && in) idx[d.start + j] = v;
    const uint32_t w0 = __ballot_sync(0xffffffffu, in && lut0[v]);
    uint32_t w1 = 0;
    if (kTwo) w1 = __ballot_sync(0xffffffffu, in && lut1[v]);
    if (lane == 0) {
      if (w0) or_bits(T0, d.start + k, w0);
      if (kTwo && w1) or_bits(T1, d.start + k, w1);
    }
  }
}

struct RowVal {
  bool valid;
  uint32_t j;  // rank among the non-null values of the slab
};

__device__ __forceinline__ RowVal row_rank(const SlabCol& c, const uint32_t* valid, const uint32_t* rank, uint32_t r) {
  RowVal o;
  if (!c.present) { o.valid = false; o.j = 0; return o; }
  if (c.all_valid) { o.valid = true; o.j = r; return o; }
  uint32_t w = valid[r >> 5];
  o.valid = (w >> (r & 31)) & 1;
  o.j = rank[r >> 5] + __popc(w & ((1u << (r & 31)) - 1u));
  return o;
}

// 8-byte value of a non-null row: dictionary entry or PLAIN slot
__device__ __forceinline__ uint64_t value_u64(const SlabCol& c, const uint8_t* arena, const uint32_t* idx, uint32_t j) {
  if (c.enc == DE_DICT) return load_u64_unaligned(arena + c.dict_off + uint64_t(idx[j]) * 8);
  if (c.enc == DE_DELTA) return reinterpret_cast<const uint64_t*>(idx)[j];  // decoded + prefix-summed in place
  return load_u64_unaligned(arena + c.val_base + uint64_t(c.vals_done + j) * 8);
}
__device__ __forceinline__ uint32_t value_bool(const SlabCol& c, const uint8_t* arena, const uint32_t* idx, uint32_t j) {
  if (c.enc == DE_RLE_BOOL) return idx[j] & 1;  // v2 pages: booleans as an RLE / bit-packed hybrid stream
  uint32_t k = c.vals_done + j;
  return (arena[c.val_base + (k >> 3)] >> (k & 7)) & 1;
}

template <typename T>
__device__ __forceinline__ T* smem_at(uint8_t* base, uint32_t off) {
  return reinterpret_cast<T*>(base + off);
}

// 64-bit integer add into an accumulator cell.  Global memory has a native 64-bit reduction; shared
// memory does not (the compiler emits a compare-and-swap spin loop, ATOMS.CAST.SPIN.64, which
// collapses under the contention of a 25-group table), so there the add is two native 32-bit
// atomics: the low word, and the high word plus the carry this very add produced.  Addition
// commutes per word and every wrap of the low word is seen by exactly one thread, so the cell is
// exact once the CTA has synchronised (it is only read at the flush).
__device__ __forceinline__ void acc_add(unsigned long long* cell, unsigned long long v) {
  if (__isShared(cell)) {
    uint32_t* w = reinterpret_cast<uint32_t*>(cell);
    const uint32_t lo = uint32_t(v), hi = uint32_t(v >> 32);
    uint32_t carry = 0;
    if (lo) {
      const uint32_t old = atomicAdd(&w[0], lo);
      carry = uint32_t(old + lo) < lo ? 1u : 0u;
    }
    if (hi + carry) atomicAdd(&w[1], hi + carry);
  } else {
    atomicAdd(cell, v);
  }
}

__device__ __forceinline__ void acc_apply(unsigned long long* cell, uint32_t fn, uint32_t kind, uint64_t bits) {
  if (fn == AG_SUM) {
    if (kind == DK_F64) atomicAdd(reinterpret_cast<double*>(cell), __longlong_as_double((long long)bits));
    else acc_add(cell, (unsigned long long)bits);  // wrapping, like DataFusion's SUM(Int64)
  } else if (fn == AG_AVG) {
    double v = kind == DK_F64 ? __longlong_as_double((long long)bits) : double((long long)bits);
    atomicAdd(reinterpret_cast<double*>(cell), v);
  } else {
    long long k = kind == DK_F64 ? (long long)f64_order_key(bits) : (long long)bits;
    // shared memory: 64-bit min / max are compare-and-swap loops; the cell only ever moves one way,
    // so a row that cannot improve the value it reads (one aligned 8-byte load) skips the atomic —
    // after the first few rows of a group that is nearly every row
    if (__isShared(cell)) {
      const long long cur = *reinterpret_cast<volatile long long*>(cell);
      if (fn == AG_MIN ? k >= cur : k <= cur) return;
    }
    if (fn == AG_MIN) atomicMin(reinterpret_cast<long long*>(cell), k);
    else atomicMax(reinterpret_cast<long long*>(cell), k);
  }
}

// merge one accumulator cell of a CTA-private (shared memory) table into the global table
__device__ __forceinline__ void acc_merge(unsigned long long* cell, uint32_t how, unsigned long long v) {
  // how: 0 integer add, 1 f64 add, 2 min (signed), 3 max (signed)
  if (how == 0) atomicAdd(cell, v);
  else if (how == 1) atomicAdd(reinterpret_cast<double*>(cell), __longlong_as_double((long long)v));
  else if (how == 2) atomicMin(reinterpret_cast<long long*>(cell), (long long)v);
  else atomicMax(reinterpret_cast<long long*>(cell), (long long)v);
}

__device__ __forceinline__ uint32_t row_mask(uint32_t w, uint32_t R) {
  uint32_t lo = w * 32;
  if (R <= lo) return 0;
  uint32_t n = R - lo;
  return n >= 32 ? 0xffffffffu : ((1u << n) - 1u);
}

// which thread walks column c: lane c of warp 0, the control warp.  All per-slab control lives on
// that one warp so the other warps park at the block barrier instead of burning issue slots.
__device__ __forceinline__ bool walker_of(uint32_t ncols, uint32_t& col) {
  col = lane_id();
  return warp_id() == 0 && col < ncols;
}


// ---- DELTA_BINARY_PACKED: miniblock directory -> deltas -> block-wide inclusive scan -> values ----
__device__ __forceinline__ void delta_decode_scan(ScanCtl& ctl, const SmemLayout& L, uint8_t* smem, uint32_t c, uint32_t buf) {
  SlabCol& s = ctl.slab[buf][c];
  const uint32_t nv = s.nv;
  int64_t* vals = smem_at<int64_t>(smem, L.idx[c]);
  const DeltaEntry* dir = smem_at<DeltaEntry>(smem, L.valdir[c][buf]);
  const uint32_t* win = smem_at<uint32_t>(smem, L.valwin[c][buf]);
  for (uint32_t e = warp_id(); e < s.nval; e += kScanWarps) {
    const DeltaEntry d = dir[e];
    for (uint32_t j = lane_id(); j < d.count; j += 32)
      vals[d.start + j] = d.kind ? d.min_delta : int64_t(uint64_t(d.min_delta) + bp_get64(win, d.bitoff, d.bw, j));
  }
  __syncthreads();
  // a slab that starts a page begins with the page's first value (absolute): no carry
  const int64_t carry = (s.nval && dir[0].kind == 1) ? 0 : ctl.dl_last[c];
  constexpr uint32_t kPer = kSlabRows / kScanThreads;
  const uint32_t b = threadIdx.x * kPer;
  int64_t loc[kPer];
  int64_t sum = 0;
#pragma unroll
  for (uint32_t i = 0; i < kPer; i++) {
    int64_t v = (b + i < nv) ? vals[b + i] : 0;
    sum = int64_t(uint64_t(sum) + uint64_t(v));
    loc[i] = sum;
  }
  int64_t incl = sum;
  for (int o = 1; o < 32; o <<= 1) {
    int64_t t = __shfl_up_sync(0xffffffffu, incl, o);
    if ((int)lane_id() >= o) incl = int64_t(uint64_t(incl) + uint64_t(t));
  }
  if (lane_id() == 31) ctl.scan_tmp[warp_id()] = incl;
  __syncthreads();
  int64_t base = carry;
  for (uint32_t w = 0; w < warp_id(); w++) base = int64_t(uint64_t(base) + uint64_t(ctl.scan_tmp[w]));
  base = int64_t(uint64_t(base) + uint64_t(incl) - uint64_t(sum));
#pragma unroll
  for (uint32_t i = 0; i < kPer; i++)
    if (b + i < nv) vals[b + i] = int64_t(uint64_t(base) + uint64_t(loc[i]));
  __syncthreads();
  if (threadIdx.x == 0 && nv) ctl.dl_last[c] = vals[nv - 1];
  __syncthreads();
}

// ---- the no-NULL fast row pass --------------------------------------------------------------
// Dictionary index of row r (== value r: the slab has no NULLs) of column c, straight from the
// staged bytes through the run directory.  Control flow is warp uniform except the (rare) walk
// across directory entries inside one 32-row word.
__device__ __forceinline__ uint32_t fast_idx(ScanCtl& ctl, const SmemLayout& L, uint8_t* smem, uint32_t c, uint32_t buf,
                                             uint32_t base_row, uint32_t r, bool in) {
  const SlabCol& s = ctl.slab[buf][c];
  const DirEntry* dir = smem_at<DirEntry>(smem, L.valdir[c][buf]);
  const uint32_t n = s.nval;
  uint32_t e = ctl.wcur[warp_id()][c];
  while (e + 1 < n && dir[e + 1].start <= base_row) e++;
  ctl.wcur[warp_id()][c] = e;
  if (!in) return 0;
  while (e + 1 < n && dir[e + 1].start <= r) e++;
  const DirEntry d = dir[e];
  return d.kind ? bp_get(smem_at<uint32_t>(smem, L.valwin[c][buf]), d.payload, s.bw, r - d.start) : d.payload;
}

__device__ __forceinline__ uint64_t fast_value_u64(ScanCtl& ctl, const SmemLayout& L, uint8_t* smem, const uint8_t* arena,
                                                   uint32_t c, uint32_t buf, uint32_t base_row, uint32_t r, bool in, bool want) {
  const SlabCol& s = ctl.slab[buf][c];
  if (PQB_ENC_HAS_STREAM(s.enc)) {
    uint32_t v = fast_idx(ctl, L, smem, c, buf, base_row, r, in);
    if (s.enc == DE_RLE_BOOL) return v & 1;
    return (in && want) ? load_u64_unaligned(arena + s.dict_off + uint64_t(v) * 8) : 0;
  }
  if (s.enc == DE_DELTA) return (in && want) ? smem_at<uint64_t>(smem, L.idx[c])[r] : 0;
  return (in && want) ? load_u64_unaligned(arena + s.val_base + uint64_t(s.vals_done + r) * 8) : 0;
}

// One 32-row word of one leaf: returns T (and N through *nw); all lanes get the same words.
__device__ __forceinline__ uint32_t fast_leaf_word(const DevPlan& plan, ScanCtl& ctl, const SmemLayout& L, uint8_t* smem,
                                                   const DevScanArgs& a, uint32_t l, uint32_t buf, uint32_t base_row,
                                                   uint32_t r, bool in, uint32_t* nw) {
  const DevLeaf& lf = plan.leaves[l];
  const uint32_t c = lf.col;
  const SlabCol& s = ctl.slab[buf][c];
  *nw = 0;
  if (!s.present) {  // column missing from this file: every row NULL
    if (lf.kind == LK_IS_NULL) return 0xffffffffu;
    if (lf.kind == LK_IS_NOT_NULL) return 0;
    *nw = 0xffffffffu;
    return 0;
  }
  if (lf.kind == LK_IS_NULL) return 0;
  if (lf.kind == LK_IS_NOT_NULL) return 0xffffffffu;
  const uint8_t kind = plan.cols[c].kind;
  bool t = false;
  if (PQB_ENC_HAS_STREAM(s.enc)) {
    uint32_t v = fast_idx(ctl, L, smem, c, buf, base_row, r, in);
    if (in) t = s.enc == DE_DICT ? a.luts[lf.lut_off + s.lut_base + v] != 0 : cmp_i64((int64_t)(v & 1), lf.lit_i64, lf.cmp);
  } else if (in) {
    if (kind == DK_BOOL) {
      uint32_t k = s.vals_done + r;
      t = cmp_i64((int64_t)((a.arena[s.val_base + (k >> 3)] >> (k & 7)) & 1), lf.lit_i64, lf.cmp);
    } else {
      uint64_t v = s.enc == DE_DELTA ? smem_at<uint64_t>(smem, L.idx[c])[r]
                                     : load_u64_unaligned(a.arena + s.val_base + uint64_t(s.vals_done + r) * 8);
      t = kind == DK_F64 ? cmp_i64(f64_order_key(v), f64_order_key((uint64_t)lf.lit_i64), lf.cmp)
                         : cmp_i64((int64_t)v, lf.lit_i64, lf.cmp);
    }
  }
  return __ballot_sync(0xffffffffu, t);
}

// Every warp owns whole 32-row words of the slab: leaves -> Kleene combine -> consume, all in
// registers / per-warp scratch.  No leaf bitmaps, no staging, no block barrier.  Returns the rows
// this thread's warp selected (lane 0 carries the count).
__device__ __forceinline__ uint32_t fast_rows(const DevPlan& plan, ScanCtl& ctl, const SmemLayout& L, uint8_t* smem,
                                              const DevScanArgs& a, const DevItem& item, uint32_t buf, uint32_t R,
                                              uint32_t r_item, unsigned long long* acc, bool agg_mode) {
  const uint32_t warp = warp_id(), lane = lane_id();
  const uint32_t nwords = (R + 31) >> 5;
  const uint32_t nslots = plan.nslots;
  if (lane < plan.ncols) ctl.wcur[warp][lane] = 0;
  __syncwarp();
  uint32_t* st = ctl.stk[warp];
  uint32_t cnt = 0;
  for (uint32_t w = warp; w < nwords; w += kScanWarps) {
    const uint32_t base_row = w * 32, r = base_row + lane;
    const bool in = r < R;
    int sp = 0;
#pragma unroll 1
    for (uint32_t i = 0; i < plan.npred; i++) {
      const DevPredOp op = plan.pred[i];
      if (op.kind == PK_LEAF) {
        uint32_t n;
        uint32_t t = fast_leaf_word(plan, ctl, L, smem, a, op.arg, buf, base_row, r, in, &n);
        st[2 * sp] = t;
        st[2 * sp + 1] = n;
        sp++;
      } else if (op.kind == PK_CONST) {
        st[2 * sp] = op.arg == 1 ? 0xffffffffu : 0u;
        st[2 * sp + 1] = op.arg == 2 ? 0xffffffffu : 0u;
        sp++;
      } else if (op.kind == PK_NOT) {
        st[2 * sp - 2] = ~(st[2 * sp - 2] | st[2 * sp - 1]);
      } else {
        uint32_t tb = st[2 * sp - 2], nb = st[2 * sp - 1], ta = st[2 * sp - 4], na = st[2 * sp - 3];
        sp--;
        if (op.kind == PK_AND) {
          uint32_t fa = ~(ta | na), fb = ~(tb | nb);
          st[2 * sp - 2] = ta & tb;
          st[2 * sp - 1] = (na | nb) & ~fa & ~fb;
        } else {
          uint32_t t = ta | tb;
          st[2 * sp - 2] = t;
          st[2 * sp - 1] = (na | nb) & ~t;
        }
      }
    }
    const uint32_t sel = (plan.npred ? st[0] : 0xffffffffu) & row_mask(w, R);
    if (!agg_mode) {
      if (lane == 0) {
        cnt += __popc(sel);
        if (plan.write_bitmap && sel) {
          uint32_t pos = r_item + base_row;
          uint32_t* dst = a.bitmap + item.bitmap_word0 + (pos >> 5);
          uint32_t sh = pos & 31;
          if (sh == 0) *dst = sel;
          else {
            atomicOr(dst, sel << sh);
            uint32_t hi = sel >> (32 - sh);
            if (hi) atomicOr(dst + 1, hi);
          }
        }
      }
      continue;
    }
    if (sel == 0) continue;  // uniform
    const bool mine = (sel >> lane) & 1;
    if (lane == 0) cnt += __popc(sel);
    uint32_t slot = 0;
    for (uint32_t k = 0; k < plan.nkeys; k++) {
      const DevKey& key = plan.keys[k];
      const SlabCol& s = ctl.slab[buf][key.col];
      uint32_t gid = key.card;  // column missing: NULL group
      if (s.present) {
        if (key.kind == KK_BOOL) {
          gid = (uint32_t)fast_value_u64(ctl, L, smem, a.arena, key.col, buf, base_row, r, in, false);
          if (!PQB_ENC_HAS_STREAM(s.enc)) {
            uint32_t kk = s.vals_done + r;
            gid = in ? (a.arena[s.val_base + (kk >> 3)] >> (kk & 7)) & 1 : 0;
          }
        } else {
          uint32_t v = fast_idx(ctl, L, smem, key.col, buf, base_row, r, in);
          gid = mine ? key.gid[s.lut_base + v] : 0;
        }
      }
      slot += gid * key.stride;
    }
    if (mine) acc_add(&acc[slot], 1ull);
    for (uint32_t g = 0; g < plan.naggs; g++) {
      const DevAgg& ag = plan.aggs[g];
      if (ag.fn == AG_COUNT_STAR) continue;
      const SlabCol& s = ctl.slab[buf][ag.col];
      if (!s.present) continue;  // all NULL: contributes nothing
      uint64_t bits;
      if (ag.kind == DK_BOOL && !PQB_ENC_HAS_STREAM(s.enc)) {
        uint32_t kk = s.vals_done + r;
        bits = in ? (a.arena[s.val_base + (kk >> 3)] >> (kk & 7)) & 1 : 0;
      } else {
        bits = fast_value_u64(ctl, L, smem, a.arena, ag.col, buf, base_row, r, in, mine && ag.fn != AG_COUNT);
      }
      if (!mine) continue;
      if (ag.update_nn) acc_add(&acc[(1 + plan.n_acc + ag.nn_slot) * nslots + slot], 1ull);
      if (ag.fn == AG_COUNT) continue;
      acc_apply(&acc[(1 + ag.acc_slot) * nslots + slot], ag.fn, ag.kind, bits);
    }
  }
  return cnt;
}

// ---- specialised row pass: WHERE leaf AND leaf AND ... over dictionary pages, no NULLs ----------
// The common log-analytics filter shape (level = 'ERROR' AND latency_ms > 100 AND ...).  Every
// thread owns 8 consecutive rows of the slab (one byte of the selection): per leaf it finds its
// run-directory entry, unpacks its 8 indices from the staged window into registers, probes the
// leaf's LUT and ANDs the byte.  No leaf bitmaps, no atomics, no block barrier inside the slab.
// The aggregate consume pass still walks 32-row words (a warp owns kWordsPerWarp consecutive ones).
// Aggregate consume of one 32-row selection word (conjunction pass): group slot from the key
// columns, then every aggregate.  Deliberately NOT inlined: the caller's loop over the warp's eight
// words is unrolled, and eight inlined copies of this body made the kernel miss the instruction
// cache (ncu: no_instruction was the top stall of a filtered group-by, issue slots 15 % busy).
__device__ __noinline__ void consume_word_agg(const DevPlan& plan, ScanCtl& ctl, const SmemLayout& L, uint8_t* smem, const DevScanArgs& a,
                                              uint32_t buf, uint32_t base_row, uint32_t sel, uint32_t R, unsigned long long* acc) {
  const uint32_t lane = lane_id();
  const uint32_t nslots = plan.nslots;
  const uint32_t r = base_row + lane;
  const bool in = r < R;
  const bool mine = (sel >> lane) & 1;
  uint32_t slot = 0;
  for (uint32_t k = 0; k < plan.nkeys; k++) {
    const DevKey& key = plan.keys[k];
    const SlabCol& s = ctl.slab[buf][key.col];
    uint32_t gid = key.card;
    if (s.present) {
      if (key.kind == KK_BOOL) {
        gid = (uint32_t)fast_value_u64(ctl, L, smem, a.arena, key.col, buf, base_row, r, in, false);
        if (!PQB_ENC_HAS_STREAM(s.enc)) {
          uint32_t kk = s.vals_done + r;
          gid = in ? (a.arena[s.val_base + (kk >> 3)] >> (kk & 7)) & 1 : 0;
        }
      } else {
        uint32_t v = fast_idx(ctl, L, smem, key.col, buf, base_row, r, in);
        gid = mine ? key.gid[s.lut_base + v] : 0;
      }
    }
    slot += gid * key.stride;
  }
  if (mine) acc_add(&acc[slot], 1ull);
  for (uint32_t g = 0; g < plan.naggs; g++) {
    const DevAgg& ag = plan.aggs[g];
    if (ag.fn == AG_COUNT_STAR) continue;
    const SlabCol& s = ctl.slab[buf][ag.col];
    if (!s.present) continue;
    uint64_t bits;
    if (ag.kind == DK_BOOL && !PQB_ENC_HAS_STREAM(s.enc)) {
      uint32_t kk = s.vals_done + r;
      bits = in ? (a.arena[s.val_base + (kk >> 3)] >> (kk & 7)) & 1 : 0;
    } else {
      bits = fast_value_u64(ctl, L, smem, a.arena, ag.col, buf, base_row, r, in, mine && ag.fn != AG_COUNT);
    }
    if (!mine) continue;
    if (ag.update_nn) acc_add(&acc[(1 + plan.n_acc + ag.nn_slot) * nslots + slot], 1ull);
    if (ag.fn == AG_COUNT) continue;
    acc_apply(&acc[(1 + ag.acc_slot) * nslots + slot], ag.fn, ag.kind, bits);
  }
}

constexpr int kWordsPerWarp = kSlabWords / kScanWarps;
constexpr int kRowsPerThread = kSlabRows / kScanThreads;
static_assert(kRowsPerThread == 8, "the octet pass gives every thread 8 consecutive rows (one selection byte)");

// One leaf over one thread's octet: rows [r, r + 8) of the slab.  Returns the LUT answers as a byte
// (bit k = row r + k); bits outside `need` are don't-care.  Parquet packs dictionary indices in
// groups of 8 values = bw bytes, so a thread that owns 8 consecutive rows reads one short byte
// range of the staged window and keeps everything else in registers: per-row cost is a shift, a
// mask, one LUT byte and one LEA, against ~2 warp-instructions per row for the ballot-per-word
// scheme this replaces (profiles/k_scan_r1c: 65 % of all executed instructions).
__device__ __forceinline__ uint32_t octet_leaf(const uint32_t* __restrict__ dirw, uint32_t nent, const uint32_t* __restrict__ win,
                                               uint32_t bw, uint32_t r, uint32_t need, bool smem_lut,
                                               const uint8_t* __restrict__ lut_s, const uint8_t* __restrict__ lut_g) {
  // directory entry holding row r: {start, count | kind << 16 | chunk0 << 24, payload}; two sentinel
  // entries (start = ~0) follow the last one
  uint32_t e = 0;
  if (nent > 6) {
#pragma unroll
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
      const uint32_t lo = __funnelshift_r(x0, x1, sh), hi = __funnelshift_r(x1, x2, sh);
      if (smem_lut) {
#pragma unroll
        for (int k = 7; k >= 0; k--) {
          const uint32_t s = uint32_t(k) * bw;
          const uint32_t v = (s < 32 ? __funnelshift_r(lo, hi, s) : (hi >> (s - 32))) & vmask;
          m = m * 2 + lut_s[v];
        }
      } else {
#pragma unroll
        for (int k = 7; k >= 0; k--) {
          const uint32_t s = uint32_t(k) * bw;
          const uint32_t v = (s < 32 ? __funnelshift_r(lo, hi, s) : (hi >> (s - 32))) & vmask;
          m = m * 2 + (((need >> k) & 1) ? uint32_t(lut_g[v]) : 0u);
        }
      }
      return m;
    }
#pragma unroll
    for (int k = 7; k >= 0; k--) {
      uint32_t t = 0;
      if ((need >> k) & 1) {
        const uint32_t bit = bit0 + uint32_t(k) * bw;
        const uint32_t wi = bit >> 5;
        const uint32_t v = __funnelshift_r(win[wi], win[wi + 1], bit & 31) & vmask;
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
          const uint32_t v = __funnelshift_r(win[wi], win[wi + 1], bit & 31) & vmask;
          const uint32_t t = smem_lut ? lut_s[v & (kLutCacheBytes - 1)] : lut_g[v];
          m |= (t ? 1u : 0u) << j;
        }
      }
    }
    k = kend;
  }
  return m;
}

__device__ __forceinline__ uint32_t fast_and_rows(const DevPlan& plan, ScanCtl& ctl, const SmemLayout& L, uint8_t* smem,
                                                  const DevScanArgs& a, const DevItem& item, uint32_t buf, uint32_t R,
                                                  uint32_t r_item, unsigned long long* acc, bool agg_mode) {
  const uint32_t warp = warp_id(), lane = lane_id();
  const uint32_t nslots = plan.nslots;
  const uint32_t w0 = warp * kWordsPerWarp;
  // ---- leaves: every thread answers its own 8 rows ----
  const uint32_t r8 = threadIdx.x * kRowsPerThread;
  uint32_t sel8 = r8 >= R ? 0u : (R - r8 >= 8 ? 0xffu : ((1u << (R - r8)) - 1u));
  for (uint32_t l = 0; l < plan.nleaves; l++) {
    if (sel8 == 0) break;  // per thread: nothing left in its octet (most octets once a selective leaf ran)
    const DevLeaf& lf = plan.leaves[l];
    const SlabCol& s = ctl.slab[buf][lf.col];
    sel8 &= octet_leaf(smem_at<uint32_t>(smem, L.valdir[lf.col][buf]), s.nval, smem_at<uint32_t>(smem, L.valwin[lf.col][buf]), s.bw, r8,
                       sel8, ctl.lut_smem[l] != 0, smem + L.lutc + l * kLutCacheBytes, a.luts + lf.lut_off + s.lut_base);
  }
  if (!agg_mode && (!plan.write_bitmap || ((r_item & 7u) == 0))) {
    // count / selection bitmap straight from the bytes (the item's bitmap region is byte addressable)
    if (sel8 && plan.write_bitmap)
      reinterpret_cast<uint8_t*>(a.bitmap + item.bitmap_word0)[(r_item + r8) >> 3] = uint8_t(sel8);
    return __popc(sel8);
  }
  // selection words for the consume pass below: word j of this warp = the bytes of lanes 4j .. 4j+3
  uint32_t selw[kWordsPerWarp];
  {
    const uint32_t src = (lane & 7u) * 4u;
    const uint32_t wv = __shfl_sync(0xffffffffu, sel8, src) | (__shfl_sync(0xffffffffu, sel8, src + 1) << 8) |
                        (__shfl_sync(0xffffffffu, sel8, src + 2) << 16) | (__shfl_sync(0xffffffffu, sel8, src + 3) << 24);
#pragma unroll
    for (int i = 0; i < kWordsPerWarp; i++) selw[i] = __shfl_sync(0xffffffffu, wv, i);
  }
  if (agg_mode) {
    if (lane < plan.ncols) ctl.wcur[warp][lane] = 0;
    __syncwarp();
  }
  uint32_t cnt = 0;
#pragma unroll
  for (int i = 0; i < kWordsPerWarp; i++) {
    const uint32_t sel = selw[i];
    if (sel == 0) continue;
    const uint32_t base_row = (w0 + i) * 32, r = base_row + lane;
    const bool in = r < R;
    if (!agg_mode) {
      if (lane == 0) {
        cnt += __popc(sel);
        if (plan.write_bitmap) {
          uint32_t pos = r_item + base_row;
          uint32_t* dst = a.bitmap + item.bitmap_word0 + (pos >> 5);
          uint32_t sh = pos & 31;
          if (sh == 0) *dst = sel;
          else {
            atomicOr(dst, sel << sh);
            uint32_t hi = sel >> (32 - sh);
            if (hi) atomicOr(dst + 1, hi);
          }
        }
      }
      continue;
    }
    if (lane == 0) cnt += __popc(sel);
    consume_word_agg(plan, ctl, L, smem, a, buf, base_row, sel, R, acc);
  }
  return cnt;
}

// The general per-slab walk (columns with NULLs, window / directory overflow): definition levels ->
// validity bitmap + ranks -> index streams, shrinking the slab until every column is covered.
// All threads call it; returns the rows of the slab (0: corrupt page).
__device__ __noinline__ uint32_t general_walk(ScanCtl& ctl, const SmemLayout& L, uint8_t* smem, uint32_t ncols,
                                              uint32_t buf, uint32_t R, const StreamState& snap_def,
                                              const StreamState& snap_val, const DeltaState& snap_dl) {
  uint32_t mycol;
  const bool walker = walker_of(ncols, mycol);
  const uint32_t tid = threadIdx.x;
  for (int attempt = 0; attempt < 4 && R > 0; attempt++) {
    if (walker) {  // definition levels
      ColCursor& c = ctl.cur[mycol];
      SlabCol& s = ctl.slab[buf][mycol];
      uint32_t got = R;
      s.ndef = 0;
      s.all_valid = 1;
      if (c.present && c.has_def) {
        Window w{smem + L.defwin[mycol][buf], c.defwin_base[buf], L.defwin_cap[mycol]};
        DirEntry* dir = smem_at<DirEntry>(smem, L.defdir[mycol]);
        uint32_t n = 0;
        got = walk_stream(c.def, w, R, dir, n, kMaxDirEntries);
        s.ndef = n;
        uint32_t allv = 1;
        for (uint32_t e = 0; e < n; e++) allv &= (dir[e].kind == 0 && (dir[e].payload & 1)) ? 1u : 0u;
        s.all_valid = allv;
      }
      ctl.rmin[mycol] = got;
    }
    for (uint32_t c = 0; c < ncols; c++) {
      uint32_t* bm = smem_at<uint32_t>(smem, L.valid[c]);
      for (uint32_t w = tid; w < (uint32_t)kSlabWords + 2; w += kScanThreads) bm[w] = 0;
    }
    __syncthreads();
    uint32_t R1 = R;
    for (uint32_t c = 0; c < ncols; c++) R1 = ctl.rmin[c] < R1 ? ctl.rmin[c] : R1;
    if (R1 < R) {  // a definition-level window / directory ran out: shrink the slab, redo
      if (walker) ctl.cur[mycol].def = snap_def;
      R = R1;
      __syncthreads();
      continue;
    }
    for (uint32_t c = 0; c < ncols; c++) {
      const SlabCol& s = ctl.slab[buf][c];
      if (s.present && !s.all_valid)
        dir_to_bitmap(smem_at<DirEntry>(smem, L.defdir[c]), s.ndef, smem_at<uint32_t>(smem, L.defwin[c][buf]),
                      smem_at<uint32_t>(smem, L.valid[c]));
    }
    __syncthreads();
    for (uint32_t c = warp_id(); c < ncols; c += kScanWarps) {
      SlabCol& s = ctl.slab[buf][c];
      if (!s.present) { if (lane_id() == 0) s.nv = 0; continue; }
      if (s.all_valid) { if (lane_id() == 0) s.nv = R; continue; }
      uint32_t* bm = smem_at<uint32_t>(smem, L.valid[c]);
      uint32_t* rk = smem_at<uint32_t>(smem, L.rank[c]);
      uint32_t w0 = lane_id() * 2, w1 = w0 + 1;
      uint32_t a0 = bm[w0] & row_mask(w0, R), a1 = bm[w1] & row_mask(w1, R);
      uint32_t p0 = __popc(a0), p1 = __popc(a1);
      uint32_t sum = p0 + p1, incl = sum;
      for (int o = 1; o < 32; o <<= 1) {
        uint32_t t = __shfl_up_sync(0xffffffffu, incl, o);
        if ((int)lane_id() >= o) incl += t;
      }
      uint32_t excl = incl - sum;
      rk[w0] = excl;
      rk[w1] = excl + p0;
      bm[w0] = a0;
      bm[w1] = a1;
      if (lane_id() == 31) s.nv = incl;
    }
    __syncthreads();
    if (walker) {  // dictionary-index streams
      ColCursor& c = ctl.cur[mycol];
      SlabCol& s = ctl.slab[buf][mycol];
      uint32_t rc = R;
      s.nval = 0;
      if (c.present && PQB_ENC_HAS_WINDOW(c.enc) && s.nv > 0) {
        Window w{smem + L.valwin[mycol][buf], c.valwin_base[buf], L.valwin_cap[mycol]};
        uint32_t n = 0;
        uint32_t got = c.enc == DE_DELTA
                           ? walk_delta(c.dl, w, s.nv, smem_at<DeltaEntry>(smem, L.valdir[mycol][buf]), n, kMaxDeltaEntries)
                           : walk_stream(c.val, w, s.nv, smem_at<DirEntry>(smem, L.valdir[mycol][buf]), n, kMaxDirEntries - 2);
        s.nval = n;
        if (c.enc != DE_DELTA) dir_sentinels(smem_at<DirEntry>(smem, L.valdir[mycol][buf]), n);
        if (got < s.nv) {  // rows [0, rc) hold exactly `got` non-null values
          if (s.all_valid) rc = got;
          else {
            const uint32_t* bm = smem_at<uint32_t>(smem, L.valid[mycol]);
            uint32_t seen = 0;
            rc = 0;
            for (uint32_t r = 0; r < R; r++) {
              uint32_t b = (bm[r >> 5] >> (r & 31)) & 1;
              if (b && seen == got) break;
              seen += b;
              rc = r + 1;
            }
          }
        }
      }
      ctl.rmin[mycol] = rc;
    }
    __syncthreads();
    uint32_t R2 = R;
    for (uint32_t c = 0; c < ncols; c++) R2 = ctl.rmin[c] < R2 ? ctl.rmin[c] : R2;
    if (R2 < R) {  // an index window / directory ran out: shrink and redo everything
      if (walker) { ctl.cur[mycol].def = snap_def; ctl.cur[mycol].val = snap_val; ctl.cur[mycol].dl = snap_dl; }
      R = R2;
      __syncthreads();
      continue;
    }
    return R;
  }
  return 0;
}

// cache this row group's leaf LUTs (one byte per dictionary entry) in shared memory (fast AND pass)
__device__ __forceinline__ void fill_lut_cache(const DevPlan& plan, ScanCtl& ctl, const SmemLayout& L, uint8_t* smem,
                                               const DevScanArgs& a, uint32_t rg) {
  if (!plan.fast_and) return;
  for (uint32_t l = 0; l < plan.nleaves; l++) {
    const DevLeaf& lf = plan.leaves[l];
    const DevChunk ch = a.chunks[rg * plan.ncols + lf.col];
    const bool fits = ch.present && ch.dict_n <= (uint32_t)kLutCacheBytes;
    if (threadIdx.x == 0) ctl.lut_smem[l] = fits;
    if (fits) {
      const uint8_t* src = a.luts + lf.lut_off + ch.lut_base;
      uint8_t* dst = smem + L.lutc + l * kLutCacheBytes;
      for (uint32_t i = threadIdx.x; i < ch.dict_n; i += kScanThreads) dst[i] = src[i];
    }
  }
}

// ---- the row phase of one slab: DELTA decode, then the row pass the slab qualifies for; adds the
// selected rows to ctl.sel_count.  All threads of the CTA call it. ----
__device__ __forceinline__ void row_phase(const DevPlan& plan, ScanCtl& ctl, const SmemLayout& L, uint8_t* smem, const DevScanArgs& a,
                                          const DevItem& item, uint32_t mode, uint32_t has_delta, uint32_t buf, uint32_t R,
                                          uint32_t r_item, unsigned long long* acc, bool agg_mode) {
  const uint32_t tid = threadIdx.x;
  const uint32_t ncols = plan.ncols;
  const uint32_t nslots = plan.nslots;
  uint32_t* selw = smem_at<uint32_t>(smem, L.sel);
  uint32_t* leafT = smem_at<uint32_t>(smem, L.leafT);
  // ---- 3b. DELTA_BINARY_PACKED columns: deltas + block scan into their staging array ----
  if (has_delta)
    for (uint32_t c = 0; c < ncols; c++)
      if (ctl.slab[buf][c].present && ctl.slab[buf][c].enc == DE_DELTA && ctl.slab[buf][c].nv) delta_decode_scan(ctl, L, smem, c, buf);
  const uint32_t nwords = (R + 31) >> 5;
  uint32_t cnt = 0;
  const bool fast_and = mode == MODE_FAST_AND;
  if (fast_and) {
    // ---- 4-6 (specialised): conjunction of dictionary-LUT leaves, registers only ----
    cnt = fast_and_rows(plan, ctl, L, smem, a, item, buf, R, r_item, acc, agg_mode);
  } else if (mode == MODE_ROW_MAJOR) {
    // ---- 4-6 (row-major variant): one warp per 32-row word, registers only ----
    cnt = fast_rows(plan, ctl, L, smem, a, item, buf, R, r_item, acc, agg_mode);
  } else {
  // ---- 4. (general) unpack: fused index -> leaf bits where possible, else stage indices ----
  for (uint32_t w = tid; w < plan.nleaves * kLeafWords; w += kScanThreads) leafT[w] = 0;
  __syncthreads();
  for (uint32_t c = 0; c < ncols; c++) {
    const SlabCol& s = ctl.slab[buf][c];
    if (!s.present || !PQB_ENC_HAS_STREAM(s.enc) || s.nv == 0) continue;
    uint32_t* idx = L.idx[c] ? smem_at<uint32_t>(smem, L.idx[c]) : nullptr;
    const DirEntry* dir = smem_at<DirEntry>(smem, L.valdir[c][buf]);
    const uint32_t* win = smem_at<uint32_t>(smem, L.valwin[c][buf]);
    // leaves of this column that a dictionary LUT answers (host precomputed lists)
    const uint32_t nlut = plan.col_nlut[c];
    if (s.enc == DE_DICT && s.all_valid && nlut >= 1 && nlut <= 2) {
      const int l0 = plan.col_l0[c], l1 = plan.col_l1[c];
      const uint8_t* lut0 = a.luts + plan.leaves[l0].lut_off + s.lut_base;
      uint32_t* i_st = plan.cols[c].need_idx ? idx : nullptr;
      if (nlut == 2)
        dir_to_leafbits<true>(dir, s.nval, win, s.bw, lut0, leafT + l0 * kLeafWords,
                              a.luts + plan.leaves[l1].lut_off + s.lut_base, leafT + l1 * kLeafWords, i_st);
      else
        dir_to_leafbits<false>(dir, s.nval, win, s.bw, lut0, leafT + l0 * kLeafWords, nullptr, nullptr, i_st);
    } else if (idx) {
      dir_to_idx(dir, s.nval, win, s.bw, idx);
    }
  }
  __syncthreads();

  // ---- 5. leaves the fused pass did not answer: PLAIN pages, NULL-carrying slabs, booleans ----
  for (uint32_t l = 0; l < plan.nleaves; l++) {
    const DevLeaf& lf = plan.leaves[l];
    if (!value_leaf(lf.kind)) continue;   // IS [NOT] NULL comes from the validity words
    const SlabCol& s = ctl.slab[buf][lf.col];
    if (!s.present) continue;                                 // all NULL: T stays 0
    if (s.enc == DE_DICT && s.all_valid && plan.col_nlut[lf.col] <= 2) continue;  // answered by the fused pass
    const uint32_t* vbm = smem_at<uint32_t>(smem, L.valid[lf.col]);
    const uint32_t* rk = smem_at<uint32_t>(smem, L.rank[lf.col]);
    const uint32_t* idx = smem_at<uint32_t>(smem, L.idx[lf.col]);
    uint32_t* Tw = leafT + l * kLeafWords;
    const uint8_t kind = plan.cols[lf.col].kind;
    const uint8_t* lut = a.luts + lf.lut_off + s.lut_base;
    const int64_t lit = lf.lit_i64;
    const int64_t litk = f64_order_key((uint64_t)lf.lit_i64);
    const uint32_t op = lf.cmp;
    for (uint32_t r0 = warp_id() * 32; r0 < R; r0 += kScanThreads) {
      uint32_t r = r0 + lane_id();
      bool t = false;
      if (r < R) {
        RowVal rv = row_rank(s, vbm, rk, r);
        if (rv.valid) {
          if (s.enc == DE_DICT) t = lut[idx[rv.j]] != 0;
          else if (kind == DK_BOOL) t = cmp_i64((int64_t)value_bool(s, a.arena, idx, rv.j), lit, op);
          else if (kind == DK_I64) t = cmp_i64((int64_t)value_u64(s, a.arena, idx, rv.j), lit, op);
          else if (kind == DK_F64) t = cmp_i64(f64_order_key(value_u64(s, a.arena, idx, rv.j)), litk, op);
        }
      }
      uint32_t tw = __ballot_sync(0xffffffffu, t);
      if (lane_id() == 0) Tw[r0 >> 5] = tw;
    }
  }
  __syncthreads();

  // ---- 6. Kleene combine on words -> selection; filter mode consumes right here ----
  for (uint32_t w = tid; w < nwords; w += kScanThreads) {
    uint32_t st_t[kPredStack], st_n[kPredStack];
    int sp = 0;
    const uint32_t rm = row_mask(w, R);
#pragma unroll 1
    for (uint32_t i = 0; i < plan.npred; i++) {
      const DevPredOp op = plan.pred[i];
      if (op.kind == PK_LEAF) {
        const DevLeaf& lf = plan.leaves[op.arg];
        const SlabCol& s = ctl.slab[buf][lf.col];
        uint32_t V = !s.present ? 0u : (s.all_valid ? 0xffffffffu : smem_at<uint32_t>(smem, L.valid[lf.col])[w]);
        uint32_t t, n;
        if (lf.kind == LK_IS_NULL) { t = ~V; n = 0; }
        else if (lf.kind == LK_IS_NOT_NULL) { t = V; n = 0; }
        else { t = leafT[op.arg * kLeafWords + w] & V; n = ~V; }
        st_t[sp] = t;
        st_n[sp] = n;
        sp++;
      } else if (op.kind == PK_CONST) {
        st_t[sp] = op.arg == 1 ? 0xffffffffu : 0u;
        st_n[sp] = op.arg == 2 ? 0xffffffffu : 0u;
        sp++;
      } else if (op.kind == PK_NOT) {
        st_t[sp - 1] = ~(st_t[sp - 1] | st_n[sp - 1]);
      } else {
        uint32_t tb = st_t[sp - 1], nb = st_n[sp - 1], ta = st_t[sp - 2], na = st_n[sp - 2];
        sp--;
        if (op.kind == PK_AND) {
          uint32_t fa = ~(ta | na), fb = ~(tb | nb);
          st_t[sp - 1] = ta & tb;
          st_n[sp - 1] = (na | nb) & ~fa & ~fb;
        } else {
          uint32_t t = ta | tb;
          st_t[sp - 1] = t;
          st_n[sp - 1] = (na | nb) & ~t;
        }
      }
    }
    uint32_t sel = (plan.npred ? st_t[0] : 0xffffffffu) & rm;
    if (agg_mode) selw[w] = sel;
    else {
      cnt += __popc(sel);
      if (plan.write_bitmap && sel) {
        uint32_t pos = r_item + w * 32;
        uint32_t* dst = a.bitmap + item.bitmap_word0 + (pos >> 5);
        uint32_t sh = pos & 31;
        if (sh == 0) *dst = sel;  // slabs are word aligned except after a pathological shrink
        else {
          atomicOr(dst, sel << sh);
          uint32_t hi = sel >> (32 - sh);
          if (hi) atomicOr(dst + 1, hi);
        }
      }
    }
  }
  if (agg_mode) {
    __syncthreads();
    for (uint32_t r = tid; r < R; r += kScanThreads) {
      if (!((selw[r >> 5] >> (r & 31)) & 1)) continue;
      cnt++;
      uint32_t slot = 0;
      for (uint32_t k = 0; k < plan.nkeys; k++) {
        const DevKey& key = plan.keys[k];
        const SlabCol& s = ctl.slab[buf][key.col];
        RowVal rv = row_rank(s, smem_at<uint32_t>(smem, L.valid[key.col]), smem_at<uint32_t>(smem, L.rank[key.col]), r);
        uint32_t gid = key.card;  // NULL is its own group (field_stats.rs:1009-1037)
        if (rv.valid) {
          if (key.kind == KK_BOOL) gid = value_bool(s, a.arena, smem_at<uint32_t>(smem, L.idx[key.col]), rv.j);
          else gid = key.gid[s.lut_base + smem_at<uint32_t>(smem, L.idx[key.col])[rv.j]];
        }
        slot += gid * key.stride;
      }
      acc_add(&acc[slot], 1ull);
      for (uint32_t g = 0; g < plan.naggs; g++) {
        const DevAgg& ag = plan.aggs[g];
        if (ag.fn == AG_COUNT_STAR) continue;
        const SlabCol& s = ctl.slab[buf][ag.col];
        RowVal rv = row_rank(s, smem_at<uint32_t>(smem, L.valid[ag.col]), smem_at<uint32_t>(smem, L.rank[ag.col]), r);
        if (!rv.valid) continue;
        if (ag.update_nn) acc_add(&acc[(1 + plan.n_acc + ag.nn_slot) * nslots + slot], 1ull);
        if (ag.fn == AG_COUNT) continue;
        uint64_t bits = ag.kind == DK_BOOL ? value_bool(s, a.arena, smem_at<uint32_t>(smem, L.idx[ag.col]), rv.j)
                                           : value_u64(s, a.arena, smem_at<uint32_t>(smem, L.idx[ag.col]), rv.j);
        acc_apply(&acc[(1 + ag.acc_slot) * nslots + slot], ag.fn, ag.kind, bits);
      }
    }
  }
  }  // general row phase
  for (int o = 16; o; o >>= 1) cnt += __shfl_xor_sync(0xffffffffu, cnt, o);
  if (lane_id() == 0 && cnt) atomicAdd(&ctl.sel_count, cnt);

}

__global__ void __launch_bounds__(kScanThreads, PQB_SCAN_MIN_BLOCKS)
k_scan(const __grid_constant__ DevPlan plan, const __grid_constant__ SmemLayout L, const DevScanArgs a) {
  extern __shared__ __align__(128) uint8_t smem[];
  ScanCtl& ctl = *reinterpret_cast<ScanCtl*>(smem);
  const uint32_t tid = threadIdx.x;
  const uint32_t ncols = plan.ncols;
  const uint32_t cells = 1 + plan.n_acc + plan.n_nn;
  const bool agg_mode = plan.mode == SM_AGG;
  uint32_t mycol;
  const bool walker = walker_of(ncols, mycol);

  if (tid == 0) {
    mbar_init(&ctl.mbar[0], 1);
    mbar_init(&ctl.mbar[1], 1);
    mbar_fence_init();
    ctl.error = 0;
  }
  unsigned long long* sacc = smem_at<unsigned long long>(smem, L.acc);
  if (agg_mode && plan.smem_acc) {
    for (uint32_t i = tid; i < cells * plan.nslots; i += kScanThreads) {
      uint32_t arr = i / plan.nslots;
      unsigned long long init = 0;
      if (arr >= 1 && arr < 1 + plan.n_acc) {
        uint8_t k = plan.acc_init[arr - 1];
        init = k == 2 ? 0x7fffffffffffffffull : (k == 3 ? 0x8000000000000000ull : 0ull);
      }
      sacc[i] = init;
    }
  }
  __syncthreads();
  unsigned long long* acc = (agg_mode && plan.smem_acc) ? sacc : a.acc;
  const uint32_t nslots = plan.nslots;

  uint32_t phases = 0;   // bit b: parity to wait for on mbar[b]

  for (;;) {
    __syncthreads();
    if (tid == 0) ctl.item = (uint32_t)atomicAdd(&a.counters[2], 1ull);
    __syncthreads();
    const uint32_t item_id = ctl.item;
    if (item_id >= plan.n_items) break;
    const DevItem& item = a.items[item_id];
    if ((item.fast & kItemFlat) && !plan.no_flat) continue;   // the flat kernels own this item
    if (a.rg_live && !a.rg_live[item.rg]) continue;            // row group pruned by statistics (counts stay 0)

    if (tid < ncols) {
      ColCursor& c = ctl.cur[tid];
      const DevChunk ch = a.chunks[item.rg * ncols + tid];
      for (uint32_t b = 0; b < 2; b++) {
        SlabCol& s = ctl.slab[b][tid];
        s.lut_base = ch.lut_base;
        s.dict_off = ch.dict_off;
        s.present = ch.present;
      }
      c.present = ch.present;
      c.page_end = ch.first_page + ch.n_pages;
      if (ch.present) page_enter(c, a.pages, item.page[tid]);
      else { c.page_rows_left = 0xffffffffu; c.enc = DE_PLAIN; c.has_def = 0; c.vals_done = 0; }
    }
    if (tid == 0) ctl.sel_count = 0;
    fill_lut_cache(plan, ctl, L, smem, a, item.rg);
    __syncthreads();

    uint32_t rows_left = item.nrows;
    uint32_t r_item = 0;
    uint32_t buf = 0;
    if (tid == 0) issue_windows(ctl, L, smem, a.arena, ncols, buf, rows_left);
    __syncthreads();

    while (rows_left > 0) {
      // ---- 1-3. control, WARP 0 ONLY (the other warps park at the barrier and spend no issue
      //      slots): wait for the staged bytes, walk the run headers (one lane per column),
      //      commit the cursors, prefetch the next slab, choose the row pass ----
      StreamState snap_def, snap_val;
      DeltaState snap_dl;
      if (warp_id() == 0) {
        if (lane_id() == 0) mbar_wait(&ctl.mbar[buf], (phases >> buf) & 1u);
        __syncwarp();
        const uint32_t R0w = ctl.target;
        if (walker) {
          ColCursor& c = ctl.cur[mycol];
          SlabCol& s = ctl.slab[buf][mycol];
          snap_def = c.def;
          snap_val = c.val;
          snap_dl = c.dl;
          uint32_t rc = R0w;
          s.ndef = 0;
          s.nval = 0;
          s.all_valid = 1;
          s.nv = c.present ? R0w : 0;
          if (c.present) {
            if (c.has_def) {
              Window w{smem + L.defwin[mycol][buf], c.defwin_base[buf], L.defwin_cap[mycol]};
              DirEntry* dir = smem_at<DirEntry>(smem, L.defdir[mycol]);
              uint32_t n = 0;
              uint32_t got = walk_stream(c.def, w, R0w, dir, n, kMaxDirEntries);
              s.ndef = n;
              uint32_t allv = 1;
              for (uint32_t e = 0; e < n; e++) allv &= (dir[e].kind == 0 && (dir[e].payload & 1)) ? 1u : 0u;
              s.all_valid = allv;
              rc = got;
              if (!allv) ctl.any_nulls = 1;
            }
            if (s.all_valid && rc == R0w && PQB_ENC_HAS_WINDOW(c.enc)) {
              Window w{smem + L.valwin[mycol][buf], c.valwin_base[buf], L.valwin_cap[mycol]};
              uint32_t n = 0;
              rc = c.enc == DE_DELTA
                       ? walk_delta(c.dl, w, R0w, smem_at<DeltaEntry>(smem, L.valdir[mycol][buf]), n, kMaxDeltaEntries)
                       : walk_stream(c.val, w, R0w, smem_at<DirEntry>(smem, L.valdir[mycol][buf]), n, kMaxDirEntries - 2);
              s.nval = n;
              if (c.enc != DE_DELTA) dir_sentinels(smem_at<DirEntry>(smem, L.valdir[mycol][buf]), n);
            }
          }
          if (rc < R0w) atomicMin(&ctl.rmin_all, rc);
        }
        __syncwarp();
        const bool general = ctl.rmin_all < R0w || ctl.any_nulls;
        if (!general) {
          if (walker) {  // freeze this slab's view, advance the cursor
            ColCursor& c = ctl.cur[mycol];
            SlabCol& s = ctl.slab[buf][mycol];
            s.val_base = c.val_base;
            s.vals_done = c.vals_done;
            s.enc = c.enc;
            s.bw = c.val.bw;
            if (c.present) {
              c.vals_done += s.nv;
              c.page_rows_left -= R0w;
              if (c.page_rows_left == 0 && rows_left > R0w) {
                if (c.page + 1 < c.page_end) page_enter(c, a.pages, c.page + 1);
                else { ctl.error = 1; atomicExch(&a.counters[1], 2ull); }
              }
            }
          }
          __syncwarp();
          if (lane_id() == 0) {
            uint32_t mode = MODE_GENERIC, has_delta = 0;
            bool fa = plan.fast_and != 0;
            for (uint32_t c = 0; c < ncols; c++) has_delta |= ctl.slab[buf][c].present && ctl.slab[buf][c].enc == DE_DELTA && ctl.slab[buf][c].nv;
            for (uint32_t l = 0; fa && l < plan.nleaves; l++) {
              const SlabCol& s = ctl.slab[buf][plan.leaves[l].col];
              fa = s.present && s.enc == DE_DICT && s.nval > 0;
            }
            if (fa) mode = MODE_FAST_AND;
            else if (plan.row_major) mode = MODE_ROW_MAJOR;
            ctl.mode = mode;
            ctl.has_delta = has_delta;
            ctl.R = R0w;
            if (!ctl.error && rows_left > R0w) issue_windows(ctl, L, smem, a.arena, ncols, buf ^ 1, rows_left - R0w);
          }
        } else if (lane_id() == 0) {
          ctl.mode = MODE_GENERAL_WALK;
          ctl.R = R0w;
        }
      }
      phases ^= 1u << buf;
      __syncthreads();
      uint32_t mode = ctl.mode;
      uint32_t R = ctl.R;
      bool has_nulls = false;
      uint32_t has_delta = ctl.has_delta;
      if (mode == MODE_GENERAL_WALK) {  // uniform: NULLs or an exhausted window -> the general walk, all threads
        if (walker) { ctl.cur[mycol].def = snap_def; ctl.cur[mycol].val = snap_val; ctl.cur[mycol].dl = snap_dl; }
        __syncthreads();
        R = general_walk(ctl, L, smem, ncols, buf, R, snap_def, snap_val, snap_dl);
        if (R == 0) {  // no progress possible: corrupt page
          if (tid == 0) { ctl.error = 1; atomicExch(&a.counters[1], 1ull); }
          break;
        }
        if (walker) {
          ColCursor& c = ctl.cur[mycol];
          SlabCol& s = ctl.slab[buf][mycol];
          s.val_base = c.val_base;
          s.vals_done = c.vals_done;
          s.enc = c.enc;
          s.bw = c.val.bw;
          if (c.present) {
            c.vals_done += s.nv;
            c.page_rows_left -= R;
            if (c.page_rows_left == 0 && rows_left > R) {
              if (c.page + 1 < c.page_end) page_enter(c, a.pages, c.page + 1);
              else { ctl.error = 1; atomicExch(&a.counters[1], 2ull); }
            }
          }
        }
        __syncthreads();
        if (!ctl.error && tid == 0 && rows_left > R) issue_windows(ctl, L, smem, a.arena, ncols, buf ^ 1, rows_left - R);
        has_delta = 0;
        for (uint32_t c = 0; c < ncols; c++) {
          has_nulls |= ctl.slab[buf][c].present && !ctl.slab[buf][c].all_valid;
          has_delta |= ctl.slab[buf][c].present && ctl.slab[buf][c].enc == DE_DELTA && ctl.slab[buf][c].nv;
        }
        mode = MODE_GENERIC;
        if (!has_nulls) {
          bool fa = plan.fast_and != 0;
          for (uint32_t l = 0; fa && l < plan.nleaves; l++) {
            const SlabCol& s = ctl.slab[buf][plan.leaves[l].col];
            fa = s.present && s.enc == DE_DICT && s.nval > 0;
          }
          if (fa) mode = MODE_FAST_AND;
          else if (plan.row_major) mode = MODE_ROW_MAJOR;
        }
      }
      if (ctl.error) break;

      row_phase(plan, ctl, L, smem, a, item, mode, has_delta, buf, R, r_item, acc, agg_mode);

      rows_left -= R;
      r_item += R;
      buf ^= 1;
      __syncthreads();
    }  // slabs
    __syncthreads();
    if (ctl.error) break;
    if (tid == 0) {
      if (a.item_counts) a.item_counts[item_id] = ctl.sel_count;
      if (ctl.sel_count) atomicAdd(&a.counters[0], (unsigned long long)ctl.sel_count);
    }
  }  // items

  // ---- flush the CTA-private accumulator table ----
  __syncthreads();
  if (agg_mode && plan.smem_acc && !ctl.error) {
    for (uint32_t slot = tid; slot < nslots; slot += kScanThreads) {
      unsigned long long rows = sacc[slot];
      if (rows == 0) continue;
      atomicAdd(&a.acc[slot], rows);
      for (uint32_t arr = 0; arr < plan.n_acc; arr++)
        acc_merge(&a.acc[(1 + arr) * nslots + slot], plan.acc_init[arr], sacc[(1 + arr) * nslots + slot]);
      for (uint32_t k = 0; k < plan.n_nn; k++) {
        unsigned long long v = sacc[(1 + plan.n_acc + k) * nslots + slot];
        if (v) atomicAdd(&a.acc[(1 + plan.n_acc + k) * nslots + slot], v);
      }
    }
  }
}

}  // namespace pqb
