// ORDER BY [... LIMIT n] on the device, over the groups of an aggregate query or the selected rows of a scan.  The
// aggregate result path lists the non-empty group slots in ascending slot order (out_slot, k_slot_compact); ordering
// permutes and cuts that list before k_agg_finish assembles the rows, so the batches, the Arrow stream and the JSON
// egress follow the new order unchanged.  A scan orders the positions of its selected rows and k_project_rows gathers
// the kept ones into the projection's result block.
//
//   k_order_encode   one thread per group: every term's order-preserving u64 (order_keys.cuh) + NULL flag, and the
//                    value range of every term (one small D2H: the pack plan is sized from it)
//   k_order_rows_encode
//                    the same for every selected row of a scan (a CTA per work item, positions as k_project finds
//                    them), plus the row's handle (item, row inside the item)
//   k_order_pack     the terms packed MSB-first into the fewest 64-bit words their ranges need
//   k_order_cta      rows <= kOrderCta: one CTA sorts (word 0, row) pairs in shared memory (bitonic, the row index as the
//                    last key: stable), then writes the kept slots
//   k_topk_hist / k_topk_pick / k_topk_tile_eq / k_item_prefix / k_topk_compact, then k_order_cta
//                    one packed word and LIMIT <= kOrderCta over more rows: radix select of the LIMIT-th key T, MSB
//                    digit first over the used bits, each digit's histogram over the rows that still match the prefix
//                    and the digit picked on the device; then the rows below T and, in row order, the first rows equal
//                    to T (exactly LIMIT candidates) are sorted by the one-CTA sort
//   k_radix_hist / k_item_prefix / k_radix_scatter
//                    anything larger: LSD radix sort of the row indices, 8-bit digits over the used bits of each word
//                    from the least significant word up; per pass tile histograms, one scan of the digit x tile matrix
//                    and a stable scatter (in-tile ranks from a __match_any_sync multisplit)
//   k_order_gather   the first `keep` rows' slots in the new order (no slot list: the row indices themselves)
// Rows equal on every term keep their slot order, or for a scan their selection order (the row index breaks every tie),
// so the ordered result is a stable sort of the unordered one.
#pragma once
#include <cuda_runtime.h>

#include "../../include/parseable_b200.h"
#include "egress_kernels.cuh"
#include "order_keys.cuh"

namespace pqb {

enum OrderSource : uint8_t { OS_VALUE = 0, OS_RANK = 1, OS_GID = 2 };   // key terms: 8-byte dictionary value | rank[gid] | gid

struct OrderTerm {
  uint8_t target;       // PQ_ORDER_KEY / PQ_ORDER_AGG
  uint8_t enc;          // OrderEnc
  uint8_t desc;
  uint8_t source;       // key terms: OrderSource
  uint8_t nn_is_rows;   // aggregate terms: as FinishArgs.nn_is_rows
  uint8_t _pad[3];
  uint32_t card;        // key terms: NULL is gid == card
  uint64_t wstride;
  const uint32_t* kd_offs;
  const uint8_t* kd_bytes;
  const uint32_t* rank;
  DevAgg agg;
};
struct OrderArgs {
  const unsigned long long* acc;
  const unsigned long long* wide;
  const uint32_t* out_slot;
  uint32_t n, nslots, n_acc, nterms;
  unsigned long long* vals;   // [nterms][n] encoded values
  uint8_t* nulls;             // [nterms][n]
  OrderRange* ranges;         // [nterms], min = ~0 / max = 0 / flags 0 on entry
  OrderTerm t[kMaxOrder];
};

constexpr int kRadixThreads = 256;
constexpr int kRadixItems = 8;
constexpr uint32_t kRadixTile = kRadixThreads * kRadixItems;

__global__ void __launch_bounds__(256) k_order_encode(const __grid_constant__ OrderArgs o) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  const bool live = i < o.n;
  const uint32_t slot = live ? o.out_slot[i] : 0u;
  const unsigned long long rows = live ? o.acc[slot] : 0ull;
  for (uint32_t t = 0; t < o.nterms; t++) {
    const OrderTerm& ot = o.t[t];
    bool valid = false;
    unsigned long long bits = 0;
    if (live) {
      if (ot.target == PQ_ORDER_AGG) {
        bits = agg_output_value(o.acc, o.nslots, o.n_acc, ot.agg, ot.nn_is_rows, slot, rows, valid);
      } else {
        const uint32_t gid = key_gid_of_slot(o.wide, slot, ot.wstride, ot.card);
        valid = gid != ot.card;
        if (valid) {
          if (ot.source == OS_RANK) bits = ot.rank[gid];
          else if (ot.source == OS_GID) bits = gid;
          else {
            const uint8_t* p = ot.kd_bytes + ot.kd_offs[gid];
            for (int b = 0; b < 8; b++) bits |= (unsigned long long)p[b] << (8 * b);
          }
        }
      }
    }
    const unsigned long long v = order_encode(bits, ot.enc, ot.desc != 0);
    if (live) {
      o.vals[size_t(t) * o.n + i] = v;
      o.nulls[size_t(t) * o.n + i] = valid ? 0 : 1;
    }
    unsigned long long mn = (live && valid) ? v : ~0ull, mx = (live && valid) ? v : 0ull;
    for (int s = 16; s > 0; s >>= 1) {
      mn = min(mn, __shfl_xor_sync(0xffffffffu, mn, s));
      mx = max(mx, __shfl_xor_sync(0xffffffffu, mx, s));
    }
    const bool any_null = __any_sync(0xffffffffu, live && !valid), any_value = __any_sync(0xffffffffu, live && valid);
    if ((threadIdx.x & 31) == 0) {
      if (any_value) {
        atomicMin(&o.ranges[t].min, mn);
        atomicMax(&o.ranges[t].max, mx);
        atomicOr(&o.ranges[t].has_value, 1u);
      }
      if (any_null) atomicOr(&o.ranges[t].has_null, 1u);
    }
  }
}

// ---- scans: the terms are columns, read for the selected rows only ----
struct RowOrderTerm {
  uint32_t slot;          // column slot of the plan
  uint8_t kind;           // DevKind
  uint8_t enc;            // OrderEnc
  uint8_t desc;
  uint8_t _pad;
  const uint32_t* gid;    // Utf8: the column's GROUP BY id of every dictionary entry (the per-row ids come as FK_IDS pages)
  const uint32_t* rank;   // Utf8: bytewise rank of every id
};
struct RowOrderArgs {
  const uint8_t* arena;
  const uint8_t* flat;
  const FlatPageRec* fpages;   // the table's flat pages; Utf8 term pages without a dictionary as FK_IDS pages
  const DevChunk* chunks;
  const DevItem* items;
  const uint32_t* bitmap;
  const uint32_t* item_counts;
  const unsigned long long* item_base;
  uint32_t n_items, plan_ncols, n, nterms;   // n: selected rows
  unsigned long long* vals;    // [nterms][n] encoded values
  uint8_t* nulls;              // [nterms][n]
  OrderRange* ranges;          // [nterms], min = ~0 / max = 0 / flags 0 on entry
  unsigned long long* handles; // [n]: item index << 32 | row inside the item
  RowOrderTerm t[kMaxOrder];
};

__global__ void __launch_bounds__(256) k_order_rows_encode(const __grid_constant__ RowOrderArgs o) {
  unsigned long long mn[kMaxOrder], mx[kMaxOrder];   // this thread's value range per term (registers: indexed by constants only)
  uint32_t met_null = 0, met_value = 0;              // bit t: term t met a NULL / a value
#pragma unroll
  for (int k = 0; k < kMaxOrder; k++) { mn[k] = ~0ull; mx[k] = 0ull; }
  for_each_selected(o.items, o.bitmap, o.item_counts, o.item_base, o.n_items,
                    [&](const DevItem& item, uint32_t it, uint32_t r, unsigned long long pos) {
    o.handles[pos] = (unsigned long long)it << 32 | r;
    for (uint32_t t = 0; t < o.nterms; t++) {
      const RowOrderTerm& ot = o.t[t];
      unsigned long long bits = 0;
      uint32_t len = 0;
      const bool valid = flat_value_at<true>(o.arena, o.flat, o.fpages, o.chunks, o.plan_ncols, item, ot.slot, ot.kind, nullptr, ot.gid, r,
                                             bits, len);
      if (valid && ot.rank) bits = ot.rank[bits];
      const unsigned long long v = order_encode(bits, ot.enc, ot.desc != 0);
      o.vals[size_t(t) * o.n + pos] = v;
      o.nulls[size_t(t) * o.n + pos] = valid ? 0 : 1;
      if (valid) {
        met_value |= 1u << t;
#pragma unroll
        for (int k = 0; k < kMaxOrder; k++)
          if (k == int(t)) { mn[k] = min(mn[k], v); mx[k] = max(mx[k], v); }
      } else {
        met_null |= 1u << t;
      }
    }
  });
  // one warp reduction per term, one set of atomics per warp
#pragma unroll
  for (int k = 0; k < kMaxOrder; k++) {
    if (k >= int(o.nterms)) break;
    unsigned long long a = mn[k], b = mx[k];
    for (int s = 16; s > 0; s >>= 1) {
      a = min(a, __shfl_xor_sync(0xffffffffu, a, s));
      b = max(b, __shfl_xor_sync(0xffffffffu, b, s));
    }
    const bool any_value = __any_sync(0xffffffffu, (met_value >> k) & 1u), any_null = __any_sync(0xffffffffu, (met_null >> k) & 1u);
    if ((threadIdx.x & 31) == 0) {
      if (any_value) {
        atomicMin(&o.ranges[k].min, a);
        atomicMax(&o.ranges[k].max, b);
        atomicOr(&o.ranges[k].has_value, 1u);
      }
      if (any_null) atomicOr(&o.ranges[k].has_null, 1u);
    }
  }
}

// words[w][n]: the packed key of every row
__global__ void __launch_bounds__(256) k_order_pack(const __grid_constant__ OrderPack p, const unsigned long long* __restrict__ vals,
                                                    const uint8_t* __restrict__ nulls, uint32_t n, unsigned long long* __restrict__ words) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  uint64_t v[kMaxOrder];
  uint8_t nl[kMaxOrder];
  for (uint32_t t = 0; t < p.nterms; t++) { v[t] = vals[size_t(t) * n + i]; nl[t] = nulls[size_t(t) * n + i]; }
  uint64_t w[kMaxOrderWords];
  for (int k = 0; k < kMaxOrderWords; k++) w[k] = 0;
  order_pack_row(p, v, nl, w);
  for (uint32_t k = 0; k < p.nwords; k++) words[size_t(k) * n + i] = w[k];
}

// row a before row b?  Word 0 is given, the other words are read from the packed keys; padding (row ~0u) goes last.
__device__ __forceinline__ bool order_row_less(const unsigned long long* __restrict__ words, uint32_t n, uint32_t nwords,
                                               unsigned long long ka, uint32_t a, unsigned long long kb, uint32_t b) {
  if (ka != kb) return ka < kb;
  if (a == ~0u || b == ~0u) return a < b;
  for (uint32_t w = 1; w < nwords; w++) {
    const unsigned long long x = words[size_t(w) * n + a], y = words[size_t(w) * n + b];
    if (x != y) return x < y;
  }
  return a < b;
}

// m <= kOrderCta rows (all n rows, or the top-K candidates cand[0, m)): bitonic sort of (word 0, row) in shared memory
// by one CTA, then the first `keep` slots
__global__ void __launch_bounds__(1024) k_order_cta(const unsigned long long* __restrict__ words, uint32_t n, uint32_t nwords,
                                                    const uint32_t* __restrict__ cand, uint32_t m, uint32_t keep,
                                                    const uint32_t* __restrict__ out_slot, uint32_t* __restrict__ new_slot) {
  extern __shared__ __align__(16) unsigned char order_smem[];
  unsigned long long* key = reinterpret_cast<unsigned long long*>(order_smem);
  uint32_t* row = reinterpret_cast<uint32_t*>(key + kOrderCta);
  uint32_t N = 2;
  while (N < m) N <<= 1;
  for (uint32_t i = threadIdx.x; i < N; i += blockDim.x) {
    const uint32_t r = i < m ? (cand ? cand[i] : i) : ~0u;
    key[i] = i < m ? words[r] : ~0ull;
    row[i] = r;
  }
  __syncthreads();
  for (uint32_t k = 2; k <= N; k <<= 1) {
    for (uint32_t j = k >> 1; j > 0; j >>= 1) {
      for (uint32_t i = threadIdx.x; i < N; i += blockDim.x) {
        const uint32_t l = i ^ j;
        if (l <= i) continue;
        const bool up = (i & k) == 0;
        const bool l_before_i = order_row_less(words, n, nwords, key[l], row[l], key[i], row[i]);
        if (l_before_i == up) {
          const unsigned long long tk = key[i]; key[i] = key[l]; key[l] = tk;
          const uint32_t tr = row[i]; row[i] = row[l]; row[l] = tr;
        }
      }
      __syncthreads();
    }
  }
  for (uint32_t r = threadIdx.x; r < keep; r += blockDim.x) new_slot[r] = out_slot ? out_slot[row[r]] : row[r];
}

// one radix pass: digit counts of every tile of kRadixTile positions, digit-major (hist[d * ntiles + tile])
__global__ void __launch_bounds__(kRadixThreads) k_radix_hist(const unsigned long long* __restrict__ key, const uint32_t* __restrict__ idx,
                                                              uint32_t n, uint32_t shift, uint32_t* __restrict__ hist, uint32_t ntiles) {
  __shared__ uint32_t h[256];
  h[threadIdx.x] = 0;
  __syncthreads();
  const uint32_t p0 = blockIdx.x * kRadixTile;
  for (int r = 0; r < kRadixItems; r++) {
    const uint32_t pos = p0 + r * kRadixThreads + threadIdx.x;
    if (pos < n) atomicAdd(&h[uint32_t(key[idx ? idx[pos] : pos] >> shift) & 255u], 1u);
  }
  __syncthreads();
  hist[threadIdx.x * ntiles + blockIdx.x] = h[threadIdx.x];
}

// one radix pass: the rows of a tile go to base[digit, tile] + their rank among the tile's rows with that digit, in
// position order (stable).  Per round of 256 positions: a warp's lanes with the same digit find each other with
// __match_any_sync, the per-warp counts are scanned across the 8 warps per digit.
__global__ void __launch_bounds__(kRadixThreads) k_radix_scatter(const unsigned long long* __restrict__ key, const uint32_t* __restrict__ idx,
                                                                 uint32_t n, uint32_t shift, const unsigned long long* __restrict__ base,
                                                                 uint32_t ntiles, uint32_t* __restrict__ idx_out) {
  constexpr int kWarps = kRadixThreads / 32;
  __shared__ uint32_t cnt[kWarps][256];
  __shared__ unsigned long long gbase[256];
  const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  gbase[threadIdx.x] = base[threadIdx.x * ntiles + blockIdx.x];
  const uint32_t p0 = blockIdx.x * kRadixTile;
  for (int r = 0; r < kRadixItems; r++) {
    for (int w = 0; w < kWarps; w++) cnt[w][threadIdx.x] = 0;
    __syncthreads();
    const uint32_t pos = p0 + r * kRadixThreads + threadIdx.x;
    const bool valid = pos < n;
    const uint32_t row = valid ? (idx ? idx[pos] : pos) : 0u;
    const uint32_t d = valid ? uint32_t(key[row] >> shift) & 255u : 256u;
    const uint32_t peers = __match_any_sync(0xffffffffu, d);
    const uint32_t rank = __popc(peers & ((1u << lane) - 1u));
    if (valid && rank == 0) cnt[warp][d] = __popc(peers);
    __syncthreads();
    uint32_t run = 0;
    for (int w = 0; w < kWarps; w++) { const uint32_t c = cnt[w][threadIdx.x]; cnt[w][threadIdx.x] = run; run += c; }
    __syncthreads();
    if (valid) idx_out[gbase[d] + cnt[warp][d] + rank] = row;
    __syncthreads();
    gbase[threadIdx.x] += run;
  }
}

// ---- top-K (one packed word, keep <= kOrderCta): radix select of the keep-th smallest key T, MSB digit first, then the
// candidates = every row below T + the first rows (in row order) equal to T, finished by k_order_cta ----
struct TopkSel {
  unsigned long long prefix, mask;   // digits of T found so far
  uint32_t k;                        // rows still wanted among those matching the prefix (1-based rank of T among them)
  uint32_t less;                     // rows known to lie strictly below T
  uint32_t hist[256];
};

// digit histogram of the rows whose key matches the prefix found so far
__global__ void __launch_bounds__(256) k_topk_hist(const unsigned long long* __restrict__ key, uint32_t n, uint32_t shift, TopkSel* sel) {
  __shared__ uint32_t h[256];
  h[threadIdx.x] = 0;
  __syncthreads();
  const unsigned long long prefix = sel->prefix, mask = sel->mask;
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const unsigned long long k = key[i];
    if ((k & mask) == prefix) atomicAdd(&h[uint32_t(k >> shift) & 255u], 1u);
  }
  __syncthreads();
  if (h[threadIdx.x]) atomicAdd(&sel->hist[threadIdx.x], h[threadIdx.x]);
}

// pick the digit holding the k-th matching row; no host round trip
__global__ void k_topk_pick(uint32_t shift, TopkSel* sel) {
  __shared__ uint32_t h[256];
  h[threadIdx.x] = sel->hist[threadIdx.x];
  sel->hist[threadIdx.x] = 0;   // ready for the next digit
  __syncthreads();
  if (threadIdx.x == 0) {
    uint32_t before = 0, d = 0;
    for (; d < 255; d++) {
      if (before + h[d] >= sel->k) break;
      before += h[d];
    }
    sel->prefix |= (unsigned long long)d << shift;
    sel->mask |= 255ull << shift;
    sel->less += before;
    sel->k -= before;
  }
}

// rows equal to T per tile of kSlotTile rows
__global__ void __launch_bounds__(256) k_topk_tile_eq(const unsigned long long* __restrict__ key, uint32_t n, const TopkSel* __restrict__ sel,
                                                      uint32_t* __restrict__ tile_counts) {
  __shared__ uint32_t ws[8];
  const unsigned long long T = sel->prefix;
  const uint32_t s0 = blockIdx.x * kSlotTile;
  uint32_t c = 0;
  for (uint32_t i = threadIdx.x; i < (uint32_t)kSlotTile; i += blockDim.x) c += (s0 + i < n && key[s0 + i] == T) ? 1u : 0u;
  c = __reduce_add_sync(0xffffffffu, c);
  if ((threadIdx.x & 31) == 0) ws[threadIdx.x >> 5] = c;
  __syncthreads();
  if (threadIdx.x == 0) {
    uint32_t t = 0;
    for (int w = 0; w < 8; w++) t += ws[w];
    tile_counts[blockIdx.x] = t;
  }
}

// the candidates: every row below T, and the rows equal to T whose rank among them in row order is below sel->k;
// their order in cand is arbitrary (k_order_cta sorts them by (key, row))
__global__ void __launch_bounds__(256) k_topk_compact(const unsigned long long* __restrict__ key, uint32_t n, const TopkSel* __restrict__ sel,
                                                      const unsigned long long* __restrict__ tile_base, uint32_t* __restrict__ cand,
                                                      uint32_t* __restrict__ count) {
  __shared__ uint32_t ws[8];
  const unsigned long long T = sel->prefix;
  const uint32_t need_eq = sel->k;
  const uint32_t s0 = blockIdx.x * kSlotTile + threadIdx.x * 4;
  uint32_t f[4], c = 0;
#pragma unroll
  for (int k = 0; k < 4; k++) { f[k] = (s0 + k < n && key[s0 + k] == T) ? 1u : 0u; c += f[k]; }
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
  unsigned long long rank = tile_base[blockIdx.x] + wbase + incl - c;   // rank of this thread's first equal row
#pragma unroll
  for (int k = 0; k < 4; k++) {
    if (s0 + k >= n) break;
    if (f[k]) {
      if (rank < need_eq) cand[atomicAdd(count, 1u)] = s0 + k;
      rank++;
    } else if (key[s0 + k] < T) {
      cand[atomicAdd(count, 1u)] = s0 + k;
    }
  }
}

__global__ void k_order_gather(const uint32_t* __restrict__ idx, uint32_t keep, const uint32_t* __restrict__ out_slot,
                               uint32_t* __restrict__ new_slot) {
  const uint32_t r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r < keep) new_slot[r] = out_slot ? out_slot[idx[r]] : idx[r];
}

// ---- ORDER BY ... LIMIT on a scan under PQ_QUERY_ALLGATHER: every rank's first rows merged alike on every rank.
// Rank r packs its first keep_r rows (order_sort's, in its order) as records of W = nterms + 2 words: the encoded term
// values (order_encode, DESC applied), a word of NULL flags (bit t: term t is NULL) and the global row id; its block
// holds keep_max records, those past keep_r are padding.  One all-gather hands every rank the same blocks in rank
// order.  The candidates (record j < keep_r of rank r is candidate pre[r] + j) are sorted by global row id (RadixSort),
// then scattered into order_sort's input in that order: order_sort breaks ties by position, so rows equal on every
// term come out in global row order, as one rank over the whole table returns them.
//   k_scan_cand_pack     this rank's send block
//   k_scan_cand_list     the global row id (the sort's key) and the record index of every candidate
//   (RadixSort)          the candidates in ascending global row id
//   k_scan_cand_scatter  the terms and NULL flags in that order, each term's value range, the record of every position
//   (order_sort)         the first `limit` positions, as record indices
//   k_scan_owned         the output rows this rank projects: their handles, ~0 for another rank's rows
struct ScanMergeArgs {
  const unsigned long long* recv;   // nranks blocks of keep_max records of nterms + 2 words
  const unsigned long long* pre;    // [nranks + 1]: the first candidate of every rank, and the total
  uint64_t keep_max;
  uint32_t nranks, n, nterms;       // n: the candidates of every rank
};

__device__ __forceinline__ uint64_t scan_cand_record(const ScanMergeArgs& a, uint32_t p) {
  uint32_t lo = 0, hi = a.nranks - 1;   // the rank r with pre[r] <= p < pre[r + 1] (a rank may have none)
  while (lo < hi) {
    const uint32_t mid = (lo + hi + 1) / 2;
    if (a.pre[mid] <= p) lo = mid;
    else hi = mid - 1;
  }
  return uint64_t(lo) * a.keep_max + (p - a.pre[lo]);
}

// record j < keep_max: this rank's row at sorted position kept[j] (kept == nullptr: j) of its selection, or padding
__global__ void k_scan_cand_pack(const unsigned long long* __restrict__ vals, const uint8_t* __restrict__ nulls, uint32_t n_sel,
                                 uint32_t nterms, const uint32_t* __restrict__ kept, uint32_t keep,
                                 const unsigned long long* __restrict__ handles, const DevItem* __restrict__ items,
                                 uint64_t keep_max, unsigned long long* __restrict__ send) {
  const uint32_t w = nterms + 2;
  for (uint64_t j = blockIdx.x * uint64_t(blockDim.x) + threadIdx.x; j < keep_max; j += uint64_t(gridDim.x) * blockDim.x) {
    unsigned long long* rec = send + j * w;
    if (j >= keep) {
      for (uint32_t t = 0; t < w; t++) rec[t] = t + 1 < w ? 0ull : ~0ull;
      continue;
    }
    const uint32_t q = kept ? kept[j] : uint32_t(j);
    unsigned long long flags = 0;
    for (uint32_t t = 0; t < nterms; t++) {
      rec[t] = vals[size_t(t) * n_sel + q];
      flags |= (unsigned long long)(nulls[size_t(t) * n_sel + q] != 0) << t;
    }
    rec[nterms] = flags;
    const unsigned long long h = handles[q];
    rec[nterms + 1] = items[uint32_t(h >> 32)].global_row0 + uint32_t(h);
  }
}

__global__ void k_scan_cand_list(const ScanMergeArgs a, unsigned long long* __restrict__ ids, uint32_t* __restrict__ rec) {
  for (uint32_t p = blockIdx.x * blockDim.x + threadIdx.x; p < a.n; p += gridDim.x * blockDim.x) {
    const uint64_t r = scan_cand_record(a, p);
    ids[p] = a.recv[r * (a.nterms + 2) + a.nterms + 1];
    rec[p] = uint32_t(r);   // nranks x keep_max < 2^32 (checked on the host)
  }
}

// one thread per position i of the global row order (candidate sorted[i]), ranges reduced as k_order_encode does
__global__ void __launch_bounds__(256) k_scan_cand_scatter(const ScanMergeArgs a, const uint32_t* __restrict__ sorted,
                                                           const uint32_t* __restrict__ rec, unsigned long long* __restrict__ vals,
                                                           uint8_t* __restrict__ nulls, OrderRange* __restrict__ ranges,
                                                           uint32_t* __restrict__ rec_at) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  const bool live = i < a.n;
  const uint64_t r = live ? rec[sorted ? sorted[i] : i] : 0;   // sorted == nullptr: the sort had no bits to sort by
  const unsigned long long* x = a.recv + r * (a.nterms + 2);
  const unsigned long long flags = live ? x[a.nterms] : 0ull;
  if (live) rec_at[i] = uint32_t(r);
  for (uint32_t t = 0; t < a.nterms; t++) {
    const bool valid = live && !((flags >> t) & 1ull);
    const unsigned long long v = live ? x[t] : 0ull;
    if (live) {
      vals[size_t(t) * a.n + i] = v;
      nulls[size_t(t) * a.n + i] = valid ? 0 : 1;
    }
    unsigned long long mn = valid ? v : ~0ull, mx = valid ? v : 0ull;
    for (int s = 16; s > 0; s >>= 1) {
      mn = min(mn, __shfl_xor_sync(0xffffffffu, mn, s));
      mx = max(mx, __shfl_xor_sync(0xffffffffu, mx, s));
    }
    const bool any_null = __any_sync(0xffffffffu, live && !valid), any_value = __any_sync(0xffffffffu, valid);
    if ((threadIdx.x & 31) == 0) {
      if (any_value) {
        atomicMin(&ranges[t].min, mn);
        atomicMax(&ranges[t].max, mx);
        atomicOr(&ranges[t].has_value, 1u);
      }
      if (any_null) atomicOr(&ranges[t].has_null, 1u);
    }
  }
}

// output row j is record order[j]: this rank's when it lies in block `me`, then projected through its handle
__global__ void k_scan_owned(const uint32_t* __restrict__ order, uint32_t keep, uint64_t keep_max, uint32_t me,
                             const uint32_t* __restrict__ kept, const unsigned long long* __restrict__ handles,
                             unsigned long long* __restrict__ owned) {
  const uint32_t j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= keep) return;
  const uint64_t r = order[j], k = r % keep_max;
  owned[j] = r / keep_max == me ? handles[kept ? kept[k] : uint32_t(k)] : ~0ull;
}

// ---- ROW_NUMBER() OVER (PARTITION BY ...) cut to a rank range, over the n rows order_sort left in (partition terms,
// order terms) order.  Sorted position p holds row perm[p] (perm == nullptr: row p).  Tiles of kSlotTile positions,
// 256 threads x 4 consecutive positions, as k_slot_compact:
//   k_window_heads    a position is a head when its partition terms' (value, NULL flag) differ from its predecessor's;
//                     heads per tile
//   k_item_prefix     heads before every tile: a position's partition id is the heads up to it, minus one
//   k_window_starts   the first position of every partition
//   k_window_count    rn = p - start + 1, kept when lo < rn <= hi; kept rows per tile
//   k_item_prefix     kept rows before every tile (and their total: the one host round trip)
//   k_window_compact  the kept rows in order, with their row_number and partition_rows
// A partition may straddle tiles and be larger than one: a position before the first head of its tile belongs to the
// last partition started in an earlier tile (id = heads before the tile - 1), and its start comes from the start table,
// which k_window_starts completes before k_window_count reads it. ----
struct WindowArgs {
  const unsigned long long* vals;        // [nterms][n]: the partition terms are the first nparts
  const uint8_t* nulls;                  // [nterms][n]
  const uint32_t* perm;                  // sorted position -> row (nullptr: identity)
  uint32_t n, nparts;
  unsigned long long lo, hi;             // kept: lo < rn <= hi
  uint8_t* heads;                        // [n]
  uint32_t* start;                       // [n]: partition id -> first sorted position
  uint32_t* tile_counts;                 // [ntiles]
  const unsigned long long* part_base;   // [ntiles]: heads before the tile
  const unsigned long long* n_part;      // partitions in all
  const unsigned long long* keep_base;   // [ntiles]: kept rows before the tile
  // k_window_compact: output row j (< cap) is kept row j
  const uint32_t* rows;                  // nullptr: kept[j] is the row itself, else rows[row]
  uint32_t* kept;
  long long* row_number;                 // nullptr: not asked for
  long long* partition_rows;
  unsigned long long cap;
};

// exclusive prefix of c over the 256 threads of the CTA (ws: 8 words of shared memory)
__device__ __forceinline__ uint32_t window_tile_excl(uint32_t c, uint32_t* ws) {
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
  return wbase + incl - c;
}

// sum of c over the CTA into tile_counts[blockIdx.x]
__device__ __forceinline__ void window_tile_count(uint32_t c, uint32_t* ws, uint32_t* tile_counts) {
  c = __reduce_add_sync(0xffffffffu, c);
  if ((threadIdx.x & 31) == 0) ws[threadIdx.x >> 5] = c;
  __syncthreads();
  if (threadIdx.x == 0) {
    uint32_t t = 0;
    for (int w = 0; w < 8; w++) t += ws[w];
    tile_counts[blockIdx.x] = t;
  }
}

__global__ void __launch_bounds__(256) k_window_heads(const __grid_constant__ WindowArgs a) {
  __shared__ uint32_t ws[8];
  const uint32_t p0 = blockIdx.x * kSlotTile + threadIdx.x * 4;
  uint32_t c = 0;
#pragma unroll
  for (int k = 0; k < 4; k++) {
    const uint32_t p = p0 + k;
    if (p >= a.n) break;
    bool head = p == 0;
    if (!head) {
      const uint32_t r = a.perm ? a.perm[p] : p, q = a.perm ? a.perm[p - 1] : p - 1;
      for (uint32_t t = 0; t < a.nparts && !head; t++) {
        const uint8_t nr = a.nulls[size_t(t) * a.n + r], nq = a.nulls[size_t(t) * a.n + q];
        head = nr != nq || (!nr && a.vals[size_t(t) * a.n + r] != a.vals[size_t(t) * a.n + q]);   // a NULL's value is not read
      }
    }
    a.heads[p] = head ? 1 : 0;
    c += head ? 1u : 0u;
  }
  window_tile_count(c, ws, a.tile_counts);
}

__global__ void __launch_bounds__(256) k_window_starts(const __grid_constant__ WindowArgs a) {
  __shared__ uint32_t ws[8];
  const uint32_t p0 = blockIdx.x * kSlotTile + threadIdx.x * 4;
  uint32_t f[4], c = 0;
#pragma unroll
  for (int k = 0; k < 4; k++) { f[k] = p0 + k < a.n ? a.heads[p0 + k] : 0u; c += f[k]; }
  unsigned long long id = a.part_base[blockIdx.x] + window_tile_excl(c, ws);
#pragma unroll
  for (int k = 0; k < 4; k++)
    if (f[k]) a.start[id++] = p0 + k;
}

// the rank of this thread's 4 positions (rn[k] = 0 past n) and their partition ids
__device__ __forceinline__ void window_ranks(const WindowArgs& a, uint32_t* ws, unsigned long long (&rn)[4], uint32_t (&pid)[4]) {
  const uint32_t p0 = blockIdx.x * kSlotTile + threadIdx.x * 4;
  uint32_t f[4], c = 0;
#pragma unroll
  for (int k = 0; k < 4; k++) { f[k] = p0 + k < a.n ? a.heads[p0 + k] : 0u; c += f[k]; }
  unsigned long long run = a.part_base[blockIdx.x] + window_tile_excl(c, ws);   // >= 1 past position 0: it is a head
#pragma unroll
  for (int k = 0; k < 4; k++) {
    run += f[k];
    pid[k] = uint32_t(run - 1);
    rn[k] = p0 + k < a.n ? uint64_t(p0 + k) - a.start[pid[k]] + 1 : 0ull;
  }
}

__global__ void __launch_bounds__(256) k_window_count(const __grid_constant__ WindowArgs a) {
  __shared__ uint32_t ws[8];
  unsigned long long rn[4];
  uint32_t pid[4], c = 0;
  window_ranks(a, ws, rn, pid);
#pragma unroll
  for (int k = 0; k < 4; k++) c += (rn[k] > a.lo && rn[k] <= a.hi) ? 1u : 0u;
  __syncthreads();   // ws is reused
  window_tile_count(c, ws, a.tile_counts);
}

__global__ void __launch_bounds__(256) k_window_compact(const __grid_constant__ WindowArgs a) {
  __shared__ uint32_t ws[8];
  unsigned long long rn[4];
  uint32_t pid[4], f[4], c = 0;
  window_ranks(a, ws, rn, pid);
#pragma unroll
  for (int k = 0; k < 4; k++) { f[k] = (rn[k] > a.lo && rn[k] <= a.hi) ? 1u : 0u; c += f[k]; }
  __syncthreads();   // ws is reused
  unsigned long long j = a.keep_base[blockIdx.x] + window_tile_excl(c, ws);
  const uint32_t p0 = blockIdx.x * kSlotTile + threadIdx.x * 4;
  const unsigned long long nparts = *a.n_part;
#pragma unroll
  for (int k = 0; k < 4; k++) {
    if (!f[k]) continue;
    if (j < a.cap) {
      const uint32_t p = p0 + k, r = a.perm ? a.perm[p] : p;
      a.kept[j] = a.rows ? a.rows[r] : r;
      if (a.row_number) a.row_number[j] = (long long)rn[k];
      if (a.partition_rows) {
        const uint32_t s = a.start[pid[k]], e = pid[k] + 1ull < nparts ? a.start[pid[k] + 1] : a.n;
        a.partition_rows[j] = (long long)(e - s);
      }
    }
    j++;
  }
}

// a window without partition terms: output row j is row offset + j of the ordered rows src (nullptr: the row order),
// rn = offset + 1 + j, and the one partition holds all n rows
__global__ void k_window_number(unsigned long long cnt, unsigned long long offset, unsigned long long n, const uint32_t* __restrict__ src,
                                uint32_t* __restrict__ kept, long long* __restrict__ row_number, long long* __restrict__ partition_rows) {
  const unsigned long long j = blockIdx.x * uint64_t(blockDim.x) + threadIdx.x;
  if (j >= cnt) return;
  kept[j] = src ? src[offset + j] : uint32_t(offset + j);
  if (row_number) row_number[j] = (long long)(offset + 1 + j);
  if (partition_rows) partition_rows[j] = (long long)n;
}

}  // namespace pqb
