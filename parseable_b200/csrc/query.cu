// Query planning and execution: the C-ABI PqQueryDesc becomes a DevPlan; work items, chunk tables
// and the per-column side tables (string entry offsets, interned GROUP BY ids) come from the
// table's caches; then  k_leaf_luts -> k_flat_filter | k_flat_agg (+ k_scan for the items the flat
// store does not cover) -> k_item_prefix / k_compact_row_ids | k_agg_compact  run on one stream.
//
// Reference behaviour restated here (all /root/reference paths):
//   * predicate pushed into the scan AND re-applied (Inexact pushdown,
//     src/query/stream_schema_provider.rs:665-683): one fused evaluation gives the
//     same rows;
//   * row-group pruning from footer min/max (ParquetFormat::with_enable_pruning,
//     :146): pruning never changes results, only rows_scanned;
//   * SQL three-valued logic, NULL group keys, COUNT -> Int64, SUM(Int64) wrapping,
//     float totalOrder (SURVEY.md §8 rows a11, a12).
#include <algorithm>
#include <charconv>
#include <chrono>
#include <cmath>
#include <cstdlib>
#include <cstring>
#include <functional>
#include <limits>
#include <map>
#include <set>
#include <string_view>
#include <unordered_map>

#include "engine.hpp"
#include "prep_kernels.cuh"
#include "scan_kernel.cuh"
#include "flat_scan.cuh"
#include "json_egress.cuh"
#include "egress_kernels.cuh"
#include "order_kernels.cuh"
#include "percentile_kernels.cuh"
#include "hash_merge.cuh"
#include "in_set.cuh"
#include "regex_compile.hpp"

namespace pqb {

namespace {

template <typename T>
struct DevBuf {
  T* p = nullptr;
  size_t n = 0;
  cudaStream_t s = nullptr;
  void alloc(size_t count, cudaStream_t stream) {
    if (p) { cudaFreeAsync(p, s); p = nullptr; }   // a second alloc (a retry with a larger capacity) replaces the first
    n = count;
    s = stream;
    if (count) PQB_CUDA(cudaMallocAsync((void**)&p, count * sizeof(T), stream));
  }
  void upload(const std::vector<T>& v, cudaStream_t stream) {
    alloc(v.size(), stream);
    if (!v.empty()) PQB_CUDA(cudaMemcpyAsync(p, v.data(), v.size() * sizeof(T), cudaMemcpyHostToDevice, stream));
  }
  void zero() { if (n) PQB_CUDA(cudaMemsetAsync(p, 0, n * sizeof(T), s)); }
  ~DevBuf() { if (p) cudaFreeAsync(p, s); }
};

constexpr uint64_t kKeepDeviceResult = 1ull << 30;   // result blocks up to this size stay on the device until the query closes
constexpr uint64_t kExactKeyBytes = 64ull << 20;     // a string key whose byte bound exceeds this is counted exactly first
// COUNT(DISTINCT): the dense presence bitmap of one distinct column may take this much HBM (and at most a quarter of
// the free HBM); above it the column gets a pair set, of at most kDistinctPairsMax 8-byte entries (2 GiB)
constexpr uint64_t kDistinctDenseBudget = 1ull << 30;
constexpr uint64_t kDistinctPairsMax = 1ull << 28;
// MEDIAN / PERCENTILE_CONT: HBM per row of the live row groups.  Every percentile column holds its emitted pairs (4-byte
// slot + 8-byte key) until its sort; one column at a time is sorted, with at most kPctSortBytes per pair (order_sort's
// [2][n] values and NULL flags 18, packed words <= 16, two index arrays 8, the kept order 4, the digit tables 2).
// The query is refused (PQ_ERR_OOM) when rows x (12 x columns + kPctSortBytes) exceeds half the free HBM.
constexpr uint64_t kPctPairBytes = 12, kPctSortBytes = 48;

struct Timer {
  cudaEvent_t a, b;
  Timer() { cudaEventCreate(&a); cudaEventCreate(&b); }
  ~Timer() { cudaEventDestroy(a); cudaEventDestroy(b); }
};

// ---- LIKE pattern classification (arrow-string like.rs fast paths) ----
struct LikePlan { uint32_t kind; std::string needle; };
LikePlan classify_like(const std::string& pat) {
  // unescaped structure: sequence of literal chars and wildcards
  std::string lit;
  std::vector<int> tokens;  // -1 '%', -2 '_', >=0 literal byte
  for (size_t i = 0; i < pat.size(); i++) {
    char c = pat[i];
    if (c == '\\' && i + 1 < pat.size()) { tokens.push_back((unsigned char)pat[++i]); }
    else if (c == '%') tokens.push_back(-1);
    else if (c == '_') tokens.push_back(-2);
    else tokens.push_back((unsigned char)c);
  }
  bool has_us = false;
  int npct = 0;
  for (int t : tokens) { has_us |= t == -2; npct += t == -1; }
  auto literal_of = [&](size_t b, size_t e) { std::string s; for (size_t i = b; i < e; i++) s.push_back(char(tokens[i])); return s; };
  if (!has_us) {
    if (npct == 0) return {LIKE_EQ, literal_of(0, tokens.size())};
    // collapse leading / trailing runs of '%'
    size_t b = 0, e = tokens.size();
    while (b < e && tokens[b] == -1) b++;
    while (e > b && tokens[e - 1] == -1) e--;
    bool inner = false;
    for (size_t i = b; i < e; i++) inner |= tokens[i] == -1;
    if (!inner) {
      bool lead = b > 0, trail = e < tokens.size();
      std::string n = literal_of(b, e);
      if (lead && trail) return {LIKE_CONTAINS, n};
      if (trail) return {LIKE_PREFIX, n};
      if (lead) return {LIKE_SUFFIX, n};
    }
  }
  return {LIKE_GENERAL, pat};
}

// FNV-1a over the bytes of a compiled plan, its literals and the batch size: equal for a repeat of the same query on the
// same table (DevPlan is zero-initialised, padding included, before the planner fills it)
uint64_t plan_hash(const DevPlan& plan, const std::vector<uint8_t>& lits, uint32_t batch_rows) {
  uint64_t h = 1469598103934665603ull;
  auto mix = [&](const void* p, size_t n) {
    const uint8_t* b = static_cast<const uint8_t*>(p);
    size_t i = 0;
    for (; i + 8 <= n; i += 8) { uint64_t w; std::memcpy(&w, b + i, 8); h = (h ^ w) * 1099511628211ull; }
    for (; i < n; i++) h = (h ^ b[i]) * 1099511628211ull;
  };
  mix(&plan, sizeof(plan));
  mix(lits.data(), lits.size());
  mix(&batch_rows, sizeof(batch_rows));
  return h;
}

uint64_t f64_bits(double d) { uint64_t b; std::memcpy(&b, &d, 8); return b; }
double bits_f64(uint64_t b) { double d; std::memcpy(&d, &b, 8); return d; }

// tri-state for pruning
enum Tri { TRI_FALSE = 0, TRI_TRUE = 1, TRI_MAYBE = 2 };

struct HostLeaf {
  DevLeaf d{};
  int qcol = -1;
  std::string str;
  // LK_IN: the distinct members, sorted in the column's order, for pruning (Int64 / Timestamp / Date32 signed, Float64 as
  // doubles, Utf8 bytewise); in_nan: some Float64 member is a NaN
  std::vector<int64_t> in_i64;
  std::vector<double> in_f64;
  std::vector<std::string> in_str;
  bool in_nan = false;
};

// min / max statistics of an Int64 / Timestamp / Date32 chunk (an INT32 (Date32) leaf's sign-extended like its values)
bool stats_i64(const ColumnStats& st, int64_t& mn, int64_t& mx) {
  if (st.min.size() == 8 && st.max.size() == 8) {
    std::memcpy(&mn, st.min.data(), 8);
    std::memcpy(&mx, st.max.data(), 8);
    return true;
  }
  if (st.min.size() == 4 && st.max.size() == 4) {
    int32_t a, b;
    std::memcpy(&a, st.min.data(), 4);
    std::memcpy(&b, st.max.data(), 4);
    mn = a;
    mx = b;
    return true;
  }
  return false;
}

// An IN leaf is FALSE on a chunk none of whose members lies in the chunk's [min, max]
Tri in_from_stats(const HostLeaf& lf, uint8_t kind, const ColumnStats& st) {
  bool hit;
  if (kind == DK_I64) {
    int64_t mn, mx;
    if (!stats_i64(st, mn, mx)) return TRI_MAYBE;
    const auto it = std::lower_bound(lf.in_i64.begin(), lf.in_i64.end(), mn);
    hit = it != lf.in_i64.end() && *it <= mx;
  } else if (kind == DK_F64) {
    if (st.min.size() != 8 || st.max.size() != 8) return TRI_MAYBE;
    double mn, mx;
    std::memcpy(&mn, st.min.data(), 8);
    std::memcpy(&mx, st.max.data(), 8);
    // as for `=`: NaN rows may lie outside [min, max], and the bounds may fold -0.0 / 0.0
    if (lf.in_nan || std::isnan(mn) || std::isnan(mx) || mn == 0.0 || mx == 0.0) return TRI_MAYBE;
    const auto it = std::lower_bound(lf.in_f64.begin(), lf.in_f64.end(), mn);
    hit = it != lf.in_f64.end() && *it <= mx;
  } else if (kind == DK_STR) {
    // (a truncated max is still an upper bound)
    auto cmps = [](const std::string& a, const std::string& b) {
      return cmp_bytes((const uint8_t*)a.data(), uint32_t(a.size()), (const uint8_t*)b.data(), uint32_t(b.size()));
    };
    const auto it = std::lower_bound(lf.in_str.begin(), lf.in_str.end(), st.min,
                                     [&](const std::string& a, const std::string& b) { return cmps(a, b) < 0; });
    hit = it != lf.in_str.end() && cmps(*it, st.max) <= 0;
  } else {
    return TRI_MAYBE;
  }
  return hit ? TRI_MAYBE : TRI_FALSE;
}

// Can `col <cmp> lit` be decided for a whole chunk from its min/max statistics?
Tri leaf_from_stats(const HostLeaf& lf, uint8_t kind, const TableChunk& ch, uint32_t rg_rows) {
  if (!ch.present) {
    // column absent: all NULL
    if (lf.d.kind == LK_IS_NULL) return TRI_TRUE;
    return TRI_FALSE;  // NULL compare is never TRUE; IS NOT NULL is FALSE
  }
  const ColumnStats& st = ch.meta->stats;
  bool no_nulls = st.null_count == 0;
  bool all_nulls = st.null_count >= 0 && uint64_t(st.null_count) == uint64_t(ch.meta->num_values);
  if (lf.d.kind == LK_IS_NULL) return no_nulls ? TRI_FALSE : (all_nulls ? TRI_TRUE : TRI_MAYBE);
  if (lf.d.kind == LK_IS_NOT_NULL) return no_nulls ? TRI_TRUE : (all_nulls ? TRI_FALSE : TRI_MAYBE);
  if (all_nulls) return TRI_FALSE;
  if (lf.d.kind == LK_IN && st.has_min && st.has_max) return in_from_stats(lf, kind, st);
  if (lf.d.kind != LK_CMP || !st.has_min || !st.has_max) return TRI_MAYBE;
  int lo_c, hi_c;  // sign of compare(min, lit), compare(max, lit)
  if (kind == DK_I64) {
    int64_t mn, mx;
    if (!stats_i64(st, mn, mx)) return TRI_MAYBE;
    lo_c = mn < lf.d.lit_i64 ? -1 : (mn > lf.d.lit_i64 ? 1 : 0);
    hi_c = mx < lf.d.lit_i64 ? -1 : (mx > lf.d.lit_i64 ? 1 : 0);
  } else if (kind == DK_F64) {
    if (st.min.size() != 8 || st.max.size() != 8) return TRI_MAYBE;
    double mn, mx, lit = bits_f64(uint64_t(lf.d.lit_i64));
    std::memcpy(&mn, st.min.data(), 8);
    std::memcpy(&mx, st.max.data(), 8);
    // footer statistics ignore NaN and may fold -0.0/+0.0: only decide on clean finite bounds
    if (std::isnan(mn) || std::isnan(mx) || std::isnan(lit)) return TRI_MAYBE;
    if (mn == 0.0 || mx == 0.0 || lit == 0.0) return TRI_MAYBE;
    lo_c = mn < lit ? -1 : (mn > lit ? 1 : 0);
    hi_c = mx < lit ? -1 : (mx > lit ? 1 : 0);
    // a chunk may still hold NaN outside [min,max], on either side: totalOrder puts a NaN with the sign bit below -inf
    // and one without it above +inf.  Only `=` against a non-NaN literal is FALSE on every NaN row.
    return (lf.d.cmp == PQ_EQ && (lo_c > 0 || hi_c < 0)) ? TRI_FALSE : TRI_MAYBE;
  } else if (kind == DK_STR) {
    auto cmpb = [&](const std::string& a) {
      int c = cmp_bytes((const uint8_t*)a.data(), uint32_t(a.size()), (const uint8_t*)lf.str.data(), uint32_t(lf.str.size()));
      return c;
    };
    lo_c = cmpb(st.min);
    hi_c = cmpb(st.max);
    // string max statistics may be truncated upper bounds: only use them to rule rows OUT
    switch (lf.d.cmp) {
      case PQ_EQ: return (lo_c > 0 || hi_c < 0) ? TRI_FALSE : TRI_MAYBE;
      case PQ_LT: return lo_c >= 0 ? TRI_FALSE : TRI_MAYBE;
      case PQ_LE: return lo_c > 0 ? TRI_FALSE : TRI_MAYBE;
      case PQ_GT: return hi_c <= 0 ? TRI_FALSE : TRI_MAYBE;
      case PQ_GE: return hi_c < 0 ? TRI_FALSE : TRI_MAYBE;
      default: return TRI_MAYBE;
    }
  } else {
    return TRI_MAYBE;
  }
  (void)rg_rows;
  Tri r = TRI_MAYBE;
  switch (lf.d.cmp) {
    case PQ_EQ: r = (lo_c > 0 || hi_c < 0) ? TRI_FALSE : ((lo_c == 0 && hi_c == 0) ? TRI_TRUE : TRI_MAYBE); break;
    case PQ_NE: r = (lo_c > 0 || hi_c < 0) ? TRI_TRUE : ((lo_c == 0 && hi_c == 0) ? TRI_FALSE : TRI_MAYBE); break;
    case PQ_LT: r = hi_c < 0 ? TRI_TRUE : (lo_c >= 0 ? TRI_FALSE : TRI_MAYBE); break;
    case PQ_LE: r = hi_c <= 0 ? TRI_TRUE : (lo_c > 0 ? TRI_FALSE : TRI_MAYBE); break;
    case PQ_GT: r = lo_c > 0 ? TRI_TRUE : (hi_c <= 0 ? TRI_FALSE : TRI_MAYBE); break;
    case PQ_GE: r = lo_c >= 0 ? TRI_TRUE : (hi_c < 0 ? TRI_FALSE : TRI_MAYBE); break;
  }
  if (r == TRI_TRUE && !no_nulls) r = TRI_MAYBE;  // NULL rows evaluate to NULL, not TRUE
  return r;
}

Tri tri_and(Tri a, Tri b) { return (a == TRI_FALSE || b == TRI_FALSE) ? TRI_FALSE : ((a == TRI_TRUE && b == TRI_TRUE) ? TRI_TRUE : TRI_MAYBE); }
Tri tri_or(Tri a, Tri b) { return (a == TRI_TRUE || b == TRI_TRUE) ? TRI_TRUE : ((a == TRI_FALSE && b == TRI_FALSE) ? TRI_FALSE : TRI_MAYBE); }
// NOT of "certainly not TRUE" is not "certainly TRUE" under NULLs: keep MAYBE
Tri tri_not(Tri a) { (void)a; return TRI_MAYBE; }

const char* type_name(int t) {
  switch (t) { case PQ_T_BOOL: return "Boolean"; case PQ_T_I64: return "Int64"; case PQ_T_F64: return "Float64";
    case PQ_T_UTF8: return "Utf8"; case PQ_T_TS_MS: return "Timestamp(ms)"; case PQ_T_DATE32: return "Date32"; default: return "Null"; }
}

uint32_t align_up(uint32_t v, uint32_t a) { return (v + a - 1) & ~(a - 1); }

// MIN / MAX over Utf8: the rows' values are their bytewise ranks (DevPlan.rank), read through the column's GROUP BY ids --
// like a key column, it reads ids, never the values themselves
bool rank_min_max(const DevAgg& ag) { return (ag.fn == AG_MIN || ag.fn == AG_MAX) && ag.kind == DK_STR; }
bool bool_min_max(const DevAgg& ag) { return (ag.fn == AG_MIN || ag.fn == AG_MAX) && ag.kind == DK_BOOL; }

// KR (rows per thread) of the k_flat_agg instantiation the launch picks for `krows` rows per thread and slab: the
// hashed ones exist for 4, the RX ones for 2 when not hashed, the others for 8, 4 and 2
uint32_t agg_kr(const DevPlan& plan, bool rx, uint32_t krows) {
  if (plan.hashed) return 4;
  if (rx) return 2;
  return krows >= 8 ? 8 : krows >= 4 ? 4 : 2;
}

}  // namespace

Query::Query(const PqQueryDesc& d) {
  run(d);
}
Query::~Query() {
  for (auto& b : dev_blocks_)
    if (b && b->dev) { cudaFree(b->dev); b->dev = nullptr; }
}

void launch_flat_store(const uint8_t* arena, const DevPage* pages, const void* jobs, uint32_t n_jobs, uint8_t* flat, uint8_t* ok,
                       uint32_t* maxlen, cudaStream_t stream) {
  if (!n_jobs) return;
  k_flat_store<<<(n_jobs + 3) / 4, 128, 0, stream>>>(arena, pages, static_cast<const FlatStoreJob*>(jobs), n_jobs, flat, ok, maxlen);
  PQB_CUDA(cudaGetLastError());
}

// ---- table-level side tables (called under Table::side_mu) -----------------------------------------
static std::vector<EntChunk> column_chunks(const Table& t, int tcol) {
  std::vector<EntChunk> v(t.row_groups.size());
  for (size_t g = 0; g < t.row_groups.size(); g++) {
    const TableChunk& tc = t.row_groups[g].chunks[tcol];
    v[g] = EntChunk{tc.dict_off, tc.dict_len, tc.dict_n, t.sides[tcol].base_per_rg[g], tc.present ? 1u : 0u};
  }
  return v;
}

void launch_dba_lengths(const uint8_t* arena, const DevPage* pages, const DbaJob* jobs, uint32_t n_jobs, uint8_t* scratch, DbaInfo* info, cudaStream_t stream) {
  if (!n_jobs) return;
  k_dba_lengths<<<(n_jobs + 3) / 4, 128, 0, stream>>>(arena, pages, jobs, n_jobs, scratch, info);
  PQB_CUDA(cudaGetLastError());
}
void launch_dba_materialise(const uint8_t* arena, const DevPage* pages, const DbaJob* jobs, const DbaInfo* info, uint32_t n_jobs,
                            const uint8_t* scratch, uint8_t* mat, cudaStream_t stream) {
  if (!n_jobs) return;
  k_dba_materialise<<<(n_jobs + 3) / 4, 128, 0, stream>>>(arena, pages, jobs, info, n_jobs, scratch, mat);
  PQB_CUDA(cudaGetLastError());
}
void launch_check_flat_indices(const uint8_t* flat, const FlatPageRec* fpages, const uint32_t* dict_n, uint32_t n_pages, uint32_t* first_bad, cudaStream_t stream) {
  if (!n_pages) return;
  k_check_flat_indices<<<(n_pages + 3) / 4, 128, 0, stream>>>(flat, fpages, dict_n, n_pages, first_bad);
  PQB_CUDA(cudaGetLastError());
}
void launch_page_has_nulls(const uint8_t* arena, const DevPage* pages, uint32_t n_pages, uint8_t* out, cudaStream_t stream) {
  if (!n_pages) return;
  k_page_has_nulls<<<(n_pages + 127) / 128, 128, 0, stream>>>(arena, pages, n_pages, out);
  PQB_CUDA(cudaGetLastError());
}

void launch_delta_to_plain8(const uint8_t* arena, const DevPage* pages, const void* jobs, uint32_t n_jobs, uint8_t* flat_base, uint8_t* ok,
                            cudaStream_t stream) {
  if (!n_jobs) return;
  k_delta_to_plain8<<<(n_jobs + 3) / 4, 128, 0, stream>>>(arena, pages, static_cast<const DeltaJob*>(jobs), n_jobs, flat_base, ok);
  PQB_CUDA(cudaGetLastError());
}

// ---- agg pages (flat_store.cuh): built once per table column, kept with the table (callers hold side_mu) ----
// Packs the jobs into one new buffer (returned; offsets relative to d_flat like every flat page) and records each page's
// new form in the table's agg page table.  The agg pages are optional: when the device memory for them is not there,
// nothing is recorded, nullptr comes back and the column keeps reading its index pages.
static bool try_alloc(void** p, size_t bytes, cudaStream_t stream) {
  if (cudaMallocAsync(p, bytes, stream) == cudaSuccess) return true;
  (void)cudaGetLastError();   // an allocation failure is not sticky: clear it, the query goes on without this form
  *p = nullptr;
  return false;
}
static uint8_t* build_agg_pages(const Table& t, std::vector<AggFormJob>& jobs, const std::vector<uint32_t>& page_of, uint8_t fkind,
                                uint64_t& bytes, cudaStream_t stream) {
  if (!t.d_agg_pages) {   // first agg pages of the table: the whole page table, every record FK_NONE (nobody reads it yet)
    FlatPageRec blank{};
    blank.voff = ~0ull;
    t.agg_pages.assign(t.pages.size(), blank);
    if (!try_alloc((void**)&t.d_agg_pages, t.agg_pages.size() * sizeof(FlatPageRec), stream)) return nullptr;
    PQB_CUDA(cudaMemcpyAsync(t.d_agg_pages, t.agg_pages.data(), t.agg_pages.size() * sizeof(FlatPageRec), cudaMemcpyHostToDevice, stream));
  }
  uint64_t off = 0;
  for (AggFormJob& j : jobs) {
    j.dst = off;
    off += (((uint64_t(j.rows) + 31) / 32) * j.w * 4 + 15) & ~15ull;
  }
  uint8_t* buf = nullptr;
  AggFormJob* dj = nullptr;
  if (!try_alloc((void**)&buf, off + 64, stream)) return nullptr;   // + the over-read of a slab's last staged word
  if (!try_alloc((void**)&dj, jobs.size() * sizeof(AggFormJob), stream)) {
    PQB_CUDA(cudaFreeAsync(buf, stream));
    return nullptr;
  }
  const uint64_t rel = uint64_t(buf) - uint64_t(t.d_flat);      // the subtraction may wrap, d_flat + offset does not
  for (AggFormJob& j : jobs) j.dst += rel;
  PQB_CUDA(cudaMemcpyAsync(dj, jobs.data(), jobs.size() * sizeof(AggFormJob), cudaMemcpyHostToDevice, stream));
  k_agg_form_pack<<<uint32_t((jobs.size() + 3) / 4), 128, 0, stream>>>(t.d_flat, dj, uint32_t(jobs.size()));
  PQB_CUDA(cudaGetLastError());
  PQB_CUDA(cudaFreeAsync(dj, stream));
  for (size_t i = 0; i < jobs.size(); i++) {
    const AggFormJob& j = jobs[i];
    FlatPageRec& r = t.agg_pages[page_of[i]];
    r = t.flat_pages[page_of[i]];
    r.off = j.dst;
    r.bw = uint8_t(j.w);
    r.fkind = fkind;
    r.dexp = uint16_t(j.e);
    r.base = uint64_t(j.base);
  }
  // only the records of this column's pages go up (runs of consecutive pages): a query running on another stream reads
  // the table's other records, and those are never written again
  for (size_t i = 0; i < page_of.size();) {
    size_t e = i + 1;
    while (e < page_of.size() && page_of[e] == page_of[e - 1] + 1) e++;
    PQB_CUDA(cudaMemcpyAsync(t.d_agg_pages + page_of[i], t.agg_pages.data() + page_of[i], (e - i) * sizeof(FlatPageRec),
                             cudaMemcpyHostToDevice, stream));
    i = e;
  }
  PQB_CUDA(cudaStreamSynchronize(stream));
  bytes = off;
  t.agg_pages_ver++;
  return buf;
}

bool Table::ensure_for_pages(int tcol, bool f64, cudaStream_t stream) const {
  std::lock_guard<std::mutex> lk(side_mu);
  ColSide& cs = sides[tcol];
  if (cs.for_ready || cs.d_ids) return cs.for_pages != 0;
  cs.for_ready = true;
  // one classification per chunk with a numeric dictionary copy
  std::vector<ForChunkJob> cj;
  std::vector<int> info_of(row_groups.size(), -1);
  for (size_t g = 0; g < row_groups.size(); g++) {
    const TableChunk& tc = row_groups[g].chunks[tcol];
    if (!tc.present || tc.dict8_off == ~0ull || !tc.dict_n) continue;
    info_of[g] = int(cj.size());
    cj.push_back(ForChunkJob{tc.dict8_off, tc.dict_n, f64 ? 1u : 0u});
  }
  std::vector<ForChunkInfo> info(cj.size());
  if (!cj.empty()) {
    DevBuf<ForChunkJob> dj;
    dj.upload(cj, stream);
    DevBuf<ForChunkInfo> di;
    di.alloc(cj.size(), stream);
    k_for_classify<<<uint32_t(cj.size()), 256, 0, stream>>>(d_flat, dj.p, di.p);
    PQB_CUDA(cudaGetLastError());
    PQB_CUDA(cudaMemcpyAsync(info.data(), di.p, info.size() * sizeof(ForChunkInfo), cudaMemcpyDeviceToHost, stream));
    PQB_CUDA(cudaStreamSynchronize(stream));
  }
  std::vector<AggFormJob> jobs;
  std::vector<uint32_t> page_of;
  uint32_t w_max = 0, rest_bw = 0;
  for (size_t g = 0; g < row_groups.size(); g++) {
    const TableChunk& tc = row_groups[g].chunks[tcol];
    if (!tc.present) continue;
    const ForChunkInfo* fi = info_of[g] >= 0 ? &info[info_of[g]] : nullptr;
    for (uint32_t k = 0; k < tc.pages.n_pages; k++) {
      const uint32_t pi = tc.pages.first_page + k;
      const FlatPageRec& fr = flat_pages[pi];
      if (fr.fkind != FK_INDEX) continue;
      if (!fi || !fi->ok) { rest_bw = std::max<uint32_t>(rest_bw, fr.bw); continue; }
      jobs.push_back(AggFormJob{fr.off, 0, fr.voff, tc.dict8_off, fi->base, fr.rows, fr.bw, tc.dict_n, fi->w, fi->e, f64 ? AF_F64 : AF_I64});
      page_of.push_back(pi);
      w_max = std::max(w_max, fi->w);
    }
  }
  if (jobs.empty()) return false;
  cs.d_for = build_agg_pages(*this, jobs, page_of, FK_FOR, cs.for_bytes, stream);
  if (!cs.d_for) return false;
  cs.for_bw = w_max;
  cs.for_rest_bw = rest_bw;
  cs.for_pages = uint32_t(jobs.size());
  return true;
}

bool Table::ensure_id_pages(int tcol, cudaStream_t stream) const {
  std::lock_guard<std::mutex> lk(side_mu);
  ColSide& cs = sides[tcol];
  if (cs.ids_ready || cs.for_pages) return cs.d_ids != nullptr;
  cs.ids_ready = true;   // one attempt: without the memory for them, the column keeps its gid LUT
  const uint32_t w = bit_width_u64(cs.card ? cs.card - 1u : 0u);
  std::vector<AggFormJob> jobs;
  std::vector<uint32_t> page_of;
  for (size_t g = 0; g < row_groups.size(); g++) {
    const TableChunk& tc = row_groups[g].chunks[tcol];
    if (!tc.present) continue;
    for (uint32_t k = 0; k < tc.pages.n_pages; k++) {
      const uint32_t pi = tc.pages.first_page + k;
      const FlatPageRec& fr = flat_pages[pi];
      if (fr.fkind != FK_INDEX) continue;
      jobs.push_back(AggFormJob{fr.off, 0, fr.voff, uint64_t(cs.d_gid + cs.base_per_rg[g]), 0, fr.rows, fr.bw, tc.dict_n, w, 0, AF_IDS});
      page_of.push_back(pi);
    }
  }
  if (jobs.empty()) return false;
  cs.d_ids = build_agg_pages(*this, jobs, page_of, FK_IDS, cs.ids_bytes, stream);
  cs.ids_bw = w;
  return cs.d_ids != nullptr;
}

TuplePages::~TuplePages() {
  if (d_buf) cudaFree(d_buf);
  if (d_wide) cudaFree(d_wide);
  if (d_order) cudaFree(d_order);
}

// Tuple id pages of the key columns `keys` (table column, mixed-radix stride), every one a dictionary key in the local
// numbering (after ensure_key) whose pages all have flat-store index pages.  The lead column is the first key present
// in every row group; none: no tuple pages.  Counts on the device, ranks on the host, packs on the device.
std::shared_ptr<const TuplePages> Table::ensure_tuple_pages(const std::vector<std::pair<int, uint64_t>>& keys, bool verbose,
                                                            cudaStream_t stream) const {
  std::lock_guard<std::mutex> lk(side_mu);
  auto it = tuples.find(keys);
  if (it != tuples.end()) return it->second;
  if (tuples.size() >= kMaxTupleEntries) return nullptr;
  std::shared_ptr<const TuplePages>& slot = tuples[keys];   // one attempt: a failure stays nullptr
  const auto t0 = std::chrono::steady_clock::now();
  const uint32_t nk = uint32_t(keys.size());
  TupleArgs ta{};
  ta.nkeys = nk;
  uint64_t space = 1;
  int lead = -1;
  for (uint32_t k = 0; k < nk; k++) {
    const ColSide& cs = sides[keys[k].first];
    if (!cs.key_ready || !cs.key_row_pages.empty()) return nullptr;
    ta.card[k] = cs.card;
    ta.stride[k] = uint32_t(keys[k].second);
    space = std::max<uint64_t>(space, keys[k].second * (uint64_t(cs.card) + 1));
    bool everywhere = true;
    for (const TableRowGroup& rg : row_groups) everywhere = everywhere && rg.chunks[keys[k].first].present;
    if (everywhere && lead < 0) lead = int(k);
  }
  if (lead < 0 || space > (1ull << 26)) return nullptr;
  const int lcol = keys[lead].first;
  // jobs: per row group, the row ranges between the page starts of all key columns
  std::vector<TupleJob> jobs;
  std::vector<uint32_t> lead_pages;
  for (size_t g = 0; g < row_groups.size(); g++) {
    std::vector<uint32_t> cuts;
    for (uint32_t k = 0; k < nk; k++) {
      const TableChunk& tc = row_groups[g].chunks[keys[k].first];
      if (!tc.present) continue;
      for (uint32_t p = 0; p < tc.pages.n_pages; p++) {
        const uint32_t pi = tc.pages.first_page + p;
        if (flat_pages[pi].fkind != FK_INDEX) return nullptr;   // every page of a key must be a flat-store index page
        cuts.push_back(pages[pi].first_row);
      }
    }
    cuts.push_back(row_groups[g].num_rows);
    std::sort(cuts.begin(), cuts.end());
    cuts.erase(std::unique(cuts.begin(), cuts.end()), cuts.end());
    std::vector<uint32_t> at(nk, 0);   // current page of each key
    for (size_t c = 0; c + 1 < cuts.size(); c++) {
      const uint32_t r0 = cuts[c], r1 = cuts[c + 1];
      if (r1 <= r0) continue;
      TupleJob j{};
      j.rows = r1 - r0;
      for (uint32_t k = 0; k < nk; k++) {
        const TableChunk& tc = row_groups[g].chunks[keys[k].first];
        if (!tc.present) continue;
        while (at[k] + 1 < tc.pages.n_pages && pages[tc.pages.first_page + at[k] + 1].first_row <= r0) at[k]++;
        const uint32_t pi = tc.pages.first_page + at[k];
        const FlatPageRec& fr = flat_pages[pi];
        if (r1 > pages[pi].first_row + fr.rows) return nullptr;   // pages must cover the row group
        j.k[k] = TupleKeySrc{fr.off, fr.voff, sides[keys[k].first].d_gid + sides[keys[k].first].base_per_rg[g], r0 - pages[pi].first_row,
                             fr.bw, tc.dict_n, 0};
        if (int(k) == lead) {
          j.row0 = r0 - pages[pi].first_row;
          if (lead_pages.empty() || lead_pages.back() != pi) lead_pages.push_back(pi);
          j.dst = pi;   // the lead page for now; its tuple page's offset below
        }
      }
      jobs.push_back(j);
    }
  }
  if (jobs.empty()) return nullptr;
  // 1. rows per group
  std::vector<unsigned int> counts(space, 0u);
  {
    DevBuf<unsigned int> d_counts;
    DevBuf<TupleJob> d_jobs;
    if (cudaMallocAsync((void**)&d_counts.p, space * 4, stream) != cudaSuccess) { (void)cudaGetLastError(); return nullptr; }
    d_counts.n = space;
    d_counts.s = stream;
    d_counts.zero();
    d_jobs.upload(jobs, stream);
    ta.jobs = d_jobs.p;
    ta.n_jobs = uint32_t(jobs.size());
    ta.counts = d_counts.p;
    k_tuple_count<<<uint32_t((jobs.size() + 3) / 4), 128, 0, stream>>>(d_flat, ta);
    PQB_CUDA(cudaGetLastError());
    PQB_CUDA(cudaMemcpyAsync(counts.data(), d_counts.p, space * 4, cudaMemcpyDeviceToHost, stream));
    PQB_CUDA(cudaStreamSynchronize(stream));
  }
  // 2. rank: count descending, mixed-radix id ascending
  std::vector<uint32_t> occurring;
  for (uint32_t m = 0; m < space; m++) if (counts[m]) occurring.push_back(m);
  if (occurring.empty()) return nullptr;
  std::vector<uint32_t> wide = occurring;
  std::stable_sort(wide.begin(), wide.end(), [&](uint32_t a, uint32_t b) { return counts[a] > counts[b]; });
  std::vector<uint32_t> rank(space, 0u);
  for (uint32_t t = 0; t < wide.size(); t++) rank[wide[t]] = t;
  std::vector<uint32_t> order(occurring.size());
  for (size_t p = 0; p < occurring.size(); p++) order[p] = rank[occurring[p]];
  auto tp = std::make_shared<TuplePages>();
  tp->n_tuples = uint32_t(wide.size());
  tp->bw = std::max<uint32_t>(1, bit_width_u64(tp->n_tuples - 1u));
  tp->lead = lcol;
  // 3. the pages: one per lead page, 16-byte aligned, zeroed (jobs that share a word OR into it)
  std::unordered_map<uint32_t, uint64_t> page_off;
  uint64_t off = 0;
  for (uint32_t pi : lead_pages) {
    page_off[pi] = off;
    off += ((uint64_t(flat_pages[pi].rows) + 31) / 32 * tp->bw * 4 + 15) & ~15ull;
  }
  std::vector<unsigned long long> wide64(wide.begin(), wide.end());
  if (!try_alloc((void**)&tp->d_buf, off + 64, stream)) return nullptr;   // + the over-read of a slab's last staged word
  if (!try_alloc((void**)&tp->d_wide, wide64.size() * 8, stream) || !try_alloc((void**)&tp->d_order, order.size() * 4, stream)) return nullptr;
  PQB_CUDA(cudaMemsetAsync(tp->d_buf, 0, off + 64, stream));
  PQB_CUDA(cudaMemcpyAsync(tp->d_wide, wide64.data(), wide64.size() * 8, cudaMemcpyHostToDevice, stream));
  PQB_CUDA(cudaMemcpyAsync(tp->d_order, order.data(), order.size() * 4, cudaMemcpyHostToDevice, stream));
  const uint64_t rel = uint64_t(tp->d_buf) - uint64_t(d_flat);   // the subtraction may wrap, d_flat + offset does not
  for (TupleJob& j : jobs) j.dst = rel + page_off[uint32_t(j.dst)];
  {
    DevBuf<uint32_t> d_rank;
    DevBuf<TupleJob> d_jobs;
    d_rank.upload(rank, stream);
    d_jobs.upload(jobs, stream);
    ta.jobs = d_jobs.p;
    ta.rank = d_rank.p;
    ta.counts = nullptr;
    ta.w = tp->bw;
    k_tuple_pack<<<uint32_t((jobs.size() + 3) / 4), 128, 0, stream>>>(d_flat, ta);
    PQB_CUDA(cudaGetLastError());
    PQB_CUDA(cudaStreamSynchronize(stream));
  }
  for (uint32_t pi : lead_pages) {
    FlatPageRec r = flat_pages[pi];
    r.off = rel + page_off[pi];
    r.voff = ~0ull;   // a NULL key is part of its tuple
    r.bw = uint8_t(tp->bw);
    r.fkind = FK_IDS;
    tp->recs.emplace_back(pi, r);
  }
  tp->bytes = off + wide64.size() * 8 + order.size() * 4;
  tp->build_ms = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
  if (verbose)
    fprintf(stderr, "[pqb] tuple pages: %u keys, lead column %s, %u tuples of %llu slots, %u bits, %zu jobs over %zu lead pages, "
            "%.1f MB, built in %.2f ms\n", nk, columns[lcol].name.c_str(), tp->n_tuples, (unsigned long long)space, tp->bw, jobs.size(),
            lead_pages.size(), double(tp->bytes) / 1e6, tp->build_ms);
  if (const char* vb = getenv("PQB_VERBOSE"); vb && vb[0] == '2')   // the numbering itself (first 4 096 tuples)
    for (uint32_t t = 0; t < std::min<uint32_t>(tp->n_tuples, 4096); t++)
      fprintf(stderr, "[pqb] tuple %u: mixed-radix id %u, %u rows\n", t, wide[t], counts[wide[t]]);
  slot = tp;
  return tp;
}

std::shared_ptr<const FlatPageRec> Table::tuple_page_table(const TuplePages& tp, cudaStream_t stream) const {
  std::lock_guard<std::mutex> lk(side_mu);
  if (tp.d_pages && tp.pages_ver == agg_pages_ver) return tp.d_pages;
  std::vector<FlatPageRec> recs = agg_pages;
  if (recs.empty()) {
    FlatPageRec blank{};
    blank.voff = ~0ull;
    recs.assign(pages.size(), blank);
  }
  for (const auto& pr : tp.recs) recs[pr.first] = pr.second;
  FlatPageRec* p = nullptr;
  if (!try_alloc((void**)&p, recs.size() * sizeof(FlatPageRec), stream)) return nullptr;
  PQB_CUDA(cudaMemcpyAsync(p, recs.data(), recs.size() * sizeof(FlatPageRec), cudaMemcpyHostToDevice, stream));
  PQB_CUDA(cudaStreamSynchronize(stream));
  tp.d_pages = std::shared_ptr<const FlatPageRec>(p, [](const FlatPageRec* q) { cudaFree(const_cast<FlatPageRec*>(q)); });
  tp.pages_ver = agg_pages_ver;
  return tp.d_pages;
}

void launch_entry_offsets(const Table& t, int tcol, uint64_t* d_out, uint32_t* max_len, cudaStream_t stream) {
  std::vector<EntChunk> ch = column_chunks(t, tcol);
  if (ch.empty()) return;
  DevBuf<EntChunk> d_ch; d_ch.upload(ch, stream);
  DevBuf<unsigned int> d_err; d_err.alloc(2, stream); d_err.zero();
  k_dict_entry_offsets<<<uint32_t((ch.size() + 3) / 4), 128, 0, stream>>>(t.d_arena, d_ch.p, uint32_t(ch.size()), t.columns[tcol].kind, d_out, d_err.p);
  PQB_CUDA(cudaGetLastError());
  unsigned int errs[2] = {0, 0};
  PQB_CUDA(cudaMemcpyAsync(errs, d_err.p, 8, cudaMemcpyDeviceToHost, stream));
  PQB_CUDA(cudaStreamSynchronize(stream));
  const unsigned int err = errs[0];
  if (max_len) *max_len = t.columns[tcol].kind == DK_STR ? errs[1] : 8u;
  if (err) throw Error(PQ_ERR_CORRUPT, "column '" + t.columns[tcol].name + "': a string dictionary page runs past its end");
}

// GROUP BY key interning of one table column: every dictionary entry of every row group gets the
// dense id of its VALUE (DataFusion's GroupValues, SURVEY §8 a12), ids numbered hot-first from a
// sample of the column, and the distinct values are packed for the result batches.
void build_key_side(const Table& t, int tcol, ColSide& side, cudaStream_t stream) {
  const uint8_t kkind = t.columns[tcol].kind;
  std::vector<EntChunk> ch = column_chunks(t, tcol);
  const uint32_t nrg = uint32_t(ch.size());
  const uint32_t n = side.total_entries;
  // ---- pages without a dictionary: their rows are entries too ----
  std::vector<RowPage> rowpages;
  side.key_row_pages.clear();
  side.n_dict_pad = (n + 3u) & ~3u;
  uint64_t row_entries = 0;
  for (uint32_t g = 0; g < nrg; g++) {
    const TableChunk& tc = t.row_groups[g].chunks[tcol];
    if (!tc.present) continue;
    for (uint32_t k = 0; k < tc.pages.n_pages; k++) {
      const uint32_t pi = tc.pages.first_page + k;
      const DevPage& dp = t.pages[pi];
      if (dp.enc == DE_DICT || dp.enc == DE_RLE_BOOL) continue;
      const FlatPageRec* fr = pi < t.flat_pages.size() ? &t.flat_pages[pi] : nullptr;
      if (!fr || (fr->fkind != FK_PLAIN8 && fr->fkind != FK_BYTES))
        throw Error(PQ_ERR_UNSUPPORTED, "GROUP BY column '" + t.columns[tcol].name + "': a page without a dictionary has no flat-store copy to take the keys from");
      rowpages.push_back(RowPage{fr->off, fr->voff, fr->base, fr->rows, uint32_t(row_entries), fr->fkind, 0u});
      side.key_row_pages.push_back({pi, uint32_t(row_entries)});
      row_entries += (uint64_t(fr->rows) + 3u) & ~3ull;
    }
  }
  if (uint64_t(side.n_dict_pad) + row_entries > 0xfffffff0ull) throw Error(PQ_ERR_UNSUPPORTED, "GROUP BY column '" + t.columns[tcol].name + "': more than 2^32 key entries");
  const uint32_t n_all = rowpages.empty() ? n : uint32_t(side.n_dict_pad + row_entries);
  side.key_entries = n_all;
  PQB_CUDA(cudaMallocAsync((void**)&side.d_gid, std::max<uint64_t>(n_all, 1) * 4, stream));
  PQB_CUDA(cudaMemsetAsync(side.d_gid, 0, std::max<uint64_t>(n_all, 1) * 4, stream));
  side.card = 0;
  side.kd = KeyDict{};
  side.kd.offs.assign(1, 0);
  if (!n_all || !nrg) { PQB_CUDA(cudaStreamSynchronize(stream)); return; }
  DevBuf<EntChunk> d_ch; d_ch.upload(ch, stream);
  DevBuf<RowPage> d_rp;
  if (!rowpages.empty()) {
    d_rp.upload(rowpages, stream);
    PQB_CUDA(cudaMallocAsync((void**)&side.d_row_ent, row_entries * 8, stream));
    PQB_CUDA(cudaMemsetAsync(side.d_row_ent, 0xff, row_entries * 8, stream));   // padding between pages: no entry
    k_row_entries<<<uint32_t(std::min<size_t>(rowpages.size(), 65535)), 256, 0, stream>>>(t.d_flat, d_rp.p, uint32_t(rowpages.size()),
                                                                                         uint64_t(t.d_flat) - uint64_t(t.d_arena), side.d_row_ent);
    PQB_CUDA(cudaGetLastError());
  }
  const EntView ent{side.d_ent_off, side.d_row_ent, rowpages.empty() ? n : side.n_dict_pad};
  const uint32_t maxn = std::max<uint32_t>(side.max_dict_n, 1);
  uint64_t cap = 64;
  while (cap < 4ull * maxn) cap <<= 1;
  while (cap < std::min<uint64_t>(2 * row_entries, 1ull << 22)) cap <<= 1;   // rows: start where a column of mostly distinct values needs few redos
  DevBuf<uint32_t> rep;
  uint32_t card = 0, rebuilds = 0;
  for (;;) {
    DevBuf<unsigned long long> slots; slots.alloc(cap, stream); slots.zero();
    DevBuf<uint32_t> gid_of_slot; gid_of_slot.alloc(cap, stream);
    DevBuf<uint32_t> rep_try; rep_try.alloc(cap, stream);
    DevBuf<uint32_t> counter; counter.alloc(2, stream); counter.zero();
    DevKeyTable kt{slots.p, gid_of_slot.p, rep_try.p, counter.p, uint32_t(cap - 1), kkind, ent, side.d_gid};
    const uint32_t gy = std::min<uint32_t>((maxn + 255) / 256, 64);
    for (int mode = 0; mode < 2; mode++) {
      for (uint32_t c0 = 0; n && c0 < nrg; c0 += 32768) {
        dim3 grid(std::min<uint32_t>(32768, nrg - c0), gy);
        k_key_intern<<<grid, 256, 0, stream>>>(t.d_arena, d_ch.p, c0, kt, mode);
      }
      if (!rowpages.empty())
        k_row_intern<<<uint32_t(std::min<size_t>(rowpages.size(), 65535)), 256, 0, stream>>>(t.d_arena, d_rp.p, uint32_t(rowpages.size()), kt, mode);
    }
    PQB_CUDA(cudaGetLastError());
    uint32_t cnt[2];
    PQB_CUDA(cudaMemcpyAsync(cnt, counter.p, 8, cudaMemcpyDeviceToHost, stream));
    PQB_CUDA(cudaStreamSynchronize(stream));
    if (cnt[1] == 1 || cnt[0] * 2ull > cap) {  // table too full: grow and redo
      if (cap > (1ull << 30)) throw Error(PQ_ERR_UNSUPPORTED, "GROUP BY key table overflow");
      cap <<= 2;
      rebuilds++;
      continue;
    }
    if (cnt[1]) throw Error(PQ_ERR_CUDA, "group key lookup failed");
    card = cnt[0];
    rep.alloc(std::max<uint32_t>(card, 1), stream);
    PQB_CUDA(cudaMemcpyAsync(rep.p, rep_try.p, size_t(card) * 4, cudaMemcpyDeviceToDevice, stream));
    PQB_CUDA(cudaStreamSynchronize(stream));
    break;
  }
  side.card = card;
  if (const char* vb = getenv("PQB_VERBOSE"); vb && vb[0] && vb[0] != '0')
    fprintf(stderr, "[pqb] key column %s: card %u, %u dictionary entries + %llu rows, table capacity %llu, %u rebuilds\n",
            t.columns[tcol].name.c_str(), card, n, (unsigned long long)row_entries, (unsigned long long)cap, rebuilds);
  // ---- hot-first numbering: occurrences of every id over a sample of the column's flat pages ----
  if (card > 1 && t.d_flat_pages) {
    std::vector<KeySamplePage> sp;
    std::vector<uint32_t> cand;
    for (uint32_t g = 0; g < nrg; g++) {
      const TableChunk& tc = t.row_groups[g].chunks[tcol];
      if (!tc.present) continue;
      for (uint32_t k = 0; k < tc.pages.n_pages; k++)
        if (t.flat_pages[tc.pages.first_page + k].fkind == FK_INDEX) { cand.push_back(g); cand.push_back(tc.pages.first_page + k); }
    }
    const size_t npg = cand.size() / 2, want = std::min<size_t>(npg, 192);
    for (size_t i = 0; i < want; i++) {
      const size_t j = i * npg / want;
      const uint32_t g = cand[2 * j], pi = cand[2 * j + 1];
      const FlatPageRec& fr = t.flat_pages[pi];
      sp.push_back({fr.off, std::min<uint32_t>(fr.rows, 2048), fr.bw, side.base_per_rg[g], t.row_groups[g].chunks[tcol].dict_n});
    }
    if (!sp.empty()) {
      DevBuf<KeySamplePage> d_sp; d_sp.upload(sp, stream);
      DevBuf<uint32_t> d_cnt; d_cnt.alloc(card, stream); d_cnt.zero();
      k_key_sample<<<uint32_t(sp.size()), 256, 0, stream>>>(t.d_flat, d_sp.p, uint32_t(sp.size()), side.d_gid, d_cnt.p);
      PQB_CUDA(cudaGetLastError());
      std::vector<uint32_t> cnt(card), hrep(card);
      PQB_CUDA(cudaMemcpyAsync(cnt.data(), d_cnt.p, size_t(card) * 4, cudaMemcpyDeviceToHost, stream));
      PQB_CUDA(cudaMemcpyAsync(hrep.data(), rep.p, size_t(card) * 4, cudaMemcpyDeviceToHost, stream));
      PQB_CUDA(cudaStreamSynchronize(stream));
      std::vector<uint32_t> order(card);
      for (uint32_t i = 0; i < card; i++) order[i] = i;
      // hot first; ties by the representative entry (deterministic for a given table)
      std::sort(order.begin(), order.end(), [&](uint32_t a, uint32_t b) { return cnt[a] != cnt[b] ? cnt[a] > cnt[b] : hrep[a] < hrep[b]; });
      std::vector<uint32_t> remap(card), nrep(card);
      for (uint32_t i = 0; i < card; i++) { remap[order[i]] = i; nrep[i] = hrep[order[i]]; }
      DevBuf<uint32_t> d_remap; d_remap.upload(remap, stream);
      k_gid_remap<<<std::min<uint32_t>(1024, (n_all + 255) / 256), 256, 0, stream>>>(side.d_gid, side.d_gid, n_all, d_remap.p, card);
      PQB_CUDA(cudaMemcpyAsync(rep.p, nrep.data(), size_t(card) * 4, cudaMemcpyHostToDevice, stream));
      PQB_CUDA(cudaStreamSynchronize(stream));
    }
  }
  // ---- pack the distinct values: lengths -> offsets (host) -> bytes ----
  KeyDict& loc = side.kd;
  loc.offs.assign(size_t(card) + 1, 0);
  if (card) {
    DevBuf<uint32_t> lens;
    lens.alloc(card, stream);
    k_key_lens<<<(card + 255) / 256, 256, 0, stream>>>(t.d_arena, ent, rep.p, card, kkind, lens.p);
    std::vector<uint32_t> hl(card);
    PQB_CUDA(cudaMemcpyAsync(hl.data(), lens.p, card * 4ull, cudaMemcpyDeviceToHost, stream));
    PQB_CUDA(cudaStreamSynchronize(stream));
    uint64_t tot = 0;
    for (uint32_t g = 0; g < card; g++) { loc.offs[g] = uint32_t(tot); tot += hl[g]; }
    loc.offs[card] = uint32_t(tot);
    if (tot > 0x7fffffffull) throw Error(PQ_ERR_UNSUPPORTED, "group key strings exceed 2 GiB");
    DevBuf<uint32_t> doffs;
    doffs.upload(loc.offs, stream);
    DevBuf<uint8_t> dbytes;
    dbytes.alloc(std::max<uint64_t>(tot, 1), stream);
    k_key_bytes<<<card, 64, 0, stream>>>(t.d_arena, ent, rep.p, card, kkind, doffs.p, dbytes.p);
    loc.bytes.resize(tot);
    if (tot) PQB_CUDA(cudaMemcpyAsync(loc.bytes.data(), dbytes.p, tot, cudaMemcpyDeviceToHost, stream));
    // the result assembly reads the dictionary on the device
    PQB_CUDA(cudaMallocAsync((void**)&side.d_kd_offs, (size_t(card) + 1) * 4, stream));
    PQB_CUDA(cudaMallocAsync((void**)&side.d_kd_bytes, std::max<uint64_t>(tot, 1), stream));
    PQB_CUDA(cudaMemcpyAsync(side.d_kd_offs, doffs.p, (size_t(card) + 1) * 4, cudaMemcpyDeviceToDevice, stream));
    if (tot) PQB_CUDA(cudaMemcpyAsync(side.d_kd_bytes, dbytes.p, tot, cudaMemcpyDeviceToDevice, stream));
    PQB_CUDA(cudaStreamSynchronize(stream));
    for (uint32_t g = 0; g < card; g++) side.kd_max_len = std::max(side.kd_max_len, hl[g]);
  }
}

// Collective: every rank of the communicator calls it for the same key column at the same time.
void unify_key_side(const Table& t, int tcol, ColSide& cs, cudaStream_t stream) {
  const KeyDict& loc = cs.kd;
  const uint32_t card_l = cs.card;
  const int nr = comm_nranks(), me = comm_rank();
  std::vector<unsigned long long> sizes(size_t(nr) * 2);
  {
    unsigned long long mine[2] = {card_l, loc.bytes.size()};
    DevBuf<unsigned long long> dsend, drecv;
    dsend.alloc(2, stream);
    drecv.alloc(size_t(nr) * 2, stream);
    PQB_CUDA(cudaMemcpyAsync(dsend.p, mine, 16, cudaMemcpyHostToDevice, stream));
    comm_allgather_bytes(dsend.p, drecv.p, 16, stream);
    PQB_CUDA(cudaMemcpyAsync(sizes.data(), drecv.p, size_t(nr) * 16, cudaMemcpyDeviceToHost, stream));
    PQB_CUDA(cudaStreamSynchronize(stream));
  }
  unsigned long long cardmax = 0, bytesmax = 0;
  for (int r = 0; r < nr; r++) { cardmax = std::max(cardmax, sizes[2 * r]); bytesmax = std::max(bytesmax, sizes[2 * r + 1]); }
  const size_t per_rank = ((4 * (cardmax + 1) + bytesmax) + 15) & ~size_t(15);
  std::vector<uint8_t> sendbuf(per_rank, 0), recvbuf(per_rank * nr);
  std::memcpy(sendbuf.data(), loc.offs.data(), loc.offs.size() * 4);
  if (!loc.bytes.empty()) std::memcpy(sendbuf.data() + 4 * (cardmax + 1), loc.bytes.data(), loc.bytes.size());
  {
    DevBuf<uint8_t> dsend, drecv;
    dsend.upload(sendbuf, stream);
    drecv.alloc(per_rank * nr, stream);
    comm_allgather_bytes(dsend.p, drecv.p, per_rank, stream);
    PQB_CUDA(cudaMemcpyAsync(recvbuf.data(), drecv.p, per_rank * nr, cudaMemcpyDeviceToHost, stream));
    PQB_CUDA(cudaStreamSynchronize(stream));
  }
  // ids by first occurrence in rank order: identical content + identical order on every rank.  Views into the received
  // bytes (no copies), one hash probe per value
  std::unordered_map<std::string_view, uint32_t> ids;
  {
    size_t total = 0;
    for (int r = 0; r < nr; r++) total += size_t(sizes[2 * r]);
    ids.reserve(total);
  }
  std::vector<uint32_t> remap(std::max<uint32_t>(card_l, 1), 0);
  KeyDict& glob = cs.glob_kd;
  glob.offs.assign(1, 0);
  glob.bytes.clear();
  for (int r = 0; r < nr; r++) {
    const uint8_t* base = recvbuf.data() + per_rank * r;
    const uint32_t* offs = reinterpret_cast<const uint32_t*>(base);
    const uint8_t* bytes = base + 4 * (cardmax + 1);
    for (unsigned long long i = 0; i < sizes[2 * r]; i++) {
      const std::string_view v(reinterpret_cast<const char*>(bytes + offs[i]), offs[i + 1] - offs[i]);
      auto it = ids.find(v);
      if (it == ids.end()) {
        it = ids.emplace(v, uint32_t(ids.size())).first;
        glob.bytes.insert(glob.bytes.end(), v.begin(), v.end());
        glob.offs.push_back(uint32_t(glob.bytes.size()));
      }
      if (r == me) remap[i] = it->second;
    }
  }
  cs.glob_card = uint32_t(ids.size());
  auto renew = [&](auto*& p, size_t bytes) {
    if (p) PQB_CUDA(cudaFreeAsync(p, stream));
    p = nullptr;
    PQB_CUDA(cudaMallocAsync((void**)&p, std::max<size_t>(bytes, 16), stream));
  };
  const uint32_t n_ent = cs.key_entries ? cs.key_entries : cs.total_entries;   // rows of pages without a dictionary are entries too
  renew(cs.d_glob_gid, size_t(n_ent) * 4);
  renew(cs.d_glob_kd_offs, glob.offs.size() * 4);
  renew(cs.d_glob_kd_bytes, glob.bytes.size());
  cs.glob_kd_rank.reset();   // ranks of the old agreement (a query still sorting with them holds its own reference)
  cs.glob_rank_luts.reset(); // likewise the MIN / MAX rank tables composed from them
  PQB_CUDA(cudaMemcpyAsync(cs.d_glob_kd_offs, glob.offs.data(), glob.offs.size() * 4, cudaMemcpyHostToDevice, stream));
  if (!glob.bytes.empty()) PQB_CUDA(cudaMemcpyAsync(cs.d_glob_kd_bytes, glob.bytes.data(), glob.bytes.size(), cudaMemcpyHostToDevice, stream));
  cs.glob_max_len = 0;
  for (size_t g = 0; g + 1 < glob.offs.size(); g++) cs.glob_max_len = std::max(cs.glob_max_len, glob.offs[g + 1] - glob.offs[g]);
  if (card_l && n_ent) {
    DevBuf<uint32_t> dremap;
    dremap.upload(remap, stream);
    k_gid_remap<<<std::min<uint32_t>(1024, (n_ent + 255) / 256), 256, 0, stream>>>(cs.d_gid, cs.d_glob_gid, n_ent, dremap.p, card_l);
    PQB_CUDA(cudaGetLastError());
  }
  PQB_CUDA(cudaStreamSynchronize(stream));
  (void)t; (void)tcol;
  cs.glob_epoch = comm_epoch();
  cs.glob_ready = true;
}

// MIN / MAX over Utf8 (callers hold side_mu): from the bytewise rank of every group id of the numbering, the rank of
// every dictionary entry (through the numbering's gid LUT) and of every group id, and the group id of every rank.  Every
// table has at least one entry, so that a column without values still hands out valid pointers.
void build_rank_luts(const ColSide& cs, bool agreed, const uint32_t* rank, RankLuts& luts, cudaStream_t stream) {
  const uint32_t card = agreed ? cs.glob_card : cs.card, n_ent = cs.total_entries;
  const uint32_t* gid = agreed ? cs.d_glob_gid : cs.d_gid;
  luts.card = card;
  auto alloc0 = [&](auto*& p, size_t n) {
    PQB_CUDA(cudaMallocAsync((void**)&p, std::max<size_t>(n, 1) * sizeof(*p), stream));
    PQB_CUDA(cudaMemsetAsync(p, 0, std::max<size_t>(n, 1) * sizeof(*p), stream));
  };
  alloc0(luts.ent, n_ent);
  alloc0(luts.ids, card);
  alloc0(luts.inv, card);
  if (card && n_ent) k_rank_compose<<<std::min<uint32_t>(1024, (n_ent + 255) / 256), 256, 0, stream>>>(gid, n_ent, rank, card, luts.ent);
  if (card) k_rank_ids<<<std::min<uint32_t>(1024, (card + 255) / 256), 256, 0, stream>>>(rank, card, luts.ids, luts.inv);
  PQB_CUDA(cudaGetLastError());
  PQB_CUDA(cudaStreamSynchronize(stream));
}

// MIN / MAX over Boolean: the "rank" of a row is its bit (false < true), read through this table like a group id
__device__ const uint64_t kBoolRank[2] = {0, 1};

namespace {

// What an ORDER BY encode step writes for n rows: [nterms][n] order-preserving values and NULL flags, and the value range
// of every term (reset here: min = ~0, max = 0, no flags).
struct OrderBufs {
  DevBuf<unsigned long long> vals;
  DevBuf<uint8_t> nulls;
  DevBuf<OrderRange> ranges;
  OrderBufs(uint32_t nterms, uint32_t n, cudaStream_t stream, PqMetrics& m) {
    vals.alloc(size_t(nterms) * n, stream);
    nulls.alloc(size_t(nterms) * n, stream);
    ranges.upload(std::vector<OrderRange>(nterms, OrderRange{~0ull, 0ull, 0u, 0u}), stream);
    m.h2d_bytes += nterms * sizeof(OrderRange);
  }
};

// LSD radix sort of n rows by 64-bit keys (key[row]), 8-bit digits: per pass tile histograms, one scan of the digit x
// tile matrix and a stable scatter.  ORDER BY sorts its packed words with it, the merge of a hashed GROUP BY under
// PQ_QUERY_ALLREDUCE its wide group ids.  Every buffer is allocated by the constructor, so a caller can time sort()
// as device work only.
struct RadixSort {
  uint32_t n, ntiles;
  DevBuf<uint32_t> hist, ia, ib;
  DevBuf<unsigned long long> base, total;
  RadixSort(uint32_t rows, cudaStream_t stream) : n(rows), ntiles(uint32_t((uint64_t(rows) + kRadixTile - 1) / kRadixTile)) {
    hist.alloc(size_t(256) * ntiles, stream);
    base.alloc(size_t(256) * ntiles, stream);
    total.alloc(1, stream);
    ia.alloc(n, stream);
    ib.alloc(n, stream);
  }
  // one pass per digit of bits [lo, hi) of key[row], the rows taken in the order `cur` (nullptr: 0 .. n - 1).  Stable,
  // so a sort by a more significant key after this one keeps this order among its ties.  Returns the sorted rows (`cur`
  // itself when there are no bits)
  const uint32_t* sort(const unsigned long long* key, const uint32_t* cur, uint32_t lo, uint32_t hi, cudaStream_t stream, uint64_t& launches) {
    for (uint32_t sh = lo; sh < hi; sh += 8) {
      uint32_t* out = cur == ia.p ? ib.p : ia.p;
      k_radix_hist<<<ntiles, kRadixThreads, 0, stream>>>(key, cur, n, sh, hist.p, ntiles);
      k_item_prefix<<<1, 1024, 0, stream>>>(hist.p, 256 * ntiles, base.p, total.p);
      k_radix_scatter<<<ntiles, kRadixThreads, 0, stream>>>(key, cur, n, sh, base.p, ntiles, out);
      launches += 3;
      cur = out;
    }
    return cur;
  }
};

// A hashed GROUP BY under PQ_QUERY_ALLREDUCE (hash_merge.cuh): every rank's groups gathered and merged into one table of
// the layout k_flat_agg leaves, which then replaces acc / hkeys, so the result tail runs on it unchanged.  Its capacity
// (plan.nslots) is the groups every rank listed; the G merged groups take the first slots in ascending wide id, the slots
// past them hold count 0.  One host round trip, on the exchange records: any rank's full table or corrupt page, and an
// exchange above half the smallest free HBM of any rank, are refused by every rank alike before the cells travel.
struct MergeRun {
  Timer t_rec, t_merge, t_sort, t_fold;
  uint64_t listed = 0, e_max = 0, total = 0;

  uint64_t run(DevPlan& plan, uint32_t cells, uint64_t key_space, uint64_t out_cap, DevBuf<unsigned long long>& acc,
               DevBuf<unsigned long long>& hkeys, const unsigned long long* counters, cudaStream_t stream, PqMetrics& m) {
    const uint32_t nr = uint32_t(comm_nranks()), me = uint32_t(comm_rank());
    // ---- this rank's groups (the cells with rows, in slot order) and its exchange record ----
    const uint32_t ntiles = (plan.nslots + kSlotTile - 1) / kSlotTile;
    DevBuf<uint32_t> tile_counts, out_slot;
    DevBuf<unsigned long long> tile_base, d_listed, rec, recs;
    tile_counts.alloc(ntiles, stream);
    tile_base.alloc(ntiles, stream);
    out_slot.alloc(out_cap, stream);
    d_listed.alloc(1, stream);
    rec.alloc(kMergeRecWords, stream);
    recs.alloc(size_t(kMergeRecWords) * nr, stream);
    size_t free_b = 0, total_b = 0;
    PQB_CUDA(cudaMemGetInfo(&free_b, &total_b));
    uint64_t budget = free_b / 2;
    if (const char* e = getenv("PQB_MERGE_BUDGET")) budget = std::min<uint64_t>(budget, strtoull(e, nullptr, 10));   // test switch: bytes
    PQB_CUDA(cudaEventRecord(t_rec.a, stream));
    k_slot_tile_counts<<<ntiles, 256, 0, stream>>>(acc.p, plan.nslots, tile_counts.p, nullptr);
    k_item_prefix<<<1, 1024, 0, stream>>>(tile_counts.p, ntiles, tile_base.p, d_listed.p);
    k_slot_compact<<<ntiles, 256, 0, stream>>>(acc.p, plan.nslots, tile_base.p, out_slot.p, nullptr);
    k_merge_record<<<1, 1, 0, stream>>>(rec.p, d_listed.p, counters, budget);
    PQB_CUDA(cudaGetLastError());
    comm_allgather_bytes(rec.p, recs.p, kMergeRecWords * 8, stream);
    PQB_CUDA(cudaEventRecord(t_rec.b, stream));
    std::vector<unsigned long long> h(size_t(kMergeRecWords) * nr);
    PQB_CUDA(cudaMemcpyAsync(h.data(), recs.p, h.size() * 8, cudaMemcpyDeviceToHost, stream));
    PQB_CUDA(cudaStreamSynchronize(stream));
    m.d2h_bytes += h.size() * 8;
    // ---- the verdicts: every rank holds the same records ----
    std::vector<unsigned long long> pre(nr + 1, 0);
    int full = -1, corrupt = -1;
    uint32_t low = 0;   // the rank with the smallest budget
    for (uint32_t r = 0; r < nr; r++) {
      const unsigned long long* x = &h[size_t(kMergeRecWords) * r];
      pre[r + 1] = pre[r] + x[kMergeListed];
      e_max = std::max<uint64_t>(e_max, x[kMergeListed]);
      if (x[kMergeFull] && full < 0) full = int(r);
      if (x[kMergeCorrupt] && corrupt < 0) corrupt = int(r);
      if (x[kMergeBudget] < h[size_t(kMergeRecWords) * low + kMergeBudget]) low = r;
    }
    listed = h[size_t(kMergeRecWords) * me + kMergeListed];
    total = pre[nr];
    if (full >= 0)
      throw Error(PQ_ERR_UNSUPPORTED, "GROUP BY: more distinct groups than the hashed accumulator table holds (2^26), on rank " + std::to_string(full));
    if (corrupt >= 0)
      throw Error(PQ_ERR_CORRUPT, "corrupt or unsupported page encoding met on the device of rank " + std::to_string(corrupt) + " (code " +
                                      std::to_string(h[size_t(kMergeRecWords) * corrupt + kMergeCorrupt]) + ")");
    if (total > 0xffffffffull) throw Error(PQ_ERR_UNSUPPORTED, "GROUP BY: the ranks' hashed tables list more than 2^32 - 1 groups together");
    // send and receive blocks, the sort's keys and its buffers, the merged table
    const uint64_t need = 8 * (1 + uint64_t(cells)) * e_max * (nr + 1) + total * (8 + 8 + 8 * (1 + uint64_t(cells))) +
                          (total / kRadixTile + 1) * 256 * 12;
    const uint64_t low_budget = h[size_t(kMergeRecWords) * low + kMergeBudget];
    if (need > low_budget)
      throw Error(PQ_ERR_OOM, "GROUP BY: merging the ranks' hashed tables needs " + std::to_string(need >> 20) +
                                  " MiB of HBM, more than its budget on rank " + std::to_string(low) + ": half the free HBM (" +
                                  std::to_string(low_budget >> 20) + " MiB)");
    // ---- the cells travel, then the merge ----
    const uint32_t n = uint32_t(total), cap = std::max<uint32_t>(n, 1), mt = (n + kSlotTile - 1) / kSlotTile;
    const uint64_t block = (1 + uint64_t(cells)) * e_max;
    DevBuf<unsigned long long> send, recv, ids, d_pre, macc, mwide, mbase, groups;
    DevBuf<uint32_t> mtiles;
    send.alloc(block, stream);
    recv.alloc(block * nr, stream);
    ids.alloc(n, stream);
    d_pre.upload(pre, stream);
    m.h2d_bytes += pre.size() * 8;
    macc.alloc(size_t(cells) * cap, stream);
    mwide.alloc(cap, stream);
    mtiles.alloc(mt, stream);
    mbase.alloc(mt, stream);
    groups.alloc(1, stream);
    RadixSort rs(n, stream);
    PQB_CUDA(cudaMemsetAsync(macc.p, 0, size_t(cap) * 8, stream));   // the count plane: slots past G hold no group
    uint64_t launches = 4;
    PQB_CUDA(cudaEventRecord(t_merge.a, stream));
    if (listed) {
      k_hash_pack<<<uint32_t(std::min<uint64_t>(2048, (listed + 255) / 256)), 256, 0, stream>>>(acc.p, hkeys.p, plan.nslots, cells, out_slot.p,
                                                                                             uint32_t(listed), e_max, send.p);
      launches++;
    }
    if (e_max) comm_allgather_bytes(send.p, recv.p, block * 8, stream);   // e_max is the same on every rank
    HashMergeArgs a{};
    a.recv = recv.p;
    a.pre = d_pre.p;
    a.ids = ids.p;
    a.acc = macc.p;
    a.wide = mwide.p;
    a.e_max = e_max;
    a.nranks = nr;
    a.n = n;
    a.cap = cap;
    a.cells = cells;
    a.n_acc = plan.n_acc;
    std::memcpy(a.acc_init, plan.acc_init, sizeof(a.acc_init));
    if (n) k_merge_list<<<std::min<uint32_t>(2048, (n + 255) / 256), 256, 0, stream>>>(a, ids.p);
    PQB_CUDA(cudaEventRecord(t_sort.a, stream));
    if (n) a.sorted = rs.sort(ids.p, nullptr, 0, 64 - __builtin_clzll(key_space - 1), stream, launches);   // wide ids < key_space
    PQB_CUDA(cudaEventRecord(t_sort.b, stream));
    PQB_CUDA(cudaEventRecord(t_fold.a, stream));
    if (n) {
      k_merge_heads<<<mt, 256, 0, stream>>>(a, mtiles.p);
      k_item_prefix<<<1, 1024, 0, stream>>>(mtiles.p, mt, mbase.p, groups.p);
      a.tile_base = mbase.p;
      k_merge_fold<<<mt, 256, 0, stream>>>(a);
      launches += 4;
    }
    PQB_CUDA(cudaEventRecord(t_fold.b, stream));
    PQB_CUDA(cudaEventRecord(t_merge.b, stream));
    PQB_CUDA(cudaGetLastError());
    std::swap(acc.p, macc.p);   // the rank's own table is freed with macc
    std::swap(acc.n, macc.n);
    std::swap(hkeys.p, mwide.p);
    std::swap(hkeys.n, mwide.n);
    plan.nslots = cap;
    return launches;
  }

  // after the caller's stream synchronise: allreduce_ms (the exchange, the all-gather and the merge kernels, without the
  // round trip between them), and with PQB_VERBOSE the sizes and the merge kernels' time
  void report(bool verbose, uint32_t groups, PqMetrics& m) {
    float rec_ms = 0, merge_ms = 0, sort_ms = 0, fold_ms = 0;
    cudaEventElapsedTime(&rec_ms, t_rec.a, t_rec.b);
    cudaEventElapsedTime(&merge_ms, t_merge.a, t_merge.b);
    cudaEventElapsedTime(&sort_ms, t_sort.a, t_sort.b);
    cudaEventElapsedTime(&fold_ms, t_fold.a, t_fold.b);
    m.allreduce_ms = double(rec_ms) + double(merge_ms);
    if (verbose)
      fprintf(stderr, "[pqb] hashed merge: E_r %llu, E_max %llu, listed by all ranks %llu, G %u, exchange %.3f ms, merge %.3f ms "
              "(sort %.3f ms, fold %.3f ms)\n", (unsigned long long)listed, (unsigned long long)e_max, (unsigned long long)total,
              groups, rec_ms, merge_ms, sort_ms, fold_ms);
  }
};

// ORDER BY [LIMIT] of n encoded rows (groups or selected scan rows), after the caller's encode step.  One round trip: the
// value ranges the pack plan is sized from.  Then `kept` becomes the first `keep` rows in the query's order, as their
// entries of `rows` (nullptr: the row indices themselves); it stays empty when every term is one value for every row
// (the row order is the order).  The kernels are timed by `t_sort` (every buffer is allocated before the events, so the
// span holds device work only); *sort_timed says whether it was recorded.  Returns the kernels it launched.
uint64_t order_sort(const OrderBufs& ob, uint32_t nterms, uint32_t n, const uint8_t* nulls_first, uint32_t keep, const uint32_t* rows,
                    DevBuf<uint32_t>& kept, cudaStream_t stream, PqMetrics& m, Timer& t_sort, bool* sort_timed,
                    const char** path_name = nullptr) {
  uint64_t launches = 0;
  *sort_timed = false;
  std::vector<OrderRange> hr(nterms);
  PQB_CUDA(cudaMemcpyAsync(hr.data(), ob.ranges.p, hr.size() * sizeof(OrderRange), cudaMemcpyDeviceToHost, stream));
  PQB_CUDA(cudaStreamSynchronize(stream));
  m.d2h_bytes += hr.size() * sizeof(OrderRange);
  OrderPack pk{};
  order_pack_plan(hr.data(), nulls_first, nterms, pk);
  if (pk.nwords == 0) return launches;   // every term is one value for every row: the row order is the order
  // the path: the one-CTA sort when every row fits it, top-K when one word holds the key and the kept rows fit the CTA
  // sort, else the radix sort.  PQB_ORDER_PATH=cta|topk|sort (experiment switch) forces a path where it is legal.
  const char* e = getenv("PQB_ORDER_PATH");
  const std::string want = e ? e : "";
  const bool cta_ok = n <= kOrderCta, topk_ok = pk.nwords == 1 && keep <= kOrderCta;
  enum { P_CTA, P_TOPK, P_SORT } path = cta_ok ? P_CTA : topk_ok ? P_TOPK : P_SORT;
  if (want == "sort") path = P_SORT;
  else if (want == "topk" && topk_ok) path = P_TOPK;
  else if (want == "cta" && cta_ok) path = P_CTA;
  if (path_name) *path_name = path == P_CTA ? "cta" : path == P_TOPK ? "topk" : "sort";
  const uint32_t grid_n = uint32_t((uint64_t(n) + 255) / 256);
  DevBuf<unsigned long long> words;
  words.alloc(size_t(pk.nwords) * n, stream);
  kept.alloc(keep, stream);
  const int smem = int(kOrderCta * (8 + 4));
  if (path != P_SORT) PQB_CUDA(cudaFuncSetAttribute(k_order_cta, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
  if (path == P_CTA) {
    PQB_CUDA(cudaEventRecord(t_sort.a, stream));
    k_order_pack<<<grid_n, 256, 0, stream>>>(pk, ob.vals.p, ob.nulls.p, n, words.p);
    k_order_cta<<<1, 1024, smem, stream>>>(words.p, n, pk.nwords, nullptr, n, keep, rows, kept.p);
    launches += 2;
  } else if (path == P_TOPK) {
    const uint32_t ntiles = uint32_t((uint64_t(n) + kSlotTile - 1) / kSlotTile);
    DevBuf<TopkSel> sel;
    DevBuf<uint32_t> tile_counts, cand, count;
    DevBuf<unsigned long long> tile_base, total;
    sel.alloc(1, stream);
    tile_counts.alloc(ntiles, stream);
    tile_base.alloc(ntiles, stream);
    total.alloc(1, stream);
    cand.alloc(keep, stream);
    count.alloc(1, stream);
    TopkSel init{};
    init.k = keep;
    PQB_CUDA(cudaMemcpyAsync(sel.p, &init, sizeof(TopkSel), cudaMemcpyHostToDevice, stream));
    count.zero();
    m.h2d_bytes += sizeof(TopkSel);
    const uint32_t hgrid = std::min<uint32_t>(grid_n, uint32_t(Context::get().sm_count()) * 8);
    PQB_CUDA(cudaEventRecord(t_sort.a, stream));
    k_order_pack<<<grid_n, 256, 0, stream>>>(pk, ob.vals.p, ob.nulls.p, n, words.p);
    launches++;
    // MSB digit first over the used bits only (MSB-first packing: bits [64 - total_bits, 64)); the lowest digit starts at
    // the lowest used bit, the highest may reach past bit 63 (those bits are zero)
    const uint32_t lo = 64 - pk.total_bits, ndig = (pk.total_bits + 7) / 8;
    for (int dg = int(ndig) - 1; dg >= 0; dg--) {
      const uint32_t sh = lo + 8u * uint32_t(dg);
      k_topk_hist<<<hgrid, 256, 0, stream>>>(words.p, n, sh, sel.p);
      k_topk_pick<<<1, 256, 0, stream>>>(sh, sel.p);
      launches += 2;
    }
    k_topk_tile_eq<<<ntiles, 256, 0, stream>>>(words.p, n, sel.p, tile_counts.p);
    k_item_prefix<<<1, 1024, 0, stream>>>(tile_counts.p, ntiles, tile_base.p, total.p);
    k_topk_compact<<<ntiles, 256, 0, stream>>>(words.p, n, sel.p, tile_base.p, cand.p, count.p);
    k_order_cta<<<1, 1024, smem, stream>>>(words.p, n, 1, cand.p, keep, keep, rows, kept.p);
    launches += 4;
  } else {
    RadixSort rs(n, stream);
    PQB_CUDA(cudaEventRecord(t_sort.a, stream));
    k_order_pack<<<grid_n, 256, 0, stream>>>(pk, ob.vals.p, ob.nulls.p, n, words.p);
    launches++;
    const uint32_t* cur = nullptr;   // the first pass reads the rows in row order
    for (int w = int(pk.nwords) - 1; w >= 0; w--) {   // least significant word first
      const uint32_t used = std::min<uint32_t>(64, pk.total_bits - 64u * uint32_t(w));   // MSB-first: the low bits of the last word are empty
      cur = rs.sort(words.p + size_t(w) * n, cur, 64 - used, 64, stream, launches);
    }
    k_order_gather<<<(keep + 255) / 256, 256, 0, stream>>>(cur, keep, rows, kept.p);
    launches++;
  }
  PQB_CUDA(cudaEventRecord(t_sort.b, stream));
  *sort_timed = true;
  PQB_CUDA(cudaGetLastError());
  return launches;
}

// ORDER BY [LIMIT] of an aggregate result: out_slot[0, n) becomes the first `keep` slots in the query's order.  The
// encode kernel is timed by `t_enc`, the sort by `t_sort` (order_sort).  Returns the kernels it launched.
uint64_t order_groups(OrderArgs oa, const uint8_t* nulls_first, uint32_t keep, DevBuf<uint32_t>& out_slot, cudaStream_t stream,
                      PqMetrics& m, Timer& t_enc, Timer& t_sort, bool* sort_timed) {
  OrderBufs ob(oa.nterms, oa.n, stream, m);
  oa.vals = ob.vals.p;
  oa.nulls = ob.nulls.p;
  oa.ranges = ob.ranges.p;
  PQB_CUDA(cudaEventRecord(t_enc.a, stream));
  k_order_encode<<<(oa.n + 255) / 256, 256, 0, stream>>>(oa);
  PQB_CUDA(cudaEventRecord(t_enc.b, stream));
  DevBuf<uint32_t> slots;
  const uint64_t launches = 1 + order_sort(ob, oa.nterms, oa.n, nulls_first, keep, out_slot.p, slots, stream, m, t_sort, sort_timed);
  if (slots.p) {
    std::swap(out_slot.p, slots.p);   // the old list is freed with `slots`
    std::swap(out_slot.n, slots.n);
  }
  return launches;
}

// ORDER BY ... LIMIT on a scan under PQ_QUERY_ALLGATHER (order_kernels.cuh): every rank's first rows gathered and
// ordered alike on every rank, each output row then projected by the rank that holds it.  exchange(): one all-gather
// of a record per rank and one host round trip, after which every rank reaches the same verdicts from the same records
// and throws the same code, naming the rank.  merge(): the candidates' all-gather and their global order.
enum : uint32_t { kScanRecKeep = 0, kScanRecTotal = 1, kScanRecCorrupt = 2, kScanRecBudget = 3, kScanRecRowEnd = 4, kScanRecWords = 5 };
struct ScanMerge {
  uint32_t nr = 0, me = 0, nterms = 0;
  uint64_t keep_r = 0, keep_max = 0, cand = 0, total = 0, keep = 0, row_end = 0;   // cand: the candidates of every rank
  std::vector<uint64_t> str_len;            // the longest string of every projected Utf8 column, over every rank
  std::vector<unsigned long long> pre;      // [nr + 1]: the first candidate of every rank
  Timer t_rec, t_cand, t_sort, t_out;
  bool sort_timed = false, out_timed = false;
  const char* path = "none";                // order_sort's path ("none": every candidate is one key)

  // keep_r / total_r / corrupt: this rank's kept and selected rows and corrupt-page code; row_end_r: one past its
  // largest global row id; str_len_r: its longest string of every projected Utf8 column; row_bytes: result block bytes
  // per output row besides the strings.  Throws the agreed verdicts.
  void exchange(uint32_t terms, uint64_t keep_rank, uint64_t total_r, uint64_t corrupt, uint64_t row_end_r,
                const std::vector<uint64_t>& str_len_r, uint64_t lim, uint64_t row_bytes, cudaStream_t stream, PqMetrics& m) {
    nr = uint32_t(comm_nranks());
    me = uint32_t(comm_rank());
    nterms = terms;
    keep_r = keep_rank;
    const size_t nw = kScanRecWords + str_len_r.size();
    std::vector<unsigned long long> rec(nw, 0), h(nw * nr);
    size_t free_b = 0, total_b = 0;
    PQB_CUDA(cudaMemGetInfo(&free_b, &total_b));
    uint64_t budget = free_b / 2;
    if (const char* e = getenv("PQB_MERGE_BUDGET")) budget = std::min<uint64_t>(budget, strtoull(e, nullptr, 10));   // test switch: bytes
    rec[kScanRecKeep] = keep_r;
    rec[kScanRecTotal] = total_r;
    rec[kScanRecCorrupt] = corrupt;
    rec[kScanRecBudget] = budget;
    rec[kScanRecRowEnd] = row_end_r;
    for (size_t c = 0; c < str_len_r.size(); c++) rec[kScanRecWords + c] = str_len_r[c];
    DevBuf<unsigned long long> d_rec, d_recs;
    d_rec.upload(rec, stream);
    d_recs.alloc(h.size(), stream);
    PQB_CUDA(cudaEventRecord(t_rec.a, stream));
    comm_allgather_bytes(d_rec.p, d_recs.p, nw * 8, stream);
    PQB_CUDA(cudaEventRecord(t_rec.b, stream));
    PQB_CUDA(cudaMemcpyAsync(h.data(), d_recs.p, h.size() * 8, cudaMemcpyDeviceToHost, stream));
    PQB_CUDA(cudaStreamSynchronize(stream));
    m.h2d_bytes += nw * 8;
    m.d2h_bytes += h.size() * 8;
    // ---- the verdicts: every rank holds the same records ----
    pre.assign(nr + 1, 0);
    str_len.assign(str_len_r.size(), 0);
    int corrupt_rank = -1, big_rank = -1;
    for (uint32_t r = 0; r < nr; r++) {
      const unsigned long long* x = &h[nw * r];
      pre[r + 1] = pre[r] + x[kScanRecKeep];
      keep_max = std::max<uint64_t>(keep_max, x[kScanRecKeep]);
      total += x[kScanRecTotal];
      row_end = std::max<uint64_t>(row_end, x[kScanRecRowEnd]);
      if (x[kScanRecCorrupt] && corrupt_rank < 0) corrupt_rank = int(r);
      if (x[kScanRecTotal] > 0xffffffffull && big_rank < 0) big_rank = int(r);
      for (size_t c = 0; c < str_len.size(); c++) str_len[c] = std::max<uint64_t>(str_len[c], x[kScanRecWords + c]);
    }
    cand = pre[nr];
    keep = std::min<uint64_t>(cand, lim);
    if (corrupt_rank >= 0)
      throw Error(PQ_ERR_CORRUPT, "corrupt or unsupported page encoding met on the device of rank " + std::to_string(corrupt_rank) + " (code " +
                                      std::to_string(h[nw * corrupt_rank + kScanRecCorrupt]) + ")");
    if (big_rank >= 0)
      throw Error(PQ_ERR_UNSUPPORTED, "row-level ORDER BY over more than 2^32 - 1 selected rows, on rank " + std::to_string(big_rank));
    if (uint64_t(nr) * keep_max > 0xffffffffull)
      throw Error(PQ_ERR_UNSUPPORTED, "ORDER BY ... LIMIT across ranks: the ranks' kept rows exceed 2^32 - 1 records: lower the LIMIT");
    if (keep > 0x7ffffff0ull) throw Error(PQ_ERR_UNSUPPORTED, "more than 2^31 projected rows in one result: add a LIMIT");
    uint64_t str_bytes = 0;
    for (uint64_t len : str_len) {
      if (keep * len > 0x7fffffffull) throw Error(PQ_ERR_UNSUPPORTED, "projected strings of one result exceed 2 GiB: add a LIMIT");
      str_bytes += keep * len;
    }
    // send and receive blocks; the candidates' ids, records and row-id sort; their terms, the global sort's packed words
    // and its radix sort; the kept order, the owners' handles and the result block
    const uint64_t w = nterms + 2;
    const uint64_t need = 8 * w * keep_max * (nr + 1) + cand * (8 + 4 + 8 + 4 + 9 * uint64_t(nterms) + 8 * (nterms + 1ull) + 8) +
                          2 * (cand / kRadixTile + 1) * 256 * 12 + keep * (4 + 8 + row_bytes) + str_bytes;
    // and on every rank its own sort, which comes first: its selected rows' terms (9 bytes per term), handles, packed words
    // (<= 8 x (nterms + 1)) and radix sort, its kept positions
    for (uint32_t r = 0; r < nr; r++) {
      const uint64_t t = h[nw * r + kScanRecTotal], budget_r = h[nw * r + kScanRecBudget];
      const uint64_t need_r = need + t * (9 * uint64_t(nterms) + 8 + 8 * (nterms + 1ull) + 8 + 4) + (t / kRadixTile + 1) * 256 * 12;
      if (need_r > budget_r)
        throw Error(PQ_ERR_OOM, "ORDER BY ... LIMIT across ranks: the rank's sort and the merge of the ranks' first rows need " +
                                    std::to_string(need_r >> 20) + " MiB of HBM, more than their budget on rank " + std::to_string(r) +
                                    ": half the free HBM (" + std::to_string(budget_r >> 20) + " MiB)");
    }
  }

  // This rank's first keep_r rows (its encoded terms vals / nulls over its n_sel selected rows, kept: their positions,
  // nullptr: 0 .. keep_r - 1) go out, every rank's come back, and owned[j] becomes the handle of output row j when this
  // rank holds it (~0 otherwise).  Returns the kernels it launched.
  uint64_t merge(const unsigned long long* vals, const uint8_t* nulls, uint32_t n_sel, const uint32_t* kept,
                 const unsigned long long* handles, const DevItem* items, const uint8_t* nulls_first,
                 DevBuf<unsigned long long>& owned, cudaStream_t stream, PqMetrics& m) {
    const uint64_t w = nterms + 2;
    const uint32_t n = uint32_t(cand);
    DevBuf<unsigned long long> send, recv, ids, d_pre;
    DevBuf<uint32_t> rec, rec_at, order;
    send.alloc(keep_max * w, stream);
    recv.alloc(nr * keep_max * w, stream);
    ids.alloc(n, stream);
    rec.alloc(n, stream);
    rec_at.alloc(n, stream);
    d_pre.upload(pre, stream);
    m.h2d_bytes += pre.size() * 8;
    owned.alloc(keep, stream);
    RadixSort rs(n, stream);
    OrderBufs ob(nterms, n, stream, m);
    uint64_t launches = 0;
    PQB_CUDA(cudaEventRecord(t_cand.a, stream));
    if (keep_max) {   // the same on every rank
      k_scan_cand_pack<<<uint32_t(std::min<uint64_t>(2048, (keep_max + 255) / 256)), 256, 0, stream>>>(
          vals, nulls, n_sel, nterms, kept, uint32_t(keep_r), handles, items, keep_max, send.p);
      comm_allgather_bytes(send.p, recv.p, keep_max * w * 8, stream);
      launches++;
    }
    ScanMergeArgs a{recv.p, d_pre.p, keep_max, nr, n, nterms};
    if (n) {
      k_scan_cand_list<<<std::min<uint32_t>(2048, (n + 255) / 256), 256, 0, stream>>>(a, ids.p, rec.p);
      const uint32_t bits = row_end > 1 ? 64 - __builtin_clzll(row_end - 1) : 0;   // global row ids < row_end
      const uint32_t* sorted = rs.sort(ids.p, nullptr, 0, bits, stream, launches);
      k_scan_cand_scatter<<<(n + 255) / 256, 256, 0, stream>>>(a, sorted, rec.p, ob.vals.p, ob.nulls.p, ob.ranges.p, rec_at.p);
      launches += 2;
    }
    PQB_CUDA(cudaEventRecord(t_cand.b, stream));
    PQB_CUDA(cudaGetLastError());
    if (keep) {
      launches += order_sort(ob, nterms, n, nulls_first, uint32_t(keep), rec_at.p, order, stream, m, t_sort, &sort_timed, &path);
      k_scan_owned<<<uint32_t((keep + 255) / 256), 256, 0, stream>>>(order.p ? order.p : rec_at.p, uint32_t(keep), keep_max, me, kept,
                                                                     handles, owned.p);
      launches++;
      PQB_CUDA(cudaGetLastError());
    }
    return launches;
  }

  // after the caller's stream synchronise: allreduce_ms, and with PQB_VERBOSE the sizes, the sort path and the times
  void report(bool verbose, PqMetrics& m) {
    float rec_ms = 0, cand_ms = 0, sort_ms = 0, out_ms = 0;
    cudaEventElapsedTime(&rec_ms, t_rec.a, t_rec.b);
    cudaEventElapsedTime(&cand_ms, t_cand.a, t_cand.b);
    if (sort_timed) cudaEventElapsedTime(&sort_ms, t_sort.a, t_sort.b);
    if (out_timed) cudaEventElapsedTime(&out_ms, t_out.a, t_out.b);
    m.allreduce_ms = double(rec_ms) + double(cand_ms) + double(sort_ms) + double(out_ms);
    if (verbose)
      fprintf(stderr, "[pqb] scan merge: keep_r %llu, keep_max %llu, candidates %llu, kept %llu, sort path %s, exchange %.3f ms, "
              "candidates %.3f ms, sort %.3f ms, projection and reductions %.3f ms\n", (unsigned long long)keep_r,
              (unsigned long long)keep_max, (unsigned long long)cand, (unsigned long long)keep, path, rec_ms, cand_ms, sort_ms, out_ms);
  }
};

// ROW_NUMBER() OVER (PARTITION BY ... ORDER BY ...) cut to a rank range, over n rows whose partition terms and then
// order terms the caller encoded into `ob`.  count() sorts and counts the kept rows; the caller sizes its result from
// that count and calls fill(), which writes the kept rows in output order (their entries of `rows`, or their positions
// with rows == nullptr) and their row_number / partition_rows straight into the caller's result buffers.
//   no partition terms: order_sort keeps the first offset + fetch rows (the top-K select when that is small), and the
//                       kept rows are those after the first `offset` (k_window_number)
//   partition terms:    order_sort orders all n rows, the k_window_* kernels rank and count them; one host round trip
//                       (beside order_sort's own) reads the kept count
struct WindowRun {
  const PqWindow& w;
  uint32_t n, nparts;
  DevBuf<uint32_t> sorted;   // order_sort's rows (empty: the row order is the order)
  WindowArgs a{};
  uint32_t ntiles = 0;
  DevBuf<uint8_t> heads;
  DevBuf<uint32_t> start, tile_counts;
  DevBuf<unsigned long long> part_base, keep_base, totals;
  Timer t_sort, t_cut, t_fill;
  bool sort_timed = false, cut_timed = false, fill_timed = false;
  uint64_t launches = 0;

  WindowRun(const PqWindow& win, uint32_t rows, uint32_t parts) : w(win), n(rows), nparts(parts) {}

  // the rows in the rank range, before any `limit`
  unsigned long long count(const OrderBufs& ob, const uint8_t* nulls_first, const uint32_t* rows, cudaStream_t stream, PqMetrics& m) {
    const unsigned long long lo = uint64_t(w.offset), hi = w.fetch < 0 ? ~0ull : uint64_t(w.offset) + uint64_t(w.fetch);
    if (nparts == 0) {
      const uint32_t keep = uint32_t(std::min<unsigned long long>(n, hi));
      if (keep <= lo) return 0;
      launches += order_sort(ob, uint32_t(ob.ranges.n), n, nulls_first, keep, rows, sorted, stream, m, t_sort, &sort_timed);
      return keep - lo;
    }
    launches += order_sort(ob, uint32_t(ob.ranges.n), n, nulls_first, n, nullptr, sorted, stream, m, t_sort, &sort_timed);
    ntiles = uint32_t((uint64_t(n) + kSlotTile - 1) / kSlotTile);
    heads.alloc(n, stream);
    start.alloc(n, stream);
    tile_counts.alloc(ntiles, stream);
    part_base.alloc(ntiles, stream);
    keep_base.alloc(ntiles, stream);
    totals.alloc(2, stream);
    a.vals = ob.vals.p;
    a.nulls = ob.nulls.p;
    a.perm = sorted.p;
    a.n = n;
    a.nparts = nparts;
    a.lo = lo;
    a.hi = hi;
    a.heads = heads.p;
    a.start = start.p;
    a.tile_counts = tile_counts.p;
    a.part_base = part_base.p;
    a.n_part = totals.p;
    a.keep_base = keep_base.p;
    PQB_CUDA(cudaEventRecord(t_cut.a, stream));
    k_window_heads<<<ntiles, 256, 0, stream>>>(a);
    k_item_prefix<<<1, 1024, 0, stream>>>(tile_counts.p, ntiles, part_base.p, totals.p);
    k_window_starts<<<ntiles, 256, 0, stream>>>(a);
    k_window_count<<<ntiles, 256, 0, stream>>>(a);
    k_item_prefix<<<1, 1024, 0, stream>>>(tile_counts.p, ntiles, keep_base.p, totals.p + 1);
    PQB_CUDA(cudaEventRecord(t_cut.b, stream));
    PQB_CUDA(cudaGetLastError());
    launches += 5;
    cut_timed = true;
    unsigned long long kept = 0;
    PQB_CUDA(cudaMemcpyAsync(&kept, totals.p + 1, 8, cudaMemcpyDeviceToHost, stream));
    PQB_CUDA(cudaStreamSynchronize(stream));
    m.d2h_bytes += 8;
    return kept;
  }

  // the first `cap` kept rows (cap <= count()) into kept[cap]; row_number / partition_rows: nullptr when not asked for
  void fill(const uint32_t* rows, unsigned long long cap, uint32_t* kept, long long* row_number, long long* partition_rows,
            cudaStream_t stream) {
    PQB_CUDA(cudaEventRecord(t_fill.a, stream));
    if (nparts == 0) {   // order_sort's rows already went through `rows`
      k_window_number<<<uint32_t((cap + 255) / 256), 256, 0, stream>>>(cap, uint64_t(w.offset), n, sorted.p ? sorted.p : rows, kept,
                                                                       row_number, partition_rows);
    } else {
      a.rows = rows;
      a.kept = kept;
      a.row_number = row_number;
      a.partition_rows = partition_rows;
      a.cap = cap;
      k_window_compact<<<ntiles, 256, 0, stream>>>(a);
    }
    PQB_CUDA(cudaEventRecord(t_fill.b, stream));
    PQB_CUDA(cudaGetLastError());
    launches++;
    fill_timed = true;
  }

  // CUDA-event time of the sort and the window's kernels (after the caller's stream synchronise)
  double ms() const {
    double t = 0;
    float x = 0;
    if (sort_timed) { cudaEventElapsedTime(&x, t_sort.a, t_sort.b); t += x; }
    if (cut_timed) { cudaEventElapsedTime(&x, t_cut.a, t_cut.b); t += x; }
    if (fill_timed) { cudaEventElapsedTime(&x, t_fill.a, t_fill.b); t += x; }
    return t;
  }
};

// MEDIAN / PERCENTILE_CONT of one column: its n emitted pairs become two ORDER BY terms (slot, key), sorted by order_sort;
// k_pct_pick then writes every non-empty group's results.  The emitted pairs are freed once staged.  The kernels are
// timed (without order_sort's one round trip) into pct_ms.  Returns the kernels it launched.
uint64_t pct_finish(DevBuf<uint32_t>& slots, DevBuf<unsigned long long>& keys, uint32_t n, PctPickArgs pk, const uint32_t* out_slot,
                    uint32_t n_out, unsigned long long* acc, uint32_t nslots, bool f64, cudaStream_t stream, PqMetrics& m, double& pct_ms) {
  OrderBufs ob(2, n, stream, m);
  Timer t_stage, t_sort, t_pick;
  PQB_CUDA(cudaEventRecord(t_stage.a, stream));
  k_pct_stage<<<std::min<uint32_t>(2048, (n + 255) / 256), 256, 0, stream>>>(slots.p, keys.p, n, ob.vals.p, ob.nulls.p, ob.ranges.p);
  PQB_CUDA(cudaEventRecord(t_stage.b, stream));
  slots.alloc(0, stream);   // stream ordered: the sort below may reuse the memory
  keys.alloc(0, stream);
  const uint8_t nulls_first[2] = {0, 0};
  DevBuf<uint32_t> sorted;
  bool sort_timed = false;
  // every pair equal (one group, one value): nothing is sorted and the emission order is the order (sorted stays empty)
  const uint64_t launches = 2 + order_sort(ob, 2, n, nulls_first, n, nullptr, sorted, stream, m, t_sort, &sort_timed);
  pk.vals = ob.vals.p;
  pk.order = sorted.p;
  pk.out_slot = out_slot;
  pk.acc = acc;
  pk.n = n;
  pk.n_out = n_out;
  pk.nslots = nslots;
  pk.f64 = f64 ? 1u : 0u;
  PQB_CUDA(cudaEventRecord(t_pick.a, stream));
  k_pct_pick<<<(n_out + 255) / 256, 256, 0, stream>>>(pk);
  PQB_CUDA(cudaEventRecord(t_pick.b, stream));
  PQB_CUDA(cudaGetLastError());
  PQB_CUDA(cudaStreamSynchronize(stream));
  float ms = 0.0f;
  cudaEventElapsedTime(&ms, t_stage.a, t_stage.b);
  pct_ms += ms;
  if (sort_timed) { cudaEventElapsedTime(&ms, t_sort.a, t_sort.b); pct_ms += ms; }
  cudaEventElapsedTime(&ms, t_pick.a, t_pick.b);
  pct_ms += ms;
  return launches;
}

// ---- the result tail: what the queued scan leaves on the device, turned into result batches ----
// A GROUP BY key of the query
struct QKey { const KeyDict* kd = nullptr; uint32_t card = 0; bool is_bin = false; };

// a window's extra columns: Int64, never NULL, after the other columns of the result
std::vector<std::string> window_columns(const PqWindow* win) {
  std::vector<std::string> names;
  if (win && (win->flags & PQ_WINDOW_ROW_NUMBER)) names.push_back("row_number");
  if (win && (win->flags & PQ_WINDOW_PARTITION_ROWS)) names.push_back("partition_rows");
  return names;
}

// A result block holds every buffer of every batch of a result, in 64-byte aligned regions taken in order: first the NULL
// counts (u32 per column and batch), then per column its validity (words per batch) and its values: 8 bytes per row (4
// for Date32), int32 offsets (rows + 1) for strings, bit-packed words per batch for booleans.  String bytes, window
// columns and the device-only scratch behind the copied part are taken where each result places them.
struct BlockCol {
  std::string name;
  int type = PQ_T_I64;      // PqType
  uint8_t kind = DK_I64;    // DevKind of the layout (DK_I32: a Date32 column, 4-byte values)
  uint64_t valid_off = 0, val_off = 0, data_off = 0;   // data_off: a string column's bytes
};
struct BlockLayout {
  uint64_t rows = 0;        // the rows the block has room for
  uint32_t batch_rows = 1, nbatches = 0, wpb = 0;
  uint32_t ncolumns = 0;    // the columns of the NULL-count table
  uint64_t off = 0, nulls_off = 0;
  uint64_t copy_bytes = 0;  // the part that is copied back
  BlockLayout() = default;
  BlockLayout(uint64_t n, uint32_t br, uint32_t ncol)
      : rows(n), batch_rows(br), nbatches(uint32_t((n + br - 1) / br)), wpb((br + 31) / 32), ncolumns(ncol) {
    nulls_off = take(uint64_t(ncol) * nbatches * 4);
  }
  uint64_t take(uint64_t bytes) { const uint64_t o = off; off = (off + bytes + 63) & ~63ull; return o; }
  uint64_t per_row(uint64_t bytes) { return take(rows * bytes); }
  void column(BlockCol& c) {   // its validity, then its values
    const uint64_t bitmap = uint64_t(nbatches) * wpb * 4;
    c.valid_off = take(bitmap);
    c.val_off = c.kind == DK_BOOL ? take(bitmap) : c.kind == DK_STR ? take((rows + 1) * 4) : per_row(c.kind == DK_I32 ? 4 : 8);
  }
};

// a zeroed block in ordinary memory, for a result laid out on the host (one row, or an empty batch)
std::shared_ptr<PinnedBlock> heap_block(uint64_t bytes) {
  auto b = std::make_shared<PinnedBlock>();
  b->heap.assign(std::max<uint64_t>(bytes / 8, 1), 0);
  b->p = reinterpret_cast<uint8_t*>(b->heap.data());
  b->bytes = b->heap.size() * 8;
  return b;
}

void host_mark(bool verbose, std::chrono::steady_clock::time_point t_begin, const char* what) {   // PQB_VERBOSE: host timeline of a query
  if (verbose)
    fprintf(stderr, "[pqb] +%.3f ms %s\n", std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t_begin).count(), what);
}

// What the result tail reads of the planned query and its queued scan (Query::run fills it), and the tail: one function
// per result shape (groups: an aggregate table; rows: a projection or an ordered scan; selection: selected row ids or
// a COUNT(*) row), then finish() for the timings
struct ResultTail {
  const PqQueryDesc& d;
  const Table* table;
  Shape& shape;
  DevPlan& plan;
  const std::vector<DevItem>& items;
  const std::vector<int>& out_type;     // query column -> its result type (PqType)
  const std::vector<int>& slot_of;      // query column -> column slot
  const std::vector<int>& shape_cols;   // column slot -> table column
  const std::vector<QKey>& qk;
  const std::vector<uint8_t>& nn_is_rows;
  const std::vector<int>& agg_out_type;
  const std::vector<double>& pct_p;
  const std::vector<std::shared_ptr<const RankLuts>>& rank_luts;
  const std::vector<uint8_t>& lit_pool;
  const std::shared_ptr<const TuplePages>& tuple;
  DevBuf<unsigned long long>& d_acc;
  DevBuf<unsigned long long>& d_hkeys;
  DevBuf<unsigned long long>& d_counters;
  DevBuf<uint32_t>& d_bitmap;
  DevBuf<uint32_t>& d_item_counts;
  DevBuf<unsigned int>& d_pct_count;
  std::vector<DevBuf<uint32_t>>& d_pct_slots;
  std::vector<DevBuf<unsigned long long>>& d_pct_keys;
  RowOrderArgs& roa;
  const uint8_t* row_nulls_first;
  DevBuf<FlatPageRec>& d_opages;
  Timer& t_all;
  Timer& t_scan;
  const uint32_t cells, ncols, nrg;
  const uint64_t key_space;
  const bool allreduce, multi, merge_rows;
  uint64_t launches;
  cudaStream_t stream;
  const bool verbose;
  const std::chrono::steady_clock::time_point t_begin;
  PqMetrics& metrics;
  std::vector<OutBatch>& batches;
  std::vector<std::shared_ptr<PinnedBlock>>& dev_blocks;   // result blocks whose device copy is kept until the query closes
  // from the query
  const PqWindow* const win = d.window;
  const uint32_t n_part = win ? win->n_partition_by : 0;
  const bool ordered = d.n_order_by > 0 || win;
  const bool row_order = ordered && !d.n_aggs;
  const bool want_rows = d.n_aggs == 0 && !(d.flags & PQ_QUERY_COUNT_ONLY);
  const uint32_t batch_rows = d.batch_size ? d.batch_size : 20000;
  const unsigned long long lim = d.limit >= 0 ? (unsigned long long)d.limit : ~0ull;
  const std::vector<std::string> win_names = window_columns(win);
  Context& ctx = Context::get();
  // the scan's counters and the rows it selected
  unsigned long long h_counters[4] = {0, 0, 0, 0};
  unsigned long long total = 0;
  DevBuf<unsigned long long> d_item_base, d_total;

  void groups();
  void rows();
  void selection();
  void finish();

  void mark(const char* what) const { host_mark(verbose, t_begin, what); }
  void count_selected();
  void check_corrupt() const;
  std::string agg_name(uint32_t a) const;
  uint8_t agg_kind(uint32_t a) const;
  void keep_device(const std::shared_ptr<PinnedBlock>& block, DevBuf<uint8_t>& d_block, uint64_t bytes);
  template <class Fill>
  unsigned long long sized_pass(unsigned long long min_cap, std::shared_ptr<PinnedBlock>& block, Fill fill, const char* then);
  void one_row(std::vector<BlockCol> cols, const std::vector<bool>& null, unsigned long long value);
  void slice(const BlockLayout& L, const std::vector<BlockCol>& cols, const std::shared_ptr<PinnedBlock>& block, uint64_t n);
};

}  // namespace

void Query::run(const PqQueryDesc& d) {
  const auto t_begin = std::chrono::steady_clock::now();
  const char* vb = getenv("PQB_VERBOSE"); const bool verbose = vb && vb[0] && vb[0] != '0';
  auto mark = [&](const char* what) { host_mark(verbose, t_begin, what); };
  struct HostTimer {
    std::chrono::steady_clock::time_point t0;
    PqMetrics* m;
    ~HostTimer() { m->host_ms = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count(); }
  } host_timer{t_begin, &metrics};
  Context& ctx = Context::get();
  ctx.ensure();
  if (d.n_columns > (uint32_t)kMaxCols) throw Error(PQ_ERR_UNSUPPORTED, "too many referenced columns");
  if (d.n_aggs > (uint32_t)kMaxAggs) throw Error(PQ_ERR_UNSUPPORTED, "too many aggregates");
  if (d.n_group_by > (uint32_t)kMaxKeys) throw Error(PQ_ERR_UNSUPPORTED, "too many GROUP BY columns");
  if (d.n_pred > (uint32_t)kMaxPredOps) throw Error(PQ_ERR_UNSUPPORTED, "predicate program too long");
  if (d.n_group_by && !d.n_aggs) throw Error(PQ_ERR_INVALID_ARG, "GROUP BY without aggregates");
  const PqWindow* win = d.window;   // ROW_NUMBER() OVER (PARTITION BY ... ORDER BY order_by), cut to a rank range
  const bool ordered = d.n_order_by > 0 || win;
  const bool row_order = ordered && !d.n_aggs;   // ORDER BY ... LIMIT on a filter / projection scan: the terms are columns
  const uint32_t n_part = win ? win->n_partition_by : 0;
  if (win) {
    if (win->offset < 0) throw Error(PQ_ERR_INVALID_ARG, "window: offset < 0");
    if (win->flags & ~(PQ_WINDOW_ROW_NUMBER | PQ_WINDOW_PARTITION_ROWS)) throw Error(PQ_ERR_INVALID_ARG, "window: unknown flags");
    if (d.flags & PQ_QUERY_COUNT_ONLY) throw Error(PQ_ERR_INVALID_ARG, "window with PQ_QUERY_COUNT_ONLY: a count has no rows to rank");
    if (n_part && !win->partition_by) throw Error(PQ_ERR_INVALID_ARG, "n_partition_by > 0 without partition_by");
    if (uint64_t(n_part) + d.n_order_by > uint64_t(kMaxOrder)) throw Error(PQ_ERR_UNSUPPORTED, "more than 8 PARTITION BY and ORDER BY terms");
  }
  if (ordered) {
    if (d.n_order_by > uint32_t(kMaxOrder)) throw Error(PQ_ERR_UNSUPPORTED, "more than 8 ORDER BY terms");
    if (d.n_order_by && !d.order_by) throw Error(PQ_ERR_INVALID_ARG, "n_order_by > 0 without order_by");
    for (uint32_t t = 0; t < n_part + d.n_order_by; t++) {   // the partition terms, then the order terms
      const PqOrderBy& ob = t < n_part ? win->partition_by[t] : d.order_by[t - n_part];
      const std::string term = t < n_part ? "PARTITION BY term " + std::to_string(t) + ": " : "ORDER BY term " + std::to_string(t - n_part) + ": ";
      if (t < n_part && !row_order && ob.target == PQ_ORDER_AGG) throw Error(PQ_ERR_INVALID_ARG, term + "a partition is a GROUP BY key or a column, not an aggregate");
      if (ob.target != PQ_ORDER_KEY && ob.target != PQ_ORDER_AGG && ob.target != PQ_ORDER_COLUMN) throw Error(PQ_ERR_INVALID_ARG, term + "unknown target");
      if (row_order && ob.target != PQ_ORDER_COLUMN)
        throw Error(PQ_ERR_UNSUPPORTED, term + "ORDER BY on a filter / projection scan orders by columns (PQ_ORDER_COLUMN), not by a GROUP BY key or an aggregate");
      if (!row_order && ob.target == PQ_ORDER_COLUMN)
        throw Error(PQ_ERR_INVALID_ARG, term + "an aggregate query orders by its GROUP BY keys and aggregates, not by a column (PQ_ORDER_COLUMN)");
      const uint32_t n = ob.target == PQ_ORDER_KEY ? d.n_group_by : ob.target == PQ_ORDER_AGG ? d.n_aggs : d.n_columns;
      if (ob.index < 0 || uint32_t(ob.index) >= n)
        throw Error(PQ_ERR_INVALID_ARG, term + (ob.target == PQ_ORDER_KEY ? "GROUP BY" : ob.target == PQ_ORDER_AGG ? "aggregate" : "column") + " index out of range");
    }
    if (row_order && (d.flags & PQ_QUERY_COUNT_ONLY)) throw Error(PQ_ERR_INVALID_ARG, "ORDER BY with PQ_QUERY_COUNT_ONLY: a count has no rows to order");
    if (row_order && d.limit < 0 && !win) throw Error(PQ_ERR_UNSUPPORTED, "row-level ORDER BY needs a LIMIT (limit >= 0)");
  }
  // PQ_QUERY_ALLGATHER: the ranks' first rows of an ordered scan merged into the whole table's (checked alike on every rank)
  if (d.flags & PQ_QUERY_ALLGATHER) {
    if (!comm_active()) throw Error(PQ_ERR_INVALID_ARG, "PQ_QUERY_ALLGATHER without pq_comm_init_rank");
    if (d.n_aggs) throw Error(PQ_ERR_INVALID_ARG, "PQ_QUERY_ALLGATHER on an aggregate query: PQ_QUERY_ALLREDUCE merges aggregates");
    if (d.flags & PQ_QUERY_COUNT_ONLY) throw Error(PQ_ERR_INVALID_ARG, "PQ_QUERY_ALLGATHER with PQ_QUERY_COUNT_ONLY: a count has no rows to merge");
    if (win) throw Error(PQ_ERR_UNSUPPORTED, "PQ_QUERY_ALLGATHER with a window: windows are not merged across ranks");
    if (!row_order) throw Error(PQ_ERR_UNSUPPORTED, "PQ_QUERY_ALLGATHER needs ORDER BY ... LIMIT: an unordered scan is not merged across ranks");
  }
  // every rank's first rows are gathered and merged (with one rank they already are the table's)
  const bool merge_rows = (d.flags & PQ_QUERY_ALLGATHER) && comm_nranks() > 1;

  cudaStream_t stream = ctx.stream_acquire();
  struct StreamGuard { cudaStream_t s; int dev; ~StreamGuard() { Context::get().stream_release(s, dev); } } sg{stream, ctx.device()};

  // ---- input: resident table, or upload the referenced columns of a file list ----
  const Table* table = reinterpret_cast<const Table*>(d.table);
  std::vector<int> tcol(d.n_columns, -1);  // query column -> table column
  if (!table) {
    if (!d.files || !d.n_files) throw Error(PQ_ERR_INVALID_ARG, "query has neither a table nor files");
    std::vector<std::string> names;
    for (uint32_t c = 0; c < d.n_columns; c++) names.push_back(d.columns[c].name ? d.columns[c].name : "");
    owned_table_ = std::make_unique<Table>();
    owned_table_->open(d.files, d.n_files, names, d.shard_index, d.shard_count, stream);
    metrics.upload_ms = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t_begin).count();
    table = owned_table_.get();
    metrics.h2d_bytes += table->h2d_bytes;
  }
  for (uint32_t c = 0; c < d.n_columns; c++) {
    if (!d.columns[c].name) throw Error(PQ_ERR_INVALID_ARG, "column without a name");
    tcol[c] = table->find_column(d.columns[c].name);
    if (tcol[c] < 0) throw Error(PQ_ERR_INVALID_ARG, std::string("column '") + d.columns[c].name + "' is not part of the resident table");
  }

  // ---- column kinds vs the plan's expectation ----
  DevPlan plan{};
  plan.ncols = d.n_columns;
  for (uint32_t c = 0; c < d.n_columns; c++) {
    const TableColumn& tc = table->columns[tcol[c]];
    uint8_t kind = tc.kind;
    int want = d.columns[c].type;
    if (kind == 0xfe) {  // in no file: all NULL, take the plan's type
      kind = want == PQ_T_F64 ? DK_F64 : want == PQ_T_UTF8 ? DK_STR : want == PQ_T_BOOL ? DK_BOOL : DK_I64;
    } else {
      bool ok = (want == PQ_T_I64 && kind == DK_I64 && !tc.is_ts && !tc.is_date) || (want == PQ_T_TS_MS && kind == DK_I64 && tc.is_ts) ||
                (want == PQ_T_F64 && kind == DK_F64) || (want == PQ_T_UTF8 && kind == DK_STR) ||
                (want == PQ_T_BOOL && kind == DK_BOOL) || (want == PQ_T_DATE32 && kind == DK_I64 && tc.is_date) || want == PQ_T_NULL;
      // Int64 plan type also accepts a timestamp column and vice versa (same physical values); a Date32 column is neither
      if (!ok && kind == DK_I64 && !tc.is_date && (want == PQ_T_I64 || want == PQ_T_TS_MS)) ok = true;
      if (!ok) throw Error(PQ_ERR_INVALID_ARG, std::string("column '") + tc.name + "' is not " + type_name(want) + " in the Parquet files");
    }
    plan.cols[c].kind = kind;
    plan.cols[c].max_def = tc.max_def;
  }
  auto out_type_of = [&](uint32_t c) -> int {
    const TableColumn& tc = table->columns[tcol[c]];
    if (d.columns[c].type != PQ_T_NULL) return d.columns[c].type;
    switch (plan.cols[c].kind) { case DK_F64: return PQ_T_F64; case DK_STR: return PQ_T_UTF8; case DK_BOOL: return PQ_T_BOOL;
      default: return tc.is_date ? PQ_T_DATE32 : tc.is_ts ? PQ_T_TS_MS : PQ_T_I64; }
  };
  // Date32 columns (by the plan's type, or the files' when the plan leaves it NULL): Int64 values in every kernel, 4-byte
  // values in the results
  auto is_date = [&](uint32_t c) { return out_type_of(c) == PQ_T_DATE32; };

  // ---- predicate compile ----
  // `col <cmp> lit` with the literal coerced into lf.d.cmp / lit_i64 / str, as PQ_OP_CMP coerces it; PQ_OP_IN coerces
  // each of its elements as the PQ_EQ case
  auto coerce_cmp = [&](HostLeaf& lf, uint32_t qc, int cmp, const PqLiteral& lit) {
    const uint8_t kind = plan.cols[qc].kind;
    lf.d.cmp = uint8_t(cmp);
    // Date32 compares with Date32 only (DataFusion rejects the other pairs or casts both sides to Timestamp)
    if (is_date(qc) != (lit.type == PQ_T_DATE32))
      throw Error(PQ_ERR_UNSUPPORTED, std::string("comparison of the ") + type_name(out_type_of(qc)) + " column '" +
                                          d.columns[qc].name + "' with a " + type_name(lit.type) + " literal is not on the GPU path");
    if (lit.type == PQ_T_DATE32 && (lit.i64 < INT32_MIN || lit.i64 > INT32_MAX))
      throw Error(PQ_ERR_INVALID_ARG, "Date32 literal outside int32 days");
    // literal coercion as DataFusion's type coercion does for column-vs-literal (SURVEY §8 a11)
    switch (kind) {
      case DK_I64:
        if (lit.type == PQ_T_I64 || lit.type == PQ_T_TS_MS || lit.type == PQ_T_DATE32) lf.d.lit_i64 = lit.i64;
        else if (lit.type == PQ_T_F64 && std::nearbyint(lit.f64) == lit.f64 && lit.f64 >= -9223372036854775808.0 && lit.f64 < 9223372036854775808.0)
          lf.d.lit_i64 = int64_t(lit.f64);
        else if (lit.type == PQ_T_F64) {
          // DataFusion coerces the COLUMN to Float64 and compares there.  Against a literal that is no int64 this
          // has an exact integer restatement (a non-integer double is < 2^52 in magnitude, where the cast of
          // any int64 at or beyond it cannot cross it):  v > 100.5  <=>  v > 100,  v < 100.5  <=>  v < 101,
          // v = 100.5 never, v != 100.5 always (for non-NULL v).  A NaN sits by its sign bit (totalOrder): above
          // every value without it, below every value (-inf included) with it.
          const double L = lit.f64;
          const int64_t kMin = std::numeric_limits<int64_t>::min();
          auto never = [&] { lf.d.cmp = PQ_LT; lf.d.lit_i64 = kMin; };    // v < INT64_MIN
          auto always = [&] { lf.d.cmp = PQ_GE; lf.d.lit_i64 = kMin; };   // v >= INT64_MIN
          const bool nan = std::isnan(L);
          const bool above = (nan && !std::signbit(L)) || L >= 9223372036854775808.0;   // greater than every int64
          const bool below = (nan && std::signbit(L)) || L < -9223372036854775808.0;     // less than every int64
          if (L == 9223372036854775808.0) {
            // 2^63: the int64 values from 2^63 - 512 up round to it when cast (to nearest, ties to even), the
            // others cast below it
            const int64_t kTop = std::numeric_limits<int64_t>::max() - 511;
            switch (cmp) {
              case PQ_EQ: case PQ_GE: lf.d.cmp = PQ_GE; lf.d.lit_i64 = kTop; break;
              case PQ_NE: case PQ_LT: lf.d.cmp = PQ_LT; lf.d.lit_i64 = kTop; break;
              case PQ_LE: always(); break;
              default: never(); break;   // PQ_GT
            }
          } else if (above || below) {
            const bool lt = cmp == PQ_LT || cmp == PQ_LE, gt = cmp == PQ_GT || cmp == PQ_GE;
            if (cmp == PQ_EQ) never();
            else if (cmp == PQ_NE) always();
            else if ((above && lt) || (below && gt)) always();
            else never();
          } else {
            const int64_t fl = int64_t(std::floor(L)), ce = fl + 1;   // |L| < 2^52
            switch (cmp) {
              case PQ_EQ: never(); break;
              case PQ_NE: always(); break;
              case PQ_GT: case PQ_GE: lf.d.cmp = PQ_GT; lf.d.lit_i64 = fl; break;
              default: lf.d.cmp = PQ_LT; lf.d.lit_i64 = ce; break;   // PQ_LT, PQ_LE
            }
          }
        } else throw Error(PQ_ERR_INVALID_ARG, "Int64 column compared with a non-numeric literal");
        break;
      case DK_F64:
        if (lit.type == PQ_T_F64) lf.d.lit_i64 = int64_t(f64_bits(lit.f64));
        else if (lit.type == PQ_T_I64) lf.d.lit_i64 = int64_t(f64_bits(double(lit.i64)));  // `status = 200` on a Float64 column
        else throw Error(PQ_ERR_INVALID_ARG, "Float64 column compared with a non-numeric literal");
        break;
      case DK_BOOL:
        if (lit.type != PQ_T_BOOL) throw Error(PQ_ERR_INVALID_ARG, "Boolean column compared with a non-boolean literal");
        lf.d.lit_i64 = lit.i64 ? 1 : 0;
        break;
      case DK_STR:
        if (lit.type != PQ_T_UTF8) throw Error(PQ_ERR_INVALID_ARG, "Utf8 column compared with a non-string literal");
        lf.str.assign(lit.str ? lit.str : "", lit.str_len);
        break;
      default: throw Error(PQ_ERR_UNSUPPORTED, "comparison on this column type");
    }
  };
  std::vector<HostLeaf> leaves;
  std::vector<DevPredOp> prog;
  std::vector<uint8_t> lit_pool(16, 0);
  bool has_null_const = false;
  auto push_leaf = [&](HostLeaf& lf) {
    if (leaves.size() >= (size_t)kMaxLeaves) throw Error(PQ_ERR_UNSUPPORTED, "too many leaf predicates");
    if ((plan.cols[lf.qcol].kind == DK_STR && value_leaf(lf.d.kind)) || lf.d.kind == LK_IN) {
      if (lit_pool.size() + lf.str.size() > 0xfffffff0ull) throw Error(PQ_ERR_UNSUPPORTED, "predicate literals too large");
      lf.d.str_off = uint32_t(lit_pool.size());   // a multiple of 8: the pool starts at 16 and every entry is padded to 8
      lf.d.str_len = uint32_t(lf.str.size());
      lit_pool.insert(lit_pool.end(), lf.str.begin(), lf.str.end());
      lit_pool.resize(align_up(uint32_t(lit_pool.size()) + 8, 8), 0);
    }
    prog.push_back({PK_LEAF, uint8_t(leaves.size())});
    leaves.push_back(std::move(lf));
  };
  // PQ_OP_IN: the Kleene OR of `col = e` over the elements.  Its distinct matching values become one LK_IN leaf (one value:
  // the LK_CMP / PQ_EQ leaf it equals; a Boolean column: a CMP leaf), the one element whose EQ restatement is a range
  // (2^63 against Int64) its CMP leaf OR'd to it, a NULL element `OR NULL`, and NOT IN a NOT.  Pushes one value.
  auto compile_in = [&](const PqPredOp& op, uint32_t qc, int depth) {
    const std::string where = std::string("IN list on '") + d.columns[qc].name + "': ";
    if (op.flags & ~(PQ_IN_NEGATED | PQ_IN_HAS_NULL)) throw Error(PQ_ERR_INVALID_ARG, where + "unknown flags");
    const bool has_null = (op.flags & PQ_IN_HAS_NULL) != 0, negated = (op.flags & PQ_IN_NEGATED) != 0;
    const PqLiteral& lit = op.lit;
    if (lit.i64 < 0) throw Error(PQ_ERR_INVALID_ARG, where + "negative element count");
    if (lit.i64 == 0 && !has_null) throw Error(PQ_ERR_INVALID_ARG, where + "no elements and no NULL");
    if (lit.i64 > int64_t(kInSetMaxElems) || lit.str_len > kInSetMaxBytes)
      throw Error(PQ_ERR_UNSUPPORTED, where + "more than 2^20 elements or 64 MiB of elements");
    const uint32_t n = uint32_t(lit.i64);
    if (n && !lit.str) throw Error(PQ_ERR_INVALID_ARG, where + "str == NULL with elements");
    const uint8_t* p = reinterpret_cast<const uint8_t*>(lit.str);
    const uint8_t kind = plan.cols[qc].kind;
    // the elements: (offset, length) in str for Utf8, else 8 bytes each
    std::vector<const uint8_t*> sp;
    std::vector<uint32_t> sl;
    if (lit.type == PQ_T_UTF8) {
      uint64_t pos = 0;
      for (uint32_t k = 0; k < n; k++) {
        if (pos + 4 > lit.str_len) throw Error(PQ_ERR_INVALID_ARG, where + "element " + std::to_string(k) + " runs past str_len");
        const uint32_t len = load_u32_unaligned(p + pos);
        if (pos + 4 + len > lit.str_len) throw Error(PQ_ERR_INVALID_ARG, where + "element " + std::to_string(k) + " runs past str_len");
        sp.push_back(p + pos + 4);
        sl.push_back(len);
        pos += 4 + uint64_t(len);
      }
      if (pos != lit.str_len) throw Error(PQ_ERR_INVALID_ARG, where + "str_len does not match the elements");
    } else if (lit.str_len != uint64_t(n) * 8) {
      throw Error(PQ_ERR_INVALID_ARG, where + "str_len is not 8 bytes per element");
    }
    // each element coerced as PQ_OP_CMP / PQ_EQ coerces its literal: a value, never equal (Int64 against a non-integral
    // Float64), or, for 2^63 against Int64, the range v >= 2^63 - 511
    std::vector<int64_t> vals;
    bool top = false;
    for (uint32_t k = 0; k < n; k++) {
      PqLiteral el{};
      el.type = lit.type;
      if (lit.type == PQ_T_UTF8) { el.str = reinterpret_cast<const char*>(sp[k]); el.str_len = sl[k]; }
      else std::memcpy(lit.type == PQ_T_F64 ? static_cast<void*>(&el.f64) : static_cast<void*>(&el.i64), p + uint64_t(k) * 8, 8);
      if (lit.type == PQ_T_NULL) throw Error(PQ_ERR_INVALID_ARG, where + "element " + std::to_string(k) + " has no type");
      HostLeaf e;
      try {
        coerce_cmp(e, qc, PQ_EQ, el);
      } catch (const Error& x) {
        throw Error(x.code, where + "element " + std::to_string(k) + ": " + x.what());
      }
      if (kind == DK_STR) break;   // every element is a Utf8 literal: their bytes are the values
      if (e.d.cmp == PQ_EQ) vals.push_back(e.d.lit_i64);
      else if (e.d.cmp == PQ_GE) top = true;
    }
    std::sort(vals.begin(), vals.end());
    vals.erase(std::unique(vals.begin(), vals.end()), vals.end());
    HostLeaf lf;
    lf.qcol = int(qc);
    lf.d.col = uint8_t(qc);
    lf.d.kind = LK_CMP;
    lf.d.cmp = PQ_EQ;
    bool has_leaf = true;
    if (n == 0) {
      has_leaf = false;
    } else if (kind == DK_BOOL) {
      if (vals.size() == 2) { lf.d.cmp = PQ_GE; lf.d.lit_i64 = 0; }   // both: every non-NULL row
      else lf.d.lit_i64 = vals[0];
    } else if (kind == DK_STR) {
      std::vector<uint32_t> ord(n);
      for (uint32_t k = 0; k < n; k++) ord[k] = k;
      auto less = [&](uint32_t a, uint32_t b) { return cmp_bytes(sp[a], sl[a], sp[b], sl[b]) < 0; };
      std::sort(ord.begin(), ord.end(), less);
      ord.erase(std::unique(ord.begin(), ord.end(), [&](uint32_t a, uint32_t b) { return !less(a, b) && !less(b, a); }), ord.end());
      if (ord.size() == 1) {
        lf.str.assign(reinterpret_cast<const char*>(sp[ord[0]]), sl[ord[0]]);
      } else {
        lf.d.kind = LK_IN;
        for (uint32_t k : ord) lf.in_str.emplace_back(reinterpret_cast<const char*>(sp[k]), sl[k]);
        const std::vector<uint8_t> blob = in_set_build_bytes(sp.data(), sl.data(), n);
        lf.str.assign(blob.begin(), blob.end());
      }
    } else if (vals.empty()) {
      if (top) has_leaf = false;
      else { lf.d.cmp = PQ_LT; lf.d.lit_i64 = std::numeric_limits<int64_t>::min(); }   // no element matches a value
    } else if (vals.size() == 1) {
      lf.d.lit_i64 = vals[0];
    } else {
      lf.d.kind = LK_IN;
      if (kind == DK_F64) {
        for (int64_t v : vals) {
          const double x = bits_f64(uint64_t(v));
          if (std::isnan(x)) lf.in_nan = true;
          else lf.in_f64.push_back(x);
        }
        std::sort(lf.in_f64.begin(), lf.in_f64.end());
      } else {
        lf.in_i64 = vals;
      }
      const std::vector<uint8_t> blob = in_set_build_u64(reinterpret_cast<const uint64_t*>(vals.data()), vals.size());
      lf.str.assign(blob.begin(), blob.end());
    }
    if (leaves.size() + (has_leaf ? 1 : 0) + (top ? 1 : 0) > (size_t)kMaxLeaves) throw Error(PQ_ERR_UNSUPPORTED, "too many leaf predicates");
    if (depth + ((has_leaf && top) || has_null ? 2 : 1) > kPredStack) throw Error(PQ_ERR_UNSUPPORTED, "predicate nesting too deep");
    if (has_leaf) push_leaf(lf);
    if (top) {
      HostLeaf t;
      t.qcol = int(qc);
      t.d.col = uint8_t(qc);
      t.d.kind = LK_CMP;
      t.d.cmp = PQ_GE;
      t.d.lit_i64 = std::numeric_limits<int64_t>::max() - 511;
      push_leaf(t);
      if (has_leaf) prog.push_back({PK_OR, 0});
    }
    if (has_null) {
      prog.push_back({PK_CONST, 2});
      has_null_const = true;
      if (has_leaf || top) prog.push_back({PK_OR, 0});
    }
    if (negated && (has_leaf || top)) prog.push_back({PK_NOT, 0});
  };
  {
    int depth = 0;
    for (uint32_t i = 0; i < d.n_pred; i++) {
      const PqPredOp& op = d.pred[i];
      switch (op.kind) {
        case PQ_OP_CMP: case PQ_OP_IS_NULL: case PQ_OP_IS_NOT_NULL: case PQ_OP_LIKE: case PQ_OP_REGEX: {
          if (op.col < 0 || uint32_t(op.col) >= d.n_columns) throw Error(PQ_ERR_INVALID_ARG, "predicate column out of range");
          if (op.kind == PQ_OP_CMP && op.lit.type == PQ_T_NULL) {   // `col <op> NULL` is NULL on every row (SQL)
            prog.push_back({PK_CONST, 2});
            has_null_const = true;
            depth++;
            break;
          }
          if (leaves.size() >= (size_t)kMaxLeaves) throw Error(PQ_ERR_UNSUPPORTED, "too many leaf predicates");
          HostLeaf lf;
          lf.qcol = op.col;
          lf.d.col = uint8_t(op.col);
          uint8_t kind = plan.cols[op.col].kind;
          if (op.kind == PQ_OP_IS_NULL) lf.d.kind = LK_IS_NULL;
          else if (op.kind == PQ_OP_IS_NOT_NULL) lf.d.kind = LK_IS_NOT_NULL;
          else if (op.kind == PQ_OP_LIKE) {
            if (kind != DK_STR) throw Error(PQ_ERR_INVALID_ARG, "LIKE needs a Utf8 column");
            if (op.lit.type != PQ_T_UTF8) throw Error(PQ_ERR_INVALID_ARG, "LIKE needs a Utf8 pattern");
            LikePlan lp = classify_like(std::string(op.lit.str ? op.lit.str : "", op.lit.str_len));
            lf.d.kind = LK_LIKE;
            lf.d.cmp = uint8_t(lp.kind);
            lf.d.flags = op.flags;
            lf.str = lp.needle;
          } else if (op.kind == PQ_OP_REGEX) {
            if (kind != DK_STR) throw Error(PQ_ERR_INVALID_ARG, "a regular expression match needs a Utf8 column");
            if (op.lit.type != PQ_T_UTF8) throw Error(PQ_ERR_INVALID_ARG, "a regular expression match needs a Utf8 pattern");
            std::vector<uint8_t> blob;
            std::string err;
            const int st = regex_compile(op.lit.str, op.lit.str ? op.lit.str_len : 0, (op.flags & PQ_REGEX_CASE_INSENSITIVE) != 0,
                                         blob, err);
            if (st != 0) throw Error(st, err);
            lf.d.kind = LK_REGEX;
            lf.d.flags = op.flags;
            lf.str.assign(blob.begin(), blob.end());   // the DFA travels in the literal pool (8-aligned: see below)
          } else {
            lf.d.kind = LK_CMP;
            if (op.cmp < PQ_EQ || op.cmp > PQ_GE) throw Error(PQ_ERR_INVALID_ARG, "bad comparison operator");
            coerce_cmp(lf, uint32_t(op.col), op.cmp, op.lit);
          }
          push_leaf(lf);
          depth++;
          break;
        }
        case PQ_OP_IN: {
          if (op.col < 0 || uint32_t(op.col) >= d.n_columns) throw Error(PQ_ERR_INVALID_ARG, "predicate column out of range");
          compile_in(op, uint32_t(op.col), depth);
          depth++;
          break;
        }
        case PQ_OP_AND: case PQ_OP_OR:
          if (depth < 2) throw Error(PQ_ERR_INVALID_ARG, "predicate program underflow");
          prog.push_back({uint8_t(op.kind == PQ_OP_AND ? PK_AND : PK_OR), 0});
          depth--;
          break;
        case PQ_OP_NOT:
          if (depth < 1) throw Error(PQ_ERR_INVALID_ARG, "predicate program underflow");
          prog.push_back({PK_NOT, 0});
          break;
        case PQ_OP_CONST:
          prog.push_back({PK_CONST, uint8_t(op.lit.type == PQ_T_NULL ? 2 : (op.lit.i64 ? 1 : 0))});
          has_null_const |= op.lit.type == PQ_T_NULL;
          depth++;
          break;
        default: throw Error(PQ_ERR_INVALID_ARG, "unknown predicate op");
      }
      if (depth > kPredStack) throw Error(PQ_ERR_UNSUPPORTED, "predicate nesting too deep");
    }
    if (d.n_pred && depth != 1) throw Error(PQ_ERR_INVALID_ARG, "predicate program does not reduce to one value");
    if (prog.size() > (size_t)kMaxPredOps) throw Error(PQ_ERR_UNSUPPORTED, "predicate program too long");
  }

  // ---- row-group pruning + constant folding of leaves that statistics decide everywhere ----
  const uint32_t nrg_table = uint32_t(table->row_groups.size());
  std::vector<uint8_t> rg_live(std::max<uint32_t>(nrg_table, 1), 0);
  uint32_t nrg = 0;   // surviving row groups
  std::vector<int> leaf_const(leaves.size(), -1);  // -1 unknown; else Tri over all survivors
  metrics.row_groups_total = nrg_table;
  {
    std::vector<Tri> lt(leaves.size()), st;
    for (uint32_t g = 0; g < nrg_table; g++) {
      const TableRowGroup& rg = table->row_groups[g];
      for (size_t l = 0; l < leaves.size(); l++) {
        const TableChunk& ch = rg.chunks[tcol[leaves[l].qcol]];
        lt[l] = leaf_from_stats(leaves[l], plan.cols[leaves[l].qcol].kind, ch, rg.num_rows);
      }
      Tri root = TRI_TRUE;
      if (!prog.empty()) {
        st.clear();
        for (const DevPredOp& op : prog) {
          if (op.kind == PK_LEAF) st.push_back(lt[op.arg]);
          else if (op.kind == PK_CONST) st.push_back(op.arg == 1 ? TRI_TRUE : TRI_FALSE);
          else if (op.kind == PK_NOT) st.back() = tri_not(st.back());
          else { Tri b = st.back(); st.pop_back(); st.back() = op.kind == PK_AND ? tri_and(st.back(), b) : tri_or(st.back(), b); }
        }
        root = st[0];
      }
      if (root == TRI_FALSE) { metrics.row_groups_pruned++; continue; }
      for (size_t l = 0; l < leaves.size(); l++) {
        if (leaf_const[l] == -1) leaf_const[l] = lt[l];
        else if (leaf_const[l] != lt[l]) leaf_const[l] = TRI_MAYBE;
      }
      rg_live[g] = 1;
      nrg++;
      metrics.rows_scanned += rg.num_rows;
    }
  }
  // a leaf that is TRUE in every surviving row group is replaced by a constant: the injected
  // p_timestamp range filter (src/query/mod.rs:774-833) usually disappears here and its column
  // is then never read.  (A NOT above it is fine: TRUE means "TRUE for every row, no NULLs".)
  std::vector<bool> leaf_live(leaves.size(), true);
  for (DevPredOp& op : prog)
    if (op.kind == PK_LEAF && leaf_const[op.arg] == TRI_TRUE) { leaf_live[op.arg] = false; op = {PK_CONST, 1}; }

  // ---- which columns does the kernel really read? ----
  std::vector<bool> col_used(d.n_columns, false);
  for (size_t l = 0; l < leaves.size(); l++) if (leaf_live[l]) col_used[leaves[l].qcol] = true;
  for (uint32_t k = 0; k < d.n_group_by; k++) {
    if (d.group_by[k] < 0 || uint32_t(d.group_by[k]) >= d.n_columns) throw Error(PQ_ERR_INVALID_ARG, "group-by column out of range");
    col_used[d.group_by[k]] = true;
  }
  for (uint32_t a = 0; a < d.n_aggs; a++) {
    if (d.aggs[a].fn == PQ_AGG_COUNT_STAR) continue;
    if (d.aggs[a].col < 0 || uint32_t(d.aggs[a].col) >= d.n_columns) throw Error(PQ_ERR_INVALID_ARG, "aggregate column out of range");
    col_used[d.aggs[a].col] = true;
  }
  std::vector<bool> col_staged = col_used;   // predicate / key / aggregate inputs: staged per slab by the flat kernels
  const bool want_rows = d.n_aggs == 0 && !(d.flags & PQ_QUERY_COUNT_ONLY);
  for (uint32_t i = 0; want_rows && i < d.n_projection; i++) {
    if (d.projection[i] < 0 || uint32_t(d.projection[i]) >= d.n_columns) throw Error(PQ_ERR_INVALID_ARG, "projection column out of range");
    col_used[d.projection[i]] = true;        // only gathered for the selected rows
  }
  for (uint32_t t = 0; row_order && t < d.n_order_by; t++) col_used[d.order_by[t].index] = true;   // likewise: read for the selected rows
  for (uint32_t t = 0; row_order && t < n_part; t++) col_used[win->partition_by[t].index] = true;
  // compact to kernel column slots
  std::vector<int> slot_of(d.n_columns, -1);
  std::vector<uint32_t> qcol_of_slot;
  for (uint32_t c = 0; c < d.n_columns; c++)
    if (col_used[c]) { slot_of[c] = int(qcol_of_slot.size()); qcol_of_slot.push_back(c); }
  const uint32_t ncols = uint32_t(qcol_of_slot.size());
  {
    DevPlan p2 = plan;
    for (uint32_t s = 0; s < ncols; s++) p2.cols[s] = plan.cols[qcol_of_slot[s]];
    plan = p2;
    plan.ncols = ncols;
  }
  std::vector<int> shape_cols(ncols);
  for (uint32_t s = 0; s < ncols; s++) {
    shape_cols[s] = tcol[qcol_of_slot[s]];
    plan.cols[s].staged = col_staged[qcol_of_slot[s]] ? 1 : 0;
    // the VALUES of a DELTA_BINARY_PACKED column are needed (a range that cuts row groups, a projection of
    // p_timestamp): its pages get row-addressable 8-byte copies, once per table
    if (table->sides[shape_cols[s]].has_delta) table->ensure_plain8(shape_cols[s], stream);
  }
  const bool flat_ok = !(getenv("PQB_FLAT_SCAN") && getenv("PQB_FLAT_SCAN")[0] == '0');   // A/B switch: every item on k_scan
  std::shared_ptr<Shape> shape = table->shape_for(shape_cols, stream, flat_ok);
  const std::vector<DevItem>& items = shape->items;

  // is the predicate a pure conjunction of leaves (folded TRUE constants are neutral)?
  bool conj = true;
  for (const DevPredOp& op : prog)
    if (!(op.kind == PK_LEAF || op.kind == PK_AND || (op.kind == PK_CONST && op.arg == 1))) conj = false;
  // renumber live leaves; a conjunction evaluates its cheapest leaves first (narrow dictionary indices:
  // the whole LUT in a register), the later ones only see the survivors
  std::vector<int> leaf_slot(leaves.size(), -1);
  uint32_t nleaves = 0;
  {
    std::vector<size_t> order;
    for (size_t l = 0; l < leaves.size(); l++) if (leaf_live[l]) order.push_back(l);
    if (conj)
      std::stable_sort(order.begin(), order.end(), [&](size_t a, size_t b) {
        auto cost = [&](size_t l) {
          const uint32_t s = uint32_t(slot_of[leaves[l].qcol]);
          if (leaves[l].d.kind == LK_IS_NULL || leaves[l].d.kind == LK_IS_NOT_NULL) return 0u;
          if (plan.cols[s].kind == DK_STR && shape->has_plain[s]) return 200u;   // PLAIN byte arrays: compared string by string, last
          return shape->flat_plain8[s] ? 64u : std::max<uint32_t>(shape->flat_max_bw[s], shape->max_bw[s]);
        };
        return cost(a) < cost(b);
      });
    for (size_t l : order) {
      leaf_slot[l] = int(nleaves);
      plan.leaves[nleaves] = leaves[l].d;
      plan.leaves[nleaves].col = uint8_t(slot_of[leaves[l].qcol]);
      nleaves++;
    }
  }
  plan.nleaves = nleaves;
  plan.conj = conj ? 1 : 0;
  if (verbose) {
    // PQB_VERBOSE: per live leaf, the flat page kinds under it and the leaf mode each flat piece selects (leaf_ctx in
    // flat_scan.cuh: a register LUT for a dictionary of <= 32 entries at an index width <= 5), with the index widths
    // seen per mode; "off-grid" counts the index pieces whose first bit is off the 128-bit grid of the staged copy
    static const char* const kLeafKind[] = {"?", "CMP", "IS_NULL", "IS_NOT_NULL", "LIKE", "REGEX", "IN"};
    for (size_t l = 0; l < leaves.size(); l++) {
      if (leaf_slot[l] < 0) continue;
      const uint32_t s = uint32_t(slot_of[leaves[l].qcol]);
      uint32_t kinds = 0, widest = 0, offgrid = 0, absent = 0;
      uint64_t bws[4] = {0, 0, 0, 0};   // REGLUT, MEMLUT, CONST (width 0 under a larger dictionary), other: bit w = width w
      for (const DevItem& it : items) {
        if (!(it.fast & kItemFlat)) continue;
        if ((it.absent >> s) & 1u) { absent++; continue; }
        const FlatPageRec& fr = table->flat_pages[it.page[s]];
        kinds |= 1u << fr.fkind;
        if (fr.fkind != FK_INDEX) continue;
        widest = std::max<uint32_t>(widest, fr.bw);
        if (fr.bw && (uint64_t(it.poff[s]) * fr.bw) % 128u) offgrid++;
        const uint32_t dn = table->row_groups[it.rg].chunks[shape_cols[s]].dict_n;
        const int m = !value_leaf(leaves[l].d.kind) ? 3 : (fr.bw <= 5 && dn <= 32) ? 0 : fr.bw == 0 ? 2 : 1;
        bws[m] |= 1ull << std::min<uint32_t>(fr.bw, 63);
      }
      std::string pk, modes;
      static const char* const kFlat[] = {"NONE", "INDEX", "PLAIN8", "BITS", "BYTES"};
      for (uint32_t k = 0; k < 5; k++) if ((kinds >> k) & 1u) pk += (pk.empty() ? "" : "+") + std::string(kFlat[k]);
      static const char* const kMode[] = {"REGLUT", "MEMLUT", "CONST"};
      for (int m = 0; m < 3; m++) {
        if (!bws[m]) continue;
        modes += std::string(" ") + kMode[m] + "{";
        for (uint32_t w = 0, first = 1; w < 64; w++) if ((bws[m] >> w) & 1ull) { modes += (first ? "" : ",") + std::to_string(w); first = 0; }
        modes += "}";
      }
      fprintf(stderr, "[pqb] leaf %d: column '%s', %s, flat pages %s, widest index %u, register LUT %s, off-grid %u, absent %u,%s\n",
              leaf_slot[l], table->columns[shape_cols[s]].name.c_str(), kLeafKind[leaves[l].d.kind < 7 ? leaves[l].d.kind : 0],
              pk.empty() ? "-" : pk.c_str(), widest, bws[0] ? (bws[1] || bws[2] ? "some" : "all") : "none", offgrid, absent,
              modes.empty() ? " -" : modes.c_str());
    }
  }
  // per column: the leaves a dictionary LUT answers (k_scan fuses up to two into the unpack)
  for (uint32_t c = 0; c < (uint32_t)kMaxCols; c++) { plan.col_nlut[c] = 0; plan.col_l0[c] = -1; plan.col_l1[c] = -1; }
  for (uint32_t l = 0; l < nleaves; l++) {
    const DevLeaf& lf = plan.leaves[l];
    if (!value_leaf(lf.kind)) continue;
    if (plan.col_nlut[lf.col] == 0) plan.col_l0[lf.col] = int8_t(l);
    else if (plan.col_nlut[lf.col] == 1) plan.col_l1[lf.col] = int8_t(l);
    plan.col_nlut[lf.col]++;
  }
  {
    const char* rm = getenv("PQB_ROW_MAJOR");  // experiment switch: register-only row-major pass for no-NULL slabs
    plan.row_major = rm && rm[0] == '1';
  }
  {
    // k_scan: conjunction of 1-4 CMP/LIKE leaves: specialised octet pass over no-NULL dictionary slabs
    bool c4 = conj && nleaves >= 1 && nleaves <= 4;
    for (uint32_t l = 0; l < nleaves; l++) c4 &= value_leaf(plan.leaves[l].kind) && plan.leaves[l].kind != LK_IN;
    const char* fa = getenv("PQB_FAST_AND");
    plan.fast_and = c4 && !(fa && fa[0] == '0');
  }
  plan.npred = uint32_t(prog.size());
  for (size_t i = 0; i < prog.size(); i++) {
    plan.pred[i] = prog[i];
    if (prog[i].kind == PK_LEAF) plan.pred[i].arg = uint8_t(leaf_slot[prog[i].arg]);
  }

  // ---- aggregates ----
  const bool has_aggs = d.n_aggs > 0;
  bool only_count_star = has_aggs && d.n_group_by == 0;
  for (uint32_t a = 0; a < d.n_aggs; a++) only_count_star &= d.aggs[a].fn == PQ_AGG_COUNT_STAR;
  const bool agg_kernel = has_aggs && !only_count_star;
  plan.mode = agg_kernel ? SM_AGG : SM_FILTER;
  std::vector<int> agg_out_type(d.n_aggs, PQ_T_I64);
  std::vector<double> pct_p(kMaxAggs, 0.0);   // PERCENTILE_CONT: the fraction of each aggregate
  if (has_aggs) {
    uint32_t n_acc = 0;
    plan.naggs = d.n_aggs;
    for (uint32_t a = 0; a < d.n_aggs; a++) {
      DevAgg& ag = plan.aggs[a];
      ag = DevAgg{};
      ag.fn = uint8_t(d.aggs[a].fn);
      if (ag.fn == AG_COUNT_STAR) { agg_out_type[a] = PQ_T_I64; continue; }
      if (ag.fn > AG_PERCENTILE_CONT) throw Error(PQ_ERR_INVALID_ARG, "unknown aggregate function");
      uint32_t qc = uint32_t(d.aggs[a].col);
      ag.col = uint8_t(slot_of[qc]);
      ag.kind = plan.cols[ag.col].kind;
      if (ag.fn == AG_MEDIAN || ag.fn == AG_PERCENTILE_CONT) {
        // the output bits go to an accumulator cell of their own (k_pct_pick writes it after the scan); the pairs of one
        // column are shared by every percentile aggregate over it
        const char* fname = ag.fn == AG_MEDIAN ? "MEDIAN" : "PERCENTILE_CONT";
        const int t = out_type_of(qc);
        if ((t != PQ_T_I64 && t != PQ_T_F64) || (ag.kind != DK_I64 && ag.kind != DK_F64))
          throw Error(PQ_ERR_UNSUPPORTED, std::string(fname) + " over " + type_name(t) + " is not on the GPU path");
        if (ag.fn == AG_PERCENTILE_CONT) {
          if (!d.agg_params) throw Error(PQ_ERR_INVALID_ARG, "PERCENTILE_CONT needs its fraction in agg_params (NULL)");
          const double p = d.agg_params[a];
          if (!std::isfinite(p) || p < 0.0 || p > 1.0)
            throw Error(PQ_ERR_INVALID_ARG, std::string("PERCENTILE_CONT(") + d.columns[qc].name + ", p): p must be finite and in [0, 1]");
          pct_p[a] = p;
        }
        agg_out_type[a] = ag.fn == AG_MEDIAN ? t : PQ_T_F64;
        ag.acc_slot = uint8_t(n_acc);
        plan.acc_init[n_acc++] = 0;
        uint32_t first = a;
        for (uint32_t b = 0; b < a; b++)
          if ((plan.aggs[b].fn == AG_MEDIAN || plan.aggs[b].fn == AG_PERCENTILE_CONT) && plan.aggs[b].col == ag.col) { first = b; break; }
        if (first != a) {
          ag.dset = plan.aggs[first].dset;
          ag.dset_owner = 0;
          continue;
        }
        ag.dset = uint8_t(plan.npct);
        ag.dset_owner = 1;
        plan.pct[plan.npct] = DevPairSet{};
        plan.pct[plan.npct].enc = ag.kind == DK_F64 ? OE_F64 : OE_I64;
        plan.npct++;
        continue;
      }
      if (ag.fn == AG_COUNT_DISTINCT) {
        // the count of first sightings is an integer-add cell; COUNT(DISTINCT) twice over one column shares the first
        // one's presence structure and cell
        if (ag.kind != DK_I64 && ag.kind != DK_F64 && ag.kind != DK_STR && ag.kind != DK_BOOL)
          throw Error(PQ_ERR_UNSUPPORTED, std::string("COUNT(DISTINCT) over ") + type_name(out_type_of(qc)) + " is not on the GPU path");
        agg_out_type[a] = PQ_T_I64;
        uint32_t first = a;
        for (uint32_t b = 0; b < a; b++)
          if (plan.aggs[b].fn == AG_COUNT_DISTINCT && plan.aggs[b].col == ag.col) { first = b; break; }
        if (first != a) {
          ag.acc_slot = plan.aggs[first].acc_slot;
          ag.dset = plan.aggs[first].dset;
          ag.dset_owner = 0;
          continue;
        }
        ag.acc_slot = uint8_t(n_acc);
        plan.acc_init[n_acc++] = 0;
        ag.dset = uint8_t(plan.ndist);
        ag.dset_owner = 1;
        plan.dist[plan.ndist] = DevDistinct{};
        plan.dist[plan.ndist].col = ag.col;
        plan.ndist++;
        continue;
      }
      if ((ag.fn == AG_MIN || ag.fn == AG_MAX) && (ag.kind == DK_STR || ag.kind == DK_BOOL)) {
        // the signed MIN / MAX cells of the numeric path: a Utf8 row contributes its bytewise rank (plan.rank, set with
        // the GROUP BY ids below), a Boolean row its bit; the result maps the cell back to the input type
        ag.acc_slot = uint8_t(n_acc);
        plan.acc_init[n_acc++] = ag.fn == AG_MIN ? 2 : 3;
        agg_out_type[a] = out_type_of(qc);
        continue;
      }
      if (ag.fn != AG_COUNT && ((ag.kind != DK_I64 && ag.kind != DK_F64) || ((ag.fn == AG_SUM || ag.fn == AG_AVG) && is_date(qc))))
        throw Error(PQ_ERR_UNSUPPORTED, std::string("SUM/AVG over ") + type_name(out_type_of(qc)) + " is not on the GPU path");
      if (ag.fn == AG_COUNT) { agg_out_type[a] = PQ_T_I64; continue; }
      ag.acc_slot = uint8_t(n_acc);
      uint8_t how = 0;
      if (ag.fn == AG_SUM) how = ag.kind == DK_F64 ? 1 : 0;
      else if (ag.fn == AG_AVG) how = 1;
      else how = ag.fn == AG_MIN ? 2 : 3;
      plan.acc_init[n_acc++] = how;
      agg_out_type[a] = ag.fn == AG_AVG ? PQ_T_F64 : out_type_of(qc);
    }
    plan.n_acc = n_acc;
    for (uint32_t a = 0; a < d.n_aggs; a++)
      if (plan.aggs[a].fn == AG_COUNT_DISTINCT && (d.flags & PQ_QUERY_ALLREDUCE))
        throw Error(PQ_ERR_UNSUPPORTED, std::string("COUNT(DISTINCT ") + d.columns[d.aggs[a].col].name +
                                            ") under PQ_QUERY_ALLREDUCE: per-rank distinct counts cannot be summed");
    if (plan.npct && (d.flags & PQ_QUERY_ALLREDUCE))
      throw Error(PQ_ERR_UNSUPPORTED, "MEDIAN / PERCENTILE_CONT under PQ_QUERY_ALLREDUCE: exact order statistics cannot be all-reduced");
    if (plan.npct && plan.ndist)
      throw Error(PQ_ERR_UNSUPPORTED, "MEDIAN / PERCENTILE_CONT together with COUNT(DISTINCT) in one query is not on the GPU path");
  }

  for (uint32_t k = 0; k < d.n_group_by; k++)
    if (d.group_exprs && d.group_exprs[k].kind == PQ_KEY_DATE_BIN && is_date(uint32_t(d.group_by[k])))
      throw Error(PQ_ERR_UNSUPPORTED, std::string("DATE_BIN over the Date32 column '") + d.columns[d.group_by[k]].name + "' is not on the GPU path");
  mark("plan compiled");
  // ---- what this query reads: bytes, NULL presence, encodings the kernels cannot take ----
  std::vector<uint8_t> col_needs_ent(ncols, 0);  // entry offsets (string leaf)
  for (uint32_t l = 0; l < nleaves; l++) {
    const DevLeaf& lf = plan.leaves[l];
    if (value_leaf(lf.kind) && plan.cols[lf.col].kind == DK_STR) col_needs_ent[lf.col] = 1;
  }
  uint64_t algo_bytes = 0, scanned_bytes = 0;
  std::vector<uint8_t> col_has_nulls(std::max<uint32_t>(ncols, 1), 0);   // statistics cannot rule NULLs out
  for (uint32_t g = 0; g < nrg_table; g++) {
    if (!rg_live[g]) continue;
    const TableRowGroup& rg = table->row_groups[g];
    for (uint32_t s = 0; s < ncols; s++) {
      const TableChunk& tc = rg.chunks[shape_cols[s]];
      if (!tc.present || tc.meta->stats.null_count != 0) col_has_nulls[s] = 1;   // absent column: every row NULL
      if (!tc.present) continue;
      scanned_bytes += tc.bytes;
      algo_bytes += uint64_t(tc.meta->total_uncompressed_size);
    }
  }
  const bool allreduce = (d.flags & PQ_QUERY_ALLREDUCE) != 0;
  if (allreduce && !comm_active()) throw Error(PQ_ERR_INVALID_ARG, "PQ_QUERY_ALLREDUCE without pq_comm_init_rank");
  const bool multi = agg_kernel && allreduce && comm_nranks() > 1;
  // every query that meets the other ranks in a collective (an aggregate table, COUNT(*)'s total, or a scan's merged
  // first rows) agrees on refusals
  const bool agree = (has_aggs && allreduce && comm_nranks() > 1) || merge_rows;
  const uint32_t n_flat = flat_ok ? shape->n_flat : 0;
  const uint32_t n_general = flat_ok ? shape->n_general : uint32_t(items.size());
  // ---- refusals that depend on what this rank's shard holds (its pages, footers and flat-store copies).  Under a
  // multi-rank all-reduce every rank must refuse together: a rank that threw while the others went on into a collective
  // would leave them waiting for it.  So they are all found here, before the first collective, and the tiny all-reduce
  // below carries "refused" words; without other ranks to meet the first one found is thrown right away ----
  std::string refusal;
  auto refuse = [&](const std::string& why) { if (refusal.empty()) refusal = why; };
  for (uint32_t s = 0; s < ncols; s++) {
    const std::string& cname = table->columns[shape_cols[s]].name;
    plan.cols[s].has_delta = shape->has_delta[s];
    plan.cols[s].has_dict = shape->has_dict[s];
    plan.cols[s].has_plain = shape->has_plain[s];
    plan.cols[s].max_bw = shape->max_bw[s];
    if (shape->has_delta[s] && plan.cols[s].kind != DK_I64)
      refuse("column '" + cname + "': DELTA_BINARY_PACKED is decoded for INT64 columns only");
    // k_scan reads no string values out of pages without a dictionary (PLAIN, and DELTA_(LENGTH_)BYTE_ARRAY rewritten
    // as PLAIN): a leaf over them would count no row.  So they are refused whenever k_scan takes items: pages without
    // a flat-store copy, or the flat kernels switched off (then every page has a copy that no kernel reads)
    if (shape->has_plain[s] && plan.cols[s].kind == DK_STR && n_general)
      refuse("column '" + cname + "': PLAIN (dictionary-fallback) string pages without a flat-store copy are not decoded on the GPU" +
             (flat_ok ? std::string() : std::string(" (the flat kernels are switched off)")));
    // k_scan reads a page's raw values at 8 bytes: a Date32 column the query reads (slot s) is read from its widened
    // flat-store copy only.  An item without a flat-store copy of any of its columns goes to k_scan whole, so one such
    // item among the query's columns refuses a query that reads a Date32 column
    if (table->columns[shape_cols[s]].is_date && n_general)
      refuse("Date32 column '" + cname + "' needs a flat-store copy of every page the query reads" +
             (shape->why_general.empty() ? std::string(" (the flat kernels are switched off)") : ": " + shape->why_general));
  }
  auto filtered_on = [&](uint32_t s) {
    for (uint32_t l = 0; l < nleaves; l++)
      if (plan.leaves[l].col == s && value_leaf(plan.leaves[l].kind)) return true;
    return false;
  };
  // DATE_BIN keys: the bins any scanned row of this rank can fall into, from the footer statistics of its live row groups
  std::vector<std::pair<int64_t, int64_t>> bin_vrange(d.n_group_by, {INT64_MAX, INT64_MIN});
  for (uint32_t k = 0; agg_kernel && k < d.n_group_by; k++) {
    const uint32_t s = uint32_t(slot_of[d.group_by[k]]);
    const std::string& cname = table->columns[tcol[d.group_by[k]]].name;
    if (d.group_exprs && d.group_exprs[k].kind == PQ_KEY_DATE_BIN) {
      const PqKeyExpr& gx = d.group_exprs[k];
      if (plan.cols[s].kind != DK_I64 || gx.width_ms <= 0) continue;   // refused below, alike on every rank
      int64_t& vmin = bin_vrange[k].first;
      int64_t& vmax = bin_vrange[k].second;
      for (uint32_t g = 0; g < nrg_table; g++) {
        if (!rg_live[g]) continue;
        const TableChunk& tc = table->row_groups[g].chunks[shape_cols[s]];
        if (!tc.present) continue;
        const ColumnStats& st = tc.meta->stats;
        if (st.null_count >= 0 && uint64_t(st.null_count) == uint64_t(tc.meta->num_values)) continue;   // all NULL: no bins
        if (!st.has_min || !st.has_max || st.min.size() != 8 || st.max.size() != 8) {
          refuse("DATE_BIN over '" + cname + "' needs min / max statistics in the file footers");
          break;
        }
        int64_t mn, mx;
        std::memcpy(&mn, st.min.data(), 8);
        std::memcpy(&mx, st.max.data(), 8);
        vmin = std::min(vmin, mn);
        vmax = std::max(vmax, mx);
      }
      if (vmin <= vmax && (vmin < gx.origin_ms - (int64_t(1) << 52) || vmax > gx.origin_ms + (int64_t(1) << 52)))
        refuse("DATE_BIN: values more than 2^52 ms away from the origin");
      if (n_general) refuse("DATE_BIN keys need a flat-store copy of every page the query reads: " + shape->why_general);
      continue;
    }
    if (plan.cols[s].kind == DK_BOOL || !(plan.cols[s].has_plain || plan.cols[s].has_delta)) continue;
    // Pages without a dictionary (PLAIN fallback of an overflowed dictionary, PLAIN / DELTA numerics): their ROWS are
    // interned next to the dictionary entries and the aggregate kernel stages the pages' ids instead of their values, so
    // nothing else of this query may read the column's values, and k_scan, which reads a dictionary index per row, cannot
    // take them
    if (filtered_on(s))
      refuse("GROUP BY column '" + cname + "' has pages without a dictionary and is also filtered on: not on the GPU path");
    for (uint32_t a = 0; a < d.n_aggs; a++)
      if (((plan.aggs[a].fn >= AG_SUM && plan.aggs[a].fn <= AG_AVG) || plan.aggs[a].fn >= AG_MEDIAN) && plan.aggs[a].col == s &&
          !rank_min_max(plan.aggs[a]))
        refuse("GROUP BY column '" + cname + "' has pages without a dictionary and is also aggregated: not on the GPU path");
    if (n_general)
      refuse("GROUP BY column '" + cname + "' has pages without a dictionary, which need a flat-store copy of every page the query reads: " +
             shape->why_general);
  }
  {
    uint64_t lut_entries = 0;   // the per-leaf LUT regions (side tables below)
    for (uint32_t l = 0; l < nleaves; l++)
      if (value_leaf(plan.leaves[l].kind)) lut_entries += table->sides[shape_cols[plan.leaves[l].col]].total_entries;
    if (lut_entries > 0xfffffff0ull) refuse("leaf LUTs too large");
  }
  for (uint32_t a = 0; agg_kernel && a < d.n_aggs; a++) {
    const DevAgg& ag = plan.aggs[a];
    if (rank_min_max(ag) && (plan.cols[ag.col].has_plain || plan.cols[ag.col].has_delta) && filtered_on(ag.col))
      refuse(std::string(ag.fn == AG_MIN ? "MIN(" : "MAX(") + table->columns[shape_cols[ag.col]].name +
             "): the column has pages without a dictionary and is also filtered on: not on the GPU path");
    // (a column in no file has nothing to read: k_scan takes it)
    if (n_general && (rank_min_max(ag) || bool_min_max(ag)) && table->columns[shape_cols[ag.col]].kind != 0xfe)
      refuse(std::string(ag.fn == AG_MIN ? "MIN(" : "MAX(") + d.columns[d.aggs[a].col].name +
             ") over Utf8 / Boolean needs a flat-store copy of every page the query reads: " + shape->why_general);
  }
  // k_scan has no IN path: its pages are read through the flat store only
  for (uint32_t l = 0; l < nleaves; l++)
    if (plan.leaves[l].kind == LK_IN && n_general) {
      refuse("IN list on '" + table->columns[shape_cols[plan.leaves[l].col]].name +
             "' needs a flat-store copy of every page the query reads" +
             (shape->why_general.empty() ? std::string(" (the flat kernels are switched off)") : ": " + shape->why_general));
      break;
    }
  if (merge_rows && n_general)   // (without other ranks: thrown with the other scan refusals below)
    refuse("ORDER BY on a scan needs a flat-store copy of every page the query reads: " + shape->why_general);
  // the merge breaks ties by __row_id, which is global only when every rank opened the same file list and scans its row
  // groups g % N == rank (under file sharding each rank numbers its own files from 0)
  if (merge_rows && (table->shard_count != uint32_t(comm_nranks()) || table->shard_index != uint32_t(comm_rank())))
    refuse("PQ_QUERY_ALLGATHER needs the table sharded by row group over the communicator (shard_count " +
           std::to_string(table->shard_count) + ", shard_index " + std::to_string(table->shard_index) + " on rank " +
           std::to_string(comm_rank()) + " of " + std::to_string(comm_nranks()) + "): only then is __row_id global");
  if (!refusal.empty() && !agree) throw Error(PQ_ERR_UNSUPPORTED, refusal);
  // k_flat_agg answers an out-of-line leaf over pages without a dictionary (a regular expression's DFA walk, an IN list's
  // set probe) only in its RX instantiations
  bool rx_bytes = false;
  for (uint32_t l = 0; l < nleaves; l++) {
    const DevLeaf& lf = plan.leaves[l];
    rx_bytes |= (lf.kind == LK_REGEX || lf.kind == LK_IN) && (plan.cols[lf.col].has_plain || plan.cols[lf.col].has_delta);
  }
  plan.n_items = uint32_t(items.size());
  metrics.bytes_scanned = scanned_bytes;
  // an aggregated column whose footers promise null_count == 0 in every row group read: its non-null
  // counter equals the group's row count, so the scan skips that atomic (and the table is 4 cells per group
  // narrower on C4).  Under PQ_QUERY_ALLREDUCE the cells are summed across ranks and every rank must make the same
  // choice: the per-rank footer verdicts are summed over the ranks first (a rank whose row groups were all pruned
  // contributes zeros).  The same tiny all-reduce carries whether every rank still holds the agreed numbering of the
  // GROUP BY key values (kept with the table column, tagged with the communicator's epoch; a rank may have reopened its
  // table): ONE collective and one round trip per query for both agreements.  Its last two words are the number of ranks
  // that refuse the query (then every rank refuses) and a mask of the refusing ranks below 63 (bit r for rank r; the bits
  // are distinct, so their sum is their union), which names one of them.  A COUNT(*)-only query runs it for the refusals
  // alone: its total's all-reduce comes after the scan.  Two more words do the same for the ranks with items that have no
  // flat-store copy, which only a hashed GROUP BY refuses (whether it is hashed is known once the key cards are agreed),
  // and the last one sums the rows of every rank's live row groups, which bound the hashed table's size alike on every rank.
  bool keys_agreed = true;
  uint64_t live_rows = 0;
  for (uint32_t g = 0; g < nrg_table; g++) if (rg_live[g]) live_rows += table->row_groups[g].num_rows;
  uint64_t rows_all = live_rows, general_ranks = n_general ? 1 : 0, general_mask = 0;
  if (agree) {
    // a merged scan adds two words: the sum and the sum of squares of every rank's file-list rows (mod 2^20), which are
    // equal on every rank when nr x (sum of squares) == sum^2: one file list for every rank
    std::vector<unsigned long long> f(6 + ncols + (merge_rows ? 2 : 0), 0ull);
    if (merge_rows) {
      const unsigned long long x = table->list_rows & 0xfffffull;
      f[6 + ncols] = x;
      f[7 + ncols] = x * x;
    }
    if (!refusal.empty()) {
      f[1 + ncols] = 1;
      if (comm_rank() < 63) f[2 + ncols] = 1ull << comm_rank();
    }
    if (n_general) {
      f[3 + ncols] = 1;
      if (comm_rank() < 63) f[4 + ncols] = 1ull << comm_rank();
    }
    f[5 + ncols] = live_rows;
    for (uint32_t k = 0; k < d.n_group_by; k++) {
      if (d.group_exprs && d.group_exprs[k].kind == PQ_KEY_DATE_BIN) continue;
      const uint32_t s = uint32_t(slot_of[d.group_by[k]]);
      if (plan.cols[s].kind == DK_BOOL) continue;
      const ColSide& cs = table->sides[shape_cols[s]];
      if (!cs.glob_ready || cs.glob_epoch != comm_epoch()) f[0] = 1;   // this rank lacks an agreement
    }
    for (uint32_t a = 0; a < d.n_aggs; a++) {   // MIN / MAX over Utf8 read their ranks in the agreed numbering too
      if (!rank_min_max(plan.aggs[a])) continue;
      const ColSide& cs = table->sides[shape_cols[plan.aggs[a].col]];
      if (!cs.glob_ready || cs.glob_epoch != comm_epoch()) f[0] = 1;
    }
    for (uint32_t t = 0; merge_rows && t < d.n_order_by; t++) {   // so do the Utf8 terms of a merged scan
      const uint32_t s = uint32_t(slot_of[d.order_by[t].index]);
      if (plan.cols[s].kind != DK_STR) continue;
      const ColSide& cs = table->sides[shape_cols[s]];
      if (!cs.glob_ready || cs.glob_epoch != comm_epoch()) f[0] = 1;
    }
    for (uint32_t s = 0; s < ncols; s++) f[1 + s] = col_has_nulls[s] ? 1ull : 0ull;
    DevBuf<unsigned long long> df;
    df.upload(f, stream);
    comm_allreduce_u64(df.p, f.size(), 0 /*sum*/, stream);
    PQB_CUDA(cudaMemcpyAsync(f.data(), df.p, f.size() * 8, cudaMemcpyDeviceToHost, stream));
    PQB_CUDA(cudaStreamSynchronize(stream));
    if (!refusal.empty()) throw Error(PQ_ERR_UNSUPPORTED, refusal);
    if (f[1 + ncols])
      throw Error(PQ_ERR_UNSUPPORTED, "refused on " + (f[2 + ncols] ? "rank " + std::to_string(__builtin_ctzll(f[2 + ncols]))
                                                                    : std::to_string(f[1 + ncols]) + " ranks") +
                                          " (its shard holds pages or footers this query cannot take on the GPU path)");
    if (merge_rows && (unsigned __int128)f[7 + ncols] * comm_nranks() != (unsigned __int128)f[6 + ncols] * f[6 + ncols])
      throw Error(PQ_ERR_UNSUPPORTED, "PQ_QUERY_ALLGATHER: the ranks opened file lists of different sizes; every rank must open the same "
                                      "list, sharded by row group");
    general_ranks = f[3 + ncols];
    general_mask = f[4 + ncols];
    rows_all = f[5 + ncols];
    if (multi || merge_rows) keys_agreed = f[0] == 0;
    if (multi)
      for (uint32_t s = 0; s < ncols; s++) col_has_nulls[s] = f[1 + s] != 0;
  }
  std::vector<uint8_t> nn_is_rows(kMaxAggs, 0);
  {
    std::map<int, int> nn_of_col;   // one non-null counter array per aggregated column that may hold NULLs
    for (uint32_t a = 0; a < d.n_aggs; a++) {
      DevAgg& ag = plan.aggs[a];
      if (ag.fn == AG_COUNT_STAR) continue;
      ag.update_nn = 0;
      if (ag.fn == AG_COUNT_DISTINCT) { nn_is_rows[a] = 1; continue; }   // no non-null counter: k_agg_finish reads only its count cell
      if (!col_has_nulls[ag.col]) { nn_is_rows[a] = 1; continue; }
      auto it = nn_of_col.find(int(ag.col));
      if (it == nn_of_col.end()) { it = nn_of_col.emplace(int(ag.col), int(nn_of_col.size())).first; ag.update_nn = 1; }
      ag.nn_slot = uint8_t(it->second);
    }
    plan.n_nn = uint32_t(nn_of_col.size());
  }
  // columns whose dictionary indices the row phase of k_scan needs (GROUP BY keys, aggregate inputs)
  for (uint32_t k = 0; k < d.n_group_by; k++) plan.cols[slot_of[d.group_by[k]]].need_idx = 1;
  for (uint32_t a = 0; a < d.n_aggs; a++)
    if (d.aggs[a].fn != PQ_AGG_COUNT_STAR) plan.cols[slot_of[d.aggs[a].col]].need_idx = 1;

  // ---- side tables: string entry offsets, per-leaf LUT regions ----
  DevPrepArgs pa{};
  uint64_t lut_total = 0;
  for (uint32_t s = 0; s < ncols; s++)
    if (col_needs_ent[s]) { table->ensure_ent_off(shape_cols[s], stream); pa.ent[s] = table->sides[shape_cols[s]].d_ent_off; }
  bool any_lut = false;
  uint32_t max_dict_n = 1;
  for (uint32_t l = 0; l < nleaves; l++) {
    DevLeaf& lf = plan.leaves[l];
    lf.lut_off = 0;
    if (!value_leaf(lf.kind)) continue;
    const ColSide& cs = table->sides[shape_cols[lf.col]];
    lf.lut_off = uint32_t(lut_total);
    lut_total += cs.total_entries;
    any_lut |= cs.total_entries != 0;
    max_dict_n = std::max(max_dict_n, cs.max_dict_n);
  }

  // ---- GROUP BY keys: interned per table column (cached with the table) ----
  std::vector<QKey> qk(d.n_group_by);
  std::vector<uint8_t> row_keys(d.n_group_by, 0);   // the key column has pages without a dictionary: per-row ids (FK_IDS pages)
  plan.nkeys = d.n_group_by;
  uint64_t launches = 0;
  for (uint32_t k = 0; agg_kernel && k < d.n_group_by; k++) {
    DevKey& key = plan.keys[k];
    key.col = uint8_t(slot_of[d.group_by[k]]);
    const uint8_t kind = plan.cols[key.col].kind;
    if (d.group_exprs && d.group_exprs[k].kind == PQ_KEY_DATE_BIN) {
      // ---- DATE_BIN(width, column, origin) (the counts / histogram API, src/query/mod.rs:623-680): the key is
      // computed from the value; the bins any scanned row can fall into come from the footer statistics (bin_vrange,
      // read with the refusals above) ----
      const PqKeyExpr& gx = d.group_exprs[k];
      const std::string& cname = table->columns[tcol[d.group_by[k]]].name;
      if (kind != DK_I64) throw Error(PQ_ERR_INVALID_ARG, "DATE_BIN needs a Timestamp / Int64 column, '" + cname + "' is neither");
      if (gx.width_ms <= 0) throw Error(PQ_ERR_INVALID_ARG, "DATE_BIN needs a positive stride");
      const int64_t vmin = bin_vrange[k].first, vmax = bin_vrange[k].second;
      auto floordiv = [](int64_t a, int64_t b) { int64_t q = a / b; return (a % b != 0 && ((a < 0) != (b < 0))) ? q - 1 : q; };
      int64_t bmin = 0, bmax = 0;
      if (vmin <= vmax) {
        bmin = floordiv(vmin - gx.origin_ms, gx.width_ms);
        bmax = floordiv(vmax - gx.origin_ms, gx.width_ms);
      }
      if (multi) {   // every rank needs the same bin 0 and the same number of bins
        long long mm[2] = {(long long)bmin, -(long long)bmax};
        if (vmin > vmax) { mm[0] = INT64_MAX; mm[1] = INT64_MAX; }
        DevBuf<unsigned long long> dmm;
        dmm.alloc(2, stream);
        PQB_CUDA(cudaMemcpyAsync(dmm.p, mm, 16, cudaMemcpyHostToDevice, stream));
        comm_allreduce_u64(dmm.p, 2, 1 /*signed min*/, stream);
        PQB_CUDA(cudaMemcpyAsync(mm, dmm.p, 16, cudaMemcpyDeviceToHost, stream));
        PQB_CUDA(cudaStreamSynchronize(stream));
        if (mm[0] == INT64_MAX) { bmin = bmax = 0; } else { bmin = mm[0]; bmax = -mm[1]; }
      }
      if (bmax - bmin + 1 > (int64_t(1) << 24)) throw Error(PQ_ERR_UNSUPPORTED, "DATE_BIN: more than 2^24 bins in the scanned range");
      key.kind = KK_BIN;
      key.bin_width = gx.width_ms;
      key.bin_base = gx.origin_ms + bmin * gx.width_ms;
      qk[k].card = uint32_t(bmax - bmin + 1);
      qk[k].is_bin = true;
      continue;
    }
    key.kind = kind == DK_BOOL ? KK_BOOL : KK_DICT_LUT;
    if (key.kind == KK_BOOL) { qk[k].card = 2; continue; }
    // pages without a dictionary: ensure_key interns their rows (the uses this rules out were refused above)
    if (plan.cols[key.col].has_plain || plan.cols[key.col].has_delta) row_keys[k] = 1;
    const int tc_i = shape_cols[key.col];
    table->ensure_key(tc_i, stream);
    const ColSide& cs = table->sides[tc_i];
    key.gid = cs.d_gid;
    qk[k].kd = &cs.kd;
    qk[k].card = cs.card;
  }
  if (multi && d.n_group_by) {
    // ---- multi-GPU: every rank must use ONE numbering of the key values.  The agreement (all-gather of the
    // packed distinct values, numbered by first occurrence in rank order: identical on every rank, and hot-first
    // because rank 0's ids are) is kept with the table column; `keys_agreed` (above) says whether EVERY rank holds it ----
    const uint32_t have = keys_agreed ? 1u : 0u;
    for (uint32_t k = 0; k < d.n_group_by; k++) {
      DevKey& key = plan.keys[k];
      if (key.kind != KK_DICT_LUT) continue;
      const int tc_i = shape_cols[key.col];
      if (!have) table->unify_key(tc_i, stream);
      const ColSide& cs = table->sides[tc_i];
      key.gid = cs.d_glob_gid;
      qk[k].kd = &cs.glob_kd;
      qk[k].card = cs.glob_card;
    }
  }
  // ---- COUNT(DISTINCT) columns: value ids are the column's GROUP BY ids (interned like a key column, NULL excluded) ----
  std::vector<const uint32_t*> ids_gid(ncols, nullptr);   // column slots whose pages without a dictionary are read as id pages
  for (uint32_t k = 0; k < d.n_group_by; k++)
    if (row_keys[k]) ids_gid[plan.keys[k].col] = plan.keys[k].gid;
  for (uint32_t i = 0; agg_kernel && i < plan.ndist; i++) {
    DevDistinct& ds = plan.dist[i];
    const int tc_i = shape_cols[ds.col];
    const std::string& cname = table->columns[tc_i].name;
    if (plan.cols[ds.col].kind == DK_BOOL) { ds.kind = KK_BOOL; ds.card = 2; continue; }
    ds.kind = KK_DICT_LUT;
    if (table->columns[tc_i].kind == 0xfe) { ds.card = 0; continue; }   // in no file: every row NULL, nothing to count
    if (plan.cols[ds.col].has_plain || plan.cols[ds.col].has_delta) {
      // the id pages stand in for the values, as for a key column: nothing else of this query may read them
      for (uint32_t l = 0; l < nleaves; l++)
        if (plan.leaves[l].col == ds.col && value_leaf(plan.leaves[l].kind))
          throw Error(PQ_ERR_UNSUPPORTED, "COUNT(DISTINCT " + cname + "): the column has pages without a dictionary and is also filtered on: not on the GPU path");
      for (uint32_t a = 0; a < d.n_aggs; a++)
        if (plan.aggs[a].fn >= AG_SUM && plan.aggs[a].fn <= AG_AVG && plan.aggs[a].col == ds.col && !rank_min_max(plan.aggs[a]))
          throw Error(PQ_ERR_UNSUPPORTED, "COUNT(DISTINCT " + cname + "): the column has pages without a dictionary and is also aggregated: not on the GPU path");
      for (uint32_t k = 0; k < d.n_group_by; k++)
        if (plan.keys[k].kind == KK_BIN && plan.keys[k].col == ds.col)
          throw Error(PQ_ERR_UNSUPPORTED, "COUNT(DISTINCT " + cname + "): the column has pages without a dictionary and is also a DATE_BIN key: not on the GPU path");
    }
    table->ensure_key(tc_i, stream);
    const ColSide& cs = table->sides[tc_i];
    ds.gid = cs.d_gid;
    ds.card = cs.card;
    if (plan.cols[ds.col].has_plain || plan.cols[ds.col].has_delta) ids_gid[ds.col] = ds.gid;
  }
  // ---- MIN / MAX over Utf8: ranks through the column's GROUP BY ids, in the numbering the keys use (the ranks' agreed one
  // under a multi-GPU all-reduce, so that every rank's cells hold ranks of the same values); pages without a dictionary
  // are read as id pages, as for a key column ----
  std::vector<std::shared_ptr<const RankLuts>> rank_luts(d.n_aggs);   // held by the query: a unify_key elsewhere may replace the column's
  {
    std::set<int> unified;   // key columns agreed on above
    for (uint32_t k = 0; multi && !keys_agreed && k < d.n_group_by; k++)
      if (plan.keys[k].kind == KK_DICT_LUT) unified.insert(shape_cols[plan.keys[k].col]);
    for (uint32_t a = 0; agg_kernel && a < d.n_aggs; a++) {
      const DevAgg& ag = plan.aggs[a];
      if (bool_min_max(ag)) {
        void* bool_rank = nullptr;
        PQB_CUDA(cudaGetSymbolAddress(&bool_rank, kBoolRank));
        plan.rank[a] = DevRankLut{nullptr, static_cast<const uint64_t*>(bool_rank), 1u, 0u};
        continue;
      }
      if (!rank_min_max(ag)) continue;
      const int tc_i = shape_cols[ag.col];
      if (table->columns[tc_i].kind == 0xfe && !multi) continue;   // in no file: every row NULL, nothing to rank
      const bool row_ids = plan.cols[ag.col].has_plain || plan.cols[ag.col].has_delta;   // (a filter on them was refused above)
      table->ensure_key(tc_i, stream);
      if (multi && !keys_agreed && unified.insert(tc_i).second) table->unify_key(tc_i, stream);
      rank_luts[a] = table->ensure_rank_luts(tc_i, multi, stream);
      const RankLuts& rl = *rank_luts[a];
      plan.rank[a] = DevRankLut{rl.ent, rl.ids, rl.card ? rl.card - 1 : 0u, 0u};
      if (row_ids) ids_gid[ag.col] = multi ? table->sides[tc_i].d_glob_gid : table->sides[tc_i].d_gid;
    }
  }
  // ---- id pages of key / COUNT(DISTINCT) columns with pages that have no dictionary: this query's copy of the flat
  // page table, with those pages pointing into the column's id array (local or agreed numbering) ----
  DevBuf<FlatPageRec> d_kpages;
  std::vector<uint32_t> key_bw32(ncols, 0);
  {
    bool any = false;
    for (uint32_t s = 0; s < ncols; s++) any = any || ids_gid[s];
    if (any) {
      std::vector<FlatPageRec> fp;
      {
        std::lock_guard<std::mutex> lk(table->side_mu);
        fp = table->flat_pages;
        for (uint32_t s = 0; s < ncols; s++) {
          if (!ids_gid[s]) continue;
          const ColSide& cs = table->sides[shape_cols[s]];
          key_bw32[s] = 32;
          for (const ColSide::KeyRowPage& rp : cs.key_row_pages) {
            FlatPageRec& r = fp[rp.page];
            r.fkind = FK_IDS;
            r.bw = 32;
            // relative to d_flat like every flat page (the subtraction may wrap, base + offset does not); 16-byte aligned: ebase is a multiple of 4
            r.off = uint64_t(ids_gid[s]) + 4ull * (uint64_t(cs.n_dict_pad) + rp.ebase) - uint64_t(table->d_flat);
          }
        }
      }
      d_kpages.upload(fp, stream);
      metrics.h2d_bytes += fp.size() * sizeof(FlatPageRec);
    }
  }
  // mixed-radix group slot: the smallest key varies fastest, so that with hot-first ids of the largest key
  // "slot < hot_slots" is "one of the hottest values of the largest key" (flat aggregate kernel)
  uint64_t nslots64 = 1;
  {
    std::vector<uint32_t> korder(d.n_group_by);
    for (uint32_t k = 0; k < d.n_group_by; k++) korder[k] = k;
    std::stable_sort(korder.begin(), korder.end(), [&](uint32_t a, uint32_t b) { return qk[a].card < qk[b].card; });
    for (uint32_t k : korder) {
      plan.keys[k].card = qk[k].card;
      plan.keys[k].stride = uint32_t(nslots64);
      plan.keys[k].wstride = nslots64;
      if (nslots64 > (1ull << 62) / (uint64_t(qk[k].card) + 1)) throw Error(PQ_ERR_UNSUPPORTED, "GROUP BY key space wider than 2^62 combinations");
      nslots64 *= uint64_t(qk[k].card) + 1;
    }
  }
  // A key space wider than the dense table (2^26 slots): the groups that actually occur are found through a hash
  // table on the wide id (DataFusion's GroupValues hashes the key tuple, SURVEY §8 a12); its capacity is twice the
  // groups that can occur (<= rows scanned, <= combinations), so it never runs full below the 2^27-slot ceiling.
  // Under PQ_QUERY_ALLREDUCE every rank's table is merged after the scan (hash_merge.cuh), and every refusal here is
  // decided from what every rank holds: the summed rows, and the ranks with items that have no flat-store copy.
  const uint64_t key_space = nslots64;   // group-id combinations (the dense table, or the groups a hashed table may meet)
  plan.hashed = 0;
  plan.hmask = 0;
  if (nslots64 > (1ull << 26)) {
    auto table_cap = [&](uint64_t rows) {
      uint64_t cap = 1024;
      while (cap < 2 * std::min<uint64_t>(nslots64, std::max<uint64_t>(rows, 1)) && cap < (1ull << 27)) cap <<= 1;
      return cap;
    };
    if (table_cap(rows_all) * (1 + plan.n_acc + plan.n_nn) * 8 > (24ull << 30))
      throw Error(PQ_ERR_UNSUPPORTED, "GROUP BY: the hashed accumulator table would exceed 24 GiB");
    if (agg_kernel && general_ranks) {
      const std::string why = "a hashed GROUP BY needs a flat-store copy of every page the query reads";
      if (n_general) throw Error(PQ_ERR_UNSUPPORTED, why + ": " + shape->why_general);
      throw Error(PQ_ERR_UNSUPPORTED, why + ": refused on " + (general_mask ? "rank " + std::to_string(__builtin_ctzll(general_mask))
                                                                            : std::to_string(general_ranks) + " ranks"));
    }
    uint64_t cap = table_cap(live_rows);
    if (const char* e = getenv("PQB_HASH_SLOTS"))   // test switch: a smaller table on this rank (a power of two, >= 64)
      while (cap > 64 && cap > strtoull(e, nullptr, 10)) cap >>= 1;
    plan.hashed = 1;
    plan.hmask = uint32_t(cap - 1);
    nslots64 = cap;
  }
  plan.nslots = uint32_t(nslots64);
  const uint32_t cells = 1 + plan.n_acc + plan.n_nn;
  // ---- COUNT(DISTINCT) presence structures: a dense bitmap (row_words words per group slot) while it fits
  // kDistinctDenseBudget and a quarter of the free HBM; above that, and always under a hashed GROUP BY (whose slots are
  // hash-table cells), a pair set on (slot << 32 | value id) with room for twice the pairs that can occur ----
  std::vector<DevBuf<unsigned int>> d_dist_bits(plan.ndist);
  std::vector<DevBuf<unsigned long long>> d_dist_pairs(plan.ndist);
  if (plan.ndist) {
    const char* fh = getenv("PQB_DISTINCT_HASH");   // experiment switch: always the pair set
    const bool force_hash = fh && fh[0] == '1';
    size_t free_b = 0, total_b = 0;
    PQB_CUDA(cudaMemGetInfo(&free_b, &total_b));
    const uint64_t budget = std::min<uint64_t>(kDistinctDenseBudget, free_b / 4);
    uint64_t rows_bound = 0;
    for (uint32_t g = 0; g < nrg_table; g++) if (rg_live[g]) rows_bound += table->row_groups[g].num_rows;
    for (uint32_t i = 0; i < plan.ndist; i++) {
      DevDistinct& ds = plan.dist[i];
      ds.row_words = std::max<uint32_t>(1, (ds.card + 31) / 32);
      const uint64_t dense_bytes = uint64_t(plan.nslots) * ds.row_words * 4;
      ds.hashed = (plan.hashed || force_hash || dense_bytes > budget) ? 1 : 0;
      if (!ds.hashed) {
        d_dist_bits[i].alloc(size_t(plan.nslots) * ds.row_words, stream);
        d_dist_bits[i].zero();
        ds.bits = d_dist_bits[i].p;
        continue;
      }
      const uint64_t pairs = std::min<uint64_t>(std::max<uint64_t>(rows_bound, 1), key_space * std::max<uint32_t>(ds.card, 1));
      uint64_t cap = 1024;
      while (cap < 2 * pairs && cap < kDistinctPairsMax) cap <<= 1;
      ds.hmask = uint32_t(cap - 1);
      d_dist_pairs[i].alloc(cap, stream);
      PQB_CUDA(cudaMemsetAsync(d_dist_pairs[i].p, 0xff, cap * 8, stream));
      ds.pairs = d_dist_pairs[i].p;
    }
  }

  // ---- MEDIAN / PERCENTILE_CONT pair sets: room for every row of the live row groups, refused above half the free HBM
  // (kPctPairBytes / kPctSortBytes) ----
  std::vector<DevBuf<uint32_t>> d_pct_slots(plan.npct);
  std::vector<DevBuf<unsigned long long>> d_pct_keys(plan.npct);
  DevBuf<unsigned int> d_pct_count;
  uint64_t pct_rows = 0;
  if (agg_kernel && plan.npct) {
    for (uint32_t g = 0; g < nrg_table; g++) if (rg_live[g]) pct_rows += table->row_groups[g].num_rows;
    if (pct_rows > 0xffffffffull)
      throw Error(PQ_ERR_UNSUPPORTED, "MEDIAN / PERCENTILE_CONT over more than 2^32 - 1 values of one column is not on the GPU path");
    size_t free_b = 0, total_b = 0;
    PQB_CUDA(cudaMemGetInfo(&free_b, &total_b));
    const uint64_t need = std::max<uint64_t>(pct_rows, 1) * (kPctPairBytes * plan.npct + kPctSortBytes);
    uint64_t budget = free_b / 2;
    if (const char* e = getenv("PQB_PCT_BUDGET")) budget = std::min<uint64_t>(budget, strtoull(e, nullptr, 10));   // test switch: a smaller budget in bytes
    if (need > budget)
      throw Error(PQ_ERR_OOM, "MEDIAN / PERCENTILE_CONT: the values and their sort need " + std::to_string(need >> 20) +
                                  " MiB of HBM, more than their budget: half the free HBM (" + std::to_string(budget >> 20) + " MiB)");
    d_pct_count.alloc(plan.npct, stream);
    d_pct_count.zero();
    for (uint32_t i = 0; i < plan.npct; i++) {
      d_pct_slots[i].alloc(std::max<uint64_t>(pct_rows, 1), stream);
      d_pct_keys[i].alloc(std::max<uint64_t>(pct_rows, 1), stream);
      plan.pct[i].slots = d_pct_slots[i].p;
      plan.pct[i].keys = d_pct_keys[i].p;
      plan.pct[i].count = d_pct_count.p + i;
    }
  }

  // ---- which kernels run ----
  (void)has_null_const;   // the flat kernels evaluate SQL three-valued logic, NULL literals included
  plan.no_flat = flat_ok ? 0 : 1;
  // (DATE_BIN keys, keys with pages without a dictionary, MIN / MAX over Utf8 / Boolean and hashed GROUP BYs were
  // refused above when some page has no flat-store copy)
  for (uint32_t i = 0; agg_kernel && i < plan.ndist; i++)
    if (n_general)
      throw Error(PQ_ERR_UNSUPPORTED, "COUNT(DISTINCT " + table->columns[shape_cols[plan.dist[i].col]].name +
                                          ") needs a flat-store copy of every page the query reads: " + shape->why_general);
  if (agg_kernel && plan.npct && n_general)
    throw Error(PQ_ERR_UNSUPPORTED, "MEDIAN / PERCENTILE_CONT need a flat-store copy of every page the query reads: " + shape->why_general);
  if (row_order && n_general)
    throw Error(PQ_ERR_UNSUPPORTED, "ORDER BY on a scan needs a flat-store copy of every page the query reads: " + shape->why_general);
  // ---- ORDER BY on a scan: a Utf8 term sorts by the bytewise rank of the column's GROUP BY ids (ensure_key, cached with
  // the table); its pages without a dictionary are read as their id pages, through this query's copy of the flat page
  // table that only the encode kernel sees.  When the ranks' rows are merged, the ids and ranks are those of the
  // numbering every rank agreed on (unify_key, a collective: every rank joins it for the same columns, also a rank whose
  // files lack the column), so that every rank encodes a value alike ----
  RowOrderArgs roa{};
  uint8_t row_nulls_first[kMaxOrder] = {};
  std::vector<std::shared_ptr<const uint32_t>> row_rank_hold;   // a query keeps the ranks it sorts with alive
  DevBuf<FlatPageRec> d_opages;
  if (row_order) {
    std::vector<std::pair<int, const uint32_t*>> id_cols;   // table columns whose pages without a dictionary are read as id pages
    std::set<int> unified;
    roa.nterms = n_part + d.n_order_by;   // a window sorts by its partition terms first
    for (uint32_t t = 0; t < roa.nterms; t++) {
      const PqOrderBy& ob = t < n_part ? win->partition_by[t] : d.order_by[t - n_part];
      RowOrderTerm& ot = roa.t[t];
      ot.slot = uint32_t(slot_of[ob.index]);
      ot.kind = plan.cols[ot.slot].kind;
      ot.desc = (ob.flags & PQ_ORDER_DESC) ? 1 : 0;
      row_nulls_first[t] = (ob.flags & PQ_ORDER_NULLS_FIRST) ? 1 : 0;
      ot.enc = ot.kind == DK_F64 ? OE_F64 : ot.kind == DK_I64 ? OE_I64 : OE_RAW;   // Boolean: 0 / 1; Utf8: the rank
      const int tc_i = shape_cols[ot.slot];
      const bool absent = table->columns[tc_i].kind == 0xfe;   // in no file: every row NULL, nothing to rank
      if (ot.kind != DK_STR || (absent && !merge_rows)) continue;
      table->ensure_key(tc_i, stream);
      if (merge_rows && !keys_agreed && unified.insert(tc_i).second) {
        if (verbose) fprintf(stderr, "[pqb] scan merge: the ranks agree on a numbering of '%s'\n", table->columns[tc_i].name.c_str());
        table->unify_key(tc_i, stream);
      }
      if (absent) continue;
      row_rank_hold.push_back(table->ensure_kd_rank(tc_i, merge_rows, stream));
      ot.gid = merge_rows ? table->sides[tc_i].d_glob_gid : table->sides[tc_i].d_gid;
      ot.rank = row_rank_hold.back().get();
      if (!table->sides[tc_i].key_row_pages.empty()) id_cols.push_back({tc_i, ot.gid});
    }
    if (!id_cols.empty()) {
      std::vector<FlatPageRec> fp;
      {
        std::lock_guard<std::mutex> lk(table->side_mu);
        fp = table->flat_pages;
        for (const auto& [tc_i, gid] : id_cols) {
          const ColSide& cs = table->sides[tc_i];
          for (const ColSide::KeyRowPage& rp : cs.key_row_pages) {
            FlatPageRec& r = fp[rp.page];
            r.fkind = FK_IDS;
            r.bw = 32;
            r.off = uint64_t(gid) + 4ull * (uint64_t(cs.n_dict_pad) + rp.ebase) - uint64_t(table->d_flat);   // as for key columns
          }
        }
      }
      d_opages.upload(fp, stream);
      metrics.h2d_bytes += fp.size() * sizeof(FlatPageRec);
    }
  }
  // ---- agg pages (k_flat_agg): a column slot whose every use in this query only looks its dictionary index up -- as
  // an aggregate input (value pages) or as a GROUP BY key (id pages) -- reads the table's agg pages instead, and its rows
  // need no dictionary or gid LUT load.  They are built once per column and kept with the table, so only a resident
  // table gets them: a file list opens its table for one query, which would pay the build every time ----
  std::vector<uint32_t> form_bw(ncols, 0);   // marked slots: widest page the slot stages
  uint32_t value_forms = 0;                  // the marked slots that read value pages (FK_FOR)
  plan.agg_forms = 0;
  // ---- tuple id pages: a GROUP BY of two or more dictionary keys whose columns have no other role reads ONE id per row,
  // the group's rank by row count in the table, from pages that follow the lead key's pages.  k_flat_agg sees a one-key
  // plan (tkey) over n_tuples slots, so the hottest GROUPS (not the hottest values of the largest key) own the hot
  // table; the result keeps the real keys, decoded from tuple->d_wide, and comes out in mixed-radix order (d_order) ----
  std::shared_ptr<const TuplePages> tuple;
  std::shared_ptr<const FlatPageRec> tuple_pages_tbl;
  DevKey tkey{};
  uint32_t tuple_keyslots = 0;   // column slots of the tuple's keys
  {
    const char* tw = getenv("PQB_TUPLE_PAGES");   // A/B switch: 0 = per-key id pages
    const char* sw = getenv("PQB_AGG_FORMS");
    bool ok = !(tw && tw[0] == '0') && !(sw && sw[0] == '0') && agg_kernel && n_flat && !n_general && d.table && !plan.ndist &&
              !plan.npct && !plan.hashed && !allreduce && !multi && d.n_group_by >= 2;
    std::vector<std::pair<int, uint64_t>> tkeys;
    for (uint32_t k = 0; ok && k < d.n_group_by; k++) {
      const DevKey& key = plan.keys[k];
      const uint32_t s = key.col;
      const ColSide& cs = table->sides[shape_cols[s]];
      ok = key.kind == KK_DICT_LUT && key.gid == cs.d_gid && cs.key_row_pages.empty() && !((tuple_keyslots >> s) & 1u);
      for (uint32_t l = 0; ok && l < nleaves; l++) ok = plan.leaves[l].col != s;
      for (uint32_t a = 0; ok && a < d.n_aggs; a++) ok = plan.aggs[a].fn == AG_COUNT_STAR || plan.aggs[a].col != s;
      tuple_keyslots |= 1u << s;
      tkeys.emplace_back(shape_cols[s], key.wstride);
    }
    if (ok) {
      std::sort(tkeys.begin(), tkeys.end());
      tuple = table->ensure_tuple_pages(tkeys, verbose, stream);
    }
    if (!tuple) tuple_keyslots = 0;
  }
  {
    const char* sw = getenv("PQB_AGG_FORMS");   // A/B switch: 0 = every slot reads its index pages
    // not with COUNT(DISTINCT) or MEDIAN / PERCENTILE_CONT: their kernel instantiations carry no agg-page paths (their
    // registers would spill there)
    if (!(sw && sw[0] == '0') && agg_kernel && n_flat && d.table && !plan.ndist && !plan.npct) {
      for (uint32_t s = 0; s < ncols; s++) {
        if ((tuple_keyslots >> s) & 1u) continue;   // the tuple pages serve the key slots
        bool as_key = false, as_value = false, other = false;
        for (uint32_t l = 0; l < nleaves; l++) other |= plan.leaves[l].col == s;
        int key = -1;
        for (uint32_t k = 0; k < d.n_group_by; k++)
          if (plan.keys[k].col == s) {
            if (plan.keys[k].kind == KK_DICT_LUT) { as_key = true; key = int(k); }
            else other = true;   // KK_BIN reads the values, KK_BOOL has no dictionary
          }
        for (uint32_t a = 0; a < d.n_aggs; a++) {
          const DevAgg& ag = plan.aggs[a];
          if (ag.fn == AG_COUNT_STAR || ag.col != s) continue;
          if (ag.fn == AG_COUNT_DISTINCT) other = true;
          else if (bool_min_max(ag)) other = true;   // reads the bits of its pages
          // MIN / MAX over Utf8 reads group ids: the id pages of a key column serve it (value pages are numeric only)
          else if (ag.fn >= AG_SUM && ag.fn <= AG_AVG && !rank_min_max(ag)) as_value = true;   // COUNT(col) reads the validity bits only: any form serves it
        }
        if (other || as_key == as_value) continue;
        const int tc_i = shape_cols[s];
        const ColSide& cs = table->sides[tc_i];
        if (as_value) {
          const uint8_t kind = plan.cols[s].kind;
          if ((kind != DK_I64 && kind != DK_F64) || !table->ensure_for_pages(tc_i, kind == DK_F64, stream)) continue;
          form_bw[s] = std::max(cs.for_bw, cs.for_rest_bw);
          value_forms |= 1u << s;
        } else {
          // id pages hold the local numbering: a query in the ranks' agreed numbering keeps the gid LUT
          if (plan.keys[key].gid != cs.d_gid || !table->ensure_id_pages(tc_i, stream)) continue;
          form_bw[s] = std::max(cs.ids_bw, key_bw32[s]);
        }
        plan.agg_forms |= 1u << s;
        if (verbose)
          fprintf(stderr, "[pqb] slot %u (%s): %s pages, %u bits, staged at %u bits (index pages: %u), %.1f MB held by the table\n", s,
                  table->columns[tc_i].name.c_str(), as_value ? "value" : "id", as_value ? cs.for_bw : cs.ids_bw, form_bw[s],
                  std::max(shape->flat_max_bw[s], key_bw32[s]),
                  double(as_value ? cs.for_bytes : cs.ids_bytes) / 1e6);
      }
    }
  }
  // the tuple query's page table copies the agg pages as they stand after this query's last ensure_* above, so that every
  // value page a marked slot's stage was sized for is in it.  Without the memory for the copy the key slots read their
  // index pages through the gid LUT (they asked for no id pages above)
  if (tuple) tuple_pages_tbl = table->tuple_page_table(*tuple, stream);
  if (tuple && tuple_pages_tbl) {
    for (uint32_t k = 0; k < d.n_group_by; k++)
      if (shape_cols[plan.keys[k].col] == tuple->lead) tkey = plan.keys[k];
    tkey.card = tuple->n_tuples;
    tkey.stride = 1;
    tkey.wstride = 1;
    for (uint32_t s = 0; s < ncols; s++)
      if (((tuple_keyslots >> s) & 1u) && s != tkey.col) plan.cols[s].staged = 0;
    plan.nslots = tuple->n_tuples;
    plan.agg_forms |= 1u << tkey.col;
    form_bw[tkey.col] = tuple->bw;
  } else {
    tuple.reset();
  }
  if (verbose && tuple)
    fprintf(stderr, "[pqb] group slots: tuple pages, lead column %s, %u tuples, %u bits, built in %.2f ms\n",
            table->columns[tuple->lead].name.c_str(), tuple->n_tuples, tuple->bw, tuple->build_ms);
  else if (verbose && agg_kernel && d.n_group_by >= 2)
    fprintf(stderr, "[pqb] group slots: per-key ids (mixed radix)\n");
  mark("side tables ready");
  // ---- shared-memory layout of k_scan (items the flat kernels do not take) ----
  SmemLayout L{};
  size_t smem_fixed = 0;
  if (n_general) {
    uint32_t off = align_up(uint32_t(sizeof(ScanCtl)), 128);
    for (uint32_t s = 0; s < ncols; s++) {
      // window = bytes of one slab at the widest index + one header per 8 values + alignment slop;
      // anything denser makes the kernel shrink the slab (always correct, only slower)
      L.defwin_cap[s] = plan.cols[s].max_def ? align_up(kSlabRows / 8 + kSlabRows / 16 + 64, 16) : 0;
      L.valwin_cap[s] = plan.cols[s].has_dict ? valwin_cap_for_bw(plan.cols[s].max_bw) : 0;
      if (plan.cols[s].has_delta) L.valwin_cap[s] = std::max<uint32_t>(L.valwin_cap[s], align_up(kDeltaWindowBytes, 16));
      for (int b = 0; b < 2; b++) { L.defwin[s][b] = off; off += align_up(L.defwin_cap[s] + 16, 128); }
      for (int b = 0; b < 2; b++) { L.valwin[s][b] = off; off += align_up(L.valwin_cap[s] + 16, 128); }
      L.valid[s] = off; off += align_up((kSlabWords + 2) * 4, 16);
      L.rank[s] = off; off += kSlabWords * 4;
      // staging: u32 dictionary indices, or i64 values of DELTA_BINARY_PACKED pages
      L.idx[s] = (plan.cols[s].has_dict || plan.cols[s].has_delta) ? off : 0;
      off += plan.cols[s].has_delta ? kSlabRows * 8 : (plan.cols[s].has_dict ? kSlabRows * 4 : 0);
      L.defdir[s] = off; off += kMaxDirEntries * sizeof(DirEntry);
      for (int b = 0; b < 2; b++) {   // DirEntry / DeltaEntry records (DeltaEntry holds an int64): 16-byte aligned
        off = align_up(off, 16);
        L.valdir[s][b] = off;
        off += std::max<uint32_t>(kMaxDirEntries * sizeof(DirEntry), plan.cols[s].has_delta ? kMaxDeltaEntries * sizeof(DeltaEntry) : 0);
      }
    }
    off = align_up(off, 16);
    L.leafT = off; off += std::max<uint32_t>(nleaves, 1) * kLeafWords * 4;
    L.sel = off; off += kSlabWords * 4;
    L.lutc = off; if (plan.fast_and) off += nleaves * kLutCacheBytes;
    off = align_up(off, 128);
    L.acc = off;
    smem_fixed = off;
  }

  // ---- shared-memory layout of the flat kernels ----
  FlatLayout FL{};
  if (n_flat) {
    // barriers, then one FlatStage record per stage (with plan.ncols column entries), then the stage buffers
    const uint32_t meta_stride = align_up(uint32_t(offsetof(FlatStage, col) + ncols * sizeof(FlatStageCol)), 16);
    const uint32_t ctl_bytes = align_up(uint32_t(sizeof(FlatCtl)), 128) + 128;   // + alignment slack of the first stage buffer
    FL.meta0 = align_up(uint32_t(sizeof(FlatCtl)), 16);
    FL.meta_stride = meta_stride;
    plan.direct8 = 0;
    plan.dbg = (getenv("PQB_FILTER_NOWORK") ? 1u : 0u) | (getenv("PQB_AGG_NOWORK") ? 2u : 0u);   // measurement: how fast can the producer + TMA feed the consumers?
    if (agg_kernel) plan.direct8 = 1;   // k_flat_agg reads 8-byte values in place (measured: 4 % faster than staging them, and room for twice the rows per slab)
    auto stage_bytes_for = [&](uint32_t S) {
      uint32_t off = 0;
      for (uint32_t s = 0; s < ncols; s++) {
        FL.col_off[s] = off;
        FL.col_voff[s] = off;
        if (!plan.cols[s].staged) continue;
        const uint32_t bw = ((plan.agg_forms >> s) & 1u) ? form_bw[s] : std::max(shape->flat_max_bw[s], key_bw32[s]);
        const uint32_t cap = std::max<uint32_t>((shape->flat_plain8[s] && !plan.direct8) ? S * 8 : 0, (S * bw + 7) / 8);
        off += align_up(cap + 48, 128);   // + the bit phase of a piece that starts inside a page, + over-read slack
        if (shape->flat_nullable[s]) { FL.col_voff[s] = off; off += align_up(S / 8 + 48, 128); }   // validity bits of pages with NULLs
      }
      return std::max<uint32_t>(off, 128);
    };
    const uint32_t avail = uint32_t(ctx.smem_optin()) - ctl_bytes - 256 - (agg_kernel ? 3 * meta_stride : 0);
    if (!agg_kernel) {
      // six CTAs per SM (160 threads, 64 registers): a CTA may use a sixth of the SM's shared memory.  A stage is one
      // warp's slab (<= 2048 rows); the ring is a power of two and at least as deep as there are consumer warps (a
      // ticket must never meet the stage's previous fill still pending: the barrier's parity has one bit)
      uint32_t ctas = 6;
      if (const char* e = getenv("PQB_FILTER_CTAS")) ctas = std::max(1, std::min(8, atoi(e)));   // experiment switch
      const uint32_t budget = (uint32_t(ctx.smem_per_sm()) - ctas * 1024) / ctas - ctl_bytes;   // the system keeps 1 KB of every CTA's share
      uint32_t S = kFilterSlabRows;
      while (S > 128 && uint32_t(kFilterConsumerWarps) * (stage_bytes_for(S) + meta_stride) > budget) S >>= 1;
      FL.stage_bytes = stage_bytes_for(S);
      const uint32_t per = FL.stage_bytes + meta_stride;
      if (uint32_t(kFilterConsumerWarps) * per > avail) throw Error(PQ_ERR_UNSUPPORTED, "query needs more shared memory than one SM has");
      uint32_t n = std::max<uint32_t>(budget, uint32_t(kFilterConsumerWarps) * per) / per;
      if (const char* e = getenv("PQB_FILTER_STAGES")) n = std::min<uint32_t>(n, uint32_t(std::max(1, atoi(e))));   // experiment switch
      n = std::max<uint32_t>(uint32_t(kFilterConsumerWarps), std::min<uint32_t>(n, uint32_t(kFlatStagesMax)));
      while (n & (n - 1)) n &= n - 1;   // largest power of two
      FL.nstages = n;
      plan.flat_slab_rows = S;
      plan.hot_slots = 0;
    } else {
      // one CTA per SM: the hot part of the accumulator table next to the stages
      const uint64_t full = plan.hashed ? 0 : uint64_t(plan.nslots) * cells * 8;   // hashed: no hot table in shared memory
      auto fit_krows = [&]() {
        uint32_t krows = plan.hashed ? 4 : 8;   // the hashed instantiation exists for 4 rows per thread (64-bit slots: registers)
        if (rx_bytes && !plan.hashed) krows = 2;   // so do the RX ones, and for 2 when not hashed
        if (const char* e = plan.hashed ? nullptr : getenv("PQB_AGG_KROWS")) krows = std::max(1, std::min(8, atoi(e)));   // experiment switch
        while (krows & (krows - 1)) krows &= krows - 1;
        while (krows > 1 && 2 * stage_bytes_for(kAggConsumers * krows) + std::min<uint64_t>(full, 96 * 1024) > avail) krows >>= 1;
        return krows;
      };
      uint32_t krows = fit_krows();
      // A thread decodes a value page for all KR rows of its instantiation, selected or not (a row mask there made the
      // <8> instantiation spill more): over a slab of fewer than KR x kAggConsumers rows its last rows would lie past
      // the stage -- in the next stage, or past the CTA's shared memory.  The hashed instantiation is <4> and the
      // narrowest dense one <2>, so a query whose stages leave room for fewer rows per thread reads index pages.
      if (agg_kr(plan, rx_bytes, krows) > krows && (plan.agg_forms & value_forms)) {
        if (verbose)
          fprintf(stderr, "[pqb] value pages off: k_flat_agg<%u> is wider than its %u-row slab\n", agg_kr(plan, rx_bytes, krows),
                  kAggConsumers * krows);
        plan.agg_forms &= ~value_forms;
        value_forms = 0;
        krows = fit_krows();
      }
      const uint32_t S = kAggConsumers * krows;
      FL.stage_bytes = stage_bytes_for(S);
      if (2 * FL.stage_bytes + cells * 8 > avail) throw Error(PQ_ERR_UNSUPPORTED, "query needs more shared memory than one SM has");
      FL.nstages = 2;
      uint32_t left = avail - 2 * FL.stage_bytes;
      if (full + FL.stage_bytes <= left && FL.nstages < (uint32_t)kFlatStagesMax) { FL.nstages = 3; left -= FL.stage_bytes; }
      if (const char* e = getenv("PQB_AGG_STAGES")) {   // experiment switch: a deeper ring at the price of hot slots
        const uint32_t want = uint32_t(std::max(2, std::min(int(kFlatStagesMax), atoi(e))));
        while (FL.nstages < want && left >= FL.stage_bytes + meta_stride + 64 * cells * 8) { FL.nstages++; left -= FL.stage_bytes + meta_stride; }
      }
      // the hottest groups own a cell per lane (no same-address lanes inside a warp): 31 more cells each
      const uint32_t cap = left / (cells * 8);
      uint32_t T = 8;
      if (const char* e = getenv("PQB_LANE_SLOTS")) T = uint32_t(std::max(0, atoi(e)));   // experiment switch
      if (const char* e = getenv("PQB_F64_GLOBAL")) if (atoi(e)) T = 0;   // that experiment sends hot f64 cells to L2 by SLOT: no per-lane cells
      T = std::min<uint32_t>(T, plan.nslots);
      while (T && cap < 64u * T) T >>= 1;
      if (plan.hashed) T = 0;
      plan.lane_slots = T;
      plan.hot_slots = plan.hashed ? 0u : uint32_t(std::min<uint64_t>(plan.nslots, cap - 31u * T));
      if (const char* hs = plan.hashed ? nullptr : getenv("PQB_HOT_SLOTS")) plan.hot_slots = std::max(T, std::min<uint32_t>(plan.hot_slots, uint32_t(atoi(hs))));   // experiment switch
      plan.flat_slab_rows = S;
      plan.flat_krows = krows;
    }
    FL.stage0 = align_up(FL.meta0 + FL.nstages * meta_stride, 128);
    FL.acc = align_up(FL.stage0 + FL.nstages * FL.stage_bytes, 128);
    FL.total = FL.acc + (agg_kernel ? (plan.hot_slots + 31u * plan.lane_slots) * cells * 8 : 0);
    if (FL.total > ctx.smem_optin()) throw Error(PQ_ERR_UNSUPPORTED, "query needs more shared memory than one SM has");
  }

  // ---- per-query device state ----
  Timer t_all, t_scan;
  PQB_CUDA(cudaEventRecord(t_all.a, stream));
  DevBuf<uint8_t> d_lit; d_lit.upload(lit_pool, stream);
  DevBuf<uint8_t> d_live;
  const bool pruned = nrg < nrg_table;
  if (pruned) d_live.upload(rg_live, stream);
  DevBuf<uint8_t> d_luts; d_luts.alloc(std::max<uint64_t>(lut_total, 16), stream);
  DevBuf<unsigned long long> d_counters; d_counters.alloc(8, stream); d_counters.zero();
  metrics.h2d_bytes += lit_pool.size() + (pruned ? rg_live.size() : 0);

  pa.arena = table->d_arena;
  pa.chunks = shape->d_chunks;
  pa.n_chunks = nrg_table * ncols;
  pa.ncols = ncols;
  pa.rg_live = pruned ? d_live.p : nullptr;
  pa.luts = d_luts.p;
  pa.lit_pool = d_lit.p;
  pa.counters = d_counters.p;
  if (nrg && ncols && any_lut) {
    dim3 grid(pa.n_chunks, std::min<uint32_t>((max_dict_n + 255) / 256, 64));
    k_leaf_luts<<<grid, 256, 0, stream>>>(pa, plan);
    launches++;
  }

  // ---- accumulators ----
  DevBuf<unsigned long long> d_acc, d_hkeys;
  size_t smem_total = smem_fixed;
  plan.replicas = 1;
  plan.smem_share = 8;
  plan.f64_global = 0;
  if (const char* e = getenv("PQB_SMEM_SHARE")) plan.smem_share = uint32_t(atoi(e));
  if (const char* e = getenv("PQB_F64_GLOBAL")) plan.f64_global = uint32_t(atoi(e));
  if (agg_kernel) {
    // Cold group slots go to L2 with fire-and-forget reductions; L2 serialises same-address atomics, so the
    // table is kept in a few copies (CTA b adds into copy b mod replicas) as long as all copies stay L2 resident:
    // together they take at most a quarter of the L2, the rest is left to the column data streaming through it
    // (H100, C4's 50 000 groups: 1-4 copies time the same, 8 copies +3 %, 17 copies +40 %).
    if (n_flat && (plan.hot_slots < plan.nslots || plan.smem_share < 8 || plan.f64_global)) {
      const uint64_t tbytes = uint64_t(plan.nslots) * cells * 8;
      const uint64_t copies_bytes = uint64_t(ctx.l2_bytes()) / 4;
      uint32_t r = uint32_t(std::min<uint64_t>(32, copies_bytes / std::max<uint64_t>(tbytes, 1)));
      if (const char* e = getenv("PQB_REPLICAS")) r = uint32_t(atoi(e));
      plan.replicas = std::max<uint32_t>(1, std::min<uint32_t>(r, uint32_t(ctx.sm_count())));
    }
    if (plan.hashed) {
      plan.replicas = 1;
      d_hkeys.alloc(plan.nslots, stream);
      PQB_CUDA(cudaMemsetAsync(d_hkeys.p, 0xff, size_t(plan.nslots) * 8, stream));
    }
    d_acc.alloc(size_t(plan.nslots) * cells * plan.replicas, stream);
    {
      const uint64_t ncell = uint64_t(plan.nslots) * cells * plan.replicas;
      k_acc_init<<<uint32_t(std::min<uint64_t>(2048, (ncell + 255) / 256)), 256, 0, stream>>>(d_acc.p, plan.nslots, plan.n_acc, cells, plan.replicas, plan);
    }
    launches++;
    size_t acc_bytes = size_t(plan.nslots) * cells * 8;
    if (n_general && smem_fixed + acc_bytes + 1024 <= ctx.smem_optin()) { plan.smem_acc = 1; smem_total = smem_fixed + acc_bytes; }
  }
  L.total = uint32_t(smem_total);
  if (smem_total > ctx.smem_optin()) throw Error(PQ_ERR_UNSUPPORTED, "query needs more shared memory than one SM has");

  // ---- selection bitmap / counts ----
  const bool projecting = want_rows && d.n_projection > 0;
  if (projecting && n_general)
    throw Error(PQ_ERR_UNSUPPORTED, "projection of column values needs a flat-store copy of every page it reads: PLAIN (dictionary-fallback) "
                                    "string pages are not projected on the GPU yet: " + shape->why_general);
  plan.write_bitmap = want_rows ? 1 : 0;
  DevBuf<uint32_t> d_bitmap, d_item_counts;
  // k_scan ORs partial words into its bitmap regions: they start zeroed.  The flat filter kernel stores
  // every word of its items, no memset needed.
  if (want_rows) { d_bitmap.alloc(std::max<uint32_t>(shape->bitmap_words, 1), stream); if (n_general) d_bitmap.zero(); }
  d_item_counts.alloc(std::max<size_t>(items.size(), 1), stream);
  d_item_counts.zero();
  if (want_rows) algo_bytes += metrics.rows_scanned / 8;
  metrics.algorithmic_bytes = algo_bytes;

  mark("prep kernels queued");
  // ---- the fused scans ----
  DevScanArgs sa{};
  sa.arena = table->d_arena;
  sa.pages = table->d_pages;
  sa.chunks = shape->d_chunks;
  sa.items = shape->d_items;
  sa.luts = d_luts.p;
  sa.lit_pool = d_lit.p;
  sa.rg_live = pruned ? d_live.p : nullptr;
  sa.flat = table->d_flat;
  sa.fpages = d_kpages.p ? d_kpages.p : table->d_flat_pages;
  sa.apages = tuple ? tuple_pages_tbl.get() : plan.agg_forms ? table->d_agg_pages : nullptr;
  sa.bitmap = d_bitmap.p;
  sa.item_counts = d_item_counts.p;
  sa.acc = d_acc.p;
  sa.hkeys = d_hkeys.p;
  sa.counters = d_counters.p;
  PQB_CUDA(cudaEventRecord(t_scan.a, stream));
  if (n_flat && nrg) {
    uint32_t grid;
    if (agg_kernel) {
      grid = std::min<uint32_t>(n_flat, uint32_t(ctx.sm_count()));
      if (const char* g = getenv("PQB_GRID")) grid = std::max(1, atoi(g));
      DevPlan kplan = plan;   // tuple pages: the kernel's plan has the one key tkey
      if (tuple) {
        kplan.nkeys = 1;
        kplan.keys[0] = tkey;
      }
      auto go = [&](auto kern) {
        PQB_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, int(ctx.smem_optin())));
        kern<<<grid, kAggThreads, FL.total, stream>>>(kplan, FL, sa);
      };
      if (rx_bytes) {   // a regular expression or an IN list over pages without a dictionary: the out-of-line leaves
        if (plan.npct) {
          if (plan.hashed) go(k_flat_agg<4, true, false, true, true>);
          else go(k_flat_agg<2, false, false, true, true>);
        } else if (plan.ndist) {
          if (plan.hashed) go(k_flat_agg<4, true, true, false, true>);
          else go(k_flat_agg<2, false, true, false, true>);
        } else if (plan.hashed) go(k_flat_agg<4, true, false, false, true>);
        else go(k_flat_agg<2, false, false, false, true>);
      }
      else if (plan.npct) {   // MEDIAN / PERCENTILE_CONT: the instantiations with the pair emission
        if (plan.hashed) go(k_flat_agg<4, true, false, true>);
        else if (plan.flat_krows >= 8) go(k_flat_agg<8, false, false, true>);
        else if (plan.flat_krows >= 4) go(k_flat_agg<4, false, false, true>);
        else go(k_flat_agg<2, false, false, true>);
      }
      else if (plan.ndist) {   // COUNT(DISTINCT): the instantiations with the presence pass
        if (plan.hashed) go(k_flat_agg<4, true, true>);
        else if (plan.flat_krows >= 8) go(k_flat_agg<8, false, true>);
        else if (plan.flat_krows >= 4) go(k_flat_agg<4, false, true>);
        else go(k_flat_agg<2, false, true>);
      }
      else if (plan.hashed) go(k_flat_agg<4, true>);           // key space wider than the dense table: cells through the hash table
      else if (plan.flat_krows >= 8) go(k_flat_agg<8, false>);   // rows per thread and slab: the widest instantiation the stages leave room for
      else if (plan.flat_krows >= 4) go(k_flat_agg<4, false>);
      else go(k_flat_agg<2, false>);
    } else {
      auto go = [&](auto kern) {
        PQB_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, int(ctx.smem_optin())));
        int occ = 1;
        PQB_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, kern, kFilterThreads, FL.total));
        if (occ < 1) occ = 1;
        grid = std::min<uint32_t>(n_flat, uint32_t(ctx.sm_count() * occ));
        if (const char* g = getenv("PQB_GRID")) grid = std::max(1, atoi(g));
        kern<<<grid, kFilterThreads, FL.total, stream>>>(plan, FL, sa);
      };
      if (plan.conj || !plan.npred) go(k_flat_filter<true>);   // conjunctions: the instantiation without the Kleene stack
      else go(k_flat_filter<false>);
    }
    PQB_CUDA(cudaGetLastError());
    launches++;
    if (verbose && agg_kernel)
      fprintf(stderr, "[pqb] k_flat_agg<%u%s%s%s%s>: %u CTAs, %u B smem/CTA, %u stages x %u B, slab %u rows, hot slots %u of %u, "
              "lane slots %u, %u copies, smem share %u, f64 global %u, value-page slots %d, id-page slots %d, %u flat items\n",
              agg_kr(plan, rx_bytes, plan.flat_krows), plan.hashed ? ",hashed" : "", plan.ndist ? ",DIST" : "", plan.npct ? ",PCT" : "",
              rx_bytes ? ",RX" : "", grid, FL.total, FL.nstages, FL.stage_bytes, plan.flat_slab_rows, plan.hot_slots, plan.nslots,
              plan.lane_slots, plan.replicas, plan.smem_share, plan.f64_global, __builtin_popcount(plan.agg_forms & value_forms),
              __builtin_popcount(plan.agg_forms & ~value_forms), n_flat);
    else if (verbose)
      fprintf(stderr, "[pqb] k_flat_filter<%s>: %u live leaves, %u CTAs, %u B smem/CTA, %u stages x %u B, slab %u rows, hot slots %u of %u, "
              "%u copies, %u flat items\n", (plan.conj || !plan.npred) ? "CONJ" : "KLEENE", plan.nleaves,
              grid, FL.total, FL.nstages, FL.stage_bytes, plan.flat_slab_rows, plan.hot_slots, plan.nslots, plan.replicas, n_flat);
  }
  if (n_general && nrg) {
    if (n_flat) { PQB_CUDA(cudaMemsetAsync(d_counters.p + 2, 0, 8, stream)); }   // the work-queue head
    PQB_CUDA(cudaFuncSetAttribute(k_scan, cudaFuncAttributeMaxDynamicSharedMemorySize, int(ctx.smem_optin())));
    int occ = 1;
    PQB_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, k_scan, kScanThreads, smem_total));
    if (occ < 1) occ = 1;
    uint32_t grid = std::min<uint32_t>(uint32_t(items.size()), uint32_t(ctx.sm_count() * occ));
    if (const char* g = getenv("PQB_GRID")) grid = std::max(1, atoi(g));   // debugging aid: forces several items per CTA
    if (verbose)
      fprintf(stderr, "[pqb] k_scan: %u CTAs x %d threads, %zu B smem/CTA, %d CTAs/SM, %u of %zu items\n", grid,
              kScanThreads, size_t(smem_total), occ, n_general, items.size());
    k_scan<<<grid, kScanThreads, smem_total, stream>>>(plan, L, sa);
    PQB_CUDA(cudaGetLastError());
    launches++;
  }
  if (agg_kernel && plan.replicas > 1) {
    k_acc_reduce<<<std::min<uint32_t>(1024, (plan.nslots * cells + 255) / 256), 256, 0, stream>>>(d_acc.p, plan.nslots, cells, plan.replicas, plan);
    launches++;
  }
  PQB_CUDA(cudaEventRecord(t_scan.b, stream));

  if (getenv("PQB_DEBUG_ITEMS")) {
    std::vector<uint32_t> ic(items.size());
    PQB_CUDA(cudaMemcpyAsync(ic.data(), d_item_counts.p, ic.size() * 4, cudaMemcpyDeviceToHost, stream));
    PQB_CUDA(cudaStreamSynchronize(stream));
    for (size_t i = 0; i < ic.size(); i++)
      fprintf(stderr, "item %zu rg %u row0 %u nrows %u g0 %llu flags %u count %u\n", i, items[i].rg, items[i].row0, items[i].nrows,
              (unsigned long long)items[i].global_row0, items[i].fast, ic[i]);
  }
  mark("scan queued");

  // ---- results ----
  batch_rows_ = d.batch_size ? d.batch_size : 20000;
  std::vector<int> out_type(d.n_columns);
  for (uint32_t c = 0; c < d.n_columns; c++) out_type[c] = out_type_of(c);
  ResultTail tail{d, table, *shape, plan, items, out_type, slot_of, shape_cols, qk, nn_is_rows, agg_out_type, pct_p, rank_luts,
                  lit_pool, tuple, d_acc, d_hkeys, d_counters, d_bitmap, d_item_counts, d_pct_count, d_pct_slots, d_pct_keys,
                  roa, row_nulls_first, d_opages, t_all, t_scan, cells, ncols, nrg, key_space, allreduce, multi, merge_rows,
                  launches, stream, verbose, t_begin, metrics, batches_, dev_blocks_};
  if (agg_kernel) tail.groups();
  else if (projecting || row_order) tail.rows();
  else tail.selection();
  tail.finish();
}

// ---- the result tail ----
void ResultTail::check_corrupt() const {
  if (h_counters[1]) throw Error(PQ_ERR_CORRUPT, "corrupt or unsupported page encoding met on the device (code " + std::to_string(h_counters[1]) + ")");
}

std::string ResultTail::agg_name(uint32_t a) const {
  static const char* fn_names[] = {"count(*)", "count", "sum", "min", "max", "avg", "count(distinct", "median", "percentile_cont"};
  const DevAgg& ag = plan.aggs[a];
  if (ag.fn == AG_PERCENTILE_CONT) {   // p in shortest round-trip form: percentile_cont(latency_ms, 0.99)
    char buf[32];
    const auto r = std::to_chars(buf, buf + sizeof(buf), pct_p[a]);
    return std::string("percentile_cont(") + d.columns[d.aggs[a].col].name + ", " + std::string(buf, r.ptr) + ")";
  }
  return ag.fn == AG_COUNT_STAR ? std::string("count(*)")
                                : std::string(fn_names[ag.fn]) + (ag.fn == AG_COUNT_DISTINCT ? " " : "(") + d.columns[d.aggs[a].col].name + ")";
}

// an aggregate's output layout: MIN / MAX over Utf8 or Boolean, or (MIN / MAX over Date32) 4-byte values, like the keys'
uint8_t ResultTail::agg_kind(uint32_t a) const {
  return rank_min_max(plan.aggs[a]) ? DK_STR : bool_min_max(plan.aggs[a]) ? DK_BOOL : agg_out_type[a] == PQ_T_DATE32 ? DK_I32 : DK_I64;
}

// a result block up to kKeepDeviceResult stays on the device until the query closes: JSON egress formats it where it is
void ResultTail::keep_device(const std::shared_ptr<PinnedBlock>& block, DevBuf<uint8_t>& d_block, uint64_t bytes) {
  if (!block || !d_block.p || bytes > kKeepDeviceResult) return;
  block->dev = d_block.p;
  d_block.p = nullptr;
  dev_blocks.push_back(block);
}

// The batches of the first n rows of a block laid out by L, which may have room for more (an empty result: one batch
// of no rows).  The NULL counts are indexed by the batches of the layout, not by the batches the rows fill.
void ResultTail::slice(const BlockLayout& L, const std::vector<BlockCol>& cols, const std::shared_ptr<PinnedBlock>& block, uint64_t n) {
  const uint32_t* nulls = reinterpret_cast<const uint32_t*>(block->p + L.nulls_off);
  for (uint64_t b = 0, r0 = 0; r0 < n || b == 0; b++, r0 += L.batch_rows) {
    OutBatch ob;
    ob.rows = int64_t(std::min<uint64_t>(L.batch_rows, n - r0));
    for (size_t c = 0; c < cols.size(); c++) {
      const BlockCol& bc = cols[c];
      OutColumn oc;
      oc.name = bc.name;
      oc.type = bc.type;
      oc.block = block;
      oc.null_count = ob.rows && c < L.ncolumns ? nulls[c * L.nbatches + b] : 0;
      oc.validity_off = bc.valid_off + b * L.wpb * 4;
      if (bc.kind == DK_STR) { oc.offsets_off = bc.val_off + r0 * 4; oc.values_off = bc.data_off; }
      else if (bc.kind == DK_BOOL) oc.values_off = bc.val_off + b * L.wpb * 4;
      else oc.values_off = bc.val_off + r0 * (bc.kind == DK_I32 ? 4 : 8);
      ob.cols.push_back(std::move(oc));
    }
    batches.push_back(std::move(ob));
  }
}

// One row built on the host (a global aggregate over zero rows, COUNT(*) alone) in a heap block: every aggregate holds
// `value`, or NULL where `null` says so, and a window's columns hold 1 (the one row of its one partition)
void ResultTail::one_row(std::vector<BlockCol> cols, const std::vector<bool>& null, unsigned long long value) {
  const size_t naggs = cols.size();
  for (const std::string& w : win_names) cols.push_back({w});
  BlockLayout L(1, batch_rows, uint32_t(cols.size()));
  for (BlockCol& c : cols) L.column(c);
  const std::shared_ptr<PinnedBlock> block = heap_block(L.off);
  for (size_t c = 0; c < cols.size(); c++) {
    const unsigned long long v = c < naggs ? value : 1;
    if (c < naggs && null[c]) reinterpret_cast<uint32_t*>(block->p + L.nulls_off)[c] = 1;   // one batch: column c's count
    else std::memcpy(block->p + cols[c].val_off, &v, 8);
  }
  slice(L, cols, block, 1);
}

// A filter scan's result sized from the rows the last scan of this shape selected.  fill(cap) queues a result for `cap`
// rows into `block` and returns the bytes it copies back.  A repeat of the query lays the result out for the previous
// answer plus a margin (at least min_cap rows) before the selected-row total is on the host, and keeps it when the rows
// fit; otherwise, and on a first run, it is laid out for the rows once the total is known.  `then` marks the verbose
// timeline once the total is on the host.  Returns the rows kept, min(total, LIMIT).
template <class Fill>
unsigned long long ResultTail::sized_pass(unsigned long long min_cap, std::shared_ptr<PinnedBlock>& block, Fill fill, const char* then) {
  const unsigned long long hint = shape.last_total.load();
  bool done = false;
  if (hint != ~0ull) {
    const unsigned long long cap = std::max(min_cap, std::min(lim, hint + hint / 8 + 1024));
    const uint64_t bytes = fill(cap);
    PQB_CUDA(cudaStreamSynchronize(stream));
    if (std::min(total, lim) <= cap) { done = true; metrics.d2h_bytes += bytes; }
    else block.reset();
  } else {
    PQB_CUDA(cudaStreamSynchronize(stream));
  }
  if (then) mark(then);
  const unsigned long long keep = std::min(total, lim);
  if (!done && keep) {
    const uint64_t bytes = fill(keep);
    PQB_CUDA(cudaStreamSynchronize(stream));
    metrics.d2h_bytes += bytes;
  }
  shape.last_total.store(total);
  return keep;
}

// bitmap-driven stream compaction on the device: per-item prefix, then one CTA per item.  The selected-row total is
// needed on the host to size the result; a repeat of the same query shape sizes it from the previous answer and skips
// that round trip (sized_pass).
void ResultTail::count_selected() {
  d_total.alloc(2, stream);   // the selected rows; under PQ_QUERY_ALLREDUCE also the ranks that met a corrupt page
  d_item_base.alloc(std::max<size_t>(items.size(), 1), stream);
  if (!items.empty()) {
    k_item_prefix<<<1, 1024, 0, stream>>>(d_item_counts.p, uint32_t(items.size()), d_item_base.p, d_total.p);
    launches++;
  } else {
    PQB_CUDA(cudaMemsetAsync(d_total.p, 0, 8, stream));
  }
  PQB_CUDA(cudaMemcpyAsync(h_counters, d_counters.p, sizeof(h_counters), cudaMemcpyDeviceToHost, stream));
  PQB_CUDA(cudaMemcpyAsync(&total, d_total.p, 8, cudaMemcpyDeviceToHost, stream));
  metrics.d2h_bytes += 8 + sizeof(h_counters);
}

// an aggregate table: the all-reduce or hashed merge of the ranks' tables, MEDIAN / PERCENTILE_CONT, ORDER BY or a
// window, the result block assembled on the device
void ResultTail::groups() {
  // multi-GPU: the partial tables meet in ONE grouped all-reduce (SURVEY §8e): one NCCL launch,
  // per array the reduction its aggregate needs
  Timer t_ar;
  std::unique_ptr<MergeRun> merge;   // a hashed GROUP BY: every rank's listed groups gathered and merged instead
  if (allreduce && plan.hashed) {
    merge = std::make_unique<MergeRun>();
    launches += merge->run(plan, cells, key_space, std::min<uint64_t>(plan.nslots, std::max<uint64_t>(metrics.rows_scanned, 1)),
                           d_acc, d_hkeys, d_counters.p, stream, metrics);
  } else if (allreduce) {
    PQB_CUDA(cudaEventRecord(t_ar.a, stream));
    comm_group_begin();
    comm_allreduce_u64(d_acc.p, plan.nslots, 0, stream);
    for (uint32_t a = 0; a < plan.n_acc; a++) {
      uint8_t how = plan.acc_init[a];
      comm_allreduce_u64(d_acc.p + size_t(1 + a) * plan.nslots, plan.nslots, how == 0 ? 0 : how == 1 ? 3 : how == 2 ? 1 : 2, stream);
    }
    if (plan.n_nn) comm_allreduce_u64(d_acc.p + size_t(1 + plan.n_acc) * plan.nslots, size_t(plan.n_nn) * plan.nslots, 0, stream);
    comm_group_end();
    PQB_CUDA(cudaEventRecord(t_ar.b, stream));
  }
  // ---- non-empty groups in ascending slot order (deterministic: the mixed radix of the group ids) ----
  const uint32_t ntiles = (plan.nslots + kSlotTile - 1) / kSlotTile;
  const uint64_t out_cap = std::min<uint64_t>(plan.nslots, std::max<uint64_t>(allreduce ? plan.nslots : metrics.rows_scanned, 1));
  DevBuf<uint32_t> d_tile_counts, d_out_slot;
  DevBuf<unsigned long long> d_tile_base, d_totals;
  d_tile_counts.alloc(ntiles, stream);
  d_tile_base.alloc(ntiles, stream);
  d_totals.alloc(2, stream);
  d_out_slot.alloc(out_cap, stream);
  const uint32_t* order = tuple ? tuple->d_order : nullptr;   // tuple slots: listed in the order of their mixed-radix ids
  k_slot_tile_counts<<<ntiles, 256, 0, stream>>>(d_acc.p, plan.nslots, d_tile_counts.p, order);
  k_item_prefix<<<1, 1024, 0, stream>>>(d_tile_counts.p, ntiles, d_tile_base.p, d_totals.p);
  k_slot_compact<<<ntiles, 256, 0, stream>>>(d_acc.p, plan.nslots, d_tile_base.p, d_out_slot.p, order);
  // rows this rank selected (its own items)
  d_item_base.alloc(std::max<size_t>(items.size(), 1), stream);
  if (!items.empty()) k_item_prefix<<<1, 1024, 0, stream>>>(d_item_counts.p, uint32_t(items.size()), d_item_base.p, d_totals.p + 1);
  else PQB_CUDA(cudaMemsetAsync(d_totals.p + 1, 0, 8, stream));
  launches += 4;
  std::unique_ptr<WindowRun> wrun;       // only for a query with a window over at least one group
  // ---- the result block: every buffer of every batch for n_out groups, assembled on the device and copied to page-locked
  // memory (no synchronise).  n_dev != nullptr: n_out is a capacity, the kernels read the group count on the device.
  // cut: ORDER BY ... LIMIT keeps a subset of the groups ----
  struct Assembled {
    BlockLayout L;       // L.rows: the groups the block has room for (0: none assembled)
    std::vector<BlockCol> cols;
    FinishArgs fa{};
    std::unique_ptr<DevBuf<uint8_t>> d_block;
    std::shared_ptr<PinnedBlock> block;
  };
  auto assemble = [&](uint32_t n_out, const unsigned long long* n_dev) -> Assembled {
    Assembled r;
    r.L = BlockLayout(n_out, batch_rows, d.n_group_by + d.n_aggs + uint32_t(win_names.size()));
    BlockLayout& L = r.L;
    FinishArgs& fa = r.fa;
    for (uint32_t k = 0; k < d.n_group_by; k++) {
      FinishKey& fk = fa.keys[k];
      const uint32_t qc = uint32_t(d.group_by[k]);
      const uint8_t kind = plan.cols[plan.keys[k].col].kind;
      fk.kind = (!qk[k].is_bin && out_type[qc] == PQ_T_DATE32) ? uint8_t(DK_I32) : kind;   // Date32: 4-byte values
      fk.stride = plan.keys[k].stride;
      fk.wstride = plan.keys[k].wstride;
      fk.card = qk[k].card;
      r.cols.push_back({qk[k].is_bin ? std::string("date_bin(") + d.columns[qc].name + ")" : std::string(d.columns[qc].name),
                        qk[k].is_bin ? PQ_T_TS_MS : out_type[qc], uint8_t(fk.kind)});
      L.column(r.cols.back());
      fk.valid_off = r.cols.back().valid_off;
      fk.val_off = r.cols.back().val_off;
      if (qk[k].is_bin) {
        fk.is_bin = 1;
        fk.bin_base = plan.keys[k].bin_base;
        fk.bin_width = plan.keys[k].bin_width;
      } else if (kind != DK_BOOL) {
        const ColSide& cs = table->sides[shape_cols[plan.keys[k].col]];
        if (multi) {   // the dictionary every rank agreed on
          fk.kd_offs = cs.d_glob_kd_offs;
          fk.kd_bytes = cs.d_glob_kd_bytes;
        } else {
          fk.kd_offs = cs.d_kd_offs;
          fk.kd_bytes = cs.d_kd_bytes;
        }
      }
    }
    for (uint32_t a = 0; a < d.n_aggs; a++) {
      fa.aggs[a] = plan.aggs[a];
      fa.nn_is_rows[a] = nn_is_rows[a];
      fa.out_kind[a] = agg_kind(a);
      r.cols.push_back({agg_name(a), agg_out_type[a], fa.out_kind[a]});
      L.column(r.cols.back());
      fa.valid_off[a] = r.cols.back().valid_off;
      fa.val_off[a] = r.cols.back().val_off;
    }
    // MIN / MAX over Utf8: the winning values' bytes, bounded by rows x the longest value of the numbering (any group may
    // hold the longest one)
    for (uint32_t a = 0; a < d.n_aggs; a++) {
      if (fa.out_kind[a] != DK_STR) continue;
      FinishAggStr& s = fa.astr[a];
      const ColSide& cs = table->sides[shape_cols[plan.aggs[a].col]];
      s.kd_offs = multi ? cs.d_glob_kd_offs : cs.d_kd_offs;
      s.kd_bytes = multi ? cs.d_glob_kd_bytes : cs.d_kd_bytes;
      s.inv = rank_luts[a] ? rank_luts[a]->inv : nullptr;   // nullptr: a column in no file, every group NULL
      const uint64_t bound = rank_luts[a] ? uint64_t(n_out) * (multi ? cs.glob_max_len : cs.kd_max_len) : 0;
      if (bound > 0x7fffffffull)
        throw Error(PQ_ERR_UNSUPPORTED, std::string(plan.aggs[a].fn == AG_MIN ? "MIN(" : "MAX(") + d.columns[d.aggs[a].col].name +
                                            "): the strings of one result may exceed 2 GiB");
      s.data_off = r.cols[d.n_group_by + a].data_off = L.take(bound);
    }
    for (const std::string& w : win_names) {
      r.cols.push_back({w});
      r.cols.back().val_off = L.per_row(8);
    }
    // string key bytes: an upper bound keeps the copy to one round trip.  Rows x the longest distinct value; or, as one
    // value of key k sits in at most prod_{j != k}(card_j + 1) groups, that many copies of all its distinct values.
    // Both hold for any subset of the groups (a result cut by ORDER BY ... LIMIT).  Where that bound is large, the
    // exact bytes of the output rows are counted on the device first (one more round trip)
    for (uint32_t k = 0; k < d.n_group_by; k++) {
      FinishKey& fk = fa.keys[k];
      if (fk.kind != DK_STR) continue;
      uint64_t max_len = 0;
      const KeyDict* kd = qk[k].kd;
      max_len = multi ? table->sides[shape_cols[plan.keys[k].col]].glob_max_len : table->sides[shape_cols[plan.keys[k].col]].kd_max_len;
      uint64_t copies = 1;
      for (uint32_t j = 0; j < d.n_group_by; j++)
        if (j != k) copies = std::min<uint64_t>(uint64_t(n_out), copies * (uint64_t(qk[j].card) + 1));
      uint64_t bound = std::min<uint64_t>(uint64_t(n_out) * max_len, copies * kd->bytes.size());
      if (bound > kExactKeyBytes && !wrun) {
        fa.wide = plan.hashed ? d_hkeys.p : tuple ? tuple->d_wide : nullptr;
        fa.out_slot = d_out_slot.p;
        fa.n_out = n_out;
        fa.n_dev = n_dev;
        DevBuf<unsigned long long> total;
        total.alloc(1, stream);
        total.zero();
        k_key_bytes_total<<<std::min<uint32_t>(1024, (n_out + 255) / 256), 256, 0, stream>>>(fa, k, total.p);
        launches++;
        PQB_CUDA(cudaGetLastError());
        unsigned long long exact = 0;
        PQB_CUDA(cudaMemcpyAsync(&exact, total.p, 8, cudaMemcpyDeviceToHost, stream));
        PQB_CUDA(cudaStreamSynchronize(stream));
        bound = exact;
      }
      if (bound > 0x7fffffffull) throw Error(PQ_ERR_UNSUPPORTED, "group key strings of one result exceed 2 GiB");
      fk.data_off = r.cols[k].data_off = L.take(bound);
    }
    L.copy_bytes = L.off;
    for (uint32_t k = 0; k < d.n_group_by; k++)
      if (fa.keys[k].kind == DK_STR) fa.keys[k].len_off = L.per_row(4);   // device-only scratch behind the copied part
    for (uint32_t a = 0; a < d.n_aggs; a++)
      if (fa.out_kind[a] == DK_STR) fa.astr[a].len_off = L.per_row(4);
    r.d_block = std::make_unique<DevBuf<uint8_t>>();
    DevBuf<uint8_t>& d_block = *r.d_block;
    d_block.alloc(L.off, stream);
    PQB_CUDA(cudaMemsetAsync(d_block.p, 0, L.copy_bytes, stream));
    if (wrun) {   // the kept groups' slots in output order, their row_number / partition_rows into the block
      DevBuf<uint32_t> slots;
      slots.alloc(n_out, stream);
      auto col = [&](uint32_t flag) -> long long* {
        if (!(win->flags & flag)) return nullptr;
        const size_t w = (flag == PQ_WINDOW_PARTITION_ROWS && (win->flags & PQ_WINDOW_ROW_NUMBER)) ? 1 : 0;
        return reinterpret_cast<long long*>(d_block.p + r.cols[d.n_group_by + d.n_aggs + w].val_off);
      };
      wrun->fill(d_out_slot.p, n_out, slots.p, col(PQ_WINDOW_ROW_NUMBER), col(PQ_WINDOW_PARTITION_ROWS), stream);
      launches++;
      std::swap(d_out_slot.p, slots.p);   // the old list is freed with `slots`
      std::swap(d_out_slot.n, slots.n);
    }
    fa.acc = d_acc.p;
    fa.wide = plan.hashed ? d_hkeys.p : tuple ? tuple->d_wide : nullptr;
    fa.out_slot = d_out_slot.p;
    fa.out = d_block.p;
    fa.nulls = reinterpret_cast<uint32_t*>(d_block.p + L.nulls_off);
    fa.n_out = n_out;
    fa.n_dev = n_dev;
    fa.nslots = plan.nslots;
    fa.n_acc = plan.n_acc;
    fa.naggs = d.n_aggs;
    fa.nkeys = d.n_group_by;
    fa.batch_rows = batch_rows;
    fa.words_per_batch = L.wpb;
    fa.nbatches = L.nbatches;
    k_agg_finish<<<(n_out + 255) / 256, 256, 0, stream>>>(fa);
    launches++;
    for (uint32_t k = 0; k < d.n_group_by; k++) {
      if (fa.keys[k].kind != DK_STR) continue;
      k_offsets_scan<<<1, 1024, 0, stream>>>(reinterpret_cast<const uint32_t*>(d_block.p + fa.keys[k].len_off), n_out, n_dev,
                                             reinterpret_cast<int32_t*>(d_block.p + fa.keys[k].val_off));
      k_key_gather<<<uint32_t((uint64_t(n_out) * 32 + 255) / 256), 256, 0, stream>>>(fa, k);
      launches += 2;
    }
    for (uint32_t a = 0; a < d.n_aggs; a++) {
      if (fa.out_kind[a] != DK_STR) continue;
      k_offsets_scan<<<1, 1024, 0, stream>>>(reinterpret_cast<const uint32_t*>(d_block.p + fa.astr[a].len_off), n_out, n_dev,
                                             reinterpret_cast<int32_t*>(d_block.p + fa.val_off[a]));
      k_agg_str_gather<<<uint32_t((uint64_t(n_out) * 32 + 255) / 256), 256, 0, stream>>>(fa, a);
      launches += 2;
    }
    PQB_CUDA(cudaGetLastError());
    r.block = std::make_shared<PinnedBlock>();
    r.block->p = ctx.pinned_acquire(L.copy_bytes);
    r.block->bytes = L.copy_bytes;
    PQB_CUDA(cudaMemcpyAsync(r.block->p, d_block.p, L.copy_bytes, cudaMemcpyDeviceToHost, stream));
    PQB_CUDA(cudaEventRecord(t_all.b, stream));
    metrics.d2h_bytes += L.copy_bytes;
    return r;
  };
  // ---- one round trip: an unordered GROUP BY whose plan this shape has answered before lays its result block out for
  // that many groups now, and the block comes back with the group count.  Should the count have grown (other ranks'
  // tables under PQ_QUERY_ALLREDUCE), the block is laid out again after the round trip.  ORDER BY / windows (the count
  // sizes their sort), MEDIAN / PERCENTILE_CONT (their pick runs on the groups) and global aggregates keep two ----
  Assembled pre;
  const bool tail_hint = d.n_group_by && !ordered && !plan.npct;
  uint64_t tail_key = 0;
  if (tail_hint) {
    tail_key = plan_hash(plan, lit_pool, batch_rows) ^ (tuple ? 0x9e3779b97f4a7c15ull : 0ull);   // a tuple plan is not its per-key plan
    uint32_t cap = 0;
    {
      std::lock_guard<std::mutex> lk(shape.hint_mu);
      auto it = shape.groups_hint.find(tail_key);
      if (it != shape.groups_hint.end()) cap = it->second;
    }
    if (const char* e = getenv("PQB_TAIL_CAP")) cap = uint32_t(atoi(e));   // test switch: the block's room in groups
    cap = uint32_t(std::min<uint64_t>(cap, out_cap));
    if (verbose) fprintf(stderr, "[pqb] result tail: %s\n", cap ? ("one round trip, block for " + std::to_string(cap) + " groups").c_str()
                                                                   : "no earlier answer of this plan: two round trips");
    if (cap) pre = assemble(cap, d_totals.p);
  }
  unsigned long long totals[2] = {0, 0};
  std::vector<unsigned int> pct_count(plan.npct, 0u);
  {   // into page-locked memory: a copy to pageable memory holds the host until it is done, and the next copy waits for
      // that.  pinned_acquire hands out any free block of the context's pool that is large enough (1 MB at least)
    PinnedBlock small;
    small.p = ctx.pinned_acquire(16 + sizeof(h_counters) + plan.npct * 4);
    PQB_CUDA(cudaMemcpyAsync(small.p, d_totals.p, 16, cudaMemcpyDeviceToHost, stream));
    PQB_CUDA(cudaMemcpyAsync(small.p + 16, d_counters.p, sizeof(h_counters), cudaMemcpyDeviceToHost, stream));
    if (plan.npct) PQB_CUDA(cudaMemcpyAsync(small.p + 16 + sizeof(h_counters), d_pct_count.p, plan.npct * 4, cudaMemcpyDeviceToHost, stream));
    PQB_CUDA(cudaStreamSynchronize(stream));
    std::memcpy(totals, small.p, 16);
    std::memcpy(h_counters, small.p + 16, sizeof(h_counters));
    if (plan.npct) std::memcpy(pct_count.data(), small.p + 16 + sizeof(h_counters), plan.npct * 4);
  }
  metrics.d2h_bytes += 16 + sizeof(h_counters) + plan.npct * 4;
  if (merge) {   // G is the same on every rank, and no collective follows: every rank throws alike
    merge->report(verbose, uint32_t(totals[0]), metrics);
    if (totals[0] > (1ull << 26)) throw Error(PQ_ERR_UNSUPPORTED, "GROUP BY: more distinct groups than the hashed accumulator table holds (2^26)");
  }
  if (plan.hashed && h_counters[1] == 100) throw Error(PQ_ERR_UNSUPPORTED, "GROUP BY: more distinct groups than the hashed accumulator table holds (2^26)");
  if (plan.ndist && h_counters[1] == kDistinctFull) throw Error(PQ_ERR_UNSUPPORTED, "COUNT(DISTINCT): more distinct (group, value) pairs than the pair set holds (2^27)");
  check_corrupt();
  uint32_t n_out = uint32_t(totals[0]);
  metrics.rows_selected = totals[1];
  if (tail_hint && n_out) {
    std::lock_guard<std::mutex> lk(shape.hint_mu);
    if (shape.groups_hint.size() >= 64 && !shape.groups_hint.count(tail_key)) shape.groups_hint.clear();   // a bound, not an LRU
    shape.groups_hint[tail_key] = n_out;
  }
  if (allreduce && !merge) { float ms = 0; cudaEventElapsedTime(&ms, t_ar.a, t_ar.b); metrics.allreduce_ms = ms; }
  // ---- MEDIAN / PERCENTILE_CONT: sort each column's pairs, pick every group's results into the aggregates' cells ----
  if (plan.npct && n_out) {
    double pct_ms = 0.0;
    for (uint32_t i = 0; i < plan.npct; i++) {
      PctPickArgs pk{};
      for (uint32_t a = 0; a < d.n_aggs; a++) {
        const DevAgg& ag = plan.aggs[a];
        if ((ag.fn != AG_MEDIAN && ag.fn != AG_PERCENTILE_CONT) || ag.dset != i) continue;
        pk.a[pk.naggs].p = pct_p[a];
        pk.a[pk.naggs].median = ag.fn == AG_MEDIAN ? 1 : 0;
        pk.a[pk.naggs].acc_slot = ag.acc_slot;
        pk.naggs++;
      }
      const uint32_t n = pct_count[i];
      if (verbose) fprintf(stderr, "[pqb] percentile column %u: %u pairs, %u aggregates\n", i, n, pk.naggs);
      if (n == 0) continue;   // every input NULL: the non-NULL counts make every result NULL
      launches += pct_finish(d_pct_slots[i], d_pct_keys[i], n, pk, d_out_slot.p, n_out, d_acc.p, plan.nslots,
                             plan.pct[i].enc == OE_F64, stream, metrics, pct_ms);
    }
    metrics.percentile_ms = pct_ms;
  }
  // ---- ORDER BY [LIMIT]: permute and cut out_slot; after the all-reduce, so every rank orders identical tables ----
  const uint64_t n_total = (d.n_group_by == 0 && n_out == 0) ? 1 : n_out;   // a global aggregate over zero rows is one row
  uint64_t keep = n_total;
  metrics.groups_total = n_total;
  std::unique_ptr<Timer> t_enc, t_sort;   // only for a query with ORDER BY
  bool sort_timed = false;
  std::unique_ptr<OrderBufs> wbufs;
  if (ordered) {
    if (d.limit >= 0) keep = std::min<uint64_t>(keep, uint64_t(d.limit));
    if (win ? n_out > 0 : keep && n_out > 1) {
      OrderArgs oa{};
      uint8_t nulls_first[kMaxOrder];
      oa.acc = d_acc.p;
      oa.wide = plan.hashed ? d_hkeys.p : tuple ? tuple->d_wide : nullptr;
      oa.out_slot = d_out_slot.p;
      oa.n = n_out;
      oa.nslots = plan.nslots;
      oa.n_acc = plan.n_acc;
      oa.nterms = n_part + d.n_order_by;   // a window sorts by its partition terms first
      std::vector<std::shared_ptr<const uint32_t>> rank_hold;   // a concurrent unify_key may replace the column's ranks
      for (uint32_t t = 0; t < oa.nterms; t++) {
        const PqOrderBy& ob = t < n_part ? win->partition_by[t] : d.order_by[t - n_part];
        OrderTerm& ot = oa.t[t];
        ot.target = uint8_t(ob.target);
        ot.desc = (ob.flags & PQ_ORDER_DESC) ? 1 : 0;
        nulls_first[t] = (ob.flags & PQ_ORDER_NULLS_FIRST) ? 1 : 0;
        if (ob.target == PQ_ORDER_AGG) {
          const DevAgg& ag = plan.aggs[ob.index];
          ot.agg = ag;
          ot.nn_is_rows = nn_is_rows[ob.index];
          ot.enc = (ag.fn == AG_AVG || ag.fn == AG_PERCENTILE_CONT ||
                    ((ag.fn == AG_SUM || ag.fn == AG_MIN || ag.fn == AG_MAX || ag.fn == AG_MEDIAN) && ag.kind == DK_F64)) ? OE_F64 : OE_I64;
          continue;
        }
        const DevKey& key = plan.keys[ob.index];
        const uint8_t kind = plan.cols[key.col].kind;
        ot.card = qk[ob.index].card;
        ot.wstride = key.wstride;
        if (qk[ob.index].is_bin || kind == DK_BOOL) { ot.enc = OE_RAW; ot.source = OS_GID; continue; }   // bins ascend with their start
        const ColSide& cs = table->sides[shape_cols[key.col]];
        ot.kd_offs = multi ? cs.d_glob_kd_offs : cs.d_kd_offs;
        ot.kd_bytes = multi ? cs.d_glob_kd_bytes : cs.d_kd_bytes;
        if (kind == DK_STR) {
          ot.enc = OE_RAW;
          ot.source = OS_RANK;
          rank_hold.push_back(table->ensure_kd_rank(shape_cols[key.col], multi, stream));
          ot.rank = rank_hold.back().get();
        } else {
          ot.enc = kind == DK_F64 ? OE_F64 : OE_I64;
          ot.source = OS_VALUE;
        }
      }
      t_enc = std::make_unique<Timer>();
      t_sort = std::make_unique<Timer>();
      if (win) {
        // the window: encode, then sort and count (WindowRun); the kept groups' slots are written once the result
        // block is allocated
        wbufs = std::make_unique<OrderBufs>(oa.nterms, oa.n, stream, metrics);
        oa.vals = wbufs->vals.p;
        oa.nulls = wbufs->nulls.p;
        oa.ranges = wbufs->ranges.p;
        PQB_CUDA(cudaEventRecord(t_enc->a, stream));
        k_order_encode<<<(oa.n + 255) / 256, 256, 0, stream>>>(oa);
        PQB_CUDA(cudaEventRecord(t_enc->b, stream));
        wrun = std::make_unique<WindowRun>(*win, n_out, n_part);
        const unsigned long long kept = wrun->count(*wbufs, nulls_first, d_out_slot.p, stream, metrics);
        launches += 1 + wrun->launches;
        keep = d.limit >= 0 ? std::min<uint64_t>(kept, uint64_t(d.limit)) : kept;
      } else {
        launches += order_groups(oa, nulls_first, uint32_t(keep), d_out_slot, stream, metrics, *t_enc, *t_sort, &sort_timed);
      }
      n_out = uint32_t(keep);
    } else if (win) {   // a global aggregate over zero rows: its one row has rn = 1
      if (!(win->offset == 0 && win->fetch != 0)) keep = 0;
    }
  }
  if (keep == 0) {   // ORDER BY ... LIMIT 0
    metrics.groups = 0;
    PQB_CUDA(cudaEventRecord(t_all.b, stream));
    PQB_CUDA(cudaStreamSynchronize(stream));
  } else if (d.n_group_by == 0 && n_out == 0) {
    // SQL: a global aggregate over zero rows still yields one row: COUNT = 0, everything else NULL
    std::vector<BlockCol> cols;
    std::vector<bool> null;
    for (uint32_t a = 0; a < d.n_aggs; a++) {
      cols.push_back({agg_name(a), agg_out_type[a], agg_kind(a)});
      null.push_back(plan.aggs[a].fn != AG_COUNT_STAR && plan.aggs[a].fn != AG_COUNT && plan.aggs[a].fn != AG_COUNT_DISTINCT);
    }
    one_row(cols, null, 0);
    metrics.groups = 1;
    PQB_CUDA(cudaEventRecord(t_all.b, stream));
    PQB_CUDA(cudaStreamSynchronize(stream));
  } else if (n_out == 0) {
    metrics.groups = 0;
    PQB_CUDA(cudaEventRecord(t_all.b, stream));
    PQB_CUDA(cudaStreamSynchronize(stream));
  } else {
    if (pre.L.rows < n_out) {   // no block yet, or one too small for the groups: lay it out for n_out
      if (pre.L.rows && verbose) fprintf(stderr, "[pqb] result tail: %u groups, the block had room for %u: second copy\n", n_out, uint32_t(pre.L.rows));
      pre = assemble(n_out, nullptr);
      PQB_CUDA(cudaStreamSynchronize(stream));
    }
    keep_device(pre.block, *pre.d_block, pre.L.copy_bytes);
    metrics.groups = n_out;
    slice(pre.L, pre.cols, pre.block, n_out);
  }
  if (t_enc) {   // the ORDER BY kernels: encode, then pack + sort (the range round trip between them is not counted)
    float ms = 0, ms2 = 0;
    cudaEventElapsedTime(&ms, t_enc->a, t_enc->b);
    if (sort_timed) cudaEventElapsedTime(&ms2, t_sort->a, t_sort->b);
    metrics.order_ms = double(ms) + double(ms2) + (wrun ? wrun->ms() : 0.0);
  }
}

// TableProvider::scan(projection): the projected columns of the selected rows, or an ordered scan (merged across ranks
// under PQ_QUERY_ALLGATHER)
void ResultTail::rows() {
  count_selected();
  // ---- TableProvider::scan(projection): gather the projected columns of the selected rows ----
  std::vector<BlockCol> pcs;   // the projected columns, then a window's
  std::vector<uint32_t> slots;
  for (uint32_t i = 0; i < d.n_projection; i++) {
    const uint32_t qc = uint32_t(d.projection[i]);
    // a Date32 column is projected as 4-byte values (DK_I32: the output layout only, read like Int64)
    pcs.push_back({d.columns[qc].name, out_type[qc], out_type[qc] == PQ_T_DATE32 ? uint8_t(DK_I32) : plan.cols[slot_of[qc]].kind});
    slots.push_back(uint32_t(slot_of[qc]));
    if (pcs.back().kind == DK_STR) table->ensure_ent_off(shape_cols[slot_of[qc]], stream);
  }
  // an ordered scan without a projection returns its selected row ordinals in order
  if ((d.flags & PQ_QUERY_EMIT_ROW_IDS) || !d.n_projection) {
    pcs.push_back({"__row_id"});
    slots.push_back(0xffffffffu);
  }
  const uint32_t npc = uint32_t(pcs.size());
  for (const std::string& w : win_names) pcs.push_back({w});
  // the longest string of every projected Utf8 column sizes its bytes (the ranks' merged rows: over every rank)
  std::vector<uint64_t> str_len(npc, 0);
  for (uint32_t c = 0; c < npc; c++)
    if (pcs[c].kind == DK_STR) {
      const ColSide& cs = table->sides[shape_cols[slots[c]]];
      str_len[c] = std::max(cs.max_ent_len, cs.max_plain_len);
    }
  std::unique_ptr<ScanMerge> smerge;   // PQ_QUERY_ALLGATHER with other ranks
  std::shared_ptr<PinnedBlock> block;
  ProjArgs pj{};
  BlockLayout L;
  uint64_t data_lo = 0, data_hi = 0;   // the string bytes of every column: [data_lo, data_hi)
  unsigned long long n_rows = 0;
  DevBuf<uint8_t> d_block;
  // a window's columns (after the projection and __row_id): `win_fill` writes them, and the kept positions, once gather
  // has allocated the block
  std::function<void(long long*, long long*)> win_fill;
  auto lay_out = [&](unsigned long long cap) {
    L = BlockLayout(cap, batch_rows, npc);
    for (uint32_t c = 0; c < npc; c++) {
      ProjCol& pc = pj.cols[c];
      pc = ProjCol{};
      pc.slot = slots[c];
      pc.kind = pcs[c].kind;
      L.column(pcs[c]);
      pc.valid_off = pcs[c].valid_off;
      pc.val_off = pcs[c].val_off;
    }
    data_lo = L.off;
    for (uint32_t c = 0; c < npc; c++) {
      ProjCol& pc = pj.cols[c];
      if (pc.kind != DK_STR) continue;
      pc.ent = table->sides[shape_cols[pc.slot]].d_ent_off;
      const uint64_t bound = cap * str_len[c];
      if (bound > 0x7fffffffull) throw Error(PQ_ERR_UNSUPPORTED, "projected strings of one result exceed 2 GiB: add a LIMIT");
      pc.data_off = pcs[c].data_off = L.take(bound);
    }
    data_hi = L.off;
    for (size_t w = 0; w < win_names.size(); w++) pcs[npc + w].val_off = L.per_row(8);
    L.copy_bytes = L.off;
    for (uint32_t c = 0; c < npc; c++)
      if (pj.cols[c].kind == DK_STR) { pj.cols[c].src_off = L.per_row(8); pj.cols[c].len_off = L.per_row(4); }
  };
  // the first `cap` selected rows, or with `handles` the rows at positions kept[0, cap) (ORDER BY ... LIMIT), or with
  // `owned` the output rows this rank holds of the ranks' merged rows: every byte of the block is then written by one
  // rank and zero on the others, and the ranks' blocks are summed (their u64 words: disjoint bytes never carry).
  // String offsets, which every rank computes alike, are computed after the lengths are summed and never summed.
  auto gather = [&](unsigned long long cap, const unsigned long long* handles, const uint32_t* kept, const unsigned long long* owned) {
    lay_out(cap);
    d_block.alloc(L.off, stream);
    PQB_CUDA(cudaMemsetAsync(d_block.p, 0, L.off, stream));
    pj.arena = table->d_arena;
    pj.flat = table->d_flat;
    pj.fpages = table->d_flat_pages;
    pj.chunks = shape.d_chunks;
    pj.items = shape.d_items;
    pj.bitmap = d_bitmap.p;
    pj.item_counts = d_item_counts.p;
    pj.item_base = d_item_base.p;
    pj.out = d_block.p;
    pj.nulls = reinterpret_cast<uint32_t*>(d_block.p + L.nulls_off);
    pj.n_out = cap;
    pj.n_items = uint32_t(items.size());
    pj.plan_ncols = ncols;
    pj.ncols = npc;
    pj.batch_rows = batch_rows;
    pj.words_per_batch = L.wpb;
    pj.nbatches = L.nbatches;
    if (win_fill) {
      long long* cols[2] = {nullptr, nullptr};
      for (size_t w = 0; w < win_names.size(); w++) cols[win_names[w] == "row_number" ? 0 : 1] = reinterpret_cast<long long*>(d_block.p + pcs[npc + w].val_off);
      win_fill(cols[0], cols[1]);
      launches++;
    }
    if (owned) {
      PQB_CUDA(cudaEventRecord(smerge->t_out.a, stream));
      k_project_owned<<<uint32_t((cap + 255) / 256), 256, 0, stream>>>(pj, owned);
      // everything but the string bytes (summed once they are written); the string offsets are still zero
      comm_allreduce_u64(d_block.p, data_lo / 8, 0 /*sum*/, stream);
      if (L.off > data_hi) comm_allreduce_u64(d_block.p + data_hi, (L.off - data_hi) / 8, 0 /*sum*/, stream);   // the lengths
    } else if (handles) {
      k_project_rows<<<uint32_t((cap + 255) / 256), 256, 0, stream>>>(pj, handles, kept);
    } else {
      const uint32_t grid = std::min<uint32_t>(uint32_t(items.size()), uint32_t(ctx.sm_count() * 8));
      k_project<<<grid, 256, 0, stream>>>(pj);
    }
    launches++;
    for (uint32_t c = 0; c < npc; c++) {
      if (pj.cols[c].kind != DK_STR) continue;
      // rows beyond the selected total have length 0: the scan over `cap` rows is exact
      k_offsets_scan<<<1, 1024, 0, stream>>>(reinterpret_cast<const uint32_t*>(d_block.p + pj.cols[c].len_off), uint32_t(cap), nullptr,
                                             reinterpret_cast<int32_t*>(d_block.p + pj.cols[c].val_off));
      k_project_bytes<<<uint32_t((cap * 32 + 255) / 256), 256, 0, stream>>>(pj, c, cap, owned);
      launches += 2;
    }
    if (owned) {
      if (data_hi > data_lo) comm_allreduce_u64(d_block.p + data_lo, (data_hi - data_lo) / 8, 0 /*sum*/, stream);
      PQB_CUDA(cudaEventRecord(smerge->t_out.b, stream));
      smerge->out_timed = true;
    }
    PQB_CUDA(cudaGetLastError());
    block = std::make_shared<PinnedBlock>();
    block->p = ctx.pinned_acquire(L.copy_bytes);
    block->bytes = L.copy_bytes;
    PQB_CUDA(cudaMemcpyAsync(block->p, d_block.p, L.copy_bytes, cudaMemcpyDeviceToHost, stream));
  };
  if (row_order && (!items.empty() || merge_rows)) {
    // ---- ORDER BY ... LIMIT: every selected row's terms and handle (k_order_rows_encode), the positions of the first
    // `keep` rows in order (order_sort), then their projection.  Under PQ_QUERY_ALLGATHER with other ranks, those
    // first rows of every rank are merged (ScanMerge) and each rank projects the merged rows it holds; without the
    // flag every shard orders and cuts its own selection.
    PQB_CUDA(cudaStreamSynchronize(stream));   // the selected-row total sizes the sort
    unsigned long long keep = std::min(total, lim);   // a window: the kept rows, known after its sort
    if (merge_rows) {   // the checks below, agreed by every rank
      uint64_t row_end = 0, row_bytes = 0;
      for (const DevItem& it : items) row_end = std::max<uint64_t>(row_end, it.global_row0 + it.nrows);
      for (uint32_t c = 0; c < npc; c++) row_bytes += 1 + (pcs[c].kind == DK_STR ? 16 : pcs[c].kind == DK_BOOL ? 1 : 8);   // validity, values / offsets and scratch
      smerge = std::make_unique<ScanMerge>();
      smerge->exchange(roa.nterms, keep, total, h_counters[1], row_end, str_len, lim, row_bytes, stream, metrics);
      str_len = smerge->str_len;
    } else {
      check_corrupt();
      if (total > 0xffffffffull) throw Error(PQ_ERR_UNSUPPORTED, "row-level ORDER BY over more than 2^32 - 1 selected rows");
      if (!win && keep > 0x7ffffff0ull) throw Error(PQ_ERR_UNSUPPORTED, "more than 2^31 projected rows in one result: add a LIMIT");
    }
    const uint32_t n = uint32_t(total);
    std::unique_ptr<OrderBufs> obuf;   // (the merge reads this rank's encoded rows)
    DevBuf<unsigned long long> handles;
    DevBuf<uint32_t> kept;
    if (win ? total > 0 : keep > 0) {
      obuf = std::make_unique<OrderBufs>(roa.nterms, n, stream, metrics);
      OrderBufs& ob = *obuf;
      handles.alloc(n, stream);
      roa.arena = table->d_arena;
      roa.flat = table->d_flat;
      roa.fpages = d_opages.p ? d_opages.p : table->d_flat_pages;
      roa.chunks = shape.d_chunks;
      roa.items = shape.d_items;
      roa.bitmap = d_bitmap.p;
      roa.item_counts = d_item_counts.p;
      roa.item_base = d_item_base.p;
      roa.n_items = uint32_t(items.size());
      roa.plan_ncols = ncols;
      roa.n = n;
      roa.vals = ob.vals.p;
      roa.nulls = ob.nulls.p;
      roa.ranges = ob.ranges.p;
      roa.handles = handles.p;
      uint32_t grid = std::min<uint32_t>(uint32_t(items.size()), uint32_t(ctx.sm_count() * 8));
      if (const char* g = getenv("PQB_GRID")) grid = std::max(1, atoi(g));   // debugging aid: several items per CTA
      Timer t_enc, t_sort;
      bool sort_timed = false;
      PQB_CUDA(cudaEventRecord(t_enc.a, stream));
      k_order_rows_encode<<<grid, 256, 0, stream>>>(roa);
      PQB_CUDA(cudaEventRecord(t_enc.b, stream));
      std::unique_ptr<WindowRun> wrun;
      if (win) {
        // the window: sort and count, then the kept positions and the extra columns in gather's block
        wrun = std::make_unique<WindowRun>(*win, n, n_part);
        keep = std::min(wrun->count(ob, row_nulls_first, nullptr, stream, metrics), lim);
        launches += 1 + wrun->launches;
        if (keep > 0x7ffffff0ull) throw Error(PQ_ERR_UNSUPPORTED, "more than 2^31 projected rows in one result: add a LIMIT");
        if (keep) {
          kept.alloc(keep, stream);
          win_fill = [&](long long* rn, long long* prows) { wrun->fill(nullptr, keep, kept.p, rn, prows, stream); };
          gather(keep, handles.p, kept.p, nullptr);
        }
      } else {
        launches += 1 + order_sort(ob, roa.nterms, n, row_nulls_first, uint32_t(keep), nullptr, kept, stream, metrics, t_sort, &sort_timed);
        if (!smerge) gather(keep, handles.p, kept.p, nullptr);
      }
      PQB_CUDA(cudaStreamSynchronize(stream));
      if (keep && !smerge) metrics.d2h_bytes += L.copy_bytes;
      float ms = 0, ms2 = 0;
      cudaEventElapsedTime(&ms, t_enc.a, t_enc.b);
      if (sort_timed) cudaEventElapsedTime(&ms2, t_sort.a, t_sort.b);
      metrics.order_ms = double(ms) + double(ms2) + (wrun ? wrun->ms() : 0.0);
    }
    shape.last_total.store(total);
    if (smerge) {
      // every rank's first rows: the same candidates and the same order on every rank, each output row projected by
      // the rank that holds it and the ranks' blocks summed
      DevBuf<unsigned long long> owned;
      launches += smerge->merge(obuf ? obuf->vals.p : nullptr, obuf ? obuf->nulls.p : nullptr, n, kept.p, handles.p, shape.d_items,
                                row_nulls_first, owned, stream, metrics);
      keep = smerge->keep;
      if (keep) {
        gather(keep, nullptr, nullptr, owned.p);
        metrics.d2h_bytes += L.copy_bytes;
      }
      PQB_CUDA(cudaStreamSynchronize(stream));
      smerge->report(verbose, metrics);
      total = smerge->total;
    }
    n_rows = keep;
  } else if (!items.empty()) {
    n_rows = sized_pass(1, block, [&](unsigned long long cap) {
      if (cap > 0x7ffffff0ull) throw Error(PQ_ERR_UNSUPPORTED, "more than 2^31 projected rows in one result: add a LIMIT");
      gather(cap, nullptr, nullptr, nullptr);
      return L.copy_bytes;
    }, nullptr);
  }
  PQB_CUDA(cudaEventRecord(t_all.b, stream));
  PQB_CUDA(cudaStreamSynchronize(stream));
  check_corrupt();
  keep_device(block, d_block, L.copy_bytes);
  metrics.rows_selected = total;
  if (!n_rows) {   // one empty batch, in a heap block
    lay_out(0);
    block = heap_block(L.off);
  }
  slice(L, pcs, block, n_rows);
}

// selected row ordinals, ascending, or the one row of SELECT COUNT(*) [, COUNT(*)...] WHERE ...
void ResultTail::selection() {
  count_selected();
  std::shared_ptr<PinnedBlock> ids_block;   // selected row ordinals land in page-locked memory, batches alias it
  unsigned long long n_ids = 0;
  DevBuf<unsigned long long> d_ids;
  if (want_rows && !items.empty()) {
    n_ids = sized_pass(0, ids_block, [&](unsigned long long cap) -> uint64_t {
      if (!cap) return 0;
      d_ids.alloc(cap, stream);
      const uint32_t grid = std::min<uint32_t>(uint32_t(items.size()), uint32_t(ctx.sm_count() * 8));
      k_compact_row_ids<<<grid, 256, 0, stream>>>(d_bitmap.p, shape.d_items, d_item_counts.p, d_item_base.p, uint32_t(items.size()), d_ids.p, cap);
      launches++;
      ids_block = std::make_shared<PinnedBlock>();
      ids_block->p = ctx.pinned_acquire(cap * 8);
      ids_block->bytes = cap * 8;
      PQB_CUDA(cudaMemcpyAsync(ids_block->p, d_ids.p, cap * 8, cudaMemcpyDeviceToHost, stream));
      return cap * 8;
    }, "scan done, selected-row total on host");
  }
  PQB_CUDA(cudaEventRecord(t_all.b, stream));
  PQB_CUDA(cudaStreamSynchronize(stream));
  mark("results on host");
  metrics.rows_selected = total;
  unsigned long long corrupt_ranks = 0;
  if (d.n_aggs && allreduce) {
    // SELECT COUNT(*) under PQ_QUERY_ALLREDUCE: the total's all-reduce also counts the ranks that met a corrupt page,
    // so that every rank throws, not only the ones that met it
    const unsigned long long bad = h_counters[1] ? 1ull : 0ull;
    PQB_CUDA(cudaMemcpyAsync(d_total.p + 1, &bad, 8, cudaMemcpyHostToDevice, stream));
    comm_allreduce_u64(d_total.p, 2, 0, stream);
    unsigned long long w[2];
    PQB_CUDA(cudaMemcpyAsync(w, d_total.p, 16, cudaMemcpyDeviceToHost, stream));
    PQB_CUDA(cudaStreamSynchronize(stream));
    total = w[0];
    corrupt_ranks = w[1];
  }
  check_corrupt();
  if (corrupt_ranks) throw Error(PQ_ERR_CORRUPT, "corrupt or unsupported page encoding met on the device of " + std::to_string(corrupt_ranks) + " other rank(s)");
  if (d.n_aggs) {
    metrics.groups_total = 1;
    // one row, ordered trivially; LIMIT 0 keeps none, and a window keeps it when its rank range holds rn = 1
    const bool win_drops = win && !(win->offset == 0 && win->fetch != 0);
    if ((ordered && d.limit == 0) || win_drops) {
      metrics.groups = 0;
    } else {
      one_row(std::vector<BlockCol>(d.n_aggs, BlockCol{"count(*)"}), std::vector<bool>(d.n_aggs, false), total);
      metrics.groups = 1;
    }
  } else if (want_rows) {
    if (!n_ids) ids_block = heap_block(0);   // one empty batch
    slice(BlockLayout(n_ids, batch_rows, 0), {BlockCol{"__row_id"}}, ids_block, n_ids);   // 8-byte ids, no NULL counts
  }
}

void ResultTail::finish() {
  float ms = 0;
  cudaEventElapsedTime(&ms, t_all.a, t_all.b);
  metrics.device_ms = ms;
  if (!items.empty() && nrg) { cudaEventElapsedTime(&ms, t_scan.a, t_scan.b); metrics.scan_kernel_ms = ms; }
  metrics.kernel_launches = launches;
}

void Query::schema(ArrowSchema* out) const {
  if (!batches_.empty()) { export_batch(batches_[0], nullptr, out); return; }
  OutBatch none;
  export_batch(none, nullptr, out);
}

// JSON egress (json_egress.cuh): all batches of the result, formatted on the device.
void Query::json(uint32_t flags, const char** out, uint64_t* len) {
  Context& ctx = Context::get();
  cudaStream_t stream = cudaStreamPerThread;
  const bool lines = (flags & PQ_JSON_LINES) != 0;
  unsigned long long n = 0;
  for (const OutBatch& b : batches_) n += uint64_t(b.rows);
  json_block_.reset();
  auto finish_empty = [&]() {
    json_block_ = std::make_shared<PinnedBlock>();
    json_block_->p = ctx.pinned_acquire(16);
    json_block_->bytes = lines ? 0 : 2;
    if (!lines) { json_block_->p[0] = '['; json_block_->p[1] = ']'; }
    *out = reinterpret_cast<const char*>(json_block_->p);
    *len = json_block_->bytes;
  };
  if (n == 0 || batches_.empty() || batches_[0].cols.empty()) { finish_empty(); return; }
  const OutBatch* first = nullptr;
  for (const OutBatch& b : batches_) if (b.rows) { first = &b; break; }
  const size_t ncols = first->cols.size();
  if (ncols > size_t(kJsonMaxCols)) throw Error(PQ_ERR_UNSUPPORTED, "JSON egress: more than 64 result columns");
  JsonArgs ja{};
  ja.ncols = uint32_t(ncols);
  ja.n_rows = n;
  ja.lines = lines ? 1u : 0u;
  ja.batch_rows = batch_rows_;
  ja.words_per_batch = (batch_rows_ + 31) / 32;
  // every column of the result is a slice of one block: its kept device copy, the mapped page-locked copy, or (a heap
  // block, one row) a copy uploaded here
  const PinnedBlock& blk = *first->cols[0].block;
  DevBuf<uint64_t> up;
  if (!blk.dev && !blk.heap.empty()) up.upload(blk.heap, stream);
  const uint8_t* base = blk.dev ? blk.dev : up.p ? reinterpret_cast<const uint8_t*>(up.p) : blk.p;
  std::vector<uint8_t> keys;
  for (size_t c = 0; c < ncols; c++) {
    const OutColumn& oc = first->cols[c];
    JsonCol& jc = ja.cols[c];
    jc.type = oc.type == PQ_T_F64 ? JT_F64 : oc.type == PQ_T_BOOL ? JT_BOOL : oc.type == PQ_T_UTF8 ? JT_UTF8 : oc.type == PQ_T_TS_MS ? JT_TS_MS
            : oc.type == PQ_T_DATE32 ? JT_DATE32 : JT_I64;
    // "name": with the name escaped like any string
    jc.key_off = uint32_t(keys.size());
    keys.push_back('"');
    { std::vector<char> e(oc.name.size() * 6 + 1);
      const uint32_t k = jf_escape(reinterpret_cast<const uint8_t*>(oc.name.data()), uint32_t(oc.name.size()), e.data());
      keys.insert(keys.end(), e.begin(), e.begin() + k); }
    keys.push_back('"'); keys.push_back(':');
    jc.key_len = uint32_t(keys.size()) - jc.key_off;
    bool any_nulls = false;
    for (const OutBatch& b : batches_) if (b.rows) any_nulls = any_nulls || b.cols[c].null_count != 0;
    jc.values = base + oc.values_off;   // values and offsets contiguous over all batches, bit-packed buffers per batch
    jc.validity = any_nulls ? reinterpret_cast<const uint32_t*>(base + oc.validity_off) : nullptr;
    jc.offsets = oc.type == PQ_T_UTF8 ? reinterpret_cast<const int32_t*>(base + oc.offsets_off) : nullptr;
  }
  DevBuf<uint8_t> d_keys; d_keys.upload(keys, stream);
  ja.keys = d_keys.p;
  DevBuf<uint32_t> d_lens; d_lens.alloc(n, stream);
  DevBuf<long long> d_offs; d_offs.alloc(n + 1, stream);
  const uint32_t grid = uint32_t((n + 255) / 256);
  k_json_sizes<<<grid, 256, 0, stream>>>(ja, d_lens.p);
  k_json_scan<<<1, 1024, 0, stream>>>(d_lens.p, n, d_offs.p, lines ? 0 : 1);
  long long total = 0;
  PQB_CUDA(cudaMemcpyAsync(&total, d_offs.p + n, 8, cudaMemcpyDeviceToHost, stream));
  PQB_CUDA(cudaStreamSynchronize(stream));
  DevBuf<char> d_out; d_out.alloc(size_t(total) + 16, stream);
  k_json_write<<<grid, 256, 0, stream>>>(ja, d_offs.p, d_out.p);
  PQB_CUDA(cudaGetLastError());
  json_block_ = std::make_shared<PinnedBlock>();
  json_block_->p = ctx.pinned_acquire(size_t(total) + 16);
  json_block_->bytes = size_t(total);
  PQB_CUDA(cudaMemcpyAsync(json_block_->p, d_out.p, size_t(total), cudaMemcpyDeviceToHost, stream));
  PQB_CUDA(cudaStreamSynchronize(stream));
  if (!lines) { json_block_->p[0] = '['; json_block_->p[total - 1] = ']'; }   // the last row's ',' closes the array
  metrics.d2h_bytes += uint64_t(total);
  metrics.kernel_launches += 3;
  *out = reinterpret_cast<const char*>(json_block_->p);
  *len = uint64_t(total);
}

int Query::next(int partition, ArrowArray* out, ArrowSchema* schema) {
  (void)partition;
  if (next_batch_ >= batches_.size()) return PQ_END_OF_STREAM;
  export_batch(batches_[next_batch_++], out, schema);
  return PQ_OK;
}

}  // namespace pqb
