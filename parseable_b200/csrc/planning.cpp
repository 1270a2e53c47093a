// Scan planning on the C side: the decisions StandardTableProvider::scan takes between the snapshot and
// create_parquet_physical_plan, so that a shim can hand the manifest to the library instead of a file list.
// Host code only.  Mirrors (paths relative to /root/reference):
//   extract_timestamp_bound / PartialTimeFilter   src/query/stream_schema_provider.rs:884-940, 698-748
//   Snapshot::manifests                           src/catalog/snapshot.rs:40-71
//   is_overlapping_query / is_within_staging_window   src/query/stream_schema_provider.rs:750-775, 842-864
//   ManifestExt::can_be_pruned / satisfy_constraints  :955-1043
//   collect_from_snapshot                         :449-510
//   TypedStatistics::update                       src/catalog/column.rs:70-140
//   supports_filters_pushdown / expr_in_boundary  src/query/stream_schema_provider.rs:665-683, 866-882
// Semantics are pinned by the reference's unit-test vectors (tests/test_planning.py runs them through this file
// and through the Python mirror).
#include <cmath>
#include <cstring>
#include <string>
#include <vector>

#include "engine.hpp"

namespace {

constexpr int64_t kNsPerSec = 1000000000ll, kNsPerMin = 60 * kNsPerSec;

int64_t days_from_civil(int64_t y, unsigned m, unsigned d) {
  y -= m <= 2;
  const int64_t era = (y >= 0 ? y : y - 399) / 400;
  const unsigned yoe = unsigned(y - era * 400);
  const unsigned doy = (153 * (m + (m > 2 ? -3 : 9)) + 2) / 5 + d - 1;
  const unsigned doe = yoe * 365 + yoe / 4 - yoe / 100 + doy;
  return era * 146097 + int64_t(doe) - 719468;
}
// "YYYY-MM-DDTHH:MM:SS[.f{1,9}]" (chrono's NaiveDateTime::from_str; a space separator is accepted as well)
bool parse_naive_datetime(const char* s, uint64_t n, int64_t& ns) {
  auto num = [&](uint64_t at, int len, int& v) {
    v = 0;
    if (at + uint64_t(len) > n) return false;
    for (int i = 0; i < len; i++) {
      const char c = s[at + i];
      if (c < '0' || c > '9') return false;
      v = v * 10 + (c - '0');
    }
    return true;
  };
  int Y, M, D, h, m, sec;
  if (!num(0, 4, Y) || n < 19 || s[4] != '-' || !num(5, 2, M) || s[7] != '-' || !num(8, 2, D)) return false;
  if (s[10] != 'T' && s[10] != ' ') return false;
  if (!num(11, 2, h) || s[13] != ':' || !num(14, 2, m) || s[16] != ':' || !num(17, 2, sec)) return false;
  if (M < 1 || M > 12 || D < 1 || D > 31 || h > 23 || m > 59 || sec > 60) return false;
  int64_t frac = 0;
  if (n > 19) {
    if (s[19] != '.' || n == 20 || n > 29) return false;
    int64_t scale = kNsPerSec;
    for (uint64_t i = 20; i < n; i++) {
      if (s[i] < '0' || s[i] > '9') return false;
      scale /= 10;
      frac += int64_t(s[i] - '0') * scale;
    }
  }
  ns = ((days_from_civil(Y, unsigned(M), unsigned(D)) * 24 + h) * 60 + m) * 60 * kNsPerSec + int64_t(sec) * kNsPerSec + frac;
  return true;
}

// (cmp, time) of `column <cmp> timestamp literal`
bool timestamp_bound(const PqPlanFilter& f, const char* time_partition, int32_t& cmp, int64_t& ns) {
  if (!f.column) return false;
  cmp = f.cmp;
  if (f.lit.type == PQ_T_TS_MS) { ns = f.lit.i64 * 1000000ll; return true; }
  if (f.lit.type == PQ_T_TS_NS) { ns = f.lit.i64; return true; }
  if (f.lit.type == PQ_T_UTF8 && time_partition && std::strcmp(f.column, time_partition) == 0)
    return parse_naive_datetime(f.lit.str, f.lit.str_len, ns);
  return false;
}

int cmp_str(const char* a, uint64_t an, const char* b, uint64_t bn) {
  const int c = std::memcmp(a, b, size_t(an < bn ? an : bn));
  if (c) return c;
  return an < bn ? -1 : (an > bn ? 1 : 0);
}

// can a file whose column spans the statistics hold a row with `column <cmp> literal`?  1 yes, 0 no, -1 cannot tell
int satisfy(const PqLiteral& lit, int32_t cmp, const PqColumnStat& st) {
  // three-way comparisons of the literal against min and max
  int vs_min, vs_max;
  switch (lit.type) {
    case PQ_T_BOOL:
      if (st.kind != PQ_STAT_BOOL) return -1;
      vs_min = (lit.i64 != 0) - (st.min_i != 0); vs_max = (lit.i64 != 0) - (st.max_i != 0);
      break;
    case PQ_T_I64: case PQ_T_TS_MS: case PQ_T_DATE32:   // TimestampMillisecond and Date32 cast to Int (stream_schema_provider.rs:1002-1015)
      if (st.kind != PQ_STAT_INT) return -1;
      vs_min = lit.i64 < st.min_i ? -1 : (lit.i64 > st.min_i ? 1 : 0);
      vs_max = lit.i64 < st.max_i ? -1 : (lit.i64 > st.max_i ? 1 : 0);
      break;
    case PQ_T_F64:
      if (st.kind != PQ_STAT_FLOAT) return -1;
      // Rust's PartialOrd on f64: every comparison with NaN is false
      if (std::isnan(lit.f64) || std::isnan(st.min_f) || std::isnan(st.max_f)) {
        // value >= min && value <= max etc. are all false -> "cannot hold" for every operator the reference answers
        return (cmp == PQ_EQ || cmp == PQ_LT || cmp == PQ_LE || cmp == PQ_GT || cmp == PQ_GE) ? 0 : -1;
      }
      vs_min = lit.f64 < st.min_f ? -1 : (lit.f64 > st.min_f ? 1 : 0);
      vs_max = lit.f64 < st.max_f ? -1 : (lit.f64 > st.max_f ? 1 : 0);
      break;
    case PQ_T_UTF8:
      if (st.kind != PQ_STAT_STRING) return -1;
      vs_min = cmp_str(lit.str, lit.str_len, st.min_s, st.min_s_len);
      vs_max = cmp_str(lit.str, lit.str_len, st.max_s, st.max_s_len);
      break;
    default: return -1;
  }
  switch (cmp) {
    case PQ_EQ: return vs_min >= 0 && vs_max <= 0;
    case PQ_LT: return vs_min > 0;     // value > min
    case PQ_LE: return vs_min >= 0;
    case PQ_GT: return vs_max < 0;     // value < max
    case PQ_GE: return vs_max <= 0;
    default: return -1;                // != never prunes
  }
}

bool can_be_pruned(const PqManifestFile& f, const PqPlanFilter& flt) {
  if (!flt.column) return false;
  for (uint32_t i = 0; i < f.n_stats; i++) {
    const PqColumnStat& st = f.stats[i];
    if (!st.column || std::strcmp(st.column, flt.column) != 0) continue;
    if (st.kind == PQ_STAT_NONE) return false;
    return satisfy(flt.lit, flt.cmp, st) == 0;
  }
  return false;
}

}  // namespace

extern "C" {

int32_t pq_plan_time_bounds(const PqPlanFilter* filters, uint32_t n, const char* time_partition, PqTimeBound* out) {
  if ((n && !filters) || !out) return PQ_ERR_INVALID_ARG;
  int32_t k = 0;
  for (uint32_t i = 0; i < n; i++) {
    int32_t cmp;
    int64_t ns;
    if (!timestamp_bound(filters[i], time_partition, cmp, ns)) continue;
    PqTimeBound b{};
    b.time_ns = ns;
    switch (cmp) {
      case PQ_GT: b.kind = PQ_BOUND_LOW; b.included = 0; break;
      case PQ_GE: b.kind = PQ_BOUND_LOW; b.included = 1; break;
      case PQ_LT: b.kind = PQ_BOUND_HIGH; b.included = 0; break;
      case PQ_LE: b.kind = PQ_BOUND_HIGH; b.included = 1; break;
      case PQ_EQ: b.kind = PQ_BOUND_EQ; b.included = 1; break;
      default: continue;
    }
    out[k++] = b;
  }
  return k;
}

int32_t pq_plan_manifests(const PqManifestItem* items, uint32_t n, const PqTimeBound* bounds, uint32_t n_bounds, uint8_t* keep) {
  if ((n && (!items || !keep)) || (n_bounds && !bounds)) return PQ_ERR_INVALID_ARG;
  for (uint32_t i = 0; i < n; i++) {
    bool k = true;
    for (uint32_t b = 0; b < n_bounds && k; b++) {
      const PqTimeBound& t = bounds[b];
      if (t.kind == PQ_BOUND_LOW) k = t.included ? items[i].time_upper_ns >= t.time_ns : items[i].time_upper_ns > t.time_ns;
      else if (t.kind == PQ_BOUND_HIGH) k = t.included ? items[i].time_lower_ns <= t.time_ns : items[i].time_lower_ns < t.time_ns;
      else k = items[i].time_lower_ns <= t.time_ns && t.time_ns <= items[i].time_upper_ns;
    }
    keep[i] = k ? 1 : 0;
  }
  return PQ_OK;
}

int32_t pq_plan_is_overlapping_query(const PqManifestItem* items, uint32_t n, const PqTimeBound* bounds, uint32_t n_bounds) {
  if ((n && !items) || (n_bounds && !bounds)) return PQ_ERR_INVALID_ARG;
  if (!n) return 1;
  int64_t first = items[0].time_lower_ns;
  for (uint32_t i = 1; i < n; i++) first = items[i].time_lower_ns < first ? items[i].time_lower_ns : first;
  for (uint32_t b = 0; b < n_bounds; b++)
    if (bounds[b].kind == PQ_BOUND_LOW && bounds[b].time_ns < first) return 1;
  return 0;
}

int32_t pq_plan_within_staging_window(const PqTimeBound* bounds, uint32_t n_bounds, int64_t now_ns) {
  if (n_bounds && !bounds) return PQ_ERR_INVALID_ARG;
  int64_t back = now_ns - 5 * kNsPerMin;
  back -= ((back % kNsPerMin) + kNsPerMin) % kNsPerMin;   // start of that minute
  bool has_high = false;
  for (uint32_t b = 0; b < n_bounds; b++) {
    if ((bounds[b].kind == PQ_BOUND_HIGH || bounds[b].kind == PQ_BOUND_EQ) && bounds[b].time_ns >= back) return 1;
    has_high = has_high || bounds[b].kind == PQ_BOUND_HIGH;
  }
  return has_high ? 0 : 1;
}

int64_t pq_plan_collect_files(const PqManifestFile* files, uint32_t n_files, const PqPlanFilter* filters, uint32_t n_filters,
                              int64_t limit, uint32_t* out_index) {
  if ((n_files && (!files || !out_index)) || (n_filters && !filters)) return PQ_ERR_INVALID_ARG;
  int64_t k = 0;
  uint64_t rows = 0;
  for (uint32_t r = 0; r < n_files; r++) {
    const uint32_t i = n_files - 1 - r;   // newest first
    bool pruned = false;
    for (uint32_t f = 0; f < n_filters && !pruned; f++) pruned = can_be_pruned(files[i], filters[f]);
    if (pruned) continue;
    out_index[k++] = i;
    rows += files[i].num_rows;
    if (limit >= 0 && rows >= uint64_t(limit)) break;
  }
  return k;
}

int32_t pq_plan_merge_stat(const PqColumnStat* a, const PqColumnStat* b, PqColumnStat* out) {
  if (!a || !b || !out) return PQ_ERR_INVALID_ARG;
  if (a->kind != b->kind || a->kind == PQ_STAT_NONE) return 0;
  PqColumnStat m = *a;
  switch (a->kind) {
    case PQ_STAT_BOOL: case PQ_STAT_INT:
      m.min_i = a->min_i < b->min_i ? a->min_i : b->min_i;
      m.max_i = a->max_i > b->max_i ? a->max_i : b->max_i;
      break;
    case PQ_STAT_FLOAT: {
      auto ok = [](double lo, double hi) { return !(std::isnan(lo) || std::isnan(hi)) && lo <= hi; };
      if (!ok(a->min_f, a->max_f) || !ok(b->min_f, b->max_f)) return 0;
      m.min_f = a->min_f < b->min_f ? a->min_f : b->min_f;
      m.max_f = a->max_f > b->max_f ? a->max_f : b->max_f;
      break;
    }
    case PQ_STAT_STRING:
      if (cmp_str(b->min_s, b->min_s_len, a->min_s, a->min_s_len) < 0) { m.min_s = b->min_s; m.min_s_len = b->min_s_len; }
      if (cmp_str(b->max_s, b->max_s_len, a->max_s, a->max_s_len) > 0) { m.max_s = b->max_s; m.max_s_len = b->max_s_len; }
      break;
    default: return 0;
  }
  *out = m;
  return 1;
}

int32_t pq_plan_pushdown(const PqPlanFilter* filters, uint32_t n, uint8_t* exact) {
  if (n && (!filters || !exact)) return PQ_ERR_INVALID_ARG;
  for (uint32_t i = 0; i < n; i++) {
    int32_t cmp;
    int64_t ns;
    exact[i] = 0;
    if (!timestamp_bound(filters[i], nullptr, cmp, ns)) continue;
    const bool aligned = ((ns % kNsPerMin) + kNsPerMin) % kNsPerMin == 0;
    if (aligned && (cmp == PQ_GT || cmp == PQ_GE || cmp == PQ_LT || cmp == PQ_LE)) exact[i] = 1;
  }
  return PQ_OK;
}

}  // extern "C"
