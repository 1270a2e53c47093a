// Result egress as JSON text, formatted on the device: what the reference does on the CPU after the query
// (/root/reference/src/utils/arrow/mod.rs:49-64 record_batches_to_json -> arrow_json::ArrayWriter, then
// /root/reference/src/response.rs:31-58 QueryResponse::to_json; SURVEY §8 rows a14 / N4).  One thread per result row:
// pass 1 sizes the row's object, a scan places it, pass 2 writes it.  Conventions of arrow-json / serde_json:
//   * a NULL value leaves its key out of the object (explicit_nulls = false)
//   * Int64 as decimal, Float64 shortest round-trip (ryu_f64.cuh), non-finite floats as null, booleans true / false
//   * Timestamp(ms) as "YYYY-MM-DDTHH:MM:SS[.mmm]" (chrono's NaiveDateTime, fraction only when non-zero)
//   * strings escaped like serde_json: \" \\ \n \r \t \b \f, other control bytes \u00XX, UTF-8 passed through
// The columns are read where the result already is: the device block the result was assembled in (kept with the query)
// or the page-locked host block (mapped: zero copy).
#pragma once
#if defined(__CUDACC__)
#include <cuda_runtime.h>
#endif

#include <cstdint>

#include "ryu_f64.cuh"

namespace pqb {

#if defined(__CUDACC__)
#define PQB_JF __host__ __device__ inline
#else
#define PQB_JF inline
#endif

PQB_JF uint32_t jf_i64(int64_t v, char* out) {
  char tmp[20];
  uint64_t u = v < 0 ? uint64_t(0) - uint64_t(v) : uint64_t(v);
  uint32_t k = 0, n = 0;
  do { tmp[k++] = char('0' + u % 10); u /= 10; } while (u);
  if (v < 0) out[n++] = '-';
  while (k) out[n++] = tmp[--k];
  return n;
}
// days since 1970-01-01 -> civil date (proleptic Gregorian)
PQB_JF void jf_civil(int64_t z, int64_t& y, uint32_t& m, uint32_t& d) {
  z += 719468;
  const int64_t era = (z >= 0 ? z : z - 146096) / 146097;
  const uint32_t doe = uint32_t(z - era * 146097);
  const uint32_t yoe = (doe - doe / 1460 + doe / 36524 - doe / 146096) / 365;
  y = int64_t(yoe) + era * 400;
  const uint32_t doy = doe - (365 * yoe + yoe / 4 - yoe / 100);
  const uint32_t mp = (5 * doy + 2) / 153;
  d = doy - (153 * mp + 2) / 5 + 1;
  m = mp < 10 ? mp + 3 : mp - 9;
  y += m <= 2;
}
// Date32 (days since 1970-01-01) without the quotes: YYYY-MM-DD, a '-' before negative years and a '+' before years above
// 9999 (chrono prints years beyond 9999 with a sign); at most 20 bytes
PQB_JF uint32_t jf_date32(int64_t days, char* out) {
  int64_t y; uint32_t mo, d;
  jf_civil(days, y, mo, d);
  uint32_t n = 0;
  if (y < 0) { out[n++] = '-'; y = -y; }
  if (y > 9999) { out[n++] = '+'; n += jf_i64(y, out + n); }
  else { out[n++] = char('0' + y / 1000); out[n++] = char('0' + y / 100 % 10); out[n++] = char('0' + y / 10 % 10); out[n++] = char('0' + y % 10); }
  auto two = [&](uint32_t v) { out[n++] = char('0' + v / 10); out[n++] = char('0' + v % 10); };
  out[n++] = '-'; two(mo); out[n++] = '-'; two(d);
  return n;
}
// Timestamp(Millisecond, None) without the quotes: the date of jf_date32, 'T', the time; at most 32 bytes
PQB_JF uint32_t jf_ts_ms(int64_t ms, char* out) {
  int64_t days = ms / 86400000, rem = ms % 86400000;
  if (rem < 0) { rem += 86400000; days -= 1; }
  uint32_t n = jf_date32(days, out);
  auto two = [&](uint32_t v) { out[n++] = char('0' + v / 10); out[n++] = char('0' + v % 10); };
  out[n++] = 'T';
  const uint32_t msod = uint32_t(rem), s = msod / 1000, f = msod % 1000;
  two(s / 3600); out[n++] = ':'; two(s / 60 % 60); out[n++] = ':'; two(s % 60);
  if (f) { out[n++] = '.'; out[n++] = char('0' + f / 100); out[n++] = char('0' + f / 10 % 10); out[n++] = char('0' + f % 10); }
  return n;
}
PQB_JF uint32_t jf_escaped_len(const uint8_t* s, uint32_t len) {
  uint32_t n = 0;
  for (uint32_t i = 0; i < len; i++) {
    const uint8_t c = s[i];
    if (c == '"' || c == '\\' || c == '\n' || c == '\r' || c == '\t' || c == 8 || c == 12) n += 2;
    else if (c < 0x20) n += 6;
    else n += 1;
  }
  return n;
}
PQB_JF uint32_t jf_escape(const uint8_t* s, uint32_t len, char* out) {
  uint32_t n = 0;
  for (uint32_t i = 0; i < len; i++) {
    const uint8_t c = s[i];
    char e = 0;
    switch (c) {
      case '"': e = '"'; break;
      case '\\': e = '\\'; break;
      case '\n': e = 'n'; break;
      case '\r': e = 'r'; break;
      case '\t': e = 't'; break;
      case 8: e = 'b'; break;
      case 12: e = 'f'; break;
      default: break;
    }
    if (e) { out[n++] = '\\'; out[n++] = e; }
    else if (c < 0x20) {
      const char* hex = "0123456789abcdef";
      out[n++] = '\\'; out[n++] = 'u'; out[n++] = '0'; out[n++] = '0'; out[n++] = hex[c >> 4]; out[n++] = hex[c & 15];
    } else out[n++] = char(c);
  }
  return n;
}

constexpr int kJsonMaxCols = 64;
enum JsonType : uint32_t { JT_I64 = 0, JT_F64 = 1, JT_BOOL = 2, JT_UTF8 = 3, JT_TS_MS = 4, JT_U64 = 5, JT_DATE32 = 6 };
struct JsonCol {
  const uint8_t* values;     // 8-byte values | 4-byte values (Date32) | bit-packed booleans (words per batch) | string bytes
  const uint32_t* validity;  // bit-packed, words per batch; nullptr: no NULLs
  const int32_t* offsets;    // strings: n_rows + 1 offsets into `values`
  uint32_t type;             // JsonType
  uint32_t key_off, key_len; // `"name":` (escaped) inside JsonArgs.keys
  uint32_t _pad;
};
struct JsonArgs {
  JsonCol cols[kJsonMaxCols];
  const uint8_t* keys;
  uint32_t ncols;
  uint32_t batch_rows, words_per_batch;   // bit-packed buffers restart every batch
  uint32_t lines;                          // 1: NDJSON (one object per line), 0: one JSON array
  unsigned long long n_rows;
};

#if defined(__CUDACC__)
__device__ __forceinline__ bool json_bit(const uint32_t* w, const JsonArgs& a, unsigned long long i) {
  const unsigned long long b = i / a.batch_rows;
  const uint32_t pos = uint32_t(i - b * a.batch_rows);
  return (w[b * a.words_per_batch + (pos >> 5)] >> (pos & 31)) & 1u;
}
// the value text of (row, col); out == nullptr: only the length
__device__ __forceinline__ uint32_t json_value(const JsonArgs& a, const JsonCol& c, unsigned long long i, char* out) {
  char tmp[40];
  char* o = out ? out : tmp;
  switch (c.type) {
    case JT_I64: return jf_i64(reinterpret_cast<const long long*>(c.values)[i], o);
    case JT_U64: {
      unsigned long long u = reinterpret_cast<const unsigned long long*>(c.values)[i];
      if (u <= 0x7fffffffffffffffull) return jf_i64((long long)u, o);
      char t2[20]; uint32_t k = 0, n = 0;
      do { t2[k++] = char('0' + u % 10); u /= 10; } while (u);
      while (k) o[n++] = t2[--k];
      return n;
    }
    case JT_F64: {
      const double v = reinterpret_cast<const double*>(c.values)[i];
      if (!(v - v == 0.0)) { o[0] = 'n'; o[1] = 'u'; o[2] = 'l'; o[3] = 'l'; return 4; }   // NaN / Inf: JSON has none
      return ryu_format_f64(v, o);
    }
    case JT_BOOL: {
      const bool v = json_bit(reinterpret_cast<const uint32_t*>(c.values), a, i);
      const char* s = v ? "true" : "false";
      const uint32_t n = v ? 4 : 5;
      for (uint32_t k = 0; k < n; k++) o[k] = s[k];
      return n;
    }
    case JT_TS_MS: {
      o[0] = '"';
      const uint32_t n = jf_ts_ms(reinterpret_cast<const long long*>(c.values)[i], o + 1);
      o[n + 1] = '"';
      return n + 2;
    }
    case JT_DATE32: {
      o[0] = '"';
      const uint32_t n = jf_date32(reinterpret_cast<const int*>(c.values)[i], o + 1);
      o[n + 1] = '"';
      return n + 2;
    }
    default: {
      const int32_t b = c.offsets[i], e = c.offsets[i + 1];
      const uint8_t* s = c.values + b;
      if (!out) return 2 + jf_escaped_len(s, uint32_t(e - b));
      out[0] = '"';
      const uint32_t n = jf_escape(s, uint32_t(e - b), out + 1);
      out[n + 1] = '"';
      return n + 2;
    }
  }
}
// bytes of row i's object (with its separator: ',' or '\n' behind every row; the host fixes the very last byte)
__global__ void k_json_sizes(const __grid_constant__ JsonArgs a, uint32_t* __restrict__ lens) {
  const unsigned long long i = blockIdx.x * (unsigned long long)blockDim.x + threadIdx.x;
  if (i >= a.n_rows) return;
  uint32_t n = 3, fields = 0;   // { } and the separator
  for (uint32_t c = 0; c < a.ncols; c++) {
    const JsonCol& col = a.cols[c];
    if (col.validity && !json_bit(col.validity, a, i)) continue;
    n += col.key_len + json_value(a, col, i, nullptr);
    fields++;
  }
  if (fields > 1) n += fields - 1;
  lens[i] = n;
}
__global__ void k_json_write(const __grid_constant__ JsonArgs a, const long long* __restrict__ offs, char* __restrict__ out) {
  const unsigned long long i = blockIdx.x * (unsigned long long)blockDim.x + threadIdx.x;
  if (i >= a.n_rows) return;
  char* o = out + offs[i];
  uint32_t n = 0;
  o[n++] = '{';
  bool first = true;
  for (uint32_t c = 0; c < a.ncols; c++) {
    const JsonCol& col = a.cols[c];
    if (col.validity && !json_bit(col.validity, a, i)) continue;
    if (!first) o[n++] = ',';
    first = false;
    for (uint32_t k = 0; k < col.key_len; k++) o[n++] = char(a.keys[col.key_off + k]);
    n += json_value(a, col, i, o + n);
  }
  o[n++] = '}';
  o[n++] = a.lines ? '\n' : ',';
}
// exclusive 64-bit prefix of the row lengths; one block
__global__ void k_json_scan(const uint32_t* __restrict__ lens, unsigned long long n, long long* __restrict__ offs, long long base) {
  __shared__ long long warp_sums[32];
  __shared__ long long carry;
  if (threadIdx.x == 0) carry = base;
  __syncthreads();
  const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = blockDim.x >> 5;
  for (unsigned long long i0 = 0; i0 < n; i0 += blockDim.x) {
    const unsigned long long i = i0 + threadIdx.x;
    long long v = i < n ? lens[i] : 0, incl = v;
    for (int o = 1; o < 32; o <<= 1) {
      const long long t = __shfl_up_sync(0xffffffffu, incl, o);
      if ((int)lane >= o) incl += t;
    }
    if (lane == 31) warp_sums[warp] = incl;
    __syncthreads();
    long long wbase = 0;
    for (uint32_t w = 0; w < warp; w++) wbase += warp_sums[w];
    if (i < n) offs[i] = carry + wbase + incl - v;
    __syncthreads();
    if (threadIdx.x == blockDim.x - 1) carry += wbase + incl;
    (void)nwarps;
    __syncthreads();
  }
  if (threadIdx.x == 0) offs[n] = carry;
}
#endif

}  // namespace pqb
