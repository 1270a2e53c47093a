// TEST HARNESS ONLY: host build of the number / timestamp / string formatting the JSON egress kernels use
// (parseable_b200/csrc/ryu_f64.cuh, json_egress.cuh), for tests/test_json_egress.py.  Never linked into the product.
#include <cstdint>
#include "json_egress.cuh"

extern "C" {
uint32_t jh_format_f64(double v, char* out) { return pqb::ryu_format_f64(v, out); }
void jh_format_f64_many(const double* v, uint64_t n, char* out /* 32 bytes each, NUL padded */) {
  for (uint64_t i = 0; i < n; i++) {
    char* o = out + i * 32;
    const uint32_t k = pqb::ryu_format_f64(v[i], o);
    for (uint32_t j = k; j < 32; j++) o[j] = 0;
  }
}
uint32_t jh_format_i64(int64_t v, char* out) { return pqb::jf_i64(v, out); }
uint32_t jh_format_ts_ms(int64_t v, char* out) { return pqb::jf_ts_ms(v, out); }
uint32_t jh_format_date32(int32_t v, char* out) { return pqb::jf_date32(v, out); }
uint32_t jh_escape(const uint8_t* s, uint32_t n, char* out) {
  const uint32_t want = pqb::jf_escaped_len(s, n), got = pqb::jf_escape(s, n, out);
  return want == got ? got : 0xffffffffu;
}
}
