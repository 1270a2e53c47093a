// Host build of the PQ_OP_REGEX compiler and DFA walk (regex_compile.cpp, regex_match.cuh) for the CPU tests.
#include <cstring>

#include "regex_compile.cpp"

extern "C" {

// Compiles `pat`; returns 0 and the blob size in *blob_len (the blob is copied to `blob` when it fits in `cap`), or the
// PqStatus of the refusal with its message in `err`.
int rx_compile(const char* pat, uint64_t n, int case_insensitive, uint8_t* blob, uint64_t cap, uint64_t* blob_len,
               char* err, uint64_t err_cap) {
  std::vector<uint8_t> b;
  std::string e;
  const int st = pqb::regex_compile(pat, n, case_insensitive != 0, b, e);
  *blob_len = b.size();
  if (st == 0 && b.size() <= cap) std::memcpy(blob, b.data(), b.size());
  if (err_cap) {
    const size_t k = std::min<size_t>(e.size(), err_cap - 1);
    std::memcpy(err, e.data(), k);
    err[k] = 0;
  }
  return st;
}

// out[i] = regex_match(data[off[i], off[i + 1]))
void rx_match_many(const uint8_t* blob, const uint8_t* data, const int64_t* off, int64_t n, uint8_t* out) {
  for (int64_t i = 0; i < n; i++) out[i] = pqb::regex_match(data + off[i], uint32_t(off[i + 1] - off[i]), blob) ? 1 : 0;
}
}
