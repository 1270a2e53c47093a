// TEST HARNESS ONLY: the membership set of PQ_OP_IN (in_set.cuh) built and probed on the CPU, for
// tests/test_in_set_core.py.  The build and the probe are the ones query.cu and the kernels use.  Never linked into
// libparseable_b200.so.
#include <cstring>
#include <vector>

#include "in_set.cuh"
using namespace pqb;

namespace {
std::vector<uint8_t> g_blob;   // the set the last build made

uint64_t keep(std::vector<uint8_t> b) {
  g_blob = std::move(b);
  return g_blob.size();
}
}  // namespace

extern "C" {
uint64_t in_empty_value() { return kInSetEmpty; }

// Builds a numeric set of v[0, n); returns the blob's size
uint64_t in_build_u64(const uint64_t* v, uint64_t n) { return keep(in_set_build_u64(v, n)); }

// Builds a bytes set of the n strings data[off[k], off[k + 1]); returns the blob's size
uint64_t in_build_bytes(const uint8_t* data, const int64_t* off, uint64_t n) {
  std::vector<const uint8_t*> p(n);
  std::vector<uint32_t> len(n);
  for (uint64_t k = 0; k < n; k++) { p[k] = data + off[k]; len[k] = uint32_t(off[k + 1] - off[k]); }
  return keep(in_set_build_bytes(p.data(), len.data(), n));
}

// Copies the last blob out (its first `cap` bytes)
void in_blob(uint8_t* out, uint64_t cap) { std::memcpy(out, g_blob.data(), std::min<uint64_t>(cap, g_blob.size())); }

// out[i] = v[i] is a member of the last set (numeric)
void in_probe_u64(const uint64_t* v, uint64_t n, uint8_t* out) {
  for (uint64_t i = 0; i < n; i++) out[i] = in_set_has(g_blob.data(), nullptr, 0, v[i]) ? 1 : 0;
}

// out[i] = data[off[i], off[i + 1]) is a member of the last set (bytes)
void in_probe_bytes(const uint8_t* data, const int64_t* off, uint64_t n, uint8_t* out) {
  for (uint64_t i = 0; i < n; i++)
    out[i] = in_set_has(g_blob.data(), data + off[i], uint32_t(off[i + 1] - off[i]), 0) ? 1 : 0;
}
}
