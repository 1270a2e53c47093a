// TEST HARNESS ONLY: the ZSTD and GZIP page decoders of parseable_b200/csrc/zstd_decode.cuh / inflate_decode.cuh
// compiled for the host (one "lane"), so that tests/test_zstd.py can check them against pyarrow's codecs on the CPU.
// Never linked into libparseable_b200.so.
#include <cstdint>
#include <cstdlib>
#include <new>
#include "inflate_decode.cuh"
#include "zstd_decode.cuh"

extern "C" int zs_host_decode(const uint8_t* src, uint32_t sn, uint8_t* dst, uint64_t dn) {
  pqb::ZstdWs* w = new (std::nothrow) pqb::ZstdWs();
  if (!w) return -1;
  const bool ok = pqb::zstd_decode(*w, src, sn, dst, dn);
  delete w;
  return ok ? 1 : 0;
}
extern "C" int gz_host_decode(const uint8_t* src, uint32_t sn, uint8_t* dst, uint64_t dn) {
  pqb::InflateWs* w = new (std::nothrow) pqb::InflateWs();
  if (!w) return -1;
  const bool ok = pqb::gzip_decode(*w, src, sn, dst, dn);
  delete w;
  return ok ? 1 : 0;
}
// A run of n pages, ZSTD (codec 6) and GZIP (codec 2) mixed, decoded one after another through ONE workspace, as a
// warp of k_decompress_zstd does: page k is src[src_off[k] ..][0 .. src_len[k]) -> dst[dst_off[k] ..][0 .. dst_len[k]).
// ok[k] = 1 when page k decoded; returns how many did, -1 without memory.
extern "C" int heavy_host_decode_run(uint32_t n, const uint32_t* codec, const uint8_t* src, const uint64_t* src_off, const uint32_t* src_len,
                                     uint8_t* dst, const uint64_t* dst_off, const uint32_t* dst_len, int32_t* ok) {
  pqb::HeavyWs* w = new (std::nothrow) pqb::HeavyWs();
  if (!w) return -1;
  int good = 0;
  for (uint32_t k = 0; k < n; k++) {
    ok[k] = pqb::heavy_page_decode(*w, codec[k], src + src_off[k], src_len[k], dst + dst_off[k], dst_len[k]) ? 1 : 0;
    good += ok[k];
  }
  delete w;
  return good;
}
