// TEST HARNESS ONLY: the LZ4_RAW, SNAPPY and stored page decoders of parseable_b200/csrc/lz_decode.cuh compiled for
// the host, every copy run lane by lane for all 32 lanes (descending when built with -DLZ_LANES_DESCENDING=1), so that
// tests/test_page_codecs.py can check them against pyarrow's codecs on the CPU.  Never linked into libparseable_b200.so.
#include <cstdint>
#include <cstdlib>
#include <cstring>

#include "lz_decode.cuh"

static constexpr uint32_t kSrcSlack = 256;   // as behind the staging buffer of table.cu
static constexpr uint32_t kMaxGuard = 64;

// Decodes src[0 .. sn) as `codec` (7 LZ4_RAW, 1 SNAPPY, 0 stored) into dn bytes.  The source is placed at byte phase
// sphase (0-63) of a 64-byte aligned buffer, the destination at phase dphase.  `out` holds guard + dn + guard bytes:
// its guards (the canaries, set by the caller) are placed on both sides of the destination before decoding, and the
// whole window comes back, so the caller sees the decoded bytes and any write outside them.
// Returns 1: decoded, 0: refused, -1: bad arguments or no memory.
extern "C" int lz_host_decode(uint32_t codec, const uint8_t* src, uint32_t sn, uint32_t sphase, uint8_t* out, uint32_t dn,
                              uint32_t dphase, uint32_t guard) {
  if (sphase >= 64 || dphase >= 64 || guard > kMaxGuard) return -1;
  const size_t sbytes = (size_t(sphase) + sn + kSrcSlack + 63) & ~size_t(63);
  const size_t dbytes = (size_t(kMaxGuard) + dphase + dn + kMaxGuard + 63) & ~size_t(63);
  uint8_t* sb = static_cast<uint8_t*>(std::aligned_alloc(64, sbytes));
  uint8_t* db = static_cast<uint8_t*>(std::aligned_alloc(64, dbytes));
  if (!sb || !db) { std::free(sb); std::free(db); return -1; }
  std::memset(sb, 0xee, sbytes);
  if (sn) std::memcpy(sb + sphase, src, sn);
  uint8_t* d = db + kMaxGuard + dphase;
  std::memset(db, 0, dbytes);
  std::memcpy(d - guard, out, size_t(guard) * 2 + dn);
  const uint8_t* s = sb + sphase;
  bool ok = false;
  if (codec == 7) ok = pqb::lz4_raw_decode(s, sn, d, dn);
  else if (codec == 1) ok = pqb::snappy_decode(s, sn, d, dn);
  else if (codec == 0) ok = pqb::stored_decode(s, sn, d, dn);
  std::memcpy(out, d - guard, size_t(guard) * 2 + dn);
  std::free(sb);
  std::free(db);
  return ok ? 1 : 0;
}
