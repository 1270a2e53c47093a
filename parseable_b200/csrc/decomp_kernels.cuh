// Page decompression on the GPU: LZ4_RAW (Parseable's default codec,
// /root/reference/src/cli.rs:441-448), SNAPPY (what the reference's CI pins,
// docker-compose-test.yaml:45), ZSTD and GZIP (zstd_decode.cuh, inflate_decode.cuh; k_decompress_zstd below).  The reference gets these from the lz4_flex 0.13 /
// snap 1.1 crates through parquet 58.1.0 (SURVEY.md §8 row a10); here one warp
// decodes one page (the formats: lz_decode.cuh).  table.cu and the test library
// tools/decomp_dev.cu both go through launch_decompress below.
//
// Output goes into the same HBM arena the scan kernel reads, so a compressed file
// costs one extra HBM write + read of the decoded pages and nothing else changes.
#pragma once
#include <cuda_runtime.h>

#include <algorithm>
#include <cstdint>
#include <vector>

#include "device_structs.hpp"
#include "inflate_decode.cuh"
#include "lz_decode.cuh"
#include "zstd_decode.cuh"

namespace pqb {

struct DecompJob {
  uint64_t src_off;   // compressed page payload inside the staging buffer
  uint64_t dst_off;   // decoded page payload inside the arena
  uint32_t src_len;
  uint32_t dst_len;   // uncompressed_page_size from the page header
  uint32_t codec;     // parquet CompressionCodec: 7 LZ4_RAW, 1 SNAPPY, 6 ZSTD, 2 GZIP, 0 plain copy (src_len must equal dst_len)
  uint32_t _pad;
};

__global__ void k_decompress_pages(const DecompJob* __restrict__ jobs, uint32_t njobs, const uint8_t* __restrict__ src_base,
                                   uint8_t* __restrict__ arena, unsigned long long* __restrict__ counters) {
  const uint32_t j = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (j >= njobs) return;
  const DecompJob job = jobs[j];
  const uint8_t* s = src_base + job.src_off;
  uint8_t* d = arena + job.dst_off;
  bool ok = false;
  if (job.codec == 7) ok = lz4_raw_decode(s, job.src_len, d, job.dst_len);
  else if (job.codec == 1) ok = snappy_decode(s, job.src_len, d, job.dst_len);
  else if (job.codec == 0) ok = stored_decode(s, job.src_len, d, job.dst_len);
  if (!ok && (threadIdx.x & 31) == 0) atomicExch(&counters[0], 1ull);
}

// ZSTD (codec 6) and GZIP (codec 2) pages: persistent warps draw pages from a counter; every warp owns one workspace
// (tables + the literals of one zstd block) in global memory.  zstd_decode.cuh / inflate_decode.cuh hold the formats.
__global__ void __launch_bounds__(128) k_decompress_zstd(const DecompJob* __restrict__ jobs, uint32_t njobs, const uint8_t* __restrict__ src_base,
                                                         uint8_t* __restrict__ arena, unsigned long long* __restrict__ counters,
                                                         HeavyWs* __restrict__ ws, unsigned int* __restrict__ next) {
  const uint32_t lane = threadIdx.x & 31;
  HeavyWs& w = ws[blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5)];
  for (;;) {
    uint32_t j = 0;
    if (lane == 0) j = atomicAdd(next, 1u);
    j = __shfl_sync(0xffffffffu, j, 0);
    if (j >= njobs) break;
    const DecompJob job = jobs[j];
    const bool ok = heavy_page_decode(w, job.codec, src_base + job.src_off, job.src_len, arena + job.dst_off, job.dst_len);
    if (!ok && lane == 0) atomicExch(&counters[0], 1ull);
    __syncwarp();
  }
}

// Queues the decoding of `djobs` on `stream`: src_base holds the compressed payloads (with 256 bytes of slack behind
// the last: the literal copy reads up to 3 bytes past a literal), arena receives the pages, *flag (zeroed by the
// caller) becomes nonzero when a page does not decode to its declared size.  djobs is reordered: ZSTD / GZIP pages
// go behind the others, their decoders are a kernel of their own (persistent warps, one workspace each).  The job
// list, the workspaces and the ticket counter are allocated here on `stream` and handed back for the caller to free
// once the stream is done; whatever this allocated is in them even when it returns an error.
inline cudaError_t launch_decompress(std::vector<DecompJob>& djobs, const uint8_t* src_base, uint8_t* arena, unsigned long long* flag,
                                     int sm_count, cudaStream_t stream, DecompJob** d_djobs, HeavyWs** d_ws, unsigned int** d_next) {
  if (djobs.empty()) return cudaSuccess;
  cudaError_t e = cudaMallocAsync((void**)d_djobs, djobs.size() * sizeof(DecompJob), stream);
  if (e != cudaSuccess) return e;
  const uint32_t n_other = uint32_t(std::stable_partition(djobs.begin(), djobs.end(), [](const DecompJob& j) { return j.codec != 6u && j.codec != 2u; }) - djobs.begin());
  const uint32_t n_heavy = uint32_t(djobs.size()) - n_other;
  if ((e = cudaMemcpyAsync(*d_djobs, djobs.data(), djobs.size() * sizeof(DecompJob), cudaMemcpyHostToDevice, stream)) != cudaSuccess) return e;
  if (n_other) k_decompress_pages<<<(n_other + 3) / 4, 128, 0, stream>>>(*d_djobs, n_other, src_base, arena, flag);
  if ((e = cudaGetLastError()) != cudaSuccess) return e;
  if (n_heavy) {
    const uint32_t blocks = std::min<uint32_t>((n_heavy + 3) / 4, uint32_t(sm_count) * 2u);
    if ((e = cudaMallocAsync((void**)d_ws, size_t(blocks) * 4 * sizeof(HeavyWs), stream)) != cudaSuccess) return e;
    if ((e = cudaMallocAsync((void**)d_next, 4, stream)) != cudaSuccess) return e;
    if ((e = cudaMemsetAsync(*d_next, 0, 4, stream)) != cudaSuccess) return e;
    k_decompress_zstd<<<blocks, 128, 0, stream>>>(*d_djobs + n_other, n_heavy, src_base, arena, flag, *d_ws, *d_next);
    if ((e = cudaGetLastError()) != cudaSuccess) return e;
  }
  return cudaSuccess;
}

// After decompression the host still does not know two bytes it normally reads from the file:
// the definition-level byte count (first 4 bytes of a v1 page) and the dictionary index bit width.
// flags: bit 0 page has a v1 definition-level block, bits 8.. DevEnc.
__global__ void k_page_fixup(DevPage* __restrict__ pages, const uint32_t* __restrict__ which, uint32_t n,
                             const uint8_t* __restrict__ arena, unsigned long long* __restrict__ counters) {
  uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  DevPage p = pages[which[i]];
  const uint8_t* payload = arena + p.off;
  uint32_t pos = p.val_off;   // v2 pages: the level bytes in front of the values (lengths from the page header); v1: 0
  if (p.def_len == 0xffffffffu) {  // v1 page of a nullable column: 4-byte length + RLE definition levels
    uint32_t dl = 0;
    if (p.len >= 4) dl = uint32_t(payload[0]) | (uint32_t(payload[1]) << 8) | (uint32_t(payload[2]) << 16) | (uint32_t(payload[3]) << 24);
    if (p.len < 4 || uint64_t(dl) + 4 > p.len) { atomicExch(&counters[0], 2ull); dl = 0; }
    p.def_off = 4;
    p.def_len = dl;
    pos = 4 + dl;
  }
  p.val_off = pos;
  if (p.enc == DE_DICT) {
    if (pos < p.len && p.num_rows) { p.bit_width = payload[pos]; p.val_off = pos + 1; }
    else p.bit_width = 0;
  } else if (p.enc == DE_RLE_BOOL) {
    p.bit_width = 1;
    if (p.num_rows && pos + 4 <= p.len) p.val_off = pos + 4;
  }
  pages[which[i]] = p;
}

}  // namespace pqb
