// TEST LIBRARY ONLY: the page decoders of parseable_b200/csrc/decomp_kernels.cuh on the GPU, launched through the
// same launch_decompress as table.cu, so that tests/test_page_codecs.py and tests/test_zstd.py can check the kernels
// the table-open path runs against pyarrow's codecs.  Never linked into libparseable_b200.so.
#include <cuda_runtime.h>

#include <cstdint>
#include <vector>

#include "decomp_kernels.cuh"

// jobs: njobs DecompJob records over a source image src[0 .. src_bytes) and a destination image dst[0 .. dst_bytes).
// Both images are uploaded (the destination with whatever the caller put around the jobs' slots), the source with the
// same 256 bytes of zeroed slack as table.cu's staging buffer; the decoders run on a stream of their own, the
// destination comes back into dst and the error flag into *flag.  Everything allocated is freed before returning.
// Returns the first CUDA error (0: none).
extern "C" int decomp_dev_run(const pqb::DecompJob* jobs, uint32_t njobs, const uint8_t* src, uint64_t src_bytes, uint8_t* dst,
                              uint64_t dst_bytes, unsigned long long* flag) {
  std::vector<pqb::DecompJob> djobs(jobs, jobs + njobs);
  int dev = 0, sms = 0;
  cudaError_t e = cudaGetDevice(&dev);
  if (e == cudaSuccess) e = cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  if (e != cudaSuccess) return int(e);
  cudaStream_t stream = nullptr;
  if ((e = cudaStreamCreateWithFlags(&stream, cudaStreamNonBlocking)) != cudaSuccess) return int(e);
  uint8_t *d_src = nullptr, *d_dst = nullptr;
  unsigned long long* d_flag = nullptr;
  pqb::DecompJob* d_jobs = nullptr;
  pqb::HeavyWs* d_ws = nullptr;
  unsigned int* d_next = nullptr;
  auto run = [&]() -> cudaError_t {
    cudaError_t r;
    if ((r = cudaMallocAsync((void**)&d_src, src_bytes + 256, stream)) != cudaSuccess) return r;
    if ((r = cudaMallocAsync((void**)&d_dst, dst_bytes ? dst_bytes : 1, stream)) != cudaSuccess) return r;
    if ((r = cudaMallocAsync((void**)&d_flag, 8, stream)) != cudaSuccess) return r;
    if ((r = cudaMemsetAsync(d_src + src_bytes, 0, 256, stream)) != cudaSuccess) return r;
    if ((r = cudaMemcpyAsync(d_src, src, src_bytes, cudaMemcpyHostToDevice, stream)) != cudaSuccess) return r;
    if ((r = cudaMemcpyAsync(d_dst, dst, dst_bytes, cudaMemcpyHostToDevice, stream)) != cudaSuccess) return r;
    if ((r = cudaMemsetAsync(d_flag, 0, 8, stream)) != cudaSuccess) return r;
    if ((r = pqb::launch_decompress(djobs, d_src, d_dst, d_flag, sms, stream, &d_jobs, &d_ws, &d_next)) != cudaSuccess) return r;
    if ((r = cudaMemcpyAsync(dst, d_dst, dst_bytes, cudaMemcpyDeviceToHost, stream)) != cudaSuccess) return r;
    return cudaMemcpyAsync(flag, d_flag, 8, cudaMemcpyDeviceToHost, stream);
  };
  e = run();
  auto step = [&](cudaError_t r) { if (e == cudaSuccess) e = r; };
  step(cudaStreamSynchronize(stream));
  for (void* p : {(void*)d_src, (void*)d_dst, (void*)d_flag, (void*)d_jobs, (void*)d_ws, (void*)d_next})
    if (p) step(cudaFree(p));
  step(cudaStreamDestroy(stream));
  return int(e);
}
