// Context + Table: footer parsing, page-header walk, and the upload of encoded
// column chunks into one HBM arena.  Only the referenced columns of the row
// groups this process owns (g % shard_count == shard_index, the GPU analogue of
// partitioned_files' round-robin, stream_schema_provider.rs:351-364) are read.
#include <fcntl.h>
#include <sys/mman.h>
#include <sys/stat.h>
#include <unistd.h>

#include <algorithm>
#include <atomic>
#include <chrono>
#include <cstring>
#include <exception>
#include <thread>

#include "decomp_kernels.cuh"
#include "engine.hpp"
#include "order_keys.cuh"

namespace pqb {

struct GatherCopy { const uint8_t* src; uint64_t dst_off; uint64_t bytes; };

// src (mapped page-locked host memory) and arena + dst_off share their 16-byte phase
__global__ void k_gather_copy(const GatherCopy* __restrict__ copies, uint8_t* __restrict__ arena) {
  const GatherCopy c = copies[blockIdx.x];
  const uint8_t* src = c.src;
  uint8_t* dst = arena + c.dst_off;
  const uint64_t head = (16 - (reinterpret_cast<uintptr_t>(src) & 15)) & 15;
  const uint64_t h = head < c.bytes ? head : c.bytes;
  if (blockIdx.y == 0 && threadIdx.x < h) dst[threadIdx.x] = src[threadIdx.x];
  const uint64_t nvec = (c.bytes - h) / 16;
  const uint4* s4 = reinterpret_cast<const uint4*>(src + h);
  uint4* d4 = reinterpret_cast<uint4*>(dst + h);
  for (uint64_t i = uint64_t(blockIdx.y) * blockDim.x + threadIdx.x; i < nvec; i += uint64_t(gridDim.y) * blockDim.x) {
    uint4 v0 = s4[i];
    d4[i] = v0;
  }
  const uint64_t tail0 = h + nvec * 16;
  if (blockIdx.y == 0 && tail0 + threadIdx.x < c.bytes) dst[tail0 + threadIdx.x] = src[tail0 + threadIdx.x];
}

// ---------------- Context ----------------
Context& Context::get() {
  static Context c;
  return c;
}

void Context::init(const int* devices, int n) {
  std::lock_guard<std::mutex> lk(mu_);
  int count = 0;
  cudaError_t e = cudaGetDeviceCount(&count);
  if (e != cudaSuccess || count == 0)
    throw Error(PQ_ERR_CUDA, std::string("no CUDA device: ") + (e != cudaSuccess ? cudaGetErrorString(e) : "count 0"));
  int dev = 0;
  if (n > 0 && devices) dev = devices[0];
  else if (inited_) dev = device_;
  else {
    const char* lr = getenv("LOCAL_RANK");
    if (lr) dev = atoi(lr) % count;
  }
  if (dev < 0 || dev >= count) throw Error(PQ_ERR_INVALID_ARG, "device id out of range");
  PQB_CUDA(cudaSetDevice(dev));
  cudaDeviceProp prop;
  PQB_CUDA(cudaGetDeviceProperties(&prop, dev));
  // the library carries sm_90a code only, which no other compute capability can run
  if (prop.major != 9 || prop.minor != 0)
    throw Error(PQ_ERR_CUDA, "parseable_b200 needs an sm_90a (Hopper) device (found sm_" +
                                 std::to_string(prop.major * 10 + prop.minor) + ")");
  device_ = dev;
  sm_count_ = prop.multiProcessorCount;
  smem_optin_ = prop.sharedMemPerBlockOptin;
  smem_per_sm_ = prop.sharedMemPerMultiprocessor;
  l2_bytes_ = size_t(prop.l2CacheSize);
  // keep freed blocks in the stream-ordered pool: query-time cudaMallocAsync stays cheap
  cudaMemPool_t pool;
  PQB_CUDA(cudaDeviceGetDefaultMemPool(&pool, dev));
  uint64_t thresh = ~0ull;
  PQB_CUDA(cudaMemPoolSetAttribute(pool, cudaMemPoolAttrReleaseThreshold, &thresh));
  inited_ = true;
}

void Context::ensure() {
  if (!inited_) init(nullptr, 0);
  PQB_CUDA(cudaSetDevice(device_));
}

void Context::shutdown() {
  std::lock_guard<std::mutex> lk(mu_);
  for (auto& p : pinned_) cudaFreeHost(p.p);
  pinned_.clear();
  for (auto& [dev, s] : free_streams_) cudaStreamDestroy(s);
  free_streams_.clear();
  inited_ = false;
}

cudaStream_t Context::stream_acquire() {
  {
    std::lock_guard<std::mutex> lk(mu_);
    for (size_t i = free_streams_.size(); i-- > 0;) {
      if (free_streams_[i].first != device_) continue;
      cudaStream_t s = free_streams_[i].second;
      free_streams_.erase(free_streams_.begin() + i);
      return s;
    }
  }
  cudaStream_t s;
  PQB_CUDA(cudaStreamCreateWithFlags(&s, cudaStreamNonBlocking));
  return s;
}

void Context::stream_release(cudaStream_t s, int device) {
  std::lock_guard<std::mutex> lk(mu_);
  free_streams_.emplace_back(device, s);
}

uint8_t* Context::pinned_acquire(size_t bytes) {
  std::lock_guard<std::mutex> lk(mu_);
  for (auto& p : pinned_)
    if (!p.busy && p.cap >= bytes) { p.busy = true; return p.p; }
  Pinned np{nullptr, std::max<size_t>(bytes, 1 << 20), true};
  cudaError_t e = cudaHostAlloc((void**)&np.p, np.cap, cudaHostAllocDefault);
  if (e != cudaSuccess) throw Error(PQ_ERR_OOM, std::string("cudaHostAlloc: ") + cudaGetErrorString(e));
  pinned_.push_back(np);
  return np.p;
}

void Context::pinned_release(uint8_t* ptr) {
  std::lock_guard<std::mutex> lk(mu_);
  for (auto& p : pinned_)
    if (p.p == ptr) p.busy = false;
}

bool Context::is_pinned(const void* p) {
  cudaPointerAttributes at;
  if (cudaPointerGetAttributes(&at, p) != cudaSuccess) { cudaGetLastError(); return false; }
  return at.type == cudaMemoryTypeHost;
}

PinnedBlock::~PinnedBlock() {
  if (p && heap.empty()) Context::get().pinned_release(p);
}

// ---------------- HostFile ----------------
HostFile::~HostFile() {
  if (mapped && data) munmap(const_cast<uint8_t*>(data), size);
}

static std::unique_ptr<HostFile> open_host_file(const PqFile& f) {
  auto hf = std::make_unique<HostFile>();
  if (f.buf) {
    hf->data = f.buf;
    hf->size = f.size;
  } else if (f.path) {
    hf->path = f.path;
    int fd = ::open(f.path, O_RDONLY);
    if (fd < 0) throw Error(PQ_ERR_IO, std::string("open ") + f.path + ": " + strerror(errno));
    struct stat st;
    if (fstat(fd, &st) != 0) { ::close(fd); throw Error(PQ_ERR_IO, std::string("stat ") + f.path); }
    hf->size = uint64_t(st.st_size);
    if (hf->size) {
      void* m = mmap(nullptr, hf->size, PROT_READ, MAP_PRIVATE, fd, 0);
      if (m == MAP_FAILED) { ::close(fd); throw Error(PQ_ERR_IO, std::string("mmap ") + f.path); }
      hf->data = static_cast<const uint8_t*>(m);
      hf->mapped = true;
    }
    ::close(fd);
  } else {
    throw Error(PQ_ERR_INVALID_ARG, "PqFile needs a path or a buffer");
  }
  try {
    hf->meta = parse_footer(hf->data, hf->size);
  } catch (const std::exception& e) {
    throw Error(PQ_ERR_CORRUPT, (hf->path.empty() ? std::string("<buffer>") : hf->path) + ": " + e.what());
  }
  return hf;
}

static void js_str(std::string& o, const std::string& s) {
  o.push_back('"');
  for (unsigned char c : s) {
    if (c == '"' || c == '\\') { o.push_back('\\'); o.push_back(char(c)); }
    else if (c < 0x20) { char b[8]; snprintf(b, sizeof b, "\\u%04x", c); o += b; }
    else o.push_back(char(c));
  }
  o.push_back('"');
}

std::string describe_file(const PqFile& f) {
  auto hf = open_host_file(f);
  std::string o = "{\"num_rows\":" + std::to_string(hf->meta.num_rows) + ",\"created_by\":";
  js_str(o, hf->meta.created_by);
  o += ",\"leaves\":[";
  for (size_t i = 0; i < hf->meta.leaves.size(); i++) {
    const LeafColumn& l = hf->meta.leaves[i];
    if (i) o += ",";
    o += "{\"name\":";
    js_str(o, l.name);
    o += ",\"phys_type\":" + std::to_string(l.phys_type) + ",\"max_def\":" + std::to_string(l.max_def) +
         ",\"max_rep\":" + std::to_string(l.max_rep) + ",\"is_timestamp_ms\":" + (l.is_timestamp_ms ? "true" : "false") +
         ",\"is_date\":" + (l.is_date ? "true" : "false") + "}";
  }
  o += "],\"row_groups\":[";
  for (size_t g = 0; g < hf->meta.row_groups.size(); g++) {
    const RowGroupMeta& rg = hf->meta.row_groups[g];
    if (g) o += ",";
    o += "{\"num_rows\":" + std::to_string(rg.num_rows) + ",\"columns\":[";
    for (size_t c = 0; c < rg.columns.size(); c++) {
      const ColumnChunkMeta& cm = rg.columns[c];
      if (c) o += ",";
      o += "{\"type\":" + std::to_string(cm.type) + ",\"codec\":" + std::to_string(cm.codec) +
           ",\"num_values\":" + std::to_string(cm.num_values) +
           ",\"total_uncompressed_size\":" + std::to_string(cm.total_uncompressed_size) +
           ",\"total_compressed_size\":" + std::to_string(cm.total_compressed_size) +
           ",\"data_page_offset\":" + std::to_string(cm.data_page_offset) +
           ",\"dictionary_page_offset\":" + std::to_string(cm.dictionary_page_offset) +
           ",\"null_count\":" + std::to_string(cm.stats.null_count);
      // PLAIN-encoded min / max statistics as hex (INT32: 4 bytes, INT64 / DOUBLE: 8)
      auto hex = [](const std::string& b) {
        static const char* d = "0123456789abcdef";
        std::string h;
        for (unsigned char c : b) { h.push_back(d[c >> 4]); h.push_back(d[c & 15]); }
        return h;
      };
      if (cm.stats.has_min) o += ",\"stats_min\":\"" + hex(cm.stats.min) + "\"";
      if (cm.stats.has_max) o += ",\"stats_max\":\"" + hex(cm.stats.max) + "\"";
      o += ",\"encodings\":[";
      for (size_t e = 0; e < cm.encodings.size(); e++) o += (e ? "," : "") + std::to_string(cm.encodings[e]);
      o += "],\"pages\":[";
      if (uint64_t(cm.start()) + uint64_t(cm.total_compressed_size) > hf->size) throw Error(PQ_ERR_CORRUPT, "column chunk outside the file");
      std::vector<PageInfo> pis;
      try { pis = walk_pages(hf->data + cm.start(), uint64_t(cm.total_compressed_size), cm.num_values); }
      catch (const std::exception& e) { throw Error(PQ_ERR_CORRUPT, e.what()); }
      for (size_t p = 0; p < pis.size(); p++) {
        const PageInfo& pi = pis[p];
        if (p) o += ",";
        o += "{\"type\":" + std::to_string(pi.type) + ",\"num_values\":" + std::to_string(pi.num_values) +
             ",\"encoding\":" + std::to_string(pi.encoding) + ",\"compressed_size\":" + std::to_string(pi.compressed_size) +
             ",\"uncompressed_size\":" + std::to_string(pi.uncompressed_size) + ",\"header_len\":" + std::to_string(pi.header_len) + "}";
      }
      o += "]}";
    }
    o += "]}";
  }
  o += "]}";
  return o;
}

// Temporary device buffers of the open path: dev_drop() frees (stream ordered) and clears the pointer; an UnwindGuard
// frees whatever it still owns when an exception leaves its scope and synchronises the stream first, so that no copy
// or kernel is in flight into memory the caller's destructor is about to hand back.
template <class T>
static void dev_drop(T*& p, cudaStream_t s) {
  if (p) { cudaFreeAsync((void*)p, s); p = nullptr; }
}
struct UnwindGuard {
  cudaStream_t s;
  int n;
  std::vector<void**> ptrs;
  explicit UnwindGuard(cudaStream_t st) : s(st), n(std::uncaught_exceptions()) {}
  template <class T> void own(T*& p) { ptrs.push_back(reinterpret_cast<void**>(&p)); }
  ~UnwindGuard() {
    if (std::uncaught_exceptions() <= n) return;
    cudaStreamSynchronize(s);
    for (void** p : ptrs) if (*p) { cudaFreeAsync(*p, s); *p = nullptr; }
  }
};

// ---------------- Table ----------------
Table::~Table() {
  // stream-ordered frees into the pool: a per-query table costs no device-wide synchronisation
  if (d_arena) cudaFreeAsync(d_arena, cudaStreamPerThread);
  if (d_pages) cudaFreeAsync(d_pages, cudaStreamPerThread);
  if (d_strmat) cudaFreeAsync(d_strmat, cudaStreamPerThread);
  if (d_flat) cudaFreeAsync(d_flat, cudaStreamPerThread);
  if (d_flat_pages) cudaFreeAsync(d_flat_pages, cudaStreamPerThread);
  if (d_agg_pages) cudaFreeAsync(d_agg_pages, cudaStreamPerThread);
  for (ColSide& cs : sides) {
    if (cs.d_for) cudaFreeAsync(cs.d_for, cudaStreamPerThread);
    if (cs.d_ids) cudaFreeAsync(cs.d_ids, cudaStreamPerThread);
    if (cs.d_ent_off) cudaFreeAsync(cs.d_ent_off, cudaStreamPerThread);
    if (cs.d_gid) cudaFreeAsync(cs.d_gid, cudaStreamPerThread);
    if (cs.d_row_ent) cudaFreeAsync(cs.d_row_ent, cudaStreamPerThread);
    if (cs.d_key_hash) cudaFreeAsync(cs.d_key_hash, cudaStreamPerThread);
    if (cs.d_glob_gid) cudaFreeAsync(cs.d_glob_gid, cudaStreamPerThread);
    if (cs.d_glob_kd_offs) cudaFreeAsync(cs.d_glob_kd_offs, cudaStreamPerThread);
    if (cs.d_glob_kd_bytes) cudaFreeAsync(cs.d_glob_kd_bytes, cudaStreamPerThread);
    if (cs.d_delta_flat) cudaFreeAsync(cs.d_delta_flat, cudaStreamPerThread);
    if (cs.d_kd_offs) cudaFreeAsync(cs.d_kd_offs, cudaStreamPerThread);
    if (cs.d_kd_bytes) cudaFreeAsync(cs.d_kd_bytes, cudaStreamPerThread);
  }
}

Shape::~Shape() {
  if (d_chunks) cudaFreeAsync(d_chunks, cudaStreamPerThread);
  if (d_items) cudaFreeAsync(d_items, cudaStreamPerThread);
}

int Table::find_column(const std::string& name) const {
  for (size_t i = 0; i < columns.size(); i++)
    if (columns[i].name == name) return int(i);
  return -1;
}

static uint8_t kind_of_leaf(const LeafColumn& l) {
  switch (l.phys_type) {
    case PT_INT64: return DK_I64;
    case PT_DOUBLE: return DK_F64;
    case PT_BYTE_ARRAY: return DK_STR;
    case PT_BOOLEAN: return DK_BOOL;
    case PT_INT32: return DK_I32;
    case PT_FLOAT: return DK_F32;
    default: return 0xff;
  }
}

static uint32_t rd_u32(const uint8_t* p) {
  uint32_t v;
  std::memcpy(&v, p, 4);
  return v;
}

void Table::open(const PqFile* in_files, uint32_t n_files, const std::vector<std::string>& col_names,
                 uint32_t shard_index, uint32_t shard_count, cudaStream_t stream) {
  Context& ctx = Context::get();
  const auto t_open = std::chrono::steady_clock::now();
  const bool verbose = getenv("PQB_VERBOSE") && getenv("PQB_VERBOSE")[0] == '2';
  auto mark = [&](const char* what) {
    if (verbose) {
      cudaStreamSynchronize(stream);
      fprintf(stderr, "[pqb] table open +%.3f ms %s\n", std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t_open).count(), what);
    }
  };
  if (shard_count == 0) shard_count = 1;
  if (shard_index >= shard_count) throw Error(PQ_ERR_INVALID_ARG, "shard_index >= shard_count");
  this->shard_index = shard_index;
  this->shard_count = shard_count;
  // footers are parsed on a few host threads (one Parquet file per ingest minute: many small footers)
  files.resize(n_files);
  {
    const unsigned nthr = std::min<unsigned>({8u, std::max(1u, std::thread::hardware_concurrency()), n_files});
    std::atomic<uint32_t> next{0};
    std::vector<std::exception_ptr> errs(n_files);
    auto work = [&]() {
      for (;;) {
        uint32_t i = next.fetch_add(1);
        if (i >= n_files) break;
        try { files[i] = open_host_file(in_files[i]); } catch (...) { errs[i] = std::current_exception(); }
      }
    };
    if (nthr <= 1) work();
    else {
      std::vector<std::thread> th;
      for (unsigned t = 0; t < nthr; t++) th.emplace_back(work);
      for (auto& t : th) t.join();
    }
    for (auto& e : errs) if (e) std::rethrow_exception(e);
  }

  // ---- resolve columns by NAME in every file (streams.rs:1024-1037: table schema is
  // sorted by name, files keep write order) ----
  columns.resize(col_names.size());
  for (size_t c = 0; c < col_names.size(); c++) {
    columns[c].name = col_names[c];
    columns[c].kind = 0xff;
  }
  // page-header walk of one column chunk -> DevPage records (runs on worker threads, after the
  // H2D copies were queued, so host parsing overlaps the PCIe transfer)
  struct WalkJob { uint32_t rg; uint32_t col; uint32_t file; std::vector<DevPage> prebuilt; bool compressed = false; };
  std::vector<WalkJob> jobs;
  auto walk_chunk = [](TableChunk& tc, const HostFile& hf, const std::string& colname, uint32_t rg_rows,
                       std::vector<DevPage>& out) {
    const ColumnChunkMeta& cm = *tc.meta;
    const LeafColumn& leaf = hf.meta.leaves[tc.leaf];
        std::vector<PageInfo> pis;
        try {
          pis = walk_pages(hf.data + tc.file_off, tc.bytes, cm.num_values);
        } catch (const std::exception& e) {
          throw Error(PQ_ERR_CORRUPT, colname + ": " + e.what());
        }
        
        uint32_t first_row = 0;
        const uint8_t max_def = uint8_t(leaf.max_def);
        for (const PageInfo& pi : pis) {
          const uint8_t* payload = hf.data + tc.file_off + pi.offset_in_chunk + pi.header_len;
          uint64_t payload_arena = tc.arena_off + pi.offset_in_chunk + pi.header_len;
          if (pi.type == PAGE_DICTIONARY) {
            if (pi.encoding != ENC_PLAIN && pi.encoding != ENC_PLAIN_DICTIONARY)
              throw Error(PQ_ERR_UNSUPPORTED, "dictionary page encoding " + std::to_string(pi.encoding));
            tc.dict_off = payload_arena;
            tc.dict_len = pi.compressed_size;
            tc.dict_n = pi.num_values;
            continue;
          }
          if (pi.type != PAGE_DATA && pi.type != PAGE_DATA_V2) continue;
          DevPage dp{};
          dp.off = payload_arena;
          dp.len = pi.compressed_size;
          dp.num_rows = pi.num_values;
          dp.first_row = first_row;
          first_row += pi.num_values;
          uint32_t pos = 0;
          if (pi.type == PAGE_DATA) {
            if (max_def > 0) {
              if (pi.def_encoding != ENC_RLE) throw Error(PQ_ERR_UNSUPPORTED, "definition levels not RLE encoded");
              if (pi.compressed_size < 4) throw Error(PQ_ERR_CORRUPT, "data page too short");
              uint32_t dl = rd_u32(payload);
              if (uint64_t(dl) + 4 > pi.compressed_size) throw Error(PQ_ERR_CORRUPT, "definition levels run past the page");
              dp.def_off = 4;
              dp.def_len = dl;
              pos = 4 + dl;
            }
          } else {
            if (pi.v2_compressed && cm.codec != CODEC_UNCOMPRESSED) throw Error(PQ_ERR_UNSUPPORTED, "compressed v2 page");
            pos = pi.v2_rep_len;
            if (max_def > 0) { dp.def_off = pos; dp.def_len = pi.v2_def_len; }
            pos += pi.v2_def_len;
          }
          dp.val_off = pos;
          switch (pi.encoding) {
            case ENC_PLAIN:
              dp.enc = DE_PLAIN;
              tc.has_plain_pages = true;
              break;
            case ENC_RLE_DICTIONARY:
            case ENC_PLAIN_DICTIONARY:
              dp.enc = DE_DICT;
              if (pos >= pi.compressed_size && pi.num_values > 0) {
                // an all-null page may legally carry no index bytes
                dp.bit_width = 0;
              } else if (pi.num_values > 0) {
                dp.bit_width = payload[pos];
                dp.val_off = pos + 1;
              }
              if (dp.bit_width > 32) throw Error(PQ_ERR_CORRUPT, "dictionary index bit width > 32");
              tc.has_dict_pages = true;
              tc.max_bw = std::max<uint32_t>(tc.max_bw, dp.bit_width);
              break;
            case ENC_RLE:
              // booleans in v2 data pages: 4-byte length + RLE / bit-packed hybrid, bit width 1
              if (leaf.phys_type != PT_BOOLEAN)
                throw Error(PQ_ERR_UNSUPPORTED, "RLE value encoding on a non-boolean column");
              dp.enc = DE_RLE_BOOL;
              dp.bit_width = 1;
              if (pi.num_values > 0 && pos + 4 <= pi.compressed_size) dp.val_off = pos + 4;
              tc.has_dict_pages = true;  // needs an index window + staging like a dictionary page
              tc.max_bw = std::max<uint32_t>(tc.max_bw, 1);
              break;
            case ENC_DELTA_BINARY_PACKED:
              if (leaf.phys_type != PT_INT64 && !leaf.is_date) throw Error(PQ_ERR_UNSUPPORTED, "column '" + colname + "': DELTA_BINARY_PACKED on a non-INT64 column");
              dp.enc = DE_DELTA;
              tc.has_delta_pages = true;
              break;
            case ENC_DELTA_BYTE_ARRAY:
            case ENC_DELTA_LENGTH_BYTE_ARRAY:
              // front-coded strings (streams.rs:614-619): rewritten as a PLAIN page once the bytes are on the device
              if (leaf.phys_type != PT_BYTE_ARRAY) throw Error(PQ_ERR_UNSUPPORTED, "column '" + colname + "': DELTA_BYTE_ARRAY on a non-BYTE_ARRAY column");
              dp.enc = pi.encoding == ENC_DELTA_BYTE_ARRAY ? DE_DELTA_BYTES : DE_DELTA_LEN_BYTES;
              tc.has_plain_pages = true;
              break;
            default:
              throw Error(PQ_ERR_UNSUPPORTED, "column '" + colname + "': page encoding " + std::to_string(pi.encoding) + " not supported");
          }
          out.push_back(dp);
        }
        
        if (first_row != rg_rows)
          throw Error(PQ_ERR_CORRUPT, colname + ": page rows do not add up to the row group's");
        if (tc.has_dict_pages && leaf.phys_type != PT_BOOLEAN && tc.dict_n == 0 && cm.num_values > 0 &&
            (cm.stats.null_count < 0 || cm.stats.null_count < cm.num_values)) {
          // dictionary-encoded pages without a dictionary page
          throw Error(PQ_ERR_CORRUPT, colname + ": dictionary-encoded pages but no dictionary page");
        }
  };
  struct Copy { uint32_t file; uint64_t src_off; uint64_t dst_off; uint64_t bytes; };
  std::vector<Copy> copies, ccopies;   // -> arena, -> compressed staging buffer
  struct PlainChunk { uint32_t file, rg, col; uint64_t file_off; };
  std::vector<PlainChunk> plain_chunks;   // uncompressed chunks waiting for their place in the arena
  std::vector<DecompJob> djobs;
  uint64_t comp = 0;
  uint64_t arena = 0;
  uint64_t global_row = 0;
  uint64_t global_rg = 0;
  for (uint32_t fi = 0; fi < files.size(); fi++) {
    HostFile& hf = *files[fi];
    std::vector<int> leaf_of(col_names.size(), -1);
    for (size_t c = 0; c < col_names.size(); c++) {
      int li = hf.meta.find_leaf(col_names[c]);
      if (li < 0) {
        // a nested column referenced by its top-level name is not a flat leaf
        for (auto& l : hf.meta.leaves)
          if (l.name.compare(0, col_names[c].size() + 1, col_names[c] + ".") == 0)
            throw Error(PQ_ERR_UNSUPPORTED, "column '" + col_names[c] + "' is nested (list/struct); only flat columns are on the GPU path");
        continue;  // missing in this file: reads as all-NULL (schema adapter behaviour, SURVEY §8 a10)
      }
      const LeafColumn& l = hf.meta.leaves[li];
      if (l.max_rep != 0 || l.depth != 1 || l.max_def > 1)
        throw Error(PQ_ERR_UNSUPPORTED, "column '" + col_names[c] + "' is nested; only flat columns are on the GPU path");
      uint8_t k = kind_of_leaf(l);
      if (k == 0xff || (k == DK_I32 && !l.is_date) || k == DK_F32)
        throw Error(PQ_ERR_UNSUPPORTED, "column '" + col_names[c] + "': physical type " + std::to_string(l.phys_type) + " not supported");
      // Date32: INT32 days, widened to the flat store's sign-extended 8-byte values when the table is opened
      // (build_flat_store, ensure_plain8), so that every kernel past the flat store sees an Int64 column
      if (k == DK_I32) k = DK_I64;
      if (columns[c].kind == 0xff) {
        columns[c].kind = k;
        columns[c].is_ts = l.is_timestamp_ms;
        columns[c].is_date = l.is_date;
      } else if (columns[c].kind != k || columns[c].is_date != l.is_date) {
        throw Error(PQ_ERR_UNSUPPORTED, "column '" + col_names[c] + "' changes physical type across files");
      }
      if (l.is_timestamp_other)
        throw Error(PQ_ERR_UNSUPPORTED, "column '" + col_names[c] + "': only Timestamp(ms) is supported");
      columns[c].max_def = std::max<uint8_t>(columns[c].max_def, uint8_t(l.max_def));
      leaf_of[c] = li;
    }
    for (uint32_t gi = 0; gi < hf.meta.row_groups.size(); gi++, global_rg++) {
      const RowGroupMeta& g = hf.meta.row_groups[gi];
      uint64_t row0 = global_row;
      global_row += uint64_t(g.num_rows);
      list_rows = global_row;
      if (global_rg % shard_count != shard_index) continue;
      if (g.num_rows == 0) continue;
      TableRowGroup trg;
      trg.file = fi;
      trg.rg_in_file = gi;
      trg.num_rows = uint32_t(g.num_rows);
      trg.global_row0 = row0;
      trg.chunks.resize(col_names.size());
      for (size_t c = 0; c < col_names.size(); c++) {
        TableChunk& tc = trg.chunks[c];
        if (leaf_of[c] < 0) continue;
        const ColumnChunkMeta& cm = g.columns[leaf_of[c]];
        const bool compressed = cm.codec != CODEC_UNCOMPRESSED;
        if (compressed && cm.codec != CODEC_LZ4_RAW && cm.codec != CODEC_SNAPPY && cm.codec != CODEC_ZSTD && cm.codec != CODEC_GZIP)
          throw Error(PQ_ERR_UNSUPPORTED, "column '" + col_names[c] + "': page compression codec " + std::to_string(cm.codec) +
                                              " is not decoded on the GPU (LZ4_RAW, SNAPPY, ZSTD, GZIP and UNCOMPRESSED are)");
        tc.present = true;
        tc.leaf = leaf_of[c];
        tc.meta = &cm;
        tc.file_off = uint64_t(cm.start());
        tc.bytes = uint64_t(cm.total_compressed_size);
        if (tc.file_off + tc.bytes > hf.size) throw Error(PQ_ERR_CORRUPT, "column chunk outside the file");
        chunk_bytes += tc.bytes;
        if (compressed) {
          // the chunk's bytes go to a staging buffer; every page is decoded into its own arena slot
          const uint64_t coff = comp + ((uintptr_t(hf.data) + tc.file_off) & 15);
          comp = (coff + tc.bytes + 255) & ~255ull;
          ccopies.push_back({fi, tc.file_off, coff, tc.bytes});
          std::vector<PageInfo> pis;
          try { pis = walk_pages(hf.data + tc.file_off, tc.bytes, cm.num_values); }
          catch (const std::exception& e) { throw Error(PQ_ERR_CORRUPT, col_names[c] + ": " + e.what()); }
          WalkJob wj{uint32_t(row_groups.size()), uint32_t(c), fi, {}, true};
          const LeafColumn& leaf = hf.meta.leaves[leaf_of[c]];
          uint32_t first_row = 0;
          tc.arena_off = arena;
          for (const PageInfo& pi : pis) {
            const uint64_t slot = (arena + 15) & ~15ull;
            arena = slot + pi.uncompressed_size + 16;
            uint64_t v2_levels = 0;
            if (pi.type == PAGE_DICTIONARY) {
              tc.dict_off = slot; tc.dict_len = pi.uncompressed_size; tc.dict_n = pi.num_values;
            } else if (pi.type == PAGE_DATA || pi.type == PAGE_DATA_V2) {
              DevPage dp{};
              dp.off = slot; dp.len = pi.uncompressed_size; dp.num_rows = pi.num_values; dp.first_row = first_row;
              first_row += pi.num_values;
              if (pi.type == PAGE_DATA) dp.def_len = leaf.max_def > 0 ? 0xffffffffu : 0;   // resolved by k_page_fixup from the decoded bytes
              else {
                // v2: the level bytes sit in front of the values, never compressed, their lengths in the header
                v2_levels = uint64_t(pi.v2_rep_len) + pi.v2_def_len;
                if (v2_levels > pi.compressed_size || v2_levels > pi.uncompressed_size) throw Error(PQ_ERR_CORRUPT, col_names[c] + ": v2 level bytes run past the page");
                if (leaf.max_def > 0) { dp.def_off = pi.v2_rep_len; dp.def_len = pi.v2_def_len; }
                dp.val_off = uint32_t(v2_levels);
              }
              switch (pi.encoding) {
                case ENC_PLAIN: dp.enc = DE_PLAIN; tc.has_plain_pages = true; break;
                case ENC_RLE_DICTIONARY: case ENC_PLAIN_DICTIONARY: dp.enc = DE_DICT; tc.has_dict_pages = true; break;
                case ENC_DELTA_BINARY_PACKED:
                  if (leaf.phys_type != PT_INT64 && !leaf.is_date) throw Error(PQ_ERR_UNSUPPORTED, "column '" + col_names[c] + "': DELTA_BINARY_PACKED on a non-INT64 column");
                  dp.enc = DE_DELTA; tc.has_delta_pages = true; break;
                case ENC_DELTA_BYTE_ARRAY: case ENC_DELTA_LENGTH_BYTE_ARRAY:
                  if (leaf.phys_type != PT_BYTE_ARRAY) throw Error(PQ_ERR_UNSUPPORTED, "column '" + col_names[c] + "': DELTA_BYTE_ARRAY on a non-BYTE_ARRAY column");
                  dp.enc = pi.encoding == ENC_DELTA_BYTE_ARRAY ? DE_DELTA_BYTES : DE_DELTA_LEN_BYTES; tc.has_plain_pages = true; break;
                case ENC_RLE:
                  if (leaf.phys_type != PT_BOOLEAN) throw Error(PQ_ERR_UNSUPPORTED, "RLE value encoding on a non-boolean column");
                  dp.enc = DE_RLE_BOOL; tc.has_dict_pages = true; break;
                default: throw Error(PQ_ERR_UNSUPPORTED, "column '" + col_names[c] + "': page encoding " + std::to_string(pi.encoding) + " not supported");
              }
              wj.prebuilt.push_back(dp);
            } else continue;
            const uint64_t src = coff + pi.offset_in_chunk + pi.header_len;
            if (pi.type == PAGE_DATA_V2) {
              const uint32_t lv = uint32_t(v2_levels);
              if (lv) djobs.push_back({src, slot, lv, lv, 0u, 0});                                     // levels: stored
              djobs.push_back({src + lv, slot + lv, pi.compressed_size - lv, pi.uncompressed_size - lv,    // values: compressed unless the header says not
                               pi.v2_compressed ? uint32_t(cm.codec) : 0u, 0});
            } else {
              djobs.push_back({src, slot, pi.compressed_size, pi.uncompressed_size, uint32_t(cm.codec), 0});
            }
          }
          if (first_row != trg.num_rows) throw Error(PQ_ERR_CORRUPT, col_names[c] + ": page rows do not add up to the row group's");
          arena = (arena + 64 + 255) & ~255ull;
          jobs.push_back(std::move(wj));
          continue;
        }
        plain_chunks.push_back({fi, uint32_t(row_groups.size()), uint32_t(c), tc.file_off});   // placed below, in file order
        jobs.push_back({uint32_t(row_groups.size()), uint32_t(c), fi, {}, false});
      }
      total_rows += trg.num_rows;
      row_groups.push_back(std::move(trg));
    }
  }
  for (size_t c = 0; c < columns.size(); c++)
    if (columns[c].kind == 0xff) columns[c].kind = 0xfe;  // present in no file: all NULL everywhere

  // ---- arena places of the uncompressed chunks: in FILE order, neighbours that are close in the file keep their
  // distance, so that one copy moves the whole span (and the unreferenced bytes in a small gap): a query over most
  // columns uploads a file in one DMA transfer (53.9 GB/s measured on this box against 47 GB/s for the gather
  // kernel's SM-issued reads); a span starts 256-byte aligned at the 16-byte phase of its source ----
  {
    std::sort(plain_chunks.begin(), plain_chunks.end(), [](const PlainChunk& a, const PlainChunk& b) {
      return a.file != b.file ? a.file < b.file : a.file_off < b.file_off;
    });
    const uint64_t kGap = 128u << 10;
    uint64_t span_src = 0, span_dst = 0, span_end = 0;   // of the open span (source offsets inside its file)
    uint32_t span_file = ~0u;
    auto close_span = [&]() {
      if (span_file == ~0u) return;
      copies.push_back({span_file, span_src, span_dst, span_end - span_src});
      arena = (span_dst + (span_end - span_src) + 64 + 255) & ~255ull;
    };
    for (const PlainChunk& pc : plain_chunks) {
      TableChunk& tc = row_groups[pc.rg].chunks[pc.col];
      if (pc.file != span_file || (tc.file_off > span_end && tc.file_off - span_end > kGap)) {
        close_span();
        span_file = pc.file;
        span_src = span_end = tc.file_off;
        span_dst = arena + ((uintptr_t(files[pc.file]->data) + tc.file_off) & 15);
      }
      tc.arena_off = span_dst + (tc.file_off - span_src);
      span_end = std::max(span_end, tc.file_off + tc.bytes);
    }
    close_span();
  }

  mark("footers parsed, chunks planned");
  // ---- one HBM arena, 64 KiB of slack so staged windows may over-read ----
  arena_bytes = arena + (64u << 10);
  PQB_CUDA(cudaMallocAsync((void**)&d_arena, arena_bytes, stream));
  // tail slack must be defined (walkers may look at it)
  PQB_CUDA(cudaMemsetAsync(d_arena + arena, 0, arena_bytes - arena, stream));
  UnwindGuard unwind(stream);   // an error below: wait for the copies in flight, free the temporaries
  uint8_t* d_comp = nullptr;   // compressed chunks wait here for k_decompress_pages
  unwind.own(d_comp);
  if (comp) PQB_CUDA(cudaMallocAsync((void**)&d_comp, comp + 256, stream));

  // ---- upload: straight from pinned caller buffers, else staged through pinned memory ----
  auto upload_to = [&](const std::vector<Copy>& copies, uint8_t* d_arena) {
  std::vector<Copy> staged;
  std::vector<size_t> staged_orig;
  std::vector<char> file_pinned(files.size(), 0);
  for (size_t f = 0; f < files.size(); f++) file_pinned[f] = !files[f]->mapped && ctx.is_pinned(files[f]->data);
  // page-locked file images: ONE gather kernel pulls every chunk over PCIe (the SMs read the
  // mapped host memory directly) instead of hundreds of cudaMemcpyAsync calls
  std::vector<GatherCopy> gathers;
  std::vector<const uint8_t*> file_dev(files.size(), nullptr);  // device-visible alias of a page-locked image
  const char* upl = getenv("PQB_UPLOAD");   // experiment switch: "memcpy" = one cudaMemcpyAsync per chunk (copy engines) instead of the gather kernel
  const bool use_gather = !(upl && upl[0] == 'm');
  const uint64_t kDmaMin = (upl && upl[0] == 'g') ? ~0ull : (2ull << 20);   // "gather": every span through the gather kernel (A/B)
  for (size_t f = 0; f < files.size(); f++) {
    if (!file_pinned[f] || !use_gather) continue;
    void* dp = nullptr;
    if (cudaHostGetDevicePointer(&dp, const_cast<uint8_t*>(files[f]->data), 0) == cudaSuccess && dp &&
        ((uintptr_t(dp) ^ uintptr_t(files[f]->data)) & 15) == 0)
      file_dev[f] = static_cast<const uint8_t*>(dp);
    else cudaGetLastError();
  }
  for (size_t k = 0; k < copies.size(); k++) {
    const Copy& cp = copies[k];
    const HostFile& hf = *files[cp.file];
    if (file_pinned[cp.file]) {
      // long spans: the copy engines (large PCIe reads); many short ones: one gather kernel (no per-copy launch cost)
      if (file_dev[cp.file] && cp.bytes < kDmaMin) {
        // pieces of 128 KiB (whole 16-byte vectors of the span's phase): the grid stays thousands of CTAs whatever the span sizes
        const uint64_t kPiece = 128u << 10;
        for (uint64_t o = 0; o < cp.bytes; o += kPiece)
          gathers.push_back({file_dev[cp.file] + cp.src_off + o, cp.dst_off + o, std::min<uint64_t>(kPiece, cp.bytes - o)});
      }
      else PQB_CUDA(cudaMemcpyAsync(d_arena + cp.dst_off, hf.data + cp.src_off, cp.bytes, cudaMemcpyHostToDevice, stream));
    } else {
      // pieces of at most 8 MiB: the staging threads below share the work copy by copy
      const uint64_t kPiece = 8ull << 20;
      for (uint64_t o = 0; o < cp.bytes; o += kPiece) {
        staged.push_back({cp.file, cp.src_off + o, cp.dst_off + o, std::min<uint64_t>(kPiece, cp.bytes - o)});
        staged_orig.push_back(k);
      }
    }
    h2d_bytes += cp.bytes;
  }
  GatherCopy* d_gathers = nullptr;
  if (!gathers.empty()) {
    PQB_CUDA(cudaMallocAsync((void**)&d_gathers, gathers.size() * sizeof(GatherCopy), stream));
    PQB_CUDA(cudaMemcpyAsync(d_gathers, gathers.data(), gathers.size() * sizeof(GatherCopy), cudaMemcpyHostToDevice, stream));
    // ~64 KiB per CTA pass keeps a few thousand 16-byte reads in flight per SM
    dim3 grid(uint32_t(gathers.size()), 4);
    k_gather_copy<<<grid, 256, 0, stream>>>(d_gathers, d_arena);
    PQB_CUDA(cudaGetLastError());
    dev_drop(d_gathers, stream);
  }
  if (!staged.empty()) {
    // gather into pinned staging slices with a few host threads, one cudaMemcpyAsync per slice;
    // three rotating slices bound the pinned footprint
    const size_t kSlice = 32u << 20;
    const int kRing = 3;
    unsigned nthr = std::min<unsigned>(8, std::max<unsigned>(1, std::thread::hardware_concurrency()));
    size_t i = 0;
    uint8_t* ring[kRing] = {nullptr, nullptr, nullptr};
    size_t ring_cap[kRing] = {0, 0, 0};
    cudaEvent_t ring_ev[kRing];
    for (int r = 0; r < kRing; r++) PQB_CUDA(cudaEventCreateWithFlags(&ring_ev[r], cudaEventDisableTiming));
    int slot = 0;
    while (i < staged.size()) {
      // pack copies that were adjacent in the arena (nothing else lives in the gaps) into one slice
      size_t j = i;
      uint64_t lo = staged[i].dst_off, hi = lo;
      while (j < staged.size() && staged[j].dst_off + staged[j].bytes - lo <= kSlice &&
             (j == i || staged_orig[j] - staged_orig[j - 1] <= 1)) {
        hi = staged[j].dst_off + staged[j].bytes;
        j++;
      }
      if (j == i) { hi = staged[i].dst_off + staged[i].bytes; j = i + 1; }
      const int r = slot % kRing;
      slot++;
      if (ring[r]) PQB_CUDA(cudaEventSynchronize(ring_ev[r]));
      if (ring_cap[r] < size_t(hi - lo)) {
        if (ring[r]) ctx.pinned_release(ring[r]);
        ring[r] = ctx.pinned_acquire(std::max<size_t>(size_t(hi - lo), kSlice));
        ring_cap[r] = std::max<size_t>(size_t(hi - lo), kSlice);
      }
      uint8_t* buf = ring[r];
      std::atomic<size_t> next{i};
      auto work = [&]() {
        for (;;) {
          size_t k = next.fetch_add(1);
          if (k >= j) break;
          const Copy& cp = staged[k];
          std::memcpy(buf + (cp.dst_off - lo), files[cp.file]->data + cp.src_off, cp.bytes);
        }
      };
      unsigned use = unsigned(std::min<size_t>(nthr, j - i));
      if (use <= 1) work();
      else {
        std::vector<std::thread> th;
        for (unsigned t = 0; t < use; t++) th.emplace_back(work);
        for (auto& t : th) t.join();
      }
      // gaps between chunks inside the slice are alignment padding: harmless to overwrite
      PQB_CUDA(cudaMemcpyAsync(d_arena + lo, buf, size_t(hi - lo), cudaMemcpyHostToDevice, stream));
      PQB_CUDA(cudaEventRecord(ring_ev[r], stream));
      i = j;
    }
    PQB_CUDA(cudaStreamSynchronize(stream));
    for (int r = 0; r < kRing; r++) {
      if (ring[r]) ctx.pinned_release(ring[r]);
      cudaEventDestroy(ring_ev[r]);
    }
  }
  };
  upload_to(copies, d_arena);
  if (!ccopies.empty()) upload_to(ccopies, d_comp);
  mark("uploads queued (synchronised for this mark)");
  DecompJob* d_djobs = nullptr;
  unsigned long long* d_dflag = nullptr;
  HeavyWs* d_zws = nullptr;
  unsigned int* d_znext = nullptr;
  unwind.own(d_djobs);
  unwind.own(d_dflag);
  unwind.own(d_zws);
  unwind.own(d_znext);
  if (!djobs.empty()) {
    PQB_CUDA(cudaMallocAsync((void**)&d_dflag, 8, stream));
    PQB_CUDA(cudaMemsetAsync(d_dflag, 0, 8, stream));
    PQB_CUDA(launch_decompress(djobs, d_comp, d_arena, d_dflag, ctx.sm_count(), stream, &d_djobs, &d_zws, &d_znext));
  }
  // ---- page walks, in parallel, while the copies above are in flight ----
  {
    std::vector<std::vector<DevPage>> out(jobs.size());
    std::vector<std::exception_ptr> errs(jobs.size());
    std::atomic<size_t> next{0};
    auto work = [&]() {
      for (;;) {
        size_t j = next.fetch_add(1);
        if (j >= jobs.size()) break;
        const WalkJob& jb = jobs[j];
        if (jb.compressed) { out[j] = jb.prebuilt; continue; }
        try {
          walk_chunk(row_groups[jb.rg].chunks[jb.col], *files[jb.file], col_names[jb.col], row_groups[jb.rg].num_rows, out[j]);
        } catch (...) { errs[j] = std::current_exception(); }
      }
    };
    const unsigned nthr = unsigned(std::min<size_t>({size_t(8), size_t(std::max(1u, std::thread::hardware_concurrency())), jobs.size() / 64 + 1}));
    if (nthr <= 1) work();
    else {
      std::vector<std::thread> th;
      for (unsigned t = 0; t < nthr; t++) th.emplace_back(work);
      for (auto& t : th) t.join();
    }
    for (auto& e : errs) if (e) std::rethrow_exception(e);
    size_t total = 0;
    for (auto& v : out) total += v.size();
    pages.reserve(total);
    for (size_t j = 0; j < jobs.size(); j++) {
      TableChunk& tc = row_groups[jobs[j].rg].chunks[jobs[j].col];
      tc.pages.first_page = uint32_t(pages.size());
      tc.pages.n_pages = uint32_t(out[j].size());
      for (DevPage& dp : out[j]) dp.chunk_slot = uint16_t(jobs[j].col);
      pages.insert(pages.end(), out[j].begin(), out[j].end());
    }
  }
  mark("page headers walked");
  if (!pages.empty()) {
    PQB_CUDA(cudaMallocAsync((void**)&d_pages, pages.size() * sizeof(DevPage), stream));
    PQB_CUDA(cudaMemcpyAsync(d_pages, pages.data(), pages.size() * sizeof(DevPage), cudaMemcpyHostToDevice, stream));
  }
  if (!djobs.empty()) {
    // decoded pages: fetch the two bytes the host normally reads from the file (def-level length, index bit width)
    std::vector<uint32_t> fix;
    for (size_t j = 0; j < jobs.size(); j++)
      if (jobs[j].compressed) {
        const TableChunk& tc = row_groups[jobs[j].rg].chunks[jobs[j].col];
        for (uint32_t k = 0; k < tc.pages.n_pages; k++) fix.push_back(tc.pages.first_page + k);
      }
    if (!fix.empty()) {
      uint32_t* d_fix = nullptr;
      PQB_CUDA(cudaMallocAsync((void**)&d_fix, fix.size() * 4, stream));
      PQB_CUDA(cudaMemcpyAsync(d_fix, fix.data(), fix.size() * 4, cudaMemcpyHostToDevice, stream));
      k_page_fixup<<<uint32_t((fix.size() + 127) / 128), 128, 0, stream>>>(d_pages, d_fix, uint32_t(fix.size()), d_arena, d_dflag);
      PQB_CUDA(cudaGetLastError());
      PQB_CUDA(cudaMemcpyAsync(pages.data(), d_pages, pages.size() * sizeof(DevPage), cudaMemcpyDeviceToHost, stream));
      dev_drop(d_fix, stream);
    }
    unsigned long long flag = 0;
    PQB_CUDA(cudaMemcpyAsync(&flag, d_dflag, 8, cudaMemcpyDeviceToHost, stream));
    PQB_CUDA(cudaStreamSynchronize(stream));
    dev_drop(d_djobs, stream);
    dev_drop(d_dflag, stream);
    dev_drop(d_zws, stream);
    dev_drop(d_znext, stream);
    dev_drop(d_comp, stream);
    if (flag) throw Error(PQ_ERR_CORRUPT, "a compressed page did not decode to its declared size (LZ4_RAW / SNAPPY / ZSTD / GZIP)");
    for (size_t j = 0; j < jobs.size(); j++)
      if (jobs[j].compressed) {
        TableChunk& tc = row_groups[jobs[j].rg].chunks[jobs[j].col];
        for (uint32_t k = 0; k < tc.pages.n_pages; k++) {
          const DevPage& dp = pages[tc.pages.first_page + k];
          if (dp.enc == DE_DICT || dp.enc == DE_RLE_BOOL) {
            if (dp.bit_width > 32) throw Error(PQ_ERR_CORRUPT, "dictionary index bit width > 32");
            tc.max_bw = std::max<uint32_t>(tc.max_bw, dp.bit_width);
          }
        }
      }
  }
  // ---- DELTA_BYTE_ARRAY / DELTA_LENGTH_BYTE_ARRAY pages -> PLAIN BYTE_ARRAY pages (device side, two passes) ----
  {
    std::vector<DbaJob> dj;
    uint64_t tmp = 0;
    for (size_t i = 0; i < pages.size(); i++)
      if (pages[i].enc == DE_DELTA_BYTES || pages[i].enc == DE_DELTA_LEN_BYTES) {
        dj.push_back({uint32_t(i), pages[i].enc == DE_DELTA_BYTES ? 1u : 0u, tmp, 0});
        tmp += (uint64_t(pages[i].num_rows) * 8 + 15) & ~15ull;
      }
    if (!dj.empty()) {
      DbaJob* d_jobs = nullptr;
      DbaInfo* d_info = nullptr;
      uint8_t* d_tmp = nullptr;
      UnwindGuard tmp_guard(stream);
      tmp_guard.own(d_jobs); tmp_guard.own(d_info); tmp_guard.own(d_tmp);
      PQB_CUDA(cudaMallocAsync((void**)&d_jobs, dj.size() * sizeof(DbaJob), stream));
      PQB_CUDA(cudaMallocAsync((void**)&d_info, dj.size() * sizeof(DbaInfo), stream));
      PQB_CUDA(cudaMallocAsync((void**)&d_tmp, tmp + 16, stream));
      PQB_CUDA(cudaMemcpyAsync(d_jobs, dj.data(), dj.size() * sizeof(DbaJob), cudaMemcpyHostToDevice, stream));
      launch_dba_lengths(d_arena, d_pages, d_jobs, uint32_t(dj.size()), d_tmp, d_info, stream);
      std::vector<DbaInfo> info(dj.size());
      PQB_CUDA(cudaMemcpyAsync(info.data(), d_info, info.size() * sizeof(DbaInfo), cudaMemcpyDeviceToHost, stream));
      PQB_CUDA(cudaStreamSynchronize(stream));
      uint64_t total = 0;
      bool bad = false;
      for (size_t j = 0; j < dj.size(); j++) {
        const DevPage& pg = pages[dj[j].page];
        if (!info[j].ok || uint64_t(pg.def_len) + info[j].bytes > 0xfffffff0ull) { bad = true; break; }
        dj[j].dst = total;
        total = (total + pg.def_len + info[j].bytes + 16 + 15) & ~15ull;
      }
      if (!bad) {
        // staged windows and the row walker over-read like they do in the arena: same slack
        PQB_CUDA(cudaMallocAsync((void**)&d_strmat, total + (64u << 10), stream));
        PQB_CUDA(cudaMemsetAsync(d_strmat + total, 0, 64u << 10, stream));
        PQB_CUDA(cudaMemcpyAsync(d_jobs, dj.data(), dj.size() * sizeof(DbaJob), cudaMemcpyHostToDevice, stream));
        launch_dba_materialise(d_arena, d_pages, d_jobs, d_info, uint32_t(dj.size()), d_tmp, d_strmat, stream);
        for (size_t j = 0; j < dj.size(); j++) {
          DevPage& pg = pages[dj[j].page];
          // the new payload lives outside the arena: offsets are relative to the arena base modulo 2^64
          pg.off = uint64_t(reinterpret_cast<uintptr_t>(d_strmat) + dj[j].dst - reinterpret_cast<uintptr_t>(d_arena));
          pg.def_off = 0;
          pg.val_off = pg.def_len;
          pg.len = uint32_t(pg.def_len + info[j].bytes);
          pg.enc = DE_PLAIN;
        }
        PQB_CUDA(cudaMemcpyAsync(d_pages, pages.data(), pages.size() * sizeof(DevPage), cudaMemcpyHostToDevice, stream));
      }
      PQB_CUDA(cudaStreamSynchronize(stream));
      dev_drop(d_jobs, stream);
      dev_drop(d_info, stream);
      dev_drop(d_tmp, stream);
      if (bad) throw Error(PQ_ERR_CORRUPT, "a DELTA_BYTE_ARRAY page does not decode (length streams / prefixes out of range)");
    }
  }
  // row groups whose columns all share their page boundaries: work items are simply the pages
  for (TableRowGroup& rg : row_groups) {
    const TableChunk* first = nullptr;
    bool same = true;
    for (const TableChunk& tc : rg.chunks) {
      if (!tc.present) continue;
      if (!first) { first = &tc; continue; }
      if (tc.pages.n_pages != first->pages.n_pages) { same = false; break; }
      for (uint32_t k = 0; k < tc.pages.n_pages && same; k++)
        same = pages[tc.pages.first_page + k].first_row == pages[first->pages.first_page + k].first_row;
      if (!same) break;
    }
    rg.pages_aligned = same && first != nullptr;
  }
  // ---- per-column entry numbering (query independent): entries of the column in earlier row groups ----
  sides.assign(columns.size(), ColSide{});
  for (size_t c = 0; c < columns.size(); c++) {
    ColSide& cs = sides[c];
    cs.base_per_rg.resize(row_groups.size());
    uint64_t tot = 0;
    for (size_t g = 0; g < row_groups.size(); g++) {
      cs.base_per_rg[g] = uint32_t(tot);
      const TableChunk& tc = row_groups[g].chunks[c];
      if (tc.present) { tot += tc.dict_n; cs.max_dict_n = std::max(cs.max_dict_n, tc.dict_n); cs.has_delta |= tc.has_delta_pages; }
      if (tot > 0xfffffff0ull) throw Error(PQ_ERR_UNSUPPORTED, "too many dictionary entries in column '" + columns[c].name + "'");
    }
    cs.total_entries = uint32_t(tot);
  }
  mark("before flat store");
  build_flat_store(stream);
  PQB_CUDA(cudaStreamSynchronize(stream));
  mark("flat store built");
}

// ---- flat store ----------------------------------------------------------------------------------
void Table::build_flat_store(cudaStream_t stream) {
  FlatPageRec blank{};
  blank.voff = ~0ull;
  flat_pages.assign(pages.size(), blank);
  if (pages.empty()) return;
  // which pages hold NULLs (their definition levels are not all 1)?
  // A chunk whose footer promises null_count == 0 (or whose column cannot hold NULLs: no definition levels) needs no
  // look at the data: when that settles every page, nothing below waits for the upload -- the jobs are built and the
  // flat store is allocated while the DMA is still in flight, and the kernels queue up behind it.  (Statistics that lie
  // make the value stream of such a page come up short: the file is refused as malformed.)
  std::vector<uint8_t> has_nulls(pages.size(), 0);
  bool need_look = false;
  for (const TableRowGroup& rg : row_groups)
    for (const TableChunk& tc : rg.chunks)
      if (tc.present && tc.meta->stats.null_count != 0)
        for (uint32_t k = 0; k < tc.pages.n_pages && !need_look; k++) need_look = pages[tc.pages.first_page + k].def_len != 0;
  if (need_look) {
    uint8_t* d_nf = nullptr;
    PQB_CUDA(cudaMallocAsync((void**)&d_nf, pages.size(), stream));
    launch_page_has_nulls(d_arena, d_pages, uint32_t(pages.size()), d_nf, stream);
    PQB_CUDA(cudaMemcpyAsync(has_nulls.data(), d_nf, pages.size(), cudaMemcpyDeviceToHost, stream));
    PQB_CUDA(cudaStreamSynchronize(stream));
    dev_drop(d_nf, stream);
  }
  struct J { uint64_t src, off, voff, toff; uint32_t page, kind, rows, zone; };
  std::vector<J> js;
  // zone 0: zeroed (hybrid outputs and validity bitmaps are merged into it with atomicOr); zone 1: plain copies;
  // zone 2: zeroed scratch for the dense values of index pages with NULLs
  uint64_t zoff[3] = {0, 0, 0};
  auto take = [&](int zone, uint64_t bytes) { uint64_t o = zoff[zone]; zoff[zone] = (zoff[zone] + bytes + 16 + 15) & ~15ull; return o; };
  const uint64_t kNone = ~0ull;
  for (TableRowGroup& rg : row_groups)
    for (size_t c = 0; c < rg.chunks.size(); c++) {
      TableChunk& tc = rg.chunks[c];
      if (!tc.present) continue;
      const uint8_t kind = columns[c].kind;
      const bool wide4 = columns[c].is_date;   // INT32 values: widened (sign-extended) to 8 bytes
      if (tc.dict_n && (kind == DK_I64 || kind == DK_F64)) {
        if (uint64_t(tc.dict_n) * (wide4 ? 4 : 8) > tc.dict_len)
          throw Error(PQ_ERR_CORRUPT, "column '" + columns[c].name + "': dictionary page shorter than its entry count");
        js.push_back({tc.dict_off, take(1, uint64_t(tc.dict_n) * 8), kNone, kNone, 0u, wide4 ? 7u /*FJ_DICT4*/ : 4u /*FJ_DICT8*/, tc.dict_n, 1u});
        tc.dict8_off = js.size() - 1;   // job index for now, resolved below
      }
      for (uint32_t k = 0; k < tc.pages.n_pages; k++) {
        const uint32_t pi = tc.pages.first_page + k;
        const DevPage& pg = pages[pi];
        FlatPageRec& fr = flat_pages[pi];
        fr.rows = pg.num_rows;
        const bool nul = has_nulls[pi] != 0;
        const uint64_t vbytes = (uint64_t(pg.num_rows) + 31) / 32 * 4;
        if (pg.enc == DE_DICT || pg.enc == DE_RLE_BOOL) {
          fr.fkind = pg.enc == DE_DICT ? FK_INDEX : FK_BITS;
          fr.bw = pg.bit_width;
          const uint64_t nb = (uint64_t(pg.num_rows) * pg.bit_width + 7) / 8;
          J j{0, take(0, nb), kNone, kNone, pi, 1u /*FJ_HYBRID*/, pg.num_rows, 0u};
          if (nul) { j.voff = take(0, vbytes); j.toff = take(2, nb); }
          js.push_back(j);
        } else if (pg.enc == DE_PLAIN && (kind == DK_I64 || kind == DK_F64)) {
          fr.fkind = FK_PLAIN8;
          fr.bw = 64;
          J j{0, take(1, uint64_t(pg.num_rows) * 8), kNone, kNone, pi, wide4 ? 8u /*FJ_WIDEN4*/ : 2u /*FJ_COPY8*/, pg.num_rows, 1u};
          if (nul) j.voff = take(0, vbytes);
          js.push_back(j);
        } else if (pg.enc == DE_PLAIN && kind == DK_BOOL) {
          fr.fkind = FK_BITS;
          fr.bw = 1;
          J j{0, take(1, vbytes), kNone, kNone, pi, 3u /*FJ_BITS*/, pg.num_rows, 1u};
          if (nul) j.voff = take(0, vbytes);
          js.push_back(j);
        } else if (pg.enc == DE_PLAIN && kind == DK_STR) {
          // dictionary-fallback strings: one u32 per row = where its bytes start inside the page
          fr.fkind = FK_BYTES;
          fr.bw = 32;
          fr.base = pg.off + pg.val_off;
          J j{0, take(1, uint64_t(pg.num_rows) * 4), kNone, kNone, pi, 6u /*FJ_BYTES*/, pg.num_rows, 1u};
          if (nul) j.voff = take(0, vbytes);
          js.push_back(j);
        } else if (pg.enc == DE_DELTA && nul) {
          // values on demand (ensure_plain8); the validity bitmap is built now
          js.push_back({0, 0, take(0, vbytes), kNone, pi, 5u /*FJ_VALID*/, pg.num_rows, 0u});
        } else {
          continue;   // DELTA pages without NULLs (decoded on demand), PLAIN strings: k_scan
        }
      }
    }
  if (js.empty()) return;
  const uint64_t zone1 = (zoff[0] + 255) & ~255ull;
  const uint64_t zone2 = (zone1 + zoff[1] + 255) & ~255ull;
  flat_bytes = zone2 + zoff[2] + 256;
  PQB_CUDA(cudaMallocAsync((void**)&d_flat, flat_bytes, stream));
  PQB_CUDA(cudaMemsetAsync(d_flat, 0, zone1, stream));
  PQB_CUDA(cudaMemsetAsync(d_flat + zone2, 0, zoff[2] + 256, stream));
  struct DevJob { uint64_t src, dst, vdst, tmp; uint32_t page, kind, rows, pad; };   // == FlatStoreJob
  std::vector<DevJob> dj(js.size());
  for (size_t i = 0; i < js.size(); i++) {
    const uint64_t dst = js[i].zone ? zone1 + js[i].off : js[i].off;
    dj[i] = {js[i].src, dst, js[i].voff, js[i].toff == kNone ? kNone : zone2 + js[i].toff, js[i].page, js[i].kind, js[i].rows, 0u};
    if (js[i].kind == 4u || js[i].kind == 7u) continue;
    FlatPageRec& fr = flat_pages[js[i].page];
    fr.voff = js[i].voff;
    if (js[i].kind != 5u) fr.off = dst;
  }
  for (TableRowGroup& rg : row_groups)
    for (size_t c = 0; c < rg.chunks.size(); c++) {
      TableChunk& tc = rg.chunks[c];
      if (!tc.present || tc.dict8_off == ~0ull) continue;
      tc.dict8_off = dj[tc.dict8_off].dst;
      if (columns[c].is_date) {
        // the readers of raw dictionary entries (entry offsets for key interning, the leaf LUTs) take 8-byte entries:
        // a Date32 chunk's dictionary is its widened copy from here on (an arena offset that wraps, like d_strmat's pages)
        tc.dict_off = uint64_t(reinterpret_cast<uintptr_t>(d_flat) + tc.dict8_off - reinterpret_cast<uintptr_t>(d_arena));
        tc.dict_len = tc.dict_n * 8;
      }
    }
  void* d_jobs = nullptr;
  uint8_t* d_ok = nullptr;
  uint32_t* d_maxlen = nullptr;
  UnwindGuard tmp_guard(stream);
  tmp_guard.own(d_jobs); tmp_guard.own(d_ok); tmp_guard.own(d_maxlen);
  bool any_bytes = false;
  for (const DevJob& j : dj) any_bytes |= j.kind == 6u;
  PQB_CUDA(cudaMallocAsync(&d_jobs, dj.size() * sizeof(DevJob), stream));
  PQB_CUDA(cudaMallocAsync((void**)&d_ok, dj.size(), stream));
  if (any_bytes) {
    PQB_CUDA(cudaMallocAsync((void**)&d_maxlen, dj.size() * 4, stream));
    PQB_CUDA(cudaMemsetAsync(d_maxlen, 0, dj.size() * 4, stream));
  }
  PQB_CUDA(cudaMemcpyAsync(d_jobs, dj.data(), dj.size() * sizeof(DevJob), cudaMemcpyHostToDevice, stream));
  launch_flat_store(d_arena, d_pages, d_jobs, uint32_t(dj.size()), d_flat, d_ok, d_maxlen, stream);
  std::vector<uint8_t> ok(dj.size());
  std::vector<uint32_t> maxlen(any_bytes ? dj.size() : 0);
  PQB_CUDA(cudaMemcpyAsync(ok.data(), d_ok, ok.size(), cudaMemcpyDeviceToHost, stream));
  if (any_bytes) PQB_CUDA(cudaMemcpyAsync(maxlen.data(), d_maxlen, maxlen.size() * 4, cudaMemcpyDeviceToHost, stream));
  PQB_CUDA(cudaStreamSynchronize(stream));
  dev_drop(d_jobs, stream);
  dev_drop(d_ok, stream);
  dev_drop(d_maxlen, stream);
  for (size_t i = 0; i < maxlen.size(); i++)
    if (dj[i].kind == 6u && ok[i]) {
      ColSide& cs = sides[pages[dj[i].page].chunk_slot];
      cs.max_plain_len = std::max(cs.max_plain_len, maxlen[i]);
    }
  size_t n_ok = 0, n_nul = 0;
  for (size_t i = 0; i < dj.size(); i++) {
    if (dj[i].kind == 4u || dj[i].kind == 7u) continue;
    if (ok[i]) { n_ok += dj[i].kind != 5u; n_nul += dj[i].vdst != kNone; }
    else {
      // a run header past the page, a length prefix past the page, a stream that stops early: the reference's reader fails such a file
      const DevPage& pg = pages[dj[i].page];
      throw Error(PQ_ERR_CORRUPT, "column '" + columns[pg.chunk_slot].name + "': the value stream of a data page (" + std::to_string(pg.num_rows) +
                                      " rows, first row " + std::to_string(pg.first_row) + " of its row group) is malformed");
    }
  }
  flat_page_count = n_ok;
  PQB_CUDA(cudaMallocAsync((void**)&d_flat_pages, flat_pages.size() * sizeof(FlatPageRec), stream));
  PQB_CUDA(cudaMemcpyAsync(d_flat_pages, flat_pages.data(), flat_pages.size() * sizeof(FlatPageRec), cudaMemcpyHostToDevice, stream));
  {
    // dictionary indices must stay inside their dictionary (checked once, here; the scan kernels only clamp)
    std::vector<uint32_t> dn(pages.size(), 0);
    for (const TableRowGroup& rg : row_groups)
      for (const TableChunk& tc : rg.chunks)
        if (tc.present)
          for (uint32_t k = 0; k < tc.pages.n_pages; k++) dn[tc.pages.first_page + k] = tc.dict_n;
    uint32_t* d_dn = nullptr;
    uint32_t* d_bad = nullptr;
    PQB_CUDA(cudaMallocAsync((void**)&d_dn, dn.size() * 4, stream));
    PQB_CUDA(cudaMallocAsync((void**)&d_bad, 4, stream));
    PQB_CUDA(cudaMemcpyAsync(d_dn, dn.data(), dn.size() * 4, cudaMemcpyHostToDevice, stream));
    PQB_CUDA(cudaMemsetAsync(d_bad, 0xff, 4, stream));
    launch_check_flat_indices(d_flat, d_flat_pages, d_dn, uint32_t(pages.size()), d_bad, stream);
    uint32_t first_bad = ~0u;
    PQB_CUDA(cudaMemcpyAsync(&first_bad, d_bad, 4, cudaMemcpyDeviceToHost, stream));
    PQB_CUDA(cudaStreamSynchronize(stream));
    dev_drop(d_dn, stream);
    dev_drop(d_bad, stream);
    if (first_bad != ~0u) {
      const DevPage& pg = pages[first_bad];
      throw Error(PQ_ERR_CORRUPT, "column '" + columns[pg.chunk_slot].name + "': a dictionary index is outside the dictionary (" +
                                      std::to_string(dn[first_bad]) + " entries)");
    }
  }
  if (getenv("PQB_VERBOSE"))
    fprintf(stderr, "[pqb] flat store: %zu of %zu pages (%zu with NULLs), %llu bytes (arena %llu)\n", n_ok, pages.size(), n_nul,
            (unsigned long long)flat_bytes, (unsigned long long)arena_bytes);
}

// ---- per column-set shape: chunk table + work items (built once, reused by every query) ----------
std::shared_ptr<Shape> Table::shape_for(const std::vector<int>& tcols, cudaStream_t stream, bool pieces) const {
  std::lock_guard<std::mutex> lk(side_mu);
  std::vector<int> key = tcols;
  if (!pieces) key.push_back(-1);   // a shape of its own
  auto it = shapes.find(key);
  if (it != shapes.end()) return it->second;
  auto sh = std::make_shared<Shape>();
  sh->tcols = tcols;
  const uint32_t ncols = uint32_t(tcols.size());
  const uint32_t nrg = uint32_t(row_groups.size());
  sh->max_bw.assign(ncols, 0); sh->flat_max_bw.assign(ncols, 0);
  sh->has_dict.assign(ncols, 0); sh->has_plain.assign(ncols, 0); sh->has_delta.assign(ncols, 0); sh->flat_plain8.assign(ncols, 0);
  sh->flat_nullable.assign(ncols, 0);
  std::vector<DevChunk> chunks(size_t(nrg) * std::max<uint32_t>(ncols, 1));
  std::vector<std::vector<uint32_t>> bounds;
  std::vector<uint32_t> common;
  const bool use_flat = d_flat_pages != nullptr || ncols == 0;
  sh->items.reserve(size_t(nrg) * 16);
  for (uint32_t g = 0; g < nrg; g++) {
    const TableRowGroup& rg = row_groups[g];
    size_t bounds_n = 0;
    int first_present = -1;
    for (uint32_t s = 0; s < ncols; s++) {
      const TableChunk& tc = rg.chunks[tcols[s]];
      DevChunk& dc = chunks[size_t(g) * ncols + s];
      dc.present = tc.present ? 1 : 0;
      dc.dict8_off = ~0ull;
      if (!tc.present) continue;
      dc.dict_off = tc.dict_off;
      dc.dict_len = tc.dict_len;
      dc.dict_n = tc.dict_n;
      dc.first_page = tc.pages.first_page;
      dc.n_pages = tc.pages.n_pages;
      dc.lut_base = sides[tcols[s]].base_per_rg[g];
      dc.dict8_off = tc.dict8_off;
      sh->max_bw[s] = std::max(sh->max_bw[s], tc.max_bw);
      sh->has_dict[s] |= tc.has_dict_pages;
      sh->has_plain[s] |= tc.has_plain_pages;
      sh->has_delta[s] |= tc.has_delta_pages;
      if (first_present < 0) first_present = int(s);
      if (!rg.pages_aligned) {
        if (bounds.size() <= bounds_n) bounds.emplace_back();
        std::vector<uint32_t>& b = bounds[bounds_n++];
        b.clear();
        for (uint32_t p = 0; p < tc.pages.n_pages; p++) b.push_back(pages[tc.pages.first_page + p].first_row);
      }
    }
    common.clear();
    const bool aligned = rg.pages_aligned && first_present >= 0;
    if (aligned) {   // the pages ARE the items
      const TableChunk& tc0 = rg.chunks[tcols[first_present]];
      for (uint32_t p = 0; p < tc0.pages.n_pages; p++) common.push_back(pages[tc0.pages.first_page + p].first_row);
    } else if (bounds_n == 0) common.push_back(0);
    else {
      common = bounds[0];
      for (size_t i = 1; i < bounds_n; i++) {
        std::vector<uint32_t> t;
        std::set_intersection(common.begin(), common.end(), bounds[i].begin(), bounds[i].end(), std::back_inserter(t));
        common.swap(t);
      }
    }
    if (common.empty() || common[0] != 0) throw Error(PQ_ERR_CORRUPT, "row group pages do not start at row 0");
    // page of column slot s that holds row r of this row group
    auto page_of = [&](uint32_t s, uint32_t r, uint32_t hint) {
      const TableChunk& tc = rg.chunks[tcols[s]];
      uint32_t lo = aligned ? hint : 0, hi = aligned ? hint + 1 : tc.pages.n_pages;
      while (hi - lo > 1) {
        uint32_t mid = (lo + hi) / 2;
        if (pages[tc.pages.first_page + mid].first_row <= r) lo = mid; else hi = mid;
      }
      return tc.pages.first_page + lo;
    };
    auto push_item = [&](DevItem& it, bool flat) {
      it.bitmap_word0 = sh->bitmap_words;
      sh->bitmap_words += (it.nrows + 31) / 32 + 1;
      if (flat)
        for (uint32_t s = 0; s < ncols; s++) {
          if ((it.absent >> s) & 1u) continue;
          const FlatPageRec& fr = flat_pages[it.page[s]];
          if (fr.fkind == FK_PLAIN8) sh->flat_plain8[s] = 1;
          else sh->flat_max_bw[s] = std::max<uint32_t>(sh->flat_max_bw[s], fr.bw);
          if (fr.voff != ~0ull) sh->flat_nullable[s] = 1;
        }
      it.fast = flat ? kItemFlat : 0u;
      sh->n_flat += flat ? 1 : 0;
      sh->n_general += flat ? 0 : 1;
      sh->items.push_back(it);
    };
    std::vector<uint32_t> cuts;
    for (size_t i = 0; i < common.size(); i++) {
      DevItem it{};
      it.rg = g;
      it.row0 = common[i];
      it.nrows = (i + 1 < common.size() ? common[i + 1] : rg.num_rows) - common[i];
      it.global_row0 = rg.global_row0 + common[i];
      const uint32_t row_end = it.row0 + it.nrows;
      bool copied = use_flat && it.nrows != 0;
      cuts.clear();
      for (uint32_t s = 0; s < ncols; s++) {
        const TableChunk& tc = rg.chunks[tcols[s]];
        if (!tc.present) { it.absent |= 1u << s; continue; }   // missing from this file: all NULL (schema adapter behaviour)
        it.page[s] = page_of(s, it.row0, uint32_t(i));
        // every page of this column under the item needs a flat copy; their starts cut the item into pieces
        for (uint32_t pi = it.page[s]; pi < tc.pages.first_page + tc.pages.n_pages && pages[pi].first_row < row_end; pi++) {
          if (flat_pages.empty() || flat_pages[pi].fkind == FK_NONE) {
            copied = false;
            if (sh->why_general.empty())
              sh->why_general = "column '" + columns[tcols[s]].name + "', row group " + std::to_string(g) + ", page " + std::to_string(pi - tc.pages.first_page) +
                                " (encoding " + std::to_string(pages[pi].enc) + ", " + std::to_string(pages[pi].num_rows) + " rows) has no flat-store copy";
          }
          if (pages[pi].first_row > it.row0) cuts.push_back(pages[pi].first_row);
        }
      }
      sh->n_uncopied += copied ? 0 : 1;
      if (!copied || !pieces) { push_item(it, false); continue; }
      // flat: one piece per stretch between page starts of ANY column (a piece lies in one page of every column)
      std::sort(cuts.begin(), cuts.end());
      cuts.erase(std::unique(cuts.begin(), cuts.end()), cuts.end());
      cuts.push_back(row_end);
      uint32_t r = it.row0;
      for (uint32_t cut : cuts) {
        DevItem pc{};
        pc.rg = g;
        pc.row0 = r;
        pc.nrows = cut - r;
        pc.global_row0 = rg.global_row0 + r;
        pc.absent = it.absent;
        for (uint32_t s = 0; s < ncols; s++) {
          if ((it.absent >> s) & 1u) continue;
          pc.page[s] = page_of(s, r, uint32_t(i));
          pc.poff[s] = r - pages[pc.page[s]].first_row;
        }
        push_item(pc, true);
        r = cut;
      }
    }
  }
  PQB_CUDA(cudaMallocAsync((void**)&sh->d_chunks, std::max<size_t>(chunks.size(), 1) * sizeof(DevChunk), stream));
  if (!chunks.empty()) PQB_CUDA(cudaMemcpyAsync(sh->d_chunks, chunks.data(), chunks.size() * sizeof(DevChunk), cudaMemcpyHostToDevice, stream));
  PQB_CUDA(cudaMallocAsync((void**)&sh->d_items, std::max<size_t>(sh->items.size(), 1) * sizeof(DevItem), stream));
  if (!sh->items.empty())
    PQB_CUDA(cudaMemcpyAsync(sh->d_items, sh->items.data(), sh->items.size() * sizeof(DevItem), cudaMemcpyHostToDevice, stream));
  PQB_CUDA(cudaStreamSynchronize(stream));
  shapes.emplace(key, sh);
  return sh;
}

void Table::ensure_ent_off(int tcol, cudaStream_t stream) const {
  std::lock_guard<std::mutex> lk(side_mu);
  ColSide& cs = sides[tcol];
  if (cs.ent_ready) return;
  PQB_CUDA(cudaMallocAsync((void**)&cs.d_ent_off, std::max<uint64_t>(cs.total_entries, 1) * 8, stream));
  launch_entry_offsets(*this, tcol, cs.d_ent_off, &cs.max_ent_len, stream);   // synchronises: later queries run on other streams
  cs.ent_ready = true;
}

void Table::ensure_plain8(int tcol, cudaStream_t stream) const {
  std::lock_guard<std::mutex> lk(side_mu);
  ColSide& cs = sides[tcol];
  if (cs.delta_ready || !cs.has_delta) return;
  struct Job { uint32_t page, sext32; uint64_t dst, vsrc, tmp; };   // == DeltaJob; offsets relative to d_flat
  std::vector<Job> jobs;
  uint64_t off = 0;
  FlatPageRec blank{};
  blank.voff = ~0ull;
  if (flat_pages.size() != pages.size()) flat_pages.assign(pages.size(), blank);
  auto take = [&](uint64_t bytes) { uint64_t o = off; off = (off + bytes + 16 + 15) & ~15ull; return o; };
  for (const TableRowGroup& rg : row_groups) {
    const TableChunk& tc = rg.chunks[tcol];
    if (!tc.present) continue;
    for (uint32_t k = 0; k < tc.pages.n_pages; k++) {
      const uint32_t pi = tc.pages.first_page + k;
      if (pages[pi].enc != DE_DELTA || flat_pages[pi].fkind != FK_NONE) continue;
      Job j{pi, columns[tcol].is_date ? 1u : 0u, take(uint64_t(pages[pi].num_rows) * 8), flat_pages[pi].voff, ~0ull};
      if (j.vsrc != ~0ull) j.tmp = take(uint64_t(pages[pi].num_rows) * 8);
      jobs.push_back(j);
    }
  }
  if (!jobs.empty()) {
    PQB_CUDA(cudaMallocAsync((void**)&cs.d_delta_flat, off + 256, stream));
    // offsets are relative to d_flat (the kernels add them to that one base); the subtraction may wrap, the sum does not
    const uint64_t rel = uint64_t(cs.d_delta_flat) - uint64_t(d_flat);
    for (Job& j : jobs) { j.dst += rel; if (j.tmp != ~0ull) j.tmp += rel; }
    void* d_jobs = nullptr;
    uint8_t* d_ok = nullptr;
    PQB_CUDA(cudaMallocAsync(&d_jobs, jobs.size() * sizeof(Job), stream));
    PQB_CUDA(cudaMallocAsync((void**)&d_ok, jobs.size(), stream));
    PQB_CUDA(cudaMemcpyAsync(d_jobs, jobs.data(), jobs.size() * sizeof(Job), cudaMemcpyHostToDevice, stream));
    launch_delta_to_plain8(d_arena, d_pages, d_jobs, uint32_t(jobs.size()), d_flat, d_ok, stream);
    std::vector<uint8_t> ok(jobs.size());
    PQB_CUDA(cudaMemcpyAsync(ok.data(), d_ok, ok.size(), cudaMemcpyDeviceToHost, stream));
    PQB_CUDA(cudaStreamSynchronize(stream));
    dev_drop(d_jobs, stream);
    dev_drop(d_ok, stream);
    for (size_t i = 0; i < jobs.size(); i++) {
      if (!ok[i]) continue;   // a stream the decoder refused: the page stays with k_scan
      FlatPageRec& fr = flat_pages[jobs[i].page];
      fr.off = jobs[i].dst;
      fr.rows = pages[jobs[i].page].num_rows;
      fr.bw = 64;
      fr.fkind = FK_PLAIN8;
    }
    if (!d_flat_pages) PQB_CUDA(cudaMallocAsync((void**)&d_flat_pages, flat_pages.size() * sizeof(FlatPageRec), stream));
    PQB_CUDA(cudaMemcpyAsync(d_flat_pages, flat_pages.data(), flat_pages.size() * sizeof(FlatPageRec), cudaMemcpyHostToDevice, stream));
    PQB_CUDA(cudaStreamSynchronize(stream));
    shapes.clear();   // column sets with this column get new work items (flat now)
  }
  cs.delta_ready = true;
}

void Table::unify_key(int tcol, cudaStream_t stream) const {
  std::lock_guard<std::mutex> lk(side_mu);
  unify_key_side(*this, tcol, sides[tcol], stream);
}

// Query-independent prep like the hot-first numbering of ensure_key: the host copy of the key dictionary is sorted once
// per column (and once per agreement of the ranks); keys interned from pages without a dictionary are in it too.
static std::shared_ptr<const uint32_t> kd_rank_locked(ColSide& cs, bool agreed, cudaStream_t stream) {
  std::shared_ptr<const uint32_t>& r = agreed ? cs.glob_kd_rank : cs.kd_rank;
  if (r) return r;
  const KeyDict& kd = agreed ? cs.glob_kd : cs.kd;
  const uint32_t card = kd.offs.empty() ? 0u : uint32_t(kd.offs.size() - 1);
  std::vector<uint32_t> rank(std::max<uint32_t>(card, 1), 0);
  order_string_ranks(kd.offs.data(), kd.bytes.data(), card, rank.data());
  uint32_t* d = nullptr;
  PQB_CUDA(cudaMallocAsync((void**)&d, rank.size() * 4, stream));
  r = std::shared_ptr<const uint32_t>(d, [](const uint32_t* p) { cudaFree(const_cast<uint32_t*>(p)); });
  PQB_CUDA(cudaMemcpyAsync(d, rank.data(), rank.size() * 4, cudaMemcpyHostToDevice, stream));
  PQB_CUDA(cudaStreamSynchronize(stream));
  return r;
}

std::shared_ptr<const uint32_t> Table::ensure_kd_rank(int tcol, bool agreed, cudaStream_t stream) const {
  std::lock_guard<std::mutex> lk(side_mu);
  return kd_rank_locked(sides[tcol], agreed, stream);
}

RankLuts::~RankLuts() {
  if (ent) cudaFree(ent);
  if (ids) cudaFree(ids);
  if (inv) cudaFree(inv);
}

std::shared_ptr<const RankLuts> Table::ensure_rank_luts(int tcol, bool agreed, cudaStream_t stream) const {
  std::lock_guard<std::mutex> lk(side_mu);
  ColSide& cs = sides[tcol];
  std::shared_ptr<const RankLuts>& r = agreed ? cs.glob_rank_luts : cs.rank_luts;
  if (r) return r;
  const std::shared_ptr<const uint32_t> rank = kd_rank_locked(cs, agreed, stream);
  auto luts = std::make_shared<RankLuts>();
  build_rank_luts(cs, agreed, rank.get(), *luts, stream);
  r = luts;
  return r;
}

void Table::ensure_key(int tcol, cudaStream_t stream) const {
  ensure_ent_off(tcol, stream);
  std::lock_guard<std::mutex> lk(side_mu);
  ColSide& cs = sides[tcol];
  if (cs.key_ready) return;
  build_key_side(*this, tcol, cs, stream);
  cs.key_ready = true;
}

}  // namespace pqb
