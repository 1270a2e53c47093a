// extern "C" surface declared in include/parseable_b200.h.  No exception crosses
// the boundary: every failure becomes a negative status plus a message
// (SURVEY.md §8b "Error convention"), which the Rust shim wraps in
// DataFusionError::External.
#include <cstring>
#include <new>
#include <string>

#include "engine.hpp"

using namespace pqb;

namespace {
thread_local std::string g_last_error;

template <typename F>
int guard(F&& f, std::string* sink = nullptr) {
  try {
    return f();
  } catch (const Error& e) {
    g_last_error = e.what();
    if (sink) *sink = e.what();
    return e.code;
  } catch (const std::bad_alloc&) {
    g_last_error = "out of host memory";
    if (sink) *sink = g_last_error;
    return PQ_ERR_OOM;
  } catch (const std::exception& e) {
    g_last_error = e.what();
    if (sink) *sink = e.what();
    return PQ_ERR_CORRUPT;
  } catch (...) {
    g_last_error = "unknown error";
    if (sink) *sink = g_last_error;
    return PQ_ERR_CUDA;
  }
}
}  // namespace

struct PqQuery {
  Query* q = nullptr;
  std::string error;
};
struct PqTable {
  Table t;
};

extern "C" {

const char* pq_version(void) { return "parseable_b200 0.1.0 (sm_90a)"; }

int pq_device_count(void) {
  int n = 0;
  if (cudaGetDeviceCount(&n) != cudaSuccess) { cudaGetLastError(); return 0; }
  return n;
}

int pq_init(const int* device_ids, int n) {
  return guard([&] { Context::get().init(device_ids, n); return PQ_OK; });
}

void pq_shutdown(void) {
  comm_destroy();
  Context::get().shutdown();
}

int pq_table_open(const PqFile* files, uint32_t n_files, const char* const* columns, uint32_t n_columns,
                  uint32_t shard_index, uint32_t shard_count, PqTable** out) {
  if (!out) return PQ_ERR_INVALID_ARG;
  *out = nullptr;
  return guard([&] {
    if (!files || !n_files || (!columns && n_columns)) throw Error(PQ_ERR_INVALID_ARG, "pq_table_open: missing files or columns");
    Context::get().ensure();
    std::vector<std::string> names;
    for (uint32_t i = 0; i < n_columns; i++) {
      if (!columns[i]) throw Error(PQ_ERR_INVALID_ARG, "pq_table_open: NULL column name");
      names.emplace_back(columns[i]);
    }
    auto* t = new PqTable;
    try {
      cudaStream_t s;
      PQB_CUDA(cudaStreamCreateWithFlags(&s, cudaStreamNonBlocking));
      try { t->t.open(files, n_files, names, shard_index, shard_count, s); } catch (...) { cudaStreamDestroy(s); throw; }
      cudaStreamDestroy(s);
    } catch (...) { delete t; throw; }
    *out = t;
    return PQ_OK;
  });
}

uint64_t pq_table_rows(const PqTable* t) { return t ? t->t.total_rows : 0; }
uint64_t pq_table_device_bytes(const PqTable* t) { return t ? t->t.arena_bytes : 0; }
void pq_table_close(PqTable* t) {
  if (!t) return;
  guard([&] { Context::get().ensure(); return PQ_OK; });
  delete t;
}

int pq_query_open(const PqQueryDesc* desc, PqQuery** out) {
  if (!out) return PQ_ERR_INVALID_ARG;
  *out = nullptr;
  if (!desc) { g_last_error = "pq_query_open: NULL descriptor"; return PQ_ERR_INVALID_ARG; }
  auto* h = new (std::nothrow) PqQuery;
  if (!h) return PQ_ERR_OOM;
  int rc = guard([&] { h->q = new Query(*desc); return PQ_OK; }, &h->error);
  if (rc != PQ_OK) { delete h; return rc; }
  *out = h;
  return PQ_OK;
}

int pq_query_next(PqQuery* q, int partition, struct ArrowArray* out, struct ArrowSchema* out_schema) {
  if (!q || !q->q) return PQ_ERR_INVALID_ARG;
  return guard([&] { return q->q->next(partition, out, out_schema); }, &q->error);
}

namespace {
struct StreamPriv {
  PqQuery* q;
  int partition;
  std::string err;
};
int stream_get_schema(struct ArrowArrayStream* s, struct ArrowSchema* out) {
  auto* p = static_cast<StreamPriv*>(s->private_data);
  try {
    p->q->q->schema(out);
    return 0;
  } catch (const std::exception& e) {
    p->err = e.what();
    return 5;  // EIO
  }
}
int stream_get_next(struct ArrowArrayStream* s, struct ArrowArray* out) {
  auto* p = static_cast<StreamPriv*>(s->private_data);
  const int rc = pq_query_next(p->q, p->partition, out, nullptr);
  if (rc == PQ_OK) return 0;
  if (rc == PQ_END_OF_STREAM) {
    std::memset(out, 0, sizeof(*out));  // release == NULL marks the end
    return 0;
  }
  p->err = pq_last_error(p->q);
  return 5;
}
const char* stream_last_error(struct ArrowArrayStream* s) { return static_cast<StreamPriv*>(s->private_data)->err.c_str(); }
void stream_release(struct ArrowArrayStream* s) {
  delete static_cast<StreamPriv*>(s->private_data);
  s->private_data = nullptr;
  s->release = nullptr;
}
}  // namespace

int pq_query_stream(PqQuery* q, int partition, struct ArrowArrayStream* out) {
  if (!q || !q->q || !out) return PQ_ERR_INVALID_ARG;
  out->get_schema = stream_get_schema;
  out->get_next = stream_get_next;
  out->get_last_error = stream_last_error;
  out->release = stream_release;
  out->private_data = new StreamPriv{q, partition, {}};
  return PQ_OK;
}

int pq_query_json(PqQuery* q, uint32_t flags, const char** out, uint64_t* len) {
  if (!q || !q->q || !out || !len) return PQ_ERR_INVALID_ARG;
  return guard([&] { q->q->json(flags, out, len); return PQ_OK; }, &q->error);
}

int pq_query_metrics(PqQuery* q, PqMetrics* out) {
  if (!q || !q->q || !out) return PQ_ERR_INVALID_ARG;
  *out = q->q->metrics;
  return PQ_OK;
}

const char* pq_last_error(PqQuery* q) { return q ? q->error.c_str() : g_last_error.c_str(); }

void pq_query_close(PqQuery* q) {
  if (!q) return;
  guard([&] { Context::get().ensure(); return PQ_OK; });
  delete q->q;
  delete q;
}

void* pq_host_alloc(uint64_t bytes) {
  void* p = nullptr;
  int rc = guard([&] {
    Context::get().ensure();
    cudaError_t e = cudaHostAlloc(&p, bytes ? bytes : 1, cudaHostAllocDefault);
    if (e != cudaSuccess) throw Error(PQ_ERR_OOM, std::string("cudaHostAlloc: ") + cudaGetErrorString(e));
    return PQ_OK;
  });
  return rc == PQ_OK ? p : nullptr;
}
void pq_host_free(void* p) {
  if (p) cudaFreeHost(p);
}

int64_t pq_file_describe(const PqFile* file, char* out, uint64_t cap) {
  if (!file) return PQ_ERR_INVALID_ARG;
  std::string js;
  int rc = guard([&] { js = describe_file(*file); return PQ_OK; });
  if (rc != PQ_OK) return rc;
  if (out && cap) {
    uint64_t n = js.size() < cap - 1 ? js.size() : cap - 1;
    std::memcpy(out, js.data(), n);
    out[n] = 0;
  }
  return int64_t(js.size());
}

int pq_comm_unique_id(uint8_t id[PQ_COMM_ID_BYTES]) {
  return guard([&] { return comm_unique_id(id); });
}
int pq_comm_init_rank(const uint8_t id[PQ_COMM_ID_BYTES], int nranks, int rank) {
  return guard([&] { Context::get().ensure(); return comm_init_rank(id, nranks, rank); });
}
int pq_comm_destroy(void) {
  return guard([&] { return comm_destroy(); });
}

}  // extern "C"
