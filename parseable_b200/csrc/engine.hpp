// Host side of the H100 query path: HBM-resident tables of encoded column
// chunks, query planning (row-group pruning, work items, predicate/aggregate
// compilation) and the kernel launch sequence.  Mirrors, on the host, what
// StandardTableProvider::scan + create_parquet_physical_plan do before
// DataFusion's operators run (/root/reference/src/query/stream_schema_provider.rs:114-189, 526-659).
#pragma once
#include <cuda_runtime.h>

#include <atomic>
#include <cstdint>
#include <map>
#include <memory>
#include <mutex>
#include <stdexcept>
#include <string>
#include <unordered_map>
#include <utility>
#include <vector>

#include "../../include/parseable_b200.h"
#include "device_structs.hpp"
#include "parquet_meta.hpp"

namespace pqb {

struct Error : std::runtime_error {
  int code;
  Error(int c, const std::string& m) : std::runtime_error(m), code(c) {}
};

#define PQB_CUDA(expr)                                                                          \
  do {                                                                                          \
    cudaError_t _e = (expr);                                                                    \
    if (_e != cudaSuccess)                                                                      \
      throw ::pqb::Error(_e == cudaErrorMemoryAllocation ? PQ_ERR_OOM : PQ_ERR_CUDA,            \
                         std::string(#expr) + ": " + cudaGetErrorString(_e));                   \
  } while (0)

// ---- process-wide state ----
class Context {
 public:
  static Context& get();
  void init(const int* devices, int n);
  void shutdown();
  void ensure();  // throws PQ_ERR_CUDA when no device is usable; binds the device to the calling thread
  int device() const { return device_; }
  int sm_count() const { return sm_count_; }
  size_t smem_optin() const { return smem_optin_; }
  size_t smem_per_sm() const { return smem_per_sm_; }
  size_t l2_bytes() const { return l2_bytes_; }
  // pinned staging buffers, grow-only cache
  uint8_t* pinned_acquire(size_t bytes);
  void pinned_release(uint8_t* p);
  bool is_pinned(const void* p);
  // non-blocking streams for queries, kept for reuse: creating and destroying one costs more host time than all the
  // other launches of a warm resident query.  A released stream may still hold queued frees; whoever takes it next
  // orders its work after them.  Each stream is kept with its device: stream_acquire hands out only the current
  // device's (a query that was running while the context moved to another device releases its stream afterwards)
  cudaStream_t stream_acquire();
  void stream_release(cudaStream_t s, int device);

 private:
  std::mutex mu_;
  bool inited_ = false;
  int device_ = 0;
  int sm_count_ = 0;
  size_t smem_optin_ = 0;
  size_t smem_per_sm_ = 0;
  size_t l2_bytes_ = 0;
  struct Pinned { uint8_t* p; size_t cap; bool busy; };
  std::vector<Pinned> pinned_;
  std::vector<std::pair<int, cudaStream_t>> free_streams_;   // (device, stream)
};

// ---- host view of a Parquet file ----
struct HostFile {
  std::string path;
  const uint8_t* data = nullptr;  // whole file image (mmap or caller buffer)
  uint64_t size = 0;
  bool mapped = false;
  FileMeta meta;
  ~HostFile();
};

struct TablePageRef {
  uint32_t first_page = 0;  // into Table::pages (data pages only)
  uint32_t n_pages = 0;
};

struct TableChunk {
  bool present = false;
  int leaf = -1;
  const ColumnChunkMeta* meta = nullptr;
  uint64_t arena_off = 0;   // where the chunk's bytes start in the arena
  uint64_t file_off = 0;
  uint64_t bytes = 0;       // compressed == uncompressed (codec NONE)
  uint64_t dict_off = 0;    // arena offset of the dictionary payload
  uint32_t dict_len = 0, dict_n = 0;
  TablePageRef pages;
  bool has_dict_pages = false, has_plain_pages = false, has_delta_pages = false;
  uint32_t max_bw = 0;
  uint64_t dict8_off = ~0ull;   // flat store: 8-byte aligned copy of a numeric dictionary
};

struct TableColumn {
  std::string name;
  uint8_t kind = 0;      // DevKind
  bool is_ts = false;
  bool is_date = false;  // Date32: INT32 leaves, kind DK_I64 with sign-extended 8-byte values in the flat store
  uint8_t max_def = 0;
};

struct TableRowGroup {
  uint32_t file = 0, rg_in_file = 0;
  uint32_t num_rows = 0;
  uint64_t global_row0 = 0;         // ordinal over ALL row groups of the file list (before sharding)
  std::vector<TableChunk> chunks;   // per table column
  bool pages_aligned = false;       // every present column has the same page boundaries (Parseable's writer: 20 000-row pages)
};

// Query-independent side tables of one table column, built on first use and kept with the table:
// string dictionary entry offsets, and (GROUP BY) the interned group ids of every dictionary entry.
struct KeyDict { std::vector<uint32_t> offs; std::vector<uint8_t> bytes; };
// MIN / MAX over a Utf8 column, one numbering (local or agreed), built from ensure_kd_rank's ranks: the bytewise rank of
// every dictionary entry (rank[gid[e]], composed once so that the aggregate pass makes one load per row) and of every group
// id (id pages), as 64-bit values like a numeric dictionary's; and the rank -> group id inverse for the result
struct RankLuts {
  uint64_t* ent = nullptr;               // per dictionary entry of the column (ColSide::total_entries)
  uint64_t* ids = nullptr;               // per group id
  uint32_t* inv = nullptr;               // per rank: its group id
  uint32_t card = 0;
  RankLuts() = default;
  RankLuts(const RankLuts&) = delete;
  ~RankLuts();
};
struct ColSide {
  std::vector<uint32_t> base_per_rg;   // dictionary entries of this column in the row groups before g
  uint32_t total_entries = 0;
  uint32_t max_dict_n = 0;
  uint64_t* d_ent_off = nullptr;       // arena offset of every dictionary entry (strings: behind the length prefix)
  bool ent_ready = false;
  // group-key interning (local numbering, hot-first)
  bool key_ready = false;
  uint32_t* d_gid = nullptr;           // group id per dictionary entry
  uint32_t card = 0;
  KeyDict kd;                          // distinct values in group-id order
  uint32_t max_ent_len = 0;            // longest dictionary entry (sizes projected string buffers)
  uint32_t max_plain_len = 0;          // longest value of the column's PLAIN byte-array pages
  bool has_delta = false;              // some page of the column is DELTA_BINARY_PACKED
  bool delta_ready = false;            // ... and its pages have aligned 8-byte copies in d_delta_flat (ensure_plain8)
  uint8_t* d_delta_flat = nullptr;
  uint32_t* d_kd_offs = nullptr;       // the same on the device (result assembly)
  uint8_t* d_kd_bytes = nullptr;
  uint32_t kd_max_len = 0;
  std::shared_ptr<const uint32_t> kd_rank;   // ORDER BY on a Utf8 key: bytewise rank of every group id, on the device (ensure_kd_rank)
  // multi-GPU: the numbering every rank of the communicator agreed on (unify_key), tagged with the communicator's epoch
  bool glob_ready = false;
  uint64_t glob_epoch = 0;
  uint32_t glob_card = 0, glob_max_len = 0;
  KeyDict glob_kd;
  uint32_t* d_glob_gid = nullptr;
  uint32_t* d_glob_kd_offs = nullptr;
  uint8_t* d_glob_kd_bytes = nullptr;
  std::shared_ptr<const uint32_t> glob_kd_rank;   // the same ranks over the agreed numbering (dropped by every unify_key)
  std::shared_ptr<const RankLuts> rank_luts, glob_rank_luts;   // MIN / MAX over Utf8 (ensure_rank_luts); the agreed one is dropped by every unify_key
  uint64_t* d_key_hash = nullptr;
  // GROUP BY on a column with pages that have no dictionary (PLAIN fallback, PLAIN / DELTA numerics): every ROW of those
  // pages is an entry behind the dictionary entries; d_gid / d_glob_gid then hold, per such page, one group id per row --
  // the page's "id page", staged by the aggregate kernel like 32-bit dictionary indices (FK_IDS)
  uint32_t key_entries = 0;            // entries d_gid covers (== total_entries when the column has only dictionary pages)
  uint32_t n_dict_pad = 0;             // first row entry (total_entries rounded up to 4)
  uint64_t* d_row_ent = nullptr;       // where every row entry's value sits (relative to the arena, ~0: NULL / padding)
  struct KeyRowPage { uint32_t page; uint32_t ebase; };   // page index, first entry of its rows relative to n_dict_pad
  std::vector<KeyRowPage> key_row_pages;
  // agg pages (Table::agg_pages): value pages of a numeric column's dictionary pages, or id pages of a GROUP BY key's.
  // A page has one other form at most: the first one a query asks for stays.
  bool for_ready = false;
  uint8_t* d_for = nullptr;
  uint32_t for_pages = 0;              // dictionary pages that have a value page
  uint32_t for_bw = 0;                 // widest value page
  uint32_t for_rest_bw = 0;            // widest index page left without one (chunks that do not qualify)
  uint64_t for_bytes = 0;
  // Id pages hold the LOCAL numbering (d_gid) only: it is fixed for the table's life, so the pages are built once and never
  // rewritten under a query that reads them.  An agreed numbering (d_glob_gid) changes with every agreement of the ranks
  // (unify_key), and a table may serve both numberings at the same time; its queries keep the gid LUT.
  bool ids_ready = false;
  uint8_t* d_ids = nullptr;
  uint32_t ids_bw = 0;
  uint64_t ids_bytes = 0;
};

// What a query needs per SET of referenced columns, built once per (table, column set): the chunk
// table, the work items (row ranges between page boundaries common to the columns) and what the
// kernels' shared-memory layouts depend on.
struct Shape {
  std::vector<int> tcols;
  std::vector<DevItem> items;
  DevChunk* d_chunks = nullptr;        // [table row group * ncols + slot]
  DevItem* d_items = nullptr;
  uint32_t n_flat = 0, n_general = 0;
  uint32_t n_uncopied = 0;             // items with a page that has no flat-store copy
  uint32_t bitmap_words = 0;
  std::vector<uint32_t> max_bw, flat_max_bw;          // per slot
  std::vector<uint8_t> has_dict, has_plain, has_delta, flat_plain8, flat_nullable;   // flat_nullable: some flat page of the slot carries a validity bitmap
  std::string why_general;             // first reason an item could not go to the flat kernels (diagnostics)
  std::atomic<unsigned long long> last_total{~0ull};   // rows the last filter scan of this shape selected (sizes the next result)
  // groups of the last answer of each aggregate plan over this shape (keyed by plan_hash): a repeat of the query lays its
  // result block out before the group count is back on the host (at most 64 plans; the map is cleared when full)
  std::mutex hint_mu;
  std::unordered_map<uint64_t, uint32_t> groups_hint;
  ~Shape();
};

// Tuple id pages of one GROUP BY key tuple (Table::ensure_tuple_pages): the groups that occur in the table, numbered by
// row count (descending, ties by mixed-radix id), and one bit-packed page of tuple ids per page of the lead key column.
// A query that holds the entry keeps its device memory alive.
struct TuplePages {
  uint32_t n_tuples = 0, bw = 0;
  int lead = -1;                        // table column whose pages the tuple pages follow
  uint8_t* d_buf = nullptr;             // the pages (FlatPageRec.off relative to d_flat, like every flat page)
  std::vector<std::pair<uint32_t, FlatPageRec>> recs;   // lead page index -> its tuple page
  unsigned long long* d_wide = nullptr; // tuple id -> mixed-radix id
  uint32_t* d_order = nullptr;          // position -> tuple id, ascending mixed-radix id
  uint64_t bytes = 0;
  double build_ms = 0;
  // the table's agg page table with the lead pages replaced by the tuple pages, for the agg pages version it copies
  // (Table::tuple_page_table; guarded by the table's side_mu)
  mutable std::shared_ptr<const FlatPageRec> d_pages;
  mutable uint64_t pages_ver = ~0ull;
  ~TuplePages();
};

// Encoded column chunks of a set of files, resident in HBM ("hot tier in HBM").
class Table {
 public:
  Table() = default;
  ~Table();
  Table(const Table&) = delete;
  void open(const PqFile* files, uint32_t n_files, const std::vector<std::string>& columns, uint32_t shard_index,
            uint32_t shard_count, cudaStream_t stream);

  std::vector<std::unique_ptr<HostFile>> files;
  std::vector<TableColumn> columns;
  std::vector<TableRowGroup> row_groups;
  std::vector<DevPage> pages;       // host copy
  uint8_t* d_arena = nullptr;
  uint64_t arena_bytes = 0;
  DevPage* d_pages = nullptr;
  uint8_t* d_strmat = nullptr;            // DELTA_BYTE_ARRAY pages rewritten as PLAIN BYTE_ARRAY pages (outside the arena: DevPage.off wraps)
  uint64_t total_rows = 0;
  uint32_t shard_index = 0, shard_count = 1;   // this process scans row groups g % shard_count == shard_index of the list
  uint64_t list_rows = 0;                      // rows of every row group of the file list (global_row0 runs over them)
  uint64_t h2d_bytes = 0;
  uint64_t chunk_bytes = 0;
  int find_column(const std::string& name) const;

  // flat store (flat_store.cuh): header-less bit-packed copies of the NULL-free dictionary-index pages,
  // aligned copies of PLAIN 8-byte pages and of numeric dictionaries
  uint8_t* d_flat = nullptr;
  uint64_t flat_bytes = 0;
  mutable std::vector<FlatPageRec> flat_pages;   // host copy, parallel to pages (ensure_plain8 adds entries later)
  mutable FlatPageRec* d_flat_pages = nullptr;
  uint64_t flat_page_count = 0;

  // lazily built, query independent (the table is immutable once opened); guarded by side_mu
  mutable std::mutex side_mu;
  mutable std::vector<ColSide> sides;
  mutable std::map<std::vector<int>, std::shared_ptr<Shape>> shapes;
  // pieces = false: no item is cut at the page starts of other columns or handed to the flat kernels (k_scan enters
  // every page of an item at its first row, so it reads only whole-page items)
  std::shared_ptr<Shape> shape_for(const std::vector<int>& tcols, cudaStream_t stream, bool pieces = true) const;
  void ensure_ent_off(int tcol, cudaStream_t stream) const;
  void ensure_key(int tcol, cudaStream_t stream) const;
  void unify_key(int tcol, cudaStream_t stream) const;        // collective over the pq_comm communicator
  // bytewise rank per group id of a Utf8 key column, local or agreed numbering (after ensure_key / unify_key)
  // (shared: a query keeps the ranks it sorts with alive even if unify_key replaces them meanwhile)
  std::shared_ptr<const uint32_t> ensure_kd_rank(int tcol, bool agreed, cudaStream_t stream) const;
  // MIN / MAX over a Utf8 column: its rank tables in the local or agreed numbering (after ensure_key / unify_key), built
  // once per numbering from ensure_kd_rank's ranks; shared like them
  std::shared_ptr<const RankLuts> ensure_rank_luts(int tcol, bool agreed, cudaStream_t stream) const;
  void ensure_plain8(int tcol, cudaStream_t stream) const;   // DELTA_BINARY_PACKED pages -> row-addressable 8-byte values
  // agg pages: a second flat page table parallel to pages[] (FK_NONE: the page has no other form), read by k_flat_agg's
  // producer for the column slots a query marks.  ensure_for_pages: value pages of a numeric column; ensure_id_pages: id
  // pages of a GROUP BY key in its local numbering (after ensure_key).  Both return false when the column has no such
  // pages (no chunk qualifies, its pages hold the other form, or the device memory for them is not there: the agg pages
  // are optional, the query then reads the index pages).  Records only ever go from FK_NONE to a form, once.
  mutable std::vector<FlatPageRec> agg_pages;
  mutable FlatPageRec* d_agg_pages = nullptr;
  bool ensure_for_pages(int tcol, bool f64, cudaStream_t stream) const;
  bool ensure_id_pages(int tcol, cudaStream_t stream) const;
  mutable uint64_t agg_pages_ver = 0;   // counts the agg page builds (a tuple entry's page table copies one version)
  // tuple id pages of a GROUP BY key tuple in the local numbering, keyed by (table column, mixed-radix stride) per key:
  // built once per tuple (nullptr: the one attempt failed, the query keeps per-key pages), at most kMaxTupleEntries
  static constexpr size_t kMaxTupleEntries = 16;
  mutable std::map<std::vector<std::pair<int, uint64_t>>, std::shared_ptr<const TuplePages>> tuples;
  std::shared_ptr<const TuplePages> ensure_tuple_pages(const std::vector<std::pair<int, uint64_t>>& keys, bool verbose,
                                                       cudaStream_t stream) const;
  // the tuple entry's page table for the current agg pages (built on first use after an agg page build)
  std::shared_ptr<const FlatPageRec> tuple_page_table(const TuplePages& tp, cudaStream_t stream) const;

 private:
  void build_flat_store(cudaStream_t stream);
};

// launches k_flat_store (flat_store.cuh); jobs are FlatStoreJob records on the device
void launch_flat_store(const uint8_t* arena, const DevPage* pages, const void* jobs, uint32_t n_jobs, uint8_t* flat, uint8_t* ok,
                       uint32_t* maxlen, cudaStream_t stream);
// side-table builders (prep_kernels.cuh), defined in query.cu
void launch_entry_offsets(const Table& t, int tcol, uint64_t* d_out, uint32_t* max_len, cudaStream_t stream);
void launch_dba_lengths(const uint8_t* arena, const DevPage* pages, const DbaJob* jobs, uint32_t n_jobs, uint8_t* scratch, DbaInfo* info, cudaStream_t stream);
void launch_dba_materialise(const uint8_t* arena, const DevPage* pages, const DbaJob* jobs, const DbaInfo* info, uint32_t n_jobs,
                            const uint8_t* scratch, uint8_t* mat, cudaStream_t stream);
void launch_check_flat_indices(const uint8_t* flat, const FlatPageRec* fpages, const uint32_t* dict_n, uint32_t n_pages, uint32_t* first_bad, cudaStream_t stream);
void launch_page_has_nulls(const uint8_t* arena, const DevPage* pages, uint32_t n_pages, uint8_t* out, cudaStream_t stream);
void launch_delta_to_plain8(const uint8_t* arena, const DevPage* pages, const void* jobs, uint32_t n_jobs, uint8_t* flat_base, uint8_t* ok,
                            cudaStream_t stream);
void build_key_side(const Table& t, int tcol, ColSide& side, cudaStream_t stream);
void unify_key_side(const Table& t, int tcol, ColSide& side, cudaStream_t stream);
void build_rank_luts(const ColSide& side, bool agreed, const uint32_t* rank, RankLuts& luts, cudaStream_t stream);

// host block that result batches alias (zero copy): page-locked from the context's pool, or (one-row and empty results)
// ordinary heap memory, so that a small result does not hold a pool block of 1 MB or more while the consumer keeps it.
// A pool block returns to the pool when the last batch that references it is released by the consumer
struct PinnedBlock {
  uint8_t* p = nullptr;
  size_t bytes = 0;
  uint8_t* dev = nullptr;        // the device block this one was copied from, while the query keeps it (JSON egress reads it there)
  std::vector<uint64_t> heap;    // a heap block: p points into it
  ~PinnedBlock();
};

// one column of one batch: a slice of a result block (laid out by query.cu's BlockLayout)
struct OutColumn {
  std::string name;
  int type = PQ_T_I64;               // PqType
  std::shared_ptr<PinnedBlock> block;
  size_t values_off = 0;             // 8-byte values (4-byte Date32), bit-packed bools, or utf8 bytes
  size_t validity_off = 0;           // validity bitmap (used when null_count != 0)
  size_t offsets_off = 0;            // utf8: int32 offsets of this batch's first row (n + 1 entries follow)
  int64_t null_count = 0;
};

struct OutBatch {
  int64_t rows = 0;
  std::vector<OutColumn> cols;
};

class Query {
 public:
  explicit Query(const PqQueryDesc& d);
  ~Query();
  int next(int partition, ArrowArray* out, ArrowSchema* schema);
  void schema(ArrowSchema* out) const;   // of the result batches (an empty struct when the query produced none)
  // every batch of the result as JSON text formatted on the device (json_egress.cuh); the bytes stay valid until the
  // next call or the query is closed
  void json(uint32_t flags, const char** out, uint64_t* len);
  PqMetrics metrics{};
  std::string error;

 private:
  void run(const PqQueryDesc& d);
  std::unique_ptr<Table> owned_table_;
  std::vector<OutBatch> batches_;
  std::vector<std::shared_ptr<PinnedBlock>> dev_blocks_;   // result blocks whose device copy is kept until the query closes
  std::shared_ptr<PinnedBlock> json_block_;
  uint32_t batch_rows_ = 20000;
  size_t next_batch_ = 0;
  bool schema_only_done_ = false;
};

void export_batch(const OutBatch& b, ArrowArray* out, ArrowSchema* schema);
std::string describe_file(const PqFile& f);

// NCCL communicator owned by the library (one process per GPU)
int comm_unique_id(uint8_t* id);
int comm_init_rank(const uint8_t* id, int nranks, int rank);
int comm_destroy();
bool comm_active();
uint64_t comm_epoch();        // changes with every communicator
void comm_group_begin();      // ncclGroupStart / End: the collectives in between launch as one
void comm_group_end();
int comm_nranks();
int comm_rank();
void comm_allreduce_u64(void* buf, size_t count, int op /*0 sum,1 min(s64),2 max(s64),3 sum f64*/, cudaStream_t s);
void comm_allgather_bytes(const void* send, void* recv, size_t bytes_per_rank, cudaStream_t s);

}  // namespace pqb
