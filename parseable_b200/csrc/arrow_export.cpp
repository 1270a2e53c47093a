// Result batches leave through the Arrow C Data Interface as a struct array
// (= RecordBatch), which arrow::ffi on the Rust side imports into the
// RecordBatch that Query::execute returns (/root/reference/src/query/mod.rs:81, 287-291).
// The producer owns the buffers until the consumer calls release.
#include <cstdlib>
#include <cstring>

#include "engine.hpp"

namespace pqb {

namespace {

struct SchemaPriv {
  std::string format, name;
  std::vector<ArrowSchema> children;
  std::vector<ArrowSchema*> child_ptrs;
};

void release_schema(ArrowSchema* s) {
  if (!s || !s->release) return;
  auto* p = static_cast<SchemaPriv*>(s->private_data);
  if (p) {
    for (auto& c : p->children)
      if (c.release) c.release(&c);
    delete p;
  }
  s->release = nullptr;
}

struct ArrayPriv {
  std::shared_ptr<PinnedBlock> keep;
  std::vector<const void*> buffers;
  std::vector<ArrowArray> children;
  std::vector<ArrowArray*> child_ptrs;
};

void release_array(ArrowArray* a) {
  if (!a || !a->release) return;
  auto* p = static_cast<ArrayPriv*>(a->private_data);
  if (p) {
    for (auto& c : p->children)
      if (c.release) c.release(&c);
    delete p;
  }
  a->release = nullptr;
}

const char* format_of(int type) {
  switch (type) {
    case PQ_T_BOOL: return "b";
    case PQ_T_I64: return "l";
    case PQ_T_F64: return "g";
    case PQ_T_UTF8: return "u";
    case PQ_T_TS_MS: return "tsm:";
    case PQ_T_DATE32: return "tdD";
    default: return "n";
  }
}

void fill_schema(ArrowSchema* s, const std::string& fmt, const std::string& name, size_t nchildren) {
  auto* p = new SchemaPriv;
  p->format = fmt;
  p->name = name;
  p->children.resize(nchildren);
  for (auto& c : p->children) { std::memset(&c, 0, sizeof(c)); p->child_ptrs.push_back(&c); }
  std::memset(s, 0, sizeof(*s));
  s->format = p->format.c_str();
  s->name = p->name.c_str();
  s->flags = ARROW_FLAG_NULLABLE;
  s->n_children = int64_t(nchildren);
  s->children = nchildren ? p->child_ptrs.data() : nullptr;
  s->release = release_schema;
  s->private_data = p;
}

}  // namespace

void export_batch(const OutBatch& b, ArrowArray* out, ArrowSchema* schema) {
  if (schema) {
    fill_schema(schema, "+s", "", b.cols.size());
    schema->flags = 0;
    for (size_t i = 0; i < b.cols.size(); i++) fill_schema(schema->children[i], format_of(b.cols[i].type), b.cols[i].name, 0);
  }
  if (!out) return;
  auto* top = new ArrayPriv;
  top->children.resize(b.cols.size());
  top->buffers.push_back(nullptr);  // struct validity
  for (size_t i = 0; i < b.cols.size(); i++) {
    const OutColumn& c = b.cols[i];
    auto* p = new ArrayPriv;
    ArrowArray& a = top->children[i];
    std::memset(&a, 0, sizeof(a));
    a.length = b.rows;
    a.null_count = c.null_count;
    // validity, [offsets], data: every buffer aliases the column's block
    p->keep = c.block;
    const uint8_t* base = c.block->p;
    p->buffers.push_back(c.null_count ? static_cast<const void*>(base + c.validity_off) : nullptr);
    if (c.type == PQ_T_UTF8) p->buffers.push_back(base + c.offsets_off);
    p->buffers.push_back(base + c.values_off);
    a.n_buffers = int64_t(p->buffers.size());
    a.buffers = p->buffers.data();
    a.release = release_array;
    a.private_data = p;
    top->child_ptrs.push_back(&a);
  }
  std::memset(out, 0, sizeof(*out));
  out->length = b.rows;
  out->null_count = 0;
  out->n_buffers = 1;
  out->buffers = top->buffers.data();
  out->n_children = int64_t(b.cols.size());
  out->children = top->child_ptrs.data();
  out->release = release_array;
  out->private_data = top;
}

}  // namespace pqb
