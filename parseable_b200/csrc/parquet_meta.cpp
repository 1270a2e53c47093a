#include "parquet_meta.hpp"

#include <cstring>
#include <stdexcept>

#include "thrift_compact.hpp"

namespace pqb {

namespace {

struct SchemaElem {
  int32_t type = -1;
  int32_t repetition = 0;  // 0 REQUIRED 1 OPTIONAL 2 REPEATED
  std::string name;
  int32_t num_children = 0;
  int32_t converted = -1;
  bool logical_string = false;
  int32_t ts_unit = -1;  // 0 ms 1 us 2 ns
  bool logical_date = false;
};

void parse_time_unit(ThriftReader& r, int32_t& unit) {
  int16_t last = 0, id; uint8_t t;
  while (r.field(last, id, t)) {
    if (t == T_STRUCT && id >= 1 && id <= 3) { unit = id - 1; r.skip_struct(); }
    else r.skip(t);
  }
}

void parse_logical_type(ThriftReader& r, SchemaElem& e) {
  int16_t last = 0, id; uint8_t t;
  while (r.field(last, id, t)) {
    if (id == 1 && t == T_STRUCT) { e.logical_string = true; r.skip_struct(); }
    else if (id == 6 && t == T_STRUCT) { e.logical_date = true; r.skip_struct(); }   // DATE
    else if (id == 8 && t == T_STRUCT) {  // TIMESTAMP
      int16_t l2 = 0, id2; uint8_t t2;
      while (r.field(l2, id2, t2)) {
        if (id2 == 2 && t2 == T_STRUCT) parse_time_unit(r, e.ts_unit);
        else r.skip(t2);
      }
    } else r.skip(t);
  }
}

SchemaElem parse_schema_elem(ThriftReader& r) {
  SchemaElem e;
  int16_t last = 0, id; uint8_t t;
  while (r.field(last, id, t)) {
    switch (id) {
      case 1: e.type = int32_t(r.zigzag()); break;
      case 3: e.repetition = int32_t(r.zigzag()); break;
      case 4: e.name = r.binary(); break;
      case 5: e.num_children = int32_t(r.zigzag()); break;
      case 6: e.converted = int32_t(r.zigzag()); break;
      case 10: if (t == T_STRUCT) parse_logical_type(r, e); else r.skip(t); break;
      default: r.skip(t);
    }
  }
  return e;
}

ColumnStats parse_stats(ThriftReader& r) {
  ColumnStats s;
  std::string old_min, old_max;
  bool has_old_min = false, has_old_max = false;
  int16_t last = 0, id; uint8_t t;
  while (r.field(last, id, t)) {
    switch (id) {
      case 1: old_max = r.binary(); has_old_max = true; break;
      case 2: old_min = r.binary(); has_old_min = true; break;
      case 3: s.null_count = r.zigzag(); break;
      case 5: s.max = r.binary(); s.has_max = true; break;
      case 6: s.min = r.binary(); s.has_min = true; break;
      default: r.skip(t);
    }
  }
  // The deprecated min / max (fields 1, 2) were written with SIGNED byte order for byte arrays by old writers:
  // they are only kept as a fallback here and only USED for signed-ordered physical types
  // (parse_column_meta drops them for BYTE_ARRAY / FIXED_LEN_BYTE_ARRAY / BOOLEAN below).
  if (!s.has_min && has_old_min) { s.min = old_min; s.has_min = true; s.deprecated_min_max = true; }
  if (!s.has_max && has_old_max) { s.max = old_max; s.has_max = true; s.deprecated_min_max = true; }
  return s;
}

ColumnChunkMeta parse_column_meta(ThriftReader& r) {
  ColumnChunkMeta c;
  int16_t last = 0, id; uint8_t t;
  while (r.field(last, id, t)) {
    switch (id) {
      case 1: c.type = int32_t(r.zigzag()); break;
      case 2: {
        uint32_t n; uint8_t et;
        r.list_header(n, et);
        for (uint32_t i = 0; i < n; i++) c.encodings.push_back(int32_t(r.zigzag()));
        break;
      }
      case 4: c.codec = int32_t(r.zigzag()); break;
      case 5: c.num_values = r.zigzag(); break;
      case 6: c.total_uncompressed_size = r.zigzag(); break;
      case 7: c.total_compressed_size = r.zigzag(); break;
      case 9: c.data_page_offset = r.zigzag(); break;
      case 11: c.dictionary_page_offset = r.zigzag(); break;
      case 12: if (t == T_STRUCT) c.stats = parse_stats(r); else r.skip(t); break;
      default: r.skip(t);
    }
  }
  // deprecated statistics order non-numeric types the wrong way round (signed bytes): never prune on them
  if (c.stats.deprecated_min_max && c.type != PT_INT32 && c.type != PT_INT64 && c.type != PT_FLOAT && c.type != PT_DOUBLE) {
    c.stats.has_min = c.stats.has_max = false;
    c.stats.min.clear();
    c.stats.max.clear();
  }
  return c;
}

ColumnChunkMeta parse_column_chunk(ThriftReader& r) {
  ColumnChunkMeta c;
  bool have = false;
  int16_t last = 0, id; uint8_t t;
  while (r.field(last, id, t)) {
    if (id == 3 && t == T_STRUCT) { c = parse_column_meta(r); have = true; }
    else r.skip(t);
  }
  if (!have) throw std::runtime_error("parquet: column chunk without meta_data");
  return c;
}

RowGroupMeta parse_row_group(ThriftReader& r) {
  RowGroupMeta g;
  int16_t last = 0, id; uint8_t t;
  while (r.field(last, id, t)) {
    switch (id) {
      case 1: {
        uint32_t n; uint8_t et;
        r.list_header(n, et);
        g.columns.reserve(n);
        for (uint32_t i = 0; i < n; i++) g.columns.push_back(parse_column_chunk(r));
        break;
      }
      case 3: g.num_rows = r.zigzag(); break;
      default: r.skip(t);
    }
  }
  return g;
}

// depth-first schema list -> leaves with definition / repetition levels
void build_leaves(const std::vector<SchemaElem>& el, size_t& pos, int def, int rep, int depth,
                  const std::string& prefix, std::vector<LeafColumn>& out) {
  const SchemaElem& e = el.at(pos++);
  int d = def + (e.repetition != 0 ? 1 : 0);
  int rp = rep + (e.repetition == 2 ? 1 : 0);
  std::string path = prefix.empty() ? e.name : prefix + "." + e.name;
  if (e.num_children > 0) {
    for (int i = 0; i < e.num_children; i++) build_leaves(el, pos, d, rp, depth + 1, path, out);
    return;
  }
  LeafColumn l;
  l.name = path;
  l.phys_type = e.type;
  l.max_def = d;
  l.max_rep = rp;
  l.depth = depth;
  // binary_as_string is on in the reference session (src/query/mod.rs:229-233), so a
  // bare BYTE_ARRAY reads as a string as well.
  l.is_string = e.type == PT_BYTE_ARRAY;
  if (e.type == PT_INT64) {
    if (e.ts_unit == 0 || (e.ts_unit < 0 && e.converted == 9)) l.is_timestamp_ms = true;
    else if (e.ts_unit > 0 || e.converted == 10) l.is_timestamp_other = true;
  }
  if (e.type == PT_INT32) l.is_date = e.logical_date || e.converted == 6;
  out.push_back(std::move(l));
}

}  // namespace

int FileMeta::find_leaf(const std::string& name) const {
  for (size_t i = 0; i < leaves.size(); i++)
    if (leaves[i].name == name) return int(i);
  return -1;
}

uint32_t footer_len_from_tail(const uint8_t tail[8]) {
  if (std::memcmp(tail + 4, "PAR1", 4) != 0) throw std::runtime_error("parquet: bad magic (encrypted or not parquet)");
  uint32_t n;
  std::memcpy(&n, tail, 4);
  return n;
}

FileMeta parse_file_metadata(const uint8_t* meta, uint64_t len) {
  FileMeta fm;
  try {
    ThriftReader r(meta, len);
    std::vector<SchemaElem> schema;
    int16_t last = 0, id; uint8_t t;
    while (r.field(last, id, t)) {
      switch (id) {
        case 2: {
          uint32_t n; uint8_t et;
          r.list_header(n, et);
          schema.reserve(n);
          for (uint32_t i = 0; i < n; i++) schema.push_back(parse_schema_elem(r));
          break;
        }
        case 3: fm.num_rows = r.zigzag(); break;
        case 4: {
          uint32_t n; uint8_t et;
          r.list_header(n, et);
          fm.row_groups.reserve(n);
          for (uint32_t i = 0; i < n; i++) fm.row_groups.push_back(parse_row_group(r));
          break;
        }
        case 6: fm.created_by = r.binary(); break;
        default: r.skip(t);
      }
    }
    if (schema.empty()) throw std::runtime_error("parquet: empty schema");
    // root: children only
    size_t pos = 1;
    for (int i = 0; i < schema[0].num_children; i++) build_leaves(schema, pos, 0, 0, 1, "", fm.leaves);
  } catch (const ThriftError& e) {
    throw std::runtime_error(std::string("parquet footer: ") + e.what());
  }
  for (auto& g : fm.row_groups)
    if (g.columns.size() != fm.leaves.size())
      throw std::runtime_error("parquet: row group column count != schema leaves");
  return fm;
}

FileMeta parse_footer(const uint8_t* file, uint64_t size) {
  if (size < 12 || std::memcmp(file, "PAR1", 4) != 0) throw std::runtime_error("parquet: bad header magic");
  uint32_t flen = footer_len_from_tail(file + size - 8);
  if (uint64_t(flen) + 12 > size) throw std::runtime_error("parquet: footer length out of range");
  return parse_file_metadata(file + size - 8 - flen, flen);
}

std::vector<PageInfo> walk_pages(const uint8_t* chunk, uint64_t len, int64_t num_values_expected) {
  std::vector<PageInfo> pages;
  uint64_t pos = 0;
  int64_t seen = 0;
  try {
    while (pos < len) {
      ThriftReader r(chunk + pos, len - pos);
      PageInfo pg;
      pg.offset_in_chunk = pos;
      int16_t last = 0, id; uint8_t t;
      while (r.field(last, id, t)) {
        switch (id) {
          case 1: pg.type = int32_t(r.zigzag()); break;
          case 2: pg.uncompressed_size = uint32_t(r.zigzag()); break;
          case 3: pg.compressed_size = uint32_t(r.zigzag()); break;
          case 5: {  // DataPageHeader
            int16_t l2 = 0, id2; uint8_t t2;
            while (r.field(l2, id2, t2)) {
              switch (id2) {
                case 1: pg.num_values = uint32_t(r.zigzag()); break;
                case 2: pg.encoding = int32_t(r.zigzag()); break;
                case 3: pg.def_encoding = int32_t(r.zigzag()); break;
                default: r.skip(t2);
              }
            }
            break;
          }
          case 7: {  // DictionaryPageHeader
            int16_t l2 = 0, id2; uint8_t t2;
            while (r.field(l2, id2, t2)) {
              switch (id2) {
                case 1: pg.num_values = uint32_t(r.zigzag()); break;
                case 2: pg.encoding = int32_t(r.zigzag()); break;
                default: r.skip(t2);
              }
            }
            break;
          }
          case 8: {  // DataPageHeaderV2
            pg.v2_compressed = true;
            int16_t l2 = 0, id2; uint8_t t2;
            while (r.field(l2, id2, t2)) {
              switch (id2) {
                case 1: pg.num_values = uint32_t(r.zigzag()); break;
                case 2: pg.v2_num_nulls = uint32_t(r.zigzag()); break;
                case 3: pg.v2_num_rows = uint32_t(r.zigzag()); break;
                case 4: pg.encoding = int32_t(r.zigzag()); break;
                case 5: pg.v2_def_len = uint32_t(r.zigzag()); break;
                case 6: pg.v2_rep_len = uint32_t(r.zigzag()); break;
                case 7: pg.v2_compressed = (t2 == T_TRUE); break;
                default: r.skip(t2);
              }
            }
            break;
          }
          default: r.skip(t);
        }
      }
      pg.header_len = uint32_t(r.consumed());
      if (pos + pg.header_len + pg.compressed_size > len)
        throw std::runtime_error("parquet: page runs past its column chunk");
      if (pg.type == PAGE_DATA || pg.type == PAGE_DATA_V2) seen += pg.num_values;
      pos += pg.header_len + pg.compressed_size;
      pages.push_back(pg);
    }
  } catch (const ThriftError& e) {
    throw std::runtime_error(std::string("parquet page header: ") + e.what());
  }
  if (seen != num_values_expected) throw std::runtime_error("parquet: page value counts do not add up to the chunk's");
  return pages;
}

}  // namespace pqb
