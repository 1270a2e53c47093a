// Host-side Parquet metadata layer: footer (FileMetaData) and page headers.
// Stands in for parquet 58.1.0's footer/page-header readers that DataFusion's
// ParquetOpener drives for the reference (SURVEY.md §8 row a10;
// call site /root/reference/src/query/stream_schema_provider.rs:146-184).
#pragma once
#include <cstdint>
#include <string>
#include <vector>

namespace pqb {

enum PhysType : int32_t {
  PT_BOOLEAN = 0, PT_INT32 = 1, PT_INT64 = 2, PT_INT96 = 3, PT_FLOAT = 4, PT_DOUBLE = 5,
  PT_BYTE_ARRAY = 6, PT_FLBA = 7
};
enum Encoding : int32_t {
  ENC_PLAIN = 0, ENC_PLAIN_DICTIONARY = 2, ENC_RLE = 3, ENC_BIT_PACKED = 4,
  ENC_DELTA_BINARY_PACKED = 5, ENC_DELTA_LENGTH_BYTE_ARRAY = 6, ENC_DELTA_BYTE_ARRAY = 7,
  ENC_RLE_DICTIONARY = 8, ENC_BYTE_STREAM_SPLIT = 9
};
enum Codec : int32_t {
  CODEC_UNCOMPRESSED = 0, CODEC_SNAPPY = 1, CODEC_GZIP = 2, CODEC_LZO = 3, CODEC_BROTLI = 4,
  CODEC_LZ4 = 5, CODEC_ZSTD = 6, CODEC_LZ4_RAW = 7
};
enum PageType : int32_t { PAGE_DATA = 0, PAGE_INDEX = 1, PAGE_DICTIONARY = 2, PAGE_DATA_V2 = 3 };

struct ColumnStats {
  bool has_min = false, has_max = false;
  std::string min, max;  // PLAIN-encoded min_value / max_value
  int64_t null_count = -1;
  bool deprecated_min_max = false;   // taken from the deprecated Statistics.min / max (fields 1, 2)
};

struct ColumnChunkMeta {
  int32_t type = -1;
  int32_t codec = 0;
  std::vector<int32_t> encodings;
  int64_t num_values = 0;
  int64_t total_uncompressed_size = 0;
  int64_t total_compressed_size = 0;
  int64_t data_page_offset = 0;
  int64_t dictionary_page_offset = -1;
  ColumnStats stats;
  // byte range of the chunk in the file
  int64_t start() const {
    return (dictionary_page_offset > 0 && (data_page_offset <= 0 || dictionary_page_offset < data_page_offset))
               ? dictionary_page_offset : data_page_offset;
  }
};

struct RowGroupMeta {
  int64_t num_rows = 0;
  std::vector<ColumnChunkMeta> columns;  // one per leaf, schema order
};

struct LeafColumn {
  std::string name;  // dotted path; top-level columns are just their name
  int32_t phys_type = -1;
  int32_t max_def = 0, max_rep = 0;
  int32_t depth = 1;
  bool is_string = false;        // converted UTF8 / logical STRING (or plain BYTE_ARRAY with binary_as_string)
  bool is_timestamp_ms = false;  // logical TIMESTAMP(MILLIS) / converted TIMESTAMP_MILLIS
  bool is_timestamp_other = false;
  bool is_date = false;          // logical DATE / converted DATE (INT32 days since 1970-01-01: Arrow Date32)
};

struct FileMeta {
  int64_t num_rows = 0;
  std::string created_by;
  std::vector<LeafColumn> leaves;
  std::vector<RowGroupMeta> row_groups;
  int find_leaf(const std::string& name) const;
};

struct PageInfo {
  int32_t type = 0;              // PageType
  uint32_t header_len = 0;       // bytes of the thrift header
  uint32_t compressed_size = 0;  // payload bytes in the file
  uint32_t uncompressed_size = 0;
  uint32_t num_values = 0;
  int32_t encoding = 0;
  int32_t def_encoding = ENC_RLE;
  // v2 only
  uint32_t v2_def_len = 0, v2_rep_len = 0, v2_num_nulls = 0, v2_num_rows = 0;
  bool v2_compressed = false;
  uint64_t offset_in_chunk = 0;  // of the header
};

// Parse the footer of a whole-file image.  Throws std::runtime_error on corruption.
FileMeta parse_footer(const uint8_t* file, uint64_t size);
// Footer location for path sources: returns footer length given the last 8 bytes.
uint32_t footer_len_from_tail(const uint8_t tail[8]);
FileMeta parse_file_metadata(const uint8_t* meta, uint64_t len);

// Walk the page headers of one column chunk (chunk = bytes [start, start+total_compressed_size)).
std::vector<PageInfo> walk_pages(const uint8_t* chunk, uint64_t len, int64_t num_values_expected);

}  // namespace pqb
