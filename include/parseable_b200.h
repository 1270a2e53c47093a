/*
 * parseable_b200.h — C ABI of the H100-native columnar query hot path for Parseable.
 *
 * This is the drop-in boundary of SURVEY.md §8(b).  Each entry point names the
 * reference interface it replaces (paths relative to /root/reference):
 *
 *   pq_init / pq_shutdown     QUERY_SESSION / QUERY_RUNTIME singletons        src/query/mod.rs:86-98
 *   pq_query_open             StandardTableProvider::scan +
 *                             create_parquet_physical_plan (+ the FilterExec /
 *                             AggregateExec DataFusion stacks on top)         src/query/stream_schema_provider.rs:114-189, 526-659
 *   pq_query_next             SendableRecordBatchStream::poll_next driven by
 *                             collect_partitioned / execute_stream_partitioned src/query/mod.rs:287, 310-334
 *   pq_query_stream           the same stream as ONE Arrow C stream object:
 *                             execute_stream_partitioned's merged
 *                             SendableRecordBatchStream (arrow-rs imports it
 *                             with ArrowArrayStreamReader)                     src/query/mod.rs:310-343
 *   pq_query_metrics          get_total_bytes_scanned ("bytes_scanned")        src/query/mod.rs:437-452
 *   pq_last_error             ExecuteError / DataFusionError::External         src/query/mod.rs:904-917
 *   pq_query_close            dropping the stream (cancellation)               src/query/mod.rs:300-340
 *   pq_table_*                the hot tier (local Parquet cache), here in HBM  src/hottier.rs:1541,1609
 *   pq_comm_*                 Partial -> RepartitionExec(Hash) -> Final merge,
 *                             here one NCCL all-reduce of partial tables       (DataFusion AggregateExec; SURVEY §8e)
 *
 * Plain C: pointers and sizes only.  Results leave through the Arrow C Data
 * Interface (ArrowArray / ArrowSchema below, ABI-identical to arrow/c/abi.h).
 * Inputs are borrowed for the duration of the call.  Every function is
 * re-entrant and thread-safe; a PqQuery may be driven from any thread but by one
 * thread at a time.  There is no CPU fallback: without a CUDA device every
 * compute entry point returns PQ_ERR_CUDA.
 */
#ifndef PARSEABLE_B200_H
#define PARSEABLE_B200_H

#include <stdint.h>
#include <stddef.h>

#ifdef __cplusplus
extern "C" {
#endif

/* ---- Arrow C Data Interface (https://arrow.apache.org/docs/format/CDataInterface.html) ---- */
#ifndef ARROW_C_DATA_INTERFACE
#define ARROW_C_DATA_INTERFACE
#define ARROW_FLAG_DICTIONARY_ORDERED 1
#define ARROW_FLAG_NULLABLE 2
#define ARROW_FLAG_MAP_KEYS_SORTED 4
struct ArrowSchema {
  const char* format;
  const char* name;
  const char* metadata;
  int64_t flags;
  int64_t n_children;
  struct ArrowSchema** children;
  struct ArrowSchema* dictionary;
  void (*release)(struct ArrowSchema*);
  void* private_data;
};
struct ArrowArray {
  int64_t length;
  int64_t null_count;
  int64_t offset;
  int64_t n_buffers;
  int64_t n_children;
  const void** buffers;
  struct ArrowArray** children;
  struct ArrowArray* dictionary;
  void (*release)(struct ArrowArray*);
  void* private_data;
};
#endif
/* ---- Arrow C Stream Interface (https://arrow.apache.org/docs/format/CStreamInterface.html) ---- */
#ifndef ARROW_C_STREAM_INTERFACE
#define ARROW_C_STREAM_INTERFACE
struct ArrowArrayStream {
  int (*get_schema)(struct ArrowArrayStream*, struct ArrowSchema* out);
  int (*get_next)(struct ArrowArrayStream*, struct ArrowArray* out); /* out->release == NULL: end of stream */
  const char* (*get_last_error)(struct ArrowArrayStream*);
  void (*release)(struct ArrowArrayStream*);
  void* private_data;
};
#endif

/* ---- status codes (SURVEY §8b "Error convention") ---- */
enum {
  PQ_OK = 0,
  PQ_END_OF_STREAM = 1,
  PQ_ERR_INVALID_ARG = -1,
  PQ_ERR_UNSUPPORTED = -2, /* plan/encoding not handled: the shim raises an error, it never falls back */
  PQ_ERR_IO = -3,
  PQ_ERR_CORRUPT = -4,
  PQ_ERR_CUDA = -5, /* CUDA or NCCL */
  PQ_ERR_OOM = -6
};

/* ---- literal / column value types ---- */
typedef enum {
  PQ_T_NULL = 0,
  PQ_T_BOOL = 1,
  PQ_T_I64 = 2,   /* Int64 */
  PQ_T_F64 = 3,   /* Float64 */
  PQ_T_UTF8 = 4,  /* Utf8 */
  PQ_T_TS_MS = 5, /* Timestamp(Millisecond, None) */
  /* Date32: days since 1970-01-01 (6 is PQ_T_TS_NS, planning only).  A Parquet INT32 leaf with the DATE logical or
   * converted type; every other INT32 leaf and FLOAT leaves stay PQ_ERR_UNSUPPORTED at open.  The flat store keeps the
   * values sign-extended to 8 bytes; results hand them out as Arrow Date32 ("tdD", 4-byte values) and JSON egress writes
   * a quoted "YYYY-MM-DD" (the date part of the Timestamp(ms) text of d * 86400000).  A literal carries the days in
   * PqLiteral.i64 (outside int32: PQ_ERR_INVALID_ARG).  PQ_OP_CMP compares a Date32 column with a Date32 literal only,
   * signed; either side against any other type returns PQ_ERR_UNSUPPORTED, and LIKE / REGEX are refused as on Int64.
   * Footer min / max (4 bytes) prune row groups.  GROUP BY keys, MIN / MAX (output Date32), COUNT, COUNT(DISTINCT) (by
   * value), ORDER BY / PARTITION BY terms and projections take it, in signed order; SUM, AVG, MEDIAN, PERCENTILE_CONT
   * and DATE_BIN over it return PQ_ERR_UNSUPPORTED, and so does a query that reads a Date32 column while some page of a
   * column it reads has no flat-store copy (PQB_FLAT_SCAN=0 included).  A Date32 column declared PQ_T_I64 or PQ_T_TS_MS
   * in columns[] returns PQ_ERR_INVALID_ARG. */
  PQ_T_DATE32 = 7
} PqType;

/* ---- predicate: flat postfix program (SURVEY §8a "Predicate vocabulary") ---- */
typedef enum {
  PQ_OP_CMP = 1,      /* push  col <cmp> literal          (NULL input -> NULL)        */
  PQ_OP_IS_NULL = 2,  /* push  col IS NULL                                            */
  PQ_OP_IS_NOT_NULL = 3,
  PQ_OP_LIKE = 4,     /* push  col LIKE pattern  ESCAPE '\'  (flags: NOT, case-insens) */
  PQ_OP_AND = 5,      /* pop 2, push Kleene AND                                       */
  PQ_OP_OR = 6,       /* pop 2, push Kleene OR                                        */
  PQ_OP_NOT = 7,      /* pop 1, push Kleene NOT                                       */
  PQ_OP_CONST = 8,    /* push literal TRUE/FALSE/NULL (lit.type BOOL or NULL)         */
  PQ_OP_REGEX = 9,    /* push  col ~ pattern  (flags: NOT, case-insens; see below)    */
  PQ_OP_IN = 10       /* push  col [NOT] IN (e1, ..., en)  (flags: NOT, has NULL; below) */
} PqOpKind;

typedef enum { PQ_EQ = 0, PQ_NE = 1, PQ_LT = 2, PQ_LE = 3, PQ_GT = 4, PQ_GE = 5 } PqCmp;

#define PQ_LIKE_NEGATED 1u
#define PQ_LIKE_CASE_INSENSITIVE 2u

/* PQ_OP_REGEX: `col ~ pattern` (`~*` with PQ_REGEX_CASE_INSENSITIVE, `!~` / `!~*` with PQ_REGEX_NEGATED), lit a PQ_T_UTF8
 * pattern.  DataFusion's regexp_is_match over the regex crate (1.12, regex-syntax 0.8), restated, not checked: an
 * unanchored search, TRUE when some substring matches.  `regexp_like(col, p, flags)` is the pattern `(?flags)p`.
 *   - NULL input -> NULL (so `!~` over NULL is NULL too); a column missing from a file reads as NULL; a column that is not
 *     Utf8 -> PQ_ERR_INVALID_ARG.  The empty pattern matches every non-NULL value, '' included.
 *   - `.` is any scalar value but `\n` (any under `s`); `^` / `$` are the text's start / end, and under `m` also after /
 *     before `\n` (`\r` is not special); `\A` / `\z` are always the text's start / end.
 *   - Syntax: UTF-8 literals; escapes \t \n \r \f \v \a \xHH \x{..} \uHHHH \u{..} \UHHHHHHHH \U{..}; an escaped ASCII
 *     punctuation character (or space) is itself, except \< and \>; groups (..) (?:..) (?P<n>..) (?<n>..); flag groups
 *     (?flags) and (?flags:..) over i m s U with `-`; alternation with empty branches; * + ? {n} {n,} {n,m}, greedy or
 *     lazy; classes [..] [^..] with ranges, escapes and Perl classes (a negated class matches `\n`); \d \s \w \D \S \W
 *     with their Unicode meanings (\p{Nd}; \p{White_Space}; Alphabetic + M + Nd + Pc + Join_Control); under `i` Unicode
 *     simple case folding orbits ((?i)k matches U+212A KELVIN SIGN).  Unicode tables are Unicode 15.0: code points first
 *     assigned later may classify differently from the regex crate's newer tables.
 *   - PQ_ERR_INVALID_ARG (the message names the byte position): unbalanced ( ) [ ], a quantifier with nothing to repeat,
 *     {m,n} with m > n, a reversed range, an unknown escape, backreferences, look-around, unknown or duplicate flags,
 *     duplicate group names, a pattern that is not UTF-8.
 *   - PQ_ERR_UNSUPPORTED: word boundaries \b \B \< \>, \p{..} / \P{..} classes, [[:alpha:]], nested classes and class
 *     set operations (&& -- ~~), the flags x R -u, {,m}, nesting deeper than 250, and patterns past the device DFA's caps
 *     (pattern 64 KiB, 65 536 NFA states, 4 096 DFA states, 1 MiB of table): "regular expression too large for the device
 *     DFA". */
#define PQ_REGEX_NEGATED 1u
#define PQ_REGEX_CASE_INSENSITIVE 2u

/* PQ_OP_IN: `col IN (e1, ..., en)` (`NOT IN` with PQ_IN_NEGATED), DataFusion's InList, restated, not checked: the Kleene
 * OR of `col = ei`, each exactly what PQ_OP_CMP with PQ_EQ computes, and NOT IN its Kleene NOT.
 *   - NULL input -> NULL; a column missing from a file reads as NULL.  PQ_IN_HAS_NULL: the list also holds a NULL, so a
 *     row that matches no element gives NULL, not FALSE (`x NOT IN (1, NULL)` is never TRUE).  Duplicates are allowed.
 *   - lit.type is the elements' PqType, lit.i64 their count n, and lit.str / lit.str_len the packed elements: for I64,
 *     TS_MS, DATE32, F64 (IEEE bits) and BOOL (0 / 1), n little-endian 8-byte values (str_len == 8 n); for UTF8, n
 *     entries of (u32 little-endian length, bytes), the PLAIN BYTE_ARRAY layout, which must fill str_len exactly.  n == 0
 *     only with PQ_IN_HAS_NULL: `x IN (NULL)` is NULL on every row.
 *   - Each element is coerced as a PQ_OP_CMP / PQ_EQ literal and refused the same way: Int64 / Timestamp(ms) take I64
 *     and TS_MS elements, and an F64 element that is integral (2^63 matches what `= 2^63` matches); Float64 takes F64
 *     and I64 elements and compares bits (-0.0 and 0.0 differ, a NaN matches only its own payload); Utf8 takes UTF8,
 *     bytewise; Date32 takes DATE32 only; Boolean takes BOOL.  An element the column cannot take returns the code
 *     PQ_OP_CMP returns for it, with a message that names the element's index.
 *   - PQ_ERR_INVALID_ARG: n == 0 without PQ_IN_HAS_NULL, n < 0, str_len that does not match n, str == NULL with n > 0,
 *     unknown flags.
 *   - PQ_ERR_UNSUPPORTED: more than 2^20 elements or 64 MiB of element bytes in one list, and a query that reads pages
 *     without a flat-store copy.
 *   - One IN is one leaf predicate whatever n is (two for an Int64 column whose list holds 2^63); PQ_IN_HAS_NULL, and
 *     2^63, add two postfix ops, and PQ_IN_NEGATED one, within the program's 40 ops and the stack depth of 8.
 * Dictionary pages answer the list once per dictionary entry; pages without a dictionary probe a hash set per row.  Row
 * groups whose footer [min, max] holds no element are pruned. */
#define PQ_IN_NEGATED 1u
#define PQ_IN_HAS_NULL 2u

typedef struct {
  int32_t type; /* PqType */
  int32_t _pad;
  int64_t i64;  /* BOOL (0/1), I64, TS_MS */
  double f64;   /* F64 */
  const char* str; /* UTF8 / LIKE pattern, not NUL-terminated */
  uint64_t str_len;
} PqLiteral;

typedef struct {
  int32_t kind;  /* PqOpKind */
  int32_t col;   /* index into PqQueryDesc.columns for leaf ops */
  int32_t cmp;   /* PqCmp for PQ_OP_CMP */
  uint32_t flags;
  PqLiteral lit;
} PqPredOp;

/* ---- aggregates (alert_enums.rs:216-223: Avg, Count, CountDistinct, Min, Max, Sum) ---- */
typedef enum {
  PQ_AGG_COUNT_STAR = 0,
  PQ_AGG_COUNT = 1,
  PQ_AGG_SUM = 2,
  /* MIN / MAX (DataFusion's min / max, restated, not checked): Int64, Timestamp(ms), Date32 (output Date32),
   * Float64 (totalOrder), and:
   *   Utf8: bytewise order, a prefix before any longer string (the order ORDER BY uses); output Utf8 with int32 offsets
   *     (the shim casts it to Utf8View, as for Utf8 keys), named "min(<col>)" / "max(<col>)".  Dictionary pages,
   *     PLAIN-fallback pages and DELTA_BYTE_ARRAY / DELTA_LENGTH_BYTE_ARRAY pages.
   *   Boolean: false < true (MIN is false if any input is false, MAX true if any is true); output Boolean.
   * NULL inputs are ignored, a group with no non-NULL input gets NULL, a column missing from a file reads as NULL, a global
   * aggregate over zero rows returns one row holding NULL.  They combine with every other aggregate (COUNT(DISTINCT) and
   * MEDIAN / PERCENTILE_CONT included), every GROUP BY form, ORDER BY [... LIMIT] and PQ_QUERY_ALLREDUCE.  Over Utf8 /
   * Boolean, PQ_ERR_UNSUPPORTED: pages without a flat-store copy (the k_scan path), a Utf8 column whose pages lack a
   * dictionary that the predicate also compares or matches (CMP / LIKE), and more than 2 GiB of result strings. */
  PQ_AGG_MIN = 3,
  PQ_AGG_MAX = 4,
  PQ_AGG_AVG = 5,
  /* COUNT(DISTINCT col) (the alerts' CountDistinct, src/alerts/mod.rs:245-251): Int64, never NULL, named
   * "count(distinct <col>)".  NULL inputs do not count; a group whose inputs are all NULL gets 0.  Values are
   * distinct as GROUP BY keys are: strings by bytes, integers / timestamps / booleans by value, Float64 by bit
   * pattern (-0.0 and 0.0 differ, as do NaNs with different payloads).  Utf8, Int64, Timestamp(ms), Date32, Float64 and
   * Boolean columns; refused (PQ_ERR_UNSUPPORTED) under PQ_QUERY_ALLREDUCE. */
  PQ_AGG_COUNT_DISTINCT = 6,
  /* Exact order statistics (DataFusion's median / percentile_cont, restated from DataFusion 53; its crates are not
   * vendored here, so the rules are restated, not checked).  Int64 and Float64 inputs (dictionary or PLAIN pages); Utf8,
   * Boolean, Timestamp and Date32 inputs return PQ_ERR_UNSUPPORTED.  NULL inputs are ignored and a column missing from a file
   * reads as NULL; a group with no non-NULL input gets NULL (a global aggregate over zero rows: one row holding NULL).
   * Values are sorted as ORDER BY sorts them: Int64 signed, Float64 by IEEE totalOrder (-NaN < -inf < ... < -0.0 < +0.0
   * < ... < +inf < +NaN).
   *   MEDIAN: output type = input type, named "median(<col>)".  n odd: the middle value.  n even: Int64 (lo + hi) as a
   *     wrapping i64 add, then / 2 truncating toward zero (add_wrapping(..).div_wrapping(2): the median of two values
   *     near INT64_MAX wraps); Float64 (lo + hi) / 2.
   *   PERCENTILE_CONT: p = agg_params[i] (finite, in [0, 1]); output Float64, named "percentile_cont(<col>, <p>)" with p
   *     in shortest round-trip form (std::to_chars: 0, 0.5, 0.95, 1).  h = p * (n - 1), lo = floor(h), f = h - lo over
   *     the sorted values as f64: v[lo] when f == 0, else v[lo] + f * (v[lo + 1] - v[lo]).
   * Float64 arithmetic on NaN follows x86-64 SSE (a NaN operand comes back quieted, the first one when both are NaN;
   * inf - inf is the default NaN 0xfff8000000000000), so the device and a CPU agree bit for bit.
   * Several of them over one column share one set of values and one sort.  They combine with every other aggregate but
   * COUNT(DISTINCT) (together: PQ_ERR_UNSUPPORTED), with every GROUP BY form and with ORDER BY.  PQ_QUERY_ALLREDUCE or
   * more than 2^32 - 1 values of one column: PQ_ERR_UNSUPPORTED; value and sort buffers above half the free HBM:
   * PQ_ERR_OOM. */
  PQ_AGG_MEDIAN = 7,
  PQ_AGG_PERCENTILE_CONT = 8
} PqAggFn;

typedef struct {
  int32_t fn;  /* PqAggFn */
  int32_t col; /* index into PqQueryDesc.columns; ignored for COUNT_STAR */
} PqAgg;

/* ---- computed GROUP BY keys: the counts / histogram API groups by DATE_BIN(<width>, p_timestamp, origin)
 *      (src/query/mod.rs:623-680); DATE_BIN over a Date32 column returns PQ_ERR_UNSUPPORTED ---- */
typedef enum { PQ_KEY_COLUMN = 0, PQ_KEY_DATE_BIN = 1 } PqKeyKind;
typedef struct {
  int32_t kind;       /* PqKeyKind */
  int32_t _pad;
  int64_t width_ms;   /* DATE_BIN: stride in milliseconds (> 0) */
  int64_t origin_ms;  /* DATE_BIN: origin, milliseconds since the epoch (the reference passes 1970-01-01) */
} PqKeyExpr;

/* ---- ORDER BY on the device: over aggregate results (the SortExec / TopK DataFusion puts above the AggregateExec), and
 *      ORDER BY ... LIMIT over the selected rows of a filter / projection scan (SortExec(fetch) above the scan) ----
 * Aggregate queries (n_aggs > 0, with or without GROUP BY and PQ_QUERY_ALLREDUCE) order by PQ_ORDER_KEY and
 * PQ_ORDER_AGG terms; a PQ_ORDER_COLUMN term there returns PQ_ERR_INVALID_ARG.  With ORDER BY, limit >= 0 keeps the
 * first `limit` rows of the ordered result (LIMIT 0: no rows, also for a global aggregate).  Without ORDER BY an
 * aggregate query ignores `limit`.
 * Scans (n_aggs == 0, with or without a projection) order by PQ_ORDER_COLUMN terms, whose column need not be projected,
 * and need a LIMIT: limit < 0 returns PQ_ERR_UNSUPPORTED.  The result is the first `limit` rows of the ordered
 * selection (LIMIT 0: no rows); the __row_id column of PQ_QUERY_EMIT_ROW_IDS follows the order, and without a
 * projection the result is the selected __row_ids in order.  rows_selected counts the rows before the cut.  Under
 * row-group or file sharding every shard orders and cuts its own selection, unless PQ_QUERY_ALLGATHER merges the
 * shards' rows (row-group sharding of one file list only): then every rank returns the whole table's first rows.
 * A PQ_ORDER_KEY / PQ_ORDER_AGG term on a scan returns PQ_ERR_UNSUPPORTED; ORDER BY with PQ_QUERY_COUNT_ONLY
 * PQ_ERR_INVALID_ARG; more than 2^32 - 1 selected rows, or pages without a flat-store copy, PQ_ERR_UNSUPPORTED.
 * Every query: an out-of-range index or an unknown target returns PQ_ERR_INVALID_ARG, more than 8 terms
 * PQ_ERR_UNSUPPORTED.
 * Value order (arrow-ord's sort, restated): Int64 / Timestamp(ms) signed; Float64 by IEEE totalOrder (-NaN < -inf <
 * ... < -0.0 < +0.0 < ... < +inf < +NaN); Utf8 bytewise, a prefix before any longer string; Boolean false < true; a
 * DATE_BIN key by bin start; an aggregate by its output value (AVG: the Float64 the result holds).  NULLs (NULL keys,
 * NULL aggregates of all-NULL groups, NULL column values, a column missing from a file) go first with
 * PQ_ORDER_NULLS_FIRST and last without it, in either direction.
 * Ties: rows equal on every term keep the order the same query returns without ORDER BY, and at the LIMIT boundary the
 * earlier of them are kept: the result is a stable sort of the unordered result, cut to the limit.  For a scan that
 * order is file order, then row order.  For an aggregate it is ascending group slot, and every rank of an all-reduced
 * query returns the same rows.  Slot order follows the group ids a table numbers when it is opened (a resident table
 * keeps them); under a hashed GROUP BY (a key space wider than 2^26) the slots are hash-table cells and their order, so
 * the order of tied rows, may differ from one query to the next.  Except under PQ_QUERY_ALLREDUCE: there the ranks'
 * tables are merged into ascending wide group id (the mixed-radix id of the key tuple in the numbering the ranks agreed
 * on), so tied rows come out in the same order on every rank, and on every run over the same resident tables.
 * Paths (all stable on that order): <= 4096 rows one CTA sorts them; a key that packs into one 64-bit word with
 * LIMIT <= 4096 takes a radix select of the LIMIT-th key; anything else an LSD radix sort. */
typedef enum { PQ_ORDER_KEY = 0, PQ_ORDER_AGG = 1, PQ_ORDER_COLUMN = 2 } PqOrderTarget;
#define PQ_ORDER_DESC 1u
#define PQ_ORDER_NULLS_FIRST 2u
typedef struct {
  int32_t target;  /* PqOrderTarget */
  int32_t index;   /* into group_by[] (PQ_ORDER_KEY), aggs[] (PQ_ORDER_AGG) or columns[] (PQ_ORDER_COLUMN) */
  uint32_t flags;  /* PQ_ORDER_DESC | PQ_ORDER_NULLS_FIRST */
  int32_t _pad;
} PqOrderBy;

/* ---- ROW_NUMBER() OVER (PARTITION BY ... ORDER BY ...) cut to a rank range, on the device: the top N rows of every
 *      partition (BoundedWindowAggExec(ROW_NUMBER / COUNT(*) OVER) + FilterExec(rn range) above the aggregate or scan) ----
 * The window's ORDER BY is the query's order_by array; partition_by holds the PARTITION BY terms in the same PqOrderBy
 * form, checked the same way: an aggregate query takes PQ_ORDER_KEY terms (GROUP BY keys, DATE_BIN included), a scan
 * PQ_ORDER_COLUMN terms (the column need not be projected).  A partition term's flags order the partitions in the
 * output.  Partition and order terms together are at most 8 (more: PQ_ERR_UNSUPPORTED).
 * Partitions: two rows share one when every partition term has the same value and NULL flag, GROUP BY equality: NULLs
 * are one partition, Float64 compares by bit pattern (-0.0 and 0.0 are two partitions, so are NaNs of different
 * payloads), Utf8 by bytes, a DATE_BIN key by bin.
 * Ranking: row_number rn counts 1, 2, ... within a partition in the order of the order_by terms; ties keep the order
 * the query has without a window (as ORDER BY states above: slot order, or file then row order), and with no order_by
 * terms that order is the ranking.  Under a hashed GROUP BY the order of tied rows may differ from one query to the next
 * (not under PQ_QUERY_ALLREDUCE: see ORDER BY above).
 * Output: the rows with offset < rn <= offset + fetch (fetch < 0: no upper bound), ordered by the partition terms and
 * then the window's order; `limit` (>= 0) then keeps the first `limit` of them (the outer LIMIT), for aggregates too.
 * PQ_WINDOW_ROW_NUMBER appends an Int64 column "row_number", PQ_WINDOW_PARTITION_ROWS an Int64 column "partition_rows"
 * (COUNT(*) OVER (PARTITION BY ...): the partition's rows before the cut), in that order: after the keys and aggregates,
 * or after a scan's projection and __row_id.  Neither is ever NULL.
 * Scans: a window needs no `limit`; the caps of a scan ORDER BY hold (2^32 - 1 selected rows, 2^31 projected rows, a
 * flat-store copy of every page read).  Under row-group or file sharding every shard ranks and cuts its own selection;
 * merging the shards' rows is the caller's (PQ_QUERY_ALLGATHER refuses a window).  Aggregates: the window runs after the all-reduce (every rank of a
 * PQ_QUERY_ALLREDUCE query returns the same rows), and takes every aggregate ORDER BY takes as a term.
 * rows_selected and groups_total count the rows before any cut; the window's kernels count into order_ms and
 * kernel_launches.  Errors: offset < 0, unknown flags, a bad term index or target, or a window with PQ_QUERY_COUNT_ONLY
 * return PQ_ERR_INVALID_ARG (a PQ_ORDER_KEY / PQ_ORDER_AGG partition term on a scan: PQ_ERR_UNSUPPORTED, as for order_by).
 * Paths: without partition terms the window is ORDER BY ... LIMIT offset + fetch with the first `offset` rows dropped;
 * with them every row is sorted by (partition terms, order terms), and one host round trip reads the kept count. */
#define PQ_WINDOW_ROW_NUMBER 1u       /* append Int64 "row_number" (1-based, within the partition) */
#define PQ_WINDOW_PARTITION_ROWS 2u   /* append Int64 "partition_rows" = COUNT(*) OVER (PARTITION BY ...), before the cut */
typedef struct {
  const PqOrderBy* partition_by;  /* PARTITION BY terms, most significant first; same targets as order_by */
  uint32_t n_partition_by;        /* 0: one partition (ROW_NUMBER() OVER (ORDER BY ...)) */
  uint32_t flags;                 /* PQ_WINDOW_ROW_NUMBER | PQ_WINDOW_PARTITION_ROWS */
  int64_t offset;                 /* keep rows whose row number rn satisfies offset < rn <= offset + fetch; >= 0 */
  int64_t fetch;                  /* < 0: no upper bound */
} PqWindow;

/* ---- inputs ---- */
typedef struct {
  const char* path;  /* file to read, or NULL when buf is given */
  const uint8_t* buf; /* whole Parquet file image in host memory, or NULL */
  uint64_t size;      /* bytes of buf (ignored for path) */
} PqFile;

typedef struct {
  const char* name; /* matched against the Parquet schema BY NAME (streams.rs:1024-1037) */
  int32_t type;     /* PqType expected by the plan; a missing column reads as all-NULL */
  int32_t _pad;
} PqColumn;

typedef struct PqTable PqTable; /* HBM-resident encoded column chunks */
typedef struct PqQuery PqQuery;

typedef struct {
  /* scan inputs: either a resident table, or a file list (host buffers / paths) */
  const PqTable* table;
  const PqFile* files;
  uint32_t n_files;

  /* every column the plan references; all indices below point into this array */
  const PqColumn* columns;
  uint32_t n_columns;

  /* output projection for non-aggregate queries (TableProvider::scan `projection`) */
  const int32_t* projection;
  uint32_t n_projection;

  /* WHERE: postfix program; n_pred == 0 means no filter */
  const PqPredOp* pred;
  uint32_t n_pred;

  /* GROUP BY + aggregates; n_aggs == 0 means a filter/projection scan */
  const int32_t* group_by;
  uint32_t n_group_by;
  const PqAgg* aggs;
  uint32_t n_aggs;

  int64_t limit;       /* < 0: none (TableProvider::scan `limit`) */
  uint32_t batch_size; /* rows per output batch; 0 -> 20000 (stream_schema_provider.rs:160) */

  /* row-group sharding for multi-GPU: this process scans row groups g with
   * g % shard_count == shard_index (mirrors partitioned_files round-robin, :351-364) */
  uint32_t shard_index;
  uint32_t shard_count; /* 0 or 1: no sharding */
  uint32_t flags;

  /* NULL, or n_group_by entries: how group_by[k] becomes a key (plain column | DATE_BIN of a Timestamp / Int64 column);
   * a DATE_BIN key comes back as a Timestamp(ms) column named date_bin(<column>) holding the bin start */
  const PqKeyExpr* group_exprs;

  /* ORDER BY terms, most significant first (see PqOrderBy); n_order_by == 0: none */
  const PqOrderBy* order_by;
  uint32_t n_order_by;
  uint32_t _pad2;

  /* NULL, or n_aggs entries: a parameter per aggregate.  Only PQ_AGG_PERCENTILE_CONT reads its entry, the fraction p
   * (finite, in [0, 1]; otherwise, or NULL here, the call returns PQ_ERR_INVALID_ARG) */
  const double* agg_params;

  /* NULL, or ROW_NUMBER() OVER (PARTITION BY ... ORDER BY order_by) cut to a rank range (see PqWindow) */
  const PqWindow* window;
} PqQueryDesc;

#define PQ_QUERY_COUNT_ONLY 1u    /* filter scan: only rows_selected is wanted, emit no batches */
/* PQ_QUERY_ALLREDUCE, aggregate: every rank returns the whole table's groups.  A key space of up to 2^26 group ids:
 * the ranks all-reduce their dense partial tables.  A wider one (a hashed GROUP BY, at any number of ranks, one
 * included): every rank lists the groups its hash table holds, the lists are all-gathered and merged on the device in
 * rank order.  The merge combines the cells as the all-reduce does: wrapping add (the row count, COUNT, non-null
 * counters, Int64 SUM), f64 add in rank order ((r0 + r1) + r2 ... for Float64 SUM / AVG), signed min / max (MIN / MAX
 * on their cell encodings); its rows come out in ascending wide group id.  Refused alike by every rank:
 *   PQ_ERR_UNSUPPORTED  more than 2^26 merged groups, or a rank's hash table ran full (the message names the rank); a
 *                       rank with pages that have no flat-store copy (named likewise); the hashed table would exceed
 *                       24 GiB for the rows of every rank
 *   PQ_ERR_CORRUPT      a rank met a corrupt page (named)
 *   PQ_ERR_OOM          the exchange and merge buffers exceed half the smallest free HBM of any rank (named)
 * COUNT(DISTINCT), MEDIAN and PERCENTILE_CONT are refused under this flag. */
#define PQ_QUERY_ALLREDUCE 2u
#define PQ_QUERY_EMIT_ROW_IDS 4u  /* filter scan: append a UInt64 `__row_id` column (global row ordinal) */
/* PQ_QUERY_ALLGATHER, a filter / projection scan with ORDER BY (PQ_ORDER_COLUMN terms) and limit >= 0, with or without
 * a projection and PQ_QUERY_EMIT_ROW_IDS, over a table that every rank opened from the SAME file list and shards by row
 * group (shard_count = the communicator's ranks, shard_index = the rank; a resident table opened so, or a file-list
 * query with those shard_* fields): every rank returns the first `limit` rows of the WHOLE table's ordered selection,
 * bit for bit and in the order one rank returns them for the same query over the unsharded list (ties in global
 * __row_id order: file order, then row order); rows_selected is the whole table's selected total on every rank.
 * __row_id is the row's ordinal over the file list the table was opened with: under file sharding (each rank opening
 * its own files) every rank's ordinals start at 0 and would collide, so the flag refuses that layout.
 * Each rank orders its own selection and keeps its first `limit` rows; one all-gather hands every rank those rows'
 * encoded terms and global row ids, every rank orders the union alike, each output row is projected by the rank that
 * holds it and the ranks' result blocks are summed (every byte is written by one rank only).  Utf8 terms sort by their
 * rank in the numbering the ranks agree on (as GROUP BY keys under PQ_QUERY_ALLREDUCE).  With one rank the result is
 * the one without the flag.
 * Errors: without pq_comm_init_rank, on an aggregate query or with PQ_QUERY_COUNT_ONLY PQ_ERR_INVALID_ARG; without
 * ORDER BY or with a window PQ_ERR_UNSUPPORTED.  Refused alike by every rank, the message naming the rank:
 *   PQ_ERR_UNSUPPORTED  a table not sharded by row group over the communicator (shard_count != ranks or
 *                       shard_index != rank), or ranks whose file lists hold different numbers of rows; a rank's shard
 *                       holds pages this scan cannot take (found before the scan: pages without a flat-store copy, ...);
 *                       more than 2^32 - 1 selected rows on a rank; ranks x the most rows any rank keeps past
 *                       2^32 - 1; more than 2^31 output rows; projected strings above 2 GiB
 *   PQ_ERR_CORRUPT      a rank met a corrupt page
 *   PQ_ERR_OOM          a rank's own sort and the exchange and merge buffers exceed half that rank's free HBM */
#define PQ_QUERY_ALLGATHER 8u

typedef struct {
  uint64_t bytes_scanned;   /* compressed bytes of the column chunks read (plan metric "bytes_scanned") */
  uint64_t rows_scanned;    /* rows in the row groups that survived pruning */
  uint64_t rows_selected;   /* rows passing the predicate (before an ORDER BY ... LIMIT cut) */
  uint64_t row_groups_total;
  uint64_t row_groups_pruned;
  uint64_t algorithmic_bytes; /* uncompressed encoded bytes of the pages read + bitmap bytes written */
  uint64_t h2d_bytes;
  uint64_t d2h_bytes;
  uint64_t kernel_launches;
  double device_ms;         /* CUDA-event time of the device work of this query */
  double scan_kernel_ms;    /* CUDA-event time of the fused scan kernel alone */
  uint64_t groups;          /* output groups (aggregate queries) */
  double host_ms;           /* wall time of pq_query_open (planning + uploads + device work + result copy) */
  double upload_ms;         /* of which: footer parse, page walk and H2D of the column chunks (file-list queries) */
  double allreduce_ms;      /* CUDA-event time of the NCCL all-reduce of the partial tables (PQ_QUERY_ALLREDUCE); a
                               hashed GROUP BY: its exchange, both all-gathers and the merge kernels, without the one
                               host round trip between them.  A scan under PQ_QUERY_ALLGATHER: its exchange record,
                               the candidates' all-gather, the merge kernels and sort, the projection by owner and
                               the reductions of the result block, without the host round trips between them */
  uint64_t groups_total;    /* aggregate queries: groups before the ORDER BY ... LIMIT cut (== groups without ORDER BY) */
  double order_ms;          /* CUDA-event time of the ORDER BY kernels, without the one host round trip between them
                               (0 without ORDER BY) */
  double percentile_ms;     /* CUDA-event time of the MEDIAN / PERCENTILE_CONT kernels (sort and pick), without the host round
                               trip of each sort (0 without them) */
} PqMetrics;

/* ---- lifecycle ---- */
int pq_init(const int* device_ids, int n); /* n == 0: current device / device 0 */
void pq_shutdown(void);
const char* pq_version(void);
int pq_device_count(void);

/* ---- HBM-resident table (hot tier) ---- */
int pq_table_open(const PqFile* files, uint32_t n_files, const char* const* columns, uint32_t n_columns,
                  uint32_t shard_index, uint32_t shard_count, PqTable** out);
uint64_t pq_table_rows(const PqTable*);
uint64_t pq_table_device_bytes(const PqTable*);
void pq_table_close(PqTable*);

/* ---- query ---- */
int pq_query_open(const PqQueryDesc* desc, PqQuery** out);
int pq_query_next(PqQuery* q, int partition, struct ArrowArray* out, struct ArrowSchema* out_schema);
/* All remaining batches of a partition as one Arrow C stream.  The stream borrows the query: release
 * it (or drain it) before pq_query_close; the batches it produced stay valid on their own. */
int pq_query_stream(PqQuery* q, int partition, struct ArrowArrayStream* out);
int pq_query_metrics(PqQuery* q, PqMetrics* out);
/* The whole result (every batch, whatever pq_query_next already handed out) as JSON text formatted on the GPU: what
 * QueryResponse::to_json builds from the batches on the CPU (src/response.rs:31-58, src/utils/arrow/mod.rs:49-64:
 * arrow_json::ArrayWriter conventions -- NULL values leave their key out, Timestamp(ms) as ISO-8601, floats shortest
 * round-trip).  flags 0: one JSON array `[{...},{...}]`; PQ_JSON_LINES: one object per line (NDJSON).  *out stays valid
 * until the next pq_query_json call on q or pq_query_close. */
#define PQ_JSON_LINES 1u
int pq_query_json(PqQuery* q, uint32_t flags, const char** out, uint64_t* len);
const char* pq_last_error(PqQuery* q); /* q == NULL: last error of the calling thread */
void pq_query_close(PqQuery* q);

/* ---- host helpers (no GPU work) ---- */
/* Page-locked host memory for file images: PqFile.buf inside such a block is DMA'd straight
 * to HBM, other host memory is staged through the library's own pinned slices. */
void* pq_host_alloc(uint64_t bytes);
void pq_host_free(void* p);
/* JSON description of a Parquet file as the host metadata layer parsed it (schema leaves, row
 * groups, column chunks, every page header).  Returns the JSON length (excluding NUL), or a
 * negative status; writes at most cap bytes.  Replaces nothing at run time: it exists so the
 * footer/page-header reader can be checked against an independent reader without a GPU. */
int64_t pq_file_describe(const PqFile* file, char* out, uint64_t cap);

/* ---- scan planning on the C side (no GPU work): which manifests / files reach the scan ----
 * What StandardTableProvider::scan does above create_parquet_physical_plan:
 *   time bounds of the filters      src/query/stream_schema_provider.rs:884-940 (extract_timestamp_bound, PartialTimeFilter)
 *   Snapshot::manifests             src/catalog/snapshot.rs:40-71
 *   is_overlapping_query            src/query/stream_schema_provider.rs:750-775
 *   is_within_staging_window        :842-864
 *   can_be_pruned / satisfy_constraints   :955-1043 (TypedStatistics, src/catalog/column.rs:52-68)
 *   collect_from_snapshot           :449-510 (newest first, pruning, LIMIT truncation)
 *   partitioned_files + statistics merge   :351-446, src/catalog/column.rs:70-198
 *   supports_filters_pushdown       :665-683, 866-882
 * The Rust host may keep doing this itself; these entry points let a shim hand the manifest over instead. */
#define PQ_T_TS_NS 6 /* planning only: Timestamp(Nanosecond) literal in PqLiteral.i64 */

typedef struct {
  const char* column; /* NULL: the filter is not `column <cmp> literal` (never prunes, never a time bound) */
  int32_t cmp;        /* PqCmp */
  int32_t _pad;
  PqLiteral lit;
} PqPlanFilter;

typedef enum { PQ_STAT_NONE = 0, PQ_STAT_BOOL = 1, PQ_STAT_INT = 2, PQ_STAT_FLOAT = 3, PQ_STAT_STRING = 4 } PqStatKind;
typedef struct {
  const char* column;
  int32_t kind; /* PqStatKind; PQ_STAT_NONE: the manifest holds no statistics for the column */
  int32_t _pad;
  int64_t min_i, max_i; /* BOOL (0/1), INT */
  double min_f, max_f;  /* FLOAT */
  const char* min_s;    /* STRING, not NUL-terminated */
  uint64_t min_s_len;
  const char* max_s;
  uint64_t max_s_len;
} PqColumnStat;

typedef struct {
  const char* path;
  uint64_t num_rows;
  uint64_t file_size;
  const PqColumnStat* stats;
  uint32_t n_stats;
  uint32_t _pad;
} PqManifestFile;

typedef struct {
  int64_t time_lower_ns; /* naive UTC, nanoseconds since the epoch */
  int64_t time_upper_ns;
} PqManifestItem;

typedef enum { PQ_BOUND_LOW = 0, PQ_BOUND_HIGH = 1, PQ_BOUND_EQ = 2 } PqBoundKind;
typedef struct {
  int32_t kind;     /* PqBoundKind */
  int32_t included; /* LOW / HIGH: the bound itself belongs to the range */
  int64_t time_ns;
} PqTimeBound;

/* One bound per filter that is `column <cmp> timestamp literal` (a Utf8 literal only on `time_partition`).
 * Returns the number of bounds written (<= n), or a negative status. */
int32_t pq_plan_time_bounds(const PqPlanFilter* filters, uint32_t n, const char* time_partition, PqTimeBound* out);
/* keep[i] = 1 when manifest item i can hold rows inside every bound */
int32_t pq_plan_manifests(const PqManifestItem* items, uint32_t n, const PqTimeBound* bounds, uint32_t n_bounds, uint8_t* keep);
int32_t pq_plan_is_overlapping_query(const PqManifestItem* items, uint32_t n, const PqTimeBound* bounds, uint32_t n_bounds);
int32_t pq_plan_within_staging_window(const PqTimeBound* bounds, uint32_t n_bounds, int64_t now_ns);
/* files in manifest order (oldest first) -> out_index: the files to scan, newest first, without those whose
 * statistics rule a filter out, cut once `limit` rows are covered (limit < 0: none).  Returns how many. */
int64_t pq_plan_collect_files(const PqManifestFile* files, uint32_t n_files, const PqPlanFilter* filters, uint32_t n_filters,
                              int64_t limit, uint32_t* out_index);
/* a [min, max] of one column merged over two files; returns 1 and fills *out, or 0 when the ranges cannot be merged
 * (different kinds, an inverted or NaN float range): the planner then skips min / max for that column */
int32_t pq_plan_merge_stat(const PqColumnStat* a, const PqColumnStat* b, PqColumnStat* out);
/* exact[i] = 1: the scan alone answers filter i (minute-aligned time comparison), 0: Inexact */
int32_t pq_plan_pushdown(const PqPlanFilter* filters, uint32_t n, uint8_t* exact);

/* ---- multi-GPU: one process per GPU, NCCL communicator owned by the library ---- */
#define PQ_COMM_ID_BYTES 128
int pq_comm_unique_id(uint8_t id[PQ_COMM_ID_BYTES]);
int pq_comm_init_rank(const uint8_t id[PQ_COMM_ID_BYTES], int nranks, int rank);
int pq_comm_destroy(void);

#ifdef __cplusplus
}
#endif
#endif /* PARSEABLE_B200_H */
