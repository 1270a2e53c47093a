"""Host-side mirror of Parseable's query surface over the C ABI.

Names follow the reference (paths relative to /root/reference):

* ``Query`` / ``execute``           src/query/mod.rs:143-157, 260-343
* ``StandardTableProvider.scan``   src/query/stream_schema_provider.rs:526-659
  (``projection``, ``filters``, ``limit``) plus ``aggregate`` for the
  FilterExec + AggregateExec stack DataFusion puts above the scan
* ``TimeRange`` filter injection   src/query/mod.rs:774-833 (``p_timestamp >= start AND p_timestamp < end``)

Everything here only builds a ``PqQueryDesc`` and hands it to
``libparseable_b200.so``; results come back through the Arrow C Data Interface
into pyarrow.  There is no CPU execution path in this module.
"""
from __future__ import annotations

import ctypes as C
import datetime as _dt
import re
import struct
from dataclasses import dataclass, field
from typing import Any, Iterable, Sequence

import pyarrow as pa

from . import _lib as L

DEFAULT_TIMESTAMP_KEY = "p_timestamp"  # src/event/mod.rs DEFAULT_TIMESTAMP_KEY
_EPOCH_DAY = _dt.date(1970, 1, 1)   # day 0 of a Date32 literal
_DATE_LITERAL = re.compile(r"\d{4}-\d{2}-\d{2}")   # DATE 'YYYY-MM-DD'


class QueryError(RuntimeError):
    """ExecuteError / DataFusionError::External of the reference (src/query/mod.rs:904-917)."""

    def __init__(self, code: int, msg: str):
        super().__init__(f"{L.ERR_NAMES.get(code, code)}: {msg}")
        self.code = code
        self.message = msg


# ----------------------------------------------------------------------------- expressions
@dataclass
class Expr:
    kind: str                      # 'col' 'lit' 'cmp' 'and' 'or' 'not' 'is_null' 'is_not_null' 'like' 'regex' 'in'
    args: tuple = ()
    op: int = 0
    flags: int = 0

    def _bin(self, other, op):
        return Expr("cmp", (self, _lit(other)), op)

    def __eq__(self, o): return self._bin(o, L.PQ_EQ)       # type: ignore[override]
    def __ne__(self, o): return self._bin(o, L.PQ_NE)       # type: ignore[override]
    def __lt__(self, o): return self._bin(o, L.PQ_LT)
    def __le__(self, o): return self._bin(o, L.PQ_LE)
    def __gt__(self, o): return self._bin(o, L.PQ_GT)
    def __ge__(self, o): return self._bin(o, L.PQ_GE)
    def __and__(self, o): return Expr("and", (self, o))
    def __or__(self, o): return Expr("or", (self, o))
    def __invert__(self): return Expr("not", (self,))
    def __hash__(self): return id(self)
    def is_null(self): return Expr("is_null", (self,))
    def is_not_null(self): return Expr("is_not_null", (self,))

    def like(self, pattern: str, negated=False, case_insensitive=False):
        f = (L.PQ_LIKE_NEGATED if negated else 0) | (L.PQ_LIKE_CASE_INSENSITIVE if case_insensitive else 0)
        return Expr("like", (self, Expr("lit", (pattern,))), flags=f)

    def ilike(self, pattern: str, negated=False):
        return self.like(pattern, negated, True)

    def regex(self, pattern: str, negated=False, case_insensitive=False):
        """``col ~ pattern`` (``~*``, ``!~``, ``!~*``): an unanchored regular-expression search (PQ_OP_REGEX)."""
        f = (L.PQ_REGEX_NEGATED if negated else 0) | (L.PQ_REGEX_CASE_INSENSITIVE if case_insensitive else 0)
        return Expr("regex", (self, Expr("lit", (pattern,))), flags=f)

    def isin(self, values: Iterable, negated=False):
        """``col [NOT] IN (values)`` (PQ_OP_IN): the Kleene OR of ``col = v``; ``None`` among the values is a NULL element."""
        return Expr("in", (self, tuple(values)), flags=L.PQ_IN_NEGATED if negated else 0)


def col(name: str) -> Expr:
    return Expr("col", (name,))


def lit(v: Any) -> Expr:
    return Expr("lit", (v,))


def _lit(v) -> Expr:
    return v if isinstance(v, Expr) else Expr("lit", (v,))


@dataclass
class Timestamp:
    """A TimestampMillisecond literal (what transform() injects, stream_schema_provider.rs:722-748)."""
    ms: int


_FLIP = {L.PQ_LT: L.PQ_GT, L.PQ_GT: L.PQ_LT, L.PQ_LE: L.PQ_GE, L.PQ_GE: L.PQ_LE, L.PQ_EQ: L.PQ_EQ, L.PQ_NE: L.PQ_NE}


def shortest_repr(v: float) -> str:
    """``std::to_chars(double)``: the shortest digits that round-trip, written fixed or scientific, whichever is shorter
    (fixed on a tie): 0, 0.5, 0.95, 1, 1e-05.  The C side names PERCENTILE_CONT columns with it."""
    from decimal import Decimal
    r = repr(float(v))
    if r in ("inf", "-inf", "nan"):
        return r
    sign, dig, exp = Decimal(r).as_tuple()
    digits = "".join(map(str, dig))
    stripped = digits.rstrip("0")
    exp += len(digits) - len(stripped)
    digits = stripped or "0"
    if digits == "0":
        exp = 0
    if exp >= 0:
        fixed = digits + "0" * exp
    elif len(digits) + exp > 0:
        fixed = digits[:len(digits) + exp] + "." + digits[len(digits) + exp:]
    else:
        fixed = "0." + "0" * -(len(digits) + exp) + digits
    e = exp + len(digits) - 1
    sci = digits[0] + ("." + digits[1:] if len(digits) > 1 else "") + f"e{'-' if e < 0 else '+'}{abs(e):02d}"
    return ("-" if sign else "") + (fixed if len(fixed) <= len(sci) else sci)


@dataclass
class Agg:
    fn: str           # count_star count sum min max avg count_distinct median percentile_cont
    column: str | None = None
    p: float | None = None   # percentile_cont: the fraction

    @property
    def name(self) -> str:
        """The result column's name (DataFusion's display names, lower case)."""
        if self.fn == "count_star":
            return "count(*)"
        if self.fn == "count_distinct":
            return f"count(distinct {self.column})"
        if self.fn == "percentile_cont":
            return f"percentile_cont({self.column}, {shortest_repr(self.p)})"
        return f"{self.fn}({self.column})"


_AGG_CODE = {"count_star": L.PQ_AGG_COUNT_STAR, "count": L.PQ_AGG_COUNT, "sum": L.PQ_AGG_SUM,
             "min": L.PQ_AGG_MIN, "max": L.PQ_AGG_MAX, "avg": L.PQ_AGG_AVG, "count_distinct": L.PQ_AGG_COUNT_DISTINCT,
             "median": L.PQ_AGG_MEDIAN, "percentile_cont": L.PQ_AGG_PERCENTILE_CONT}


@dataclass(frozen=True)
class DateBin:
    """GROUP BY DATE_BIN(width, column, origin): the counts / histogram API of the reference
    (src/query/mod.rs:623-680 builds `DATE_BIN('1m', p_timestamp, TIMESTAMP '1970-01-01 00:00:00+00')`)."""
    width_ms: int
    column: str = DEFAULT_TIMESTAMP_KEY
    origin_ms: int = 0

    @property
    def name(self) -> str:
        return f"date_bin({self.column})"


_INTERVALS = {"s": 1000, "m": 60_000, "h": 3_600_000, "d": 86_400_000}


def date_bin(width: str | int, column: str = DEFAULT_TIMESTAMP_KEY, origin_ms: int = 0) -> DateBin:
    """``date_bin("5m")``: widths like the reference's '1m' | '5m' | '1h' | '1d', or milliseconds."""
    if isinstance(width, str):
        width = int(width[:-1]) * _INTERVALS[width[-1]]
    return DateBin(int(width), column, origin_ms)


def count_star(): return Agg("count_star")
def count(c): return Agg("count", c)
def sum_(c): return Agg("sum", c)
def min_(c): return Agg("min", c)
def max_(c): return Agg("max", c)
def avg(c): return Agg("avg", c)
def count_distinct(c): return Agg("count_distinct", c)
def median(c): return Agg("median", c)
def percentile_cont(c, p): return Agg("percentile_cont", c, float(p))


# ----------------------------------------------------------------------------- descriptor builder
class _Desc:
    """Keeps every ctypes object alive for the duration of the call."""

    def __init__(self):
        self.keep: list = []
        self.columns: list[str] = []

    def col_index(self, name: str) -> int:
        if name not in self.columns:
            self.columns.append(name)
        return self.columns.index(name)

    def literal(self, v) -> L.PqLiteral:
        out = L.PqLiteral()
        if v is None:
            out.type = L.PQ_T_NULL
        elif isinstance(v, bool):
            out.type, out.i64 = L.PQ_T_BOOL, int(v)
        elif isinstance(v, Timestamp):
            out.type, out.i64 = L.PQ_T_TS_MS, int(v.ms)
        elif isinstance(v, _dt.date) and not isinstance(v, _dt.datetime):
            out.type, out.i64 = L.PQ_T_DATE32, (v - _EPOCH_DAY).days
        elif isinstance(v, int):
            out.type, out.i64 = L.PQ_T_I64, v
        elif isinstance(v, float):
            out.type, out.f64 = L.PQ_T_F64, v
        elif isinstance(v, (str, bytes)):
            b = v.encode() if isinstance(v, str) else v
            buf = C.create_string_buffer(b, len(b) + 1)
            self.keep.append(buf)
            out.type = L.PQ_T_UTF8
            out.str = C.cast(buf, C.c_char_p)
            out.str_len = len(b)
        else:
            raise TypeError(f"unsupported literal {v!r}")
        return out

    def in_list(self, col: int, values: list, flags: int) -> L.PqPredOp:
        """One PQ_OP_IN over elements of one literal type, packed as the header lays them out."""
        t = self.literal(values[0]).type if values else L.PQ_T_NULL
        if t == L.PQ_T_UTF8:
            bs = [v.encode() if isinstance(v, str) else v for v in values]
            data = b"".join(struct.pack("<I", len(b)) + b for b in bs)
            return self._in_op(col, flags, t, len(bs), data)
        if any(isinstance(v, int) and not -(1 << 63) <= v < (1 << 63) for v in values):
            raise QueryError(L.PQ_ERR_INVALID_ARG, "IN list element outside int64")
        lits = [self.literal(v) for v in values]
        if t == L.PQ_T_F64:
            data = struct.pack(f"<{len(lits)}d", *(x.f64 for x in lits))
        else:
            data = struct.pack(f"<{len(lits)}q", *(x.i64 for x in lits))
        return self._in_op(col, flags, t, len(lits), data)

    def _in_op(self, col: int, flags: int, t: int, n: int, data: bytes) -> L.PqPredOp:
        buf = C.create_string_buffer(data, len(data) + 1)
        self.keep.append(buf)
        lit = L.PqLiteral()
        lit.type, lit.i64, lit.str, lit.str_len = t, n, C.cast(buf, C.c_char_p), len(data)
        return L.PqPredOp(kind=L.PQ_OP_IN, col=col, flags=flags, lit=lit)

    def compile_pred(self, e: Expr, ops: list):
        if e.kind in ("and", "or"):
            self.compile_pred(e.args[0], ops)
            self.compile_pred(e.args[1], ops)
            ops.append(L.PqPredOp(kind=L.PQ_OP_AND if e.kind == "and" else L.PQ_OP_OR))
        elif e.kind == "not":
            self.compile_pred(e.args[0], ops)
            ops.append(L.PqPredOp(kind=L.PQ_OP_NOT))
        elif e.kind in ("is_null", "is_not_null"):
            c = e.args[0]
            if c.kind != "col":
                raise QueryError(L.PQ_ERR_UNSUPPORTED, "IS NULL on a non-column expression")
            ops.append(L.PqPredOp(kind=L.PQ_OP_IS_NULL if e.kind == "is_null" else L.PQ_OP_IS_NOT_NULL,
                                  col=self.col_index(c.args[0])))
        elif e.kind in ("like", "regex"):
            c, p = e.args
            if c.kind != "col":
                raise QueryError(L.PQ_ERR_UNSUPPORTED, f"{e.kind.upper()} on a non-column expression")
            if p.kind != "lit" or not isinstance(p.args[0], (str, bytes)):
                raise QueryError(L.PQ_ERR_UNSUPPORTED, f"{e.kind.upper()} with a pattern that is not a string literal")
            ops.append(L.PqPredOp(kind=L.PQ_OP_LIKE if e.kind == "like" else L.PQ_OP_REGEX, col=self.col_index(c.args[0]),
                                  flags=e.flags, lit=self.literal(p.args[0])))
        elif e.kind == "cmp":
            a, b = e.args
            op = e.op
            if a.kind == "lit" and b.kind == "col":
                a, b, op = b, a, _FLIP[op]
            if a.kind != "col" or b.kind != "lit":
                raise QueryError(L.PQ_ERR_UNSUPPORTED, "only column <op> literal comparisons are pushed to the GPU")
            ops.append(L.PqPredOp(kind=L.PQ_OP_CMP, col=self.col_index(a.args[0]), cmp=op, lit=self.literal(b.args[0])))
        elif e.kind == "in":
            c, values = e.args
            if c.kind != "col":
                raise QueryError(L.PQ_ERR_UNSUPPORTED, "IN on a non-column expression")
            ci = self.col_index(c.args[0])
            # one PQ_OP_IN per literal type, OR'd together; the NULL element and NOT go with the whole list
            groups: dict = {}
            for v in values:
                if v is not None:
                    t = L.PQ_T_UTF8 if isinstance(v, (str, bytes)) else self.literal(v).type
                    groups.setdefault(t, []).append(v)
            has_null = L.PQ_IN_HAS_NULL if any(v is None for v in values) else 0
            if not groups:
                if not has_null:
                    raise QueryError(L.PQ_ERR_INVALID_ARG, "IN with an empty list")
                groups[L.PQ_T_NULL] = []
            for i, vs in enumerate(groups.values()):
                ops.append(self.in_list(ci, vs, has_null if i == 0 else 0))
                if i:
                    ops.append(L.PqPredOp(kind=L.PQ_OP_OR))
            if e.flags & L.PQ_IN_NEGATED:
                if len(groups) == 1:
                    ops[-1].flags |= L.PQ_IN_NEGATED
                else:
                    ops.append(L.PqPredOp(kind=L.PQ_OP_NOT))
        elif e.kind == "lit":
            ops.append(L.PqPredOp(kind=L.PQ_OP_CONST, lit=self.literal(e.args[0])))
        else:
            raise QueryError(L.PQ_ERR_UNSUPPORTED, f"expression {e.kind} in a predicate")


def _order_flags(direction, nulls_first) -> int:
    """PqOrderBy flags of ``asc`` / ``desc`` and NULLS FIRST (True) / LAST (False) / the default (None)."""
    if str(direction).lower() not in ("asc", "desc"):
        raise QueryError(L.PQ_ERR_INVALID_ARG, f"ORDER BY direction {direction!r}: asc or desc")
    desc = str(direction).lower() == "desc"
    if nulls_first is None:
        nulls_first = desc               # DataFusion: ASC -> NULLS LAST, DESC -> NULLS FIRST
    return (L.PQ_ORDER_DESC if desc else 0) | (L.PQ_ORDER_NULLS_FIRST if nulls_first else 0)


def _order_term(group_by: list, aggs: list, term) -> tuple[int, int, int]:
    """One ORDER BY term of ``aggregate`` -> (PqOrderTarget, index, PqOrderBy flags)."""
    item, direction, *rest = term
    flags = _order_flags(direction, rest[0] if rest else None)
    if isinstance(item, Agg):
        if item in aggs:
            return L.PQ_ORDER_AGG, aggs.index(item), flags
    else:
        for i, k in enumerate(group_by):
            if item == k or (isinstance(k, DateBin) and item == k.name):
                return L.PQ_ORDER_KEY, i, flags
        for i, a in enumerate(aggs):
            if item == a.name:
                return L.PQ_ORDER_AGG, i, flags
    raise QueryError(L.PQ_ERR_INVALID_ARG, f"ORDER BY {item!r}: neither a GROUP BY key nor an aggregate of the query")


@dataclass
class Window:
    """``ROW_NUMBER() OVER (PARTITION BY partition_by ORDER BY <the query's order_by>)`` cut to ``offset < rn <= offset +
    fetch`` (``fetch=None``: no upper bound), ranked on the GPU (PqWindow).  ``partition_by`` items are written like
    ``order_by`` items, ``item`` or ``(item, "asc" | "desc"[, nulls_first])``: GROUP BY keys (names or DateBin) for
    ``aggregate``, column names for ``scan``; their direction orders the partitions in the output.  ``row_number`` /
    ``partition_rows`` append the Int64 columns ``row_number`` and ``partition_rows`` (COUNT(*) OVER the partition)."""
    partition_by: Sequence = ()
    offset: int = 0
    fetch: int | None = None
    row_number: bool = False
    partition_rows: bool = False


def _window_desc(w: "Window", terms: list):
    """The PqWindow of ``w`` over its partition terms [(PqOrderTarget, index, flags)] (the caller keeps both alive)."""
    arr = (L.PqOrderBy * max(1, len(terms)))()
    for i, (target, index, fl) in enumerate(terms):
        arr[i].target, arr[i].index, arr[i].flags = target, index, fl
    pw = L.PqWindow(partition_by=arr if terms else None, n_partition_by=len(terms),
                    flags=(L.PQ_WINDOW_ROW_NUMBER if w.row_number else 0) | (L.PQ_WINDOW_PARTITION_ROWS if w.partition_rows else 0),
                    offset=int(w.offset), fetch=-1 if w.fetch is None else int(w.fetch))
    return pw, arr


def _partition_items(w: "Window") -> list:
    """``partition_by`` items as order terms: a bare item is ascending with the default NULL placement."""
    return [tuple(p) if isinstance(p, (tuple, list)) else (p, "asc") for p in w.partition_by]


_ARROW_TO_PQ = {pa.int64(): L.PQ_T_I64, pa.float64(): L.PQ_T_F64, pa.string(): L.PQ_T_UTF8,
                pa.large_string(): L.PQ_T_UTF8, pa.bool_(): L.PQ_T_BOOL, pa.timestamp("ms"): L.PQ_T_TS_MS}


def _pq_type(t: pa.DataType | None) -> int:
    if t is None:
        return L.PQ_T_NULL
    if pa.types.is_dictionary(t):
        t = t.value_type
    if pa.types.is_timestamp(t):
        return L.PQ_T_TS_MS
    if pa.types.is_date32(t):
        return L.PQ_T_DATE32
    return _ARROW_TO_PQ.get(t, L.PQ_T_NULL)


# ----------------------------------------------------------------------------- files / tables
class HostFile:
    """A Parquet file image in host memory (page-locked when ``pinned``) or a path."""

    def __init__(self, path: str | None = None, data: bytes | None = None, pinned: bool = False):
        self.path = path
        self._pinned_ptr = None
        self._buf = None
        self.size = 0
        if data is not None or pinned:
            if data is None:
                with open(path, "rb") as f:
                    data = f.read()
            self.size = len(data)
            if pinned:
                lib = L.load()
                p = lib.pq_host_alloc(self.size)
                if not p:
                    raise QueryError(L.PQ_ERR_OOM, "pq_host_alloc failed")
                C.memmove(p, data, self.size)
                self._pinned_ptr = p
            else:
                self._buf = C.create_string_buffer(data, len(data))

    def as_pq(self) -> L.PqFile:
        f = L.PqFile()
        if self._pinned_ptr:
            f.buf, f.size = self._pinned_ptr, self.size
        elif self._buf is not None:
            f.buf, f.size = C.cast(self._buf, C.c_void_p), self.size
        else:
            self._path_b = self.path.encode()
            f.path = self._path_b
        return f

    def close(self):
        if self._pinned_ptr:
            L.load().pq_host_free(self._pinned_ptr)
            self._pinned_ptr = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def _files_array(files: Sequence[HostFile | str]):
    hfs = [f if isinstance(f, HostFile) else HostFile(path=f) for f in files]
    arr = (L.PqFile * len(hfs))(*[h.as_pq() for h in hfs])
    return hfs, arr


def _staging_image(batches: list) -> "HostFile":
    """In-RAM staging record batches -> one Parquet file image (newest row first)."""
    import io

    import pyarrow.parquet as pq

    from . import synth
    rev = [b.take(pa.array(range(b.num_rows - 1, -1, -1), pa.int64())) for b in reversed(batches)]
    t = pa.Table.from_batches(rev)
    buf = io.BytesIO()
    kw = synth.parseable_writer_kwargs(t.column_names, time_col=DEFAULT_TIMESTAMP_KEY)
    pq.write_table(t, buf, row_group_size=synth.ROW_GROUP, **kw)
    return HostFile(data=buf.getvalue())


def field_stats(provider: "StandardTableProvider", field: str, max_field_statistics: int = 50, filters: Iterable[Expr] = ()):
    """Field statistics of one column like the reference's per-upload job (src/storage/field_stats.rs:298-330):
    ``GROUP BY field -> COUNT(*) ORDER BY count(*) DESC LIMIT max_field_statistics`` is one GPU query: the groups are
    ordered and cut on the device (ties keep the scan's order, as ROW_NUMBER() over a stable sort does), the total is
    the selected rows and the distinct count the groups before the cut -- what SUM / COUNT OVER () compute.
    Returns (total_count, distinct_count, [(value, count), ...] for the max_field_statistics most frequent values)."""
    res = provider.aggregate([field], [count_star()], list(filters), order_by=[(count_star(), "desc")], limit=max_field_statistics)
    top = []
    if res.batches:
        t = res.table()
        top = list(zip(t[field].to_pylist(), t["count(*)"].to_pylist()))
    return res.metrics["rows_selected"], res.metrics["groups_total"], top


def dataset_stats(provider: "StandardTableProvider", dataset_name: str, fields: Sequence[str] | None = None, offset: int = 0,
                  limit: int = 5) -> dict:
    """The dataset-stats API over a pstats-shaped table (``get_dataset_stats`` / ``build_stats_sql``,
    src/storage/field_stats.rs:530-757 in the reference) in two GPU queries:
      * ``GROUP BY field_name, distinct_value`` -> ``SUM(count)`` over the dataset's rows with a non-NULL distinct value
        (and one of ``fields``), ranked per field by ``SUM DESC, distinct_value ASC`` and cut to ``offset < rn <= offset
        + limit`` on the device, with each field's distinct count (COUNT(*) OVER (PARTITION BY field_name));
      * the ``field_totals``: ``GROUP BY field_name`` -> ``SUM(field_stats_count)`` over the dataset's rows.
    Their join on the field name is the host's.  Returns ``{field: {"field_count", "distinct_count",
    "distinct_values": {value: count}}}``, the values in rank order."""
    fname, dval, dcount = "field_stats_field_name", "field_stats_distinct_stats_distinct_value", "field_stats_distinct_stats_count"
    in_dataset = col("dataset_name") == dataset_name
    flt = [in_dataset, col(dval).is_not_null()]
    if fields:
        any_field = None
        for f in fields:
            any_field = (col(fname) == f) if any_field is None else (any_field | (col(fname) == f))
        flt.append(any_field)
    total = sum_(dcount)
    ranked = provider.aggregate([fname, dval], [total], flt, order_by=[(total, "desc"), (dval, "asc")],
                                window=Window(partition_by=[fname], offset=offset, fetch=limit, partition_rows=True))
    totals = provider.aggregate([fname], [sum_("field_stats_count")], [in_dataset])
    field_count = {}
    if totals.batches:
        t = totals.table()
        field_count = dict(zip(t[fname].to_pylist(), t["sum(field_stats_count)"].to_pylist()))
    out: dict = {}
    if ranked.batches:
        t = ranked.table()
        for f, v, c, dc in zip(t[fname].to_pylist(), t[dval].to_pylist(), t[total.name].to_pylist(), t["partition_rows"].to_pylist()):
            if f is None or f not in field_count:   # the inner join (NULL joins nothing)
                continue
            st = out.setdefault(f, {"field_count": field_count[f], "distinct_count": dc, "distinct_values": {}})
            st["distinct_values"][v] = c
    return out


class DeviceTable:
    """Encoded column chunks resident in HBM (pq_table_open): the hot tier of
    src/hottier.rs, one level closer to the kernels."""

    def __init__(self, files: Sequence[HostFile | str], columns: Sequence[str], shard_index=0, shard_count=1):
        lib = L.load()
        self._hfs, arr = _files_array(files)
        names = (C.c_char_p * len(columns))(*[c.encode() for c in columns])
        h = C.c_void_p()
        rc = lib.pq_table_open(arr, len(self._hfs), names, len(columns), shard_index, shard_count, C.byref(h))
        if rc != L.PQ_OK:
            raise QueryError(rc, (lib.pq_last_error(None) or b"").decode())
        self.handle = h
        self.columns = list(columns)

    @property
    def rows(self) -> int:
        return L.load().pq_table_rows(self.handle)

    @property
    def device_bytes(self) -> int:
        return L.load().pq_table_device_bytes(self.handle)

    def close(self):
        if self.handle:
            L.load().pq_table_close(self.handle)
            self.handle = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


# ----------------------------------------------------------------------------- execution
@dataclass
class QueryResult:
    batches: list[pa.RecordBatch]
    metrics: dict
    fields: list[str] = field(default_factory=list)
    json_text: bytes | None = None      # the result as JSON text formatted on the GPU (pq_query_json), when asked for

    def to_json(self, with_fields: bool = False, fill_null: bool = False):
        """QueryResponse::to_json (src/response.rs:31-58) over the GPU-formatted records: the list of row objects,
        optionally with every field present (NULL filled in) and wrapped with the field list."""
        import json as _json
        if self.json_text is None:
            raise ValueError("run the query with json='array' or json='lines'")
        txt = self.json_text.decode()
        rows = _json.loads(txt) if txt.startswith("[") else [_json.loads(line) for line in txt.splitlines() if line]
        if fill_null:
            for r in rows:
                for f in self.fields:
                    r.setdefault(f, None)
        return {"fields": self.fields, "records": rows} if with_fields else rows

    def table(self) -> pa.Table:
        if not self.batches:
            return pa.table({})
        return pa.Table.from_batches(self.batches)


class StandardTableProvider:
    """scan()/aggregate() over a file list or a resident DeviceTable.

    ``schema`` maps column name -> Arrow type the plan expects (the table schema
    Parseable keeps per stream); columns the plan names but a file lacks read as NULL.
    """

    def __init__(self, source: DeviceTable | Sequence[HostFile | str], schema: pa.Schema | dict | None = None,
                 shard_index: int = 0, shard_count: int = 1, staging_batches: Sequence[pa.RecordBatch] = (),
                 staging_parquet: Sequence[str] = ()):
        # ---- get_staging_execution_plan (stream_schema_provider.rs:242-298): data still in staging ----
        # staging Parquet files: newest first by file name, scanned like any other file; in-RAM staging batches: reversed
        # (batch order and row order, `reversed_mem_table` :686-695) and turned into ONE in-memory Parquet image with the
        # stream's writer properties -- the conversion Parseable itself runs when it flushes staging
        # (streams.rs:572-631) -- so that the GPU path stays the only reader.  They come first in the file list, like
        # the reference's plan order (staging arrow, staging parquet, then hot tier / object store).
        extra: list = []
        if staging_batches:
            extra.append(_staging_image(list(staging_batches)))
        extra += sorted(staging_parquet, reverse=True)
        if extra:
            if isinstance(source, DeviceTable):
                raise QueryError(L.PQ_ERR_INVALID_ARG, "staging data joins a file list, not a resident table")
            source = extra + list(source)
        self.source = source
        if isinstance(schema, pa.Schema):
            schema = {f.name: f.type for f in schema}
        self.schema = schema or {}
        self.shard_index, self.shard_count = shard_index, shard_count

    # -- TableProvider::scan -------------------------------------------------
    def scan(self, projection: Sequence[str] | None = None, filters: Iterable[Expr] = (), limit: int | None = None,
             count_only: bool = False, row_ids: bool | None = None, batch_size: int = 0, flags: int = 0,
             poll: bool = False, json: str | None = None, order_by: Sequence | None = None,
             window: Window | None = None) -> QueryResult:
        """``projection``: the columns to return for the selected rows (TableProvider::scan's projection);
        without one the scan returns the selected row ordinals (``__row_id``).  ``row_ids=True`` appends
        ``__row_id`` to a projection.  ``order_by``: ``[(column, "asc" | "desc"[, nulls_first]), ...]``, most
        significant first, with a ``limit``: the first ``limit`` selected rows in that order, selected and sorted on
        the GPU (the SortExec(fetch) / TopK above the scan); the columns need not be projected.  ``nulls_first=None``
        follows the same default as ``aggregate``.  ``window``: the top rows of every partition of columns
        (Window), ranked by ``order_by``; it needs no ``limit``, which then cuts its output."""
        def term(c, direction, *rest):
            return L.PQ_ORDER_COLUMN, c, _order_flags(direction, rest[0] if rest else None)
        order = [term(*t) for t in (order_by or [])]
        part = [term(*t) for t in _partition_items(window)] if window is not None else None
        f = 0
        if row_ids is None:
            row_ids = not projection
        if count_only:
            f |= L.PQ_QUERY_COUNT_ONLY
        elif row_ids:
            f |= L.PQ_QUERY_EMIT_ROW_IDS
        win = {} if window is None else {"window": window, "partition": part}
        return self._run(list(filters), [], [], list(projection or []), limit, batch_size, f | flags, poll=poll, json=json, order=order,
                         **win)

    # -- FilterExec + AggregateExec folded into the same call ----------------
    def aggregate(self, group_by: Sequence[str], aggs: Sequence[Agg], filters: Iterable[Expr] = (),
                  batch_size: int = 0, flags: int = 0, json: str | None = None, order_by: Sequence | None = None,
                  limit: int | None = None, window: Window | None = None) -> QueryResult:
        """``order_by``: ``[(item, "asc" | "desc"[, nulls_first]), ...]``, most significant first, sorted on the GPU
        (the SortExec / TopK above the AggregateExec).  An item is a GROUP BY key (its name or DateBin), an aggregate
        (an Agg of ``aggs`` or its output name).  ``nulls_first=None`` follows DataFusion's default (restated, not
        checked here): ASC puts NULLs last, DESC first.  With ``order_by``, ``limit`` keeps the first rows of the
        ordered result; without it the C ABI ignores ``limit`` on an aggregate.  ``window``: the top groups of every
        partition of GROUP BY keys (Window), ranked by ``order_by``; ``limit`` then cuts its output."""
        group_by, aggs = list(group_by), list(aggs)
        order = [_order_term(group_by, aggs, t) for t in (order_by or [])]
        win = {}
        if window is not None:
            part = [_order_term(group_by, aggs, t) for t in _partition_items(window)]
            for (target, _, _), (item, *_) in zip(part, _partition_items(window)):
                if target != L.PQ_ORDER_KEY:
                    raise QueryError(L.PQ_ERR_INVALID_ARG, f"PARTITION BY {item!r}: not a GROUP BY key of the query")
            win = {"window": window, "partition": part}
        return self._run(list(filters), group_by, aggs, [], limit, batch_size, flags, json=json, order=order, **win)

    def count_distinct(self, group_by: Sequence[str], column: str, filters: Iterable[Expr] = ()) -> pa.Table:
        """``SELECT keys, COUNT(DISTINCT column)`` (Parseable's alerts use it: src/alerts/alert_enums.rs:216-223), one
        native aggregate (PQ_AGG_COUNT_DISTINCT).  NULLs do not count, an empty input yields 0 for the global form."""
        name = f"count(distinct {column})"
        res = self.aggregate(list(group_by), [count_distinct(column)], filters)
        if res.batches:
            return res.table()
        return pa.table({**{k: pa.array([], pa.null()) for k in group_by}, name: pa.array([], pa.int64())})

    def _run(self, filters, group_by, aggs, projection, limit, batch_size, flags, poll: bool = False, json: str | None = None,
             order: Sequence[tuple] = (), window: Window | None = None, partition: Sequence[tuple] | None = None) -> QueryResult:
        lib = L.load()
        d = _Desc()
        ops: list = []
        pred = None
        for e in filters:                      # conjunction(filters), stream_schema_provider.rs:126
            pred = e if pred is None else Expr("and", (pred, e))
        if pred is not None:
            d.compile_pred(pred, ops)
        gb = [d.col_index(c.column if isinstance(c, DateBin) else c) for c in group_by]
        gx = None
        if any(isinstance(c, DateBin) for c in group_by):
            gx = (L.PqKeyExpr * len(group_by))()
            for i, c in enumerate(group_by):
                if isinstance(c, DateBin):
                    gx[i].kind, gx[i].width_ms, gx[i].origin_ms = L.PQ_KEY_DATE_BIN, c.width_ms, c.origin_ms
        ag = []
        for a in aggs:
            ag.append(L.PqAgg(fn=_AGG_CODE[a.fn], col=d.col_index(a.column) if a.column is not None else -1))
        # agg_params: PERCENTILE_CONT's fraction, one entry per aggregate (the others ignore theirs)
        params = (C.c_double * len(aggs))(*[a.p if a.p is not None else 0.0 for a in aggs]) if any(a.fn == "percentile_cont" for a in aggs) else None
        proj = [d.col_index(c) for c in projection]
        # PQ_ORDER_COLUMN terms name their column: it joins the referenced columns
        order = [(t, d.col_index(i) if isinstance(i, str) else i, fl) for t, i, fl in order]
        if window is not None:   # partition terms resolve like order terms
            partition = [(t, d.col_index(i) if isinstance(i, str) else i, fl) for t, i, fl in (partition or [])]

        desc = L.PqQueryDesc()
        hfs = None
        if isinstance(self.source, DeviceTable):
            desc.table = self.source.handle
        else:
            hfs, arr = _files_array(self.source)
            desc.files, desc.n_files = arr, len(hfs)
        names = [c.encode() for c in d.columns]
        cols = (L.PqColumn * max(1, len(names)))()
        for i, n in enumerate(names):
            cols[i].name = n
            cols[i].type = _pq_type(self.schema.get(d.columns[i]))
        desc.columns, desc.n_columns = cols, len(names)
        if ops:
            arr_ops = (L.PqPredOp * len(ops))(*ops)
            desc.pred, desc.n_pred = arr_ops, len(ops)
        if gb:
            arr_gb = (C.c_int32 * len(gb))(*gb)
            desc.group_by, desc.n_group_by = arr_gb, len(gb)
            if gx is not None:
                desc.group_exprs = gx
        if ag:
            arr_ag = (L.PqAgg * len(ag))(*ag)
            desc.aggs, desc.n_aggs = arr_ag, len(ag)
        if proj:
            arr_pj = (C.c_int32 * len(proj))(*proj)
            desc.projection, desc.n_projection = arr_pj, len(proj)
        if order:
            arr_ob = (L.PqOrderBy * len(order))()
            for i, (target, index, fl) in enumerate(order):
                arr_ob[i].target, arr_ob[i].index, arr_ob[i].flags = target, index, fl
            desc.order_by, desc.n_order_by = arr_ob, len(order)
        if params is not None:
            desc.agg_params = params
        if window is not None:
            pw, _parr = _window_desc(window, partition)
            desc.window = C.pointer(pw)
        desc.limit = -1 if limit is None else int(limit)
        desc.batch_size = batch_size
        desc.shard_index, desc.shard_count = self.shard_index, self.shard_count
        desc.flags = flags

        h = C.c_void_p()
        rc = lib.pq_query_open(C.byref(desc), C.byref(h))
        if rc != L.PQ_OK:
            raise QueryError(rc, (lib.pq_last_error(None) or b"").decode())
        try:
            # every batch through ONE Arrow C stream (pq_query_stream): what arrow-rs does with
            # ArrowArrayStreamReader; pq_query_next stays for consumers that poll batch by batch
            batches = []
            while poll:   # poll_next, one batch per call
                arr_c, sch_c = L.ArrowArray(), L.ArrowSchema()
                rc = lib.pq_query_next(h, 0, C.byref(arr_c), C.byref(sch_c))
                if rc == L.PQ_END_OF_STREAM:
                    break
                if rc != L.PQ_OK:
                    raise QueryError(rc, (lib.pq_last_error(h) or b"").decode())
                batches.append(pa.RecordBatch._import_from_c(C.addressof(arr_c), C.addressof(sch_c)))
            if not poll:
                stream_c = L.ArrowArrayStream()
                rc = lib.pq_query_stream(h, 0, C.byref(stream_c))
                if rc != L.PQ_OK:
                    raise QueryError(rc, (lib.pq_last_error(h) or b"").decode())
                try:
                    batches = list(pa.RecordBatchReader._import_from_c(C.addressof(stream_c)))
                except pa.ArrowException as e:
                    raise QueryError(L.PQ_ERR_CUDA, (lib.pq_last_error(h) or str(e).encode()).decode()) from e
            json_text = None
            if json is not None:      # the same result as JSON text, formatted on the GPU
                jp, jn = C.c_void_p(), C.c_uint64()
                rc = lib.pq_query_json(h, L.PQ_JSON_LINES if json == "lines" else 0, C.byref(jp), C.byref(jn))
                if rc != L.PQ_OK:
                    raise QueryError(rc, (lib.pq_last_error(h) or b"").decode())
                json_text = C.string_at(jp.value, jn.value) if jn.value else b""
            m = L.PqMetrics()
            lib.pq_query_metrics(h, C.byref(m))
        finally:
            lib.pq_query_close(h)
        return QueryResult(batches, m.as_dict(), [f.name for f in batches[0].schema] if batches else [], json_text)


def flatten_objects_for_count(objects: list[dict]) -> list[dict]:
    """src/query/mod.rs:858-902 (kept "for later" by the reference; its six unit tests pin it): JSON rows that all carry
    the one same ``COUNT...`` key -- per-partition / per-node COUNT results -- fold into one row with their sum; anything
    else passes through untouched.  On the GPU path the same fold is the all-reduce of the partial tables."""
    if not objects:
        return objects
    first_key = next(iter(objects[0]), None)
    if all(all(k.startswith("COUNT") for k in o) for o in objects) and all(all(k == first_key for k in o) for o in objects):
        return [{first_key: sum(int(v) for o in objects for v in o.values())}]
    return objects


# ----------------------------------------------------------------------------- Query / execute
@dataclass
class TimeRange:
    start_ms: int
    end_ms: int


class Query:
    """``SELECT <cols | aggs> FROM <stream> [WHERE ...] [GROUP BY ...] [ORDER BY ...] [LIMIT n]`` — the subset of SQL the
    GPU path executes (ORDER BY on a query without aggregates only with a LIMIT).  It parses no subqueries, CTEs or window
    calls (``ROW_NUMBER() OVER (...)``): windows are reached through ``aggregate`` / ``scan(window=Window(...))``.  The reference hands SQL to DataFusion's planner (src/query/mod.rs:261-264);
    that planner is out of scope (SURVEY §2), so this small recursive-descent parser only exists
    to let tests and the bench state their queries the way Parseable users do."""

    def __init__(self, sql: str, time_range: TimeRange | None = None):
        self.sql = sql
        self.time_range = time_range
        self._parse(sql)

    # --- tokenizer / parser ---
    _TOK = re.compile(r"\s*(?:(-?\d+\.\d+(?:[eE][-+]?\d+)?|-?\d+)|'((?:[^']|'')*)'|\"([^\"]+)\"|([A-Za-z_][A-Za-z_0-9]*)|(<=|>=|<>|!~\*|!~|~\*|!=|~|[=<>(),*]))")

    def _parse(self, sql: str):
        toks, pos = [], 0
        sql = sql.strip().rstrip(";")
        while pos < len(sql):
            m = self._TOK.match(sql, pos)
            if not m:
                raise QueryError(L.PQ_ERR_INVALID_ARG, f"cannot tokenise SQL at: {sql[pos:pos+20]!r}")
            pos = m.end()
            if m.group(1) is not None:
                toks.append(("num", m.group(1)))
            elif m.group(2) is not None:
                toks.append(("str", m.group(2).replace("''", "'")))
            elif m.group(3) is not None:
                toks.append(("id", m.group(3)))
            elif m.group(4) is not None:
                w = m.group(4)
                toks.append(("kw", w.upper()) if w.upper() in _KEYWORDS else ("id", w))
            else:
                toks.append(("op", m.group(5)))
        self._t, self._i = toks, 0
        self._expect("kw", "SELECT")
        self.select: list = []
        while True:
            self.select.append(self._select_item())
            if not self._accept("op", ","):
                break
        self._expect("kw", "FROM")
        self.stream = self._next("id")[1]
        self.where = None
        self.group_by: list[str] = []
        self.limit = None
        if self._accept("kw", "WHERE"):
            self.where = self._or()
        if self._accept("kw", "GROUP"):
            self._expect("kw", "BY")
            while True:
                self.group_by.append(self._next("id")[1])
                if not self._accept("op", ","):
                    break
        # ORDER BY item [ASC | DESC] [NULLS FIRST | LAST], ...: these words are matched here only, never reserved, so
        # columns named `order`, `last`, ... keep parsing everywhere else
        self.order_by: list = []
        if self._word() == "ORDER" and self._peek(1) == ("kw", "BY"):
            self._i += 2
            while True:
                self.order_by.append(self._order_item())
                if not self._accept("op", ","):
                    break
        if self._accept("kw", "LIMIT"):
            self.limit = int(self._next("num")[1])
        if self.order_by and not any(it[0] == "agg" for it in self.select):
            # rows are ordered on the GPU as a top-K of the selection (SortExec(fetch)), never as a full sort
            if self.limit is None:
                raise QueryError(L.PQ_ERR_UNSUPPORTED, "ORDER BY on a query without aggregates needs a LIMIT: a full row-level sort is not on the GPU path")
            if any(item[0] == "agg" for item, _, _ in self.order_by):
                raise QueryError(L.PQ_ERR_UNSUPPORTED, "an aggregate in ORDER BY of a query without aggregates")
        if self._i != len(self._t):
            raise QueryError(L.PQ_ERR_UNSUPPORTED, f"unsupported SQL near {self._t[self._i]!r}")

    def _peek(self, k: int = 0):
        return self._t[self._i + k] if self._i + k < len(self._t) else (None, None)

    def _word(self, k: int = 0):
        """The upper-cased identifier k tokens ahead (a non-reserved word such as ORDER or NULLS), else None."""
        t = self._peek(k)
        return t[1].upper() if t[0] == "id" else None

    def _order_item(self):
        t = self._peek()
        if t[0] == "num" and t[1].isdigit():
            self._i += 1
            item = ("pos", int(t[1]))                       # 1-based position in the SELECT list
        elif t[0] == "kw" and t[1] in ("COUNT", "SUM", "MIN", "MAX", "AVG"):
            item = ("agg", self._agg_call())
        elif self._pct_ahead():
            item = ("agg", self._pct_call())
        else:
            item = ("name", self._next("id")[1])            # a SELECT alias or a GROUP BY column
        direction = "asc"
        if self._word() in ("ASC", "DESC"):
            direction = self._next("id")[1].lower()
        nulls_first = None
        if self._word() == "NULLS" and self._word(1) in ("FIRST", "LAST"):
            self._i += 1
            nulls_first = self._next("id")[1].upper() == "FIRST"
        return (item, direction, nulls_first)

    def _agg_call(self) -> Agg:
        t = self._next("kw")
        self._expect("op", "(")
        if t[1] == "COUNT" and self._accept("op", "*"):
            item = Agg("count_star")
        elif t[1] == "COUNT" and self._accept("kw", "DISTINCT"):
            item = Agg("count_distinct", self._next("id")[1])
        else:
            item = Agg(t[1].lower(), self._next("id")[1])
        self._expect("op", ")")
        return item

    # MEDIAN / PERCENTILE_CONT (and the refused approximate forms) are an identifier followed by "(": never reserved, so a
    # column named `median` still parses as a column
    _PCT_WORDS = ("MEDIAN", "PERCENTILE_CONT", "APPROX_MEDIAN", "APPROX_PERCENTILE_CONT", "APPROX_PERCENTILE_CONT_WITH_WEIGHT")

    def _pct_ahead(self) -> bool:
        return self._word() in self._PCT_WORDS and self._peek(1) == ("op", "(")

    def _fraction(self) -> float:
        t = self._next("num")
        return float(t[1])

    def _pct_call(self) -> Agg:
        """MEDIAN(col) | PERCENTILE_CONT(col, p) | PERCENTILE_CONT(p) WITHIN GROUP (ORDER BY col [ASC])."""
        w = self._next("id")[1].upper()
        if w.startswith("APPROX_"):
            raise QueryError(L.PQ_ERR_UNSUPPORTED, f"{w.lower()}: approximate percentiles (t-digest) are not on the GPU path; "
                                                   "the exact MEDIAN / PERCENTILE_CONT would answer differently")
        self._expect("op", "(")
        if w == "MEDIAN":
            item = Agg("median", self._next("id")[1])
            self._expect("op", ")")
            return item
        if self._peek()[0] == "num":                      # PERCENTILE_CONT(p) WITHIN GROUP (ORDER BY col [ASC])
            p = self._fraction()
            self._expect("op", ")")
            if self._word() != "WITHIN":
                raise QueryError(L.PQ_ERR_INVALID_ARG, "PERCENTILE_CONT(p) needs WITHIN GROUP (ORDER BY col)")
            self._i += 1
            self._expect("kw", "GROUP")
            self._expect("op", "(")
            if self._word() != "ORDER":
                raise QueryError(L.PQ_ERR_INVALID_ARG, "WITHIN GROUP needs (ORDER BY col)")
            self._i += 1
            self._expect("kw", "BY")
            c = self._next("id")[1]
            if self._word() == "DESC":
                raise QueryError(L.PQ_ERR_UNSUPPORTED, "PERCENTILE_CONT ... WITHIN GROUP (ORDER BY col DESC) is not on the GPU path")
            if self._word() == "ASC":
                self._i += 1
            self._expect("op", ")")
            return Agg("percentile_cont", c, p)
        c = self._next("id")[1]
        self._expect("op", ",")
        p = self._fraction()
        self._expect("op", ")")
        return Agg("percentile_cont", c, p)

    def _next(self, kind):
        t = self._peek()
        if t[0] != kind:
            raise QueryError(L.PQ_ERR_INVALID_ARG, f"expected {kind}, found {t!r}")
        self._i += 1
        return t

    def _accept(self, kind, val):
        t = self._peek()
        if t[0] == kind and t[1] == val:
            self._i += 1
            return True
        return False

    def _expect(self, kind, val):
        if not self._accept(kind, val):
            raise QueryError(L.PQ_ERR_INVALID_ARG, f"expected {val}, found {self._peek()!r}")

    def _select_item(self):
        t = self._peek()
        if t == ("op", "*"):
            self._i += 1
            return ("star",)
        if t[0] == "kw" and t[1] in ("COUNT", "SUM", "MIN", "MAX", "AVG"):
            item = self._agg_call()
            alias = self._next("id")[1] if self._accept("kw", "AS") else None
            return ("agg", item, alias)
        if self._pct_ahead():
            item = self._pct_call()
            alias = self._next("id")[1] if self._accept("kw", "AS") else None
            return ("agg", item, alias)
        if self._peek()[0] == "id" and self._peek(1) == ("op", "(") and self._peek()[1].lower().startswith("regexp_"):
            raise QueryError(L.PQ_ERR_UNSUPPORTED, f"{self._peek()[1]}(...) as a projected value is not on the GPU path")
        name = self._next("id")[1]
        alias = self._next("id")[1] if self._accept("kw", "AS") else None
        return ("col", name, alias)

    def _or(self):
        e = self._and()
        while self._accept("kw", "OR"):
            e = e | self._and()
        return e

    def _and(self):
        e = self._not()
        while self._accept("kw", "AND"):
            e = e & self._not()
        return e

    def _not(self):
        if self._accept("kw", "NOT"):
            return ~self._not()
        return self._primary()

    def _value(self):
        t = self._peek()
        self._i += 1
        if t[0] == "num":
            return lit(float(t[1]) if any(c in t[1] for c in ".eE") else int(t[1]))
        if t[0] == "str":
            return lit(t[1])
        if t[0] == "id" and t[1].upper() == "DATE" and self._peek()[0] == "str":   # DATE 'YYYY-MM-DD': a Date32 literal
            s = self._next("str")[1]
            try:   # fromisoformat alone also takes 20200102 and ISO week dates
                if not _DATE_LITERAL.fullmatch(s):
                    raise ValueError
                return lit(_dt.date.fromisoformat(s))
            except ValueError:
                raise QueryError(L.PQ_ERR_INVALID_ARG, f"DATE {s!r} is not a YYYY-MM-DD date") from None
        if t[0] == "id":
            return col(t[1])
        if t == ("kw", "TRUE"):
            return lit(True)
        if t == ("kw", "FALSE"):
            return lit(False)
        if t == ("kw", "NULL"):
            return lit(None)
        raise QueryError(L.PQ_ERR_INVALID_ARG, f"unexpected token {t!r}")

    def _regexp_like(self):
        """``regexp_like(col, 'pattern' [, 'flags'])``: the pattern with ``(?flags)`` in front, as arrow-string builds it."""
        self._i += 1
        self._expect("op", "(")
        t = self._next("id") if self._peek()[0] == "id" else None
        if t is None:
            raise QueryError(L.PQ_ERR_UNSUPPORTED, "regexp_like over an expression that is not a column")
        self._expect("op", ",")
        if self._peek()[0] != "str" or self._peek(1) not in (("op", ","), ("op", ")")):
            raise QueryError(L.PQ_ERR_UNSUPPORTED, "regexp_like with a pattern that is not a string literal")
        p = self._next("str")[1]
        if self._accept("op", ","):
            if self._peek()[0] != "str":
                raise QueryError(L.PQ_ERR_UNSUPPORTED, "regexp_like with flags that are not a string literal")
            flags = self._next("str")[1]
            if "g" in flags:
                raise QueryError(L.PQ_ERR_INVALID_ARG, "regexp_like() does not support the \"global\" option")
            if not flags:
                raise QueryError(L.PQ_ERR_UNSUPPORTED, "regexp_like with an empty flags string")
            p = f"(?{flags}){p}"
        self._expect("op", ")")
        return col(t[1]).regex(p)

    def _primary(self):
        if self._accept("op", "("):
            e = self._or()
            self._expect("op", ")")
            return e
        if self._peek()[0] == "id" and self._peek()[1].lower() == "regexp_like" and self._peek(1) == ("op", "("):
            return self._regexp_like()
        a = self._value()
        t = self._peek()
        if t[0] == "op" and t[1] in _REGEX_OPS:
            self._i += 1
            b = self._value()
            if a.kind != "col" or b.kind != "lit" or not isinstance(b.args[0], str):
                raise QueryError(L.PQ_ERR_UNSUPPORTED, f"{t[1]} needs a column on the left and a string literal pattern")
            neg, ci = _REGEX_OPS[t[1]]
            return a.regex(b.args[0], negated=neg, case_insensitive=ci)
        if t[0] == "op" and t[1] in _CMP:
            self._i += 1
            b = self._value()
            return Expr("cmp", (a, b), _CMP[t[1]])
        if self._accept("kw", "IS"):
            neg = self._accept("kw", "NOT")
            self._expect("kw", "NULL")
            return a.is_not_null() if neg else a.is_null()
        neg = self._accept("kw", "NOT")
        if t := self._peek():
            if t == ("kw", "LIKE") or t == ("kw", "ILIKE"):
                self._i += 1
                p = self._next("str")[1]
                if self._accept("kw", "ESCAPE"):
                    esc = self._next("str")[1]
                    if esc != "\\":     # the matcher's escape character is the backslash (arrow-string's default)
                        raise QueryError(L.PQ_ERR_UNSUPPORTED, f"LIKE ... ESCAPE {esc!r}: only the backslash is supported")
                return a.like(p, negated=neg, case_insensitive=(t[1] == "ILIKE"))
        raise QueryError(L.PQ_ERR_UNSUPPORTED, f"unsupported predicate near {self._peek()!r}")

    # --- src/query/mod.rs:774-856: wrap the scan in the time-range filter unless the user
    #     already filtered on the time column ---
    def final_filters(self) -> list[Expr]:
        filters = [] if self.where is None else [self.where]
        if self.time_range is not None and not _mentions(self.where, DEFAULT_TIMESTAMP_KEY):
            filters.append(col(DEFAULT_TIMESTAMP_KEY) >= Timestamp(self.time_range.start_ms))
            filters.append(col(DEFAULT_TIMESTAMP_KEY) < Timestamp(self.time_range.end_ms))
        return filters


_KEYWORDS = {"SELECT", "FROM", "WHERE", "GROUP", "BY", "AND", "OR", "NOT", "LIKE", "ILIKE", "IS", "NULL", "COUNT",
             "SUM", "MIN", "MAX", "AVG", "AS", "LIMIT", "TRUE", "FALSE", "ESCAPE",
             "DISTINCT"}
_REGEX_OPS = {"~": (False, False), "~*": (False, True), "!~": (True, False), "!~*": (True, True)}   # (negated, case-insens)
_CMP = {"=": L.PQ_EQ, "!=": L.PQ_NE, "<>": L.PQ_NE, "<": L.PQ_LT, "<=": L.PQ_LE, ">": L.PQ_GT, ">=": L.PQ_GE}


def _mentions(e: Expr | None, name: str) -> bool:
    if e is None:
        return False
    if e.kind == "col":
        return e.args[0] == name
    return any(_mentions(a, name) for a in e.args if isinstance(a, Expr))


def execute(query: Query, provider: StandardTableProvider, is_streaming: bool = False) -> QueryResult:
    """query::execute (src/query/mod.rs:143-149).  ``is_streaming`` only changes how the
    reference hands batches over (Vec vs stream); the batches are the same."""
    aggs = [it[1] for it in query.select if it[0] == "agg"]
    cols = [it[1] for it in query.select if it[0] == "col"]
    star = any(it[0] == "star" for it in query.select)
    filters = query.final_filters()
    if aggs:
        if star:
            raise QueryError(L.PQ_ERR_INVALID_ARG, "SELECT * next to an aggregate")
        extra = [c for c in cols if c not in query.group_by]
        if extra:
            raise QueryError(L.PQ_ERR_INVALID_ARG, f"column {extra[0]} must appear in GROUP BY")
        # ORDER BY items -> GROUP BY keys / aggregates; an aggregate only ORDER BY names is computed and then dropped
        order, hidden = [], []
        for (kind, v), direction, nulls_first in query.order_by:
            if kind == "pos":
                if not 1 <= v <= len(query.select):
                    raise QueryError(L.PQ_ERR_INVALID_ARG, f"ORDER BY {v}: the SELECT list has {len(query.select)} items")
                target = query.select[v - 1][1]
            elif kind == "agg":
                target = v
                if v not in aggs and v not in hidden:
                    hidden.append(v)
            else:
                alias = [it[1] for it in query.select if it[0] != "star" and it[2] == v]
                target = alias[0] if alias else v
            order.append((target, direction, nulls_first))
        # ORDER BY ... LIMIT runs on the GPU; a grouped LIMIT without ORDER BY keeps n groups in the unordered result
        res = provider.aggregate(query.group_by, aggs + hidden, filters, order_by=order or None,
                                 limit=query.limit if order else None)
        # output columns in SELECT order under their aliases
        if res.batches:
            t = res.table()
            names, picked = [], []
            for it in query.select:
                if it[0] == "col":
                    src = it[1]
                else:
                    src = it[1].name
                picked.append(t.column(src))
                names.append(it[2] or src)
            t = pa.table(picked, names=names)
            if query.limit is not None and not order:
                t = t.slice(0, query.limit)
            res.batches = t.to_batches(max_chunksize=20000) or res.batches[:1]
            res.fields = names
        return res
    if query.group_by:
        raise QueryError(L.PQ_ERR_UNSUPPORTED, "GROUP BY without aggregates")
    if star:
        if not provider.schema:
            raise QueryError(L.PQ_ERR_INVALID_ARG, "SELECT * needs the table schema")
        cols = list(provider.schema.keys())
    # ORDER BY items -> columns: a position in the SELECT list (SELECT * counts as the schema's columns), a SELECT alias,
    # or any column of the stream
    listed = [c for it in query.select for c in (list(provider.schema.keys()) if it[0] == "star" else [it[1]])]
    order = []
    for (kind, v), direction, nulls_first in query.order_by:
        if kind == "pos":
            if not 1 <= v <= len(listed):
                raise QueryError(L.PQ_ERR_INVALID_ARG, f"ORDER BY {v}: the SELECT list has {len(listed)} items")
            target = listed[v - 1]
        else:
            alias = [it[1] for it in query.select if it[0] == "col" and it[2] == v]
            target = alias[0] if alias else v
        order.append((target, direction, nulls_first))
    res = provider.scan(cols, filters, query.limit, order_by=order or None)
    aliases = {it[1]: it[2] for it in query.select if it[0] == "col" and it[2]}
    if aliases and res.batches:
        names = [aliases.get(n, n) for n in res.batches[0].schema.names]
        res.batches = [b.rename_columns(names) for b in res.batches]
        res.fields = names
    return res
