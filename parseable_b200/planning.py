"""Host-side scan planning, mirrored from the reference so that the same files reach the GPU scan
that reach DataFusion's: nothing here touches the GPU.

Mirrors (paths relative to /root/reference):

* ``supports_filters_pushdown`` / ``expr_in_boundary``      src/query/stream_schema_provider.rs:665-683, 866-882
* ``extract_timestamp_bound`` / ``PartialTimeFilter``         :884-936, 698-748
* ``Snapshot::manifests`` (time pruning of manifest items)     src/catalog/snapshot.rs:40-71
* ``is_overlapping_query`` / ``is_within_staging_window``      src/query/stream_schema_provider.rs:750-775, 842-864
* ``ManifestExt::can_be_pruned`` / ``satisfy_constraints``     :955-1043   (per-file min / max pruning, TypedStatistics)
* ``collect_from_snapshot`` (pruning + LIMIT truncation)       :449-510
* ``partitioned_files`` (file i -> partition i % n, stats merge)  :351-446, src/catalog/column.rs:52-198

The Rust host keeps doing this itself in a drop-in build (nothing above ``scan()`` changes); the mirror
exists so that the Python harness plans like the reference and so that the semantics are pinned by the
reference's own unit-test vectors (tests/test_planning.py).
"""
from __future__ import annotations

import datetime as _dt
import math
from dataclasses import dataclass, field
from typing import Any, Iterable, Sequence

from . import _lib as L
from .query import DEFAULT_TIMESTAMP_KEY, Expr, Timestamp

EXACT, INEXACT = "Exact", "Inexact"      # TableProviderFilterPushDown


@dataclass(frozen=True)
class TimestampNs:
    """A TimestampNanosecond literal (extract_timestamp_bound accepts both units)."""
    ns: int


def _naive(ms: int) -> _dt.datetime:
    return _dt.datetime(1970, 1, 1) + _dt.timedelta(milliseconds=ms)


def extract_timestamp_bound(e: Expr, time_partition: str | None = None):
    """(op, naive UTC datetime) of ``<column> <op> <timestamp literal>``, else None.
    A Utf8 literal only counts on the time-partition column (stream_schema_provider.rs:884-920)."""
    if not isinstance(e, Expr) or e.kind != "cmp":
        return None
    left, right = e.args
    if right.kind != "lit":
        return None
    v = right.args[0]
    is_tp = left.kind == "col" and time_partition is not None and left.args[0] == time_partition
    if isinstance(v, Timestamp):
        return e.op, _naive(v.ms)
    if isinstance(v, TimestampNs):
        return e.op, _dt.datetime(1970, 1, 1) + _dt.timedelta(microseconds=v.ns // 1000)
    if isinstance(v, str) and is_tp:
        try:
            return e.op, _dt.datetime.fromisoformat(v)
        except ValueError:
            return None
    return None


def expr_in_boundary(e: Expr) -> bool:
    """Minute-aligned time comparisons can be answered by the minute-long prefixes alone (:866-882)."""
    b = extract_timestamp_bound(e, None)
    if b is None:
        return False
    op, t = b
    return t.second == 0 and t.microsecond == 0 and op in (L.PQ_GT, L.PQ_GE, L.PQ_LT, L.PQ_LE)


def supports_filters_pushdown(filters: Iterable[Expr]) -> list[str]:
    """Exact: the scan alone answers the filter (no FilterExec is kept above it); Inexact: evaluated in the scan
    AND re-applied.  The GPU scan evaluates every filter exactly either way, so the classification only tells the
    host which FilterExec it may drop (:665-683)."""
    return [EXACT if expr_in_boundary(f) else INEXACT for f in filters]


@dataclass(frozen=True)
class PartialTimeFilter:
    kind: str                  # "low" | "high" | "eq"
    time: _dt.datetime
    included: bool = True

    @staticmethod
    def try_from_expr(e: Expr, time_partition: str | None = None):
        b = extract_timestamp_bound(e, time_partition)
        if b is None:
            return None
        op, t = b
        return {L.PQ_GT: PartialTimeFilter("low", t, False), L.PQ_GE: PartialTimeFilter("low", t, True),
                L.PQ_LT: PartialTimeFilter("high", t, False), L.PQ_LE: PartialTimeFilter("high", t, True),
                L.PQ_EQ: PartialTimeFilter("eq", t, True)}.get(op)


def extract_primary_filter(filters: Iterable[Expr], time_partition: str | None = None) -> list[PartialTimeFilter]:
    """First time bound found in each filter expression (pre-order), like the reference's TreeNode walk (:922-940)."""
    out = []

    def walk(e):
        if not isinstance(e, Expr):
            return None
        t = PartialTimeFilter.try_from_expr(e, time_partition)
        if t is not None:
            return t
        for a in e.args:
            r = walk(a)
            if r is not None:
                return r
        return None

    for f in filters:
        t = walk(f)
        if t is not None:
            out.append(t)
    return out


@dataclass
class ManifestItem:            # src/catalog/snapshot.rs
    manifest_path: str
    time_lower_bound: _dt.datetime
    time_upper_bound: _dt.datetime


def snapshot_manifests(items: Sequence[ManifestItem], time_predicates: Iterable[PartialTimeFilter]) -> list[ManifestItem]:
    """Snapshot::manifests (src/catalog/snapshot.rs:40-71)."""
    out = list(items)
    for p in time_predicates:
        if p.kind == "low":
            out = [m for m in out if (m.time_upper_bound >= p.time if p.included else m.time_upper_bound > p.time)]
        elif p.kind == "high":
            out = [m for m in out if (m.time_lower_bound <= p.time if p.included else m.time_lower_bound < p.time)]
        else:
            out = [m for m in out if m.time_lower_bound <= p.time <= m.time_upper_bound]
    return out


def is_overlapping_query(items: Sequence[ManifestItem], time_filters: Iterable[PartialTimeFilter]) -> bool:
    """Backwards compatibility with the listing-based table format (:750-775)."""
    if not items:
        return True
    first = min(m.time_lower_bound for m in items)
    return any(f.kind == "low" and f.time < first for f in time_filters)


def is_within_staging_window(time_filters: Sequence[PartialTimeFilter], now: _dt.datetime | None = None) -> bool:
    """Staging data matters when the query's period ends within 5 minutes from now, or has no upper bound (:842-864)."""
    now = now or _dt.datetime.utcnow()
    back = (now - _dt.timedelta(minutes=5)).replace(second=0, microsecond=0)
    if any(f.kind in ("high", "eq") and f.time >= back for f in time_filters):
        return True
    return not any(f.kind == "high" for f in time_filters)


# ---- per-file statistics (src/catalog/column.rs TypedStatistics) ----
@dataclass
class TypedStatistics:
    kind: str                  # "bool" | "int" | "float" | "string"
    min: Any
    max: Any

    def update(self, other: "TypedStatistics"):
        """Merge two ranges; None when the variants disagree or a float range is invalid (column.rs:70-140)."""
        if self.kind != other.kind:
            return None
        if self.kind == "float":
            ok = lambda a, b: not (math.isnan(a) or math.isnan(b)) and a <= b   # noqa: E731
            if not ok(self.min, self.max) or not ok(other.min, other.max):
                return None
        return TypedStatistics(self.kind, min(self.min, other.min), max(self.max, other.max))


@dataclass
class ManifestColumn:
    name: str
    stats: TypedStatistics | None = None


@dataclass
class ManifestFileEntry:       # src/catalog/manifest.rs File
    file_path: str
    num_rows: int
    file_size: int = 0
    columns: list[ManifestColumn] = field(default_factory=list)


def _cast_or_none(v):
    if v is None:
        return None
    if isinstance(v, bool):
        return "bool", v
    if isinstance(v, Timestamp):
        return "int", v.ms
    if isinstance(v, _dt.date) and not isinstance(v, _dt.datetime):   # Date32 casts to Int (days): :1011
        return "int", (v - _dt.date(1970, 1, 1)).days
    if isinstance(v, int):
        return "int", v
    if isinstance(v, float):
        return "float", v
    if isinstance(v, str):
        return "string", v
    return None


def satisfy_constraints(kind: str, value, op: int, stats: TypedStatistics):
    """Can a file whose column spans [min, max] hold a row with ``column <op> value``?  None: cannot tell (:1017-1043)."""
    if kind != stats.kind:
        return None
    lo, hi = stats.min, stats.max
    if op == L.PQ_EQ:
        return lo <= value <= hi
    if op == L.PQ_LT:
        return value > lo
    if op == L.PQ_LE:
        return value >= lo
    if op == L.PQ_GT:
        return value < hi
    if op == L.PQ_GE:
        return value <= hi
    return None


def can_be_pruned(f: ManifestFileEntry, partial_filter: Expr) -> bool:
    """ManifestExt::can_be_pruned (:955-1000): only ``column <op> literal`` with statistics present prunes."""
    if not isinstance(partial_filter, Expr) or partial_filter.kind != "cmp":
        return False
    left, right = partial_filter.args
    if left.kind != "col" or right.kind != "lit":
        return False
    c = next((c for c in f.columns if c.name == left.args[0]), None)
    if c is None or c.stats is None:
        return False
    cast = _cast_or_none(right.args[0])
    if cast is None:
        return False
    ok = satisfy_constraints(cast[0], cast[1], partial_filter.op, c.stats)
    return not (True if ok is None else ok)


def collect_from_snapshot(manifest_files: Sequence[Sequence[ManifestFileEntry]], filters: Iterable[Expr], limit: int | None = None):
    """Files of the surviving manifests, newest first, minus the prunable ones, truncated once LIMIT rows are covered (:478-508)."""
    files = [f for m in manifest_files for f in m][::-1]
    for flt in filters:
        files = [f for f in files if not can_be_pruned(f, flt)]
    if limit is not None:
        total = 0
        for i, f in enumerate(files):
            total += f.num_rows
            if total >= limit:
                return files[: i + 1]
    return files


def partitioned_files(files: Sequence[ManifestFileEntry], target_partitions: int):
    """file i -> partition i % n; merged column statistics and the exact row count (:351-446).  With GPUs the
    partitions are the ranks: bench.py shards its file list the same way."""
    parts = [[] for _ in range(target_partitions)]
    stats: dict[str, TypedStatistics | None] = {}
    rows = 0
    for i, f in enumerate(files):
        parts[i % target_partitions].append(f)
        for c in f.columns:
            if c.name in stats:
                if stats[c.name] is not None and c.stats is not None:
                    stats[c.name] = stats[c.name].update(c.stats)
            else:
                stats[c.name] = c.stats
        rows += f.num_rows
    return parts, stats, rows


def final_time_filters(filters: Sequence[Expr], start_ms: int, end_ms: int) -> list[Expr]:
    """Query::final_logical_plan (src/query/mod.rs:774-856): ``p_timestamp >= start AND p_timestamp < end`` unless the
    user already filtered on the time column."""
    from .query import _mentions, col
    if any(_mentions(f, DEFAULT_TIMESTAMP_KEY) for f in filters):
        return list(filters)
    return list(filters) + [col(DEFAULT_TIMESTAMP_KEY) >= Timestamp(start_ms), col(DEFAULT_TIMESTAMP_KEY) < Timestamp(end_ms)]
