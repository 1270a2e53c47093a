"""ORDER BY ... LIMIT on filter / projection scans: the first rows of the ordered selection, selected and sorted on the
device (PqQueryDesc.order_by with PQ_ORDER_COLUMN terms).

Two oracles for every case:
  * the ordered result equals a stable host sort of the same scan's unordered GPU result (with __row_id), cut to the
    limit, in every column and every row;
  * independently of the GPU, its __row_id sequence equals the C oracle's selected row ids, stably sorted on the
    pyarrow-decoded values and cut.
Each case runs under every PQB_ORDER_PATH (a path that is not legal for the case falls back to the planner's choice)."""
import os
import struct

import numpy as np
import pyarrow as pa
import pyarrow.parquet as pq
import pytest

from oracle.oracle import Oracle
from parseable_b200 import _lib as L
from parseable_b200 import synth
from parseable_b200.query import (DeviceTable, Query, QueryError, QueryResult, StandardTableProvider, Timestamp, col, count_star,
                                  execute)
from test_order_by import canon, env_var, host_order

PATHS = ("", "cta", "topk", "sort")
TS0 = 1_700_000_000_000


def _nan(payload, neg=False):
    return struct.unpack("<d", struct.pack("<Q", (1 << 63 if neg else 0) | 0x7FF0000000000000 | payload))[0]


def _sortable(t: pa.Table) -> pa.Table:
    """Timestamps as their Int64 milliseconds (the host sort then never goes through datetime)."""
    for i, f in enumerate(t.schema):
        if pa.types.is_timestamp(f.type):
            t = t.set_column(i, f.name, t.column(i).cast(pa.int64()))
    return t


def _terms(order):
    return [(c, d == "desc", (d == "desc") if len(o) < 3 or o[2] is None else o[2]) for o in order for c, d in [o[:2]]]


def _table(res: QueryResult) -> pa.Table:
    return res.table() if res.batches else pa.table({})


def check_rows(prov, ora, order, limit, projection=("s", "i"), flt=(), paths=PATHS, batch_size=0):
    """One ordered scan under every path against the stable host sort of the unordered scan (and the C oracle)."""
    projection = list(projection)
    names = [o[0] for o in order]
    base = prov.scan(projection + [c for c in names if c not in projection], list(flt), row_ids=True)
    unordered = _sortable(_table(base)) if base.batches and base.batches[0].num_rows else None
    n = base.metrics["rows_selected"]
    want_n = min(limit, n)
    terms = _terms(order)
    want = None
    if want_n:
        idx = host_order(unordered, terms)[:want_n]
        want = canon(unordered.take(pa.array(idx, pa.int64())).select(projection + ["__row_id"]))
        # the C oracle: the selected rows in scan order, sorted on their pyarrow-decoded values
        if ora is not None:
            ids = ora.row_ids(list(flt))
            assert len(ids) == n
            vals = _sortable(ora.table.take(pa.array(ids)).select(list(dict.fromkeys(names))))
            oidx = host_order(vals, terms)[:want_n]
            oracle_ids = ids[np.array(oidx, np.int64)].tolist()
    results = []
    for path in paths:
        with env_var("PQB_ORDER_PATH", path or None):
            res = prov.scan(projection, list(flt), limit, row_ids=True, order_by=order, batch_size=batch_size)
        assert res.metrics["rows_selected"] == n
        got = _table(res)
        assert sum(b.num_rows for b in res.batches) == want_n, (path, order, limit)
        if want_n == 0:
            continue
        assert got.column_names == projection + ["__row_id"]
        assert canon(_sortable(got)) == want, (path, order, limit)
        if ora is not None:
            assert got["__row_id"].to_pylist() == oracle_ids, (path, order, limit)
        if batch_size:
            assert all(b.num_rows <= batch_size for b in res.batches)
        results.append(res)
    return results


# ---- data ---------------------------------------------------------------------------------------------------------------
def _columns(rng, n, with_i=True):
    svals = np.array(["", "a", "ab", "abc", "b", "zz", "δ-x"] + [f"user-{k:03d}" for k in range(200)], dtype=object)
    s = svals[rng.integers(0, len(svals), n)]
    s[rng.random(n) < 0.03] = None
    fvals = np.array([-0.0, 0.0, np.inf, -np.inf, _nan(1), _nan(3, True), _nan(1 << 51), 1.5, -2.25, 3.0, 100.0], dtype=np.float64)
    f = fvals[rng.integers(0, len(fvals), n)].astype(object)
    f[rng.random(n) < 0.02] = None
    b = (rng.random(n) < 0.4).astype(object)
    b[rng.random(n) < 0.1] = None
    t2 = (TS0 + rng.integers(-5_000, 5_000, n)).astype(object)
    t2[rng.random(n) < 0.05] = None
    msg = np.array([f"req-{k:06d} {'x' * (k % 13)}" for k in rng.integers(0, 130_000, n)], dtype=object)
    cols = {"p_timestamp": pa.array(TS0 + rng.integers(0, 50_000, n), pa.timestamp("ms")),   # ~4 rows per value: ties
            "s": pa.array(s, pa.string()), "msg": pa.array(msg, pa.string()), "f": pa.array(f, pa.float64()),
            "b": pa.array(b, pa.bool_()), "t2": pa.array(t2, pa.timestamp("ms")),
            "grp": pa.array(rng.integers(0, 5, n)), "u": pa.array(rng.integers(0, 150_000, n)), "v": pa.array(rng.integers(-9, 9, n))}
    if with_i:
        ivals = np.array([-(1 << 63), (1 << 63) - 1, -5, 0, 7] + list(range(100, 160)), dtype=object)
        i = ivals[rng.integers(0, len(ivals), n)]
        i[rng.random(n) < 0.02] = None
        cols["i"] = pa.array(i, pa.int64())
    return pa.table(cols)


@pytest.fixture(scope="module")
def data(data_dir, built):
    rng = np.random.default_rng(2026)
    # file A: two row groups, `msg` overflows its dictionary into PLAIN pages, p_timestamp PLAIN
    ta = _columns(rng, 160_000)
    pa_path = os.path.join(data_dir, "order_rows_a.parquet")
    pq.write_table(ta, pa_path, compression="NONE", row_group_size=80_000,
                   use_dictionary=[c for c in ta.column_names if c != "p_timestamp"], dictionary_pagesize_limit=256 << 10,
                   data_page_size=128 << 10)
    assert "PLAIN" in pq.ParquetFile(pa_path).metadata.row_group(0).column(ta.column_names.index("msg")).encodings
    # file B: Parseable's writer properties (DELTA_BINARY_PACKED p_timestamp), and no column `i`: its rows read as NULL
    tb = _columns(rng, 40_000, with_i=False)
    pb_path = os.path.join(data_dir, "order_rows_b.parquet")
    pq.write_table(tb, pb_path, row_group_size=40_000, **synth.parseable_writer_kwargs(tb.column_names))
    assert "DELTA_BINARY_PACKED" in pq.ParquetFile(pb_path).metadata.row_group(0).column(0).encodings
    files = [pa_path, pb_path]
    schema = ta.schema
    ora = Oracle(pa.concat_tables([ta, tb.append_column("i", pa.nulls(tb.num_rows, pa.int64())).select(ta.column_names)]))
    table = DeviceTable(files, schema.names)
    yield ora, StandardTableProvider(table, schema=schema), StandardTableProvider(files, schema=schema), files, schema
    table.close()


KINDS = ["s", "msg", "i", "f", "b", "t2", "p_timestamp"]
FILTERS = {"all": [], "sel": [col("u") < 2_500]}   # every row (top-K / radix) and ~3 300 rows (the one-CTA sort is legal)


@pytest.mark.gpu
@pytest.mark.parametrize("flt", FILTERS, ids=list(FILTERS))
@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("direction,nulls_first", [("asc", False), ("asc", True), ("desc", False), ("desc", True)])
def test_every_column_kind(data, kind, direction, nulls_first, flt):
    ora, prov, _, _, _ = data
    check_rows(prov, ora, [(kind, direction, nulls_first)], 1000, projection=["s", kind] if kind != "s" else ["s", "v"],
               flt=FILTERS[flt])


@pytest.mark.gpu
def test_multi_term_orders(data):
    ora, prov, _, _, _ = data
    # packs into one word: a Boolean with NULLs and a 5-value integer
    check_rows(prov, ora, [("b", "asc"), ("grp", "desc")], 3000)
    # two words (full-range Int64 with NULLs + Float64 + 150 000 values): the radix sort
    for limit in (10, 5000):
        check_rows(prov, ora, [("i", "desc", False), ("f", "asc", True), ("u", "asc")], limit, projection=["i", "f", "u", "msg"])
    check_rows(prov, ora, [("s", "asc"), ("p_timestamp", "desc"), ("t2", "asc", True)], 777, projection=["s", "p_timestamp"],
               flt=[col("grp") != 2])


@pytest.mark.gpu
def test_topk_ties_straddle_the_cut(data):
    """200 000 selected rows over 5 values: the kept tied rows are the first in scan order."""
    ora, prov, _, _, _ = data
    for limit in (1, 7, 1000, 4096):
        check_rows(prov, ora, [("grp", "asc")], limit, projection=["grp", "u"], paths=("", "topk", "sort"))
    check_rows(prov, ora, [("p_timestamp", "desc")], 4096, projection=["p_timestamp"], paths=("", "topk", "sort"))


@pytest.mark.gpu
def test_limits(data):
    ora, prov, _, _, _ = data
    flt = [col("u") < 2_500]
    n = ora.count(flt)
    assert 1000 < n <= 4096
    for limit in (0, 1, 17, n, n + 5):
        check_rows(prov, ora, [("f", "desc")], limit, projection=["f", "msg"], flt=flt)
    res = prov.scan(["s"], flt, 0, order_by=[("s", "asc")])
    assert res.metrics["rows_selected"] == n and sum(b.num_rows for b in res.batches) == 0


@pytest.mark.gpu
def test_selection_shapes(data):
    ora, prov, files_prov, files, schema = data
    # the log-search shape: a 0.1 % filter, newest first, every column
    c5 = [col("u") < 150, col("p_timestamp") >= Timestamp(TS0 + 1_000)]
    check_rows(prov, ora, [("p_timestamp", "desc")], 100, projection=schema.names, flt=c5)
    # the order column not projected; string projections; the column missing from file B (`i`: NULL there)
    check_rows(prov, ora, [("u", "desc")], 50, projection=["msg", "s"])
    check_rows(prov, ora, [("i", "asc", True)], 2000, projection=["i", "msg"])
    check_rows(prov, ora, [("i", "desc", False)], 45_000, projection=["i"], paths=("", "sort"))
    # a file list: the table is opened (and its Utf8 ids numbered) for this query alone
    check_rows(files_prov, ora, [("msg", "desc"), ("p_timestamp", "asc")], 300, projection=["msg", "p_timestamp"])
    # two row-group shards on one GPU: each orders and cuts its own selection
    for k in range(2):
        shard = StandardTableProvider(files, schema=schema, shard_index=k, shard_count=2)
        check_rows(shard, None, [("s", "asc"), ("f", "desc")], 500, projection=["s", "f"])


@pytest.mark.gpu
def test_output_forms(data):
    ora, prov, _, _, _ = data
    check_rows(prov, ora, [("msg", "asc")], 2500, projection=["msg", "s", "b"], batch_size=97)
    res = prov.scan(["s", "i", "grp", "msg"], [col("v") > 5], 300, order_by=[("s", "desc"), ("u", "asc")], json="array")
    assert res.to_json(fill_null=True) == res.table().to_pylist()
    # no projection: the selected __row_ids, in order
    flt = [col("grp") == 3]
    ids = ora.row_ids(flt)
    vals = _sortable(ora.table.take(pa.array(ids)).select(["t2"]))
    want = ids[np.array(host_order(vals, [("t2", True, False)])[:999], np.int64)].tolist()
    for path in PATHS:
        with env_var("PQB_ORDER_PATH", path or None):
            got = prov.scan(None, flt, 999, order_by=[("t2", "desc", False)])
        assert got.table().column_names == ["__row_id"] and got.table()["__row_id"].to_pylist() == want


@pytest.mark.gpu
def test_small_grid(data):
    """A forced small grid: every CTA of the encode kernel walks several work items."""
    ora, prov, _, _, _ = data
    with env_var("PQB_GRID", "3"):
        check_rows(prov, ora, [("s", "desc"), ("u", "asc")], 1500, projection=["s", "u"], flt=[col("v") < 0])


@pytest.mark.gpu
def test_metrics(data):
    ora, prov, _, _, _ = data
    flt = [col("v") < 0]
    plain = prov.scan(["s"], flt, 10)
    assert plain.metrics["order_ms"] == 0
    res = prov.scan(["s"], flt, 10, order_by=[("u", "desc")])
    assert res.metrics["rows_selected"] == ora.count(flt) == plain.metrics["rows_selected"]
    assert res.metrics["order_ms"] > 0 and res.metrics["kernel_launches"] > plain.metrics["kernel_launches"]
    assert res.metrics["groups"] == 0 and res.metrics["groups_total"] == 0


@pytest.mark.gpu
def test_refusals(data):
    ora, prov, _, _, _ = data

    def code(*args, **kw):
        with pytest.raises(QueryError) as e:
            prov._run(*args, **kw)
        return e.value

    # a GROUP BY key or an aggregate term on a scan
    e = code([], [], [], ["s"], 10, 0, 0, order=[(L.PQ_ORDER_KEY, 0, 0)])
    assert e.code == L.PQ_ERR_UNSUPPORTED and "ORDER BY" in e.message
    assert code([], [], [], ["s"], 10, 0, 0, order=[(L.PQ_ORDER_AGG, 0, 0)]).code == L.PQ_ERR_UNSUPPORTED
    # no LIMIT
    e = code([], [], [], ["s"], None, 0, 0, order=[(L.PQ_ORDER_COLUMN, "s", 0)])
    assert e.code == L.PQ_ERR_UNSUPPORTED and "LIMIT" in e.message
    # a column term on an aggregate query; a column index out of range; with COUNT_ONLY
    assert code([], ["s"], [count_star()], [], 5, 0, 0, order=[(L.PQ_ORDER_COLUMN, 0, 0)]).code == L.PQ_ERR_INVALID_ARG
    for index in (1, -1, 12):
        assert code([], [], [], ["s"], 5, 0, 0, order=[(L.PQ_ORDER_COLUMN, index, 0)]).code == L.PQ_ERR_INVALID_ARG
    assert code([], [], [], [], 5, 0, L.PQ_QUERY_COUNT_ONLY, order=[(L.PQ_ORDER_COLUMN, "s", 0)]).code == L.PQ_ERR_INVALID_ARG
    # more than 8 terms
    assert code([], [], [], ["s"], 5, 0, 0, order=[(L.PQ_ORDER_COLUMN, "s", 0)] * 9).code == L.PQ_ERR_UNSUPPORTED
    # items the flat kernels do not take (k_scan): not ordered on the GPU
    with env_var("PQB_FLAT_SCAN", "0"):
        assert code([], [], [], ["s"], 5, 0, 0, order=[(L.PQ_ORDER_COLUMN, "u", 0)]).code == L.PQ_ERR_UNSUPPORTED
    check_rows(prov, ora, [("u", "desc")], 3, projection=["u"], paths=("",))   # still answers


@pytest.mark.gpu
def test_sql_front(data):
    ora, prov, _, _, schema = data
    res = execute(Query("SELECT * FROM logs WHERE msg LIKE '%xxxxxxxxxxx%' ORDER BY p_timestamp DESC LIMIT 100"), prov)
    want = prov.scan(schema.names, [col("msg").like("%xxxxxxxxxxx%")], 100, order_by=[("p_timestamp", "desc")])
    assert canon(res.table()) == canon(want.table()) and res.table().num_rows == 100
    res = execute(Query("SELECT s AS name, u FROM logs WHERE v > 0 ORDER BY 2 DESC, name NULLS FIRST LIMIT 20"), prov)
    want = prov.scan(["s", "u"], [col("v") > 0], 20, order_by=[("u", "desc"), ("s", "asc", True)])
    assert res.table().column_names == ["name", "u"] and canon(res.table()) == canon(want.table())


# ---- the SQL front on the CPU: what execute hands to scan --------------------------------------------------------------
class _Recorder(StandardTableProvider):
    def __init__(self, schema):
        super().__init__([], schema=schema)
        self.calls = []

    def scan(self, projection=None, filters=(), limit=None, order_by=None, **kw):
        self.calls.append((list(projection or []), limit, order_by))
        return QueryResult([], {})


SCHEMA = {"p_timestamp": pa.timestamp("ms"), "host": pa.string(), "latency_ms": pa.int64(), "message": pa.string()}


@pytest.mark.parametrize("sql,projection,limit,order", [
    ("SELECT * FROM logs WHERE message LIKE '%timeout%' ORDER BY p_timestamp DESC LIMIT 100",
     list(SCHEMA), 100, [("p_timestamp", "desc", None)]),
    ("SELECT host, latency_ms FROM logs ORDER BY latency_ms DESC LIMIT 10", ["host", "latency_ms"], 10, [("latency_ms", "desc", None)]),
    ("SELECT host AS h, message FROM logs ORDER BY h ASC NULLS FIRST, 2 DESC NULLS LAST LIMIT 5", ["host", "message"], 5,
     [("host", "asc", True), ("message", "desc", False)]),
    ("SELECT * FROM logs ORDER BY 3, 1 DESC LIMIT 0", list(SCHEMA), 0, [("latency_ms", "asc", None), ("p_timestamp", "desc", None)]),
    ("SELECT message FROM logs WHERE host = 'a' ORDER BY p_timestamp DESC LIMIT 10", ["message"], 10, [("p_timestamp", "desc", None)]),
    ("SELECT message FROM logs LIMIT 10", ["message"], 10, None),
])
def test_sql_row_order_reaches_scan(sql, projection, limit, order):
    prov = _Recorder(SCHEMA)
    execute(Query(sql), prov)
    assert prov.calls == [(projection, limit, order)]


@pytest.mark.parametrize("sql", ["SELECT a FROM t ORDER BY a", "SELECT * FROM t WHERE a > 1 ORDER BY a DESC",
                                 "SELECT a FROM t ORDER BY COUNT(*) LIMIT 3"])
def test_sql_row_order_refusals(sql):
    with pytest.raises(QueryError) as e:
        Query(sql)
    assert e.value.code == L.PQ_ERR_UNSUPPORTED


def test_sql_row_order_bad_position():
    with pytest.raises(QueryError) as e:
        execute(Query("SELECT host FROM logs ORDER BY 2 LIMIT 3"), _Recorder(SCHEMA))
    assert e.value.code == L.PQ_ERR_INVALID_ARG


def test_scan_order_terms_reach_the_descriptor():
    """scan(order_by=...) names columns; the NULL defaults follow aggregate's (ASC: last, DESC: first)."""
    seen = {}

    class _Desc(StandardTableProvider):
        def _run(self, filters, group_by, aggs, projection, limit, batch_size, flags, poll=False, json=None, order=()):
            seen.update(order=order, limit=limit, flags=flags, projection=projection)

    _Desc([]).scan(["a"], [], 7, order_by=[("b", "asc"), ("c", "desc"), ("d", "desc", False), ("e", "asc", True)])
    assert seen["order"] == [(L.PQ_ORDER_COLUMN, "b", 0), (L.PQ_ORDER_COLUMN, "c", L.PQ_ORDER_DESC | L.PQ_ORDER_NULLS_FIRST),
                             (L.PQ_ORDER_COLUMN, "d", L.PQ_ORDER_DESC), (L.PQ_ORDER_COLUMN, "e", L.PQ_ORDER_NULLS_FIRST)]
    assert seen["limit"] == 7 and seen["projection"] == ["a"]
