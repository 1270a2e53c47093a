"""ROW_NUMBER() OVER (PARTITION BY ... ORDER BY ...) cut to a rank range, ranked on the device (PqQueryDesc.window).

The central oracle, for every case: the windowed result equals the host restatement over the same query's unordered GPU
result (whose values the rest of the suite checks against the C oracle), in every row and column:
  1. stable-sort the unordered rows by (partition terms, order terms);
  2. number each partition's rows 1, 2, ... (row_number) and count them (partition_rows);
  3. keep offset < rn <= offset + fetch, then the first `limit`.
Scans are also checked against the C oracle's selected row ids, ranked the same way on pyarrow-decoded values.  Every
case runs under every PQB_ORDER_PATH (a path that is not legal for the case falls back to the planner's choice)."""
import collections
import os
import struct

import numpy as np
import pyarrow as pa
import pyarrow.parquet as pq
import pytest

from oracle.oracle import Oracle
from parseable_b200 import _lib as L
from parseable_b200 import synth
from parseable_b200.query import (Agg, DateBin, DeviceTable, QueryError, StandardTableProvider, Window, col, count_distinct,
                                  count_star, dataset_stats, date_bin, median, min_, sum_)
from test_order_by import canon, env_var, host_order

PATHS = ("", "cta", "topk", "sort")
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def _nan(payload, neg=False):
    return struct.unpack("<d", struct.pack("<Q", (1 << 63 if neg else 0) | 0x7FF0000000000000 | payload))[0]


def _name(item):
    return item.name if isinstance(item, (Agg, DateBin)) else item


def _terms(items):
    """[(item, dir[, nulls_first])] -> host_order terms [(column, desc, nulls_first)], DataFusion's NULL default."""
    out = []
    for it in items:
        it = tuple(it) if isinstance(it, (tuple, list)) else (it, "asc")
        desc = it[1] == "desc"
        out.append((_name(it[0]), desc, desc if len(it) < 3 or it[2] is None else it[2]))
    return out


def _pkey(v):
    return struct.pack("<d", v) if isinstance(v, float) else v   # Float64 partitions by bit pattern


def host_window(t: pa.Table, part, order, offset=0, fetch=None, limit=None):
    """(row indices, row_number, partition_rows) of the restated window over t."""
    idx = host_order(t, _terms(part) + _terms(order))
    pcols = [t[name].to_pylist() for name, _, _ in _terms(part)]
    keys = [tuple(_pkey(c[i]) for c in pcols) for i in idx]
    sizes = collections.Counter(keys)
    out, rns, szs = [], [], []
    rn, prev = 0, object()
    for pos, i in enumerate(idx):
        rn = rn + 1 if pos and keys[pos] == prev else 1
        prev = keys[pos]
        if rn > offset and (fetch is None or rn <= offset + fetch):
            out.append(i)
            rns.append(rn)
            szs.append(sizes[keys[pos]])
    if limit is not None:
        out, rns, szs = out[:limit], rns[:limit], szs[:limit]
    return out, rns, szs


def _with_window_cols(t: pa.Table, idx, rns, szs):
    t = t.take(pa.array(idx, pa.int64()))
    return t.append_column("row_number", pa.array(rns, pa.int64())).append_column("partition_rows", pa.array(szs, pa.int64()))


def _table(res):
    return res.table() if res.batches else None


def check_agg(prov, keys, aggs, part, order, offset=0, fetch=None, limit=None, flt=(), paths=PATHS, tie_multiset=False):
    """One windowed aggregate under every path against the host restatement over the unordered result."""
    base = prov.aggregate(keys, aggs, list(flt))
    unordered = _table(base)
    n_total = max(base.metrics["groups"], 0 if keys else 1)
    results = []
    for path in paths:
        with env_var("PQB_ORDER_PATH", path or None):
            res = prov.aggregate(keys, aggs, list(flt), order_by=order, limit=limit,
                                 window=Window(part, offset, fetch, row_number=True, partition_rows=True))
        assert res.metrics["groups_total"] == n_total
        got = _table(res)
        if unordered is None or unordered.num_rows == 0:
            assert got is None or got.num_rows == 0
            continue
        idx, rns, szs = host_window(unordered, part, order, offset, fetch, limit)
        assert res.metrics["groups"] == len(idx)
        if not idx:
            assert got is None or got.num_rows == 0
            continue
        want = _with_window_cols(unordered, idx, rns, szs)
        assert got.column_names == want.column_names
        if tie_multiset:
            # hashed slots: tied rows may come in another order; every tie group holds rows of the unordered result and
            # the tie keys, row numbers and partition sizes follow the restatement exactly
            tie = [n for n, _, _ in _terms(part) + _terms(order)]
            assert canon(got.select(tie + ["row_number", "partition_rows"])) == canon(want.select(tie + ["row_number", "partition_rows"]))
            assert set(canon(got.drop_columns(["row_number", "partition_rows"]))) <= set(canon(unordered))
        else:
            assert canon(got) == canon(want), (path, part, order, offset, fetch, limit)
        assert res.metrics["order_ms"] >= 0
        results.append(res)
    return results


def check_scan(prov, ora, projection, part, order, offset=0, fetch=None, limit=None, flt=(), paths=PATHS, rid_oracle=None):
    """One windowed scan under every path against the host restatement over the unordered scan, and the C oracle's ids."""
    projection = list(projection)
    names = [n for n, _, _ in _terms(part) + _terms(order)]
    base = prov.scan(projection + [c for c in dict.fromkeys(names) if c not in projection], list(flt), row_ids=True)
    unordered = _table(base)
    n = base.metrics["rows_selected"]
    want = None
    if unordered is not None and unordered.num_rows:
        unordered = _sortable(unordered)
        idx, rns, szs = host_window(unordered, part, order, offset, fetch, limit)
        want = _with_window_cols(unordered.select(projection + ["__row_id"]), idx, rns, szs)
        if ora is not None:   # the C oracle: selected ids in scan order, ranked on pyarrow-decoded values
            ids = ora.row_ids(list(flt))
            assert len(ids) == n
            vals = _sortable(ora.table.take(pa.array(ids)).select(list(dict.fromkeys(names)))) if names else pa.table({"_": np.zeros(len(ids))})
            oidx, _, _ = host_window(vals, part, order, offset, fetch, limit)
            assert ids[np.array(oidx, np.int64)].tolist() == want["__row_id"].to_pylist()
    results = []
    for path in paths:
        with env_var("PQB_ORDER_PATH", path or None):
            res = prov.scan(projection, list(flt), limit, row_ids=True, order_by=order,
                            window=Window(part, offset, fetch, row_number=True, partition_rows=True))
        assert res.metrics["rows_selected"] == n
        got = _table(res)
        if want is None or want.num_rows == 0:
            assert got is None or got.num_rows == 0
            continue
        assert got.column_names == projection + ["__row_id", "row_number", "partition_rows"]
        assert canon(_sortable(got)) == canon(want), (path, part, order, offset, fetch, limit)
        results.append(res)
    return results


def _sortable(t: pa.Table) -> pa.Table:
    for i, f in enumerate(t.schema):
        if pa.types.is_timestamp(f.type):
            t = t.set_column(i, f.name, t.column(i).cast(pa.int64()))
    return t


# ---- data ---------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def logs(small_files, built):
    """The small logs16 files as resident tables (group ids, so slot order, are numbered once) with their oracles."""
    out = {}
    for tag, path in small_files.items():
        ora = Oracle.from_parquet(path)
        table = DeviceTable([path], ora.table.column_names)
        out[tag] = (ora, StandardTableProvider(table, schema=ora.table.schema), table, path)
    yield out
    for _, _, table, _ in out.values():
        table.close()


@pytest.fixture(scope="module")
def floats(data_dir, built):
    """A Float64 key whose -0.0 / 0.0 and NaN payloads are distinct groups and so distinct partitions."""
    rng = np.random.default_rng(11)
    n = 60_000
    fvals = np.array([-0.0, 0.0, np.inf, -np.inf, _nan(1), _nan(3), _nan(3, True), 1.5, -2.25], dtype=np.float64)
    f = fvals[rng.integers(0, len(fvals), n)].astype(object)
    f[rng.random(n) < 0.03] = None
    t = pa.table({"f": pa.array(f, pa.float64()), "g": pa.array(rng.integers(0, 40, n)), "v": pa.array(rng.integers(-9, 9, n))})
    p = os.path.join(data_dir, "window_floats.parquet")
    pq.write_table(t, p, compression="NONE", row_group_size=30_000)
    table = DeviceTable([p], t.column_names)
    yield StandardTableProvider(table, schema=t.schema)
    table.close()


# ---- aggregates ---------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_aggregate_partitions(logs):
    _, prov, _, _ = logs["nn"]
    check_agg(prov, ["status", "host"], [sum_("bytes"), count_star()], ["status"], [(sum_("bytes"), "desc")], fetch=3)
    check_agg(prov, ["level", "status", "service"], [count_star()], ["level", "status"], [(count_star(), "desc")], offset=2, fetch=2)
    db = date_bin("1m")
    check_agg(prov, [db, "service"], [count_star()], [db], [(count_star(), "desc")], fetch=5)


@pytest.mark.gpu
def test_many_partitions_and_large_partitions(logs):
    """> 4 096 groups (the radix sort) in thousands of partitions, many straddling the 1 024-position tiles; and
    partitions of several thousand groups (larger than a tile)."""
    _, prov, _, _ = logs["nn"]
    res = check_agg(prov, ["host", "service"], [count_star(), sum_("bytes")], ["host"], [(count_star(), "desc"), ("service", "asc")],
                    fetch=2, paths=("", "sort"))
    assert res[0].metrics["groups_total"] > 4096
    assert len(set(res[0].table()["host"].to_pylist())) > 2000
    res = check_agg(prov, ["status", "host"], [count_star()], ["status"], [(count_star(), "desc")], offset=1000, fetch=1500)
    assert max(res[0].table()["partition_rows"].to_pylist()) > 1024
    check_agg(prov, ["status", "host"], [count_star()], [("status", "desc")], [("host", "desc")], offset=0, fetch=None, limit=5000)


@pytest.mark.gpu
def test_nullable_partition_key(logs):
    _, prov, _, _ = logs["nulls"]
    for nulls_first in (False, True):
        check_agg(prov, ["level", "status"], [count_star()], [("level", "asc", nulls_first)], [(count_star(), "desc")], fetch=2)
        check_agg(prov, ["status", "region"], [count_star()], [("status", "desc", nulls_first)], [("region", "asc", nulls_first)],
                  offset=1, fetch=3)


@pytest.mark.gpu
def test_float_partitions_by_bit_pattern(floats):
    prov = floats
    res = check_agg(prov, ["f", "g"], [count_star(), sum_("v")], ["f"], [(count_star(), "desc"), ("g", "asc")], fetch=2)
    parts = {struct.pack("<d", v) if v is not None else None for v in res[0].table()["f"].to_pylist()}
    assert struct.pack("<d", -0.0) in parts and struct.pack("<d", 0.0) in parts
    assert struct.pack("<d", _nan(3)) in parts and struct.pack("<d", _nan(3, True)) in parts and None in parts


@pytest.mark.gpu
def test_order_terms_of_every_aggregate_kind(logs):
    _, prov, _, _ = logs["nulls"]
    check_agg(prov, ["status", "service"], [min_("host"), count_star()], ["status"], [(min_("host"), "asc")], fetch=3)
    check_agg(prov, ["level", "service"], [median("latency_ms")], ["level"], [(median("latency_ms"), "desc")], fetch=4)
    check_agg(prov, ["region", "service"], [count_distinct("host")], ["region"], [(count_distinct("host"), "desc")], offset=1, fetch=2)


@pytest.mark.gpu
def test_hashed_group_by(logs):
    _, prov, _, _ = logs["nn"]
    check_agg(prov, ["host", "message", "pod"], [count_star()], ["host"], [(count_star(), "desc")], fetch=2,
              paths=("", "sort"), tie_multiset=True)


@pytest.mark.gpu
def test_edges(logs):
    _, prov, _, _ = logs["nn"]
    keys, aggs = ["status", "service"], [count_star()]
    check_agg(prov, keys, aggs, ["status"], [(count_star(), "desc")], fetch=0)
    check_agg(prov, keys, aggs, ["status"], [(count_star(), "desc")], offset=7, fetch=None)
    past = prov.aggregate(keys, aggs, order_by=[(count_star(), "desc")], window=Window(["status"], 10_000, 3, row_number=True))
    assert past.metrics["groups"] == 0 and (past.batches == [] or past.table().num_rows == 0)   # past every partition
    check_agg(prov, keys, aggs, ["status"], [(count_star(), "desc")], offset=10_000, fetch=3)
    check_agg(prov, keys, aggs, ["status"], [(count_star(), "desc")], fetch=10, limit=23)   # the outer LIMIT cuts across partitions
    check_agg(prov, keys, aggs, ["status"], [], fetch=4)                                     # no order terms: slot order ranks
    check_agg(prov, keys, aggs, [], [], offset=5, fetch=6)
    check_agg(prov, ["status"], aggs, ["status"], [(count_star(), "desc")], fetch=2, flt=[col("status") == 404])   # one group
    check_agg(prov, [], [count_star(), sum_("bytes")], [], [(count_star(), "desc")], fetch=1)                     # a global aggregate
    check_agg(prov, [], [count_star(), sum_("bytes")], [], [], offset=1, fetch=1)
    g = prov.aggregate([], [count_star(), sum_("bytes")], [col("status") == 7], window=Window(row_number=True, partition_rows=True))
    assert g.table().to_pylist() == [{"count(*)": 0, "sum(bytes)": None, "row_number": 1, "partition_rows": 1}]
    c = prov.aggregate([], [count_star()], [col("status") == 404], window=Window(row_number=True, partition_rows=True))
    assert c.table().column_names == ["count(*)", "row_number", "partition_rows"] and c.table()["row_number"].to_pylist() == [1]
    assert prov.aggregate([], [count_star()], window=Window(offset=1)).batches == []


@pytest.mark.gpu
def test_no_partition_equals_order_by_limit_with_offset(logs):
    _, prov, _, _ = logs["nn"]
    keys, aggs, order = ["host"], [count_star(), sum_("bytes")], [(count_star(), "desc"), (sum_("bytes"), "asc")]
    for offset, fetch in ((0, 10), (7, 20), (3000, 50), (0, None), (9000, 5)):
        for path in PATHS:
            with env_var("PQB_ORDER_PATH", path or None):
                w = prov.aggregate(keys, aggs, order_by=order, window=Window([], offset, fetch, row_number=True, partition_rows=True))
                lim = prov.aggregate(keys, aggs, order_by=order, limit=None if fetch is None else offset + fetch)
            base = lim.table().slice(offset)
            got = _table(w)
            if base.num_rows == 0:
                assert got is None or got.num_rows == 0
                continue
            assert canon(got.select(base.column_names)) == canon(base), (offset, fetch, path)
            assert got["row_number"].to_pylist() == list(range(offset + 1, offset + 1 + base.num_rows))
            assert set(got["partition_rows"].to_pylist()) == {lim.metrics["groups_total"]}


@pytest.mark.gpu
def test_window_json_and_metrics(logs):
    _, prov, _, _ = logs["nulls"]
    res = prov.aggregate(["level", "service"], [count_star()], order_by=[(count_star(), "desc")], json="array",
                         window=Window(["level"], 1, 3, row_number=True, partition_rows=True))
    assert res.to_json(fill_null=True) == res.table().to_pylist()
    plain = prov.aggregate(["level", "service"], [count_star()])
    assert res.metrics["groups_total"] == plain.metrics["groups"] and res.metrics["order_ms"] > 0
    assert res.metrics["kernel_launches"] > plain.metrics["kernel_launches"]
    res = prov.scan(["host", "status"], [col("level") == "ERROR"], json="lines", order_by=[("status", "desc")],
                    window=Window(["service"], 0, 2, row_number=True, partition_rows=True))
    assert res.to_json(fill_null=True) == res.table().to_pylist()
    assert res.metrics["rows_selected"] > res.table().num_rows


# ---- scans --------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_scan_latest_errors_per_service(logs):
    ora, prov, _, path = logs["nn"]
    flt = [col("level") == "ERROR"]
    check_scan(prov, ora, ["p_timestamp", "host", "message"], ["service"], [("p_timestamp", "desc")], fetch=3, flt=flt)
    # the same over a file list, and with several work items per CTA in the encode kernel
    files = StandardTableProvider([path], schema=ora.table.schema)
    check_scan(files, ora, ["p_timestamp", "host", "message"], ["service"], [("p_timestamp", "desc")], fetch=3, flt=flt)
    with env_var("PQB_GRID", "2"):
        check_scan(prov, ora, ["host"], ["service"], [("p_timestamp", "desc"), ("latency_ms", "asc")], offset=1, fetch=2, flt=flt,
                   paths=("", "sort"))


@pytest.mark.gpu
def test_scan_shapes(logs):
    ora, prov, _, _ = logs["nulls"]
    flt = [col("status") == 503]
    for nulls_first in (False, True):   # a nullable partition column
        check_scan(prov, ora, ["host", "status"], [("region", "asc", nulls_first)], [("latency_ms", "desc")], fetch=4, flt=flt)
    check_scan(prov, ora, ["host"], ["region"], [], offset=2, fetch=3, flt=flt)                  # no order terms: file order
    check_scan(prov, ora, [], ["level"], [("bytes", "asc")], fetch=5, flt=flt)                  # no projection: ordered row ids
    check_scan(prov, ora, ["service"], ["level", "method"], [("cpu", "desc")], fetch=1, limit=17, flt=flt)
    check_scan(prov, ora, ["service"], [], [("bytes", "desc")], offset=10, fetch=20, flt=flt)   # one partition
    check_scan(prov, ora, ["service"], ["region"], [("bytes", "desc")], offset=10_000, fetch=2, flt=flt)   # past every partition
    with pytest.raises(QueryError) as e:   # a window needs no LIMIT, a plain ORDER BY still does
        prov.scan(["host"], flt, order_by=[("bytes", "asc")])
    assert e.value.code == L.PQ_ERR_UNSUPPORTED


@pytest.mark.gpu
def test_scan_shards_rank_their_own_selection(small_files, built):
    path = small_files["nn"]
    schema = synth.logs16_schema()
    for shard in range(2):
        prov = StandardTableProvider([path], schema=schema, shard_index=shard, shard_count=2)
        res = check_scan(prov, None, ["host"], ["service"], [("p_timestamp", "desc")], fetch=3, flt=[col("level") == "ERROR"],
                         paths=("",))
        assert res and max(res[0].table()["row_number"].to_pylist()) <= 3


# ---- known answers ------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_field_stats_fixtures_through_the_window(built):
    prov = StandardTableProvider([os.path.join(GOLD, "field_stats_10rows.parquet")], schema={"name": pa.string()})
    res = prov.aggregate(["name"], [count_star()], order_by=[(count_star(), "desc")],
                         window=Window(row_number=True, partition_rows=True))
    t = res.table()
    assert t["row_number"].to_pylist() == list(range(1, 8)) and set(t["partition_rows"].to_pylist()) == {7}
    assert list(zip(t["name"].to_pylist(), t["count(*)"].to_pylist()))[:3] == [("Alice", 3), ("Bob", 2), ("Charlie", 1)]
    prov = StandardTableProvider([os.path.join(GOLD, "field_stats_1000rows.parquet")], schema={"category": pa.string()})
    t = prov.aggregate(["category"], [count_star()], order_by=[(count_star(), "desc")],
                       window=Window(fetch=10, partition_rows=True)).table()
    assert t["count(*)"].to_pylist() == [100] * 10 and t["partition_rows"].to_pylist() == [10] * 10
    prov = StandardTableProvider([os.path.join(GOLD, "field_stats_empty.parquet")], schema={"name": pa.string()})
    res = prov.aggregate(["name"], [count_star()], order_by=[(count_star(), "desc")], window=Window(fetch=5, row_number=True))
    assert res.batches == [] or res.table().num_rows == 0


def _pstats(rng, n):
    datasets = np.array(["web", "db", "q\"x"], dtype=object)
    fields = np.array(["host", "level", "status", "user"], dtype=object)
    values = np.array([f"v{k:02d}" for k in range(30)], dtype=object)
    dv = values[rng.integers(0, len(values), n)]
    dv[rng.random(n) < 0.08] = None
    fn = fields[rng.integers(0, len(fields), n)]
    fn[rng.random(n) < 0.01] = None
    return pa.table({"dataset_name": pa.array(datasets[rng.integers(0, len(datasets), n)], pa.string()),
                     "field_stats_field_name": pa.array(fn, pa.string()),
                     "field_stats_count": pa.array(rng.integers(1, 50, n)),
                     "field_stats_distinct_stats_distinct_value": pa.array(dv, pa.string()),
                     "field_stats_distinct_stats_count": pa.array(rng.integers(1, 4, n))})   # small counts: tied sums


def host_dataset_stats(t: pa.Table, dataset, fields, offset, limit):
    """build_stats_sql (src/storage/field_stats.rs in the reference), restated in Python."""
    rows = t.to_pylist()
    sums, totals = collections.defaultdict(int), collections.defaultdict(int)
    for r in rows:
        if r["dataset_name"] != dataset:
            continue
        if r["field_stats_field_name"] is not None:
            totals[r["field_stats_field_name"]] += r["field_stats_count"]
        if r["field_stats_distinct_stats_distinct_value"] is None or (fields and r["field_stats_field_name"] not in fields):
            continue
        sums[(r["field_stats_field_name"], r["field_stats_distinct_stats_distinct_value"])] += r["field_stats_distinct_stats_count"]
    per_field = collections.defaultdict(list)
    for (f, v), s in sums.items():
        per_field[f].append((v, s))
    out = {}
    for f, vs in per_field.items():
        if f is None or f not in totals:
            continue
        vs.sort(key=lambda x: (-x[1], x[0].encode()))
        top = vs[offset:offset + limit]
        if top:
            out[f] = {"field_count": totals[f], "distinct_count": len(vs), "distinct_values": dict(top)}
    return out


@pytest.mark.gpu
def test_dataset_stats(data_dir, built):
    t = _pstats(np.random.default_rng(5), 40_000)
    p = os.path.join(data_dir, "pstats.parquet")
    pq.write_table(t, p, row_group_size=20_000)
    prov = StandardTableProvider([p], schema=t.schema)
    for dataset in ("web", "q\"x", "none"):
        for fields in (None, ["level", "user", "nope"]):
            for offset in (0, 2):
                got = dataset_stats(prov, dataset, fields, offset, 5)
                want = host_dataset_stats(t, dataset, fields, offset, 5)
                assert got == want, (dataset, fields, offset)
                for f, st in got.items():   # rank order: SUM DESC, then distinct_value ASC
                    assert list(st["distinct_values"]) == list(want[f]["distinct_values"])
    assert dataset_stats(prov, "web", None, 0, 5)["host"]["distinct_count"] == 30


# ---- refusals -----------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_refusals(logs):
    _, prov, _, _ = logs["nn"]

    def agg(window, order=(), flags=0, partition=None):
        return prov._run([], ["status", "service"], [count_star()], [], None, 0, flags, order=list(order), window=window,
                         partition=partition)

    def code(fn):
        with pytest.raises(QueryError) as e:
            fn()
        return e.value.code

    nine = [(L.PQ_ORDER_KEY, 0, 0)] * 5
    assert code(lambda: agg(Window(), order=[(L.PQ_ORDER_AGG, 0, 0)] * 4, partition=nine)) == L.PQ_ERR_UNSUPPORTED
    assert code(lambda: prov._run([], [], [], ["host"], None, 0, 0, window=Window(), partition=[(L.PQ_ORDER_KEY, 0, 0)])) == L.PQ_ERR_UNSUPPORTED
    assert code(lambda: agg(Window(), partition=[(L.PQ_ORDER_COLUMN, 0, 0)])) == L.PQ_ERR_INVALID_ARG
    assert code(lambda: agg(Window(), partition=[(L.PQ_ORDER_KEY, 2, 0)])) == L.PQ_ERR_INVALID_ARG
    assert code(lambda: agg(Window(), partition=[(L.PQ_ORDER_AGG, 0, 0)])) == L.PQ_ERR_INVALID_ARG
    assert code(lambda: agg(Window(offset=-1), partition=[])) == L.PQ_ERR_INVALID_ARG
    assert code(lambda: prov.scan(["host"], [], window=Window(offset=-1))) == L.PQ_ERR_INVALID_ARG
    assert code(lambda: prov.scan(count_only=True, window=Window(["host"]))) == L.PQ_ERR_INVALID_ARG

    # unknown flag bits: through the raw descriptor
    import parseable_b200.query as Q
    orig = Q._window_desc

    def bad_desc(w, terms):
        pw, arr = orig(w, terms)
        pw.flags |= 8
        return pw, arr
    Q._window_desc = bad_desc
    try:
        assert code(lambda: agg(Window(), partition=[])) == L.PQ_ERR_INVALID_ARG
    finally:
        Q._window_desc = orig
    # still answers
    check_agg(prov, ["status", "service"], [count_star()], ["status"], [(count_star(), "desc")], fetch=1, paths=("",))


def test_window_mirror():
    """The ctypes mirror: PqWindow is appended after agg_params, its flags are the header's."""
    assert L.PqQueryDesc._fields_[-1][0] == "window" and L.PqQueryDesc._fields_[-2][0] == "agg_params"
    assert (L.PQ_WINDOW_ROW_NUMBER, L.PQ_WINDOW_PARTITION_ROWS) == (1, 2)
    from parseable_b200.query import _partition_items, _window_desc
    w = Window(["a", ("b", "desc", True)], offset=2, fetch=None, partition_rows=True)
    assert _partition_items(w) == [("a", "asc"), ("b", "desc", True)]
    pw, _ = _window_desc(w, [(L.PQ_ORDER_COLUMN, 0, 0), (L.PQ_ORDER_COLUMN, 1, 3)])
    assert (pw.n_partition_by, pw.flags, pw.offset, pw.fetch) == (2, L.PQ_WINDOW_PARTITION_ROWS, 2, -1)
    assert pw.partition_by[1].flags == 3
