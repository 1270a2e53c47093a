"""MEDIAN / PERCENTILE_CONT (PQ_AGG_MEDIAN / PQ_AGG_PERCENTILE_CONT) on the GPU.

Every result is compared with `restate` (tests/test_percentile_core.py), run over pyarrow-decoded values of the rows the
C oracle selects (`Oracle.select`), so the expectation does not depend on the GPU: Int64 results and medians bit for
bit, PERCENTILE_CONT equal to the restatement's f64 formula (also bit for bit: the kernel spells out the same
operations).  The other aggregates of a query are compared with the oracle's GROUP BY."""
import ctypes as C
import math
import os
import struct

import numpy as np
import pyarrow as pa
import pyarrow.compute as pc
import pyarrow.parquet as pq
import pytest

from oracle.oracle import Oracle
from parseable_b200 import _lib as L
from parseable_b200.query import (Agg, DateBin, DeviceTable, Query, QueryError, StandardTableProvider, _files_array, avg, col,
                                  count, count_distinct, count_star, date_bin, execute, max_, median, min_, percentile_cont,
                                  sum_)
from test_order_by import canon, check_ordered, env_var
from test_percentile_core import bits_f64, f64_bits, nan, restate

PCT = ("median", "percentile_cont")
I64_MIN, I64_MAX = -(1 << 63), (1 << 63) - 1


# ---- the expectation -----------------------------------------------------------------------------------------------
def _norm(v):
    return ("nan",) if isinstance(v, float) and math.isnan(v) else v


def _key_values(t: pa.Table, k, n):
    if isinstance(k, DateBin):
        v = pc.cast(t[k.column], pa.int64()).to_numpy(zero_copy_only=False)
        valid = t[k.column].is_valid().to_numpy(zero_copy_only=False)
        b = np.floor_divide(v - k.origin_ms, k.width_ms) * k.width_ms + k.origin_ms
        return pa.array(np.where(valid, b, 0), pa.int64()).cast(pa.timestamp("ms")).to_pylist() if n else [], valid
    if k not in t.column_names:
        return [None] * n, None
    return t[k].to_pylist(), None


def expect(ora: Oracle, keys, aggs, flt=()) -> dict:
    """key tuple -> {result column: value}: percentile results (as bits: f64 results as u64 patterns) from the
    restatement over the selected rows, everything else from the oracle's GROUP BY."""
    t = ora.table.filter(pa.array(ora.select(list(flt)).astype(bool)))
    n = t.num_rows
    kv = []
    for k in keys:
        vals, valid = _key_values(t, k, n)
        if valid is not None:
            vals = [v if ok else None for v, ok in zip(vals, valid)]
        kv.append(vals)
    groups: dict = {}
    for r in range(n):
        groups.setdefault(tuple(_norm(kv[i][r]) for i in range(len(keys))), []).append(r)
    if not keys and not groups:
        groups[()] = []                                   # a global aggregate over zero rows: one row
    plain = [a for a in aggs if a.fn not in PCT]
    out = {key: {} for key in groups}
    if plain:
        base = ora.group_by(list(keys), plain, list(flt))
        nk = len(keys)
        bk = [base.column(i).to_pylist() for i in range(nk)]
        for j, a in enumerate(plain):
            vals = base.column(nk + j).to_pylist()
            for r in range(base.num_rows):
                out[tuple(_norm(bk[i][r]) for i in range(nk))][a.name] = vals[r]
        if not keys and base.num_rows == 0:
            for a in plain:
                out[()][a.name] = 0 if a.fn in ("count", "count_star") else None
    for a in aggs:
        if a.fn not in PCT:
            continue
        f64 = a.column in t.column_names and pa.types.is_floating(t[a.column].type)
        vals = t[a.column].to_pylist() if a.column in t.column_names else [None] * n
        for key, rows in groups.items():
            out[key][a.name] = restate([vals[r] for r in rows], a.fn, a.p, f64)
    return out


def rows_of(t: pa.Table, nk) -> dict:
    names = t.column_names
    cols = [t.column(i).to_pylist() for i in range(t.num_columns)]
    return {tuple(_norm(cols[k][r]) for k in range(nk)): {names[c]: cols[c][r] for c in range(nk, len(names))} for r in range(t.num_rows)}


def assert_matches(got: pa.Table, exp: dict, keys, aggs):
    assert got.column_names == [k.name if isinstance(k, DateBin) else k for k in keys] + [a.name for a in aggs]
    g = rows_of(got, len(keys))
    assert set(g) == set(exp), (len(g), len(exp))
    for i, a in enumerate(aggs):
        typ = got.column(len(keys) + i).type
        if a.fn == "percentile_cont":
            assert typ == pa.float64()
        for key, row in g.items():
            v, e = row[a.name], exp[key][a.name]
            if a.fn in PCT:
                if e is None or v is None:
                    assert v is None and e is None, (a.name, key, v, e)
                elif pa.types.is_floating(typ):
                    assert f64_bits(v) == e, (a.name, key, v, bits_f64(e))
                else:
                    assert v == e, (a.name, key, v, e)
            elif isinstance(e, float) and isinstance(v, float) and a.fn in ("sum", "avg"):
                assert math.isclose(v, e, rel_tol=1e-9, abs_tol=1e-9), (a.name, key, v, e)
            else:
                assert v == e or (isinstance(v, float) and math.isnan(v) and math.isnan(e)), (a.name, key, v, e)


def check(prov, ora, keys, aggs, flt=(), **kw):
    res = prov.aggregate(keys, aggs, list(flt), **kw)
    got = res.table() if res.batches else pa.table({})
    assert_matches(got, expect(ora, keys, aggs, flt), keys, aggs)
    return res


# ---- the logs16 files (70 000-row row groups; `nulls`: 2 % NULLs) ---------------------------------------------------
@pytest.fixture(scope="module")
def logs(built, small_files):
    out = {}
    for tag, path in small_files.items():
        ora = Oracle.from_parquet(path)
        out[tag] = (ora, StandardTableProvider([path], schema=ora.table.schema), path)
    return out


P = percentile_cont
CASES = {
    "global": ([], [median("latency_ms"), P("latency_ms", 0.99), P("cpu", 0.5)], []),
    "global_zero_rows": ([], [count_star(), median("latency_ms"), P("duration_s", 0.9)], [col("level") == "NOPE"]),
    "one_key": (["host"], [median("latency_ms"), P("duration_s", 0.95), P("cpu", 0.5)], []),
    "two_keys": (["host", "status"], [count_star(), median("latency_ms"), P("latency_ms", 0.99), P("duration_s", 0.95)], []),
    "date_bin": ([date_bin("1m")], [P("latency_ms", 0.5), P("latency_ms", 0.95), P("latency_ms", 0.99)], []),
    "selective": (["level"], [median("cpu"), P("duration_s", 1 / 3), count_star()], [col("latency_ms") > 990]),
    "every_aggregate": (["level"], [count_star(), count("cpu"), sum_("bytes"), min_("latency_ms"), max_("cpu"), avg("latency_ms"),
                                    median("duration_s"), P("latency_ms", 0.0)], []),
}


@pytest.mark.gpu
@pytest.mark.parametrize("tag", ["nn", "nulls"])
@pytest.mark.parametrize("name", sorted(CASES))
def test_percentile_logs(logs, tag, name):
    ora, prov, _ = logs[tag]
    keys, aggs, flt = CASES[name]
    res = check(prov, ora, keys, aggs, flt)
    if name not in ("global_zero_rows", "selective"):
        assert res.metrics["percentile_ms"] > 0


@pytest.mark.gpu
def test_percentile_shares_one_sort(logs):
    """p50 / p95 / p99 of one column: one set of pairs, one sort, one pick -- the same kernels as p50 alone."""
    ora, prov, _ = logs["nulls"]
    one = check(prov, ora, ["host"], [P("latency_ms", 0.5)])
    three = check(prov, ora, ["host"], [P("latency_ms", 0.5), P("latency_ms", 0.95), P("latency_ms", 0.99), median("latency_ms")])
    assert three.metrics["kernel_launches"] == one.metrics["kernel_launches"]
    two_cols = check(prov, ora, ["host"], [P("latency_ms", 0.5), P("duration_s", 0.5)])
    assert two_cols.metrics["kernel_launches"] > one.metrics["kernel_launches"]
    plain = prov.aggregate(["host"], [count_star()])
    assert plain.metrics["percentile_ms"] == 0.0


@pytest.mark.gpu
@pytest.mark.parametrize("limit", [None, 1, 7])
def test_percentile_order_by(logs, limit):
    """ORDER BY a percentile DESC [LIMIT k] under every PQB_ORDER_PATH: a stable host sort of the unordered result (of a
    resident table, whose group numbering -- the order of tied rows -- is the same for every query)."""
    ora, _, path = logs["nulls"]
    dt = DeviceTable([path], ["host", "status", "latency_ms", "duration_s"])
    try:
        prov = StandardTableProvider(dt, schema=ora.table.schema)
        aggs = [count_star(), median("latency_ms"), P("duration_s", 0.99)]
        check_ordered(prov, None, ["host", "status"], aggs, [(P("duration_s", 0.99), "desc")], limit=limit)
        check_ordered(prov, None, ["host"], aggs, [(median("latency_ms"), "desc"), ("host", "asc")], limit=limit)
    finally:
        dt.close()


@pytest.mark.gpu
def test_percentile_small_batches_and_json(logs):
    ora, prov, _ = logs["nulls"]
    keys, aggs = ["host", "status"], [median("latency_ms"), P("cpu", 0.95)]
    res = check(prov, ora, keys, aggs, batch_size=7)
    assert len(res.batches) > 1
    res = prov.aggregate(keys, aggs, json="array")
    assert res.to_json(fill_null=True) == res.table().to_pylist()


@pytest.mark.gpu
def test_percentile_resident_table_and_shards(logs):
    ora, _, path = logs["nulls"]
    cols = ["host", "status", "latency_ms", "duration_s", "cpu", "level"]
    dt = DeviceTable([path], cols)
    try:
        prov = StandardTableProvider(dt, schema=ora.table.schema)
        for _ in range(2):   # the second query runs on the table's cached side tables
            check(prov, ora, ["host"], [median("latency_ms"), P("duration_s", 0.95), P("cpu", 0.5), sum_("latency_ms")])
    finally:
        dt.close()
    # two row-group shards: shard i scans row groups g with g % 2 == i
    t = ora.table
    n_rg = pq.ParquetFile(path).metadata.num_row_groups
    bounds = np.cumsum([0] + [pq.ParquetFile(path).metadata.row_group(g).num_rows for g in range(n_rg)])
    for shard in range(2):
        part = pa.concat_tables([t.slice(bounds[g], bounds[g + 1] - bounds[g]) for g in range(n_rg) if g % 2 == shard])
        prov = StandardTableProvider([path], schema=t.schema, shard_index=shard, shard_count=2)
        check(prov, Oracle(part), ["level"], [median("latency_ms"), P("cpu", 0.99)])


@pytest.mark.gpu
def test_percentile_small_grid(logs):
    ora, prov, _ = logs["nn"]
    with env_var("PQB_GRID", "3"):   # every CTA takes many items
        check(prov, ora, ["status"], [median("latency_ms"), P("duration_s", 0.5)], [col("latency_ms") > 10])


@pytest.mark.gpu
def test_percentile_edge_values_and_missing_column(data_dir, built):
    """Bit-exact on the edges: the wrapping Int64 median, -0.0 / +0.0, +-inf at and between ranks, NaN payloads of both
    signs; an all-NULL group; a column missing from one file; a PLAIN Float64 column; dictionary Int64 / Float64."""
    rng = np.random.default_rng(5)
    groups = {
        "wrap": ([I64_MAX, I64_MAX - 1], [1.0, 2.0]),
        "wrap2": ([I64_MIN, I64_MIN, 5], [-0.0, 0.0]),
        "zeros": ([0, 0], [0.0, -0.0, -0.0, 0.0]),
        "inf": ([1, 2, 3], [-math.inf, math.inf]),
        "inf3": ([4, 5], [-math.inf, 1.0, math.inf]),
        "nan": ([7], [nan(5), nan(9, True), 1.0, 2.0]),
        "nanonly": ([8, 9], [nan(3), nan(1)]),
        "allnull": ([None, None], [None, None]),
    }
    k, i, f = [], [], []
    for name, (iv, fv) in groups.items():
        m = max(len(iv), len(fv))
        for r in range(m):
            k.append(name)
            i.append(iv[r] if r < len(iv) else None)
            f.append(fv[r] if r < len(fv) else None)
    # a larger random body in group "body", with NULLs
    nb = 60_000
    k += ["body"] * nb
    i += [None if x < 0.03 else int(v) for x, v in zip(rng.random(nb), rng.integers(-10**6, 10**6, nb))]
    f += [None if x < 0.03 else float(v) for x, v in zip(rng.random(nb), np.round(rng.normal(0, 100, nb), 2))]
    ne = len(k) - nb   # the edge groups stay first (in the file that has `i`), the body is shuffled
    perm = np.concatenate([np.arange(ne), ne + rng.permutation(nb)])
    t = pa.table({"k": pa.array([k[j] for j in perm], pa.string()), "i": pa.array([i[j] for j in perm], pa.int64()),
                  "f": pa.array([f[j] for j in perm], pa.float64()), "pf": pa.array([f[j] for j in perm], pa.float64())})
    p1, p2 = (os.path.join(data_dir, f"pct_edges_{j}.parquet") for j in range(2))
    half = t.num_rows // 2
    kw = dict(row_group_size=20_000, use_dictionary=["k", "i", "f"], column_encoding={"pf": "PLAIN"}, compression="NONE")
    pq.write_table(t.slice(0, half), p1, **kw)
    pq.write_table(t.slice(half).drop_columns(["i"]), p2, **kw)         # `i` missing from this file: NULL
    ora = Oracle.from_parquet([p1, p2])   # the values as the files hold them (a dictionary may merge NaN payloads)
    prov = StandardTableProvider([p1, p2], schema=t.schema)
    for aggs in ([median("i"), P("i", 0.5), median("f"), P("f", 0.0), P("f", 1.0), P("f", 0.5), P("f", 0.99), P("pf", 1 / 3)],
                 [median("pf"), P("i", 0.0), P("i", 1.0), P("pf", 0.95), count_star()]):
        check(prov, ora, ["k"], aggs)
        check(prov, ora, [], aggs, [col("k") != "body"])
    # the wrapping median, read back directly
    got = prov.aggregate([], [median("i")], [col("k") == "wrap"]).table().to_pydict()
    assert got == {"median(i)": [-1]}


@pytest.mark.gpu
def test_percentile_hashed_group_by(data_dir, built):
    """A key space wider than the dense table (100 000 x 1 000 ids): the pairs carry hash-table cells."""
    rng = np.random.default_rng(9)
    n = 150_000
    t = pa.table({"id": pa.array(rng.integers(0, 100_000, n).astype(np.int64)),
                  "tag": pa.array(np.array([f"t{j}" for j in range(1000)], dtype=object)[rng.integers(0, 1000, n)], pa.string()),
                  "v": pa.array(np.where(rng.random(n) < 0.02, None, rng.integers(0, 10_000, n)), pa.int64()),
                  "x": pa.array(rng.normal(0, 1, n), pa.float64())})
    p = os.path.join(data_dir, "pct_hashed.parquet")
    pq.write_table(t, p, row_group_size=50_000, use_dictionary=["id", "tag", "v"], compression="NONE")
    ora = Oracle(t)
    prov = StandardTableProvider([p], schema=t.schema)
    check(prov, ora, ["id", "tag"], [count_star(), median("v"), P("x", 0.9)])


@pytest.mark.gpu
def test_percentile_sql(logs):
    ora, prov, _ = logs["nulls"]
    res = execute(Query("SELECT host, median(latency_ms), percentile_cont(latency_ms, 0.99) AS p99 FROM logs "
                        "GROUP BY host ORDER BY 3 DESC LIMIT 10"), prov)
    t = res.table()
    assert t.column_names == ["host", "median(latency_ms)", "p99"] and t.num_rows == 10
    exp = expect(ora, ["host"], [median("latency_ms"), P("latency_ms", 0.99)])
    vals = [v["percentile_cont(latency_ms, 0.99)"] for v in exp.values()]   # DESC: NULLs first
    want = sorted(vals, key=lambda b: (b is not None, -bits_f64(b) if b is not None else 0.0))[:10]
    assert [None if b is None else bits_f64(b) for b in want] == t["p99"].to_pylist()
    res = execute(Query("SELECT PERCENTILE_CONT(0.5) WITHIN GROUP (ORDER BY duration_s) AS p50, median(duration_s) FROM logs"), prov)
    t = res.table()
    e = expect(ora, [], [P("duration_s", 0.5), median("duration_s")])[()]
    assert f64_bits(t["p50"][0].as_py()) == e["percentile_cont(duration_s, 0.5)"]
    assert f64_bits(t["median(duration_s)"][0].as_py()) == e["median(duration_s)"]


# ---- refusals --------------------------------------------------------------------------------------------------------
def _raw_open(path, cols, aggs, params):
    """pq_query_open on a hand-built descriptor: columns [(name, PqType)], aggs [(fn, col)], params None or a list."""
    lib = L.load()
    hfs, arr = _files_array([path])
    c = (L.PqColumn * len(cols))()
    names = [n.encode() for n, _ in cols]
    for j, (n, ty) in enumerate(cols):
        c[j].name, c[j].type = names[j], ty
    a = (L.PqAgg * len(aggs))(*[L.PqAgg(fn=fn, col=ci) for fn, ci in aggs])
    d = L.PqQueryDesc()
    d.files, d.n_files = arr, 1
    d.columns, d.n_columns = c, len(cols)
    d.aggs, d.n_aggs = a, len(aggs)
    d.limit = -1
    if params is not None:
        d.agg_params = (C.c_double * len(params))(*params)
    h = C.c_void_p()
    rc = lib.pq_query_open(C.byref(d), C.byref(h))
    msg = (lib.pq_last_error(None) or b"").decode()
    if rc == L.PQ_OK:
        lib.pq_query_close(h)
    return rc, msg


@pytest.mark.gpu
def test_percentile_refusals(logs):
    ora, prov, path = logs["nulls"]
    for aggs in ([median("host")], [P("p_timestamp", 0.5)], [median("level")]):
        with pytest.raises(QueryError) as e:
            prov.aggregate([], aggs)
        assert e.value.code == L.PQ_ERR_UNSUPPORTED and "not on the GPU path" in e.value.message
    with pytest.raises(QueryError) as e:
        prov.aggregate([], [median("latency_ms")], flags=L.PQ_QUERY_ALLREDUCE)
    assert e.value.code == L.PQ_ERR_UNSUPPORTED and "PQ_QUERY_ALLREDUCE" in e.value.message
    with pytest.raises(QueryError) as e:
        prov.aggregate(["level"], [median("latency_ms"), count_distinct("host")])
    assert e.value.code == L.PQ_ERR_UNSUPPORTED and "COUNT(DISTINCT)" in e.value.message
    for p in (1.5, -0.1, math.nan, math.inf):
        with pytest.raises(QueryError) as e:
            prov.aggregate([], [P("latency_ms", p)])
        assert e.value.code == L.PQ_ERR_INVALID_ARG and "p must be finite" in e.value.message
    rc, msg = _raw_open(path, [("latency_ms", L.PQ_T_I64)], [(L.PQ_AGG_PERCENTILE_CONT, 0)], None)
    assert rc == L.PQ_ERR_INVALID_ARG and "agg_params" in msg
    rc, msg = _raw_open(path, [("latency_ms", L.PQ_T_I64)], [(L.PQ_AGG_MEDIAN, 0)], None)   # MEDIAN reads no parameter
    assert rc == L.PQ_OK, msg
    rc, msg = _raw_open(path, [("latency_ms", L.PQ_T_I64)], [(9, 0)], None)
    assert rc == L.PQ_ERR_INVALID_ARG
    with env_var("PQB_PCT_BUDGET", "1000000"):
        with pytest.raises(QueryError) as e:
            prov.aggregate(["host"], [median("latency_ms")])
        assert e.value.code == L.PQ_ERR_OOM and "HBM" in e.value.message
    check(prov, ora, ["level"], [median("latency_ms")])      # the context still answers
