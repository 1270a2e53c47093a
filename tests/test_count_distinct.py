"""COUNT(DISTINCT col) (PQ_AGG_COUNT_DISTINCT, the alerts' CountDistinct: src/alerts/mod.rs:245-251).

GPU tests go through the C ABI and are compared with `expect_count_distinct`, a CPU restatement built on the C oracle:
GROUP BY keys + col -> COUNT(*) over the selected rows (f64 keys group by bit pattern), then the number of non-NULL
`col` groups per key.  That restatement is itself checked against Acero's count_distinct (only_valid) on the CPU."""
import math
import os
import struct
from contextlib import contextmanager

import numpy as np
import pyarrow as pa
import pyarrow.compute as pc
import pyarrow.parquet as pq
import pytest

from oracle.oracle import Oracle
from parseable_b200 import _lib as L
from parseable_b200.query import (Agg, DateBin, Query, QueryError, StandardTableProvider, avg, col, count, count_distinct,
                                  count_star, date_bin, execute, max_, min_, sum_)

F64_REL = 1e-9


# ---- the CPU restatement -----------------------------------------------------------------------------------------
def _norm(v):
    """Key values as dictionary keys: NaN keys compare equal to each other."""
    return ("nan",) if isinstance(v, float) and math.isnan(v) else v


def _key_name(k):
    return k.name if isinstance(k, DateBin) else k


def expect_count_distinct(ora: Oracle, keys, column: str, filters=()) -> dict:
    """key tuple -> distinct non-NULL values of `column` among the selected rows of that group."""
    g = ora.group_by(list(keys) + [column], [count_star()], list(filters))
    nk = len(keys)
    cols = [g.column(i).to_pylist() for i in range(nk + 1)]
    out: dict = {}
    for r in range(g.num_rows):
        key = tuple(_norm(cols[k][r]) for k in range(nk))
        out[key] = out.get(key, 0) + (0 if cols[nk][r] is None else 1)
    if not keys and not out:
        out[()] = 0          # a global aggregate over zero rows: one row holding 0
    return out


def expect(ora: Oracle, keys, aggs, filters=()) -> dict:
    """key tuple -> {result column: value} for a mix of COUNT(DISTINCT) and the other aggregates."""
    plain = [a for a in aggs if a.fn != "count_distinct"]
    base = ora.group_by(list(keys), plain or [count_star()], list(filters))
    nk = len(keys)
    kcols = [base.column(i).to_pylist() for i in range(nk)]
    rows = {tuple(_norm(kcols[k][r]) for k in range(nk)): {} for r in range(base.num_rows)}
    for j, a in enumerate(plain):
        vals = base.column(nk + j).to_pylist()
        for r, key in enumerate(rows):
            rows[key][a.name] = vals[r]
    for a in aggs:
        if a.fn == "count_distinct":
            cd = expect_count_distinct(ora, keys, a.column, filters)
            for key in rows:
                rows[key][a.name] = cd.get(key, 0)
    return rows


def rows_of(t: pa.Table, keys) -> dict:
    nk = len(keys)
    names = t.column_names
    cols = [t.column(i).to_pylist() for i in range(t.num_columns)]
    return {tuple(_norm(cols[k][r]) for k in range(nk)): {names[c]: cols[c][r] for c in range(nk, len(names))}
            for r in range(t.num_rows)}


def assert_matches(got: pa.Table, exp: dict, keys, aggs):
    assert got.column_names == [_key_name(k) for k in keys] + [a.name for a in aggs]
    for i, a in enumerate(aggs):
        if a.fn == "count_distinct":
            c = got.column(len(keys) + i)
            assert c.type == pa.int64() and c.null_count == 0, a.name
    g = rows_of(got, keys)
    assert g.keys() == exp.keys()
    for key, vals in exp.items():
        for name, want in vals.items():
            have = g[key][name]
            if isinstance(want, float) and (name.startswith("sum(") or name.startswith("avg(")):
                assert have is not None and (math.isclose(have, want, rel_tol=F64_REL) or (math.isnan(have) and math.isnan(want))), (key, name)
            else:
                assert _norm(have) == _norm(want), (key, name, have, want)


@contextmanager
def env_var(name, value):
    old = os.environ.get(name)
    os.environ[name] = value
    try:
        yield
    finally:
        if old is None:
            del os.environ[name]
        else:
            os.environ[name] = old


def check(prov, ora, keys, aggs, flt=(), both_forms=True):
    """Oracle parity, and the dense bitmap and the pair set give the same table."""
    exp = expect(ora, keys, aggs, flt)
    got = prov.aggregate(keys, aggs, list(flt)).table()
    assert_matches(got, exp, keys, aggs)
    if both_forms:
        with env_var("PQB_DISTINCT_HASH", "1"):
            got_h = prov.aggregate(keys, aggs, list(flt)).table()
        assert_matches(got_h, exp, keys, aggs)


# ---- CPU: the restatement against Acero, hand vectors, SQL parsing --------------------------------------------------
def _acero(t: pa.Table, keys, column):
    if keys:
        r = t.group_by(keys).aggregate([(column, "count_distinct", pc.CountOptions(mode="only_valid"))])
        kc = [r[k].to_pylist() for k in keys]
        vc = r[f"{column}_count_distinct"].to_pylist()
        return {tuple(_norm(kc[i][j]) for i in range(len(keys))): vc[j] for j in range(r.num_rows)}
    return {(): pc.count_distinct(t[column], mode="only_valid").as_py()}


def test_oracle_count_distinct_matches_acero(built):
    rng = np.random.default_rng(7)
    n = 20_000
    t = pa.table({
        "k": pa.array(np.array(["a", "b", "c", None], dtype=object)[rng.integers(0, 4, n)], pa.string()),
        "k2": pa.array(rng.integers(0, 3, n).astype(np.int64)),
        "s": pa.array(np.where(rng.random(n) < 0.1, None, np.array([f"v{i}" for i in rng.integers(0, 500, n)], dtype=object)), pa.string()),
        "i": pa.array(np.where(rng.random(n) < 0.05, None, rng.integers(-50, 50, n)), pa.int64()),
        "f": pa.array(np.where(rng.random(n) < 0.05, None, np.round(rng.standard_normal(n), 2) + 10.0), pa.float64()),
        "b": pa.array(np.where(rng.random(n) < 0.3, None, rng.random(n) < 0.5), pa.bool_()),
        "nul": pa.nulls(n, pa.int64()),
    })
    ora = Oracle(t)
    for keys in ([], ["k"], ["k", "k2"]):
        for c in ("s", "i", "f", "b", "nul"):
            assert expect_count_distinct(ora, keys, c) == _acero(t, keys, c), (keys, c)
    # with a filter: only the selected rows count
    flt = [col("k2") == 1]
    sel = t.filter(pc.equal(t["k2"], 1))
    assert expect_count_distinct(ora, ["k"], "s", flt) == _acero(sel, ["k"], "s")
    assert expect_count_distinct(ora, [], "s", [col("k2") == 9]) == {(): 0}


def test_oracle_count_distinct_f64_bit_patterns(built):
    """f64 values are distinct by bit pattern: -0.0 and 0.0 differ, and so do NaNs with different payloads."""
    def nan(payload):
        return struct.unpack("<d", struct.pack("<Q", 0x7ff8000000000000 | payload))[0]
    vals = [-0.0, 0.0, nan(1), nan(2), nan(1), None, 1.0, 0.0, -0.0]
    t = pa.table({"k": pa.array(["x", "x", "x", "y", "y", "y", "y", "z", "z"]), "f": pa.array(vals, pa.float64())})
    ora = Oracle(t)
    assert expect_count_distinct(ora, [], "f") == {(): 5}
    assert expect_count_distinct(ora, ["k"], "f") == {("x",): 3, ("y",): 3, ("z",): 2}


def test_sql_count_distinct_parses():
    q = Query("SELECT status, COUNT(DISTINCT host) AS n, count(distinct \"path\"), COUNT(*) FROM logs WHERE level = 'ERROR' GROUP BY status")
    assert q.select[0] == ("col", "status", None)
    assert q.select[1] == ("agg", Agg("count_distinct", "host"), "n")
    assert q.select[2] == ("agg", Agg("count_distinct", "path"), None)
    assert q.select[3] == ("agg", Agg("count_star"), None)
    assert Agg("count_distinct", "path").name == "count(distinct path)"
    assert q.group_by == ["status"]
    assert Query("SELECT COUNT(DISTINCT host) FROM logs").select == [("agg", count_distinct("host"), None)]
    assert L.PQ_AGG_COUNT_DISTINCT == 6


# ---- GPU ----------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def logs(built, small_files):
    out = {}
    for tag, path in small_files.items():
        ora = Oracle.from_parquet(path)
        out[tag] = (ora, StandardTableProvider([path], schema=ora.table.schema))
    return out


CD = count_distinct
LOGS_CASES = {
    "global": ([], [CD("host")], []),
    "global_where": ([], [CD("host")], [col("level") == "ERROR"]),          # the alert form
    "global_zero_rows": ([], [CD("host"), count_star()], [col("level") == "NOPE"]),
    "grouped_status": (["status"], [CD("host")], []),
    "two_keys": (["region", "level"], [CD("path")], [col("latency_ms") > 30]),
    "date_bin_hosts_per_minute": ([date_bin("1m")], [CD("host")], []),
    "with_count_sum": (["host"], [count_star(), sum_("bytes"), CD("path")], []),
    "every_aggregate": (["level"], [count_star(), count("cpu"), sum_("bytes"), min_("latency_ms"), max_("cpu"), avg("score"),
                                    CD("host"), CD("status")], []),
    "same_column_twice": (["level"], [CD("host"), count("host"), CD("host")], []),
    "group_by_itself": (["status"], [CD("status"), count_star()], []),
    "plain_f64_and_delta_ts": (["level"], [CD("cpu"), CD("p_timestamp")], [col("status") == 200]),
    "contention_every_row": ([], [CD("status")], []),
}


@pytest.mark.gpu
@pytest.mark.parametrize("tag", ["nn", "nulls"])
@pytest.mark.parametrize("name", sorted(LOGS_CASES))
def test_count_distinct_logs(logs, tag, name):
    ora, prov = logs[tag]
    keys, aggs, flt = LOGS_CASES[name]
    check(prov, ora, keys, aggs, flt)


@pytest.mark.gpu
def test_count_distinct_zero_rows_and_small_grid(logs):
    ora, prov = logs["nulls"]
    assert prov.aggregate([], [CD("host")], [col("level") == "NOPE"]).table().to_pydict() == {"count(distinct host)": [0]}
    with env_var("PQB_GRID", "3"):   # every CTA takes many items, in every order
        check(prov, ora, ["level"], [CD("host"), count_star()], [col("latency_ms") > 10])


@pytest.mark.gpu
def test_count_distinct_column_kinds(data_dir, built):
    """Dictionary Utf8 / Int64, PLAIN Int64 / Float64, DELTA timestamps, Boolean, a column missing from one file, f64
    bit patterns, and one LZ4_RAW file."""
    rng = np.random.default_rng(41)
    n = 120_000

    def nan(payload):
        return struct.unpack("<d", struct.pack("<Q", 0x7ff8000000000000 | payload))[0]
    fvals = np.array([-0.0, 0.0, nan(1), nan(2), 1.5, -2.25], dtype=np.float64)
    f = fvals[rng.integers(0, len(fvals), n)]
    t = pa.table({
        "p_timestamp": pa.array((1_700_000_000_000 + np.cumsum(rng.integers(0, 3, n))).astype(np.int64), pa.timestamp("ms")),
        "g": pa.array(np.array(["a", "b", "c", None], dtype=object)[rng.integers(0, 4, n)], pa.string()),
        "s": pa.array(np.where(rng.random(n) < 0.05, None, np.array([f"user-{i}" for i in rng.integers(0, 3000, n)], dtype=object)), pa.string()),
        "di": pa.array(np.where(rng.random(n) < 0.05, None, rng.integers(0, 700, n)), pa.int64()),
        "pi": pa.array(rng.integers(-10**6, 10**6, n).astype(np.int64)),
        "pf": pa.array(np.where(rng.random(n) < 0.05, None, f), pa.float64()),
        "b": pa.array(np.where(rng.random(n) < 0.2, None, rng.random(n) < 0.3), pa.bool_()),
        "allnull": pa.nulls(n, pa.string()),
    })
    p1, p2, p3 = (os.path.join(data_dir, f"cd_kinds_{i}.parquet") for i in range(3))
    kw = dict(row_group_size=50_000, use_dictionary=["g", "s", "di", "b", "allnull"],
              column_encoding={"p_timestamp": "DELTA_BINARY_PACKED", "pi": "PLAIN", "pf": "PLAIN"}, data_page_size=64 << 10)
    half = n // 2
    pq.write_table(t.slice(0, half), p1, compression="NONE", **kw)
    pq.write_table(t.slice(half).drop_columns(["s"]), p2, compression="NONE", **kw)        # `s` missing from this file: NULL
    pq.write_table(t.slice(half), p3, compression="LZ4_RAW", **kw)
    schema = t.schema
    for files in ([p1, p2], [p3]):
        ora = Oracle.from_parquet(files)
        prov = StandardTableProvider(files, schema=schema)
        for keys, aggs, flt in (([], [CD("s"), CD("di"), CD("pi"), CD("pf"), CD("p_timestamp"), CD("b"), CD("allnull")], []),
                                (["g"], [CD("s"), CD("di"), CD("pf"), CD("b"), count_star()], [col("di") < 300]),
                                (["b"], [CD("g"), CD("pi"), sum_("di")], []),
                                ([date_bin("1m")], [CD("s"), CD("g")], [])):
            check(prov, ora, keys, aggs, flt)
    # -0.0 / 0.0 / NaN payloads: six distinct bit patterns
    prov = StandardTableProvider([p1, p2], schema=schema)
    assert prov.aggregate([], [CD("pf")]).table()["count(distinct pf)"].to_pylist() == [6]


@pytest.mark.gpu
def test_count_distinct_plain_fallback_and_refusals(data_dir, built):
    """The `message` chunk that flips from RLE_DICTIONARY to PLAIN mid-way (pages without a dictionary read as id
    pages), the hashed GROUP BY (70 001 x 978 combinations), and the refusals: the context answers afterwards."""
    rng = np.random.default_rng(23)
    n = 180_000
    words = np.array(["timeout", "retry", "upstream", "cache", "db", "panic", "ok", "queued", "δ-error", "reset"])
    uniq = np.array([f"req-{i:06d} " + " ".join(words[rng.integers(0, len(words), 4)]) for i in range(70_000)], dtype=object)
    msg = uniq[rng.integers(0, len(uniq), n)]
    msg[rng.random(n) < 0.03] = None
    tag = np.array([f"t{i % 977}-{'x' * (i % 7)}" for i in range(n)], dtype=object)
    tag[rng.random(n) < 0.01] = None
    t = pa.table({"id": pa.array(np.arange(n, dtype=np.int64)), "message": pa.array(msg, pa.string()), "tag": pa.array(tag, pa.string()),
                  "v": pa.array(rng.integers(0, 100, n).astype(np.int64))})
    p = os.path.join(data_dir, "cd_plain_strings.parquet")
    pq.write_table(t, p, compression="NONE", row_group_size=90_000, use_dictionary=["message", "v"], dictionary_pagesize_limit=1 << 20,
                   data_page_size=256 << 10)
    encs = {c.path_in_schema: set(c.encodings) for rg in range(2) for c in [pq.ParquetFile(p).metadata.row_group(rg).column(i) for i in range(4)]}
    assert "PLAIN" in encs["message"] and "RLE_DICTIONARY" in encs["message"], encs
    ora = Oracle(t)
    prov = StandardTableProvider([p], schema=t.schema)
    check(prov, ora, [], [CD("message"), CD("tag")], [col("v") < 50])
    check(prov, ora, ["v"], [CD("message"), count("message")], [])
    check(prov, ora, ["message"], [CD("message"), CD("tag")], [])
    check(prov, ora, ["message", "tag"], [count_star(), CD("v")], [])     # hashed GROUP BY: the pair set
    for aggs, flt in (([CD("message")], [col("message").like("%ok%")]),      # the id pages stand in for the values
                      ([CD("tag"), max_("id")], [col("tag") == "t5-xxxxx"])):
        with pytest.raises(QueryError) as e:
            prov.aggregate(["v"], aggs, flt)
        assert e.value.code == L.PQ_ERR_UNSUPPORTED and "COUNT(DISTINCT" in e.value.message
    with pytest.raises(QueryError) as e:
        prov.aggregate([], [CD("v")], [], flags=L.PQ_QUERY_ALLREDUCE)
    assert e.value.code == L.PQ_ERR_UNSUPPORTED and "COUNT(DISTINCT v)" in e.value.message
    check(prov, ora, ["v"], [CD("tag")], [], both_forms=False)            # still answers


@pytest.mark.gpu
def test_count_distinct_sql_and_json(logs):
    ora, prov = logs["nulls"]
    res = execute(Query("SELECT status, COUNT(DISTINCT host) AS n FROM logs GROUP BY status"), prov)
    t = res.table()
    assert t.column_names == ["status", "n"]
    exp = expect_count_distinct(ora, ["status"], "host")
    assert {(s,): v for s, v in zip(t["status"].to_pylist(), t["n"].to_pylist())} == exp
    res = prov.aggregate(["level"], [count_star(), CD("host")], json="array")
    t = res.table()
    assert res.to_json(fill_null=True) == t.to_pylist()
