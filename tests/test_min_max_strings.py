"""MIN / MAX over Utf8 and Boolean columns (PQ_AGG_MIN / PQ_AGG_MAX), reduced on the GPU.

GPU results are compared with `expect`, a CPU restatement built on the C oracle: every Utf8 input becomes the code of its
value in a bytewise-sorted dictionary (a prefix before any longer string), every Boolean input 0 / 1, the C oracle's
GROUP BY takes Int64 MIN / MAX of the codes over the rows it selects, and the codes are decoded back.  On the CPU that
restatement is checked against Acero's hash_min_max and against hand vectors."""
import math
import os
import subprocess
import sys

import numpy as np
import pyarrow as pa
import pyarrow.compute as pc
import pyarrow.parquet as pq
import pytest

from oracle.oracle import Oracle
from parseable_b200 import _lib as L
from parseable_b200.query import (Agg, DateBin, DeviceTable, Query, QueryError, StandardTableProvider, avg, col, count,
                                  count_distinct, count_star, date_bin, execute, max_, median, min_, sum_)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")


# ---- the CPU restatement -------------------------------------------------------------------------------------------
def _norm(v):
    return ("nan",) if isinstance(v, float) and math.isnan(v) else v


def _ranked(t: pa.Table, aggs):
    """t plus one Int64 code column per Utf8 / Boolean MIN / MAX input; returns (table, aggs over the codes, decoders)."""
    extra, mapped, decode = {}, [], {}
    for a in aggs:
        if a.fn not in ("min", "max") or a.column is None:
            mapped.append(a)
            continue
        typ = t.schema.field(a.column).type if a.column in t.column_names else None
        if typ is not None and pa.types.is_dictionary(typ):
            typ = typ.value_type
        if typ is None or not (pa.types.is_string(typ) or pa.types.is_large_string(typ) or pa.types.is_boolean(typ)):
            mapped.append(a)
            continue
        code = f"__code_{a.column}"
        if code not in extra:
            vals = t[a.column].to_pylist()
            if pa.types.is_boolean(typ):
                extra[code] = pa.array([None if v is None else int(v) for v in vals], pa.int64())
                decode[code] = lambda c: bool(c)
            else:
                # bytewise order: Python compares bytes lexicographically, a prefix first
                uniq = sorted({v.encode() for v in vals if v is not None})
                idx = {b: i for i, b in enumerate(uniq)}
                extra[code] = pa.array([None if v is None else idx[v.encode()] for v in vals], pa.int64())
                decode[code] = lambda c, u=uniq: u[c].decode()
        mapped.append(Agg(a.fn, code))
    for name, arr in extra.items():
        t = t.append_column(name, arr)
    return t, mapped, decode


def expect(ora: Oracle, keys, aggs, flt=()) -> dict:
    """key tuple -> {result column: value}."""
    t, mapped, decode = _ranked(ora.table, aggs)
    base = Oracle(t).group_by(list(keys), mapped, list(flt))
    nk = len(keys)
    cols = [base.column(i).to_pylist() for i in range(base.num_columns)]
    out = {}
    for r in range(base.num_rows):
        row = {}
        for j, (a, m) in enumerate(zip(aggs, mapped)):
            v = cols[nk + j][r]
            row[a.name] = decode[m.column](v) if (m.column in decode and v is not None) else v
        out[tuple(_norm(cols[k][r]) for k in range(nk))] = row
    return out


def rows_of(t: pa.Table, nk) -> dict:
    names = t.column_names
    cols = [t.column(i).to_pylist() for i in range(t.num_columns)]
    return {tuple(_norm(cols[k][r]) for k in range(nk)): {names[c]: cols[c][r] for c in range(nk, len(names))} for r in range(t.num_rows)}


def assert_matches(got: pa.Table, exp: dict, keys, aggs, types=None):
    assert got.column_names == [k.name if isinstance(k, DateBin) else k for k in keys] + [a.name for a in aggs]
    for i, a in enumerate(aggs):
        if types and a.name in types:
            assert got.column(len(keys) + i).type == types[a.name], (a.name, got.column(len(keys) + i).type)
    g = rows_of(got, len(keys))
    assert set(g) == set(exp), (len(g), len(exp))
    for key, vals in exp.items():
        for name, want in vals.items():
            have = g[key][name]
            if isinstance(want, float) and name.startswith(("sum(", "avg(")):
                assert have is not None and math.isclose(have, want, rel_tol=1e-9, abs_tol=1e-9), (key, name, have, want)
            else:
                assert _norm(have) == _norm(want), (key, name, have, want)


def check(prov, ora, keys, aggs, flt=(), types=None, **kw):
    res = prov.aggregate(keys, aggs, list(flt), **kw)
    got = res.table()
    assert_matches(got, expect(ora, keys, aggs, flt), keys, aggs, types)
    return res


# ---- CPU: the restatement against Acero and hand vectors, SQL parsing ----------------------------------------------
EDGE = ["", "a", "ab", "abc", "Z", "a\x00b", "a\x00", "é", "zz", "日本", "\U0001F600", "A", " ", "ab\x00"]


def _acero(t: pa.Table, keys, c):
    if keys:
        r = t.group_by(keys).aggregate([(c, "min"), (c, "max")])
        kc = [r[k].to_pylist() for k in keys]
        mn, mx = r[f"{c}_min"].to_pylist(), r[f"{c}_max"].to_pylist()
        return {tuple(kc[i][j] for i in range(len(keys))): {f"min({c})": mn[j], f"max({c})": mx[j]} for j in range(r.num_rows)}
    mm = pc.min_max(t[c]).as_py()
    return {(): {f"min({c})": mm["min"], f"max({c})": mm["max"]}}


def test_oracle_min_max_matches_acero(built):
    rng = np.random.default_rng(11)
    n = 20_000
    edge = np.array(EDGE, dtype=object)
    t = pa.table({
        "k": pa.array(np.array(["a", "b", "c", "d", None], dtype=object)[rng.integers(0, 5, n)], pa.string()),
        "k2": pa.array(rng.integers(0, 3, n).astype(np.int64)),
        "s": pa.array(np.where(rng.random(n) < 0.1, None, edge[rng.integers(0, len(edge), n)]), pa.string()),
        "w": pa.array(np.where(rng.random(n) < 0.05, None, np.array([f"v{i}" for i in rng.integers(0, 500, n)], dtype=object)), pa.string()),
        "b": pa.array(np.where(rng.random(n) < 0.3, None, rng.random(n) < 0.5), pa.bool_()),
    })
    # a group ("d") whose inputs are all NULL
    dmask = np.array([v == "d" for v in t["k"].to_pylist()])
    t = t.set_column(2, "s", pa.array([None if m else v for m, v in zip(dmask, t["s"].to_pylist())], pa.string()))
    t = t.set_column(4, "b", pa.array([None if m else v for m, v in zip(dmask, t["b"].to_pylist())], pa.bool_()))
    ora = Oracle(t)
    for keys in ([], ["k"], ["k", "k2"]):
        for c in ("s", "w", "b"):
            assert expect(ora, keys, [min_(c), max_(c)]) == _acero(t, keys, c), (keys, c)
    assert expect(ora, ["k"], [min_("s"), max_("b")])[("d",)] == {"min(s)": None, "max(b)": None}
    # with a filter: only the selected rows count; zero rows: one row holding NULL
    sel = t.filter(pc.equal(t["k2"], 1))
    assert expect(ora, ["k"], [min_("s"), max_("s")], [col("k2") == 1]) == _acero(sel, ["k"], "s")
    assert expect(ora, [], [min_("s"), max_("b"), count_star()], [col("k2") == 9]) == {(): {"min(s)": None, "max(b)": None, "count(*)": 0}}


def test_oracle_min_max_hand_vectors(built):
    """Bytewise order: "" first, a prefix before its extensions, "Z" < "a", NUL bytes, UTF-8 above ASCII; false < true."""
    t = pa.table({"g": ["x"] * len(EDGE), "s": EDGE})
    e = expect(Oracle(t), ["g"], [min_("s"), max_("s")])[("x",)]
    assert e == {"min(s)": "", "max(s)": "\U0001F600"}
    for vals, lo, hi in ((["ab", "abc", "abd"], "ab", "abd"), (["a", "Z"], "Z", "a"), (["a\x00b", "a\x00", "a"], "a", "a\x00b"),
                         (["z", "é"], "z", "é"), (["é", "日本"], "é", "日本"), ([None, "q", None], "q", "q"), ([None, None], None, None)):
        tt = pa.table({"s": pa.array(vals, pa.string())})
        assert expect(Oracle(tt), [], [min_("s"), max_("s")]) == {(): {"min(s)": lo, "max(s)": hi}}, vals
    for vals, lo, hi in (([True, None, False], False, True), ([True, None], True, True), ([None], None, None), ([False, False], False, False)):
        tt = pa.table({"b": pa.array(vals, pa.bool_())})
        assert expect(Oracle(tt), [], [min_("b"), max_("b")]) == {(): {"min(b)": lo, "max(b)": hi}}, vals


def test_sql_min_max_strings_parse():
    q = Query("SELECT host, MIN(level), max(path) AS last_path, MIN(active) FROM logs WHERE status = 200 GROUP BY host ORDER BY 3 DESC LIMIT 5")
    assert q.select[1] == ("agg", Agg("min", "level"), None)
    assert q.select[2] == ("agg", Agg("max", "path"), "last_path")
    assert q.select[3] == ("agg", Agg("min", "active"), None)
    assert q.group_by == ["host"]
    assert Agg("max", "path").name == "max(path)"
    assert L.PQ_AGG_MIN == 3 and L.PQ_AGG_MAX == 4


# ---- GPU: the logs16 files ------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def logs(built, small_files):
    out = {}
    for tag, path in small_files.items():
        ora = Oracle.from_parquet(path)
        out[tag] = (ora, StandardTableProvider([path], schema=ora.table.schema), path)
    return out


CASES = {
    "global": ([], [min_("host"), max_("host"), min_("path"), max_("message")], []),
    "global_zero_rows": ([], [count_star(), min_("host"), max_("level")], [col("level") == "NOPE"]),
    "one_key": (["status"], [min_("host"), max_("host")], []),
    "two_keys": (["region", "level"], [min_("pod"), max_("path"), count_star()], []),
    "date_bin": ([date_bin("1m")], [min_("service"), max_("service")], []),
    "selective": (["level"], [max_("path"), min_("pod")], [col("latency_ms") > 990]),
    "first_last_pod_per_region": (["region"], [min_("pod"), max_("pod")], []),
    "mixed": (["host"], [count_star(), min_("level"), sum_("bytes"), max_("level"), avg("latency_ms"), count("path"), min_("latency_ms")], []),
    "key_is_input": (["service"], [min_("service"), max_("service"), max_("method")], []),
}
STR = {a.name: pa.string() for _, aggs, _ in CASES.values() for a in aggs if a.fn in ("min", "max") and a.column not in ("latency_ms",)}


@pytest.mark.gpu
@pytest.mark.parametrize("tag", ["nn", "nulls"])
@pytest.mark.parametrize("name", sorted(CASES))
def test_min_max_strings_logs(logs, tag, name):
    ora, prov, _ = logs[tag]
    keys, aggs, flt = CASES[name]
    check(prov, ora, keys, aggs, flt, types=STR)


@pytest.mark.gpu
def test_min_max_with_distinct_median_hashed_grid_batches(logs):
    ora, prov, _ = logs["nulls"]
    aggs = [min_("host"), max_("host"), count_distinct("host"), max_("path")]
    exp = expect(ora, ["level"], [a for a in aggs if a.fn != "count_distinct"])
    got = rows_of(prov.aggregate(["level"], aggs).table(), 1)
    assert set(got) == set(exp)
    for k, v in exp.items():
        for name, want in v.items():
            assert got[k][name] == want, (k, name)
    want_cd = {tuple([lv]): len({h for h, l2 in zip(ora.table["host"].to_pylist(), ora.table["level"].to_pylist()) if l2 == lv and h is not None})
               for (lv,) in exp}
    assert {k: got[k]["count(distinct host)"] for k in got} == want_cd
    # next to MEDIAN (its own instantiation): the MEDIAN matches the plain query's
    res = prov.aggregate(["region"], [min_("service"), median("latency_ms"), max_("pod")]).table()
    assert_matches(res.select(["region", "min(service)", "max(pod)"]), expect(ora, ["region"], [min_("service"), max_("pod")]), ["region"],
                   [min_("service"), max_("pod")])
    ref = prov.aggregate(["region"], [median("latency_ms")]).table()
    assert dict(zip(res["region"].to_pylist(), res["median(latency_ms)"].to_pylist())) == dict(zip(ref["region"].to_pylist(), ref["median(latency_ms)"].to_pylist()))
    # a hashed GROUP BY (host x pod x path: a key space wider than the dense table)
    check(prov, ora, ["host", "pod", "path"], [min_("level"), max_("service"), count_star()])
    # a small grid (every CTA takes many items) and batches smaller than the result
    old = os.environ.get("PQB_GRID")
    os.environ["PQB_GRID"] = "3"
    try:
        check(prov, ora, ["status"], [min_("path"), max_("path")], [col("latency_ms") > 10])
    finally:
        if old is None:
            del os.environ["PQB_GRID"]
        else:
            os.environ["PQB_GRID"] = old
    res = check(prov, ora, ["status", "level"], [min_("host"), max_("message")], batch_size=7)
    assert len(res.batches) > 1


@pytest.mark.gpu
def test_min_max_resident_table_and_shards(logs):
    ora, _, path = logs["nulls"]
    dt = DeviceTable([path], ["host", "status", "level", "path", "pod", "bytes"])
    try:
        prov = StandardTableProvider(dt, schema=ora.table.schema)
        for _ in range(2):   # the second query reads the rank tables the table column keeps
            check(prov, ora, ["status"], [min_("host"), max_("path"), sum_("bytes")], types=STR)
            check(prov, ora, ["host"], [min_("host"), max_("level"), max_("bytes")])   # the key's id pages serve its MIN
    finally:
        dt.close()
    t = ora.table
    n_rg = pq.ParquetFile(path).metadata.num_row_groups
    bounds = np.cumsum([0] + [pq.ParquetFile(path).metadata.row_group(g).num_rows for g in range(n_rg)])
    for shard in range(2):
        part = pa.concat_tables([t.slice(bounds[g], bounds[g + 1] - bounds[g]) for g in range(n_rg) if g % 2 == shard])
        prov = StandardTableProvider([path], schema=t.schema, shard_index=shard, shard_count=2)
        check(prov, Oracle(part), ["level"], [min_("host"), max_("pod")])


@pytest.mark.gpu
def test_min_max_dictionaries_in_different_orders(data_dir, built):
    """Two files whose dictionaries hold the same strings in opposite orders (and row groups of one file, too): the
    answer is over the whole table, not per chunk."""
    vals = ["delta", "alpha", "Charlie", "bravo", "", "echo", "alpha-2", "ä"]
    rng = np.random.default_rng(3)
    n = 40_000
    def table(order):
        v = np.array(order, dtype=object)[rng.integers(0, len(order), n)]
        v[: len(order)] = order    # first occurrences fix the dictionary order
        return pa.table({"g": pa.array(rng.integers(0, 5, n).astype(np.int64)), "s": pa.array(v, pa.string())})
    p1, p2 = (os.path.join(data_dir, f"mm_order_{i}.parquet") for i in range(2))
    pq.write_table(table(vals), p1, row_group_size=n, use_dictionary=True, compression="NONE")
    pq.write_table(table(vals[::-1]), p2, row_group_size=n // 2, use_dictionary=True, compression="NONE")
    ora = Oracle.from_parquet([p1, p2])
    prov = StandardTableProvider([p1, p2], schema=ora.table.schema)
    check(prov, ora, [], [min_("s"), max_("s")])
    check(prov, ora, ["g"], [min_("s"), max_("s")])
    assert prov.aggregate([], [min_("s"), max_("s")]).table().to_pydict() == {"min(s)": [""], "max(s)": ["ä"]}


@pytest.mark.gpu
def test_min_max_pages_without_dictionary(data_dir, built):
    """A column whose dictionary overflows into PLAIN pages and one written as DELTA_BYTE_ARRAY: MIN / MAX read their id
    pages, together with GROUP BY and COUNT(DISTINCT) on the same column; filtering on it as well is refused."""
    rng = np.random.default_rng(23)
    n = 150_000
    # ~40 bytes x 60 000 values: the dictionary outgrows its 1 MiB limit and the chunk falls back to PLAIN pages
    uniq = np.array([f"req-{i:06d}-{'é' * (i % 3)} upstream timeout retry cache-miss" for i in range(60_000)], dtype=object)
    msg = uniq[rng.integers(0, len(uniq), n)]
    msg[rng.random(n) < 0.03] = None
    dba = np.array([f"k{i % 911:04d}{'z' * (i % 5)}" for i in range(n)], dtype=object)
    dba[rng.random(n) < 0.02] = None
    t = pa.table({"v": pa.array(rng.integers(0, 50, n).astype(np.int64)), "message": pa.array(msg, pa.string()),
                  "dba": pa.array(dba, pa.string())})
    p = os.path.join(data_dir, "mm_plain_strings.parquet")
    pq.write_table(t, p, compression="NONE", row_group_size=75_000, use_dictionary=["message", "v"], dictionary_pagesize_limit=1 << 20,
                   data_page_size=256 << 10, column_encoding={"dba": "DELTA_BYTE_ARRAY"})
    from test_meta import describe
    pages = [[pg["encoding"] for pg in c["pages"]] for c in describe(L.load(), p)["row_groups"][0]["columns"]]
    assert 8 in pages[1] and 0 in pages[1][2:], pages[1]     # message: RLE_DICTIONARY pages, then the PLAIN fallback
    assert set(pages[2]) == {7}, pages[2]                     # dba: DELTA_BYTE_ARRAY only
    ora = Oracle(t)
    prov = StandardTableProvider([p], schema=t.schema)
    check(prov, ora, [], [min_("message"), max_("message"), min_("dba"), max_("dba")], [col("v") < 25])
    check(prov, ora, ["v"], [min_("message"), max_("dba"), count("message")])
    check(prov, ora, ["message"], [min_("message"), max_("message"), count_star()])
    check(prov, ora, ["dba"], [max_("dba"), min_("message")])
    res = prov.aggregate(["v"], [min_("message"), count_distinct("message"), max_("dba"), count_distinct("dba")]).table()
    exp = expect(ora, ["v"], [min_("message"), max_("dba")])
    for r in res.to_pylist():
        assert r["min(message)"] == exp[(r["v"],)]["min(message)"] and r["max(dba)"] == exp[(r["v"],)]["max(dba)"]
        sub = [m for m, v in zip(t["message"].to_pylist(), t["v"].to_pylist()) if v == r["v"] and m is not None]
        assert r["count(distinct message)"] == len(set(sub))
    for aggs, flt in (([min_("message")], [col("message").like("%req-00%")]), ([max_("dba")], [col("dba") == "k0001z"])):
        try:
            r = prov.aggregate(["v"], aggs, flt)
            raise AssertionError(f"{aggs[0].name} filtered on its own column was not refused: {r.metrics}")
        except QueryError as e:
            assert e.code == L.PQ_ERR_UNSUPPORTED and aggs[0].name.split("(")[0].upper() + "(" in e.message, e.message
    check(prov, ora, ["v"], [max_("message")])   # still answers


@pytest.mark.gpu
def test_min_max_booleans_and_missing_columns(data_dir, built):
    gold = os.path.join(GOLDEN, "field_stats_10rows.parquet")
    ora = Oracle.from_parquet(gold, columns=["id", "name", "active", "score"])
    prov = StandardTableProvider([gold], schema=ora.table.schema)
    b = {"min(active)": pa.bool_(), "max(active)": pa.bool_(), "min(name)": pa.string(), "max(name)": pa.string()}
    check(prov, ora, [], [min_("active"), max_("active"), min_("name"), max_("name")], types=b)
    check(prov, ora, ["name"], [min_("active"), max_("active"), count_star()], types=b)
    check(prov, ora, ["active"], [min_("name"), max_("name"), max_("id")], types=b)
    assert prov.aggregate([], [min_("active"), max_("active"), min_("name")]).table().to_pydict() == {
        "min(active)": [False], "max(active)": [True], "min(name)": ["Alice"]}
    # a generated Boolean with NULLs and an all-NULL group; a Utf8 column missing from one file, another from every file
    rng = np.random.default_rng(8)
    n = 90_000
    g = rng.integers(0, 6, n)
    flag = np.where(rng.random(n) < 0.2, None, rng.random(n) < 0.1)
    flag[g == 5] = None
    t = pa.table({"g": pa.array(g.astype(np.int64)), "flag": pa.array(flag, pa.bool_()),
                  "s": pa.array(np.where(rng.random(n) < 0.05, None, np.array([f"s{i}" for i in rng.integers(0, 300, n)], dtype=object)), pa.string())})
    p1, p2 = (os.path.join(data_dir, f"mm_bool_{i}.parquet") for i in range(2))
    pq.write_table(t.slice(0, n // 2), p1, row_group_size=30_000, compression="NONE")
    pq.write_table(t.slice(n // 2).drop_columns(["s"]), p2, row_group_size=30_000, compression="NONE")   # `s` missing: NULL
    schema = pa.schema(list(t.schema) + [pa.field("nowhere", pa.string())])
    ora = Oracle.from_parquet([p1, p2])
    prov = StandardTableProvider([p1, p2], schema=schema)
    types = {"min(flag)": pa.bool_(), "max(flag)": pa.bool_(), "min(s)": pa.string(), "max(s)": pa.string()}
    check(prov, ora, ["g"], [min_("flag"), max_("flag"), min_("s"), max_("s")], types=types)
    check(prov, ora, [], [min_("flag"), max_("flag"), min_("s"), max_("s")], [col("g") < 3], types=types)
    got = prov.aggregate(["g"], [min_("nowhere"), max_("nowhere"), max_("flag")]).table()
    assert got["min(nowhere)"].type == pa.string() and got["min(nowhere)"].null_count == got.num_rows
    assert got["max(nowhere)"].null_count == got.num_rows
    assert prov.aggregate([], [max_("nowhere")]).table().to_pydict() == {"max(nowhere)": [None]}


@pytest.mark.gpu
@pytest.mark.parametrize("limit", [None, 1, 7])
def test_min_max_order_by(logs, limit):
    """ORDER BY max(path) DESC [LIMIT n] and min(level) NULLS FIRST under every ORDER BY path: a stable host sort of the
    unordered result (of a resident table: its group numbering, the order of tied rows, is the same for every query)."""
    from test_order_by import check_ordered
    ora, _, path = logs["nulls"]
    dt = DeviceTable([path], ["host", "status", "level", "path", "region"])
    try:
        prov = StandardTableProvider(dt, schema=ora.table.schema)
        aggs = [count_star(), max_("path"), min_("level")]
        check_ordered(prov, None, ["host"], aggs, [(max_("path"), "desc")], limit=limit)
        check_ordered(prov, None, ["region", "status"], aggs, [(min_("level"), "asc", True), (max_("path"), "asc")], limit=limit)
    finally:
        dt.close()


@pytest.mark.gpu
def test_min_max_boolean_order_by(built):
    from test_order_by import check_ordered
    gold = os.path.join(GOLDEN, "field_stats_10rows.parquet")
    ora = Oracle.from_parquet(gold, columns=["id", "name", "active"])
    prov = StandardTableProvider([gold], schema=ora.table.schema)
    for limit in (None, 2):
        check_ordered(prov, None, ["name"], [min_("active"), max_("id")], [(min_("active"), "asc", True)], limit=limit)
        check_ordered(prov, None, ["name"], [max_("active")], [(max_("active"), "desc")], limit=limit)


@pytest.mark.gpu
def test_min_max_json_and_sql(logs):
    ora, prov, _ = logs["nulls"]
    for fmt in ("array", "lines"):
        res = prov.aggregate(["level"], [min_("host"), max_("path"), count_star()], json=fmt)
        assert res.to_json(fill_null=True) == res.table().to_pylist()
    res = prov.aggregate([], [min_("host"), max_("level")], [col("level") == "NOPE"], json="array")
    assert res.to_json(fill_null=True) == res.table().to_pylist() == [{"min(host)": None, "max(level)": None}]
    res = execute(Query("SELECT service, MAX(path) AS last_path, MIN(host) FROM logs GROUP BY service ORDER BY 2 DESC LIMIT 5"), prov)
    t = res.table()
    assert t.column_names == ["service", "last_path", "min(host)"] and t.num_rows == 5
    exp = expect(ora, ["service"], [max_("path"), min_("host")])
    want = sorted(exp.items(), key=lambda kv: (kv[1]["max(path)"] is not None, kv[1]["max(path)"] or ""), reverse=True)
    assert t["last_path"].to_pylist() == [v["max(path)"] for _, v in want[:5]]
    for r in t.to_pylist():
        assert r["min(host)"] == exp[(r["service"],)]["min(host)"]


@pytest.mark.gpu
def test_min_max_refusals(logs):
    ora, prov, _ = logs["nulls"]
    old = os.environ.get("PQB_FLAT_SCAN")
    os.environ["PQB_FLAT_SCAN"] = "0"   # every item goes to the k_scan path
    try:
        for aggs in ([min_("host")], [max_("level"), count_star()]):
            with pytest.raises(QueryError) as e:
                prov.aggregate(["status"], aggs)
            assert e.value.code == L.PQ_ERR_UNSUPPORTED and "flat-store copy" in e.value.message, e.value.message
    finally:
        if old is None:
            del os.environ["PQB_FLAT_SCAN"]
        else:
            os.environ["PQB_FLAT_SCAN"] = old
    for aggs in ([sum_("host")], [avg("level")], [median("host")]):
        with pytest.raises(QueryError) as e:
            prov.aggregate([], aggs)
        assert e.value.code == L.PQ_ERR_UNSUPPORTED and "not on the GPU path" in e.value.message
    check(prov, ora, ["level"], [min_("host")])   # the context still answers


# ---- multi-GPU: PQ_QUERY_ALLREDUCE --------------------------------------------------------------------------------
def _mgpu(tmp_path, n, files):
    idfile = str(tmp_path / f"nccl_id_{n}")
    procs = [subprocess.Popen([sys.executable, os.path.join(ROOT, "tests", "scripts", "mgpu_minmax_check.py"), str(r), str(n), idfile] + files,
                              stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True) for r in range(n)]
    outs = [p.communicate(timeout=600)[0] for p in procs]
    for r, (p, o) in enumerate(zip(procs, outs)):
        assert p.returncode == 0, f"rank {r}:\n{o[-3000:]}"
        assert "parity OK" in o


@pytest.mark.gpu
def test_min_max_allreduce_one_rank(small_files, tmp_path, built):
    _mgpu(tmp_path, 1, [small_files["nulls"], small_files["nn"]])


@pytest.mark.gpu
def test_min_max_allreduce_two_ranks(small_files, tmp_path, built):
    if L.load().pq_device_count() < 2:
        pytest.skip("needs 2 GPUs")
    _mgpu(tmp_path, 2, [small_files["nulls"], small_files["nn"]])
