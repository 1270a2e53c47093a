"""ORDER BY [... LIMIT n] over aggregate results, sorted on the device (PqQueryDesc.order_by).

The central oracle: for every case the ordered result equals a stable host sort of the same query's unordered GPU
result (whose values the rest of the suite checks against the C oracle), cut to the limit, in every column and every
row.  The sort-key tuples are also checked against the C oracle's GROUP BY result sorted the same way.  Float64 SUM /
AVG terms run on integer-valued data, so their sums are exact and the order is well defined."""
import math
import os
import struct
from contextlib import contextmanager

import numpy as np
import pyarrow as pa
import pyarrow.parquet as pq
import pytest

from oracle.oracle import Oracle
from parseable_b200 import _lib as L
from parseable_b200.query import (Agg, DateBin, DeviceTable, Query, QueryError, StandardTableProvider, avg, col, count, count_distinct,
                                  count_star, date_bin, execute, field_stats, max_, min_, sum_)


@contextmanager
def env_var(name, value):
    old = os.environ.get(name)
    if value is None:
        os.environ.pop(name, None)
    else:
        os.environ[name] = value
    try:
        yield
    finally:
        if old is None:
            os.environ.pop(name, None)
        else:
            os.environ[name] = old


# ---- the host restatement of the order -------------------------------------------------------------------------------
def _total_order(x: float) -> int:
    b = struct.unpack("<Q", struct.pack("<d", x))[0]
    mag = b & ((1 << 63) - 1)
    return -mag - 1 if b >> 63 else mag


def _vkey(v):
    if isinstance(v, bool):
        return int(v)
    if isinstance(v, float):
        return _total_order(v)
    if isinstance(v, str):
        return v.encode()
    if hasattr(v, "timestamp"):          # Timestamp(ms) values come back as datetimes
        return int(v.timestamp() * 1000)
    return v


def host_order(t: pa.Table, terms):
    """Row indices of a stable sort of t; terms = [(column, desc, nulls_first)]."""
    cols = []
    for name, desc, nulls_first in terms:
        vals = t[name].to_pylist()
        distinct = sorted({_vkey(v) for v in vals if v is not None})
        rank = {k: i for i, k in enumerate(distinct)}
        cols.append([(0 if nulls_first else 2, 0) if v is None else (1, -rank[_vkey(v)] if desc else rank[_vkey(v)]) for v in vals])
    return sorted(range(t.num_rows), key=lambda i: tuple(c[i] for c in cols))


def canon(t: pa.Table):
    """Rows as tuples, floats by bit pattern (NaN == NaN, -0.0 != 0.0)."""
    cols = [[struct.pack("<d", v) if isinstance(v, float) else v for v in t.column(i).to_pylist()] for i in range(t.num_columns)]
    return list(zip(*cols)) if cols else []


def _name(item, aggs):
    if isinstance(item, Agg):
        return item.name
    if isinstance(item, DateBin):
        return item.name
    return item


def check_ordered(prov, ora, keys, aggs, order, limit=None, flt=(), paths=("", "cta", "topk", "sort"), batch_size=0):
    base = prov.aggregate(keys, aggs, list(flt))
    unordered = base.table() if base.batches else None
    terms = [(_name(it, aggs), d == "desc", (d == "desc") if len(o) < 3 or o[2] is None else o[2])
             for o in order for it, d in [o[:2]]]
    results = []
    for path in paths:
        with env_var("PQB_ORDER_PATH", path or None):
            res = prov.aggregate(keys, aggs, list(flt), order_by=order, limit=limit, batch_size=batch_size)
        n_total = unordered.num_rows if unordered is not None else 0
        want_n = n_total if limit is None else min(limit, n_total)
        assert res.metrics["groups_total"] == max(n_total, base.metrics["groups"])
        assert res.metrics["groups"] == want_n
        if want_n == 0:
            assert res.batches == [] or res.table().num_rows == 0
            continue
        got = res.table()
        idx = host_order(unordered, terms)[:want_n]
        assert got.column_names == unordered.column_names
        assert canon(got) == canon(unordered.take(pa.array(idx, pa.int64()))), (path, order, limit)
        assert res.metrics["order_ms"] >= 0
        results.append(got)
    # the sort-key tuples against the C oracle's GROUP BY, sorted the same way
    if (ora is not None and unordered is not None and all(not isinstance(k, DateBin) for k in keys)
            and all(a.fn != "count_distinct" for a in aggs)):
        exp = ora.group_by(list(keys), list(aggs), list(flt))
        names = [t[0] for t in terms]
        if all(n in exp.column_names for n in names) and all(not n.startswith(("sum(", "avg(")) for n in names):
            eidx = host_order(exp, terms)[: (exp.num_rows if limit is None else min(limit, exp.num_rows))]
            want = canon(exp.take(pa.array(eidx, pa.int64())).select(names))
            for got in results:
                assert canon(got.select(names)) == want
    return results


# ---- data ----------------------------------------------------------------------------------------------------------------
def nan(payload, neg=False):
    return struct.unpack("<d", struct.pack("<Q", (1 << 63 if neg else 0) | 0x7FF0000000000000 | payload))[0]


@pytest.fixture(scope="module")
def data(data_dir, built):
    rng = np.random.default_rng(77)
    n = 240_000
    svals = np.array(["", "a", "ab", "abc", "b", "zz", "δ-x", "user-%03d"] + [f"user-{i:03d}" for i in range(200)], dtype=object)
    s = svals[rng.integers(0, len(svals), n)]
    s[rng.random(n) < 0.03] = None
    ivals = np.array([-(1 << 63), (1 << 63) - 1, -5, 0, 7] + list(range(100, 160)), dtype=object)
    i = ivals[rng.integers(0, len(ivals), n)]
    i[rng.random(n) < 0.02] = None
    fvals = np.array([-0.0, 0.0, math.inf, -math.inf, nan(1), nan(3, True), 1.5, -2.25, 3.0, 100.0], dtype=np.float64)
    f = fvals[rng.integers(0, len(fvals), n)].astype(object)
    f[rng.random(n) < 0.02] = None
    b = (rng.random(n) < 0.4).astype(object)
    b[rng.random(n) < 0.1] = None
    ts = (1_700_000_000_000 + np.sort(rng.integers(0, 3_600_000, n))).astype(np.int64)
    msg = np.array([f"req-{k:06d} {'x' * (k % 13)}" for k in rng.integers(0, 130_000, n)], dtype=object)
    v = rng.integers(-1000, 1000, n).astype(np.int64)
    v[rng.random(n) < 0.01] = (1 << 62)                                  # SUM(v) wraps in a few groups
    x = rng.integers(-50, 50, n).astype(np.float64)                       # integer-valued: exact sums
    nv = np.where(np.isin(s, ["a", "zz"]) | (rng.random(n) < 0.3), None, rng.integers(-9, 9, n)).astype(object)   # all-NULL groups
    last = rng.integers(0, 5, n).astype(np.int64)
    t = pa.table({"p_timestamp": pa.array(ts, pa.timestamp("ms")), "s": pa.array(s, pa.string()), "i": pa.array(i, pa.int64()),
                  "f": pa.array(f, pa.float64()), "b": pa.array(b, pa.bool_()), "msg": pa.array(msg, pa.string()),
                  "v": pa.array(v), "x": pa.array(x), "nv": pa.array(nv, pa.int64()), "last": pa.array(last),
                  "u": pa.array(rng.integers(0, 150_000, n).astype(np.int64))})
    p = os.path.join(data_dir, "order_by.parquet")
    pq.write_table(t, p, compression="NONE", row_group_size=120_000, use_dictionary=["s", "i", "f", "b", "msg", "nv", "last", "u"],
                   dictionary_pagesize_limit=256 << 10, data_page_size=128 << 10)
    md = pq.ParquetFile(p).metadata
    assert "PLAIN" in md.row_group(0).column(5).encodings                   # `msg` falls back to PLAIN pages
    # a resident table: its group ids (numbered hot-first) and so the slot order that breaks ties are built once;
    # a file list opens, and numbers, the table anew for every query
    table = DeviceTable([p], t.column_names)
    yield Oracle(t), StandardTableProvider(table, schema=t.schema), t
    table.close()


KEY_TERMS = ["s", "msg", "i", "f", "p_timestamp", "b", "db"]


@pytest.mark.gpu
@pytest.mark.parametrize("key", KEY_TERMS)
@pytest.mark.parametrize("direction,nulls_first", [("asc", False), ("asc", True), ("desc", False), ("desc", True)])
def test_every_key_kind(data, key, direction, nulls_first):
    ora, prov, _ = data
    k = date_bin("1m") if key == "db" else key
    kname = k.name if key == "db" else key
    limit = None if key not in ("msg", "p_timestamp") else 3000
    check_ordered(prov, ora if key != "db" else None, [k], [count_star()], [(kname, direction, nulls_first)], limit)


AGG_TERMS = [count_star(), count("nv"), count_distinct("i"), sum_("v"), sum_("x"), avg("x"), min_("v"), max_("v"),
             min_("f"), max_("f"), sum_("nv"), min_("nv")]


@pytest.mark.gpu
@pytest.mark.parametrize("agg", AGG_TERMS, ids=lambda a: a.name)
@pytest.mark.parametrize("direction,nulls_first", [("asc", None), ("desc", None), ("asc", True), ("desc", False)])
def test_every_aggregate_term(data, agg, direction, nulls_first):
    ora, prov, _ = data
    aggs = [agg] if agg.fn == "count_star" else [agg, count_star()]
    check_ordered(prov, ora, ["s"], aggs, [(agg, direction, nulls_first)], 40)


@pytest.mark.gpu
def test_multi_term_shapes_and_limits(data):
    ora, prov, _ = data
    # the counts / histogram shape, and status-like ASC + count DESC
    check_ordered(prov, None, [date_bin("5m"), "s"], [count_star()], [("date_bin(p_timestamp)", "asc"), ("s", "asc")])
    check_ordered(prov, ora, ["b", "s"], [count_star(), sum_("v")], [("b", "asc"), (count_star(), "desc")])
    # a multi-word pack: full-range Int64 key with NULLs, f64 key, two aggregates
    for limit in (None, 0, 1, 17, 10_000):
        check_ordered(prov, ora, ["i", "f", "b"], [count_star(), min_("v")],
                      [("i", "desc", False), ("f", "asc", True), (min_("v"), "desc"), ("b", "asc")], limit)
    # ties straddling the limit: many groups share a count
    res = check_ordered(prov, ora, ["last", "b"], [count_star()], [("last", "asc")], 4)
    assert res[0].num_rows == 4


@pytest.mark.gpu
def test_many_groups_radix_and_batches(data):
    """> 100 000 groups: the multi-tile radix passes; small batches carry the order across batch boundaries."""
    ora, prov, _ = data
    for limit in (None, 5, 4096, 4097):
        check_ordered(prov, ora, ["u"], [count_star(), sum_("x")], [(count_star(), "desc"), (sum_("x"), "asc")], limit,
                      paths=("", "topk", "sort"), batch_size=997)
    # top-K with ties straddling the cut: ~150 000 groups share a handful of counts, the tied groups kept are the first
    # in slot order; one term, so the key is one word and `topk` is the default for these limits
    for limit in (1, 7, 1000, 4096):
        check_ordered(prov, ora, ["u"], [count_star()], [(count_star(), "desc")], limit, paths=("", "topk", "sort"))
        check_ordered(prov, None, ["msg"], [count_star()], [(count_star(), "asc")], limit, paths=("", "topk"))
    res = prov.aggregate(["u"], [count_star()], order_by=[("u", "desc")], batch_size=1000)
    assert len(res.batches) > 100 and res.table()["u"].to_pylist() == sorted(res.table()["u"].to_pylist(), reverse=True)


@pytest.mark.gpu
def test_hashed_group_by_with_limit(data):
    ora, prov, _ = data
    # a hashed table's slots are hash-table cells, placed by insertion races: the unordered order, and so the order of
    # tied rows, may differ from one query to the next.  These orders are total (every key is a term).
    total = [("msg", "asc"), ("s", "asc", True), ("i", "desc", False)]
    check_ordered(prov, None, ["msg", "s", "i"], [count_star(), max_("x")], [(count_star(), "desc")] + total, 100,
                  paths=("", "topk", "sort"))
    check_ordered(prov, None, ["msg", "s", "i"], [count_star()], [(count_star(), "desc")] + total, 3000, paths=("", "topk", "sort"))


@pytest.mark.gpu
def test_global_aggregate_json_and_metrics(data):
    ora, prov, _ = data
    one = prov.aggregate([], [count_star(), sum_("v")], order_by=[(sum_("v"), "desc")], limit=5)
    assert one.table().num_rows == 1 and one.metrics["groups_total"] == 1
    for aggs in ([count_star()], [count_star(), sum_("v")]):
        zero = prov.aggregate([], aggs, order_by=[(count_star(), "asc")], limit=0)
        assert zero.metrics["groups"] == 0 and zero.metrics["groups_total"] == 1 and (zero.batches == [] or zero.table().num_rows == 0)
    plain = prov.aggregate(["s"], [count_star()])
    assert plain.metrics["order_ms"] == 0 and plain.metrics["groups_total"] == plain.metrics["groups"]
    # without ORDER BY the aggregate path ignores `limit`, and the kernels it launches are the same
    lim = prov.aggregate(["s"], [count_star()], limit=3)
    assert lim.metrics["groups"] == plain.metrics["groups"] and lim.metrics["kernel_launches"] == plain.metrics["kernel_launches"]
    res = prov.aggregate(["s"], [count_star(), avg("x")], order_by=[(count_star(), "desc"), ("s", "asc")], limit=25, json="array")
    assert res.to_json(fill_null=True) == res.table().to_pylist()


@pytest.mark.gpu
def test_refusals(data):
    ora, prov, _ = data
    with pytest.raises(QueryError) as e:
        prov._run([], [], [], ["s"], None, 0, 0, order=[(L.PQ_ORDER_KEY, 0, 0)])
    assert e.value.code == L.PQ_ERR_UNSUPPORTED and "ORDER BY" in e.value.message
    for order in ([(L.PQ_ORDER_KEY, 1, 0)], [(L.PQ_ORDER_AGG, 2, 0)], [(7, 0, 0)], [(L.PQ_ORDER_KEY, -1, 0)]):
        with pytest.raises(QueryError) as e:
            prov._run([], ["s"], [count_star()], [], None, 0, 0, order=order)
        assert e.value.code == L.PQ_ERR_INVALID_ARG
    with pytest.raises(QueryError) as e:
        prov._run([], ["s"], [count_star()], [], None, 0, 0, order=[(L.PQ_ORDER_AGG, 0, 0)] * 9)
    assert e.value.code == L.PQ_ERR_UNSUPPORTED
    with pytest.raises(QueryError) as e:
        prov.aggregate(["s"], [count_star()], order_by=[("nope", "asc")])
    assert e.value.code == L.PQ_ERR_INVALID_ARG
    check_ordered(prov, ora, ["s"], [count_star()], [(count_star(), "desc")], 3)   # still answers


@pytest.mark.gpu
def test_sql_front(data):
    ora, prov, _ = data
    res = execute(Query("SELECT last, COUNT(*) AS c FROM t GROUP BY last ORDER BY c DESC, last NULLS FIRST LIMIT 3"), prov)
    t = res.table()
    base = prov.aggregate(["last"], [count_star()]).table()
    idx = host_order(base, [("count(*)", True, True), ("last", False, True)])[:3]
    assert t.column_names == ["last", "c"] and canon(t) == canon(base.take(pa.array(idx, pa.int64())))
    # a position, an aggregate only ORDER BY names (computed, then dropped), and a grouped LIMIT without ORDER BY
    res = execute(Query("SELECT s AS name, COUNT(*) FROM t GROUP BY s ORDER BY SUM(v) DESC, 1 LIMIT 5"), prov)
    t = res.table()
    base = prov.aggregate(["s"], [count_star(), sum_("v")]).table()
    idx = host_order(base, [("sum(v)", True, True), ("s", False, False)])[:5]
    assert t.column_names == ["name", "count(*)"]
    assert canon(t) == canon(base.take(pa.array(idx, pa.int64())).select(["s", "count(*)"]))
    assert execute(Query("SELECT s, COUNT(*) FROM t GROUP BY s LIMIT 4"), prov).table().num_rows == 4
    with pytest.raises(QueryError) as e:
        execute(Query("SELECT s FROM t ORDER BY s"), prov)
    assert e.value.code == L.PQ_ERR_UNSUPPORTED


def test_sql_order_by_parses():
    q = Query("SELECT last, count(*) AS c FROM logs WHERE last > 1 GROUP BY last ORDER BY c desc, last ASC NULLS LAST, 2, "
              "SUM(bytes) LIMIT 7")
    assert q.group_by == ["last"] and q.limit == 7
    assert q.order_by == [(("name", "c"), "desc", None), (("name", "last"), "asc", False), (("pos", 2), "asc", None),
                          (("agg", sum_("bytes")), "asc", None)]
    # the words stay column names everywhere else
    q = Query("SELECT nulls, COUNT(*) FROM t GROUP BY nulls ORDER BY nulls")
    assert q.group_by == ["nulls"] and q.order_by == [(("name", "nulls"), "asc", None)]
    assert Query("SELECT COUNT(*) FROM t WHERE last = 1").order_by == []


@pytest.mark.gpu
def test_field_stats_high_cardinality(data):
    """field_stats is one ordered, cut device query; it returns exactly what the host computation it replaces did:
    GROUP BY field -> COUNT(*), a stable sort by count descending on the host, the sum and number of the groups."""
    ora, prov, _ = data

    def old_field_stats(provider, field, k, filters=()):
        t = provider.aggregate([field], [count_star()], list(filters)).table()
        vals, cnts = t[field].to_pylist(), t["count(*)"].to_pylist()
        order = sorted(range(len(vals)), key=lambda i: -cnts[i])
        return sum(cnts), len(vals), [(vals[i], cnts[i]) for i in order[:k]]

    for field, k in (("msg", 50), ("u", 50), ("s", 1000), ("b", 50), ("i", 3)):
        got = field_stats(prov, field, k)
        assert got == old_field_stats(prov, field, k), field
    assert field_stats(prov, "msg", 50)[1] > 50_000
    assert field_stats(prov, "s", 10, [col("v") > 10 ** 6]) == old_field_stats(prov, "s", 10, [col("v") > 10 ** 6])
