"""GPU parity tests: every query goes through the C ABI (pq_query_open / pq_query_next) and is
compared with the CPU oracle on the same files.  Bit-exact for counts, row ids, integer aggregates,
MIN/MAX; 1e-9 relative for f64 SUM/AVG (BASELINE.json north_star: accumulation order differs)."""
import ctypes as C
import json
import math
import os

import numpy as np
import pyarrow as pa
import pyarrow.parquet as pq
import pytest

from oracle.oracle import Oracle
from parseable_b200 import _lib as L
from parseable_b200 import synth
from parseable_b200.query import (DeviceTable, HostFile, Query, QueryError, StandardTableProvider, TimeRange,
                                  Window, avg, col, count, count_star, execute, lit, max_, min_, sum_)

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(__file__), "golden")
F64_REL = 1e-9


def assert_tables_equal(got: pa.Table, exp: pa.Table, keys):
    assert got.num_rows == exp.num_rows
    assert got.column_names == exp.column_names
    if keys and got.num_rows:
        order = [(k, "ascending") for k in keys]
        got, exp = got.sort_by(order), exp.sort_by(order)
    for name in exp.column_names:
        a, b = got[name].to_pylist(), exp[name].to_pylist()
        f64_sum = pa.types.is_floating(exp[name].type) and (name.startswith("sum(") or name.startswith("avg("))
        if f64_sum:
            for x, y in zip(a, b):
                assert (x is None) == (y is None), name
                if x is not None:
                    assert math.isclose(x, y, rel_tol=F64_REL, abs_tol=0.0) or (math.isnan(x) and math.isnan(y)), (name, x, y)
        else:
            a = [None if (isinstance(v, float) and math.isnan(v)) else v for v in a]
            b = [None if (isinstance(v, float) and math.isnan(v)) else v for v in b]
            assert a == b, name


@pytest.fixture(scope="module")
def env(built, small_files):
    out = {}
    for tag, path in small_files.items():
        ora = Oracle.from_parquet(path)
        out[tag] = (path, ora, StandardTableProvider([path], schema=ora.table.schema))
    return out


FILTERS = {
    "c2_level_and_latency": [(col("level") == "ERROR") & (col("latency_ms") > 100)],
    "c1_status_eq": [col("status") == 200],
    "f64_vs_int_literal": [col("duration_s") >= 1],
    "i64_vs_fraction_gt": [col("latency_ms") > 100.5],               # the column is cast to Float64 (DataFusion): v > 100.5 <=> v > 100
    "i64_vs_fraction_le_ne": [(col("latency_ms") <= 99.5) & (col("bytes") != 7.5)],
    "i64_vs_fraction_eq_or": [(col("status") == 200.5) | (col("latency_ms") >= 1e19) | (col("bytes") < -0.5) | (col("status") > float("nan"))],   # all never true
    "i64_vs_nan_lt": [(col("status") < float("nan")) & (col("latency_ms") < 3.25)],
    "or_mixed": [(col("level") == "FATAL") | (col("bytes") < 1000)],
    "not": [~(col("level") == "INFO")],
    "not_or": [~((col("status") == 200) | (col("cpu") >= 0.25))],
    "plain_f64": [col("cpu") > 0.5],
    "plain_f64_and_dict": [(col("mem_gb") <= 32.0) & (col("method") != "GET")],
    "is_null": [col("host").is_null()],
    "is_not_null_and": [col("pod").is_not_null() & (col("region") == "region-03")],
    "like_contains": [col("message").like("%timeout-xyzzy%")],
    "like_prefix": [col("host").like("host-000%")],
    "like_suffix": [col("host").like("%7")],
    "like_underscore": [col("path").like("/api/v1/resource/00_1")],
    "not_like": [col("service").like("svc-00%", negated=True)],
    "ilike": [col("level").ilike("err%")],
    "str_range": [(col("host") >= "host-05000") & (col("host") < "host-05100")],
    "conjunction_list": [col("level") == "WARN", col("latency_ms") <= 20, col("score") < 0.0],
    "never": [col("level") == "NOPE"],
    "always": [],
    "deep": [((col("level") == "ERROR") | (col("level") == "FATAL")) & ((col("status") == 500) | (col("status") == 503))
             & ~(col("region") == "region-00") & (col("bytes") > 10)],
}


@pytest.mark.parametrize("tag", ["nn", "nulls"])
@pytest.mark.parametrize("name", sorted(FILTERS))
def test_filter_count(env, tag, name):
    path, ora, prov = env[tag]
    flt = FILTERS[name]
    got = prov.scan(filters=flt, count_only=True)
    assert got.metrics["rows_selected"] == ora.count(flt)
    assert got.metrics["rows_scanned"] + 70_000 * got.metrics["row_groups_pruned"] == ora.n


@pytest.mark.parametrize("tag", ["nn", "nulls"])
@pytest.mark.parametrize("name", ["c2_level_and_latency", "like_contains", "or_mixed", "never", "is_null"])
def test_filter_row_ids(env, tag, name):
    path, ora, prov = env[tag]
    flt = FILTERS[name]
    res = prov.scan(filters=flt)
    ids = np.concatenate([b.column(0).to_numpy() for b in res.batches]) if res.batches else np.array([], np.int64)
    assert np.array_equal(ids, ora.row_ids(flt))
    assert all(b.num_rows <= 20000 for b in res.batches)          # batch size of the reference scan


def test_limit(env):
    path, ora, prov = env["nn"]
    flt = FILTERS["or_mixed"]
    res = prov.scan(filters=flt, limit=37)
    ids = np.concatenate([b.column(0).to_numpy() for b in res.batches])
    assert np.array_equal(ids, ora.row_ids(flt)[:37])


AGGS = {
    "c3_host": (["host"], [count_star(), sum_("bytes")], []),
    "c4_host_status_6aggs": (["host", "status"], [count_star(), sum_("bytes"), min_("latency_ms"), max_("latency_ms"),
                                                  sum_("duration_s"), max_("cpu")], []),
    "level_avg_count": (["level"], [count_star(), avg("latency_ms"), count("cpu"), avg("score")], [col("status") == 200]),
    "global": ([], [count_star(), sum_("bytes"), min_("cpu"), max_("score"), avg("mem_gb")], [col("level") == "ERROR"]),
    "global_empty": ([], [count_star(), sum_("bytes"), min_("cpu")], [col("level") == "NOPE"]),
    "grouped_empty": (["region"], [count_star()], [col("level") == "NOPE"]),
    "count_star_only": ([], [count_star()], [col("status") == 404]),
    "three_keys": (["region", "method", "level"], [count_star(), max_("bytes")], [col("latency_ms") > 30]),
    "numeric_key": (["status"], [count_star(), min_("score"), max_("mem_gb")], []),
    "f64_key": (["duration_s"], [count_star()], [col("latency_ms") < 40]),
    "filtered_c3": (["host"], [count_star(), sum_("bytes")], [(col("level") == "ERROR") & (col("latency_ms") > 100)]),
    "ts_minmax": (["service"], [min_("latency_ms"), max_("latency_ms"), count("host")], []),
    # key space 10 000 x 1 000 x 5 000 (x NULL): wider than the dense table, the groups that occur are hashed
    "hashed_wide_keys": (["host", "path", "pod"], [count_star(), sum_("bytes"), min_("latency_ms"), max_("cpu"), sum_("duration_s"),
                                                    avg("score"), count("mem_gb")], [col("level") != "DEBUG"]),
    "hashed_four_keys": (["pod", "path", "service", "status"], [count_star(), max_("latency_ms")], []),
}


@pytest.mark.parametrize("tag", ["nn", "nulls"])
@pytest.mark.parametrize("name", sorted(AGGS))
def test_group_by(env, tag, name):
    path, ora, prov = env[tag]
    keys, aggs, flt = AGGS[name]
    got = prov.aggregate(keys, aggs, flt)
    exp = ora.group_by(keys, aggs, flt)
    assert_tables_equal(got.table() if got.batches else exp.slice(0, 0), exp, keys)


def test_golden_field_stats_through_gpu(built):
    """The reference's own known answers (src/storage/field_stats.rs:927-1327) through the GPU path."""
    exp = json.load(open(os.path.join(GOLD, "expected.json")))
    path = os.path.join(GOLD, "field_stats_10rows.parquet")
    schema = {"name": pa.string(), "score": pa.float64(), "active": pa.bool_(), "created_at": pa.timestamp("ms"),
              "single_value": pa.string(), "id": pa.int64()}
    prov = StandardTableProvider([path], schema=schema)

    def stats(field):
        t = prov.aggregate([field], [count_star()]).table()
        return dict(zip(t[field].to_pylist(), t["count(*)"].to_pylist())), t

    name, t = stats("name")
    assert t["count(*)"].type == pa.int64()
    assert sum(name.values()) == 10 and len(name) == 7
    assert name["Alice"] == 3 and name["Bob"] == 2 and name["Charlie"] == 1 and name[None] == 1
    score, _ = stats("score")
    assert len(score) == 9 and score[95.5] == 2 and sum(score.values()) == 10
    active, _ = stats("active")
    assert active == {True: 6, False: 3, None: 1}
    created, t = stats("created_at")
    assert len(created) == 9 and max(created.values()) == 2 and pa.types.is_timestamp(t["created_at"].type)
    single, _ = stats("single_value")
    assert single == {"constant": 10}

    prov = StandardTableProvider([os.path.join(GOLD, "field_stats_1000rows.parquet")], schema={"category": pa.string()})
    cat = prov.aggregate(["category"], [count_star()]).table()
    assert cat.num_rows == 10 and set(cat["count(*)"].to_pylist()) == {100}
    prov = StandardTableProvider([os.path.join(GOLD, "field_stats_empty.parquet")], schema={"name": pa.string()})
    assert prov.aggregate(["name"], [count_star()]).batches == []
    # nested (list) columns are outside the GPU path and say so instead of guessing
    prov = StandardTableProvider([path], schema={})
    with pytest.raises(QueryError) as ei:
        prov.aggregate(["int_list"], [count_star()])
    assert ei.value.code == L.PQ_ERR_UNSUPPORTED


def test_sql_front_and_time_range_elision(env):
    path, ora, prov = env["nn"]
    ts = ora.table["p_timestamp"].cast(pa.int64()).to_numpy()
    tr = TimeRange(int(ts.min()), int(ts.max()) + 1)                 # covers everything: elided by statistics
    q = Query("SELECT host, COUNT(*), SUM(bytes) FROM logs16 WHERE level = 'ERROR' AND latency_ms > 100 GROUP BY host", tr)
    got = execute(q, prov)
    exp = ora.group_by(["host"], [count_star(), sum_("bytes")], FILTERS["c2_level_and_latency"])
    assert_tables_equal(got.table(), exp, ["host"])
    q = Query("SELECT COUNT(*) FROM demo WHERE status=200", tr)
    got = execute(q, prov)
    assert got.table()["count(*)"].to_pylist() == [ora.count([col("status") == 200])]
    # a range that excludes every row group prunes them all
    q = Query("SELECT COUNT(*) FROM demo WHERE status=200", TimeRange(0, 1000))
    got = execute(q, prov)
    assert got.table()["count(*)"].to_pylist() == [0]
    assert got.metrics["row_groups_pruned"] == got.metrics["row_groups_total"] == 3


def test_resident_table_and_host_buffers(env):
    path, ora, _ = env["nulls"]
    cols = ["level", "latency_ms", "host", "bytes"]
    flt = FILTERS["c2_level_and_latency"]
    want = ora.count(flt)
    tbl = DeviceTable([path], cols)
    assert tbl.rows == ora.n and tbl.device_bytes > 0
    prov = StandardTableProvider(tbl, schema=ora.table.schema)
    for _ in range(3):
        assert prov.scan(filters=flt, count_only=True).metrics["rows_selected"] == want
    got = prov.aggregate(["host"], [count_star(), sum_("bytes")], flt)
    assert got.metrics["h2d_bytes"] < 1 << 20                      # the column chunks were already in HBM
    assert_tables_equal(got.table(), ora.group_by(["host"], [count_star(), sum_("bytes")], flt), ["host"])
    tbl.close()
    data = open(path, "rb").read()
    for pinned in (False, True):
        hf = HostFile(data=data, pinned=pinned)
        prov = StandardTableProvider([hf], schema=ora.table.schema)
        r = prov.scan(filters=flt, count_only=True)
        assert r.metrics["rows_selected"] == want
        assert r.metrics["h2d_bytes"] >= r.metrics["bytes_scanned"] > 0
        hf.close()


def test_multiple_files_missing_columns_and_shards(env, data_dir):
    """Several files (one per minute in Parseable), one of them written before a column existed:
    the missing column reads as NULL; shards partition the row groups."""
    p0, ora0, _ = env["nn"]
    p1 = os.path.join(data_dir, "older.parquet")
    cols = [c for c in synth.LOGS16_COLUMNS if c not in ("pod", "score")]
    synth.write_logs16(p1, n_row_groups=2, first_rg=7, rows_per_group=50_000, null_rate=0.01, columns=cols)
    ora = Oracle.from_parquet([p0, p1])
    schema = {f.name: f.type for f in ora0.table.schema}
    prov = StandardTableProvider([p0, p1], schema=schema)
    for flt in ([col("pod").is_null()], [col("pod") == "pod-0007-4e0f"], [(col("score") < 0.0) | (col("level") == "ERROR")]):
        assert prov.scan(filters=flt, count_only=True).metrics["rows_selected"] == ora.count(flt)
    keys, aggs = ["level"], [count_star(), count("score"), max_("score"), sum_("bytes")]
    assert_tables_equal(prov.aggregate(keys, aggs).table(), ora.group_by(keys, aggs), keys)
    flt = FILTERS["c2_level_and_latency"]
    ids = []
    total = 0
    for s in range(3):
        sp = StandardTableProvider([p0, p1], schema=schema, shard_index=s, shard_count=3)
        r = sp.scan(filters=flt)
        total += r.metrics["rows_scanned"]
        ids += [b.column(0).to_numpy() for b in r.batches]
    assert total == ora.n
    assert np.array_equal(np.sort(np.concatenate(ids)), ora.row_ids(flt))


def test_stream_and_poll_next_agree(env):
    """pq_query_stream (one Arrow C stream) and pq_query_next (batch by batch) hand out the same batches."""
    path, ora, prov = env["nn"]
    flt = FILTERS["c2_level_and_latency"]
    a = prov.scan(filters=flt, batch_size=500)
    b = prov.scan(filters=flt, batch_size=500, poll=True)
    assert len(a.batches) == len(b.batches) > 1
    for x, y in zip(a.batches, b.batches):
        assert x.equals(y)
    assert np.array_equal(np.concatenate([x.column(0).to_numpy() for x in a.batches]), ora.row_ids(flt))


def test_arrow_default_pages_and_v2(data_dir, built):
    """Files NOT written the Parseable way: pyarrow defaults (1 MiB pages, misaligned across columns),
    data page v2, required (non-nullable) columns, small dictionaries with long RLE runs."""
    rng = np.random.default_rng(5)
    n = 300_000
    t = pa.table({
        "k": pa.array(np.repeat(rng.integers(0, 50, n // 100), 100).astype(np.int64)),            # long RLE runs
        "v": pa.array(rng.integers(-10**12, 10**12, n).astype(np.int64)),                           # PLAIN
        "f": pa.array(rng.standard_normal(n)),
        "s": pa.array(rng.choice(["a", "bb", "ccc", "dddd"], n)),
        "b": pa.array(rng.random(n) < 0.3),
    })
    t = t.set_column(2, "f", pa.array(np.where(rng.random(n) < 0.1, None, t["f"].to_numpy()), pa.float64(), from_pandas=True))
    req = pa.schema([pa.field("k", pa.int64(), False), pa.field("v", pa.int64(), False), pa.field("f", pa.float64(), True),
                     pa.field("s", pa.string(), False), pa.field("b", pa.bool_(), True)])
    t = t.cast(req)
    # v2 pages keep their level bytes uncompressed in front of the (compressed) values
    for ver, kw in (("1.0", {}), ("2.0", {}), ("1.0", {"use_dictionary": ["k", "s"], "data_page_size": 64 << 10}),
                    ("2.0", {"compression": "LZ4"}), ("2.0", {"compression": "SNAPPY", "data_page_size": 64 << 10}),
                    ("2.0", {"compression": "ZSTD"}), ("1.0", {"compression": "ZSTD", "compression_level": 9, "data_page_size": 64 << 10}),
                    ("2.0", {"compression": "GZIP", "data_page_size": 256 << 10})):
        p = os.path.join(data_dir, f"arrow_default_{ver}_{len(kw)}_{kw.get('compression', 'NONE')}.parquet")
        kw = dict({"compression": "NONE"}, **kw)
        pq.write_table(t, p, data_page_version=ver, row_group_size=120_000, **kw)
        ora = Oracle.from_parquet(p)
        prov = StandardTableProvider([p], schema=ora.table.schema)
        for flt in ([col("k") == 7], [(col("v") > 0) & (col("s") == "ccc")], [col("f") < -1.0], [col("b") == True],  # noqa: E712
                    [~(col("b") == True) | col("f").is_null()]):                                                       # noqa: E712
            assert prov.scan(filters=flt, count_only=True).metrics["rows_selected"] == ora.count(flt), (ver, kw, flt)
        # with the default page size, one 120 000-row page per row group: a work item of 59 slabs over
        # long RLE runs; the row ids must come out exactly
        for flt in ([col("k") == 7], [(col("k") == 7) & (col("s") == "ccc")]):
            res = prov.scan(filters=flt)
            ids = np.concatenate([b.column(0).to_numpy() for b in res.batches]) if res.batches else np.array([], np.int64)
            assert np.array_equal(ids, ora.row_ids(flt)), (ver, kw, flt)
        keys, aggs = ["k"], [count_star(), sum_("v"), min_("f"), max_("f"), count("f")]
        assert_tables_equal(prov.aggregate(keys, aggs, [col("s") != "a"]).table(), ora.group_by(keys, aggs, [col("s") != "a"]), keys)
        keys, aggs = ["b", "s"], [count_star(), avg("f")]
        assert_tables_equal(prov.aggregate(keys, aggs).table(), ora.group_by(keys, aggs), keys)


def test_edge_values_total_order_and_wrapping(data_dir, built):
    nan = float("nan")
    t = pa.table({
        "g": pa.array(["a", "a", "a", "b", "b", None, None, "c"]),
        "x": pa.array([nan, 1.0, -0.0, 0.0, None, 5.0, nan, None]),
        "big": pa.array([2**62, 2**62, 2**62, -2**63, -1, 7, None, None]),
    })
    p = os.path.join(data_dir, "edge.parquet")
    pq.write_table(t, p, compression="NONE")
    ora = Oracle(t)
    prov = StandardTableProvider([p], schema=t.schema)
    for flt in ([col("x") == nan], [col("x") > 1e308], [col("x") < 0.0], [col("x") == 0.0], [col("x") >= -0.0],
                [col("big") < 0], [col("g").is_null() & col("x").is_not_null()]):
        assert prov.scan(filters=flt, count_only=True).metrics["rows_selected"] == ora.count(flt), flt
    keys, aggs = ["g"], [count_star(), sum_("big"), min_("x"), max_("x"), count("x"), sum_("x")]
    got = prov.aggregate(keys, aggs).table().sort_by("g")
    exp = ora.group_by(keys, aggs).sort_by("g")
    assert got["sum(big)"].to_pylist() == exp["sum(big)"].to_pylist()            # wrapping SUM(Int64)
    assert [str(v) for v in got["min(x)"].to_pylist()] == [str(v) for v in exp["min(x)"].to_pylist()]
    assert [str(v) for v in got["max(x)"].to_pylist()] == [str(v) for v in exp["max(x)"].to_pylist()]
    assert got["count(x)"].to_pylist() == exp["count(x)"].to_pylist()
    assert got["g"].to_pylist() == exp["g"].to_pylist()


def test_errors_are_codes_not_crashes(env, data_dir):
    path, ora, prov = env["nn"]
    with pytest.raises(QueryError) as ei:
        StandardTableProvider([os.path.join(data_dir, "missing.parquet")]).scan(filters=[col("a") == 1], count_only=True)
    assert ei.value.code == L.PQ_ERR_IO
    with pytest.raises(QueryError) as ei:
        prov.aggregate(["host"], [sum_("level")])
    assert ei.value.code == L.PQ_ERR_UNSUPPORTED
    with pytest.raises(QueryError) as ei:
        prov.scan(filters=[col("level") == 5], count_only=True)
    assert ei.value.code == L.PQ_ERR_INVALID_ARG
    gz = os.path.join(data_dir, "brotli.parquet")
    synth.write_logs16(gz, n_row_groups=1, rows_per_group=10_000, compression="BROTLI", columns=["level", "status"])
    with pytest.raises(QueryError) as ei:
        StandardTableProvider([gz], schema={"level": pa.string()}).scan(filters=[col("level") == "INFO"], count_only=True)
    assert ei.value.code == L.PQ_ERR_UNSUPPORTED and "codec" in ei.value.message


@pytest.mark.parametrize("codec", ["LZ4_RAW", "SNAPPY", "ZSTD", "GZIP"])
@pytest.mark.parametrize("null_rate", [0.0, 0.02])
def test_compressed_pages_decoded_on_gpu(data_dir, built, codec, null_rate):
    """Parseable's default codec is lz4_raw (src/cli.rs:441-448), its CI pins snappy
    (docker-compose-test.yaml:45), zstd and gzip are other legal P_PARQUET_COMPRESSION_ALGO values (src/option.rs:62-86):
    pages are decompressed on the GPU (one warp per page) into the arena, then the same scan runs."""
    p = os.path.join(data_dir, f"comp_{codec}_{int(null_rate * 100)}.parquet")
    synth.write_logs16(p, n_row_groups=2, rows_per_group=60_000, null_rate=null_rate, compression=codec)
    ora = Oracle.from_parquet(p)
    prov = StandardTableProvider([p], schema=ora.table.schema)
    for name in ("c2_level_and_latency", "plain_f64", "like_contains", "is_null", "deep", "c1_status_eq"):
        flt = FILTERS[name]
        got = prov.scan(filters=flt, count_only=True)
        assert got.metrics["rows_selected"] == ora.count(flt), (codec, name)
    assert got.metrics["bytes_scanned"] < got.metrics["algorithmic_bytes"]      # compressed bytes read < decoded bytes
    flt = FILTERS["c2_level_and_latency"]
    res = prov.scan(filters=flt)
    ids = np.concatenate([b.column(0).to_numpy() for b in res.batches]) if res.batches else np.array([], np.int64)
    assert np.array_equal(ids, ora.row_ids(flt))
    keys, aggs, f = AGGS["c4_host_status_6aggs"]
    assert_tables_equal(prov.aggregate(keys, aggs, f).table(), ora.group_by(keys, aggs, f), keys)
    ts = ora.table["p_timestamp"].cast(pa.int64()).drop_null().to_numpy()
    from parseable_b200.query import Timestamp
    rng = [col("p_timestamp") >= Timestamp(int(np.quantile(ts, 0.4))), col("p_timestamp") < Timestamp(int(np.quantile(ts, 0.9)))]
    assert prov.scan(filters=rng, count_only=True).metrics["rows_selected"] == ora.count(rng)


def test_concurrent_queries_from_threads(env):
    """The reference drives partitions and several queries concurrently from tokio workers
    (src/query/mod.rs:287, 317-334): the C ABI must be re-entrant."""
    import threading
    path, ora, prov = env["nulls"]
    names = ["c2_level_and_latency", "or_mixed", "like_contains", "plain_f64", "deep", "not_or"]
    want = {n: ora.count(FILTERS[n]) for n in names}
    errs = []

    def work(n):
        try:
            for _ in range(3):
                got = prov.scan(filters=FILTERS[n], count_only=True).metrics["rows_selected"]
                if got != want[n]:
                    errs.append((n, got, want[n]))
        except Exception as e:  # pragma: no cover
            errs.append((n, repr(e)))

    th = [threading.Thread(target=work, args=(n,)) for n in names]
    [t.start() for t in th]
    [t.join() for t in th]
    assert not errs


@pytest.mark.parametrize("tag", ["nn", "nulls"])
def test_delta_binary_packed_time_column(env, tag):
    """p_timestamp is DELTA_BINARY_PACKED in every Parseable file (streams.rs:587-590).  A time range that
    cuts THROUGH row groups cannot be decided by footer statistics: the column is decoded on the GPU
    (miniblock unpack + block-wide prefix scan)."""
    path, ora, prov = env[tag]
    ts = ora.table["p_timestamp"].cast(pa.int64()).drop_null().to_numpy()
    lo, hi = int(np.quantile(ts, 0.31)), int(np.quantile(ts, 0.78))
    from parseable_b200.query import Timestamp
    rng = [col("p_timestamp") >= Timestamp(lo), col("p_timestamp") < Timestamp(hi)]
    got = prov.scan(filters=rng, count_only=True)
    assert got.metrics["rows_selected"] == ora.count(rng)
    flt = rng + [col("level") == "ERROR"]
    res = prov.scan(filters=flt)
    ids = np.concatenate([b.column(0).to_numpy() for b in res.batches]) if res.batches else np.array([], np.int64)
    assert np.array_equal(ids, ora.row_ids(flt))
    keys, aggs = ["level"], [count_star(), min_("p_timestamp"), max_("p_timestamp"), count("p_timestamp")]
    assert_tables_equal(prov.aggregate(keys, aggs, rng).table(), ora.group_by(keys, aggs, rng), keys)
    q = Query("SELECT COUNT(*) FROM t WHERE status = 200", TimeRange(lo, hi))
    assert execute(q, prov).table()["count(*)"].to_pylist() == [ora.count(rng + [col("status") == 200])]
    # equality / inequality on the raw values as well
    probe = int(ts[len(ts) // 2])
    for f in ([col("p_timestamp") == Timestamp(probe)], [col("p_timestamp") != Timestamp(probe)], [col("p_timestamp") > Timestamp(probe)]):
        assert prov.scan(filters=f, count_only=True).metrics["rows_selected"] == ora.count(f)


# ---- TableProvider::scan(projection, filters, limit): values of the selected rows (stream_schema_provider.rs:526-659) ----
def _project_expect(ora, flt, cols, limit=None):
    ids = ora.row_ids(flt)
    if limit is not None:
        ids = ids[:limit]
    t = ora.table.take(pa.array(ids)).select(cols)
    # dictionary-typed Utf8 columns of the synthetic files compare as plain strings
    return pa.table([c.cast(pa.string()) if pa.types.is_dictionary(c.type) else c for c in t.columns], names=cols), ids


@pytest.mark.parametrize("name", ["c2_level_and_latency", "like_contains", "or_mixed", "never", "plain_f64"])
def test_projection_values(env, name):
    """Every column kind of logs16: Timestamp (DELTA_BINARY_PACKED), Int64 / Float64 (dictionary and PLAIN
    fallback pages inside one chunk), Utf8 dictionaries; rows, order and batch size as the reference's scan."""
    path, ora, prov = env["nn"]
    flt = FILTERS[name]
    cols = ["p_timestamp", "host", "message", "latency_ms", "cpu", "duration_s", "level", "status"]
    res = prov.scan(projection=cols, filters=flt)
    exp, ids = _project_expect(ora, flt, cols)
    got = res.table() if res.batches else pa.table({})
    assert [f.name for f in res.batches[0].schema] == cols
    assert got.num_rows == len(ids)
    assert all(b.num_rows <= 20000 for b in res.batches)
    for c in cols:
        assert got[c].to_pylist() == exp[c].to_pylist(), c
    # a second run of the same shape sizes its result from the first answer (one round trip less): same rows
    again = prov.scan(projection=cols, filters=flt)
    assert (again.table() if again.batches else pa.table({})).num_rows == len(ids)


def test_projection_limit_row_ids_and_small_batches(env):
    path, ora, prov = env["nn"]
    flt = FILTERS["or_mixed"]
    res = prov.scan(projection=["host", "bytes"], filters=flt, limit=1234, row_ids=True, batch_size=500)
    exp, ids = _project_expect(ora, flt, ["host", "bytes"], limit=1234)
    got = res.table()
    assert got.column_names == ["host", "bytes", "__row_id"]
    assert got["host"].to_pylist() == exp["host"].to_pylist() and got["bytes"].to_pylist() == exp["bytes"].to_pylist()
    assert np.array_equal(got["__row_id"].to_numpy(), ids)
    assert all(b.num_rows <= 500 for b in res.batches) and len(res.batches) == 3


def test_projection_bool_plain_and_time_range(data_dir, built):
    """Booleans (bit-packed PLAIN), PLAIN Int64 / Float64, a time range that cuts a row group (the DELTA pages
    are decoded to row-addressable values), SELECT * through the SQL front."""
    rng = np.random.default_rng(11)
    n = 150_000
    ts = (1_700_000_000_000 - np.cumsum(rng.integers(0, 3, n))).astype(np.int64)
    t = pa.table({
        "p_timestamp": pa.array(ts, pa.timestamp("ms")),
        "flag": pa.array(rng.random(n) < 0.4),
        "v": pa.array(rng.integers(-10**15, 10**15, n).astype(np.int64)),
        "x": pa.array(rng.standard_normal(n)),
        "s": pa.array(rng.choice(["alpha", "", "gamma-gamma-gamma", "δέλτα"], n)),
    })
    p = os.path.join(data_dir, "proj_bool.parquet")
    pq.write_table(t, p, compression="NONE", row_group_size=60_000, use_dictionary=["s"],
                   column_encoding={"p_timestamp": "DELTA_BINARY_PACKED"}, data_page_size=128 << 10)
    ora = Oracle(t)
    prov = StandardTableProvider([p], schema=t.schema)
    lo, hi = int(ts[100_000]), int(ts[20_000])
    q = Query("SELECT * FROM t WHERE flag = TRUE AND x > 0.5", TimeRange(lo, hi))
    res = execute(q, prov)
    from parseable_b200.query import Timestamp
    flt = [(col("flag") == True) & (col("x") > 0.5), col("p_timestamp") >= Timestamp(lo), col("p_timestamp") < Timestamp(hi)]  # noqa: E712
    exp, ids = _project_expect(ora, flt, t.column_names)
    got = res.table()
    assert got.num_rows == len(ids) > 0
    for c in t.column_names:
        assert got[c].to_pylist() == exp[c].to_pylist(), c


@pytest.mark.parametrize("name", ["c1_status_eq", "is_null", "or_mixed", "not_or"])
def test_projection_with_nulls(env, name):
    """2 % NULLs in every column: validity bitmaps and values of the selected rows equal the oracle's take()."""
    path, ora, prov = env["nulls"]
    flt = FILTERS[name]
    cols = ["p_timestamp", "host", "message", "latency_ms", "cpu", "duration_s", "level", "status"]
    res = prov.scan(projection=cols, filters=flt, row_ids=True)
    exp, ids = _project_expect(ora, flt, cols)
    got = res.table()
    assert got.num_rows == len(ids) > 0
    assert np.array_equal(got["__row_id"].to_numpy(), ids)
    for c in cols:
        assert got[c].to_pylist() == exp[c].to_pylist(), c
        assert got[c].null_count == exp[c].null_count, c


def test_projection_of_a_column_missing_from_one_file(data_dir, built):
    """Schema evolution: a column that only newer files have reads as NULL for the old ones (schema adapter
    behaviour of the reference's scan), in filters, group keys, aggregates and projections."""
    a = pa.table({"k": pa.array(["x", "y", "x", "z"] * 500), "v": pa.array(np.arange(2000, dtype=np.int64))})
    b = pa.table({"k": pa.array(["y", "z"] * 800), "v": pa.array(np.arange(1600, dtype=np.int64) * 3),
                  "extra": pa.array(np.where(np.arange(1600) % 5 == 0, None, np.arange(1600) * 0.5), pa.float64(), from_pandas=True)})
    pa_, pb_ = os.path.join(data_dir, "evo_a.parquet"), os.path.join(data_dir, "evo_b.parquet")
    pq.write_table(a, pa_, compression="NONE")
    pq.write_table(b, pb_, compression="NONE")
    full = pa.concat_tables([a.append_column("extra", pa.nulls(a.num_rows, pa.float64())), b])
    ora = Oracle(full)
    prov = StandardTableProvider([pa_, pb_], schema=full.schema)
    for flt in ([col("extra") > 100.0], [col("extra").is_null()], [~(col("extra") > 100.0) | (col("k") == "x")]):
        assert prov.scan(filters=flt, count_only=True).metrics["rows_selected"] == ora.count(flt), flt
    flt = [col("v") >= 1500]
    got = prov.scan(projection=["k", "extra", "v"], filters=flt).table()
    exp, ids = _project_expect(ora, flt, ["k", "extra", "v"])
    for c in ["k", "extra", "v"]:
        assert got[c].to_pylist() == exp[c].to_pylist(), c
    keys, aggs = ["k"], [count_star(), count("extra"), sum_("extra"), max_("extra")]
    assert_tables_equal(prov.aggregate(keys, aggs).table(), ora.group_by(keys, aggs, []), keys)


@pytest.mark.parametrize("variant", ["v1_none", "v2_lz4", "v1_snappy_small_pages"])
def test_delta_byte_array_pages(data_dir, built, variant):
    """Front-coded strings: DELTA_BYTE_ARRAY is the fallback encoding Parseable sets on custom-partition columns
    (streams.rs:614-619), DELTA_LENGTH_BYTE_ARRAY its prefix-less sibling.  The pages are rewritten as PLAIN BYTE_ARRAY
    pages on the device at table open; filters, projections and COUNTs then see the same strings as the oracle.
    Sorted values (long shared prefixes), random values (no prefixes), empty strings, NULLs, multi-byte characters."""
    rng = np.random.default_rng(31)
    n = 150_000
    part = np.array([f"tenant-{i // 37:05d}/zone-{i % 5}/δ{i % 3}" for i in range(n)], dtype=object)       # sorted: long shared prefixes
    part[rng.random(n) < 0.02] = None
    rnd = np.array(["".join(chr(97 + int(c)) for c in rng.integers(0, 26, int(k))) for k in rng.integers(0, 24, n)], dtype=object)   # incl. ""
    rnd[rng.random(n) < 0.05] = None
    t = pa.table({"id": pa.array(np.arange(n, dtype=np.int64)), "part": pa.array(part, pa.string()), "rnd": pa.array(rnd, pa.string()),
                  "dl": pa.array(rnd, pa.string()), "v": pa.array(rng.integers(0, 100, n).astype(np.int64))})
    kw = {"v1_none": dict(compression="NONE", data_page_version="1.0"),
          "v2_lz4": dict(compression="LZ4", data_page_version="2.0"),
          "v1_snappy_small_pages": dict(compression="SNAPPY", data_page_version="1.0", data_page_size=16 << 10)}[variant]
    p = os.path.join(data_dir, f"delta_byte_array_{variant}.parquet")
    pq.write_table(t, p, row_group_size=60_000, use_dictionary=["v"],
                   column_encoding={"part": "DELTA_BYTE_ARRAY", "rnd": "DELTA_BYTE_ARRAY", "dl": "DELTA_LENGTH_BYTE_ARRAY"}, **kw)
    md = pq.ParquetFile(p).metadata.row_group(0)
    encs = {md.column(i).path_in_schema: set(md.column(i).encodings) for i in range(5)}
    assert "DELTA_BYTE_ARRAY" in encs["part"] and "DELTA_LENGTH_BYTE_ARRAY" in encs["dl"], encs
    ora = Oracle(t)
    prov = StandardTableProvider([p], schema=t.schema)
    flts = {
        "eq": [col("part") == "tenant-00123/zone-4/δ1"],
        "range": [(col("part") >= "tenant-02000") & (col("part") < "tenant-02010")],
        "like_multibyte": [col("part").like("%/zone-3/δ0")],
        "rnd_prefix": [col("rnd").like("ab%")],
        "empty_string": [col("rnd") == ""],
        "dl_suffix_and_dict": [col("dl").like("%zz") & (col("v") < 50)],
        "is_null_or": [col("part").is_null() | (col("dl") == "q")],
        "not_like": [col("rnd").like("%a%", negated=True)],
    }
    for name, flt in flts.items():
        assert prov.scan(filters=flt, count_only=True).metrics["rows_selected"] == ora.count(flt), (variant, name)
    for name in ("range", "rnd_prefix", "is_null_or"):
        flt = flts[name]
        got = prov.scan(projection=["id", "part", "rnd", "dl"], filters=flt, row_ids=True).table()
        exp, ids = _project_expect(ora, flt, ["id", "part", "rnd", "dl"])
        assert len(ids) > 10 and np.array_equal(got["__row_id"].to_numpy(), ids), (variant, name)
        for c in ["id", "part", "rnd", "dl"]:
            assert got[c].to_pylist() == exp[c].to_pylist(), (variant, name, c)
    keys, aggs = ["v"], [count_star(), count("part"), count("dl")]
    assert_tables_equal(prov.aggregate(keys, aggs, flts["rnd_prefix"]).table(), ora.group_by(keys, aggs, flts["rnd_prefix"]), keys)


def test_corrupt_dictionary_index_is_refused(data_dir, built):
    """A dictionary index outside the dictionary: the reference's Parquet reader fails the file; so does the table
    open (every index of the flat store is checked once, on the device) -- never a read outside a LUT."""
    rng = np.random.default_rng(41)
    n = 50_000
    t = pa.table({"k": pa.array(np.array(["a", "b", "c", "d", "e"])[rng.integers(0, 5, n)]), "v": pa.array(np.arange(n, dtype=np.int64))})
    p = os.path.join(data_dir, "corrupt_index.parquet")
    pq.write_table(t, p, compression="NONE", use_dictionary=["k"], data_page_size=1 << 20)
    schema = pa.schema([pa.field("k", pa.string()), pa.field("v", pa.int64())])
    assert StandardTableProvider([p], schema=schema).scan(filters=[col("k") == "c"], count_only=True).metrics["rows_selected"] == int((np.array(t["k"].to_pylist()) == "c").sum())
    cm = pq.ParquetFile(p).metadata.row_group(0).column(0)
    raw = bytearray(open(p, "rb").read())
    mid = cm.data_page_offset + (cm.total_compressed_size - (cm.data_page_offset - (cm.dictionary_page_offset or cm.data_page_offset))) // 2
    raw[mid:mid + 3] = b"\xff\xff\xff"          # 3-bit indices of a 5-entry dictionary: eight 7s
    bad = os.path.join(data_dir, "corrupt_index_bad.parquet")
    open(bad, "wb").write(bytes(raw))
    with pytest.raises(QueryError) as e:
        StandardTableProvider([bad], schema=schema).scan(filters=[col("k") == "c"], count_only=True)
    assert e.value.code == L.PQ_ERR_CORRUPT and "dictionary" in str(e.value)
    # a later query on a good file still works (the context is not poisoned)
    assert StandardTableProvider([p], schema=schema).scan(filters=[col("v") < 10], count_only=True).metrics["rows_selected"] == 10


def test_garbled_pages_fail_cleanly(data_dir, built):
    """Bytes flipped inside dictionary and data pages (run headers, bit widths, definition levels, PLAIN values, LZ4
    and Snappy sequences, ZSTD / GZIP streams): every open either answers or returns an error code -- no fault, no hang, and the CUDA context serves the
    next query.  (What a reader must answer for garbled VALUES is undefined; that it survives is not.)"""
    rng = np.random.default_rng(53)
    n = 60_000
    t = pa.table({
        "k": pa.array(np.array(["a", "bb", "ccc", "dddd", "e"])[rng.integers(0, 5, n)]),
        "v": pa.array(rng.integers(0, 1 << 40, n).astype(np.int64)),
        "d": pa.array(np.where(rng.random(n) < 0.1, None, rng.integers(0, 300, n)), pa.int64(), from_pandas=True),
        "s": pa.array([f"msg-{i % 4000:05d}-{'x' * (i % 9)}" for i in range(n)]),
    })
    schema = t.schema
    good = {}
    for codec in ("NONE", "LZ4", "SNAPPY", "ZSTD", "GZIP"):
        p = os.path.join(data_dir, f"garble_{codec}.parquet")
        pq.write_table(t, p, compression=codec, use_dictionary=["k", "d"], data_page_size=32 << 10, row_group_size=30_000,
                       column_encoding={"s": "DELTA_BYTE_ARRAY"})
        good[codec] = p
    flt = [(col("k") == "ccc") & (col("d") > 10) & col("s").like("%-x%")]
    keys, aggs = ["k"], [count_star(), sum_("v"), max_("d")]
    want = Oracle(t).count(flt)
    outcomes = {"ok": 0, "error": 0}
    for codec, p in good.items():
        raw = open(p, "rb").read()
        md = pq.ParquetFile(p).metadata
        spans = [(md.row_group(g).column(c).dictionary_page_offset or md.row_group(g).column(c).data_page_offset,
                  md.row_group(g).column(c).total_compressed_size) for g in range(md.num_row_groups) for c in range(md.num_columns)]
        for trial in range(24):
            b = bytearray(raw)
            for _ in range(int(rng.integers(1, 4))):
                lo, ln = spans[int(rng.integers(0, len(spans)))]
                pos = lo + int(rng.integers(0, ln))
                b[pos] = int(rng.integers(0, 256)) if trial % 3 else (b[pos] ^ 0xFF)
            bad = os.path.join(data_dir, f"garbled_{codec}_{trial}.parquet")
            open(bad, "wb").write(bytes(b))
            try:
                prov = StandardTableProvider([bad], schema=schema)
                prov.scan(filters=flt, count_only=True)
                prov.aggregate(keys, aggs, [col("v") >= 0])
                prov.scan(projection=["s", "d"], filters=[col("k") == "e"], limit=50)
                outcomes["ok"] += 1
            except QueryError as e:
                assert e.code < 0
                outcomes["error"] += 1
            os.remove(bad)
            # the context still answers, exactly
            assert StandardTableProvider([p], schema=schema).scan(filters=flt, count_only=True).metrics["rows_selected"] == want, (codec, trial)
    assert outcomes["ok"] + outcomes["error"] == 24 * len(good) and outcomes["error"] > 0, outcomes


def test_staging_branch_and_field_stats(data_dir, built):
    """get_staging_execution_plan (stream_schema_provider.rs:242-298): in-RAM staging batches (reversed, as one Parquet
    image) and staging Parquet files (newest name first) join the scan; field statistics (field_stats.rs:298-330):
    GROUP BY + COUNT(*) on the GPU, total / distinct / top-k above it."""
    from parseable_b200.query import field_stats
    rng = np.random.default_rng(61)

    def mk(n, t0):
        return pa.table({"p_timestamp": pa.array((t0 - np.arange(n)).astype(np.int64), pa.timestamp("ms")),
                         "k": pa.array(np.array(["x", "y", "z", None], dtype=object)[rng.integers(0, 4, n)], pa.string()),
                         "v": pa.array(rng.integers(0, 1000, n).astype(np.int64))})
    old, s1, s2 = mk(5000, 1_700_000_000_000), mk(700, 1_700_000_300_000), mk(900, 1_700_000_400_000)
    ram = [mk(40, 1_700_000_500_000 + i * 1000).to_batches()[0] for i in range(5)]
    paths = {}
    for name, tab in (("old", old), ("stage-0001", s1), ("stage-0002", s2)):
        paths[name] = os.path.join(data_dir, f"{name}.parquet")
        pq.write_table(tab, paths[name], compression="NONE")
    prov = StandardTableProvider([paths["old"]], schema=old.schema, staging_batches=ram,
                                 staging_parquet=[paths["stage-0001"], paths["stage-0002"]])
    # the reference's plan order: reversed in-RAM batches, staging files newest name first, then the rest
    rev = pa.Table.from_batches([b.take(pa.array(range(b.num_rows - 1, -1, -1), pa.int64())) for b in reversed(ram)])
    full = pa.concat_tables([rev, s2, s1, old])
    ora = Oracle(full)
    flt = [(col("v") < 300) & col("k").is_not_null()]
    assert prov.scan(filters=flt, count_only=True).metrics["rows_selected"] == ora.count(flt)
    got = prov.scan(projection=["p_timestamp", "k", "v"], filters=flt, row_ids=True).table()
    exp, ids = _project_expect(ora, flt, ["p_timestamp", "k", "v"])
    assert np.array_equal(got["__row_id"].to_numpy(), ids)
    for c in ["p_timestamp", "k", "v"]:
        assert got[c].to_pylist() == exp[c].to_pylist(), c
    keys, aggs = ["k"], [count_star(), sum_("v")]
    assert_tables_equal(prov.aggregate(keys, aggs).table(), ora.group_by(keys, aggs, []), keys)
    # field statistics: the reference's own known answers (field_stats.rs:927-1066)
    gold = StandardTableProvider([os.path.join(GOLD, "field_stats_10rows.parquet")],
                                 schema={"name": pa.string(), "score": pa.float64(), "active": pa.bool_(), "created_at": pa.timestamp("ms"),
                                         "single_value": pa.string(), "id": pa.int64()})
    total, distinct, top = field_stats(gold, "name", 3)
    assert (total, distinct) == (10, 7) and top[0] == ("Alice", 3) and top[1] == ("Bob", 2) and len(top) == 3
    total, distinct, top = field_stats(gold, "single_value")
    assert (total, distinct, top) == (10, 1, [("constant", 10)])
    total, distinct, top = field_stats(gold, "active")
    assert (total, distinct) == (10, 3) and top[0] == (True, 6)
    # COUNT(DISTINCT ...) of the alerts (alert_enums.rs:216-223): distinct values are interned ids
    cd = prov.count_distinct(["k"], "v", [col("v") < 50]).sort_by([("k", "ascending")])
    import pyarrow.compute as pc
    ft = full.filter(pc.less(full["v"], 50))
    ref = ft.group_by(["k"]).aggregate([("v", "count_distinct")]).sort_by([("k", "ascending")])
    assert cd["k"].to_pylist() == ref["k"].to_pylist() and cd["count(distinct v)"].to_pylist() == ref["v_count_distinct"].to_pylist()
    assert prov.count_distinct([], "k").column(0).to_pylist() == [3]          # NULL does not count
    assert prov.count_distinct([], "k", [col("v") < 0]).column(0).to_pylist() == [0]
    total, distinct, top = field_stats(prov, "k", 2)
    cnt = {k: c for k, c in zip(*[x.to_pylist() for x in ora.group_by(["k"], [count_star()], []).columns])}
    assert total == full.num_rows and distinct == 4 and top[0][1] == max(cnt.values())


def test_plain_byte_array_pages(data_dir, built):
    """Dictionary-fallback strings (streams.rs:584-631: dictionary on, 1 MiB limit): a `message` column whose chunk
    flips from RLE_DICTIONARY to PLAIN BYTE_ARRAY pages mid-way, a column written PLAIN from the start, NULLs in both;
    LIKE / comparisons / IS NULL on the raw bytes, projection of the strings, COUNT over them."""
    rng = np.random.default_rng(23)
    n = 180_000
    words = np.array(["timeout", "retry", "upstream", "cache", "db", "panic", "ok", "queued", "δ-error", "reset"])
    uniq = np.array([f"req-{i:06d} " + " ".join(words[rng.integers(0, len(words), 4)]) for i in range(70_000)], dtype=object)
    msg = uniq[rng.integers(0, len(uniq), n)]                        # ~36-byte strings, 70 000 distinct: the dictionary passes 1 MiB
    msg[rng.random(n) < 0.03] = None
    tag = np.array([f"t{i % 977}-{'x' * (i % 7)}" for i in range(n)], dtype=object)
    tag[rng.random(n) < 0.01] = None
    t = pa.table({"id": pa.array(np.arange(n, dtype=np.int64)), "message": pa.array(msg, pa.string()), "tag": pa.array(tag, pa.string()),
                  "v": pa.array(rng.integers(0, 100, n).astype(np.int64))})
    p = os.path.join(data_dir, "plain_strings.parquet")
    pq.write_table(t, p, compression="NONE", row_group_size=90_000, use_dictionary=["message", "v"], dictionary_pagesize_limit=1 << 20,
                   data_page_size=256 << 10)
    encs = {c.path_in_schema: set(c.encodings) for rg in range(2) for c in [pq.ParquetFile(p).metadata.row_group(rg).column(i) for i in range(4)]}
    assert "PLAIN" in encs["message"] and "RLE_DICTIONARY" in encs["message"], encs      # the chunk really flips
    ora = Oracle(t)
    prov = StandardTableProvider([p], schema=t.schema)
    flts = {
        "like_contains": [col("message").like("%panic%")],
        "like_and_dict": [col("message").like("%timeout%") & (col("v") < 10)],
        "eq_plain_only": [col("tag") == "t5-xxxxx"],
        "range": [(col("tag") >= "t90") & (col("tag") < "t91")],
        "ilike_prefix": [col("message").ilike("REQ-0000%")],
        "not_like_or_null": [col("message").like("%ok%", negated=True) | col("tag").is_null()],
        "is_null": [col("message").is_null()],
        "multibyte": [col("message").like("%δ-error%δ-error%")],
    }
    for name, flt in flts.items():
        assert prov.scan(filters=flt, count_only=True).metrics["rows_selected"] == ora.count(flt), name
    flt = flts["like_and_dict"]
    got = prov.scan(projection=["id", "message", "tag"], filters=flt).table()
    exp, ids = _project_expect(ora, flt, ["id", "message", "tag"])
    assert len(ids) > 100
    for c in ["id", "message", "tag"]:
        assert got[c].to_pylist() == exp[c].to_pylist(), c
    keys, aggs = ["v"], [count_star(), count("message"), count("tag")]
    assert_tables_equal(prov.aggregate(keys, aggs, flts["like_contains"]).table(), ora.group_by(keys, aggs, flts["like_contains"]), keys)
    # GROUP BY on pages without a dictionary: the rows are interned next to the dictionary entries of the chunk that
    # flipped (one numbering for both page kinds), NULL is its own group
    for keys, aggs, flt in ((["message"], [count_star(), sum_("v"), count("tag")], []),
                            (["tag"], [count_star(), max_("id")], [col("v") < 50]),
                            (["tag", "v"], [count_star(), min_("id")], [col("message").like("%db%")]),
                            (["message", "tag"], [count_star()], [])):                     # 70 001 x 978 combinations: hashed
        assert_tables_equal(prov.aggregate(keys, aggs, flt).table(), ora.group_by(keys, aggs, flt), keys)
    with pytest.raises(QueryError) as e:       # the id pages stand in for the values: filtering the same column is refused, never mis-evaluated
        prov.aggregate(["message"], [count_star()], [col("message").like("%ok%")])
    assert e.value.code == L.PQ_ERR_UNSUPPORTED


def test_group_by_numeric_columns_without_dictionary(data_dir, built):
    """GROUP BY on PLAIN Int64 / Float64 pages and on the DELTA_BINARY_PACKED time column (no dictionary anywhere):
    every row is interned by value; field statistics run exactly such queries over every field
    (src/storage/field_stats.rs:298-330)."""
    rng = np.random.default_rng(31)
    n = 150_000
    ts = (1_700_000_000_000 - np.cumsum(rng.integers(0, 2, n))).astype(np.int64)          # long runs of equal stamps
    x = np.round(rng.standard_normal(n), 1) + 0.0                                          # ~80 distinct doubles (no -0.0: it would sort next to 0.0)
    v = rng.integers(-40, 40, n).astype(np.int64) * 10**12
    xs = pa.array(np.where(rng.random(n) < 0.05, None, x), pa.float64(), from_pandas=True)
    t = pa.table({"p_timestamp": pa.array(ts, pa.timestamp("ms")), "v": pa.array(v), "x": xs,
                  "s": pa.array(rng.choice(["a", "bb", "ccc"], n)), "w": pa.array(rng.integers(0, 1000, n).astype(np.int64))})
    p = os.path.join(data_dir, "plain_numeric_keys.parquet")
    pq.write_table(t, p, compression="NONE", row_group_size=60_000, use_dictionary=["s"],
                   column_encoding={"p_timestamp": "DELTA_BINARY_PACKED", "v": "PLAIN", "x": "PLAIN", "w": "PLAIN"}, data_page_size=128 << 10)
    ora = Oracle(t)
    prov = StandardTableProvider([p], schema=t.schema)
    for keys, aggs, flt in ((["v"], [count_star(), sum_("w"), min_("x")], []),
                            (["x"], [count_star(), max_("w")], [col("s") != "a"]),
                            (["p_timestamp"], [count_star(), sum_("w")], []),
                            (["s", "v"], [count_star(), avg("w"), min_("x")], [col("w") < 500]),   # (AVG of the symmetric x cancels to ~1e-17: no relative tolerance fits)
                            (["v", "w", "p_timestamp"], [count_star(), max_("x")], [])):    # 80 x 1000 x ~75 000 combinations: hashed
        assert_tables_equal(prov.aggregate(keys, aggs, flt).table(), ora.group_by(keys, aggs, flt), keys)


# ---- the counts / histogram API: GROUP BY DATE_BIN(width, p_timestamp, origin) (src/query/mod.rs:623-680) ----
@pytest.mark.parametrize("tag", ["nn", "nulls"])
def test_date_bin_counts(env, tag):
    from parseable_b200.query import date_bin
    path, ora, prov = env[tag]
    for width, extra, flt in (("1m", [], []), ("5m", ["level"], [col("status") == 200]), (7_000, ["status", "region"], [col("latency_ms") > 50])):
        keys = [date_bin(width)] + extra
        aggs = [count_star(), sum_("bytes"), max_("cpu")]
        got = prov.aggregate(keys, aggs, flt).table()
        exp = ora.group_by(keys, aggs, flt)
        assert got.column_names[0] == "date_bin(p_timestamp)" and pa.types.is_timestamp(got.schema.field(0).type)
        assert_tables_equal(got, exp, ["date_bin(p_timestamp)"] + extra)
    # a time range that cuts the table plus bins: what the UI histogram asks for
    ts = ora.table["p_timestamp"].drop_null().cast(pa.int64()).to_numpy()
    lo, hi = int(np.quantile(ts, 0.2)), int(np.quantile(ts, 0.7))
    from parseable_b200.query import Timestamp
    rng_f = [col("p_timestamp") >= Timestamp(lo), col("p_timestamp") < Timestamp(hi)]
    got = prov.aggregate([date_bin("1m")], [count_star()], rng_f).table()
    assert_tables_equal(got, ora.group_by([date_bin("1m")], [count_star()], rng_f), ["date_bin(p_timestamp)"])


# ---- JSON egress formatted on the device (pq_query_json; the reference: record_batches_to_json + QueryResponse::to_json,
#      src/utils/arrow/mod.rs:49-64, src/response.rs:31-58) ----
def _json_expect(table: pa.Table):
    """Rows the way arrow_json::ArrayWriter writes them: NULL values leave their key out, non-finite floats are null,
    Timestamp(ms) is chrono's NaiveDateTime text."""
    import datetime as dt
    cols = {n: table[n].to_pylist() for n in table.column_names}
    ts_cols = {n for n in table.column_names if pa.types.is_timestamp(table.schema.field(n).type)}
    raw_ts = {n: table[n].cast(pa.int64()).to_pylist() for n in ts_cols}
    rows = []
    for i in range(table.num_rows):
        r = {}
        for n in table.column_names:
            v = cols[n][i]
            if v is None:
                continue
            if n in ts_cols:
                ms = raw_ts[n][i]
                t = dt.datetime(1970, 1, 1) + dt.timedelta(milliseconds=ms)
                v = t.strftime("%Y-%m-%dT%H:%M:%S") + (f".{ms % 1000:03d}" if ms % 1000 else "")
            elif isinstance(v, float) and (math.isnan(v) or math.isinf(v)):
                v = None
            r[n] = v
        rows.append(r)
    return rows


@pytest.mark.gpu
def test_json_egress_on_device(data_dir, built):
    rng = np.random.default_rng(41)
    n = 50_000
    ts = (1_700_000_000_000 - np.cumsum(rng.integers(0, 3, n)) * 250).astype(np.int64)      # some stamps on whole seconds, some not
    x = rng.standard_normal(n) * 10.0 ** rng.integers(-8, 18, n)
    x[rng.random(n) < 0.01] = np.nan
    x[rng.random(n) < 0.005] = np.inf
    s = rng.choice(np.array(['plain', 'quote " \\ back', "tab\tnl\n", "δέλτα ✓ 😀", "", "ctl\x01\x1f", "a/b"], dtype=object), n)
    s[rng.random(n) < 0.05] = None
    t = pa.table({"p_timestamp": pa.array(ts, pa.timestamp("ms")),
                  "x": pa.array(np.where(rng.random(n) < 0.03, None, x), pa.float64(), from_pandas=False),
                  "v": pa.array(rng.integers(-2**62, 2**62, n).astype(np.int64)),
                  "flag": pa.array(np.where(rng.random(n) < 0.1, None, rng.random(n) < 0.5), pa.bool_()),
                  "s": pa.array(s, pa.string()), "k": pa.array(rng.integers(0, 7, n).astype(np.int64))})
    p = os.path.join(data_dir, "json_egress.parquet")
    pq.write_table(t, p, compression="NONE", row_group_size=20_000, use_dictionary=["s", "k"],
                   column_encoding={"p_timestamp": "DELTA_BINARY_PACKED", "x": "PLAIN", "v": "PLAIN"}, data_page_size=64 << 10)
    ora = Oracle(t)
    prov = StandardTableProvider([p], schema=t.schema)
    flt = [col("k") < 5]
    for mode in ("array", "lines"):
        res = prov.scan(projection=t.column_names, filters=flt, batch_size=7_000, json=mode)       # several batches, one text
        assert res.json_text[:1] == (b"[" if mode == "array" else b"{")
        got = res.to_json()
        exp = _json_expect(res.table())
        assert len(got) == len(exp) == ora.count(flt) > 30_000
        assert got == exp
    # floats print shortest round-trip: the text parses back to the very same doubles (checked above through ==), and no
    # longer than repr
    txt = prov.scan(projection=["x"], filters=[col("k") == 1], json="lines").json_text.decode()
    for line, v in zip(txt.splitlines()[:2000], [r for r in prov.scan(projection=["x"], filters=[col("k") == 1]).table()["x"].to_pylist()][:2000]):
        if v is not None and math.isfinite(v):
            assert len(line) <= len('{"x":' + repr(v) + "}") + 2, (line, v)
    # aggregate results (assembled on the device, formatted where they are), NULL group included; row ids; empty results
    keys, aggs = ["s", "flag"], [count_star(), sum_("v"), min_("x"), avg("k"), max_("v")]
    res = prov.aggregate(keys, aggs, [col("k") > 0], json="array")
    srt = lambda rows: sorted(rows, key=lambda r: json.dumps(r, sort_keys=True))   # noqa: E731
    assert srt(res.to_json()) == srt(_json_expect(res.table()))
    filled = res.to_json(with_fields=True, fill_null=True)
    assert filled["fields"] == res.table().column_names and all(set(r) == set(filled["fields"]) for r in filled["records"])
    res = prov.scan(filters=[col("k") == 6], json="lines")
    assert [r["__row_id"] for r in res.to_json()] == list(ora.row_ids([col("k") == 6]))
    assert prov.scan(projection=["v"], filters=[col("k") == 99], json="array").json_text == b"[]"
    assert prov.scan(projection=["v"], filters=[col("k") == 99], json="lines").json_text == b""
    res = prov.aggregate([], [count_star(), sum_("v")], [col("k") == 99], json="array")              # one host-built row: COUNT 0, SUM NULL
    assert res.to_json() == [{"count(*)": 0}]
    # results laid out on the host, as JSON and as Arrow (twice: the second run of a scan sizes its result from the first)
    none = [col("k") == 99]
    aggs = [count_star(), count("x"), sum_("v"), min_("s"), max_("flag"), avg("x")]
    res = prov.aggregate([], aggs, none, json="array")                                    # a global aggregate over zero rows
    assert res.to_json() == [{"count(*)": 0, "count(x)": 0}]
    assert res.table().to_pylist() == [{"count(*)": 0, "count(x)": 0, "sum(v)": None, "min(s)": None, "max(flag)": None, "avg(x)": None}]
    assert [f.type for f in res.table().schema] == [pa.int64(), pa.int64(), pa.int64(), pa.string(), pa.bool_(), pa.float64()]
    n1 = ora.count([col("k") == 1])
    for window, extra in ((None, {}), (Window(row_number=True, partition_rows=True), {"row_number": 1, "partition_rows": 1})):
        for mode in ("array", "lines"):
            res = prov.aggregate([], [count_star()], [col("k") == 1], json=mode, window=window)   # COUNT(*) alone
            assert res.to_json() == res.table().to_pylist() == [{"count(*)": n1, **extra}]
    for _ in range(2):
        res = prov.scan(projection=["v", "s", "flag", "p_timestamp"], filters=none, json="array")   # an empty projection
        assert res.json_text == b"[]" and len(res.batches) == 1
        assert res.table().num_rows == 0 and res.table().schema.types == [pa.int64(), pa.string(), pa.bool_(), pa.timestamp("ms")]
        res = prov.scan(filters=none, json="lines")                                                  # empty row ids
        assert res.json_text == b"" and len(res.batches) == 1
        assert res.table().num_rows == 0 and res.table().column_names == ["__row_id"]
