"""Regular-expression filters (PQ_OP_REGEX: `~`, `~*`, `!~`, `!~*`, `regexp_like`) matched on the GPU by a DFA.

The reference is RE2 (pyarrow.compute.match_substring_regex), an engine independent of ours, wrapped into the C oracle's
Kleene logic by `RxOracle`.  RE2 takes \\d \\w as ASCII and its \\s lacks \\v, so the patterns here that use Perl classes
run over ASCII columns without \\v only; the Unicode meanings are checked on the CPU (test_regex_core.py)."""
import os

import numpy as np
import pyarrow as pa
import pyarrow.compute as pc
import pyarrow.parquet as pq
import pytest

from oracle.oracle import Oracle
from parseable_b200 import _lib as L
from parseable_b200 import synth
from parseable_b200.query import (DeviceTable, Query, QueryError, StandardTableProvider, avg, col, count, count_star,
                                  execute, lit, max_, min_, sum_)


class RxOracle(Oracle):
    """The C oracle plus a `regex` leaf evaluated by RE2: NULL input -> NULL, NOT / AND / OR in the oracle's Kleene logic."""

    def _eval(self, e):
        if e.kind != "regex":
            return super()._eval(e)
        name, pat = e.args[0].args[0], e.args[1].args[0]
        arr = self.table[name] if name in self.table.column_names else pa.nulls(self.n, pa.string())
        arr = arr.combine_chunks() if isinstance(arr, pa.ChunkedArray) else arr
        if pa.types.is_dictionary(arr.type):
            arr = arr.cast(arr.type.value_type)
        if pa.types.is_null(arr.type):
            arr = arr.cast(pa.string())
        if e.flags & L.PQ_REGEX_CASE_INSENSITIVE:
            pat = "(?i)" + pat
        m = pc.match_substring_regex(arr, pat)
        T = np.asarray(m.fill_null(False)).astype(np.uint8)
        N = np.asarray(m.is_null()).astype(np.uint8)
        if e.flags & L.PQ_REGEX_NEGATED:
            T = ((1 - T) & (1 - N)).astype(np.uint8)
        return np.ascontiguousarray(T), np.ascontiguousarray(N)


def ids_of(res) -> np.ndarray:
    return np.concatenate([b.column(0).to_numpy() for b in res.batches]) if res.batches else np.array([], np.int64)


def check_rows(prov, ora, flt):
    res = prov.scan(filters=flt)
    want = ora.row_ids(flt)
    got = ids_of(res)
    assert np.array_equal(np.sort(got), want), (len(got), len(want))
    assert prov.scan(filters=flt, count_only=True).metrics["rows_selected"] == len(want)
    return len(want)


LOG_PATTERNS = {
    "token": [col("message").regex(r"timeout-xy+zzy")],
    "anchored_path": [col("path").regex(r"^/api/v[12]/resource/00[0-4]\d$")],
    "host_class": [col("host").regex(r"^host-0[0-9]{3}7$")],
    "level_ci_alt": [col("level").regex(r"err|fatal", case_insensitive=True)],
    "negated": [col("level").regex(r"^(INFO|DEBUG)$", negated=True)],
    "negated_ci": [col("message").regex(r"RETRY|panic", negated=True, case_insensitive=True)],
    "and_cmp": [(col("level") == "ERROR") & col("message").regex(r"upstream (cache|db)")],
    "or_like": [col("message").regex(r"^\[000[0-7]\]") | col("path").like("%/0999")],
    "not_regex": [~col("host").regex(r"[13579]$") & (col("latency_ms") > 500)],
    "two_regex": [col("message").regex(r"session.*expired") & col("host").regex(r"-00\d\d\d$")],
    "like_same_col": [col("message").like("%retry%") & col("message").regex(r"retry (ok|queued)")],
    "empty_pattern": [col("pod").regex("")],
    "dot_star": [col("pod").regex(r"^pod-0.*-f")],
}


@pytest.fixture(scope="module")
def logs(built, small_files):
    out = {}
    for tag, path in small_files.items():
        ora = RxOracle.from_parquet(path)
        out[tag] = (ora, StandardTableProvider([path], schema=ora.table.schema), path)
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("tag", ["nn", "nulls"])
@pytest.mark.parametrize("name", sorted(LOG_PATTERNS))
def test_regex_logs_rows(logs, tag, name):
    ora, prov, _ = logs[tag]
    check_rows(prov, ora, LOG_PATTERNS[name])


@pytest.mark.gpu
def test_regex_logs_lz4_aggregates_order_projection(data_dir, built):
    """logs16 written LZ4_RAW with 2 % NULLs: counts, C4's aggregates, ORDER BY ... LIMIT and a projection under a regex."""
    path = os.path.join(data_dir, "rx_logs_lz4.parquet")
    synth.write_logs16(path, n_row_groups=3, rows_per_group=60_000, null_rate=0.02, compression="LZ4_RAW")
    ora = RxOracle.from_parquet(path)
    prov = StandardTableProvider([path], schema=ora.table.schema)
    flt = [col("message").regex(r"(?i)FAILED|panic") & col("host").regex(r"^host-0\d{3}[0-4]$")]
    n = check_rows(prov, ora, flt)
    assert 0 < n < ora.n
    aggs = [count_star(), sum_("bytes"), min_("latency_ms"), max_("latency_ms"), sum_("duration_s"), max_("cpu")]
    got = prov.aggregate(["status"], aggs, flt).table().sort_by("status")
    exp = ora.group_by(["status"], aggs, flt).sort_by("status")
    for name in exp.column_names:
        a, b = got[name].to_pylist(), exp[name].to_pylist()
        if name == "sum(duration_s)":
            assert np.allclose(np.array(a, float), np.array(b, float), rtol=1e-9), name
        else:
            assert a == b, name
    # ORDER BY p_timestamp DESC LIMIT 100 under the regex
    res = prov.scan(projection=["p_timestamp", "message"], filters=flt, order_by=[("p_timestamp", "desc")], limit=100)
    t = res.table()
    sel = ora.select(flt).astype(bool)
    ts = ora.table["p_timestamp"].cast(pa.int64())
    valid = np.asarray(ts.is_valid())
    vals = ts.fill_null(0).to_numpy(zero_copy_only=False)
    want = [None] * int((sel & ~valid).sum()) + np.sort(vals[sel & valid])[::-1].tolist()   # DESC: NULLS FIRST
    assert t["p_timestamp"].cast(pa.int64()).to_pylist() == want[:100]
    # a projection of the selected rows
    res = prov.scan(projection=["host", "message"], filters=flt)
    t = res.table()
    want = ora.table.filter(pa.array(sel)).select(["host", "message"])
    assert t["host"].cast(pa.string()).to_pylist() == want["host"].cast(pa.string()).to_pylist()
    assert t["message"].cast(pa.string()).to_pylist() == want["message"].cast(pa.string()).to_pylist()
    # the SQL front end, every operator
    for sql in ["SELECT COUNT(*) FROM s WHERE message ~ 'timeout-xy+zzy'",
                "SELECT COUNT(*) FROM s WHERE level ~* 'err|FATAL'",
                "SELECT COUNT(*) FROM s WHERE host !~ '[02468]$' AND level = 'WARN'",
                "SELECT COUNT(*) FROM s WHERE message !~* 'RETRY'",
                "SELECT COUNT(*) FROM s WHERE regexp_like(path, '^/API/v1/resource/01', 'i')",
                "SELECT COUNT(*) FROM s WHERE NOT regexp_like(host, '^host-0[0-9]{3}1$')"]:
        q = Query(sql)
        got = execute(q, prov).table().column(0).to_pylist()[0]
        assert got == ora.count([q.where]), sql


@pytest.mark.gpu
def test_regex_resident_table_kscan_noflat_and_shards(logs):
    ora, _, path = logs["nulls"]
    flt = [col("message").regex(r"(completed|failed) (user|session)") & (col("latency_ms") > 100)]
    dt = DeviceTable([path], ["message", "latency_ms", "level", "host"])
    try:
        prov = StandardTableProvider(dt, schema=ora.table.schema)
        for _ in range(2):
            check_rows(prov, ora, flt)
    finally:
        dt.close()
    prov = StandardTableProvider([path], schema=ora.table.schema)
    old = os.environ.get("PQB_FLAT_SCAN")
    os.environ["PQB_FLAT_SCAN"] = "0"   # every item on the k_scan path
    try:
        check_rows(prov, ora, flt)
        check_rows(prov, ora, [col("level").regex("^(WARN|ERROR)$") | col("host").regex("0$")])
    finally:
        if old is None:
            del os.environ["PQB_FLAT_SCAN"]
        else:
            os.environ["PQB_FLAT_SCAN"] = old
    # a NULL literal elsewhere in the predicate
    nf = [col("message").regex(r"retry") | lit(None)]
    check_rows(prov, ora, nf)
    got = prov.aggregate(["level"], [count_star()], nf).table().sort_by("level")
    exp = ora.group_by(["level"], [count_star()], nf).sort_by("level")
    assert got["count(*)"].to_pylist() == exp["count(*)"].to_pylist()
    # row-group shards 0/2 and 1/2 give the whole answer between them
    total = 0
    for shard in range(2):
        p = StandardTableProvider([path], schema=ora.table.schema, shard_index=shard, shard_count=2)
        total += p.scan(filters=flt, count_only=True).metrics["rows_selected"]
    assert total == ora.count(flt)


def _no_dict_table(rng, n):
    words = ["alpha", "beta", "gamma", "δέλτα", "Ε", "naïve", "日本語", "🙂", "x\ny", "", "K", "ſ", "timeout after 17 ms",
             "timeout after ms", "path/api/v2/", "/api/v1/x"]
    msg = np.array([" ".join(words[j] for j in rng.integers(0, len(words), int(rng.integers(0, 4)))) + f" #{i % 70_000:05d}"
                    for i in range(n)], dtype=object)
    msg[rng.random(n) < 0.03] = None
    msg[5] = ""
    msg[6] = "a\nb"
    msg[7] = "long " + "é" * 40_000 + " timeout after 99 ms"   # one value over 64 KiB
    dba = np.array([f"k{i % 911:04d}{'z' * (i % 5)}{'ä' if i % 7 == 0 else ''}" for i in range(n)], dtype=object)
    dba[rng.random(n) < 0.02] = None
    return pa.table({"v": pa.array(rng.integers(0, 50, n).astype(np.int64)), "message": pa.array(msg, pa.string()),
                     "dba": pa.array(dba, pa.string()), "dlba": pa.array(dba[::-1], pa.string())})


NO_DICT_PATTERNS = [
    [col("message").regex(r"timeout after [0-9]+ ms")],
    [col("message").regex(r"(?i)δέλτα|naÏve")],
    [col("message").regex(r"^$")],
    [col("message").regex(r"(?m)^y")],
    [col("message").regex(r"(?m)x$")],
    [col("message").regex(r"(?s)x.y")],
    [col("message").regex(r"日本.|🙂 #0001")],
    [col("message").regex(r"(?i)k|S", negated=True)],
    [col("dba").regex(r"z{3}ä?$") & (col("v") < 25)],
    [col("dlba").regex(r"^k0[0-4]\d\dz?$") | col("message").regex("beta gamma")],
    [~col("dba").regex(r"ä") & col("message").like("%alpha%")],
]


@pytest.fixture(scope="module")
def no_dict(data_dir, built):
    rng = np.random.default_rng(41)
    n = 150_000
    t = _no_dict_table(rng, n)
    p = os.path.join(data_dir, "rx_plain_strings.parquet")
    pq.write_table(t, p, compression="NONE", row_group_size=75_000, use_dictionary=["message", "v"], dictionary_pagesize_limit=1 << 20,
                   data_page_size=256 << 10, column_encoding={"dba": "DELTA_BYTE_ARRAY", "dlba": "DELTA_LENGTH_BYTE_ARRAY"})
    # a second file without the `dba` column: it reads as NULL there
    p2 = os.path.join(data_dir, "rx_plain_strings_2.parquet")
    pq.write_table(_no_dict_table(rng, 20_000).drop_columns(["dba"]), p2, compression="NONE", use_dictionary=["v"])
    return p, p2


@pytest.mark.gpu
@pytest.mark.parametrize("k", range(len(NO_DICT_PATTERNS)))
def test_regex_pages_without_dictionary(no_dict, k):
    p, p2 = no_dict
    from test_meta import describe
    pages = [[pg["encoding"] for pg in c["pages"]] for c in describe(L.load(), p)["row_groups"][0]["columns"]]
    assert 8 in pages[1] and 0 in pages[1][2:], pages[1]     # message: RLE_DICTIONARY pages, then the PLAIN fallback
    flt = NO_DICT_PATTERNS[k]
    for files in ([p], [p, p2]):
        ora = RxOracle.from_parquet(files)
        prov = StandardTableProvider(files, schema=ora.table.schema)
        check_rows(prov, ora, flt)
        # the aggregate kernel walks the DFA per row, with GROUP BY, in its own instantiations
        got = prov.aggregate(["v"], [count_star(), sum_("v"), count("message")], flt).table().sort_by("v")
        exp = ora.group_by(["v"], [count_star(), sum_("v"), count("message")], flt).sort_by("v")
        for name in exp.column_names:
            assert got[name].to_pylist() == exp[name].to_pylist(), (name, files)
        g = prov.aggregate([], [count_star(), min_("v"), max_("v"), avg("v")], flt).table()
        e = ora.group_by([], [count_star(), min_("v"), max_("v"), avg("v")], flt)
        assert g["count(*)"].to_pylist() == e["count(*)"].to_pylist()


@pytest.mark.gpu
def test_regex_refusals_leave_the_context_usable(logs):
    ora, prov, _ = logs["nulls"]
    good = [col("level").regex("^ERR")]
    want = ora.count(good)
    cases = [
        ([col("message").regex("(unclosed")], L.PQ_ERR_INVALID_ARG),
        ([col("message").regex(r"\bword\b")], L.PQ_ERR_UNSUPPORTED),
        ([col("latency_ms").regex("1")], L.PQ_ERR_INVALID_ARG),
        ([col("message").regex("(a|b)*a(a|b){20}")], L.PQ_ERR_UNSUPPORTED),
        ([col("message").regex(r"\p{Greek}")], L.PQ_ERR_UNSUPPORTED),
    ]
    for flt, code in cases:
        with pytest.raises(QueryError) as ei:
            prov.scan(filters=flt, count_only=True)
        assert ei.value.code == code, ei.value
        assert prov.scan(filters=good, count_only=True).metrics["rows_selected"] == want
    with pytest.raises(QueryError) as ei:
        prov.scan(filters=[col("message").regex("(a|b)*a(a|b){20}")], count_only=True)
    assert "too large for the device DFA" in str(ei.value)
