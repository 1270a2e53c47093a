"""Date32 columns (Parquet INT32 leaves with the DATE logical type) through the C ABI.

The flat store widens them to sign-extended 8-byte values when a table is opened; the results narrow them back to Arrow
Date32.  Every GPU case runs over a resident table and over a file list, against a numpy reference over the same rows
(days as int64):
  - page forms RLE_DICTIONARY, PLAIN, a dictionary that falls back to PLAIN mid-chunk and DELTA_BINARY_PACKED, in data
    page v1 and v2, without NULLs, with NULLs and with one all-NULL row group, several pages per chunk;
  - values before 1970, 0, +-(2^31 - 1) and years above 9999;
  - every comparison and IS [NOT] NULL (row ids exact), GROUP BY d alone and with a Utf8 key (dense and hashed), COUNT,
    COUNT(DISTINCT d), MIN / MAX(d), ORDER BY d / MIN(d) LIMIT under every PQB_ORDER_PATH, ROW_NUMBER by d, projections
    and JSON egress;
  - the codecs, a column missing from one file, pruning by footer statistics and the refusals.
CPU: the footer parse, the JSON date formatter through the host harness and the manifest pruning with a Date32 literal.
"""
import contextlib
import ctypes as C
import datetime as dt
import json
import os
import subprocess

import numpy as np
import pyarrow as pa
import pyarrow.parquet as pq
import pytest

from parseable_b200 import _lib as L
from parseable_b200.query import (DeviceTable, QueryError, StandardTableProvider, Timestamp, Window, avg, col, count,
                                  count_distinct, count_star, date_bin, max_, median, min_, percentile_cont, sum_)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EPOCH = dt.date(1970, 1, 1)
I32MAX = 2**31 - 1
Y10000 = (dt.date(9999, 12, 31) - EPOCH).days + 1          # 10000-01-01
EXTREMES = [-I32MAX, I32MAX, 0, -1, (dt.date(1, 1, 1) - EPOCH).days, Y10000 - 1, Y10000, Y10000 + 400_000, -800_000]
RG_ROWS = 6000
N_RG = 4


@contextlib.contextmanager
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


def make_data(nulls: str, seed=7):
    """(pyarrow table, days int64, valid bool).  nulls: 'none' | 'some' | 'rg' (some, and row group 1 all NULL)."""
    rng = np.random.default_rng(seed)
    n = RG_ROWS * N_RG
    pool = np.concatenate([rng.integers(-3000, 25_000, 300), np.array(EXTREMES)]).astype(np.int64)
    days = pool[rng.integers(0, len(pool), n)]
    days[rng.integers(0, n, 40)] = np.array(EXTREMES)[rng.integers(0, len(EXTREMES), 40)]
    valid = np.ones(n, bool)
    if nulls != "none":
        valid = rng.random(n) > 0.1
    if nulls == "rg":
        valid[RG_ROWS:2 * RG_ROWS] = False
    d = pa.array(days.astype(np.int32), pa.int32(), mask=~valid).cast(pa.date32())
    s = pa.array([f"s{int(x)}" for x in rng.integers(0, 7, n)])
    w = pa.array(rng.integers(0, 300_000, n).astype(np.int64))
    i = pa.array(np.arange(n, dtype=np.int64))
    t = pa.array(np.where(valid, days * 86_400_000, 0), pa.int64(), mask=~valid).cast(pa.timestamp("ms"))
    return pa.table({"d": d, "s": s, "w": w, "i": i, "t": t}), days, valid


FORMS = {
    "dict": dict(),
    "plain": dict(use_dictionary=["s", "w", "i", "t"]),
    "fallback": dict(dictionary_pagesize_limit=256),
    "delta": dict(use_dictionary=["s", "w", "i", "t"], column_encoding={"d": "DELTA_BINARY_PACKED"}),
}


def write(path, table, form, page_version, compression="none", **kw):
    args = dict(FORMS[form])
    args.update(kw)
    pq.write_table(table, path, row_group_size=RG_ROWS, data_page_size=4096, data_page_version=page_version,
                   compression=compression, **args)
    return path


SCHEMA = {"d": pa.date32(), "s": pa.string(), "w": pa.int64(), "i": pa.int64(), "t": pa.timestamp("ms")}
COLS = list(SCHEMA)


@pytest.fixture(scope="module")
def cases(tmp_path_factory):
    base = tmp_path_factory.mktemp("date32")
    out = {}
    for nulls in ("none", "some", "rg"):
        tbl, days, valid = make_data(nulls)
        for form in FORMS:
            for pv in ("1.0", "2.0"):
                p = write(str(base / f"{form}_{pv}_{nulls}.parquet"), tbl, form, pv)
                out[(form, pv, nulls)] = (p, days, valid)
    return out


CASE_IDS = [(f, v, n) for n in ("none", "some", "rg") for f in FORMS for v in ("1.0", "2.0")]


def providers(path):
    """(name, provider) over a resident table and over the file list."""
    yield "resident", StandardTableProvider(DeviceTable([path] if isinstance(path, str) else path, COLS), schema=SCHEMA)
    yield "files", StandardTableProvider([path] if isinstance(path, str) else list(path), schema=SCHEMA)


def row_ids(res):
    return np.concatenate([b.column(b.schema.get_field_index("__row_id")).to_numpy() for b in res.batches]) \
        if res.batches else np.array([], np.int64)


def days_of(arr):
    """Date32 array -> list of int days / None."""
    assert arr.type == pa.date32(), arr.type
    return arr.cast(pa.int32()).to_pylist()


CMP = {L.PQ_EQ: np.equal, L.PQ_NE: np.not_equal, L.PQ_LT: np.less, L.PQ_LE: np.less_equal, L.PQ_GT: np.greater,
       L.PQ_GE: np.greater_equal}
OPS = {L.PQ_EQ: "__eq__", L.PQ_NE: "__ne__", L.PQ_LT: "__lt__", L.PQ_LE: "__le__", L.PQ_GT: "__gt__", L.PQ_GE: "__ge__"}


class DateLit:
    """A Date32 literal of any int32 day count (datetime.date stops at year 9999)."""
    def __init__(self, days):
        self.days = days


def _cmp_expr(c, op, days):
    lit = EPOCH + dt.timedelta(days=days) if -719162 <= days <= 2932896 else None
    if lit is None:
        from parseable_b200.query import Expr
        e = Expr("cmp", (col(c), Expr("lit", (DateLit(days),))), op)
        return e
    return getattr(col(c), OPS[op])(lit)


@pytest.fixture(autouse=True)
def _date_lit_support(monkeypatch):
    """DateLit -> a PQ_T_DATE32 literal (days outside datetime.date's years)."""
    from parseable_b200 import query as Q
    orig = Q._Desc.literal

    def literal(self, v):
        if isinstance(v, DateLit):
            out = L.PqLiteral()
            out.type, out.i64 = L.PQ_T_DATE32, v.days
            return out
        return orig(self, v)
    monkeypatch.setattr(Q._Desc, "literal", literal)


# ------------------------------------------------------------------------------------------------------------- CPU
def test_footer_parse_finds_date_leaves(tmp_path):
    lib = L.load()
    tbl, days, valid = make_data("some")
    p = write(str(tmp_path / "f.parquet"), tbl, "dict", "1.0")
    f = L.PqFile(path=p.encode())
    n = lib.pq_file_describe(C.byref(f), None, 0)
    buf = C.create_string_buffer(n + 1)
    assert lib.pq_file_describe(C.byref(f), buf, n + 1) == n
    meta = json.loads(buf.value.decode())
    leaves = {lf["name"]: lf for lf in meta["leaves"]}
    assert leaves["d"]["is_date"] and leaves["d"]["phys_type"] == 1
    assert not any(leaves[c]["is_date"] for c in ("s", "w", "i", "t"))
    di = [lf["name"] for lf in meta["leaves"]].index("d")
    for g, rg in enumerate(meta["row_groups"]):
        c = rg["columns"][di]
        assert len(c["stats_min"]) == 8 and len(c["stats_max"]) == 8     # 4 bytes each
        sl = slice(g * RG_ROWS, (g + 1) * RG_ROWS)
        v = days[sl][valid[sl]]
        mn = int.from_bytes(bytes.fromhex(c["stats_min"]), "little", signed=True)
        mx = int.from_bytes(bytes.fromhex(c["stats_max"]), "little", signed=True)
        assert (mn, mx) == (int(v.min()), int(v.max()))


@pytest.fixture(scope="module")
def jh():
    so = os.path.join(ROOT, "tools", "libjson_host.so")
    if not os.path.exists(so):
        subprocess.check_call(["make", "-C", ROOT, "tools"])
    lib = C.CDLL(so)
    lib.jh_format_date32.argtypes = [C.c_int32, C.c_char_p]
    lib.jh_format_ts_ms.argtypes = [C.c_int64, C.c_char_p]
    return lib


def test_json_date_formatter(jh):
    buf = C.create_string_buffer(64)
    rng = np.random.default_rng(5)
    cases = EXTREMES + [-2**31, 59, 60, -719163, -719162, 2932896] + [int(x) for x in rng.integers(-2**31, 2**31, 4000)]
    for d in cases:
        n = jh.jh_format_date32(d, buf)
        got = buf.raw[:n].decode()
        if -719162 <= d <= 2932896:              # years 1..9999
            assert got == (EPOCH + dt.timedelta(days=d)).isoformat(), d
        m = jh.jh_format_ts_ms(d * 86_400_000, buf)
        assert got == buf.raw[:m].decode().split("T")[0], d


def test_plan_collect_files_with_date_literal():
    """pq_plan_collect_files takes a PQ_T_DATE32 literal as an Int against PQ_STAT_INT statistics (the expected answers
    restate satisfy_constraints: EQ lo <= v <= hi, LT v > lo, LE v >= lo, GT v < hi, GE v <= hi)."""
    lib = L.load()
    lo, hi = 18_000, 18_100
    st = L.PqColumnStat()
    st.column, st.kind, st.min_i, st.max_i = b"d", L.PQ_STAT_INT, lo, hi
    stats = (L.PqColumnStat * 1)(st)
    files = (L.PqManifestFile * 1)()
    files[0].path, files[0].num_rows, files[0].stats, files[0].n_stats = b"a", 10, stats, 1
    want = {L.PQ_EQ: lambda v: lo <= v <= hi, L.PQ_LT: lambda v: v > lo, L.PQ_LE: lambda v: v >= lo,
            L.PQ_GT: lambda v: v < hi, L.PQ_GE: lambda v: v <= hi}
    for v in (lo - 1, lo, lo + 50, hi, hi + 1):
        for op, keep in want.items():
            flt = (L.PqPlanFilter * 1)()
            flt[0].column, flt[0].cmp = b"d", op
            flt[0].lit.type, flt[0].lit.i64 = L.PQ_T_DATE32, v
            out = (C.c_uint32 * 1)()
            n = lib.pq_plan_collect_files(files, 1, flt, 1, -1, out)
            assert n == (1 if keep(v) else 0), (op, v)
    # a Date32 literal against Float / String statistics cannot tell: the file stays
    stats[0].kind = L.PQ_STAT_FLOAT
    flt = (L.PqPlanFilter * 1)()
    flt[0].column, flt[0].cmp = b"d", L.PQ_EQ
    flt[0].lit.type, flt[0].lit.i64 = L.PQ_T_DATE32, lo - 100
    assert lib.pq_plan_collect_files(files, 1, flt, 1, -1, (C.c_uint32 * 1)()) == 1
    from parseable_b200.planning import ManifestColumn, ManifestFileEntry, TypedStatistics, can_be_pruned
    f = ManifestFileEntry("a", 10, columns=[ManifestColumn("d", TypedStatistics("int", lo, hi))])
    assert can_be_pruned(f, col("d") < EPOCH + dt.timedelta(days=lo)) and not can_be_pruned(f, col("d") <= EPOCH + dt.timedelta(days=lo))


def test_sql_date_literal():
    from parseable_b200.query import Query
    q = Query("SELECT d FROM t WHERE d >= DATE '2020-01-02'")
    e = q.where
    assert e.kind == "cmp" and e.args[1].args[0] == dt.date(2020, 1, 2)
    for bad in ("2020-13-02", "20200102", "2020-W01-1", "2020-1-2"):
        with pytest.raises(QueryError):
            Query(f"SELECT d FROM t WHERE d >= DATE '{bad}'")


# ------------------------------------------------------------------------------------------------------------- GPU
def lits_for(days, valid):
    v = days[valid] if valid.any() else np.array([0])
    return sorted({int(v.min()) - 1, int(v.min()), int(np.median(v)), int(v.max()), int(v.max()) + (1 if v.max() < I32MAX else 0), 5_000})


@pytest.mark.gpu
@pytest.mark.parametrize("case", CASE_IDS, ids=["-".join(c) for c in CASE_IDS])
def test_filters(cases, case):
    path, days, valid = cases[case]
    for name, prov in providers(path):
        for lit in lits_for(days, valid):
            for op, fn in CMP.items():
                want = np.nonzero(valid & fn(days, lit))[0]
                res = prov.scan(filters=[_cmp_expr("d", op, lit)])
                assert res.metrics["rows_selected"] == len(want), (name, op, lit)
                assert np.array_equal(row_ids(res), want), (name, op, lit)
        for e, want in ((col("d").is_null(), ~valid), (col("d").is_not_null(), valid)):
            res = prov.scan(filters=[e])
            assert np.array_equal(row_ids(res), np.nonzero(want)[0]), name


@pytest.mark.gpu
@pytest.mark.parametrize("case", CASE_IDS, ids=["-".join(c) for c in CASE_IDS])
def test_group_by(cases, case, capfd):
    """GROUP BY d alone and with a Utf8 key, dense, hashed and (resident, dictionary pages) tuple pages.  MIN / MAX of a
    GROUP BY column whose pages lack a dictionary is refused for every numeric type (the key's pages then carry ids, not
    values), and so are MIN / MAX next to COUNT(DISTINCT) over such a column: MIN / MAX(d) run as a query of their own,
    grouped by d only over the dictionary form."""
    path, days, valid = cases[case]
    tbl = pq.read_table(path)
    s = tbl["s"].to_pylist()
    w = tbl["w"].to_numpy()
    dict_form = case[0] == "dict"
    counts = [count_star(), count("d"), count_distinct("d")]
    for name, prov in providers(path):
        for keys in (["d"], ["d", "s"], ["s", "d"], ["s"]):
            by = [(days[k] if valid[k] else None, s[k]) for k in range(len(days))]
            pick = [(0,), (0, 1), (1, 0), (1,)][[["d"], ["d", "s"], ["s", "d"], ["s"]].index(keys)]
            ref = {}
            for k, row in enumerate(by):
                key = tuple(None if row[j] is None else (int(row[j]) if j == 0 else row[j]) for j in pick)
                c = ref.setdefault(key, [0, 0, set()])
                c[0] += 1
                if valid[k]:
                    c[1] += 1
                    c[2].add(int(days[k]))

            def got_of(r):
                kcols = [days_of(r[k]) if k == "d" else r[k].to_pylist() for k in keys]
                return [tuple(kc[k] for kc in kcols) for k in range(r.num_rows)]
            r = prov.aggregate(keys, counts).table()
            if "d" in keys:
                assert r.schema.field("d").type == pa.date32()
            got = dict(zip(got_of(r), zip(r["count(*)"].to_pylist(), r["count(d)"].to_pylist(), r["count(distinct d)"].to_pylist())))
            assert got == {k: (a, b, len(st)) for k, (a, b, st) in ref.items()}, (name, keys)
            if "d" in keys and not dict_form:
                continue
            r = prov.aggregate(keys, [min_("d"), max_("d")]).table()
            assert r.schema.field("min(d)").type == pa.date32() and r.schema.field("max(d)").type == pa.date32()
            got = dict(zip(got_of(r), zip(days_of(r["min(d)"]), days_of(r["max(d)"]))))
            assert got == {k: (min(st) if st else None, max(st) if st else None) for k, (a, b, st) in ref.items()}, (name, keys)
        # hashed: (card(d) + 1) x (card(w) + 1) x (card(i) + 1) > 2^26 slots (i is the row number)
        with env_var("PQB_VERBOSE", "1"):
            capfd.readouterr()
            r = prov.aggregate(["d", "w", "i"], [count_star()] + ([max_("d")] if dict_form else [])).table()
            assert ",hashed" in capfd.readouterr().err, name
        dd = days_of(r["d"])
        ii = r["i"].to_pylist()
        assert sorted(ii) == list(range(len(days))), name
        for k in range(r.num_rows):
            row = ii[k]
            assert dd[k] == (int(days[row]) if valid[row] else None) and r["w"][k].as_py() == int(w[row]), (name, k)
            assert r["count(*)"][k].as_py() == 1
        if dict_form:
            assert days_of(r["max(d)"]) == dd, name
        # tuple pages: a resident table, two dictionary keys with no other role, COUNT(*) only
        if dict_form and name == "resident":
            with env_var("PQB_VERBOSE", "1"):
                capfd.readouterr()
                r = prov.aggregate(["d", "s"], [count_star()]).table()
                assert "group slots: tuple pages" in capfd.readouterr().err
            dd, ss = days_of(r["d"]), r["s"].to_pylist()
            ref = {}
            for k in range(len(days)):
                key = (int(days[k]) if valid[k] else None, s[k])
                ref[key] = ref.get(key, 0) + 1
            assert {(dd[k], ss[k]): r["count(*)"][k].as_py() for k in range(r.num_rows)} == ref
        # global MIN / MAX and COUNT(DISTINCT) (together only over dictionary pages, as for every numeric column)
        v = days[valid]
        g = prov.aggregate([], [min_("d"), max_("d")] + ([count_distinct("d")] if dict_form else [])).table()
        assert days_of(g["min(d)"]) == [int(v.min()) if len(v) else None]
        assert days_of(g["max(d)"]) == [int(v.max()) if len(v) else None]
        g = prov.aggregate([], [count_distinct("d")]).table()
        assert g["count(distinct d)"].to_pylist() == [len(set(v.tolist()))]


ORDER_PATHS = [None, "cta", "topk", "sort"]


def _ref_order(days, valid, desc, n):
    idx = np.arange(len(days))
    key = np.where(valid, days, 0)
    if desc:   # DESC: NULLs first, then descending, ties in row order
        order = sorted(idx, key=lambda k: (valid[k], -key[k], k))
    else:      # ASC: NULLs last
        order = sorted(idx, key=lambda k: (not valid[k], key[k], k))
    return np.array(order[:n], np.int64)


@pytest.mark.gpu
@pytest.mark.parametrize("case", [c for c in CASE_IDS if c[1] == "1.0"], ids=lambda c: "-".join(c))
def test_order_window_project_json(cases, case):
    path, days, valid = cases[case]
    svals = pq.read_table(path)["s"].to_pylist()
    for name, prov in providers(path):
        for path_env in ORDER_PATHS:
            with env_var("PQB_ORDER_PATH", path_env):
                for desc in (False, True):
                    for n in (1, 37, 5000):
                        res = prov.scan(projection=["d"], row_ids=True, order_by=[("d", "desc" if desc else "asc")], limit=n)
                        want = _ref_order(days, valid, desc, n)
                        assert np.array_equal(row_ids(res), want), (name, path_env, desc, n)
                        got = days_of(res.table()["d"])
                        assert got == [int(days[k]) if valid[k] else None for k in want]
                # ORDER BY MIN(d) over groups of s (a group with no date: NULL, last)
                r = prov.aggregate(["s"], [min_("d")], order_by=[("min(d)", "asc")], limit=4).table()
                per_s = {}
                for sv, dv, ok in zip(svals, days, valid):
                    per_s.setdefault(sv, None)
                    if ok:
                        per_s[sv] = int(dv) if per_s[sv] is None else min(per_s[sv], int(dv))
                allm = sorted(m for m in per_s.values() if m is not None) + [None] * sum(m is None for m in per_s.values())
                assert days_of(r["min(d)"]) == allm[:4], (name, path_env)
        # ROW_NUMBER() OVER (PARTITION BY d ORDER BY i) <= 1: the first row of every date
        res = prov.scan(projection=["d"], row_ids=True, order_by=[("i", "asc")],
                        window=Window(partition_by=["d"], fetch=1, row_number=True))
        first = {}
        for k in range(len(days)):
            first.setdefault(int(days[k]) if valid[k] else None, k)
        assert sorted(row_ids(res).tolist()) == sorted(first.values()), name
        assert set(res.table()["row_number"].to_pylist()) == {1}
        # projection with a filter on another column
        res = prov.scan(projection=["d", "s"], filters=[col("i") >= 100], row_ids=True)
        t = res.table()
        assert t.schema.field("d").type == pa.date32()
        ids = row_ids(res)
        assert np.array_equal(ids, np.arange(100, len(days)))
        assert days_of(t["d"]) == [int(days[k]) if valid[k] else None for k in ids]
        assert t["d"].null_count == int((~valid[100:]).sum())
        # JSON egress: the date part of the Timestamp(ms) text of d * 86400000, and isoformat() for years 1..9999
        res = prov.scan(projection=["d", "t"], json="lines")
        lines = [json.loads(x) for x in res.json_text.decode().splitlines() if x]
        assert len(lines) == len(days)
        for k, obj in enumerate(lines):
            if not valid[k]:
                assert "d" not in obj and "t" not in obj
                continue
            assert obj["d"] == obj["t"].split("T")[0], (k, obj)
            if -719162 <= days[k] <= 2932896:
                assert obj["d"] == (EPOCH + dt.timedelta(days=int(days[k]))).isoformat()


@pytest.mark.gpu
@pytest.mark.parametrize("codec", ["none", "lz4", "snappy", "zstd", "gzip"])
def test_codecs_and_missing_column(tmp_path, codec):
    tbl, days, valid = make_data("some", seed=11)
    p1 = write(str(tmp_path / "a.parquet"), tbl, "fallback", "2.0", compression=codec)
    p2 = write(str(tmp_path / "b.parquet"), tbl.drop_columns(["d"]), "dict", "1.0", compression=codec)
    all_days = np.concatenate([days, np.zeros_like(days)])
    all_valid = np.concatenate([valid, np.zeros_like(valid)])
    lit = int(np.median(days[valid]))
    for name, prov in providers([p1, p2]):
        res = prov.scan(filters=[_cmp_expr("d", L.PQ_GE, lit)])
        assert np.array_equal(row_ids(res), np.nonzero(all_valid & (all_days >= lit))[0]), name
        res = prov.scan(filters=[col("d").is_null()])
        assert np.array_equal(row_ids(res), np.nonzero(~all_valid)[0]), name
        r = prov.aggregate(["d"], [count_star()]).table()
        ref = {}
        for k in range(len(all_days)):
            key = int(all_days[k]) if all_valid[k] else None
            ref[key] = ref.get(key, 0) + 1
        dd = days_of(r["d"])
        assert {dd[k]: r["count(*)"][k].as_py() for k in range(r.num_rows)} == ref, name


@pytest.mark.gpu
def test_pruning_by_footer_statistics(tmp_path):
    n = RG_ROWS * N_RG
    days = (np.arange(n) // RG_ROWS * 1000 + np.arange(n) % 997).astype(np.int64)   # row group g: [1000 g, 1000 g + 996]
    tbl = pa.table({"d": pa.array(days.astype(np.int32)).cast(pa.date32()), "s": pa.array(["x"] * n), "w": pa.array(days),
                    "i": pa.array(np.arange(n)), "t": pa.array(days * 86_400_000).cast(pa.timestamp("ms"))})
    with_stats = write(str(tmp_path / "s.parquet"), tbl, "dict", "1.0")
    no_stats = write(str(tmp_path / "n.parquet"), tbl, "dict", "1.0", write_statistics=False)
    lo = EPOCH + dt.timedelta(days=2000)
    for op, fn in ((L.PQ_GE, np.greater_equal), (L.PQ_LT, np.less)):
        got = {}
        for tag, p in (("stats", with_stats), ("bare", no_stats)):
            for name, prov in providers(p):
                res = prov.scan(filters=[getattr(col("d"), OPS[op])(lo)])
                assert np.array_equal(row_ids(res), np.nonzero(fn(days, 2000))[0]), (tag, name)
                got[(tag, name)] = res.metrics["rows_scanned"]
        for name in ("resident", "files"):
            assert got[("stats", name)] == 2 * RG_ROWS and got[("bare", name)] == n, got


@pytest.mark.gpu
def test_refusals(tmp_path):
    tbl, days, valid = make_data("some", seed=3)
    p = write(str(tmp_path / "r.parquet"), tbl, "dict", "1.0")
    plain32 = str(tmp_path / "i32.parquet")
    pq.write_table(pa.table({"x": pa.array(np.arange(100, dtype=np.int32))}), plain32)
    ok_days = int(np.median(days[valid]))

    def answered(prov):
        res = prov.scan(filters=[_cmp_expr("d", L.PQ_LE, ok_days)], count_only=True)
        assert res.metrics["rows_selected"] == int((valid & (days <= ok_days)).sum())

    for name, prov in providers(p):
        refusals = [
            (L.PQ_ERR_UNSUPPORTED, lambda: prov.aggregate(["s"], [sum_("d")])),
            (L.PQ_ERR_UNSUPPORTED, lambda: prov.aggregate(["s"], [avg("d")])),
            (L.PQ_ERR_UNSUPPORTED, lambda: prov.aggregate(["s"], [median("d")])),
            (L.PQ_ERR_UNSUPPORTED, lambda: prov.aggregate(["s"], [percentile_cont("d", 0.5)])),
            (L.PQ_ERR_UNSUPPORTED, lambda: prov.aggregate([date_bin("1d", "d")], [count_star()])),
            (L.PQ_ERR_UNSUPPORTED, lambda: prov.scan(filters=[col("d") >= 5], count_only=True)),
            (L.PQ_ERR_UNSUPPORTED, lambda: prov.scan(filters=[col("d") >= Timestamp(5)], count_only=True)),
            (L.PQ_ERR_UNSUPPORTED, lambda: prov.scan(filters=[col("d") >= 5.0], count_only=True)),
            (L.PQ_ERR_UNSUPPORTED, lambda: prov.scan(filters=[col("d") == "2020-01-01"], count_only=True)),
            (L.PQ_ERR_UNSUPPORTED, lambda: prov.scan(filters=[col("i") >= dt.date(2020, 1, 1)], count_only=True)),
            (L.PQ_ERR_INVALID_ARG, lambda: prov.scan(filters=[col("d").like("2020%")], count_only=True)),
            (L.PQ_ERR_INVALID_ARG, lambda: prov.scan(filters=[_cmp_expr("d", L.PQ_EQ, 2**31)], count_only=True)),
        ]
        for code, q in refusals:
            with pytest.raises(QueryError) as ei:
                q()
            assert ei.value.code == code, (name, ei.value)
            answered(prov)
        with env_var("PQB_FLAT_SCAN", "0"):
            with pytest.raises(QueryError) as ei:
                prov.scan(filters=[_cmp_expr("d", L.PQ_LE, ok_days)], count_only=True)
            assert ei.value.code == L.PQ_ERR_UNSUPPORTED, name
        answered(prov)
    # a Date32 column declared Int64 or Timestamp(ms) in the plan
    for t in (pa.int64(), pa.timestamp("ms")):
        with pytest.raises(QueryError) as ei:
            StandardTableProvider([p], schema={**SCHEMA, "d": t}).scan(filters=[col("d") >= 5], count_only=True)
        assert ei.value.code == L.PQ_ERR_INVALID_ARG, t
    with pytest.raises(QueryError) as ei:
        DeviceTable([plain32], ["x"])
    assert ei.value.code == L.PQ_ERR_UNSUPPORTED and "physical type 1" in str(ei.value)
