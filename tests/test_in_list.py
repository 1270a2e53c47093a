"""`col [NOT] IN (list)` (PQ_OP_IN) on the GPU, through the C ABI, over a resident table and a file list.

Every column kind and page form: Int64 dictionary / PLAIN / DELTA, Float64 dictionary / PLAIN, Utf8 dictionary /
dictionary-fallback PLAIN / DELTA_BYTE_ARRAY, Timestamp(ms), Date32 and Boolean, with NULLs, and a second file without the
PLAIN string column.  Lists of 1, 2, 16, 17, 1 000 and 100 000 elements with duplicates, IN and NOT IN, with and without
a NULL element, are checked against a numpy restatement of the Kleene OR of `col = e`; lists of at most 16 elements also
row for row against the same predicate written as an OR chain of PQ_EQ leaves, on the GPU and in the C oracle.  Then: IN
inside AND / OR / NOT trees, scans (row ids, COUNT_ONLY, a projection, ORDER BY ... LIMIT), aggregates (dense, hashed,
COUNT(DISTINCT), MEDIAN), forced small grids and stage counts, row-group pruning, and every refusal."""
import datetime as dt
import os
from contextlib import contextmanager
from functools import reduce

import numpy as np
import pyarrow as pa
import pyarrow.compute as pc
import pyarrow.parquet as pq
import pytest

from oracle.oracle import Oracle
from parseable_b200 import _lib as L
from parseable_b200.query import (DeviceTable, QueryError, StandardTableProvider, Timestamp, _Desc, col, count,
                                  count_distinct, count_star, median, sum_)

SEED = 20261019
RG_ROWS, N_RG = 40_000, 3
N1 = RG_ROWS * N_RG
N2 = 30_000
TOP = 9223372036854775808.0   # 2^63
COLS = ["i_dict", "i_plain", "i_delta", "f_dict", "f_plain", "s_dict", "s_plain", "s_dba", "ts", "d32", "b", "g", "k1",
        "k2", "x", "seq"]
F_VOCAB = [0.0, -0.0, 1.5, -2.25, np.inf, -np.inf, np.nan, 1e300, 3.0, 7.0]


def _table(rng, n, seq0):
    def nulls(a, rate=0.04):
        m = rng.random(n) < rate
        return pa.array(a, mask=m)
    s_vocab = np.array([f"host-{i:04d}" for i in range(300)] + ["", "é", "日本", "a\0b"], dtype=object)
    trace = np.array([f"{int(v):016x}" for v in rng.integers(0, 1 << 62, n)], dtype=object)
    trace[::97] = ""
    trace[5::97] = "ß" * 3000      # longer than 4 KiB in UTF-8
    i_plain = rng.integers(-(1 << 63), (1 << 63) - 1, n, dtype=np.int64, endpoint=True)
    i_plain[::50] = rng.integers(-500, 500, len(i_plain[::50]))
    i_plain[7::1000] = (1 << 63) - 1
    i_plain[9::1000] = (1 << 63) - 300
    i_plain[11::1000] = -(1 << 63)
    days = rng.integers(-800, 20_000, n).astype(np.int32)
    return pa.table({
        "i_dict": nulls(rng.integers(0, 1000, n).astype(np.int64)),
        "i_plain": nulls(i_plain),
        "i_delta": nulls(np.cumsum(rng.integers(0, 5, n)).astype(np.int64)),
        "f_dict": nulls(np.array(F_VOCAB)[rng.integers(0, len(F_VOCAB), n)]),
        "f_plain": nulls(np.round(rng.normal(0, 100, n), 1)),
        "s_dict": nulls(s_vocab[rng.integers(0, len(s_vocab), n)]),
        "s_plain": nulls(trace),
        "s_dba": nulls(np.array([f"k{i % 911:04d}{'z' * (i % 5)}" for i in range(n)], dtype=object)),
        "ts": nulls(pa.array(1_700_000_000_000 + rng.integers(0, 5000, n) * 1000, pa.timestamp("ms")).to_numpy(False)),
        "d32": nulls(pa.array(days, pa.date32()).to_numpy(False)),
        "b": nulls(rng.random(n) < 0.3),
        "g": pa.array(rng.integers(0, 20, n).astype(np.int64)),
        "k1": pa.array(rng.integers(0, 40_000, n).astype(np.int64)),
        "k2": pa.array(rng.integers(0, 40_000, n).astype(np.int64)),
        "x": pa.array(rng.normal(0, 1, n)),
        "seq": pa.array(np.arange(seq0, seq0 + n, dtype=np.int64)),
    })


@pytest.fixture(scope="module")
def data(data_dir, built):
    rng = np.random.default_rng(SEED)
    t1 = _table(rng, N1, 0)
    t1 = t1.set_column(t1.schema.get_field_index("ts"), "ts", t1["ts"].cast(pa.timestamp("ms")))
    t1 = t1.set_column(t1.schema.get_field_index("d32"), "d32", t1["d32"].cast(pa.date32()))
    p1 = os.path.join(data_dir, "in_list_1.parquet")
    pq.write_table(t1, p1, row_group_size=RG_ROWS, compression="NONE", data_page_size=64 << 10,
                   use_dictionary=["i_dict", "f_dict", "s_dict", "s_plain", "ts", "d32", "g", "k1", "k2"],
                   dictionary_pagesize_limit=256 << 10,
                   column_encoding={"i_plain": "PLAIN", "f_plain": "PLAIN", "i_delta": "DELTA_BINARY_PACKED",
                                    "s_dba": "DELTA_BYTE_ARRAY", "b": "PLAIN", "x": "PLAIN", "seq": "PLAIN"})
    t2 = _table(rng, N2, N1).drop_columns(["s_plain"])
    t2 = t2.set_column(t2.schema.get_field_index("ts"), "ts", t2["ts"].cast(pa.timestamp("ms")))
    t2 = t2.set_column(t2.schema.get_field_index("d32"), "d32", t2["d32"].cast(pa.date32()))
    p2 = os.path.join(data_dir, "in_list_2.parquet")
    pq.write_table(t2, p2, compression="NONE")
    table = pa.concat_tables([t1, t2], promote_options="default")
    return [p1, p2], table


@pytest.fixture(scope="module")
def provs(data):
    files, table = data
    dtab = DeviceTable(files, COLS)
    yield {"resident": StandardTableProvider(dtab, schema=table.schema),
           "files": StandardTableProvider(files, schema=table.schema)}, table
    dtab.close()


@contextmanager
def env(**kw):
    old = {k: os.environ.get(k) for k in kw}
    os.environ.update({k: str(v) for k, v in kw.items()})
    try:
        yield
    finally:
        for k, v in old.items():
            if v is None:
                del os.environ[k]
            else:
                os.environ[k] = v


# ---- the reference: the Kleene OR of `col = e` -------------------------------------------------------------------------
def _valid(a):
    return np.asarray(a.is_valid()) if a.null_count else np.ones(len(a), bool)


def member(a: pa.ChunkedArray, values) -> np.ndarray:
    """Rows (non-NULL or not) whose value some element equals, as PQ_OP_CMP / PQ_EQ coerces the element."""
    a = a.combine_chunks()
    vals = [v for v in values if v is not None]
    t = a.type
    if pa.types.is_string(t):
        return np.asarray(pc.is_in(a, value_set=pa.array(vals, pa.string())).fill_null(False))
    if pa.types.is_boolean(t):
        return np.asarray(pc.is_in(a, value_set=pa.array(vals, pa.bool_())).fill_null(False))
    if pa.types.is_floating(t):
        bits = a.fill_null(0.0).to_numpy(zero_copy_only=False).view(np.int64)
        els = np.array([float(v) for v in vals], np.float64).view(np.int64)
        return np.isin(bits, els)
    if pa.types.is_date32(t):
        v = a.cast(pa.int32()).fill_null(0).to_numpy(zero_copy_only=False).astype(np.int64)
        return np.isin(v, np.array([(d - dt.date(1970, 1, 1)).days for d in vals], np.int64))
    v = a.cast(pa.int64()).fill_null(0).to_numpy(zero_copy_only=False)
    ints = [x.ms if isinstance(x, Timestamp) else x for x in vals
            if not isinstance(x, float) or (x == x and float(x).is_integer() and -TOP <= x < TOP)]
    m = np.isin(v, np.array([int(x) for x in ints], np.int64))
    if any(isinstance(x, float) and x == TOP for x in vals):
        m |= v >= (1 << 63) - 511       # the int64 values that round to 2^63 as doubles
    return m


def expected(table, name, values, negated):
    a = table[name] if name in table.column_names else pa.chunked_array([pa.nulls(table.num_rows, pa.int64())])
    valid = _valid(a.combine_chunks())
    m = member(a, values) & valid
    has_null = any(v is None for v in values)
    t = m if not negated else (valid & ~m & (not has_null))
    return t


# ---- the lists ----------------------------------------------------------------------------------------------------------
def domain(table, name, rng, k):
    """k elements for column `name`: about half drawn from the column (duplicates included), the rest not in it."""
    a = table[name].combine_chunks().drop_null()
    present = a.to_pylist()
    kind = a.type
    half = [present[int(i)] for i in rng.integers(0, len(present), max(1, k - k // 2))]
    if pa.types.is_string(kind):
        other = [f"absent-{int(i)}" for i in rng.integers(0, 1 << 40, k // 2)]
    elif pa.types.is_floating(kind):
        other = [float(v) for v in rng.normal(0, 1e6, k // 2)]
    elif pa.types.is_timestamp(kind):
        ms = a.cast(pa.int64()).to_pylist()
        half = [Timestamp(ms[int(i)]) for i in rng.integers(0, len(ms), len(half))]
        other = [Timestamp(int(v)) for v in rng.integers(0, 1 << 40, k // 2)]
    elif pa.types.is_date32(kind):
        other = [dt.date(1970, 1, 1) + dt.timedelta(days=int(v)) for v in rng.integers(30_000, 60_000, k // 2)]
    else:
        other = [int(v) for v in rng.integers(-(1 << 62), 1 << 62, k // 2)]
    out = half + other
    if k >= 2:
        out[-1] = out[0]      # a duplicate
    return out[:k]


KINDS = ["i_dict", "i_plain", "i_delta", "f_dict", "f_plain", "s_dict", "s_plain", "s_dba", "ts", "d32"]
SIZES = [1, 2, 16, 17, 1000, 100_000]


def ids_of(res):
    return np.concatenate([b.column(0).to_numpy() for b in res.batches]) if res.batches else np.array([], np.int64)


def check_scan(prov, table, flt, want_mask):
    want = np.flatnonzero(want_mask)
    got = ids_of(prov.scan(filters=flt))
    assert np.array_equal(np.sort(got), want), (len(got), len(want))
    assert prov.scan(filters=flt, count_only=True).metrics["rows_selected"] == len(want)
    return want


def or_chain(name, values, negated):
    vals = [v for v in values if v is not None]
    e = reduce(lambda a, b: a | b, [col(name) == v for v in vals])
    if any(v is None for v in values):
        e = e | (col(name) == None)   # noqa: E711  (`col = NULL`: NULL on every row)
    return ~e if negated else e


@pytest.mark.gpu
@pytest.mark.parametrize("name", KINDS)
@pytest.mark.parametrize("k", SIZES)
def test_in_every_kind_and_size(provs, name, k):
    pv, table = provs
    rng = np.random.default_rng(hash((name, k)) % (1 << 32))
    base = domain(table, name, rng, k)
    for negated in (False, True):
        for has_null in (False, True):
            values = base + [None] if has_null else base
            flt = [col(name).isin(values, negated=negated)]
            want = expected(table, name, values, negated)
            for prov in pv.values():
                ids = check_scan(prov, table, flt, want)
            if k <= 16:
                # the same predicate as an OR chain of PQ_EQ leaves: bit for bit on the GPU, and in the C oracle
                chain = [or_chain(name, values, negated)]
                assert np.array_equal(np.sort(ids_of(pv["resident"].scan(filters=chain))), ids)
                if name not in ("d32",):
                    ora = Oracle(table.select([name]) if name in table.column_names else table)
                    assert np.array_equal(ora.row_ids(chain), ids)


@pytest.mark.gpu
def test_boolean_lists(provs):
    pv, table = provs
    for values in ([True], [False], [True, False, True], [None], [False, None], [True, False, None]):
        for negated in (False, True):
            flt = [col("b").isin(values, negated=negated)]
            check_scan(pv["resident"], table, flt, expected(table, "b", values, negated))


@pytest.mark.gpu
def test_int64_with_float_elements(provs):
    pv, table = provs
    for name in ("i_dict", "i_plain", "i_delta"):
        for values in ([1.5, 2.0, -3.0, 7.25], [TOP], [TOP, 3.0, 17.0, 0.5], [TOP, 0.5, None], [0.5, float("nan")],
                       [-TOP, 5.0], [float("inf"), 12.0, 13.0]):
            for negated in (False, True):
                flt = [col(name).isin(values, negated=negated)]
                want = expected(table, name, values, negated)
                ids = check_scan(pv["resident"], table, flt, want)
                chain = [or_chain(name, values, negated)]
                assert np.array_equal(np.sort(ids_of(pv["resident"].scan(filters=chain))), ids)


@pytest.mark.gpu
def test_in_inside_trees_and_missing_column(provs):
    pv, table = provs
    rng = np.random.default_rng(3)
    hosts = domain(table, "s_dict", rng, 40)
    traces = domain(table, "s_plain", rng, 300) + [None]
    n = table.num_rows
    m_h = expected(table, "s_dict", hosts, False)
    x = table["i_dict"].combine_chunks()
    lt = np.asarray(pc.less(x, 500).fill_null(False))
    lt_null = ~_valid(x)
    t_tr = expected(table, "s_plain", traces, False)
    # s_plain IN (...) is NULL where s_plain is NULL (the second file too) or misses with the NULL element
    valid_tr = _valid(table["s_plain"].combine_chunks())
    n_tr = ~valid_tr | (valid_tr & ~t_tr)
    cases = [
        ([col("s_dict").isin(hosts) & (col("i_dict") < 500)], m_h & lt),
        ([col("s_dict").isin(hosts) | col("s_plain").isin(traces)], m_h | t_tr),
        ([~(col("s_plain").isin(traces) & (col("i_dict") < 500))],
         # NOT (a AND b): TRUE where a or b is FALSE
         (valid_tr & ~t_tr & ~n_tr) | (~lt & ~lt_null)),
        ([col("s_plain").isin(traces, negated=True) | col("s_dict").isin(hosts, negated=True)],
         np.zeros(n, bool) | expected(table, "s_dict", hosts, True)),
    ]
    for flt, want in cases:
        for prov in pv.values():
            check_scan(prov, table, flt, want)


@pytest.mark.gpu
def test_scan_shapes(provs):
    pv, table = provs
    rng = np.random.default_rng(5)
    a, b = domain(table, "s_plain", rng, 1000), domain(table, "i_plain", rng, 17)
    flt = [col("s_plain").isin(a) | col("i_plain").isin(b)]
    want = expected(table, "s_plain", a, False) | expected(table, "i_plain", b, False)
    for prov in pv.values():
        ids = check_scan(prov, table, flt, want)
        res = prov.scan(projection=["seq", "s_plain"], filters=flt)
        got = pa.Table.from_batches(res.batches) if res.batches else None
        assert got is not None and np.array_equal(np.sort(got["seq"].to_numpy()), np.sort(table["seq"].to_numpy()[ids]))
        top = prov.scan(projection=["seq"], filters=flt, order_by=[("seq", "desc")], limit=25)
        got_top = pa.Table.from_batches(top.batches)["seq"].to_pylist()
        assert got_top == sorted(table["seq"].to_numpy()[ids].tolist(), reverse=True)[:25]


def _agg_ref(table, mask, keys, fn):
    t = table.filter(pa.array(mask))
    return t.group_by(keys).aggregate(fn) if keys else t


@pytest.mark.gpu
@pytest.mark.parametrize("name,k", [("s_plain", 1000), ("s_dict", 17), ("i_plain", 100_000), ("f_plain", 16),
                                    ("i_delta", 1000), ("d32", 17)])
def test_aggregates_with_in(provs, name, k):
    pv, table = provs
    rng = np.random.default_rng(k)
    values = domain(table, name, rng, k)
    for negated in (False, True):
        flt = [col(name).isin(values, negated=negated)]
        mask = expected(table, name, values, negated)
        ft = table.filter(pa.array(mask))
        for prov in pv.values():
            # dense GROUP BY
            got = prov.aggregate(["g"], [count_star(), sum_("seq"), count("i_dict")], flt).table().sort_by("g")
            ref = ft.group_by(["g"]).aggregate([([], "count_all"), ("seq", "sum"), ("i_dict", "count")]).sort_by("g")
            assert got["g"].to_pylist() == ref["g"].to_pylist()
            assert got["count(*)"].to_pylist() == ref["count_all"].to_pylist()
            assert got["sum(seq)"].to_pylist() == ref["seq_sum"].to_pylist()
            assert got["count(i_dict)"].to_pylist() == ref["i_dict_count"].to_pylist()
            # hashed GROUP BY (40 000 x 40 000 key values)
            got = prov.aggregate(["k1", "k2"], [count_star(), sum_("seq")], flt).table().sort_by([("k1", "ascending"), ("k2", "ascending")])
            ref = ft.group_by(["k1", "k2"]).aggregate([([], "count_all"), ("seq", "sum")]).sort_by([("k1", "ascending"), ("k2", "ascending")])
            assert got["count(*)"].to_pylist() == ref["count_all"].to_pylist()
            assert got["sum(seq)"].to_pylist() == ref["seq_sum"].to_pylist()
            # COUNT(DISTINCT)
            got = prov.aggregate(["g"], [count_distinct("k1")], flt).table().sort_by("g")
            ref = ft.group_by(["g"]).aggregate([("k1", "count_distinct")]).sort_by("g")
            assert got["count(distinct k1)"].to_pylist() == ref["k1_count_distinct"].to_pylist()
            # MEDIAN over a Float64 column without NaN
            got = prov.aggregate([], [median("x"), count_star()], flt).table()
            xs = ft["x"].to_numpy()
            assert got["count(*)"].to_pylist() == [len(xs)]
            if len(xs):
                assert got["median(x)"].to_pylist()[0] == pytest.approx(float(np.median(xs)), rel=1e-12, abs=1e-15)


@pytest.mark.gpu
@pytest.mark.parametrize("switches", [{"PQB_GRID": 1}, {"PQB_GRID": 3}, {"PQB_FILTER_STAGES": 4}, {"PQB_FILTER_CTAS": 8},
                                      {"PQB_AGG_KROWS": 2}, {"PQB_AGG_STAGES": 2}])
def test_forced_configurations(provs, switches):
    pv, table = provs
    rng = np.random.default_rng(11)
    a, b = domain(table, "s_plain", rng, 1000), domain(table, "i_delta", rng, 17)
    flt = [col("s_plain").isin(a) | col("i_delta").isin(b, negated=True)]
    la, lb = expected(table, "s_plain", a, False), expected(table, "i_delta", b, True)
    want = la | lb
    with env(**switches):
        for prov in pv.values():
            check_scan(prov, table, flt, want)
            got = prov.aggregate(["g"], [count_star()], flt).table().sort_by("g")
            ref = table.filter(pa.array(want)).group_by(["g"]).aggregate([([], "count_all")]).sort_by("g")
            assert got["count(*)"].to_pylist() == ref["count_all"].to_pylist()


@pytest.mark.gpu
def test_row_group_pruning(provs):
    pv, table = provs
    # seq rises with the row: every row group of the first file holds a disjoint range
    values = [5, 17, RG_ROWS + 3, N1 + 10, 10 ** 12]
    flt = [col("seq").isin(values)]
    want = expected(table, "seq", values, False)
    for prov in pv.values():
        res = prov.scan(filters=flt)
        assert res.metrics["row_groups_pruned"] > 0, res.metrics
        assert np.array_equal(np.sort(ids_of(res)), np.flatnonzero(want))
    for name, vals in (("s_dba", ["zzz-after-all", "0-before-all"]), ("d32", [dt.date(2200, 1, 1)]),
                       ("f_plain", [1e9, -1e9])):
        res = pv["files"].scan(filters=[col(name).isin(vals)], count_only=True)
        assert res.metrics["rows_selected"] == 0 and res.metrics["row_groups_pruned"] == res.metrics["row_groups_total"], (name, res.metrics)


def _raw_in(prov, name, typ, n, data, flags=0):
    """A PQ_OP_IN with hand-packed elements, through the provider's scan."""
    import parseable_b200.query as Q
    orig = Q._Desc.compile_pred

    def patched(self, e, ops):
        if e.kind == "raw_in":
            ops.append(self._in_op(self.col_index(name), flags, typ, n, data))
        else:
            orig(self, e, ops)
    Q._Desc.compile_pred = patched
    try:
        return prov.scan(filters=[Q.Expr("raw_in")], count_only=True)
    finally:
        Q._Desc.compile_pred = orig


@pytest.mark.gpu
def test_refusals(provs, data):
    pv, table = provs
    prov = pv["resident"]
    good = [col("s_dict").isin(["host-0001", "host-0002"])]
    want = int(expected(table, "s_dict", ["host-0001", "host-0002"], False).sum())
    import struct
    cases = [
        (lambda: _raw_in(prov, "i_dict", L.PQ_T_I64, 0, b""), L.PQ_ERR_INVALID_ARG, "no elements"),
        (lambda: _raw_in(prov, "i_dict", L.PQ_T_I64, 2, struct.pack("<q", 1)), L.PQ_ERR_INVALID_ARG, "8 bytes"),
        (lambda: _raw_in(prov, "s_dict", L.PQ_T_UTF8, 2, struct.pack("<I", 1) + b"a" + struct.pack("<I", 5) + b"ab"),
         L.PQ_ERR_INVALID_ARG, "element 1"),
        (lambda: _raw_in(prov, "s_dict", L.PQ_T_UTF8, 1, struct.pack("<I", 1) + b"ab"), L.PQ_ERR_INVALID_ARG, "str_len"),
        (lambda: _raw_in(prov, "i_dict", L.PQ_T_I64, 1, struct.pack("<q", 1), flags=4), L.PQ_ERR_INVALID_ARG, "flags"),
        (lambda: prov.scan(filters=[col("i_dict").isin([1, 2, "x"])], count_only=True), L.PQ_ERR_INVALID_ARG, "element 0"),
        (lambda: prov.scan(filters=[col("s_dict").isin(["a", 3])], count_only=True), L.PQ_ERR_INVALID_ARG, "element 0"),
        (lambda: prov.scan(filters=[col("d32").isin([1, 2])], count_only=True), L.PQ_ERR_UNSUPPORTED, "element 0"),
        (lambda: prov.scan(filters=[col("i_dict").isin([dt.date(2020, 1, 1)])], count_only=True), L.PQ_ERR_UNSUPPORTED, "element 0"),
        (lambda: prov.scan(filters=[col("b").isin([1])], count_only=True), L.PQ_ERR_INVALID_ARG, "element 0"),
        (lambda: prov.scan(filters=[col("i_dict").isin(range((1 << 20) + 1))], count_only=True), L.PQ_ERR_UNSUPPORTED, "2^20"),
        (lambda: prov.scan(filters=[col("s_plain").isin(["x" * (1 << 16)] * 1100)], count_only=True), L.PQ_ERR_UNSUPPORTED, "64 MiB"),
        # 16 leaves: one IN counts once whatever its length, but a 17th leaf is refused
        (lambda: prov.scan(filters=[reduce(lambda a, b: a | b, [col("i_dict").isin(range(i, i + 100)) for i in range(17)])],
                           count_only=True), L.PQ_ERR_UNSUPPORTED, "too many leaf"),
    ]
    for run, code, text in cases:
        with pytest.raises(QueryError) as ei:
            run()
        assert ei.value.code == code and text in str(ei.value), ei.value
        assert prov.scan(filters=good, count_only=True).metrics["rows_selected"] == want
    ok = [reduce(lambda a, b: a | b, [col("i_dict").isin(range(i, i + 100)) for i in range(16)])]
    assert prov.scan(filters=ok, count_only=True).metrics["rows_selected"] == int(
        expected(table, "i_dict", list(range(115)), False).sum())
    # 2^63 against Int64 is a second leaf: eight such lists fit in 16 leaves, nine do not
    with pytest.raises(QueryError) as ei:
        prov.scan(filters=[reduce(lambda a, b: a & b, [col("i_dict").isin([TOP, 1.0, 2.0, None], negated=True)] * 9)],
                  count_only=True)
    assert ei.value.code == L.PQ_ERR_UNSUPPORTED and "too many leaf" in str(ei.value)
    # pages without a flat-store copy (the flat kernels switched off): refused
    with env(PQB_FLAT_SCAN=0):
        with pytest.raises(QueryError) as ei:
            pv["files"].scan(filters=[col("s_dict").isin(["host-0001", "host-0002"])], count_only=True)
        assert ei.value.code == L.PQ_ERR_UNSUPPORTED and "flat-store copy" in str(ei.value)
    # x IN (NULL) is NULL on every row; NOT IN too
    for neg in (False, True):
        assert prov.scan(filters=[col("i_dict").isin([None], negated=neg)], count_only=True).metrics["rows_selected"] == 0


@pytest.mark.gpu
def test_program_limits(provs):
    pv, table = provs
    prov = pv["resident"]
    # IN with a NULL element and NOT: leaf, CONST NULL, OR, NOT (4 ops, stack 2) per list; 10 such lists with 9 ANDs is
    # 49 ops: over the 40-op program although the descriptor holds only 19
    e = reduce(lambda a, b: a & b, [col("i_dict").isin([i, i + 1, None], negated=True) for i in range(10)])
    with pytest.raises(QueryError) as ei:
        prov.scan(filters=[e], count_only=True)
    assert ei.value.code == L.PQ_ERR_UNSUPPORTED and "program too long" in str(ei.value)
    # right-nested ANDs 7 deep, the innermost an IN with a NULL element: its `OR NULL` needs a ninth stack slot
    e = col("i_dict").isin([1, 2, None])
    for _ in range(7):
        e = (col("g") == 3) & e
    with pytest.raises(QueryError) as ei:
        prov.scan(filters=[e], count_only=True)
    assert ei.value.code == L.PQ_ERR_UNSUPPORTED and "nesting too deep" in str(ei.value)
