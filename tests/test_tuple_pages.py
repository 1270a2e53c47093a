"""Tuple id pages: a GROUP BY of two or more dictionary keys on a resident table reads one id per row, the rank of its
key tuple by row count, so that k_flat_agg's hot table holds the hottest groups rather than the hottest values of the
largest key.

CPU: a numpy restatement of the numbering (rows per tuple, descending, ties by mixed-radix id ascending) and of the
coverage it buys on the generator's distributions.
GPU: every query with and without PQB_TUPLE_PAGES=0 on one resident table, equal row for row (order included) and equal
to the oracle after a canonical sort; the same under the kernel's experiment switches; which queries take the path;
two threads asking for the same tuple at once; a fresh table whose first query is a tuple query with value pages; key
columns whose pages do not line up (jobs that start inside a lead page and share words with their neighbours); the
ranking the library builds, read from PQB_VERBOSE=2, against the restatement.

One-line mutations and the test that catches each:
- ties ranked the other way (count descending, mixed-radix id DEScending): test_ranking_built_on_the_device;
- `order` ignored by k_slot_tile_counts / k_slot_compact (slots listed by tuple id): every case of
  test_tuple_pages_equal_per_key_ids_and_oracle, which compares with PQB_TUPLE_PAGES=0 row for row;
- a NULL key written as id 0 instead of card in tuple_mixed: the oracle checks of host_status and three_keys (the first
  file has 2 % NULL keys, which then merge into another group);
- the page width one bit short: the oracle checks of every case (tuple ids lose their top bit and groups merge)."""
import math
import os
import re
import threading
import time
from contextlib import contextmanager

import numpy as np
import pyarrow as pa
import pyarrow.parquet as pq
import pytest

from oracle.oracle import Oracle
from parseable_b200 import synth
from parseable_b200.query import (DeviceTable, StandardTableProvider, Window, col, count, count_distinct, count_star,
                                  date_bin, max_, median, min_, sum_)


# ---- CPU ----------------------------------------------------------------------------------------------------------
def tuple_numbering(mixed: np.ndarray, space: int):
    """(wide, order, rank) of the groups that occur: wide[t] = mixed-radix id of tuple t, ranked by rows descending and
    mixed-radix id ascending; order[p] = the tuple ids in ascending mixed-radix order; rank[m] = tuple id of id m."""
    counts = np.bincount(mixed, minlength=space)
    occurring = np.flatnonzero(counts)
    wide = occurring[np.lexsort((occurring, -counts[occurring]))]
    rank = np.zeros(space, np.int64)
    rank[wide] = np.arange(len(wide))
    return wide, rank[occurring], rank


def test_ranking_ties_by_mixed_radix_id():
    mixed = np.array([7, 3, 3, 9, 7, 1, 1, 5, 5, 5])
    wide, order, rank = tuple_numbering(mixed, 16)
    assert wide.tolist() == [5, 1, 3, 7, 9]           # 5 has three rows; 1, 3 and 7 two each, in id order; 9 one
    assert order.tolist() == [1, 2, 0, 3, 4]          # ids 1, 3, 5, 7, 9 -> their tuple ids
    assert wide[order].tolist() == sorted(wide.tolist())
    assert rank[wide].tolist() == list(range(5))


def test_ranking_on_generated_keys():
    """host x status of two generated row groups: the numbering is a bijection onto the occurring groups, ranks are by
    count and the first 8 tuples are the 8 largest groups."""
    t = pa.concat_tables([synth.logs16_row_group(g, 50_000, columns=["host", "status"]) for g in range(2)])
    host = t.column("host").combine_chunks().indices.to_numpy()
    status = np.searchsorted(synth.STATUS, t.column("status").to_numpy())
    mixed = host * 6 + status
    wide, order, rank = tuple_numbering(mixed, 10_000 * 6)
    counts = np.bincount(mixed, minlength=60_000)
    assert len(wide) == len(np.unique(mixed))
    c = counts[wide]
    assert np.all(c[:-1] >= c[1:])
    assert np.all((c[:-1] > c[1:]) | (wide[:-1] < wide[1:]))
    assert np.array_equal(np.sort(wide), wide[order])
    assert set(wide[:8].tolist()) == set(np.argsort(-counts, kind="stable")[:8].tolist())


def test_coverage_of_the_hot_table():
    """C4's groups (Zipf 1.1 over 10 000 hosts x 5 statuses, NULL status id included in the radix): rows outside 2 856
    hot slots and rows on the 8 lane slots, in slot order and in tuple order."""
    w = 1.0 / np.arange(1, 10_001) ** 1.1
    ph = w / w.sum()
    ps = np.array(sorted(synth.STATUS_P, reverse=True))
    slot = np.zeros(10_000 * 6)
    slot.reshape(10_000, 6)[:, :5] = np.outer(ph, ps)   # slot = host * 6 + status, hot-first ids; id 5 is NULL
    tup = np.sort(slot[slot > 0])[::-1]
    assert math.isclose(1 - slot[:2856].sum(), 0.215, abs_tol=5e-4)
    assert math.isclose(1 - tup[:2856].sum(), 0.137, abs_tol=5e-4)
    assert math.isclose(slot[:8].sum(), 0.214, abs_tol=5e-4)
    assert math.isclose(tup[:8].sum(), 0.306, abs_tol=5e-4)
    assert len(tup) == 50_000


# ---- GPU ----------------------------------------------------------------------------------------------------------
RG = 70_000
COLS = ["p_timestamp", "host", "status", "level", "service", "bytes", "latency_ms", "duration_s", "cpu"]


@contextmanager
def env(**kv):
    old = {k: os.environ.get(k) for k in kv}
    os.environ.update({k: str(v) for k, v in kv.items()})
    try:
        yield
    finally:
        for k, v in old.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v


@pytest.fixture(scope="module")
def files(built, tmp_path_factory):
    """Two files: three row groups with 2 % NULLs in every column, and two row groups without `service`."""
    td = tmp_path_factory.mktemp("tuple_pages")
    p1, p2 = str(td / "a.parquet"), str(td / "b.parquet")
    synth.write_logs16(p1, n_row_groups=3, rows_per_group=RG, null_rate=0.02, columns=COLS)
    synth.write_logs16(p2, n_row_groups=2, first_rg=3, rows_per_group=RG, columns=[c for c in COLS if c != "service"])
    t1 = pq.read_table(p1)
    t2 = pq.read_table(p2)
    t2 = t2.append_column(pa.field("service", t1.schema.field("service").type), pa.nulls(t2.num_rows, t1.schema.field("service").type))
    both = pa.concat_tables([t1, t2.select(t1.column_names)])
    return [p1, p2], Oracle(both), t1.schema


@pytest.fixture(scope="module")
def resident(files):
    paths, ora, schema = files
    table = DeviceTable(paths, COLS)
    yield StandardTableProvider(table, schema=schema), ora, table
    table.close()


AGGS = [count_star(), sum_("bytes"), min_("latency_ms"), max_("latency_ms"), sum_("duration_s"), max_("cpu")]
TS_LO = synth.TS_BASE - 2 * synth.RG_TS_STRIDE_MS - 1
CASES = {
    "host_status": (["host", "status"], AGGS, [], {}),
    "status_host": (["status", "host"], AGGS, [], {}),
    "level_status": (["level", "status"], [count_star(), sum_("bytes")], [], {}),
    "three_keys": (["level", "status", "host"], [count_star(), max_("cpu")], [], {}),
    "absent_in_one_file_wide": (["host", "service"], [count_star(), sum_("bytes")], [], {}),
    "where_filter": (["host", "status"], AGGS, [col("latency_ms") > 40], {}),
    "time_range_prunes": (["host", "status"], [count_star(), sum_("bytes")], [col("p_timestamp") >= TS_LO], {}),
    "order_limit_ties": (["host", "status"], [count_star()], [], {"order_by": [(count_star(), "desc")], "limit": 25}),
    "row_number_no_order": (["level", "status"], [count_star()], [], {"window": Window((), 0, None, row_number=True)}),
}


def _canon(t: pa.Table):
    rows = list(zip(*[t.column(i).to_pylist() for i in range(t.num_columns)]))
    return sorted(rows, key=lambda r: tuple((v is None, v) for v in r))


def _close_rows(a, b):
    assert len(a) == len(b)
    for ra, rb in zip(a, b):
        for x, y in zip(ra, rb):
            if isinstance(y, float):
                assert x is not None and math.isclose(x, y, rel_tol=1e-9, abs_tol=1e-12), (ra, rb)
            else:
                assert x == y, (ra, rb)


def _run(prov, case, **kv):
    keys, aggs, flt, extra = CASES[case]
    with env(**kv):
        return prov.aggregate(keys, aggs, flt, **extra).table()


def _rows(t: pa.Table):
    return list(zip(*[c.to_pylist() for c in t.columns]))


@pytest.mark.gpu
@pytest.mark.parametrize("case", list(CASES))
def test_tuple_pages_equal_per_key_ids_and_oracle(resident, case, capfd):
    prov, ora, _ = resident
    keys, aggs, flt, extra = CASES[case]
    got = _run(prov, case, PQB_VERBOSE=1)
    log = capfd.readouterr().err
    assert "group slots: tuple pages" in log, log
    off = _run(prov, case, PQB_TUPLE_PAGES=0)
    assert got.column_names == off.column_names
    # row for row, order included; SUM over Float64 to 1e-9 (its accumulation order follows the hot table)
    _close_rows(_rows(got), _rows(off))
    if "window" in extra or "order_by" in extra:
        return   # the cut is checked against the per-key path above, row for row
    want = ora.group_by(keys, aggs, flt)
    _close_rows(_canon(got), _canon(want))


SWITCHES = [{"PQB_HOT_SLOTS": 64}, {"PQB_LANE_SLOTS": 0}, {"PQB_TAIL_CAP": 3}, {"PQB_GRID": 1}, {"PQB_GRID": 3}]


@pytest.mark.gpu
@pytest.mark.parametrize("sw", SWITCHES, ids=lambda d: "-".join(f"{k}={v}" for k, v in d.items()))
@pytest.mark.parametrize("case", ["host_status", "three_keys", "absent_in_one_file_wide"])
def test_switches(resident, case, sw):
    prov, ora, _ = resident
    keys, aggs, flt, _ = CASES[case]
    got = _run(prov, case, **sw)
    off = _run(prov, case, PQB_TUPLE_PAGES=0, **sw)
    _close_rows(_rows(got), _rows(off))
    _close_rows(_canon(got), _canon(ora.group_by(keys, aggs, flt)))


NOT_ELIGIBLE = {
    "key_also_min": (["host", "status"], [count_star(), min_("host")], []),
    "count_distinct": (["host", "status"], [count_distinct("level")], []),
    "median": (["level", "status"], [median("latency_ms")], []),
    "date_bin": ([date_bin(60_000), "status"], [count_star()], []),
    "key_also_filtered": (["host", "status"], [count_star()], [col("status") == 200]),
    "one_key": (["host"], [count_star()], []),
}


@pytest.mark.gpu
@pytest.mark.parametrize("case", list(NOT_ELIGIBLE))
def test_not_taken(resident, case, capfd):
    prov, _, _ = resident
    keys, aggs, flt = NOT_ELIGIBLE[case]
    with env(PQB_VERBOSE=1):
        prov.aggregate(keys, aggs, flt).table()
    assert "group slots: tuple pages" not in capfd.readouterr().err, case


@pytest.mark.gpu
def test_file_list_not_taken(files, capfd):
    paths, ora, schema = files
    keys, aggs, flt, _ = CASES["host_status"]
    with env(PQB_VERBOSE=1):
        got = StandardTableProvider(paths, schema=schema).aggregate(keys, aggs, flt).table()
    assert "group slots: tuple pages" not in capfd.readouterr().err
    _close_rows(_canon(got), _canon(ora.group_by(keys, aggs, flt)))


@pytest.mark.gpu
def test_two_threads_build_once(files, capfd):
    """Both threads wait at a barrier and then send the table's first tuple query; the calls overlap in time (ctypes
    drops the GIL inside the library) and the pages are built once."""
    paths, ora, schema = files
    table = DeviceTable(paths, COLS)
    try:
        prov = StandardTableProvider(table, schema=schema)
        keys, aggs, flt, _ = CASES["level_status"]
        out, span = [None, None], [None, None]
        gate = threading.Barrier(2)

        def go(i):
            gate.wait()
            t0 = time.perf_counter()
            out[i] = prov.aggregate(keys, aggs, flt).table()
            span[i] = (t0, time.perf_counter())

        with env(PQB_VERBOSE=1):
            th = [threading.Thread(target=go, args=(i,)) for i in range(2)]
            for t in th:
                t.start()
            for t in th:
                t.join()
        log = capfd.readouterr().err
        assert max(a for a, _ in span) < min(b for _, b in span), span   # the two queries were in flight together
        assert len(re.findall(r"\[pqb\] tuple pages: ", log)) == 1, log
        assert len(re.findall(r"group slots: tuple pages", log)) == 2, log
        assert _rows(out[0]) == _rows(out[1])
        _close_rows(_canon(out[0]), _canon(ora.group_by(keys, aggs, flt)))
    finally:
        table.close()


# ---- key columns whose pages do not line up, constant numeric columns, a fresh table -------------------------------
@pytest.fixture(scope="module")
def ragged(built, tmp_path_factory):
    """Three row groups written with 2 KB data pages and no row limit per page: `host` pages hold a few hundred rows,
    `status` / `level` pages many more, so the other keys' page starts cut the lead pages.  `k` and `z` are
    the same value in every row (value pages of width 0 over an index page of width 1)."""
    td = tmp_path_factory.mktemp("tuple_ragged")
    path = str(td / "ragged.parquet")
    parts = []
    for g in range(3):
        t = synth.logs16_row_group(20 + g, 60_000, null_rate=0.01, columns=["host", "status", "level", "bytes"])
        parts.append(t.append_column("k", pa.array(np.full(t.num_rows, 7), pa.int64()))
                      .append_column("z", pa.array(np.full(t.num_rows, 2.5), pa.float64())))
    t = pa.concat_tables([p.cast(parts[0].schema) for p in parts]).combine_chunks()
    pq.write_table(t, path, row_group_size=60_000, use_dictionary=True, data_page_size=2048, write_batch_size=128,
                   max_rows_per_page=1 << 30)
    back = pq.read_table(path)
    return path, Oracle(back), back.schema


RAGGED_AGGS = [count_star(), sum_("k"), min_("k"), max_("z"), sum_("z"), sum_("bytes")]


@pytest.mark.gpu
def test_fresh_table_first_query_with_value_pages(ragged, capfd):
    """The table's first query is a tuple query whose aggregate inputs get value pages in that same query."""
    path, ora, schema = ragged
    cols = ["status", "host", "level", "bytes", "k", "z"]   # `status` (the fewest pages) leads: host's page starts cut it
    for keys in (["host", "status"], ["status", "level", "host"]):
        table = DeviceTable([path], cols)
        try:
            prov = StandardTableProvider(table, schema=schema)
            with env(PQB_VERBOSE=1):
                got = prov.aggregate(keys, RAGGED_AGGS).table()
            log = capfd.readouterr().err
            assert "group slots: tuple pages" in log and "(k): value pages, 0 bits" in log, log
            m = re.search(r"tuple pages: \d+ keys, lead column \w+, \d+ tuples of \d+ slots, \d+ bits, (\d+) jobs over (\d+) lead pages", log)
            assert m and int(m.group(1)) > int(m.group(2)), log   # jobs start inside lead pages
            off = StandardTableProvider(table, schema=schema)
            with env(PQB_TUPLE_PAGES=0):
                ref = off.aggregate(keys, RAGGED_AGGS).table()
            _close_rows(_rows(got), _rows(ref))
            _close_rows(_canon(got), _canon(ora.group_by(keys, RAGGED_AGGS)))
        finally:
            table.close()


@pytest.fixture(scope="module")
def ties(built, tmp_path_factory):
    """12 groups of (a, b) plus NULL-key groups with few distinct row counts: ties everywhere in the ranking."""
    rng = np.random.default_rng(3)
    rows = []
    sizes = [40, 40, 40, 25, 25, 25, 25, 10, 10, 10, 10, 10]
    for i, n in enumerate(sizes):
        rows += [(f"a{i % 4}", f"b{i // 4}")] * n
    rows += [(None, "b0")] * 25 + [("a1", None)] * 10
    rows = [rows[i] for i in rng.permutation(len(rows))]
    t = pa.table({"a": [r[0] for r in rows], "b": [r[1] for r in rows], "v": np.arange(len(rows), dtype=np.int64)})
    path = str(tmp_path_factory.mktemp("tuple_ties") / "ties.parquet")
    pq.write_table(t, path, use_dictionary=True, data_page_size=256, write_batch_size=16)
    return path, Oracle(pq.read_table(path)), pq.read_table(path).schema


@pytest.mark.gpu
def test_ranking_built_on_the_device(ties, capfd):
    """The library's numbering (PQB_VERBOSE=2 lists tuple id, mixed-radix id and rows) is the restatement's: rows
    descending, ties by mixed-radix id ascending, one tuple per group that occurs."""
    path, ora, schema = ties
    table = DeviceTable([path], ["a", "b", "v"])
    try:
        with env(PQB_VERBOSE=2):
            got = StandardTableProvider(table, schema=schema).aggregate(["a", "b"], [count_star(), sum_("v")]).table()
        log = capfd.readouterr().err
        listed = [tuple(map(int, m)) for m in re.findall(r"\[pqb\] tuple (\d+): mixed-radix id (\d+), (\d+) rows", log)]
        assert [t for t, _, _ in listed] == list(range(len(listed))), log
        want = ora.group_by(["a", "b"], [count_star()])
        assert sorted(n for _, _, n in listed) == sorted(want.column("count(*)").to_pylist())
        mixed = np.repeat([m for _, m, _ in listed], [n for _, _, n in listed])
        wide, _, _ = tuple_numbering(mixed, int(mixed.max()) + 1)
        assert wide.tolist() == [m for _, m, _ in listed]
        _close_rows(_canon(got), _canon(ora.group_by(["a", "b"], [count_star(), sum_("v")])))
    finally:
        table.close()
