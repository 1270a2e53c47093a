"""Aggregate queries on a resident table run on streams the library keeps for reuse: the same query repeated, then other
queries, on one thread, and two threads querying one table at the same time.  The results have tens of thousands of
string groups (string offsets over several passes of the one-CTA scan).  GPU answers are compared with Acero's."""
import threading

import numpy as np
import pyarrow as pa
import pyarrow.compute as pc
import pyarrow.parquet as pq
import pytest

from parseable_b200.query import DeviceTable, StandardTableProvider, col, count_star, max_, min_, sum_

N_ROWS = 400_000
N_KEYS = 40_000


@pytest.fixture(scope="module")
def data(tmp_path_factory):
    rng = np.random.default_rng(7)
    # keys of 1 .. 40 bytes, so that the offsets of one pass differ from a fixed stride
    lens = rng.integers(1, 41, N_KEYS)
    words = [(f"k{i:05d}-" + "x" * int(n))[: max(int(n), 6)] + f"{i}" for i, n in enumerate(lens)]
    key = pa.array([words[i] for i in rng.integers(0, N_KEYS, N_ROWS)], pa.string())
    lvl = pa.array(np.array(["INFO", "WARN", "ERROR"])[rng.integers(0, 3, N_ROWS)], pa.string())
    val = pa.array(rng.integers(-1000, 1000, N_ROWS), pa.int64())
    t = pa.table({"host": key, "level": lvl, "bytes": val})
    path = str(tmp_path_factory.mktemp("tail") / "tail.parquet")
    pq.write_table(t, path, row_group_size=100_000, use_dictionary=True)
    return path, t


SCHEMA = {"host": pa.string(), "level": pa.string(), "bytes": pa.int64()}


def _want(t: pa.Table, keys, level=None):
    if level is not None:
        t = t.filter(pc.equal(t["level"], level))
    g = t.group_by(keys).aggregate([([], "count_all"), ("bytes", "sum"), ("level", "min"), ("level", "max")])
    g = g.rename_columns({"count_all": "count(*)", "bytes_sum": "sum(bytes)", "level_min": "min(level)", "level_max": "max(level)"})
    return g.select(keys + ["count(*)", "sum(bytes)", "min(level)", "max(level)"]).sort_by([(k, "ascending") for k in keys])


def _got(prov, keys, level=None):
    flt = [col("level") == level] if level is not None else []
    r = prov.aggregate(keys, [count_star(), sum_("bytes"), min_("level"), max_("level")], flt).table()
    return r.select(keys + ["count(*)", "sum(bytes)", "min(level)", "max(level)"]).sort_by([(k, "ascending") for k in keys])


def _same(a: pa.Table, b: pa.Table):
    assert a.num_rows == b.num_rows
    for name in a.column_names:
        assert a[name].cast(b.schema.field(name).type).to_pylist() == b[name].to_pylist(), name


@pytest.mark.gpu
def test_many_string_groups_repeated(data):
    path, t = data
    table = DeviceTable([path], list(SCHEMA))
    try:
        prov = StandardTableProvider(table, schema=SCHEMA)
        want = _want(t, ["host"])
        assert want.num_rows > 2 * 16_384
        for _ in range(3):
            _same(_got(prov, ["host"]), want)
        _same(_got(prov, ["host"], "ERROR"), _want(t, ["host"], "ERROR"))
        _same(_got(prov, ["level"]), _want(t, ["level"]))
    finally:
        table.close()


@pytest.mark.gpu
def test_two_threads_one_table(data):
    path, t = data
    table = DeviceTable([path], list(SCHEMA))
    try:
        prov = StandardTableProvider(table, schema=SCHEMA)
        want = {"host": _want(t, ["host"]), "level": _want(t, ["level"], "WARN")}
        for name, level in (("host", None), ("level", "WARN")):   # the side tables each query builds once
            _same(_got(prov, [name], level), want[name])
        errors = []

        def run(name, level):
            try:
                for _ in range(8):
                    _same(_got(prov, [name], level), want[name])
            except Exception as e:  # pragma: no cover - reported below
                errors.append(e)

        th = [threading.Thread(target=run, args=("host", None)), threading.Thread(target=run, args=("level", "WARN"))]
        for x in th:
            x.start()
        for x in th:
            x.join()
        assert not errors, errors
    finally:
        table.close()


def _tail_lines(capfd):
    return [l for l in capfd.readouterr().err.splitlines() if l.startswith("[pqb] result tail:")]


@pytest.mark.gpu
def test_repeat_takes_one_round_trip(data, capfd, monkeypatch):
    """A repeat of a plan lays its result block out for the previous answer's groups before the count is back; another
    literal, another aggregate or another key is another plan.  Every answer equals Acero's."""
    path, t = data
    monkeypatch.setenv("PQB_VERBOSE", "1")
    table = DeviceTable([path], list(SCHEMA))
    try:
        prov = StandardTableProvider(table, schema=SCHEMA)
        want = _want(t, ["host"])
        capfd.readouterr()
        _same(_got(prov, ["host"]), want)
        assert _tail_lines(capfd) == ["[pqb] result tail: no earlier answer of this plan: two round trips"]
        for _ in range(2):
            _same(_got(prov, ["host"]), want)
            assert _tail_lines(capfd) == [f"[pqb] result tail: one round trip, block for {want.num_rows} groups"]
        for level in ("ERROR", "WARN"):   # another literal: another plan
            _same(_got(prov, ["host"], level), _want(t, ["host"], level))
            assert _tail_lines(capfd) == ["[pqb] result tail: no earlier answer of this plan: two round trips"]
        _same(_got(prov, ["level"]), _want(t, ["level"]))   # another key
        assert _tail_lines(capfd) == ["[pqb] result tail: no earlier answer of this plan: two round trips"]
        r = prov.aggregate(["host"], [count_star(), sum_("bytes"), min_("level"), max_("level"), max_("bytes")]).table()   # one more aggregate
        assert _tail_lines(capfd) == ["[pqb] result tail: no earlier answer of this plan: two round trips"]
        want_max = t.group_by(["host"]).aggregate([("bytes", "max")]).sort_by("host")
        assert r.sort_by("host")["max(bytes)"].to_pylist() == want_max["bytes_max"].to_pylist()
        _same(_got(prov, ["host"], "ERROR"), _want(t, ["host"], "ERROR"))
        assert _tail_lines(capfd)[0].startswith("[pqb] result tail: one round trip")
    finally:
        table.close()


@pytest.mark.gpu
@pytest.mark.parametrize("cap", [100, 1_000_000])
def test_block_capacity_differs_from_the_count(data, capfd, monkeypatch, cap):
    """A block laid out for fewer groups than the answer has is laid out again after the round trip (a second copy); one
    with room for more groups than the answer has holds the answer in its first rows."""
    path, t = data
    monkeypatch.setenv("PQB_VERBOSE", "1")
    monkeypatch.setenv("PQB_TAIL_CAP", str(cap))
    table = DeviceTable([path], list(SCHEMA))
    try:
        prov = StandardTableProvider(table, schema=SCHEMA)
        for level in (None, "ERROR"):
            want = _want(t, ["host"], level)
            capfd.readouterr()
            _same(_got(prov, ["host"], level), want)
            lines = _tail_lines(capfd)
            assert lines[0].startswith("[pqb] result tail: one round trip"), lines
            if cap < want.num_rows:
                assert lines[1:] == [f"[pqb] result tail: {want.num_rows} groups, the block had room for {cap}: second copy"]
            else:
                assert lines[1:] == []
    finally:
        table.close()
