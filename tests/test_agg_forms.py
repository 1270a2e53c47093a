"""Agg pages of k_flat_agg: value pages (FK_FOR) of numeric dictionary pages and bit-packed id pages (FK_IDS) of GROUP BY
keys, which a resident table builds once and the aggregate kernel reads instead of looking every row up.

CPU: the encode / decode pair of decode_core.cuh through the host harness (the same source the kernels compile).
GPU: oracle parity on resident tables, and the same answers with the forms switched off (PQB_AGG_FORMS=0)."""
import ctypes as C
import math
import os
import re
import struct
from contextlib import contextmanager

import numpy as np
import pyarrow as pa
import pyarrow.parquet as pq
import pytest

from oracle.oracle import Oracle
from parseable_b200.query import (DeviceTable, StandardTableProvider, avg, col, count, count_distinct, count_star, max_,
                                  min_, sum_)

F64_REL = 1e-9


def f64_bits(x: float) -> int:
    return struct.unpack("<Q", struct.pack("<d", x))[0]


def bits_f64(b: int) -> float:
    return struct.unpack("<d", struct.pack("<Q", b))[0]


@pytest.fixture(scope="module")
def dc(built):
    lib = C.CDLL(os.path.join(built, "tools", "libdecode_core_host.so"))
    lib.dc_dec_encode_f64.argtypes = [C.c_uint64, C.c_uint32, C.POINTER(C.c_int64)]
    lib.dc_dec_encode_f64.restype = C.c_int
    lib.dc_dec_decode_f64.argtypes = [C.c_int64, C.c_uint32]
    lib.dc_dec_decode_f64.restype = C.c_uint64
    lib.dc_dec_decode_many.argtypes = [C.c_void_p, C.c_uint64, C.c_uint32, C.c_void_p]
    lib.dc_dec_decode_many.restype = None
    lib.dc_for_encode.argtypes = [C.c_int64, C.c_int64]
    lib.dc_for_encode.restype = C.c_uint64
    lib.dc_for_decode.argtypes = [C.c_int64, C.c_uint32]
    lib.dc_for_decode.restype = C.c_int64
    lib.dc_bit_width.argtypes = [C.c_uint64]
    lib.dc_bit_width.restype = C.c_uint32
    return lib


def encode(dc, v: float, e: int):
    k = C.c_int64(0)
    return k.value if dc.dc_dec_encode_f64(f64_bits(v), e, C.byref(k)) else None


# ---- CPU ----------------------------------------------------------------------------------------------------------
def test_decode_equals_ieee_division(dc):
    """The decode is k / 10^e rounded to nearest: identical to IEEE division over the whole |k| < 2^53 range."""
    rng = np.random.default_rng(11)
    for e in range(10):
        for lim in (10, 10**4, 10**9, 10**15, 2**53 - 1):
            k = rng.integers(-lim, lim, size=100_000, dtype=np.int64)
            out = np.empty(k.size, np.uint64)
            dc.dc_dec_decode_many(k.ctypes.data, k.size, e, out.ctypes.data)
            assert np.array_equal(out, (k.astype(np.float64) / 10.0**e).view(np.uint64)), (e, lim)


@pytest.mark.parametrize("e", range(10))
def test_random_decimals_round_trip(dc, e):
    rng = np.random.default_rng(100 + e)
    k = rng.integers(-10**12, 10**12, size=20_000)
    for kk in k[:2000]:
        v = int(kk) / 10**e                       # what a writer of decimal values produces
        got = encode(dc, v, e)
        assert got is not None, (v, e)
        assert dc.dc_dec_decode_f64(got, e) == f64_bits(v)
    # negative decimals and values next to 2^53
    for v, ee in ((-0.5, 1), (-123.45, 2), (-1e-9, 9), (float(2**53 - 1), 0), (-float(2**53 - 1), 0), ((2**53 - 1) / 1000, 3)):
        got = encode(dc, v, ee)
        assert got is not None and dc.dc_dec_decode_f64(got, ee) == f64_bits(v), (v, ee)


def test_refused_values(dc):
    sub = bits_f64(1)                                               # the smallest subnormal
    for v in (-0.0, float("nan"), float("inf"), float("-inf"), sub, -sub, 2.0**53, -(2.0**53), 1e300, math.pi):
        for e in range(10):
            assert encode(dc, v, e) is None, (v, e)
    # a NaN with a payload, and +0.0 which is fine
    assert encode(dc, bits_f64(0x7ff8000000000001), 0) is None
    assert encode(dc, 0.0, 0) == 0 and dc.dc_dec_decode_f64(0, 0) == f64_bits(0.0)


def test_frame_of_reference_i64_extremes(dc):
    lo, hi = -(2**63), 2**63 - 1
    assert dc.dc_for_encode(hi, lo) == 2**64 - 1 and dc.dc_bit_width(dc.dc_for_encode(hi, lo)) == 64
    for base, v in ((lo, lo), (lo, lo + 2**32 - 1), (hi - 5, hi), (-3, 7), (hi, hi), (2**62, 2**62 + 12345)):
        bits = dc.dc_for_encode(v, base)
        assert bits < 2**32
        assert dc.dc_for_decode(base, bits) == v
    # base + bits wraps exactly (the kernel adds in 64 bits, two's complement)
    assert dc.dc_for_decode(hi, 1) == lo
    assert dc.dc_bit_width(0) == 0 and dc.dc_bit_width(1) == 1 and dc.dc_bit_width(2**32 - 1) == 32 and dc.dc_bit_width(2**32) == 33


# ---- GPU ----------------------------------------------------------------------------------------------------------
ROWS = 200_000
RG = 100_000


def _keys(rng, card, n, null_rate=0.0):
    v = np.array([f"k{card}_{i:06d}" for i in range(card)], dtype=object)[rng.integers(0, card, n)]
    v[: min(card, n)] = np.array([f"k{card}_{i:06d}" for i in range(min(card, n))], dtype=object)   # every value occurs
    if null_rate:
        v[rng.random(n) < null_rate] = None
    return pa.array(v, pa.string())


def _with_nulls(rng, a, rate):
    return np.where(rng.random(a.size) < rate, None, a)


def _write(path, t):
    pq.write_table(t, path, row_group_size=RG, use_dictionary=True, data_page_size=64 * 1024)


@pytest.fixture(scope="module")
def forms_files(built, tmp_path_factory):
    """Two files; the second lacks column `d`.  Row group 0 of `d` holds decimals (qualifies), row group 1 random doubles
    (keeps the dictionary); `i` spans the whole Int64 range in row group 1 (more than 32 bits: keeps the dictionary)."""
    rng = np.random.default_rng(5)
    d0 = np.round(rng.integers(-10**6, 10**6, RG) / 100.0, 2)
    d1 = rng.standard_normal(RG) * 1e3
    i0 = rng.integers(-5000, 5000, RG)
    i1 = np.where(rng.random(RG) < 0.5, rng.integers(-(2**63), -(2**62), RG), rng.integers(2**62, 2**63 - 1, RG))
    i1[:2] = [-(2**63), 2**63 - 1]
    t1 = pa.table({
        "k1": _keys(rng, 2, ROWS),
        "k13": _keys(rng, 5000, ROWS, 0.01),
        "k14": _keys(rng, 10000, ROWS),
        "k17": _keys(rng, 70000, ROWS),
        "d": pa.array(_with_nulls(rng, np.concatenate([d0, d1]), 0.02), pa.float64()),
        "i": pa.array(_with_nulls(rng, np.concatenate([i0, i1]), 0.02), pa.int64()),
        "m": pa.array(rng.integers(0, 1000, ROWS) * 1000 + 1_700_000_000_000, pa.int64()),
    })
    t2 = t1.slice(0, RG).drop_columns(["d"])
    td = tmp_path_factory.mktemp("agg_forms")
    p1, p2 = str(td / "f1.parquet"), str(td / "f2.parquet")
    _write(p1, t1)
    _write(p2, t2)
    both = pa.concat_tables([t1, t2.append_column("d", pa.nulls(t2.num_rows, pa.float64())).select(t1.column_names)])
    return [p1, p2], Oracle(both), t1.schema


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


def _rows(t: pa.Table, nk: int) -> dict:
    cols = [t.column(i).to_pylist() for i in range(t.num_columns)]
    return {tuple(cols[k][r] for k in range(nk)): [cols[c][r] for c in range(nk, t.num_columns)] for r in range(t.num_rows)}


def _oracle(ora: Oracle, keys, aggs, flt) -> pa.Table:
    """The oracle's table; COUNT(DISTINCT c) as the non-NULL `c` groups under each key (GROUP BY keys + c)."""
    plain = [a for a in aggs if a.fn != "count_distinct"]
    base = ora.group_by(keys, plain, flt)
    kc = [base.column(i).to_pylist() for i in range(len(keys))]
    cols = {k: base.column(i) for i, k in enumerate(keys)}
    for a in aggs:
        if a.fn != "count_distinct":
            cols[a.name] = base.column(a.name)
            continue
        g = ora.group_by(keys + [a.column], [count_star()], flt)
        n: dict = {}
        for r in range(g.num_rows):
            row = tuple(g.column(i)[r].as_py() for i in range(len(keys)))
            n[row] = n.get(row, 0) + (g.column(len(keys))[r].as_py() is not None)
        cols[a.name] = pa.array([n.get(tuple(c[r] for c in kc), 0) for r in range(base.num_rows)], pa.int64())
    return pa.table(cols)


def _same(got: pa.Table, want: pa.Table, nk: int, what: str):
    assert got.column_names == want.column_names, what
    g, w = _rows(got, nk), _rows(want, nk)
    assert g.keys() == w.keys(), what
    names = got.column_names[nk:]
    for key, wv in w.items():
        for name, a, b in zip(names, g[key], wv):
            if isinstance(b, float) and (name.startswith("sum(") or name.startswith("avg(")):
                assert a is not None and math.isclose(a, b, rel_tol=F64_REL, abs_tol=1e-300), (what, key, name, a, b)
            elif isinstance(b, float):
                assert a is not None and f64_bits(a) == f64_bits(b), (what, key, name, a, b)   # MIN / MAX: bit exact
            else:
                assert a == b, (what, key, name, a, b)


CASES = {
    "values_mixed_chunks": (["k1"], [count_star(), sum_("d"), min_("d"), max_("d"), sum_("i"), min_("i"), max_("i"), avg("m")], []),
    "key_13_bits_nulls": (["k13"], [count_star(), sum_("d"), count("d"), max_("i")], []),
    "key_14_bits": (["k14"], [sum_("m"), min_("d")], []),
    "key_17_bits": (["k17"], [count_star(), max_("d"), sum_("i")], []),
    "filtered_and_aggregated": (["k13"], [sum_("i"), max_("i"), sum_("d")], [col("i") > 0]),
    "key_also_filtered": (["k13"], [sum_("d")], [col("k13") != "k5000_000001"]),
    "with_count_distinct": (["k1"], [count_distinct("k14"), sum_("d"), min_("m")], []),
    "hashed_group_by": (["k17", "k14"], [count_star(), sum_("d"), max_("i")], []),
}


@pytest.fixture(scope="module")
def resident(forms_files):
    files, ora, schema = forms_files
    table = DeviceTable(files, schema.names)
    yield StandardTableProvider(table, schema=schema), ora
    table.close()


@pytest.mark.gpu
@pytest.mark.parametrize("case", list(CASES))
def test_oracle_parity_and_forms_off(resident, case, capfd):
    prov, ora = resident
    keys, aggs, flt = CASES[case]
    want = _oracle(ora, keys, aggs, flt)
    with env_var("PQB_VERBOSE", "1"):
        got = prov.aggregate(keys, aggs, flt).table()
    log = capfd.readouterr().err
    _same(got, want, len(keys), f"{case}: GPU vs oracle")
    with env_var("PQB_AGG_FORMS", "0"):
        off = prov.aggregate(keys, aggs, flt).table()
    _same(off, got, len(keys), f"{case}: PQB_AGG_FORMS=0 vs forms")
    for slot, kind, bits in FORMS[case]:
        m = re.search(rf"\({slot}\): {kind} pages, (\d+) bits", log)
        assert m, (case, slot, log)
        assert bits is None or int(m.group(1)) == bits, (case, slot, m.group(0))
    for slot in NO_FORMS.get(case, []):
        assert f"({slot}):" not in log, (case, slot, log)   # a filtered column reads its index pages
    if case == "with_count_distinct":
        assert "pages," not in log, log                     # a query with COUNT(DISTINCT) reads index pages only


# the agg pages each case must read (PQB_VERBOSE line of the marked slot): Float64 value pages of `d` (its decimal chunks;
# the random doubles keep the dictionary), Int64 value pages of `i` (the narrow chunks) and `m`, id pages of every key
# at bits(card - 1) bits.  `k17`'s dictionary overflows into PLAIN pages: those keep their 32-bit id pages, so the slot
# mixes both kinds of id page (and is staged at 32 bits)
FORMS = {
    "values_mixed_chunks": [("k1", "id", 1), ("d", "value", None), ("i", "value", None), ("m", "value", None)],
    "key_13_bits_nulls": [("k13", "id", 13), ("d", "value", None)],
    "key_14_bits": [("k14", "id", 14), ("m", "value", None), ("d", "value", None)],
    "key_17_bits": [("k17", "id", 17), ("d", "value", None), ("i", "value", None)],
    "filtered_and_aggregated": [("k13", "id", 13), ("d", "value", None)],
    "key_also_filtered": [("d", "value", None)],
    "with_count_distinct": [],
    "hashed_group_by": [("k17", "id", 17), ("k14", "id", 14), ("d", "value", None)],
}
NO_FORMS = {"filtered_and_aggregated": ["i"], "key_also_filtered": ["k13"]}


@pytest.mark.gpu
def test_file_list_builds_no_forms(forms_files, capfd):
    """A file list opens its table for one query: no agg pages are built, the answer is the same."""
    files, ora, schema = forms_files
    prov = StandardTableProvider(files, schema=schema)
    keys, aggs, flt = CASES["values_mixed_chunks"]
    with env_var("PQB_VERBOSE", "1"):
        got = prov.aggregate(keys, aggs, flt).table()
    assert "value pages" not in capfd.readouterr().err
    _same(got, _oracle(ora, keys, aggs, flt), len(keys), "file list vs oracle")
