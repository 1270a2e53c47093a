"""MEDIAN / PERCENTILE_CONT on the CPU: the Python restatement of both aggregates, and the arithmetic the kernel runs.

`restate` is the rule of include/parseable_b200.h (DataFusion 53's median / percentile_cont, restated, not checked): the
non-NULL values sorted by Int64 order or IEEE totalOrder; median = the middle value, or for an even count (lo + hi)
wrapping / 2 toward zero (Int64) or (lo + hi) / 2 (Float64); percentile_cont = v[lo] + f * (v[lo + 1] - v[lo]) with
h = p * (n - 1), lo = floor(h), f = h - lo, and v[lo] itself when f == 0.  Float64 operations on NaN follow x86-64 SSE:
a NaN operand comes back quieted (the first one when both are), an invalid operation gives 0xfff8000000000000.

The restatement is checked against numpy.quantile(method="linear") and pyarrow.compute.quantile on random finite
vectors, and against hand vectors exactly.  The host build of percentile_core.cuh (tools/liborder_keys_host.so: the
decode, median and interpolation k_pct_pick runs) must agree with it bit for bit on edge vectors.  The SQL front's three
forms and its refusals are parsed here too."""
import ctypes as C
import math
import os
import struct

import numpy as np
import pyarrow as pa
import pyarrow.compute as pc
import pytest

from parseable_b200 import _lib as L
from parseable_b200.query import Agg, Query, QueryError, median, percentile_cont, shortest_repr

OE_I64, OE_F64 = 0, 1
I64_MIN, I64_MAX = -(1 << 63), (1 << 63) - 1
QUIET = 1 << 51
DEFAULT_NAN = 0xFFF8000000000000


# ---- the restatement -----------------------------------------------------------------------------------------------
def f64_bits(x: float) -> int:
    return struct.unpack("<Q", struct.pack("<d", x))[0]


def bits_f64(b: int) -> float:
    return struct.unpack("<d", struct.pack("<Q", b))[0]


def nan(payload: int, neg: bool = False) -> float:
    return bits_f64((1 << 63 if neg else 0) | 0x7FF0000000000000 | payload)


def total_order(x: float) -> int:
    b = f64_bits(x)
    mag = b & ((1 << 63) - 1)
    return -mag - 1 if b >> 63 else mag


def _is_nan_bits(b: int) -> bool:
    return (b & ((1 << 63) - 1)) > 0x7FF0000000000000


def x86_op(a: int, b: int, op: str) -> int:
    """a op b on f64 bits with x86-64 SSE NaN results."""
    if _is_nan_bits(a):
        return a | QUIET
    if _is_nan_bits(b):
        return b | QUIET
    x, y = bits_f64(a), bits_f64(b)
    r = {"+": lambda: x + y, "-": lambda: x - y, "*": lambda: x * y, "/": lambda: x / y}[op]()
    return DEFAULT_NAN if math.isnan(r) else f64_bits(r)


def _wrap(v: int) -> int:
    return (v + (1 << 63)) % (1 << 64) - (1 << 63)


def restate(values, fn: str, p: float | None = None, f64: bool = False):
    """The result of median / percentile_cont over `values` (None = NULL) as bits: Int64 results as a signed int, Float64
    results as their u64 bit pattern; None for no non-NULL value."""
    vals = [v for v in values if v is not None]
    if not vals:
        return None
    vals.sort(key=total_order if f64 else None)
    n = len(vals)
    as_bits = (lambda v: f64_bits(v)) if f64 else (lambda v: f64_bits(float(v)))
    if fn == "median":
        lo = vals[(n - 1) // 2]
        if n % 2:
            return f64_bits(lo) if f64 else lo
        hi = vals[n // 2]
        if f64:
            return x86_op(x86_op(f64_bits(lo), f64_bits(hi), "+"), f64_bits(2.0), "/")
        s = _wrap(lo + hi)
        return -((-s) // 2) if s < 0 else s // 2          # toward zero
    h = p * float(n - 1)
    r = math.floor(h)
    f = h - r
    vlo = as_bits(vals[r])
    if f == 0.0:
        return vlo
    d = x86_op(as_bits(vals[r + 1]), vlo, "-")
    return x86_op(vlo, x86_op(f64_bits(f), d, "*"), "+")


def as_value(bits, f64_out: bool):
    return None if bits is None else (bits_f64(bits) if f64_out else bits)


# ---- the restatement against numpy / pyarrow and hand vectors --------------------------------------------------------
@pytest.mark.parametrize("seed", range(6))
def test_restatement_matches_numpy_and_arrow(seed):
    rng = np.random.default_rng(seed)
    for n in (1, 2, 3, 10, 101, 1000):
        xs = rng.normal(0, 1e3, n) if seed % 2 else rng.integers(-10**9, 10**9, n).astype(np.float64)
        ints = rng.integers(-10**12, 10**12, n)
        for p in (0.0, 0.01, 0.25, 0.5, 0.95, 0.99, 1.0, 1 / 3, float(rng.random())):
            got = bits_f64(restate(list(xs), "percentile_cont", p, f64=True))
            assert math.isclose(got, np.quantile(xs, p, method="linear"), rel_tol=1e-12, abs_tol=1e-300)
            assert math.isclose(got, pc.quantile(pa.array(xs), q=p, interpolation="linear")[0].as_py(), rel_tol=1e-12, abs_tol=1e-300)
            got_i = bits_f64(restate([int(v) for v in ints], "percentile_cont", p))
            assert math.isclose(got_i, np.quantile(ints.astype(np.float64), p, method="linear"), rel_tol=1e-12)
        assert math.isclose(bits_f64(restate(list(xs), "median", f64=True)), float(np.median(xs)), rel_tol=1e-12, abs_tol=1e-300)


def test_restatement_hand_vectors():
    assert restate([3, 1, 2], "median") == 2
    assert restate([4, 1, 2, 3], "median") == 2                   # (2 + 3) / 2 toward zero
    assert restate([-4, -1, -2, -3], "median") == -2              # (-3 + -2) / 2 = -2.5 -> -2
    assert restate([None, None], "median") is None
    assert restate([None, 7, None], "median") == 7
    assert restate([I64_MAX, I64_MAX - 1], "median") == -1        # wraps: add_wrapping(..).div_wrapping(2)
    assert restate([I64_MIN, I64_MIN], "median") == 0
    assert restate([I64_MIN, I64_MAX], "median") == 0             # -1 / 2 toward zero
    assert as_value(restate([1.0, 2.0, 4.0, 8.0], "median", f64=True), True) == 3.0
    assert as_value(restate([1, 2, 3, 4], "percentile_cont", 0.5), True) == 2.5
    assert as_value(restate([10, 20, 30], "percentile_cont", 0.0), True) == 10.0
    assert as_value(restate([10, 20, 30], "percentile_cont", 1.0), True) == 30.0
    assert as_value(restate([10, 20, 30, 40], "percentile_cont", 0.25), True) == 17.5
    inf = math.inf
    assert as_value(restate([-inf, 1.0, inf], "percentile_cont", 0.0, True), True) == -inf   # exact ranks: no inf - inf
    assert as_value(restate([-inf, 1.0, inf], "percentile_cont", 1.0, True), True) == inf
    assert restate([-inf, inf], "percentile_cont", 0.5, True) == DEFAULT_NAN                  # -inf + 0.5 * inf
    assert restate([-inf, inf], "median", None, True) == DEFAULT_NAN
    assert restate([nan(5), 1.0], "median", None, True) == f64_bits(nan(5)) | QUIET           # +NaN sorts last
    assert restate([nan(5, True), 1.0], "median", None, True) == f64_bits(nan(5, True)) | QUIET
    assert f64_bits(as_value(restate([0.0, -0.0], "median", None, True), True)) == f64_bits(0.0)
    assert restate([0.0, -0.0, 0.0], "median", None, True) == f64_bits(0.0)
    assert restate([-0.0, -0.0, 0.0], "median", None, True) == f64_bits(-0.0)


# ---- the kernel's arithmetic on the CPU ----------------------------------------------------------------------------
@pytest.fixture(scope="module")
def pk(built):
    lib = C.CDLL(os.path.join(built, "tools", "liborder_keys_host.so"))
    lib.ok_encode.restype = C.c_uint64
    lib.ok_encode.argtypes = [C.c_uint64, C.c_uint32, C.c_int]
    lib.pk_pick.restype = C.c_uint64
    lib.pk_pick.argtypes = [C.POINTER(C.c_uint64), C.c_uint64, C.c_int, C.c_double, C.c_int]
    lib.pk_key_bits.restype = C.c_uint64
    lib.pk_key_bits.argtypes = [C.c_uint64, C.c_int]
    return lib


def device_pick(pk, values, fn, p, f64):
    """What k_pct_pick computes for one group: the values' order keys sorted ascending, then pct_pick."""
    raw = [(f64_bits(v) if f64 else v & ((1 << 64) - 1)) for v in values if v is not None]
    keys = sorted(pk.ok_encode(b, OE_F64 if f64 else OE_I64, 0) for b in raw)
    arr = (C.c_uint64 * len(keys))(*keys)
    out = pk.pk_pick(arr, len(keys), 1 if fn == "median" else 0, 0.0 if p is None else p, 1 if f64 else 0)
    if fn == "median" and not f64:
        out = out - (1 << 64) if out >> 63 else out
    return out


def nan_bits(v):
    return f64_bits(v)


EDGE_I64 = [[5], [7, -7], [I64_MAX], [I64_MAX, I64_MAX - 1], [I64_MIN, I64_MIN], [I64_MIN, I64_MAX], [I64_MAX, I64_MAX],
            [-3, 0], [1, 2, 3, 4, 5, 6], [2**53 + 1, 2**53 + 3], list(range(-50, 51, 7)), [I64_MIN, 0, I64_MAX]]
EDGE_F64 = [[1.5], [1.0, 2.0], [-0.0], [0.0, -0.0], [-0.0, 0.0, -0.0], [math.inf], [-math.inf, math.inf],
            [-math.inf, 1.0, 2.0, math.inf], [math.inf, math.inf], [-math.inf, -math.inf, 3.0],
            [nan(1), 1.0], [nan(3, True), 1.0, 2.0], [nan(7), nan(9, True)], [nan(2), nan(4), 5.0, -5.0], [nan(0x8000000000000 - 1)],
            [1e308, 1.7e308], [-1e308, 1e308], [0.1, 0.2, 0.3], [5e-324, -5e-324], [1.0, math.inf, nan(11)]]
PS = [0.0, 1.0, 0.5, 0.95, 0.99, 1 / 3]


@pytest.mark.parametrize("vec", range(len(EDGE_I64)))
def test_host_pick_int64_edges(pk, vec):
    vals = EDGE_I64[vec]
    assert device_pick(pk, vals, "median", None, False) == restate(vals, "median")
    for p in PS:
        assert device_pick(pk, vals, "percentile_cont", p, False) == restate(vals, "percentile_cont", p), p


@pytest.mark.parametrize("vec", range(len(EDGE_F64)))
def test_host_pick_float64_edges(pk, vec):
    vals = EDGE_F64[vec]
    assert device_pick(pk, vals, "median", None, True) == restate(vals, "median", None, True)
    for p in PS:
        assert device_pick(pk, vals, "percentile_cont", p, True) == restate(vals, "percentile_cont", p, True), p


def test_host_pick_random(pk):
    rng = np.random.default_rng(7)
    for _ in range(200):
        n = int(rng.integers(1, 40))
        f = [float(x) for x in rng.normal(0, 10, n)]
        i = [int(x) for x in rng.integers(-1000, 1000, n)]
        p = float(rng.random())
        assert device_pick(pk, f, "percentile_cont", p, True) == restate(f, "percentile_cont", p, True)
        assert device_pick(pk, i, "percentile_cont", p, False) == restate(i, "percentile_cont", p)
        assert device_pick(pk, f, "median", None, True) == restate(f, "median", None, True)
        assert device_pick(pk, i, "median", None, False) == restate(i, "median")


def test_key_decode_round_trip(pk):
    for v in [0, 1, -1, I64_MIN, I64_MAX, 12345]:
        assert pk.pk_key_bits(pk.ok_encode(v & ((1 << 64) - 1), OE_I64, 0), 0) == v & ((1 << 64) - 1)
    for x in [0.0, -0.0, 1.5, -2.5, math.inf, -math.inf, nan(1), nan(2, True), 5e-324]:
        assert pk.pk_key_bits(pk.ok_encode(f64_bits(x), OE_F64, 0), 1) == f64_bits(x)


# ---- the Python mirror and the SQL front ---------------------------------------------------------------------------
def test_abi_values_and_names():
    assert (L.PQ_AGG_MEDIAN, L.PQ_AGG_PERCENTILE_CONT) == (7, 8)
    assert median("latency_ms").name == "median(latency_ms)"
    assert [percentile_cont("x", p).name for p in (0, 0.5, 0.95, 1, 0.0001)] == [
        "percentile_cont(x, 0)", "percentile_cont(x, 0.5)", "percentile_cont(x, 0.95)", "percentile_cont(x, 1)",
        "percentile_cont(x, 1e-04)"]
    assert shortest_repr(1 / 3) == "0.3333333333333333" and shortest_repr(1e20) == "1e+20"


def test_sql_three_forms():
    q = Query("SELECT host, MEDIAN(latency_ms), percentile_cont(latency_ms, 0.99) AS p99, "
              "PERCENTILE_CONT(0.5) WITHIN GROUP (ORDER BY cpu ASC) FROM logs GROUP BY host ORDER BY 3 DESC LIMIT 10")
    assert q.select == [("col", "host", None), ("agg", Agg("median", "latency_ms"), None),
                        ("agg", Agg("percentile_cont", "latency_ms", 0.99), "p99"), ("agg", Agg("percentile_cont", "cpu", 0.5), None)]
    assert q.order_by == [(("pos", 3), "desc", None)] and q.limit == 10
    q = Query("SELECT status, median(duration_s) FROM logs GROUP BY status ORDER BY median(duration_s) DESC")
    assert q.order_by == [(("agg", Agg("median", "duration_s")), "desc", None)]
    q = Query("SELECT percentile_cont(0.95) within group (order by latency_ms) FROM logs")
    assert q.select == [("agg", Agg("percentile_cont", "latency_ms", 0.95), None)]


def test_sql_words_stay_identifiers():
    q = Query("SELECT median, within FROM logs WHERE median > 3 ORDER BY median LIMIT 5")
    assert q.select == [("col", "median", None), ("col", "within", None)]
    assert q.order_by == [(("name", "median"), "asc", None)]
    q = Query("SELECT percentile_cont, COUNT(*) FROM logs GROUP BY percentile_cont")
    assert q.group_by == ["percentile_cont"]


@pytest.mark.parametrize("sql", [
    "SELECT approx_percentile_cont(latency_ms, 0.9) FROM logs",
    "SELECT APPROX_MEDIAN(latency_ms) FROM logs",
    "SELECT approx_percentile_cont(0.9) WITHIN GROUP (ORDER BY latency_ms) FROM logs",
    "SELECT percentile_cont(0.9) WITHIN GROUP (ORDER BY latency_ms DESC) FROM logs",
])
def test_sql_refusals(sql):
    with pytest.raises(QueryError) as e:
        Query(sql)
    assert e.value.code == L.PQ_ERR_UNSUPPORTED
