"""The membership set of PQ_OP_IN (in_set.cuh) on the CPU, through its host build tools/libin_set_host.so: the build and
the probe the kernels run, against a Python `set`.

* random numeric sets of 1 to 2^20 members, Int64 extremes, Float64 bit patterns (+-0, +-inf, several NaN payloads), and
  the one value that marks a free slot, as a member and not;
* byte strings: empty, embedded NUL, multi-byte UTF-8, longer than 4 KiB;
* members chosen so that they all hash to one slot (long probe runs that wrap around the table's end), for both kinds;
* the Python packing of `Expr.isin` into PQ_OP_IN literals."""
import ctypes as C
import os
import struct

import numpy as np
import pytest

from parseable_b200 import _lib as L
from parseable_b200.query import QueryError, _Desc, col

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
M64 = (1 << 64) - 1


def mix64(x):   # decode_core.cuh
    x ^= x >> 30
    x = (x * 0xbf58476d1ce4e5b9) & M64
    x ^= x >> 27
    x = (x * 0x94d049bb133111eb) & M64
    return x ^ (x >> 31)


def hash_bytes(b):   # decode_core.cuh
    h = 0xcbf29ce484222325 ^ ((len(b) * 0x9e3779b97f4a7c15) & M64)
    for c in b:
        h = ((h ^ c) * 0x100000001b3) & M64
    return mix64(h)


@pytest.fixture(scope="module")
def ins(built):
    lib = C.CDLL(os.path.join(ROOT, "tools", "libin_set_host.so"))
    lib.in_empty_value.restype = C.c_uint64
    lib.in_build_u64.restype = C.c_uint64
    lib.in_build_u64.argtypes = [C.c_void_p, C.c_uint64]
    lib.in_build_bytes.restype = C.c_uint64
    lib.in_build_bytes.argtypes = [C.c_void_p, C.c_void_p, C.c_uint64]
    lib.in_blob.argtypes = [C.c_void_p, C.c_uint64]
    lib.in_probe_u64.argtypes = [C.c_void_p, C.c_uint64, C.c_void_p]
    lib.in_probe_bytes.argtypes = [C.c_void_p, C.c_void_p, C.c_uint64, C.c_void_p]
    return lib


def _u64(vals):
    return np.ascontiguousarray(np.asarray(vals, dtype=np.uint64))


def probe_u64(ins, members, queries):
    m = _u64(members)
    size = ins.in_build_u64(m.ctypes.data, len(m))
    q = _u64(queries)
    out = np.zeros(len(q), np.uint8)
    ins.in_probe_u64(q.ctypes.data, len(q), out.ctypes.data)
    return out.astype(bool), size


def _packed(strs):
    off = np.zeros(len(strs) + 1, np.int64)
    off[1:] = np.cumsum([len(s) for s in strs])
    data = np.frombuffer(b"".join(strs) + b"\0", np.uint8).copy()
    return data, off


def probe_bytes(ins, members, queries):
    d, o = _packed(members)
    size = ins.in_build_bytes(d.ctypes.data, o.ctypes.data, len(members))
    qd, qo = _packed(queries)
    out = np.zeros(len(queries), np.uint8)
    ins.in_probe_bytes(qd.ctypes.data, qo.ctypes.data, len(queries), out.ctypes.data)
    return out.astype(bool), size


def f64_bits(xs):
    return [int(b) for b in np.asarray(xs, np.float64).view(np.uint64)]


@pytest.mark.parametrize("n", [1, 2, 3, 17, 1000, 65_537, 1 << 20])
def test_random_numeric_sets(ins, n):
    rng = np.random.default_rng(n)
    members = rng.integers(0, M64, size=n, dtype=np.uint64, endpoint=True)
    members[: n // 4] = members[n // 2: n // 2 + n // 4]        # duplicates
    others = rng.integers(0, M64, size=max(2 * n, 1000), dtype=np.uint64, endpoint=True)
    queries = np.concatenate([members, others])
    got, size = probe_u64(ins, members, queries)
    want = set(int(v) for v in members)
    assert np.array_equal(got, np.array([int(v) in want for v in queries]))
    cap = (size - 16) // 8
    assert cap & (cap - 1) == 0 and cap >= 2 * len(want)         # load factor at most 1/2


def test_numeric_extremes_and_float_bits(ins):
    i64 = [-(1 << 63), -(1 << 63) + 1, -1, 0, 1, (1 << 63) - 1, (1 << 63) - 512]
    members = [v & M64 for v in i64[::2]]
    floats = f64_bits([0.0, -0.0, np.inf, -np.inf, 1.5, -2.25, 5e-324])
    nans = [0x7FF8000000000000, 0xFFF8000000000000, 0x7FF8000000000001, 0x7FF0000000000001, 0xFFFFFFFFFFFFFFFF]
    members += floats[::2] + nans[::2]
    queries = [v & M64 for v in i64] + floats + nans
    got, _ = probe_u64(ins, members, queries)
    assert list(got) == [q in set(members) for q in queries]


@pytest.mark.parametrize("with_empty", [False, True])
def test_free_slot_value(ins, with_empty):
    empty = ins.in_empty_value()
    members = [1, 2, 3] + ([empty] if with_empty else [])
    got, _ = probe_u64(ins, members, [empty, 1, 4, empty ^ 1])
    assert list(got) == [with_empty, True, False, False]
    # the free-slot value alone: a set with no slot taken
    got, _ = probe_u64(ins, [empty], [empty, 0, 1])
    assert list(got) == [True, False, False]


def test_numeric_one_slot_runs(ins):
    # 40 members whose mix64 share the low bits of a 128-slot table's last slot: one run that wraps past the end
    target, members, x = 127, [], 0
    while len(members) < 40:
        if mix64(x) & 127 == target:
            members.append(x)
        x += 1
    queries = list(range(x)) + [x + k for k in range(100)]
    got, size = probe_u64(ins, members, queries)
    assert (size - 16) // 8 == 128
    assert list(got) == [q in set(members) for q in queries]


def test_random_byte_sets(ins):
    rng = np.random.default_rng(7)
    alphabet = [b"a", b"b", b"\0", "é".encode(), "日本".encode(), "😀".encode(), b"\xff"]
    def word():
        k = int(rng.integers(0, 12))
        return b"".join(alphabet[int(i)] for i in rng.integers(0, len(alphabet), size=k))
    members = [word() for _ in range(3000)] + [b"", b"\0", b"\0\0", b"x" * 5000, b"x" * 4999 + b"y", "ß".encode()]
    members += members[:100]
    queries = members + [word() for _ in range(5000)] + [b"x" * 5001, b"x" * 4999, "SS".encode(), b"\0\0\0"]
    got, _ = probe_bytes(ins, members, queries)
    want = set(members)
    assert list(got) == [q in want for q in queries]


def test_bytes_without_empty_string(ins):
    got, _ = probe_bytes(ins, [b"a", b"bb"], [b"", b"a", b"b", b"bb", b"\0"])
    assert list(got) == [False, True, False, True, False]


@pytest.mark.parametrize("n", [1, 2, 100_000])
def test_byte_sets_sizes(ins, n):
    members = [b"id-%08x" % (i * 2654435761 % (1 << 32)) for i in range(n)]
    queries = members[::3] + [b"id-%08x" % i for i in range(3 * n)]
    got, size = probe_bytes(ins, members, queries)
    want = set(members)
    assert list(got) == [q in want for q in queries]
    cap = (size - 16 - sum(len(m) for m in want)) // 16
    assert cap & (cap - 1) == 0 and cap >= 2 * len(want)


def test_bytes_one_slot_runs(ins):
    # strings whose hash_bytes share the low 6 bits: one probe run through a 64-slot table, and equal lengths, so the
    # probe has to tell them apart by hash and bytes
    members, k = [], 0
    while len(members) < 30:
        s = b"k%05d" % k
        if hash_bytes(s) & 63 == 5:
            members.append(s)
        k += 1
    queries = [b"k%05d" % i for i in range(k + 50)]
    got, _ = probe_bytes(ins, members, queries)
    assert list(got) == [q in set(members) for q in queries]


def _ops(e):
    d, ops = _Desc(), []
    d.compile_pred(e, ops)
    _ops.keep = d   # the packed elements live as long as the descriptor
    return ops


def _raw(op):
    """The packed elements of a PQ_OP_IN (lit.str is not NUL-terminated)."""
    p = C.c_void_p.from_buffer(op.lit, L.PqLiteral.str.offset).value
    return C.string_at(p, op.lit.str_len)


def test_isin_packing():
    ops = _ops(col("a").isin([3, -1, 3]))
    assert len(ops) == 1 and ops[0].kind == L.PQ_OP_IN and ops[0].flags == 0
    lit = ops[0].lit
    assert (lit.type, lit.i64, lit.str_len) == (L.PQ_T_I64, 3, 24)
    assert struct.unpack("<3q", _raw(ops[0])) == (3, -1, 3)
    ops = _ops(col("s").isin(["", "é", None], negated=True))
    lit = ops[0].lit
    assert ops[0].flags == L.PQ_IN_NEGATED | L.PQ_IN_HAS_NULL and (lit.type, lit.i64) == (L.PQ_T_UTF8, 2)
    assert _raw(ops[0]) == struct.pack("<I", 0) + struct.pack("<I", 2) + "é".encode()
    ops = _ops(col("f").isin([1.5, -0.0]))
    assert struct.unpack("<2d", _raw(ops[0])) == (1.5, -0.0)
    ops = _ops(col("x").isin([None]))
    assert ops[0].flags == L.PQ_IN_HAS_NULL and ops[0].lit.i64 == 0
    # mixed literal types: one IN per type, OR'd, and NOT over the whole
    ops = _ops(col("x").isin([1, "a", 2.5, None], negated=True))
    assert [o.kind for o in ops] == [L.PQ_OP_IN, L.PQ_OP_IN, L.PQ_OP_OR, L.PQ_OP_IN, L.PQ_OP_OR, L.PQ_OP_NOT]
    assert [o.flags for o in ops if o.kind == L.PQ_OP_IN] == [L.PQ_IN_HAS_NULL, 0, 0]
    with pytest.raises(QueryError):
        _ops(col("x").isin([]))
    with pytest.raises(QueryError):
        _ops(col("x").isin([1 << 63]))
