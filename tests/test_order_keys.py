"""CPU tests of the ORDER BY key functions (csrc/order_keys.cuh) through the test-only harness
tools/liborder_keys_host.so: encode -> value ranges -> pack plan -> packed words, the sequence k_order_encode and
k_order_pack run on the device.  Sorting rows by their packed words (ties by row index) must equal Python's stable sort
under the stated value order: Int64 signed, Float64 by IEEE totalOrder, Utf8 bytewise with a prefix first, Boolean
false < true, NULLs first or last as asked in either direction."""
import ctypes as C
import itertools
import math
import os
import struct

import numpy as np
import pytest

OE_I64, OE_F64, OE_RAW = 0, 1, 2
I64_MIN, I64_MAX = -(1 << 63), (1 << 63) - 1


@pytest.fixture(scope="module")
def ok(built):
    lib = C.CDLL(os.path.join(built, "tools", "liborder_keys_host.so"))
    lib.ok_encode.restype = C.c_uint64
    lib.ok_encode.argtypes = [C.c_uint64, C.c_uint32, C.c_int]
    lib.ok_pack.restype = C.c_int32
    lib.ok_max_words.restype = C.c_uint32
    return lib


def f64_bits(x: float) -> int:
    return struct.unpack("<Q", struct.pack("<d", x))[0]


def nan(payload: int, neg: bool = False) -> float:
    return struct.unpack("<d", struct.pack("<Q", (1 << 63 if neg else 0) | 0x7FF0000000000000 | payload))[0]


def total_order(x: float) -> int:
    """IEEE 754 totalOrder as an integer, stated from the definition: the sign first, then the magnitude (exponent and
    significand, NaN payloads included), reversed for negative values."""
    b = f64_bits(x)
    mag = b & ((1 << 63) - 1)
    return -mag - 1 if b >> 63 else mag


def py_key(kind, v):
    if kind == "f64":
        return total_order(v)
    if kind == "str":
        return v.encode()
    return int(v)


def expected_order(terms, n):
    """Python's stable sort: per term (NULL rank, value) with the value order reversed for DESC."""
    ranked = []
    for kind, vals, desc, nulls_first in terms:
        distinct = sorted({py_key(kind, v) for v in vals if v is not None})
        rank = {k: i for i, k in enumerate(distinct)}
        col = []
        for v in vals:
            if v is None:
                col.append((0 if nulls_first else 2, 0))
            else:
                r = rank[py_key(kind, v)]
                col.append((1, -r if desc else r))
        ranked.append(col)
    return sorted(range(n), key=lambda i: tuple(c[i] for c in ranked))


def pack(ok, terms, n):
    """Raw bits per term as the device sees them (strings: their bytewise rank from ok_string_ranks)."""
    nt = len(terms)
    raw = np.zeros((nt, n), np.uint64)
    nulls = np.zeros((nt, n), np.uint8)
    enc = np.zeros(nt, np.uint8)
    desc = np.zeros(nt, np.uint8)
    nfirst = np.zeros(nt, np.uint8)
    for t, (kind, vals, d, nf) in enumerate(terms):
        desc[t], nfirst[t] = d, nf
        if kind == "str":
            dict_vals = sorted({v for v in vals if v is not None}, key=lambda s: hash(s))   # group ids are not in value order
            ranks = string_ranks(ok, dict_vals)
            gid = {v: i for i, v in enumerate(dict_vals)}
        for i, v in enumerate(vals):
            if v is None:
                nulls[t, i] = 1
                continue
            if kind == "i64":
                raw[t, i] = v & ((1 << 64) - 1)
            elif kind == "f64":
                raw[t, i] = f64_bits(v)
            elif kind == "str":
                raw[t, i] = ranks[gid[v]]
            else:
                raw[t, i] = int(v)
        enc[t] = {"i64": OE_I64, "f64": OE_F64}.get(kind, OE_RAW)
    mw = ok.ok_max_words()
    words = np.zeros((n, mw), np.uint64)
    plan = np.zeros(2 + 3 * nt, np.uint32)
    p = lambda a: a.ctypes.data_as(C.c_void_p)
    nw = ok.ok_pack(n, nt, p(raw), p(nulls), p(enc), p(desc), p(nfirst), p(words), p(plan))
    assert nw >= 0
    return words, plan, nw


def string_ranks(ok, vals):
    b = [v.encode() for v in vals]
    offs = np.zeros(len(b) + 1, np.uint32)
    offs[1:] = np.cumsum([len(x) for x in b])
    data = np.frombuffer(b"".join(b) or b"\0", np.uint8).copy()
    rank = np.zeros(max(len(b), 1), np.uint32)
    ok.ok_string_ranks(offs.ctypes.data_as(C.c_void_p), data.ctypes.data_as(C.c_void_p), C.c_uint32(len(b)), rank.ctypes.data_as(C.c_void_p))
    return [int(r) for r in rank[:len(b)]]


def check_plan(plan, nw, nterms):
    total = int(plan[1])
    assert int(plan[0]) == nw == (total + 63) // 64
    pos = 0
    for t in range(nterms):
        p, nb, vb = (int(x) for x in plan[2 + 3 * t: 5 + 3 * t])
        assert p == pos and nb in (0, 1) and 0 <= vb <= 64      # terms follow each other, MSB first, no overlap
        pos += nb + vb
    assert pos == total <= 64 * nw


def check(ok, terms):
    n = len(terms[0][1])
    words, plan, nw = pack(ok, terms, n)
    check_plan(plan, nw, len(terms))
    got = sorted(range(n), key=lambda i: (tuple(int(w) for w in words[i, :nw]), i))
    assert got == expected_order(terms, n)
    return nw


I64_EDGE = [I64_MIN, I64_MIN + 1, -1, 0, 1, I64_MAX - 1, I64_MAX, None]
F64_EDGE = [-math.inf, math.inf, -0.0, 0.0, 1.5, -1.5, 5e-324, -5e-324, 1.7976931348623157e308, nan(1), nan(0x8000000000000),
            nan(7, neg=True), nan(0x8000000000000, neg=True), None]
STR_EDGE = ["", "a", "ab", "abc", "b", "\xff", "ab\x00", "δ", "Z", None]


@pytest.mark.parametrize("desc,nulls_first", list(itertools.product([0, 1], [0, 1])))
def test_edge_values_every_direction(ok, desc, nulls_first):
    for kind, edge in (("i64", I64_EDGE), ("f64", F64_EDGE), ("str", STR_EDGE), ("bool", [False, True, None])):
        vals = edge * 3
        check(ok, [(kind, vals, desc, nulls_first)])


def test_full_i64_range_with_null_needs_65_bits(ok):
    vals = [I64_MIN, I64_MAX, None, 0]
    for d, nf in itertools.product([0, 1], [0, 1]):
        words, plan, nw = pack(ok, [("i64", vals, d, nf)], 4)
        assert int(plan[1]) == 65 and nw == 2           # 64 value bits + the NULL bit straddle two words
        check(ok, [("i64", vals, d, nf)])


def test_random_multi_term_multi_word(ok):
    rng = np.random.default_rng(5)
    n = 3000
    widths = []
    for trial in range(40):
        nt = int(rng.integers(1, 9))
        terms = []
        for _ in range(nt):
            kind = ["i64", "f64", "str", "bool"][int(rng.integers(0, 4))]
            nullp = [0.0, 0.1, 1.0][int(rng.integers(0, 3))] if trial % 5 else 0.05
            if kind == "i64":
                span = [3, 1000, 1 << 40, None][int(rng.integers(0, 4))]
                base = [int(x) for x in (rng.integers(-(1 << 62), 1 << 62, n) if span is None else rng.integers(-span, span, n))]
                pool = base + I64_EDGE[:-1] if span is None else base
                vals = [pool[int(rng.integers(0, len(pool)))] for _ in range(n)]
            elif kind == "f64":
                pool = [float(x) for x in rng.integers(-20, 20, 40)] + F64_EDGE[:-1]
                vals = [pool[int(rng.integers(0, len(pool)))] for _ in range(n)]
            elif kind == "str":
                pool = ["".join(chr(97 + int(c)) for c in rng.integers(0, 3, int(rng.integers(0, 5)))) for _ in range(60)]
                vals = [pool[int(rng.integers(0, len(pool)))] for _ in range(n)]
            else:
                vals = [bool(x) for x in rng.integers(0, 2, n)]
            vals = [None if rng.random() < nullp else v for v in vals]
            terms.append((kind, vals, int(rng.integers(0, 2)), int(rng.integers(0, 2))))
        widths.append(check(ok, terms))
    assert max(widths) >= 3 and min(widths) <= 1     # single-word and multi-word packs were both exercised


def test_count_desc_fits_one_word(ok):
    """The field statistics form: ORDER BY count(*) DESC over counts up to 10^8 takes 27 bits of one word."""
    rng = np.random.default_rng(9)
    vals = [int(x) for x in rng.integers(1, 10 ** 8, 500)] + [1, 10 ** 8 - 1]
    words, plan, nw = pack(ok, [("i64", vals, 1, 1)], len(vals))
    assert nw == 1 and int(plan[1]) == 27
    check(ok, [("i64", vals, 1, 1)])


def test_string_ranks_bytewise(ok):
    vals = ["b", "", "ab", "a", "abc", "\xff", "A", "δ", "a\x00"]
    ranks = string_ranks(ok, vals)
    want = sorted(range(len(vals)), key=lambda i: vals[i].encode())
    assert [vals[i] for i in sorted(range(len(vals)), key=lambda i: ranks[i])] == [vals[i] for i in want]


def test_encode_is_order_preserving(ok):
    i64 = sorted(v for v in I64_EDGE if v is not None)
    e = [ok.ok_encode(v & ((1 << 64) - 1), OE_I64, 0) for v in i64]
    assert e == sorted(e) and len(set(e)) == len(e)
    f = sorted((v for v in F64_EDGE if v is not None), key=total_order)
    e = [ok.ok_encode(f64_bits(v), OE_F64, 0) for v in f]
    assert e == sorted(e) and len(set(e)) == len(e)
    assert [ok.ok_encode(f64_bits(v), OE_F64, 1) for v in f] == sorted((ok.ok_encode(f64_bits(v), OE_F64, 1) for v in f), reverse=True)
