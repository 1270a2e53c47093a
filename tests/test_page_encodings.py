"""The device decoders that build the flat store, on hand-built Parquet pages in the stream shapes the format allows and
pyarrow's writer does not emit.

pyarrow writes DELTA_BINARY_PACKED as blocks of 128 values in 4 miniblocks, groups hybrid runs its own way and never
writes PLAIN_DICTIONARY data pages; other writers (the Rust `parquet` crate, parquet-mr) do.  `parquet_forge` writes
pages from explicit plans: dictionary indices at bit widths 0 .. 32 (wider than the dictionary needs too) with RLE runs of
1, page-long RLE runs, bit-packed runs with 1- and 2-byte headers, a bit-packed run longer than the 4 KB walker tile,
more than 96 runs in one tile and run headers / RLE values that straddle the tile end; definition levels as bit-packed
groups padded with 1s or 0s; RLE Booleans; DELTA_BINARY_PACKED in eight block geometries (up to 64 miniblocks) with
widths 0 .. 64, extreme min deltas and wrapping sums; DELTA_(LENGTH_)BYTE_ARRAY over those length streams; PLAIN values
at every byte phase; chunks with and without statistics, and dictionary pages without `dictionary_page_offset`.  Each
family is written twice: uncompressed, and under ZSTD (v2 pages with `is_compressed` true and false).

CPU: pyarrow reads every file back to the source values (floats by bit pattern), the Python reference decoders read the
same values out of the page bytes and the run layouts each case promises, `pq_file_describe` finds the pages as built,
and the k_scan walkers of the CPU harness decode every stream within their limits and refuse the rest.

GPU, over a resident table and a file list: projections of every column with __row_id (default batches and 97 rows)
value for value, filters and GROUP BY against numpy, no k_scan launch (PQB_VERBOSE=1), the flat store's count of pages
with NULLs, and the same filters on k_scan alone (PQB_FLAT_SCAN=0): the reference answer or a clean refusal."""
import ctypes as C
import datetime as dt
import json
import os
import re

import numpy as np
import pyarrow as pa
import pyarrow.parquet as pq
import pytest

import parquet_forge as F
from parquet_forge import Chunk, Column, DeltaPlan, Page
from parseable_b200 import _lib as L
from parseable_b200.query import DeviceTable, QueryError, StandardTableProvider, col, count, count_star, max_, min_, sum_
from test_project_paths import assert_same as _assert_same, check_batches

SEED = 20261019
I64_MIN, I64_MAX = -(1 << 63), (1 << 63) - 1
I32_MIN, I32_MAX = -(1 << 31), (1 << 31) - 1
WIDTHS = [0, 1, 2, 3, 5, 8, 9, 13, 16, 17, 24, 31, 32]
DICT_N = {0: 1, 1: 2, 2: 4, 3: 8, 5: 32, 8: 256, 9: 512, 13: 8192, 16: 65536, 17: 5000, 24: 3000, 31: 700, 32: 300}
GEOMS = [(128, 4), (128, 1), (128, 2), (256, 8), (512, 16), (1024, 32), (4096, 8), (2048, 64)]
CODECS = ("NONE", "ZSTD")
EPOCH = dt.date(1970, 1, 1)
KIND_CYCLE = ["i64", "str", "f64", "ts", "date"]
SWEEP_W = (8, 13, 24)    # widths of the tile-end sweep: 1-, 2- and 3-byte RLE values


# ---- value pools -------------------------------------------------------------------------------------------------------
def _dictionary(kind, n, rng, tag):
    if kind == "str":
        return [f"{tag}-{i}".encode() for i in range(n)]
    if kind == "f64":
        bits = [int(x) for x in rng.integers(0, 1 << 64, n, dtype=np.uint64)]
        special = [0x8000000000000000, 0x7FF8000000000001, 0xFFF00000DEADBEEF, 0x7FF0000000000000]
        return [b for b in (special + bits)[:n]] if n > 1 else [0x8000000000000000]
    if kind == "date":
        return [int(x) for x in rng.choice(np.arange(-400_000, 400_000), n, replace=False)]
    lo, hi = (-(1 << 62), 1 << 62) if kind == "i64" else (-2_200_000_000_000, 4_000_000_000_000)
    v = list(dict.fromkeys(int(x) for x in rng.integers(lo, hi, n + 16)))[:n]
    if kind == "i64" and n > 2:
        v[0], v[1] = I64_MIN, I64_MAX
    return v


def _valid(n, rng, rate):
    return list(rng.random(n) >= rate) if rate else [True] * n


def _rows(idx, valid, dictionary):
    it = iter(idx)
    return [dictionary[next(it)] if v else None for v in valid]


class Builder:
    """Pages of one column filled up to a row group's row count: `gen` proposes pages; the last page of a chunk takes
    whatever rows are left."""

    def __init__(self, rng):
        self.rng = rng

    def chunks(self, rg_rows, gen, tail, **kw):
        out = []
        for rows in rg_rows:
            pages, left = [], rows
            while left:
                pg = gen(len(pages), left)
                if pg is None or len(pg.values) > left:
                    pg = tail(left)
                pages.append(pg)
                left -= len(pg.values)
            out.append(Chunk(pages=pages, **{k: (v(len(out)) if callable(v) else v) for k, v in kw.items()}))
        return out


# ---- family: dictionary indices ----------------------------------------------------------------------------------------
def _sweep_prefix(target, bw, vals):
    """Runs whose bytes add up to `target`: bit-packed runs of 63 groups, then RLE runs with 1- and 2-byte headers."""
    vb = (bw + 7) // 8
    runs, size = [], 0
    while target - size > 64 * bw + 40:
        runs.append(("bp", [int(x) for x in vals(504)], 63))
        size += 1 + 63 * bw
    rest = target - size
    b = next(b for b in range(vb + 1) if (rest - b * (2 + vb)) >= 0 and (rest - b * (2 + vb)) % (1 + vb) == 0)
    runs += [("rle", int(vals(1)[0]), 70)] * b
    runs += [("rle", int(vals(1)[0]), 1)] * ((rest - b * (2 + vb)) // (1 + vb))
    assert len(F.encode_hybrid(runs, bw)) == target
    return runs


def family_hybrid(rng):
    rg_rows = [100_000, 90_000]
    b = Builder(rng)
    cols = []
    v = Column("v", "i64", required=True)
    v.chunks = b.chunks(rg_rows, lambda i, left: F.plain_page("i64", [int(x) for x in rng.integers(-1000, 1000, min(left, 7001))]),
                        lambda left: F.plain_page("i64", [int(x) for x in rng.integers(-1000, 1000, left)]), stats=True)
    cols.append(v)
    for wi, w in enumerate(WIDTHS):
        kind = KIND_CYCLE[wi % len(KIND_CYCLE)]
        n = DICT_N[w]
        dct = _dictionary(kind, n, rng, f"w{w}")
        mx = (1 << w) - 1

        def page(i, left, w=w, n=n, dct=dct, mx=mx):
            style = i % 5
            rows = int(min(left, [3001, 1000, 777, 2049, 96][style]))
            valid = _valid(rows, rng, 0.1 if style in (0, 2, 3) else 0)
            nn = sum(valid)
            if style == 0:    # mixed runs, bit-packed runs with 1- and 2-byte headers
                idx = [int(x) for x in np.repeat(rng.integers(0, n, nn), rng.integers(1, 12, nn))[:nn]]
                runs = F.runs_for(idx, w, rng, max_bp_groups=100)
            elif style == 1:  # one RLE run over the whole page
                idx = [int(rng.integers(0, n))] * nn
                runs = [("rle", idx[0], nn)]
            elif style == 2:  # RLE runs of 1
                idx = [int(x) for x in rng.integers(0, n, nn)]
                runs = [("rle", x, 1) for x in idx]
            elif style == 3:  # bit-packed, the last group padded with 1 bits
                idx = [int(x) for x in rng.integers(0, n, nn)]
                runs = [("bp", idx, (nn + 7) // 8, mx)] if nn else []
            else:             # 2-byte RLE headers split by 1-group bit-packed runs
                idx = [int(x) for x in rng.integers(0, n, nn)]
                runs, k = [], 0
                while k < nn:
                    take = min(nn - k, 8)
                    runs.append(("bp", idx[k:k + take], 1)) if k % 16 == 0 else runs.append(("rle", idx[k], take))
                    if runs[-1][0] == "rle":
                        idx[k:k + take] = [idx[k]] * take
                    k += take
            return F.dict_page(_rows(idx, valid, dct), dct, runs, w, v2=i % 2 == 1, compressed=i % 4 != 1)

        c = Column(f"h{w}", kind)
        c.chunks = b.chunks(rg_rows, page, lambda left, w=w, n=n, dct=dct: F.dict_page(
            [dct[0]] * left, dct, [("rle", 0, left)], w), dictionary=dct, stats=lambda g: g == 0,
            dict_offset_field=lambda g, w=w: not (w in (3, 17) and g == 1))
        cols.append(c)

    # a bit-packed run longer than the 4 KB tile: width 32, 200 groups
    dct = _dictionary("i64", DICT_N[32], rng, "t")

    def tile_page(i, left):
        if i % 2:
            return None
        idx = [int(x) for x in rng.integers(0, len(dct), 1600)]
        tail = [int(x) for x in rng.integers(0, len(dct), 400)]
        return F.dict_page(_rows(idx + tail, [True] * 2000, dct), dct, [("bp", idx, 200)] + [("rle", x, 1) for x in tail], 32)
    c = Column("tile32", "i64", required=True)
    c.chunks = b.chunks(rg_rows, tile_page, lambda left: F.dict_page([dct[1]] * left, dct, [("rle", 1, left)], 32), dictionary=dct)
    cols.append(c)

    # more than 96 runs inside one tile: RLE runs of 1 at width 1 (2 bytes each), with NULLs
    dct1 = [b"no", b"yes"]

    def runs1(i, left):
        rows = min(left, 5000)
        valid = _valid(rows, rng, 0.05 if i % 2 else 0)
        idx = [int(x) for x in rng.integers(0, 2, sum(valid))]
        return F.dict_page(_rows(idx, valid, dct1), dct1, [("rle", x, 1) for x in idx], 1, v2=i % 3 == 0)
    c = Column("runs1", "str")
    c.chunks = b.chunks(rg_rows, runs1, lambda left: F.dict_page([b"no"] * left, dct1, [("rle", 0, left)], 1), dictionary=dct1)
    cols.append(c)

    # a run header / RLE value at stream bytes 4064 .. 4112, widths 8, 13 and 24 in one chunk
    dct8 = _dictionary("i64", 256, rng, "s")
    targets = [(t, SWEEP_W[t % 3]) for t in range(4064, 4113)]

    def sweep(i, left):
        if not targets:
            return None
        t, w = targets.pop(0)
        vals = lambda k: rng.integers(0, 256, k)  # noqa: E731
        runs = _sweep_prefix(t, w, vals)
        runs += [("rle", int(vals(1)[0]), 300), ("bp", [int(x) for x in vals(20)], 3)] if t % 2 else \
                [("bp", [int(x) for x in vals(32)], 4), ("rle", int(vals(1)[0]), 300)]
        idx = []
        for r in runs:
            idx += [r[1]] * r[2] if r[0] == "rle" else list(r[1])
        if len(idx) > left:
            targets.insert(0, (t, w))
            return None
        return F.dict_page(_rows(idx, [True] * len(idx), dct8), dct8, runs, w, plan=("sweep", w, t))
    c = Column("sweep", "i64", required=True)
    c.chunks = b.chunks(rg_rows, sweep, lambda left: F.dict_page([dct8[5]] * left, dct8, [("rle", 5, left)], 13), dictionary=dct8)
    assert not targets
    cols.append(c)

    # PLAIN_DICTIONARY on the dictionary page and the data pages, widths changing from page to page
    dctp = _dictionary("str", 8, rng, "pd")

    def pdict(i, left):
        w = (3, 5, 9, 4)[i % 4]
        rows = min(left, 1234)
        valid = _valid(rows, rng, 0.2)
        idx = [int(x) for x in rng.integers(0, 8, sum(valid))]
        return F.dict_page(_rows(idx, valid, dctp), dctp, F.runs_for(idx, w, rng), w, enc=F.PLAIN_DICTIONARY, v2=i % 2 == 0)
    c = Column("pdict", "str")
    c.chunks = b.chunks(rg_rows, pdict, lambda left: F.dict_page([dctp[2]] * left, dctp, [("rle", 2, left)], 3, enc=F.PLAIN_DICTIONARY),
                        dictionary=dctp, dict_enc=F.PLAIN_DICTIONARY, dict_offset_field=lambda g: g == 0)
    cols.append(c)
    return cols


# ---- family: definition levels and Booleans ----------------------------------------------------------------------------
LEVEL_STYLES = ["bp_pad1", "bp_pad0", "last_null", "all_null", "no_null_bp", "no_null_bp_pad1", "mixed"]
LEVEL_ROWS = [1, 7, 8, 31, 33, 97, 1000, 2049, 4103, 40]


def _level_page(kind, i, left, rng, make):
    style = LEVEL_STYLES[i % len(LEVEL_STYLES)]
    rows = min(left, LEVEL_ROWS[(i // len(LEVEL_STYLES) + i) % len(LEVEL_ROWS)])
    if style in ("bp_pad1", "bp_pad0", "mixed"):
        valid = _valid(rows, rng, 0.3)
    elif style == "last_null":
        valid = [True] * rows
        for r in range(7, rows, 8 * 5):
            valid[r] = False
        valid[rows - 1] = False
    elif style == "all_null":
        valid = [False] * rows
    else:
        valid = [True] * rows
    lv = [int(x) for x in valid]
    defs = None if style == "mixed" else [("bp", lv, (rows + 7) // 8, 0 if style in ("bp_pad0", "no_null_bp") else 1)]
    pg = make(valid)
    pg.defs, pg.v2, pg.compressed = defs, i % 2 == 1, i % 3 != 0
    pg.plan = ("levels", style)
    return pg


def family_levels(rng):
    rg_rows = [30_000, 21_111]
    b = Builder(rng)
    cols = []
    v = Column("v", "i64", required=True)
    v.chunks = b.chunks(rg_rows, lambda i, left: None, lambda left: F.plain_page("i64", [int(x) for x in rng.integers(-500, 500, left)]))
    cols.append(v)

    def plain_values(kind, n):
        if kind in ("i64", "ts"):
            return [int(x) for x in rng.integers(-(1 << 50), 1 << 50, n)]
        if kind == "f64":
            return [int(x) for x in rng.integers(0, 1 << 64, n, dtype=np.uint64)]
        if kind == "date":
            return [int(x) for x in rng.integers(I32_MIN, I32_MAX, n, endpoint=True)]
        if kind == "bool":
            return [bool(x) for x in rng.random(n) < 0.5]
        return [bytes(rng.integers(97, 123, int(k)).astype(np.uint8)) for k in rng.integers(0, 20, n)]

    def fill(valid, vals):
        it = iter(vals)
        return [next(it) if x else None for x in valid]

    for kind in ("i64", "f64", "str", "bool", "date", "ts"):
        def make(valid, kind=kind):
            return F.plain_page(kind, fill(valid, plain_values(kind, sum(valid))))
        c = Column(f"l_{kind}", kind)
        c.chunks = b.chunks(rg_rows, lambda i, left, kind=kind, make=make: _level_page(kind, i, left, rng, make),
                            lambda left, make=make: make([True] * left), stats=lambda g: g == 1)
        cols.append(c)

    def rle_bool(valid):
        vals = [int(x) for x in rng.random(sum(valid)) < 0.4]
        pg = Page(values=fill(valid, [bool(x) for x in vals]), enc=F.RLE, body=F.encode_hybrid(F.runs_for(vals, 1, rng, rle_min=5), 1))
        return pg
    c = Column("l_rlebool", "bool")
    c.chunks = b.chunks(rg_rows, lambda i, left: _level_page("bool", i, left, rng, rle_bool), lambda left: rle_bool([True] * left))
    cols.append(c)

    dct = _dictionary("i64", 20, rng, "ld")

    def dict_make(valid):
        idx = [int(x) for x in rng.integers(0, 20, sum(valid))]
        return F.dict_page(_rows(idx, valid, dct), dct, F.runs_for(idx, 5, rng), 5)
    c = Column("l_dict", "i64")
    c.chunks = b.chunks(rg_rows, lambda i, left: _level_page("i64", i, left, rng, dict_make), lambda left: dict_make([True] * left),
                        dictionary=dct)
    cols.append(c)
    return cols


# ---- family: DELTA_BINARY_PACKED ---------------------------------------------------------------------------------------
def _delta_cases(bits):
    """(plan, count) of every page: each geometry at value counts 1, 31, 32, 33, a miniblock +- 1 and a block +- 1, the
    widths and min deltas the format allows, and junk in the unused widths of the last block."""
    w_all = [0, 1, 31, 32, 33, 63, 64] if bits == 64 else [0, 1, 31, 32]
    md_all = [0, -1, I64_MIN, I64_MAX] if bits == 64 else [0, -1, I32_MIN, I32_MAX]
    out = []
    for gi, (bs, nm) in enumerate(GEOMS):
        vpm = bs // nm
        for ci, n in enumerate(sorted({1, 31, 32, 33, vpm - 1, vpm + 1, bs - 1, bs + 1, 3 * bs + vpm + 5})):
            k = gi * 16 + ci
            plan = DeltaPlan(bs, nm, widths=lambda b, m, k=k: w_all[(k + b * 3 + m) % len(w_all)],
                             min_delta=lambda b, k=k: md_all[(k + b) % len(md_all)], junk=(0, 0xFF, 0x41, 7)[k % 4])
            out.append((plan, n))
    return out


def family_delta(rng):
    b = Builder(rng)
    cols = []
    specs = [("d_i64", "i64", True, 64, 0.0), ("d_i64n", "i64", False, 64, 0.15), ("d_ts", "ts", False, 64, 0.1),
             ("d_date", "date", False, 32, 0.1), ("d_daten", "date", True, 32, 0.0)]
    cases = {64: _delta_cases(64), 32: _delta_cases(32)}
    rows_per = [int(sum(n for _, n in cases[64]) * 1.3) + 5000]
    rg_rows = [rows_per[0] // 2, rows_per[0] - rows_per[0] // 2]
    v = Column("v", "i64", required=True)
    v.chunks = b.chunks(rg_rows, lambda i, left: None, lambda left: F.plain_page("i64", [int(x) for x in rng.integers(-99, 99, left)]))
    cols.append(v)
    for name, kind, req, bits, rate in specs:
        todo = list(cases[bits])

        def page(i, left, todo=todo, kind=kind, req=req, bits=bits, rate=rate):
            if not todo:
                return None
            plan, n = todo[0]
            valid = [True] * n if req or i % 3 == 0 else None
            if valid is None:   # NULLs between the values: the page holds more rows than values
                valid = [True] * n
                for _ in range(max(1, int(n * rate))):
                    valid.insert(int(rng.integers(0, len(valid) + 1)), False)
            if len(valid) > left:
                return None
            todo.pop(0)
            first = {0: None, 1: I64_MAX if bits == 64 else I32_MAX, 2: I64_MIN if bits == 64 else I32_MIN}[i % 3]
            vals, body = F.delta_stream(n, plan, rng, bits, first)
            it = iter(vals)
            return Page(values=[next(it) if x else None for x in valid], enc=F.DELTA_BINARY_PACKED, body=body, v2=i % 2 == 1,
                        compressed=i % 4 != 3, plan=("delta", plan.block, plan.minis, n))

        def tail(left, bits=bits):
            vals, body = F.delta_stream(left, DeltaPlan(128, 4), rng, bits)
            return Page(values=vals, enc=F.DELTA_BINARY_PACKED, body=body)
        c = Column(name, kind, required=req)
        c.chunks = b.chunks(rg_rows, page, tail, stats=lambda g: g == 0)
        assert not todo, name
        cols.append(c)
    return cols


# ---- family: DELTA_LENGTH_BYTE_ARRAY / DELTA_BYTE_ARRAY ---------------------------------------------------------------
def _strings(rng, n, style):
    if style == "empty":
        return [b""] * n
    if style == "repeat":   # prefix = the whole previous value
        base = b"same-value"
        return [base + (b"x" * int(k)) for k in np.cumsum(rng.integers(0, 2, n))]
    if style == "long32":
        return sorted(b"tenant/" + b"p" * 40 + b"/" + bytes(rng.integers(97, 100, int(k)).astype(np.uint8)) for k in rng.integers(0, 6, n))
    if style == "long4k":
        head = b"L" * 4500
        return [head + bytes(rng.integers(97, 99, int(k)).astype(np.uint8)) for k in rng.integers(0, 4, n)]
    return [bytes(rng.integers(97, 123, int(k)).astype(np.uint8)) for k in rng.integers(0, 30, n)]


def family_dba(rng):
    rg_rows = [12_000]
    b = Builder(rng)
    cols = []
    v = Column("v", "i64", required=True)
    v.chunks = b.chunks(rg_rows, lambda i, left: None, lambda left: F.plain_page("i64", [int(x) for x in rng.integers(-9, 9, left)]))
    cols.append(v)
    styles = ["random", "empty", "repeat", "long32", "long4k", "allnull"]
    for name, enc, req in (("s_dlba", F.DELTA_LENGTH_BYTE_ARRAY, False), ("s_dba", F.DELTA_BYTE_ARRAY, False),
                           ("s_dbar", F.DELTA_BYTE_ARRAY, True)):
        def page(i, left, enc=enc, req=req):
            bs, nm = GEOMS[i % len(GEOMS)]
            style = styles[i % len(styles)] if not (req and styles[i % len(styles)] == "allnull") else "random"
            n = min(left, [1, 31, 33, 97, 300, 1000, 61][i % 7] if style != "long4k" else 40)
            valid = [False] * n if style == "allnull" else _valid(n, rng, 0 if req else 0.1)
            strs = _strings(rng, sum(valid), style)
            plan = DeltaPlan(bs, nm, junk=(0, 0x99)[i % 2])
            body = (F.encode_dlba if enc == F.DELTA_LENGTH_BYTE_ARRAY else F.encode_dba)(strs, plan)
            it = iter(strs)
            return Page(values=[next(it) if x else None for x in valid], enc=enc, body=body, v2=style == "allnull" or i % 2 == 1,
                        compressed=i % 3 != 0, plan=("dba", bs, nm, style))

        def tail(left, enc=enc):
            strs = _strings(rng, left, "random")
            return Page(values=strs, enc=enc, body=(F.encode_dlba if enc == F.DELTA_LENGTH_BYTE_ARRAY else F.encode_dba)(strs, DeltaPlan()))
        c = Column(name, "str", required=req)
        c.chunks = b.chunks(rg_rows, lambda i, left, page=page: page(i, left) if i < 60 else None, tail)
        cols.append(c)
    return cols


def family_dba_empty(rng):
    """All-NULL DELTA_(LENGTH_)BYTE_ARRAY pages that carry no value bytes at all (v1 and v2) between pages with values.
    pyarrow's reader refuses such a page, so this file is checked against the Python reference decoders only."""
    rg_rows = [5_000]
    b = Builder(rng)
    cols = []
    v = Column("v", "i64", required=True)
    v.chunks = b.chunks(rg_rows, lambda i, left: None, lambda left: F.plain_page("i64", [int(x) for x in rng.integers(-9, 9, left)]))
    cols.append(v)
    for name, enc in (("e_dlba", F.DELTA_LENGTH_BYTE_ARRAY), ("e_dba", F.DELTA_BYTE_ARRAY)):
        encode = F.encode_dlba if enc == F.DELTA_LENGTH_BYTE_ARRAY else F.encode_dba

        def page(i, left, enc=enc, encode=encode):
            n = min(left, (97, 33, 250, 1)[i % 4])
            if i % 2 == 0:   # all NULL, no value bytes; v2 uncompressed (a codec would add a frame), or v1
                return Page(values=[None] * n, enc=enc, body=b"", v2=i % 4 == 0, compressed=False, plan=("dba_empty", i % 4 == 0))
            valid = _valid(n, rng, 0.2)
            strs = _strings(rng, sum(valid), "long32")
            it = iter(strs)
            return Page(values=[next(it) if x else None for x in valid], enc=enc, body=encode(strs, DeltaPlan(2048, 64)), v2=i % 3 == 0)
        c = Column(name, "str")
        c.chunks = b.chunks(rg_rows, page, lambda left, page=page: page(1, left))
        cols.append(c)
    return cols


# ---- family: PLAIN -----------------------------------------------------------------------------------------------------
def family_plain(rng):
    rg_rows = [20_000, 9_999]
    b = Builder(rng)
    cols = []
    v = Column("v", "i64", required=True)
    v.chunks = b.chunks(rg_rows, lambda i, left: None, lambda left: F.plain_page("i64", [int(x) for x in rng.integers(-9, 9, left)]))
    cols.append(v)

    # strings: a first value of 4070 .. 4105 bytes puts the next length prefix at every offset around the tile end
    def spage(i, left):
        n = min(left, 50)
        valid = _valid(n, rng, 0.1 if i % 2 else 0)
        valid[0] = valid[1] = True
        strs = [b"S" * (4070 + i % 36)] + [bytes(rng.integers(97, 123, int(k)).astype(np.uint8)) for k in rng.integers(0, 9, n)]
        strs[2] = b""
        if i % 7 == 0:
            strs[3] = b"Z" * 9000
        it = iter(strs)
        return F.plain_page("str", [next(it) if x else None for x in valid], v2=i % 2 == 0)
    c = Column("p_str", "str")
    c.chunks = b.chunks(rg_rows, spage, lambda left: F.plain_page("str", [b"tail"] * left), stats=True)
    cols.append(c)

    for kind, gap in (("i64", 1), ("f64", 3), ("date", 6), ("ts", 13), ("i64", 0)):
        def page(i, left, kind=kind):
            n = min(left, 97 + (i * 37) % 500)
            valid = _valid(n, rng, 0.1 if i % 3 else 0)
            if kind == "f64":
                pool = [0x8000000000000000, 0x7FF8000000000001, 0xFFF00000DEADBEEF, 0x7FF0000000000000, 0, 1]
                vals = [pool[int(k)] if k < 6 else int(x) for k, x in zip(rng.integers(0, 20, n), rng.integers(0, 1 << 64, n, dtype=np.uint64))]
            elif kind == "date":
                vals = [int(x) for x in rng.integers(I32_MIN, I32_MAX, n, endpoint=True)]
            else:
                vals = [int(x) for x in rng.integers(I64_MIN, I64_MAX, n, endpoint=True)]
            it = iter(vals)
            return F.plain_page(kind, [next(it) if x else None for x in valid], v2=i % 2 == 1, compressed=i % 4 == 1)
        c = Column(f"p_{kind}{gap}", kind)
        c.chunks = b.chunks(rg_rows, page, lambda left, page=page: page(0, left), stats=lambda g, gap=gap: gap % 2 == 1,
                            gap=lambda g, gap=gap: gap + g)
        cols.append(c)

    def bpage(i, left):
        n = min(left, [1, 31, 32, 33, 100, 1000][i % 6])
        valid = _valid(n, rng, 0.3 if i % 2 else 0)
        vals = [bool(x) for x in rng.random(n) < 0.5]
        it = iter(vals)
        return F.plain_page("bool", [next(it) if x else None for x in valid], v2=i % 3 == 0)
    c = Column("p_bool", "bool")
    c.chunks = b.chunks(rg_rows, bpage, lambda left: F.plain_page("bool", [True] * left))
    cols.append(c)
    return cols


FAMILIES = {"hybrid": family_hybrid, "levels": family_levels, "delta": family_delta, "dba": family_dba, "plain": family_plain,
            "dba_empty": family_dba_empty}
PYARROW_REFUSES = {"dba_empty"}   # an all-NULL DELTA_(LENGTH_)BYTE_ARRAY page without value bytes


@pytest.fixture(scope="module")
def forged(tmp_path_factory):
    d = tmp_path_factory.mktemp("forged")
    out = {}
    for fi, (fam, make) in enumerate(FAMILIES.items()):
        cols = make(np.random.default_rng(SEED + fi))
        paths = {}
        for codec in CODECS:
            p = str(d / f"{fam}_{codec.lower()}.parquet")
            F.write_file(p, cols, codec)
            paths[codec] = p
        out[fam] = (cols, paths)
    return out


def _schema(cols):
    return pa.schema([(c.name, F.KINDS[c.kind][1]) for c in cols])


def _source(cols):
    return pa.table({c.name: F.to_arrow(c) for c in cols})


CASES = [(fam, codec) for fam in FAMILIES for codec in CODECS]


def assert_same(got, want, what):
    """By validity and by bits; Date32 as its int32 day counts."""
    if pa.types.is_date32(want.type):
        assert got.type == want.type, (what, got.type)
        got, want = got.cast(pa.int32()).cast(pa.int64()), want.cast(pa.int32()).cast(pa.int64())
    _assert_same(got, want, what)


# ---- CPU ---------------------------------------------------------------------------------------------------------------
def _describe(path):
    lib = L.load()
    f = L.PqFile(path=path.encode())
    n = lib.pq_file_describe(C.byref(f), None, 0)
    buf = C.create_string_buffer(n + 1)
    lib.pq_file_describe(C.byref(f), buf, n + 1)
    return json.loads(buf.value.decode())


def _pages(path):
    """(row group, column, page record, payload offset in the file) of every page, from the library's own page walk."""
    out = []
    for g, rgd in enumerate(_describe(path)["row_groups"]):
        for j, cc in enumerate(rgd["columns"]):
            dpo, dto = cc["dictionary_page_offset"], cc["data_page_offset"]
            off = dpo if 0 < dpo < dto else dto
            for p in cc["pages"]:
                start = off + p["header_len"]
                out.append((g, j, p, start))
                off = start + p["compressed_size"]
    return out


def test_total_size(forged):
    total = sum(os.path.getsize(p) for _, paths in forged.values() for p in paths.values())
    assert 10 << 20 < total < 200 << 20, total


@pytest.mark.parametrize("fam,codec", [c for c in CASES if c[0] not in PYARROW_REFUSES])
def test_pyarrow_reads_the_source(forged, fam, codec):
    """pyarrow's reader (an independent decoder) returns exactly the values the pages were built from."""
    cols, paths = forged[fam]
    got = pq.read_table(paths[codec])
    want = _source(cols)
    assert got.column_names == want.column_names
    for c in cols:
        assert_same(got[c.name], want[c.name], f"{fam} {codec} {c.name}")


@pytest.mark.parametrize("fam", FAMILIES)
def test_pages_as_built(forged, built, fam):
    """pq_file_describe finds the pages each case was built with (type, encoding, value count), and the Python
    reference decoders read every page's bytes back to its values and its promised shape: hybrid run layouts and bit
    widths, DELTA block geometries, PLAIN payloads at every byte phase."""
    cols, paths = forged[fam]
    raw = open(paths["NONE"], "rb").read()
    pages = _pages(paths["NONE"])
    shapes, phases, seen = set(), set(), {}
    for g, j, rec, start in pages:
        col_ = cols[j]
        ch = col_.chunks[g]
        if rec["type"] == F.DICTIONARY_PAGE:
            assert ch.dictionary is not None and rec["encoding"] == ch.dict_enc and rec["num_values"] == len(ch.dictionary)
            assert F.decode_plain(col_.kind, raw, len(ch.dictionary), start) == ch.dictionary
            continue
        k = seen[g, j] = seen.get((g, j), -1) + 1
        pg = ch.pages[k]
        assert rec["type"] == (F.DATA_PAGE_V2 if pg.v2 else F.DATA_PAGE) and rec["encoding"] == pg.enc
        assert rec["num_values"] == len(pg.values)
        valid = [x is not None for x in pg.values]
        pos = start
        if not col_.required:
            if pg.v2:
                dlen = len(F.encode_hybrid(pg.defs, 1)) if pg.defs is not None else None
                lv, runs, end = F.decode_hybrid(raw, 1, len(valid), pos)
                pos = end if dlen is None else pos + dlen
            else:
                dlen = int.from_bytes(raw[pos:pos + 4], "little")
                lv, runs, _ = F.decode_hybrid(raw, 1, len(valid), pos + 4)
                pos += 4 + dlen
            assert lv == [int(x) for x in valid]
            if pg.plan and pg.plan[0] == "levels":
                shapes.add(pg.plan)
                if pg.defs is not None:
                    assert runs == [("bp", 8 * ((len(valid) + 7) // 8))]
        nn = [x for x in pg.values if x is not None]
        phases.add((col_.kind, pos % 16))
        if pg.enc in (F.RLE_DICTIONARY, F.PLAIN_DICTIONARY):
            if not nn and pos >= start + rec["compressed_size"]:
                continue
            bw = raw[pos]
            assert bw == pg.bw
            idx, runs, _ = F.decode_hybrid(raw, bw, len(nn), pos + 1)
            assert [ch.dictionary[i] for i in idx] == nn
            if pg.plan[0] == "hybrid":
                assert runs == pg.plan[2], (col_.name, k)
                shapes.add(("width", bw))
                shapes.update(("run", kind, cnt == 1, cnt > 63 * 8 if kind == "bp" else cnt >= 64) for kind, cnt in runs)
                if runs and runs[0][0] == "bp" and runs[0][1] >= 1600 and bw == 32:
                    shapes.add("bp_longer_than_tile")
            else:
                shapes.add(pg.plan)
        elif pg.enc == F.RLE:
            n = int.from_bytes(raw[pos:pos + 4], "little")
            bits, _, end = F.decode_hybrid(raw, 1, len(nn), pos + 4)
            assert bits == [int(x) for x in nn] and end <= pos + 4 + n
            shapes.add(("rlebool", pg.v2, len(pg.values) % 32 != 0, len(nn) < len(pg.values)))
        elif pg.enc == F.DELTA_BINARY_PACKED:
            vals, geom, widths, _ = F.decode_delta(raw, pos, 32 if col_.kind == "date" else 64)
            assert vals == nn
            if pg.plan:
                assert geom == pg.plan[1:3]
                shapes.add(("delta", col_.kind, geom, len(nn) < len(pg.values)))
                shapes.update(("dwidth", w) for ws in widths for w in ws)
        elif pg.enc in (F.DELTA_LENGTH_BYTE_ARRAY, F.DELTA_BYTE_ARRAY):
            if nn or pos < start + rec["compressed_size"]:
                dec = F.decode_dlba if pg.enc == F.DELTA_LENGTH_BYTE_ARRAY else F.decode_dba
                assert dec(raw, pos) == nn
            if pg.plan and pg.plan[0] == "dba_empty":
                assert not nn and pos == start + rec["compressed_size"], (col_.name, k)   # no value bytes at all
                shapes.add(pg.plan)
            elif pg.plan:
                shapes.add(pg.plan)
        else:
            assert F.decode_plain(col_.kind, raw, len(nn), pos) == nn
    if fam == "hybrid":
        assert {("width", w) for w in WIDTHS} <= shapes, sorted(s for s in shapes if s[0] == "width")
        for s in [("run", "rle", True, False), ("run", "rle", False, True), ("run", "bp", False, True), ("run", "bp", False, False),
                  "bp_longer_than_tile"]:
            assert s in shapes, s
        assert {("sweep", SWEEP_W[t % 3], t) for t in range(4064, 4113)} <= shapes
    if fam == "levels":
        assert {("levels", s) for s in LEVEL_STYLES} <= shapes
        assert {("rlebool", v2, True, True) for v2 in (False, True)} <= shapes
    if fam == "delta":
        for kind in ("i64", "ts", "date"):
            assert {("delta", kind, gm, True) for gm in GEOMS} <= shapes, kind
        assert {("delta", "i64", gm, False) for gm in GEOMS} <= shapes
        assert {("dwidth", w) for w in (0, 1, 31, 32, 33, 63, 64)} <= shapes
    if fam == "dba":
        for style in ("random", "empty", "repeat", "long32", "long4k", "allnull"):
            assert any(s[0] == "dba" and s[3] == style for s in shapes), style
        assert {s[1:3] for s in shapes if s[0] == "dba"} == set(GEOMS)
    if fam == "dba_empty":
        assert {("dba_empty", True), ("dba_empty", False)} <= shapes
    if fam == "plain":
        for kind in ("i64", "f64", "date"):
            assert {p for k, p in phases if k == kind} == set(range(16)), kind


@pytest.mark.parametrize("fam", ["hybrid", "levels", "delta"])
def test_cpu_walkers(forged, built, fam):
    """k_scan's walkers in the CPU harness: every hybrid and DELTA stream within their limits decodes to the source
    values; a DELTA stream with more than 8 miniblocks per block is refused."""
    dc = C.CDLL(os.path.join(built, "tools", "libdecode_core_host.so"))
    dc.dc_decode_hybrid.restype = C.c_int64
    dc.dc_decode_delta.restype = C.c_int64
    cols, _ = forged[fam]
    n_h = n_d = n_refused = 0
    for c in cols:
        for ch in c.chunks:
            for pg in ch.pages:
                nn = [x for x in pg.values if x is not None]
                if pg.enc in (F.RLE_DICTIONARY, F.PLAIN_DICTIONARY) and nn and pg.bw:
                    out = np.zeros(len(nn), np.uint32)
                    slab = 2048
                    cap = ((slab * pg.bw // 8 + slab // 8 + 64 + 15) // 16) * 16
                    got = dc.dc_decode_hybrid(pg.body, C.c_uint64(len(pg.body)), pg.bw, len(nn), slab, cap, 64, out.ctypes.data_as(C.c_void_p))
                    assert got == len(nn), (c.name, got)
                    assert [ch.dictionary[i] for i in out] == nn, c.name
                    n_h += 1
                elif pg.enc == F.DELTA_BINARY_PACKED and nn and c.kind != "date":
                    out = np.zeros(len(nn), np.int64)
                    got = dc.dc_decode_delta(pg.body, C.c_uint64(len(pg.body)), len(nn), 2048, 8192 + 64, 80, out.ctypes.data_as(C.c_void_p))
                    if pg.plan and pg.plan[2] > 8:
                        assert got < 0, (c.name, pg.plan)
                        n_refused += 1
                    else:
                        assert got == len(nn), (c.name, pg.plan, got)
                        assert out.tolist() == nn, (c.name, pg.plan)
                        n_d += 1
    assert n_h > 50 if fam != "delta" else n_d > 50 and n_refused > 10


# ---- GPU ---------------------------------------------------------------------------------------------------------------
def _ints(arr: pa.Array) -> list:
    """Source values of a column as Python values comparable with the forge's (ints / f64 bits / bytes / bools)."""
    t = arr.type
    if pa.types.is_string(t):
        return arr.cast(pa.binary()).to_pylist()
    if pa.types.is_timestamp(t) or pa.types.is_date32(t):
        return arr.cast(pa.int64() if pa.types.is_timestamp(t) else pa.int32()).to_pylist()
    if pa.types.is_floating(t):
        bits = np.frombuffer(arr.buffers()[1], np.uint64, count=arr.offset + len(arr))[arr.offset:]
        return [int(b) if ok else None for b, ok in zip(bits, arr.is_valid().to_pylist())]
    return arr.to_pylist()


def _groups(cols):
    names = [c.name for c in cols]
    return [names[i:i + 10] for i in range(0, len(names), 10)]


def _lit(kind, v):
    return v.decode() if kind == "str" else v


def _filters(cols):
    """(name, expr, numpy mask) per column: IS NULL, IS NOT NULL, = an existing value, < the median (not Booleans).
    Timestamp literals are ms since the epoch, Date32 literals dates."""
    out = []
    for c in cols:
        vals = c.values()
        valid = np.array([x is not None for x in vals])
        out.append((f"{c.name} is null", col(c.name).is_null(), ~valid))
        out.append((f"{c.name} not null", col(c.name).is_not_null(), valid))
        nn = [x for x in vals if x is not None]
        if not nn or c.kind == "bool":
            continue
        if c.kind == "f64":   # in IEEE totalOrder (DataFusion's): -NaN below every value, +NaN above, -0.0 < 0.0
            b = np.array([0 if y is None else y for y in vals], np.uint64)
            key = np.where(b >> np.uint64(63) == 1, ~b, b | np.uint64(1 << 63))
            d = b.view(np.float64)
            fin = np.isfinite(d) & (d != 0) & valid
            if fin.any():
                x = float(d[fin][int(fin.sum()) // 3])
                out.append((f"{c.name} = x", col(c.name) == x, fin & (d == x)))
                m = float(np.median(d[fin]))
                km = np.array([m]).view(np.uint64)[0]
                km = ~km if km >> np.uint64(63) == 1 else km | np.uint64(1 << 63)
                out.append((f"{c.name} < m", col(c.name) < m, valid & (key < km)))
            continue
        if c.kind == "date":  # literals inside datetime.date's years
            lo, hi = (dt.date(1, 1, 1) - EPOCH).days, (dt.date(9999, 12, 31) - EPOCH).days
            days = [y for y in nn if lo <= y <= hi]
            if days:
                x = days[len(days) // 3]
                out.append((f"{c.name} = x", col(c.name) == EPOCH + dt.timedelta(days=x), np.array([y == x for y in vals])))
                m = sorted(days)[len(days) // 2]
                out.append((f"{c.name} < m", col(c.name) < EPOCH + dt.timedelta(days=m), np.array([y is not None and y < m for y in vals])))
            continue
        x = nn[len(nn) // 3]
        out.append((f"{c.name} = x", col(c.name) == _lit(c.kind, x), np.array([y == x for y in vals])))
        if c.kind in ("i64", "ts"):
            m = sorted(nn)[len(nn) // 2]
            out.append((f"{c.name} < m", col(c.name) < m, np.array([y is not None and y < m for y in vals])))
    return out


def _expected_null_pages(cols):
    return sum(1 for c in cols for ch in c.chunks for p in ch.pages if any(x is None for x in p.values))


@pytest.fixture(scope="module")
def gpu_tables(forged):
    out = {}
    yield out
    for t in out.values():
        t.close()


def _provider(gpu_tables, forged, fam, codec, source):
    cols, paths = forged[fam]
    schema = _schema(cols)
    if source == "files":
        return StandardTableProvider([paths[codec]], schema=schema)
    key = (fam, codec)
    if key not in gpu_tables:
        gpu_tables[key] = DeviceTable([paths[codec]], schema.names)
    return StandardTableProvider(gpu_tables[key], schema=schema)


def _assert_no_k_scan(capfd, what):
    err = capfd.readouterr().err
    assert "[pqb] k_scan:" not in err, (what, [ln for ln in err.splitlines() if "k_scan" in ln][:3])
    return err


@pytest.mark.gpu
@pytest.mark.parametrize("source", ["resident", "files"])
@pytest.mark.parametrize("fam,codec", CASES)
def test_gpu_project_filter_group(forged, gpu_tables, fam, codec, source, monkeypatch, capfd):
    """Every column projected with __row_id at the default batch size and at 97 rows, value for value; filters per
    column and GROUP BY over the dictionary columns against numpy; no k_scan launch anywhere."""
    cols, _ = forged[fam]
    monkeypatch.setenv("PQB_VERBOSE", "1")
    capfd.readouterr()
    prov = _provider(gpu_tables, forged, fam, codec, source)
    if source == "resident":
        err = capfd.readouterr().err
        m = re.search(r"\[pqb\] flat store: (\d+) of (\d+) pages \((\d+) with NULLs\)", err)
        assert m and int(m.group(3)) == _expected_null_pages(cols), (fam, codec, m and m.group(0), _expected_null_pages(cols))
    ref = _source(cols)
    n = ref.num_rows
    ids = np.arange(n)
    for bs in (0, 97):
        for cs in _groups(cols):
            res = prov.scan(projection=cs, row_ids=True, batch_size=bs)
            check_batches(res, bs)
            got = res.table()
            assert got.num_rows == n and got.column_names == cs + ["__row_id"], (fam, cs, got.num_rows)
            for c in cs:
                assert_same(got[c], ref[c], f"{fam} {codec} {source} {c} batch {bs}")
            assert np.array_equal(got["__row_id"].to_numpy(), ids)
    _assert_no_k_scan(capfd, f"{fam} {codec} {source} projections")
    for what, e, m in _filters(cols):
        assert prov.scan(filters=[e], count_only=True).metrics["rows_selected"] == int(m.sum()), (fam, codec, source, what)
        if "=" in what or "<" in what:
            res = prov.scan(filters=[e])
            got = np.concatenate([b.column(0).to_numpy() for b in res.batches]) if res.batches else np.zeros(0, np.int64)
            assert np.array_equal(got, np.flatnonzero(m)), (fam, codec, source, what)
    _assert_no_k_scan(capfd, f"{fam} {codec} {source} filters")
    v = np.array(cols[0].values(), np.int64)
    assert cols[0].name == "v"
    for c in cols:
        if c.chunks[0].dictionary is None or c.kind == "f64":
            continue
        keys = c.values()
        aggs = [count_star(), count(c.name), sum_("v"), min_("v"), max_("v")]
        if c.kind in ("i64", "str"):
            aggs += [min_(c.name), max_(c.name)]
        t = prov.aggregate([c.name], aggs).table()
        got = {}
        for row in t.to_pylist():
            k = row[c.name]
            k = k.encode() if isinstance(k, str) else k
            if c.kind in ("ts", "date") and k is not None:
                k = pa.scalar(k, F.KINDS[c.kind][1]).cast(pa.int64() if c.kind == "ts" else pa.int32()).as_py()
            got[k] = row
        code = {}
        codes = np.array([code.setdefault(x, len(code)) for x in keys], np.int64)
        ng = len(code)
        cnt, sm = np.bincount(codes, minlength=ng), np.bincount(codes, weights=v, minlength=ng).astype(np.int64)
        lo, hi = np.full(ng, I64_MAX), np.full(ng, I64_MIN)
        np.minimum.at(lo, codes, v)
        np.maximum.at(hi, codes, v)
        want = {k: (int(cnt[i]), int(sm[i]), int(lo[i]), int(hi[i])) for k, i in code.items()}
        assert set(got) == set(want), (fam, codec, source, c.name, len(got), len(want))
        for k, (cnt, s, lo, hi) in want.items():
            r = got[k]
            assert (r["count(*)"], r[f"count({c.name})"], r["sum(v)"], r["min(v)"], r["max(v)"]) == \
                (cnt, cnt if k is not None else 0, s, lo, hi), (fam, codec, source, c.name, k)
            if c.kind in ("i64", "str"):
                kk = k.decode() if isinstance(k, bytes) else k
                assert r[f"min({c.name})"] == kk and r[f"max({c.name})"] == kk, (c.name, k)
    _assert_no_k_scan(capfd, f"{fam} {codec} {source} group by")


def _plain_str_col(cols, what):
    """The string column without a dictionary (PLAIN or DELTA_(LENGTH_)BYTE_ARRAY pages) a filter reads, or None."""
    for c in cols:
        if what.split(" ")[0] == c.name and c.kind == "str" and c.chunks[0].dictionary is None:
            return c.name
    return None


@pytest.mark.gpu
@pytest.mark.parametrize("fam,codec", CASES)
def test_gpu_k_scan_walkers(forged, gpu_tables, fam, codec, monkeypatch):
    """The same filters with every item on k_scan (PQB_FLAT_SCAN=0): its own walkers over the same streams give the
    reference count or refuse the query cleanly; a wrong count is never an answer.  k_scan reads no string values out of
    pages without a dictionary: every filter over such a column is refused with PQ_ERR_UNSUPPORTED naming it."""
    cols, _ = forged[fam]
    prov = _provider(gpu_tables, forged, fam, codec, "resident")
    monkeypatch.setenv("PQB_FLAT_SCAN", "0")
    wrong, refused = [], 0
    for what, e, m in _filters(cols):
        plain = _plain_str_col(cols, what)
        try:
            got = prov.scan(filters=[e], count_only=True).metrics["rows_selected"]
        except QueryError as ex:
            assert ex.code in (L.PQ_ERR_UNSUPPORTED, L.PQ_ERR_CORRUPT), (what, ex)
            if plain:
                assert ex.code == L.PQ_ERR_UNSUPPORTED and f"'{plain}'" in ex.message, (what, ex)
                refused += 1
            continue
        assert plain is None, (fam, codec, what, "k_scan answered a filter over string pages without a dictionary", got)
        if got != int(m.sum()):
            wrong.append((what, got, int(m.sum())))
    assert not wrong, (fam, codec, wrong)
    assert refused == sum(_plain_str_col(cols, w) is not None for w, _, _ in _filters(cols))
    # the table still answers once the flat kernels are back
    monkeypatch.delenv("PQB_FLAT_SCAN")
    what, e, m = _filters(cols)[-1]
    assert prov.scan(filters=[e], count_only=True).metrics["rows_selected"] == int(m.sum()), (fam, codec, what)
