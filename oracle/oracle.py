"""TEST INFRASTRUCTURE ONLY — CPU oracle for the GPU query path.

Decodes Parquet with pyarrow (an independent implementation of the Parquet
spec; the reference's decoder is the un-vendored `parquet` crate 58.1.0) and
evaluates predicates / GROUP BY with the scalar C restatement in oracle.c.
Only tests/, __graft_entry__.smoke() and bench.py (cpu_baseline and
--impl reference) may import this module; the product package never does.
See oracle.c's header for the reference call sites and the pinning status.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np
import pyarrow as pa
import pyarrow.parquet as pq

_HERE = os.path.dirname(os.path.abspath(__file__))
_SO = os.path.join(_HERE, "liboracle.so")
_lib = None

_U8P = C.POINTER(C.c_uint8)


def build():
    src = os.path.join(_HERE, "oracle.c")
    if not os.path.exists(_SO) or os.path.getmtime(_SO) < os.path.getmtime(src):
        subprocess.check_call(["gcc", "-O2", "-std=c11", "-fPIC", "-shared", "-o", _SO, src, "-lm"])


def lib():
    global _lib
    if _lib is None:
        build()
        _lib = C.CDLL(_SO)
        _lib.or_count.restype = C.c_int64
        _lib.or_groupby.restype = C.c_int64
    return _lib


def _ptr(a: np.ndarray | None, typ=C.c_void_p):
    if a is None:
        return None
    return a.ctypes.data_as(typ)


class Column:
    """One decoded column as flat numpy buffers."""

    def __init__(self, arr: pa.ChunkedArray | pa.Array):
        if isinstance(arr, pa.ChunkedArray):
            arr = arr.combine_chunks() if arr.num_chunks != 1 else arr.chunk(0)
        if pa.types.is_dictionary(arr.type):
            arr = arr.cast(arr.type.value_type)
        self.n = len(arr)
        self.type = arr.type
        self.valid = None
        if arr.null_count:
            self.valid = np.ascontiguousarray(np.asarray(arr.is_valid()).astype(np.uint8))
        if pa.types.is_string(arr.type) or pa.types.is_large_string(arr.type):
            arr = arr.cast(pa.string())
            bufs = arr.buffers()
            off = np.frombuffer(bufs[1], dtype=np.int32, count=self.n + 1 + arr.offset)[arr.offset:]
            self.offsets = np.ascontiguousarray(off)
            self.data = np.frombuffer(bufs[2], dtype=np.uint8) if bufs[2] is not None else np.zeros(1, np.uint8)
            self.kind = "str"
        elif pa.types.is_floating(arr.type):
            self.values = np.ascontiguousarray(arr.fill_null(0.0).to_numpy(zero_copy_only=False).astype(np.float64))
            self.kind = "f64"
        elif pa.types.is_boolean(arr.type):
            self.values = np.ascontiguousarray(arr.fill_null(False).to_numpy(zero_copy_only=False).astype(np.int64))
            self.kind = "bool"
        elif pa.types.is_timestamp(arr.type):
            self.values = np.ascontiguousarray(arr.cast(pa.int64()).fill_null(0).to_numpy(zero_copy_only=False).astype(np.int64))
            self.kind = "i64"
        elif pa.types.is_integer(arr.type):
            self.values = np.ascontiguousarray(arr.fill_null(0).to_numpy(zero_copy_only=False).astype(np.int64))
            self.kind = "i64"
        elif pa.types.is_null(arr.type):
            self.values = np.zeros(self.n, np.int64)
            self.valid = np.zeros(self.n, np.uint8)
            self.kind = "i64"
        else:
            raise TypeError(f"oracle: unsupported column type {arr.type}")


class Oracle:
    def __init__(self, table: pa.Table):
        self.table = table
        self.n = table.num_rows
        self._cols: dict[str, Column] = {}

    @classmethod
    def from_parquet(cls, paths, columns=None):
        if isinstance(paths, (str, bytes)):
            paths = [paths]
        tables = [pq.read_table(p, columns=columns) for p in paths]
        # files may lack columns (schema evolution): promote to the union with NULLs
        return cls(pa.concat_tables(tables, promote_options="default"))

    def col(self, name: str) -> Column:
        if name not in self._cols:
            if name in self.table.column_names:
                self._cols[name] = Column(self.table[name])
            else:  # missing column reads as all NULL
                self._cols[name] = Column(pa.nulls(self.n))
        return self._cols[name]

    # ---- predicate ----
    def _eval(self, e) -> tuple[np.ndarray, np.ndarray]:
        from parseable_b200.query import Timestamp  # the Expr syntax tree only
        L = lib()
        n = self.n
        T = np.zeros(n, np.uint8)
        N = np.zeros(n, np.uint8)
        if e.kind in ("and", "or"):
            Ta, Na = self._eval(e.args[0])
            Tb, Nb = self._eval(e.args[1])
            (L.or_and if e.kind == "and" else L.or_or)(_ptr(Ta), _ptr(Na), _ptr(Tb), _ptr(Nb), C.c_int64(n))
            return Ta, Na
        if e.kind == "not":
            Ta, Na = self._eval(e.args[0])
            L.or_not(_ptr(Ta), _ptr(Na), C.c_int64(n))
            return Ta, Na
        if e.kind in ("is_null", "is_not_null"):
            c = self.col(e.args[0].args[0])
            L.or_is_null(_ptr(c.valid), C.c_int64(n), 1 if e.kind == "is_not_null" else 0, _ptr(T), _ptr(N))
            return T, N
        if e.kind == "like":
            c = self.col(e.args[0].args[0])
            p = e.args[1].args[0].encode()
            if c.kind != "str":
                raise TypeError("LIKE on non-string")
            L.or_like(_ptr(c.offsets), _ptr(c.data), _ptr(c.valid), C.c_int64(n), p, len(p), C.c_uint32(e.flags), _ptr(T), _ptr(N))
            return T, N
        if e.kind == "lit":
            v = e.args[0]
            if v is None:
                N[:] = 1
            elif v:
                T[:] = 1
            return T, N
        if e.kind == "cmp":
            a, b, op = e.args[0], e.args[1], e.op
            if a.kind == "lit":
                flip = {2: 4, 4: 2, 3: 5, 5: 3, 0: 0, 1: 1}
                a, b, op = b, a, flip[op]
            c = self.col(a.args[0])
            v = b.args[0]
            if isinstance(v, Timestamp):
                v = v.ms
            if v is None:   # a comparison with NULL is NULL on every row
                N[:] = 1
                return T, N
            if c.kind == "str":
                s = v.encode() if isinstance(v, str) else v
                L.or_cmp_str(_ptr(c.offsets), _ptr(c.data), _ptr(c.valid), C.c_int64(n), op, s, len(s), _ptr(T), _ptr(N))
            elif c.kind == "f64":
                L.or_cmp_f64(_ptr(c.values), _ptr(c.valid), C.c_int64(n), op, C.c_double(float(v)), _ptr(T), _ptr(N))
            elif c.kind == "i64" and isinstance(v, float) and not (v == v and float(v).is_integer() and -2.0 ** 63 <= v < 2.0 ** 63):
                # Int64 column vs a Float64 literal that is no integer: DataFusion's comparison coercion casts the COLUMN
                # to Float64 (datafusion-expr type_coercion/binary: Int64 x Float64 -> Float64) and compares in totalOrder
                vals = np.ascontiguousarray(c.values.astype(np.float64))
                L.or_cmp_f64(_ptr(vals), _ptr(c.valid), C.c_int64(n), op, C.c_double(v), _ptr(T), _ptr(N))
            else:
                L.or_cmp_i64(_ptr(c.values), _ptr(c.valid), C.c_int64(n), op, C.c_int64(int(v)), _ptr(T), _ptr(N))
            return T, N
        raise TypeError(e.kind)

    def select(self, filters) -> np.ndarray:
        """Byte mask of rows whose predicate is TRUE (conjunction of `filters`)."""
        sel = np.ones(self.n, np.uint8)
        for f in filters or []:
            T, _ = self._eval(f)
            sel &= T
        return sel

    def count(self, filters) -> int:
        return int(self.select(filters).sum())

    def row_ids(self, filters) -> np.ndarray:
        return np.flatnonzero(self.select(filters)).astype(np.int64)

    # ---- GROUP BY ----
    def group_by(self, keys, aggs, filters=None) -> pa.Table:
        """aggs: list of parseable_b200.query.Agg.  Returns key columns then aggregates, named like
        the GPU result (count(*), sum(col), ...)."""
        L = lib()
        n = self.n
        sel = self.select(filters) if filters else None
        key_codes, key_valid, key_decode = [], [], []
        keys = list(keys)
        for ki, k in enumerate(keys):
            if hasattr(k, "width_ms"):
                # DATE_BIN(width, column, origin): DataFusion's date_bin floors towards minus infinity
                # (datafusion-functions 53.1.0 date_bin.rs: a negative remainder moves one stride down);
                # /root/reference/src/query/mod.rs:623-680 is the call site (the counts API)
                c = self.col(k.column)
                codes = np.ascontiguousarray(np.floor_divide(c.values.astype(np.int64) - k.origin_ms, k.width_ms) * k.width_ms + k.origin_ms)
                key_decode.append(("i64", pa.timestamp("ms")))
                key_codes.append(codes)
                key_valid.append(c.valid)
                keys[ki] = k.name
                continue
            c = self.col(k)
            if c.kind == "str":
                arr = self.table[k].combine_chunks()
                if pa.types.is_dictionary(arr.type):
                    arr = arr.cast(arr.type.value_type)
                enc = arr.dictionary_encode()
                codes = np.ascontiguousarray(enc.indices.fill_null(0).to_numpy(zero_copy_only=False).astype(np.int64))
                key_decode.append(("str", enc.dictionary))
            elif c.kind == "f64":
                codes = np.ascontiguousarray(c.values.view(np.int64))
                key_decode.append(("f64", None))
            else:
                codes = c.values
                key_decode.append((c.kind, self.table.schema.field(k).type if k in self.table.column_names else pa.int64()))
            key_codes.append(codes)
            key_valid.append(c.valid)
        fn_code = {"count_star": 0, "count": 1, "sum": 2, "min": 3, "max": 4, "avg": 5}
        na = len(aggs)
        fns = (C.c_int * max(na, 1))()
        tys = (C.c_int * max(na, 1))()
        vals = (C.c_void_p * max(na, 1))()
        valids = (_U8P * max(na, 1))()
        agg_cols = []
        for i, a in enumerate(aggs):
            fns[i] = fn_code[a.fn]
            if a.fn == "count_star":
                agg_cols.append(None)
                continue
            c = self.col(a.column)
            agg_cols.append(c)
            if c.kind == "str":
                if a.fn != "count":
                    raise TypeError("oracle: only COUNT over strings")
                tys[i] = 0
                vals[i] = None
            else:
                tys[i] = 1 if c.kind == "f64" else 0
                vals[i] = c.values.ctypes.data
            valids[i] = _ptr(c.valid, _U8P) if c.valid is not None else None
        nk = len(keys)
        kc = (C.c_void_p * max(nk, 1))(*[k.ctypes.data for k in key_codes]) if nk else (C.c_void_p * 1)()
        kv = (_U8P * max(nk, 1))()
        for i, v in enumerate(key_valid):
            kv[i] = _ptr(v, _U8P) if v is not None else None
        max_groups = 1024
        while True:
            out_keys = np.zeros(max_groups * max(nk, 1), np.int64)
            out_null = np.zeros(max_groups * max(nk, 1), np.uint8)
            out_i = np.zeros(max(na, 1) * max_groups, np.int64)
            out_f = np.zeros(max(na, 1) * max_groups, np.float64)
            out_v = np.zeros(max(na, 1) * max_groups, np.uint8)
            g = L.or_groupby(C.c_int64(n), _ptr(sel), nk, kc, kv, na, fns, tys, vals, valids, C.c_int64(max_groups),
                             _ptr(out_keys), _ptr(out_null), _ptr(out_i), _ptr(out_f), _ptr(out_v))
            if g == -2:
                max_groups *= 8
                continue
            if g < 0:
                raise MemoryError("oracle group-by")
            break
        if nk == 0 and g == 0:
            g = 1  # SQL: a global aggregate over zero rows yields one row (COUNT 0, others NULL)
            for i, a in enumerate(aggs):
                out_v[i * max_groups] = 1 if a.fn in ("count_star", "count") else 0
        cols, names = [], []
        for ki, k in enumerate(keys):
            codes = out_keys[: g * nk].reshape(g, nk)[:, ki]
            nulls = out_null[: g * nk].reshape(g, nk)[:, ki].astype(bool)
            kind, aux = key_decode[ki]
            if kind == "str":
                arr = pa.DictionaryArray.from_arrays(pa.array(codes, mask=nulls), aux).cast(pa.string())
            elif kind == "f64":
                arr = pa.array(codes.view(np.float64), mask=nulls)
            elif kind == "bool":
                arr = pa.array(codes.astype(bool), mask=nulls)
            else:
                arr = pa.array(codes, mask=nulls).cast(aux if aux is not None else pa.int64())
            cols.append(arr)
            names.append(k)
        for i, a in enumerate(aggs):
            valid = out_v[i * max_groups: i * max_groups + g].astype(bool)
            c = agg_cols[i]
            if a.fn in ("count_star", "count"):
                arr = pa.array(out_i[i * max_groups: i * max_groups + g])
            elif a.fn == "avg" or (c is not None and c.kind == "f64"):
                arr = pa.array(out_f[i * max_groups: i * max_groups + g], mask=~valid)
            else:
                arr = pa.array(out_i[i * max_groups: i * max_groups + g], mask=~valid)
                if a.fn in ("min", "max") and a.column in self.table.column_names and pa.types.is_timestamp(self.table.schema.field(a.column).type):
                    arr = arr.cast(pa.timestamp("ms"))
            cols.append(arr)
            names.append("count(*)" if a.fn == "count_star" else f"{a.fn}({a.column})")
        return pa.table(cols, names=names)
