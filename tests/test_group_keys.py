"""Every GROUP BY key kind, page form and NULL layout, checked group for group against a numpy reference.

A row reaches its group through three stages, and an error in any of them puts the row in another group without changing
a sum: interning per table column (`build_key_side`: k_key_intern over the dictionary entries, k_row_entries /
k_row_intern over the rows of PLAIN, DELTA and DELTA_(LENGTH_)BYTE_ARRAY pages, the grow-and-redo loop of the key table,
k_key_sample / k_gid_remap for the hot-first numbering); the slot of every row in k_flat_agg (dictionary ids through the
gid LUT, FK_IDS id pages, Booleans, KK_BIN's double reciprocal and its fix-up, NULL as slot `card`, the mixed radix, the
hashed table above 2^26 slots, tuple pages) or in k_scan; and the result assembly (key_gid_of_slot, k_agg_finish,
k_offsets_scan, k_key_gather).  So every query here fingerprints membership: COUNT(*), COUNT / wrapping SUM / MIN / MAX
of `rid` (the global row index) and the wrapping SUM of `rnd` (random Int64).  If these agree for every key tuple, every
row sits in the right group.

Three files: v1 uncompressed, v2, v1 SNAPPY; row groups of 100 003 rows, write batches of 97 rows, 4 KB pages of at most
3 000 rows (pages end off the 32-row grid and start at other rows in other columns); dictionaries fall back to PLAIN at
512 KiB.  Every key column exists NULL-free (`_nn`) and with ~3 % NULLs, a run of NULL pages and one all-NULL row group
(`_n`); `opt` is absent from the last file.  Utf8 keys with 1, 2, 33 and 5 000 values, one of ~70 000 values whose
dictionary falls back mid-chunk, PLAIN-only, DELTA_BYTE_ARRAY and DELTA_LENGTH_BYTE_ARRAY columns, all holding values
that stress equality ("" next to NULL, a / ab, a\\0 / a\\0b, multi-byte UTF-8, 4 093 .. 4 100 and 9 000 bytes that
share a 4 KiB prefix and differ in their last byte); a request-id column whose dictionaries never overlap (the key
table fills and is rebuilt); Int64 keys in dictionary, PLAIN and DELTA form with INT64_MIN / MAX, 0, -1; Float64 keys
with +-0.0, NaNs of both signs with distinct payloads, +-inf and subnormals; Timestamp(ms) keys before 1970 in
dictionary, PLAIN, DELTA and dictionary-fallback form; PLAIN and RLE Booleans; an Int64 DATE_BIN column whose values sit
at k * w - 1, k * w, k * w + 1 for w = 2^29 + 1 and that spans exactly origin +- 2^52 ms.  Beside them: a file of more
than 2^21 distinct PLAIN strings (the row-sized key table regrows), a file whose Int64 key pairs span exactly 2^26 slots
(dense) and 2^26 + 8 192 (hashed), and a file without statistics.

The reference is numpy over `pq.read_table` of the files (the absent column read as NULL), grouping by (validity, bits):
Float64 as uint64 bits, Timestamp and Int64 as int64, strings as bytes, Booleans as bits, DATE_BIN as an exact int64
floor division.

CPU: the reference equals Oracle.group_by; the files hold what they promise (encodings, the mid-chunk fallback with the
same values in dictionary and PLAIN pages, disjoint dictionaries, the boundary cards, the DATE_BIN edge values, which
Float64 bit patterns each form keeps).  GPU: every single key and a generated set of 2-4 key tuples on the resident
table and the file list (NULLs in every position, Booleans inside tuples, DATE_BIN with a Utf8 key in a hashed table,
GROUP BY k, k); keys that are also aggregated or filtered; a subset again under PQB_AGG_FORMS=0, PQB_TUPLE_PAGES=0,
PQB_FLAT_SCAN=0, PQB_GRID=1 / 3, PQB_AGG_KROWS=2 / 4 / 8 and two row-group shards, each configuration proven from its
PQB_VERBOSE line; the key table's rebuilds from its own verbose line; the 2^26 boundary; result batches of 1, 7, 1 000
rows and the default; DATE_BIN widths, origins, page forms, pruning and limits; refusals followed by a correct answer.

Bugs found here, each with its own regression test:
- the string key bytes of a result were sized as (groups / card + 1) x the key's distinct bytes, which holds for one key
  only: in a tuple one long value can sit in far more groups than the average, and k_key_gather wrote past the block
  (test_string_key_bytes_of_tuples);
- with every item on k_scan (PQB_FLAT_SCAN=0), a key column with pages without a dictionary was read through its
  dictionary index, out of bounds; it is now refused (test_kscan_refuses_row_keys).

One-line mutants, each run alone against the named test on the resident table (the first failure reported):
- `key_gid_of_slot` taking `% card` for `% (card + 1)`: test_single_keys (the NULL group of a NULL-bearing key);
- `k_key_gather` taking `% card`: test_tuples (string bytes of another group: invalid UTF-8);
- the DATE_BIN fix-up `rem < 0` dropped, or `rem >= w` dropped: test_date_bin_edges (dbin at FIX_WIDTHS);
- the NULL check dropped from the Boolean key pass: test_single_keys (bp_n: the NULL group vanishes);
- `k_offsets_scan` not carrying across its 1 024-row passes: test_result_batches (non-monotonic offsets);
- `k_gid_remap` over the dictionary entries only (`n` for `n_all`): test_single_keys (sfb_nn: the PLAIN rows of a
  fallback chunk keep the old numbering).
String `entry_equal` without its length check survives: an entry is compared only when the upper 32 bits of the two
values' 64-bit hashes agree, so "a" and "ab" meet in that test only on a hash collision."""
import os
import re

import numpy as np
import pyarrow as pa
import pyarrow.compute as pc
import pyarrow.parquet as pq
import pytest

from oracle.oracle import Oracle
from parseable_b200 import _lib as L
from parseable_b200.query import (DateBin, DeviceTable, QueryError, StandardTableProvider, col, count, count_distinct,
                                  count_star, date_bin, max_, min_, sum_)
from test_agg_tiers import env_vars
from test_project_paths import (F_SPECIALS, FILE_KW, FILE_ROWS, I64_MAX, I64_MIN, PAGE_KW, RG, _rg_index, _words,
                                check_batches, data_pages)

SEED = 20261019
N = sum(FILE_ROWS)
DICT_LIMIT = 512 * 1024               # dictionary pages fall back to PLAIN above this
ALL_NULL_RG = 1                       # every `_n` key column is NULL in this (global) row group
NULL_RUN = 7_000                      # `_n` columns: a run of NULLs (>= two whole pages) in row group 4
W29 = (1 << 29) + 1                   # 2^24 bins of this width span 2^53 + 2^24 ms
P52 = 1 << 52
ORIGIN = -123_456_789_013             # dbin's origin: negative and not on a whole second
# widths near 2^30 for which double(x) * (1 / w) rounds across an integer for some x < 2^53 above the bin base: upwards
# (the kernel's `rem < 0` fix-up) and downwards (`rem >= w`)
FIX_WIDTHS = (1_073_740_826, 1_073_740_824)
REQ_PER_RG = 20_000                   # sreq: distinct request ids per row group, never repeated in another one
BIG_ROWS = 2_200_000                  # sbig: > 2^21 distinct PLAIN strings in a file of its own
BIG_RG = 1_100_000

# values that stress byte equality: "" next to NULL, prefixes, embedded NUL bytes, multi-byte UTF-8, and strings of
# 4 093 .. 4 100 and 9 000 bytes that share a 4 KiB prefix and differ only in their last byte
EQ = ["", "a", "ab", "a\0", "a\0b", "\u00e9", "e\u0301", "日本", "𝄞", "A"]   # é composed and decomposed
LONGS = ["Q" * (n - 1) + t for n in (4093, 4094, 4095, 4096, 4097, 4098, 4099, 4100, 9000) for t in "xy"]
STRESS = EQ + LONGS

# base -> (type, encoding form); every base is written as `<base>_nn` (NULL-free) and `<base>_n` (NULLs)
BASES = {
    "s1": ("str", "dict"), "s2": ("str", "dict"), "s33": ("str", "dict"), "s5000": ("str", "dict"),
    "sfb": ("str", "fallback"), "splain": ("str", "PLAIN"), "sdba": ("str", "DELTA_BYTE_ARRAY"),
    "sdlba": ("str", "DELTA_LENGTH_BYTE_ARRAY"), "sreq": ("str", "dict"),
    "idict": ("i64", "dict"), "ip": ("i64", "PLAIN"), "idelta": ("i64", "DELTA_BINARY_PACKED"),
    "fdict": ("f64", "dict"), "fp": ("f64", "PLAIN"),
    "tdict": ("ts", "dict"), "tp": ("ts", "PLAIN"), "tdelta": ("ts", "DELTA_BINARY_PACKED"), "tfb": ("ts", "fallback"),
    "bp": ("bool", "PLAIN"), "brle": ("bool", "RLE"),
    "dbin": ("i64", "dict"),
}
TYPES = {"str": pa.string(), "i64": pa.int64(), "f64": pa.float64(), "ts": pa.timestamp("ms"), "bool": pa.bool_()}
VARIANTS = [f"{b}_{v}" for b in BASES for v in ("nn", "n")]
KEYS = VARIANTS + ["opt"]
COLUMNS = KEYS + ["rid", "rnd"]
FORCED = {"rid": "PLAIN", "rnd": "PLAIN"}


def _base(name):
    return name.rsplit("_", 1)[0]


# ---- data ------------------------------------------------------------------------------------------------------------
def _pool_str(rng, n, width=0):
    """n distinct Utf8 values, the STRESS values first."""
    return STRESS[:min(n, len(STRESS))] + [f"v{i:06d}-" + "w" * width for i in range(max(0, n - len(STRESS)))]


def _take(pool, codes):
    return pa.array(np.array(pool, dtype=object)[codes], pa.string())


def fix_up_rows(w):
    """(x - bin base, the quotient of the kernel's double multiply) near the top of dbin's range at width w."""
    base = ORIGIN + (-P52 // w) * w
    ks = np.arange((ORIGIN + P52 - base) // w - 20_000, (ORIGIN + P52 - base) // w + 1, dtype=np.int64)
    x = np.concatenate([ks * w + d for d in range(-3, 4)])
    x = x[(x >= 0) & (x <= ORIGIN + P52 - base)]
    return base, x, (x.astype(np.float64) * (1.0 / w)).astype(np.int64)


def dbin_values():
    """The DATE_BIN edge values: k * w - 1, k * w, k * w + 1 (w = 2^29 + 1) for k near 0, +-2^23 and 2^24 - 1 bins up from
    the lowest bin, the exact limits origin +- 2^52, and for FIX_WIDTHS the values whose quotient the fix-up corrects."""
    lo_bin = -(P52 // W29) - 1                       # floor(-2^52 / w)
    ks = set()
    for c in (0, 1, -1, 2, -2, 1 << 22, -(1 << 22), (1 << 23) - 2, -(1 << 23) + 2):
        ks.update(range(c - 2, c + 3))
    for rel in (0, 1, 2, 1 << 23, (1 << 23) + 1, (1 << 24) - 3, (1 << 24) - 2, (1 << 24) - 1):
        ks.add(lo_bin + rel)
    vals = {ORIGIN - P52, ORIGIN + P52}
    for w in FIX_WIDTHS:
        base, x, q = fix_up_rows(w)
        rem = x - q * w
        for r in x[(rem < 0) | (rem >= w)][:40].tolist():
            vals.update((base + r - 1, base + r, base + r + 1))
    for k in ks:
        for d in (-1, 0, 1):
            x = k * W29 + d
            if -P52 <= x <= P52:
                vals.add(ORIGIN + x)
    return np.array(sorted(vals), np.int64)


def _values(base, rng, rg):
    """One key column's N values (a pyarrow array without NULLs)."""
    kind, form = BASES[base]
    if base in ("s1", "s2", "s33", "s5000"):
        card = {"s1": 1, "s2": 2, "s33": 33, "s5000": 5000}[base]
        pool = ["only-é"] if card == 1 else _pool_str(rng, card)
        return _take(pool, rng.integers(0, card, N))
    if base in ("sfb", "splain", "sdba", "sdlba"):
        # sfb: ~70 000 values of ~50 bytes: every chunk's dictionary passes 512 KiB early and falls back to PLAIN, so
        # the same values sit in dictionary entries and in PLAIN rows, in one file and in another
        pool = _pool_str(rng, 70_000 if base == "sfb" else 3_000, 40)
        codes = rng.integers(0, len(pool), N)
        hot = rng.random(N) < 0.04
        codes[hot] = rng.integers(0, len(STRESS), hot.sum())
        return _take(pool, codes)
    if base == "sreq":   # request ids: a row group's values never occur in another row group
        ids = rng.integers(0, REQ_PER_RG, N)
        return pa.array([f"req-{g:02d}-{i:05d}" for g, i in zip(rg.tolist(), ids.tolist())], pa.string())
    if kind == "i64" and base != "dbin":
        pool = np.concatenate([[I64_MIN, I64_MAX, 0, -1, 1, I64_MIN + 1], rng.integers(-10**12, 10**12, 294)]).astype(np.int64)
        return pa.array(pool[rng.integers(0, len(pool), N)])
    if kind == "f64":
        pool = np.concatenate([F_SPECIALS, np.round(rng.standard_normal(100) * 100, 2)])
        return pa.array(pool[rng.integers(0, len(pool), N)])
    if base in ("tdict", "tp"):
        pool = np.concatenate([[-1, 0, 1, -86_400_000, -2_208_988_800_001, 1_700_000_000_000],
                               rng.integers(-2_200_000_000_000, 4_000_000_000_000, 394)]).astype(np.int64)
        return pa.array(pool[rng.integers(0, len(pool), N)], pa.timestamp("ms"))
    if base == "tdelta":   # Parseable's p_timestamp: newest first, starting before 1970 in the last file
        return pa.array(100_000 - np.cumsum(rng.integers(0, 3, N)), pa.timestamp("ms"))
    if base == "tfb":      # nearly distinct: 8-byte dictionary entries pass 512 KiB and fall back
        return pa.array(rng.integers(-50_000_000_000, 50_000_000_000, N), pa.timestamp("ms"))
    if kind == "bool":
        return pa.array(rng.random(N) < 0.5)
    if base == "dbin":
        v = dbin_values()
        x = v[rng.integers(0, len(v), N)]
        x[:len(v)] = v                      # every edge value at least once
        return pa.array(x)
    raise AssertionError(base)


def make_data():
    rng = np.random.default_rng(SEED)
    rg, starts = _rg_index()
    cols, valid = {}, {}
    run0 = np.flatnonzero(rg == 4)[0] + 11_111
    for i, base in enumerate(BASES):
        arr = _values(base, rng, rg)
        for var in ("nn", "n"):
            v = np.ones(N, bool)
            if var == "n":
                v = rng.random(N) >= 0.03
                lo = run0 + 1_009 * i
                v[lo:lo + NULL_RUN] = False
                v[rg == ALL_NULL_RG] = False
                if base == "dbin":          # the edge values stay valid
                    v[:len(dbin_values())] = True
            cols[f"{base}_{var}"], valid[f"{base}_{var}"] = arr, v
    opt = rng.random(N) >= 0.03
    opt[starts[2]:] = False
    cols["opt"], valid["opt"] = _take(_pool_str(rng, 9), rng.integers(0, 9, N)), opt
    cols["rid"], valid["rid"] = pa.array(np.arange(N, dtype=np.int64)), np.ones(N, bool)
    cols["rnd"], valid["rnd"] = pa.array(rng.integers(I64_MIN, I64_MAX, N, dtype=np.int64, endpoint=True)), np.ones(N, bool)
    return cols, valid


def _masked(arr, v):
    return arr if v.all() else pc.if_else(pa.array(v), arr, pa.scalar(None, arr.type))


def _encodings(names):
    enc = {c: BASES[_base(c)][1] for c in names if c in VARIANTS and BASES[_base(c)][1] not in ("dict", "fallback")}
    enc.update({c: e for c, e in FORCED.items() if c in names})
    return enc


def _write(path, t, enc, **kw):
    pq.write_table(t, path, use_dictionary=[c for c in t.column_names if c not in enc], column_encoding=enc or None,
                   dictionary_pagesize_limit=DICT_LIMIT, **kw)


def _reference(paths, schema):
    parts = []
    for p in paths:
        t = pq.read_table(p)
        for f in schema:
            if f.name not in t.column_names:
                t = t.append_column(f.name, pa.nulls(t.num_rows, f.type))
        parts.append(t.select(schema.names))
    return pa.concat_tables(parts).combine_chunks()


@pytest.fixture(scope="module")
def gdata(built, data_dir):
    cols, valid = make_data()
    paths, lo = [], 0
    for i, n in enumerate(FILE_ROWS):
        names = [c for c in COLUMNS if not (c == "opt" and i == 2)]
        t = pa.table({c: _masked(cols[c].slice(lo, n), valid[c][lo:lo + n]) for c in names})
        p = os.path.join(data_dir, f"group_keys_{i}.parquet")
        _write(p, t, _encodings(names), row_group_size=RG, **FILE_KW[i], **PAGE_KW)
        paths.append(p)
        lo += n
    schema = pa.schema([(c, TYPES[BASES[_base(c)][0]]) if c in VARIANTS else (c, pa.string() if c == "opt" else pa.int64())
                        for c in COLUMNS])
    return paths, schema, _reference(paths, schema)


@pytest.fixture(scope="module")
def side_files(built, data_dir):
    """name -> (paths, schema, reference table): the > 2^21 distinct PLAIN strings, the 2^26 boundary keys, no statistics."""
    rng = np.random.default_rng(SEED + 1)
    out = {}
    # sbig: nearly every value distinct, 3 % NULL, PLAIN pages only
    ids = rng.permutation(BIG_ROWS)
    v = rng.random(BIG_ROWS) >= 0.03
    sbig = pa.array([f"{i:07x}/{i * 2654435761 % 1000003:06d}" for i in ids.tolist()], pa.string())
    t = pa.table({"sbig": _masked(sbig, v), "rid": pa.array(np.arange(BIG_ROWS, dtype=np.int64)),
                  "rnd": pa.array(rng.integers(I64_MIN, I64_MAX, BIG_ROWS, dtype=np.int64, endpoint=True))})
    p = os.path.join(data_dir, "group_keys_big.parquet")
    _write(p, t, {"sbig": "PLAIN", "rid": "PLAIN", "rnd": "PLAIN"}, row_group_size=BIG_RG)
    out["big"] = ([p], t.schema, _reference([p], t.schema))
    # ba, bb: 8 191 distinct values each ((8 191 + 1)^2 = 2^26 slots: dense); bc: 8 192 (8 193 x 8 192 slots: hashed)
    n = 3 * 8192
    i = np.arange(n, dtype=np.int64)
    t = pa.table({"ba": pa.array(i % 8191 - 4000), "bb": pa.array((i * 3) % 8191 * 1_000_003), "bc": pa.array(i % 8192 + 10**15),
                  "rid": pa.array(i), "rnd": pa.array(rng.integers(I64_MIN, I64_MAX, n, dtype=np.int64, endpoint=True))})
    p = os.path.join(data_dir, "group_keys_bound.parquet")
    _write(p, t, {"rid": "PLAIN", "rnd": "PLAIN"}, row_group_size=10_000)
    out["bound"] = ([p], t.schema, _reference([p], t.schema))
    # a Timestamp key in a file written without statistics: DATE_BIN over it is refused, GROUP BY it answers
    n = 5_000
    t = pa.table({"ts": pa.array(rng.integers(0, 1_000_000, n), pa.timestamp("ms")), "rid": pa.array(np.arange(n, dtype=np.int64)),
                  "rnd": pa.array(rng.integers(I64_MIN, I64_MAX, n, dtype=np.int64, endpoint=True))})
    p = os.path.join(data_dir, "group_keys_nostats.parquet")
    _write(p, t, {"rid": "PLAIN", "rnd": "PLAIN"}, write_statistics=False)
    out["nostats"] = ([p], t.schema, _reference([p], t.schema))
    return out


# ---- reference -------------------------------------------------------------------------------------------------------
def _valid(a):
    return a.is_valid().to_numpy(zero_copy_only=False)


def _num(a):
    """(validity, int64 bits) of a non-string array: Float64 as its bits, Timestamp / Int64 as int64, Booleans as 0 / 1."""
    a = a.combine_chunks() if isinstance(a, pa.ChunkedArray) else a
    v = _valid(a)
    return v, np.where(v, _words(a).view(np.int64), 0)


class Ref:
    """The reference table, grouped in numpy by (validity, bits) of every key."""

    def __init__(self, t: pa.Table):
        self.t = t
        self.n = t.num_rows
        self.rid = t["rid"].to_numpy()
        self.rnd = t["rnd"].to_numpy()
        self._keys = {}
        self._groups = {}

    def key(self, k):
        """(validity, int64 value) per row; strings as their code in `self.dicts[name]` (bytes)."""
        if k in self._keys:
            return self._keys[k]
        if isinstance(k, DateBin):
            v, x, _ = self.key(k.column)
            b = np.where(v, np.floor_divide(x - k.origin_ms, k.width_ms) * k.width_ms + k.origin_ms, 0)
            out = (v, b, None)
        else:
            a = self.t[k].combine_chunks()
            if pa.types.is_string(a.type):
                enc = pc.dictionary_encode(a.cast(pa.binary()))
                codes = enc.indices.fill_null(0).to_numpy(zero_copy_only=False).astype(np.int64)
                out = (_valid(a), codes, enc.dictionary)
            else:
                out = _num(a) + (None,)
        self._keys[k] = out
        return out

    def result_codes(self, k, arr):
        """The same (validity, value) of a result key column."""
        arr = arr.combine_chunks() if isinstance(arr, pa.ChunkedArray) else arr
        _, _, dictionary = self.key(k)
        if dictionary is not None:
            v = _valid(arr)
            idx = pc.index_in(arr.cast(pa.binary()), value_set=dictionary)
            found = _valid(idx)
            assert not (v & ~found).any(), (k, "a key value the reference does not hold",
                                            arr.filter(pa.array(v & ~found))[0].as_py()[:80])
            return v, np.where(v, idx.fill_null(-1).to_numpy(zero_copy_only=False), 0).astype(np.int64)
        if isinstance(k, DateBin):
            arr = arr.cast(pa.int64())
        return _num(arr)

    def groups(self, keys, sel=None):
        """(unique (validity, value) rows, fingerprint columns) of the selected rows; kept for the next query over all
        rows with the same keys."""
        if sel is None and tuple(keys) in self._groups:
            return self._groups[tuple(keys)]
        out = self._grouped(keys, sel)
        if sel is None:
            self._groups[tuple(keys)] = out
        return out

    def _grouped(self, keys, sel):
        rows = np.arange(self.n) if sel is None else np.flatnonzero(sel)
        cols = []
        for k in keys:
            v, x, _ = self.key(k)
            cols += [v[rows].astype(np.int64), x[rows]]
        if not keys:
            cols = [np.zeros(len(rows), np.int64)]
        uniq, inv = np.unique(np.stack(cols, 1), axis=0, return_inverse=True)
        inv = inv.reshape(-1)
        order = np.argsort(inv, kind="stable")
        starts = np.searchsorted(inv[order], np.arange(len(uniq)))
        r = rows[order]
        fp = {
            "count": np.diff(np.append(starts, len(r))).astype(np.int64),
            "sum_rid": np.add.reduceat(self.rid[r].astype(np.uint64), starts).view(np.int64),
            "min_rid": np.minimum.reduceat(self.rid[r], starts),
            "max_rid": np.maximum.reduceat(self.rid[r], starts),
            "sum_rnd": np.add.reduceat(self.rnd[r].astype(np.uint64), starts).view(np.int64),
        }
        return uniq, fp


FP_AGGS = [count_star(), count("rid"), sum_("rid"), min_("rid"), max_("rid"), sum_("rnd")]
FP_COLS = ["count", "count", "sum_rid", "min_rid", "max_rid", "sum_rnd"]
# a query takes at most 8 aggregates: beside 5 more, a shorter fingerprint
FP_SHORT = ([count_star(), sum_("rid"), sum_("rnd")], ["count", "sum_rid", "sum_rnd"])


def check_groups(R: Ref, got: pa.Table, keys, what, sel=None, extra=None, fp_cols=FP_COLS):
    """got: keys, then the fingerprint aggregates named by fp_cols, then `extra` aggregates, checked by
    extra[1](unique key rows, [first key column] + extra result columns, fingerprints, what)."""
    uniq, fp = R.groups(keys, sel)
    nk = len(keys)
    assert got.num_columns == nk + len(fp_cols) + (len(extra[0]) if extra else 0), (what, got.column_names)
    assert got.num_rows == len(uniq), (what, "groups", got.num_rows, len(uniq))
    if not len(uniq):
        return
    cols = []
    for i, k in enumerate(keys):
        v, x = R.result_codes(k, got.column(i))
        cols += [v.astype(np.int64), x]
    if not keys:
        cols = [np.zeros(got.num_rows, np.int64)]
    guniq, idx = np.unique(np.stack(cols, 1), axis=0, return_index=True)
    assert len(guniq) == len(uniq), (what, "duplicate groups in the result", got.num_rows - len(guniq))
    bad = np.flatnonzero((guniq != uniq).any(1))
    assert bad.size == 0, (what, "group keys differ", bad.size, guniq[bad[0]].tolist(), uniq[bad[0]].tolist())
    for j, name in enumerate(fp_cols):
        g = got.column(nk + j).combine_chunks().take(pa.array(idx))
        assert g.null_count == 0, (what, got.column_names[nk + j], "NULL")
        g = g.to_numpy(zero_copy_only=False).astype(np.int64)
        bad = np.flatnonzero(g != fp[name])
        if bad.size:
            i = int(bad[0])
            raise AssertionError(f"{what}: {got.column_names[nk + j]}: {bad.size} of {len(uniq)} groups differ; group "
                                 f"{uniq[i].tolist()}: got {g[i]}, want {fp[name][i]}")
    if extra:
        cols = [got.column(j).combine_chunks().take(pa.array(idx)) for j in [0] + list(range(nk + len(fp_cols), got.num_columns))]
        extra[1](uniq, cols, fp, what)


# ---- queries ---------------------------------------------------------------------------------------------------------
def tuples():
    """A generated set of 2-4 key tuples (every key kind in some position, NULLs in every position) and the named cases."""
    rng = np.random.default_rng(SEED + 2)
    small = [k for k in KEYS if _base(k) not in ("sreq", "sfb", "tfb", "dbin")]
    out = []
    for i in range(18):
        n = 2 + i % 3
        out.append(tuple(str(k) for k in rng.choice(small, n, replace=False)))
    out += [
        ("bp_n", "s33_n"), ("brle_n", "bp_n", "idict_n"), ("s2_n", "bp_nn", "brle_n", "fdict_n"),   # Booleans inside tuples
        ("s33_n", "s33_n"), ("ip_n", "ip_n", "s2_n"),                                               # the same key twice
        ("opt", "s5000_n"), ("sfb_n", "s2_n"), ("sreq_n", "bp_n"), ("sdba_n", "sdlba_n"),
        ("s5000_n", "idict_n", "fdict_n"),                                                          # 5 001 x 301 x 118: hashed
    ]
    return out


TUPLES = tuples()
BIN_HASHED = (date_bin(1, "tdelta_n"), "s5000_n")          # ~1.5 M bins x 5 001 values: hashed


def _key_id(keys):
    return ",".join(k.name + f"/{k.width_ms}/{k.origin_ms}" if isinstance(k, DateBin) else k for k in keys)


VERBOSE_AGG = re.compile(r"\[pqb\] k_flat_agg<(\d+)((?:,\w+)*)>: (\d+) CTAs")
VERBOSE_KEY = re.compile(r"\[pqb\] key column (\w+): card (\d+), (\d+) dictionary entries \+ (\d+) rows, table capacity (\d+), (\d+) rebuilds")


def run(prov, keys, aggs=FP_AGGS, filters=(), env=None, capfd=None, **kw):
    """(result table, PQB_VERBOSE log)."""
    if capfd is not None:
        capfd.readouterr()
    with env_vars({**(env or {}), "PQB_VERBOSE": 1}):
        res = prov.aggregate(list(keys), list(aggs), list(filters), **kw)
    log = capfd.readouterr().err if capfd is not None else ""
    return res, log


@pytest.fixture(scope="module")
def R(gdata):
    return Ref(gdata[2])


@pytest.fixture(scope="module")
def gpu(gdata):
    paths, schema, _ = gdata
    table = DeviceTable(paths, schema.names)
    yield {"resident": StandardTableProvider(table, schema=schema), "files": StandardTableProvider(paths, schema=schema)}
    table.close()


SOURCES = ["resident", "files"]


# ---- CPU -------------------------------------------------------------------------------------------------------------
def _chunk_encodings(paths):
    enc = {}
    for p in paths:
        md = pq.ParquetFile(p).metadata
        for g in range(md.num_row_groups):
            for j in range(md.num_columns):
                c = md.row_group(g).column(j)
                enc.setdefault(c.path_in_schema, []).append(set(c.encodings))
    return enc


def test_data_layout(gdata, R):
    """Encodings per column, the mid-chunk fallback holding the same values in dictionary and PLAIN pages across files,
    NULL layouts, the absent column, the equality-stress values."""
    paths, schema, ref = gdata
    assert ref.num_rows == N and "opt" not in pq.ParquetFile(paths[2]).schema_arrow.names
    enc = _chunk_encodings(paths)
    for name in VARIANTS:
        form = BASES[_base(name)][1]
        for e in enc[name]:
            if form in ("dict", "fallback"):
                assert "RLE_DICTIONARY" in e, (name, e)
            else:
                assert "RLE_DICTIONARY" not in e and form in e, (name, e)
    pages = data_pages(paths, schema)
    codes = {"PLAIN": 0, "RLE_DICTIONARY": 8}
    for name in VARIANTS:
        form = BASES[_base(name)][1]
        kinds = {pe for _, _, pe in pages[name]}
        if form == "dict":
            assert kinds == {codes["RLE_DICTIONARY"]}, (name, kinds)
        elif form == "fallback":   # every chunk with values: dictionary pages first, then PLAIN pages
            assert kinds == {0, 8}, (name, kinds)
    # the fallback column: values in dictionary pages of one file and in PLAIN pages of another
    for name in ("sfb_nn", "sfb_n", "tfb_nn"):
        a = ref[name].cast(pa.binary()) if name.startswith("s") else ref[name].cast(pa.int64())
        in_dict, in_plain = {}, {}
        for r0, n, pe in pages[name]:
            f = int(np.searchsorted(np.cumsum(FILE_ROWS), r0, side="right"))
            vals = set(x for x in a.slice(r0, n).to_pylist() if x is not None)
            (in_dict if pe == 8 else in_plain).setdefault(f, set()).update(vals)
        cross = any(in_dict[f] & in_plain[g] for f in in_dict for g in in_plain if f != g)
        assert cross, name
        if name.startswith("s"):
            for s in (b"a", b"ab", b"", LONGS[0].encode()):
                assert any(s in in_dict[f] for f in in_dict) and any(s in in_plain[f] for f in in_plain), (name, s[:8])
    # the stress values in every Utf8 form, "" next to NULL
    for b in ("s33", "s5000", "sfb", "splain", "sdba", "sdlba"):
        vals = set(pc.unique(ref[f"{b}_n"].cast(pa.binary())).to_pylist())
        assert {s.encode() for s in STRESS} <= vals and None in vals, b
    # NULL layouts: an all-NULL row group, a run of NULL pages; the NULL-free variants hold no NULL
    rg, _ = _rg_index()
    for name in VARIANTS:
        v = _valid(ref[name])
        if name.endswith("_nn"):
            assert v.all(), name
        else:
            assert not v[rg == ALL_NULL_RG].any() and 0.02 < 1 - v[rg != ALL_NULL_RG].mean() < 0.06, name
    # Int64 extremes and Timestamps before 1970
    for name in ("idict_nn", "ip_nn", "idelta_nn"):
        x = R.key(name)[1]
        assert {I64_MIN, I64_MAX, 0, -1} <= set(x.tolist()), name
    for name in ("tdict_nn", "tp_nn", "tdelta_nn", "tfb_nn"):
        assert (R.key(name)[1] < 0).any(), name


def test_float_bit_patterns(gdata, R):
    """Which Float64 bit patterns each form keeps through the writer (Arrow's dictionary builder may fold NaN payloads
    or -0.0 / 0.0); the reference takes the read-back, and every form keeps both zeros and NaNs of both signs."""
    want = set(F_SPECIALS.view(np.int64).tolist())
    kept = {}
    for name in ("fdict_nn", "fp_nn"):
        v, x, _ = R.key(name)
        got = set(x[v].tolist())
        kept[name] = sorted(hex(b & (2**64 - 1)) for b in want & got)
        assert {0, -(1 << 63)} <= got, name                                   # +0.0 and -0.0
        nan = (np.array(sorted(got)) >> 52) & 0x7FF == 0x7FF
        bits = np.array(sorted(got))[nan]
        assert (bits < 0).any() and (bits > 0).any(), name                    # NaN / inf of both signs
    print("Float64 specials kept:", kept)
    assert set(kept["fp_nn"]) == {hex(b & (2**64 - 1)) for b in want}        # PLAIN keeps every pattern


def test_disjoint_dictionaries(gdata, R):
    """sreq: no value in two row groups, ~20 000 per row group over >= 7 row groups, so the distinct count is more than
    4 x the largest chunk dictionary (the key table's first capacity); sbig: > 2^21 distinct PLAIN values."""
    paths, _, ref = gdata
    rg, _ = _rg_index()
    for name in ("sreq_nn", "sreq_n"):
        seen, per = {}, []
        for g in range(int(rg.max()) + 1):
            s = set(pc.unique(ref[name].filter(pa.array(rg == g))).drop_null().to_pylist())
            for x in s:
                assert x not in seen, (name, x)
                seen[x] = g
            per.append(len(s))
        assert sum(1 for n in per if n > 15_000) >= 7, per
        assert len(seen) > 4 * max(per), (len(seen), max(per))
        assert len(seen) * 2 > 4 * 65_536, len(seen)   # the first table (4 x 20 000 -> 131 072 slots) runs too full


def test_side_files(side_files):
    """sbig holds > 2^21 distinct PLAIN values; the boundary keys have exactly 8 191 / 8 191 / 8 192 distinct values;
    the no-statistics file has no statistics."""
    _, _, big = side_files["big"]
    assert pc.count_distinct(big["sbig"]).as_py() > (1 << 21)
    assert all(e == {"PLAIN"} or e <= {"PLAIN", "RLE"} for e in _chunk_encodings(side_files["big"][0])["sbig"])
    _, _, b = side_files["bound"]
    assert [pc.count_distinct(b[c]).as_py() for c in ("ba", "bb", "bc")] == [8191, 8191, 8192]
    assert (8191 + 1) * (8191 + 1) == 1 << 26 and (8192 + 1) * (8191 + 1) > 1 << 26
    md = pq.ParquetFile(side_files["nostats"][0][0]).metadata
    assert all(md.row_group(g).column(0).statistics is None or not md.row_group(g).column(0).statistics.has_min_max
               for g in range(md.num_row_groups))


def bin_span(R, column, w, o, sel=None):
    """(accepted, bins) of DATE_BIN(w, column, o) over the rows' values (the footer statistics are exact for them)."""
    v, x, _ = R.key(column)
    m = v if sel is None else v & sel
    if not m.any():
        return True, 1
    lo, hi = int(x[m].min()), int(x[m].max())
    if lo < o - P52 or hi > o + P52:
        return False, None
    bins = (hi - o) // w - (lo - o) // w + 1
    return bins <= (1 << 24), bins


def test_date_bin_edges_data(R):
    """dbin: every edge value, the exact +-2^52 limits, 2^24 bins at w = 2^29 + 1 and 2^24 + 1 at w = 2^29; the values
    for which double(x) * (1 / w) rounds across an integer are there, so the kernel's fix-up must run."""
    v, x, _ = R.key("dbin_nn")
    assert x.min() == ORIGIN - P52 and x.max() == ORIGIN + P52
    assert bin_span(R, "dbin_nn", W29, ORIGIN) == (True, 1 << 24)
    assert bin_span(R, "dbin_nn", 1 << 29, ORIGIN) == (False, (1 << 24) + 1)
    assert bin_span(R, "dbin_nn", W29, ORIGIN + 1)[0] is False and bin_span(R, "dbin_nn", W29, ORIGIN - 1)[0] is False
    # the kernel's arithmetic without its fix-up, over dbin's own values: at FIX_WIDTHS[0] the quotient comes out one too
    # high (rem < 0), at FIX_WIDTHS[1] one too low (rem >= w); both widths keep < 2^24 bins
    for w, sign in zip(FIX_WIDTHS, (-1, 1)):
        base = ORIGIN + ((int(x.min()) - ORIGIN) // w) * w
        d = x - base
        q = (d.astype(np.float64) * (1.0 / w)).astype(np.int64)
        rem = d - q * w
        off = (rem < 0) if sign < 0 else (rem >= w)
        assert off.sum() >= 20 and ((rem < 0) | (rem >= w)).sum() == off.sum(), (w, off.sum())
        assert np.array_equal(q + np.where(rem < 0, -1, np.where(rem >= w, 1, 0)), np.floor_divide(d, w))
        assert bin_span(R, "dbin_nn", w, ORIGIN)[0]


def test_reference_matches_oracle(gdata, R):
    """The numpy reference equals Oracle.group_by for every key kind the oracle takes (Utf8, Int64, Float64, Timestamp,
    Boolean, DATE_BIN) and a few tuples."""
    ref = gdata[2]
    cases = [[k] for k in ("s2_n", "s33_n", "sfb_n", "sdba_n", "idict_n", "ip_n", "idelta_n", "fdict_n", "fp_n", "tdict_n",
                           "tdelta_n", "bp_n", "brle_n", "opt")]
    cases += [["bp_n", "s33_n"], ["fdict_n", "tp_n", "brle_n"], [date_bin("1h", "tp_n", -1_234_567)], [date_bin(7_000, "tdelta_n"), "s2_n"],
              [date_bin(W29, "dbin_n", ORIGIN)]]
    for keys in cases:
        names = sorted({k.column if isinstance(k, DateBin) else k for k in keys} | {"rid", "rnd"})
        ora = Oracle(ref.select(names))
        got = ora.group_by(keys, FP_AGGS)
        check_groups(R, got, keys, f"oracle {_key_id(keys)}")


# ---- GPU: single keys and tuples --------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("source", SOURCES)
def test_single_keys(R, gpu, source, capfd):
    """Every key column alone: its groups and their fingerprints; a NULL-free key still has no NULL group."""
    prov = gpu[source]
    for k in KEYS:
        res, log = run(prov, [k], capfd=capfd)
        check_batches(res)
        check_groups(R, res.table(), [k], f"{source} {k}")
        assert VERBOSE_AGG.search(log), (k, log)


@pytest.mark.gpu
@pytest.mark.parametrize("source", SOURCES)
def test_tuples(R, gpu, source, capfd):
    """2-4 key tuples: NULLs in every position, Booleans inside tuples, GROUP BY k, k, a hashed tuple, DATE_BIN with a
    Utf8 key in a hashed table.  On the resident table the tuples of dictionary-only keys take tuple pages."""
    prov = gpu[source]
    for keys in TUPLES + [BIN_HASHED]:
        res, log = run(prov, keys, capfd=capfd)
        check_batches(res)
        check_groups(R, res.table(), list(keys), f"{source} {_key_id(keys)}")
        m = VERBOSE_AGG.search(log)
        assert m, (keys, log)
        if keys in (BIN_HASHED, ("s5000_n", "idict_n", "fdict_n")):
            assert "hashed" in m.group(2), (keys, m.group(0))
        dict_only = all(_dict_key(k) for k in keys) and len(set(keys)) == len(keys) and "hashed" not in m.group(2)
        if source == "resident" and dict_only:
            assert "group slots: tuple pages" in log, (keys, log)
        elif len(keys) >= 2 and "hashed" not in m.group(2):
            assert "group slots: per-key ids" in log, (keys, log)


def _dict_key(k):
    """A key whose every page has a dictionary (not a Boolean, not DATE_BIN)."""
    return isinstance(k, str) and (k == "opt" or BASES[_base(k)][1] == "dict" and BASES[_base(k)][0] != "bool")


def _kscan_key(k):
    """A key k_scan stages itself: dictionary ids and Booleans."""
    return _dict_key(k) or isinstance(k, str) and BASES[_base(k)][0] == "bool"


def _key_input_check(key, kind):
    def check(uniq, cols, fp, what):
        v = uniq[:, 0].astype(bool)
        n = fp["count"]
        key, mn, mx, cnt, dist = cols[:5]
        assert np.array_equal(cnt.to_numpy(zero_copy_only=False), np.where(v, n, 0)), (what, "count(k)")
        assert np.array_equal(dist.to_numpy(zero_copy_only=False), v.astype(np.int64)), (what, "count(distinct k)")
        for a in (mn, mx):
            assert np.array_equal(_valid(a), v), (what, "min/max NULLs")
        if kind == "str":
            for a in (mn, mx):
                assert pc.all(pc.equal(a.cast(pa.binary()), key.cast(pa.binary())).fill_null(True)).as_py(), (what, "min/max(k) != k")
        else:
            assert np.array_equal(_num(mn)[1][v], uniq[v, 1]) and np.array_equal(_num(mx)[1][v], uniq[v, 1]), what
        if len(cols) > 5:   # SUM of an Int64 key: count x key, wrapping
            s = cols[5]
            want = (n.astype(np.uint64) * uniq[:, 1].astype(np.uint64)).view(np.int64)
            assert np.array_equal(_valid(s), v) and np.array_equal(_num(s)[1][v], want[v]), (what, "sum(k)")
    return check


@pytest.mark.gpu
@pytest.mark.parametrize("source", SOURCES)
def test_key_roles(R, gpu, source):
    """A key that is also an input (MIN / MAX / COUNT / COUNT(DISTINCT) of it, SUM of an Int64 key) and a dictionary key
    that is also filtered; a key with pages without a dictionary in either role is refused, never answered wrongly."""
    prov = gpu[source]
    for k, kind in (("s33_n", "str"), ("idict_n", "i64"), ("s5000_nn", "str")):
        aggs = [min_(k), max_(k), count(k), count_distinct(k)] + ([sum_(k)] if kind == "i64" else [])
        res = prov.aggregate([k], FP_SHORT[0] + aggs)
        check_groups(R, res.table(), [k], f"{source} {k} as input", extra=(aggs, _key_input_check(k, kind)), fp_cols=FP_SHORT[1])
    v, x, d = R.key("s33_n")
    a_code = d.to_pylist().index(b"a")
    for flt, sel in (([col("s33_n") != "a"], v & (x != a_code)), ([col("s33_n") == "ab"], v & (x == d.to_pylist().index(b"ab"))),
                     ([col("s33_n").is_null()], ~v)):
        res = prov.aggregate(["s33_n"], FP_AGGS, flt)
        check_groups(R, res.table(), ["s33_n"], f"{source} s33_n filtered", sel=sel)
    for k, aggs, flt in (("ip_n", [sum_("ip_n")], []), ("sfb_n", [count_star()], [col("sfb_n") == "a"])):
        with pytest.raises(QueryError) as e:
            prov.aggregate([k], aggs, flt)
        assert e.value.code == L.PQ_ERR_UNSUPPORTED, (k, e.value)
    res = prov.aggregate(["s33_n"], FP_AGGS)      # the context still answers
    check_groups(R, res.table(), ["s33_n"], f"{source} after refusals")


# ---- GPU: configurations ---------------------------------------------------------------------------------------------
CFG_KEYS = [("s33_n",), ("sfb_n",), ("sdba_n",), ("sdlba_nn",), ("ip_n",), ("fp_n",), ("idelta_n",), ("tdelta_n",), ("tfb_n",),
            ("bp_n",), ("brle_nn",), ("sreq_n",), ("opt",), ("s33_n", "bp_n"), ("idict_n", "s5000_n", "brle_n"),
            ("fdict_n", "tdict_n"), ("s2_n", "s2_n"), ("s5000_n", "idict_n", "fdict_n"), BIN_HASHED]
CFG_HASHED = {("s5000_n", "idict_n", "fdict_n"), BIN_HASHED}   # a hashed table needs a flat-store copy of every page
CONFIGS = {
    "forms0": {"PQB_AGG_FORMS": 0},
    "tuple0": {"PQB_TUPLE_PAGES": 0},
    "kscan": {"PQB_FLAT_SCAN": 0},
    "grid1": {"PQB_GRID": 1},
    "grid3": {"PQB_GRID": 3},
    "krows2": {"PQB_AGG_KROWS": 2},
    "krows4": {"PQB_AGG_KROWS": 4},
    "krows8": {"PQB_AGG_KROWS": 8},
}
# k_scan stages dictionary and Boolean keys itself
KSCAN_KINDS = {"dict"}


@pytest.mark.gpu
@pytest.mark.parametrize("cfg", list(CONFIGS))
def test_configs(R, gpu, cfg, capfd):
    """The subset under each switch, on the resident table; the verbose line proves the configuration ran."""
    env = CONFIGS[cfg]
    prov = gpu["resident"]
    answered = 0
    for keys in CFG_KEYS:
        what = f"{cfg} {_key_id(keys)}"
        try:
            res, log = run(prov, keys, env=env, capfd=capfd)
        except QueryError as e:
            # only k_scan may refuse a key it does not stage (pages without a dictionary, DATE_BIN, hashed tables)
            assert cfg == "kscan" and e.code == L.PQ_ERR_UNSUPPORTED, (what, e)
            assert keys in CFG_HASHED or not all(_kscan_key(k) for k in keys), (what, "a dictionary / Boolean key refused by k_scan", e)
            continue
        answered += 1
        check_batches(res)
        check_groups(R, res.table(), list(keys), what)
        m = VERBOSE_AGG.search(log)
        hashed = bool(m and "hashed" in m.group(2))
        if cfg == "kscan":
            assert "[pqb] k_scan:" in log and not m, (what, log)
            continue
        assert m, (what, log)
        if cfg.startswith("grid"):
            assert int(m.group(3)) == env["PQB_GRID"], (what, m.group(0))
        if cfg.startswith("krows") and not hashed:
            assert int(m.group(1)) == env["PQB_AGG_KROWS"], (what, m.group(0))
        if cfg == "forms0":
            assert "pages, " not in "".join(l for l in log.splitlines() if "[pqb] slot " in l), (what, log)
        if cfg in ("forms0", "tuple0") and len(keys) >= 2 and not hashed:
            assert "group slots: per-key ids" in log and "tuple pages" not in log, (what, log)
    assert answered >= (5 if cfg == "kscan" else len(CFG_KEYS)), (cfg, answered)


@pytest.mark.gpu
@pytest.mark.parametrize("shard", [0, 1])
def test_shards(gdata, R, shard):
    """Two row-group shards (global row group g % 2 == shard), each against the reference over its own row groups."""
    paths, schema, _ = gdata
    rg, _ = _rg_index()
    sel = rg % 2 == shard
    for source in SOURCES:
        if source == "resident":
            table = DeviceTable(paths, schema.names, shard_index=shard, shard_count=2)
            prov = StandardTableProvider(table, schema=schema)
        else:
            table, prov = None, StandardTableProvider(paths, schema=schema, shard_index=shard, shard_count=2)
        try:
            for keys in CFG_KEYS:
                res = prov.aggregate(list(keys), FP_AGGS)
                check_groups(R, res.table(), list(keys), f"shard {shard} {source} {_key_id(keys)}", sel=sel)
        finally:
            if table is not None:
                table.close()


@pytest.mark.gpu
def test_key_table_rebuilds(gdata, side_files, capfd):
    """The disjoint-dictionary key overfills the first key table (sized from the largest chunk dictionary) and the
    table is rebuilt; so does the row-sized table of > 2^21 distinct PLAIN rows.  Both answers stay exact."""
    paths, schema, ref = gdata
    prov = StandardTableProvider(paths, schema=schema)
    R = Ref(ref)
    for k in ("sreq_nn", "sreq_n"):
        res, log = run(prov, [k], capfd=capfd)
        check_groups(R, res.table(), [k], k)
        lines = [m for m in VERBOSE_KEY.findall(log) if m[0] == k]
        assert len(lines) == 1, log
        card, ndict, rows, cap, rebuilds = map(int, lines[0][1:])
        assert rows == 0 and rebuilds >= 1 and 2 * card <= cap and card > 4 * REQ_PER_RG, lines
    bpaths, bschema, bref = side_files["big"]
    bprov = StandardTableProvider(bpaths, schema=bschema)
    res, log = run(bprov, ["sbig"], capfd=capfd)
    check_groups(Ref(bref), res.table(), ["sbig"], "sbig")
    lines = [m for m in VERBOSE_KEY.findall(log) if m[0] == "sbig"]
    assert len(lines) == 1, log
    card, rows, cap, rebuilds = int(lines[0][1]), int(lines[0][3]), int(lines[0][4]), int(lines[0][5])
    assert card > (1 << 21) and rows >= BIG_ROWS and rebuilds >= 1 and 2 * card <= cap, lines[0]


@pytest.mark.gpu
def test_dense_hashed_boundary(side_files, capfd):
    """(8 191 + 1) x (8 191 + 1) = 2^26 slots stay in the dense table; (8 192 + 1) x (8 191 + 1) go to the hashed one."""
    paths, schema, ref = side_files["bound"]
    R = Ref(ref)
    table = DeviceTable(paths, schema.names)
    try:
        for source, prov, env in (("files", StandardTableProvider(paths, schema=schema), {}),
                                  ("resident", StandardTableProvider(table, schema=schema), {"PQB_TUPLE_PAGES": 0})):
            for keys, hashed in ((["ba", "bb"], False), (["bc", "bb"], True), (["bb", "bc"], True)):
                res, log = run(prov, keys, env=env, capfd=capfd)
                check_groups(R, res.table(), keys, f"{source} {keys}")
                m = VERBOSE_AGG.search(log)
                assert m and ("hashed" in m.group(2)) == hashed, (source, keys, log)
    finally:
        table.close()


# ---- GPU: result assembly --------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("source", SOURCES)
def test_result_batches(R, gpu, source, capfd):
    """More than 3 000 string-keyed groups (several k_offsets_scan passes) in batches of 1, 7, 1 000 rows and the default:
    every batch valid Arrow data whose key null_count equals its own bitmap; a repeated query on the resident table takes
    the one-round-trip result tail."""
    prov = gpu[source]
    for keys in (["s5000_n"], ["s5000_n", "s33_n"], ["sfb_n"]):
        for bs in (1, 7, 1000, 0):
            if keys != ["s5000_n"] and bs in (1, 7):
                continue
            res = prov.aggregate(keys, FP_AGGS, batch_size=bs)
            check_batches(res, bs)
            if bs:
                assert all(b.num_rows == bs for b in res.batches[:-1]), (keys, bs)
            check_groups(R, res.table(), keys, f"{source} {keys} batch {bs}")
    if source == "resident":
        for i in range(2):
            res, log = run(prov, ["s5000_n", "bp_n"], capfd=capfd)
            check_groups(R, res.table(), ["s5000_n", "bp_n"], f"repeat {i}")
        assert "result tail: one round trip" in log, log


# ---- GPU: DATE_BIN ---------------------------------------------------------------------------------------------------
BIN_WIDTHS = [1, 3, 7_000, 60_000, 3_600_000, 86_400_000, 86_400_001, W29]
BIN_COLUMNS = ["tdict_n", "tp_nn", "tdelta_n", "tfb_n", "dbin_n", "ip_nn"]


def _origins(R):
    after = max(int(R.key(c)[1].max()) for c in ("tdict_nn", "tp_nn", "tdelta_nn", "tfb_nn")) + 12_345
    return [0, -7_777_777_777, after, 1_234_567]


def check_bin(R, prov, keys, what, filters=(), sel=None):
    [b] = [k for k in keys if isinstance(k, DateBin)]
    ok, _ = bin_span(R, b.column, b.width_ms, b.origin_ms, sel)
    if not ok:
        with pytest.raises(QueryError) as e:
            prov.aggregate(list(keys), FP_AGGS, list(filters))
        assert e.value.code == L.PQ_ERR_UNSUPPORTED, (what, e.value)
        return False
    res = prov.aggregate(list(keys), FP_AGGS, list(filters))
    check_batches(res)
    check_groups(R, res.table(), list(keys), what, sel=sel)
    return True


@pytest.mark.gpu
@pytest.mark.parametrize("source", SOURCES)
def test_date_bin(R, gpu, source):
    """Widths 1 ms .. 2^29 + 1 ms, origins 0, negative, after every value and off the whole second, over dictionary, PLAIN,
    DELTA and fallback Timestamps and an Int64 column; a range that prunes row groups.  Where the bins in the scanned
    range exceed 2^24 or a value lies more than 2^52 ms from the origin the query is refused, else exact."""
    prov = gpu[source]
    verdicts = {True: 0, False: 0}
    for c in BIN_COLUMNS:
        for w in BIN_WIDTHS:
            for o in (_origins(R) if source == "resident" else _origins(R)[::3]) if c != "dbin_n" else [ORIGIN]:
                verdicts[check_bin(R, prov, [date_bin(w, c, o)], f"{source} {c} {w} {o}")] += 1
    assert verdicts[True] >= 30 and verdicts[False] >= 10, verdicts
    # a range that prunes row groups (tdelta falls row by row): bin 0 moves to the first live row group
    v, x, _ = R.key("tdelta_nn")
    cut = int(x[FILE_ROWS[0] + 150_000])
    sel = v & (x < cut)
    for w in (1, 7_000):
        assert check_bin(R, prov, [date_bin(w, "tdelta_nn", 5)], f"{source} pruned {w}", [col("tdelta_nn") < cut], sel)
        assert check_bin(R, prov, [date_bin(w, "tdelta_nn", 5), "s2_n"], f"{source} pruned {w} s2", [col("tdelta_nn") < cut], sel)


@pytest.mark.gpu
@pytest.mark.parametrize("source", SOURCES)
def test_date_bin_edges(R, gpu, source):
    """dbin at w = 2^29 + 1: exactly 2^24 bins over origin +- 2^52 ms (values at k * w - 1, k * w, k * w + 1, where the
    double reciprocal rounds both ways); w = 2^29 (2^24 + 1 bins) refused; the origin moved 1 ms either way puts a value
    outside 2^52 ms: refused.  Each refusal is followed by a correct answer."""
    prov = gpu[source]
    for c in ("dbin_nn", "dbin_n"):
        assert check_bin(R, prov, [date_bin(W29, c, ORIGIN)], f"{source} {c}")
        for w in FIX_WIDTHS:
            assert check_bin(R, prov, [date_bin(w, c, ORIGIN)], f"{source} {c} fix-up {w}")
        assert check_bin(R, prov, [date_bin(W29, c, ORIGIN), "bp_n"], f"{source} {c} bp_n")
        for w, o in ((1 << 29, ORIGIN), (W29, ORIGIN + 1), (W29, ORIGIN - 1)):
            assert not check_bin(R, prov, [date_bin(w, c, o)], f"{source} {c} {w} {o}")
            assert check_bin(R, prov, [date_bin(W29, c, ORIGIN)], f"{source} {c} after refusal")


@pytest.mark.gpu
def test_refusals(R, gpu, side_files):
    """Refused queries return an error code, and the context then answers the next query correctly: DATE_BIN over a
    file without statistics, DATE_BIN over a Float64 / Utf8 column, a non-positive width."""
    paths, schema, nref = side_files["nostats"]
    nprov = StandardTableProvider(paths, schema=schema)
    cases = [(nprov, [date_bin(1000, "ts")], L.PQ_ERR_UNSUPPORTED), (gpu["resident"], [date_bin(1000, "fp_n")], L.PQ_ERR_INVALID_ARG),
             (gpu["resident"], [date_bin(1000, "s33_n")], L.PQ_ERR_INVALID_ARG), (gpu["files"], [date_bin(0, "tp_nn")], L.PQ_ERR_INVALID_ARG)]
    for prov, keys, code in cases:
        with pytest.raises(QueryError) as e:
            prov.aggregate(keys, FP_AGGS)
        assert e.value.code == code, (keys, e.value)
        res = prov.aggregate(["ts"] if prov is nprov else ["s33_n"], FP_AGGS)
        check_groups(Ref(nref) if prov is nprov else R, res.table(), ["ts"] if prov is nprov else ["s33_n"], f"after {keys}")


# ---- regression tests ------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("source", SOURCES)
def test_string_key_bytes_of_tuples(R, gpu, source):
    """A Utf8 key in a tuple whose long values (4 KiB .. 9 000 bytes) occur in far more groups than the key's average
    value: the result block must hold their bytes in every group (it was sized as groups / card + 1 copies of the
    key's distinct bytes, and the gather wrote past it)."""
    prov = gpu[source]
    for keys in (["fdict_n", "s1_n", "splain_n", "brle_n"], ["splain_nn", "fdict_nn"], ["sdba_n", "idict_n", "bp_nn"]):
        res = prov.aggregate(keys, FP_AGGS)
        check_batches(res)
        check_groups(R, res.table(), keys, f"{source} {keys}")


@pytest.mark.gpu
def test_kscan_refuses_row_keys(R, gpu):
    """With every item on k_scan, a key column with pages without a dictionary (PLAIN fallback, PLAIN, DELTA) is
    refused with PQ_ERR_UNSUPPORTED, never read through a dictionary index it does not have; the next query answers."""
    prov = gpu["resident"]
    with env_vars({"PQB_FLAT_SCAN": 0}):
        for keys in (["sfb_n"], ["splain_nn"], ["sdba_n"], ["ip_n"], ["idelta_nn"], ["tfb_n"], ["s33_n", "tp_n"]):
            with pytest.raises(QueryError) as e:
                prov.aggregate(keys, FP_AGGS)
            assert e.value.code == L.PQ_ERR_UNSUPPORTED, (keys, e.value)
            res = prov.aggregate(["s33_n", "bp_n"], FP_AGGS)
            check_groups(R, res.table(), ["s33_n", "bp_n"], f"after {keys}")
