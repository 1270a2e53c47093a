"""Every value a projection returns, checked bit for bit against pyarrow's own reading of the same files.

A scan with a projection reads each selected row straight out of the flat store (`flat_value_at`), so it is the one
consumer that sees every value the flat-store build kernels write: dictionary indices of width 0 .. 17 (FJ_HYBRID),
8-byte PLAIN values (FJ_COPY8), PLAIN and RLE Booleans (FJ_BITS, FJ_HYBRID), PLAIN strings (FJ_BYTES, also the pages
after a dictionary falls back, and DELTA_(LENGTH_)BYTE_ARRAY pages rewritten as PLAIN), DELTA_BINARY_PACKED pages
(decoded on demand; FJ_VALID when they hold NULLs), each with and without NULLs, in all-NULL pages and an all-NULL row
group, and a column absent from one file.

Three files: v1 pages uncompressed, v2 pages, v1 pages under SNAPPY (pages sit in the arena at decompressed offsets).
Row groups of 100 003 rows, write batches of 97 rows, 4 KB pages of at most 3 000 rows: pages end off the 32-row grid
and start at other rows in other columns.  Two selectors choose the rows: `q` (PLAIN, uniform in 0 .. 999) and `blk`
(clustered: equal values run in blocks of 1 .. 5 000 rows).

The reference is `pq.read_table` of the files (the absent column filled with NULLs); the selected rows are computed in
numpy from `q` / `blk`.  Columns compare by validity and by bits: Float64 as uint64 (NaN sign and payload, -0.0),
Timestamp as int64, strings as bytes, Booleans as bits; values under NULL slots are not compared.  Every result batch
is also checked against itself: `validate(full=True)`, and its null_count against its own validity bitmap.

CPU: the files hold what the cases promise (encodings, page geometry, NULL layouts, long strings, long DBA prefixes,
NaN sign bits), and the numpy selection equals the C oracle's.  GPU: k_project at every selection density, batch
size, LIMIT and with __row_id; k_project_rows through ORDER BY ... LIMIT; the JSON egress against rows built from the
reference; and predicates, GROUP BY and MIN / MAX over NULL-free Boolean pages, whose last word holds bits past the
page's last row."""
import ctypes as C
import json
import os
import struct

import numpy as np
import pyarrow as pa
import pyarrow.compute as pc
import pyarrow.parquet as pq
import pytest

from oracle.oracle import Oracle
from parseable_b200 import _lib as L
from parseable_b200.query import DeviceTable, StandardTableProvider, col, count, count_star, max_, min_
from test_gpu_parity import _json_expect

SEED = 20261018
FILE_ROWS = (300_000, 260_000, 190_000)
N = sum(FILE_ROWS)
RG = 100_003                        # odd row groups
MAX_PAGE_ROWS = 3_000               # pages of narrow columns end here (3000 % 32 == 24)
PAGE_KW = dict(data_page_size=4096, write_batch_size=97, max_rows_per_page=MAX_PAGE_ROWS)
FILE_KW = (dict(data_page_version="1.0", compression="NONE"), dict(data_page_version="2.0", compression="NONE"),
           dict(data_page_version="1.0", compression="SNAPPY"))
I64_MIN, I64_MAX = -(1 << 63), (1 << 63) - 1
ALL_NULL_RG = 1                     # every column but the selectors and `k` is NULL in this (global) row group
NULL_RUN = 7_000                    # NULL-bearing variants: a run of NULLs (>= two whole pages) in row group 4
PREF = ["", "a", "A", "ab", "é", "x%", "日本", "𝄞"]
LONG_LENS = (4093, 4094, 4095, 4096, 4097, 4098, 4099, 4100, 4200, 9000)   # around the 4 KiB walker tile (kFlatTile)
DBA_PREFIX = "tenant/" + "p" * 34 + "/zone-"                                 # sorted DBA values share > 32 bytes


def _bits(x: float) -> int:
    return struct.unpack("<Q", struct.pack("<d", x))[0]


def _f64(bits: int) -> float:
    return struct.unpack("<d", struct.pack("<Q", bits))[0]


# NaNs of both signs with distinct payloads (a signalling one too), subnormals, zeros of both signs, infinities
F_SPECIALS = np.array([_f64(b) for b in (0x7FF8000000000000, 0xFFF8000000000000, 0x7FF0000000000001, 0xFFF00000DEADBEEF,
                                          0x7FFFFFFFFFFFFFFF, 0xFFF8000000012345)] +
                      [0.0, -0.0, np.inf, -np.inf, 5e-324, -5e-324, 2.2250738585072009e-308, -2.2250738585072014e-308,
                       1.7976931348623157e308, -1.5, 0.1])

# base name -> (kind, flat-store case); every base is written twice: `<base>_nn` (NULL-free) and `<base>_n` (~3 % NULLs)
BASES = {
    "s1": ("str", "index0"), "i1": ("i64", "index0"), "f1": ("f64", "index0"),
    "s2": ("str", "index"), "s3": ("str", "index"), "s33": ("str", "index"), "s600": ("str", "index"),
    "s5000": ("str", "index"), "s70k": ("str", "index"),
    "idict": ("i64", "dict8"), "fdict": ("f64", "dict8"), "tdict": ("ts", "dict8"),
    "sfb": ("str", "fallback"), "splain": ("str", "bytes"),
    "sdba": ("str", "dba"), "sdlba": ("str", "dlba"),
    "ip": ("i64", "plain8"), "fp": ("f64", "plain8"), "tp": ("ts", "plain8"),
    "tdelta": ("ts", "delta"), "idelta": ("i64", "delta"),
    "bp": ("bool", "bits"), "brle": ("bool", "rlebits"),
}
ENCODING = {"ip": "PLAIN", "fp": "PLAIN", "tp": "PLAIN", "splain": "PLAIN", "bp": "PLAIN", "sdba": "DELTA_BYTE_ARRAY",
            "sdlba": "DELTA_LENGTH_BYTE_ARRAY", "tdelta": "DELTA_BINARY_PACKED", "idelta": "DELTA_BINARY_PACKED", "brle": "RLE"}
CARDS = {"s1": 1, "s2": 2, "s3": 3, "s33": 33, "s600": 600, "s5000": 5000, "s70k": 70_000}
WIDTHS = {"s1": 0, "s2": 1, "s3": 2, "s33": 6, "s600": 10, "s5000": 13, "s70k": 17}   # index bit width per chunk
VARIANTS = [f"{b}_{v}" for b in BASES for v in ("nn", "n")]
SELECTORS = {"q": "PLAIN", "blk": "PLAIN"}
COLUMNS = VARIANTS + ["opt", "k", "q", "blk"]
# A query references at most 12 columns (kMaxCols): the projections go in groups of <= 10 (the selectors beside them).
# The strings over 4 KiB have a group of their own: a projection sizes its string bytes as rows x the column's longest
# value and refuses more than 2 GiB, so that group's scans keep at most LONG_CAP rows.
LONG = ["sfb_nn", "sfb_n", "splain_nn", "splain_n"]
LONG_CAP = 49_999
_SHORT = [c for c in VARIANTS if c not in LONG] + ["opt", "k"]
GROUPS = [_SHORT[i:i + 10] for i in range(0, len(_SHORT), 10)] + [LONG]


def _capped(cols, ids, limit=None):
    """(LIMIT, rows kept) of a scan of `cols` over the selection `ids`."""
    if cols == LONG and len(ids) > LONG_CAP and (limit is None or limit > LONG_CAP):
        limit = LONG_CAP
    return limit, ids if limit is None else ids[:limit]


# every flat-store case and the column types that must reach it
CASES = {"index0": {"str", "i64", "f64"}, "index": {"str"}, "dict8": {"i64", "f64", "ts"}, "fallback": {"str"}, "bytes": {"str"},
         "dba": {"str"}, "dlba": {"str"}, "plain8": {"i64", "f64", "ts"}, "delta": {"ts", "i64"}, "bits": {"bool"},
         "rlebits": {"bool"}}
TYPES = {"str": pa.string(), "i64": pa.int64(), "f64": pa.float64(), "ts": pa.timestamp("ms"), "bool": pa.bool_()}


def _base(name):
    return name.rsplit("_", 1)[0]


# ---- data ------------------------------------------------------------------------------------------------------------
def _rg_index():
    """Global row group of every row, and the first row of every file."""
    rg, starts, base, s = np.empty(N, np.int64), [], 0, 0
    for n in FILE_ROWS:
        rg[s:s + n] = base + np.arange(n) // RG
        starts.append(s)
        base += -(-n // RG)
        s += n
    return rg, starts


def _vocab(n):
    if n == 1:
        return ["only-value-é"]
    return [""] + [f"{PREF[i % len(PREF)]}{i:x}" for i in range(1, n)]


def _str_array(codes, vocab):
    return pa.DictionaryArray.from_arrays(pa.array(codes, pa.int32()), pa.array(vocab, pa.string())).cast(pa.string())


def _values(base, rng, rg):
    """One column's N values (a pyarrow array without NULLs) and the rows that must stay valid."""
    kind, case = BASES[base]
    keep = np.zeros(N, bool)
    if base in CARDS:
        card = CARDS[base]
        if card == 70_000:   # every value in every row group: 17-bit indices
            codes = (np.arange(N) * 7919 + rg * 13) % card
        else:
            codes = rng.integers(0, card, N)
        return _str_array(codes, _vocab(card)), keep
    if base == "i1":
        return pa.array(np.full(N, I64_MIN, np.int64)), keep
    if base == "f1":
        return pa.array(np.full(N, -0.0)), keep
    if base == "idict":
        pool = np.concatenate([[I64_MIN, I64_MAX, 0, -1, 1], rng.integers(-10**12, 10**12, 295)]).astype(np.int64)
        return pa.array(pool[rng.integers(0, len(pool), N)]), keep
    if base == "fdict":
        pool = np.concatenate([F_SPECIALS, np.round(rng.standard_normal(200) * 100, 2)])
        return pa.array(pool[rng.integers(0, len(pool), N)]), keep
    if base == "tdict":
        pool = np.concatenate([[-1, 0, -86_400_000, -2_208_988_800_000, 1_700_000_000_000],
                               rng.integers(-2_200_000_000_000, 4_000_000_000_000, 495)]).astype(np.int64)
        return pa.array(pool[rng.integers(0, len(pool), N)], pa.timestamp("ms")), keep
    if base in ("sfb", "splain"):
        # long, nearly distinct strings: the dictionary passes 1 MB early in every chunk and falls back to PLAIN; strings
        # longer than the walker tile at fixed rows late in every row group (inside the PLAIN pages)
        tails = ["", "ü", "€", "𝄞", "common/prefix/", "日本語"]
        vocab = [""] + [f"{tails[i % 6]}{'ab' * (i % 17)}{i:07d}{tails[(i // 6) % 6]}" for i in range(1, 300_000)]
        # they start with the largest leading bytes of the column, so that an ORDER BY ... DESC LIMIT keeps them
        longs = ["𝄞é" + (("é" * ((n - 6) // 2) + "x" * (n % 2)) if j % 3 == 1 else ("Z" * (n - 6))) for j, n in enumerate(LONG_LENS)]
        codes = rng.integers(0, len(vocab), N)
        for s in np.flatnonzero(np.diff(rg, prepend=-1)):
            rows = s + 60_000 + 97 * np.arange(len(longs)) + 13
            rows = rows[rows < N]
            rows = rows[rg[rows] == rg[s]]
            codes[rows] = len(vocab) + np.arange(len(rows))
            keep[rows] = True
        return _str_array(codes, vocab + longs), keep
    if base in ("sdba", "sdlba"):
        pool = [""] + ["".join(chr(97 + int(c)) for c in rng.integers(0, 26, int(k))) for k in rng.integers(0, 24, 20_000)]
        codes = rng.integers(0, len(pool), N)
        out = np.array(pool, dtype=object)[codes]
        srt = (np.arange(N) // 4000) % 2 == 0      # sorted blocks: neighbours share > 32 bytes
        out[srt] = [f"{DBA_PREFIX}{i // 7:07d}/δ" for i in np.flatnonzero(srt)]
        return pa.array(out, pa.string()), keep
    if base == "ip":
        v = rng.integers(I64_MIN, I64_MAX, N, dtype=np.int64, endpoint=True)
        v[rng.integers(0, N, 300)] = I64_MIN
        v[rng.integers(0, N, 300)] = I64_MAX
        v[rng.integers(0, N, 300)] = 0
        return pa.array(v), keep
    if base == "fp":
        v = rng.standard_normal(N) * 10.0 ** rng.integers(-300, 300, N)
        sp = rng.integers(0, N, N // 50)
        v[sp] = F_SPECIALS[rng.integers(0, len(F_SPECIALS), len(sp))]
        return pa.array(v), keep
    if base == "tp":
        return pa.array(rng.integers(-2_200_000_000_000, 4_000_000_000_000, N), pa.timestamp("ms")), keep
    if base == "tdelta":   # Parseable's p_timestamp: newest first
        return pa.array(1_700_000_000_000 - np.cumsum(rng.integers(0, 5, N)), pa.timestamp("ms")), keep
    if base == "idelta":   # random over the whole range: the deltas wrap
        return pa.array(rng.integers(I64_MIN, I64_MAX, N, dtype=np.int64, endpoint=True)), keep
    if kind == "bool":
        return pa.array(rng.random(N) < 0.5), keep
    raise AssertionError(base)


def _blocks(rng):
    """blk: block ids in row order, block lengths 1 .. 5000 (one in six of length 1)."""
    lens = rng.integers(1, 5001, N // 1000 + 10)
    lens[rng.random(len(lens)) < 1 / 6] = 1
    return np.repeat(np.arange(len(lens), dtype=np.int64), lens)[:N]


def make_data():
    rng = np.random.default_rng(SEED)
    rg, starts = _rg_index()
    cols, valid = {}, {}
    run0 = np.flatnonzero(rg == 4)[0] + 11_111
    for i, base in enumerate(BASES):
        arr, keep = _values(base, rng, rg)
        for var in ("nn", "n"):
            v = np.ones(N, bool)
            if var == "n":
                v = rng.random(N) >= 0.03
                lo = run0 + 1_009 * i                     # the all-NULL pages start at other rows in other columns
                v[lo:lo + NULL_RUN] = False
                v[keep] = True
            v[rg == ALL_NULL_RG] = False
            cols[f"{base}_{var}"], valid[f"{base}_{var}"] = arr, v
    opt = rng.random(N) >= 0.03
    opt[starts[2]:] = False
    cols["opt"], valid["opt"] = _str_array(rng.integers(0, 9, N), _vocab(9)), opt
    cols["k"], valid["k"] = _str_array(rng.integers(0, 7, N), [f"k{i}" for i in range(7)]), np.ones(N, bool)
    cols["q"], valid["q"] = pa.array(rng.integers(0, 1000, N)), np.ones(N, bool)
    cols["blk"], valid["blk"] = pa.array(_blocks(rng)), np.ones(N, bool)
    return cols, valid


def _masked(arr: pa.Array, v: np.ndarray) -> pa.Array:
    if v.all():
        return arr
    return pc.if_else(pa.array(v), arr, pa.scalar(None, arr.type))


@pytest.fixture(scope="module")
def pdata(built, data_dir):
    cols, valid = make_data()
    paths, lo = [], 0
    for i, n in enumerate(FILE_ROWS):
        names = [c for c in COLUMNS if not (c == "opt" and i == 2)]
        t = pa.table({c: _masked(cols[c].slice(lo, n), valid[c][lo:lo + n]) for c in names})
        enc = {c: ENCODING[_base(c)] for c in names if _base(c) in ENCODING}
        enc.update(SELECTORS)
        p = os.path.join(data_dir, f"project_paths_{i}.parquet")
        pq.write_table(t, p, row_group_size=RG, use_dictionary=[c for c in names if c not in enc], column_encoding=enc,
                       **FILE_KW[i], **PAGE_KW)
        paths.append(p)
        lo += n
    schema = pa.schema([(c, TYPES[BASES[_base(c)][0]] if c in VARIANTS else pa.string() if c in ("opt", "k") else pa.int64())
                        for c in COLUMNS])
    return cols, valid, paths, schema


def reference(paths, schema) -> pa.Table:
    """pyarrow's reading of the files, concatenated; the column absent from a file reads as NULL."""
    parts = []
    for p in paths:
        t = pq.read_table(p)
        for f in schema:
            if f.name not in t.column_names:
                t = t.append_column(f.name, pa.nulls(t.num_rows, f.type))
        parts.append(t.select(schema.names))
    return pa.concat_tables(parts).combine_chunks()


@pytest.fixture(scope="module")
def ref(pdata):
    return reference(pdata[2], pdata[3])


# ---- selections ------------------------------------------------------------------------------------------------------
def selections(ref: pa.Table):
    """name -> (predicate, selected rows).  Densities none, one row, 0.1 %, 50 %, 99.9 %, all, and clustered ones whose
    runs start and end inside words, pages and work items."""
    q, blk = ref["q"].to_numpy(), ref["blk"].to_numpy()
    lens = np.bincount(blk)
    starts = np.r_[0, np.cumsum(lens)[:-1]]
    one = int(np.flatnonzero((lens == 1) & (starts > FILE_ROWS[0] + 1000))[0])
    lo, hi = int(blk[FILE_ROWS[0] - 40_000]), int(blk[FILE_ROWS[0] + 30_000])   # across the first file boundary
    rng = np.random.default_rng(SEED + 1)
    few = sorted(int(b) for b in rng.choice(int(blk.max()) + 1, 6, replace=False))
    e_few = col("blk") == few[0]
    for b in few[1:]:
        e_few = e_few | (col("blk") == b)
    cases = {
        "none": (col("q") < 0, q < 0),
        "one": (col("blk") == one, blk == one),
        "sparse": (col("q") == 7, q == 7),
        "half": (col("q") < 500, q < 500),
        "dense": (col("q") != 7, q != 7),
        "all": (col("q") >= 0, q >= 0),
        "cluster": ((col("blk") >= lo) & (col("blk") <= hi), (blk >= lo) & (blk <= hi)),
        "blocks": (e_few, np.isin(blk, few)),
        "cluster_half": ((col("blk") >= lo) & (col("blk") <= hi) & (col("q") < 500), (blk >= lo) & (blk <= hi) & (q < 500)),
    }
    return {k: (e, np.flatnonzero(m)) for k, (e, m) in cases.items()}


# ---- comparison ------------------------------------------------------------------------------------------------------
def _valid(a: pa.Array) -> np.ndarray:
    return a.is_valid().to_numpy(zero_copy_only=False)


def _words(a: pa.Array) -> np.ndarray:
    """The raw value of every slot: uint64 bits of 8-byte values, 0 / 1 for Booleans."""
    buf = a.buffers()[1]
    if pa.types.is_boolean(a.type):
        return np.unpackbits(np.frombuffer(buf, np.uint8), bitorder="little")[a.offset:a.offset + len(a)].astype(np.uint64)
    return np.frombuffer(buf, np.uint64, count=a.offset + len(a))[a.offset:]


def assert_same(got, want, what):
    """got and want: the same values by validity and by bits; slots under NULL are not compared."""
    got = got.combine_chunks() if isinstance(got, pa.ChunkedArray) else got
    want = want.combine_chunks() if isinstance(want, pa.ChunkedArray) else want
    assert got.type == want.type, (what, got.type, want.type)
    assert len(got) == len(want), (what, len(got), len(want))
    gv, wv = _valid(got), _valid(want)
    bad = np.flatnonzero(gv != wv)
    assert bad.size == 0, (what, "validity", bad.size, int(bad[0]))
    if pa.types.is_string(want.type):
        va = pa.array(wv)
        g = pc.if_else(va, got.cast(pa.binary()), pa.scalar(b"", pa.binary()))
        w = pc.if_else(va, want.cast(pa.binary()), pa.scalar(b"", pa.binary()))
        if not g.equals(w):
            bad = np.flatnonzero(~pc.equal(g, w).to_numpy(zero_copy_only=False))
            i = int(bad[0])
            raise AssertionError(f"{what}: {bad.size} strings differ, first at {i}: {g[i].as_py()[:80]!r} vs {w[i].as_py()[:80]!r}")
        return
    g, w = np.where(gv, _words(got), 0), np.where(wv, _words(want), 0)
    bad = np.flatnonzero(g != w)
    if bad.size:
        i = int(bad[0])
        raise AssertionError(f"{what}: {bad.size} values differ, first at {i}: {int(g[i]):#018x} vs {int(w[i]):#018x}")


def check_batches(res, batch_size=0):
    """Every batch on its own: valid Arrow data, and each column's null_count equals the zero bits of its own bitmap."""
    for bi, b in enumerate(res.batches):
        b.validate(full=True)
        if batch_size:
            assert b.num_rows <= batch_size, (bi, b.num_rows, batch_size)
        for ci, c in enumerate(b.columns):
            vb = c.buffers()[0]
            zeros = 0 if vb is None else len(c) - int(np.unpackbits(np.frombuffer(vb, np.uint8), bitorder="little")[c.offset:c.offset + len(c)].sum())
            assert c.null_count == zeros, (bi, b.schema.names[ci], c.null_count, zeros)


def _table(res) -> pa.Table:
    return res.table() if res.batches else pa.table({})


def check_projection(res, ref, cols, ids, row_ids, batch_size=0, what=""):
    check_batches(res, batch_size)
    got = _table(res)
    assert sum(b.num_rows for b in res.batches) == len(ids), (what, "rows", got.num_rows, len(ids))
    if not len(ids):
        return
    assert got.column_names == cols + (["__row_id"] if row_ids else []), (what, got.column_names)
    want = ref.select(cols).take(pa.array(ids))
    for c in cols:
        assert_same(got[c], want[c], f"{what} {c}")
    if row_ids:
        assert np.array_equal(got["__row_id"].to_numpy(), ids), (what, "__row_id")


# ---- CPU -------------------------------------------------------------------------------------------------------------
ENC_CODE = {"PLAIN": 0, "PLAIN_DICTIONARY": 2, "RLE": 3, "DELTA_BINARY_PACKED": 5, "DELTA_LENGTH_BYTE_ARRAY": 6,
            "DELTA_BYTE_ARRAY": 7, "RLE_DICTIONARY": 8}


def _describe(path):
    lib = L.load()
    f = L.PqFile(path=path.encode())
    n = lib.pq_file_describe(C.byref(f), None, 0)
    buf = C.create_string_buffer(n + 1)
    lib.pq_file_describe(C.byref(f), buf, n + 1)
    return json.loads(buf.value.decode())


def data_pages(paths, schema):
    """name -> [(first global row, rows, encoding code)] of every data page, from the library's own page walk."""
    out, base = {}, 0
    for p, n in zip(paths, FILE_ROWS):
        d = _describe(p)
        names = pq.ParquetFile(p).schema_arrow.names
        r0 = base
        for rgd in d["row_groups"]:
            nrows = None
            for j, name in enumerate(names):
                r = r0
                for pg in rgd["columns"][j]["pages"]:
                    if pg["type"] in (0, 3):
                        out.setdefault(name, []).append((r, pg["num_values"], pg["encoding"]))
                        r += pg["num_values"]
                assert nrows is None or r - r0 == nrows, (p, name)
                nrows = r - r0
            r0 += nrows
        assert r0 == base + n, p
        base += n
    return out


def test_data_layout(pdata, ref):
    """The files hold every case of the table: encodings, pages off the 32-row grid, all-NULL / NULL-free /
    NULL-bearing pages per case, strings over 4 KiB in PLAIN pages, DBA prefixes over 32 bytes, NaN sign bits."""
    cols, valid, paths, schema = pdata
    assert ref.num_rows == N and ref.column_names == COLUMNS
    covered = {}
    for base, (kind, case) in BASES.items():
        covered.setdefault(case, set()).add(kind)
        for name in (f"{base}_nn", f"{base}_n"):
            assert ref.schema.field(name).type == TYPES[kind], name
    assert covered == CASES, covered
    assert sorted(WIDTHS.values()) == [0, 1, 2, 6, 10, 13, 17]
    assert "opt" not in pq.ParquetFile(paths[2]).schema_arrow.names
    pages = data_pages(paths, schema)
    enc = {}
    for p in paths:
        md = pq.ParquetFile(p).metadata
        for g in range(md.num_row_groups):
            for j in range(md.num_columns):
                c = md.row_group(g).column(j)
                enc.setdefault(c.path_in_schema, set()).update(c.encodings)
    for name in VARIANTS:
        base = _base(name)
        case = BASES[base][1]
        e = enc[name]
        if case in ("index0", "index", "dict8"):
            assert "RLE_DICTIONARY" in e, (name, e)
            assert all(pe == ENC_CODE["RLE_DICTIONARY"] for _, _, pe in pages[name]), name
        elif case == "fallback":
            assert {"RLE_DICTIONARY", "PLAIN"} <= e, (name, e)
        elif case in ("bytes", "plain8", "bits"):
            assert "RLE_DICTIONARY" not in e and all(pe == 0 for _, _, pe in pages[name]), (name, e)
        else:
            want = {"dba": "DELTA_BYTE_ARRAY", "dlba": "DELTA_LENGTH_BYTE_ARRAY", "delta": "DELTA_BINARY_PACKED", "rlebits": "RLE"}[case]
            assert all(pe == ENC_CODE[want] for _, _, pe in pages[name]), (name, e)
    for s in ("q", "blk"):
        assert all(pe == 0 for _, _, pe in pages[s]), s
    # index widths: one chunk's dictionary holds the distinct values it met
    rg, _ = _rg_index()
    sel = rg == 0
    for base, w in WIDTHS.items():
        k = len(pc.unique(ref[f"{base}_nn"].filter(pa.array(sel))))
        assert (k - 1).bit_length() == w, (base, k, w)
    # pages per case: off the 32-row grid (not only the last of a chunk), all-NULL, NULL-free and NULL-bearing ones
    vmask = {c: _valid(ref[c]) for c in VARIANTS}
    rg_ends = set(np.flatnonzero(np.diff(rg)) + 1) | {N}
    for base in BASES:
        kinds = set()
        offgrid = 0
        for name in (f"{base}_nn", f"{base}_n"):
            v = vmask[name]
            cum = np.r_[0, np.cumsum(~v)]
            for r0, n, _ in pages[name]:
                nulls = int(cum[r0 + n] - cum[r0])
                kinds.add("all_null" if nulls == n else "null_free" if nulls == 0 else "nulls")
                offgrid += n % 32 != 0 and r0 + n not in rg_ends and r0 % 32 != 0   # not the last page of a chunk
        assert kinds == {"all_null", "null_free", "nulls"}, (base, kinds)
        assert offgrid >= 10, (base, offgrid)
    # all-NULL pages inside an otherwise valid chunk (not the all-NULL row group)
    for name in (f"{b}_n" for b in BASES):
        v = vmask[name]
        assert any(not v[r0:r0 + n].any() and rg[r0] != ALL_NULL_RG for r0, n, _ in pages[name]), name
    # PLAIN Booleans: the NULL-free pages end inside a 32-bit word (bits after the last row are not the page's)
    assert any(n % 32 and vmask["bp_nn"][r0:r0 + n].all() for r0, n, _ in pages["bp_nn"])
    # strings over 4 KiB, some at 4093 .. 4100 bytes, in PLAIN pages of the fallback and the PLAIN-only columns
    for name in ("sfb_nn", "sfb_n", "splain_nn", "splain_n"):
        lens = pc.binary_length(ref[name].cast(pa.binary())).to_numpy(zero_copy_only=False)
        lens = np.nan_to_num(lens.astype(np.float64)).astype(np.int64)
        plain = [(r0, n) for r0, n, pe in pages[name] if pe == 0]
        long_rows = {int(r) for r in np.flatnonzero(lens >= min(LONG_LENS))}
        in_plain = {r for r in long_rows if any(r0 <= r < r0 + n for r0, n in plain)}
        assert len(in_plain) >= 30 and {int(lens[r]) for r in in_plain} == set(LONG_LENS), name
        assert (lens == 0).sum() > 0 and ref[name].null_count >= (RG if name.endswith("_nn") else RG + NULL_RUN), name
    # DELTA_BYTE_ARRAY: neighbours in the same page share prefixes longer than 32 bytes
    for name in ("sdba_nn", "sdba_n"):
        vals = ref[name].to_pylist()
        best = max(len(os.path.commonprefix([a.encode(), b.encode()])) for a, b in zip(vals[:50_000], vals[1:50_001])
                   if a is not None and b is not None)
        assert best > 32, (name, best)
        assert "" in vals[:50_000], name
    # the read-back keeps every NaN's sign and payload, and -0.0
    for name in ("fp_nn", "fp_n"):
        w = _words(ref[name].combine_chunks())
        v = vmask[name]
        src = np.where(valid[name], _words(cols[name]), 0)
        assert np.array_equal(np.where(v, w, 0), src), name
        for b in (0xFFF8000000000000, 0x7FF0000000000001, 0xFFF00000DEADBEEF, 0x8000000000000000):
            assert (w[v] == b).any(), (name, hex(b))
    fd = _words(ref["fdict_nn"].combine_chunks())[vmask["fdict_nn"]]
    assert (fd == 0x8000000000000000).any() and ((fd >> 63 == 1) & ((fd >> 52) & 0x7FF == 0x7FF) & (fd & ((1 << 52) - 1) != 0)).any()
    assert (_words(ref["f1_nn"].combine_chunks())[vmask["f1_nn"]] == 0x8000000000000000).all()
    # Timestamps before 1970 in the PLAIN and the dictionary column; INT64_MIN / MAX in the PLAIN Int64
    for name in ("tp_nn", "tdict_nn"):
        assert (ref[name].cast(pa.int64()).to_numpy(zero_copy_only=False)[vmask[name]] < 0).any(), name
    ip = _words(ref["ip_nn"].combine_chunks()).view(np.int64)[vmask["ip_nn"]]
    assert (ip == I64_MIN).any() and (ip == I64_MAX).any()
    td = ref["tdelta_nn"].cast(pa.int64()).to_numpy(zero_copy_only=False)[vmask["tdelta_nn"]]
    assert (np.diff(td) <= 0).all()
    # the selections: every density, a single row, runs cut inside words and pages
    sels = selections(ref)
    sizes = {k: len(ids) for k, (_, ids) in sels.items()}
    assert sizes["none"] == 0 and sizes["one"] == 1 and sizes["all"] == N
    assert 0 < sizes["sparse"] < N // 500 and N // 3 < sizes["half"] < 2 * N // 3 and N - N // 500 < sizes["dense"] < N
    ids = sels["cluster"][1]
    assert ids[0] % 32 and (ids[-1] + 1) % 32 and ids[0] < FILE_ROWS[0] < ids[-1]
    assert 1 in np.bincount(ref["blk"].to_numpy())


def test_reference_matches_oracle(pdata, ref):
    """The C oracle's row ids for the selector predicates equal the numpy selection."""
    ora = Oracle(ref.select(["q", "blk"]))
    for name, (e, ids) in selections(ref).items():
        assert np.array_equal(ora.row_ids([e]), ids), name


# ---- GPU -------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def gpu(pdata):
    _, _, paths, schema = pdata
    table = DeviceTable(paths, schema.names)
    yield {"resident": StandardTableProvider(table, schema=schema), "files": StandardTableProvider(paths, schema=schema)}
    table.close()


SOURCES = ["resident", "files"]


@pytest.mark.gpu
@pytest.mark.parametrize("source", SOURCES)
def test_project_every_density(ref, gpu, source):
    """k_project: every column at every selection density, with and without __row_id."""
    prov = gpu[source]
    for k, (name, (e, ids)) in enumerate(selections(ref).items()):
        for gi, cols in enumerate(GROUPS):
            row_ids = (k + gi) % 2 == 1
            limit, want = _capped(cols, ids)
            res = prov.scan(projection=cols, filters=[e], row_ids=row_ids, limit=limit)
            assert res.metrics["rows_selected"] == len(ids) if limit is None else res.metrics["rows_selected"] >= len(want), (source, name)
            check_projection(res, ref, cols, want, row_ids, what=f"{source} {name} group {gi}")


@pytest.mark.gpu
@pytest.mark.parametrize("source", SOURCES)
def test_project_batches_and_limits(ref, gpu, source):
    """Batches of 97 and 500 rows over whole selections; 1, 31, 32 and 33 rows under a LIMIT; LIMITs that end inside a
    word and inside a batch; one run polled batch by batch."""
    prov = gpu[source]
    sels = selections(ref)
    for name in ("half", "cluster_half"):
        e, ids = sels[name]
        for bs in (97, 500):
            for gi, cols in enumerate(GROUPS):
                limit, want = _capped(cols, ids)
                res = prov.scan(projection=cols, filters=[e], batch_size=bs, row_ids=gi == 0, limit=limit)
                check_projection(res, ref, cols, want, gi == 0, bs, f"{source} {name} batch {bs} group {gi}")
    e, ids = sels["dense"]
    for bs, limit in ((1, 2345), (31, 2345), (32, 3001), (33, 2048), (0, 1000), (500, 4321)):
        for gi, cols in enumerate(GROUPS):
            res = prov.scan(projection=cols, filters=[e], limit=limit, batch_size=bs, row_ids=True)
            check_projection(res, ref, cols, ids[:limit], True, bs, f"{source} limit {limit} batch {bs} group {gi}")
    e, ids = sels["blocks"]
    assert 3 < len(ids) < LONG_CAP
    for gi, cols in enumerate(GROUPS):
        res = prov.scan(projection=cols, filters=[e], limit=len(ids) - 3, row_ids=True)
        check_projection(res, ref, cols, ids[:len(ids) - 3], True, 0, f"{source} blocks limit group {gi}")
    e, ids = sels["cluster"]
    res = prov.scan(projection=GROUPS[1], filters=[e], batch_size=777, poll=True, row_ids=True)
    assert len(res.batches) == -(-len(ids) // 777)
    check_projection(res, ref, GROUPS[1], ids, True, 777, f"{source} poll")


def _desc_order(vals):
    """Stable DESC NULLS LAST order over Python values (bytes for strings); equal values keep scan order."""
    return sorted(range(len(vals)), key=lambda i: (vals[i] is not None, vals[i] if vals[i] is not None else b""), reverse=True)


@pytest.mark.gpu
@pytest.mark.parametrize("source", SOURCES)
def test_project_rows_ordered(ref, gpu, source):
    """k_project_rows / k_project_bytes: ORDER BY q (and a string column) ... LIMIT gathers every column kind through
    row handles; the expected rows are a stable host sort of the reference selection."""
    prov = gpu[source]
    sels = selections(ref)
    q = ref["q"].to_numpy()
    for name, limit in (("half", 3000), ("all", 4097), ("cluster", 2500)):
        e, ids = sels[name]
        want = ids[np.argsort(q[ids], kind="stable")[:limit]]
        for gi, cols in enumerate(GROUPS):
            res = prov.scan(projection=cols, filters=[e], limit=limit, row_ids=True, order_by=[("q", "asc")],
                            batch_size=1000 if gi == 1 else 0)
            check_projection(res, ref, cols, want, True, 1000 if gi == 1 else 0, f"{source} order q {name} group {gi}")
    e, ids = sels["half"]
    sv = ref["sfb_n"].take(pa.array(ids)).cast(pa.binary()).to_pylist()
    want = ids[np.array(_desc_order(sv)[:2000], np.int64)]
    lens = pc.binary_length(ref["sfb_n"].take(pa.array(want)).cast(pa.binary())).to_numpy(zero_copy_only=False)
    assert (lens > 4096).sum() >= 10      # the strings longer than the walker tile are among the kept rows
    for gi, cols in enumerate(GROUPS):
        res = prov.scan(projection=cols, filters=[e], limit=2000, row_ids=True, order_by=[("sfb_n", "desc", False)])
        check_projection(res, ref, cols, want, True, 0, f"{source} order sfb_n group {gi}")


def _json_rows_expect(ref, cols, ids, row_ids):
    t = ref.take(pa.array(ids)).select(cols)
    if row_ids:
        t = t.append_column("__row_id", pa.array(ids, pa.int64()))
    return _json_expect(t)


def check_json(res, ref, cols, ids, row_ids, what):
    got = res.to_json()
    want = _json_rows_expect(ref, cols, ids, row_ids)
    assert len(got) == len(want), (what, len(got), len(want))
    fcols = [c for c in cols if pa.types.is_floating(ref.schema.field(c).type)]
    for i, (g, w) in enumerate(zip(got, want)):
        assert g == w, (what, i, {k: (g.get(k), w.get(k)) for k in set(g) | set(w) if g.get(k) != w.get(k)})
        for c in fcols:   # -0.0 == 0.0: compare the parsed doubles by their bits
            if w.get(c) is not None:
                assert _bits(float(g[c])) == _bits(w[c]), (what, i, c, g[c], w[c])


@pytest.mark.gpu
@pytest.mark.parametrize("source", SOURCES)
def test_json_egress(ref, gpu, source):
    """json='array' / 'lines' over the same projections, parsed and compared with rows built from the reference: NULLs
    leave their key out, non-finite floats are null, -0.0 stays -0.0, Timestamp(ms) in chrono's text (before 1970
    too), __row_id when asked for."""
    prov = gpu[source]
    sels = selections(ref)
    cases = [("sparse", 0), ("cluster_half", 1)] if source == "resident" else [("sparse", 0)]
    for name, batch_rows in cases:
        e, ids = sels[name]
        ids = ids[:20_000]
        for gi, cols in enumerate(GROUPS):
            for mode in ("array", "lines"):
                row_ids = (gi + (mode == "lines")) % 2 == 1
                res = prov.scan(projection=cols, filters=[e], limit=len(ids), row_ids=row_ids, json=mode,
                                batch_size=977 if batch_rows else 0)
                assert res.json_text[:1] == (b"[" if mode == "array" else b"{"), (name, mode)
                check_json(res, ref, cols, ids, row_ids, f"{source} {name} {mode} group {gi}")


# ---- NULL-free Boolean pages: the bits after a page's last row --------------------------------------------------------
BOOLS = ["bp_nn", "brle_nn", "bp_n", "brle_n"]


def _bool_planes(ref, name):
    a = ref[name].combine_chunks()
    return _valid(a), _words(a).astype(bool)


def _k_codes(ref):
    return np.array([int(s[1:]) for s in ref["k"].to_pylist()], np.int64)


@pytest.mark.gpu
@pytest.mark.parametrize("source", SOURCES)
def test_boolean_page_tails(ref, gpu, source):
    """PLAIN Boolean pages without NULLs are copied as whole 32-bit words, so the bits after a page's last row are
    whatever bytes follow the page.  Every reader must mask them: predicates (count, row ids, grouped COUNT), GROUP BY
    the Boolean, and MIN / MAX of it per group, against numpy on the reference."""
    prov = gpu[source]
    kc = _k_codes(ref)
    q = ref["q"].to_numpy()
    for name in BOOLS:
        v, x = _bool_planes(ref, name)
        preds = {
            "true": (col(name) == True, v & x),                       # noqa: E712
            "false": (col(name) == False, v & ~x),                    # noqa: E712
            "not_true": (~(col(name) == True), v & ~x),               # noqa: E712
            "ne_false": (col(name) != False, v & x),                  # noqa: E712
            "is_null": (col(name).is_null(), ~v),
            "false_half": ((col(name) == False) & (col("q") < 500), v & ~x & (q < 500)),   # noqa: E712
            "not_or": (~((col(name) == True) | (col("q") < 100)), v & ~x & (q >= 100)),      # noqa: E712
        }
        for pname, (e, m) in preds.items():
            what = f"{source} {name} {pname}"
            ids = np.flatnonzero(m)
            assert prov.scan(filters=[e], count_only=True).metrics["rows_selected"] == len(ids), what
            res = prov.scan(filters=[e])
            got = np.concatenate([b.column(0).to_numpy() for b in res.batches]) if res.batches else np.zeros(0, np.int64)
            assert np.array_equal(got, ids), (what, len(got), len(ids))
            t = prov.aggregate(["k"], [count_star(), count(name)], [e]).table()
            want_n = np.bincount(kc[m], minlength=7)
            want_c = np.bincount(kc[m & v], minlength=7)
            got_n, got_c = np.zeros(7, np.int64), np.zeros(7, np.int64)
            if t.num_rows:
                for key, n, c in zip(t["k"].to_pylist(), t["count(*)"].to_pylist(), t[f"count({name})"].to_pylist()):
                    got_n[int(key[1:])], got_c[int(key[1:])] = n, c
            assert np.array_equal(got_n, want_n) and np.array_equal(got_c, want_c), (what, got_n, want_n, got_c, want_c)
        # GROUP BY the Boolean itself
        t = prov.aggregate([name], [count_star(), count(name)]).table()
        got = {key: (n, c) for key, n, c in zip(t[name].to_pylist(), t["count(*)"].to_pylist(), t[f"count({name})"].to_pylist())}
        want = {True: (int((v & x).sum()), int((v & x).sum())), False: (int((v & ~x).sum()), int((v & ~x).sum())),
                None: (int((~v).sum()), 0)}
        assert got == want, (source, name, got, want)
        # MIN / MAX per group
        t = prov.aggregate(["k"], [min_(name), max_(name)]).table()
        got = {key: (lo, hi) for key, lo, hi in zip(t["k"].to_pylist(), t[f"min({name})"].to_pylist(), t[f"max({name})"].to_pylist())}
        want = {}
        for g in range(7):
            vals = x[(kc == g) & v]
            want[f"k{g}"] = (bool(vals.min()), bool(vals.max())) if vals.size else (None, None)
        assert got == want, (source, name, got, want)
        # MIN / MAX where only FALSE (or only TRUE) rows are selected: a stray tail bit would show as TRUE (FALSE)
        for flag in (False, True):
            t = prov.aggregate(["k"], [min_(name), max_(name)], [col(name) == flag]).table()
            got = {key: (lo, hi) for key, lo, hi in zip(t["k"].to_pylist(), t[f"min({name})"].to_pylist(), t[f"max({name})"].to_pylist())}
            assert got == {f"k{g}": (flag, flag) for g in range(7) if ((kc == g) & v & (x == flag)).any()}, (source, name, flag, got)
