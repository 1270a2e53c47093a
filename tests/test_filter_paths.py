"""Every way k_flat_filter (and the two other device evaluators of a predicate) can decide a row, checked against a plain
numpy restatement of SQL three-valued logic.

A leaf is answered per flat piece in one of the modes of `leaf_ctx` (flat_scan.cuh): a register LUT (dictionary of <= 32
entries at an index width <= 5), a LUT in memory (any other index page), PLAIN8 values, BITS (Boolean) or BYTES (PLAIN
strings).  The data below reach each of them by construction: dictionary Utf8 columns of 1 .. 70 000 values (index
widths 1 - 17), a column whose first pages are written while its dictionary is still small (narrow pages under a
dictionary of more than 32 entries), a dictionary that falls back to PLAIN in mid-chunk, PLAIN / DELTA Int64 and Float64
columns, DELTA string columns, a v2-page file, an all-NULL row group and a column absent from one file.  Pages are cut
every 97 rows at 4 KB, so every column's pages start at other rows and pieces start inside pages, off the 32-bit grid.

The reference (`Ref`) holds a TRUE and a NULL plane per row; leaves on Utf8 columns are evaluated once per distinct
value and mapped through the codes; floats compare by the totalOrder key; strings bytewise; LIKE / ILIKE become Python
regular expressions (ILIKE folds ASCII only, like the device); regex leaves use `re.search`.  Int64 against a Float64
literal follows the project's rule: an integral literal inside the int64 range compares as that integer (exactly, also
beyond 2^53), any other literal compares with the column cast to Float64 in totalOrder (DataFusion's coercion), a NaN by
its sign bit: below every value with it, above every value without it.

CPU: the reference against the C oracle on every generated predicate (regex leaves excepted: the oracle has none), and
the data and generator coverage.  GPU: count, row ids, LIMIT and a grouped COUNT per predicate, resident and over the
file list, and a subset under forced configurations whose PQB_VERBOSE lines show that they ran."""
import os
import re
from contextlib import ExitStack, contextmanager

import numpy as np
import pyarrow as pa
import pyarrow.parquet as pq
import pytest

from oracle.oracle import Oracle
from parseable_b200 import _lib as L
from parseable_b200.query import DeviceTable, Expr, QueryError, StandardTableProvider, _Desc, col, count, count_star, lit

SEED = 20261017
FILE_ROWS = (800_000, 700_000, 500_000)
N = sum(FILE_ROWS)
RG = 200_003                        # odd row groups: short last slabs and last words
PAGE_KW = dict(data_page_size=4096, write_batch_size=97)
I64_MIN, I64_MAX = -(1 << 63), (1 << 63) - 1
NEG_NAN = np.array([0xFFF8000000000001], np.uint64).view(np.float64)[0]
POS_NAN = np.array([0x7FF8000000000002], np.uint64).view(np.float64)[0]
STACK, MAX_LEAVES, MAX_OPS = 8, 16, 40     # kPredStack, kMaxLeaves, kMaxPredOps (device_structs.hpp)
CARDS = {"s1": 1, "s2": 2, "s3": 3, "s5": 5, "s9": 9, "s17": 17, "s32": 32, "s33": 33, "s65": 65, "s200": 200, "s600": 600,
         "s1500": 1500, "s3000": 3000, "s5000": 5000, "s70k": 70_000}
PREF = ["", "a", "A", "ab", "Ab", "aB_", "é", "x%", "日本"]
PLAIN_STR = ("sfb", "sdba", "sdlba")       # Utf8 columns with PLAIN pages (k_scan does not read them)
ALL_NULL_RG, NEG_NAN_RGS = 1, (4, 7)
ENCODING = {"iplain": "PLAIN", "fplain": "PLAIN", "fclu": "PLAIN", "ts": "DELTA_BINARY_PACKED", "sdba": "DELTA_BYTE_ARRAY",
            "sdlba": "DELTA_LENGTH_BYTE_ARRAY"}


@contextmanager
def env_var(name, value):
    old = os.environ.get(name)
    os.environ[name] = str(value)
    try:
        yield
    finally:
        if old is None:
            del os.environ[name]
        else:
            os.environ[name] = old


@contextmanager
def env_vars(env: dict):
    with ExitStack() as st:
        for k, v in env.items():
            st.enter_context(env_var(k, v))
        yield


# ---- data ------------------------------------------------------------------------------------------------------------
class Col:
    def __init__(self, kind, values, valid, vocab=None):
        self.kind, self.values, self.valid, self.vocab = kind, values, valid, vocab
        if vocab is not None:
            self.vbytes = [v.encode() for v in vocab]


def _vocab(n):
    return [f"{PREF[i % len(PREF)]}{i:x}" for i in range(n)]


def _rg_index():
    """Global row group of every row, and the first row of every file."""
    rg, starts, base, s = np.empty(N, np.int64), [], 0, 0
    for n in FILE_ROWS:
        rg[s:s + n] = base + np.arange(n) // RG
        starts.append(s)
        base += -(-n // RG)
        s += n
    return rg, starts


def make_data(rng):
    rg, starts = _rg_index()
    D = {}
    valid = lambda p: rng.random(N) >= p   # noqa: E731
    for name, card in CARDS.items():
        if name == "s5":   # skewed: `s5 = v0` keeps ~2 % of the rows (sparse survivors), `s5 != v0` ~98 %
            codes = rng.choice(5, N, p=[0.02, 0.49, 0.29, 0.15, 0.05])
        else:
            codes = rng.integers(0, card, N)
        D[name] = Col("str", codes, valid(0.03), _vocab(card))
    # mem: the first 40 000 rows of a row group see 2 .. 32 values, the rest 100: narrow pages under a wide dictionary
    codes = rng.integers(0, 100, N)
    first = np.zeros(N, bool)
    for g in np.unique(rg):
        rows = np.flatnonzero(rg == g)[:40_000]
        codes[rows] = rng.integers(0, 2 ** (1 + g % 5), len(rows))
        first[rows] = True
    D["mem"] = Col("str", codes, valid(0.02), [f"m{i:02d}" for i in range(100)])
    # sfb: long, nearly distinct strings: the dictionary passes 1 MB inside every chunk and falls back to PLAIN
    tails = ["", "ü", "€", "𝄞", "common/prefix/", "common/prefixes/"]
    sfb = [""] + [f"{tails[i % 6]}{'ab' * (i % 17)}{i:07d}{tails[(i // 6) % 6]}" for i in range(1, 400_000)]
    D["sfb"] = Col("str", rng.integers(0, len(sfb), N), valid(0.02), sfb)
    pool = [f"{PREF[i % len(PREF)]}{'z' * (i % 5)}{i:05d}" for i in range(50_000)]
    D["sdba"] = Col("str", rng.integers(0, len(pool), N), valid(0.02), pool)
    D["sdlba"] = Col("str", rng.integers(0, len(pool), N), valid(0.02), pool)
    D["k7"] = Col("str", rng.integers(0, 7, N), valid(0.01), [f"k{i}" for i in range(7)])
    opt = Col("str", rng.integers(0, 9, N), valid(0.02), _vocab(9))
    opt.valid[starts[2]:] = False      # absent from the third file
    D["opt"] = opt
    # Int64
    ipool = np.concatenate([rng.integers(-10**6, 10**6, 390), [0, 1, -1, 2**40, -2**40, 7, 8, 9, 10, 11]]).astype(np.int64)
    idict = Col("i64", ipool[rng.integers(0, len(ipool), N)], valid(0.03))
    idict.valid[rg == ALL_NULL_RG] = False
    D["idict"] = idict
    ip = rng.integers(I64_MIN, I64_MAX, N, dtype=np.int64, endpoint=True)
    ip[rng.integers(0, N, 200)] = I64_MIN
    ip[rng.integers(0, N, 200)] = I64_MAX
    D["iplain"] = Col("i64", ip, valid(0.02))
    big = np.array([2**53 + k for k in range(-3, 4)] + [-(2**53) + k for k in range(-3, 4)] + [2**62, 5], np.int64)
    D["ibig"] = Col("i64", big[rng.integers(0, len(big), N)], valid(0.02))
    D["ts"] = Col("i64", 1_700_000_000_000 + np.cumsum(rng.integers(0, 4, N)), np.ones(N, bool))
    # Float64
    specials = np.array([0.0, -0.0, np.inf, -np.inf, 5e-324, -5e-324, 2.2250738585072009e-308, NEG_NAN, POS_NAN, 1.5, -1.5])
    fpool = np.concatenate([specials, np.round(rng.standard_normal(289) * 100, 2)])
    D["fdict"] = Col("f64", fpool[rng.integers(0, len(fpool), N)], valid(0.03))
    fp = rng.standard_normal(N) * 10.0 ** rng.integers(-3, 6, N)
    sp = rng.integers(0, N, N // 100)
    fp[sp] = specials[rng.integers(0, len(specials), len(sp))]
    D["fplain"] = Col("f64", fp, valid(0.02))
    # fclu: row group g holds [10 g, 10 g + 10): statistics prune and fold; negative NaN inside two row groups far above
    # the literals, a positive NaN in a third
    fc = 10.0 * rg + rng.random(N) * 10.0
    for g in NEG_NAN_RGS:
        rows = np.flatnonzero(rg == g)
        fc[rng.choice(rows, 1000, replace=False)] = NEG_NAN
    rows = np.flatnonzero(rg == 6)
    fc[rng.choice(rows, 1000, replace=False)] = POS_NAN
    D["fclu"] = Col("f64", fc, valid(0.01))
    D["b"] = Col("bool", rng.integers(0, 2, N).astype(np.int64), valid(0.05))
    return D, first


def _arrow(c: Col, lo, hi):
    if c.kind == "str":
        return pa.DictionaryArray.from_arrays(pa.array(c.values[lo:hi], pa.int32(), mask=~c.valid[lo:hi]),
                                              pa.array(c.vocab, pa.string())).cast(pa.string())
    typ = {"i64": pa.int64(), "f64": pa.float64(), "bool": pa.bool_()}[c.kind]
    v = c.values[lo:hi].astype(bool) if c.kind == "bool" else c.values[lo:hi]
    return pa.array(v, typ, mask=~c.valid[lo:hi])


@pytest.fixture(scope="module")
def fdata(built, data_dir):
    D, first = make_data(np.random.default_rng(SEED))
    names = list(D)
    paths, lo = [], 0
    for i, n in enumerate(FILE_ROWS):
        cols = [c for c in names if not (c == "opt" and i == 2)]
        t = pa.table({c: _arrow(D[c], lo, lo + n) for c in cols})
        p = os.path.join(data_dir, f"filter_paths_{i}.parquet")
        pq.write_table(t, p, row_group_size=RG, use_dictionary=[c for c in cols if c not in ENCODING and c != "b"],
                       column_encoding={c: e for c, e in ENCODING.items()}, data_page_version="2.0" if i == 1 else "1.0", **PAGE_KW)
        paths.append(p)
        lo += n
    schema = pa.schema([(c, pa.string() if D[c].kind == "str" else pa.int64() if D[c].kind == "i64" else
                         pa.float64() if D[c].kind == "f64" else pa.bool_()) for c in names])
    return D, first, paths, schema


# ---- reference -------------------------------------------------------------------------------------------------------
def _okey(bits):
    return bits ^ ((bits >> 63) & np.int64(0x7FFFFFFFFFFFFFFF))


def _fkey(x):
    return _okey(np.asarray(x, np.float64).view(np.int64))


_CMP = {L.PQ_EQ: np.equal, L.PQ_NE: np.not_equal, L.PQ_LT: np.less, L.PQ_LE: np.less_equal, L.PQ_GT: np.greater,
        L.PQ_GE: np.greater_equal}
_FLIP = {L.PQ_LT: L.PQ_GT, L.PQ_GT: L.PQ_LT, L.PQ_LE: L.PQ_GE, L.PQ_GE: L.PQ_LE, L.PQ_EQ: L.PQ_EQ, L.PQ_NE: L.PQ_NE}
_ASCII_LOWER = {c: c + 32 for c in range(65, 91)}


def like_regex(pattern: str, ci: bool):
    """LIKE pattern -> a compiled full-match regex: % any run, _ one character, backslash escapes the next one."""
    out, i = [], 0
    while i < len(pattern):
        ch = pattern[i]
        if ch == "\\" and i + 1 < len(pattern):
            i += 1
            out.append(re.escape(pattern[i]))
        elif ch == "%":
            out.append(".*")
        elif ch == "_":
            out.append(".")
        else:
            out.append(re.escape(ch))
        i += 1
    rx = "".join(out)
    return re.compile(rx.translate(_ASCII_LOWER) if ci else rx, re.DOTALL)


class Ref:
    def __init__(self, D):
        self.D = D

    def _str_leaf(self, c: Col, fn):
        per_value = np.fromiter((fn(i) for i in range(len(c.vocab))), bool, len(c.vocab))
        return per_value[c.values]

    def leaf(self, e: Expr) -> np.ndarray:
        """TRUE per row of a value leaf, ignoring validity."""
        if e.kind in ("like", "regex"):
            c = self.D[e.args[0].args[0]]
            pat = e.args[1].args[0]
            neg = bool(e.flags & 1)
            ci = bool(e.flags & 2)
            if e.kind == "like":
                rx = like_regex(pat, ci)
                fold = (lambda s: s.translate(_ASCII_LOWER)) if ci else (lambda s: s)
                t = self._str_leaf(c, lambda i: rx.fullmatch(fold(c.vocab[i])) is not None)
            else:
                rx = re.compile(pat, re.IGNORECASE if ci else 0)
                t = self._str_leaf(c, lambda i: rx.search(c.vocab[i]) is not None)
            return ~t if neg else t
        a, b, op = e.args[0], e.args[1], e.op
        if a.kind == "lit":
            a, b, op = b, a, _FLIP[op]
        c, v = self.D[a.args[0]], b.args[0]
        if c.kind == "str":
            lb = v.encode()
            cmp = {L.PQ_EQ: lambda x: x == lb, L.PQ_NE: lambda x: x != lb, L.PQ_LT: lambda x: x < lb,
                   L.PQ_LE: lambda x: x <= lb, L.PQ_GT: lambda x: x > lb, L.PQ_GE: lambda x: x >= lb}[op]
            return self._str_leaf(c, lambda i: cmp(c.vbytes[i]))
        if c.kind == "f64":
            return _CMP[op](_fkey(c.values), _fkey(float(v)))
        if c.kind == "bool":
            return _CMP[op](c.values, int(v))
        if isinstance(v, float) and not (v == v and v.is_integer() and -2.0 ** 63 <= v < 2.0 ** 63):
            return _CMP[op](_fkey(c.values.astype(np.float64)), _fkey(v))   # the column cast to Float64, totalOrder
        return _CMP[op](c.values, np.int64(int(v)))

    def eval(self, e: Expr):
        """(TRUE plane, NULL plane)."""
        if e.kind in ("and", "or"):
            ta, na = self.eval(e.args[0])
            tb, nb = self.eval(e.args[1])
            if e.kind == "and":
                fa, fb = ~(ta | na), ~(tb | nb)
                return ta & tb, (na | nb) & ~fa & ~fb
            t = ta | tb
            return t, (na | nb) & ~t
        if e.kind == "not":
            t, n = self.eval(e.args[0])
            return ~(t | n), n
        if e.kind == "lit":
            v = e.args[0]
            return np.full(N, v is True), np.full(N, v is None)
        if e.kind in ("is_null", "is_not_null"):
            v = self.D[e.args[0].args[0]].valid
            return (~v if e.kind == "is_null" else v.copy()), np.zeros(N, bool)
        if e.kind == "cmp" and (e.args[1].kind == "lit" and e.args[1].args[0] is None):
            return np.zeros(N, bool), np.ones(N, bool)   # col <op> NULL: NULL on every row
        valid = self.D[(e.args[1] if e.args[0].kind == "lit" else e.args[0]).args[0]].valid
        return self.leaf(e) & valid, ~valid

    def select(self, e: Expr) -> np.ndarray:
        """The TRUE rows; kept per predicate (by its repr) for the module's later tests."""
        key = (id(self.D), repr(e))
        if key not in _SELECTED:
            _SELECTED[key] = self.eval(e)[0]
        return _SELECTED[key]


_SELECTED: dict = {}


# ---- predicates ------------------------------------------------------------------------------------------------------
def program(e: Expr):
    """(ops, leaves, max stack depth, columns) of the postfix program the host compiles."""
    d, ops = _Desc(), []
    d.compile_pred(e, ops)
    depth = best = leaves = 0
    for op in ops:
        if op.kind in (L.PQ_OP_AND, L.PQ_OP_OR):
            depth -= 1
        elif op.kind != L.PQ_OP_NOT:
            depth += 1
            leaves += op.kind != L.PQ_OP_CONST
        best = max(best, depth)
    return len(ops), leaves, best, d.columns


def kinds(e: Expr) -> set:
    out = {e.kind}
    for a in e.args:
        if isinstance(a, Expr):
            out |= kinds(a)
    if e.kind == "like":
        out.add(("ilike" if e.flags & 2 else "like") + ("_neg" if e.flags & 1 else ""))
        p = e.args[1].args[0]
        out.add("like_" + ("prefix" if re.fullmatch(r"[^%_\\]+%", p) else "suffix" if re.fullmatch(r"%[^%_\\]+", p) else
                           "contains" if re.fullmatch(r"%[^%_\\]+%", p) else "under" if "_" in p else "general"))
    if e.kind == "cmp":
        out.add(("op", e.op))
    if e.kind == "lit":
        out.add(("const", e.args[0]))
    return out


def is_conj(e: Expr) -> bool:
    if e.kind == "and":
        return is_conj(e.args[0]) and is_conj(e.args[1])
    if e.kind == "lit":
        return e.args[0] is True
    return e.kind not in ("or", "not")


NUMERIC = ["idict", "iplain", "ibig", "ts", "fdict", "fplain", "fclu", "b"]
STRS = list(CARDS) + ["mem", "sfb", "sdba", "sdlba", "opt", "k7"]


class Gen:
    def __init__(self, D, rng):
        self.D, self.rng = D, rng

    def _pick(self, seq):
        return seq[int(self.rng.integers(0, len(seq)))]

    def _num_lit(self, c: Col):
        v = c.values[c.valid]
        if c.kind == "bool":
            return bool(self.rng.integers(0, 2))
        if c.kind == "i64":
            lo, hi = int(v.min()), int(v.max())
            cands = [lo, hi, int(self._pick(v)), min(hi + 1, I64_MAX), max(lo - 1, I64_MIN), float(self._pick(v)) + 0.5,
                     NEG_NAN, POS_NAN, 2.0 ** 53, -(2.0 ** 53), 2.0 ** 63]
        else:
            fin = v[np.isfinite(v)]
            lo, hi = float(fin.min()), float(fin.max())
            cands = [lo, hi, float(self._pick(v)), np.nextafter(lo, -np.inf), np.nextafter(hi, np.inf), 0.0, -0.0, np.inf,
                     -np.inf, NEG_NAN, POS_NAN, 5e-324, 0.25, 7]
        x = cands[int(self.rng.integers(0, len(cands)))]
        return float(x) if isinstance(x, (float, np.floating)) else int(x)

    def _str_lit(self, c: Col):
        present = [c.vocab[i] for i in np.unique(c.values[:2000])]
        lo, hi = min(present, key=str.encode), max(present, key=str.encode)
        v = self._pick(present)
        return self._pick([lo, hi, v, v[:-1], v + "0", "", hi + "\U0010ffff", "A"])

    def leaf(self, name):
        c, r = self.D[name], self.rng.random()
        if r < 0.08:
            return col(name).is_null() if self.rng.random() < 0.5 else col(name).is_not_null()
        op = int(self.rng.integers(0, 6))
        if c.kind != "str":
            return Expr("cmp", (col(name), lit(self._num_lit(c))), op)
        if r < 0.55:
            return Expr("cmp", (col(name), lit(self._str_lit(c))), op)
        v = self._pick(c.vocab)
        frag = v[1:3] or "a"
        if r < 0.92:
            pat = self._pick([v[:2] + "%", "%" + v[-2:], "%" + frag + "%", "_" + v[1:] if len(v) > 1 else "_", "a%1%",
                              "%\\%%", "A_%", "%é%", "日%", v])
            return col(name).like(pat, negated=self.rng.random() < 0.25, case_insensitive=self.rng.random() < 0.3)
        return col(name).regex(self._pick(["^a", "1$", "[0-4]7", "ab|Ab", "^[0-9a-f]+$", "z{2}"]), negated=self.rng.random() < 0.3)

    def const(self):
        return lit(self._pick([True, False, None]))

    def tree(self, names, n_leaves):
        """A random tree over `n_leaves` leaves of the columns `names`, with NOTs and constants."""
        if n_leaves == 1:
            e = self.const() if self.rng.random() < 0.06 else self.leaf(self._pick(names))
        else:
            k = int(self.rng.integers(1, n_leaves))
            a, b = self.tree(names, k), self.tree(names, n_leaves - k)
            e = a & b if self.rng.random() < 0.5 else a | b
        return ~e if self.rng.random() < 0.15 else e

    def chain(self, names, n, ops, right_deep):
        leaves = [self.leaf(self._pick(names)) for _ in range(n)]
        e = leaves[-1] if right_deep else leaves[0]
        for i, x in enumerate(leaves[-2::-1] if right_deep else leaves[1:]):
            o = ops[i % len(ops)]
            e = (x & e if o == "and" else x | e) if right_deep else (e & x if o == "and" else e | x)
        return e

    def columns(self, k):
        pool = NUMERIC + STRS
        return [pool[i] for i in self.rng.choice(len(pool), k, replace=False)]


def predicates(D, n_random=40):
    """The generated set: random trees, pure conjunctions (sparse and dense survivors after the first leaf), stack-deep
    chains and 16-leaf programs; every one within the caps and at most 10 columns."""
    g = Gen(D, np.random.default_rng(SEED + 1))
    out = []
    while len(out) < n_random:
        e = g.tree(g.columns(int(g.rng.integers(1, 8))), int(g.rng.integers(1, 12)))
        n_ops, n_leaves, depth, cols = program(e)
        if n_ops <= MAX_OPS and n_leaves <= MAX_LEAVES and depth <= STACK and len(cols) <= 10:
            out.append(("random", e))
    for i in range(8):   # conjunctions: `s5 = v0` (2 %) first leaves sparse survivors, `s5 != v0` (98 %) dense ones
        first = (col("s5") == D["s5"].vocab[0]) if i % 2 == 0 else (col("s5") != D["s5"].vocab[0])
        e = first
        for name in g.columns(int(g.rng.integers(1, 5))):
            e = e & g.leaf(name)
        out.append(("conj_sparse" if i % 2 == 0 else "conj_dense", e))
    for i in range(4):   # plain random conjunctions
        out.append(("conj", g.chain(g.columns(6), int(g.rng.integers(2, 9)), ["and"], False)))
    for i in range(4):   # stack depth exactly 8 (right-deep), OR / AND mixes: the Kleene stack full
        out.append(("deep", g.chain(g.columns(6), STACK, ["or", "and"] if i % 2 else ["or"], True)))
    for i in range(3):   # 16 leaves (left-deep: depth 2)
        out.append(("wide", g.chain(g.columns(8), MAX_LEAVES, ["and", "or", "or"], False)))
    return out


def hand_cases(D):
    ts0 = int(D["ts"].values.min())
    return [
        # NaN literals against Int64: by the sign bit (negative NaN below every value)
        ("nan_i64_gt", col("iplain") > NEG_NAN), ("nan_i64_lt", col("iplain") < NEG_NAN),
        ("nan_i64_ge_dict", col("idict") >= NEG_NAN), ("nan_i64_le_pos", col("ibig") <= POS_NAN),
        ("nan_i64_ne", col("ibig") != NEG_NAN), ("nan_i64_eq", col("idict") == POS_NAN),
        # Float64 pruning: negative NaN rows in row groups whose min lies far above the literal
        ("nan_f64_lt", col("fclu") < 0.25), ("nan_f64_le", col("fclu") <= 0.25), ("nan_f64_lt_neg", col("fclu") < -1e300),
        ("nan_f64_eq", col("fclu") == 5.0), ("nan_f64_gt", col("fclu") > 55.5),
        # integral literals beyond 2^53 compare as integers
        ("big_eq", col("ibig") == 2.0 ** 53), ("big_lt", col("ibig") < float(2 ** 53 + 2)), ("big_ge", col("ibig") >= -(2.0 ** 53)),
        ("big_gt_half", col("ibig") > 4.5),
        # 2^63 is no int64: the column is cast, and the int64 values from 2^63 - 512 up round to it
        ("top_eq", col("iplain") == 2.0 ** 63), ("top_ge", col("iplain") >= 2.0 ** 63), ("top_lt", col("iplain") < 2.0 ** 63),
        ("top_ne", col("iplain") != 2.0 ** 63), ("top_le", col("iplain") <= 2.0 ** 63), ("top_gt", col("iplain") > 2.0 ** 63),
        # conjunctions whose cheapest leaf (the planner evaluates it first) is `s5`: after it the PLAIN8 and 10-bit leaves
        # see ~1 survivor in 64 rows (one at a time) or ~63 (dense)
        ("first_sparse", (col("s5") == D["s5"].vocab[0]) & (col("iplain") > 0) & (col("s600") < "b")),
        ("first_dense", (col("s5") != D["s5"].vocab[0]) & (col("iplain") > 0) & (col("s600") < "b")),
        # leaves that statistics decide TRUE everywhere, folded under NOT and OR
        ("fold_not", ~(col("ts") >= ts0)), ("fold_or", (col("ts") >= ts0) | (col("s9") == "a1")),
        ("fold_not_or", ~((col("ts") >= ts0) | col("fplain").is_null())), ("fold_is_not_null", ~col("ts").is_not_null()),
        # NULL constants
        ("eq_null", Expr("cmp", (col("s9"), lit(None)), L.PQ_EQ)), ("not_null_const", ~lit(None)),
        ("null_or", lit(None) | (col("b") == True)), ("not_eq_null_and", ~(Expr("cmp", (col("idict"), lit(None)), L.PQ_LT) & (col("s2") == "a1"))),
        # the all-NULL row group and the absent column
        ("allnull_is_null", col("idict").is_null()), ("allnull_not", ~(col("idict") == 7)), ("allnull_not_nn", ~col("idict").is_not_null()),
        ("absent_is_null", col("opt").is_null()), ("absent_not", ~(col("opt") == "a1")), ("absent_nn", col("opt").is_not_null()),
        ("absent_or", (col("opt") != "a1") | col("opt").is_null()),
    ]


def _cap_chain(n, op):
    e = col("s2").is_null()
    for i in range(n - 1):
        e = (col(["s3", "s9", "b"][i % 3]).is_null() | e) if op == "or_right" else (e & (col("s17") != f"x{i}"))
    return e


def caps():
    """(name, predicate, within the caps?) at each cap and one past it."""
    def ops40(n):   # 16 leaves + 15 ANDs + NOT NOT pairs: n ops in all
        e = _cap_chain(MAX_LEAVES, "and")
        extra = n - (2 * MAX_LEAVES - 1)
        for _ in range(extra):
            e = ~e
        return e
    return [("depth8", _cap_chain(STACK, "or_right"), True), ("depth9", _cap_chain(STACK + 1, "or_right"), False),
            ("leaves16", _cap_chain(MAX_LEAVES, "and"), True), ("leaves17", _cap_chain(MAX_LEAVES + 1, "and"), False),
            ("ops40", ops40(MAX_OPS), True), ("ops41", ops40(MAX_OPS + 1), False)]


# ---- CPU -------------------------------------------------------------------------------------------------------------
def _has_regex(e):
    return "regex" in kinds(e)


def _oracle_table(paths, schema):
    t = [pq.read_table(p) for p in paths]
    t[2] = t[2].append_column("opt", pa.nulls(t[2].num_rows, pa.string()))
    return pa.concat_tables([x.select(schema.names) for x in t])


def test_reference_matches_oracle(fdata):
    """The numpy reference and the C oracle agree on every generated and hand-written predicate without a regex leaf;
    no predicate is a legitimate difference."""
    D, _, paths, schema = fdata
    # the oracle walks its rows one by one: the first 300 000 rows (the all-NULL row group) and 150 000 rows of the third
    # file (the absent column)
    rows = np.r_[0:300_000, N - 150_000:N]
    ora, ref = Oracle(_oracle_table(paths, schema).take(pa.array(rows))), Ref(D)
    cases = predicates(D) + hand_cases(D)
    checked = 0
    for name, e in cases:
        if _has_regex(e):
            continue
        want = ref.select(e)[rows]
        got = ora.select([e]).astype(bool)
        bad = np.flatnonzero(want != got)
        assert bad.size == 0, (name, e, bad.size, int(bad[0]))
        checked += 1
    assert checked >= 60


def test_data_layout(fdata):
    """The files hold what the modes need: encodings, dictionary sizes, fallback, v2 pages, NaN sign bits, the all-NULL
    row group, the absent column, and pages that start at different rows in different columns."""
    D, first, paths, schema = fdata
    md = [pq.ParquetFile(p).metadata for p in paths]
    enc = {}
    for m in md:
        for g in range(m.num_row_groups):
            rgm = m.row_group(g)
            assert rgm.num_rows in (RG, FILE_ROWS[0] - 3 * RG, FILE_ROWS[1] - 3 * RG, FILE_ROWS[2] - 2 * RG)
            for j in range(rgm.num_columns):
                c = rgm.column(j)
                enc.setdefault(c.path_in_schema, set()).update(c.encodings)
    for name in CARDS:
        assert "RLE_DICTIONARY" in enc[name], name
    assert {"RLE_DICTIONARY", "PLAIN"} <= enc["sfb"]              # the dictionary falls back in mid-chunk
    assert "DELTA_BYTE_ARRAY" in enc["sdba"] and "DELTA_LENGTH_BYTE_ARRAY" in enc["sdlba"]
    assert "DELTA_BINARY_PACKED" in enc["ts"]
    assert "RLE_DICTIONARY" not in enc["iplain"] | enc["fplain"] | enc["fclu"]
    assert "RLE_DICTIONARY" in enc["idict"] and "RLE_DICTIONARY" in enc["fdict"] and "RLE_DICTIONARY" in enc["ibig"]
    assert "opt" not in pq.ParquetFile(paths[2]).schema_arrow.names
    # dictionary sizes per chunk (a chunk's dictionary holds the distinct values it met): both sides of 32 entries,
    # and wider than 2^16 for the widest
    rg, _ = _rg_index()
    sel = rg == 0
    for name, card in CARDS.items():
        k = len(np.unique(D[name].values[sel & D[name].valid]))
        assert k == card or (card > 30_000 and k > 65_536), (name, k)
    assert len(np.unique(D["mem"].values[sel & D["mem"].valid])) == 100 and first.sum() == 40_000 * (rg.max() + 1)
    # the read-back keeps every NaN's sign bit (the reference reads the arrays, the kernels the files)
    t = _oracle_table(paths, schema)
    for name in ("fdict", "fplain", "fclu"):
        got = t[name].to_numpy(zero_copy_only=False)
        v = D[name].valid
        assert np.array_equal(np.asarray(got, np.float64)[v].view(np.int64), D[name].values[v].view(np.int64)), name
        assert (np.signbit(D[name].values[v]) & np.isnan(D[name].values[v])).any(), name
    # the all-NULL row group, and the negative NaN only where fclu's other values lie far above 0.25
    m0 = md[0].row_group(ALL_NULL_RG).column(schema.names.index("idict")).statistics
    assert m0.null_count == md[0].row_group(ALL_NULL_RG).num_rows and not m0.has_min_max
    for g in NEG_NAN_RGS:
        st = md[g // 4 if g < 4 else 1].row_group(g % 4 if g < 4 else g - 4).column(schema.names.index("fclu")).statistics
        assert st.min >= 10.0, (g, st.min)
    # page starts differ between columns: a 4 KB page holds ~500 PLAIN8 rows but tens of thousands of narrow indices
    pf = pq.ParquetFile(paths[0])
    starts = {}
    for name in ("iplain", "s3", "s600"):
        j = schema.names.index(name)
        ci = pf.metadata.row_group(0).column(j)
        starts[name] = ci.total_compressed_size
    assert starts["iplain"] > 4 * starts["s3"]


def test_generator_coverage(fdata):
    """The generated set reaches every operator, LIKE kind, constant and the three caps; its conjunctions put both
    sparse (<= 12 of 64 rows) and dense survivors after the first leaf."""
    D = fdata[0]
    cases = predicates(D)
    seen, depth, leaves, n_ops = set(), 0, 0, 0
    for _, e in cases:
        seen |= kinds(e)
        o, lv, dp, cols = program(e)
        assert o <= MAX_OPS and lv <= MAX_LEAVES and dp <= STACK and len(cols) <= 10
        depth, leaves, n_ops = max(depth, dp), max(leaves, lv), max(n_ops, o)
    assert depth == STACK and leaves == MAX_LEAVES
    want = {"and", "or", "not", "is_null", "is_not_null", "like", "regex", "like_prefix", "like_suffix", "like_contains",
            "like_under", "like_general", "ilike", "like_neg", ("const", True), ("const", False), ("const", None)}
    want |= {("op", op) for op in range(6)}
    assert want <= seen, want - seen
    assert sum(is_conj(e) for _, e in cases) >= 12
    ref = Ref(D)
    sparse = ref.select(col("s5") == D["s5"].vocab[0]).mean()
    dense = ref.select(col("s5") != D["s5"].vocab[0]).mean()
    assert sparse < 0.03 and dense > 0.9
    for name, e, ok in caps():
        o, lv, dp, _ = program(e)
        assert (o <= MAX_OPS and lv <= MAX_LEAVES and dp <= STACK) == ok, name
        assert (o, lv, dp) in ((MAX_OPS, MAX_LEAVES, 2), (MAX_OPS + 1, MAX_LEAVES, 2), (2 * MAX_LEAVES - 1, MAX_LEAVES, 2),
                               (2 * MAX_LEAVES + 1, MAX_LEAVES + 1, 2), (2 * STACK - 1, STACK, STACK),
                               (2 * STACK + 1, STACK + 1, STACK + 1)), (name, o, lv, dp)


# ---- GPU -------------------------------------------------------------------------------------------------------------
FILTER_LINE = re.compile(r"\[pqb\] k_flat_filter<(CONJ|KLEENE)>: (\d+) live leaves, (\d+) CTAs, \d+ B smem/CTA, (\d+) stages x \d+ B, "
                         r"slab (\d+) rows")
AGG_LINE = re.compile(r"\[pqb\] k_flat_agg<(\d+)((?:,\w+)*)>")
LEAF_LINE = re.compile(r"\[pqb\] leaf (\d+): column '(\w+)', (\w+), flat pages ([\w+-]+), widest index (\d+), register LUT (\w+), "
                       r"off-grid (\d+), absent (\d+),(.*)")


@pytest.fixture(scope="module")
def gpu(fdata):
    D, _, paths, schema = fdata
    table = DeviceTable(paths, schema.names)
    yield {"resident": StandardTableProvider(table, schema=schema), "files": StandardTableProvider(paths, schema=schema)}
    table.close()


def _ids(res):
    if not res.batches:
        return np.zeros(0, np.int64)
    return np.concatenate([b.column(b.schema.names.index("__row_id")).to_numpy() for b in res.batches]).astype(np.int64)


def _count_col(e):
    return next((c for c in program(e)[3] if c != "k7"), "fplain")


def check_group(D, prov, e, want, what):
    """GROUP BY k7 -> COUNT(*), COUNT(col) through k_flat_agg, against the reference's selection."""
    cc = _count_col(e)
    t = prov.aggregate(["k7"], [count_star(), count(cc)], [e]).table()
    k7 = D["k7"]
    codes = np.where(k7.valid, k7.values, 7)[want]
    want_n = np.bincount(codes, minlength=8)
    want_c = np.bincount(codes, weights=D[cc].valid[want], minlength=8).astype(np.int64)
    got_n, got_c = np.zeros(8, np.int64), np.zeros(8, np.int64)
    if t.num_rows:
        for k, n, c in zip(t["k7"].to_pylist(), t["count(*)"].to_pylist(), t[f"count({cc})"].to_pylist()):
            i = 7 if k is None else k7.vocab.index(k)
            assert got_n[i] == 0, (what, "group twice", k)
            got_n[i], got_c[i] = n, c
    assert np.array_equal(got_n, want_n), (what, got_n, want_n)
    assert np.array_equal(got_c, want_c), (what, got_c, want_c)


def check_pred(D, prov, e, want, what, limit=True, group=True):
    ids = np.flatnonzero(want)
    n = prov.scan(filters=[e], count_only=True).metrics["rows_selected"]
    assert n == len(ids), (what, "count", n, len(ids))
    got = _ids(prov.scan(filters=[e]))
    if not np.array_equal(got, ids):
        diff = np.setxor1d(got, ids)
        raise AssertionError(f"{what}: row ids differ: {len(got)} vs {len(ids)}, first differing row {diff[:1]}")
    if limit:
        k = int(min(len(ids), 1 + (len(ids) * 7) // 13)) or 5
        got = _ids(prov.scan(filters=[e], limit=k))
        assert np.array_equal(got, ids[:k]), (what, "limit", k)
    if group:
        check_group(D, prov, e, want, what)


def _all_cases(D):
    return predicates(D) + hand_cases(D)


@pytest.mark.gpu
def test_predicates_resident(fdata, gpu, capfd):
    """Every predicate on the resident table: count, row ids, LIMIT, grouped counts; the filter kernel's line names the
    instantiation the program asks for, and its leaf lines show every leaf mode and index width over the set."""
    D = fdata[0]
    ref = Ref(D)
    modes = {}
    kernels = set()
    for name, e in _all_cases(D):
        want = ref.select(e)
        capfd.readouterr()
        with env_var("PQB_VERBOSE", 1):
            n = gpu["resident"].scan(filters=[e], count_only=True).metrics["rows_selected"]
        log = capfd.readouterr().err
        assert n == want.sum(), (name, e, n, want.sum())
        lines = FILTER_LINE.findall(log)
        if lines:
            kern, live = lines[0][0], int(lines[0][1])
            kernels.add(kern)
            assert kern == ("CONJ" if is_conj(e) else "KLEENE"), (name, log)
            assert live == len(LEAF_LINE.findall(log)) <= program(e)[1], (name, log)
        if name.startswith("first_"):   # the planner put `s5` first, and the two selectivities hold
            assert [c for slot, c, *_ in LEAF_LINE.findall(log) if slot == "0"] == ["s5"], (name, log)
            assert (want.mean() < 0.01) == (name == "first_sparse"), (name, want.mean())
        for slot, cname, kind, pages, widest, reg, offgrid, absent, rest in LEAF_LINE.findall(log):
            for m, ws in re.findall(r"(\w+)\{([\d,]+)\}", rest):
                for w in ws.split(","):
                    modes.setdefault(m, set()).add(int(w))
            for p in pages.split("+"):
                modes.setdefault("pages", set()).add(p)
            if int(offgrid):
                modes.setdefault("offgrid", set()).add(cname)
            if int(absent):
                modes.setdefault("absent", set()).add(cname)
        check_pred(D, gpu["resident"], e, want, name)
    assert kernels == {"CONJ", "KLEENE"}
    assert {"INDEX", "PLAIN8", "BITS", "BYTES"} <= modes["pages"], modes
    assert set(range(1, 13)) <= modes["MEMLUT"] | modes["REGLUT"], modes
    assert {1, 2, 3, 4, 5} <= modes["MEMLUT"] and {0, 1, 2, 5} <= modes["REGLUT"], modes   # width 0: the all-NULL row group
    assert "opt" in modes.get("absent", set()) and modes.get("offgrid"), modes


@pytest.mark.gpu
def test_predicates_files(fdata, gpu):
    """A subset over the file list (a table opened per query)."""
    D = fdata[0]
    ref = Ref(D)
    for name, e in _all_cases(D)[::4]:
        check_pred(D, gpu["files"], e, ref.select(e), "files " + name, limit=False)


@pytest.mark.gpu
def test_nan_literals_and_float_pruning(fdata, gpu):
    """The two NaN cases on their own: Int64 against a NaN literal by its sign; Float64 statistics that leave the
    negative-NaN rows out of min must not prune them."""
    D = fdata[0]
    ref = Ref(D)
    for name, e in hand_cases(D):
        if name.startswith("nan_"):
            want = ref.select(e)
            assert want.any() or name in ("nan_i64_lt", "nan_i64_eq", "nan_f64_eq"), name
            check_pred(D, gpu["resident"], e, want, name, limit=False, group=False)


@pytest.mark.gpu
def test_caps(fdata, gpu):
    """Stack depth 8, 16 leaves and a 40-op program run; one past each cap is PQ_ERR_UNSUPPORTED."""
    D = fdata[0]
    ref = Ref(D)
    for name, e, ok in caps():
        if ok:
            check_pred(D, gpu["resident"], e, ref.select(e), name, limit=False)
        else:
            with pytest.raises(QueryError) as ei:
                gpu["resident"].scan(filters=[e], count_only=True)
            assert ei.value.code == L.PQ_ERR_UNSUPPORTED, (name, ei.value)


def _subset(D):
    cases = _all_cases(D)
    return [c for c in cases if c[0] in ("conj_sparse", "deep", "wide")][::2] + [c for c in cases if c[0] == "conj_dense"][::2] + \
        cases[:6:2] + [c for c in cases if c[0] in ("nan_f64_lt", "fold_not_or", "allnull_not", "absent_or", "first_sparse",
                                                    "first_dense", "top_ge")]


def _no_plain_str(e):
    return not set(program(e)[3]) & set(PLAIN_STR)


TWELVE = (col("s1") != "x") & (col("s2").is_not_null() | (col("s3") == "a1")) & ~(col("s9") < "A") & (col("s33") >= "") & \
    (col("mem") != "m05") & (col("iplain") > -(2 ** 62)) & (col("fplain") != 1.5) & (col("b") == True) & \
    ((col("sfb").like("%ab%")) | (col("ts") > 0)) & (col("fdict") < np.inf)

CONFIGS = {
    "grid1": ({"PQB_GRID": 1}, dict(ctas=1)),
    "grid3": ({"PQB_GRID": 3}, dict(ctas=3)),
    "stages4": ({"PQB_FILTER_STAGES": 4}, dict(stages=4)),
    "ctas8_twelve": ({"PQB_FILTER_CTAS": 8}, dict(short_slab=True)),
    "kscan": ({"PQB_FLAT_SCAN": 0}, dict(kscan=True)),
    "krows2": ({"PQB_AGG_KROWS": 2}, dict(kr=2)),
    "krows4": ({"PQB_AGG_KROWS": 4}, dict(kr=4)),
    "krows8": ({"PQB_AGG_KROWS": 8}, dict(kr=8)),
}


@pytest.mark.gpu
@pytest.mark.parametrize("cfg", list(CONFIGS))
def test_config(fdata, gpu, cfg, capfd):
    D = fdata[0]
    ref = Ref(D)
    env, expect = CONFIGS[cfg]
    cases = [("twelve", TWELVE)] if cfg == "ctas8_twelve" else _subset(D)
    if expect.get("kscan"):
        cases = [c for c in cases if _no_plain_str(c[1])]
    assert len(program(TWELVE)[3]) == 12
    lines = 0   # the kernel lines that showed the configuration: at least one over the subset
    for name, e in cases:
        want = ref.select(e)
        capfd.readouterr()
        with env_vars({**env, "PQB_VERBOSE": 1}):
            if "kr" in expect:
                check_group(D, gpu["resident"], e, want, f"{cfg} {name}")
            else:
                check_pred(D, gpu["resident"], e, want, f"{cfg} {name}", limit=False, group=False)
        log = capfd.readouterr().err
        if "kr" in expect:
            a = AGG_LINE.findall(log)
            # a regex leaf over PLAIN pages takes the RX instantiation, which exists for 2 rows per thread only
            assert all(int(k) == (2 if ",RX" in f else expect["kr"]) for k, f in a), (cfg, name, log)
            lines += sum(int(k) == expect["kr"] for k, f in a)
            continue
        if expect.get("kscan"):
            assert "k_flat_filter" not in log and ("k_scan" in log or not want.any()), (cfg, name, log)
            lines += "k_scan" in log
            continue
        for kern, live, ctas, stages, slab in FILTER_LINE.findall(log):
            lines += 1
            if "ctas" in expect:
                assert int(ctas) == expect["ctas"], (cfg, log)
            if "stages" in expect:
                assert int(stages) == expect["stages"], (cfg, log)
            if expect.get("short_slab"):
                assert int(slab) < 2048, (cfg, log)
    assert lines >= (1 if cfg == "ctas8_twelve" else 3), (cfg, lines)


@pytest.mark.gpu
def test_regex_over_plain_pages_rx(fdata, gpu, capfd):
    """A regex leaf on PLAIN pages in a grouped COUNT: the RX instantiation of k_flat_agg walks the DFA per row."""
    D = fdata[0]
    ref = Ref(D)
    for e in (col("sfb").regex("^common/prefix/"), col("sdba").regex("1$") & (col("s5") != D["s5"].vocab[0]),
              ~col("sdlba").regex("z{2}") | col("b").is_null()):
        capfd.readouterr()
        with env_var("PQB_VERBOSE", 1):
            check_group(D, gpu["resident"], e, ref.select(e), f"rx {e}")
        log = capfd.readouterr().err
        assert any("RX" in f for _, f in AGG_LINE.findall(log)), log


@pytest.mark.gpu
def test_two_shards(fdata):
    """Row-group shards 0/2 and 1/2: their row ids and counts together are the whole."""
    D, _, paths, schema = fdata
    ref = Ref(D)
    for name, e in _subset(D)[:6]:
        want = np.flatnonzero(ref.select(e))
        ids, total = [], 0
        for k in range(2):
            prov = StandardTableProvider(paths, schema=schema, shard_index=k, shard_count=2)
            total += prov.scan(filters=[e], count_only=True).metrics["rows_selected"]
            ids.append(_ids(prov.scan(filters=[e])))
        assert total == len(want), (name, total, len(want))
        assert np.array_equal(np.sort(np.concatenate(ids)), want), name


@pytest.mark.gpu
def test_piece_layout(fdata, gpu, capfd):
    """Pieces start inside pages: the items of a PLAIN8 + narrow-index query include starts off the 32-row grid."""
    capfd.readouterr()
    with env_var("PQB_DEBUG_ITEMS", 1):
        gpu["resident"].scan(filters=[(col("iplain") > 0) & (col("s3") != "a1") & (col("s600") < "b")], count_only=True)
    rows = [int(r) for r in re.findall(r"item \d+ rg \d+ row0 (\d+) nrows", capfd.readouterr().err)]
    assert rows and any(r % 32 for r in rows), rows[:20]
