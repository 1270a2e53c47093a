"""Every place a k_flat_agg cell update can land, checked against exact arithmetic.

A row's update goes to a per-lane cell of one of the `lane_slots` hottest groups, to a hot shared-memory cell (slot <
hot_slots), to a cold cell in L2 (one of `replicas` copies that k_acc_reduce merges), to L2 for whole warps
(PQB_SMEM_SHARE) or for the f64 sums (PQB_F64_GLOBAL), or to a hash-table cell; through the <2>, <4> and <8> rows-per-
thread instantiations and their DIST / PCT / RX variants.  Each configuration below forces one combination with the
planner's own switches and asserts from the PQB_VERBOSE line that it is the one that ran.

The data make every order of summation exact: the Float64 columns `xd`, `xp` and `v*` hold k / 8 with |k| <= 2^30, and
with n <= 2^22 rows every partial sum is a multiple of 1/8 below 2^50.  So SUM and AVG over them must match math.fsum
bit for bit, whatever the tier, the replicas or the atomics' order; a lost, doubled or misplaced update shows.  `xr`
(random doubles) is held to the bound that holds for any summation tree.

CPU: the reference (plain numpy / math.fsum, not the oracle's arithmetic) against Oracle.group_by, and the exactness
argument itself.  GPU: the configuration table."""
import math
import os
import re
from contextlib import ExitStack, contextmanager

import numpy as np
import pyarrow as pa
import pyarrow.compute as pc
import pyarrow.parquet as pq
import pytest

from oracle.oracle import Oracle
from parseable_b200.query import (DeviceTable, StandardTableProvider, avg, col, count, count_distinct, count_star, max_,
                                  median, min_, sum_)

SEED = 20261016
N1, N2 = 1_200_000, 800_000   # two files, six and four row groups; the second one lacks `u`
RG = 200_000
N = N1 + N2
ROWS_PER_SLAB_THREAD = 992    # consumer threads of k_flat_agg: a slab holds krows x 992 rows
U53 = 2.0 ** -53
I64_MIN, I64_MAX = -(1 << 63), (1 << 63) - 1
NV = 10                       # v0 .. v9: wide value-page columns for the wide-stage queries


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
def _dyadic_pool(rng, size, kmax):
    k = rng.integers(-kmax, kmax + 1, size)
    k[0] = 0
    return k / 8.0


def _strings(codes, valid, dictionary):
    return pa.DictionaryArray.from_arrays(pa.array(codes, pa.int32(), mask=~valid), pa.array(dictionary, pa.string())).cast(pa.string())


def make_data(rng):
    """Columns as numpy arrays over all N rows: Utf8 columns as (codes, dictionary), every column with a validity mask."""
    D = {}
    # g: ~5 000 values, Zipf-skewed (the hottest ~20 % of rows), 3 % NULL; its values' names do not follow their heat
    card_g = 5000
    w = 1.0 / np.arange(1, card_g + 1) ** 1.2
    names = rng.permutation(card_g)
    D["g"] = (names[rng.choice(card_g, N, p=w / w.sum())], rng.random(N) >= 0.03, [f"g{i:04d}" for i in range(card_g)])
    D["h"] = (rng.integers(0, 7, N), rng.random(N) >= 0.01, [f"h{i}" for i in range(7)])
    # w1 x w2: 10 000 x 10 000 values (a hashed GROUP BY), but few pairs actually occur
    w1 = rng.integers(0, 10_000, N)
    D["w1"] = (w1, rng.random(N) >= 0.01, [f"w{i:05d}" for i in range(10_000)])
    D["w2"] = ((w1 * 37 + rng.integers(0, 8, N)) % 10_000, np.ones(N, bool), [f"x{i:05d}" for i in range(10_000)])
    # xd: k / 8 from a pool of 3 000, |k| <= 2^20 (a dictionary; decimal with e = 3 inside 32 bits: value pages);
    # -0.0 only in the last row group of the first file, which therefore keeps its index pages
    xd = _dyadic_pool(rng, 3000, 2**20)[rng.integers(0, 3000, N)]
    nz = np.zeros(N, bool)
    nz[N1 - RG:N1] = rng.random(RG) < 0.01
    xd[nz] = -0.0
    D["xd"] = (xd, rng.random(N) >= 0.03)
    # xp: k / 8, |k| <= 2^30, nearly all distinct: the dictionary falls back to PLAIN (read in place as plain-8)
    D["xp"] = (rng.integers(-2**30, 2**30 + 1, N) / 8.0, rng.random(N) >= 0.02)
    D["xr"] = (rng.standard_normal(N) * 10.0 ** rng.uniform(-3, 8, N), rng.random(N) >= 0.02)
    iw_pool = np.where(rng.random(2000) < 0.7, 1, -1) * (2**62 + rng.integers(0, 2**40, 2000))
    D["iw"] = (iw_pool[rng.integers(0, 2000, N)].astype(np.int64), rng.random(N) >= 0.02)
    D["in"] = (rng.integers(0, 16, N).astype(np.int64), rng.random(N) >= 0.02)
    i32_pool = rng.integers(-(2**31) + 1, 2**31, 3000)
    i32_pool[:2] = [-(2**31) + 1, 2**31 - 1]
    D["i32"] = (i32_pool[rng.integers(0, 3000, N)].astype(np.int64), rng.random(N) >= 0.02)
    # s: bytewise order matters (prefixes, upper / lower case, digits)
    sd = sorted({"".join(rng.choice(list("aAbB0z~"), int(rng.integers(0, 6)))) for _ in range(600)})
    D["s"] = (rng.integers(0, len(sd), N), rng.random(N) >= 0.02, sd)
    # u: nearly distinct strings (PLAIN pages: the regex filter walks their bytes); absent from the second file
    u = rng.integers(0, 10**9, N)
    ud = [f"a{v:09d}" for v in u[:N1]]
    D["u"] = (np.concatenate([np.arange(N1), np.zeros(N2, np.int64)]), np.concatenate([np.ones(N1, bool), np.zeros(N2, bool)]), ud)
    for i in range(NV):   # 31-bit value pages: k / 8, |k| <= 2^23 from a pool of 3 000
        D[f"v{i}"] = (_dyadic_pool(rng, 3000, 2**23)[rng.integers(0, 3000, N)], np.ones(N, bool))
    return D


def _arrow(D, name, lo, hi):
    v = D[name]
    if len(v) == 3:
        return _strings(v[0][lo:hi], v[1][lo:hi], v[2])
    arr = v[0][lo:hi]
    return pa.array(arr, pa.float64() if arr.dtype == np.float64 else pa.int64(), mask=~v[1][lo:hi])


@pytest.fixture(scope="module")
def tiers(built, data_dir):
    D = make_data(np.random.default_rng(SEED))
    names = list(D)
    p1, p2 = os.path.join(data_dir, "tiers_1.parquet"), os.path.join(data_dir, "tiers_2.parquet")
    t1 = pa.table({c: _arrow(D, c, 0, N1) for c in names})
    t2 = pa.table({c: _arrow(D, c, N1, N) for c in names if c != "u"})
    for p, t in ((p1, t1), (p2, t2)):
        pq.write_table(t, p, row_group_size=RG, use_dictionary=True, data_page_size=64 * 1024)
    return D, [p1, p2], t1.schema


# ---- reference -------------------------------------------------------------------------------------------------------
def _okey(bits_i64):
    """totalOrder key of f64 bit patterns (as int64); its own inverse."""
    return bits_i64 ^ ((bits_i64 >> 63) & np.int64(0x7FFFFFFFFFFFFFFF))


def _key_codes(D, k):
    codes, valid, dictionary = D[k]
    return np.where(valid, codes, len(dictionary)).astype(np.int64), len(dictionary) + 1


def _filter_mask(D, flt):
    sel = np.ones(N, bool)
    for f in flt:
        if f == "in<6":
            sel &= D["in"][1] & (D["in"][0] < 6)
        elif f == "u~7$":
            codes, valid, ud = D["u"]
            m = np.asarray(pc.match_substring_regex(pa.array(ud), "7$").to_numpy(zero_copy_only=False))
            sel &= valid & m[np.where(valid, codes, 0)]
        else:
            c, value = f.split("!=")
            codes, valid, dictionary = D[c]
            sel &= valid & (codes != dictionary.index(value))
    return sel


def _gpu_filter(f):
    if "!=" in f:
        c, value = f.split("!=")
        return col(c) != value
    return {"in<6": col("in") < 6, "u~7$": col("u").regex("7$")}[f]


class Groups:
    """The selected rows grouped by the key columns: sorted, with the start of every group."""

    def __init__(self, D, keys, sel):
        comb = np.zeros(N, np.int64)
        for k in keys:
            c, card = _key_codes(D, k)
            comb = comb * card + c
        self.rows = np.flatnonzero(sel)
        self.uniq, inv = np.unique(comb[self.rows], return_inverse=True)
        order = np.argsort(inv, kind="stable")
        self.rows, self.inv = self.rows[order], inv[order]
        self.G = len(self.uniq)
        self.starts = np.searchsorted(self.inv, np.arange(self.G))
        self.ends = np.append(self.starts[1:], len(self.rows))


def _fsums(vals, valid, gr):
    """math.fsum over each group's non-NULL values; the empty sum and -0.0 sums as the +0.0 every accumulator starts at."""
    v = np.where(valid, vals, 0.0).tolist()
    out = np.array([math.fsum(v[a:b]) for a, b in zip(gr.starts, gr.ends)], np.float64)
    return out + 0.0


def _reduce(fn, vals, gr):
    return fn.reduceat(vals, gr.starts) if len(vals) else vals


_GROUPS: dict = {}
_FSUMS: dict = {}


def reference(D, keys, aggs, flt=()):
    """{result column: (values, null mask, how)} over the groups in ascending key-code order; `how` says how a result must
    compare: 'exact' (bit for bit), ('bound', tol) or 'str'.  Groups and fsums are kept for the next query over the same
    data, keys and filters."""
    gkey = (id(D), tuple(keys), tuple(flt))
    if gkey not in _GROUPS:
        _GROUPS[gkey] = Groups(D, keys, _filter_mask(D, flt))
    gr = _GROUPS[gkey]
    r = gr.rows
    out = {"__groups__": gr}
    for a in aggs:
        if a.fn == "count_star":
            out[a.name] = (np.bincount(gr.inv, minlength=gr.G).astype(np.int64), np.zeros(gr.G, bool), "exact")
            continue
        v = D[a.column]
        valid = v[1][r]
        nn = np.bincount(gr.inv, weights=valid, minlength=gr.G).astype(np.int64)
        empty = nn == 0
        if a.fn == "count":
            out[a.name] = (nn, np.zeros(gr.G, bool), "exact")
        elif a.fn == "count_distinct":
            pairs = np.unique(gr.inv[valid].astype(np.int64) * (1 << 32) + v[0][r][valid])
            out[a.name] = (np.bincount(pairs >> 32, minlength=gr.G).astype(np.int64), np.zeros(gr.G, bool), "exact")
        elif len(v) == 3:   # MIN / MAX over Utf8: bytewise
            dictionary = v[2]
            rank = np.empty(len(dictionary), np.int64)
            rank[sorted(range(len(dictionary)), key=lambda i: dictionary[i].encode())] = np.arange(len(dictionary))
            rk = rank[np.where(valid, v[0][r], 0)]
            if a.fn == "min":
                best = _reduce(np.minimum, np.where(valid, rk, I64_MAX), gr)
            else:
                best = _reduce(np.maximum, np.where(valid, rk, -1), gr)
            inv_rank = np.argsort(rank)
            out[a.name] = (np.array([dictionary[inv_rank[b]] if not e else None for b, e in zip(best, empty)], object), empty, "str")
        elif v[0].dtype == np.float64:
            x = v[0][r]
            if a.fn in ("sum", "avg"):
                if gkey + (a.column,) not in _FSUMS:
                    _FSUMS[gkey + (a.column,)] = _fsums(x, valid, gr)
                s = _FSUMS[gkey + (a.column,)]
                if a.column == "xr":
                    ab = _reduce(np.add, np.where(valid, np.abs(x), 0.0), gr)
                    m = np.maximum(nn - 1, 0) * U53
                    tol = m * ab / (1 - m) * 1.0001
                    how = ("bound", tol / np.maximum(nn, 1) + 2 * U53 * np.abs(s / np.maximum(nn, 1))) if a.fn == "avg" else ("bound", tol)
                else:
                    how = "exact"
                out[a.name] = ((s / np.maximum(nn, 1)) if a.fn == "avg" else s, empty, how)
            elif a.fn in ("min", "max"):
                k = _okey(x.view(np.int64))
                if a.fn == "min":
                    best = _reduce(np.minimum, np.where(valid, k, I64_MAX), gr)
                else:
                    best = _reduce(np.maximum, np.where(valid, k, I64_MIN), gr)
                out[a.name] = (_okey(best).view(np.float64), empty, "exact")
            elif a.fn == "median":
                xv = x[valid]
                gi = gr.inv[valid]
                o = np.lexsort((_okey(xv.view(np.int64)), gi))
                xs = xv[o]
                st = np.searchsorted(gi[o], np.arange(gr.G))
                lo, hi = st + (nn - 1) // 2, st + nn // 2
                lo_v = xs[np.clip(lo, 0, max(len(xs) - 1, 0))] if len(xs) else np.zeros(gr.G)
                hi_v = xs[np.clip(hi, 0, max(len(xs) - 1, 0))] if len(xs) else np.zeros(gr.G)
                out[a.name] = (np.where(nn % 2 == 1, lo_v, (lo_v + hi_v) / 2.0), empty, "exact")
            else:
                raise ValueError(a)
        else:
            x = v[0][r]
            if a.fn == "sum":   # wrapping, like DataFusion's SUM(Int64)
                s = _reduce(np.add, np.where(valid, x, 0).astype(np.uint64), gr).view(np.int64)
                out[a.name] = (s, empty, "exact")
            elif a.fn == "avg":
                xf = np.where(valid, x, 0).tolist()
                sums = [sum(xf[a0:b0]) for a0, b0 in zip(gr.starts, gr.ends)]
                if a.column == "iw":   # the kernel sums doubles: the order-free bound over the converted values
                    fv = np.where(valid, x.astype(np.float64), 0.0)
                    s = _fsums(fv, valid, gr)
                    ab = _reduce(np.add, np.abs(fv), gr)
                    m = np.maximum(nn - 1, 0) * U53
                    q = s / np.maximum(nn, 1)
                    out[a.name] = (q, empty, ("bound", m * ab / (1 - m) * 1.0001 / np.maximum(nn, 1) + 2 * U53 * np.abs(q)))
                else:                  # |x| < 2^31: the sum is exact, the quotient rounded once
                    out[a.name] = (np.array([sm / n if n else 0.0 for sm, n in zip(sums, nn)], np.float64), empty, "exact")
            elif a.fn in ("min", "max"):
                if a.fn == "min":
                    best = _reduce(np.minimum, np.where(valid, x, I64_MAX), gr)
                else:
                    best = _reduce(np.maximum, np.where(valid, x, I64_MIN), gr)
                out[a.name] = (best, empty, "exact")
            else:
                raise ValueError(a)
    return out


def _result_codes(D, t: pa.Table, keys):
    comb = np.zeros(t.num_rows, np.int64)
    for k in keys:
        _, valid, dictionary = D[k]
        c = pc.index_in(t[k], value_set=pa.array(dictionary, pa.string())).to_numpy(zero_copy_only=False)
        c = np.where(np.isnan(c.astype(np.float64)), len(dictionary), c).astype(np.int64)
        comb = comb * (len(dictionary) + 1) + c
    return comb


def assert_result(D, got: pa.Table, keys, aggs, ref, what):
    gr = ref["__groups__"]
    assert got.column_names == list(keys) + [a.name for a in aggs], what
    assert got.num_rows == gr.G, (what, got.num_rows, gr.G)
    comb = _result_codes(D, got, keys)
    perm = np.argsort(comb, kind="stable")
    assert np.array_equal(comb[perm], gr.uniq), (what, "group keys differ")
    for a in aggs:
        want, null, how = ref[a.name]
        arr = got[a.name].combine_chunks().take(pa.array(perm))
        gnull = arr.is_null().to_numpy(zero_copy_only=False)
        bad = np.flatnonzero(gnull != null)
        assert bad.size == 0, (what, a.name, "NULLs differ", int(bad[0]))
        ok = ~null
        if how == "str":
            g = np.array(arr.to_pylist(), object)
            bad = np.flatnonzero(ok & (g != want))
        elif pa.types.is_floating(arr.type):
            g = arr.fill_null(0.0).to_numpy(zero_copy_only=False)
            if how == "exact":
                bad = np.flatnonzero(ok & (g.view(np.uint64) != np.asarray(want, np.float64).view(np.uint64)))
            else:
                bad = np.flatnonzero(ok & ~(np.abs(g - want) <= how[1]))
        else:
            g = arr.fill_null(0).to_numpy(zero_copy_only=False).astype(np.int64)
            bad = np.flatnonzero(ok & (g != want))
        if bad.size:
            i = int(bad[0])
            raise AssertionError(f"{what}: {a.name}: {bad.size} of {gr.G} groups differ; group code {gr.uniq[i]}: got {g[i]!r}, "
                                 f"want {want[i]!r}")


# ---- queries ---------------------------------------------------------------------------------------------------------
# a query takes at most 8 aggregates: the full list runs as four queries
AGGS_FULL = [
    [count_star(), count("xd"), sum_("xd"), avg("xd"), min_("xd"), max_("xd"), sum_("xp"), avg("xp")],
    [count_star(), min_("xp"), max_("xp"), sum_("xr"), avg("xr"), min_("xr"), max_("xr"), sum_("iw")],
    [count_star(), avg("iw"), min_("iw"), max_("iw"), sum_("i32"), avg("i32"), min_("i32"), max_("i32")],
    [count_star(), sum_("in"), max_("in"), avg("in"), min_("s"), max_("s"), count("xr"), sum_("xd")],
]
AGGS_SMALL = [[count_star(), count("xd"), sum_("xd"), avg("xd"), min_("xd"), max_("xd"), sum_("in"), max_("in")]]

QUERIES = {   # name: (keys, [aggregates of one query, ...], filters)
    "global": ([], AGGS_FULL, ()),
    "g": (["g"], AGGS_FULL, ()),
    "gh": (["g", "h"], AGGS_FULL, ()),
    "hashed": (["w1", "w2"], AGGS_FULL, ()),
    "g_filtered": (["g"], AGGS_FULL, ("in<6",)),
    "g_small": (["g"], AGGS_SMALL, ()),
    "h_small": (["h"], AGGS_SMALL, ()),
    "dist": (["g"], [[count_star(), count_distinct("in"), sum_("xd"), max_("iw")]], ()),
    "pct": (["g"], [[count_star(), median("xd"), sum_("xp"), min_("i32")]], ()),
    "dist_hashed": (["w1", "w2"], [[count_star(), count_distinct("in"), sum_("xp")]], ()),
    "rx": (["g"], [[count_star(), sum_("xd"), avg("i32"), max_("iw")]], ("u~7$",)),
    # wide stages, ~280 and ~300 staged bits per row with value pages: two 14-bit id pages + eight 31-bit value pages;
    # 13 + 3-bit id pages, two 14-bit filtered columns and eight 31-bit value pages next to a hot table of 40 008 groups
    "wide_hashed": (["w1", "w2"], [[sum_(f"v{i}") for i in range(8)]], ()),
    "wide_dense": (["g", "h"], [[sum_(f"v{i}") for i in range(8)]], ("w1!=w00001", "w2!=x00001")),
}
NSLOTS = {"g_small": 5001, "h_small": 8}

VERBOSE = re.compile(r"\[pqb\] k_flat_agg<(\d+)((?:,\w+)*)>: (\d+) CTAs, \d+ B smem/CTA, (\d+) stages x \d+ B, slab (\d+) rows, "
                     r"hot slots (\d+) of (\d+), lane slots (\d+), (\d+) copies, smem share (\d+), f64 global (\d+), "
                     r"value-page slots (\d+), id-page slots (\d+), \d+ flat items")
OFF = re.compile(r"\[pqb\] value pages off: k_flat_agg<(\d+)> is wider than its (\d+)-row slab")


def parse_line(log: str) -> dict:
    lines = VERBOSE.findall(log)
    assert len(lines) == 1, log
    kr, flags, ctas, stages, slab, hot, nslots, lane, copies, share, f64g, vp, ip = lines[0]
    return dict(kr=int(kr), flags=set(f for f in flags.split(",") if f), ctas=int(ctas), stages=int(stages), slab=int(slab),
                hot=int(hot), nslots=int(nslots), lane=int(lane), copies=int(copies), share=int(share), f64g=int(f64g),
                vpages=int(vp), idpages=int(ip))


def check_line(v: dict, query: str, env: dict, expect: dict, what: str):
    keys, parts, flt = QUERIES[query]
    fns = {a.fn for aggs in parts for a in aggs}
    want_flags = set()
    if keys == ["w1", "w2"]:
        want_flags.add("hashed")
    if "count_distinct" in fns:
        want_flags.add("DIST")
    if "median" in fns:
        want_flags.add("PCT")
    if "u~7$" in flt:
        want_flags.add("RX")
    assert v["flags"] == want_flags, (what, v)
    # the planner's invariants: a value page is decoded for all KR rows of a thread, so only over full slabs
    assert v["kr"] in (2, 4, 8) and v["slab"] % ROWS_PER_SLAB_THREAD == 0 and v["slab"] <= v["kr"] * ROWS_PER_SLAB_THREAD, (what, v)
    if v["vpages"]:
        assert v["slab"] == v["kr"] * ROWS_PER_SLAB_THREAD, (what, v)
    if "hashed" in v["flags"]:
        assert v["kr"] == 4 and v["hot"] == 0 and v["lane"] == 0 and v["copies"] == 1, (what, v)
    else:
        assert v["lane"] in (0, 1, 2, 4, 8) and v["lane"] <= v["hot"] <= v["nslots"], (what, v)
        if v["hot"] == v["nslots"] and v["share"] >= 8 and not v["f64g"]:
            assert v["copies"] == 1, (what, v)
    assert v["share"] == int(env.get("PQB_SMEM_SHARE", 8)) and v["f64g"] == int(env.get("PQB_F64_GLOBAL", 0)), (what, v)
    if "PQB_GRID" in env:
        assert v["ctas"] == int(env["PQB_GRID"]), (what, v)
    if query in NSLOTS:
        assert v["nslots"] == NSLOTS[query], (what, v)
    for k, want in expect.items():
        if k == "vpages" and want == ">0":
            assert v["vpages"] > 0, (what, v)
        else:
            assert v[k] == want, (what, k, v)


def kr_of(krows):
    return max(2, krows)


def _krows(k, query="g_small", T=None, hot=None, **more):
    """A row forcing PQB_AGG_KROWS = k on a light query (its stages leave room for 8 rows per thread), optionally with
    PQB_LANE_SLOTS = T and PQB_HOT_SLOTS = hot; krows = 1 runs <2> over 992-row slabs, without value pages."""
    env = {"PQB_AGG_KROWS": k}
    exp = dict(kr=kr_of(k), slab=k * ROWS_PER_SLAB_THREAD, vpages=0 if k == 1 else ">0")
    if T is not None:
        env["PQB_LANE_SLOTS"] = T
        exp["lane"] = min(T, NSLOTS[query])
    if hot is not None:
        env["PQB_HOT_SLOTS"] = hot
        exp["hot"] = max(exp["lane"], min(hot, NSLOTS[query]))
    elif T is not None and query == "h_small":
        exp["hot"] = NSLOTS[query]      # the default: every slot of a small table is hot
    env.update(more)
    return query, env, "resident", exp


H_N1 = NSLOTS["h_small"] - 1
CONFIGS = {
    # rows per thread
    "krows1": _krows(1),
    "krows2": _krows(2),
    "krows4": _krows(4),
    "krows8": _krows(8),
    # lane slots x hot slots (T, T + 1, nslots - 1, default), pairwise with the rows per thread
    "lane0_hotT_k1": _krows(1, T=0, hot=0),
    "lane0_hotT1_k2": _krows(2, T=0, hot=1),
    "lane0_hotN1_k4": _krows(4, "h_small", T=0, hot=H_N1),
    "lane0_hotdef_k8": _krows(8, T=0),
    "lane1_hotT_k2": _krows(2, T=1, hot=1),
    "lane1_hotT1_k4": _krows(4, T=1, hot=2),
    "lane1_hotN1_k8": _krows(8, "h_small", T=1, hot=H_N1),
    "lane1_hotdef_k1": _krows(1, T=1),
    "lane8_hotT_k4": _krows(4, T=8, hot=8),
    "lane8_hotT1_k8": _krows(8, T=8, hot=9),
    "lane8_hotN1_k1": _krows(1, "h_small", T=8, hot=H_N1),
    "lane8_hotdef_k2": _krows(2, T=8),
    # L2 copies: only with a cold slot, whole warps in L2 or the f64 sums in L2
    "replicas1": ("g", {"PQB_REPLICAS": 1}, "resident", dict(copies=1)),
    "replicas3_grid3": ("g", {"PQB_REPLICAS": 3, "PQB_GRID": 3}, "resident", dict(copies=3)),
    "replicas32": ("g", {"PQB_REPLICAS": 32}, "resident", dict(copies=32)),
    "share0_replicas3": ("h_small", {"PQB_SMEM_SHARE": 0, "PQB_REPLICAS": 3}, "resident", dict(copies=3, hot=8)),
    "share3": ("gh", {"PQB_SMEM_SHARE": 3}, "resident", {}),
    "share8_lane8": ("g_small", {"PQB_SMEM_SHARE": 8, "PQB_LANE_SLOTS": 8}, "resident", dict(lane=8)),
    "f64global_replicas32": ("h_small", {"PQB_F64_GLOBAL": 1, "PQB_REPLICAS": 32}, "resident", dict(lane=0, hot=8, copies=32)),
    "f64global_gh": ("gh", {"PQB_F64_GLOBAL": 1}, "resident", dict(lane=0)),
    "f64global0_g": ("g", {"PQB_F64_GLOBAL": 0}, "resident", {}),
    # ring depth and forced grids (each CTA takes many items)
    "stages2": ("g_small", {"PQB_AGG_STAGES": 2, "PQB_AGG_KROWS": 8}, "resident", dict(stages=2, kr=8)),
    "stages4": ("g_small", {"PQB_AGG_STAGES": 4, "PQB_AGG_KROWS": 2}, "resident", dict(stages=4, kr=2)),
    "grid1": ("h_small", {"PQB_GRID": 1}, "resident", dict(hot=8, copies=1)),
    "grid3_hashed": ("hashed", {"PQB_GRID": 3}, "resident", dict(slab=3968)),
    # the forms off, and a file list (no agg pages)
    "forms0_g": ("g", {"PQB_AGG_FORMS": 0}, "resident", dict(vpages=0, idpages=0)),
    "files_g": ("g", {}, "files", dict(vpages=0, idpages=0)),
    "files_hashed": ("hashed", {}, "files", dict(vpages=0, kr=4)),
    # the queries with the planner's defaults
    "global": ("global", {}, "resident", dict(nslots=1)),
    "g": ("g", {}, "resident", {}),
    "gh": ("gh", {}, "resident", {}),
    "hashed": ("hashed", {}, "resident", dict(slab=3968)),
    "g_filtered": ("g_filtered", {}, "resident", {}),
    # COUNT(DISTINCT) and MEDIAN at 1, 2, 4 and 8 rows per thread (no agg pages in those instantiations)
    **{f"dist_k{k}": ("dist", {"PQB_AGG_KROWS": k}, "resident", dict(kr=kr_of(k), slab=k * ROWS_PER_SLAB_THREAD, vpages=0)) for k in (1, 2, 4, 8)},
    **{f"pct_k{k}": ("pct", {"PQB_AGG_KROWS": k}, "resident", dict(kr=kr_of(k), slab=k * ROWS_PER_SLAB_THREAD, vpages=0)) for k in (1, 2, 4, 8)},
    "dist_hashed": ("dist_hashed", {}, "resident", dict(vpages=0)),
    # a regular expression over PLAIN strings: the RX instantiation
    "rx": ("rx", {}, "resident", dict(kr=2)),
}


@pytest.fixture(scope="module")
def providers(tiers):
    D, files, schema = tiers
    table = DeviceTable(files, schema.names)
    yield {"resident": StandardTableProvider(table, schema=schema), "files": StandardTableProvider(files, schema=schema)}
    table.close()


_REF_CACHE: dict = {}


def _ref(D, query, part):
    if (query, part) not in _REF_CACHE:
        keys, parts, flt = QUERIES[query]
        _REF_CACHE[query, part] = reference(D, keys, parts[part], flt)
    return _REF_CACHE[query, part]


def run(providers, query, env, src, capfd):
    """Every query of the row: (its aggregates, result, PQB_VERBOSE log)."""
    keys, parts, flt = QUERIES[query]
    out = []
    for aggs in parts:
        capfd.readouterr()
        with env_vars({**env, "PQB_VERBOSE": 1}):
            got = providers[src].aggregate(keys, aggs, [_gpu_filter(f) for f in flt]).table()
        out.append((aggs, got, capfd.readouterr().err))
    return out


# ---- CPU: the reference against the oracle, and the exactness argument ---------------------------------------------
def test_reference_matches_oracle(tiers):
    D, files, schema = tiers
    t = pa.concat_tables([pq.read_table(files[0]), pq.read_table(files[1]).append_column("u", pa.nulls(N2, pa.string())).select(schema.names)])
    ora = Oracle(t)
    aggs = [count_star(), count("xd"), sum_("xd"), sum_("xp"), min_("xd"), max_("xd"), min_("xp"), max_("xp"), min_("xr"),
            max_("xr"), min_("iw"), max_("iw"), min_("i32"), max_("i32"), count("iw")]
    for keys, flt in ((["g"], ()), (["g", "h"], ()), ([], ())):
        ref = reference(D, keys, aggs, flt)
        assert_result(D, ora.group_by(keys, aggs), keys, aggs, ref, f"oracle vs reference {keys}")


def test_dyadic_sums_are_order_free(tiers):
    """Permuted numpy sums (pairwise within a group, in any row order) equal math.fsum bit for bit on `xd` and `xp`."""
    D, _, _ = tiers
    rng = np.random.default_rng(7)
    for c in ("xd", "xp"):
        x, valid = D[c]
        want = math.fsum(x[valid].tolist())
        for _ in range(3):
            p = rng.permutation(N)
            assert np.sum(np.where(valid, x, 0.0)[p]) == want
            assert np.cumsum(np.where(valid, x, 0.0)[p])[-1] == want
        gr = Groups(D, ["g"], np.ones(N, bool))
        fs = _fsums(x[gr.rows], valid[gr.rows], gr)
        p = rng.permutation(len(gr.rows))
        # the same groups, rows in a random order inside each group
        o = np.lexsort((p, gr.inv))
        sums = np.add.reduceat(np.where(valid[gr.rows], x[gr.rows], 0.0)[o], gr.starts) + 0.0
        assert np.array_equal(sums.view(np.uint64), fs.view(np.uint64)), c


# ---- GPU -------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("cfg", list(CONFIGS))
def test_tier(tiers, providers, cfg, capfd):
    D, _, _ = tiers
    query, env, src, expect = CONFIGS[cfg]
    keys = QUERIES[query][0]
    for part, (aggs, got, log) in enumerate(run(providers, query, env, src, capfd)):
        what = f"{cfg} / {part}"
        check_line(parse_line(log), query, {k: str(v) for k, v in env.items()}, expect, what)
        off = OFF.findall(log)
        if env.get("PQB_AGG_KROWS") == 1 and src == "resident" and query in ("g_small", "h_small"):
            assert off == [("2", "992")], (what, log)   # the <2> instantiation over 992-row slabs: value pages off
        assert_result(D, got, keys, aggs, _ref(D, query, part), what)


@pytest.mark.gpu
@pytest.mark.parametrize("query,kr", [("wide_hashed", 4), ("wide_dense", 2)])
def test_wide_stages_read_index_pages(tiers, providers, query, kr, capfd):
    """Planner-chosen plans (no switches) whose stages leave room for fewer rows per thread than the launched
    instantiation decodes: the query qualifies for value pages, the planner turns them off, the answer is exact."""
    D, _, _ = tiers
    keys = QUERIES[query][0]
    [(aggs, got, log)] = run(providers, query, {}, "resident", capfd)
    assert "(v0): value pages" in log, log                  # the columns qualify for value pages ...
    off = OFF.findall(log)
    assert len(off) == 1 and int(off[0][0]) == kr and int(off[0][1]) < kr * ROWS_PER_SLAB_THREAD, log
    v = parse_line(log)                                     # ... and the kernel ran without them
    check_line(v, query, {}, dict(kr=kr, vpages=0), query)
    if query == "wide_dense":
        assert int(off[0][1]) == ROWS_PER_SLAB_THREAD, log
    assert_result(D, got, keys, aggs, _ref(D, query, 0), query)
