"""The multi-rank path (PQ_QUERY_ALLREDUCE with more than one rank) on ONE device: 2, 3, 4 and 8 ranks as processes over
the host-staged communicator build (tools/comm_host.cpp), every key kind, aggregate and refusal checked three ways:

(a) every rank's result is identical to rank 0's, valid values bit for bit and rows in the same order;
(b) it is the whole table's answer: the oracle's GROUP BY for the numeric aggregates, a restated reference for MIN / MAX
    over Utf8 and Boolean, and the NULL groups, wrapping Int64 sums and Float64 bit patterns of the keys;
(c) without the flag, each rank's answer is the one over its own row groups g % n == rank (g global across files),
    with global __row_id ordinals.

The data is built so that the ranks disagree: a different hottest `s` per row group, `s` values of one row group only
and an all-NULL row group; `sp` falls back to PLAIN pages in one row group only; `i` has a dictionary in one file and
PLAIN pages in the other; `opt` is absent from the second file; the second file also has a copy without statistics.
Queries that only some ranks can answer (the PLAIN `sp` row group, DATE_BIN without statistics) must be refused by
EVERY rank, well within the communicator's timeout, and the next query must still be answered."""
import ctypes as C
import json
import math
import os
import shutil
import struct
import subprocess
import sys

import numpy as np
import pyarrow as pa
import pyarrow.parquet as pq
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests", "scripts"))
import ranks_worker as W  # noqa: E402

HOSTCOMM = os.path.join(ROOT, "tools", "libparseable_b200_hostcomm.so")
NRANKS = (2, 3, 4, 8)
RG_ROWS = [20_000, 33_000, 27_000, 40_000, 24_000, 36_000, 30_000]
FILE_RGS = (4, 3)              # row groups of the first and the second file
SP_PLAIN_RG, S_NULL_RG, X_NULL_RG, B_TRUE_RG = 5, 3, 1, 2
TIMEOUT_MS = 20_000            # the communicator's bound on one wait; refusals must come back well within it
SEED = 20261017


# ---- data ------------------------------------------------------------------------------------------------------------
def _nan(bits):
    return np.array([bits], np.uint64).view(np.float64)[0]


F_POOL = np.array([0.0, -0.0, np.inf, -np.inf, 1.5, -2.25, 3.0, 0.375, -6.5, 7.125], np.float64)   # finite ones: k / 8
F_NANS = [_nan(0x7FF8000000000001), _nan(0xFFF8000000000002), _nan(0x7FF8000000000F00), _nan(0xFFF0000000000007)]


def _rg_table(g, r0, m, rng):
    def nulls(rate):
        return rng.random(m) < rate
    s_common = np.array([f"s{j:03d}" for j in range(40)], object)
    s = s_common[rng.integers(0, 40, m)]
    s[rng.random(m) < 0.5] = f"hot{g}"
    only = rng.random(m) < 0.05
    s[only] = [f"only{g}_{j:02d}" for j in rng.integers(0, 60, int(only.sum()))]
    s_mask = np.ones(m, bool) if g == S_NULL_RG else nulls(0.02)
    if g == SP_PLAIN_RG:   # unique values past the dictionary page limit: this chunk falls back to PLAIN pages
        sp = np.array([f"v{g}_{k:08d}_{'x' * (k % 7)}" for k in range(m)], object)
    else:
        sp = np.array([f"v{j:02d}" for j in range(60)], object)[rng.integers(0, 60, m)]
    f = F_POOL[rng.integers(0, len(F_POOL), m)]
    nan_rows = rng.random(m) < 0.04
    f[nan_rows] = np.array(F_NANS)[rng.integers(0, len(F_NANS), int(nan_rows.sum()))]
    ts = W.ts_bound(g) + np.sort(rng.integers(0, 20 * W.HOUR, m))
    x = rng.integers(-4000, 4000, m) / 8.0           # k / 8: every SUM / AVG is exact in any order
    w = rng.integers(-300, 300, m) + np.where(rng.random(m) < 0.5, 1, -1) * (1 << 62)   # near +-2^62: partial sums wrap
    b = np.ones(m, bool) if g == B_TRUE_RG else rng.random(m) < 0.4
    cols = {
        "rid": pa.array(np.arange(r0, r0 + m, dtype=np.int64)),
        "rnd": pa.array(rng.integers(-(1 << 63), (1 << 63) - 1, m, dtype=np.int64)),
        "s": pa.array(s, pa.string(), mask=s_mask),
        "sp": pa.array(sp, pa.string(), mask=nulls(0.01)),
        "i": pa.array(rng.integers(-300, 300, m) * 7, pa.int64(), mask=nulls(0.01)),
        "f": pa.array(f, pa.float64(), mask=nulls(0.01)),
        "b": pa.array(b, pa.bool_(), mask=nulls(0.03)),
        "ts": pa.array(ts, pa.timestamp("ms"), mask=nulls(0.005)),
        "x": pa.array(x, pa.float64(), mask=nulls(0.05) if g == X_NULL_RG else None),
        "w": pa.array(w.astype(np.int64)),
    }
    if g < FILE_RGS[0]:
        cols["opt"] = pa.array(rng.integers(0, 10, m), pa.int64(), mask=nulls(0.1))
    return pa.table(cols)


def _write(path, tables, use_dictionary, stats=True):
    kw = dict(use_dictionary=use_dictionary, column_encoding={"ts": "DELTA_BINARY_PACKED"}, data_page_size=8192,
              dictionary_pagesize_limit=100_000, write_statistics=stats, compression="snappy")
    with pq.ParquetWriter(path, tables[0].schema, **kw) as wr:
        for t in tables:
            wr.write_table(t, row_group_size=t.num_rows)


@pytest.fixture(scope="module")
def data(tmp_path_factory):
    d = tmp_path_factory.mktemp("ranks")
    rng = np.random.default_rng(SEED)
    rgs, r0 = [], 0
    for g, m in enumerate(RG_ROWS):
        rgs.append(_rg_table(g, r0, m, rng))
        r0 += m
    a, b, b_nostats = str(d / "a.parquet"), str(d / "b.parquet"), str(d / "b_nostats.parquet")
    _write(a, rgs[:FILE_RGS[0]], ["s", "sp", "i", "f", "x", "opt"])
    _write(b, rgs[FILE_RGS[0]:], ["s", "sp", "f", "x"])          # `i` has PLAIN pages in this file
    _write(b_nostats, rgs[FILE_RGS[0]:], ["s", "sp", "f", "x"], stats=False)
    table = pa.concat_tables(rgs, promote_options="default")
    starts = np.cumsum([0] + RG_ROWS)
    return {"dir": str(d), "files": [a, b], "nostats": [a, b_nostats], "table": table, "starts": starts}


def test_data_layout(data):
    """The row groups hold what the cases rely on: 7 of them across two files, `i` with a dictionary in the first file
    only, `ts` DELTA, no statistics in the copy, `opt` in the first file only.  (That `sp` has PLAIN pages in one row
    group only shows in which rank refuses the `sp` cases.)"""
    g = 0
    for path, nostats in zip(data["files"], data["nostats"]):
        md = pq.ParquetFile(path).metadata
        for r in range(md.num_row_groups):
            cc = {md.row_group(r).column(c).path_in_schema: md.row_group(r).column(c) for c in range(md.num_columns)}
            assert ("RLE_DICTIONARY" in cc["i"].encodings) == (g < FILE_RGS[0]), (g, cc["i"].encodings)
            assert "DELTA_BINARY_PACKED" in cc["ts"].encodings
            assert cc["ts"].is_stats_set
            assert ("opt" in cc) == (g < FILE_RGS[0])
            g += 1
        if nostats != path:
            md2 = pq.ParquetFile(nostats).metadata
            assert not any(md2.row_group(r).column(c).is_stats_set for r in range(md2.num_row_groups) for c in range(md2.num_columns))
    assert g == len(RG_ROWS)


# ---- canonical results -----------------------------------------------------------------------------------------------
def _bits(v):
    return struct.unpack("<q", struct.pack("<d", v))[0]


def _canon_value(v, fn=None):
    if isinstance(v, float):
        if fn in ("sum", "avg") and math.isnan(v):
            return "nan"      # the payload of a NaN that arithmetic made is not specified
        return ("f", _bits(v))
    return v


def _columns(t):
    out = []
    for c in t.columns:
        c = c.combine_chunks() if isinstance(c, pa.ChunkedArray) else c
        if pa.types.is_timestamp(c.type):
            c = c.cast(pa.int64())
        out.append(c.to_pylist())
    return out


def canon_rows(t, fns):
    """Rows of a result as tuples, Float64 values as their bits (NaN of SUM / AVG as one value)."""
    if t.num_rows == 0:
        return []
    cols = _columns(t)
    assert len(cols) == len(fns), (t.column_names, fns)
    return [tuple(_canon_value(v, fn) for v, fn in zip(row, fns)) for row in zip(*cols)]


def _fns(keys, aggs):
    return [None] * len(keys) + [a.fn for a in aggs]


def _str_or_bool(t, a):
    return a.fn in ("min", "max") and (pa.types.is_string(t.schema.field(a.column).type) or pa.types.is_boolean(t.schema.field(a.column).type))


def reference(t, keys, aggs, flt):
    """{key tuple: aggregate tuple} of table `t`, canonical like canon_rows."""
    from oracle.oracle import Oracle
    from parseable_b200.query import count_star
    ora = Oracle(t)
    filters = W.filters_of(flt)
    numeric = [a for a in aggs if not _str_or_bool(t, a)]
    got = ora.group_by(keys, numeric or [count_star()], filters)
    rows = canon_rows(got, _fns(keys, numeric or [count_star()]))
    nk = len(keys)
    groups = {r[:nk]: dict(zip([id(a) for a in numeric], r[nk:])) for r in rows}
    special = [a for a in aggs if _str_or_bool(t, a)]
    if special:
        sel = ora.select(filters).astype(bool)
        kcols = []
        for k in keys:
            if hasattr(k, "width_ms"):
                kcols.append([None if x is None else (x - k.origin_ms) // k.width_ms * k.width_ms + k.origin_ms
                              for x in t[k.column].cast(pa.int64()).to_pylist()])
            else:
                kcols.append([_canon_value(v) for v in _columns(t.select([k]))[0]])
        for a in special:
            vals = t[a.column].to_pylist()
            acc = {}
            for r in np.flatnonzero(sel):
                kt = tuple(c[r] for c in kcols)
                v = vals[r]
                if v is None:
                    acc.setdefault(kt, None)
                    continue
                cur = acc.get(kt)
                acc[kt] = v if cur is None else (min(cur, v) if a.fn == "min" else max(cur, v))
            if not keys and not acc:
                acc[()] = None
            for kt, v in acc.items():
                assert kt in groups, (kt, "a group the oracle lacks")
                groups[kt][id(a)] = v
    return {kt: tuple(g.get(id(a)) for a in aggs) for kt, g in groups.items()}


def as_groups(rows, nk, what):
    out = {}
    for r in rows:
        assert r[:nk] not in out, (what, "duplicate group", r[:nk])
        out[r[:nk]] = r[nk:]
    return out


def check_groups(got_rows, want, nk, what):
    got = as_groups(got_rows, nk, what)
    assert len(got) == len(want), (what, "groups", len(got), len(want), sorted(set(want) - set(got), key=repr)[:3],
                                   sorted(set(got) - set(want), key=repr)[:3])
    for kt, v in want.items():
        assert kt in got, (what, "missing group", kt)
        assert got[kt] == v, (what, kt, got[kt], v)


def _sort_key(v, desc=False, nulls_last=True):
    """A Python sort key of one canonical value (ASC NULLS LAST unless told otherwise)."""
    if v is None:
        return (1 if nulls_last else -1, 0)
    if isinstance(v, tuple):
        v = struct.unpack("<d", struct.pack("<q", v[1]))[0]
    return (0, -v if desc else v)


# ---- runs ------------------------------------------------------------------------------------------------------------
def _spawn(data, n):
    out = os.path.join(data["dir"], f"out{n}")
    comm = os.path.join(data["dir"], f"comm{n}")
    os.makedirs(out, exist_ok=True)
    os.makedirs(comm, exist_ok=True)
    spec = os.path.join(out, "spec.json")
    with open(spec, "w") as f:
        json.dump({"files": data["files"], "nostats": data["nostats"], "out": out, "idfile": os.path.join(comm, "id")}, f)
    env = {**os.environ, "PQB_LIB": HOSTCOMM, "PQB_COMM_DIR": comm, "PQB_COMM_TIMEOUT_MS": str(TIMEOUT_MS)}
    env.pop("PQB_VERBOSE", None)
    procs = [subprocess.Popen([sys.executable, os.path.join(ROOT, "tests", "scripts", "ranks_worker.py"), str(r), str(n), spec],
                              stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, env=env) for r in range(n)]
    return out, comm, procs


def _ensure_hostcomm():
    if not os.path.exists(HOSTCOMM):
        subprocess.check_call(["make", "-C", ROOT, "-j4", os.path.relpath(HOSTCOMM, ROOT)])


@pytest.fixture(scope="module")
def runs(data, built):
    """The rank counts one after another (a shared device keeps each rank's latency predictable), each in its own exchange
    directory; the workers are always reaped."""
    _ensure_hostcomm()
    started = []
    res = {}
    try:
        for n in NRANKS:
            out, comm, procs = _spawn(data, n)
            started.append(procs)
            logs = [p.communicate(timeout=600)[0] for p in procs]
            for r, (p, log) in enumerate(zip(procs, logs)):
                assert p.returncode == 0, f"n={n} rank {r}:\n{log[-4000:]}"
            # the exchange directory: no half-written file, and at most the last collective's file of each rank and session
            left = [x for x in os.listdir(comm) if not x.startswith("id")]
            assert not [x for x in left if x.endswith(".tmp")], left
            per = {}
            for x in left:
                tag, _, rank = x.split(".")
                per[(tag, rank)] = per.get((tag, rank), 0) + 1
            assert all(v == 1 for v in per.values()), per
            assert len(per) <= 2 * n, per          # two sessions: the first communicator and the one after re-init
            shutil.rmtree(comm)
            res[n] = out
        return res
    finally:
        for procs in started:
            for p in procs:
                if p.poll() is None:
                    p.kill()
                p.wait()


def load(out, name, src, rank):
    base = os.path.join(out, f"{name}.{src}.{rank}")
    if os.path.exists(base + ".json"):
        return json.load(open(base + ".json"))
    assert os.path.exists(base + ".arrow"), f"{base}: no result"
    with pa.memory_map(base + ".arrow") as f:
        return pa.ipc.open_file(f).read_all()


SOURCES = ("table", "files")


def _case_results(out, n, name, src, fns):
    res = [load(out, name, src, r) for r in range(n)]
    for r in range(n):
        assert not isinstance(res[r], dict), (name, src, f"rank {r} refused", res[r])
    rows = [canon_rows(t, fns) if "json" not in t.column_names else t["json"].to_pylist() for t in res]
    for r in range(1, n):
        assert rows[r] == rows[0], (name, src, f"rank {r} differs from rank 0")
    return res[0], rows[0]


@pytest.fixture(scope="module")
def refs(data):
    """Whole-table references by case name, computed once for every rank count."""
    return {}


def _want(data, refs, name):
    if name not in refs:
        keys, aggs, flt, _ = W.CASES[name]
        refs[name] = reference(data["table"], keys, aggs, flt)
    return refs[name]


@pytest.mark.gpu
@pytest.mark.parametrize("n", NRANKS)
def test_allreduce_cases(runs, data, refs, n):
    """(a) and (b) for every case under PQ_QUERY_ALLREDUCE, on a resident table and on a file list."""
    for src in SOURCES:
        for name, (keys, aggs, flt, kw) in W.CASES.items():
            what = f"n={n} {src} {name}"
            t, rows = _case_results(runs[n], n, name, src, _fns(keys, aggs) + (["rn"] if "window" in kw else []))
            want = _want(data, refs, name)
            nk = len(keys)
            if "json" in kw:
                recs = [json.loads(x) for x in rows[0].splitlines() if x]
                got = {}
                for r in recs:
                    kt = tuple(r.get(k) for k in keys)
                    got[kt] = tuple(_canon_value(r.get(a.name), a.fn) for a in aggs)
                assert got == want, what
            elif kw.get("order_by") and "window" not in kw:
                # count(*) DESC, s ASC NULLS LAST, first `limit` groups
                order = sorted(want.items(), key=lambda kv: (-kv[1][0], _sort_key(kv[0][0])))[: kw["limit"]]
                assert [r[:nk] + r[nk:] for r in rows] == [k + v for k, v in order], what
            elif "window" in kw:
                # ROW_NUMBER() OVER (PARTITION BY b ORDER BY count(*) DESC, s ASC), rn <= 3
                parts = {}
                for k, v in want.items():
                    parts.setdefault(k[0], []).append((k, v))
                exp = []
                for b in sorted(parts, key=_sort_key):
                    top = sorted(parts[b], key=lambda kv: (-kv[1][0], _sort_key(kv[0][1])))[:3]
                    exp += [k + v + (i + 1,) for i, (k, v) in enumerate(top)]
                assert sorted(rows, key=repr) == sorted(exp, key=repr), what
                for b in parts:   # within a partition, in rank order
                    got_b = [r for r in rows if r[0] == b]
                    assert [r[-1] for r in got_b] == list(range(1, len(got_b) + 1)), what
            else:
                check_groups(rows, want, nk, what)


def _shard_table(data, n, r):
    starts = data["starts"]
    parts = [data["table"].slice(starts[g], RG_ROWS[g]) for g in range(len(RG_ROWS)) if g % n == r]
    return pa.concat_tables(parts) if parts else data["table"].slice(0, 0)


@pytest.mark.gpu
@pytest.mark.parametrize("n", NRANKS)
def test_local_shards(runs, data, n):
    """(c) without PQ_QUERY_ALLREDUCE: each rank answers for its own row groups, __row_id global."""
    for r in range(n):
        t = _shard_table(data, n, r)
        for name in W.LOCAL:
            keys, aggs, flt, _ = W.CASES[name]
            want = reference(t, keys, aggs, flt) if t.num_rows else {}
            for src in SOURCES:
                got = load(runs[n], "local_" + name, src, r)
                assert not isinstance(got, dict), (n, r, name, src, got)
                check_groups(canon_rows(got, _fns(keys, aggs)), want, len(keys), f"n={n} rank {r} {src} local {name}")
        x = t["x"].to_numpy(zero_copy_only=False) if t.num_rows else np.zeros(0)
        valid = t["x"].is_valid().to_numpy(zero_copy_only=False) if t.num_rows else np.zeros(0, bool)
        want_ids = t["rid"].to_numpy()[valid & (np.nan_to_num(x) > 0)] if t.num_rows else np.zeros(0, np.int64)
        for src in SOURCES:
            got = load(runs[n], "local_rowids", src, r)
            ids = got.column(0).to_numpy() if got.num_rows else np.zeros(0, np.int64)
            assert np.array_equal(ids, want_ids), (n, r, src, "__row_id", len(ids), len(want_ids))


@pytest.mark.gpu
@pytest.mark.parametrize("n", NRANKS)
def test_refusals_are_collective(runs, data, refs, n):
    """Every rank refuses together, with the cause from the rank that met it, well within the timeout; the next query
    on the same communicator is answered."""
    own = {"refuse_distinct": "COUNT(DISTINCT", "refuse_median": "MEDIAN",
           "refuse_sp_like": "without a dictionary", "refuse_minmax_sp_like": "without a dictionary",
           "refuse_bin_nostats": "min / max statistics"}
    divergent = {"refuse_sp_like", "refuse_minmax_sp_like", "refuse_bin_nostats"}
    nostats_ranks = {g % n for g in range(FILE_RGS[0], len(RG_ROWS))}
    for name in own:
        for src in (SOURCES if name != "refuse_bin_nostats" else ("files",)):
            errs = [load(runs[n], name, src, r) for r in range(n)]
            for r, e in enumerate(errs):
                what = f"n={n} {src} {name} rank {r}"
                assert isinstance(e, dict), (what, "answered")
                assert e["code"] == -2, (what, e)        # PQ_ERR_UNSUPPORTED, never a communicator timeout
                assert e["seconds"] < TIMEOUT_MS / 4000, (what, e["seconds"])
                if name not in divergent:
                    assert own[name] in e["message"], (what, e)
                    continue
                cause = {SP_PLAIN_RG % n} if name != "refuse_bin_nostats" else nostats_ranks
                if r in cause:
                    assert own[name] in e["message"], (what, e)
                else:
                    assert "refused on rank" in e["message"], (what, e)
            key = "after_" + name
            keys, aggs, flt, _ = W.CASES["fp_s" if name != "refuse_bin_nostats" else "fp_bin"]
            _, rows = _case_results(runs[n], n, key, src, _fns(keys, aggs))
            check_groups(rows, _want(data, refs, "fp_s" if name != "refuse_bin_nostats" else "fp_bin"), len(keys), f"n={n} {src} {key}")


@pytest.mark.gpu
@pytest.mark.parametrize("n", NRANKS)
def test_agreement_cache(runs, data, refs, n):
    """The agreed numbering kept with the table: the same query again, after rank 1 alone reopens its table, and on a new
    communicator (a new epoch)."""
    for step in ("again", "reopen", "epoch"):
        for name in ("fp_s", "minmax_str_by_s"):
            keys, aggs, _, _ = W.CASES[name]
            _, rows = _case_results(runs[n], n, f"cache_{step}_{name}", "table", _fns(keys, aggs))
            check_groups(rows, _want(data, refs, name), len(keys), f"n={n} cache {step} {name}")


def test_hostcomm_exports_header(built):
    """The host-staged build exports every symbol the header declares, and does not link NCCL."""
    import re
    from parseable_b200 import _lib as L
    _ensure_hostcomm()
    hdr = open(os.path.join(ROOT, "include", "parseable_b200.h")).read()
    declared = set(re.findall(r"\b(pq_[a-z_0-9]+)\s*\(", hdr))
    assert declared == set(L.EXPORTS)
    lib = C.CDLL(HOSTCOMM)
    for name in declared:
        assert hasattr(lib, name), name
    needed = _elf_needed(HOSTCOMM)
    assert any("libcudart" in x for x in needed), needed
    assert not [x for x in needed if "nccl" in x], needed


def _elf_needed(path):
    """DT_NEEDED entries of a 64-bit little-endian ELF shared object."""
    with open(path, "rb") as f:
        blob = f.read()
    assert blob[:4] == b"\x7fELF" and blob[4] == 2 and blob[5] == 1
    shoff, = struct.unpack_from("<Q", blob, 0x28)
    shentsize, shnum = struct.unpack_from("<HH", blob, 0x3A)
    secs = [struct.unpack_from("<IIQQQQIIQQ", blob, shoff + i * shentsize) for i in range(shnum)]
    dyn = [s for s in secs if s[1] == 6]          # SHT_DYNAMIC
    assert dyn
    _, _, _, _, off, size, link, _, _, entsize = dyn[0]
    stroff = secs[link][4]
    out = []
    for e in range(size // entsize):
        tag, val = struct.unpack_from("<qQ", blob, off + e * entsize)
        if tag == 1:                              # DT_NEEDED
            end = blob.index(b"\0", stroff + val)
            out.append(blob[stroff + val:end].decode())
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("n", (2, 3))
@pytest.mark.parametrize("script", ("mgpu_check.py", "mgpu_order_check.py", "mgpu_minmax_check.py"))
def test_multi_gpu_scripts_on_one_device(small_files, tmp_path, built, script, n):
    """The two-GPU parity scripts, with every rank on device 0 over the host-staged communicator (mgpu_check.py with
    its split files, one NULL-free)."""
    from parseable_b200 import synth
    _ensure_hostcomm()
    args = [small_files["nulls"], small_files["nn"]]
    if script == "mgpu_check.py":
        split = []
        for tag, rate, rg in (("nn", 0.0, 5), ("nulls", 0.02, 7), ("nn2", 0.0, 9))[:n]:
            p = str(tmp_path / f"one_{tag}.parquet")
            synth.write_logs16(p, n_row_groups=1, first_rg=rg, rows_per_group=50_000, null_rate=rate)
            split.append(p)
        args += ["--"] + split
    comm = tmp_path / "comm"
    comm.mkdir()
    env = {**os.environ, "PQB_LIB": HOSTCOMM, "PQB_COMM_DIR": str(comm), "PQB_COMM_TIMEOUT_MS": str(TIMEOUT_MS),
           "PQB_RANK_DEVICE": "0"}
    procs = [subprocess.Popen([sys.executable, os.path.join(ROOT, "tests", "scripts", script), str(r), str(n), str(comm / "id")] + args,
                              stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, env=env) for r in range(n)]
    try:
        outs = [p.communicate(timeout=300)[0] for p in procs]
    finally:
        for p in procs:
            if p.poll() is None:
                p.kill()
            p.wait()
    for r, (p, o) in enumerate(zip(procs, outs)):
        assert p.returncode == 0, f"{script} n={n} rank {r}:\n{o[-3000:]}"
