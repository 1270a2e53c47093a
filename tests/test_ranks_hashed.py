"""A hashed GROUP BY under PQ_QUERY_ALLREDUCE on ONE device: 1, 2, 3 and 8 ranks as processes over the host-staged
communicator build (tools/comm_host.cpp), each key tuple wider than 2^26 combinations in the ranks' agreed numbering.
Every rank's listed groups are gathered and merged on the device (hash_merge.cuh).  Each case is checked three ways:

(a) every rank's result is identical to rank 0's, bit for bit and rows in the same order, and a second run over the
    resident table gives the same order;
(b) it is the whole table's answer, with the references of test_ranks_one_gpu.py;
(c) the PQB_VERBOSE lines show the hashed table and its merge; GROUP BY u, i is dense on every rank alone (n >= 2).

The data (7 row groups in two files): `u` with ~12 000 values, most of them in one row group only; `i` with a dictionary
in the first file and PLAIN pages in the second; `f` with +-0.0 and NaN payloads; a Boolean `b`; DATE_BIN over `ts` at a
1-minute bin; NULLs in every key; `opt` absent from the second file.  One rank owns nothing at n = 8.  A table that runs
full on one rank, and an exchange above one rank's budget, are refused by every rank with the same code, naming that
rank, well within the communicator's timeout, and the next query is answered."""
import json
import os
import re
import shutil
import subprocess
import sys

import numpy as np
import pyarrow as pa
import pyarrow.parquet as pq
import pytest

import test_ranks_one_gpu as R

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests", "scripts"))
import ranks_hashed_worker as HW  # noqa: E402
import ranks_worker as W  # noqa: E402

NRANKS = (1, 2, 3, 8)
RG_ROWS = [12_000, 15_000, 11_000, 14_000, 10_000, 13_000, 12_000]
FILE_RGS = (4, 3)
U_COMMON, U_OWN = 4000, 1200        # `u`: values every row group draws from, and values of one row group only
I_COMMON, I_OWN = 1500, 700
SEED = 20261018
TIMEOUT_MS = R.TIMEOUT_MS


# ---- data ------------------------------------------------------------------------------------------------------------
def _rg_table(g, r0, m, rng):
    def nulls(rate):
        return rng.random(m) < rate
    own = rng.random(m) < 0.4
    u = np.where(own, np.char.add(f"g{g}_", rng.integers(0, U_OWN, m).astype(str)),
                 np.char.add("c", rng.integers(0, U_COMMON, m).astype(str))).astype(object)
    i = np.where(rng.random(m) < 0.4, 100_000 + g * 1000 + rng.integers(0, I_OWN, m), rng.integers(0, I_COMMON, m) * 7)
    f = rng.integers(-3000, 3000, m) / 8.0
    f[rng.random(m) < 0.02] = -0.0
    nan_rows = rng.random(m) < 0.02
    f[nan_rows] = np.array(R.F_NANS)[rng.integers(0, len(R.F_NANS), int(nan_rows.sum()))]
    fn = rng.integers(-4000, 4000, m) / 8.0
    fn[rng.random(m) < 0.01] = np.inf
    nan_rows = rng.random(m) < 0.01
    fn[nan_rows] = np.array(R.F_NANS)[rng.integers(0, len(R.F_NANS), int(nan_rows.sum()))]
    w = rng.integers(-300, 300, m) + np.where(rng.random(m) < 0.5, 1, -1) * (1 << 62)
    cols = {
        "rid": pa.array(np.arange(r0, r0 + m, dtype=np.int64)),
        "rnd": pa.array(rng.integers(-(1 << 63), (1 << 63) - 1, m, dtype=np.int64)),
        "u": pa.array(u, pa.string(), mask=nulls(0.02)),
        "i": pa.array(i.astype(np.int64), pa.int64(), mask=nulls(0.01)),
        "f": pa.array(f, pa.float64(), mask=nulls(0.01)),
        "b": pa.array(rng.random(m) < 0.4, pa.bool_(), mask=nulls(0.03)),
        "ts": pa.array(W.ts_bound(g) + np.sort(rng.integers(0, 20 * W.HOUR, m)), pa.timestamp("ms"), mask=nulls(0.005)),
        "sp": pa.array(np.array([f"v{j:02d}" for j in range(60)], object)[rng.integers(0, 60, m)], pa.string(), mask=nulls(0.01)),
        "x": pa.array(rng.integers(-4000, 4000, m) / 8.0, pa.float64(), mask=nulls(0.05)),
        "fn": pa.array(fn, pa.float64(), mask=nulls(0.02)),
        "w": pa.array(w.astype(np.int64)),
    }
    if g < FILE_RGS[0]:
        cols["opt"] = pa.array(rng.integers(0, 10, m), pa.int64(), mask=nulls(0.1))
    return pa.table(cols)


def _write(path, tables, use_dictionary):
    kw = dict(use_dictionary=use_dictionary, column_encoding={"ts": "DELTA_BINARY_PACKED"}, data_page_size=8192,
              dictionary_pagesize_limit=1 << 20, compression="snappy")
    with pq.ParquetWriter(path, tables[0].schema, **kw) as wr:
        for t in tables:
            wr.write_table(t, row_group_size=t.num_rows)


@pytest.fixture(scope="module")
def data(tmp_path_factory):
    d = tmp_path_factory.mktemp("ranks_hashed")
    rng = np.random.default_rng(SEED)
    rgs, r0 = [], 0
    for g, m in enumerate(RG_ROWS):
        rgs.append(_rg_table(g, r0, m, rng))
        r0 += m
    a, b = str(d / "a.parquet"), str(d / "b.parquet")
    _write(a, rgs[:FILE_RGS[0]], ["u", "i", "f", "sp", "x", "fn", "opt"])
    _write(b, rgs[FILE_RGS[0]:], ["u", "f", "sp", "x", "fn"])          # `i` has PLAIN pages in this file
    return {"dir": str(d), "files": [a, b], "table": pa.concat_tables(rgs, promote_options="default"), "rgs": rgs}


def _card(tables, col):
    return len({v for t in tables for v in t[col].to_pylist() if v is not None})


def test_data_layout(data):
    """The key spaces the cases rely on: (u, i) wider than 2^26 in the agreed numbering and narrower on every rank alone
    at n >= 2; `i` with a dictionary in the first file only; `opt` in the first file only."""
    rgs = data["rgs"]
    assert (_card(rgs, "u") + 1) * (_card(rgs, "i") + 1) > 1 << 26
    for n in NRANKS[1:]:
        for r in range(n):
            mine = [t for g, t in enumerate(rgs) if g % n == r]
            if mine:
                assert (_card(mine, "u") + 1) * (_card(mine, "i") + 1) <= 1 << 26, (n, r)
    assert (_card(rgs, "u") + 1) * (_card(rgs, "f") + 1) > 1 << 26
    g = 0
    for path in data["files"]:
        md = pq.ParquetFile(path).metadata
        for r in range(md.num_row_groups):
            cc = {md.row_group(r).column(c).path_in_schema: md.row_group(r).column(c) for c in range(md.num_columns)}
            assert ("RLE_DICTIONARY" in cc["i"].encodings) == (g < FILE_RGS[0]), (g, cc["i"].encodings)
            assert ("opt" in cc) == (g < FILE_RGS[0])
            assert "RLE_DICTIONARY" in cc["u"].encodings
            g += 1
    assert g == len(RG_ROWS)


# ---- runs ------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def runs(data, built):
    """The rank counts one after another, each in its own exchange directory, with PQB_VERBOSE on and each rank's stderr
    in <out>/log.<rank>; the workers are always reaped."""
    R._ensure_hostcomm()
    started, res = [], {}
    try:
        for n in NRANKS:
            out = os.path.join(data["dir"], f"out{n}")
            comm = os.path.join(data["dir"], f"comm{n}")
            os.makedirs(out, exist_ok=True)
            os.makedirs(comm, exist_ok=True)
            spec = os.path.join(out, "spec.json")
            with open(spec, "w") as f:
                json.dump({"files": data["files"], "out": out, "idfile": os.path.join(comm, "id")}, f)
            env = {**os.environ, "PQB_LIB": R.HOSTCOMM, "PQB_COMM_DIR": comm, "PQB_COMM_TIMEOUT_MS": str(TIMEOUT_MS), "PQB_VERBOSE": "1"}
            for var, _ in HW.REFUSALS.values():
                env.pop(var, None)
            logs = [open(os.path.join(out, f"log.{r}"), "w") for r in range(n)]
            procs = [subprocess.Popen([sys.executable, os.path.join(ROOT, "tests", "scripts", "ranks_hashed_worker.py"), str(r), str(n), spec],
                                      stdout=subprocess.PIPE, stderr=logs[r], text=True, env=env) for r in range(n)]
            started.append(procs)
            outs = [p.communicate(timeout=900)[0] for p in procs]
            for f in logs:
                f.close()
            for r, (p, o) in enumerate(zip(procs, outs)):
                assert p.returncode == 0, f"n={n} rank {r}:\n{o[-3000:]}\n{open(os.path.join(out, f'log.{r}')).read()[-3000:]}"
            shutil.rmtree(comm)
            res[n] = out
        return res
    finally:
        for procs in started:
            for p in procs:
                if p.poll() is None:
                    p.kill()
                p.wait()


def _sections(out, rank):
    """stderr of one rank, split at the worker's "== <case>.<source>" lines."""
    sec, cur = {}, None
    for line in open(os.path.join(out, f"log.{rank}")):
        if line.startswith("== "):
            cur = line[3:].strip()
            sec[cur] = []
        elif cur:
            sec[cur].append(line)
    return {k: "".join(v) for k, v in sec.items()}


@pytest.fixture(scope="module")
def refs():
    return {}


def _want(data, refs, name):
    if name not in refs:
        keys, aggs, flt, _ = HW.CASES[name]
        refs[name] = R.reference(data["table"], keys, aggs, flt)
    return refs[name]


def _results(out, n, name, src, fns):
    return R._case_results(out, n, name, src, fns)


@pytest.mark.gpu
@pytest.mark.parametrize("n", NRANKS)
def test_hashed_allreduce_cases(runs, data, refs, n):
    """(a), (b) and (c) for every case, on a resident table and on a file list."""
    out = runs[n]
    secs = [_sections(out, r) for r in range(n)]
    for src in R.SOURCES:
        for name, (keys, aggs, flt, kw) in HW.CASES.items():
            what = f"n={n} {src} {name}"
            fns = R._fns(keys, aggs) + (["rn"] if "window" in kw else [])
            _, rows = _results(out, n, name, src, fns)
            for r in range(n):   # the hashed table on every rank that scanned, and its merge on every rank
                s = secs[r][f"{name}.{src}"]
                for m in re.finditer(r"k_flat_agg<([^>]*)>", s):
                    assert ",hashed" in m.group(1), (what, r, m.group(0))
                mg = re.search(r"hashed merge: E_r (\d+), E_max (\d+), listed by all ranks (\d+), G (\d+)", s)
                assert mg, (what, r, "no merge line")
                assert int(mg.group(4)) == len(rows) or kw.get("order_by") or kw.get("json"), (what, mg.group(0), len(rows))
            if name in HW.AGAIN:
                # the same rows in the same order on every rank (checked by _results) and, on the resident table, whose key
                # numbering is kept, on every run.  A file list numbers its keys anew at every open.
                _, again = _results(out, n, "again_" + name, src, fns)
                if src == "table":
                    assert again == rows, (what, "a second run differs")
            want = _want(data, refs, name)
            nk = len(keys)
            if "json" in kw:
                recs = [json.loads(x) for x in rows[0].splitlines() if x]
                got = {tuple(r.get(k) for k in keys): tuple(R._canon_value(r.get(a.name), a.fn) for a in aggs) for r in recs}
                assert len(got) == len(recs) and got == want, what
            elif "window" in kw:
                # ROW_NUMBER() OVER (PARTITION BY b ORDER BY count(*) DESC, u, i), rn <= 3
                parts = {}
                for k, v in want.items():
                    parts.setdefault(k[0], []).append((k, v))
                exp = []
                for b in sorted(parts, key=R._sort_key):
                    top = sorted(parts[b], key=lambda kv: (-kv[1][0], R._sort_key(kv[0][1]), R._sort_key(kv[0][2])))[:3]
                    exp += [k + v + (i + 1,) for i, (k, v) in enumerate(top)]
                assert sorted(rows, key=repr) == sorted(exp, key=repr), what
                for b in parts:   # within a partition, in rank order
                    assert [r[-1] for r in rows if r[0] == b] == list(range(1, len([r for r in rows if r[0] == b]) + 1)), what
            elif name == "order_limit":
                order = sorted(want.items(), key=lambda kv: (-kv[1][0], R._sort_key(kv[0][0]), R._sort_key(kv[0][1])))[: kw["limit"]]
                assert rows == [k + v for k, v in order], what
            elif name == "order_ties":
                # count(*) DESC only: ties broken alike on every rank and every run (checked above); the counts are the top
                # ones and every row is a whole-table group
                top = sorted((v[0] for v in want.values()), reverse=True)[: kw["limit"]]
                assert [r[nk] for r in rows] == top, what
                assert len({r[:nk] for r in rows}) == len(rows), what
                for r in rows:
                    assert want[r[:nk]] == r[nk:], (what, r)
            else:
                R.check_groups(rows, want, nk, what)


@pytest.mark.gpu
@pytest.mark.parametrize("n", NRANKS[1:])
def test_dense_on_each_rank_alone(runs, n):
    """GROUP BY u, i without PQ_QUERY_ALLREDUCE: the dense table on every rank that scans (the same query under the flag
    is hashed, test_hashed_allreduce_cases)."""
    for r in range(n):
        for src in R.SOURCES:
            s = _sections(runs[n], r)[f"local_fp_u_i.{src}"]
            lines = re.findall(r"k_flat_agg<([^>]*)>", s)
            if any(g % n == r for g in range(len(RG_ROWS))):
                assert lines, (n, r, src)
            assert all(",hashed" not in x for x in lines), (n, r, src, lines)


@pytest.mark.gpu
@pytest.mark.parametrize("n", NRANKS)
def test_hashed_refusals_are_collective(runs, data, refs, n):
    """One rank's table runs full (PQB_HASH_SLOTS), or its merge budget is too small (PQB_MERGE_BUDGET): every rank
    returns the same code naming that rank, well within the timeout, and the next query is answered."""
    want_code = {"refuse_full": -2, "refuse_budget": -6}   # PQ_ERR_UNSUPPORTED, PQ_ERR_OOM
    text = {"refuse_full": "hashed accumulator table", "refuse_budget": "budget"}
    v = HW.victim(n)
    keys, aggs, _, _ = HW.CASES["fp_u_i"]
    for name in HW.REFUSALS:
        for src in R.SOURCES:
            for r in range(n):
                e = R.load(runs[n], name, src, r)
                what = f"n={n} {src} {name} rank {r}"
                assert isinstance(e, dict), (what, "answered")
                assert e["code"] == want_code[name], (what, e)
                assert text[name] in e["message"] and f"rank {v}" in e["message"], (what, e)
                assert e["seconds"] < TIMEOUT_MS / 4000, (what, e["seconds"])
            _, rows = _results(runs[n], n, "after_" + name, src, R._fns(keys, aggs))
            R.check_groups(rows, _want(data, refs, "fp_u_i"), len(keys), f"n={n} {src} after {name}")
