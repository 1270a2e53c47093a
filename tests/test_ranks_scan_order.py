"""ORDER BY ... LIMIT scans under PQ_QUERY_ALLGATHER on ONE device: 1, 2, 3 and 8 ranks as processes over the
host-staged communicator build (tools/comm_host.cpp).  Every rank's first rows are gathered, ordered alike on every rank
and projected by the rank that holds each (order_kernels.cuh, ScanMerge in query.cu).  Each case runs on a resident
table and on a file list, and is checked three ways:

(a) every rank's result and rows_selected are identical to rank 0's, Float64 by bit pattern, rows in the same order;
(b) they equal the same query without sharding and without the flag (one rank over all files, run by the worker);
(c) the __row_id sequence equals the C oracle's selected row ids, stably sorted on their pyarrow values and cut.

The data is test_ranks_one_gpu.py's: 7 row groups in two files (one rank owns nothing at n = 8), `sp` PLAIN in one row
group, an all-NULL `s` row group, `opt` absent from the second file, +-0.0, +-inf and NaN payloads in `f`, DELTA `ts`;
here also a Utf8 `sopt` in the first file only and a Utf8 `ghost` in no file.  A merge budget too small on one rank, one
rank whose items have no flat-store copies (found before the scan), a table not sharded by row group over the
communicator and ranks with lists of different sizes are refused by every rank, well within the communicator's timeout,
and the next query is answered."""
import json
import os
import shutil
import subprocess
import sys

import numpy as np
import pyarrow as pa
import pytest

import test_ranks_one_gpu as R
from test_order_by import canon, host_order
from test_order_rows import _sortable

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests", "scripts"))
import ranks_scan_worker as SW  # noqa: E402
import ranks_worker as W  # noqa: E402

NRANKS = (1, 2, 3, 8)
TIMEOUT_MS = R.TIMEOUT_MS
SEED = 20261018


@pytest.fixture(scope="module")
def data(tmp_path_factory):
    d = tmp_path_factory.mktemp("ranks_scan")
    rng = np.random.default_rng(SEED)
    rgs, r0 = [], 0
    for g, m in enumerate(R.RG_ROWS):
        t = R._rg_table(g, r0, m, rng)
        if g < R.FILE_RGS[0]:   # `sopt`: a Utf8 column of the first file only
            sopt = np.array([f"o{k:03d}" for k in range(300)], object)[rng.integers(0, 300, m)]
            t = t.append_column("sopt", pa.array(sopt, pa.string(), mask=rng.random(m) < 0.05))
        rgs.append(t)
        r0 += m
    a, b = str(d / "a.parquet"), str(d / "b.parquet")
    R._write(a, rgs[:R.FILE_RGS[0]], ["s", "sp", "i", "f", "x", "opt", "sopt"])
    R._write(b, rgs[R.FILE_RGS[0]:], ["s", "sp", "f", "x"])
    table = pa.concat_tables(rgs, promote_options="default")
    table = table.append_column("ghost", pa.nulls(table.num_rows, pa.string()))   # in no file (the worker's schema adds it)
    return {"dir": str(d), "files": [a, b], "table": table}


def test_flag_matches_header():
    """The Python mirror of PQ_QUERY_ALLGATHER is the header's value, a bit no other query flag uses."""
    import re
    from parseable_b200 import _lib as L
    hdr = open(os.path.join(ROOT, "include", "parseable_b200.h")).read()
    flags = {m.group(1): int(m.group(2)) for m in re.finditer(r"#define (PQ_QUERY_\w+) (\d+)u", hdr)}
    assert flags["PQ_QUERY_ALLGATHER"] == L.PQ_QUERY_ALLGATHER == 8
    assert sum(flags.values()) == 1 | 2 | 4 | 8 and all(getattr(L, k) == v for k, v in flags.items())


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
            for var, _ in SW.REFUSALS.values():
                env.pop(var, None)
            logs = [open(os.path.join(out, f"log.{r}"), "w") for r in range(n)]
            procs = [subprocess.Popen([sys.executable, os.path.join(ROOT, "tests", "scripts", "ranks_scan_worker.py"), str(r), str(n), spec],
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


def _meta(out, name, src, rank):
    return json.load(open(os.path.join(out, f"{name}.{src}.{rank}.meta.json")))


def _rows(t):
    return t["json"].to_pylist() if "json" in t.column_names else canon(t)


@pytest.fixture(scope="module")
def oracle_ids(data):
    """Per case: the C oracle's selected row ids, stably sorted on their pyarrow values and cut, and the selected total."""
    from oracle.oracle import Oracle
    ora = Oracle(data["table"])
    memo = {}

    def get(name):
        if name not in memo:
            case = SW.CASES[name]
            ids = np.asarray(ora.row_ids(W.filters_of(case.get("filters", []))), np.int64)
            terms = [(c, d == "desc", (d == "desc") if len(o) < 3 else o[2]) for o in case["order_by"] for c, d in [o[:2]]]
            want = []
            if len(ids) and case["limit"]:
                vals = _sortable(data["table"].take(pa.array(ids)).select(list(dict.fromkeys(t[0] for t in terms))))
                want = ids[np.array(host_order(vals, terms)[: case["limit"]], np.int64)].tolist()
            memo[name] = (want, len(ids))
        return memo[name]
    return get


def _check_case(out, n, name, src, what):
    """(a): every rank's result and rows_selected are rank 0's; returns rank 0's table, rows and rows_selected."""
    got = [R.load(out, name, src, r) for r in range(n)]
    for r in range(n):
        assert not isinstance(got[r], dict), (what, f"rank {r} refused", got[r])
    rows0 = _rows(got[0])
    sel = [_meta(out, name, src, r)["rows_selected"] for r in range(n)]
    for r in range(1, n):
        assert got[r].schema == got[0].schema, (what, r)
        assert _rows(got[r]) == rows0, (what, f"rank {r} differs from rank 0")
        assert sel[r] == sel[0], (what, r, sel)
    return got[0], rows0, sel[0]


@pytest.mark.gpu
@pytest.mark.parametrize("n", NRANKS)
def test_scan_merge_cases(runs, data, oracle_ids, n):
    """(a), (b) and (c) for every case, on a resident table and on a file list; the merge line on every rank (n >= 2)."""
    out = runs[n]
    secs = [_sections(out, r) for r in range(n)]
    for src in R.SOURCES:
        for name, case in SW.CASES.items():
            what = f"n={n} {src} {name}"
            if SW.REFUSED_AT.get(name) == (n, src):
                _check_refused(out, n, name, src, -2, "flat-store copy", FILE_B_ONLY_RANKS, what)
                continue
            t0, rows0, sel = _check_case(out, n, name, src, what)
            ref = R.load(out, name, "ref", 0)
            assert t0.schema == ref.schema, what
            assert rows0 == _rows(ref), (what, "differs from one rank over the unsharded table")   # (b)
            want_ids, want_sel = oracle_ids(name)
            assert sel == want_sel, (what, sel, want_sel)
            if "json" in case:
                recs = [json.loads(x) for x in rows0[0].splitlines() if x]
                assert len(recs) == len(want_ids), what
            else:   # (c)
                rid = "__row_id" if "__row_id" in t0.column_names else "rid"   # `rid` holds every row's global ordinal
                ids = t0[rid].to_pylist() if t0.num_rows else []
                assert ids == want_ids, (what, "__row_id order", ids[:5], want_ids[:5])
            for r in range(n):   # the merge ran on every rank, and its sizes agree
                line = [x for x in secs[r][f"{name}.{src}"].splitlines() if "scan merge: keep_r" in x]
                assert len(line) == (1 if n > 1 else 0), (what, r, line)
                if line:
                    assert f"kept {min(case['limit'], want_sel)}," in line[0], (what, r, line[0])


# at n = 8 the ranks whose row groups all lie in the second file
FILE_B_ONLY_RANKS = {g % 8 for g in range(R.FILE_RGS[0], len(R.RG_ROWS))}


def _check_refused(out, n, name, src, code, own, cause, what):
    """Every rank refuses with `code`, well within the timeout: the ranks in `cause` with their own message `own`, the
    others naming the lowest of them."""
    for r in range(n):
        e = R.load(out, name, src, r)
        assert isinstance(e, dict), (what, r, "answered")
        assert e["code"] == code, (what, r, e)
        assert e["seconds"] < TIMEOUT_MS / 4000, (what, r, e["seconds"])
        if r in cause:
            assert own in e["message"], (what, r, e)
        else:
            assert f"refused on rank {min(cause)}" in e["message"], (what, r, e)


@pytest.mark.gpu
@pytest.mark.parametrize("n", NRANKS[1:])
def test_scan_merge_needs_one_row_group_sharded_list(runs, n):
    """__row_id is global only when every rank opens the same file list and scans its row groups g % n == rank: an
    unsharded provider, and rank 0 opening a shorter list, are refused by every rank; the next query is answered."""
    _check_refused(runs[n], n, "refuse_unsharded", "files", -2, "sharded by row group", set(range(n)), f"n={n} unsharded")
    for r in range(n):
        e = R.load(runs[n], "refuse_lists", "files", r)
        assert isinstance(e, dict) and e["code"] == -2 and "file lists of different sizes" in e["message"], (n, r, e)
        assert e["seconds"] < TIMEOUT_MS / 4000, (n, r, e["seconds"])
    _, rows, _ = _check_case(runs[n], n, "after_refuse_lists", "files", f"n={n} after refuse_lists")
    assert rows == _rows(R.load(runs[n], "log_search", "ref", 0)), n


@pytest.mark.gpu
@pytest.mark.parametrize("n", NRANKS[1:])
def test_scan_merge_refusals_are_collective(runs, n):
    """One rank's merge budget is too small (PQ_ERR_OOM), or its items have no flat-store copy (PQ_ERR_UNSUPPORTED before
    the scan): every rank returns the same code naming that rank, well within the timeout, and the next query is
    answered."""
    want_code = {"refuse_budget": -6, "refuse_flat": -2}   # PQ_ERR_OOM, PQ_ERR_UNSUPPORTED
    v = SW.victim(n)
    for name in SW.REFUSALS:
        for src in R.SOURCES:
            for r in range(n):
                e = R.load(runs[n], name, src, r)
                what = f"n={n} {src} {name} rank {r}"
                assert isinstance(e, dict), (what, "answered")
                assert e["code"] == want_code[name], (what, e)
                if name == "refuse_flat" and r == v:
                    assert "flat-store copy" in e["message"], (what, e)
                else:
                    assert f"rank {v}" in e["message"], (what, e)
                assert e["seconds"] < TIMEOUT_MS / 4000, (what, e["seconds"])
            _, rows, _ = _check_case(runs[n], n, "after_" + name, src, f"n={n} {src} after {name}")
            assert rows == _rows(R.load(runs[n], "log_search", "ref", 0)), (n, src, name)


@pytest.mark.gpu
@pytest.mark.parametrize("n", NRANKS)
def test_scan_merge_agreement_cache(runs, n):
    """The agreed Utf8 numbering kept with the resident table: the same queries again, and after rank 1 alone reopens its
    table, give the unsharded answer on every rank.  A repeat reuses the agreement (no rank agrees anew); after the reopen
    every rank agrees anew (the PQB_VERBOSE line)."""
    secs = [_sections(runs[n], r) for r in range(n)]
    for step in ("again", "reopen"):
        for name in SW.AGAIN:
            _, rows, _ = _check_case(runs[n], n, f"{step}_{name}", "table", f"n={n} {step} {name}")
            assert rows == _rows(R.load(runs[n], name, "ref", 0)), (n, step, name)
            for r in range(n):
                agreed = "the ranks agree on a numbering" in secs[r][f"{step}_{name}.table"]
                assert agreed == (step == "reopen" and n > 1), (n, step, name, r)


@pytest.mark.gpu
@pytest.mark.parametrize("n", NRANKS)
def test_scan_merge_misuse(runs, n):
    """The flag on an aggregate, with COUNT_ONLY, with a window, without ORDER BY, and without a communicator."""
    L_INVALID, L_UNSUPPORTED = -1, -2
    want = {"aggregate": L_INVALID, "count_only": L_INVALID, "window": L_UNSUPPORTED, "no_order_by": L_UNSUPPORTED}
    for r in range(n):
        got = json.load(open(os.path.join(runs[n], f"misuse.{r}.json")))
        assert {k: v and v[0] for k, v in got.items()} == want, (n, r, got)
    got = json.load(open(os.path.join(runs[n], "misuse_nocomm.0.json")))
    assert got["no_comm"][0] == L_INVALID and "pq_comm_init_rank" in got["no_comm"][1], got
