"""Date32 across ranks on ONE device: 2 and 3 ranks as processes over the host-staged communicator build
(tools/comm_host.cpp, PQB_LIB / PQB_COMM_DIR, as test_ranks_one_gpu.py runs them), each over a resident table and a file
list sharded by row group (tests/scripts/date32_ranks_worker.py).

- GROUP BY d / s / (d, s) with COUNT and MIN / MAX(d) under PQ_QUERY_ALLREDUCE, dense and hashed (the merge of the
  ranks' hashed tables), and the global form: identical on every rank, bit for bit and in row order, and equal to the
  whole table's groups.
- A scan ORDER BY d [DESC] LIMIT n under PQ_QUERY_ALLGATHER: every rank returns the whole table's first n rows (ties in
  global row order), with their Date32 values."""
import json
import os
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
import date32_ranks_worker as DW  # noqa: E402

NRANKS = (2, 3)
RG_ROWS = [8000, 7000, 9000, 6000, 8000]
EXTREMES = [-(2**31 - 1), 2**31 - 1, 0, -1, -719162, 2932897, -800_000]


@pytest.fixture(scope="module")
def data(tmp_path_factory):
    d = tmp_path_factory.mktemp("date32_ranks")
    rng = np.random.default_rng(20261019)
    n = sum(RG_ROWS)
    pool = np.concatenate([rng.integers(-2000, 20_000, 250), EXTREMES]).astype(np.int64)
    days = pool[rng.integers(0, len(pool), n)]
    valid = rng.random(n) > 0.1
    valid[RG_ROWS[0]:RG_ROWS[0] + RG_ROWS[1]] &= rng.random(RG_ROWS[1]) > 0.9   # a mostly-NULL row group
    table = pa.table({"d": pa.array(days.astype(np.int32), pa.int32(), mask=~valid).cast(pa.date32()),
                      "s": pa.array([f"s{int(x)}" for x in rng.integers(0, 9, n)]),
                      "w": pa.array(rng.integers(0, 1 << 40, n)),
                      "i": pa.array(np.arange(n, dtype=np.int64))})
    files, r0 = [], 0
    for name, rgs in (("a", RG_ROWS[:3]), ("b", RG_ROWS[3:])):
        p = str(d / f"{name}.parquet")
        with pq.ParquetWriter(p, table.schema, data_page_size=8192) as wr:
            for k in rgs:
                wr.write_table(table.slice(r0, k), row_group_size=k)
                r0 += k
        files.append(p)
    return {"dir": str(d), "files": files, "days": days, "valid": valid, "table": table}


@pytest.fixture(scope="module")
def runs(data, built):
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
            env = {**os.environ, "PQB_LIB": R.HOSTCOMM, "PQB_COMM_DIR": comm, "PQB_COMM_TIMEOUT_MS": str(R.TIMEOUT_MS),
                   "PQB_VERBOSE": "1"}
            logs = [open(os.path.join(out, f"log.{r}"), "w") for r in range(n)]
            procs = [subprocess.Popen([sys.executable, os.path.join(ROOT, "tests", "scripts", "date32_ranks_worker.py"), str(r), str(n), spec],
                                      stdout=subprocess.PIPE, stderr=logs[r], text=True, env=env) for r in range(n)]
            started.append(procs)
            outs = [p.communicate(timeout=600)[0] for p in procs]
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


def _read(out, name, src, rank):
    base = os.path.join(out, f"{name}.{src}.{rank}")
    if os.path.exists(base + ".json"):
        raise AssertionError(f"{name}.{src} refused on rank {rank}: {open(base + '.json').read()}")
    with pa.memory_map(base + ".arrow") as f:
        return pa.ipc.open_file(f).read_all()


def _days(col):
    assert col.type == pa.date32(), col.type
    return col.cast(pa.int32()).to_pylist()


def _ref(data, keys):
    """{key tuple: (count(*), count(d), min(d), max(d))} over the whole table."""
    days, valid = data["days"], data["valid"]
    t = data["table"]
    cols = {"d": [int(x) if v else None for x, v in zip(days, valid)], "s": t["s"].to_pylist(), "w": t["w"].to_pylist(),
            "i": t["i"].to_pylist()}
    acc = {}
    for k in range(len(days)):
        key = tuple(cols[c][k] for c in keys)
        a = acc.setdefault(key, [0, 0, None, None])
        a[0] += 1
        if valid[k]:
            x = int(days[k])
            a[1] += 1
            a[2] = x if a[2] is None else min(a[2], x)
            a[3] = x if a[3] is None else max(a[3], x)
    return {k: tuple(v) for k, v in acc.items()}


@pytest.mark.gpu
@pytest.mark.parametrize("n", NRANKS)
@pytest.mark.parametrize("src", ["table", "files"])
@pytest.mark.parametrize("name", list(DW.AGGS))
def test_allreduce_groups(runs, data, n, src, name):
    out = runs[n]
    keys, aggs = DW.AGGS[name]
    t0 = _read(out, name, src, 0)
    for r in range(1, n):
        assert _read(out, name, src, r).equals(t0), (name, src, r)   # bit for bit, same row order
    ref = _ref(data, keys)
    kcols = [_days(t0[k]) if k == "d" else t0[k].to_pylist() for k in keys]
    acols = [_days(t0[a.name]) if a.fn in ("min", "max") else t0[a.name].to_pylist() for a in aggs]
    got = {tuple(kc[k] for kc in kcols): tuple(ac[k] for ac in acols) for k in range(t0.num_rows)}
    want = {}
    for key, (cs, cd, mn, mx) in ref.items():
        want[key] = tuple({"count_star": cs, "count": cd, "min": mn, "max": mx}[a.fn] for a in aggs)
    assert got == want, (name, src, n)
    if name == "hashed":
        log = open(os.path.join(out, "log.0")).read()
        assert "hashed merge" in log


def _ref_order(data, desc, limit):
    days, valid = data["days"], data["valid"]
    idx = range(len(days))
    if desc:   # DESC: NULLs first
        order = sorted(idx, key=lambda k: (bool(valid[k]), -int(days[k]) if valid[k] else 0, k))
    else:
        order = sorted(idx, key=lambda k: (not valid[k], int(days[k]) if valid[k] else 0, k))
    return order[:limit]


@pytest.mark.gpu
@pytest.mark.parametrize("n", NRANKS)
@pytest.mark.parametrize("src", ["table", "files"])
@pytest.mark.parametrize("name", list(DW.SCANS))
def test_allgather_order(runs, data, n, src, name):
    out = runs[n]
    kw = DW.SCANS[name]
    t0 = _read(out, name, src, 0)
    for r in range(1, n):
        assert _read(out, name, src, r).equals(t0), (name, src, r)
    want = _ref_order(data, kw["order_by"][0][1] == "desc", kw["limit"])
    assert t0["__row_id"].to_pylist() == want, (name, src, n)
    days, valid = data["days"], data["valid"]
    assert _days(t0["d"]) == [int(days[k]) if valid[k] else None for k in want]
