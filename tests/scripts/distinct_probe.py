"""Development probe (GPU box): COUNT(DISTINCT) on the synthetic logs16 files -- oracle parity on the first file,
then timing over a resident table of (a) the alert form, (b) distinct hosts per status, (c) COUNT(DISTINCT) next to
COUNT / SUM, and (d) what (a) and (b) cost through the old composition (GROUP BY [status,] host -> COUNT(*), counted
on the host).  Not a bench line: bench.py is the contract.

    python tests/scripts/distinct_probe.py [row_groups=96] [steps=20]
"""
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

COLS = ["p_timestamp", "level", "host", "bytes", "status", "path"]
DIR = os.environ.get("PQB_PROBE_DIR", "/tmp/pqb_distinct_probe")
RGS_PER_FILE = 8


def _gen(args):
    path, first, n = args
    from parseable_b200 import synth
    if not os.path.exists(path):
        synth.write_logs16(path, n_row_groups=n, first_rg=first, columns=COLS)
    return path


def ensure(nrg):
    import multiprocessing as mp
    os.makedirs(DIR, exist_ok=True)
    jobs, g = [], 0
    while g < nrg:
        n = min(RGS_PER_FILE, nrg - g)
        jobs.append((os.path.join(DIR, f"probe_{g:05d}_{n}.parquet"), g, n))
        g += n
    missing = [j for j in jobs if not os.path.exists(j[0])]
    if missing:
        t = time.time()
        with mp.get_context("spawn").Pool(max(1, min(len(missing), (os.cpu_count() or 2) - 1, 64))) as pool:
            pool.map(_gen, missing, chunksize=1)
        print(f"generated {len(missing)} files in {time.time() - t:.1f}s", flush=True)
    return [j[0] for j in jobs]


def main():
    nrg = int(sys.argv[1]) if len(sys.argv) > 1 else 96
    steps = int(sys.argv[2]) if len(sys.argv) > 2 else 20
    import pyarrow as pa
    from oracle.oracle import Oracle
    from parseable_b200.query import DeviceTable, StandardTableProvider, col, count_distinct, count_star, sum_
    from test_count_distinct import assert_matches, expect
    files = ensure(nrg)
    schema = {"p_timestamp": pa.timestamp("ms"), "level": pa.string(), "host": pa.string(), "bytes": pa.int64(),
              "status": pa.int64(), "path": pa.string()}
    err = [col("level") == "ERROR"]
    q = {
        "(a) COUNT(DISTINCT host) WHERE level='ERROR'": ([], [count_distinct("host")], err),
        "(b) status, COUNT(DISTINCT host) GROUP BY status": (["status"], [count_distinct("host")], []),
        "(c) host, COUNT(*), SUM(bytes), COUNT(DISTINCT path) GROUP BY host": (["host"], [count_star(), sum_("bytes"), count_distinct("path")], []),
    }
    # ---- parity on the first file, both presence forms ----
    ora = Oracle.from_parquet(files[0], columns=COLS)
    p1 = StandardTableProvider([files[0]], schema=schema)
    for name, (keys, aggs, flt) in q.items():
        exp = expect(ora, keys, aggs, flt)
        assert_matches(p1.aggregate(keys, aggs, flt).table(), exp, keys, aggs)
        os.environ["PQB_DISTINCT_HASH"] = "1"
        assert_matches(p1.aggregate(keys, aggs, flt).table(), exp, keys, aggs)
        del os.environ["PQB_DISTINCT_HASH"]
        print("parity ok:", name, flush=True)
    # ---- timing, table resident ----
    t0 = time.perf_counter()
    table = DeviceTable(files, COLS)
    print(f"table open: {1e3 * (time.perf_counter() - t0):.1f} ms, {table.rows} rows", flush=True)
    prov = StandardTableProvider(table, schema=schema)

    def run(name, fn):
        for _ in range(3):
            r = fn()
        ms = []
        for _ in range(steps):
            t = time.perf_counter()
            r = fn()
            ms.append(1e3 * (time.perf_counter() - t))
        ms.sort()
        m = r.metrics
        print(f"{name}: p50 {ms[len(ms) // 2]:.3f} ms = {table.rows / ms[len(ms) // 2] / 1e6:.1f} G rows/s | scan {m['scan_kernel_ms']:.3f} ms "
              f"device {m['device_ms']:.3f} host {m['host_ms']:.3f} | groups {m['groups']} launches {m['kernel_launches']}", flush=True)
        return r

    class Composed:   # the old mirror: (keys x host) groups to the host, counted there
        def __init__(self, keys, flt):
            self.keys, self.flt = keys, flt

        def __call__(self):
            r = prov.aggregate(self.keys + ["host"], [count_star()], self.flt)
            t = r.table()
            seen = {}
            kc = [t[k].to_pylist() for k in self.keys]
            for i, h in enumerate(t["host"].to_pylist()):
                key = tuple(c[i] for c in kc)
                seen[key] = seen.get(key, 0) + (h is not None)
            return r

    for name, (keys, aggs, flt) in q.items():
        run(name, lambda: prov.aggregate(keys, aggs, flt))
        if name.startswith("(a)") or name.startswith("(b)"):
            os.environ["PQB_DISTINCT_HASH"] = "1"
            run(name + " [pair set]", lambda: prov.aggregate(keys, aggs, flt))
            del os.environ["PQB_DISTINCT_HASH"]
    run("(d) (a) composed: GROUP BY host -> COUNT(*), counted on the host", Composed([], err))
    run("(d) (b) composed: GROUP BY status, host -> COUNT(*), counted on the host", Composed(["status"], []))
    table.close()


if __name__ == "__main__":
    main()
