"""Development probe (GPU box): ORDER BY ... LIMIT on filter / projection scans, ordered and cut on the device, against
the same scan without ORDER BY plus a pyarrow sort_indices on the host, over resident logs16 tables:
  (a) SELECT * ... WHERE message LIKE '%timeout-xyzzy%' ORDER BY p_timestamp DESC LIMIT 100   (C5's 0.1 % selection)
  (b) SELECT p_timestamp, host, level, message ... ORDER BY p_timestamp DESC LIMIT 1000       (no filter, one bench file)
  (c) SELECT p_timestamp, host, latency_ms ... ORDER BY latency_ms DESC LIMIT 10               (no filter)
  (d) SELECT p_timestamp, host, message ... WHERE level = 'ERROR' ORDER BY host, p_timestamp DESC LIMIT 100
      (a Utf8 term: its first query on a table also builds the column's ids and bytewise ranks, reported on their own)
(a), (c), (d) run over `row_groups` row groups; (b) over the first 16 (one bench file: the unordered form projects
every row's message, which must fit one result).  Every device result is first checked against the host-sorted one.
Reports order_ms (CUDA events of the ordering kernels), the query p50 and the unordered scan + host sort p50.  Not a
bench line: bench.py is the contract.

    python tests/scripts/row_order_probe.py [row_groups=96] [steps=20]
"""
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

COLS = ["p_timestamp", "host", "level", "message", "latency_ms", "status"]
DIR = os.environ.get("PQB_PROBE_DIR", "/tmp/pqb_row_order_probe")
RGS_PER_FILE = 8
SHARD_RGS = 16


def _gen(args):
    path, first, n = args
    from parseable_b200 import synth
    if not os.path.exists(path):
        synth.write_logs16(path, n_row_groups=n, first_rg=first, columns=COLS)
    return path


def ensure(nrg):
    import multiprocessing as mp
    os.makedirs(DIR, exist_ok=True)
    jobs = [(os.path.join(DIR, f"probe_{g:05d}.parquet"), g, min(RGS_PER_FILE, nrg - g)) for g in range(0, nrg, RGS_PER_FILE)]
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
    import pyarrow.compute as pc
    from parseable_b200 import synth
    from parseable_b200.query import DeviceTable, StandardTableProvider, col
    from test_order_by import canon
    files = ensure(max(nrg, SHARD_RGS))
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    print("gpu:", smi, flush=True)
    schema = {"p_timestamp": pa.timestamp("ms"), "host": pa.string(), "level": pa.string(), "message": pa.string(),
              "latency_ms": pa.int64(), "status": pa.int64()}
    big = DeviceTable(files[: (nrg + RGS_PER_FILE - 1) // RGS_PER_FILE], COLS)
    shard = DeviceTable(files[: SHARD_RGS // RGS_PER_FILE], COLS)
    print(f"tables: {big.rows} rows, bench file {shard.rows} rows", flush=True)
    provs = {"big": StandardTableProvider(big, schema=schema), "shard": StandardTableProvider(shard, schema=schema)}
    q = {
        "(a) SELECT * LIKE 0.1% ORDER BY p_timestamp DESC LIMIT 100":
            ("big", COLS, [col("message").like(f"%{synth.TOKEN}%")], [("p_timestamp", "desc")], 100),
        "(b) ts,host,level,message ORDER BY p_timestamp DESC LIMIT 1000":
            ("shard", ["p_timestamp", "host", "level", "message"], [], [("p_timestamp", "desc")], 1000),
        "(c) ORDER BY latency_ms DESC LIMIT 10":
            ("big", ["p_timestamp", "host", "latency_ms"], [], [("latency_ms", "desc")], 10),
        "(d) level='ERROR' ORDER BY host, p_timestamp DESC LIMIT 100":
            ("big", ["p_timestamp", "host", "message"], [col("level") == "ERROR"], [("host", "asc"), ("p_timestamp", "desc")], 100),
    }

    def p50(fn):
        for _ in range(3):
            r = fn()
        ms = []
        for _ in range(steps):
            t = time.perf_counter()
            r = fn()
            ms.append(1e3 * (time.perf_counter() - t))
        ms.sort()
        return ms[len(ms) // 2], r

    for name, (which, proj, flt, order, limit) in q.items():
        prov = provs[which]
        need = proj + [c for c, _ in order if c not in proj]
        keys = [(c, "descending" if d == "desc" else "ascending") for c, d in order]

        def host_form():
            r = prov.scan(need, flt)
            t = r.table()
            idx = pc.sort_indices(t, sort_keys=keys, null_placement="at_end")   # stable; these columns hold no NULLs
            return t.take(idx[:limit]).select(proj), r

        dev = lambda: prov.scan(proj, flt, limit, order_by=order)
        want, base = host_form()   # first: the column set's work items exist before the first ordered query is timed
        t0 = time.perf_counter()
        dev()
        first_ms = 1e3 * (time.perf_counter() - t0)
        for path in ("", "topk", "sort"):   # "": the planner's choice
            if path:
                os.environ["PQB_ORDER_PATH"] = path
            got = dev().table()
            assert canon(got) == canon(want), (name, path)
            ms_dev, r = p50(dev)
            m = r.metrics
            print(f"{name}{' [' + path + ']' if path else ''}: selected {m['rows_selected']} -> {got.num_rows} | order_ms {m['order_ms']:.3f} "
                  f"| query p50 {ms_dev:.3f} ms (device {m['device_ms']:.3f}), launches {m['kernel_launches']} "
                  f"(unordered {base.metrics['kernel_launches']})", flush=True)
            os.environ.pop("PQB_ORDER_PATH", None)
        ms_host, _ = p50(lambda: host_form()[1])
        ms_scan, _ = p50(lambda: prov.scan(need, flt))
        print(f"    first ordered query {first_ms:.3f} ms (a Utf8 term's first: + its ids and ranks) | unordered scan p50 "
              f"{ms_scan:.3f} ms; unordered scan + host sort_indices p50 {ms_host:.3f} ms", flush=True)
    big.close()
    shard.close()


if __name__ == "__main__":
    main()
