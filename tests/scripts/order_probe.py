"""Development probe (GPU box): ORDER BY [LIMIT] on the device against the same query without ORDER BY plus the sort on
the host, over a resident logs16 table.  Reports order_ms (CUDA events of the ordering kernels) and the whole-query p50
of both forms for
  (a) C4's keys: GROUP BY host, status -> COUNT(*) ORDER BY count(*) DESC LIMIT 10
  (b) the same groups fully ordered by SUM(bytes)
  (c) field statistics of `pod` and `message` (ORDER BY count(*) DESC LIMIT 50)
  (d) a hashed GROUP BY host, pod, status -> COUNT(*) ORDER BY count(*) DESC LIMIT 100.
Queries with a LIMIT run once per path (the planner's choice, then PQB_ORDER_PATH=topk and =sort).
Every device result is first checked against the host-sorted one.  Not a bench line: bench.py is the contract.

    python tests/scripts/order_probe.py [row_groups=96] [steps=20]
"""
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

COLS = ["p_timestamp", "host", "status", "bytes", "pod", "message"]
DIR = os.environ.get("PQB_PROBE_DIR", "/tmp/pqb_order_probe")
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
    import subprocess

    import pyarrow as pa
    from parseable_b200.query import DeviceTable, StandardTableProvider, count_star, sum_
    from test_order_by import canon, host_order
    files = ensure(nrg)
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    print("gpu:", smi, flush=True)
    schema = {"p_timestamp": pa.timestamp("ms"), "host": pa.string(), "status": pa.int64(), "bytes": pa.int64(), "pod": pa.string(),
              "message": pa.string()}
    table = DeviceTable(files, COLS)
    print(f"table: {table.rows} rows", flush=True)
    prov = StandardTableProvider(table, schema=schema)
    cs = count_star()
    q = {
        "(a) host,status count(*) DESC LIMIT 10": (["host", "status"], [cs, sum_("bytes")], [(cs, "desc")], 10),
        "(b) host,status ORDER BY sum(bytes)": (["host", "status"], [cs, sum_("bytes")], [(sum_("bytes"), "asc")], None),
        "(c) field stats pod": (["pod"], [cs], [(cs, "desc")], 50),
        "(c) field stats message": (["message"], [cs], [(cs, "desc")], 50),
        "(d) hashed host,pod,status LIMIT 100": (["host", "pod", "status"], [cs], [(cs, "desc")], 100),
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

    for name, (keys, aggs, order, limit) in q.items():
        terms = [(a.name if hasattr(a, "fn") else a, d == "desc", d == "desc") for a, d in order]

        def host_form():
            r = prov.aggregate(keys, aggs)
            t = r.table()
            idx = host_order(t, terms)
            return t.take(pa.array(idx[:limit] if limit is not None else idx, pa.int64())), r

        want, base = host_form()
        for path in (("", "topk", "sort") if limit is not None else ("",)):   # "": the planner's choice
            if path:
                os.environ["PQB_ORDER_PATH"] = path
            dev = lambda: prov.aggregate(keys, aggs, order_by=order, limit=limit)
            got = dev().table()
            assert canon(got) == canon(want), name
            ms_dev, r = p50(dev)
            m = r.metrics
            print(f"{name}{' [' + path + ']' if path else ''}: groups {m['groups_total']} -> {m['groups']} | order_ms {m['order_ms']:.3f} "
                  f"| device p50 {ms_dev:.3f} ms, launches {m['kernel_launches']} (unordered {base.metrics['kernel_launches']})", flush=True)
            os.environ.pop("PQB_ORDER_PATH", None)
        ms_host, _ = p50(lambda: host_form()[1])
        ms_plain, _ = p50(lambda: prov.aggregate(keys, aggs))
        print(f"    unordered query p50 {ms_plain:.3f} ms; unordered + host sort p50 {ms_host:.3f} ms", flush=True)
    table.close()


if __name__ == "__main__":
    main()
