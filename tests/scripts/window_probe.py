"""Development probe (GPU box): ROW_NUMBER() OVER (PARTITION BY ...) cut to a rank range, ranked on the device.
  (a) top 10 hosts per status by SUM(bytes): GROUP BY host, status (C4's ~50 000 groups) over bench.py's resident files
  (b) latest 3 ERROR rows per service: WHERE level = 'ERROR', partitioned by service, ordered by p_timestamp DESC,
      projecting p_timestamp, host, over `scan_row_groups` logs16 row groups of its own (bench files lack `service`)
Every device result is first checked against the same query without a window, ranked on the host.  Reports order_ms
(CUDA events of the sort and window kernels), the windowed query's p50 and the unwindowed query's p50.  Not a bench
line: bench.py is the contract.

    python tests/scripts/window_probe.py [agg_row_groups=480] [scan_row_groups=480] [steps=10]
"""
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

SCAN_COLS = ["p_timestamp", "level", "service", "host"]
SCAN_DIR = os.environ.get("PQB_PROBE_DIR", "/tmp/pqb_window_probe")
RGS_PER_FILE = 16


def _gen(args):
    path, first, n = args
    from parseable_b200 import synth
    if not os.path.exists(path):
        synth.write_logs16(path, n_row_groups=n, first_rg=first, columns=SCAN_COLS)
    return path


def scan_files(nrg):
    import multiprocessing as mp
    os.makedirs(SCAN_DIR, exist_ok=True)
    jobs = [(os.path.join(SCAN_DIR, f"w_{g:05d}.parquet"), g, min(RGS_PER_FILE, nrg - g)) for g in range(0, nrg, RGS_PER_FILE)]
    missing = [j for j in jobs if not os.path.exists(j[0])]
    if missing:
        with mp.get_context("spawn").Pool(max(1, min(len(missing), (os.cpu_count() or 2) - 1, 64))) as pool:
            pool.map(_gen, missing, chunksize=1)
    return [j[0] for j in jobs]


def timed(fn, steps):
    fn()
    ts = []
    for _ in range(steps):
        t = time.perf_counter()
        res = fn()
        ts.append((time.perf_counter() - t) * 1e3)
    return res, statistics.median(ts)


def main():
    agg_rg = int(sys.argv[1]) if len(sys.argv) > 1 else 480
    scan_rg = int(sys.argv[2]) if len(sys.argv) > 2 else 480
    steps = int(sys.argv[3]) if len(sys.argv) > 3 else 10
    import pyarrow as pa
    import bench
    from parseable_b200.query import DeviceTable, StandardTableProvider, Window, col, sum_
    from test_order_by import canon
    from test_window import _sortable, _with_window_cols, host_window
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    print("gpu:", smi, flush=True)

    # (a) top 10 hosts per status by SUM(bytes)
    files = bench.ensure_data(agg_rg)
    table = DeviceTable(files, bench.C4_COLS)
    prov = StandardTableProvider(table, schema={"host": pa.string(), "status": pa.int64(), "bytes": pa.int64()})
    keys, aggs, order = ["host", "status"], [sum_("bytes")], [(sum_("bytes"), "desc")]
    win = Window(["status"], 0, 10, row_number=True, partition_rows=True)
    res, p50 = timed(lambda: prov.aggregate(keys, aggs, order_by=order, window=win), steps)
    base, p50_base = timed(lambda: prov.aggregate(keys, aggs), steps)
    t = base.table()
    idx, rns, szs = host_window(t, ["status"], order, 0, 10)
    assert canon(res.table()) == canon(_with_window_cols(t, idx, rns, szs)), "(a) differs from the host ranking"
    print(f"(a) top 10 hosts per status by SUM(bytes): {table.rows} rows, {res.metrics['groups_total']} groups, "
          f"{res.metrics['groups']} kept; order_ms {res.metrics['order_ms']:.3f}; query p50 {p50:.2f} ms "
          f"(without the window {p50_base:.2f} ms)", flush=True)
    table.close()

    # (b) latest 3 ERROR rows per service
    files = scan_files(scan_rg)
    table = DeviceTable(files, SCAN_COLS)
    prov = StandardTableProvider(table, schema={"p_timestamp": pa.timestamp("ms"), "level": pa.string(), "service": pa.string(),
                                                "host": pa.string()})
    flt = [col("level") == "ERROR"]
    win = Window(["service"], 0, 3, row_number=True, partition_rows=True)
    order = [("p_timestamp", "desc")]
    res, p50 = timed(lambda: prov.scan(["p_timestamp", "host"], flt, row_ids=True, order_by=order, window=win), steps)
    base, p50_base = timed(lambda: prov.scan(["p_timestamp", "host", "service"], flt, row_ids=True), steps)
    t = _sortable(base.table())
    idx, rns, szs = host_window(t, ["service"], order, 0, 3)
    want = _with_window_cols(t.select(["p_timestamp", "host", "__row_id"]), idx, rns, szs)
    assert canon(_sortable(res.table())) == canon(want), "(b) differs from the host ranking"
    print(f"(b) latest 3 ERROR rows per service: {table.rows} rows, {res.metrics['rows_selected']} selected, "
          f"{res.table().num_rows} kept; order_ms {res.metrics['order_ms']:.3f}; query p50 {p50:.2f} ms "
          f"(the unwindowed scan of the selected rows {p50_base:.2f} ms)", flush=True)
    table.close()


if __name__ == "__main__":
    main()
