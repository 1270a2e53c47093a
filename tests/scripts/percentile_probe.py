"""Development probe (GPU box): MEDIAN / PERCENTILE_CONT over the bench's logs16 data (bench.ensure_data, table
resident, the bench's C4 columns).  Parity against the CPU restatement on one whole file, then, for
`GROUP BY host, status` with COUNT(*), median(latency_ms), percentile_cont(latency_ms, 0.99) and
percentile_cont(duration_s, 0.95) and the same query without the percentile aggregates: the step time, scan_kernel_ms,
percentile_ms, the pairs per column and the extra HBM the percentile buffers take.  Prints the card's name and power
limit.  Not a bench line: bench.py is the contract.

    python tests/scripts/percentile_probe.py [row_groups=bench default] [steps=20]
"""
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def main():
    import bench
    nrg = int(sys.argv[1]) if len(sys.argv) > 1 else bench.RGS_PER_GPU
    steps = int(sys.argv[2]) if len(sys.argv) > 2 else 20
    import pyarrow.parquet as pq
    from oracle.oracle import Oracle
    from parseable_b200.query import DeviceTable, StandardTableProvider, count_star, median, percentile_cont
    from test_percentile import assert_matches, expect
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    print(f"card: {card}", flush=True)
    files = bench.ensure_data(nrg)
    schema = {f.name: f.type for f in pq.read_schema(files[0])}
    keys = ["host", "status"]
    pct = [count_star(), median("latency_ms"), percentile_cont("latency_ms", 0.99), percentile_cont("duration_s", 0.95)]
    plain = [count_star()]
    # ---- parity on one whole file ----
    ora = Oracle.from_parquet(files[0], columns=bench.C4_COLS)
    p1 = StandardTableProvider([files[0]], schema=schema)
    assert_matches(p1.aggregate(keys, pct).table(), expect(ora, keys, pct), keys, pct)
    print(f"parity ok on {files[0]} ({ora.table.num_rows} rows)", flush=True)
    # ---- timing, table resident ----
    table = DeviceTable(files, bench.C4_COLS)
    prov = StandardTableProvider(table, schema=schema)
    print(f"table: {table.rows} rows, {table.device_bytes / 1e9:.2f} GB", flush=True)

    def run(name, aggs):
        for _ in range(3):
            r = prov.aggregate(keys, aggs)
        ms, scan, pms = [], [], []
        for _ in range(steps):
            t = time.perf_counter()
            r = prov.aggregate(keys, aggs)
            ms.append(1e3 * (time.perf_counter() - t))
            scan.append(r.metrics["scan_kernel_ms"])
            pms.append(r.metrics["percentile_ms"])
        med = lambda v: sorted(v)[len(v) // 2]
        m = r.metrics
        print(f"{name}: step p50 {med(ms):.3f} ms | scan_kernel_ms p50 {med(scan):.3f} | percentile_ms p50 {med(pms):.3f} | "
              f"groups {m['groups']} launches {m['kernel_launches']} rows_selected {m['rows_selected']}", flush=True)
        return r

    run("without percentiles: COUNT(*)", plain)
    run("with percentiles: COUNT(*), median(latency_ms), p99(latency_ms), p95(duration_s)", pct)
    run("without percentiles: COUNT(*)", plain)
    run("with percentiles", pct)
    # pairs per column: every non-NULL input row (no filter); the buffers' HBM by the rule of query.cu
    t = pq.read_table(files[0], columns=["latency_ms", "duration_s"])
    nn = {c: t[c].length() - t[c].null_count for c in ("latency_ms", "duration_s")}
    rows = table.rows
    print(f"pairs per column: about {rows} x non-NULL share {', '.join(f'{c} {v / t.num_rows:.4f}' for c, v in nn.items())}", flush=True)
    print(f"percentile HBM (2 columns): emitted pairs {2 * 12 * rows / 1e9:.2f} GB + one sort <= {48 * rows / 1e9:.2f} GB "
          f"(rule: rows x (12 x columns + 48) = {(24 + 48) * rows / 1e9:.2f} GB)", flush=True)
    table.close()


if __name__ == "__main__":
    main()
