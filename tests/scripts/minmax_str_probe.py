"""Development probe (GPU box): MIN / MAX over Utf8 at bench size (bench.ensure_data, table resident).  Parity against
the CPU restatement on one whole file, then `GROUP BY status` with MIN(host), MAX(host) against the same query with
MIN(bytes), MAX(bytes): the step time, scan_kernel_ms and device_ms of each, alternated.  Prints the card's name and
power limit.  Not a bench line: bench.py is the contract.

    python tests/scripts/minmax_str_probe.py [row_groups=bench default] [steps=20]
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
    from parseable_b200.query import DeviceTable, StandardTableProvider, max_, min_
    from test_min_max_strings import assert_matches, expect
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    print(f"card: {card}", flush=True)
    files = bench.ensure_data(nrg)
    schema = {f.name: f.type for f in pq.read_schema(files[0])}
    keys = ["status"]
    strs = [min_("host"), max_("host")]
    nums = [min_("bytes"), max_("bytes")]
    # ---- parity on one whole file ----
    ora = Oracle.from_parquet(files[0], columns=["status", "host", "bytes"])
    p1 = StandardTableProvider([files[0]], schema=schema)
    assert_matches(p1.aggregate(keys, strs + nums).table(), expect(ora, keys, strs + nums), keys, strs + nums)
    print(f"parity ok on {files[0]} ({ora.table.num_rows} rows)", flush=True)
    # ---- timing, table resident ----
    table = DeviceTable(files, ["status", "host", "bytes"])
    prov = StandardTableProvider(table, schema=schema)
    print(f"table: {table.rows} rows, {table.device_bytes / 1e9:.2f} GB", flush=True)

    def run(name, aggs):
        for _ in range(3):
            r = prov.aggregate(keys, aggs)
        ms, scan, dev = [], [], []
        for _ in range(steps):
            t = time.perf_counter()
            r = prov.aggregate(keys, aggs)
            ms.append(1e3 * (time.perf_counter() - t))
            scan.append(r.metrics["scan_kernel_ms"])
            dev.append(r.metrics["device_ms"])
        med = lambda v: sorted(v)[len(v) // 2]
        print(f"{name}: step p50 {med(ms):.3f} ms | scan_kernel_ms p50 {med(scan):.3f} (min {min(scan):.3f}, max {max(scan):.3f}) | "
              f"device_ms p50 {med(dev):.3f} | groups {r.metrics['groups']}", flush=True)

    for _ in range(2):
        run("MIN(bytes), MAX(bytes)", nums)
        run("MIN(host), MAX(host)  ", strs)
    table.close()


if __name__ == "__main__":
    main()
